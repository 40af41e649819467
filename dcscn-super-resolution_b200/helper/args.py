"""
Flag definitions shared by train.py / evaluate.py / sr.py.

Same flag names and defaults as the reference's helper/args.py:16-98, without TensorFlow: a small absl-compatible parser (`--name=value`, `--name value`, `--bool`, `--nobool`,
`--bool=true|false`).  Scripts may add their own flags through `args.flags.DEFINE_*` before calling
`args.get()`, exactly like the reference (evaluate.py:38-39, sr.py:34).
"""

import sys

import numpy as np


class _Flags:
    def __init__(self):
        object.__setattr__(self, "_defs", {})
        object.__setattr__(self, "_values", {})
        object.__setattr__(self, "_parsed", False)
        object.__setattr__(self, "_unparsed", [])

    def _define(self, name, default, help_text, kind):
        self._defs[name] = (kind, default, help_text)
        self._values[name] = default

    def __getattr__(self, name):
        values = object.__getattribute__(self, "_values")
        if name in values:
            return values[name]
        raise AttributeError("Unknown flag '%s'" % name)

    def __setattr__(self, name, value):
        if name not in self._defs:
            raise AttributeError("Unknown flag '%s'" % name)
        self._values[name] = value

    def _convert(self, name, text):
        kind = self._defs[name][0]
        if kind == "int":
            return int(text)
        if kind == "float":
            return float(text)
        if kind == "bool":
            t = text.lower()
            if t in ("true", "t", "1", "yes", "y"):
                return True
            if t in ("false", "f", "0", "no", "n"):
                return False
            raise ValueError("flag --%s: '%s' is not a boolean" % (name, text))
        return text

    def parse(self, argv):
        """Parses argv[1:]; returns [argv[0]] + arguments that are not flags (absl behaviour)."""
        rest = [argv[0]] if argv else [""]
        i = 1
        while i < len(argv):
            a = argv[i]
            if a == "--":
                rest.extend(argv[i + 1:])
                break
            if a.startswith("-") and len(a) > 1 and not _is_number(a):
                body = a.lstrip("-")
                if "=" in body:
                    name, text = body.split("=", 1)
                    if name not in self._defs:
                        raise SystemExit("FATAL Flags parsing error: Unknown command line flag '%s'" % name)
                    self._values[name] = self._convert(name, text)
                else:
                    name = body
                    if name in self._defs:
                        if self._defs[name][0] == "bool":
                            self._values[name] = True
                        else:
                            if i + 1 >= len(argv):
                                raise SystemExit("FATAL Flags parsing error: Missing value for flag --%s" % name)
                            i += 1
                            self._values[name] = self._convert(name, argv[i])
                    elif name.startswith("no") and name[2:] in self._defs and self._defs[name[2:]][0] == "bool":
                        self._values[name[2:]] = False
                    elif name in ("help", "helpfull", "h"):
                        self.print_help()
                        raise SystemExit(0)
                    else:
                        raise SystemExit("FATAL Flags parsing error: Unknown command line flag '%s'" % name)
            else:
                rest.append(a)
            i += 1
        object.__setattr__(self, "_parsed", True)
        object.__setattr__(self, "_unparsed", rest)
        return rest

    def print_help(self):
        for name, (kind, default, help_text) in self._defs.items():
            print("  --%s: %s\n    (default: %r)" % (name, help_text, default))

    def flag_values_dict(self):
        return dict(self._values)


def _is_number(s):
    try:
        float(s)
        return True
    except ValueError:
        return False


FLAGS = _Flags()


class _FlagModule:
    """The `flags` object of the reference (tf.app.flags): DEFINE_* + FLAGS."""
    FLAGS = FLAGS

    @staticmethod
    def DEFINE_integer(name, default, help_text):
        FLAGS._define(name, default, help_text, "int")

    @staticmethod
    def DEFINE_float(name, default, help_text):
        FLAGS._define(name, float(default), help_text, "float")

    @staticmethod
    def DEFINE_string(name, default, help_text):
        FLAGS._define(name, default, help_text, "str")

    @staticmethod
    def DEFINE_boolean(name, default, help_text):
        FLAGS._define(name, default, help_text, "bool")

    DEFINE_bool = DEFINE_boolean


flags = _FlagModule()

# The reference's flag set (helper/args.py:16-98): identical names and defaults, so every command line of the reference
# parses unchanged; the descriptions are this engine's.  One row per flag: name, default, description - the kind is
# the default's Python type.
_REFERENCE_FLAGS = [
    # --- network ---
    ("scale", 2, "upscaling factor, 2 to 8"),
    ("layers", 12, "depth of the feature-extraction stack (CNN1..CNNn)"),
    ("filters", 196, "output channels of CNN1"),
    ("min_filters", 48, "output channels of the last feature-extraction layer"),
    ("filters_decay_gamma", 1.5, "shape of the channel decay from `filters` down to `min_filters`"),
    ("use_nin", True, "reconstruction through the A1 / B1-B2 network-in-network branches"),
    ("nin_filters", 64, "channels of branch A1"),
    ("nin_filters2", 32, "channels of branch B1 and B2"),
    ("cnn_size", 3, "spatial size of the feature-extraction filters"),
    ("reconstruct_layers", 1, "R-CNN layers after the up-sampler (0 or 1 here)"),
    ("reconstruct_filters", 32, "channels of intermediate R-CNN layers"),
    ("dropout_rate", 0.8, "keep probability during training (1 disables dropout)"),
    ("activator", "prelu", "activation of CNN1..CNNL, A1, B1, B2: prelu, relu, leaky_relu, sigmoid, tanh or selu"),
    ("pixel_shuffler", True, "sub-pixel (depth_to_space) up-sampling; false: one bilinear-initialised transposed convolution"),
    ("pixel_shuffler_filters", 0, "channels after the pixel shuffler; 0 keeps the channel count of its input"),
    ("self_ensemble", 8, "how many of the 8 flip / rotate variants are averaged at inference (1..8)"),
    ("batch_norm", False, "not supported by this engine (rejected when set)"),
    ("depthwise_separable", False, "every layer as depthwise k x k followed by pointwise 1 x 1"),
    # --- training ---
    ("bicubic_init", True, "the network predicts the residual over the bicubic up-scale x2"),
    ("clipping_norm", 5.0, "global-norm gradient clipping threshold; <= 0 turns clipping off"),
    ("initializer", "he", "weight initialiser: uniform, stddev, xavier, he, identity or zero"),
    ("weight_dev", 0.01, "standard deviation for the `stddev` initialiser"),
    ("l2_decay", 0.0001, "weight of the L2 penalty on the convolution filters"),
    ("optimizer", "adam", "gd, momentum, adadelta, adagrad, adam or rmsprop (TF1 optimizers at TF's defaults)"),
    ("beta1", 0.9, "Adam first-moment decay"),
    ("beta2", 0.999, "Adam second-moment decay"),
    ("epsilon", 1e-8, "Adam epsilon"),
    ("momentum", 0.9, "momentum of the momentum and rmsprop optimisers"),
    ("batch_num", 20, "patches per training step"),
    ("batch_image_size", 48, "edge length of a low-resolution training patch"),
    ("stride_size", 0, "patch grid stride when building batches; 0 = half a patch"),
    ("training_images", 24000, "patches per epoch"),
    ("use_l1_loss", False, "mean absolute error instead of mean squared error as the image loss"),
    # --- learning-rate schedule ---
    ("initial_lr", 0.002, "learning rate of the first epoch"),
    ("lr_decay", 0.5, "factor applied to the learning rate at each decay"),
    ("lr_decay_epoch", 9, "epochs between two decays"),
    ("end_lr", 2e-5, "training stops once the learning rate falls below this"),
    # --- data sets ---
    ("dataset", "bsd200", "training set folder under data_dir (yang91, general100, bsd200, ...)"),
    ("test_dataset", "set5", "evaluation set folder (set5, set14, bsd100, urban100) or `all`"),
    ("tests", 1, "independent training runs"),
    ("do_benchmark", False, "after training also evaluate set5, set14 and bsd100"),
    # --- image handling ---
    ("max_value", 255.0, "pixel range the network works in"),
    ("channels", 1, "image channels fed to the network (1: luma only)"),
    ("psnr_calc_border_size", -1, "pixels shaved before PSNR / SSIM; negative = 2 + scale"),
    ("build_batch", False, "pre-cut grid patches to disk instead of sampling them on the fly"),
    # --- folders and names (no trailing slash) ---
    ("checkpoint_dir", "models", "where checkpoints are read and written"),
    ("graph_dir", "graphs", "kept for command-line compatibility"),
    ("data_dir", "data", "root of the image data sets"),
    ("batch_dir", "batch_data", "where pre-cut training patches live"),
    ("output_dir", "output", "where result images go"),
    ("tf_log_dir", "tf_log", "kept for command-line compatibility (no tensorboard here)"),
    ("log_filename", "log.txt", "text log"),
    ("model_name", "", "overrides the generated model name"),
    ("load_model_name", "", "checkpoint to start from (`default` = the generated model name)"),
    # --- logging switches of the reference (accepted, mostly without effect here) ---
    ("initialize_tf_log", True, "accepted for compatibility"),
    ("enable_log", True, "accepted for compatibility"),
    ("save_weights", True, "accepted for compatibility"),
    ("save_images", False, "accepted for compatibility"),
    ("save_images_num", 20, "accepted for compatibility"),
    ("save_meta_data", False, "accepted for compatibility"),
    ("gpu_device_id", 0, "CUDA device to run on"),
    # --- frozen GraphDef deployment: not part of this engine, the flags only have to parse ---
    ("frozenInference", False, "rejected when set"),
    ("frozen_graph_path", "./model_to_freeze/frozen_model_optimized.pb", "unused"),
    # --- additions of this engine; the defaults reproduce the reference's fp32 results ---
    ("precision", "f16x3", "tensor-core arithmetic: f16x3 (fp32-equivalent) or f16x1 (single pass, PSNR-neutral)"),
    ("gpus", 1, "GPUs the self-ensemble / training batch is spread over (one process each)"),
    ("workspace_mb", 0, "MiB of GPU workspace one inference batch may use; larger images run as overlapping windows, "
                        "bit-identical to the whole image (0 = no limit)"),
]

for _name, _default, _help in _REFERENCE_FLAGS:
    _kind = {bool: "bool", int: "int", float: "float", str: "str"}[type(_default)]
    FLAGS._define(_name, _default, _help, _kind)


def get(argv=None):
    print("Python Interpreter version:%s" % sys.version[:3])
    print("engine: dcscn_b200 (sm_90a CUDA, no TensorFlow)")
    print("numpy version:%s" % np.__version__)
    if not FLAGS._parsed:
        FLAGS.parse(sys.argv if argv is None else argv)
    return FLAGS


def run(main):
    """tf.app.run(): parse flags, call main(not_parsed_args)."""
    if not FLAGS._parsed:
        FLAGS.parse(sys.argv)
    sys.exit(main(FLAGS._unparsed))
