"""
DCSCN.SuperResolution - drop-in for the reference's model class (reference: DCSCN.py:28-769 and its base
class helper/tf_graph.py:17-305), with the TensorFlow graph / session replaced by the H100 engine
(hand-written sm_90a CUDA kernels behind the C-ABI of include/dcscn_b200.h).

Kept from the reference: constructor arguments (the FLAGS object), the model-name grammar, the call order used
by the CLIs (`build_graph` -> [`build_optimizer`] -> `build_summary_saver` -> `init_all_variables` ->
`load_model`), `do` / `do_for_file` / `do_for_evaluate[_with_output]` / `evaluate` / `evaluate_bicubic`,
`train_batch` / `build_input_batch` and the learning-rate / status bookkeeping, and the log lines.
Replaced: everything `sess.run` did.  Not carried over (TensorFlow-specific, SURVEY.md section 2 rows 15-17):
tensorboard summaries, frozen-graph loading, batch-norm.
"""

import logging
import math
import os
import sys
import time

import numpy as np

from helper import engine as eng
from helper import loader, tf_bundle, utilty as util

BICUBIC_METHOD_STRING = "bicubic"


def bilinear_kernel(size):
    """The size x size bilinear interpolation kernel: the outer product of a tent that falls linearly from 1 at the
    kernel's centre to 0 one factor = ceil(size / 2) away (the centre sits between two taps when size is even)."""
    factor = (size + 1) // 2
    center = factor - 1 if size % 2 == 1 else factor - 0.5
    tent = 1.0 - np.abs(np.arange(size) - center) / factor
    return np.outer(tent, tent)


def upscale_weight(shape):
    """Initial Up-TCNN/Tconv_W [K, K, C, C]: the bilinear kernel on every channel's own diagonal entry, zero across
    channels, so the untrained layer is a bilinear up-scaler (utilty.py:366-390)."""
    k, _, c, _ = shape
    w = np.zeros(shape, np.float32)
    kern = bilinear_kernel(k).astype(np.float32)
    for i in range(c):
        w[:, :, i, i] = kern
    return w


def _dist_rank_world():
    """(rank, world_size) of the torch.distributed job this process belongs to, (0, 1) outside one.  A plain
    single-process command line never imports torch: it is only consulted when the caller already loaded it or the
    process was started by torchrun (WORLD_SIZE in the environment)."""
    if "torch" not in sys.modules and int(os.environ.get("WORLD_SIZE", "1")) <= 1:
        return 0, 1
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except ImportError:
        pass
    return 0, 1


def init_distributed(flags):
    """train.py / evaluate.py under torchrun (WORLD_SIZE > 1): one process per GPU.  Joins the NCCL job, pins this
    process to GPU LOCAL_RANK (overriding --gpu_device_id) and gives every rank its own crop / flip random stream.
    Returns (rank, world); (0, 1) and no torch import for a plain single-process command line."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1 and getattr(flags, "gpus", 1) > 1:
        # --gpus=N on a plain command line: re-launch this script as N ranks (127.0.0.1 rendezvous, one node)
        import subprocess
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(flags.gpus),
               "--master-addr", "127.0.0.1", "--master-port", os.environ.get("MASTER_PORT", "29517")] + sys.argv
        sys.exit(subprocess.call(cmd))
    if world <= 1:
        return 0, 1
    import random
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not dist.is_initialized():
        if torch.cuda.is_available():
            torch.cuda.set_device(local)
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        else:
            dist.init_process_group("gloo")
    flags.gpu_device_id = local
    rank = dist.get_rank()
    random.seed(0x5EED + 7919 * rank)
    np.random.seed(0x5EED + 7919 * rank)
    return rank, dist.get_world_size()


def _nccl_job():
    import torch.distributed as dist
    return dist.is_available() and dist.is_initialized() and dist.get_backend() == "nccl"


def _all_reduce_sum(array):
    """Sum a float64 numpy array over all ranks (one NCCL all-reduce when the backend is nccl, gloo on CPU)."""
    import torch
    import torch.distributed as dist
    t = torch.from_numpy(np.ascontiguousarray(array))
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t.cpu().numpy()


class SuperResolution:
    # defaults of --optimizer / --momentum, for instances whose attributes are set without the constructor
    optimizer = "adam"
    momentum = 0.9

    def __init__(self, flags, model_name=""):
        # ---- TensorflowGraph.__init__ (tf_graph.py:19-63) ----
        self.dropout_rate = flags.dropout_rate
        self.activator = flags.activator
        self.batch_norm = flags.batch_norm
        self.cnn_size = flags.cnn_size
        self.cnn_stride = 1
        self.initializer = flags.initializer
        self.weight_dev = flags.weight_dev
        self.enable_log = flags.enable_log
        self.save_weights = flags.save_weights and flags.enable_log
        self.save_images = flags.save_images and flags.enable_log
        self.save_images_num = flags.save_images_num
        self.save_meta_data = flags.save_meta_data and flags.enable_log
        self.checkpoint_dir = flags.checkpoint_dir
        self.tf_log_dir = flags.tf_log_dir
        self.features = ""
        self.receptive_fields = 0
        self.complexity = 0
        self.pix_per_input = 1
        self.gpu_device_id = flags.gpu_device_id

        # ---- SuperResolution.__init__ (DCSCN.py:33-106) ----
        self.scale = flags.scale
        self.layers = flags.layers
        self.filters = flags.filters
        self.min_filters = min(flags.filters, flags.min_filters)
        self.filters_decay_gamma = flags.filters_decay_gamma
        self.use_nin = flags.use_nin
        self.nin_filters = flags.nin_filters
        self.nin_filters2 = flags.nin_filters2
        self.reconstruct_layers = max(flags.reconstruct_layers, 1)
        self.reconstruct_filters = flags.reconstruct_filters
        self.resampling_method = BICUBIC_METHOD_STRING
        self.pixel_shuffler = flags.pixel_shuffler
        self.pixel_shuffler_filters = flags.pixel_shuffler_filters
        self.self_ensemble = flags.self_ensemble
        self.depthwise_separable = flags.depthwise_separable

        self.l2_decay = flags.l2_decay
        self.optimizer = flags.optimizer
        self.beta1 = flags.beta1
        self.beta2 = flags.beta2
        self.epsilon = flags.epsilon
        self.momentum = flags.momentum
        self.batch_num = flags.batch_num
        self.batch_image_size = flags.batch_image_size
        self.stride_size = flags.batch_image_size // 2 if flags.stride_size == 0 else flags.stride_size
        self.clipping_norm = flags.clipping_norm
        self.use_l1_loss = flags.use_l1_loss

        self.initial_lr = flags.initial_lr
        self.lr_decay = flags.lr_decay
        self.lr_decay_epoch = flags.lr_decay_epoch

        self.training_images = int(math.ceil(flags.training_images / flags.batch_num) * flags.batch_num)
        self.train = None
        self.test = None

        self.max_value = flags.max_value
        self.channels = flags.channels
        self.output_channels = 1
        self.psnr_calc_border_size = flags.psnr_calc_border_size
        if self.psnr_calc_border_size < 0:
            self.psnr_calc_border_size = self.scale

        self.batch_dir = flags.batch_dir
        self.precision = getattr(flags, "precision", "f16x3")
        self.workspace_mb = getattr(flags, "workspace_mb", 0)

        self.name = self.get_model_name(model_name)
        self.total_epochs = 0
        lr = self.initial_lr
        while lr > flags.end_lr:
            self.total_epochs += self.lr_decay_epoch
            lr *= self.lr_decay

        util.make_dir(self.checkpoint_dir)
        util.make_dir(flags.graph_dir)
        util.make_dir(self.tf_log_dir)
        if flags.initialize_tf_log:
            util.clean_dir(self.tf_log_dir)
        util.set_logging(flags.log_filename, stream_log_level=logging.INFO, file_log_level=logging.INFO)
        logging.info("\nDCSCN v2-------------------------------------")
        logging.info("%s [%s]" % (util.get_now_date(), self.name))

        self.engine = None
        self.optimizer_built = False
        self.init_train_step()
        self._check_supported()
        print("Session and graph initialized.")

    # ------------------------------------------------------------------ naming ----
    def get_model_name(self, model_name, name_postfix=""):
        """DCSCN.py:108-144 - the grammar evaluate.py / sr.py rely on to find `models/<name>.ckpt`."""
        if model_name != "":
            return "dcscn_%s" % model_name
        parts = ["dcscn", "L%d" % self.layers,
                 "F%d" % self.filters + ("to%d" % self.min_filters if self.min_filters != 0 else "")]
        if self.filters_decay_gamma != 1.5:
            parts.append("G%2.2f" % self.filters_decay_gamma)
        if self.cnn_size != 3:
            parts.append("C%d" % self.cnn_size)
        if self.scale != 2:
            parts.append("Sc%d" % self.scale)
        if self.use_nin:
            parts.append("NIN")
            if self.nin_filters != 0:
                parts.append("A%d" % self.nin_filters)
            if self.nin_filters2 != self.nin_filters // 2:
                parts.append("B%d" % self.nin_filters2)
        if self.pixel_shuffler:
            parts.append("PS")
        if self.max_value != 255.0:
            parts.append("M%2.1f" % self.max_value)
        if self.activator != "prelu":
            parts.append(self.activator)
        if self.batch_norm:
            parts.append("BN")
        if self.depthwise_separable:
            parts.append("DS")
        tail = "R%d" % self.reconstruct_layers  # reconstruct_layers >= 1 always (DCSCN.py:42)
        if self.reconstruct_filters != 1:
            tail += "F%d" % self.reconstruct_filters
        parts.append(tail)
        if name_postfix != "":
            parts.append(name_postfix)
        return "_".join(parts)

    def _check_supported(self):
        """Flag values the reference accepts but no shipped checkpoint uses are rejected with a clear message."""
        problems = []
        if self.batch_norm:
            problems.append("--batch_norm")
        if not self.use_nin:
            problems.append("--use_nin=false")
        if self.channels != 1:
            problems.append("--channels=%d" % self.channels)
        if self.reconstruct_layers != 1:
            problems.append("--reconstruct_layers=%d" % self.reconstruct_layers)
        if problems:
            raise NotImplementedError("not supported by the H100 engine: " + ", ".join(problems))

    # ------------------------------------------------------------------ graph ----
    def _engine_config(self):
        if self.activator not in eng.ACTIVATORS:
            raise NameError("Not implemented activator:%s" % self.activator)   # tf_graph.py:98, at build_graph
        if self.optimizer not in eng.OPTIMIZERS:   # the message of add_optimizer_op (DCSCN.py:391)
            raise ValueError("Optimizer arg should be one of [gd, adadelta, adagrad, adam, momentum, rmsprop].")
        prec = {"f16x3": eng.PRECISION_F16X3, "f16x1": eng.PRECISION_F16X1}[self.precision]
        return eng.make_config(
            scale=self.scale, layers=self.layers, filters=self.filters, min_filters=self.min_filters,
            filters_decay_gamma=self.filters_decay_gamma, use_nin=self.use_nin, nin_filters=self.nin_filters,
            nin_filters2=self.nin_filters2, cnn_size=self.cnn_size, reconstruct_layers=self.reconstruct_layers,
            reconstruct_filters=self.reconstruct_filters, pixel_shuffler_filters=self.pixel_shuffler_filters,
            depthwise_separable=self.depthwise_separable, channels=self.channels, dropout_keep=self.dropout_rate,
            l2_decay=self.l2_decay, clipping_norm=self.clipping_norm, beta1=self.beta1, beta2=self.beta2,
            epsilon=self.epsilon, device_id=self.gpu_device_id, precision=prec, activator=self.activator,
            optimizer=self.optimizer, momentum=self.momentum, transposed_upsampler=not self.pixel_shuffler)

    def build_graph(self):
        """DCSCN.py:222-332: creates the engine (variables at their initial values) and the bookkeeping strings."""
        self.engine = eng.Engine(self._engine_config())
        if self.workspace_mb > 0:   # inference above this workspace runs as overlapping windows (bit-identical)
            self.engine.set_option("workspace_mb", self.workspace_mb)
        shapes = self.engine.param_shapes()
        # complexity / receptive-field bookkeeping of tf_graph.py:100-110,143-147 and DCSCN.py:267-275
        self.features = ""
        self.complexity = 0
        self.receptive_fields = 0
        pix = 1
        total = 0
        for name, shape in shapes.items():
            if name == "Up-TCNN/Tconv_W":   # build_transposed_conv: s*s times the pixels, K x K x C x C, +1 field
                k, _, c, _ = shape
                pix *= self.scale * self.scale
                self.complexity += pix * k * k * c * c
                self.receptive_fields += 1
                continue
            if not name.endswith("/conv_W"):
                continue
            scope = name[:-len("/conv_W")]
            k, _, cin, cout = shape
            if scope.startswith("Up-PS2"):
                pix = 4
            self.complexity += pix * k * k * cin * cout
            if (scope + "/conv_B") in shapes:
                self.complexity += pix * cout
            if scope.startswith("CNN") or scope in ("A1", "B1", "B2"):   # build_activator, whatever the activator
                self.complexity += pix * cout
            if scope == "B1":
                pass  # A1 and B1 are parallel: DCSCN.py:275 takes the 1x1 back out
            self.receptive_fields = k if self.receptive_fields == 0 else self.receptive_fields + (k - 1)
            if scope == "A1":
                self.receptive_fields -= (self.cnn_size - 1)
            self.features += "%d " % cout
            if scope.startswith("CNN"):
                total += cout
                if scope == "CNN%d" % self.layers:
                    self.features += " Total: (%d)" % total
        logging.info("Feature:%s Complexity:%s Receptive Fields:%d" % (
            self.features, "{:,}".format(self.complexity), self.receptive_fields))

    def build_optimizer(self):
        """DCSCN.py:334-369: the loss / clip / --optimizer step lives inside the engine's train_step."""
        self.optimizer_built = True
        if self.use_l1_loss:
            self.engine.set_option("l1_loss", 1)
        util.print_num_of_total_parameters(self, output_detail=True)

    def build_summary_saver(self, with_saver=True):
        """tf_graph.py:298-305: tensorboard writers are not carried over; the 'saver' is helper/tf_bundle."""
        self.saver = with_saver

    def init_all_variables(self):
        """tf_graph.py:73-75: (re-)initialise weights - 'he' truncated normal (utilty.py:360-363), bias 0, alpha 0.1,
        and the transposed upsampler's Tconv_W as a bilinear up-scaler (upscale_weight)."""
        if self.engine is None:
            raise RuntimeError("call build_graph() first")
        rng = np.random.RandomState()
        for name, shape in self.engine.param_shapes().items():
            if name.endswith("/Tconv_W"):
                self.engine.set_param(name, upscale_weight(shape))
            elif name.endswith("conv_W"):
                k, _, cin, _ = shape
                std = {"he": math.sqrt(2.0 / (k * k * cin))}.get(self.initializer, self.weight_dev)
                w = rng.randn(*shape)
                bad = np.abs(w) > 2
                while bad.any():  # tf.truncated_normal re-draws beyond 2 sigma
                    w[bad] = rng.randn(int(bad.sum()))
                    bad = np.abs(w) > 2
                self.engine.set_param(name, (w * std).astype(np.float32))
            elif name.endswith("conv_B"):
                self.engine.set_param(name, np.zeros(shape, np.float32))
            else:
                self.engine.set_param(name, np.full(shape, 0.1, np.float32))
        # the reference re-runs tf.global_variables_initializer(), which also re-initialises the optimizer's slots and
        # the beta powers: trials of train.py (--tests > 1) must not inherit the previous trial's moments
        self.engine.reset_optimizer()
        print("Model initialized.")

    def broadcast_variables(self, src=0):
        """Data-parallel start: every rank takes rank `src`'s variables (the ranks drew different random initial
        weights), like the replicated variables of a mirrored strategy.  No-op outside a torch.distributed job."""
        rank, world = _dist_rank_world()
        if world <= 1:
            return
        import torch
        import torch.distributed as dist
        on_gpu = dist.get_backend() == "nccl"
        for name in self.engine.param_shapes():
            t = torch.from_numpy(np.ascontiguousarray(self.engine.get_param(name)))
            if on_gpu:
                t = t.cuda()
            dist.broadcast(t, src=src)
            if rank != src:
                self.engine.set_param(name, t.cpu().numpy())
        step = torch.tensor([self.engine.adam_step], dtype=torch.int64)
        if on_gpu:
            step = step.cuda()
        dist.broadcast(step, src=src)
        if rank != src and int(step.item()) != self.engine.adam_step:
            self.engine.adam_step = int(step.item())

    def trainable_shapes(self):
        return self.engine.param_shapes() if self.engine is not None else {}

    # ------------------------------------------------------------------ checkpoints ----
    def _ckpt_filename(self, name, trial):
        if name == "" or name == "default":
            name = self.name
        if trial > 0:
            return self.checkpoint_dir + "/" + name + "_" + str(trial) + ".ckpt"
        return self.checkpoint_dir + "/" + name + ".ckpt"

    def load_model(self, name="", trial=0, output_log=False, restore_optimizer=False):
        """tf_graph.py:263-280: restore from the TF V2 bundle `<checkpoint_dir>/<name>.ckpt`.  With
        `restore_optimizer` (train.py resuming a run) the Adam slots `<var>/Adam`, `<var>/Adam_1` and the update count
        behind `beta1_power` are restored too, as tf.train.Saver.restore does for the graph train.py builds; for the
        other optimizers, their slots (engine.OPTIMIZER_SLOTS) that the file holds."""
        filename = self._ckpt_filename(name, trial)
        if not os.path.isfile(filename + ".index"):
            print("Error. [%s] is not exist!" % filename)
            exit(-1)
        reader = tf_bundle.BundleReader(filename)
        weights = {}
        for var in self.engine.param_shapes():
            if not reader.has_tensor(var):
                raise eng.EngineError("checkpoint %s has no variable '%s' (model flags do not match the file)"
                                      % (filename, var))
            weights[var] = reader.get_tensor(var)
        self.engine.set_params(weights)
        self.engine.reset_optimizer()   # weights from a file never keep moments of whatever was trained before
        if restore_optimizer and self.optimizer == "adam" and reader.has_tensor("beta1_power"):
            for var in weights:
                for slot, suffix in enumerate(("/Adam", "/Adam_1")):
                    if reader.has_tensor(var + suffix):
                        self.engine.set_adam_slot(var, slot, reader.get_tensor(var + suffix))
            self.engine.adam_step = self._adam_step_from_powers(reader)
        elif restore_optimizer and self.optimizer != "adam":
            for var in weights:
                for slot, (suffix, _) in enumerate(eng.OPTIMIZER_SLOTS[self.optimizer]):
                    if reader.has_tensor(var + suffix):
                        self.engine.set_optimizer_slot(var, slot, reader.get_tensor(var + suffix))
        if output_log:
            logging.info("Model restored [ %s ]." % filename)
        else:
            print("Model restored [ %s ]." % filename)

    def _adam_step_from_powers(self, reader):
        """Update count t behind the stored beta powers (TF keeps beta^(t+1)).  beta2_power = 0.999^(t+1) stays a normal
        float32 for ~1e5 updates, beta1_power = 0.9^(t+1) underflows after ~980 - so beta2_power is read first and
        beta1_power only when the file has no usable beta2_power."""
        for key, beta in (("beta2_power", self.beta2), ("beta1_power", self.beta1)):
            if not reader.has_tensor(key) or not 0.0 < beta < 1.0:
                continue
            p = float(np.asarray(reader.get_tensor(key)).reshape(-1)[0])
            if 1e-30 < p < 1.0:
                return max(0, int(round(math.log(p) / math.log(beta))) - 1)
            if p >= 1.0:
                return 0
        return 10 ** 6   # every stored power underflowed (a very long run): both bias corrections are 1

    def save_model(self, name="", trial=0, output_log=False):
        """tf_graph.py:282-296: write `<name>.ckpt.index` + `.data-00000-of-00001` (TF V2 bundle) with everything the
        reference's tf.train.Saver() writes: the trainables, the --optimizer's slots (engine.OPTIMIZER_SLOTS) and, for
        Adam, beta1_power / beta2_power - so the file restores in the reference's sr.py / train.py graphs (which build
        the optimizer) as well as here."""
        filename = self._ckpt_filename(name, trial)
        if _dist_rank_world()[0] != 0:
            return      # data-parallel ranks hold identical weights: rank 0 writes the file
        shapes = self.engine.param_shapes()
        tensors = {var: self.engine.get_param(var) for var in shapes}
        if self.optimizer != "adam":
            for var in shapes:   # the engine returns a slot's initial value until the first step
                for slot, (suffix, _) in enumerate(eng.OPTIMIZER_SLOTS[self.optimizer]):
                    tensors[var + suffix] = self.engine.get_optimizer_slot(var, slot)
        else:
            steps = self.engine.adam_step
            for var, shape in shapes.items():
                for slot, suffix in enumerate(("/Adam", "/Adam_1")):
                    tensors[var + suffix] = (self.engine.get_adam_slot(var, slot) if steps > 0
                                             else np.zeros(shape, dtype=np.float32))
            tensors["beta1_power"] = np.asarray(self.beta1 ** (steps + 1), dtype=np.float32)
            tensors["beta2_power"] = np.asarray(self.beta2 ** (steps + 1), dtype=np.float32)
        tf_bundle.write_bundle(filename, tensors)
        if output_log:
            logging.info("Model saved [%s]." % filename)
        else:
            print("Model saved [%s]." % filename)

    # ------------------------------------------------------------------ data sets ----
    def load_dynamic_datasets(self, data_dir, batch_image_size):
        """DCSCN.py:146-153"""
        self.train = loader.DynamicDataSets(self.scale, batch_image_size, channels=self.channels,
                                            resampling_method=self.resampling_method)
        self.train.set_data_dir(data_dir)
        self._images_on_device = False    # uploaded to HBM by init_epoch_index once the engine exists

    def load_datasets(self, data_dir, batch_dir, batch_image_size, stride_size=0):
        """DCSCN.py:155-173"""
        batch_dir += "/scale%d" % self.scale
        self.train = loader.BatchDataSets(self.scale, batch_dir, batch_image_size, stride_size, channels=self.channels,
                                          resampling_method=self.resampling_method)
        if not self.train.is_batch_exist():
            self.train.build_batch(data_dir)
        else:
            self.train.load_batch_counts()
        self.train.load_all_batch_images()
        self._patches_on_device = False   # uploaded to HBM by init_epoch_index once the engine exists

    def init_epoch_index(self):
        """DCSCN.py:175-184"""
        rank, world = _dist_rank_world()
        if world > 1 and self.batch_num % world != 0:
            raise ValueError("--batch_num=%d must be a multiple of the %d data-parallel ranks (every rank normalises its "
                             "gradient by its own patch count; equal shards keep the reference's global mean)"
                             % (self.batch_num, world))
        # data parallel: this rank loads and trains on batch_num / world patches of every mini-batch
        self.local_batch = self.batch_num // world
        if world > 1 and getattr(self.train, "shard_world", 1) != world:
            self.train.set_shard(rank, world, seed=0xDC5C)
        self.batch_input = self.local_batch * [None]
        self.batch_input_bicubic = self.local_batch * [None]
        self.batch_true = self.local_batch * [None]
        # grid-patch data sets (--build_batch): the uint8 patch arrays move to HBM once and a mini-batch becomes an index
        # list + one gather launch per tensor (helper/engine.py: set_patch_store / train_step_indexed)
        self.batch_indices = None
        if isinstance(self.train, loader.BatchDataSets) and self.engine is not None and self.train.count > 0:
            if not getattr(self, "_patches_on_device", False):
                self.engine.set_patch_store(self.train.input_images, self.train.input_interpolated_images,
                                            self.train.true_images)
                self._patches_on_device = True
            self.batch_indices = np.zeros(self.local_batch, dtype=np.int64)
        # random-crop data sets (the default): the decoded images move to HBM once and a mini-batch becomes a list of crop
        # descriptors (image, top, left, mirror) drawn on the host (helper/engine.py: set_image_store / train_step_crops)
        self.batch_crops = None
        if isinstance(self.train, loader.DynamicDataSets) and self.engine is not None and self.train.count > 0:
            if not getattr(self, "_images_on_device", False):
                self.engine.set_image_store(self.train.decoded_images())
                self._images_on_device = True
            self.batch_crops = np.zeros((self.local_batch, 4), dtype=np.int32)
        self.training_psnr_sum = 0
        self.training_loss_sum = 0
        self.training_step = 0
        self.train.init_batch_index()

    def build_input_batch(self):
        """DCSCN.py:186-190"""
        if getattr(self, "batch_indices", None) is not None:            # patches already live in HBM: draw the indices only
            for i in range(len(self.batch_indices)):
                self.batch_indices[i] = self.train.get_next_image_no()
            return
        if getattr(self, "batch_crops", None) is not None:              # images already live in HBM: draw the crops only
            for i in range(len(self.batch_crops)):
                self.batch_crops[i] = self.train.draw_crop()
            return
        for i in range(len(self.batch_input)):
            self.batch_input[i], self.batch_input_bicubic[i], self.batch_true[i] = self.train.load_batch_image(
                self.max_value)

    # ------------------------------------------------------------------ training ----
    def train_batch(self):
        """DCSCN.py:415-425: one optimisation step on the current mini-batch."""
        # data parallel: every rank holds its own batch_num / world patches (init_epoch_index); the gradients meet in
        # one flat all-reduce before the (identical) clip + optimizer update on every rank
        rank, world = _dist_rank_world()
        if getattr(self, "batch_indices", None) is not None:
            if world > 1:
                image_loss, mse = self.engine.train_step_data_parallel(None, None, None, lr=self.lr, seed=self.step * world + rank,
                                                                       indices=self.batch_indices, max_value=self.max_value)
            else:
                image_loss, mse = self.engine.train_step_indexed(self.batch_indices, lr=self.lr, seed=self.step,
                                                                 max_value=self.max_value)
        elif getattr(self, "batch_crops", None) is not None:
            if world > 1:
                image_loss, mse = self.engine.train_step_data_parallel(None, None, None, lr=self.lr, seed=self.step * world + rank,
                                                                       crops=self.batch_crops, patch_size=self.train.batch_image_size,
                                                                       max_value=self.max_value)
            else:
                image_loss, mse = self.engine.train_step_crops(self.batch_crops, self.train.batch_image_size, lr=self.lr,
                                                               seed=self.step, max_value=self.max_value)
        else:
            x = np.ascontiguousarray(np.stack(self.batch_input), dtype=np.float32)
            x2 = np.ascontiguousarray(np.stack(self.batch_input_bicubic), dtype=np.float32)
            y = np.ascontiguousarray(np.stack(self.batch_true), dtype=np.float32)
            if x.ndim == 3:
                x, x2, y = x[..., None], x2[..., None], y[..., None]
            if world > 1:
                image_loss, mse = self.engine.train_step_data_parallel(x, x2, y, lr=self.lr, seed=self.step * world + rank)
            else:
                image_loss, mse = self.engine.train_step_host(x, x2, y, lr=self.lr, seed=self.step, apply_update=True)
        self.training_loss_sum += image_loss
        self.training_psnr_sum += util.get_psnr(mse, max_value=self.max_value)
        self.training_step += 1
        self.step += 1

    def log_to_tensorboard(self, test_filename, psnr, save_meta_data=True):
        """DCSCN.py:427-482: tensorboard summaries are not carried over (SURVEY.md section 5.5)."""
        return

    def update_epoch_and_lr(self):
        """DCSCN.py:484-495"""
        self.epochs_completed_in_stage += 1
        if self.epochs_completed_in_stage >= self.lr_decay_epoch:
            self.lr *= self.lr_decay
            self.epochs_completed_in_stage = 0
            return True
        return False

    def print_status(self, psnr, ssim, log=False):
        """DCSCN.py:497-524"""
        if self.step == 0:
            logging.info("Initial PSNR:%f SSIM:%f" % (psnr, ssim))
            return
        processing_time = (time.time() - self.start_time) / self.step
        line_a = "%s Step:%s PSNR:%f SSIM:%f (Training PSNR:%0.3f)" % (
            util.get_now_date(), "{:,}".format(self.step), psnr, ssim, self.training_psnr_sum / self.training_step)
        estimated = processing_time * (self.total_epochs - self.epochs_completed) * (
            self.training_images // self.batch_num)
        h = estimated // (60 * 60)
        estimated -= h * 60 * 60
        m = estimated // 60
        s = estimated - m * 60
        line_b = "Epoch:%d LR:%f (%2.3fsec/step) Estimated:%d:%d:%d" % (
            self.epochs_completed, self.lr, processing_time, h, m, s)
        if log:
            logging.info(line_a)
            logging.info(line_b)
        else:
            print(line_a)
            print(line_b)

    def init_train_step(self):
        """DCSCN.py:727-735"""
        self.lr = self.initial_lr
        self.epochs_completed = 0
        self.epochs_completed_in_stage = 0
        self.min_validation_mse = -1
        self.min_validation_epoch = -1
        self.step = 0
        self.start_time = time.time()

    def end_train_step(self):
        self.total_time = time.time() - self.start_time

    def print_steps_completed(self, output_to_logging=False):
        """DCSCN.py:740-757"""
        if self.step == 0:
            return
        processing_time = self.total_time / self.step
        h = self.total_time // (60 * 60)
        m = (self.total_time - h * 60 * 60) // 60
        s = (self.total_time - h * 60 * 60 - m * 60)
        status = "Finished at Total Epoch:%d Steps:%s Time:%02d:%02d:%02d (%2.3fsec/step) %d x %d x %d patches" % (
            self.epochs_completed, "{:,}".format(self.step), h, m, s, processing_time,
            self.batch_image_size, self.batch_image_size, self.training_images)
        (logging.info if output_to_logging else print)(status)

    def copy_log_to_archive(self, archive_name):
        """tf_graph.py:251-261: nothing to archive (no tensorboard log is written)."""
        return

    # ------------------------------------------------------------------ inference ----
    def evaluate(self, test_filenames):
        """DCSCN.py:534-545.  On the device path (_device_evaluation) the test images are decoded once and kept in the
        engine's evaluation store while the files stay the same (train.py evaluates after every epoch): each later call
        uploads nothing and makes one engine call per image."""
        total_psnr = total_ssim = 0
        if len(test_filenames) == 0:
            return 0, 0
        slots = self._eval_store(test_filenames) if self._device_evaluation() else [None] * len(test_filenames)
        for filename, slot in zip(test_filenames, slots):
            if slot is None:
                psnr, ssim = self.do_for_evaluate(filename, print_console=False)
            else:
                psnr, ssim = self.engine.evaluate_image(slot, self.self_ensemble, self.max_value, self.psnr_calc_border_size)
            total_psnr += psnr
            total_ssim += ssim
        return total_psnr / len(test_filenames), total_ssim / len(test_filenames)

    # ---- evaluation on the device (helper/engine.py: set_eval_images / evaluate_image) ----
    def _device_evaluation(self):
        """do_for_evaluate / evaluate_bicubic / evaluate run on the device in a single process with an engine that has
        the evaluation call; under torchrun the host path keeps its flip sharding."""
        return (_dist_rank_world()[1] == 1 and getattr(self, "engine", None) is not None
                and hasattr(self.engine, "evaluate_image") and getattr(self, "channels", 1) == 1
                and self.resampling_method == BICUBIC_METHOD_STRING)

    def _device_eval_image(self, file_path):
        """The decoded image the device path evaluates, or None for one it leaves to the host path (not 1 or 3 uint8
        channels, or smaller than one scale x scale block)."""
        image = util.load_image(file_path, print_console=False)
        if (image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] not in (1, 3)
                or image.shape[0] < self.scale or image.shape[1] < self.scale):
            return None
        return image

    @staticmethod
    def _file_key(file_path):
        st = os.stat(file_path)
        return file_path, st.st_size, st.st_mtime_ns

    def _eval_store(self, test_filenames):
        """Store slot (or None: host path) of every file.  The store is rebuilt only when a file's (path, size, mtime)
        changes; it does not depend on the weights."""
        keys = [self._file_key(f) for f in test_filenames]
        cached = getattr(self, "_eval_cache", None)
        if cached is None or cached[0] != keys or cached[2] is not self.engine:
            images, slots = [], []
            for filename in test_filenames:
                image = self._device_eval_image(filename)
                slots.append(None if image is None else len(images))
                if image is not None:
                    images.append(image)
            if images:
                self.engine.set_eval_images(images)
            self._eval_cache = cached = (keys, slots, self.engine)
        return cached[1]

    def _run(self, image, bicubic):
        """What `sess.run(self.y_, {x:[1,h,w,1], x2:[1,sh,sw,1], dropout:1, is_training:0})` returned."""
        h, w = image.shape[:2]
        x = np.ascontiguousarray(image, dtype=np.float32).reshape(1, h, w, 1)
        x2 = np.ascontiguousarray(bicubic, dtype=np.float32).reshape(1, self.scale * h, self.scale * w, 1)
        return self.engine.forward_host(x, x2)

    def do(self, input_image, bicubic_input_image=None):
        """DCSCN.py:547-586: self-ensemble of up to 8 flips, float64 mean."""
        h, w = input_image.shape[:2]
        if bicubic_input_image is None:
            rank, world = _dist_rank_world()
            on_device = (self.max_value == 255.0 and self.resampling_method == BICUBIC_METHOD_STRING and world == 1
                         and input_image.dtype != np.uint8 and getattr(self, "engine", None) is not None
                         and hasattr(self.engine, "forward_ensemble_host"))
            if not on_device:
                bicubic_input_image = util.resize_image_by_pil(input_image, self.scale,
                                                               resampling_method=self.resampling_method)
            # else: the engine forms Pillow's bicubic up-scale in HBM (bit for bit the same values) - only the LR image
            # crosses PCIe and no host-side resize sits in front of the GPU
        if self.max_value != 255.0:
            input_image = np.multiply(input_image, self.max_value / 255.0)
            bicubic_input_image = np.multiply(bicubic_input_image, self.max_value / 255.0)
        if bicubic_input_image is None:      # device-side bicubic (single process)
            if self.self_ensemble > 1:
                return self.engine.forward_ensemble_host(input_image, None, self.self_ensemble)
            x = np.ascontiguousarray(input_image, dtype=np.float32).reshape(1, h, w, 1)
            return self.engine.forward_host(x, None)[0]

        if self.self_ensemble > 1:
            # The flips are independent: rank r of a torch.distributed job computes flips r, r + world, ... and the
            # inverse-flipped partial sums meet in ONE all-reduce (NCCL over NVLink on GPUs); single process = the
            # reference's serial loop.  float64 accumulation like the reference's np.zeros default (DCSCN.py:560).
            rank, world = _dist_rank_world()
            if world == 1 and getattr(self, "channels", 1) == 1:
                # one process: flips, two batched forwards (transforms 0..3 and 4..7) and the float64 mean all on the GPU
                output = self.engine.forward_ensemble_host(input_image, bicubic_input_image, self.self_ensemble)
            elif world > 1 and _nccl_job() and getattr(self, "engine", None) is not None:
                # one process per GPU: this rank's transforms as batched forwards, float64 partial sum on the device,
                # ONE NCCL all-reduce, mean (helper/engine.py: forward_ensemble_sharded)
                import torch
                dev = "cuda:%d" % self.engine.config.device_id
                xd = torch.from_numpy(np.ascontiguousarray(input_image, dtype=np.float32).reshape(h, w)).to(dev)
                x2d = torch.from_numpy(np.ascontiguousarray(bicubic_input_image, dtype=np.float32).reshape(
                    self.scale * h, self.scale * w)).to(dev)
                output = self.engine.forward_ensemble_sharded(xd, x2d, self.self_ensemble).cpu().numpy()[..., None]
            else:
                output = np.zeros([self.scale * h, self.scale * w, 1])
                for i in range(rank, self.self_ensemble, world):
                    image = util.flip(input_image, i)
                    bicubic_image = util.flip(bicubic_input_image, i)
                    y = self._run(image, bicubic_image)
                    output += util.flip(y[0], i, invert=True)
                if world > 1:
                    output = _all_reduce_sum(output)
                output /= self.self_ensemble
        else:
            output = self._run(input_image, bicubic_input_image)[0]

        if self.max_value != 255.0:
            return np.multiply(output, 255.0 / self.max_value)
        return output

    # ---- file-level drivers (host glue around `do`) ----
    def _save(self, folder, stem, suffix, extension, image):
        util.save_image(folder + stem + suffix + extension, image)

    def _upscale(self, image):
        return util.resize_image_by_pil(image, self.scale, resampling_method=self.resampling_method)

    def do_for_file(self, file_path, output_folder="output"):
        """DCSCN.py:588-614: one image file -> original, bicubic, bicubic_y, result_y and result PNGs under
        `<output_folder>/<model name>/`.  Colour images are super-resolved on Y and merged with bicubic CbCr."""
        org_image = util.load_image(file_path)
        stem, extension = os.path.splitext(os.path.basename(file_path))
        folder = output_folder + "/" + self.name + "/"
        self._save(folder, stem, "", extension, org_image)
        self._save(folder, stem, "_bicubic", extension, self._upscale(org_image))

        is_color = len(org_image.shape) >= 3 and org_image.shape[2] == 3 and self.channels == 1
        if is_color:
            y_plane = util.convert_rgb_to_y(org_image)
            self._save(folder, stem, "_bicubic_y", extension, self._upscale(y_plane))
            result_y = self.do(y_plane)
            self._save(folder, stem, "_result_y", extension, result_y)
            cbcr = util.convert_rgb_to_ycbcr(self._upscale(org_image))[:, :, 1:3]
            result = util.convert_y_and_cbcr_to_rgb(result_y, cbcr)
        else:
            self._save(folder, stem, "_bicubic_y", extension, self._upscale(org_image))
            result = self.do(org_image)
        self._save(folder, stem, "_result", extension, result)

    def _evaluation_set(self, file_path):
        """Host half of DCSCN.py:672-696 / :616-661 / :705-717, shared by the three evaluate entry points.
        Returns None for images the reference skips (neither 3- nor 1-channel), else a dict with the aligned
        ground truth, the network input (LR luma), its bicubic up-scale and the luma ground truth."""
        true_image = util.set_image_alignment(util.load_image(file_path, print_console=False), self.scale)
        if self.channels != 1 or true_image.shape[2] not in (1, 3):
            return None
        color = true_image.shape[2] == 3
        lr = loader.build_input_image(true_image, channels=self.channels, scale=self.scale, alignment=self.scale,
                                      convert_ycbcr=True if color else True)
        return {"true": true_image, "color": color, "lr": lr, "bicubic": self._upscale(lr),
                "true_y": util.convert_rgb_to_y(true_image) if color else true_image}

    def do_for_evaluate(self, file_path, print_console=False):
        """DCSCN.py:672-703: PSNR / SSIM of the super-resolved luma against the ground truth (border = scale).  In a
        single process the image is decoded here and everything after the decode runs on the device, equal to the host
        path (_do_for_evaluate_host) bit for bit."""
        image = self._device_eval_image(file_path) if self._device_evaluation() else None
        if image is None:
            return self._do_for_evaluate_host(file_path, print_console)
        psnr, ssim = self.engine.evaluate_image(image, self.self_ensemble, self.max_value, self.psnr_calc_border_size)
        if print_console:
            print("[%s] PSNR:%f, SSIM:%f" % (file_path, psnr, ssim))
        return psnr, ssim

    def _do_for_evaluate_host(self, file_path, print_console=False):
        """do_for_evaluate with the inputs and the metric formed on the host (numpy, scipy, Pillow)."""
        s = self._evaluation_set(file_path)
        if s is None:
            return None, None
        output = self.do(s["lr"], s["bicubic"])
        psnr, ssim = util.compute_psnr_and_ssim(s["true_y"], output, border_size=self.psnr_calc_border_size)
        if print_console:
            print("[%s] PSNR:%f, SSIM:%f" % (file_path, psnr, ssim))
        return psnr, ssim

    def do_for_evaluate_with_output(self, file_path, output_directory, print_console=False):
        """DCSCN.py:616-670: do_for_evaluate plus the result / bicubic / loss images on disk
        (`<output_directory>/<model name>/<file_path stem>_*.png`, same names as the reference)."""
        if _dist_rank_world()[0] != 0:
            return self.do_for_evaluate(file_path, print_console=False)   # same collectives, rank 0 writes the images
        stem, extension = os.path.splitext(file_path)
        folder = output_directory + "/" + self.name + "/"
        util.make_dir(folder)
        s = self._evaluation_set(file_path)
        if s is None:
            return None, None
        # bicubic of the (colour) input, written first like the reference (DCSCN.py:623-625)
        whole_lr = util.resize_image_by_pil(s["true"], 1.0 / self.scale, resampling_method=self.resampling_method)
        self._save(folder, stem, "_input_bicubic", extension, self._upscale(whole_lr))

        output = self.do(s["lr"], s["bicubic"])
        border = self.psnr_calc_border_size
        if s["color"]:
            ycbcr = util.convert_rgb_to_ycbcr(s["true"])
            true_y = ycbcr[:, :, 0:1]
            psnr, ssim = util.compute_psnr_and_ssim(true_y, output, border_size=border)
            util.save_image(folder + file_path, s["true"])
            self._save(folder, stem, "_input", extension, s["lr"])
            self._save(folder, stem, "_input_bicubic_y", extension, s["bicubic"])
            self._save(folder, stem, "_true_y", extension, true_y)
            self._save(folder, stem, "_result", extension, output)
            self._save(folder, stem, "_result_c", extension, util.convert_y_and_cbcr_to_rgb(output, ycbcr[:, :, 1:3]))
            self._save(folder, stem, "_loss", extension, util.get_loss_image(true_y, output, border_size=border))
        else:
            psnr, ssim = util.compute_psnr_and_ssim(s["true"], output, border_size=border)
            util.save_image(folder + file_path, s["true"])
            self._save(folder, stem, "_result", extension, output)
        if print_console:
            print("[%s] PSNR:%f, SSIM:%f" % (stem, psnr, ssim))
        return psnr, ssim

    def evaluate_bicubic(self, file_path, print_console=False):
        """DCSCN.py:705-725: the bicubic baseline through the same metric (on the device like do_for_evaluate)."""
        image = self._device_eval_image(file_path) if self._device_evaluation() else None
        if image is None:
            return self._evaluate_bicubic_host(file_path, print_console)
        psnr, ssim = self.engine.evaluate_image(image, 1, self.max_value, self.psnr_calc_border_size, bicubic=True)
        if print_console:
            print("PSNR:%f, SSIM:%f" % (psnr, ssim))
        return psnr, ssim

    def _evaluate_bicubic_host(self, file_path, print_console=False):
        """evaluate_bicubic on the host."""
        s = self._evaluation_set(file_path)
        if s is None:
            return None, None
        psnr, ssim = util.compute_psnr_and_ssim(s["true_y"], s["bicubic"], border_size=self.psnr_calc_border_size)
        if print_console:
            print("PSNR:%f, SSIM:%f" % (psnr, ssim))
        return psnr, ssim


def create(flags, with_optimizer=False):
    """The construction sequence every CLI of the reference spells out (evaluate.py:49-58, sr.py:39-43, train.py:27-36):
    SuperResolution(...) -> build_graph -> [build_optimizer] -> build_summary_saver -> init_all_variables."""
    model = SuperResolution(flags, model_name=flags.model_name)
    model.build_graph()
    if with_optimizer:
        model.build_optimizer()
    model.build_summary_saver()
    model.init_all_variables()
    return model
