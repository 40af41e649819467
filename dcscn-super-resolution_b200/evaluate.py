"""
Evaluate a trained DCSCN model on a test data set (drop-in for the reference's evaluate.py).

  python evaluate.py --test_dataset=set14 --save_results=true
  python evaluate.py --scale=2 --layers=7 --filters=32 --min_filters=8 --filters_decay_gamma=1.2 \
      --nin_filters=24 --nin_filters2=8 --reconstruct_layers=0 --self_ensemble=1 --pixel_shuffler_filters=1

Same flags as the reference (helper/args.py) plus --save_results / --compute_bicubic (evaluate.py:38-39);
the model flags must match the ones the checkpoint was trained with.  Per data set it logs
"Model Average [<set>] PSNR:..., SSIM:..., Time (s): ..." (evaluate.py:106), the time being wall-clock
seconds per image around the whole per-image pipeline exactly like the reference (evaluate.py:94-101).
"""

import logging
import time

import DCSCN
from helper import args, utilty as util

args.flags.DEFINE_boolean("save_results", True, "Save result, bicubic and loss images.")
args.flags.DEFINE_boolean("compute_bicubic", False, "Compute bicubic performance.")

FLAGS = args.get()


def build_model():
    if FLAGS.frozenInference:
        raise NotImplementedError("--frozenInference loads a TensorFlow GraphDef; not supported by the H100 engine")
    # under torchrun / --gpus=N the flips of the self-ensemble are shared out over one process per GPU (DCSCN.do)
    DCSCN.init_distributed(FLAGS)
    return DCSCN.create(FLAGS)


def evaluate_bicubic(model, test_data):
    files = util.get_files_in_directory(FLAGS.data_dir + "/" + test_data)
    scores = [model.evaluate_bicubic(f, print_console=False) for f in files]
    logging.info("Bicubic Average [%s] PSNR:%f, SSIM:%f" % (
        test_data, sum(s[0] for s in scores) / len(files), sum(s[1] for s in scores) / len(files)))


def evaluate_model(model, test_data):
    files = util.get_files_in_directory(FLAGS.data_dir + "/" + test_data)
    total_psnr = total_ssim = total_time = 0
    for filename in files:
        start = time.time()
        if FLAGS.save_results:
            psnr, ssim = model.do_for_evaluate_with_output(filename, output_directory=FLAGS.output_dir,
                                                           print_console=False)
        else:
            psnr, ssim = model.do_for_evaluate(filename, print_console=False)
        total_time += time.time() - start
        total_psnr += psnr
        total_ssim += ssim
    logging.info("Model Average [%s] PSNR:%f, SSIM:%f, Time (s): %f" % (
        test_data, total_psnr / len(files), total_ssim / len(files), total_time / len(files)))
    return total_psnr / len(files), total_ssim / len(files), total_time / len(files)


def main(not_parsed_args):
    if len(not_parsed_args) > 1:
        print("Unknown args:%s" % not_parsed_args)
        exit()
    model = build_model()
    test_list = ['set5', 'set14', 'bsd100'] if FLAGS.test_dataset == "all" else [FLAGS.test_dataset]
    for trial in range(FLAGS.tests):
        model.load_model(FLAGS.load_model_name, trial=trial, output_log=FLAGS.tests > 1)
        if FLAGS.compute_bicubic:
            for test_data in test_list:
                print(test_data)
                evaluate_bicubic(model, test_data)
        for test_data in test_list:
            evaluate_model(model, test_data)


if __name__ == '__main__':
    args.run(main)
