"""
Super-resolve one image file: the reference's `sr.py` command line on the H100 engine.

  python sr.py --file=your_file.png [--scale=3 --layers=8 --filters=96 ...]

The original, the bicubic up-scale and the result (Y and colour) land in `<output_dir>/<model name>/`
(`SuperResolution.do_for_file`).  The model flags select the checkpoint `<checkpoint_dir>/<model name>.ckpt` and have to
be the ones it was trained with.
"""

import DCSCN
from helper import args

args.flags.DEFINE_string("file", "image.jpg", "image to up-scale")
FLAGS = args.get()


def main(_unused):
    # the optimizer is part of the graph here as in the reference (sr.py:41), so a checkpoint's Adam slots are accepted
    engine_model = DCSCN.create(FLAGS, with_optimizer=True)
    engine_model.load_model()
    engine_model.do_for_file(FLAGS.file, FLAGS.output_dir)


if __name__ == '__main__':
    args.run(main)
