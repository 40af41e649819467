"""
Host-side input preparation for training and evaluation (what the reference's helper/loader.py provides).

Only what the callers of the replaced path need, restated: `build_input_image` / `build_image_set` (the LR / bicubic /
HR triple of `do_for_evaluate`, loader.py:23-67), a grid-patch training set kept in RAM (`BatchDataSets`, loader.py:70-275;
the reference caches the same patches as BMP files) and a random-crop training set (`DynamicDataSets`, loader.py:278-355).
Data loading is CPU work outside the GPU path (SURVEY.md section 2, row 8).
"""

import logging
import random

import numpy as np
from PIL import Image

from helper import utilty as util


def _to_luma_or_ycbcr(image, channels, convert_ycbcr):
    """RGB -> Y for a one-channel model, RGB -> YCbCr otherwise (loader.py:55-61)."""
    if not convert_ycbcr:
        return image
    wants_luma = channels == 1 and image.shape[2] == 3
    return util.convert_rgb_to_y(image) if wants_luma else util.convert_rgb_to_ycbcr(image)


def build_input_image(image, width=0, height=0, channels=1, scale=1, alignment=0, convert_ycbcr=True):
    """loader.py:42-67: optional centre crop to (height, width), size alignment, colour conversion and a bicubic
    down-scale by `scale`."""
    if width and height and image.shape[:2] != (height, width):
        top, left = (image.shape[0] - height) // 2, (image.shape[1] - width) // 2
        image = image[top:top + height, left:left + width, :]
    if alignment > 1:
        image = util.set_image_alignment(image, alignment)
    image = _to_luma_or_ycbcr(image, channels, convert_ycbcr)
    return image if scale == 1 else util.resize_image_by_pil(image, 1.0 / scale)


def load_input_image(filename, width=0, height=0, channels=1, scale=1, alignment=0, convert_ycbcr=True, print_console=True):
    return build_input_image(util.load_image(filename, print_console=print_console), width, height, channels, scale,
                             alignment, convert_ycbcr)


def build_image_set(file_path, channels=1, scale=1, convert_ycbcr=True, resampling_method="bicubic", print_console=True):
    """loader.py:23-33: (LR input, its bicubic up-scale, ground truth) of one image file."""
    truth = util.set_image_alignment(util.load_image(file_path, print_console=print_console), scale)
    if convert_ycbcr and channels == 1 and truth.shape[2] == 3:
        truth = util.convert_rgb_to_y(truth)
    small = util.resize_image_by_pil(truth, 1.0 / scale, resampling_method=resampling_method)
    return small, util.resize_image_by_pil(small, scale, resampling_method=resampling_method), truth


class _ShuffledOrder:
    """Serves 0..count-1 in a fresh random permutation per pass (loader.py:259-275, 300-308)."""

    count = 0
    shard_rank, shard_world, order_rng = 0, 1, None

    def set_shard(self, rank, world, seed):
        """Data-parallel training: all ranks draw the SAME permutation (private generator, shared seed) and rank r
        serves its elements r, r + world, ... - the ranks' patches are disjoint and together cover a pass."""
        self.shard_rank, self.shard_world, self.order_rng = rank, world, random.Random(seed)
        self.batch_index = None

    def init_batch_index(self, shuffle=True):
        order = list(range(self.count))
        if shuffle:
            (self.order_rng or random).shuffle(order)
        self.batch_index, self.index = order, self.shard_rank

    def get_next_image_no(self):
        if getattr(self, "batch_index", None) is None or self.index >= self.count:
            self.init_batch_index()
        number = self.batch_index[min(self.index, self.count - 1)]
        self.index += self.shard_world
        return number


def _rescaled(arrays, max_value):
    if max_value == 255:
        return arrays
    return tuple(np.multiply(a, max_value / 255.0) for a in arrays)


class BatchDataSets(_ShuffledOrder):
    """Every grid patch of every image of a directory, as uint8 (the reference stores them as BMP files,
    loader.py:236-249), served in shuffled order."""

    def __init__(self, scale, batch_dir, batch_image_size, stride_size=0, channels=1, resampling_method="bicubic"):
        self.scale, self.channels, self.resampling_method = scale, channels, resampling_method
        self.batch_dir = batch_dir
        self.batch_image_size = batch_image_size
        self.stride = stride_size or batch_image_size // 2
        self.input_images = self.input_interpolated_images = self.true_images = None
        self.batch_index, self.index, self.count = None, 0, 0

    def is_batch_exist(self):
        return self.input_images is not None

    def build_batch(self, data_dir):
        print("Building batch images for %s..." % self.batch_dir)
        hr_size, hr_stride = self.batch_image_size * self.scale, self.stride * self.scale
        stacks = ([], [], [])
        for filename in util.get_files_in_directory(data_dir):
            small, bicubic, truth = build_image_set(filename, channels=self.channels, scale=self.scale,
                                                    resampling_method=self.resampling_method, print_console=False)
            patches = (util.get_split_images(small, self.batch_image_size, stride=self.stride),
                       util.get_split_images(bicubic, hr_size, stride=hr_stride),
                       util.get_split_images(truth, hr_size, stride=hr_stride))
            if patches[0] is None or patches[1] is None:
                continue                                   # image smaller than one patch
            for stack, p in zip(stacks, patches):
                stack.append(p)
        if not stacks[0]:
            self.count = 0
            return
        # uint8 like the reference's BMP cache: the same truncation of the float patches
        self.input_images, self.input_interpolated_images, self.true_images = (
            np.concatenate(stack).astype(np.uint8) for stack in stacks)
        self.count = self.input_images.shape[0]
        print("%d mini-batch images are built(saved)." % self.count)

    def load_batch_counts(self):
        """The reference re-reads its on-disk cache here; the RAM set needs nothing."""

    def load_all_batch_images(self):
        print("Allocating memory for all batch images.")

    def load_batch_image(self, max_value):
        k = self.get_next_image_no()
        return _rescaled((self.input_images[k], self.input_interpolated_images[k], self.true_images[k]), max_value)


class DynamicDataSets(_ShuffledOrder):
    """A random HR crop per request, mirrored left-right half of the time (loader.py:278-355).  A crop is drawn as a
    descriptor (image, top, left, mirror) by `draw_crop`; `load_batch_image` cuts and resamples it on the host, the engine
    does the same from its image store (SuperResolution.init_epoch_index / train_batch)."""

    def __init__(self, scale, batch_image_size, channels=1, resampling_method="bicubic"):
        self.scale, self.channels, self.resampling_method = scale, channels, resampling_method
        self.batch_image_size = batch_image_size
        self.filenames, self.sizes, self.batch_index, self.index, self.count = [], [], None, 0, 0

    def set_data_dir(self, data_dir):
        self.filenames = util.get_files_in_directory(data_dir)
        self.count = len(self.filenames)
        if self.count <= 0:
            logging.error("Data Directory is empty.")
            exit(-1)
        self.sizes = []
        for filename in self.filenames:            # PIL reads the header only; pixels are decoded on demand
            with Image.open(filename) as im:
                self.sizes.append((im.height, im.width))

    def init_batch_index(self, shuffle=True):
        super().init_batch_index(True)

    def draw_crop(self):
        """(image number, top, left, mirror) of the next patch, drawing from `random` exactly as the reference's
        load_batch_image / load_random_patch do (loader.py:310-355); images smaller than one HR patch are skipped."""
        edge = self.batch_image_size * self.scale
        while True:
            number = self.get_next_image_no()
            rows, cols = self.sizes[number]
            if rows < edge or cols < edge:
                print("Error: %s should have more than %d x %d size." % (self.filenames[number], edge, edge))
                continue
            top = random.randrange(rows - edge) if rows > edge else 0
            left = random.randrange(cols - edge) if cols > edge else 0
            return number, top, left, int(random.randrange(2) == 0)

    def decoded_images(self):
        """Every image of the set decoded once (util.load_image), in image-number order: the engine's image store."""
        return [util.load_image(filename, print_console=False) for filename in self.filenames]

    def load_batch_image(self, max_value):
        """loader.py:310-330"""
        number, top, left, mirror = self.draw_crop()
        edge = self.batch_image_size * self.scale
        image = util.load_image(self.filenames[number], print_console=False)
        truth = build_input_image(image[top:top + edge, left:left + edge, :], channels=self.channels, convert_ycbcr=True)
        if mirror:
            truth = np.fliplr(truth)
        small = util.resize_image_by_pil(truth, 1 / self.scale)
        return _rescaled((small, util.resize_image_by_pil(small, self.scale), truth), max_value)
