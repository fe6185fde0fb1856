"""Image readers (reference: neuralmonkey/readers/image_reader.py:14-226).  Host-side
data format code next to the path (SURVEY.md section 8, row f): a list file names one image
per line; `.npy` arrays are taken as they are, anything else is opened with PIL."""
import os
from typing import Callable, Iterable, List

import numpy as np

from neuralmonkey_b200.logging import warn

VGG_RGB_MEANS = [[[123.68, 116.779, 103.939]]]  # image_reader.py:99


def _center_crop(image: np.ndarray, width: int, height: int) -> np.ndarray:
    """_crop (:206-216): symmetric crop, the odd pixel is dropped on the right / bottom."""
    h, w = image.shape[:2]
    w_shift, h_shift = max(w - width, 0) // 2, max(h - height, 0) // 2
    even_w, even_h = max(w - width, 0) % 2, max(h - height, 0) % 2
    return image[h_shift:h - h_shift - even_h, w_shift:w - w_shift - even_w]


def single_image_for_imagenet(path: str, target_height: int, target_width: int,
                              vgg_normalization: bool, zero_one_normalization: bool) -> np.ndarray:
    """The reference computes a rescaled image and discards it (:153-165: the result of
    `_rescale_or_crop` is never assigned), so what reaches the network is the centre crop of
    the ORIGINAL image, zero-padded to the target size.  Same here."""
    if path.endswith(".npy"):
        image = np.load(path)
    else:
        from PIL import Image
        image = np.array(Image.open(path).convert("RGB"))
    cropped = _center_crop(image, target_width, target_height)
    res = np.zeros((target_height, target_width, 3))
    res[:cropped.shape[0], :cropped.shape[1], :] = cropped
    if vgg_normalization:
        res -= VGG_RGB_MEANS
    if zero_one_normalization:
        res /= 255.
    return res


def imagenet_reader(prefix: str, target_width: int = 227, target_height: int = 227,
                    vgg_normalization: bool = False,
                    zero_one_normalization: bool = False) -> Callable:
    def load(list_files: List[str]) -> Iterable[np.ndarray]:
        for list_file in list_files:
            with open(list_file) as f_list:
                for i, image_file in enumerate(f_list):
                    path = os.path.join(prefix, image_file.rstrip())
                    if not os.path.exists(path):
                        raise Exception("Image file '{}' no. {} does not exist.".format(path, i + 1))
                    yield single_image_for_imagenet(path, target_height, target_width,
                                                    vgg_normalization, zero_one_normalization)
    return load


def image_reader(pad_w: int, pad_h: int, channels: int = 3, prefix: str = "", rescale_w: bool = False,
                 rescale_h: bool = False, keep_aspect_ratio: bool = False, mode: str = "RGB") -> Callable:
    """Reader of the images named in list files (:14-95): each is converted to the PIL `mode`, rescaled and / or
    centre-cropped to at most pad_h x pad_w (_rescale_or_crop), and zero-padded at the bottom / right to
    [pad_h, pad_w, channels] float64.  An image PIL cannot read becomes a blank one, with a warning."""
    if not rescale_w and not rescale_h and keep_aspect_ratio:
        raise ValueError("It does not make sense to keep the aspect ratio while not rescaling the image.")
    if rescale_w != rescale_h and not keep_aspect_ratio:
        raise ValueError("While rescaling only one side, aspect ratio must be kept, was set to false.")
    from PIL import Image, ImageFile
    ImageFile.LOAD_TRUNCATED_IMAGES = True

    def load(list_files: List[str]) -> Iterable[np.ndarray]:
        for list_file in list_files:
            with open(list_file) as f_list:
                for i, image_file in enumerate(f_list):
                    path = os.path.join(prefix, image_file.rstrip())
                    if not os.path.exists(path):
                        raise Exception("Image file '{}' no.{}  does not exist.".format(path, i + 1))
                    try:
                        image = Image.open(path).convert(mode)
                    except IOError:
                        warn("Skipping image from file '{}' no. '{}'.".format(path, i + 1))
                        image = Image.new(mode, (pad_w, pad_h))
                    image = _rescale_or_crop(image, pad_w, pad_h, rescale_w, rescale_h, keep_aspect_ratio)
                    image_np = np.array(image)
                    if image_np.ndim == 2:
                        img_channels = 1
                        image_np = np.expand_dims(image_np, 2)
                    elif image_np.ndim == 3:
                        img_channels = image_np.shape[2]
                    else:
                        raise ValueError("Image should have either 2 (black and white) or three dimensions (color "
                                         "channels), has {} dimension.".format(image_np.ndim))
                    if channels != img_channels:
                        raise ValueError("Image does not have the pre-declared number of channels {}, but {}."
                                         .format(channels, img_channels))
                    padded = np.zeros((pad_h, pad_w, channels))
                    padded[:image_np.shape[0], :image_np.shape[1], :] = image_np
                    yield padded
    return load


def _rescale_or_crop(image, pad_w: int, pad_h: int, rescale_w: bool, rescale_h: bool, keep_aspect_ratio: bool):
    """(:180-203) PIL's default resampling where the reference uses it, bilinear for the both-sides rescale."""
    from PIL import Image
    orig_w, orig_h = image.size
    if orig_w == pad_w and orig_h == pad_h:
        return image
    if rescale_w and rescale_h and not keep_aspect_ratio:
        image = image.resize((pad_w, pad_h), Image.BILINEAR)
    elif rescale_w and rescale_h and keep_aspect_ratio:
        ratio = min(pad_h / orig_h, pad_w / orig_w)
        image = image.resize((int(orig_w * ratio), int(orig_h * ratio)))
    elif rescale_w and not rescale_h:
        if orig_w != pad_w:
            ratio = pad_w / orig_w
            image = image.resize((pad_w, int(orig_h * ratio)))
    elif rescale_h and not rescale_w:
        if orig_h != pad_h:
            ratio = pad_h / orig_h
            image = image.resize((int(orig_w * ratio), pad_h))
    width, height = image.size
    w_shift, h_shift = max(width - pad_w, 0) // 2, max(height - pad_h, 0) // 2
    even_w, even_h = max(width - pad_w, 0) % 2, max(height - pad_h, 0) % 2
    return image.crop((w_shift, h_shift, width - w_shift - even_w, height - h_shift - even_h))
