"""The data side of the robustness evaluation (mce/eval_robustness.py, --robustness_type ce): the
ImageNet-C directory walk, the label mapping, the split of the distortions over GPUs and the decoding of
one image to uint8.  The device side is metrics.CorruptionError and model_fns.corruption_error.

  get_synsets2idx     :151-158  each line of the label file, stripped, ' ' -> '_', lowercased -> its index
  distortion_images   :190-196  data_dir/<distortion>/<severity 1..5>/<synset dir>/* (every file, any
                      extension), label = synsets2idx[parent dir name] + label_offset (:217-219)
  distortion_quota    :249-278  the first n % g GPUs take one distortion more, in ALEXNET_CE order
  decode_image        :123-135  3-channel uint8, exactly image_size x image_size (the reference's set_shape)
"""
from __future__ import annotations

import glob
import os

import numpy as np

from .metrics import DISTORTIONS

# preprocessing/imagenet_preprocessing.py:46-49 (R, G, B), subtracted from every pixel (:122-149)
CHANNEL_MEANS = (123.68, 116.78, 103.94)
SEVERITIES = (1, 2, 3, 4, 5)


def get_synsets2idx(label_file):
    with open(label_file, "r") as f:
        synsets = [l.strip().replace(" ", "_").lower() for l in f.readlines()]
    return {s: i for i, s in enumerate(synsets)}


def distortion_images(data_dir, distortion, synsets2idx, label_offset=1):
    """(files, labels) of one distortion pooled over its five severities, in a fixed (sorted) order."""
    distortion_dir = os.path.join(data_dir, distortion)
    if not os.path.isdir(distortion_dir):
        raise FileNotFoundError("robustness evaluation: missing distortion directory %s" % distortion_dir)
    files, labels = [], []
    for severity in SEVERITIES:
        severity_dir = os.path.join(distortion_dir, str(severity))
        if not os.path.isdir(severity_dir):
            raise FileNotFoundError("robustness evaluation: missing severity directory %s" % severity_dir)
        for d in sorted(os.listdir(severity_dir)):
            for f in sorted(glob.glob(os.path.join(severity_dir, d) + "/*")):
                synset = os.path.basename(os.path.dirname(os.path.splitext(f)[0]))
                if synset not in synsets2idx:
                    raise ValueError("robustness evaluation: %s: synset %r is not in the label file" % (f, synset))
                files.append(f)
                labels.append(synsets2idx[synset] + label_offset)
    return files, labels


def distortion_quota(num_gpus, distortions=DISTORTIONS):
    """The distortions each of num_gpus GPUs evaluates (process() of mce/eval_robustness.py:249-278)."""
    base, extra = divmod(len(distortions), num_gpus)
    out, start = [], 0
    for i in range(num_gpus):
        n = base + (1 if i < extra else 0)
        out.append(list(distortions[start:start + n]))
        start += n
    return out


def decode_rgb(src):
    """uint8 [H, W, 3] of an encoded image at its own size: `src` a path or a binary file object (PIL,
    converted to RGB; for a JPEG, libjpeg's ISLOW DCT, TF's INTEGER_ACCURATE).  Image.draft is never
    used: it trades pixels for speed."""
    from PIL import Image
    with Image.open(src) as im:
        return np.array(im.convert("RGB"), dtype=np.uint8)


def decode_image(path, image_size):
    """uint8 [image_size, image_size, 3] of an image file (PIL, converted to RGB)."""
    a = decode_rgb(path)
    if a.shape != (image_size, image_size, 3):
        raise ValueError("robustness evaluation: %s is %dx%d, expected %dx%d"
                         % (path, a.shape[1], a.shape[0], image_size, image_size))
    return a
