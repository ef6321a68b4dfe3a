"""TFRecord shards from raw image folders, without TensorFlow: the reference's dataset builders.

  imagenet          datasets/build_imagenet_data.py (+ preprocess_imagenet_validation_data.py's file list)
  food101           datasets/build_ethz_food101.py
  cub_200_2011      datasets/build_cub_bird200_zeroshot.py
  cars196_zeroshot  datasets/build_cars196_zeroshot.py
  SOP               datasets/build_sop.py

    python -m assembled_cnn_b200.build_data <dataset> [the reference script's flags] [--num_workers N]
                                            [--check device|pil]

Each builder writes the shards its reference script writes: the same file names ('%s-%.5d-of-%.5d'), the
same records in the same order and the same Example features.  The order is the reference's: its listing
(sorted where the reference's tf.gfile.Glob leaves it to the file system), its Python `random` shuffles
seeded 12345, and its record-to-shard assignment, which depends on its `num_threads` flag (np.linspace
ranges per thread, then per shard).  `num_threads` therefore only sets the layout; the work runs on a pool
of `num_workers` host threads and on the GPU, and the bytes do not depend on either.

Every image is checked as the reference's decode_jpeg checks it: its scan is decoded, on the device by
jpeg.JpegDecoder in batches on a copy stream (PIL for the images the device does not decode or whose scan
fails its checks, on the host pool), or by PIL alone with check='pil'.  The height and width come from that
decode.  An image that is not a JPEG, PNG or one-frame GIF (what tf.image.decode_jpeg decodes), or that PIL
cannot decode, raises ValueError with its path; food101 and SOP skip it with a log line, as their reference
scripts do.  Only converted images are re-encoded (encode_jpeg): the ImageNet PNG and CMYK files
of the reference's lists and the CUB / Cars bounding-box crops.  Everything that can be checked before the
images are read is checked before any shard exists: the label directories and files, the bbox and logit
files, the shard counts, the listed files and the outputs.  Each shard is written under a hidden temporary
name and renamed when complete; after a failure the shards already completed stay (a log line says so), and
a new build into the same directory is refused until they are removed.
"""
from __future__ import annotations

import argparse
import fnmatch
import io
import logging
import os
import random
import sys
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, List, NamedTuple, Optional

import numpy as np

from .imagenet_c import decode_rgb
from .imagenet_eval import serialize_example, write_record
from .staging import read_ahead

log = logging.getLogger("assembled_cnn_b200.build_data")

BATCH = 64          # images per device decode

# build_imagenet_data.py _is_png / _is_cmyk
IMAGENET_PNG = ("n02105855_2933.JPEG",)
IMAGENET_CMYK = ("n01739381_1309.JPEG", "n02077923_14822.JPEG", "n02447366_23489.JPEG", "n02492035_15739.JPEG",
                 "n02747177_10752.JPEG", "n03018349_4028.JPEG", "n03062245_4620.JPEG", "n03347037_9675.JPEG",
                 "n03467068_12171.JPEG", "n03529860_11437.JPEG", "n03544143_17228.JPEG", "n03633091_5218.JPEG",
                 "n03710637_5125.JPEG", "n03961711_5286.JPEG", "n04033995_2932.JPEG", "n04258138_17003.JPEG",
                 "n04264628_27969.JPEG", "n04336792_7448.JPEG", "n04371774_5854.JPEG", "n04596742_4225.JPEG",
                 "n07583066_647.JPEG", "n13037406_4650.JPEG")
LOGIT_COLUMNS = 1002            # file name + 1001 logits per line of a logits CSV
# build_imagenet_data.py's flag defaults, used by the command line when the flag is not given and they exist
IMAGENET_BBOX_DEFAULT = "./imagenet_2012_bounding_boxes.csv"
IMAGENET_LOGITS_DEFAULT = "amoebanet_logits"


class Item(NamedTuple):
    path: str
    example: Callable           # (image bytes, height, width) -> {key: (kind, values)}
    convert: Optional[str] = None   # 'png' / 'cmyk': decoded and re-encoded before the check
    bbox: Optional[list] = None     # [xmin, ymin, xmax, ymax]: the image is cropped to it and re-encoded


class Split(NamedTuple):
    name: str                   # 'train' / 'validation'
    items: List[Item]           # in record order
    shards: list                # [(file name, first item, end item)] in shard order
    skip_invalid: bool          # log and skip an image PIL cannot decode instead of raising


# ---------------------------------------------------------------------------------------- layout
def shard_layout(name, total, num_threads, num_shards):
    """[(file name, start, end)] of every shard: the items split into num_threads np.linspace ranges, each
    into num_shards / num_threads np.linspace ranges (build_imagenet_data.py _process_image_files(_batch),
    dataset_utils.make_shard_offsets / make_shard_filenames)."""
    if num_threads < 1 or num_shards < 1:
        raise ValueError("num_threads (%d) and the shard count (%d) must be positive" % (num_threads, num_shards))
    if num_shards % num_threads:
        raise ValueError("the shard count of %s (%d) is not a multiple of num_threads (%d)"
                         % (name, num_shards, num_threads))
    per = num_shards // num_threads
    spacing = np.linspace(0, total, num_threads + 1).astype(int)
    out = []
    for t in range(num_threads):
        r = np.linspace(spacing[t], spacing[t + 1], per + 1).astype(int)
        for s in range(per):
            out.append(("%s-%.5d-of-%.5d" % (name, t * per + s, num_shards), int(r[s]), int(r[s + 1])))
    return out


def shuffled(*lists):
    """The lists permuted by the reference's `random.seed(12345); random.shuffle(range(n))`."""
    idx = list(range(len(lists[0])))
    random.Random(12345).shuffle(idx)
    return [[l[i] for i in idx] for l in lists]


def glob_files(directory, pattern="*"):
    """The entries of `directory` matching `pattern` (tf.gfile.Glob(directory/pattern): fnmatch without
    special treatment of a leading dot), sorted: TF 1.14's GetMatchingPaths returns them in the file system's
    readdir order, which it does not fix."""
    return [os.path.join(directory, f) for f in sorted(os.listdir(directory)) if fnmatch.fnmatchcase(f, pattern)]


def _lines(path, what):
    if not os.path.isfile(path):
        raise ValueError("%s %s does not exist" % (what, path))
    with open(path, "r") as f:
        return f.readlines()


# -------------------------------------------------------------------------------------- features
def encode_jpeg(pixels):
    """JPEG bytes of uint8 [h, w, 3] RGB pixels with tf.image.encode_jpeg's defaults at quality 100: 4:2:0,
    no optimisation, baseline, JFIF at 300 dpi (PIL's libjpeg)."""
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(pixels, dtype=np.uint8), "RGB").save(
        b, "JPEG", quality=100, subsampling=2, optimize=False, progressive=False, dpi=(300, 300))
    return b.getvalue()


def example_without_bbox(label):
    """utils/data_util.py convert_to_example_without_bbox(image, 'jpg', label, height, width)."""
    def make(data, h, w):
        return {"image/encoded": ("bytes", [data]), "image/height": ("int64", [h]), "image/width": ("int64", [w]),
                "image/class/label": ("int64", [label]), "image/format": ("bytes", [b"jpg"])}
    return make


def imagenet_example(path, label, synset, human, bbox, logit):
    """build_imagenet_data.py _convert_to_example; logit None leaves out image/logit."""
    cols = list(zip(*bbox)) if bbox else [(), (), (), ()]

    def make(data, h, w):
        f = {"image/height": ("int64", [h]), "image/width": ("int64", [w]),
                "image/colorspace": ("bytes", [b"RGB"]), "image/channels": ("int64", [3]),
                "image/class/label": ("int64", [label]), "image/class/synset": ("bytes", [synset.encode()]),
                "image/class/text": ("bytes", [human.encode()]),
                "image/object/bbox/xmin": ("float", list(cols[0])), "image/object/bbox/xmax": ("float", list(cols[2])),
                "image/object/bbox/ymin": ("float", list(cols[1])), "image/object/bbox/ymax": ("float", list(cols[3])),
                "image/logit": ("float", logit), "image/object/bbox/label": ("int64", [label] * len(bbox)),
                "image/format": ("bytes", [b"JPEG"]), "image/filename": ("bytes", [os.path.basename(path).encode()]),
                "image/encoded": ("bytes", [data])}
        if logit is None:
            del f["image/logit"]
        return f
    return make


def crop_window(bbox, height, width, path):
    """(y, x, h, w) of the bbox [xmin, ymin, xmax, ymax] clipped at the image's bottom and right edges, as the
    CUB / Cars builders' _process_image clip it."""
    y, x, h, w = bbox[1], bbox[0], bbox[3] - bbox[1], bbox[2] - bbox[0]
    h -= max(0, y + h - height)
    w -= max(0, x + w - width)
    if h <= 0 or w <= 0 or y < 0 or x < 0:
        raise ValueError("%s: bbox %s is outside the %dx%d image" % (path, bbox, height, width))
    return y, x, h, w


# ---------------------------------------------------------------------------------------- ImageNet
def imagenet_synsets(labels_file):
    synsets = [l.strip() for l in _lines(labels_file, "labels_file")]
    if any(not s for s in synsets) or len(set(synsets)) != len(synsets):
        raise ValueError("labels_file %s: every line must be one distinct synset" % labels_file)
    return synsets


def synset_lookup(metadata_file):
    """_build_synset_lookup: '<synset>\\t<human readable label>' per line."""
    out = {}
    for n, l in enumerate(_lines(metadata_file, "imagenet_metadata_file")):
        parts = l.strip().split("\t")
        if len(parts) != 2:
            raise ValueError("imagenet_metadata_file %s line %d: expected <synset>\\t<text>: %r"
                             % (metadata_file, n + 1, l))
        out[parts[0]] = parts[1]
    return out


def bounding_box_lookup(bounding_box_file):
    """_build_bounding_box_lookup: '<file name>,<xmin>,<ymin>,<xmax>,<ymax>' per line, several per image."""
    out = {}
    for n, l in enumerate(_lines(bounding_box_file, "bounding_box_file")):
        parts = l.split(",")
        try:
            if len(parts) != 5:
                raise ValueError("expected 5 fields")
            box = [float(parts[1]), float(parts[2]), float(parts[3]), float(parts[4])]
        except ValueError as e:
            raise ValueError("bounding_box_file %s line %d: %s: %r" % (bounding_box_file, n + 1, e, l))
        out.setdefault(parts[0], []).append(box)
    return out


def logits_lookup(prefix):
    """_build_kd_embbeddings_lookup(prefix): every file matching prefix*, '<file name>,<1001 logits>' per
    line; a file name seen twice raises."""
    d = os.path.dirname(prefix) or "."
    files = glob_files(d, os.path.basename(prefix) + "*") if os.path.isdir(d) else []
    if not files:
        raise ValueError("logits_file_path: no file matches %s*" % prefix)
    out = {}
    for path in files:
        for n, l in enumerate(_lines(path, "logits file")):
            parts = l.split(",")
            try:
                if len(parts) != LOGIT_COLUMNS:
                    raise ValueError("expected %d fields, got %d" % (LOGIT_COLUMNS, len(parts)))
                vals = [float(v) for v in parts[1:LOGIT_COLUMNS]]
            except ValueError as e:
                raise ValueError("logits file %s line %d: %s" % (path, n + 1, e))
            if parts[0] in out:
                raise ValueError("logits file %s line %d: duplicated image %s" % (path, n + 1, parts[0]))
            out[parts[0]] = vals
    return out


def imagenet_files(data_dir, synsets, validation_labels_file=None):
    """(files, synsets, labels) of _find_image_files before its shuffle: for each synset of the labels file
    in order (label 1, 2, ...; 0 is the background class), data_dir/<synset>/*.JPEG.  With
    validation_labels_file (imagenet_2012_validation_synset_labels.txt), data_dir is the flat validation
    directory and <synset>'s files are the ILSVRC2012_val_%08d.JPEG (line number) of its lines, the list
    preprocess_imagenet_validation_data.py would leave in data_dir/<synset>/ without moving a file."""
    index = {s: i + 1 for i, s in enumerate(synsets)}
    by_synset = {s: [] for s in synsets}
    if validation_labels_file is not None:
        for n, l in enumerate(_lines(validation_labels_file, "validation labels file")):
            s = l.strip()
            if s not in index:
                raise ValueError("%s line %d: synset %r is not in the labels file" % (validation_labels_file, n + 1, s))
            by_synset[s].append(os.path.join(data_dir, "ILSVRC2012_val_%08d.JPEG" % (n + 1)))
        for s in synsets:
            by_synset[s].sort()
    else:
        if not os.path.isdir(data_dir):
            raise ValueError("%s is not a directory" % data_dir)
        dirs = {d for d in os.listdir(data_dir) if os.path.isdir(os.path.join(data_dir, d))}
        unknown, missing = sorted(dirs - set(synsets)), [s for s in synsets if s not in dirs]
        if unknown or missing:
            raise ValueError("%s: label directories not in the labels file: %s; labels without a directory: %s"
                             % (data_dir, unknown[:10], missing[:10]))
        for s in synsets:
            by_synset[s] = glob_files(os.path.join(data_dir, s), "*.JPEG")
    files, syn, labels = [], [], []
    for s in synsets:
        files += by_synset[s]
        syn += [s] * len(by_synset[s])
        labels += [index[s]] * len(by_synset[s])
    return files, syn, labels


def imagenet_splits(train_directory, validation_directory, *, train_shards=1024, validation_shards=128,
                    num_threads=8, make_val=True, make_train=True, labels_file="imagenet_lsvrc_2015_synsets.txt",
                    imagenet_metadata_file="imagenet_metadata.txt", bounding_box_file=None, logits_file_path=None,
                    validation_labels_file=None):
    """The splits of build_imagenet_data.py (validation first).  bounding_box_file None: no boxes;
    logits_file_path None: no image/logit feature (model_fns.extract_teacher_logits can add it), else every
    image needs a line in <logits_file_path>/<split>*."""
    synsets = imagenet_synsets(labels_file)
    human = synset_lookup(imagenet_metadata_file)
    missing = [s for s in synsets if s not in human]
    if missing:
        raise ValueError("imagenet_metadata_file %s has no text for %s" % (imagenet_metadata_file, missing[:10]))
    boxes = bounding_box_lookup(bounding_box_file) if bounding_box_file is not None else {}
    splits = []
    for name, directory, shards, make, vlabels in (
            ("validation", validation_directory, validation_shards, make_val, validation_labels_file),
            ("train", train_directory, train_shards, make_train, None)):
        if not make:
            continue
        shard_layout(name, 0, num_threads, shards)          # the shard counts, before the listing
        files, syn, labels = imagenet_files(directory, synsets, vlabels)
        files, syn, labels = shuffled(files, syn, labels)
        logits = logits_lookup(os.path.join(logits_file_path, name)) if logits_file_path is not None else None
        items = []
        for f, s, lab in zip(files, syn, labels):
            base = os.path.basename(f)
            if logits is not None and base not in logits:
                raise ValueError("There is missing logits: %s" % base)
            convert = "png" if base in IMAGENET_PNG else "cmyk" if base in IMAGENET_CMYK else None
            ex = imagenet_example(f, lab, s, human[s], boxes.get(base, []), logits[base] if logits is not None else None)
            items.append(Item(f, ex, convert))
        splits.append(Split(name, items, shard_layout(name, len(items), num_threads, shards), False))
    return splits


# -------------------------------------------------------------------------------------- Food-101
def food101_splits(data_dir, *, train_shards=128, validation_shards=16, num_threads=8):
    """build_ethz_food101.py: meta/labels.txt (lower-cased, ' ' -> '_', label = line index), meta/train.txt
    shuffled and meta/test.txt in order, images/<line>.jpg."""
    ids = {l.strip().lower().replace(" ", "_"): i
           for i, l in enumerate(_lines(os.path.join(data_dir, "meta", "labels.txt"), "labels file"))}
    splits = []
    for name, txt, shards, shuffle in (("train", "train.txt", train_shards, True),
                                       ("validation", "test.txt", validation_shards, False)):
        shard_layout(name, 0, num_threads, shards)
        path = os.path.join(data_dir, "meta", txt)
        files = [os.path.join(data_dir, "images", l.strip() + ".jpg") for l in _lines(path, "file list")]
        labels = []
        for f in files:
            label = os.path.basename(os.path.dirname(f))
            if label not in ids:
                raise ValueError("%s: label %r of %s is not in meta/labels.txt" % (path, label, f))
            labels.append(ids[label])
        if shuffle:
            files, labels = shuffled(files, labels)
        splits.append(_plain_split(name, files, labels, num_threads, shards, True))
    return splits


def _plain_split(name, files, labels, num_threads, shards, skip_invalid, bboxes=None):
    if not files:
        raise ValueError("no image for the %s split" % name)
    items = [Item(f, example_without_bbox(l), None, None if bboxes is None else bboxes[i])
             for i, (f, l) in enumerate(zip(files, labels))]
    return Split(name, items, shard_layout(name, len(items), num_threads, shards), skip_invalid)


# ----------------------------------------------------------------------------------- CUB-200-2011
CUB_RANGES = {"train": range(0, 100), "validation": range(100, 200)}


def cub_bboxes(data_dir):
    """_get_bbox_info: file id (base name without extension) -> [xmin, ymin, xmax, ymax] (int of x, y, x + w,
    y + h) from images.txt and bounding_boxes.txt."""
    names = {}
    for l in _lines(os.path.join(data_dir, "images.txt"), "images.txt"):
        t = l.strip().split()
        if len(t) != 2:
            raise ValueError("images.txt: expected '<image id> <path>': %r" % l)
        names[t[0]] = t[1]
    out = {}
    for l in _lines(os.path.join(data_dir, "bounding_boxes.txt"), "bounding_boxes.txt"):
        t = l.strip().split()
        try:
            if len(t) != 5:
                raise ValueError("expected 5 fields")
            x, y, w, h = (float(v) for v in t[1:])
        except ValueError as e:
            raise ValueError("bounding_boxes.txt: %s: %r" % (e, l))
        if t[0] not in names:
            raise ValueError("bounding_boxes.txt: image id %s is not in images.txt" % t[0])
        out[os.path.splitext(os.path.basename(names[t[0]]))[0]] = [int(x), int(y), int(x + w), int(y + h)]
    return out


def cub_files(name, image_dir):
    """_find_image_files: the sorted entries of image_dir numbered from 0, those of the split's class range
    that are directories read with their files (Glob '*', sorted) shuffled per class, then all shuffled."""
    files, labels, label_index = [], [], 0
    for label_name in sorted(os.listdir(image_dir)):
        if label_index not in CUB_RANGES[name]:
            label_index += 1
            continue
        path = os.path.join(image_dir, label_name)
        if os.path.isdir(path):
            f = glob_files(path)
            f, l = shuffled(f, [label_index] * len(f)) if f else ([], [])
            files += f
            labels += l
            label_index += 1
    return shuffled(files, labels) if files else ([], [])


def cub_splits(data_dir, *, num_threads=16, use_bbox=False):
    """build_cub_bird200_zeroshot.py: classes 0-99 train (128 shards), 100-199 validation (16 shards)."""
    bbox = cub_bboxes(data_dir) if use_bbox else None
    splits = []
    for name, shards in (("train", 128), ("validation", 16)):
        shard_layout(name, 0, num_threads, shards)
        files, labels = cub_files(name, os.path.join(data_dir, "images"))
        splits.append(_plain_split(name, files, labels, num_threads, shards, False, _bboxes_of(files, bbox)))
    return splits


def _bboxes_of(files, bbox):
    if bbox is None:
        return None
    ids = [os.path.splitext(os.path.basename(f))[0] for f in files]
    missing = [f for f, i in zip(files, ids) if i not in bbox]
    if missing:
        raise ValueError("no bounding box for %s" % missing[:10])
    return [bbox[i] for i in ids]


# ---------------------------------------------------------------------------------------- Cars196
CARS_RANGES = {"train": range(0, 98), "validation": range(98, 196)}


def cars_annotations(data_dir):
    """cars_annos.mat's annotations sorted by relative_im_path: [(path, [xmin, ymin, xmax, ymax], class)]."""
    from scipy.io import loadmat
    path = os.path.join(data_dir, "cars_annos.mat")
    if not os.path.isfile(path):
        raise ValueError("%s does not exist" % path)
    ann = sorted(loadmat(path)["annotations"].ravel(), key=lambda a: str(a[0][0]))
    scalar = lambda v: np.asarray(v).reshape(-1)[0]
    return [(str(a[0][0]), [int(scalar(a[k])) for k in (1, 2, 3, 4)], int(scalar(a[5]))) for a in ann]


def cars_files(name, data_dir, ann, archive_basename="car_ims"):
    """_find_image_files: the sorted .jpg names of <archive_basename>.tgz paired in order with the sorted
    annotations' classes (label = class - 1), grouped by label in the split's range, then shuffled."""
    import tarfile
    tgz = os.path.join(data_dir, archive_basename + ".tgz")
    if not os.path.isfile(tgz):
        raise ValueError("%s does not exist" % tgz)
    with tarfile.open(tgz, "r") as t:
        jpgs = sorted(fn for fn in t.getnames() if fn.endswith(".jpg"))
    if len(jpgs) != len(ann):
        raise ValueError("%s holds %d .jpg files, cars_annos.mat %d annotations" % (tgz, len(jpgs), len(ann)))
    classes = [c for _, _, c in ann]
    per = [[] for _ in range(max(classes))]
    for fn, c in zip(jpgs, classes):
        if c - 1 in CARS_RANGES[name]:
            per[c - 1].append(os.path.join(data_dir, fn))
    files, labels = [], []
    for label in range(len(per)):
        if label in CARS_RANGES[name]:
            if not per[label]:
                raise ValueError("cars_annos.mat: class %d (below the largest, %d) has no image" % (label + 1, len(per)))
            files += per[label]
            labels += [label] * len(per[label])
    return shuffled(files, labels) if files else ([], [])


def cars_splits(data_dir, *, num_threads=16, use_bbox=False):
    """build_cars196_zeroshot.py: labels 0-97 train, 98-195 validation, 128 shards each."""
    ann = cars_annotations(data_dir)
    bbox = {os.path.splitext(os.path.basename(p))[0]: b for p, b, _ in ann} if use_bbox else None
    splits = []
    for name in ("train", "validation"):
        shard_layout(name, 0, num_threads, 128)
        files, labels = cars_files(name, data_dir, ann)
        splits.append(_plain_split(name, files, labels, num_threads, 128, False, _bboxes_of(files, bbox)))
    return splits


# -------------------------------------------------------------------------------------------- SOP
def sop_splits(input_dir, *, train_shards=128, validation_shards=16, num_threads=8):
    """build_sop.py: Ebay_train.txt (shuffled) and Ebay_test.txt, 'image_id class_id super_class_id path'
    per line after the header, label class_id - 1."""
    splits = []
    for name, txt, shards, shuffle in (("train", "Ebay_train.txt", train_shards, True),
                                       ("validation", "Ebay_test.txt", validation_shards, False)):
        shard_layout(name, 0, num_threads, shards)
        files, labels = [], []
        for n, l in enumerate(_lines(input_dir + "/" + txt, "file list")):
            t = l.strip().split()
            if t and t[0] == "image_id":
                continue
            try:
                if len(t) != 4:
                    raise ValueError("expected 4 fields")
                labels.append(int(t[1]) - 1)
            except ValueError as e:
                raise ValueError("%s line %d: %s: %r" % (txt, n + 1, e, l))
            files.append(os.path.join(input_dir, t[3]))
        if shuffle:
            files, labels = shuffled(files, labels)
        splits.append(_plain_split(name, files, labels, num_threads, shards, True))
    return splits


# ------------------------------------------------------------------------------------------ writer
class _Checked(NamedTuple):
    data: bytes                 # the bytes the record holds (re-encoded for a converted image)
    shape: Optional[tuple]      # (h, w) of the decode; None while the device has not checked the image
    crop: Optional[np.ndarray]  # the uint8 pixels of the item's bbox crop, None without a bbox
    error: Optional[str]        # why the image cannot be decoded


# the formats tf.image.decode_jpeg decodes, by the magic bytes TF 1.14's DecodeImageOp classifies them by
TF_DECODE_MAGIC = (b"\xff\xd8\xff", b"\x89PNG\r\n\x1a\n", b"GIF8")


def _pil(data):
    """(uint8 [h, w, 3] pixels, None) of what tf.image.decode_jpeg accepts -- a JPEG, a PNG or a GIF of one
    frame -- decoded by PIL, or (None, why not).  Other formats PIL opens (BMP, TIFF, WebP, ...) are refused,
    as TF refuses them."""
    if not bytes(data[:8]).startswith(TF_DECODE_MAGIC):
        return None, "not a JPEG, PNG or GIF (the formats tf.image.decode_jpeg decodes)"
    try:
        if data[:4] == b"GIF8":
            from PIL import Image
            with Image.open(io.BytesIO(data)) as im:
                if getattr(im, "n_frames", 1) > 1:
                    return None, "an animated GIF (tf.image.decode_jpeg refuses it)"
        return decode_rgb(io.BytesIO(data)), None
    except Exception as e:      # PIL raises OSError, ValueError, SyntaxError, ... for a bad image
        return None, "%s: %s" % (type(e).__name__, e)


def _pil_check(item, data):
    """_Checked of the PIL check of `data`: the height and width, and only the crop's pixels are kept."""
    a, err = _pil(data)
    if err is not None:
        return _Checked(data, None, None, err)
    crop = None
    if item.bbox is not None:
        y, x, h, w = crop_window(item.bbox, a.shape[0], a.shape[1], item.path)
        crop = np.ascontiguousarray(a[y:y + h, x:x + w])
    return _Checked(data, a.shape[:2], crop, None)


def _load(item, pil_check):
    """Runs on the pool: reads the file, converts a PNG / CMYK image and, with pil_check, checks it."""
    with open(item.path, "rb") as f:
        data = f.read()
    if item.convert is not None:
        a, err = _pil(data)
        if err is not None:
            return _Checked(data, None, None, err)
        data = encode_jpeg(a)
    return _pil_check(item, data) if pil_check else _Checked(data, None, None, None)


class _Shards:
    """Writes the records of a split shard by shard, in order; every shard, empty ones too, is written
    under a hidden temporary name and renamed once complete."""

    def __init__(self, out_dir, shards):
        self.out_dir, self.shards, self.k, self.f = out_dir, shards, -1, None

    def _open_next(self):
        self._close()
        self.k += 1
        name = self.shards[self.k][0]
        self.tmp = os.path.join(self.out_dir, ".%s.partial" % name)
        self.f = open(self.tmp, "wb")

    def _close(self):
        if self.f is not None:
            self.f.flush()
            os.fsync(self.f.fileno())
            self.f.close()
            self.f = None
            os.replace(self.tmp, os.path.join(self.out_dir, self.shards[self.k][0]))

    def write(self, i, features):
        while self.f is None or i >= self.shards[self.k][2]:
            self._open_next()
        write_record(self.f, [serialize_example(features)])

    def close(self):
        while self.k + 1 < len(self.shards):
            self._open_next()
        self._close()

    def abort(self):
        if self.f is not None:
            self.f.close()
            self.f = None
            os.remove(self.tmp)


def _decode_failed(split, item, error):
    if split.skip_invalid:
        log.warning("%s: invalid image %s (%s) - skipped", split.name, item.path, error)
        return True
    raise ValueError("build_data: cannot decode %s: %s" % (item.path, error))


class _DeviceCheck:
    """The device check of batches of encoded images: two jpeg.JpegDecoder alternate on one copy stream, so
    batch j + 1 is parsed and enqueued before the statuses of batch j are read."""

    def __init__(self, device):
        import torch
        from .jpeg import JpegDecoder
        if not torch.cuda.is_available():
            raise RuntimeError("build_data: check='device' needs a CUDA device (check='pil' checks with PIL)")
        self.torch, self.dev = torch, torch.device(device)
        self.decoders = [JpegDecoder(self.dev), JpegDecoder(self.dev)]
        self.stream = torch.cuda.Stream(self.dev)
        self.status = [torch.zeros(BATCH, dtype=torch.int32).pin_memory() for _ in range(2)]
        self.j = 0

    def enqueue(self, buffers):
        torch, slot = self.torch, self.j % 2
        self.j += 1
        _, jobs, out, status = self.decoders[slot].enqueue(buffers, stream=self.stream)
        st = self.status[slot][:len(buffers)]
        with torch.cuda.stream(self.stream):
            st.copy_(status[:len(buffers)], non_blocking=True)
            done = torch.cuda.Event()
            done.record(self.stream)
        return jobs, out, st, done

    def results(self, pending, windows):
        """[(ok, h, w, uint8 pixels of windows[i] or None)] of an enqueued batch; windows[i] is a function
        of (h, w) giving (y, x, h, w), or None when the pixels are not needed."""
        jobs, out, st, done = pending
        done.synchronize()
        res = []
        for i, s in enumerate(st.numpy()):
            if s != 0:
                res.append((False, 0, 0, None))
                continue
            h, w = int(jobs[i]["win_h"]), int(jobs[i]["win_w"])
            px = None
            if windows[i] is not None:
                y, x, ch, cw = windows[i](h, w)
                o = int(jobs[i]["out"])
                px = out[o:o + h * w * 3].view(h, w, 3)[y:y + ch, x:x + cw].cpu().numpy()
            res.append((True, h, w, px))
        return res


def _run_split(split, out_dir, check, pool, device):
    shards = _Shards(out_dir, split.shards)
    batches = [list(range(a, min(a + BATCH, len(split.items)))) for a in range(0, len(split.items), BATCH)]
    dc = _DeviceCheck(device) if check == "device" else None
    written = 0

    def finish(idx, loaded, pending):
        nonlocal written
        items = [split.items[i] for i in idx]
        if dc is not None:
            windows = [None if it.bbox is None or c.error is not None
                       else (lambda h, w, it=it: crop_window(it.bbox, h, w, it.path)) for it, c in zip(items, loaded)]
            dev = dc.results(pending, windows)
            # the images the device refused go to PIL on the pool
            refused = {k: pool.submit(_pil_check, items[k], c.data) for k, c in enumerate(loaded)
                       if c.error is None and not dev[k][0]}
            loaded = [refused[k].result() if k in refused else
                      c if c.error is not None else c._replace(shape=dev[k][1:3], crop=dev[k][3])
                      for k, c in enumerate(loaded)]
        crops = {k: pool.submit(encode_jpeg, c.crop) for k, c in enumerate(loaded) if c.crop is not None}
        for k, (i, it, c) in enumerate(zip(idx, items, loaded)):
            if c.error is not None:
                if _decode_failed(split, it, c.error):
                    continue
            data, (h, w) = c.data, c.shape
            if k in crops:
                data, (h, w) = crops[k].result(), c.crop.shape[:2]
            shards.write(i, it.example(data, int(h), int(w)))
            written += 1

    try:
        pending = None
        for idx, loaded in read_ahead(pool, batches, lambda i: _load(split.items[i], dc is None)):
            if dc is not None:
                nxt = (idx, loaded, dc.enqueue([c.data for c in loaded]))
                if pending is not None:
                    finish(*pending)
                pending = nxt
            else:
                finish(idx, loaded, None)
        if pending is not None:
            finish(*pending)
        shards.close()
    except BaseException:
        shards.abort()
        raise
    log.info("%s: wrote %d of %d images to %d shards", split.name, written, len(split.items), len(split.shards))
    return written


def write_splits(splits, output_dir, *, check="device", num_workers=None, device="cuda"):
    """Writes the shards of `splits` to output_dir (made if missing) after checking that none exists yet.
    Returns {split name: records written}."""
    if check not in ("device", "pil"):
        raise ValueError("check must be 'device' or 'pil' (got %r)" % (check,))
    names = [s[0] for sp in splits for s in sp.shards]
    if os.path.exists(output_dir) and not os.path.isdir(output_dir):
        raise ValueError("output directory %s is not a directory" % output_dir)
    existing = [n for n in names if os.path.lexists(os.path.join(output_dir, n))]
    if existing:
        raise ValueError("output %s already exists" % os.path.join(output_dir, existing[0]))
    missing = [it.path for sp in splits for it in sp.items if not os.path.isfile(it.path)]
    if missing:
        raise ValueError("%d listed image(s) do not exist, e.g. %s" % (len(missing), missing[0]))
    os.makedirs(output_dir, exist_ok=True)
    pool = ThreadPoolExecutor(max_workers=num_workers or min(32, os.cpu_count() or 1))
    try:
        return {sp.name: _run_split(sp, output_dir, check, pool, device) for sp in splits}
    except BaseException:
        done = [n for n in names if os.path.exists(os.path.join(output_dir, n))]
        if done:
            log.error("build_data: %d shard(s) of this build were completed in %s before it failed (%s, ...); they "
                      "are kept, and a new build into %s is refused until they are removed",
                      len(done), output_dir, done[0], output_dir)
        raise
    finally:
        pool.shutdown(wait=True, cancel_futures=True)


BUILDERS = {"imagenet": imagenet_splits, "food101": food101_splits, "cub_200_2011": cub_splits,
            "cars196_zeroshot": cars_splits, "SOP": sop_splits}


def build(dataset, output_dir, *args, check="device", num_workers=None, device="cuda", **flags):
    """Lists dataset (a BUILDERS key) with the reference script's flags, checks it and writes its shards to
    output_dir.  Returns {split name: records written}."""
    if dataset not in BUILDERS:
        raise ValueError("unknown dataset %r: one of %s" % (dataset, sorted(BUILDERS)))
    splits = BUILDERS[dataset](*args, **flags)
    return write_splits(splits, output_dir, check=check, num_workers=num_workers, device=device)


# --------------------------------------------------------------------------------------------- CLI
def str2bool(v):
    """dataset_utils.str2bool (and TF's boolean flag values)."""
    if v.lower() in ("yes", "true", "t", "y", "1"):
        return True
    if v.lower() in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError("Boolean value expected.")


def _parser():
    p = argparse.ArgumentParser(prog="python -m assembled_cnn_b200.build_data",
                                description="Build the reference's TFRecord shards from raw image folders.")
    sub = p.add_subparsers(dest="dataset", required=True)

    def common(sp):
        sp.add_argument("--num_workers", type=int, default=None, help="host threads (default: cores, at most 32)")
        sp.add_argument("--check", choices=("device", "pil"), default="device",
                        help="decode the scans on the GPU (PIL for the rest) or with PIL only")
        sp.add_argument("--device", default="cuda")

    b = lambda sp, name, default: sp.add_argument("--" + name, type=str2bool, nargs="?", const=True, default=default)
    im = sub.add_parser("imagenet")
    for name, default in (("train_directory", "/tmp/"), ("validation_directory", "/tmp/"),
                          ("output_directory", "/tmp/"), ("labels_file", "imagenet_lsvrc_2015_synsets.txt"),
                          ("imagenet_metadata_file", "imagenet_metadata.txt")):
        im.add_argument("--" + name, default=default)
    im.add_argument("--bounding_box_file", default=None,
                    help="default: %s if it exists, else no boxes" % IMAGENET_BBOX_DEFAULT)
    im.add_argument("--logits_file_path", default=None,
                    help="default: %s if it is a directory, else no image/logit" % IMAGENET_LOGITS_DEFAULT)
    im.add_argument("--train_shards", type=int, default=1024)
    im.add_argument("--validation_shards", type=int, default=128)
    im.add_argument("--num_threads", type=int, default=8)
    for name in ("make_val", "make_train"):          # tf.app.flags.DEFINE_boolean: --x, --x=False, --nox
        b(im, name, True)
        im.add_argument("--no" + name, dest=name, action="store_false")
    im.add_argument("--validation_labels_file", default=None,
                    help="imagenet_2012_validation_synset_labels.txt: validation_directory is the flat directory")
    for name, threads, shards in (("food101", 8, True), ("SOP", 8, True), ("cub_200_2011", 16, False),
                                  ("cars196_zeroshot", 16, False)):
        sp = sub.add_parser(name)
        if name == "SOP":
            sp.add_argument("-i", "--input_dir", default=None)
        else:
            sp.add_argument("-d", "--data_dir", default=None)
        sp.add_argument("-o", "--output_dir", default=None)
        if shards:
            sp.add_argument("--train_shards", type=int, default=128)
            sp.add_argument("--validation_shards", type=int, default=16)
        else:
            b(sp, "use_bbox", False)
        sp.add_argument("--num_threads", type=int, default=threads)
    for sp in sub.choices.values():
        common(sp)
    return p


def main(argv=None):
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(message)s")
    a = vars(_parser().parse_args(argv))
    dataset = a.pop("dataset")
    run = {k: a.pop(k) for k in ("check", "num_workers", "device")}
    if dataset == "imagenet":
        out = a.pop("output_directory")
        # a path on the command line must exist (build raises before any shard otherwise); without the flag
        # the reference's default is used where it exists
        if a["bounding_box_file"] is None:
            if os.path.isfile(IMAGENET_BBOX_DEFAULT):
                a["bounding_box_file"] = IMAGENET_BBOX_DEFAULT
            else:
                log.info("no --bounding_box_file and no %s: no boxes", IMAGENET_BBOX_DEFAULT)
        if a["logits_file_path"] is None:
            if os.path.isdir(IMAGENET_LOGITS_DEFAULT):
                a["logits_file_path"] = IMAGENET_LOGITS_DEFAULT
            else:
                log.info("no --logits_file_path and no %s: no image/logit", IMAGENET_LOGITS_DEFAULT)
        args = (a.pop("train_directory"), a.pop("validation_directory"))
    else:
        data_dir = a.pop("input_dir" if dataset == "SOP" else "data_dir")
        out = a.pop("output_dir")
        if data_dir is None or out is None:
            _parser().parse_args([dataset, "--help"])
        args = (data_dir,)
    written = build(dataset, out, *args, **run, **a)
    for name, n in written.items():
        log.info("%s: %d records", name, n)
    return written


if __name__ == "__main__":
    main(sys.argv[1:])
