"""The data side of the ImageNet classification evaluation (classifier.evaluate(input_fn_eval),
nets/run_loop_classification.py:397-402,446-448): the validation shards, the TFRecord / tf.train.Example
reader, the eval preprocessing geometry and the descriptors of acnn_resize_crop_u8.  The device side is
model_fns.evaluate_classification; the zero-shot retrieval evaluation (model_fns.evaluate_retrieval) reads
the same shards with missing_label=-1.

  validation_files      utils/data_util.py:161-170      sorted(glob(data_dir/val_regex))
  read_records          utils/data_util.py:173-208      image/encoded and image/class/label of every record
  eval_geometry         utils/data_util.py:267-345,     the imagenet-family preprocessing_type dispatch,
                        preprocessing/imagenet_preprocessing.py:100-119,158-226,295-313
                                                        _smallest_size_at_least, central_crop
Decoding is imagenet_c.decode_rgb (PIL); the channel means are imagenet_c.CHANNEL_MEANS.
"""
from __future__ import annotations

import glob
import os
import re
import struct

import numpy as np

from .imagenet_c import CHANNEL_MEANS, decode_rgb  # noqa: F401  (re-exported for the evaluation)

# include/acnn.h acnn_resize_desc
DESC_DTYPE = np.dtype([("src", "<u8"), ("src_h", "<i4"), ("src_w", "<i4"), ("rsz_h", "<i4"), ("rsz_w", "<i4"),
                       ("crop_y", "<i4"), ("crop_x", "<i4")])
assert DESC_DTYPE.itemsize == 32

# ------------------------------------------------------------------------------------------ CRC32C
_CRC_TABLE = []
for _n in range(256):
    _c = _n
    for _ in range(8):
        _c = (_c >> 1) ^ 0x82F63B78 if _c & 1 else _c >> 1
    _CRC_TABLE.append(_c)


def crc32c(data):
    """CRC-32C (Castagnoli, reflected polynomial 0x82F63B78) of `data`."""
    c = 0xFFFFFFFF
    for b in data:
        c = _CRC_TABLE[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def masked_crc32c(data):
    """The TFRecord checksum: the CRC rotated right by 15 bits plus 0xa282ead8."""
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


# ---------------------------------------------------------------------------------------- TFRecord
def validation_files(data_dir, val_regex="validation-*"):
    """get_filenames(is_training=False): the shards matching data_dir/val_regex, sorted."""
    files = sorted(glob.glob(os.path.join(data_dir, val_regex)))
    if not files:
        raise FileNotFoundError("evaluation: no file matches %s" % os.path.join(data_dir, val_regex))
    return files


def _varint(buf, pos, end):
    v, shift = 0, 0
    while True:
        if pos >= end or shift > 63:
            raise ValueError("bad varint")
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        if not b & 0x80:
            return v, pos
        shift += 7


def _fields(buf, pos, end):
    """(field number, wire type, value) of each field of the protobuf message buf[pos:end]: a varint's
    value, a length-delimited field's (start, end), a fixed-width field's start."""
    while pos < end:
        key, pos = _varint(buf, pos, end)
        field, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos, end)
        elif wt == 1:
            v, pos = pos, pos + 8
        elif wt == 2:
            n, pos = _varint(buf, pos, end)
            v, pos = (pos, pos + n), pos + n
        elif wt == 5:
            v, pos = pos, pos + 4
        else:
            raise ValueError("unsupported wire type %d" % wt)
        if pos > end:
            raise ValueError("field runs past its message")
        yield field, wt, v


def _float_list(buf, feature):
    """float32 array of a Feature's float_list(2) -> value(1), packed (fixed32 run) or not."""
    vals = []
    for f, wt, v in _fields(buf, *feature):
        if f == 2 and wt == 2:                       # FloatList
            for f2, wt2, v2 in _fields(buf, *v):
                if f2 == 1 and wt2 == 5:
                    vals.append(bytes(buf[v2:v2 + 4]))
                elif f2 == 1 and wt2 == 2:
                    if (v2[1] - v2[0]) % 4:
                        raise ValueError("packed FloatList of %d bytes" % (v2[1] - v2[0]))
                    vals.append(bytes(buf[v2[0]:v2[1]]))
    return np.frombuffer(b"".join(vals), dtype="<f4").astype(np.float32)


def parse_example(buf, logits=False, missing_label=None):
    """(label, (start, end) of the encoded image in buf) of a serialised tf.train.Example: the
    'image/class/label' int64 and 'image/encoded' bytes features (parse_example_proto).  Only the
    protobuf wire format is read: Example.features(1) -> Features.feature(1) map entries {key(1),
    value(2)} -> Feature.bytes_list(1) / int64_list(3) -> value(1).  A repeated key keeps its last
    value, as protobuf's map parsing does.  logits=True appends the float32 values of the
    'image/logit' FloatList (the knowledge-distillation teacher logits; empty when the feature is
    absent, as tf.VarLenFeature).  An Example without 'image/class/label' raises ValueError unless
    missing_label is given, which is then its label (-1: the reference's default_value, the
    distractor label of the retrieval evaluation)."""
    feats = {}
    for f, wt, v in _fields(buf, 0, len(buf)):
        if f != 1 or wt != 2:
            continue
        for f2, wt2, entry in _fields(buf, *v):
            if f2 != 1 or wt2 != 2:
                continue
            key = value = None
            for f3, wt3, kv in _fields(buf, *entry):
                if f3 == 1 and wt3 == 2:
                    key = bytes(buf[kv[0]:kv[1]])
                elif f3 == 2 and wt3 == 2:
                    value = kv
            if key in (b"image/encoded", b"image/class/label", b"image/logit"):
                feats[key] = value
    if b"image/encoded" not in feats or (b"image/class/label" not in feats and missing_label is None):
        raise ValueError("Example without image/encoded or image/class/label")
    enc = []
    for f, wt, v in _fields(buf, *feats[b"image/encoded"]):
        if f == 1 and wt == 2:                       # BytesList
            enc += [v2 for f2, wt2, v2 in _fields(buf, *v) if f2 == 1 and wt2 == 2]
    labels = [] if b"image/class/label" in feats else [int(missing_label)]
    for f, wt, v in _fields(buf, *feats.get(b"image/class/label", (0, 0))):
        if f == 3 and wt == 2:                       # Int64List, packed or not
            for f2, wt2, v2 in _fields(buf, *v):
                if f2 == 1 and wt2 == 0:
                    labels.append(v2)
                elif f2 == 1 and wt2 == 2:
                    p, e = v2
                    while p < e:
                        x, p = _varint(buf, p, e)
                        labels.append(x)
    if len(enc) != 1 or len(labels) != 1:
        raise ValueError("image/encoded and image/class/label must hold one value each (got %d, %d)"
                         % (len(enc), len(labels)))
    label = labels[0] - (1 << 64) if labels[0] >= 1 << 63 else labels[0]
    if logits:
        lg = _float_list(buf, feats[b"image/logit"]) if feats.get(b"image/logit") else np.zeros(0, np.float32)
        return label, enc[0], lg
    return label, enc[0]


def read_records(path, logits=False, missing_label=None):
    """[(label, offset, length)] of every record of a TFRecord file: the label and the byte range of the
    encoded image in the file (logits=True: [(label, offset, length, float32 image/logit values)];
    missing_label: the label of a record without one, as parse_example).  A
    record is u64 length, u32 masked CRC32C of the length, the data, u32 masked CRC32C of the data.  The
    length's CRC is verified; the data's is not (a pure-Python CRC over the 6.4 GB of ImageNet validation
    JPEGs would take far longer than the evaluation).  A truncated or corrupt record raises ValueError
    naming the file and the record's byte offset."""
    with open(path, "rb") as f:
        data = f.read()
    out, pos, n = [], 0, len(data)
    while pos < n:
        if pos + 12 > n:
            raise ValueError("%s: truncated record header at byte offset %d" % (path, pos))
        head = data[pos:pos + 8]
        (length,) = struct.unpack("<Q", head)
        (crc,) = struct.unpack("<I", data[pos + 8:pos + 12])
        if masked_crc32c(head) != crc:
            raise ValueError("%s: corrupt record length at byte offset %d" % (path, pos))
        start = pos + 12
        if start + length + 4 > n:
            raise ValueError("%s: truncated record at byte offset %d" % (path, pos))
        try:
            ex = parse_example(memoryview(data)[start:start + length], logits, missing_label)
        except ValueError as e:
            raise ValueError("%s: bad tf.train.Example in the record at byte offset %d: %s" % (path, pos, e))
        label, (a, b) = ex[:2]
        out.append((label, start + a, b - a) + tuple(ex[2:]))
        pos = start + length + 4
    return out


def read_encoded(path, offset, length):
    with open(path, "rb") as f:
        f.seek(offset)
        return f.read(length)


# ---------------------------------------------------------------------------------------- geometry
_TYPE_NNN_A = re.compile("imagenet_[0-9]{3}a")
_TYPE_NNN = re.compile("imagenet_[0-9]{3}")
_OUT_OF_SCOPE = ("reid", "reid_224", "inception_331", "inception_600")


def eval_size(preprocessing_type, image_size=224):
    """(S, crop_type) of preprocess_image(is_training=False) for an imagenet-family preprocessing_type
    (utils/data_util.py:267-345, the same regular expressions in the same order).  S must be a multiple
    of 32 (the model's constraint): ValueError otherwise."""
    if preprocessing_type == "imagenet":
        s, crop_type = image_size, 0
    elif preprocessing_type == "imagenet_224_256":
        s, crop_type = 256, 0
    elif preprocessing_type == "imagenet_224_256a":
        s, crop_type = 256, 1
    elif _TYPE_NNN_A.match(preprocessing_type):
        s, crop_type = int(preprocessing_type.split("_")[1][0:3]), 1
    elif _TYPE_NNN.match(preprocessing_type):
        s, crop_type = int(preprocessing_type.split("_")[1]), 0
    elif preprocessing_type in _OUT_OF_SCOPE:
        raise NotImplementedError("preprocessing_type %r (reid / inception preprocessing) is not supported by "
                                  "the classification evaluation" % preprocessing_type)
    else:
        raise NotImplementedError("unknown preprocessing_type %r" % preprocessing_type)
    s = int(s)
    if s < 32 or s % 32:
        raise ValueError("preprocessing_type %r evaluates at %d px; the model needs a multiple of 32"
                         % (preprocessing_type, s))
    return s, crop_type


def smallest_size_at_least(height, width, resize_min):
    """_smallest_size_at_least in float32, as the reference computes it in tf.float32: the product can
    round below the integer (a 256 target on a 107-pixel side gives 255)."""
    resize_min = np.float32(resize_min)
    h, w = np.float32(height), np.float32(width)
    scale = resize_min / np.minimum(h, w)
    return int(np.int32(h * scale)), int(np.int32(w * scale))


def eval_geometry(h, w, preprocessing_type="imagenet", image_size=224):
    """(S, rsz_h, rsz_w, crop_y, crop_x) of the eval preprocessing of an h x w image: the aspect-preserving
    resize to resize_min = int(S * (1.0 / 0.875)) (crop_type 0) or S + 1 (crop_type 1), then the central
    S x S crop at ((rsz - S) // 2)."""
    s, crop_type = eval_size(preprocessing_type, image_size)
    resize_min = s + 1 if crop_type == 1 else int(s * (1.0 / 0.875))
    rh, rw = smallest_size_at_least(h, w, resize_min)
    return s, rh, rw, (rh - s) // 2, (rw - s) // 2


def check_descriptors(desc, n_valid, S):
    """The host-side check of descriptors before they go to the device (acnn_resize_crop_u8 does not
    read them on the host): rows < n_valid need a source address, source sizes >= 1 and the S x S crop
    inside the resized image."""
    d = desc[:n_valid]
    bad = (d["src"] == 0) | (d["src_h"] < 1) | (d["src_w"] < 1) | (d["crop_y"] < 0) | (d["crop_x"] < 0) \
        | (d["crop_y"].astype(np.int64) + S > d["rsz_h"]) | (d["crop_x"].astype(np.int64) + S > d["rsz_w"])
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError("resize descriptor %d is invalid for S=%d: %s" % (i, S, d[i]))


def decode_record(path, offset, length, preprocessing_type="imagenet", image_size=224):
    """(uint8 [H, W, 3], eval_geometry) of the image stored at path[offset:offset + length]."""
    import io
    a = decode_rgb(io.BytesIO(read_encoded(path, offset, length)))
    return a, eval_geometry(a.shape[0], a.shape[1], preprocessing_type, image_size)
