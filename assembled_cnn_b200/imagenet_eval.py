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

The TFRecord writer of the knowledge-distillation shards (model_fns.extract_teacher_logits, the reference's
datasets/build_imagenet_data.py --logits_file_path) is here too, so the record format lives in one module:
write_record frames a record, add_float_feature adds a float feature to a serialised Example and
FloatFeatureWriter copies whole files with one added to every record.  serialize_example writes a whole
Example (the dataset builders, build_data).
"""
from __future__ import annotations

import glob
import os
import re
import struct

import numpy as np

from . import native
from .imagenet_c import CHANNEL_MEANS, decode_rgb  # noqa: F401  (re-exported for the evaluation)

# include/acnn.h acnn_resize_desc
DESC_DTYPE = np.dtype([("src", "<u8"), ("src_h", "<i4"), ("src_w", "<i4"), ("rsz_h", "<i4"), ("rsz_w", "<i4"),
                       ("crop_y", "<i4"), ("crop_x", "<i4")])
assert DESC_DTYPE.itemsize == 32

# the knowledge-distillation teacher logits of a record (utils/data_util.py parse_record_sup)
LOGIT_KEY = b"image/logit"

# ------------------------------------------------------------------------------------------ CRC32C
def crc32c(data, crc=0):
    """CRC-32C (Castagnoli, reflected polynomial 0x82F63B78) of `data`, continued from `crc` (0 starts a
    new one): libacnn's host acnn_crc32c."""
    return native.crc32c(data, crc)


def _mask(c):
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def masked_crc32c(data):
    """The TFRecord checksum: the CRC rotated right by 15 bits plus 0xa282ead8."""
    return _mask(crc32c(data))


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
    length's CRC is verified; the data's is not (FloatFeatureWriter verifies it when it copies a record).
    A truncated or corrupt record raises ValueError naming the file and the record's byte offset."""
    data = _read_file(path)
    out = []
    for pos, start, length in record_frames(data, path):
        try:
            ex = parse_example(memoryview(data)[start:start + length], logits, missing_label)
        except ValueError as e:
            raise ValueError("%s: bad tf.train.Example in the record at byte offset %d: %s" % (path, pos, e))
        label, (a, b) = ex[:2]
        out.append((label, start + a, b - a) + tuple(ex[2:]))
    return out


def _read_file(path):
    with open(path, "rb") as f:
        return f.read()


def record_frames(data, path):
    """(byte offset, data start, data length) of every record of the TFRecord file contents `data`, in
    order.  The length's CRC is verified: a truncated record or a corrupt length raises ValueError naming
    `path` and the record's byte offset.  The data's CRC sits at data[start + length:][:4]."""
    pos, n = 0, len(data)
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
        yield pos, start, length
        pos = start + length + 4


# ------------------------------------------------------------------------------- TFRecord writer
def write_record(f, pieces):
    """Writes one TFRecord record to the binary file `f`: u64 length, masked CRC32C of the length, the data
    (the bytes-like `pieces` back to back, not joined in memory), masked CRC32C of the data."""
    head = struct.pack("<Q", sum(len(p) for p in pieces))
    c = 0
    for p in pieces:
        c = crc32c(p, c)
    f.write(head + struct.pack("<I", masked_crc32c(head)))
    for p in pieces:
        f.write(p)
    f.write(struct.pack("<I", _mask(c)))


def _encode_varint(v):
    out = bytearray()
    while v > 0x7F:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _len_field(field, payload_len):
    """The key and length of a length-delimited field (wire type 2) of payload_len bytes."""
    return _encode_varint(field << 3 | 2) + _encode_varint(payload_len)


def serialize_example(features):
    """A serialised tf.train.Example of `features` {key: (kind, values)}, kind 'bytes' (a list of bytes),
    'int64' or 'float' (a list of numbers; float32 on the wire).  The map entries go in key order and the
    numeric lists packed, as proto3 writes them; an empty list still sets the Feature's kind, as
    tf.train.Feature(float_list=tf.train.FloatList(value=[])) does."""
    entries = []
    for key in sorted(features):
        kind, values = features[key]
        kb = key.encode() if isinstance(key, str) else key
        if kind == "bytes":
            body = b"".join(_len_field(1, len(v)) + v for v in values)
            feature = _len_field(1, len(body)) + body                       # Feature.bytes_list
        elif kind == "float":
            vals = np.asarray(values, dtype="<f4").tobytes()
            body = _len_field(1, len(vals)) + vals if vals else b""
            feature = _len_field(2, len(body)) + body                       # Feature.float_list
        elif kind == "int64":
            vals = b"".join(_encode_varint(int(v) & 0xFFFFFFFFFFFFFFFF) for v in values)
            body = _len_field(1, len(vals)) + vals if vals else b""
            feature = _len_field(3, len(body)) + body                       # Feature.int64_list
        else:
            raise ValueError("unknown feature kind %r of %s" % (kind, key))
        entry = _len_field(1, len(kb)) + kb + _len_field(2, len(feature)) + feature
        entries.append(_len_field(1, len(entry)) + entry)                   # Features.feature map entry
    feats = b"".join(entries)
    return _len_field(1, len(feats)) + feats                                 # Example.features


def features_span(example, key):
    """(start, end) of the Features message inside the serialised tf.train.Example `example`.  ValueError
    unless the Example is exactly one `features` field, or when one of its map entries has `key`."""
    fields = list(_fields(example, 0, len(example)))
    if len(fields) != 1 or fields[0][:2] != (1, 2):
        raise ValueError("the Example is not one features message")
    span = fields[0][2]
    for f, wt, entry in _fields(example, *span):
        if f == 1 and wt == 2:
            for f2, wt2, kv in _fields(example, *entry):
                if f2 == 1 and wt2 == 2 and bytes(example[kv[0]:kv[1]]) == key:
                    raise ValueError("the Example already holds %s" % key.decode())
    return span


def add_float_feature(example, key, values):
    """The serialised tf.train.Example `example` with one more Features map entry, {key: Feature{float_list
    {value: float32 `values`, packed}}}, as pieces for write_record: (the Example's key and new length, its
    Features message as it is, the new entry).  The input's features keep their bytes and order, so a
    protobuf parser reads the input's features plus the new one.  ValueError as features_span."""
    a, b = features_span(example, key)
    vals = np.ascontiguousarray(values, dtype="<f4").tobytes()
    flist = _len_field(1, len(vals)) + vals                          # FloatList.value (packed)
    feature = _len_field(2, len(flist)) + flist                      # Feature.float_list
    entry = _len_field(1, len(key)) + key + _len_field(2, len(feature)) + feature
    entry = _len_field(1, len(entry)) + entry                        # Features.feature map entry
    return _len_field(1, (b - a) + len(entry)), example[a:b], entry  # Example.features


def appendable_records(path, key):
    """[(offset, length)] of the encoded image of every record of the TFRecord file `path`, each record
    checked as add_float_feature's input (one features message without `key`) and as parse_example's (an
    image/encoded; a missing label is allowed).  ValueError naming the file and the record's byte offset."""
    data = _read_file(path)
    out = []
    for pos, start, length in record_frames(data, path):
        ex = memoryview(data)[start:start + length]
        try:
            features_span(ex, key)
            _, (a, b) = parse_example(ex, missing_label=-1)
        except ValueError as e:
            raise ValueError("%s: the record at byte offset %d: %s" % (path, pos, e))
        out.append((start + a, b - a))
    return out


class FloatFeatureWriter:
    """Writes a copy of each TFRecord file of `jobs` [(input path, output path)] with one float feature
    `key` added to every record (add_float_feature), fed the values record by record across the files in
    order (`add`).  While a file is copied, the data CRC of each of its input records is verified (a
    mismatch raises ValueError naming the file and the record's byte offset), so a fresh checksum never
    covers corrupt bytes.  Each output is written under a hidden temporary name in its directory and
    renamed once complete; `abort` removes the one being written.  One input file is held in memory."""

    def __init__(self, jobs, key):
        self.jobs, self.key = list(jobs), key
        self.j, self.f = -1, None

    def add(self, rows):
        """Appends one record per row of the float32 [n, k] `rows` (copied before the call returns)."""
        for row in np.asarray(rows, dtype=np.float32):
            while self.f is None or self.i == len(self.frames):
                self._next_file()
            pos, start, length = self.frames[self.i]
            src = self.jobs[self.j][0]
            data = memoryview(self.data)[start:start + length]
            (crc,) = struct.unpack("<I", self.data[start + length:start + length + 4])
            if masked_crc32c(data) != crc:
                raise ValueError("%s: corrupt record data at byte offset %d" % (src, pos))
            try:
                pieces = add_float_feature(data, self.key, row)
            except ValueError as e:
                raise ValueError("%s: the record at byte offset %d: %s" % (src, pos, e))
            write_record(self.f, pieces)
            self.i += 1

    def close(self):
        """Completes the files after the last one fed, which must hold no record."""
        while self.f is None or self.i == len(self.frames):
            if self.j + 1 == len(self.jobs):
                break
            self._next_file()
        if self.f is not None and self.i < len(self.frames):
            raise ValueError("%s: %d of its %d records were given values"
                             % (self.jobs[self.j][0], self.i, len(self.frames)))
        if self.f is not None:
            self._finish()

    def abort(self):
        """Removes the output being written, if any."""
        if self.f is not None:
            self.f.close()
            self.f = None
            os.remove(self.tmp)

    def _next_file(self):
        if self.f is not None:
            self._finish()
        if self.j + 1 == len(self.jobs):
            raise ValueError("more values than records in %s" % [s for s, _ in self.jobs])
        self.j += 1
        src, dst = self.jobs[self.j]
        self.data = _read_file(src)
        self.frames, self.i = list(record_frames(self.data, src)), 0
        self.tmp = os.path.join(os.path.dirname(dst), ".%s.partial" % os.path.basename(dst))
        self.f = open(self.tmp, "wb")

    def _finish(self):
        self.f.flush()
        os.fsync(self.f.fileno())
        self.f.close()
        self.f = None
        os.replace(self.tmp, self.jobs[self.j][1])


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
