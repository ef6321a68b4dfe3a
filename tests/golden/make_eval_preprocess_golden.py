#!/usr/bin/env python
"""Golden data of the classification evaluation's preprocessing, produced by EXECUTING the reference's own
code (by its AST) from a checkout of the original project:

    python tests/golden/make_eval_preprocess_golden.py REFERENCE_DIR
        # rewrites eval_preprocess_golden.json and eval_golden.tfrecord

It records
  * for every imagenet-family preprocessing_type and a grid of image sizes, the eval geometry the
    reference asks for: utils/data_util.py preprocess_image (the preprocessing_type dispatch) ->
    preprocessing/imagenet_preprocessing.py preprocess_image(is_training=False, crop_type 0 | 1) ->
    _aspect_preserving_resize / _smallest_size_at_least / _resize_image / central_crop /
    mean_image_subtraction, run against a stand-in `tf` that computes shapes in numpy float32 / int32 (as
    tf.float32 / tf.int32) and records the requested resize size and slice window;
  * a small TFRecord shard of tiny JPEGs (eval_golden.tfrecord): tf.train.Example messages serialised by
    the protobuf runtime from a descriptor built here (the product's parser is not involved), framed with a
    CRC-32C written here bit by bit; the JSON holds its labels and the SHA-256 of each JPEG.
tests/test_eval_preprocess_cpu.py checks the product against these files; it does not need the original
project.
"""
import ast
import hashlib
import io
import json
import os
import re
import struct
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "eval_preprocess_golden.json")
SHARD = os.path.join(HERE, "eval_golden.tfrecord")
PRE = os.path.join("preprocessing", "imagenet_preprocessing.py")
DATA = os.path.join("utils", "data_util.py")

TYPES = [("imagenet", 224), ("imagenet", 256), ("imagenet", 160), ("imagenet_224_256", 224),
         ("imagenet_224_256a", 224), ("imagenet_256", 224), ("imagenet_320", 224), ("imagenet_256a", 224),
         ("imagenet_288a", 224)]
SIZES = [(500, 375), (375, 500), (500, 333), (333, 500), (2592, 1944), (1944, 2592), (224, 224), (256, 256),
         (300, 300), (100, 100), (50, 80), (80, 50), (1, 500), (500, 1), (1, 1), (2, 3), (257, 1000)]
# smaller sides whose float32 product rounds down: 256 -> 255 and 292 -> 291
SIZES += [(s, 400) for s in (107, 109, 110, 121, 165, 145, 275, 290, 550)]
SIZES += [(400, s) for s in (107, 109, 110, 121, 165, 145, 275, 290, 550)]

# (height, width, label) of the JPEGs of the shard
SHARD_IMAGES = [(17, 23, 0), (40, 31, 999), (8, 8, 1000), (1, 5, 5), (33, 64, 123), (50, 20, 7)]


# ------------------------------------------------------------------------------ the stand-in tf
class FakeImage:
    def __init__(self, h, w, log):
        self.h, self.w, self.log = int(h), int(w), log

    def set_shape(self, shape):
        assert [self.h, self.w] == [int(shape[0]), int(shape[1])], (self.h, self.w, shape)
        self.log["set_shape"] = [int(s) for s in shape]

    def get_shape(self):
        return types.SimpleNamespace(ndims=3)

    def __sub__(self, other):
        self.log["mean"] = [float(v) for v in other]
        return self


def stub_tf(log):
    def cast(x, dt):
        return x if isinstance(x, FakeImage) else dt(x)

    def resize_images(image, size, method, align_corners):
        assert method == "BILINEAR" and align_corners is False
        log["resize"] = [int(size[0]), int(size[1])]
        return FakeImage(size[0], size[1], log)

    def slice_(image, begin, size):
        log["slice"] = [int(b) for b in begin[:2]] + [int(s) for s in size[:2]]
        return FakeImage(size[0], size[1], log)

    image = types.SimpleNamespace(
        decode_jpeg=lambda buf, channels, dct_method="": FakeImage(buf[0], buf[1], log),
        resize_images=resize_images, ResizeMethod=types.SimpleNamespace(BILINEAR="BILINEAR"))
    return types.SimpleNamespace(
        float32=np.float32, int32=np.int32, cast=cast, minimum=np.minimum, image=image, slice=slice_,
        shape=lambda img: [np.int32(img.h), np.int32(img.w), np.int32(3)],
        broadcast_to=lambda means, shape: means, zeros=lambda shape, dtype=None: None,
        logging=types.SimpleNamespace(info=lambda *a, **k: None))


def module_nodes(path, names):
    tree = ast.parse(open(path).read())
    keep = []
    for n in tree.body:
        if isinstance(n, ast.FunctionDef) and n.name in names:
            keep.append(n)
        elif isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id in names for t in n.targets):
            keep.append(n)
    return ast.Module(body=keep, type_ignores=[])


def reference_geometry(ref_root, h, w, preprocessing_type, image_size):
    log = {}
    tf = stub_tf(log)
    pre = {"tf": tf}
    exec(compile(module_nodes(os.path.join(ref_root, PRE),
                              {"_R_MEAN", "_G_MEAN", "_B_MEAN", "CHANNEL_MEANS", "central_crop",
                               "mean_image_subtraction", "_smallest_size_at_least", "_aspect_preserving_resize",
                               "_resize_image", "preprocess_image"}), PRE, "exec"), pre)
    data = {"tf": tf, "re": re, "imagenet_preprocessing": types.SimpleNamespace(**pre)}
    exec(compile(module_nodes(os.path.join(ref_root, DATA), {"preprocess_image"}), DATA, "exec"), data)
    out = data["preprocess_image"](image_buffer=(h, w), is_training=False, num_channels=3, dtype=np.float32,
                                   image_size=image_size, preprocessing_type=preprocessing_type)
    s = log["set_shape"][0]
    assert log["slice"][2:] == [s, s] and isinstance(out, FakeImage)
    return {"type": preprocessing_type, "image_size": image_size, "h": h, "w": w, "S": s, "rsz": log["resize"],
            "crop": log["slice"][:2], "mean": log["mean"]}


# ------------------------------------------------------------------------------ the TFRecord shard
def crc32c_bitwise(data):
    c = 0xFFFFFFFF
    for b in data:
        c ^= b
        for _ in range(8):
            c = (c >> 1) ^ (0x82F63B78 * (c & 1))
    return c ^ 0xFFFFFFFF


def masked(data):
    c = crc32c_bitwise(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def example_class():
    """tf.train.Example (tensorflow/core/example/{example,feature}.proto) built as a runtime descriptor."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="golden_example.proto", package="golden", syntax="proto3")

    def msg(name, fields, nested=()):
        m = fd.message_type.add(name=name)
        for fname, num, ftype, label, tname in fields:
            f = m.field.add(name=fname, number=num, type=ftype, label=label)
            if tname:
                f.type_name = tname
        for n in nested:
            m.nested_type.add().CopyFrom(n)
        return m

    rep, opt = F.LABEL_REPEATED, F.LABEL_OPTIONAL
    msg("BytesList", [("value", 1, F.TYPE_BYTES, rep, None)])
    msg("FloatList", [("value", 1, F.TYPE_FLOAT, rep, None)])
    msg("Int64List", [("value", 1, F.TYPE_INT64, rep, None)])
    feat = msg("Feature", [("bytes_list", 1, F.TYPE_MESSAGE, opt, ".golden.BytesList"),
                           ("float_list", 2, F.TYPE_MESSAGE, opt, ".golden.FloatList"),
                           ("int64_list", 3, F.TYPE_MESSAGE, opt, ".golden.Int64List")])
    feat.oneof_decl.add(name="kind")
    for f in feat.field:
        f.oneof_index = 0
    entry = descriptor_pb2.DescriptorProto(name="FeatureEntry")
    entry.field.add(name="key", number=1, type=F.TYPE_STRING, label=opt)
    entry.field.add(name="value", number=2, type=F.TYPE_MESSAGE, label=opt, type_name=".golden.Feature")
    entry.options.map_entry = True
    msg("Features", [("feature", 1, F.TYPE_MESSAGE, rep, ".golden.Features.FeatureEntry")], nested=[entry])
    msg("Example", [("features", 1, F.TYPE_MESSAGE, opt, ".golden.Features")])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("golden.Example"))


def write_shard():
    from PIL import Image
    Example = example_class()
    rng = np.random.default_rng(2024)
    records, meta = [], []
    for i, (h, w, label) in enumerate(SHARD_IMAGES):
        buf = io.BytesIO()
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(buf, format="JPEG", quality=90)
        jpeg = buf.getvalue()
        ex = Example()
        f = ex.features.feature
        f["image/format"].bytes_list.value.append(b"JPEG")
        f["image/encoded"].bytes_list.value.append(jpeg)
        f["image/height"].int64_list.value.append(h)
        f["image/class/label"].int64_list.value.append(label)
        f["image/object/bbox/xmin"].float_list.value.extend([0.25, 0.5])
        f["image/filename"].bytes_list.value.append(b"ILSVRC2012_val_%08d.JPEG" % (i + 1))
        data = ex.SerializeToString()
        head = struct.pack("<Q", len(data))
        records.append(head + struct.pack("<I", masked(head)) + data + struct.pack("<I", masked(data)))
        meta.append({"label": label, "h": h, "w": w, "sha256": hashlib.sha256(jpeg).hexdigest()})
    with open(SHARD, "wb") as fh:
        fh.write(b"".join(records))
    return meta


def main(ref_root):
    cases = [reference_geometry(ref_root, h, w, t, s) for t, s in TYPES for h, w in SIZES]
    gold = {"cases": cases, "shard": write_shard()}
    json.dump(gold, open(OUT, "w"), sort_keys=True, indent=0)
    print("wrote", OUT, "and", SHARD)


if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isfile(os.path.join(sys.argv[1], PRE)):
        sys.exit("usage: python tests/golden/make_eval_preprocess_golden.py REFERENCE_DIR\n"
                 "  REFERENCE_DIR: a checkout of clovaai/assembled-cnn (the directory holding preprocessing/)")
    main(os.path.abspath(sys.argv[1]))
