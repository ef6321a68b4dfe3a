"""The dataset builders (assembled_cnn_b200.build_data) against the records of the reference's own builder code
(tests/golden/build_data_golden.json, generator tests/golden/make_build_data_golden.py): shard names, per-shard
record order and feature maps for every builder at num_threads 1, 2 and 8, checked here with the PIL check
(check='pil'; the device check is compared with it in test_build_data_gpu.py).  Every record is read back
through a protobuf schema built from example.proto's field numbers and through the project's own reader.
Re-encoded images (the ImageNet PNG / CMYK files, the CUB / Cars crops) must be build_data.encode_jpeg of
PIL's decode of the source (cropped to the golden window)."""
import hashlib
import importlib.util
import io
import json
import os
import shutil
import struct

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("make_build_data_golden",
                                              os.path.join(HERE, "golden", "make_build_data_golden.py"))
mg = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mg)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "build_data_golden.json")))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("raw"))
    mg.make_tree(root, GOLDEN["seed"])
    return root


def imagenet_flags(tree, t, logits=True):
    im = os.path.join(tree, "imagenet")
    return dict(train_shards=mg.SHARDS, validation_shards=mg.SHARDS, num_threads=t,
                labels_file=im + "/synsets.txt", imagenet_metadata_file=im + "/metadata.txt",
                bounding_box_file=im + "/bboxes.csv", logits_file_path=im + "/logits" if logits else None)


def build_args(name, tree, t):
    """(dataset, positional args, flags) of a golden configuration at num_threads t."""
    im = os.path.join(tree, "imagenet")
    if name.startswith("imagenet"):
        return "imagenet", (im + "/train", im + "/validation"), imagenet_flags(tree, t, name == "imagenet")
    if name == "food101":
        return name, (os.path.join(tree, "food101"),), dict(train_shards=mg.SHARDS, validation_shards=mg.SHARDS,
                                                            num_threads=t)
    if name.startswith("cub_200_2011"):
        return "cub_200_2011", (os.path.join(tree, "cub"),), dict(num_threads=t, use_bbox=name == "cub_200_2011")
    if name == "cars196_zeroshot":
        return name, (os.path.join(tree, "cars196"),), dict(num_threads=t, use_bbox=True)
    return "SOP", (os.path.join(tree, "sop"),), dict(train_shards=mg.SHARDS, validation_shards=mg.SHARDS,
                                                     num_threads=t)


def example_class():
    """tf.train.Example from example.proto / feature.proto's field numbers."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="test_example.proto", package="tfex", syntax="proto3")
    opt, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED
    for name, typ in (("BytesList", F.TYPE_BYTES), ("FloatList", F.TYPE_FLOAT), ("Int64List", F.TYPE_INT64)):
        fd.message_type.add(name=name).field.add(name="value", number=1, type=typ, label=rep)
    f = fd.message_type.add(name="Feature")
    f.oneof_decl.add(name="kind")
    for name, num, typ in (("bytes_list", 1, "BytesList"), ("float_list", 2, "FloatList"),
                           ("int64_list", 3, "Int64List")):
        f.field.add(name=name, number=num, type=F.TYPE_MESSAGE, label=opt, type_name=".tfex." + typ, oneof_index=0)
    fs = fd.message_type.add(name="Features")
    entry = fs.nested_type.add(name="FeatureEntry")
    entry.options.map_entry = True
    entry.field.add(name="key", number=1, type=F.TYPE_STRING, label=opt)
    entry.field.add(name="value", number=2, type=F.TYPE_MESSAGE, label=opt, type_name=".tfex.Feature")
    fs.field.add(name="feature", number=1, type=F.TYPE_MESSAGE, label=rep, type_name=".tfex.Features.FeatureEntry")
    e = fd.message_type.add(name="Example")
    e.field.add(name="features", number=1, type=F.TYPE_MESSAGE, label=opt, type_name=".tfex.Features")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("tfex.Example"))


def read_shards(out_dir):
    """{shard file name: [{key: (kind, values)}]} of every shard in out_dir, each record's data CRC checked and
    its Example parsed by protobuf and, for the label and the image, by imagenet_eval.read_records."""
    from assembled_cnn_b200.imagenet_eval import masked_crc32c, read_records, record_frames
    Example = example_class()
    out = {}
    for name in sorted(os.listdir(out_dir)):
        path = os.path.join(out_dir, name)
        data = open(path, "rb").read()
        recs = []
        for _, start, length in record_frames(data, path):
            body = data[start:start + length]
            assert struct.unpack("<I", data[start + length:start + length + 4])[0] == masked_crc32c(body)
            ex = Example()
            ex.ParseFromString(body)
            feats = {}
            for key, f in ex.features.feature.items():
                kind = f.WhichOneof("kind")
                feats[key] = (kind.split("_")[0], list(getattr(f, kind).value))
            recs.append(feats)
        ours = read_records(path)
        assert [(r["image/class/label"][1][0], r["image/encoded"][1][0]) for r in recs] == \
               [(lab, data[o:o + n]) for lab, o, n in ours]
        out[name] = recs
    return out


def expected_image(tree, desc):
    """The bytes a golden image/encoded descriptor stands for."""
    from assembled_cnn_b200.build_data import encode_jpeg
    from assembled_cnn_b200.imagenet_c import decode_rgb
    if "crop" in desc:
        y, x, h, w = desc["crop"]
        return encode_jpeg(decode_rgb(os.path.join(tree, desc["file"]))[y:y + h, x:x + w])
    if "file" in desc:
        return open(os.path.join(tree, desc["file"]), "rb").read()
    (src,) = desc.values()
    return encode_jpeg(decode_rgb(os.path.join(tree, src)))


def golden_form(tree, feats, golden_records):
    """(record id, the record in the golden JSON form) of a product record; its image bytes are checked
    against the golden descriptor of the record with the same file name and class, found by content."""
    out = {}
    for key, (kind, values) in feats.items():
        if kind == "bytes":
            values = [v if key == "image/encoded" else v.decode() for v in values]
        elif kind == "float":
            values = mg._value("float", values)
        out[key] = [kind, values]
    data = out["image/encoded"][1][0]
    for rid, rec in golden_records.items():
        desc = rec["image/encoded"][1]
        if (desc.get("file") and "crop" not in desc and open(os.path.join(tree, desc["file"]), "rb").read() == data) \
                or (("crop" in desc or "file" not in desc) and expected_image(tree, desc) == data
                    and rec["image/height"] == out["image/height"]):
            out["image/encoded"] = ["image", desc]
            return rid, out
    raise AssertionError("a record's image matches no golden record (%d bytes, sha256 %s)"
                         % (len(data), hashlib.sha256(data).hexdigest()))


def check_against_golden(tree, name, t, out_dir):
    g = GOLDEN["datasets"][name]
    shards = read_shards(out_dir)
    layout = g["layouts"][str(t)]
    assert list(shards) == [s for s, _ in layout]
    for (shard, ids) in layout:
        got = [golden_form(tree, f, g["records"]) for f in shards[shard]]
        assert [rid for rid, _ in got] == ids, shard
        for rid, rec in got:
            assert rec == g["records"][rid], (shard, rid)


CONFIGS = [(name, int(t)) for name, g in GOLDEN["datasets"].items() for t in g["layouts"]]


@pytest.mark.parametrize("name,t", CONFIGS, ids=["%s-threads%d" % c for c in CONFIGS])
def test_shards_equal_reference_records(tree, tmp_path, name, t):
    from assembled_cnn_b200 import build_data
    dataset, args, flags = build_args(name, tree, t)
    out = str(tmp_path / "out")
    build_data.build(dataset, out, *args, check="pil", num_workers=3, **flags)
    assert not [f for f in os.listdir(out) if f.startswith(".")]
    check_against_golden(tree, name, t, out)


def test_worker_count_does_not_change_bytes(tree, tmp_path):
    from assembled_cnn_b200 import build_data
    dataset, args, flags = build_args("imagenet", tree, 2)
    outs = []
    for w in (1, 7):
        out = str(tmp_path / ("w%d" % w))
        build_data.build(dataset, out, *args, check="pil", num_workers=w, **flags)
        outs.append({f: open(os.path.join(out, f), "rb").read() for f in sorted(os.listdir(out))})
    assert outs[0] == outs[1]


def test_flat_validation_directory(tree, tmp_path):
    """The flat validation directory + imagenet_2012_validation_synset_labels.txt gives the shards of the
    per-synset directories (what preprocess_imagenet_validation_data.py would make), moving no file."""
    from assembled_cnn_b200 import build_data
    im = os.path.join(tree, "imagenet")
    flat = tmp_path / "flat"
    flat.mkdir()
    for s in os.listdir(im + "/validation"):
        for f in os.listdir(os.path.join(im, "validation", s)):
            shutil.copy(os.path.join(im, "validation", s, f), flat / f)
    before = sorted(os.listdir(flat))
    flags = imagenet_flags(tree, 2)
    outs = []
    for vdir, vlabels in ((im + "/validation", None), (str(flat), im + "/val_labels.txt")):
        out = str(tmp_path / ("out%d" % len(outs)))
        build_data.build("imagenet", out, im + "/train", vdir, check="pil", make_train=False,
                         validation_labels_file=vlabels, **flags)
        outs.append({f: open(os.path.join(out, f), "rb").read() for f in sorted(os.listdir(out))})
    assert outs[0] == outs[1] and len(outs[0]) == mg.SHARDS
    assert sorted(os.listdir(flat)) == before


def test_command_line(tree, tmp_path):
    from assembled_cnn_b200 import build_data
    out = str(tmp_path / "out")
    build_data.main(["SOP", "-i", os.path.join(tree, "sop"), "-o", out, "--train_shards", "8",
                     "--validation_shards", "8", "--num_threads", "2", "--check", "pil", "--num_workers", "2"])
    check_against_golden(tree, "SOP", 2, out)
    a = build_data._parser().parse_args(["imagenet"])
    assert (a.train_shards, a.validation_shards, a.num_threads, a.make_val, a.make_train, a.labels_file,
            a.imagenet_metadata_file) == (1024, 128, 8, True, True, "imagenet_lsvrc_2015_synsets.txt",
                                          "imagenet_metadata.txt")
    # not given: the reference's default paths are used where they exist (test_cli_default_paths)
    assert (a.bounding_box_file, a.logits_file_path) == (None, None)
    assert (build_data.IMAGENET_BBOX_DEFAULT, build_data.IMAGENET_LOGITS_DEFAULT) == \
        ("./imagenet_2012_bounding_boxes.csv", "amoebanet_logits")
    assert build_data._parser().parse_args(["imagenet", "--make_train=False"]).make_train is False
    for arg, want in (("--nomake_train", (True, False)), ("--nomake_val", (False, True)),
                      ("--make_val", (True, True))):
        a = build_data._parser().parse_args(["imagenet", arg])
        assert (a.make_val, a.make_train) == want
    for ds, threads in (("food101", 8), ("SOP", 8), ("cub_200_2011", 16), ("cars196_zeroshot", 16)):
        assert build_data._parser().parse_args([ds]).num_threads == threads
    assert build_data._parser().parse_args(["cub_200_2011", "--use_bbox"]).use_bbox is True


def test_layout_rules():
    from assembled_cnn_b200.build_data import shard_layout, shuffled
    import random
    lay = shard_layout("train", 10, 2, 4)
    assert lay == [("train-00000-of-00004", 0, 2), ("train-00001-of-00004", 2, 5),
                   ("train-00002-of-00004", 5, 7), ("train-00003-of-00004", 7, 10)]
    idx = list(range(50))
    random.seed(12345)
    random.shuffle(idx)
    assert shuffled(list(range(50)))[0] == idx


def test_example_serialisation_round_trip():
    from assembled_cnn_b200.imagenet_eval import serialize_example
    Example = example_class()
    feats = {"a": ("bytes", [b"xy", b""]), "b": ("float", []), "c": ("int64", [0, -3, 1 << 40]),
             "d": ("float", [1.5, -2.25])}
    ex = Example()
    ex.ParseFromString(serialize_example(feats))
    assert ex.SerializeToString(deterministic=True) == serialize_example(feats)
    assert ex.features.feature["b"].WhichOneof("kind") == "float_list"
    assert list(ex.features.feature["c"].int64_list.value) == [0, -3, 1 << 40]


# --------------------------------------------------------------------------------- errors, before writing
def _copy(tree, tmp_path, sub):
    dst = tmp_path / sub
    shutil.copytree(os.path.join(tree, sub), dst)
    return str(dst)


def _edit(path, fn):
    with open(path) as f:
        text = f.read()
    with open(path, "w") as f:
        f.write(fn(text))


def _imagenet_case(case):
    def run(tree, tmp_path):
        im = _copy(tree, tmp_path, "imagenet")
        flags = imagenet_flags(tree, 2)
        flags.update(labels_file=im + "/synsets.txt", imagenet_metadata_file=im + "/metadata.txt",
                     bounding_box_file=im + "/bboxes.csv", logits_file_path=im + "/logits")
        if case == "unknown_dir":
            os.makedirs(im + "/train/n09999999")
        elif case == "missing_dir":
            shutil.rmtree(im + "/validation/n03000001")
        elif case == "label_file":
            _edit(im + "/synsets.txt", lambda t: t + "n03000001\n")
        elif case == "metadata":
            _edit(im + "/metadata.txt", lambda t: t.replace("n03000001\tthing\n", ""))
        elif case == "bbox":
            _edit(im + "/bboxes.csv", lambda t: t + "x.JPEG,0.1,0.2,0.3\n")
        elif case == "bbox_value":
            _edit(im + "/bboxes.csv", lambda t: t + "x.JPEG,0.1,0.2,0.3,zero\n")
        elif case == "logit_columns":
            _edit(im + "/logits/train_1.csv", lambda t: t + "x.JPEG,1.0\n")
        elif case == "logit_duplicate":
            _edit(im + "/logits/train_1.csv", lambda t: t + open(im + "/logits/train_0.csv").readline())
        elif case == "logit_missing":
            _edit(im + "/logits/validation_1.csv", lambda t: "".join(t.splitlines(True)[1:]))
        elif case == "shards":
            flags.update(train_shards=6, num_threads=4)
        return "imagenet", (im + "/train", im + "/validation"), flags
    return run


def _other_case(case):
    def run(tree, tmp_path):
        if case == "food_label":
            d = _copy(tree, tmp_path, "food101")
            _edit(d + "/meta/train.txt", lambda t: t + "pizza/1\n")
            return "food101", (d,), dict(train_shards=8, validation_shards=8)
        if case == "food_missing_file":
            d = _copy(tree, tmp_path, "food101")
            _edit(d + "/meta/test.txt", lambda t: t + "apple_pie/424242\n")
            return "food101", (d,), dict(train_shards=8, validation_shards=8)
        if case == "sop_line":
            d = _copy(tree, tmp_path, "sop")
            _edit(d + "/Ebay_test.txt", lambda t: t + "99 x\n")
            return "SOP", (d,), dict(train_shards=8, validation_shards=8)
        if case == "sop_shards":
            return "SOP", (os.path.join(tree, "sop"),), dict(train_shards=8, validation_shards=12, num_threads=8)
        if case == "cub_bbox":
            d = _copy(tree, tmp_path, "cub")
            _edit(d + "/bounding_boxes.txt", lambda t: "".join(t.splitlines(True)[:-1]))
            return "cub_200_2011", (d,), dict(use_bbox=True)
        if case == "cub_bbox_line":
            d = _copy(tree, tmp_path, "cub")
            _edit(d + "/bounding_boxes.txt", lambda t: t + "1 2 3\n")
            return "cub_200_2011", (d,), dict(use_bbox=True)
        if case == "cars_count":
            d = _copy(tree, tmp_path, "cars196")
            import tarfile
            with tarfile.open(d + "/car_ims.tgz", "w:gz") as t:
                t.add(d + "/car_ims/000001.jpg", arcname="car_ims/000001.jpg")
            return "cars196_zeroshot", (d,), dict(use_bbox=True)
    return run


ERRORS = {**{"imagenet_" + c: _imagenet_case(c) for c in
             ("unknown_dir", "missing_dir", "label_file", "metadata", "bbox", "bbox_value", "logit_columns",
              "logit_duplicate", "logit_missing", "shards")},
          **{c: _other_case(c) for c in ("food_label", "food_missing_file", "sop_line", "sop_shards", "cub_bbox",
                                         "cub_bbox_line", "cars_count")}}


@pytest.mark.parametrize("case", sorted(ERRORS))
def test_errors_before_any_file(tree, tmp_path, case):
    from assembled_cnn_b200 import build_data
    dataset, args, flags = ERRORS[case](tree, tmp_path)
    out = tmp_path / "out"
    with pytest.raises(ValueError):
        build_data.build(dataset, str(out), *args, check="pil", **flags)
    assert not out.exists()


def test_existing_output_refused(tree, tmp_path):
    from assembled_cnn_b200 import build_data
    dataset, args, flags = build_args("SOP", tree, 2)
    out = tmp_path / "out"
    out.mkdir()
    (out / "validation-00007-of-00008").write_bytes(b"keep")
    with pytest.raises(ValueError, match="already exists"):
        build_data.build(dataset, str(out), *args, check="pil", **flags)
    assert os.listdir(out) == ["validation-00007-of-00008"]
    assert (out / "validation-00007-of-00008").read_bytes() == b"keep"


def test_undecodable_image_raises_with_its_path(tree, tmp_path):
    """ImageNet, CUB and Cars raise on an image PIL cannot decode (food101 and SOP skip it: golden above);
    the shard being written is removed."""
    from assembled_cnn_b200 import build_data
    im = _copy(tree, tmp_path, "imagenet")
    bad = os.path.join(im, "train", "n03000001", "n03000001_100.JPEG")
    data = open(bad, "rb").read()
    open(bad, "wb").write(data[:len(data) // 2])
    out = tmp_path / "out"
    flags = imagenet_flags(tree, 2)
    with pytest.raises(ValueError, match=bad):
        build_data.build("imagenet", str(out), im + "/train", im + "/validation", check="pil", make_val=False,
                         **flags)
    assert not [f for f in os.listdir(out) if f.startswith(".")]


def test_device_check_needs_a_device(tree, tmp_path, monkeypatch):
    import torch
    from assembled_cnn_b200 import build_data
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    dataset, args, flags = build_args("SOP", tree, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        build_data.build(dataset, str(tmp_path / "out"), *args, check="device", **flags)


def test_encode_jpeg_settings():
    from PIL import Image
    from assembled_cnn_b200.build_data import encode_jpeg
    a = (np.arange(24 * 40 * 3) % 251).astype(np.uint8).reshape(24, 40, 3)
    with Image.open(io.BytesIO(encode_jpeg(a))) as im:
        assert im.format == "JPEG" and im.mode == "RGB" and im.size == (40, 24)
        assert im.info.get("dpi") == (300, 300) and not im.info.get("progressive")
        assert [c[1:3] for c in im.layer] == [(2, 2), (1, 1), (1, 1)]          # 4:2:0
        assert im.quantization[0] == [1] * 64                                 # quality 100


def _imagenet_argv(tree, out, *extra):
    im = os.path.join(tree, "imagenet")
    return ["imagenet", "--train_directory", im + "/train", "--validation_directory", im + "/validation",
            "--output_directory", out, "--labels_file", im + "/synsets.txt", "--imagenet_metadata_file",
            im + "/metadata.txt", "--train_shards", "8", "--validation_shards", "8", "--num_threads", "2",
            "--check", "pil"] + list(extra)


@pytest.mark.parametrize("flag", ["--bounding_box_file", "--logits_file_path"])
def test_cli_given_paths_must_exist(tree, tmp_path, monkeypatch, flag):
    """A bbox file or logits path given on the command line that does not exist raises before any shard, even
    where the reference's default exists."""
    from assembled_cnn_b200 import build_data
    monkeypatch.chdir(tmp_path)
    shutil.copy(os.path.join(tree, "imagenet", "bboxes.csv"), build_data.IMAGENET_BBOX_DEFAULT)
    shutil.copytree(os.path.join(tree, "imagenet", "logits"), build_data.IMAGENET_LOGITS_DEFAULT)
    out = tmp_path / "out"
    with pytest.raises(ValueError, match="typo"):
        build_data.main(_imagenet_argv(tree, str(out), flag, str(tmp_path / "typo")))
    assert not out.exists()


def test_cli_default_paths(tree, tmp_path, monkeypatch):
    """Without the flags: no boxes and no image/logit where the reference's default paths do not exist, the
    default files where they do."""
    from assembled_cnn_b200 import build_data
    monkeypatch.chdir(tmp_path)
    im = os.path.join(tree, "imagenet")
    out = str(tmp_path / "no_logits")
    build_data.main(_imagenet_argv(tree, out, "--bounding_box_file", im + "/bboxes.csv"))
    check_against_golden(tree, "imagenet_no_logits", 2, out)
    out = str(tmp_path / "no_boxes")
    build_data.main(_imagenet_argv(tree, out, "--nomake_train"))
    recs = [r for f in read_shards(out).values() for r in f]
    assert recs and all("image/logit" not in r and r["image/object/bbox/xmin"] == ("float", []) for r in recs)
    shutil.copy(im + "/bboxes.csv", build_data.IMAGENET_BBOX_DEFAULT)
    shutil.copytree(im + "/logits", build_data.IMAGENET_LOGITS_DEFAULT)
    out = str(tmp_path / "defaults")
    build_data.main(_imagenet_argv(tree, out))
    check_against_golden(tree, "imagenet", 2, out)


def _image_bytes(fmt, frames=1):
    from PIL import Image
    ims = [Image.fromarray(np.full((9, 11, 3), 40 * k, dtype=np.uint8)) for k in range(frames)]
    b = io.BytesIO()
    ims[0].save(b, fmt, **({"save_all": True, "append_images": ims[1:]} if frames > 1 else {}))
    return b.getvalue()


def test_pil_check_takes_what_decode_jpeg_takes():
    """JPEG, PNG and one-frame GIF decode; BMP, TIFF, WebP and an animated GIF are refused as
    tf.image.decode_jpeg refuses them."""
    from assembled_cnn_b200.build_data import _pil
    for fmt in ("JPEG", "PNG", "GIF"):
        a, err = _pil(_image_bytes(fmt))
        assert err is None and a.shape == (9, 11, 3), fmt
    for fmt in ("BMP", "TIFF", "WEBP"):
        a, err = _pil(_image_bytes(fmt))
        assert a is None and "not a JPEG, PNG or GIF" in err, fmt
    a, err = _pil(_image_bytes("GIF", frames=2))
    assert a is None and "animated" in err


def test_other_formats_skipped_or_raised(tree, tmp_path):
    """A BMP under a listed name is skipped by SOP (the reference logs and skips what decode_jpeg refuses)
    and raises with its path in CUB."""
    from assembled_cnn_b200 import build_data
    sop = _copy(tree, tmp_path, "sop")
    bmp = os.path.join(sop, "bicycle_final", "112_0.JPG")
    open(bmp, "wb").write(_image_bytes("BMP"))
    n = build_data.build("SOP", str(tmp_path / "sop_out"), sop, train_shards=8, validation_shards=8, check="pil")
    assert n == {"train": 8, "validation": 6}                      # the truncated one and the BMP skipped
    cub = _copy(tree, tmp_path, "cub")
    d = os.path.join(cub, "images", "001.Bird_0")
    bmp = os.path.join(d, sorted(os.listdir(d))[0])
    open(bmp, "wb").write(_image_bytes("BMP"))
    with pytest.raises(ValueError, match=bmp):
        build_data.build("cub_200_2011", str(tmp_path / "cub_out"), cub, check="pil")


def test_pil_check_keeps_no_full_image(tree):
    """What the pool hands back holds the height and width, and pixels only for a bbox crop."""
    from assembled_cnn_b200 import build_data
    sop = build_data.sop_splits(os.path.join(tree, "sop"), train_shards=8, validation_shards=8)
    c = build_data._load(sop[1].items[0], True)
    assert c.error is None and c.crop is None and len(c.shape) == 2
    cub = build_data.cub_splits(os.path.join(tree, "cub"), use_bbox=True)
    it = cub[0].items[0]
    c = build_data._load(it, True)
    y, x, h, w = build_data.crop_window(it.bbox, c.shape[0], c.shape[1], it.path)
    assert c.crop.shape == (h, w, 3)


def test_failed_build_keeps_completed_shards_and_says_so(tree, tmp_path, caplog):
    from assembled_cnn_b200 import build_data
    cub = _copy(tree, tmp_path, "cub")
    d = os.path.join(cub, "images", "102.Bird_101")                 # validation, written after train
    bad = os.path.join(d, sorted(os.listdir(d))[0])
    open(bad, "wb").write(b"junk")
    out = tmp_path / "out"
    with pytest.raises(ValueError, match=bad):
        build_data.build("cub_200_2011", str(out), cub, check="pil")
    assert len([f for f in os.listdir(out) if f.startswith("train-")]) == 128
    assert not [f for f in os.listdir(out) if f.startswith(".")]
    done = len([f for f in os.listdir(out) if not f.startswith(".")])
    assert done >= 128 and "%d shard(s) of this build were completed" % done in caplog.text
    with pytest.raises(ValueError, match="already exists"):
        build_data.build("cub_200_2011", str(out), _copy(tree, tmp_path / "again", "cub"), check="pil")
