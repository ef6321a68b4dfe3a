"""CPU checks of the knowledge-distillation shard writer: libacnn's host acnn_crc32c against the bitwise CRC of
the golden generator, the TFRecord framing against tests/golden/eval_golden.tfrecord, the Example with an
added image/logit against the protobuf runtime and parse_example, imagenet_eval.FloatFeatureWriter (record
order across files, the data CRC check, no partial output), and every refusal of
model_fns.extract_teacher_logits before any output file exists."""
import io
import os
import struct
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(ROOT, "golden", "eval_golden.tfrecord")
sys.path.insert(0, os.path.join(ROOT, "golden"))
import make_eval_preprocess_golden as mk  # noqa: E402

NUM_CLASSES, DATASET = 37, "oxford_iiit_pet"


def _crc(data, crc=0):
    from assembled_cnn_b200 import native
    return native.crc32c(data, crc)


def test_crc32c_known_answer():
    from assembled_cnn_b200.imagenet_eval import crc32c
    assert crc32c(b"123456789") == 0xE3069283
    assert crc32c(b"") == 0 and crc32c(b"", 0x1234) == 0x1234


def test_crc32c_equals_bitwise_oracle():
    """Every length 0..64 and random lengths up to 100 000, at starts 0..7 bytes past an 8-byte boundary."""
    rng = np.random.default_rng(7)
    buf = rng.integers(0, 256, 100_008, dtype=np.uint8).tobytes()
    lengths = list(range(65)) + [int(n) for n in rng.integers(65, 100_000, 12)] + [100_000]
    for n in lengths:
        for start in range(8) if n < 65 else (0, 3, 7):
            piece = memoryview(buf)[start:start + n]
            assert _crc(piece) == mk.crc32c_bitwise(bytes(piece)), (n, start)


def test_crc32c_chained():
    rng = np.random.default_rng(8)
    data = rng.integers(0, 256, 20_000, dtype=np.uint8).tobytes()
    whole = mk.crc32c_bitwise(data)
    for cuts in ([0, 20_000], [1, 5, 9, 4096, 19_999], sorted(int(c) for c in rng.integers(0, 20_000, 6))):
        c = 0
        for a, b in zip([0] + cuts, cuts + [len(data)]):
            c = _crc(memoryview(data)[a:b], c)
        assert c == whole, cuts


def test_reframing_reproduces_the_golden_shard():
    from assembled_cnn_b200.imagenet_eval import record_frames, write_record
    data = open(GOLDEN, "rb").read()
    out = io.BytesIO()
    frames = list(record_frames(data, GOLDEN))
    assert len(frames) > 1
    for _, start, length in frames:
        write_record(out, [memoryview(data)[start:start + length]])
    assert out.getvalue() == data


def _golden_examples():
    from assembled_cnn_b200.imagenet_eval import record_frames
    data = open(GOLDEN, "rb").read()
    return [data[s:s + n] for _, s, n in record_frames(data, GOLDEN)]


def test_added_logits_parse_with_protobuf_and_parse_example():
    from assembled_cnn_b200.imagenet_eval import LOGIT_KEY, add_float_feature, parse_example, write_record
    Example = mk.example_class()
    rng = np.random.default_rng(9)
    for ex in _golden_examples():
        vals = (rng.standard_normal(1001) * 5).astype(np.float32)
        vals[:4] = [0.0, -0.0, np.float32(1e-40), np.float32(-3.4e38)]     # zeros, a subnormal, a large one
        out = io.BytesIO()
        write_record(out, add_float_feature(memoryview(ex), LOGIT_KEY, vals))
        rec = out.getvalue()
        # both checksums, by the bitwise oracle
        (n,) = struct.unpack("<Q", rec[:8])
        assert rec[8:12] == struct.pack("<I", mk.masked(rec[:8]))
        new = rec[12:12 + n]
        assert len(rec) == 16 + n and rec[12 + n:] == struct.pack("<I", mk.masked(new))
        a, b = Example(), Example()
        a.ParseFromString(ex)
        b.ParseFromString(new)
        assert set(b.features.feature) == set(a.features.feature) | {"image/logit"}
        for k in a.features.feature:
            assert b.features.feature[k] == a.features.feature[k], k
        got = np.array(b.features.feature["image/logit"].float_list.value, dtype=np.float32)
        assert got.tobytes() == vals.tobytes()
        label, enc, lg = parse_example(memoryview(new), logits=True)
        assert (label, bytes(memoryview(new)[enc[0]:enc[1]])) == (
            a.features.feature["image/class/label"].int64_list.value[0],
            a.features.feature["image/encoded"].bytes_list.value[0])
        assert lg.tobytes() == vals.tobytes()
        # a second image/logit is refused
        with pytest.raises(ValueError, match="already holds image/logit"):
            add_float_feature(memoryview(new), LOGIT_KEY, vals)


# ------------------------------------------------------------------------------------------ shards
def _record(Example, rng, logits=False, label=True):
    from PIL import Image
    h, w = int(rng.integers(20, 60)), int(rng.integers(20, 60))
    buf = io.BytesIO()
    Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(buf, format="JPEG", quality=90)
    ex = Example()
    ex.features.feature["image/encoded"].bytes_list.value.append(buf.getvalue())
    if label:
        ex.features.feature["image/class/label"].int64_list.value.append(int(rng.integers(0, NUM_CLASSES)))
    if logits:
        ex.features.feature["image/logit"].float_list.value.extend([1.0] * NUM_CLASSES)
    data = ex.SerializeToString()
    head = struct.pack("<Q", len(data))
    return head + struct.pack("<I", mk.masked(head)) + data + struct.pack("<I", mk.masked(data))


def _shards(root, counts=(3, 0, 4), val=2, seed=0):
    Example = mk.example_class()
    rng = np.random.default_rng(seed)
    root.mkdir(parents=True, exist_ok=True)
    for i, n in enumerate(counts):
        (root / ("train-%05d-of-%05d" % (i, len(counts)))).write_bytes(
            b"".join(_record(Example, rng) for _ in range(n)))
    (root / "validation-00000-of-00001").write_bytes(b"".join(_record(Example, rng, label=False) for _ in range(val)))
    return root


def _jobs(src, dst):
    dst.mkdir(exist_ok=True)
    names = sorted(os.listdir(src))
    return [(str(src / n), str(dst / n)) for n in names]


def test_writer_adds_values_in_order_across_files(tmp_path):
    from assembled_cnn_b200.imagenet_eval import LOGIT_KEY, FloatFeatureWriter, read_records
    src = _shards(tmp_path / "in")
    jobs = _jobs(src, tmp_path / "out")
    total = sum(len(read_records(s, missing_label=-1)) for s, _ in jobs)
    vals = np.arange(total * NUM_CLASSES, dtype=np.float32).reshape(total, NUM_CLASSES) / 7
    w = FloatFeatureWriter(jobs, LOGIT_KEY)
    for a, b in ((0, 2), (2, 2), (2, 6), (6, total)):      # batches across file boundaries and an empty one
        w.add(vals[a:b])
    w.close()
    assert sorted(os.listdir(tmp_path / "out")) == sorted(os.listdir(src))
    row = 0
    for s, d in jobs:
        before = read_records(s, logits=True, missing_label=-1)
        after = read_records(d, logits=True, missing_label=-1)
        assert len(after) == len(before)
        for (la, _, na, lga), (lb, _, nb, lgb) in zip(before, after):
            assert (la, na, len(lga)) == (lb, nb, 0)
            assert lgb.tobytes() == vals[row].tobytes()
            row += 1
    assert row == total


def test_writer_refuses_corrupt_data_and_leaves_no_partial_file(tmp_path):
    from assembled_cnn_b200.imagenet_eval import LOGIT_KEY, FloatFeatureWriter, record_frames
    src = _shards(tmp_path / "in", counts=(3,), val=1)
    path = src / "train-00000-of-00001"
    data = bytearray(path.read_bytes())
    frames = list(record_frames(bytes(data), str(path)))
    pos, start, length = frames[1]
    data[start + length // 2] ^= 0x10                       # a flipped bit inside the second record's JPEG
    path.write_bytes(bytes(data))
    jobs = _jobs(src, tmp_path / "out")
    w = FloatFeatureWriter(jobs, LOGIT_KEY)
    with pytest.raises(ValueError, match="%s: corrupt record data at byte offset %d" % (path, pos)):
        try:
            w.add(np.zeros((3, NUM_CLASSES), np.float32))
        except ValueError:
            w.abort()
            raise
    assert os.listdir(tmp_path / "out") == []
    # too few values for the records
    w = FloatFeatureWriter(_jobs(src, tmp_path / "out2")[1:], LOGIT_KEY)
    with pytest.raises(ValueError, match="0 of its 1 records"):
        w.close()
    w.abort()
    assert os.listdir(tmp_path / "out2") == []


def _teacher(num_classes=NUM_CLASSES):
    return types.SimpleNamespace(num_classes=num_classes, use_resnet_d=False)


@pytest.mark.parametrize("case", ["empty_train_glob", "empty_val_glob", "corrupt_frame", "has_logit", "classes",
                                  "same_dir", "exists", "shard_index"])
def test_refusals_before_any_output(tmp_path, case):
    from assembled_cnn_b200.model_fns import extract_teacher_logits
    src = _shards(tmp_path / "in")
    out = tmp_path / "out"
    kw = dict(dataset_name=DATASET)
    teacher = _teacher()
    if case == "empty_train_glob":
        err, match, kw["train_regex"] = FileNotFoundError, "no file matches", "nothing-*"
    elif case == "empty_val_glob":
        err, match, kw["val_regex"] = FileNotFoundError, "no file matches", "nothing-*"
    elif case == "corrupt_frame":
        p = src / "train-00002-of-00003"
        data = bytearray(p.read_bytes())
        data[3] ^= 1                                          # the first record's length
        p.write_bytes(bytes(data))
        err, match = ValueError, "%s: corrupt record length at byte offset 0" % p
    elif case == "has_logit":
        Example = mk.example_class()
        p = src / "train-00002-of-00003"
        p.write_bytes(p.read_bytes() + _record(Example, np.random.default_rng(1), logits=True))
        err, match = ValueError, "already holds image/logit"
    elif case == "classes":
        err, match, teacher = ValueError, "the teacher has 1001 classes", _teacher(1001)
    elif case == "same_dir":
        err, match, out = ValueError, "out_dir is data_dir", tmp_path / "in" / "."
    elif case == "exists":
        out.mkdir()
        (out / "validation-00000-of-00001").write_bytes(b"")
        err, match = ValueError, "already exists"
    else:
        err, match, kw["shard_index"], kw["num_shards"] = ValueError, "shard_index 2 outside", 2, 2
    before = sorted(os.listdir(src))
    with pytest.raises(err, match=match):
        extract_teacher_logits(teacher, str(src), str(out), **kw)
    assert sorted(os.listdir(src)) == before
    left = sorted(os.listdir(out)) if out.is_dir() and case != "same_dir" else []
    assert left == (["validation-00000-of-00001"] if case == "exists" else [])


def test_default_dataset_is_imagenet(tmp_path):
    from assembled_cnn_b200.model_fns import extract_teacher_logits
    src = _shards(tmp_path / "in")
    with pytest.raises(ValueError, match="the teacher has 37 classes; imagenet has 1001"):
        extract_teacher_logits(_teacher(), str(src), str(tmp_path / "out"))
    with pytest.raises(ValueError, match="unknown dataset_name"):
        extract_teacher_logits(_teacher(), str(src), str(tmp_path / "out"), dataset_name="nope")
    assert not (tmp_path / "out").exists()
