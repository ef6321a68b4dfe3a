"""GPU checks of model_fns.extract_teacher_logits on synthetic shards (three train shards and one validation
shard of mixed image sizes; batches of 16 over 40 records, so the short last batch spans two shards): every
written image/logit equals teacher(x, False) on the PIL-decoded, float32-restated eval batches bit for bit
(bf16 / fp32 teachers, two preprocessing types), every other feature and both checksums of every record,
eager launches and a two-process split give the same files, and the output trains a student with
kd_temp > 0 (read_train_records returns the teacher's logits; one train_and_evaluate cycle)."""
import io
import os
import struct
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "golden"))
import make_eval_preprocess_golden as mk  # noqa: E402

NUM_CLASSES, DATASET, BATCH = 37, "oxford_iiit_pet", 16
COUNTS = {"train-00000-of-00003": 13, "train-00001-of-00003": 11, "train-00002-of-00003": 9,
          "validation-00000-of-00001": 7}


def _write_shard(path, Example, rng, n):
    from PIL import Image
    recs = []
    for _ in range(n):
        h, w = int(rng.integers(20, 150)), int(rng.integers(20, 150))
        base = rng.integers(0, 256, 3)
        img = np.clip(base + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        ex = Example()
        ex.features.feature["image/encoded"].bytes_list.value.append(buf.getvalue())
        ex.features.feature["image/class/label"].int64_list.value.append(int(rng.integers(0, NUM_CLASSES)))
        ex.features.feature["image/height"].int64_list.value.append(h)
        ex.features.feature["image/filename"].bytes_list.value.append(b"img_%d_%d.jpg" % (h, w))
        data = ex.SerializeToString()
        head = len(data).to_bytes(8, "little")
        recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
    path.write_bytes(b"".join(recs))


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    Example = mk.example_class()
    root = tmp_path_factory.mktemp("data")
    rng = np.random.default_rng(0)
    for name, n in COUNTS.items():
        _write_shard(root / name, Example, rng, n)
    return root


def _frames(path):
    """The data of every record of `path`, each record's two checksums verified with the bitwise oracle."""
    data = open(path, "rb").read()
    out, pos = [], 0
    while pos < len(data):
        (n,) = struct.unpack("<Q", data[pos:pos + 8])
        assert data[pos + 8:pos + 12] == struct.pack("<I", mk.masked(data[pos:pos + 8]))
        rec = data[pos + 12:pos + 12 + n]
        assert data[pos + 12 + n:pos + 16 + n] == struct.pack("<I", mk.masked(rec))
        out.append(rec)
        pos += 16 + n
    return out


def _oracle_logits(teacher, root, ptype, image_size):
    """teacher(x, False) on the extraction's batches, x through the host path: PIL decode, the float32
    restatement of the eval preprocessing."""
    from assembled_cnn_b200 import imagenet_eval as ie
    from oracle import eval_preprocess as O
    recs = [(str(root / f), off, n) for f in sorted(COUNTS) for _, off, n in ie.read_records(str(root / f))]
    out = []
    for a in range(0, len(recs), BATCH):
        x = np.stack([O.preprocess(ie.decode_record(f, off, n, ptype, image_size)[0], ptype, image_size)
                      for f, off, n in recs[a:a + BATCH]])
        out.append(teacher(torch.from_numpy(x), False).float().cpu().clone())
    return torch.cat(out).numpy()


CASES = [("bf16", "imagenet", 64), ("fp32", "imagenet", 64), ("bf16", "imagenet_128a", 224),
         ("fp32", "imagenet_128a", 224)]


@pytest.mark.parametrize("dtype,ptype,image_size", CASES)
def test_logits_equal_teacher_on_pil_batches(shards, tmp_path, dtype, ptype, image_size):
    from assembled_cnn_b200.model_fns import build_model, extract_teacher_logits
    teacher = build_model(resnet_size=50, num_classes=NUM_CLASSES, dtype=dtype, seed=5)
    kw = dict(preprocessing_type=ptype, image_size=image_size, batch_size=BATCH, dataset_name=DATASET,
              num_workers=4)
    out = tmp_path / "kd"
    written = extract_teacher_logits(teacher, str(shards), str(out), **kw)
    assert written == [str(out / f) for f in sorted(COUNTS)] and sorted(os.listdir(out)) == sorted(COUNTS)
    want = _oracle_logits(teacher, shards, ptype, image_size)
    assert want.shape == (sum(COUNTS.values()), NUM_CLASSES) and np.isfinite(want).all()
    Example = mk.example_class()
    row = 0
    for f in sorted(COUNTS):
        before, after = _frames(shards / f), _frames(out / f)
        assert len(before) == len(after) == COUNTS[f]
        for a_bytes, b_bytes in zip(before, after):
            a, b = Example(), Example()
            a.ParseFromString(a_bytes)
            b.ParseFromString(b_bytes)
            assert set(b.features.feature) == set(a.features.feature) | {"image/logit"}
            assert all(b.features.feature[k] == a.features.feature[k] for k in a.features.feature)
            got = np.array(b.features.feature["image/logit"].float_list.value, dtype=np.float32)
            assert got.tobytes() == want[row].tobytes(), (f, row)
            row += 1
    # eager launches write the same bytes
    eager = tmp_path / "eager"
    extract_teacher_logits(teacher, str(shards), str(eager), use_cuda_graph=False, **kw)
    assert all((eager / f).read_bytes() == (out / f).read_bytes() for f in COUNTS)
    # two processes' worth of calls write the same files between them, each file once
    split = tmp_path / "split"
    parts = [extract_teacher_logits(teacher, str(shards), str(split), shard_index=i, num_shards=2, **kw)
             for i in range(2)]
    names = [[os.path.basename(d) for d in part] for part in parts]
    assert names == [sorted(COUNTS)[0::2], sorted(COUNTS)[1::2]]
    assert all((split / f).read_bytes() == (out / f).read_bytes() for f in COUNTS)
    assert sorted(os.listdir(split)) == sorted(COUNTS)          # no temporary file left


def test_student_trains_on_the_output(shards, tmp_path):
    from assembled_cnn_b200 import imagenet_train as it
    from assembled_cnn_b200.model_fns import build_model, extract_teacher_logits, train_and_evaluate
    teacher = build_model(resnet_size=50, num_classes=NUM_CLASSES, dtype="bf16", seed=6)
    out = tmp_path / "kd"
    extract_teacher_logits(teacher, str(shards), str(out), image_size=64, batch_size=BATCH, dataset_name=DATASET)
    want = _oracle_logits(teacher, shards, "imagenet", 64)
    records, counts = it.read_train_records(it.train_files(str(out)), NUM_CLASSES, kd=True)
    assert counts == [COUNTS[f] for f in sorted(COUNTS) if f.startswith("train")]
    assert np.array_equal(np.stack([r[4] for r in records]), want[:len(records)])
    orig, _ = it.read_train_records(it.train_files(str(shards)), NUM_CLASSES)
    assert [r[3] for r in records] == [r[3] for r in orig]
    res = train_and_evaluate(str(out), str(tmp_path / "run"), batch_size=8, dataset_name=DATASET, train_epochs=1,
                             image_size=64, seed=3, num_workers=4, dtype="bf16", kd_temp=2.0,
                             base_learning_rate=0.01, num_best_ckpt_to_keep=1)
    assert len(res) == 1 and res[0]["global_step"] == 33 // 8
    assert np.isfinite(res[0]["loss"]) and 0.0 <= res[0]["accuracy"] <= 1.0
