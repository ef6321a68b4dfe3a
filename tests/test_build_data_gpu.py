"""GPU checks of the dataset builders (assembled_cnn_b200.build_data): the device check (jpeg.JpegDecoder on a
copy stream, PIL for the rest) writes the same bytes as the PIL check for every builder and matches the
reference's golden records; a damaged scan raises with its path and leaves no partial shard; and shards
built from synthetic ImageNet-, SOP- and CUB-style trees run through train_and_evaluate,
evaluate_classification, extract_teacher_logits and evaluate_retrieval."""
import importlib.util
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("test_build_data_cpu", os.path.join(HERE, "test_build_data_cpu.py"))
cpu = importlib.util.module_from_spec(spec)
spec.loader.exec_module(cpu)
mg = cpu.mg


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("raw"))
    mg.make_tree(root, cpu.GOLDEN["seed"])
    return root


def _files(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


CASES = [("imagenet", 2), ("imagenet_no_logits", 2), ("food101", 8), ("cub_200_2011", 8),
         ("cub_200_2011_no_bbox", 8), ("cars196_zeroshot", 1), ("SOP", 2)]


@pytest.mark.parametrize("name,t", CASES, ids=["%s-threads%d" % c for c in CASES])
def test_device_check_equals_pil_check(tree, tmp_path, name, t):
    from assembled_cnn_b200 import build_data
    dataset, args, flags = cpu.build_args(name, tree, t)
    out = {}
    for check in ("device", "pil"):
        out[check] = str(tmp_path / check)
        build_data.build(dataset, out[check], *args, check=check, num_workers=4, **flags)
    assert _files(out["device"]) == _files(out["pil"])
    cpu.check_against_golden(tree, name, t, out["device"])


def test_device_check_decodes_on_the_device(tree, monkeypatch):
    """The baseline JPEGs of the tree are checked by the device decoder, not by the PIL fallback."""
    from assembled_cnn_b200 import build_data
    calls = []
    real = build_data._pil
    monkeypatch.setattr(build_data, "_pil", lambda data: calls.append(len(data)) or real(data))
    dataset, args, flags = cpu.build_args("cars196_zeroshot", tree, 8)
    splits = build_data.BUILDERS[dataset](*args, **flags)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        build_data.write_splits(splits, os.path.join(d, "out"), check="device", num_workers=4)
    assert sum(len(s.items) for s in splits) > 100 and calls == []


def test_damaged_scan_raises_with_its_path(tree, tmp_path):
    from assembled_cnn_b200 import build_data, jpeg
    im = str(tmp_path / "imagenet")
    shutil.copytree(os.path.join(tree, "imagenet"), im)
    bad = os.path.join(im, "validation", "n01739381")
    bad = os.path.join(bad, sorted(os.listdir(bad))[0])
    data = open(bad, "rb").read()
    assert jpeg.parse([data])[0]["supported"]                       # a scan the device decodes
    open(bad, "wb").write(data[:len(data) * 2 // 3])
    out = tmp_path / "out"
    with pytest.raises(ValueError, match=bad):
        build_data.build("imagenet", str(out), im + "/train", im + "/validation", check="device",
                         make_train=False, **cpu.imagenet_flags(tree, 2))
    assert not [f for f in os.listdir(out) if f.startswith(".")]


# --------------------------------------------------------------------------------- downstream loops
def _imagenet_tree(root, rng, n_per_class=(14, 12, 14), n_val=12):
    """An ImageNet-style tree of 375 x 500 and 333 x 250 JPEGs over three synsets."""
    from PIL import Image
    import io
    synsets = ["n01440764", "n01443537", "n01484850"]
    os.makedirs(root)
    with open(os.path.join(root, "synsets.txt"), "w") as f:
        f.write("\n".join(synsets) + "\n")
    with open(os.path.join(root, "metadata.txt"), "w") as f:
        f.write("".join("%s\tclass %d\n" % (s, i) for i, s in enumerate(synsets)))

    def jpg(h, w):
        base = rng.integers(0, 256, size=(6, 8, 3), dtype=np.uint8)
        b = io.BytesIO()
        Image.fromarray(base).resize((w, h), Image.BILINEAR).save(b, "JPEG", quality=85)
        return b.getvalue()

    for split, counts in (("train", n_per_class), ("validation", (n_val // 3,) * 3)):
        for s, n in zip(synsets, counts):
            os.makedirs(os.path.join(root, split, s))
            for j in range(n):
                h, w = (375, 500) if j % 2 else (333, 250)
                with open(os.path.join(root, split, s, "%s_%d.JPEG" % (s, j)), "wb") as f:
                    f.write(jpg(h, w))


def test_imagenet_shards_run_through_the_loops(tmp_path):
    from assembled_cnn_b200 import build_data
    from assembled_cnn_b200.imagenet_train import read_train_records, train_files
    from assembled_cnn_b200.model_fns import (build_model, evaluate_classification, extract_teacher_logits,
                                              train_and_evaluate)
    raw = str(tmp_path / "raw")
    _imagenet_tree(raw, np.random.default_rng(4))
    data = str(tmp_path / "shards")
    n = build_data.build("imagenet", data, raw + "/train", raw + "/validation", train_shards=4, validation_shards=2,
                         num_threads=2, labels_file=raw + "/synsets.txt", imagenet_metadata_file=raw + "/metadata.txt")
    assert n == {"validation": 12, "train": 40}
    records, counts = read_train_records(train_files(data), 1001)
    assert sorted(r[3] for r in records) == [1] * 14 + [2] * 12 + [3] * 14
    model = build_model(resnet_size=50, num_classes=1001, dtype="bf16", seed=2)
    ev = evaluate_classification(model, data, image_size=64, batch_size=8, num_workers=4)
    assert 0.0 <= ev["accuracy"] <= 1.0 and np.isfinite(ev["loss"])
    kd = str(tmp_path / "kd")
    written = extract_teacher_logits(model, data, kd, image_size=64, batch_size=8, dataset_name="imagenet")
    assert sorted(os.path.basename(p) for p in written) == sorted(os.listdir(data))
    res = train_and_evaluate(data, str(tmp_path / "run"), batch_size=8, dataset_name="imagenet", train_epochs=1,
                             image_size=64, seed=3, num_workers=4, dtype="bf16", base_learning_rate=0.01,
                             num_best_ckpt_to_keep=1)
    assert len(res) == 1 and res[0]["global_step"] == 40 // 8
    assert np.isfinite(res[0]["loss"]) and 0.0 <= res[0]["accuracy"] <= 1.0


@pytest.mark.parametrize("name", ["SOP", "cub_200_2011"])
def test_retrieval_shards_run_through_evaluate_retrieval(tree, tmp_path, name):
    from assembled_cnn_b200 import build_data
    from assembled_cnn_b200.imagenet_eval import read_records, validation_files
    from assembled_cnn_b200.model_fns import build_model, evaluate_retrieval
    dataset, args, flags = cpu.build_args(name, tree, 8)
    data = str(tmp_path / "shards")
    build_data.build(dataset, data, *args, **flags)
    labels = [r[0] for f in validation_files(data) for r in read_records(f)]
    model = build_model(resnet_size=50, num_classes=100, embedding_size=32, dtype="bf16", seed=1)
    res = evaluate_retrieval(model, data, image_size=64, batch_size=8, recall_at_k=(1, 2), num_workers=4)
    assert len(labels) >= 3 and set(res) == {"recall_at_1", "recall_at_2", "global_step"}
    assert 0.0 <= res["recall_at_1"] <= res["recall_at_2"] <= 1.0
