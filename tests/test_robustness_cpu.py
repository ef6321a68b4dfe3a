"""CPU checks of the robustness evaluation (mce/eval_robustness.py, --robustness_type ce): the product's
AlexNet table, distortion quota and label mapping against golden data of the reference's own code
(tests/golden/make_robustness_golden.py), the oracle's mCE arithmetic, the ImageNet-C tree walk and its
errors, the host-side argument checks of acnn_images_from_u8 / acnn_softmax_top1_count /
acnn_set_images_u8, and the new kernels in the library's SASS."""
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "robustness_golden.json")))


def test_alexnet_table_matches_reference():
    from assembled_cnn_b200.metrics import ALEXNET_CE, DISTORTIONS
    from oracle import robustness as R
    assert [[k, v] for k, v in ALEXNET_CE.items()] == GOLD["alexnet_ce"]
    assert list(R.ALEXNET_CE.items()) == [tuple(kv) for kv in GOLD["alexnet_ce"]]
    assert list(DISTORTIONS) == [k for k, _ in GOLD["alexnet_ce"]] and len(DISTORTIONS) == 19


@pytest.mark.parametrize("g", range(1, 9))
def test_distortion_quota_matches_reference(g):
    from assembled_cnn_b200.imagenet_c import distortion_quota
    from oracle import robustness as R
    assert distortion_quota(g) == GOLD["quota"][str(g)]
    assert R.quota(g) == GOLD["quota"][str(g)]


def test_label_mapping_matches_reference(tmp_path):
    from assembled_cnn_b200.imagenet_c import get_synsets2idx
    path = tmp_path / "labels.txt"
    path.write_text("".join(GOLD["label_lines"]))
    assert get_synsets2idx(str(path)) == GOLD["synsets2idx"]


def test_oracle_mce_arithmetic_on_fixed_counts():
    from oracle import robustness as R
    names = list(R.ALEXNET_CE)
    count = {d: 1000 + 7 * i for i, d in enumerate(names)}
    correct = {d: 400 + 13 * i for i, d in enumerate(names)}
    m, mu, per = R.mce(correct, count)
    errs = [1 - (400 + 13 * i) / (1000 + 7 * i) for i in range(19)]
    ces = [e / R.ALEXNET_CE[d] for e, d in zip(errs, names)]
    assert per["gaussian_noise"] == (0.6, 0.6 / 0.8864)
    assert m == pytest.approx(sum(ces) / 19, rel=1e-15) and mu == pytest.approx(sum(errs) / 19, rel=1e-15)
    # all correct: zero error; none correct: the mean of 1 / ALEXNET_CE
    assert R.mce(count, count)[:2] == (0.0, 0.0)
    zero = {d: 0 for d in names}
    assert R.mce(zero, count)[0] == pytest.approx(np.mean([1 / v for v in R.ALEXNET_CE.values()]), rel=1e-15)


def test_product_result_equals_oracle():
    from assembled_cnn_b200.metrics import corruption_error_result
    from oracle import robustness as R
    rng = np.random.default_rng(3)
    count = {d: int(rng.integers(1, 50000)) for d in R.ALEXNET_CE}
    correct = {d: int(rng.integers(0, count[d] + 1)) for d in R.ALEXNET_CE}
    got = corruption_error_result(correct, count)
    m, mu, per = R.mce(correct, count)
    assert got["mCE"] == m and got["mCE_unnormalized"] == mu
    for d, (err, ce) in per.items():
        assert got[d] == {"error": err, "ce": ce}
    with pytest.raises(ValueError, match="frost"):
        corruption_error_result(correct, dict(count, frost=0))
    del count["fog"]
    with pytest.raises(ValueError, match="fog"):
        corruption_error_result(correct, count)


def test_corruption_error_metric_refuses_empty_distortions():
    import torch
    from assembled_cnn_b200.metrics import CorruptionError, DISTORTIONS
    metric = CorruptionError(device="cpu")
    for d in DISTORTIONS[:-1]:
        metric.add_counts(d, 3, 4)
    with pytest.raises(ValueError, match="saturate"):
        metric.result()
    metric.add_counts("saturate", 1, 4)
    r = metric.result()
    assert r["saturate"]["error"] == 0.75 and r["fog"]["error"] == 0.25
    with pytest.raises(ValueError):
        metric.add_counts("rotate", 1, 1)
    assert metric.correct.dtype == torch.int64


def _jpeg(path, size, color=(10, 200, 30)):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.new("RGB", (size[0], size[1]), color).save(path, format="JPEG")


def _tree(root, synsets, per_dir=2, size=(16, 16), distortions=None):
    from assembled_cnn_b200.metrics import DISTORTIONS
    for d in distortions or DISTORTIONS:
        for s in range(1, 6):
            for k, syn in enumerate(synsets):
                for j in range(per_dir):
                    # any extension is taken, as by the reference's glob
                    _jpeg(os.path.join(root, d, str(s), syn, "img%d%s" % (j, ".JPEG" if j else ".png.jpg")), size)


def test_tree_walk_and_labels(tmp_path):
    from assembled_cnn_b200.imagenet_c import distortion_images, get_synsets2idx, decode_image
    (tmp_path / "labels.txt").write_text("Background\nn01440764\nN01443537\nGold Fish\n")
    syn = get_synsets2idx(str(tmp_path / "labels.txt"))
    _tree(str(tmp_path / "c"), ["n01440764", "n01443537", "gold_fish"], distortions=["fog"])
    (tmp_path / "c" / "fog" / "3" / "stray_file.txt").write_text("not a synset dir")   # skipped, as by glob
    files, labels = distortion_images(str(tmp_path / "c"), "fog", syn, label_offset=1)
    assert len(files) == 5 * 3 * 2
    assert sorted(set(labels)) == [2, 3, 4]
    for f, y in zip(files, labels):
        assert y == syn[os.path.basename(os.path.dirname(f))] + 1
    files0, labels0 = distortion_images(str(tmp_path / "c"), "fog", syn, label_offset=0)
    assert files0 == files and [y + 1 for y in labels0] == labels
    a = decode_image(files[0], 16)
    assert a.dtype == np.uint8 and a.shape == (16, 16, 3)


def test_tree_errors(tmp_path):
    from assembled_cnn_b200.imagenet_c import distortion_images, decode_image
    syn = {"n01440764": 0}
    _tree(str(tmp_path / "c"), ["n01440764"], per_dir=1, distortions=["fog"])
    with pytest.raises(FileNotFoundError, match="frost"):
        distortion_images(str(tmp_path / "c"), "frost", syn)
    _jpeg(str(tmp_path / "c" / "fog" / "2" / "n99999999" / "x.jpg"), (16, 16))
    with pytest.raises(ValueError, match="n99999999"):
        distortion_images(str(tmp_path / "c"), "fog", syn)
    _jpeg(str(tmp_path / "wrong.jpg"), (16, 12))
    with pytest.raises(ValueError, match="expected 16x16"):
        decode_image(str(tmp_path / "wrong.jpg"), 16)
    import shutil
    shutil.rmtree(tmp_path / "c" / "fog" / "4")
    with pytest.raises(FileNotFoundError, match="severity"):
        distortion_images(str(tmp_path / "c"), "fog", {"n01440764": 0, "n99999999": 1})


def test_corruption_error_checks_before_any_gpu_work(tmp_path):
    """robustness_type errors with the reference's messages, a missing distortion, and an empty one are
    all raised before a runtime is built (no GPU is touched)."""
    from assembled_cnn_b200.model_fns import build_model, corruption_error
    from assembled_cnn_b200.metrics import DISTORTIONS
    model = build_model(resnet_size=50, num_classes=10)
    (tmp_path / "labels.txt").write_text("a\nb\n")
    with pytest.raises(ValueError) as e:
        corruption_error(model, str(tmp_path), str(tmp_path / "labels.txt"), robustness_type="fr")
    assert str(e.value) == "not yet supported (fr"
    with pytest.raises(ValueError) as e:
        corruption_error(model, str(tmp_path), str(tmp_path / "labels.txt"), robustness_type="mfr")
    assert str(e.value) == "invalid type (mfr)"
    _tree(str(tmp_path / "c"), ["a"], per_dir=1, distortions=DISTORTIONS[:-1])
    with pytest.raises(FileNotFoundError, match="saturate"):
        corruption_error(model, str(tmp_path / "c"), str(tmp_path / "labels.txt"))
    for s in range(1, 6):
        os.makedirs(tmp_path / "c" / "saturate" / str(s))
    with pytest.raises(ValueError, match="saturate"):
        corruption_error(model, str(tmp_path / "c"), str(tmp_path / "labels.txt"))


def test_argument_errors_without_gpu():
    """The host-side checks of the new entry points run before any CUDA call."""
    from assembled_cnn_b200 import _lib, native
    lib = _lib.load()
    INVALID = 1
    p = 1 << 20          # never dereferenced: the checks fail first

    def top1(logits=p, B=4, ld=16, NC=10, labels=p, n_valid=4, pred=p, correct=p):
        return lib.acnn_softmax_top1_count(logits, B, ld, NC, labels, n_valid, pred, correct, None)

    for kw in (dict(logits=None), dict(labels=None), dict(pred=None), dict(correct=None), dict(B=0),
               dict(NC=0), dict(ld=9), dict(n_valid=5), dict(n_valid=-1), dict(B=-2, n_valid=0)):
        assert top1(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    assert top1(n_valid=0) == 0          # nothing to count: nothing is launched

    def u8(images=p, mean=p, out=p, B=2, H=4, W=4):
        return lib.acnn_images_from_u8(images, mean, out, B, H, W, None)

    for kw in (dict(images=None), dict(mean=None), dict(out=None), dict(B=0), dict(H=-1), dict(W=0),
               dict(images=p + 4), dict(out=p + 8)):
        assert u8(**kw) == INVALID, kw
    nl = native.lib()
    assert nl.acnn_set_images_u8(None, p, p, None) == INVALID


def test_new_kernels_in_sass():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from assembled_cnn_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for kernel in ("images_from_u8_kernel", "softmax_top1_count_kernel"):
        assert kernel in sass, kernel
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
