"""CPU checks of the classification evaluation (classifier.evaluate(input_fn_eval)): the eval geometry
against golden data of the reference's own code (tests/golden/make_eval_preprocess_golden.py), the
oracle's legacy bilinear resize against hand-computed answers and scipy, the TFRecord reader against a
shard written by the protobuf runtime, the oracle's in_top_k rule, classification_result against
EvalMetrics, the host-side argument checks of the new entry points and the new kernels in the SASS."""
import hashlib
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLD_DIR = os.path.join(ROOT, "golden")
GOLD = json.load(open(os.path.join(GOLD_DIR, "eval_preprocess_golden.json")))
SHARD = os.path.join(GOLD_DIR, "eval_golden.tfrecord")
# smaller sides whose float32 product rounds 256 down to 255 (107 ... 165) and 292 down to 291 (145 ... 550)
ROUND_DOWN = (107, 109, 110, 121, 165, 145, 275, 290, 550)


def test_eval_geometry_matches_reference():
    from assembled_cnn_b200.imagenet_eval import CHANNEL_MEANS, eval_geometry
    from oracle import eval_preprocess as O
    assert len(GOLD["cases"]) >= 300
    rounded = 0
    for c in GOLD["cases"]:
        want = (c["S"], c["rsz"][0], c["rsz"][1], c["crop"][0], c["crop"][1])
        assert eval_geometry(c["h"], c["w"], c["type"], c["image_size"]) == want, c
        assert O.geometry(c["h"], c["w"], c["type"], c["image_size"]) == want, c
        assert tuple(c["mean"]) == CHANNEL_MEANS == O.CHANNEL_MEANS
        rounded += min(c["rsz"]) in (255, 291) and min(c["h"], c["w"]) in ROUND_DOWN
    assert rounded >= 9 * 2             # the float32 round-down cases are in the golden


def test_eval_size_refusals():
    from assembled_cnn_b200.imagenet_eval import eval_size
    assert eval_size("imagenet", 224) == (224, 0) and eval_size("imagenet_224_256a") == (256, 1)
    assert eval_size("imagenet_320") == (320, 0) and eval_size("imagenet_288a") == (288, 1)
    for t in ("cub", "imagenet_22", "foo"):
        with pytest.raises(NotImplementedError, match="unknown"):
            eval_size(t)
    for t in ("reid", "reid_224", "inception_331", "inception_600"):
        with pytest.raises(NotImplementedError, match="reid / inception"):
            eval_size(t)
    for t, s in (("imagenet_300", 224), ("imagenet_299a", 224), ("imagenet", 200), ("imagenet", 16)):
        with pytest.raises(ValueError, match="multiple of 32"):
            eval_size(t, s)


def test_oracle_resize_known_answers():
    from oracle.eval_preprocess import resize_bilinear
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (7, 5, 3)).astype(np.uint8)
    assert np.array_equal(resize_bilinear(img, 7, 5), img.astype(np.float32))      # identity
    ramp = np.array([[0, 10], [20, 30]], dtype=np.float32)[:, :, None]
    want = np.array([[0, 5, 10, 10], [10, 15, 20, 20], [20, 25, 30, 30], [20, 25, 30, 30]], np.float32)
    assert np.array_equal(resize_bilinear(ramp, 4, 4)[:, :, 0], want)              # clamped edge repeats


@pytest.mark.parametrize("shape,out", [((13, 17), (29, 11)), ((64, 48), (256, 192)), ((500, 375), (224, 168)),
                                       ((1, 9), (4, 36))])
def test_oracle_resize_matches_scipy(shape, out):
    from scipy.ndimage import map_coordinates
    from oracle.eval_preprocess import resize_bilinear
    rng = np.random.default_rng(sum(shape))
    img = rng.integers(0, 256, shape + (3,)).astype(np.float64)
    got = resize_bilinear(img.astype(np.uint8), *out)
    # the sample coordinates i * in / out as TF forms them (fp32); the interpolation itself is scipy's
    yy = (np.arange(out[0], dtype=np.float32) * (np.float32(shape[0]) / np.float32(out[0]))).astype(np.float64)
    xx = (np.arange(out[1], dtype=np.float32) * (np.float32(shape[1]) / np.float32(out[1]))).astype(np.float64)
    Y, X = np.meshgrid(yy, xx, indexing="ij")
    for c in range(3):
        want = map_coordinates(img[:, :, c], [Y, X], order=1, mode="nearest")
        assert np.abs(got[:, :, c] - want).max() < 1e-3


def test_crc32c_known_answer():
    from assembled_cnn_b200.imagenet_eval import crc32c
    assert crc32c(b"123456789") == 0xE3069283
    assert crc32c(b"") == 0


def test_reader_matches_golden_shard():
    from assembled_cnn_b200.imagenet_eval import read_encoded, read_records, decode_rgb
    import io
    recs = read_records(SHARD)
    assert [r[0] for r in recs] == [m["label"] for m in GOLD["shard"]]
    for (label, off, n), m in zip(recs, GOLD["shard"]):
        jpeg = read_encoded(SHARD, off, n)
        assert hashlib.sha256(jpeg).hexdigest() == m["sha256"]
        assert decode_rgb(io.BytesIO(jpeg)).shape == (m["h"], m["w"], 3)


def test_reader_errors_name_the_offset(tmp_path):
    from assembled_cnn_b200.imagenet_eval import read_records, validation_files
    data = open(SHARD, "rb").read()
    first_len = int.from_bytes(data[:8], "little")
    second = 12 + first_len + 4
    flipped = bytearray(data)
    flipped[second] ^= 0x01                       # a length byte of the second record
    (tmp_path / "validation-00000-of-00002").write_bytes(bytes(flipped))
    with pytest.raises(ValueError, match="validation-00000-of-00002: corrupt record length at byte offset %d"
                       % second):
        read_records(str(tmp_path / "validation-00000-of-00002"))
    (tmp_path / "validation-00001-of-00002").write_bytes(data[:second + 40])
    with pytest.raises(ValueError, match="truncated record at byte offset %d" % second):
        read_records(str(tmp_path / "validation-00001-of-00002"))
    (tmp_path / "validation-00001-of-00002").write_bytes(data[:second + 5])
    with pytest.raises(ValueError, match="truncated record header at byte offset %d" % second):
        read_records(str(tmp_path / "validation-00001-of-00002"))
    assert validation_files(str(tmp_path)) == sorted(str(p) for p in tmp_path.glob("validation-*"))
    with pytest.raises(FileNotFoundError):
        validation_files(str(tmp_path), "train-*")


def test_oracle_in_top_k_ties_and_non_finite():
    from oracle.eval_preprocess import argmax, in_top_k
    x = np.full((5, 8), -1.0)
    x[0, [1, 2, 3, 4, 5, 6]] = 2.0                 # six-way tie with the target: in for any k
    x[1, :6] = [5, 4, 3, 2, 1, 1]                  # target 5 ties with 4 at the 5th place
    x[2, 3] = np.nan
    x[3, 0] = np.inf
    x[4, 7] = 9.0
    labels = np.array([6, 5, 0, 0, 8])
    assert in_top_k(x, labels, 1).tolist() == [True, False, False, False, False]
    assert in_top_k(x, labels, 5).tolist() == [True, True, False, False, False]
    assert in_top_k(x[:2], [6, 6], 5).tolist() == [True, False]
    assert argmax(x).tolist() == [1, 0, -1, -1, 7]


def test_classification_result_equals_eval_metrics():
    import torch
    from assembled_cnn_b200.metrics import EvalMetrics, classification_result
    from oracle import eval_preprocess as O
    rng = np.random.default_rng(1)
    logits = (rng.standard_normal((300, 50)) * 3).astype(np.float32)
    labels = rng.integers(0, 50, 300)
    labels[::4] = logits[::4].argmax(1)
    em = EvalMetrics()
    sizes = [128, 128, 44]
    for a, b in ((0, 128), (128, 256), (256, 300)):
        em.update(torch.from_numpy(logits[a:b]), torch.from_numpy(labels[a:b]))
    want = em.result()
    conf = torch.softmax(torch.from_numpy(logits), 1).max(1).values.numpy()
    ce = O.cross_entropy(logits, labels, 0.1)
    got = classification_result(O.argmax(logits), conf, O.in_top_k(logits, labels, 5), ce, labels, sizes)
    assert got["accuracy"] == want["accuracy"] and got["accuracy_top_5"] == want["accuracy_top_5"]
    assert abs(got["ece"] - want["ece"]) < 1e-6
    assert got["ece"] == pytest.approx(O.ece(conf, O.argmax(logits), labels), abs=1e-12)
    assert got["cross_entropy"] == pytest.approx(np.mean([ce[:128].mean(), ce[128:256].mean(), ce[256:].mean()]),
                                                 rel=1e-14)
    with pytest.raises(ValueError):
        classification_result(O.argmax(logits), conf, O.in_top_k(logits, labels, 5), ce, labels, [128, 128])


def test_descriptor_check():
    from assembled_cnn_b200.imagenet_eval import DESC_DTYPE, check_descriptors
    d = np.zeros(4, DESC_DTYPE)
    d[:] = (1 << 20, 375, 500, 256, 341, 16, 58)
    check_descriptors(d, 4, 224)
    for field, v in (("src", 0), ("src_h", 0), ("src_w", -1), ("crop_y", 33), ("crop_x", -1), ("rsz_w", 281)):
        bad = d.copy()
        bad[2][field] = v
        with pytest.raises(ValueError, match="descriptor 2"):
            check_descriptors(bad, 4, 224)
        check_descriptors(bad, 2, 224)            # rows >= n_valid are not read


def test_evaluate_classification_checks_before_any_gpu_work(tmp_path):
    from assembled_cnn_b200.model_fns import build_model, evaluate_classification
    model = build_model(resnet_size=50, num_classes=1000)
    with pytest.raises(FileNotFoundError):
        evaluate_classification(model, str(tmp_path))
    shutil.copy(SHARD, tmp_path / "validation-00000-of-00001")
    # the golden shard holds label 1000: outside [0, 1000)
    with pytest.raises(ValueError, match="label 1000"):
        evaluate_classification(model, str(tmp_path))
    with pytest.raises(NotImplementedError):
        evaluate_classification(model, str(tmp_path), preprocessing_type="inception_331")
    with pytest.raises(ValueError, match="multiple of 32"):
        evaluate_classification(model, str(tmp_path), preprocessing_type="imagenet_300")
    (tmp_path / "validation-00000-of-00001").write_bytes(open(SHARD, "rb").read()[:100])
    with pytest.raises(ValueError, match="byte offset 0"):
        evaluate_classification(build_model(resnet_size=50), str(tmp_path))


def test_hparams_defaults():
    from assembled_cnn_b200.hparams import DEFAULTS
    assert DEFAULTS["preprocessing_type"] == "imagenet" and DEFAULTS["val_regex"] == "validation-*"


def test_argument_errors_without_gpu():
    """The host-side checks of the new entry points run before any CUDA call."""
    from assembled_cnn_b200 import _lib, native
    lib = _lib.load()
    INVALID = 1
    p = 1 << 20          # never dereferenced: the checks fail first

    def rows(logits=p, B=4, ld=16, NC=10, labels=p, n_valid=4, k=5, ls=0.1, pred=p, conf=p, hit=p, ce=p):
        return lib.acnn_classify_rows(logits, B, ld, NC, labels, n_valid, k, ls, pred, conf, hit, ce, None)

    for kw in (dict(logits=None), dict(labels=None), dict(pred=None), dict(conf=None), dict(hit=None),
               dict(ce=None), dict(B=0), dict(NC=0), dict(ld=9), dict(n_valid=5), dict(n_valid=-1), dict(k=0),
               dict(ls=float("nan")), dict(ls=float("inf"))):
        assert rows(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    assert rows(n_valid=0) == 0

    def resize(desc=p, B=4, n_valid=4, S=224, mean=p, out=p):
        return lib.acnn_resize_crop_u8(desc, B, n_valid, S, mean, out, None)

    for kw in (dict(desc=None), dict(mean=None), dict(out=None), dict(B=0), dict(S=0), dict(S=-32),
               dict(n_valid=5), dict(n_valid=-1), dict(out=p + 2), dict(desc=p + 4)):
        assert resize(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    nl = native.lib()
    assert nl.acnn_set_images_resized(None, p, 1, p, None) == INVALID


def test_new_kernels_in_sass():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from assembled_cnn_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for kernel in ("resize_crop_u8_kernel", "classify_rows_kernel"):
        assert kernel in sass, kernel
