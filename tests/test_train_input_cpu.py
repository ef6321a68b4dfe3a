"""CPU checks of training from TFRecord shards: the dispatch, sampler arguments, order of operations,
input_fn_cls's mixup doubling and the epoch schedules against golden data of the reference's own code
(tests/golden/make_train_preprocess_golden.py); the crop window sampler against the oracle on scripted and
seeded draws and its properties; the record stream against the oracle's order (permutations, rank slices,
worker independence, resume); the KD logit parsing and its errors; the flag errors; the host-side argument
errors of the new entry points and the new kernel in the SASS."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(ROOT, "golden", "train_preprocess_golden.json")))


# ------------------------------------------------------------------------------- golden: reference code
def test_dispatch_sampler_arguments_and_order_match_reference():
    from assembled_cnn_b200.imagenet_train import CHANNEL_MEANS, train_size
    assert len(GOLD["cases"]) >= 150
    for c in GOLD["cases"]:
        assert train_size(c["type"], c["image_size"]) == c["S"], c
        s = c["sampler"]
        assert s["min_object_covered"] == (0.1 if c["use_random_crop"] else 1.0)
        assert s["aspect_ratio_range"] == [0.75, 1.33] and s["area_range"] == [0.05, 1.0]
        assert s["max_attempts"] == 100 and s["use_image_if_no_bounding_boxes"] is True
        assert s["image_size"] == [c["h"], c["w"], 3] and c["bbox_zeros"] == [0, 0, 4]
        assert c["crop_window"] == c["box"]                   # the sampled box is the decode window
        assert c["ops"] == ["sample", "decode_and_crop", "flip", "resize", "mean"]
        assert c["flipped"] == (c["u_flip"] < 0.5)
        assert tuple(c["mean"]) == CHANNEL_MEANS


def test_input_fn_cls_mixup_doubles_batch_and_epochs():
    for c in GOLD["input_fn_cls"]:
        k = 2 if c["mixup_type"] == 1 else 1
        assert c["train"]["batch_size"] == k * c["batch_size"] // c["num_gpus"]
        assert c["train"]["num_epochs"] == k * c["num_epochs"]
        assert c["eval"]["batch_size"] == c["batch_size"] // c["num_gpus"] and c["eval"]["num_epochs"] == 1
        assert c["train"]["shuffle_buffer"] == 10000


def test_epoch_schedule_matches_reference():
    from assembled_cnn_b200.imagenet_train import epoch_schedule
    assert len(GOLD["schedules"]) >= 10
    for c in GOLD["schedules"]:
        cur = c["resume_step"] // int(c["num_images"] / c["batch_size"])
        got = epoch_schedule(c["train_epochs"], c["epochs_between_evals"], c["ratio_fine_eval"], cur)
        assert got == c["schedule"], c
        # a resumed schedule is a suffix of the fresh one: the cycle index is its position in the fresh one
        full = epoch_schedule(c["train_epochs"], c["epochs_between_evals"], c["ratio_fine_eval"])
        assert full[len(full) - len(got):] == got


def test_train_size_refusals():
    from assembled_cnn_b200.imagenet_train import train_size
    assert train_size("imagenet_224_256a", 64) == 224 and train_size("imagenet_288a") == 288
    for t in ("reid", "reid_224", "inception_331", "inception_600"):
        with pytest.raises(NotImplementedError, match="reid / inception"):
            train_size(t)
    with pytest.raises(NotImplementedError, match="unknown"):
        train_size("cub")
    with pytest.raises(ValueError, match="multiple of 32"):
        train_size("imagenet", 200)


# ------------------------------------------------------------------------------------------- sampler
class Script:
    def __init__(self, values):
        self.values, self.i = list(values), 0

    def __call__(self):
        v = self.values[self.i % len(self.values)]
        self.i += 1
        return v


SAMPLER_SIZES = [(1, 1), (1, 7), (7, 1), (1, 500), (500, 1), (2, 3), (3, 1000), (1000, 3), (375, 500),
                 (500, 375), (2592, 1944), (64, 64), (17, 23), (10, 2000), (2000, 10)]


@pytest.mark.parametrize("h,w", SAMPLER_SIZES)
def test_sampler_matches_oracle_on_scripted_draws(h, w):
    from assembled_cnn_b200.imagenet_train import sample_distorted_bounding_box
    from oracle.train_preprocess import sample_box
    rng = np.random.default_rng(h * 7919 + w)
    for trial in range(60):
        draws = list(rng.random(int(rng.integers(1, 12))))
        if trial % 5 == 0:
            draws += [0.0, 0.999999, 0.5]
        for moc in (0.1, 1.0, 0.5):
            a = Script(draws)
            b = Script(draws)
            got = sample_distorted_bounding_box(h, w, a, moc)
            assert got == sample_box(h, w, b, moc), (h, w, draws, moc)
            assert a.i == b.i                              # the same draws consumed


@pytest.mark.parametrize("h,w", SAMPLER_SIZES)
def test_sampler_properties(h, w):
    from assembled_cnn_b200.imagenet_train import crop_window, example_rng, sample_distorted_bounding_box
    from oracle.train_preprocess import example
    rng = np.random.default_rng(5)
    fallback = 0
    for _ in range(200):
        y, x, ch, cw = sample_distorted_bounding_box(h, w, rng.random)
        assert 0 <= y and 0 <= x and ch >= 1 and cw >= 1 and y + ch <= h and x + cw <= w
        whole = (y, x, ch, cw) == (0, 0, h, w)
        assert whole or np.float32(ch * cw) / np.float32(h * w) >= np.float32(0.1)
        fallback += whole
        # min_object_covered = 1.0: only the whole image covers the whole object
        assert sample_distorted_bounding_box(h, w, rng.random, 1.0) == (0, 0, h, w)
    for p in range(20):
        assert crop_window(h, w, example_rng(3, 1, p)) == example(h, w, 3, 1, p)
        assert crop_window(h, w, example_rng(3, 1, p), False)[:4] == (0, 0, h, w)


def test_sampler_draws_and_fallback():
    from assembled_cnn_b200.imagenet_train import sample_distorted_bounding_box
    # aspect 0.75 + 0 (draw 0), min area 0.05 * 100 * 100: height lrintf(sqrt(500 / 0.75)) = 26, max_height
    # 115 clamped to 100; height 26 + Uniform(75) at draw 0 = 26, width lrintf(19.5) = 20, area 520;
    # y = Uniform(74), x = Uniform(80) at draw 0.5 -> (37, 40); it covers 0.052 of the image: accepted at
    # min_object_covered 0.05, rejected by every attempt (the same draws) at 0.1
    assert sample_distorted_bounding_box(100, 100, Script([0.0, 0.0, 0.5, 0.5]), 0.05) == (37, 40, 26, 20)
    assert sample_distorted_bounding_box(100, 100, Script([0.0, 0.0, 0.5, 0.5]), 0.1) == (0, 0, 100, 100)
    # every attempt of a 1 x 1 image at min coverage 1.0 gives the whole image
    assert sample_distorted_bounding_box(1, 1, Script([0.3]), 1.0) == (0, 0, 1, 1)


# ------------------------------------------------------------------------------------------- stream
COUNTS = [7, 0, 13, 5, 1, 9, 11, 2, 6, 8, 3, 4, 10, 12, 1, 5, 7, 3, 2, 6, 9, 4, 8]     # 23 files, 135 records


@pytest.mark.parametrize("buffer", [1, 16, 1000])
def test_epoch_order_matches_oracle_and_is_a_permutation(buffer):
    from assembled_cnn_b200.imagenet_train import epoch_order
    from oracle import train_preprocess as O
    n = sum(COUNTS)
    for cycle in range(3):
        for e in range(2):
            got = epoch_order(COUNTS, 9, cycle, e, buffer)
            assert got.tolist() == O.epoch(COUNTS, 9, cycle, e, buffer)
            assert sorted(got.tolist()) == list(range(n))
    # buffer 1: no record shuffle, the interleave order itself
    order = O.interleave(COUNTS, list(range(len(COUNTS))))
    assert order[:3] == [(0, 0), (2, 0), (3, 0)] and len(order) == n


def test_interleave_rules():
    from oracle.train_preprocess import interleave
    # 21 files of 2 records: the 21st waits for the first slot that empties, then starts at once
    out = interleave([2] * 21, list(range(21)))
    assert out[:20] == [(f, 0) for f in range(20)] and out[20:40] == [(f, 1) for f in range(20)]
    assert out[40:] == [(20, 0), (20, 1)]


@pytest.mark.parametrize("epochs,ib", [(1, 8), (3, 16), (2, 5)])
def test_cycle_stream_ranks_resume_and_oracle(epochs, ib):
    from assembled_cnn_b200.imagenet_train import CycleStream
    from oracle import train_preprocess as O
    n = sum(COUNTS)
    full = O.stream(COUNTS, 4, 2, epochs, 16)
    one = CycleStream(COUNTS, 4, 2, epochs, 16, 2 * ib)
    assert one.steps == epochs * n // (2 * ib)             # the partial last batch is dropped
    two = [CycleStream(COUNTS, 4, 2, epochs, 16, ib, world=2, rank=r) for r in range(2)]
    assert two[0].steps == two[1].steps == one.steps
    for t in range(one.steps):
        g = [r for _, r in one.records(t)]
        assert g == full[t * 2 * ib:(t + 1) * 2 * ib]
        assert [r for _, r in two[0].records(t)] + [r for _, r in two[1].records(t)] == g
    # a fresh object (a resumed run) gives the same cycle; a different cycle another order
    again = CycleStream(COUNTS, 4, 2, epochs, 16, 2 * ib)
    assert [again.records(t) for t in range(one.steps)] == [one.records(t) for t in range(one.steps)]
    assert O.stream(COUNTS, 4, 3, epochs, 16) != full
    with pytest.raises(IndexError):
        one.records(one.steps)


def _shards(tmp_path, n_files=3, per_file=7, kd_classes=None, bad_logits_at=None):
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "golden"))
    import make_eval_preprocess_golden as mk
    Example = mk.example_class()
    rng = np.random.default_rng(1)
    for f in range(n_files):
        recs = []
        for i in range(per_file):
            h, w = int(rng.integers(8, 60)), int(rng.integers(8, 60))
            buf = io.BytesIO()
            Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(buf, format="JPEG", quality=90)
            ex = Example()
            ex.features.feature["image/encoded"].bytes_list.value.append(buf.getvalue())
            ex.features.feature["image/class/label"].int64_list.value.append(int(rng.integers(0, 10)))
            if kd_classes:
                k = kd_classes - 1 if (f, i) == bad_logits_at else kd_classes
                ex.features.feature["image/logit"].float_list.value.extend(
                    rng.standard_normal(k).astype(np.float32).tolist())
            data = ex.SerializeToString()
            head = len(data).to_bytes(8, "little")
            recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
        (tmp_path / ("train-%05d-of-%05d" % (f, n_files))).write_bytes(b"".join(recs))
    return tmp_path


def test_decode_window_is_worker_independent(tmp_path):
    from concurrent.futures import ThreadPoolExecutor
    from assembled_cnn_b200.imagenet_eval import decode_rgb, read_encoded
    from assembled_cnn_b200.imagenet_train import decode_window, read_train_records, train_files
    from oracle import train_preprocess as O
    root = _shards(tmp_path)
    records, counts = read_train_records(train_files(str(root)), 10)
    assert counts == [7, 7, 7] and len(records) == 21
    jobs = [(r[0], r[1], r[2], 5, 1, p) for p, r in enumerate(records)]
    outs = []
    for workers in (1, 4):
        with ThreadPoolExecutor(workers) as pool:
            outs.append([pool.submit(decode_window, *j) for j in jobs])
        outs[-1] = [f.result() for f in outs[-1]]
    for (a, fa), (b, fb), j in zip(outs[0], outs[1], jobs):
        assert fa == fb and np.array_equal(a, b) and a.flags["C_CONTIGUOUS"]
        img = decode_rgb(io.BytesIO(read_encoded(*j[:3])))
        y, x, ch, cw, flip = O.example(img.shape[0], img.shape[1], 5, 1, j[5])
        assert flip == fa and np.array_equal(a, img[y:y + ch, x:x + cw])


def test_kd_logits_parsing_and_errors(tmp_path):
    from assembled_cnn_b200.imagenet_eval import read_records
    from assembled_cnn_b200.imagenet_train import read_train_records, train_files
    root = _shards(tmp_path, n_files=1, per_file=4, kd_classes=10)
    path = train_files(str(root))[0]
    recs, _ = read_train_records([path], 10, kd=True)
    assert all(r[4].dtype == np.float32 and r[4].shape == (10,) for r in recs)
    # current callers see the three-field records
    assert [len(r) for r in read_records(path)] == [3] * 4
    assert [r[:3] for r in read_records(path, logits=True)] == read_records(path)
    with pytest.raises(ValueError, match="image/logit holds 10 values.*num_classes = 11"):
        read_train_records([path], 11, kd=True)
    with pytest.raises(ValueError, match="label .* outside \\[0, 3\\)"):
        read_train_records([path], 3)
    bad = tmp_path / "bad"
    bad.mkdir()
    _shards(bad, n_files=1, per_file=4, kd_classes=10, bad_logits_at=(0, 2))
    off = read_records(train_files(str(bad))[0])[2][1]
    with pytest.raises(ValueError, match="train-00000-of-00001: image/logit holds 9 values \\(image at byte "
                                         "offset %d\\)" % off):
        read_train_records(train_files(str(bad)), 10, kd=True)
    with pytest.raises(FileNotFoundError):
        train_files(str(tmp_path / "nothing"))


def test_float_list_packed_and_unpacked():
    from assembled_cnn_b200.imagenet_eval import parse_example
    import struct
    vals = np.float32([1.5, -2.25, 3e-8])

    def ld(field, payload):
        return bytes([(field << 3) | 2]) + bytes([len(payload)]) + payload

    def feature_entry(key, feature):
        return ld(1, ld(1, key) + ld(2, feature))

    packed = ld(2, ld(1, vals.tobytes()))
    unpacked = ld(2, b"".join(bytes([(1 << 3) | 5]) + struct.pack("<f", v) for v in vals))
    for fl in (packed, unpacked):
        feats = feature_entry(b"image/encoded", ld(1, ld(1, b"JPEG"))) \
            + feature_entry(b"image/class/label", ld(3, bytes([8, 4]))) + feature_entry(b"image/logit", fl)
        label, _, lg = parse_example(memoryview(ld(1, feats)), logits=True)
        assert label == 4 and np.array_equal(lg, vals)


def test_mixup_lambdas_are_a_function_of_seed_step_rank():
    from assembled_cnn_b200.imagenet_train import mixup_lambdas
    a = mixup_lambdas(1, 10, 0, 8)
    assert a.dtype == np.float32 and a.shape == (8,) and ((a >= 0) & (a <= 1)).all()
    assert np.array_equal(a, mixup_lambdas(1, 10, 0, 8)) and not np.array_equal(a, mixup_lambdas(1, 11, 0, 8))


def test_flag_errors_and_defaults(tmp_path):
    from assembled_cnn_b200.hparams import DEFAULTS
    from assembled_cnn_b200.model_fns import train_and_evaluate
    want = {"train_regex": "train-*", "training_random_crop": True, "autoaugment_type": None,
            "num_best_ckpt_to_keep": 3, "keep_ckpt_every_eval": True, "keep_checkpoint_max": 20,
            "eval_only": False, "save_checkpoints_epochs": 1.0, "ratio_fine_eval": 1.0,
            "pretrained_model_checkpoint_path": None}
    assert {k: DEFAULTS[k] for k in want} == want
    with pytest.raises(NotImplementedError, match="autoaugment_type"):
        train_and_evaluate(str(tmp_path), str(tmp_path / "m"), autoaugment_type="imagenet")
    with pytest.raises(NotImplementedError, match="reid / inception"):
        train_and_evaluate(str(tmp_path), str(tmp_path / "m"), preprocessing_type="reid")
    with pytest.raises(KeyError, match="unknown flag"):
        train_and_evaluate(str(tmp_path), str(tmp_path / "m"), no_such_flag=1)
    with pytest.raises(FileNotFoundError):              # the shards are read before any GPU work
        train_and_evaluate(str(tmp_path), str(tmp_path / "m"))


# ------------------------------------------------------------------------------------ native entry points
def test_argument_errors_without_gpu():
    """The host-side checks of the new entry points run before any CUDA call."""
    from assembled_cnn_b200 import _lib, native
    lib = _lib.load()
    INVALID = 1
    p = 1 << 20          # never dereferenced: the checks fail first

    def crop(desc=p, B=4, n_valid=4, S=224, mean=p, out=p):
        return lib.acnn_crop_resize_u8(desc, B, n_valid, S, mean, out, None)

    for kw in (dict(desc=None), dict(mean=None), dict(out=None), dict(B=0), dict(S=0), dict(S=-32),
               dict(n_valid=5), dict(n_valid=-1), dict(out=p + 2), dict(desc=p + 4), dict(S=1 << 16)):
        assert crop(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    nl = native.lib()
    assert nl.acnn_set_images_cropped(None, p, p, None) == INVALID


def test_crop_descriptor_check():
    from assembled_cnn_b200.imagenet_train import CROP_DESC_DTYPE, check_crop_descriptors
    d = np.zeros(3, CROP_DESC_DTYPE)
    d[:] = (1 << 20, 5, 7, 1, (0, 0, 0))
    check_crop_descriptors(d)
    for field, v in (("src", 0), ("h", 0), ("w", -1)):
        bad = d.copy()
        bad[1][field] = v
        with pytest.raises(ValueError, match="crop descriptor 1"):
            check_crop_descriptors(bad)


def test_new_kernel_in_sass():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from assembled_cnn_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "crop_resize_u8_kernel" in sass
