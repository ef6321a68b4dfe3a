"""CPU checks of AutoAugment: the product's policy tables and resolved arguments, and the oracle's outputs,
against tests/golden/autoaugment_golden.json (the reference's autoaugment.py executed against a numpy
stand-in for tf); the oracle's Equalize / Posterize / Solarize / Invert against PIL's ImageOps; host cos / sin
against libm; the draws; the descriptor check; the argument errors of the C entries without a GPU."""
import ctypes
import ctypes.util
import hashlib
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "golden", "autoaugment_golden.json")) as f:
        return json.load(f)


def _maker():
    sys.path.insert(0, os.path.join(ROOT, "golden"))
    import make_autoaugment_golden
    return make_autoaugment_golden


def _applies(u, prob):
    return bool(np.floor(f32(f32(u) + f32(prob))) != 0)


def test_tables_match_reference(golden):
    from assembled_cnn_b200 import autoaugment as A
    assert set(golden["policies"]) == set(A.POLICIES)
    for name, subs in golden["policies"].items():
        assert [[list(op) for op in sub] for sub in A.policy(name)] == subs, name
    with pytest.raises(ValueError, match="Invalid augmentation_name: v9"):
        A.policy("v9")


def test_resolved_arguments_match_reference(golden):
    from assembled_cnn_b200 import autoaugment as A
    S = 224
    seen = set()
    for key, (args, sign_draws) in golden["args"].items():
        op, level, neg = key.split("/")
        level, neg = int(level), neg == "1"
        r = A.op_record(op, level, S, negate=neg, centre=(3, 4))
        assert r["op"] == A.OP_CODE[op]
        assert sign_draws == (1 if op in A.SIGNED else 0)
        a = args[0] if args else None
        if op in A.SIGNED:
            assert a == float(-f32(A.level_to_arg(op, level)) if neg else f32(A.level_to_arg(op, level)))
        else:
            assert a == A.level_to_arg(op, level) or (a is None and not args), (op, level, a)
        if op == "Posterize":
            assert r["i"][0] == min(max(8 - a, 0), 7)
        elif op == "Solarize":
            assert r["i"][0] == int(np.array(a).astype(np.uint8))
        elif op == "SolarizeAdd":
            assert r["i"][0] == a
        elif op in A.BLENDS:
            assert r["f"][0] == f32(a)
        elif op == "Rotate":
            assert list(r["f"]) == A.rotate_transform(f32(a), S)
        elif op in ("ShearX", "ShearY"):
            assert list(r["f"]) == ([1, a, 0, 0, 1, 0] if op == "ShearX" else [1, 0, 0, a, 1, 0])
        elif op in ("TranslateX", "TranslateY"):           # translate([-pixels, 0]): t2 = -dx
            assert list(r["f"]) == ([1, 0, a, 0, 1, 0] if op == "TranslateX" else [1, 0, 0, 0, 1, a])
        elif op == "Cutout":
            assert list(r["i"]) == [3, 4, a]
        seen.add((op, level))
    # every (operation, level) of the four tables is covered, and v0's two corners resolve as documented
    assert seen == {(op, lv) for subs in A.POLICIES.values() for sub in subs for op, _, lv in sub}
    assert A.op_record("Posterize", 2, S)["i"][0] == 7                     # bits 0: shift 8 clamped to 7
    assert A.op_record("Solarize", 10, S)["i"][0] == 0                     # threshold 256 as uint8
    assert A.op_record("Contrast", 8, 224)["i"][0] == 196 and A.op_record("Contrast", 8, 256)["i"][0] == 255
    assert A.op_record("Color", 5, S)["f"][0] == 1.0


def test_oracle_matches_reference_outputs(golden):
    """One digest per (S, policy, sub-policy) over the outputs of its cases, which the generator's images()
    and cases() rebuild."""
    from oracle import autoaugment as O
    M = _maker()
    n = 0
    for key, want in golden["digests"].items():
        S, policy, k = key.split("/")
        S, k = int(S), int(k)
        sub = golden["policies"][policy][k]
        imgs = M.images(S)
        h = hashlib.sha256()
        for u, neg, centres, name in M.cases(S, policy, k, sub):
            applied = [_applies(x, prob) for x, (_, prob, _) in zip(u, sub)]
            h.update(O.augment(imgs[name], sub, applied, neg, centres).tobytes())
            n += 1
        assert h.hexdigest()[:32] == want, key
    assert n == golden["cases"] > 5000
    assert len(golden["digests"]) == 2 * sum(len(s) for s in golden["policies"].values())
    # Cutout's centre is drawn as a uniform int32 in [0, S)
    assert golden["cutout_draws"] == [[S, 0.0, float(S), "int32"] for S in (32, 64)]


def test_apply_rule_matches_reference(golden):
    from assembled_cnn_b200 import autoaugment as A
    for u in golden["u"].values():
        for prob in [i / 10 for i in range(11)]:
            assert A.applies(f32(u), prob) == _applies(u, prob), (u, prob)
    assert A.applies(f32(1 - 2 ** -24), 1.0)                 # u + 1.0 rounds to 2.0: still applies
    assert not A.applies(f32(1 - 2 ** -24), 0.0) and A.applies(f32(0), 1.0) and not A.applies(f32(0), 0.9)


def test_oracle_against_pil():
    from PIL import Image, ImageOps
    from oracle import autoaugment as O
    rng = np.random.default_rng(0)
    for k in range(20):
        h, w = int(rng.integers(1, 70)), int(rng.integers(1, 70))
        a = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
        if k % 3 == 1:
            a = (a // 37 * 37).astype(np.uint8)          # few bins
        if k % 5 == 2:
            a[:] = a[0, 0]                               # one bin per channel
        im = Image.fromarray(a)
        assert np.array_equal(O.equalize(a), np.asarray(ImageOps.equalize(im)))
        assert np.array_equal(O.apply_op(a, "Invert", 0), np.asarray(ImageOps.invert(im)))
        for level in (3, 5, 6, 7, 8):                    # bits >= 1
            bits = int(level / 10 * 4)
            assert np.array_equal(O.apply_op(a, "Posterize", level), np.asarray(ImageOps.posterize(im, bits)))
        for level in range(10):                          # thresholds below 256
            t = int(level / 10 * 256)
            assert np.array_equal(O.apply_op(a, "Solarize", level), np.asarray(ImageOps.solarize(im, t)))


def test_host_cos_sin_equal_libm():
    from assembled_cnn_b200 import autoaugment as A
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    for fn in (libm.cosf, libm.sinf):
        fn.restype, fn.argtypes = ctypes.c_float, [ctypes.c_float]
    levels = sorted({lv for subs in A.POLICIES.values() for sub in subs for op, _, lv in sub if op == "Rotate"})
    assert levels == [0, 2, 3, 5, 7, 8, 9]
    for lv in levels:
        for neg in (False, True):
            deg = f32(A.level_to_arg("Rotate", lv))
            deg = -deg if neg else deg
            rad = f32(deg * f32(math.pi / 180.0))
            t = A.rotate_transform(deg, 224)
            assert t[0] == f32(libm.cosf(rad)) and t[3] == f32(libm.sinf(rad)), (lv, neg)


def test_draws_depend_only_on_rng():
    from assembled_cnn_b200 import autoaugment as A
    np.random.seed(1)
    state = np.random.get_state()[1].copy()
    for name in ("v0", "imagenet", "good", "test"):
        a = [A.resolve(name, 224, np.random.default_rng([7, i])) for i in range(200)]
        b = [A.resolve(name, 224, np.random.default_rng([7, i])) for i in range(200)]
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        A.check_autoaugment_descriptors(np.array(a, A.AUTOAUG_DESC_DTYPE), 224)
        ks = {int(x["subpolicy"]) for x in a}
        assert ks <= set(range(len(A.policy(name)))) and len(ks) > min(10, len(A.policy(name)) - 1)
        assert any(x["slot"][0]["op"] == 0 for x in a) or name == "test"
    assert np.array_equal(np.random.get_state()[1], state)          # the global numpy stream is untouched
    # the draw order: sub-policy index, then per slot the apply draw and the sign draw / the centre
    rng = np.random.default_rng(3)
    d = A.resolve("good", 64, rng)
    rng = np.random.default_rng(3)
    k = int(rng.integers(0, 95))
    assert d["subpolicy"] == k
    for j, (op, prob, level) in enumerate(A.policy("good")[k]):
        app = A.applies(A.uniform(rng), prob)
        neg = op in A.SIGNED and np.floor(f32(A.uniform(rng) + f32(0.5))) == 0
        cen = (int(rng.integers(0, 64)), int(rng.integers(0, 64))) if op == "Cutout" else (0, 0)
        want = A.op_record(op, level, 64, neg, cen) if app else np.zeros((), A.AUTOAUG_OP_DTYPE)
        assert d["slot"][j].tobytes() == want.tobytes()


def test_descriptor_check():
    from assembled_cnn_b200 import autoaugment as A
    good = np.array([A.subpolicy_record("good", k, 32, (True, True), (True, False), ((31, 0), (0, 31)))
                     for k in range(95)], A.AUTOAUG_DESC_DTYPE)
    A.check_autoaugment_descriptors(good, 32)
    for field, v, op in (("op", 17, 0), ("op", -1, 0), ("i", (8, 0, 0), 5), ("i", (256, 0, 0), 6),
                         ("f", (np.nan,) + (0,) * 5, 8), ("f", (-0.5,) + (0,) * 5, 10), ("i", (300, 0, 0), 9),
                         ("f", (np.inf,) + (0,) * 5, 4), ("i", (32, 0, 10), 16), ("i", (0, -1, 10), 16)):
        bad = np.zeros(3, A.AUTOAUG_DESC_DTYPE)
        bad[1]["slot"][1]["op"] = op
        bad[1]["slot"][1][field] = v
        with pytest.raises(ValueError, match="autoaugment descriptor 1 slot 1"):
            A.check_autoaugment_descriptors(bad, 32)


def test_argument_errors_without_gpu():
    from assembled_cnn_b200 import _lib, native
    lib = _lib.load()
    INVALID = 1
    p = 1 << 20          # never dereferenced: the checks fail first

    def aug(desc=p, a=p, B=4, n_valid=4, S=224, mean=p, work=p, out=p):
        return lib.acnn_crop_resize_autoaugment_u8(desc, a, B, n_valid, S, mean, work, out, None)

    for kw in (dict(desc=None), dict(a=None), dict(mean=None), dict(work=None), dict(out=None), dict(B=0),
               dict(S=0), dict(S=-32), dict(n_valid=5), dict(n_valid=-1), dict(out=p + 2), dict(desc=p + 4),
               dict(a=p + 4), dict(work=p + 8), dict(S=1 << 15)):
        assert aug(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    assert lib.acnn_autoaugment_work_bytes(512, 224) == 512 * 2 * 150528
    assert lib.acnn_autoaugment_work_bytes(3, 33) == 3 * 2 * 3280          # 33 * 33 * 3 = 3267 -> 3280
    for B, S in ((0, 224), (4, 0), (-1, 5), (4, 1 << 15)):
        assert lib.acnn_autoaugment_work_bytes(B, S) == -1
    nl = native.lib()
    assert nl.acnn_set_images_augmented(None, p, p, p, p, None) == INVALID


def test_new_kernel_in_sass():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from assembled_cnn_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "crop_resize_autoaugment_kernel" in sass
