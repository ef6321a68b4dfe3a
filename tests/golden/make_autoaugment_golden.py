#!/usr/bin/env python
"""Golden data of AutoAugment, produced by EXECUTING the reference's preprocessing/autoaugment.py (by its AST)
from a checkout of the original project:

    python tests/golden/make_autoaugment_golden.py REFERENCE_DIR
        # rewrites autoaugment_golden.json

The module's functions run against a stand-in `tf` whose tensors are numpy arrays with TF's dtype rules
(a Python scalar operand becomes a tensor of the other operand's dtype, uint8 constants wrap as TF 1.14's
make_tensor_proto did) and whose primitives are numpy restatements of TF 1.14's kernels:
histogram_fixed_width (the double-precision bin formula), rgb_to_grayscale (convert_image_dtype x * (1/255),
tensordot left to right, trunc(g * 255.5)), depthwise_conv2d VALID (taps left to right, float32),
contrib.image.transform / rotate / translate (NEAREST, std::round, fill 0; rotate's cos / sin in float64
rounded to float32), bitwise shifts clamped to [0, 7], cast (truncation), clip_by_value, cond, where.
random_uniform returns scripted values and records its arguments.  The primitives' semantics are an
assumption stated here; what this file pins is the reference's composition: the tables, level-to-argument,
the blend special cases, the Contrast "mean", wrap / unwrap, the cutout geometry and the order of operations.

It records
  * the four policy tables (v0, imagenet, good, test);
  * the arguments each (operation, level) of the tables resolves to, with the sign draw forced both ways, and
    the number of sign draws it makes ("op/level/negated": [args, draws]);
  * the output of every sub-policy of every policy, apply draws forced both ways and signs both ways, on
    structured and random S x S images at S = 32 and 64 (images() and cases() below): the first 128 bits of
    the SHA-256 of the concatenated outputs per (S, policy, sub-policy);
  * the ranges of Cutout's centre draws.
tests/test_autoaugment_cpu.py checks the product and the oracle against this file; it does not need the
original project.
"""
import ast
import hashlib
import inspect
import json
import math
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "autoaugment_golden.json")
SRC = os.path.join("preprocessing", "autoaugment.py")
POLICY_FUNCS = {"v0": "policy_v0", "imagenet": "imagenet_policies", "good": "good_policies", "test": "policy_vtest"}
SIZES = (32, 64)
U_LO, U_HI = 0.0, 1.0 - 2.0 ** -24          # apply draws: applies iff prob == 1 / iff prob > 0
U_NEG, U_POS = 0.0, 0.75                     # sign draws: floor(u + 0.5) == 0 negates
f32 = np.float32


# ------------------------------------------------------------------------------------ stand-in tensors
class T:
    """A tensor: a numpy array of a fixed dtype."""
    def __init__(self, a, dtype=None):
        self.a = np.asarray(a, dtype=dtype)

    dtype = property(lambda self: self.a.dtype.type)

    def _other(self, o):
        if isinstance(o, T):
            assert o.a.dtype == self.a.dtype, (o.a.dtype, self.a.dtype)
            return o.a
        return const(o, self.a.dtype.type).a

    def __add__(self, o): return T(self.a + self._other(o))
    def __radd__(self, o): return T(self._other(o) + self.a)
    def __sub__(self, o): return T(self.a - self._other(o))
    def __rsub__(self, o): return T(self._other(o) - self.a)
    def __mul__(self, o): return T(self.a * self._other(o))
    def __rmul__(self, o): return T(self._other(o) * self.a)
    def __truediv__(self, o): return T(self.a / self._other(o))
    def __rtruediv__(self, o): return T(self._other(o) / self.a)
    def __floordiv__(self, o): return T(self.a // self._other(o))
    def __neg__(self): return T(-self.a)
    def __lt__(self, o): return T(self.a < self._other(o))
    def __gt__(self, o): return T(self.a > self._other(o))
    def __getitem__(self, k): return T(self.a[k])
    def __bool__(self): return bool(self.a)


def const(v, dtype=None):
    """convert_to_tensor: a Python value of `dtype` (uint8 wraps, as np.array(256, np.uint8) did in TF 1.14's
    days); without dtype, Python floats are float32 and ints int32."""
    if isinstance(v, T):
        return v
    if isinstance(v, (list, tuple)):
        parts = [const(x, dtype).a for x in v]
        return T(np.stack(parts) if parts else np.zeros(0, dtype or f32))
    if dtype is None:
        dtype = f32 if isinstance(v, float) else np.int32
    return T(np.array(int(v) if np.issubdtype(dtype, np.integer) else v).astype(dtype))


def _round_half_away(v):
    a = np.abs(v.astype(np.float64))
    return np.sign(v) * np.floor(a + 0.5)


def _transform(images, transforms):
    img = images.a
    H, W = img.shape[:2]
    t = [f32(x) for x in np.asarray(const(list(transforms), f32).a).reshape(-1)]
    y, x = np.meshgrid(np.arange(H, dtype=f32), np.arange(W, dtype=f32), indexing="ij")
    proj = (t[6] * x + t[7] * y) + f32(1)
    ix = _round_half_away(((t[0] * x + t[1] * y) + t[2]) / proj)
    iy = _round_half_away(((t[3] * x + t[4] * y) + t[5]) / proj)
    inside = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    out = np.zeros_like(img)
    out[inside] = img[iy[inside].astype(np.int64), ix[inside].astype(np.int64)]
    return T(out)


def _rotate(images, angles):
    H, W = images.a.shape[:2]
    ang = f32(np.asarray(const(angles, f32).a))
    c, s = f32(math.cos(float(ang))), f32(math.sin(float(ang)))
    h1, w1 = f32(H) - f32(1), f32(W) - f32(1)
    xo = (w1 - (c * w1 - s * h1)) / f32(2.0)
    yo = (h1 - (s * w1 + c * h1)) / f32(2.0)
    return _transform(images, [c, -s, xo, s, c, yo, f32(0), f32(0)])


def _translate(images, translations):
    dx, dy = [f32(v) for v in const(list(translations), f32).a]
    return _transform(images, [f32(1), f32(0), -dx, f32(0), f32(1), -dy, f32(0), f32(0)])


def _grayscale(images):
    x = images.a.astype(f32) * f32(1.0 / 255)
    g = x[..., 0] * f32(0.2989) + x[..., 1] * f32(0.5870)
    g = g + x[..., 2] * f32(0.1140)
    return T((g * f32(255.5)).astype(np.uint8)[..., None])


def _histogram(values, value_range, nbins):
    lo, hi = [float(v) for v in np.asarray(const(value_range).a)]
    step = (hi - lo) / float(nbins)
    idx = np.minimum((np.maximum(values.a, lo) - lo).astype(np.float64) / step, nbins - 1).astype(np.int32)
    return T(np.bincount(idx.reshape(-1), minlength=nbins).astype(np.int32))


def _depthwise(image, kernel, strides, padding, rate):
    assert padding == "VALID" and list(strides) == [1, 1, 1, 1]
    x, k = image.a, kernel.a
    kh, kw = k.shape[:2]
    H, W = x.shape[1] - kh + 1, x.shape[2] - kw + 1
    acc = np.zeros((1, max(H, 0), max(W, 0), x.shape[3]), f32)
    for i in range(kh):
        for j in range(kw):
            acc = acc + x[:, i:i + H, j:j + W, :] * k[i, j, :, 0]
    return T(acc)


def _shift(op):
    def f(x, y):
        s = np.clip(np.asarray(const(y, x.dtype).a).astype(np.int64), 0, 8 * x.a.itemsize - 1)
        return T(op(x.a, s.astype(x.a.dtype)).astype(x.a.dtype))
    return f


def stub_tf(draws, log):
    """`draws`: the scripted random_uniform values, in call order."""
    def random_uniform(shape, minval=0, maxval=None, dtype=f32, seed=None):
        log.append({"shape": list(shape), "minval": float(minval),
                    "maxval": None if maxval is None else float(const(maxval).a), "dtype": np.dtype(dtype).name})
        return T(np.array(draws.pop(0)).astype(dtype))

    def cond(pred, a, b):
        return const(a() if bool(const(pred).a) else b())

    def where(c, x=None, y=None):
        if x is None:
            return T(np.argwhere(c.a).astype(np.int64))
        x, y = const(x).a, const(y).a
        cond_ = c.a
        if cond_.ndim == 1 and x.ndim > 1:         # TF 1.x: a vector condition selects rows
            cond_ = cond_.reshape((-1,) + (1,) * (x.ndim - 1))
        return T(np.where(cond_, x, y))

    def cast(x, dtype):
        x = const(x)
        if dtype is bool:
            return T(x.a != 0)
        return T(x.a.astype(dtype))

    def pad(x, paddings, constant_values=0):
        p = [[int(const(v).a) for v in row] for row in paddings]
        return T(np.pad(const(x).a, p, constant_values=constant_values))

    image = types.SimpleNamespace(rgb_to_grayscale=_grayscale,
                                  grayscale_to_rgb=lambda g: T(np.repeat(g.a, 3, axis=-1)))
    contrib = types.SimpleNamespace(
        image=types.SimpleNamespace(transform=_transform, rotate=_rotate, translate=_translate),
        training=types.SimpleNamespace(HParams=lambda **kw: types.SimpleNamespace(**kw)))
    return types.SimpleNamespace(
        uint8=np.uint8, int32=np.int32, int64=np.int64, float32=f32, bool=bool,
        random_uniform=random_uniform, cond=cond, where=where, cast=cast, pad=pad, image=image, contrib=contrib,
        floor=lambda x: T(np.floor(const(x).a)), to_float=lambda x: T(const(x).a.astype(f32)),
        convert_to_tensor=lambda x: const(x), clip_by_value=lambda x, lo, hi: T(np.clip(x.a, *[
            const(v, x.dtype).a for v in (lo, hi)])),
        equal=lambda x, y: T(const(x).a == const(y, const(x).dtype).a),
        not_equal=lambda x, y: T(const(x).a != const(y, const(x).dtype).a),
        maximum=lambda x, y: T(np.maximum(const(x, const(y).dtype).a, const(y).a)),
        shape=lambda x: T(np.array(x.a.shape, np.int32)),
        ones=lambda shape, dtype: T(np.ones([int(const(s).a) for s in shape], dtype)),
        zeros=lambda shape, dtype=f32: T(np.zeros([int(const(s).a) for s in shape], dtype)),
        ones_like=lambda x, dtype=None: T(np.ones_like(x.a, dtype=dtype)),
        zeros_like=lambda x: T(np.zeros_like(x.a)),
        concat=lambda xs, axis: T(np.concatenate([np.atleast_1d(const(x, xs[-1].dtype if isinstance(xs[-1], T)
                                                                        else None).a) for x in xs], axis)),
        stack=lambda xs, axis: T(np.stack([x.a for x in xs], axis)),
        reshape=lambda x, shape: T(x.a.reshape([int(const(s).a) for s in const(shape).a.reshape(-1)])),
        slice=lambda x, begin, size: T(x.a[tuple(slice(int(b), int(b) + int(s)) for b, s in
                                                 zip(const(begin).a, const(size).a))]),
        expand_dims=lambda x, axis: T(np.expand_dims(x.a, axis)),
        squeeze=lambda x, axis: T(np.squeeze(x.a, tuple(axis))),
        tile=lambda x, m: T(np.tile(x.a, list(m))),
        constant=lambda v, dtype, shape: T(np.array(v, dtype).reshape(shape)),
        reduce_sum=lambda x: T(x.a.sum(dtype=x.a.dtype)), reduce_min=lambda x: T(x.a.min()),
        reduce_max=lambda x: T(x.a.max()), cumsum=lambda x: T(np.cumsum(x.a, dtype=x.a.dtype)),
        gather=lambda p, i: T(p.a[i.a]), histogram_fixed_width=_histogram,
        nn=types.SimpleNamespace(depthwise_conv2d=_depthwise),
        bitwise=types.SimpleNamespace(left_shift=_shift(np.left_shift), right_shift=_shift(np.right_shift)))


_CODE = {}


def load(ref_root, draws, log):
    if ref_root not in _CODE:
        tree = ast.parse(open(os.path.join(ref_root, SRC)).read())
        keep = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.Assign))]
        _CODE[ref_root] = compile(ast.Module(body=keep, type_ignores=[]), SRC, "exec")
    g = {"tf": stub_tf(draws, log), "math": math,
         "inspect": types.SimpleNamespace(getargspec=inspect.getfullargspec)}
    exec(_CODE[ref_root], g)
    return g


# ------------------------------------------------------------------------------------------ cases
# tests/test_autoaugment_cpu.py imports images() and cases() to rebuild the inputs the digests cover.
def images(S):
    """The S x S uint8 test images: random, constant, two-valued, one dominant bin, full range."""
    rng = np.random.default_rng(S)
    yy, xx = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    dominant = np.full((S, S, 3), 100, np.uint8)
    m = rng.random((S, S)) < 0.05
    dominant[m] = rng.integers(0, 256, (int(m.sum()), 3))
    full = np.stack([(yy * S + xx) * 255 // (S * S - 1), 255 - (xx * 255 // (S - 1)), (yy * 255 // (S - 1))], -1)
    return {"random": rng.integers(0, 256, (S, S, 3)).astype(np.uint8),
            "constant": np.full((S, S, 3), 77, np.uint8),
            "two_valued": np.where(((yy // 3 + xx // 5) % 2 == 0)[..., None], 30, 200).astype(np.uint8)
            .repeat(3, -1).reshape(S, S, 3),
            "dominant": dominant, "full_range": full.astype(np.uint8)}


def cases(S, policy, k, sub):
    """[(apply draws, negated, centres, image name)] of sub-policy k of `policy` at S, in digest order: the
    apply draws forced both ways per slot, the signs of signed operations both ways, Cutout centres drawn
    from a generator keyed by (S, policy, k)."""
    rng = np.random.default_rng([S, list(POLICY_FUNCS).index(policy), k])
    signed = [op in ("Rotate", "ShearX", "ShearY", "TranslateX", "TranslateY") for op, _, _ in sub]
    out = []
    for u in ((U_LO, U_LO), (U_LO, U_HI), (U_HI, U_LO), (U_HI, U_HI)):
        for neg in ((False, False), (True, False), (False, True), (True, True)):
            if any(n and not s for n, s in zip(neg, signed)):
                continue
            centres = [(int(rng.integers(0, S)), int(rng.integers(0, S))) for _ in range(2)]
            out += [(u, neg, centres, name) for name in sorted(images(S))]
    return out


def _plain(v):
    v = v.a if isinstance(v, T) else v
    if isinstance(v, np.ndarray):
        return _plain(v.item()) if v.ndim == 0 else [_plain(x) for x in v.tolist()]
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, (float, np.floating)):
        return float(v)
    if isinstance(v, (int, np.integer)):
        return int(v)
    return v


def reference_args(ref_root, name, level, negate):
    """(args, number of sign draws) of _parse_policy_info for operation `name` at `level`."""
    draws, log = [U_NEG if negate else U_POS] * 2, []
    g = load(ref_root, draws, log)
    hp = types.SimpleNamespace(cutout_max_pad_fraction=0.75, cutout_const=100, translate_const=250)
    func, prob, args = g["_parse_policy_info"](name, 0.5, level, [128, 128, 128], hp)
    assert func.__name__ == g["NAME_TO_FUNC"][name].__name__
    return [_plain(a) for a in args], len(log)


def run_subpolicy(ref_root, policy, k, img, u_apply, negated, centres):
    """distort_image_with_autoaugment(img, policy) with sub-policy k drawn and the given draws."""
    subs = load(ref_root, [], [])[POLICY_FUNCS[policy]]()
    draws = []
    for j, sub in enumerate(subs):             # build time: one sign draw per signed operation
        for s, (op, _, _) in enumerate(sub):
            if op in ("Rotate", "ShearX", "ShearY", "TranslateX", "TranslateY"):
                draws.append(U_NEG if (j == k and negated[s]) else U_POS)
    draws.append(k)
    for s, (op, prob, _) in enumerate(subs[k]):
        draws.append(u_apply[s])
        if op == "Cutout" and math.floor(f32(f32(u_apply[s]) + f32(prob))) != 0:
            draws += list(centres[s])
    log = []
    g = load(ref_root, draws, log)
    out = g["distort_image_with_autoaugment"](T(img), policy)
    assert not draws, draws
    return np.asarray(out.a, np.uint8), log


def main(ref_root):
    g = load(ref_root, [], [])
    tables = {p: [[[op, float(prob), int(level)] for op, prob, level in sub] for sub in g[f]()]
              for p, f in POLICY_FUNCS.items()}
    ops = sorted({(op, level) for subs in tables.values() for sub in subs for op, _, level in sub})
    args = {"%s/%d/%d" % (op, level, neg): reference_args(ref_root, op, level, neg)
            for op, level in ops for neg in (False, True)}
    digests, cutout_draws, n = {}, set(), 0
    for S in SIZES:
        imgs = images(S)
        for p, subs in tables.items():
            for k, sub in enumerate(subs):
                h = hashlib.sha256()
                for u, neg, centres, name in cases(S, p, k, sub):
                    out, log = run_subpolicy(ref_root, p, k, imgs[name], u, neg, centres)
                    h.update(out.tobytes())
                    n += 1
                    cutout_draws |= {(S, e["minval"], e["maxval"], e["dtype"]) for e in log
                                     if e["dtype"] == "int32" and e["maxval"] != len(subs)}
                digests["%d/%s/%d" % (S, p, k)] = h.hexdigest()[:32]
    json.dump({"policies": tables, "args": args, "digests": digests, "cases": n,
               "cutout_draws": sorted(list(c) for c in cutout_draws), "u": {"lo": U_LO, "hi": U_HI}},
              open(OUT, "w"), sort_keys=True, separators=(",", ":"))
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", n, "cases")


if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isfile(os.path.join(sys.argv[1], SRC)):
        sys.exit("usage: python tests/golden/make_autoaugment_golden.py REFERENCE_DIR\n"
                 "  REFERENCE_DIR: a checkout of clovaai/assembled-cnn (the directory holding preprocessing/)")
    main(os.path.abspath(sys.argv[1]))
