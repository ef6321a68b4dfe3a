"""Per-element checks of the 16-bit conv GEMMs (csrc/gemm.cu: fprop, dgrad, wgrad) against float64
references: tests/test_conv_plan_bf16_gpu.py and tests/test_conv_plan_fp16_gpu.py run them at the
training plans' geometries (the fp16 file also at fp16's overflow and subnormal edges) and
tests/test_conv_checks_cpu.py shows on synthetic data that they reject the errors they are meant to find.

TEST INFRASTRUCTURE ONLY.

The references are computed in float64 from the kernel's own 16-bit-representable operands, so every
difference is the kernel's rounding -- or a bug.  Every bound is derived from the arithmetic the kernel
does, not fitted to what it returns:

  * Accumulation.  An output element is a sum of K products of 16-bit operands (exact in fp32) added in
    fp32: wgmma chains and the register adds after them.  Each add rounds by at most 2u (u = 2^-24; the
    tensor cores' fp32 accumulation truncates instead of rounding to nearest), so the fp32 sum differs
    from the exact one by at most  acc = 2 K u mag,  mag = the same GEMM on |operands| (Higham, Accuracy
    and Stability of Numerical Algorithms, 2nd ed., sec. 3.1, with 2u per operation).  The add epilogue
    adds one more fp32 rounding of the sum, at most u (mag + acc + |add|).
  * Storage.  A 16-bit store rounds the fp32 value to nearest even: at most half a 16-bit ulp.  So
    |got - ref| <= acc + ulp(|ref| + acc) for every element (one full ulp: the fp32 value may sit
    across a binade boundary from the reference).
  * Exact rounding.  That per-element bound cannot tell round-to-nearest-even from truncation, nor a
    one-ulp systematic error from a correct result.  Call an element *decided* when every real number in
    [ref - acc, ref + acc] rounds to the same 16-bit value (the interval holds no rounding midpoint).
    The kernel's fp32 value lies in that interval, so a kernel that accumulates within acc and rounds to
    nearest even stores exactly round16(ref) there; the check requires it bit for bit on every decided
    element.  It cannot fail on a correct kernel, and it fails on truncation, on a one-ulp bias, on an
    add epilogue rounded twice (through 16 bits before the add) and on an fp32 add done in 16 bits.  How
    many elements are decided depends on the data: with K products of one sign per output element
    mag = |ref| and acc / |ref| = 2 K u, so at K = 4608 (3x3x512) about four in five bf16 outputs are.
    fp16's spacing is eight times finer: at that K next to none are (the per-element bound still holds
    every element), at the fp16 range edges of tests/test_conv_plan_fp16_gpu.py at least a third are.
  * fp16's range.  The store overflows as round to nearest even does: |fp32 value| >= 65520 is +-inf
    (the dynamic loss scale's overflow check reads those infs; a saturating store would hide them), and
    below 2^-14 it keeps fp16's subnormals (spacing 2^-24) instead of flushing them to zero.  An
    element whose interval lies beyond 65520 must be the inf of its sign; one whose interval crosses
    65520 may be the inf of that side or finite within the bound.
  * ReLU mask.  Wherever mask <= 0 (+0, -0 and negatives) the output is exactly 0, also where the
    value before the mask overflowed (a mask applied as a multiply gives inf x 0 = NaN there).
  * Batch-norm partial statistics.  Every CTA row stores its column sums and sums of squares of the
    stored 16-bit output in fp32.  Summed over the rows they are within n u sum|y| (sums) and 2 n u
    sum y^2 (squares: one more rounding per term) of the float64 sums of the stored output, n = rows of
    the output (the longest possible fp32 chain; Higham eq. 4.4).  A column whose stored output holds
    an inf sums to that inf (its squares to +inf).
  * Weight gradient.  dw (fp32) += sum over the P output pixels of x (*) dy.  Per element
    |got - ref| <= 2 P u mag_w + u (|dw0| + mag_w) (the P-term sum, then the add into the running dw0).
    At P = 200k - 3.2M that bound is loose: it grows with P where the actual rounding error grows with
    sqrt(P), and a missing pixel changes an element by one product in sqrt(P) of them.  So dw is also
    checked tile by tile: viewed as [Cout][kh kw Cin], every block of the wgrad GEMM's N tile of Cout
    (wgrad_bn) by its 128-row M tile of kh kw Cin must be within wgrad_tile_tol(n) norm-relative of the
    reference, n = the pixels one split sums in one chain (acnn_conv_wgrad_plan: all P in deterministic
    mode), so one wrong tile cannot hide in a whole-tensor norm.  That tolerance is 1e-3 up to n = 268k
    pixels and n u / 16 beyond: the tensor cores' fp32 accumulation truncates, so every update of the
    accumulator (one per 16-pixel wgmma k-step, n / 16 of them in one chain) moves the running sum toward
    zero by up to one ulp, and on random-sign operands that adds up to a shrink of dw that grows linearly
    with n, not with sqrt(n) (a random-walk partial sum |S_k| ~ sqrt(k) losing about u |S_k| per update:
    about (n / 16) u / 1.5 = n u / 24).  Measured on an H100 80GB HBM3 (700 W) at every wgrad geometry of
    the c3 / c5 plans at B = 256, 224 px (random-sign bf16 operands; worst tile over the geometries of one
    pixel count), default split-K / deterministic (one chain of all P pixels):
        P = 12544 (7 x 7):                 7.0e-6 / 1.4e-5
        P = 50176 (14 x 14):               1.9e-5 / 5.8e-5
        P = 200704 (28 x 28):              1.6e-5 / 2.3e-4
        P = 802816 (56 x 56):              3.6e-5 / 9.4e-4
        P = 3211264 (112 x 112, the stem): 1.4e-4 / 3.7e-3
    -- one chain of n pixels comes out about n u / 51 off, a third of the tolerance; the default split-K
    keeps every chain short and stays below 1.5e-4.  At P = 200k a tile without one pixel's contribution
    is 2.2e-3 off (tests/test_conv_checks_cpu.py).
"""
from __future__ import annotations

import torch

U32 = 2.0 ** -24

# significant bits, smallest normal exponent (2^emin), largest finite value of the 16-bit storage formats
FORMATS = {"bf16": (8, -126, (2.0 - 2.0 ** -7) * 2.0 ** 127), "fp16": (11, -14, 65504.0)}

# the NaN that the statistics rows are poisoned with before a launch (stats_poison): a stored row
# never holds this payload, while a sum over an inf and a -inf would be the default NaN
STATS_POISON_BITS = 0x7FC0DEAD

WGRAD_TILE_TOL = 1e-3


def ulp16(x: torch.Tensor, fmt: str = "bf16") -> torch.Tensor:
    """Spacing of the 16-bit format's numbers at |x|, float64 (the subnormal spacing below the
    smallest normal, the spacing of the largest binade at and beyond the largest finite value, inf
    included)."""
    p, emin, top = FORMATS[fmt]
    x = x.double().abs().clamp(2.0 ** emin, top)
    _, e = torch.frexp(x)              # x = m * 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(x), (e - p).to(torch.int64))


def round16(x: torch.Tensor, fmt: str = "bf16") -> torch.Tensor:
    """x (float64) rounded to the nearest 16-bit value, ties to even, computed in float64 (one
    rounding; torch's float64 -> bf16 conversion goes through fp32 and can round twice).  Beyond the
    largest finite value it overflows as round to nearest even does: fp16 |x| >= 65520 (half an ulp
    above 65504) is +-inf, 65504 < |x| < 65520 is +-65504 (bf16 alike at its own limit)."""
    x = x.double()
    q = ulp16(x, fmt)
    r = torch.round(x / q) * q         # x / q is exact (a power of two); torch.round: half to even
    top = FORMATS[fmt][2]
    return torch.where(r.abs() > top, torch.copysign(torch.full_like(r, float("inf")), x), r)


def acc_bound(mag: torch.Tensor, K: int) -> torch.Tensor:
    """Bound of the fp32 accumulation of K products against the exact sum: 2 K u mag."""
    return 2.0 * K * U32 * mag.double()


def add_epilogue_bound(acc: torch.Tensor, mag: torch.Tensor, add: torch.Tensor) -> torch.Tensor:
    """acc plus the fp32 rounding of (accumulated sum + add): u (mag + acc + |add|)."""
    return acc + U32 * (mag.double() + acc + add.double().abs())


def decided(ref: torch.Tensor, acc: torch.Tensor, fmt: str = "bf16") -> torch.Tensor:
    """Elements whose whole interval [ref - acc, ref + acc] rounds to one 16-bit value.  Rounding is
    monotone, so comparing the two ends decides it; the ends are widened by a relative 2^-40 for the
    float64 rounding of ref -+ acc."""
    lo, hi = _rounded_ends(ref, acc, fmt)
    return lo == hi


def _rounded_ends(ref, acc, fmt):
    ref, acc = ref.double(), acc.double()
    w = acc + ref.abs() * 2.0 ** -40
    return round16(ref - w, fmt), round16(ref + w, fmt)


def _first_bad(bad, got, ref):
    idx = int(torch.nonzero(bad.flatten())[0])
    return "first at flat index %d: got %.9g, ref %.9g" % (idx, float(got.flatten()[idx]), float(ref.flatten()[idx]))


def check_16bit(got: torch.Tensor, ref: torch.Tensor, acc: torch.Tensor, what: str,
                fmt: str = "bf16") -> float:
    """The per-element bound and the exact-rounding check of a 16-bit output; returns the decided
    fraction.  got: the kernel's 16-bit output, ref / acc: float64, same shape.

    Overflow (fp16): an element whose whole interval [ref - acc, ref + acc] rounds to +-inf must be
    that inf (not the saturated 65504); one whose interval reaches half an ulp beyond the largest
    finite value on one side only may be that inf or, within the bound, finite; every finite element
    is under the bound, so an inf anywhere else fails."""
    g = got.double()
    ref, acc = ref.double(), acc.double()
    lo, hi = _rounded_ends(ref, acc, fmt)
    over = (lo == hi) & torch.isinf(lo)
    bad = over & (g != lo)
    if bool(bad.any()):
        raise AssertionError("%s: %d of %d elements that overflow are not the inf of their sign; %s" % (
            what, int(bad.sum()), int(over.sum()), _first_bad(bad, g, ref)))
    # the straddling elements that stored the inf of the side whose end overflows
    inf_ok = ~over & torch.isinf(g) & ((torch.isinf(lo) & (g == lo)) | (torch.isinf(hi) & (g == hi)))
    tol = acc + ulp16(ref.abs() + acc, fmt)
    bad = ~over & ~inf_ok & ~((g - ref).abs() <= tol)
    if bool(bad.any()):
        raise AssertionError("%s: %d of %d elements outside acc + ulp; %s" % (
            what, int(bad.sum()), bad.numel(), _first_bad(bad, g, ref)))
    dec = lo == hi
    wrong = dec & (g != lo)
    if bool(wrong.any()):
        raise AssertionError("%s: %d of %d decided elements are not round-to-nearest-even of the "
                             "reference; %s" % (what, int(wrong.sum()), int(dec.sum()),
                                                _first_bad(wrong, g, ref)))
    return float(dec.double().mean())


def check_mask(got: torch.Tensor, mask: torch.Tensor, what: str) -> None:
    """Exactly 0 (+0 or -0) wherever mask <= 0 (+0, -0 and negatives), whatever the value before the
    mask was: a mask applied as a multiply leaves NaN where that value overflowed to inf."""
    off = ~(mask > 0)
    bad = off & (got != 0)
    if bool(bad.any()):
        raise AssertionError("%s: %d of %d masked elements are not 0; %s" % (
            what, int(bad.sum()), int(off.sum()), _first_bad(bad, got.double(), torch.zeros_like(got.double()))))


def stats_poison(shape, device="cuda") -> torch.Tensor:
    """fp32 statistics rows filled with the STATS_POISON_BITS NaN, for check_stats."""
    return torch.full(shape, STATS_POISON_BITS, dtype=torch.int32, device=device).view(torch.float32)


def check_stats(rows: torch.Tensor, y: torch.Tensor, what: str) -> None:
    """rows [parts][2][C] (fp32, poisoned with stats_poison before the launch): every row stored (no
    element keeps the poison payload), and the row sums within n u sum|y| / 2 n u sum y^2 of the
    float64 column sums of the stored output y [..., C].  A column whose stored output holds an inf
    (fp16 overflow; one sign per column) must total exactly that inf, its squares +inf."""
    C = rows.shape[-1]
    left = (rows.contiguous().view(torch.int32) == STATS_POISON_BITS).flatten(1).any(1)
    if bool(left.any()):
        raise AssertionError("%s: %d of %d statistics rows not stored (poison left)" % (
            what, int(left.sum()), rows.shape[0]))
    yd = y.double().reshape(-1, C)
    n = yd.shape[0]
    pos, neg = (yd == float("inf")).any(0), (yd == -float("inf")).any(0)
    if bool((pos & neg).any()):
        raise AssertionError("%s: columns with both +inf and -inf outputs (the check needs one overflow "
                             "sign per column)" % what)
    inf_col = pos | neg
    s, q = rows.double().sum(0)
    want = torch.where(pos, float("inf"), -float("inf"))
    for got, ref, name in ((s, want, "column sums"), (q, torch.full_like(q, float("inf")), "column sums of squares")):
        bad = inf_col & (got != ref)
        if bool(bad.any()):
            raise AssertionError("%s %s: %d of %d columns with an inf output do not total that inf; %s" % (
                what, name, int(bad.sum()), int(inf_col.sum()), _first_bad(bad, got, ref)))
    yf = torch.where(inf_col, torch.zeros_like(yd), yd)
    for got, ref, tol, name in ((s, yf.sum(0), n * U32 * yf.abs().sum(0), "column sums"),
                                (q, (yf * yf).sum(0), 2 * n * U32 * (yf * yf).sum(0), "column sums of squares")):
        bad = ~inf_col & ~((got - ref).abs() <= tol + 1e-30)
        if bool(bad.any()):
            raise AssertionError("%s %s: %d of %d channels outside the bound; %s" % (
                what, name, int(bad.sum()), C, _first_bad(bad, got, ref)))


def wgrad_bn(Cout: int) -> int:
    """N tile (output channels) of the wgrad GEMM (csrc/gemm.cu wgrad tiling, bf16 / fp16 operands)."""
    return 256 if Cout >= 256 else 128 if Cout >= 128 else 64 if Cout >= 64 else 32


def wgrad_tile_errors(got: torch.Tensor, ref: torch.Tensor, bm: int = 128, bn: int | None = None) -> torch.Tensor:
    """Norm-relative error of every bn x bm block of dw viewed as [Cout][kh kw Cin] (the wgrad GEMM's
    N tile x M tile; ragged last blocks included), float64 [Cout blocks][row blocks]."""
    Cout = got.shape[0]
    bn = bn or wgrad_bn(Cout)
    d = (got.double() - ref.double()).reshape(Cout, -1)
    r = ref.double().reshape(Cout, -1)
    Kr = r.shape[1]
    pn, pk = -Cout % bn, -Kr % bm

    def blocks(t):
        t = torch.nn.functional.pad(t, (0, pk, 0, pn))
        return t.reshape(t.shape[0] // bn, bn, t.shape[1] // bm, bm).pow(2).sum((1, 3)).sqrt()
    return blocks(d) / blocks(r).clamp_min(1e-300)


def wgrad_tile_tol(chain: int) -> float:
    """Norm-relative tolerance of a tile of dw whose splits each sum `chain` pixels in one chain: 1e-3,
    or the truncating accumulation's shrink bound chain u / 16 where that is larger (chain > 268k)."""
    return max(WGRAD_TILE_TOL, chain * U32 / 16)


def check_wgrad(got: torch.Tensor, ref: torch.Tensor, mag: torch.Tensor, dw0: torch.Tensor, P: int,
                what: str, chain: int | None = None) -> float:
    """The per-element bound and the tile-local norm check of an fp32 weight gradient accumulated into
    dw0 over P pixels, in splits of at most `chain` pixels (default P: one split); returns the worst
    tile's norm-relative error."""
    g, ref, mag = got.double(), ref.double(), mag.double()
    tol = 2.0 * P * U32 * mag + U32 * (dw0.double().abs() + mag)
    bad = ~((g - ref).abs() <= tol + 1e-30)
    if bool(bad.any()):
        raise AssertionError("%s: %d of %d elements outside 2 P u mag; %s" % (
            what, int(bad.sum()), bad.numel(), _first_bad(bad, g, ref)))
    # the tiles of the gradient's own sum (dw0 is common to both sides)
    e = wgrad_tile_errors(g - dw0.double(), ref - dw0.double())
    worst = float(e.max())
    tile_tol = wgrad_tile_tol(min(P, chain or P))
    if not worst < tile_tol:
        i = int(torch.argmax(e.flatten()))
        raise AssertionError("%s: tile (%d, %d) of %s has norm-relative error %.3e >= %.3e" % (
            what, i // e.shape[1], i % e.shape[1], tuple(e.shape), worst, tile_tol))
    return worst


# ---------------------------------------------------------------------------------------------------
# The conv GEMM launches of a training plan
# ---------------------------------------------------------------------------------------------------
class ConvCase(tuple):
    """One distinct conv GEMM launch of a plan: (kind, geom, stats, add, mask, bias, out_f32, x_wpad,
    src).  geom is the plan's 12-tuple (B, H, W, Cin, Cout, kh, kw, stride, pads); x_wpad the stem's
    W padding of its space-to-depth input (None elsewhere); src, for a dgrad on a zero-inserted
    gradient, the strided forward geometry whose data gradient it computes (None elsewhere)."""
    __slots__ = ()
    _fields = ("kind", "geom", "stats", "add", "mask", "bias", "out_f32", "x_wpad", "src")

    def __new__(cls, *a):
        return tuple.__new__(cls, a)

    def __getattr__(self, k):
        return self[self._fields.index(k)]

    def id(self):
        s = "%s-%s" % (self.kind, "x".join(map(str, self.geom)))
        for f in ("stats", "add", "mask", "bias", "out_f32"):
            if getattr(self, f):
                s += "-" + f
        if self.x_wpad:
            s += "-wpad%d%d" % tuple(self.x_wpad)
        if self.src:
            s += "-zi_s%d" % self.src[7]
        return s


def plan_cases(plans) -> list:
    """Distinct conv / conv_dgrad / conv_wgrad launches of the given plans, sorted."""
    seen = set()
    for plan in plans:
        wgrad_geom = {}                   # dy -> the (strided) geometry of the conv it belongs to
        zi_src = {}                       # zero-inserted dy -> that geometry
        for op in plan.all_ops():
            a = op.a
            if op.kind == "conv_wgrad":
                wgrad_geom[a["dy"]] = tuple(op.geom.astuple())
            if op.kind == "zero_insert":
                zi_src[a["out"]] = wgrad_geom[a["dy"]]
            if op.kind not in ("conv", "conv_dgrad", "conv_wgrad"):
                continue
            wp = a.get("x_wpad")
            seen.add(ConvCase(op.kind, tuple(op.geom.astuple()), a.get("stats") is not None,
                              a.get("add_src") is not None, a.get("mask_src") is not None,
                              a.get("bias") is not None, bool(a.get("out_f32")),
                              tuple(wp) if wp is not None else None,
                              zi_src.get(a["dy"]) if op.kind == "conv_dgrad" else None))
    return sorted(seen, key=lambda c: (c.kind, c.geom, c.id()))


def launch_geom(geom, x_wpad=None):
    """The acnn_conv_geom the library launches for a plan geometry (csrc/model_exec.cu geom()): with
    x_wpad the W-padded space-to-depth stem input, read as W pixels of kw * Cin channels that overlap
    (x_pix_stride = Cin)."""
    from assembled_cnn_b200._lib import ConvGeom
    if x_wpad is None:
        return ConvGeom(*geom)
    B, H, W, Cin, Cout, kh, kw, stride, phl, phh, _, _ = geom
    lo, hi = x_wpad
    row = (W + lo + hi) * Cin
    return ConvGeom(B, H, W, Cin * kw, Cout, kh, 1, 1, phl, phh, 0, 0, Cin, row, H * row, 0)
