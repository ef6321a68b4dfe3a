"""Per-element tolerances for the op-level tests of the HBM-bound kernels (batch norm, SK, pooling,
head, optimizer: tests/test_stream_ops_cpu.py and tests/test_stream_ops_gpu.py).

TEST INFRASTRUCTURE ONLY.

Every bound is derived from the arithmetic the kernel does, not fitted to what it returns:

  * u = 2^-24, the unit roundoff of fp32.  An fp32 expression of k rounded operations (an FMA counts
    once) over exact inputs differs from its exact value by at most ~k * u * M, where M is the sum of
    the magnitudes of its terms (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed.,
    sec. 3.1); `elementwise_tol` takes k ("ops") and M ("mag").
  * A sum of terms added along chains of at most n_eff sequential fp32 additions -- the rows one
    thread adds one after another, then the sequential lanes of the kernel's fixed combination tree --
    differs from the exact sum by at most n_eff * u * sum|terms| (Higham eq. 4.4: gamma_(n-1) bounds
    recursive summation; a tree of chains is bounded by its longest chain).  `reduction_tol`.
  * A bf16 store adds at most half a bf16 ulp of the fp32 value; the tolerance allows one bf16 ulp
    of the reference (the fp32 value may sit across a binade boundary from the reference).

The references are computed in float64 from the kernel's own (bf16- or fp32-representable) inputs,
so every difference is the kernel's rounding -- or a bug.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |x| (8 significant bits), float64; the subnormal spacing at 0."""
    x = x.double().abs().clamp_min(2.0 ** -126)
    _, e = torch.frexp(x)              # x = m * 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int64))


def ulp_f32(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp32 numbers at |x| (24 significant bits), float64."""
    x = x.double().abs().clamp_min(2.0 ** -126)
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int64))


def elementwise_tol(ref, mag, bf16_out: bool, ops: int = 4):
    """|got - ref| bound of an fp32 expression of `ops` roundings over terms of total magnitude `mag`,
    stored as bf16 (one bf16 ulp on top, at the largest magnitude the fp32 value can have) or fp32."""
    t = ops * U32 * mag.double()
    return t + ulp_bf16(ref.double().abs() + t) if bf16_out else t


def reduction_tol(abs_sum, n_eff, extra_ops: int = 0):
    """|got - ref| bound of a sum whose longest sequential fp32 chain has n_eff additions, over terms
    of total magnitude abs_sum; `extra_ops` roundings of each term (e.g. g * xhat) add to the chain."""
    return (n_eff + extra_ops) * U32 * abs_sum.double()


def violations(got, ref, tol) -> torch.Tensor:
    """Boolean mask of the elements outside the tolerance (NaN counts as outside)."""
    d = (got.double() - ref.double()).abs()
    return ~(d <= tol.double())


def assert_within(got, ref, tol, what: str) -> None:
    bad = violations(got, ref, tol)
    if bool(bad.any()):
        idx = int(torch.nonzero(bad.flatten())[0])
        g, r, t = (float(v.flatten()[idx]) for v in (got.double(), ref.double(), tol.double()))
        raise AssertionError("%s: %d of %d elements outside the tolerance; first at flat index %d: "
                             "got %.9g, ref %.9g, |d| %.3g > tol %.3g"
                             % (what, int(bad.sum()), bad.numel(), idx, g, r, abs(g - r), t))


# ---------------------------------------------------------------------------------------------------
# Work decompositions the partial-row outputs follow (include/acnn.h: one partial row per CTA)
# ---------------------------------------------------------------------------------------------------
def bn_bwd_reduce_owner(M: int, C: int, nparts: int) -> torch.Tensor:
    """Partial row of every input row of acnn_bn_bwd_reduce / reduce2: CTA x starts at row x * RPB (RPB
    = 256 / (C / 8) rows per pass, one per thread of an 8-channel group) and strides by nparts * RPB, so
    row r belongs to CTA (r // RPB) % nparts."""
    rpb = 256 // (C // 8)
    return (torch.arange(M) // rpb) % nparts


def bn_bwd_reduce_chain(M: int, C: int, nparts: int) -> int:
    """Longest fp32 chain of one partial: rows per thread, then the RPB thread sums added in order."""
    rpb = 256 // (C // 8)
    return -(-M // (nparts * rpb)) + rpb


def row_slabs(B: int, HW: int, rpb: int, ctas_per_sm: int) -> int:
    """Row slabs per image of the SK kernels (csrc/bn_ops.cu row_slabs): about ctas_per_sm CTAs per SM
    of the H100's 132, at least one trip of 4 * rpb rows per slab."""
    s = (132 * ctas_per_sm + B - 1) // B
    max_s = (HW + 4 * rpb - 1) // (4 * rpb)
    return max(min(s, max_s), 1)


def sk_slabs(B: int, HW: int, f: int, ctas_per_sm: int):
    """(slabs, rows per slab, rows per trip) of sk_combine (ctas_per_sm 8: 2 rows of an f-wide thread
    layout per trip) and sk_bn_bwd_reduce / apply (2 resp. 8: 4 rows of a 2f-wide layout per trip) --
    both trips are 4096 / f rows."""
    rpb = 1024 // f
    s = row_slabs(B, HW, rpb, ctas_per_sm)
    return s, -(-HW // s), 4 * rpb


def slab_trips(HW: int, slabs: int, rows_per: int, rt: int):
    """Trips of every slab of an image (0 for a slab that starts past the last row)."""
    out = []
    for x in range(slabs):
        n = min(x * rows_per + rows_per, HW) - x * rows_per
        out.append(-(-n // rt) if n > 0 else 0)
    return out


def sk_slab_edges(B: int, HW: int, f: int, ctas_per_sm: int) -> set:
    """Which pipeline edges the SK slab kernels meet at (B, HW, f): 'empty' (a slab past the last row:
    zero trips, a zero partial row still written), 'wrap' (a slab with more trips than the 3 stages of
    the ring) and 'partial' (a slab whose last trip has fewer rows than a full one)."""
    s, rows_per, rt = sk_slabs(B, HW, f, ctas_per_sm)
    out = set()
    for x, t in enumerate(slab_trips(HW, s, rows_per, rt)):
        n = min(x * rows_per + rows_per, HW) - x * rows_per
        if t == 0:
            out.add("empty")
        if t > 3:
            out.add("wrap")
        if n > 0 and n % rt:
            out.add("partial")
    return out


# (B, HW, f) of the SK kernels' pipeline edges, the smallest (fewest elements of y) found by a search
# over f in {8, 64, 512, 1024}, B <= 64, HW < 400 for each edge of sk_slab_edges and each slab layout
# (8 and 2 CTAs per SM); plus (4, 49, 512), where the one-CTA-per-image reductions (sk_gap,
# sk_bwd_gate: trips of 2 * 256 / (f / 8) rows) wrap their ring with a partial last trip.
# tests/test_stream_ops_cpu.py checks that they still reach every edge.
SK_EDGE_SHAPES = [(1, 1, 8), (4, 49, 512), (6, 353, 512), (8, 397, 1024), (22, 385, 512), (32, 397, 1024)]


# ---------------------------------------------------------------------------------------------------
# float64 restatements of the pools with the kernels' explicit geometry (pad_lo before, the rest
# implied by the output size); tests/test_stream_ops_cpu.py pins them to oracle/tf_ops.py where that
# defines the same pool
# ---------------------------------------------------------------------------------------------------
def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def _pool_geom(H, k, s, pad_lo, Ho):
    return max((Ho - 1) * s + k - H - pad_lo, 0)


def avgpool_ref(x, k, s, pad_lo, Ho, Wo, count_pad):
    """float64 NHWC average pool with zero padding pad_lo before (and what Ho / Wo imply after),
    divided by k*k (count_pad) or by the number of in-bounds cells (TF 'SAME')."""
    B, H, W, C = x.shape
    ph, pw = _pool_geom(H, k, s, pad_lo, Ho), _pool_geom(W, k, s, pad_lo, Wo)
    xp = F.pad(x.permute(0, 3, 1, 2), (pad_lo, pw, pad_lo, ph))
    sm = F.avg_pool2d(xp, k, s)[:, :, :Ho, :Wo] * (k * k)
    if count_pad:
        return _nhwc(sm / (k * k))
    ones = F.pad(torch.ones(1, 1, H, W, dtype=x.dtype), (pad_lo, pw, pad_lo, ph))
    cnt = F.avg_pool2d(ones, k, s)[:, :, :Ho, :Wo] * (k * k)
    return _nhwc(sm / cnt)


def maxpool_ref(x, k, s, pad_lo, Ho, Wo, dout=None):
    """float64 max pool with -inf padding; the gradient goes to the FIRST maximum of every window (row-
    major), as torch.argmax picks it."""
    B, H, W, C = x.shape
    ph, pw = _pool_geom(H, k, s, pad_lo, Ho), _pool_geom(W, k, s, pad_lo, Wo)
    Hp, Wp = H + pad_lo + ph, W + pad_lo + pw
    xp = F.pad(x.permute(0, 3, 1, 2), (pad_lo, pw, pad_lo, ph), value=float("-inf"))
    cols = F.unfold(xp, k, stride=s).view(B, C, k * k, -1)
    L = cols.shape[-1]
    nh, nw = (Hp - k) // s + 1, (Wp - k) // s + 1
    mx, am = cols.max(2)
    out = _nhwc(mx.view(B, C, nh, nw)[:, :, :Ho, :Wo])
    if dout is None:
        return out
    d = torch.zeros(B, C, nh, nw, dtype=x.dtype)
    d[:, :, :Ho, :Wo] = dout.permute(0, 3, 1, 2)
    onehot = torch.zeros_like(cols).scatter_(2, am[:, :, None, :], d.view(B, C, 1, L))
    dxp = F.fold(onehot.view(B, C * k * k, L), (Hp, Wp), k, stride=s)
    return out, _nhwc(dxp[:, :, pad_lo:pad_lo + H, pad_lo:pad_lo + W])
