"""Layer plan of the assembled-ResNet hot path: a static list of kernel launches over named buffers.

The reference builds a TF graph once and then runs `session.run(train_op)` per step
; here the "graph" is this plan -- forward, backward and SGD ops in execution order over
statically shaped NHWC bf16 buffers -- built once by walking the same topology as
nets/resnet_model.py:305-599 / functions/model_fns.py:98-198, and executed by runtime.py through
the C ABI (optionally captured into one CUDA graph).

Backward is emitted explicitly (the reference relies on tf.gradients): each forward module pushes
a closure on a tape; closures run in reverse.  A tensor read by several ops accumulates its
gradient through the consumers' fused epilogues (`add_src`), and the LAST contribution also applies
the ReLU mask of the tensor (`mask_src`), so a gradient buffer always holds dL/d(pre-ReLU).

Parameters are enumerated in the reference's variable creation order with TF-style names
; the flat fp32 master buffer stores conv kernels as OHWI ([Cout][kh][kw][Cin]).
"""
from __future__ import annotations

import os
import math
from collections import OrderedDict
from dataclasses import dataclass, field

BLOCK_SIZES = {   # functions/model_fns.py:113-127
    1: {50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3], 200: [3, 24, 36, 3]},
    2: {50: [3, 4, 6, 3], 101: [4, 8, 18, 3], 152: [5, 12, 30, 3]},
}
ALIGN = 256   # every tensor of a flat buffer starts at a multiple of 256 elements
def _sk_job_floats(M, N, K, share):
    tiles = -(-M // 64) * -(-N // 64)
    s = max(1, min(share // tiles, K // 32, 8))
    kper = -(-(-(-K // s)) // 16) * 16
    return -(-K // kper) * M * N


def sk_fc_scratch_floats(B, f, d, G=132):
    """Mirror of acnn_sk_fc_scratch_floats (csrc/small_fc.cu; tests/test_abi_cpu.py compares them):
    da [B,2f] + dz [B,d] + the K-split partial tiles of the widest phase of the fused SK chains."""
    fwd = max(_sk_job_floats(B, d, f, G), _sk_job_floats(B, 2 * f, d, G))
    bwd = max(_sk_job_floats(2 * f, d, B, G // 2) + _sk_job_floats(B, d, 2 * f, G // 2),
              _sk_job_floats(d, f, B, G // 2) + _sk_job_floats(B, f, d, G // 2))
    return B * (2 * f + d) + max(fwd, bwd)


# capacities (rows) of the per-CTA partial-sum buffers the reductions write (include/acnn.h:
# acnn_conv_stats_parts / acnn_bn_bwd_reduce_parts / acnn_sk_bn_bwd_reduce_parts give the real counts)
# (the H100 SXM's 132 SMs: csrc/common.h kMaxSms)
STATS_PARTS_CAP = 132
BWD_PARTS_CAP = 2 * 132
SGD_SCRATCH = 132 * 8 + 1


def _round_up(n, a=ALIGN):
    return (n + a - 1) // a * a


@dataclass
class Tensor:
    name: str
    shape: tuple
    dtype: str = "bf16"
    relu: bool = False          # output of a ReLU: its gradient gets masked by (t > 0)
    consumers: int = 0          # forward readers that will send a gradient back
    contribs: int = 0
    grad: str | None = None     # name of the buffer holding the accumulated gradient so far


@dataclass
class Param:
    name: str            # TF-style variable name
    tf_shape: tuple      # shape in the reference's layout (HWIO kernels, [in,out] dense)
    kind: str            # conv_kernel | dense_kernel | dense_bias | gamma | beta | moving_mean | moving_variance
    offset: int          # element offset in the flat buffer it lives in ("params" or "state")
    size: int            # elements actually used
    store_shape: tuple   # shape as stored (OHWI for kernels; padded for dense)
    trainable: bool = True
    decay: bool = False  # weight decay applies (run_loop_classification.py:166-177)
    zero_init: bool = False
    dgrad_off: int = -1  # offset in the bf16 dgrad-layout buffer, -1 if never needed


@dataclass
class Slot:
    """A small fp32 vector inside one of the flat work buffers."""
    buf: str     # "zero" (cleared every step) or "work"
    offset: int
    size: int


@dataclass
class Geom:
    B: int
    H: int
    W: int
    Cin: int
    Cout: int
    kh: int
    kw: int
    stride: int
    pad_h_lo: int
    pad_h_hi: int
    pad_w_lo: int
    pad_w_hi: int

    @property
    def Ho(self):
        return (self.H + self.pad_h_lo + self.pad_h_hi - self.kh) // self.stride + 1

    @property
    def Wo(self):
        return (self.W + self.pad_w_lo + self.pad_w_hi - self.kw) // self.stride + 1

    def astuple(self):
        return (self.B, self.H, self.W, self.Cin, self.Cout, self.kh, self.kw, self.stride,
                self.pad_h_lo, self.pad_h_hi, self.pad_w_lo, self.pad_w_hi)


@dataclass
class Op:
    kind: str
    a: dict = field(default_factory=dict)

    def __getattr__(self, k):
        try:
            return self.__dict__["a"][k]
        except KeyError:
            raise AttributeError(k)


@dataclass
class BN:
    """A batch-norm layer instance: parameters + per-step work slots."""
    C: int
    gamma: str
    beta: str
    mm: str
    mv: str
    count: int
    stats: Slot | None      # bf16 mode: [parts][sum | sumsq] partial rows written by the conv
                            # epilogue; fp32 mode: [mean | var] from bn_stats (training only)
    work: Slot              # [scale | shift | mean | rstd]


@dataclass
class ConvOut:
    x: Tensor
    y: Tensor
    geom: Geom
    w: str                 # param name
    bn: BN | None
    stem: dict | None = None   # space-to-depth stem bookkeeping


@dataclass
class ModelConfig:
    """Constructor flags of functions/model_fns.py:141-157 + call-time use_resnet_d."""
    resnet_size: int = 50
    num_classes: int = 1001
    resnet_version: int = 1
    no_downsample: bool = False
    zero_gamma: bool = False
    use_se_block: bool = False
    use_sk_block: bool = False
    bn_momentum: float = 0.997
    embedding_size: int = 0
    anti_alias_filter_size: int = 0
    anti_alias_type: str = ""
    pool_type: str = "gap"
    loss_type: str = "softmax"
    bl_alpha: int = 2
    bl_beta: int = 4
    use_resnet_d: bool = False

    def validate(self):
        if self.resnet_version not in (1, 2):
            raise ValueError("Resnet version should be 1 or 2. See README for citations.")
        if self.resnet_size < 50:
            raise NotImplementedError("non-bottleneck ResNets (nets/resnet_model.py:211-212)")
        if self.resnet_size not in BLOCK_SIZES[self.resnet_version]:
            raise ValueError("Could not find layers for selected Resnet size.\nSize received: {}; "
                             "sizes allowed: {}.".format(
                                 self.resnet_size, BLOCK_SIZES[self.resnet_version].keys()))
        if self.pool_type not in ("gap", "gem", "flatten"):
            raise NotImplementedError("pool_type=%r (nets/resnet_model.py:560-573)" % self.pool_type)
        e = self.embedding_size
        if e and (e < 32 or e > 2048 or e & (e - 1)):
            raise ValueError("embedding_size must be a power of two between 32 and 2048 (tensor-core N tile, "
                             "channel groups of the batch-norm kernels)")
        if self.loss_type != "softmax":
            raise NotImplementedError("only the softmax loss is on the hot path")
        if self.anti_alias_type and self.anti_alias_filter_size not in range(1, 8):
            raise ValueError("anti_alias_filter_size must be in 1..7")
        if self.resnet_version == 2 and (self.bl_alpha < 1 or self.bl_beta < 1 or (64 // self.bl_alpha) % 32):
            raise NotImplementedError("bl_alpha=%r: the little branches would have %d channels, below the "
                                      "32-channel tensor-core tile (bl_alpha 1 or 2)"
                                      % (self.bl_alpha, 64 // max(self.bl_alpha, 1)))


class Plan:
    """Result of PlanBuilder: buffers, parameters and the op lists."""

    def __init__(self):
        self.tensors: "OrderedDict[str, Tensor]" = OrderedDict()
        self.params: "OrderedDict[str, Param]" = OrderedDict()      # trainables, creation order
        self.state: "OrderedDict[str, Param]" = OrderedDict()       # moving statistics
        self.param_elems = 0
        self.state_elems = 0
        self.dgrad_elems = 0
        self.zero_elems = 0
        self.work_elems = 0
        self.forward: list[Op] = []
        self.backward: list[Op] = []
        self.update: list[Op] = []
        self.bns: list[BN] = []
        self.meta = {}

    def all_ops(self):
        return self.forward + self.backward + self.update

    def python_mirror(self):
        return self

    _GRAD_WRITERS = ("conv_wgrad", "sk_fc_bwd", "se_fc_bwd", "s2d_wgrad_unpack")

    def grad_done_at(self):
        """name -> index of the backward op after which that variable's gradient is final (the
        data-parallel schedule of dp.py; acnn_variable_info.grad_ready_op of the native plan)."""
        done_at = {}
        for i, op in enumerate(self.backward):
            a = op.a
            if op.kind in self._GRAD_WRITERS:
                for key in ("w", "w1", "w2"):
                    if isinstance(a.get(key), str) and a[key] in self.params:
                        done_at[a[key]] = i
            if op.kind in ("bn_bwd_finalize", "sk_fc_bwd") and a.get("bn") is not None:
                for n in (a["bn"].gamma, a["bn"].beta):
                    if n in self.params:
                        done_at[n] = i
        return done_at


class PlanBuilder:
    def __init__(self, cfg: ModelConfig, batch: int, height: int = 224, width: int = 224, *,
                 training: bool = True, mixup_type: int = 0, label_smoothing: float = 0.0,
                 with_loss: bool = True, dtype: str = "bf16", use_dropblock: bool = False,
                 kd_temp: float = 0.0):
        cfg.validate()
        # DropBlock (nets/blocks.py:187-251) is active in training only; its keep probability is a
        # device scalar (hp[4]) because it follows a schedule (functions/model_fns.py:221-228)
        self.use_dropblock = bool(use_dropblock) and training
        if self.use_dropblock and cfg.use_se_block:
            raise NotImplementedError("use_dropblock together with use_se_block")
        self.kd_temp = float(kd_temp) if training else 0.0
        # backward of the two batch norms of a projection block's output in one pass each
        # (bn_backward2; ACNN_FUSE_BN_PAIRS=0 keeps the separate kernels for A/B runs)
        self.fuse_bn_pairs = os.environ.get("ACNN_FUSE_BN_PAIRS", "1") == "1"
        self._identity_bns = {}
        if dtype not in ("bf16", "fp32"):
            raise ValueError("dtype must be one of: ('bf16', 'fp32')")
        # fp32 = the reference's default dtype (nets/resnet_model.py:30-33): fp32 activation storage,
        # conv GEMMs on 3-way bf16-split operands, deterministic reductions -- the parity mode
        self.fp32 = dtype == "fp32"
        self.adt = "f32" if self.fp32 else "bf16"
        self._planes = {}
        if height % 32 or width % 32:
            raise ValueError("input size must be a multiple of 32 (got %dx%d)" % (height, width))
        if mixup_type not in (0, 1, 2):
            raise ValueError("mixup_type must be 0, 1 or 2")
        self.cfg = cfg
        self.B = batch
        self.training = training
        self.mixup_type = mixup_type if training else 0
        self.with_loss = with_loss or training
        self.plan = Plan()
        self.tape = []
        self._scope = ["resnet_model"]
        self._counters = {}
        self._tid = 0
        self.ops = self.plan.forward
        p = self.plan
        p.meta.update(batch=batch, height=height, width=width, training=training,
                      mixup_type=self.mixup_type, label_smoothing=label_smoothing,
                      num_classes=cfg.num_classes, ld_logits=_round_up(cfg.num_classes, 128),
                      bn_momentum=cfg.bn_momentum, dtype=dtype, use_dropblock=self.use_dropblock,
                      kd_temp=self.kd_temp, dropblock_u=[], ones=[],
                      input_batch=batch * 2 if self.mixup_type == 1 else batch)
        self._build(height, width)

    # ---------------------------------------------------------------- naming (TF-1.x style)
    def _unique(self, base):
        key = ("/".join(self._scope), base)
        n = self._counters.get(key, 0)
        self._counters[key] = n + 1
        return base if n == 0 else "%s_%d" % (base, n)

    class _Scope:
        def __init__(self, b, name):
            self.b, self.name = b, name

        def __enter__(self):
            self.b._scope.append(self.b._unique(self.name))

        def __exit__(self, *a):
            self.b._scope.pop()

    def scope(self, name):
        return PlanBuilder._Scope(self, name)

    def _full(self, name):
        return "/".join(self._scope + [name])

    # ---------------------------------------------------------------- allocation helpers
    def tensor(self, base, shape, dtype=None, relu=False):
        dtype = dtype or self.adt
        self._tid += 1
        name = "%s#%d" % (base, self._tid)
        t = Tensor(name, tuple(shape), dtype, relu)
        self.plan.tensors[name] = t
        return t

    def _param(self, name, tf_shape, kind, store_shape, *, trainable=True, decay=False,
               zero_init=False, need_dgrad=False):
        p = self.plan
        size = 1
        for s in store_shape:
            size *= s
        if trainable:
            par = Param(name, tuple(tf_shape), kind, p.param_elems, size, tuple(store_shape), True,
                        decay, zero_init)
            p.param_elems += _round_up(size)
            if need_dgrad:
                par.dgrad_off = p.dgrad_elems
                p.dgrad_elems += _round_up(size)
            assert name not in p.params, name
            p.params[name] = par
        else:
            par = Param(name, tuple(tf_shape), kind, p.state_elems, size, tuple(store_shape), False)
            p.state_elems += _round_up(size)
            p.state[name] = par
        return par

    def slot(self, buf, size):
        p = self.plan
        if buf == "zero":
            s = Slot("zero", p.zero_elems, size)
            p.zero_elems += _round_up(size, 32)
        else:
            s = Slot("work", p.work_elems, size)
            p.work_elems += _round_up(size, 32)
        return s

    def emit(self, kind, **a):
        self.ops.append(Op(kind, a))

    def planes(self, name):
        """fp32 mode: the (hi, mid, lo) bf16 operand planes of a GEMM operand tensor, split once
        (op `split3`) right before its first consumer and reused by later ones (fprop + wgrad)."""
        if not self.fp32:
            return None
        pl = self._planes.get(name)
        if pl is None:
            t = self.plan.tensors[name]
            n = 1
            for d in t.shape:
                n *= d
            pt = self.tensor("planes", (3,) + tuple(t.shape), "bf16")
            self.emit("split3", src=name, dst=pt.name, n=n)
            self._planes[name] = pl = pt.name
        return pl

    # ---------------------------------------------------------------- gradient accumulation
    def use(self, t: Tensor):
        t.consumers += 1
        return t

    def contribute(self, t: Tensor, emit_fn):
        """emit_fn(out_name, add_src, mask_src) must emit one op writing the new running sum."""
        t.contribs += 1
        last = t.contribs == t.consumers
        assert t.contribs <= t.consumers, t.name
        out = self.tensor("d_" + t.name.split("#")[0], t.shape)
        emit_fn(out.name, t.grad, t.name if (last and t.relu) else None)
        t.grad = out.name

    def contribute_alias(self, t: Tensor, buf: str):
        """The gradient flowing into t is an existing buffer (identity shortcut)."""
        t.contribs += 1
        last = t.contribs == t.consumers
        if t.grad is None and not (last and t.relu):
            t.grad = buf
            return
        out = self.tensor("d_" + t.name.split("#")[0], t.shape)
        self.emit("grad_combine", a=buf, add_src=t.grad, mask_src=t.name if (last and t.relu) else None,
                  out=out.name, shape=t.shape)
        t.grad = out.name

    def grad_of(self, t: Tensor) -> str:
        assert t.contribs == t.consumers and t.grad is not None, \
            "gradient of %s incomplete (%d/%d)" % (t.name, t.contribs, t.consumers)
        return t.grad

    # ---------------------------------------------------------------- layers
    def _geom(self, x: Tensor, cout, k, stride):
        B, H, W, C = x.shape
        lo = (k - 1) // 2
        hi = k - 1 - lo
        return Geom(B, H, W, C, cout, k, k, stride, lo, hi, lo, hi)

    def bn_layer(self, C, count, zero_gamma=False, layer=None):
        layer = layer or self._unique("batch_normalization")
        g = self._param(self._full(layer + "/gamma"), (C,), "gamma", (C,), zero_init=zero_gamma)
        b = self._param(self._full(layer + "/beta"), (C,), "beta", (C,))
        mm = self._param(self._full(layer + "/moving_mean"), (C,), "moving_mean", (C,), trainable=False)
        mv = self._param(self._full(layer + "/moving_variance"), (C,), "moving_variance", (C,),
                         trainable=False)
        stats = None
        if self.training:
            stats = self.slot("work", 2 * C if self.fp32 else STATS_PARTS_CAP * 2 * C)
        bn = BN(C, g.name, b.name, mm.name, mv.name, count, stats, self.slot("work", 4 * C))
        self.plan.bns.append(bn)
        return bn

    def conv(self, x: Tensor, filters, k, stride, *, with_bn=True, zero_gamma=False,
             need_dgrad=True) -> ConvOut:
        """conv2d_fixed_padding (+ the batch-norm that always follows it in the reference)."""
        B, H, W, Cin = x.shape
        if filters % 32 or Cin % 16:
            # e.g. bl_alpha=4: the little branches would have 16 channels
            raise NotImplementedError("conv %d -> %d channels: the tensor-core tiles need input channels in "
                                      "multiples of 16 and output channels in multiples of 32" % (Cin, filters))
        layer = self._unique("conv2d")
        g = self._geom(x, filters, k, stride)
        w = self._param(self._full(layer + "/kernel"), (k, k, Cin, filters), "conv_kernel",
                        (filters, k, k, Cin), decay=True, need_dgrad=need_dgrad and self.training)
        y = self.tensor("y", (B, g.Ho, g.Wo, filters))
        bn = self.bn_layer(filters, B * g.Ho * g.Wo, zero_gamma) if with_bn else None
        self.emit("conv", x=x.name, xp=self.planes(x.name), w=w.name, y=y.name, geom=g,
                  stats=bn.stats if (bn and self.training and not self.fp32) else None, bias=None,
                  out_f32=False)
        if bn:
            self.emit_bn_finalize(bn, y, g)
        if need_dgrad:
            self.use(x)
        return ConvOut(x, y, g, w.name, bn)

    def emit_bn_finalize(self, bn: BN, y: Tensor, geom: Geom, x_wpad=None):
        """Batch statistics -> scale / shift / mean / rstd (+ moving statistics).  bf16 mode: the
        conv epilogue left partial (sum, sumsq) rows (stats_mode 0); fp32 mode: a separate two-pass
        kernel computes mean / variance of the fp32 conv output (stats_mode 1)."""
        mode = 0
        if self.training and self.fp32:
            self.emit("bn_stats", x=y.name, bn=bn, M=bn.count, C=bn.C)
            mode = 1
        self.emit("bn_finalize", bn=bn, stats_mode=mode, geom=geom, x_wpad=x_wpad)

    @staticmethod
    def stem_s2d_taps(k):
        """k x k stride-2 conv with padding (k-1)//2 == k2 x k2 stride-1 conv on the
        space-to-depth(2) image with padding (lo2, hi2): input offset u - p = 2*r + a."""
        p = (k - 1) // 2
        rmin = math.floor(-p / 2)
        rmax = math.floor((k - 1 - p) / 2)
        return p, rmax - rmin + 1, -rmin, rmax

    def stem_conv(self, x0: Tensor, filters, k) -> ConvOut:
        """First conv (k x k, stride 2, 3 input channels) run as a stride-1 conv on the
        space-to-depth(2) input that pack_input produced."""
        B, H2, Wp, C16 = x0.shape
        layer = self._unique("conv2d")
        p, k2, lo2, hi2 = self.stem_s2d_taps(k)
        W2 = Wp - lo2 - hi2
        w = self._param(self._full(layer + "/kernel"), (k, k, 3, filters), "conv_kernel",
                        (filters, k, k, 3), decay=True)
        g = Geom(B, H2, W2, 16, filters, k2, k2, 1, lo2, hi2, lo2, hi2)
        assert g.Ho == H2 and g.Wo == W2
        y = self.tensor("y", (B, H2, W2, filters))
        bn = self.bn_layer(filters, B * H2 * W2)
        stem = dict(k=k, pad=p, k2=k2, pad2=lo2, w2=self.tensor("w_stem", (filters, k2, k2, 16)),
                    dw2=self.slot("zero", filters * k2 * k2 * 16) if self.training else None)
        self.emit("s2d_weight_pack", w=w.name, w2=stem["w2"].name, cout=filters, **{
            "k": k, "pad": p, "k2": k2, "pad2": lo2})
        stem["x_wpad"] = (lo2, hi2)
        self.emit("conv", x=x0.name, xp=self.planes(x0.name), w=stem["w2"].name,
                  wp=self.planes(stem["w2"].name), y=y.name, geom=g,
                  stats=bn.stats if (self.training and not self.fp32) else None, bias=None,
                  out_f32=False, w_is_tensor=True, x_wpad=(lo2, hi2),
                  alg_macs=B * H2 * W2 * filters * k * k * 3)   # the k x k x 3 conv, not its
        # zero-padded k2 x k2 x 16 space-to-depth form (bench.py's roofline counts algorithmic work)
        stem["alg_macs"] = B * H2 * W2 * filters * k * k * 3
        self.emit_bn_finalize(bn, y, g, (lo2, hi2))
        return ConvOut(x0, y, g, w.name, bn, stem)

    def bn_act(self, co: ConvOut, *, relu, b=None, b_mode=0, gate=None, name="u") -> Tensor:
        """b: ConvOut (b_mode 1) or Tensor (b_mode 2 identity / 3 upsample)."""
        out = self.tensor(name, co.y.shape, relu=relu)
        self.emit("bn_act", a=co.y.name, bn_a=co.bn,
                  b=(b.y.name if b_mode == 1 else (b.name if b is not None else None)),
                  bn_b=(b.bn if b_mode == 1 else None), b_mode=b_mode, gate=gate, relu=relu,
                  out=out.name, shape=co.y.shape)
        return out

    # -- DropBlock -----------------------------------------------------------------------------
    def identity_bn(self, C):
        """scale = 1, shift = 0: lets bn_act consume an already-normalised tensor."""
        bn = self._identity_bns.get(C)
        if bn is None:
            work = self.slot("work", 4 * C)
            self.plan.meta["ones"].append((work.offset, C))        # runtime presets scale = 1
            bn = self._identity_bns[C] = BN(C, None, None, None, None, 0, None, work)
        return bn

    def dropblock_mask(self, H, W, C, gamma_scale, block_size=7):
        """One DropBlock call of the reference = one mask [H,W,C] shared by the batch + its
        renormalisation factor (op `dropblock_mask`, forward list)."""
        if H < block_size or W < block_size:
            raise ValueError("dropblock: feature map %dx%d smaller than block_size %d (the reference "
                             "fails the same way: nets/blocks.py:222-229)" % (H, W, block_size))
        hs, ws = H - block_size + 1, W - block_size + 1
        u = self.tensor("dropblock_u", (hs, ws, C), "f32")
        index = len(self.plan.meta["dropblock_u"])
        self.plan.meta["dropblock_u"].append(u.name)
        m = dict(keep=self.slot("work", H * W * C), scale=self.slot("work", 1),
                 scratch=self.slot("work", hs * ws * C + (H * W * C + 255) // 256),
                 H=H, W=W, C=C, gamma_scale=gamma_scale, block_size=block_size, u=u.name,
                 index=index)
        self.emit("dropblock_mask", **m)
        return m

    def dropblock_apply(self, x: Tensor, m, relu, name="db") -> Tensor:
        """out = relu?(x * keep * scale); registers the backward (same kernel, no relu)."""
        B, H, W, C = x.shape
        out = self.tensor(name, x.shape, relu=relu)
        self.emit("dropblock_apply", x=x.name, keep=m["keep"], scale=m["scale"], relu=relu,
                  out=out.name, B=B, HW=H * W, C=C)
        return out

    def dropblock_bwd(self, g: str, m, shape) -> str:
        B, H, W, C = shape
        dt = self.tensor("d_db", shape)
        self.emit("dropblock_apply", x=g, keep=m["keep"], scale=m["scale"], relu=False,
                  out=dt.name, B=B, HW=H * W, C=C)
        return dt.name

    def cbr_db(self, x: Tensor, filters, k, stride, gamma_scale) -> Tensor:
        """conv -> BN -> dropblock -> ReLU (nets/resnet_model.py:49-56,65-72)."""
        co = self.conv(x, filters, k, stride)
        t = self.bn_act(co, relu=False, name="t")
        m = self.dropblock_mask(t.shape[1], t.shape[2], t.shape[3], gamma_scale)
        u = self.dropblock_apply(t, m, relu=True, name="u")
        self.tape.append(lambda: self.conv_backward(co, self.bn_backward(
            co, self.dropblock_bwd(self.grad_of(u), m, t.shape))))
        return u

    # -- backward helpers ----------------------------------------------------------------------
    def bn_backward(self, co: ConvOut, g: str, gate=None, addbc=None) -> str:
        bn, y = co.bn, co.y
        sums = self.slot("work", BWD_PARTS_CAP * 2 * bn.C)   # per-CTA partial rows
        coef = self.slot("work", 3 * bn.C)
        dy = self.tensor("dy", y.shape)
        self.emit("bn_bwd_reduce", g=g, y=y.name, bn=bn, gate=gate, addbc=addbc, sums=sums,
                  shape=y.shape)
        self.emit("bn_bwd_finalize", bn=bn, sums=sums, coef=coef)
        self.emit("bn_bwd_apply", g=g, y=y.name, coef=coef, gate=gate, addbc=addbc, dy=dy.name,
                  shape=y.shape)
        return dy.name

    def bn_backward2(self, co_a: ConvOut, co_b: ConvOut, g: str):
        """Backward of the two batch norms summed into one residual output (block-final BN and
        projection-shortcut BN, same gradient g, same shape): g is read once per pass instead of
        twice (ops bn_bwd_reduce2 / bn_bwd_apply2; bit-identical to two bn_backward calls)."""
        assert co_a.y.shape == co_b.y.shape
        outs = []
        for co in (co_a, co_b):
            outs.append((self.slot("work", BWD_PARTS_CAP * 2 * co.bn.C), self.slot("work", 3 * co.bn.C),
                         self.tensor("dy", co.y.shape)))
        (sa, ca, da), (sb, cb, db) = outs
        self.emit("bn_bwd_reduce2", g=g, y=co_a.y.name, bn=co_a.bn, sums=sa, y2=co_b.y.name,
                  bn2=co_b.bn, sums2=sb, shape=co_a.y.shape)
        self.emit("bn_bwd_finalize", bn=co_a.bn, sums=sa, coef=ca)
        self.emit("bn_bwd_finalize", bn=co_b.bn, sums=sb, coef=cb)
        self.emit("bn_bwd_apply2", g=g, y=co_a.y.name, coef=ca, dy=da.name, y2=co_b.y.name, coef2=cb,
                  dy2=db.name, shape=co_a.y.shape)
        return da.name, db.name

    def conv_backward(self, co: ConvOut, dy: str, need_dgrad=True):
        g = co.geom
        dyp = self.planes(dy)
        if co.stem is not None:
            self.emit("conv_wgrad", x=co.x.name, xp=self.planes(co.x.name), dy=dy, dyp=dyp, geom=g,
                      dw_slot=co.stem["dw2"], x_wpad=co.stem["x_wpad"],
                      alg_macs=co.stem["alg_macs"])
            self.emit("s2d_wgrad_unpack", dw2=co.stem["dw2"], w=co.w, cout=g.Cout, k=co.stem["k"],
                      pad=co.stem["pad"], k2=co.stem["k2"], pad2=co.stem["pad2"])
            return
        self.emit("conv_wgrad", x=co.x.name, xp=self.planes(co.x.name), dy=dy, dyp=dyp, geom=g,
                  w=co.w)
        if not need_dgrad:
            return
        if g.stride == 1:
            self.contribute(co.x, lambda out, add, mask: self.emit_dgrad(
                dy, co.w, out, g, add, mask))
        else:
            assert g.stride == 2
            dyz = self.tensor("dyz", (g.B, g.H, g.W, g.Cout))
            self.emit("zero_insert", dy=dy, out=dyz.name, B=g.B, Ho=g.Ho, Wo=g.Wo, H=g.H, W=g.W,
                      C=g.Cout)
            g1 = Geom(g.B, g.H, g.W, g.Cin, g.Cout, g.kh, g.kw, 1, g.pad_h_lo,
                      g.kh - 1 - g.pad_h_lo, g.pad_w_lo, g.kw - 1 - g.pad_w_lo)
            # executed on the zero-inserted dy (4x the MACs of the stride-2 transposed conv)
            alg = g.B * g.Ho * g.Wo * g.Cout * g.kh * g.kw * g.Cin
            self.contribute(co.x, lambda out, add, mask: self.emit_dgrad(
                dyz.name, co.w, out, g1, add, mask, alg_macs=alg))

    def emit_dgrad(self, dy, w, out, g, add, mask, alg_macs=None):
        """dx = conv_transpose(dy) (+ add_src) (* relu mask).  bf16 mode fuses the accumulate / mask
        into the GEMM epilogue; fp32 mode (fp32 output straight from the accumulators) runs them as one extra
        elementwise pass."""
        if self.fp32 and (add is not None or mask is not None):
            shape = self.plan.tensors[out].shape
            tmp = self.tensor("dx_raw", shape)
            self.emit("conv_dgrad", dy=dy, dyp=self.planes(dy), w=w, dx=tmp.name, geom=g,
                      add_src=None, mask_src=None, alg_macs=alg_macs)
            self.emit("grad_combine", a=tmp.name, add_src=add, mask_src=mask, out=out, shape=shape)
        else:
            self.emit("conv_dgrad", dy=dy, dyp=self.planes(dy), w=w, dx=out, geom=g, add_src=add,
                      mask_src=mask, alg_macs=alg_macs)

    # -- composite modules -----------------------------------------------------------------------
    def cbr(self, x: Tensor, filters, k, stride, need_dgrad=True) -> Tensor:
        """conv -> BN -> ReLU."""
        co = self.conv(x, filters, k, stride, need_dgrad=need_dgrad)
        u = self.bn_act(co, relu=True)
        self.tape.append(lambda: self.conv_backward(co, self.bn_backward(co, self.grad_of(u)),
                                                    need_dgrad))
        return u

    def stem_cbr(self, x0: Tensor, filters, k) -> Tensor:
        co = self.stem_conv(x0, filters, k)
        u = self.bn_act(co, relu=True)
        self.tape.append(lambda: self.conv_backward(co, self.bn_backward(co, self.grad_of(u))))
        return u

    def sk(self, t: Tensor, filters, stride) -> Tensor:
        """nets/blocks.py:110-154."""
        B = t.shape[0]
        co = self.conv(t, 2 * filters, 3, stride)
        H, W = co.y.shape[1:3]
        f, d = filters, max(int(filters / 2), 32)
        with self.scope("sk_block"):
            w1 = self._param(self._full("sk_fc_1/kernel"), (1, 1, f, d), "conv_kernel", (d, 1, 1, f),
                             decay=True)
            bnz = self.bn_layer(d, B, layer="batch_normalization")
            w2 = self._param(self._full("sk_fc_2/kernel"), (1, 1, d, 2 * f), "conv_kernel",
                             (2 * f, 1, 1, d), decay=True)
        s = self.slot("work", B * f)
        zpre = self.slot("work", B * d)
        z = self.slot("work", B * d)
        att = self.slot("work", B * f)
        scratch = self.slot("work", sk_fc_scratch_floats(B, f, d))
        v = self.tensor("v", (B, H, W, f))
        dims = dict(B=B, HW=H * W, f=f, d=d)
        self.emit("sk_gap", y=co.y.name, bn=co.bn, s=s, **dims)
        self.emit("sk_fc", s=s, w1=w1.name, bn=bnz, w2=w2.name, zpre=zpre, z=z, att=att,
                  scratch=scratch, **dims)
        self.emit("sk_combine", y=co.y.name, bn=co.bn, att=att, v=v.name, **dims)

        def bwd():
            gv = self.grad_of(v)
            dA = self.slot("work", B * f)
            ds = self.slot("work", B * f)
            sums = self.slot("work", (BWD_PARTS_CAP + B) * 4 * f)   # per-CTA partial rows
            coef = self.slot("work", 6 * f)
            dy = self.tensor("dy", co.y.shape)
            self.emit("sk_bwd_gate", dv=gv, y=co.y.name, bn=co.bn, dA=dA, **dims)
            self.emit("sk_fc_bwd", dA=dA, att=att, z=z, zpre=zpre, bn=bnz, s=s, w1=w1.name,
                      w2=w2.name, ds=ds, scratch=scratch, **dims)
            self.emit("sk_bn_bwd_reduce", dv=gv, y=co.y.name, bn=co.bn, att=att, ds=ds, sums=sums,
                      **dims)
            self.emit("bn_bwd_finalize", bn=co.bn, sums=sums, coef=coef)
            self.emit("sk_bn_bwd_apply", dv=gv, y=co.y.name, bn=co.bn, att=att, ds=ds, coef=coef,
                      dy=dy.name, **dims)
            self.conv_backward(co, dy.name)
        self.tape.append(bwd)
        return v

    def blurpool(self, x: Tensor, filt, stride) -> Tensor:
        B, H, W, C = x.shape
        pad = (filt - 1) // 2
        if pad >= H or pad >= W:
            raise ValueError("anti-alias filter %d on a %dx%d feature map: REFLECT padding of %d needs a larger "
                             "map (tf.pad fails the same way, nets/blocks.py:70-75)" % (filt, H, W, pad))
        Ho, Wo = (H + 2 * pad - filt) // stride + 1, (W + 2 * pad - filt) // stride + 1
        out = self.tensor("blur", (B, Ho, Wo, C))
        a = dict(B=B, H=H, W=W, C=C, filt=filt, stride=stride)
        self.emit("blurpool", x=x.name, out=out.name, **a)
        self.use(x)
        self.tape.append(lambda: self.contribute(x, lambda o, add, mask: self.emit(
            "blurpool_bwd", dout=self.grad_of(out), dx=o, add_src=add, mask_src=mask, **a)))
        return out

    def avgpool(self, x: Tensor, k, stride, pad_lo, Ho, Wo, count_pad) -> Tensor:
        B, H, W, C = x.shape
        out = self.tensor("avgp", (B, Ho, Wo, C))
        a = dict(B=B, H=H, W=W, C=C, k=k, stride=stride, pad_lo=pad_lo, Ho=Ho, Wo=Wo,
                 count_pad=count_pad)
        self.emit("avgpool", x=x.name, out=out.name, **a)
        self.use(x)
        self.tape.append(lambda: self.contribute(x, lambda o, add, mask: self.emit(
            "avgpool_bwd", dout=self.grad_of(out), dx=o, add_src=add, mask_src=mask, **a)))
        return out

    def maxpool(self, x: Tensor, k, stride) -> Tensor:
        B, H, W, C = x.shape
        Ho, Wo = -(-H // stride), -(-W // stride)
        total = max((Ho - 1) * stride + k - H, 0)
        pad_lo = total // 2          # TF SAME: the odd cell goes after
        out = self.tensor("maxp", (B, Ho, Wo, C))
        a = dict(B=B, H=H, W=W, C=C, k=k, stride=stride, pad_lo=pad_lo, Ho=Ho, Wo=Wo)
        self.emit("maxpool", x=x.name, out=out.name, **a)
        self.use(x)
        self.tape.append(lambda: self.contribute(x, lambda o, add, mask: self.emit(
            "maxpool_bwd", dout=self.grad_of(out), x=x.name, dx=o, add_src=add, mask_src=mask, **a)))
        return out

    def residual_tail_db(self, co3: ConvOut, *, shortcut, mode, relu, gamma_scale, ms=None) -> Tensor:
        """Block tail with DropBlock (nets/resnet_model.py:42-47,84-95): out = act(db(bn(y3)) + R),
        R = db(bn(shortcut conv)) for a projection shortcut, x for an identity shortcut."""
        B, H, W, C = co3.y.shape
        t3 = self.bn_act(co3, relu=False, name="t3")
        m3 = self.dropblock_mask(H, W, C, gamma_scale)
        t3d = self.dropblock_apply(t3, m3, relu=False, name="t3d")
        if mode == "bn":
            # ms: the shortcut's mask, drawn by the caller where the reference draws it (first in
            # the block, :42-47), so that meta['dropblock_u'] lists the draws in the reference's order
            ts = self.bn_act(shortcut, relu=False, name="ts")
            r = self.dropblock_apply(ts, ms, relu=False, name="tsd")
        else:
            assert mode == "identity"
            r = shortcut
            self.use(shortcut)
        ident = ConvOut(None, t3d, None, None, self.identity_bn(C))
        out = self.bn_act(ident, relu=relu, b=r, b_mode=2, name="out")

        def bwd():
            g = self.grad_of(out)
            self.conv_backward(co3, self.bn_backward(co3, self.dropblock_bwd(g, m3, co3.y.shape)))
            if mode == "bn":
                self.conv_backward(shortcut, self.bn_backward(
                    shortcut, self.dropblock_bwd(g, ms, co3.y.shape)))
            else:
                self.contribute_alias(shortcut, g)
        self.tape.append(bwd)
        return out

    def residual_tail(self, co3: ConvOut, *, shortcut, mode, relu, se=None) -> Tensor:
        """out = act(bn(y3) [*gate] + R); mode: 'bn' (ConvOut), 'identity' / 'up2' (Tensor)."""
        b_mode = {"bn": 1, "identity": 2, "up2": 3, None: 0}[mode]
        gate = se["e"] if se else None
        out = self.bn_act(co3, relu=relu, b=shortcut, b_mode=b_mode, gate=gate, name="out")
        if mode in ("identity", "up2"):
            self.use(shortcut)

        def bwd():
            g = self.grad_of(out)
            if se:
                B, H, W, C = co3.y.shape
                dims = dict(B=B, HW=H * W, C=C, r=se["r"])
                de = self.slot("work", B * C)
                dq = self.slot("work", B * C)
                self.emit("se_bwd_gate", g=g, y=co3.y.name, bn=co3.bn, de=de, **dims)
                self.emit("se_fc_bwd", de=de, e=se["e"], h=se["h"], q=se["q"], w1=se["w1"],
                          w2=se["w2"], dq=dq, scratch=se["scratch"], **dims)
                dy3 = self.bn_backward(co3, g, gate=se["e"], addbc=dq)
            elif mode == "bn" and self.fuse_bn_pairs:
                dy3, dys = self.bn_backward2(co3, shortcut, g)
                self.conv_backward(co3, dy3)
                self.conv_backward(shortcut, dys)
                return
            else:
                dy3 = self.bn_backward(co3, g)
            self.conv_backward(co3, dy3)
            if mode == "bn":
                self.conv_backward(shortcut, self.bn_backward(shortcut, g))
            elif mode == "identity":
                self.contribute_alias(shortcut, g)
            elif mode == "up2":
                B, H, W, C = shortcut.shape
                self.contribute(shortcut, lambda o, add, mask: self.emit(
                    "upsample2x_bwd", dout=g, dx=o, add_src=add, mask_src=mask, B=B, H=H, W=W, C=C))
        self.tape.append(bwd)
        return out

    def se(self, co3: ConvOut) -> dict:
        """nets/blocks.py:156-184 on t = bn(y3): returns the gate bookkeeping."""
        B, H, W, C = co3.y.shape
        r = C // 16
        with self.scope("se_block"):
            w1 = self._param(self._full("seblock_dense_1/kernel"), (1, 1, C, r), "conv_kernel",
                             (r, 1, 1, C), decay=True)
            w2 = self._param(self._full("seblock_dense_2/kernel"), (1, 1, r, C), "conv_kernel",
                             (C, 1, 1, r), decay=True)
        q, h, e = self.slot("work", B * C), self.slot("work", B * r), self.slot("work", B * C)
        scratch = self.slot("work", B * (C + r))
        dims = dict(B=B, HW=H * W, C=C, r=r)
        self.emit("se_gap", y=co3.y.name, bn=co3.bn, q=q, **dims)
        self.emit("se_fc", q=q, w1=w1.name, w2=w2.name, h=h, e=e, **dims)
        return dict(q=q, h=h, e=e, w1=w1.name, w2=w2.name, r=r, scratch=scratch)

    def bottleneck(self, x: Tensor, filters, shortcut_kind, strides, last_relu=True, db=None) -> Tensor:
        """nets/resnet_model.py:35-97 (_bottleneck_block_v1); db = DropBlock gamma_scale of this
        stage (None: off)."""
        cfg = self.cfg
        if not self.use_dropblock:
            db = None
        sconv = "sconv" in cfg.anti_alias_type
        sc = None
        if shortcut_kind is not None:
            xs = x
            k_s = 1
            if shortcut_kind == "proj":
                if "proj" in cfg.anti_alias_type and strides != 1:
                    xs = self.blurpool(x, cfg.anti_alias_filter_size, strides)
                else:
                    k_s = strides
            elif shortcut_kind == "resnet_d":
                B, H, W, C = x.shape
                if strides > 1:
                    xs = self.avgpool(x, 2, strides, 0, H // strides, W // strides, 1)
                else:
                    xs = self.avgpool(x, 2, 1, 0, H, W, 0)
            elif shortcut_kind == "bl":
                B, H, W, C = x.shape
                if strides > 1:
                    xs = self.avgpool(x, 3, strides, 1, (H + 2 - 3) // strides + 1,
                                      (W + 2 - 3) // strides + 1, 1)
            sc = self.conv(xs, filters * 4, 1, k_s)
        ms = None
        if db is not None and sc is not None:
            ms = self.dropblock_mask(sc.y.shape[1], sc.y.shape[2], sc.y.shape[3], db)
        t = self.cbr(x, filters, 1, 1) if db is None else self.cbr_db(x, filters, 1, 1, db)
        s3 = 1 if sconv else strides
        if cfg.use_sk_block:
            t = self.sk(t, filters, s3)
            if db is not None:                                   # :57-63 dropblock on the SK output
                v = t
                m = self.dropblock_mask(v.shape[1], v.shape[2], v.shape[3], db)
                t = self.dropblock_apply(v, m, relu=False, name="vd")
                self.use(v)
                self.tape.append(lambda v=v, m=m, t=t: self.contribute(
                    v, lambda out, add, mask: self._emit_db_contrib(self.grad_of(t), m, v, out, add,
                                                                     mask)))
        else:
            t = self.cbr(t, filters, 3, s3) if db is None else self.cbr_db(t, filters, 3, s3, db)
        if sconv and strides != 1:
            t = self.blurpool(t, cfg.anti_alias_filter_size, strides)
        co3 = self.conv(t, filters * 4, 1, 1, zero_gamma=cfg.zero_gamma)
        if db is not None:
            return self.residual_tail_db(co3, shortcut=sc if sc is not None else x,
                                         mode="bn" if sc is not None else "identity",
                                         relu=last_relu, gamma_scale=db, ms=ms)
        se = self.se(co3) if cfg.use_se_block else None
        if sc is not None:
            return self.residual_tail(co3, shortcut=sc, mode="bn", relu=last_relu, se=se)
        return self.residual_tail(co3, shortcut=x, mode="identity", relu=last_relu, se=se)

    def _emit_db_contrib(self, g, m, v, out, add, mask):
        assert add is None and mask is None
        B, H, W, C = v.shape
        self.emit("dropblock_apply", x=g, keep=m["keep"], scale=m["scale"], relu=False, out=out,
                  B=B, HW=H * W, C=C)

    def block_layer(self, x, filters, num_blocks, strides, *, use_resnet_d=False, use_bl=False,
                    last_relu=True, db=None):
        """nets/resnet_model.py:99-163: the first block always projects and never sees last_relu."""
        kind = "resnet_d" if use_resnet_d else ("bl" if use_bl else "proj")
        x = self.bottleneck(x, filters, kind, strides, db=db)
        for i in range(1, num_blocks):
            x = self.bottleneck(x, filters, None, 1,
                                last_relu=last_relu if i == num_blocks - 1 else True, db=db)
        return x

    # ---------------------------------------------------------------- the network
    def _build(self, H, W):
        cfg, p, B = self.cfg, self.plan, self.B
        meta = p.meta
        nf = 64
        Bin = meta["input_batch"]
        images = self.tensor("images", (Bin, H, W, 3), "f32")
        meta["images"] = images.name
        # the W axis of the packed input is physically zero-padded for the stem's taps
        _, _, wlo, whi = self.stem_s2d_taps(3 if cfg.use_resnet_d else 7)
        x0 = self.tensor("x0", (B, H // 2, W // 2 + wlo + whi, 16))
        self.emit("prep_weights")
        lam1 = lam2 = None
        if self.mixup_type:
            lam1 = self.tensor("lam1", (Bin // 2,), "f32")
            meta["lam1"] = lam1.name
            if self.mixup_type == 2:
                lam2 = self.tensor("lam2", (Bin // 2,), "f32")
                meta["lam2"] = lam2.name
        self.emit("pack_input", images=images.name, lam1=lam1 and lam1.name,
                  lam2=lam2 and lam2.name, mode=self.mixup_type, out=x0.name, Bin=Bin, H=H, W=W,
                  wpad=(wlo, whi))

        d = cfg.use_resnet_d
        if d and cfg.resnet_version == 1:
            x = self.stem_cbr(x0, nf // 2, 3)
            x = self.cbr(x, nf // 2, 3, 1)
            co = self.conv(x, nf, 3, 1, with_bn=False)
            co.bn = self.bn_layer(nf, B * (H // 2) * (W // 2))
            self._attach_bn(co)
        elif d:
            with self.scope("stage0"):
                x = self.stem_cbr(x0, nf // 2, 3)
                x = self.cbr(x, nf // 2, 3, 1)
                co = self.conv(x, nf, 3, 1, with_bn=False)
            with self.scope("stage0"):
                co.bn = self.bn_layer(nf, B * (H // 2) * (W // 2))
                self._attach_bn(co)
        elif cfg.resnet_version == 2:
            with self.scope("stage0"):
                co = self.stem_conv(x0, nf, 7)
                stem_bn_ops = self._detach_last_bn(co)
            with self.scope("stage0"):
                self._rename_bn(co, stem_bn_ops)
        else:
            co = self.stem_conv(x0, nf, 7)
        x = self.bn_act(co, relu=True)
        self.tape.append(lambda co=co, x=x: self.conv_backward(
            co, self.bn_backward(co, self.grad_of(x))))

        if cfg.resnet_version == 1:
            x = self.maxpool(x, 3, 2)
        else:
            with self.scope("stage0/pool"):             # BL module 0, resnet_model.py:385-419
                big0 = self.conv(x, nf, 3, 2)
                l0 = self.cbr(x, nf // cfg.bl_alpha, 3, 1)
                l0 = self.cbr(l0, nf // cfg.bl_alpha, 3, 2)
                l0c = self.conv(l0, nf, 1, 1)
                x = self.residual_tail(big0, shortcut=l0c, mode="bn", relu=True)
                x = self.cbr(x, nf, 1, 1)

        sizes = BLOCK_SIZES[cfg.resnet_version][cfg.resnet_size]
        strides = [2, 2, 1, 2] if cfg.resnet_version == 2 else [1, 2, 2, 2]
        if cfg.no_downsample:
            strides[-1] = 1
        for i, nb in enumerate(sizes):
            f = nf * (2 ** i)
            # dropblock_for_group3 (gamma_scale 0.25) / group4 (1.0): nets/resnet_model.py:432-453
            db = {2: 0.25, 3: 1.0}.get(i)
            if cfg.resnet_version == 2 and i < 3:
                with self.scope("stage%d" % (i + 1)):
                    with self.scope("big%d" % (i + 1)):
                        big = self.block_layer(x, f, nb - 1, 2, use_bl=True, last_relu=False, db=db)
                    with self.scope("little%d" % (i + 1)):
                        little = self.block_layer(x, f // cfg.bl_alpha,
                                                  max(1, nb // cfg.bl_beta - 1), 1, use_bl=True,
                                                  db=db)
                        le = self.conv(little, f * 4, 1, 1)
                    with self.scope("merge%d" % (i + 1)):
                        x = self.residual_tail(le, shortcut=big, mode="up2", relu=True)
                        x = self.block_layer(x, f, 1, strides[i], use_bl=True, db=db)
            elif cfg.resnet_version == 2:
                with self.scope("stage%d" % (i + 1)):
                    x = self.block_layer(x, f, nb, strides[i], use_resnet_d=d, use_bl=True, db=db)
            else:
                x = self.block_layer(x, f, nb, strides[i], use_resnet_d=d, db=db)

        # head: pool -> [embedding conv + BN] -> dense (nets/resnet_model.py:552-599)
        Bx, Hx, Wx, Cx = x.shape
        nc, ld = cfg.num_classes, meta["ld_logits"]
        self.use(x)
        if cfg.pool_type == "gap":
            pooled = self.tensor("pooled", (B, Cx))
            self.emit("gap", x=x.name, out=pooled.name, B=B, HW=Hx * Wx, C=Cx)
        elif cfg.pool_type == "gem":
            pooled = self.tensor("pooled", (B, Cx))
            gem_s = self.slot("work", B * Cx)
            self.emit("gem", x=x.name, out=pooled.name, ssum=gem_s, B=B, HW=Hx * Wx, C=Cx)
        else:                                            # flatten, NHWC order (:568-571)
            pooled = self.tensor("pooled", (B, Hx * Wx * Cx))
            self.emit("grad_combine", a=x.name, add_src=None, mask_src=None, out=pooled.name,
                      shape=x.shape)
        Cf = pooled.shape[1]
        feat, emb_co = pooled, None
        if cfg.embedding_size > 0:
            # 1x1 conv 'embedding_dense' (no bias) + BN 'embedding_dense_batch_normalization' on the
            # [B,1,1,Cf] pooled tensor (:575-584); return_embedding = the BN output; ReLU before dense
            E = cfg.embedding_size
            we = self._param("resnet_model/embedding_dense/kernel", (1, 1, Cf, E), "conv_kernel",
                             (E, 1, 1, Cf), decay=True, need_dgrad=self.training)
            ge = Geom(B, 1, 1, Cf, E, 1, 1, 1, 0, 0, 0, 0)
            ye = self.tensor("y", (B, 1, 1, E))
            bne = self.bn_layer(E, B, layer="embedding_dense_batch_normalization")
            self.emit("conv", x=pooled.name, xp=self.planes(pooled.name), w=we.name, y=ye.name,
                      geom=ge, stats=bne.stats if (self.training and not self.fp32) else None,
                      bias=None, out_f32=False)
            self.emit_bn_finalize(bne, ye, ge)
            self.use(pooled)
            emb_co = ConvOut(pooled, ye, ge, we.name, bne)
            emb = self.bn_act(emb_co, relu=False, name="embedding")
            feat = self.bn_act(emb_co, relu=True, name="embedding_relu")
            meta["embedding"] = emb.name
            Cf = E
        wk = self._param("resnet_model/dense/kernel", (Cf, nc), "dense_kernel", (ld, 1, 1, Cf),
                         decay=True, need_dgrad=self.training)
        bk = self._param("resnet_model/dense/bias", (nc,), "dense_bias", (ld,), decay=True)
        logits = self.tensor("logits", (B, ld), "f32")
        gd = Geom(B, 1, 1, Cf, ld, 1, 1, 1, 0, 0, 0, 0)
        self.emit("conv", x=feat.name, xp=self.planes(feat.name), w=wk.name, y=logits.name,
                  geom=gd, stats=None, bias=bk.name, out_f32=True)
        self.use(feat)
        meta.update(logits=logits.name, pooled=pooled.name, feature_shape=x.shape)
        if not self.with_loss:
            return
        labels = self.tensor("labels", (Bin,), "i32")
        ysoft = self.tensor("ysoft", (B, nc), "f32")
        lam_names = dict(lam1=lam1 and lam1.name, lam2=lam2 and lam2.name)
        self.emit("mix_labels", labels=labels.name, mode=self.mixup_type, y=ysoft.name, Bin=Bin,
                  NC=nc, **lam_names)
        yt = None
        if self.kd_temp > 0:
            # knowledge distillation (nets/run_loop_classification.py:86-96): the labels carry the
            # teacher's logits; teacher labels = softmax(. / T), mixed like the supervised labels
            tlog = self.tensor("teacher_logits", (Bin, nc), "f32")
            yt = self.tensor("yteacher", (B, nc), "f32")
            meta["teacher_logits"] = tlog.name
            self.emit("kd_teacher", teacher_logits=tlog.name, labels=labels.name,
                      mode=self.mixup_type, kd_temp=self.kd_temp, yt=yt.name, Bin=Bin, NC=nc,
                      **lam_names)
        loss = self.slot("zero", 4)          # [cross_entropy, l2_loss, kd_loss, -]
        dlogits = self.tensor("dlogits", (B, ld))
        meta.update(labels=labels.name, ysoft=ysoft.name, loss=loss)
        self.emit("softmax_ce", logits=logits.name, y=ysoft.name, yt=yt and yt.name,
                  kd_temp=self.kd_temp, B=B, NC=nc, ld=ld,
                  label_smoothing=meta["label_smoothing"], loss=loss, dlogits=dlogits.name,
                  dbias=bk.name if self.training else None,
                  work=self.slot("work", 2 * _round_up(B, 32) + B * ld))
        if not self.training:
            return

        # ---------------- backward ----------------
        self.ops = p.backward
        self.emit("conv_wgrad", x=feat.name, xp=self.planes(feat.name), dy=dlogits.name,
                  dyp=self.planes(dlogits.name), geom=gd, w=wk.name)
        self.contribute(feat, lambda out, add, mask: self.emit_dgrad(
            dlogits.name, wk.name, out, gd, add, mask))
        if emb_co is not None:
            self.conv_backward(emb_co, self.bn_backward(emb_co, self.grad_of(feat)))
        dpooled = self.grad_of(pooled)

        def pool_bwd(out, add, mask):
            assert add is None
            if cfg.pool_type == "gap":
                self.emit("gap_bwd", dpooled=dpooled, mask_src=mask, dx=out, B=B, HW=Hx * Wx, C=Cx)
            elif cfg.pool_type == "gem":
                # x <= 0 is outside GeM's clip range: the ReLU mask is implied
                self.emit("gem_bwd", dpooled=dpooled, ssum=gem_s, x=x.name, dx=out, B=B,
                          HW=Hx * Wx, C=Cx)
            else:
                self.emit("grad_combine", a=dpooled, add_src=None, mask_src=mask, out=out,
                          shape=x.shape)
        self.contribute(x, pool_bwd)
        for fn in reversed(self.tape):
            fn()
        # ---------------- update ----------------
        self.ops = p.update
        self.emit("sgd", loss=loss, scratch=self.slot("work", SGD_SCRATCH))
        for t in p.tensors.values():
            assert t.contribs == t.consumers or t.name == x0.name, (t.name, t.contribs, t.consumers)

    # stem BN bookkeeping for rv=2: the BN after the first conv lives in a second 'stage0' scope
    # (nets/resnet_model.py:359-381), so its variable names differ from the conv's scope.
    def _detach_last_bn(self, co: ConvOut):
        bn = co.bn
        for n in (bn.gamma, bn.beta):
            self._stash = getattr(self, "_stash", {})
            self._stash[n] = self.plan.params.pop(n)
        for n in (bn.mm, bn.mv):
            self._stash[n] = self.plan.state.pop(n)
        key = ("/".join(self._scope), "batch_normalization")
        self._counters[key] -= 1
        return bn

    def _rename_bn(self, co: ConvOut, bn: BN):
        layer = self._unique("batch_normalization")
        for attr, table in (("gamma", self.plan.params), ("beta", self.plan.params),
                            ("mm", self.plan.state), ("mv", self.plan.state)):
            old = getattr(bn, attr)
            par = self._stash.pop(old)
            par.name = self._full(layer + "/" + old.rsplit("/", 1)[1])
            table[par.name] = par
            setattr(bn, attr, par.name)

    def _attach_bn(self, co: ConvOut):
        """BN created after a with_bn=False conv: add the statistics to the conv op, finalize."""
        for op in reversed(self.ops):
            if op.kind == "conv" and op.y == co.y.name:
                op.a["stats"] = co.bn.stats if (self.training and not self.fp32) else None
                break
        self.emit_bn_finalize(co.bn, co.y, co.geom)


def build_plan(cfg: ModelConfig, batch: int, height: int = 224, width: int = 224, **kw) -> Plan:
    return PlanBuilder(cfg, batch, height, width, **kw).plan


# ------------------------------------------------------------------------------------------------
# Canonical text of a plan -- the same format as acnn_plan_dump() of the model-level C ABI
# (csrc/model_plan.cu builds the plan natively; tests/test_native_plan_cpu.py compares the two texts)
def _fmt(v):
    if v is None:
        return "-"
    if isinstance(v, bool):
        return "1" if v else "0"
    if isinstance(v, int):
        return str(v)
    if isinstance(v, float):
        return "%.9g" % v
    if isinstance(v, str):
        return v
    if isinstance(v, Slot):
        return "%s:%d:%d" % (v.buf, v.offset, v.size)
    if isinstance(v, BN):
        return "bn(C=%d,count=%d,gamma=%s,beta=%s,mm=%s,mv=%s,stats=%s,work=%s)" % (
            v.C, v.count, _fmt(v.gamma), _fmt(v.beta), _fmt(v.mm), _fmt(v.mv), _fmt(v.stats),
            _fmt(v.work))
    if isinstance(v, Geom):
        return "g" + _fmt(v.astuple())
    if isinstance(v, (tuple, list)):
        return "(" + ",".join(_fmt(x) for x in v) + ")"
    raise TypeError("plan dump: cannot format %r" % (v,))


def dump(plan: Plan) -> str:
    out = ["sizes param_elems=%d state_elems=%d dgrad_elems=%d zero_elems=%d work_elems=%d" % (
        plan.param_elems, plan.state_elems, plan.dgrad_elems, plan.zero_elems, plan.work_elems)]
    for k in sorted(plan.meta):
        if plan.meta[k] is not None:
            out.append("meta %s=%s" % (k, _fmt(plan.meta[k])))
    for buffer, table in (("params", plan.params), ("state", plan.state)):
        for p in table.values():
            out.append("var %s buffer=%s kind=%s tf_shape=%s store_shape=%s offset=%d size=%d decay=%d "
                       "zero_init=%d dgrad_off=%d" % (
                           p.name, buffer, p.kind, _fmt(p.tf_shape), _fmt(p.store_shape), p.offset,
                           p.size, p.decay, p.zero_init, p.dgrad_off))
    for t in plan.tensors.values():
        out.append("tensor %s shape=%s dtype=%s relu=%d" % (t.name, _fmt(t.shape), t.dtype, t.relu))
    for tag, ops in (("F", plan.forward), ("B", plan.backward), ("U", plan.update)):
        for i, op in enumerate(ops):
            kv = " ".join("%s=%s" % (k, _fmt(op.a[k])) for k in sorted(op.a) if op.a[k] is not None)
            out.append(("op %s %d %s %s" % (tag, i, op.kind, kv)).rstrip())
    return "\n".join(out) + "\n"
