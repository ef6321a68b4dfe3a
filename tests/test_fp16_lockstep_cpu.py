"""CPU checks that make the fp16 lock-step (tests/test_fp16_lockstep_gpu.py) trustworthy:

  * coverage: its runs contain every op kind an fp16 plan can contain (over the flag space the plan
    builder accepts), and test_plan_gpu._outputs knows the outputs of every one of them;
  * rounding: the interpreter emulating an fp16 plan's storage leaves every stored fp16 tensor and every
    GEMM weight fp16-representable; on a bf16 plan it computes what the bf16-only emulation computed,
    bit for bit;
  * sharpness: an interpreter that rounds the fp16 plan's storage to bf16 instead differs from the right
    one by more than the lock-step's 2^-10 on the stem conv, the first bn_act and the logit gradient, so
    a kernel that stored the wrong 16-bit type fails the GPU lock-step.
"""
import itertools
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import pytest
import torch

import test_fp16_lockstep_gpu as L
import test_plan_gpu as P
from oracle import model as M, plan_interp as PI
from assembled_cnn_b200.plan import ModelConfig, build_plan

FP32_ONLY = {"split3", "bn_stats"}


def _flag_space_plans():
    """fp16 plans over the builder's flags: shortcut kinds x SK / SE x anti-alias variants x pooling /
    embedding heads x no_downsample x train (mixup 0 / 1 / 2, with and without KD) / eval, and DropBlock
    (224 px, not with SE); combinations the builder refuses are skipped."""
    models = itertools.product([1, 2], ["", "sk", "se"], ["", "sconv", "proj", "sconv,proj"],
                               ["gap", "gem", "flatten"], [0, 64], [False, True], [False, True])
    for i, (ver, block, aa, pool, emb, d, nd) in enumerate(models):
        kw = dict(resnet_size=50, resnet_version=ver, use_sk_block=block == "sk", use_se_block=block == "se",
                  anti_alias_type=aa, anti_alias_filter_size=3 if aa else 0, pool_type=pool,
                  embedding_size=emb, no_downsample=nd, use_resnet_d=d)
        runs = [dict(training=True, mixup_type=i % 3, kd_temp=float(i % 2)), dict(training=False)]
        if block != "se" and i % 4 == 0:
            runs.append(dict(training=True, mixup_type=i % 3, use_dropblock=True, hw=224))
        for r in runs:
            hw = r.pop("hw", 64)
            try:
                yield build_plan(ModelConfig(**kw), 4, hw, hw, label_smoothing=0.1, dtype="fp16", **r)
            except (ValueError, NotImplementedError):
                continue


def test_fp16_lockstep_runs_cover_every_fp16_op_kind():
    possible = set()
    for plan in _flag_space_plans():
        assert plan.meta["dtype"] == "fp16"
        for op in plan.all_ops():
            possible.add(op.kind)
            P._outputs(op)                      # KeyError for a kind the lock-step cannot compare
    assert not possible & FP32_ONLY, possible & FP32_ONLY
    covered = set()
    for name in L.RUNS:
        for op in L.build_run_plan(name).all_ops():
            covered.add(op.kind)
            P._outputs(op)
    assert covered == possible, ("fp16 op kinds without a lock-step run: %s; run kinds no plan of the flag "
                                 "space has: %s" % (sorted(possible - covered), sorted(covered - possible)))


# ---------------------------------------------------------------------------------------------------
# rounding
# ---------------------------------------------------------------------------------------------------
SMALL = (dict(resnet_size=50, resnet_version=1), 2, 64)       # rv1: stem maxpool, projection shortcuts


def _small_plan(dtype, mix=1, B=None):
    kw, B0, hw = SMALL
    B = B or B0
    return build_plan(ModelConfig(**kw), B, hw, hw, training=True, mixup_type=mix, label_smoothing=0.1,
                      dtype=dtype)


def _inputs(plan, seed=3):
    g = torch.Generator().manual_seed(seed)
    m = plan.meta
    Bin = m["input_batch"]
    x = (torch.randn(Bin, m["height"], m["width"], 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (Bin,), generator=g).int()
    lam = torch.rand(Bin // 2, generator=g) if m["mixup_type"] else None
    return x, lab, lam


def _interp(plan, dtype, **emu):
    _, vs = M.build(seed=42, input_hw=plan.meta["height"], **SMALL[0])
    it = PI.PlanInterpreter(plan, dtype=dtype, **emu)
    it.set_weights(vs.vars)
    it.hp.update(lr=0.05, momentum=0.9, weight_decay=1e-4, grad_scale=128.0, sgd_grad_scale=1.0 / 128)
    return it


def _f16_representable(v):
    return bool(torch.equal(v.half().to(v.dtype), v)) and not bool(torch.isnan(v).any())


def test_fp16_emulation_stores_fp16_values():
    plan = _small_plan("fp16")
    it = _interp(plan, torch.float64, emulate_storage=True)
    assert it.adt == "f16"
    weights = []
    wq = it.wq
    it.wq = lambda w: weights.append(wq(w)) or weights[-1]
    x, lab, lam = _inputs(plan)
    it.train_step(x, lab, lam)
    f16 = [n for n, t in plan.tensors.items() if t.dtype == "f16"]
    assert len(f16) > 100 and len(weights) > 50
    for n in f16:
        assert n in it.t and _f16_representable(it.t[n]), n
        assert not bool(it.t[n].isinf().any()), n              # nothing overflows in this step
    for w in weights:
        assert _f16_representable(w)
    # the values really carry fp16's 11 significant bits, not bf16's 8
    stem = next(op for op in plan.forward if op.kind == "conv").a["y"]
    assert not bool(torch.equal(it.t[stem].bfloat16().double(), it.t[stem]))


class _Bf16OnlyInterpreter(PI.PlanInterpreter):
    """The emulation as it was before fp16 plans existed: "bf16" tensors and every GEMM weight to bf16."""

    def store(self, name, value):
        t = self.plan.tensors[name]
        value = value.to(self.dtype)
        if self.emu and t.dtype == "bf16":
            value = value.bfloat16().to(self.dtype)
        self.t[name] = value

    def wq(self, w):
        return w.bfloat16().to(self.dtype) if self.emu else w


@pytest.mark.parametrize("kw", [dict(emulate_storage=True), dict(emulate_bf16=True)],
                         ids=["emulate_storage", "emulate_bf16"])
def test_bf16_plan_results_unchanged(kw):
    plan = _small_plan("bf16")
    x, lab, lam = _inputs(plan)
    new = _interp(plan, torch.float32, **kw)
    old = _interp(plan, torch.float32, emulate_storage=False)
    old.__class__ = _Bf16OnlyInterpreter
    old.emu = True
    out_new = new.train_step(x, lab, lam)
    out_old = old.train_step(x, lab, lam)
    assert torch.equal(out_new[0], out_old[0]) and out_new[1:] == out_old[1:]
    for n in plan.tensors:
        if n in old.t:
            assert torch.equal(new.t[n], old.t[n]), n
    for a in ("params", "grads", "momentum", "state", "zero", "work"):
        assert torch.equal(getattr(new, a), getattr(old, a)), a


# ---------------------------------------------------------------------------------------------------
# sharpness
# ---------------------------------------------------------------------------------------------------
def test_wrong_16bit_type_fails_the_fp16_tolerance():
    """The fp16 plan's forward in lock-step between the right emulation and one that rounds to bf16 (the
    wrong one's outputs are reset to the right one's after every op, as the GPU lock-step resets the
    kernels'): the stem conv, the first bn_act and dlogits differ by more than 2^-10.  (Batch 4 with mixup
    1: 16 logit gradients near the largest magnitude, the label terms, whose bf16 roundings set dlogits'
    error.)"""
    plan = _small_plan("fp16", B=4)
    right = _interp(plan, torch.float64, emulate_storage=True)
    wrong = _interp(plan, torch.float64, emulate_storage="bf16")
    x, lab, lam = _inputs(plan)
    m = plan.meta
    for it in (right, wrong):
        it.zero_step_buffers()
        it.t[m["images"]], it.t[m["labels"]], it.t[m["lam1"]] = x.double(), lab, lam.double()
    stem = next(op for op in plan.forward if op.kind == "conv")
    assert stem.a.get("x_wpad")
    first_bn_act = next(op for op in plan.forward if op.kind == "bn_act")
    watch = {id(stem): "stem conv", id(first_bn_act): "first bn_act"}
    errs = {}
    for op in plan.forward:
        right.run([op])
        wrong.run([op])
        for out in P._outputs(op):
            if out[0] != "t":
                if out[0] in ("slot", "parts"):
                    wrong.slot(out[1]).copy_(right.slot(out[1]))
                elif out[0] == "state":
                    wrong.pview(out[1]).copy_(right.pview(out[1]))
                elif out[0] == "grad":
                    wrong.pview(out[1], wrong.grads).copy_(right.pview(out[1], right.grads))
                continue
            name = out[1]
            e, _ = P._err(wrong.t[name].reshape(-1), right.t[name].reshape(-1))
            if id(op) in watch:
                errs[watch[id(op)]] = e
            if op.kind == "softmax_ce":
                errs["dlogits"] = e
            wrong.t[name] = right.t[name].clone()
    assert set(errs) == {"stem conv", "first bn_act", "dlogits"}, errs
    for k, e in errs.items():
        assert e > P.F16_TOL, (k, e)
