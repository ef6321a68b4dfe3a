"""GPU parity, op by op: the CUDA runtime is run in lock-step with the CPU plan interpreter
(oracle/plan_interp.py, same bf16 rounding points) on small configurations; after every op the
op's outputs are compared and then overwritten with the oracle's values, so each kernel is checked
in isolation on identical inputs.

Tolerances (relative to the output's max magnitude): bf16 tensors 2^-7 (one bf16 ulp at the top
of the range: accumulation-order differences can flip a rounding), fp32 vectors 2e-3 where sums
of bf16 data cancel (BN backward sums), 1e-4 otherwise.

The fp32 parity mode (dtype='fp32': fp32 storage, 3-plane wgmma GEMMs) runs the same lock-step
against the exact fp32 interpreter with every tensor at 2e-5 and the reductions at 2e-4.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_TOL = 2.0 ** -7
F32_TOL = 2e-3


def _outputs(op):
    k, a = op.kind, op.a
    T = lambda key: [("t", a[key])]
    S = lambda key: [("slot", a[key])]
    G = lambda *names: [("grad", n) for n in names]
    if k in ("prep_weights", "split3"):
        return []
    if k == "bn_stats":
        return [("slot", a["bn"].stats)]
    if k == "pack_input":
        return T("out")
    if k == "mix_labels":
        return T("y")
    if k == "s2d_weight_pack":
        return T("w2")
    if k == "conv":
        return T("y") + ([("parts", a["stats"], 2 * a["geom"].Cout)]
                         if a.get("stats") is not None else [])
    if k == "bn_finalize":
        bn = a["bn"]
        return [("slot", bn.work), ("state", bn.mm), ("state", bn.mv)]
    if k in ("bn_act", "blurpool", "avgpool", "maxpool", "gap", "zero_insert", "grad_combine",
             "dropblock_apply"):
        return T("out")
    if k == "gem":
        return T("out") + S("ssum")
    if k == "gem_bwd":
        return T("dx")
    if k == "dropblock_mask":
        return S("keep") + S("scale")
    if k == "kd_teacher":
        return T("yt")
    if k == "sk_gap":
        return S("s")
    if k == "sk_fc":
        bn = a["bn"]
        return S("zpre") + S("z") + S("att") + [("slot", bn.work), ("state", bn.mm), ("state", bn.mv)]
    if k == "sk_combine":
        return T("v")
    if k == "se_gap":
        return S("q")
    if k == "se_fc":
        return S("h") + S("e")
    if k == "softmax_ce":
        return T("dlogits") + S("loss") + (G(a["dbias"]) if a.get("dbias") else [])
    if k == "conv_wgrad":
        return S("dw_slot") if a.get("dw_slot") is not None else G(a["w"])
    if k in ("conv_dgrad", "blurpool_bwd", "avgpool_bwd", "maxpool_bwd", "upsample2x_bwd", "gap_bwd"):
        return T("dx")
    if k == "s2d_wgrad_unpack":
        return G(a["w"])
    if k in ("bn_bwd_reduce", "sk_bn_bwd_reduce"):
        return [("parts", a["sums"], 2 * a["bn"].C)]
    if k == "bn_bwd_reduce2":
        return [("parts", a["sums"], 2 * a["bn"].C), ("parts", a["sums2"], 2 * a["bn2"].C)]
    if k == "bn_bwd_apply2":
        return T("dy") + T("dy2")
    if k == "bn_bwd_finalize":
        return S("coef") + G(a["bn"].gamma, a["bn"].beta)
    if k in ("bn_bwd_apply", "sk_bn_bwd_apply"):
        return T("dy")
    if k == "sk_bwd_gate":
        return S("dA")
    if k == "sk_fc_bwd":
        return S("ds") + G(a["w1"], a["w2"], a["bn"].gamma, a["bn"].beta)
    if k == "se_bwd_gate":
        return S("de")
    if k == "se_fc_bwd":
        return S("dq") + G(a["w1"], a["w2"])
    if k == "sgd":
        return [("all_params",), ("all_momentum",), ("slot", a["loss"])]
    raise KeyError(k)


def _err(got, ref):
    ref = ref.double()
    got = got.double().cpu()
    scale = max(ref.abs().max().item(), 1e-20)
    return (got - ref).abs().max().item() / scale, scale


def lockstep(cfg_kw, use_resnet_d=False, B=4, HW=64, mix=0, training=True, verbose=False,
             dtype="bf16", use_dropblock=False, kd_temp=0.0, keep_prob=0.9):
    H, W = (HW, HW) if isinstance(HW, int) else HW
    from oracle import model as M, plan_interp as PI
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from assembled_cnn_b200.runtime import Runtime

    cfg = ModelConfig(use_resnet_d=use_resnet_d, **cfg_kw)
    fp32 = dtype == "fp32"
    bf16_tol, f32_tol = (2e-5, 2e-4) if fp32 else (BF16_TOL, F32_TOL)
    plan = build_plan(cfg, B, H, W, training=training, mixup_type=mix, label_smoothing=0.1,
                      dtype=dtype, use_dropblock=use_dropblock, kd_temp=kd_temp)
    _, vs = M.build(seed=42, input_hw=64, use_resnet_d=use_resnet_d, **cfg_kw)
    g = torch.Generator().manual_seed(3)
    for n in vs.vars:       # non-trivial BN parameters / statistics
        if n.endswith("gamma"):
            vs.vars[n] = 0.5 + torch.rand(vs.vars[n].shape, generator=g)
        elif n.endswith("beta") or n.endswith("moving_mean"):
            vs.vars[n] = 0.1 * torch.randn(vs.vars[n].shape, generator=g)
        elif n.endswith("moving_variance"):
            vs.vars[n] = 0.5 + torch.rand(vs.vars[n].shape, generator=g)
    it = PI.PlanInterpreter(plan, dtype=torch.float64 if fp32 else torch.float32,
                            emulate_bf16=not fp32)
    rt = Runtime(plan)
    it.set_weights(vs.vars)
    rt.set_weights(vs.vars)
    hp = dict(lr=0.05, momentum=0.9, weight_decay=1e-4, keep_prob=keep_prob)
    it.hp.update(hp)
    rt.set_hparams(**hp)
    rt.dropblock_feed = True          # masks from the fed uniforms (identical on both sides)
    m = plan.meta
    Bin = m["input_batch"]
    x = (torch.randn(Bin, H, W, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (Bin,), generator=g).int()
    it.zero_step_buffers()
    rt.zero_step_buffers()
    feeds = {m["images"]: x}
    if "labels" in m:
        feeds[m["labels"]] = lab
    if mix:
        feeds[m["lam1"]] = torch.rand(Bin // 2, generator=g)
    if mix == 2:
        feeds[m["lam2"]] = torch.rand(Bin // 2, generator=g)
    for name in m.get("dropblock_u", []):
        feeds[name] = torch.rand(plan.tensors[name].shape, generator=g)
    if "teacher_logits" in m:
        feeds[m["teacher_logits"]] = 3.0 * torch.randn(Bin, 1001, generator=g)
    for name, v in feeds.items():
        it.t[name] = v.to(it.dtype) if v.is_floating_point() else v
        rt.t[name].copy_(v)

    worst = {}
    failures = []
    for idx, op in enumerate(plan.all_ops()):
        it.run([op])
        rt.run([op])
        torch.cuda.synchronize()
        for out in _outputs(op):
            kind = out[0]
            if kind == "t":
                ref, got = it.t[out[1]], rt.t[out[1]]
                tol = bf16_tol if plan.tensors[out[1]].dtype == "bf16" else (2e-5 if fp32 else 1e-4)
                force = lambda r=ref, gt=got: gt.copy_(r)
            elif kind == "slot":
                ref, got = it.slot(out[1]), rt.slot_view(out[1])
                tol = f32_tol
                force = lambda r=ref, gt=got: gt.copy_(r)
            elif kind == "parts":
                # [parts][ncols] per-CTA partial rows on the GPU (unused rows stay zero); the
                # interpreter keeps the total in row 0
                ncols = out[2]
                full = rt.slot_view(out[1])
                ref = it.slot(out[1])[:ncols]
                got = full.view(-1, ncols).double().sum(0)
                tol = f32_tol

                def force(r=ref, f=full, n=ncols):
                    f.zero_()
                    f[:n].copy_(r)
            elif kind == "grad":
                ref, got = it.pview(out[1], it.grads), rt.pview(out[1], rt.grads)
                tol = f32_tol
                force = lambda r=ref, gt=got: gt.copy_(r)
            elif kind == "state":
                ref, got = it.pview(out[1]), rt.pview(out[1])
                tol = 1e-4
                force = lambda r=ref, gt=got: gt.copy_(r)
            elif kind == "all_params":
                ref, got, tol, force = it.params, rt.params, 1e-5, (lambda: None)
            elif kind == "all_momentum":
                ref, got, tol, force = it.momentum, rt.momentum, 1e-4, (lambda: None)
            e, scale = _err(got.float().reshape(-1), ref.float().reshape(-1))
            key = op.kind + ":" + kind
            worst[key] = max(worst.get(key, 0.0), e)
            if not (e <= tol):
                failures.append("op %d %s output %s: rel err %.3e (tol %.1e, scale %.3e)"
                                % (idx, op.kind, out[1:] if len(out) > 1 else "", e, tol, scale))
                if verbose:
                    print(failures[-1], flush=True)
            force()
    if verbose:
        for k_, v_ in sorted(worst.items()):
            print("%-28s %.3e" % (k_, v_))
    return failures, worst


CONFIGS = {
    "vanilla_rv1": (dict(resnet_size=50, resnet_version=1), False, 0),
    "assemble_rv2_sk_sconv_mix1": (dict(resnet_size=50, resnet_version=2, use_sk_block=True,
                                        anti_alias_type="sconv", anti_alias_filter_size=3), False, 1),
    "rv1_d_sk_sconv_mix2": (dict(resnet_size=50, resnet_version=1, use_sk_block=True,
                                 anti_alias_type="sconv", anti_alias_filter_size=3), True, 2),
    "rv2_se_proj5": (dict(resnet_size=50, resnet_version=2, use_se_block=True,
                          anti_alias_type="proj", anti_alias_filter_size=5), False, 0),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_train_step_lockstep(name):
    kw, d, mix = CONFIGS[name]
    failures, _ = lockstep(kw, d, B=4, HW=64, mix=mix, training=True)
    assert not failures, "\n".join(failures[:20])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_train_step_lockstep_fp32_mode(name):
    """dtype='fp32' (the reference's default dtype): every op against the exact interpreter."""
    kw, d, mix = CONFIGS[name]
    failures, _ = lockstep(kw, d, B=4, HW=64, mix=mix, training=True, dtype="fp32")
    assert not failures, "\n".join(failures[:20])


FEATURE_CONFIGS = {
    # GeM pooling + embedding head + KD (mixup 2: the teacher-label quirk);
    # flatten pooling + KD in the fp32 mode; DropBlock on both block kinds (needs 224 px: the
    # stage-4 feature map must be >= the 7 x 7 block)
    "gem_embedding_kd_mix2": dict(cfg=dict(pool_type="gem", embedding_size=64, resnet_size=50,
                                           resnet_version=2, use_sk_block=True,
                                           anti_alias_type="sconv", anti_alias_filter_size=3),
                                  mix=2, kd_temp=2.0),
    "flatten_kd_fp32": dict(cfg=dict(resnet_size=50, resnet_version=1, pool_type="flatten"), mix=1,
                            kd_temp=1.0, dtype="fp32"),
    "dropblock_assemble": dict(cfg=dict(resnet_size=50, resnet_version=2, use_sk_block=True,
                                        anti_alias_type="sconv", anti_alias_filter_size=3),
                               use_dropblock=True, B=4, HW=224),
    "dropblock_vanilla_fp32": dict(cfg=dict(resnet_size=50, resnet_version=1), use_dropblock=True,
                                   B=4, HW=224, dtype="fp32"),
}


@pytest.mark.parametrize("name", list(FEATURE_CONFIGS))
def test_feature_rows_lockstep(name):
    kw = dict(FEATURE_CONFIGS[name])
    cfg = kw.pop("cfg")
    failures, _ = lockstep(cfg, False, training=True, **kw)
    assert not failures, "\n".join(failures[:20])


def test_non_square_odd_batch_lockstep():
    """Ragged shapes: 64 x 96 input, batch 3 (no dimension is a multiple of a tile size)."""
    kw, d, _ = CONFIGS["assemble_rv2_sk_sconv_mix1"]
    failures, _ = lockstep(kw, d, B=3, HW=(64, 96), mix=0, training=True)
    assert not failures, "\n".join(failures[:20])


def test_eval_forward_lockstep():
    kw, d, _ = CONFIGS["assemble_rv2_sk_sconv_mix1"]
    failures, _ = lockstep(kw, d, B=2, HW=64, mix=0, training=False)
    assert not failures, "\n".join(failures[:20])


if __name__ == "__main__":
    dtype = "fp32" if "--fp32" in sys.argv else "bf16"
    names = [a for a in sys.argv[1:] if not a.startswith("--")] or list(CONFIGS)
    for n in names:
        kw, d, mix = CONFIGS[n]
        print("=====", n, dtype, flush=True)
        f, w = lockstep(kw, d, mix=mix, verbose=True, dtype=dtype)
        print("FAILURES:", len(f))
