"""GPU parity of the fp32 mode (dtype='fp32', the reference's default dtype) against the CPU oracle
(oracle/model.py, autograd) -- the north-star tolerance: 1e-3 relative.

What is asserted, per BASELINE configuration family (C1 eval forward, C2 forward + loss, C3 full
training step, C5 topology):

  * logits, cross-entropy, L2 loss, BN moving statistics and the SGD-updated weights: norm-relative
    error <= 1e-3 against BOTH the fp32 and the fp64 oracle (measured: ~1e-5);
  * every gradient tensor, "backward given the forward": the whole CUDA backward chain (no teacher
    forcing of gradients) against the fp64 plan interpreter run on the SAME forward activations:
    <= 1e-3 (measured ~1e-5).  This is the well-posed gradient comparison: see next point;
  * every gradient tensor end to end against the fp64 autograd oracle: <= max(1e-3, 4 x yardstick),
    where the yardstick is the fp32 autograd oracle's own distance from the fp64 oracle on that
    tensor, measured in the same test.  A ReLU network's gradient is discontinuous in the forward
    activations: forward round-off of ~1e-5 (unavoidable in ANY fp32 implementation, including the
    reference's TF kernels with a different summation order) flips the sign of a ~1e-5 fraction of
    pre-activations, which moves every upstream gradient tensor by ~sqrt(1e-5) ~ 1e-2.  The fp32
    oracle itself is 1-2e-2 away from the fp64 oracle on these shapes, so 1e-3 end to end on
    gradients is not a property any fp32 implementation can have; the test reports both numbers;
  * two runs of the step are bit-identical (all reductions ordered, no split-K in this mode);
  * the bf16 production path's error on the same inputs is printed beside each fp32 number.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-3
ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)
R152 = dict(resnet_size=152, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
            anti_alias_filter_size=3, bl_alpha=1, bl_beta=2)


def _nrel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _inputs(n, hw, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, hw, hw, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (n,), generator=g).int()
    return x, lab, g


def _randomise_bn(vs, seed):
    g = torch.Generator().manual_seed(seed)
    for n in vs.vars:
        if n.endswith("moving_mean") or n.endswith("beta"):
            vs.vars[n] = (0.1 * torch.randn(vs.vars[n].shape, generator=g)).to(vs.vars[n].dtype)
        elif n.endswith("moving_variance") or n.endswith("gamma"):
            vs.vars[n] = (0.5 + torch.rand(vs.vars[n].shape, generator=g)).to(vs.vars[n].dtype)


def _oracle_vars(kw, hw, dt, seed_bn=None, **build_kw):
    from oracle import model as M
    omodel, vs = M.build(seed=42, dtype=torch.float32, input_hw=min(hw, 64), **kw, **build_kw)
    if seed_bn is not None:
        _randomise_bn(vs, seed_bn)
    for n in vs.vars:
        vs.vars[n] = vs.vars[n].to(dt)
    vs.dtype = dt
    return omodel, vs


def test_c1_vanilla_resnet50_eval_batch1_224():
    """BASELINE config 1: vanilla ResNet-50 (rv=1), eval forward, batch 1, 224 x 224."""
    from assembled_cnn_b200.model_fns import build_model
    from oracle import model as M
    kw = dict(resnet_size=50, resnet_version=1)
    x, _, _ = _inputs(1, 224, seed=5)
    want = {}
    for dt in (torch.float32, torch.float64):
        omodel, vs = _oracle_vars(kw, 224, dt, seed_bn=11)
        want[dt] = M.forward(omodel, vs, x.to(dt), training=False).detach()
    _, vs32 = _oracle_vars(kw, 224, torch.float32, seed_bn=11)
    errs = {}
    for dtype in ("fp32", "bf16"):
        model = build_model(dtype=dtype, **kw)
        model.set_weights(vs32.vars)
        logits = model(x, training=False).float().cpu()
        assert logits.shape == (1, 1001)
        errs[dtype] = (_nrel(logits, want[torch.float32]), _nrel(logits, want[torch.float64]))
    print("C1 eval logits norm-rel: fp32 mode %.2e (vs fp32 oracle) %.2e (vs fp64 oracle); "
          "bf16 mode %.2e / %.2e; oracle fp32-vs-fp64 %.2e"
          % (errs["fp32"] + errs["bf16"] + (_nrel(want[torch.float32], want[torch.float64]),)))
    assert errs["fp32"][0] < TOL and errs["fp32"][1] < TOL
    assert errs["bf16"][1] < 3e-2


def test_c2_assemble_forward_and_loss():
    """BASELINE config 2 family: Assemble-ResNet-50 forward + loss.  Training-mode forward (batch
    statistics) through Model.__call__, and the EVAL loss (CE + L2) through model_fn_cls."""
    from assembled_cnn_b200 import model_fns as F
    from oracle import model as M
    hw, B = 128, 8
    x, lab, _ = _inputs(B, hw, seed=2)
    onehot = torch.nn.functional.one_hot(lab.long(), 1001)
    ref = {}
    for dt in (torch.float32, torch.float64):
        omodel, vs = _oracle_vars(ASSEMBLE, hw, dt, seed_bn=21)
        tr_logits = M.forward(omodel, vs, x.to(dt), training=True).detach()
        loss, ce, l2, ev_logits = M.loss_fn(omodel, vs, x.to(dt), onehot.to(dt), training=False,
                                            label_smoothing=0.1, weight_decay=1e-4)
        ref[dt] = (tr_logits, ev_logits.detach(), float(ce), float(l2))
    _, vs32 = _oracle_vars(ASSEMBLE, hw, torch.float32, seed_bn=21)
    for dtype in ("fp32", "bf16"):
        model = F.Model(50, num_classes=1001, resnet_version=2, use_sk_block=True,
                        anti_alias_type="sconv", anti_alias_filter_size=3, dtype=dtype)
        model.set_weights(vs32.vars)
        got_tr = model(x, training=True).float().cpu()
        e32, e64 = _nrel(got_tr, ref[torch.float32][0]), _nrel(got_tr, ref[torch.float64][0])
        # EVAL-mode forward + loss (moving statistics) on the same model
        model.set_weights(vs32.vars)          # the training-mode call moved the moving statistics
        rt = model.runtime(B, hw, hw, training=False, label_smoothing=0.1, with_loss=True)
        m = rt.plan.meta
        rt.t[m["images"]].copy_(x)
        rt.t[m["labels"]].copy_(lab)
        rt.run_forward()
        ce = float(rt.slot_view(m["loss"])[0])
        ev = rt.t[m["logits"]][:, :1001].float().cpu()
        print("C2 %s mode: train-mode logits %.2e / %.2e (vs fp32 / fp64 oracle); eval logits %.2e; "
              "CE %.6f vs %.6f" % (dtype, e32, e64, _nrel(ev, ref[torch.float64][1]), ce,
                                   ref[torch.float64][2]))
        if dtype == "fp32":
            assert e32 < TOL and e64 < TOL
            assert _nrel(ev, ref[torch.float64][1]) < TOL
            assert abs(ce - ref[torch.float64][2]) < TOL * abs(ref[torch.float64][2])
            assert abs(ce - ref[torch.float32][2]) < TOL * abs(ref[torch.float32][2])
        else:
            assert _nrel(ev, ref[torch.float64][1]) < 3e-2


def test_c2_full_size_batch256_224():
    """BASELINE config 2 AT ITS OWN SIZE: Assemble-ResNet-50 forward + loss, batch 256, 224 x 224,
    against the fp32 CPU oracle run on the same 256 images (forward only, torch.no_grad: seconds).
      * fp32 mode, eval-mode forward + loss at batch 256: logits and CE within 1e-3;
      * fp32 mode, training-mode forward (batch statistics) at batch 64 (its training runtime at 256
        would not leave room for the other models of this test): logits within 1e-3;
      * bf16 production mode at batch 256 -- the benchmarked configuration: training-mode logits and
        eval-mode logits / CE, reported and bounded (bf16 storage: ~1e-2)."""
    import gc
    from assembled_cnn_b200 import model_fns as F
    from oracle import model as M
    hw, B, Bs = 224, 256, 64
    x, lab, _ = _inputs(B, hw, seed=12)
    onehot = torch.nn.functional.one_hot(lab.long(), 1001).float()
    omodel, vs = _oracle_vars(ASSEMBLE, hw, torch.float32, seed_bn=23)
    with torch.no_grad():
        ref_tr = M.forward(omodel, vs, x, training=True)
        ref_tr_s = M.forward(omodel, vs, x[:Bs], training=True)
        _, ref_ce, _, ref_ev = M.loss_fn(omodel, vs, x, onehot, training=False, label_smoothing=0.1,
                                         weight_decay=1e-4)
    ref_ce = float(ref_ce)
    _, vs32 = _oracle_vars(ASSEMBLE, hw, torch.float32, seed_bn=23)

    def eval_forward(model):
        rt = model.runtime(B, hw, hw, training=False, label_smoothing=0.1, with_loss=True)
        m = rt.plan.meta
        rt.t[m["images"]].copy_(x)
        rt.t[m["labels"]].copy_(lab)
        rt.run_forward()
        return rt.t[m["logits"]][:, :1001].float().cpu(), float(rt.slot_view(m["loss"])[0])

    ctor = dict(num_classes=1001, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)
    # fp32 mode
    model = F.Model(50, dtype="fp32", **ctor)
    model.set_weights(vs32.vars)
    ev, ce = eval_forward(model)
    e_ev, e_ce = _nrel(ev, ref_ev), abs(ce - ref_ce) / abs(ref_ce)
    got = model(x[:Bs], training=True).float().cpu()
    e_tr = _nrel(got, ref_tr_s)
    print("C2 full size, fp32 mode: eval logits B=256 %.2e, CE %.6f vs %.6f (rel %.2e); training-mode "
          "logits B=64 %.2e" % (e_ev, ce, ref_ce, e_ce, e_tr))
    assert e_ev < TOL and e_ce < TOL and e_tr < TOL
    del model
    gc.collect()
    torch.cuda.empty_cache()
    # bf16 production mode, batch 256
    model = F.Model(50, dtype="bf16", **ctor)
    model.set_weights(vs32.vars)
    ev, ce = eval_forward(model)
    got = model(x, training=True).float().cpu()
    b_ev, b_ce, b_tr = _nrel(ev, ref_ev), abs(ce - ref_ce) / abs(ref_ce), _nrel(got, ref_tr)
    print("C2 full size, bf16 mode B=256: eval logits %.2e, CE rel %.2e; training-mode logits %.2e; "
          "argmax agreement eval %.3f / train %.3f"
          % (b_ev, b_ce, b_tr, float((ev.argmax(1) == ref_ev.argmax(1)).float().mean()),
             float((got.argmax(1) == ref_tr.argmax(1)).float().mean())))
    assert b_ev < 3e-2 and b_ce < 1e-2 and b_tr < 1e-1
    del model
    gc.collect()
    torch.cuda.empty_cache()


def _train_step_parity(kw, model_ctor_kw, B, hw, label, e2e_grad_check=True):
    from assembled_cnn_b200.model_fns import Model, Trainer
    from assembled_cnn_b200.hparams import params_from_flags
    from oracle import model as M, plan_interp as PI, tf_ops as T
    x, lab, g = _inputs(2 * B, hw, seed=0)
    lam = torch.rand(B, generator=g)
    onehot = torch.nn.functional.one_hot(lab.long(), 1001)
    hp = dict(lr=0.05, momentum=0.9, weight_decay=1e-4)

    # ---- autograd oracle, fp32 and fp64 -------------------------------------------------------
    ref = {}
    for dt in (torch.float32, torch.float64):
        omodel, vs = _oracle_vars(kw, hw, dt)
        names = [n for n in vs.vars if vs.trainable[n]]
        mom = {n: torch.zeros_like(vs.vars[n]) for n in names}
        before = {n: vs.vars[n].clone() for n in vs.vars}
        xm, ym = T.mixup(x.to(dt), onehot.to(dt), lam.to(dt), keep_batch_size=False)
        out = M.train_step(omodel, vs, mom, xm, ym, lr=hp["lr"], momentum=hp["momentum"],
                           label_smoothing=0.1, weight_decay=hp["weight_decay"])
        # product convention: rt.grads excludes the weight-decay term (folded into the SGD kernel)
        grads = {n: out["grads"][n] - (hp["weight_decay"] * before[n] if M.decayed(n) else 0)
                 for n in names}
        ref[dt] = dict(out=out, grads=grads, after={n: vs.vars[n].clone() for n in vs.vars})
    r32, r64 = ref[torch.float32], ref[torch.float64]
    _, vs32 = _oracle_vars(kw, hw, torch.float32)
    names = list(r64["grads"])

    results = {}
    for dtype in ("fp32", "bf16"):
        model = Model(kw["resnet_size"], num_classes=1001, dtype=dtype, **model_ctor_kw)
        model.set_weights(vs32.vars)
        params = params_from_flags(batch_size=B, mixup_type=1, label_smoothing=0.1,
                                   weight_decay=hp["weight_decay"], base_learning_rate=hp["lr"],
                                   learning_rate_decay_type="fixed", dtype=dtype, **kw)
        tr = Trainer(model, params, hw, hw, use_cuda_graph=False)
        rt = tr.rt
        loss = tr.train_step(x, lab, lam1=lam).tolist()
        torch.cuda.synchronize()
        m = rt.plan.meta
        logits = rt.t[m["logits"]][:, :1001].float().cpu()
        grads = {n: rt.get_tf(n, rt.grads).float().cpu().clone() for n in names}
        after = model.get_weights()
        results[dtype] = dict(loss=loss, logits=logits, grads=grads, after=after, rt=rt, tr=tr)

    # ---- forward quantities: tight against both oracles ----------------------------------------
    for dtype in ("fp32", "bf16"):
        r = results[dtype]
        e_log = (_nrel(r["logits"], r32["out"]["logits"]), _nrel(r["logits"], r64["out"]["logits"]))
        ce64, l264 = float(r64["out"]["cross_entropy"]), float(r64["out"]["l2_loss"])
        e_ce = abs(r["loss"][0] - ce64) / abs(ce64)
        e_l2 = abs(r["loss"][1] - l264) / abs(l264)
        e_mm = max(_nrel(r["after"][n], r64["after"][n]) for n in r64["after"]
                   if n.endswith("moving_mean") or n.endswith("moving_variance"))
        ge = sorted(((_nrel(r["grads"][n], r64["grads"][n]), n) for n in names), reverse=True)
        print("%s %s mode: logits %.2e / %.2e (vs fp32 / fp64 oracle), CE rel %.2e, L2 rel %.2e, "
              "moving stats worst %.2e, e2e gradients vs fp64 oracle worst %.2e median %.2e"
              % (label, dtype, e_log[0], e_log[1], e_ce, e_l2, e_mm, ge[0][0], ge[len(ge) // 2][0]))
        if dtype == "fp32":
            assert e_log[0] < TOL and e_log[1] < TOL, e_log
            assert e_ce < TOL and e_l2 < TOL
            assert abs(r["loss"][0] - float(r32["out"]["cross_entropy"])) < TOL * abs(ce64)
            assert e_mm < TOL
        else:
            assert e_l2 < 1e-4

    # ---- gradients, end to end, against the oracle's own fp32 round-off yardstick --------------
    r = results["fp32"]
    if e2e_grad_check:
        yard = {n: _nrel(r32["grads"][n], r64["grads"][n]) for n in names}
        ys = sorted(yard.values())
        print("%s oracle fp32-vs-fp64 gradient yardstick: worst %.2e median %.2e"
              % (label, ys[-1], ys[len(ys) // 2]))
        bad = []
        for n in names:
            e = _nrel(r["grads"][n], r64["grads"][n])
            if not (e <= max(TOL, 4.0 * yard[n])) and r64["grads"][n].abs().max() > 1e-12:
                bad.append((n, e, yard[n]))
        assert not bad, bad[:10]
        # SGD-updated weights (momentum step on those gradients).  Variables that start at zero
        # (beta, dense bias) ARE lr * gradient afterwards, so the same yardstick applies
        bad_w, worst_w = [], 0.0
        for n in names:
            e = _nrel(r["after"][n], r64["after"][n])
            yw = _nrel(r32["after"][n], r64["after"][n])
            worst_w = max(worst_w, e)
            if not (e <= max(TOL, 4.0 * yw)):
                bad_w.append((n, e, yw))
        print("%s fp32 mode: updated weights worst norm-rel %.2e" % (label, worst_w))
        assert not bad_w, bad_w[:10]

    # ---- gradients, backward given the forward: the CUDA backward chain vs the fp64 interpreter
    #      on the same forward activations (identical ReLU masks) ---------------------------------
    for dtype in ("fp32", "bf16"):
        rt = results[dtype]["rt"]
        plan = rt.plan
        # the oracle's interpreter walks the Python plan: the same plan as the library's, op for op
        # (tests/test_native_plan_cpu.py)
        pyplan = plan.python_mirror()
        it = PI.PlanInterpreter(pyplan, dtype=torch.float64, emulate_bf16=False)
        # re-run forward + backward on the GPU from the ORIGINAL weights (the step above updated them)
        rt.set_weights(vs32.vars)
        it.set_weights(vs32.vars)
        m = plan.meta
        rt.t[m["images"]].copy_(x)
        rt.t[m["labels"]].copy_(lab)
        rt.t[m["lam1"]].copy_(lam)
        rt.run_forward()
        torch.cuda.synchronize()
        for name, t in plan.tensors.items():
            if name.startswith("planes"):
                continue
            v = rt.t[name]
            it.t[name] = v.cpu() if not v.is_floating_point() else v.double().cpu()
        it.work.copy_(rt.work.double().cpu())
        it.zero.copy_(rt.zero.double().cpu())
        it.state.copy_(rt.state.double().cpu())
        it.hp.update(grad_scale=1.0)
        rt.run(plan.backward)
        torch.cuda.synchronize()
        it.grads.zero_()
        # dbias is accumulated by the forward's softmax_ce op on both sides
        it.run([op for op in pyplan.forward if op.kind == "softmax_ce"])
        it.run(pyplan.backward)
        ge = sorted(((_nrel(rt.get_tf(n, rt.grads), it.get_tf(n, it.grads)), n) for n in names),
                    reverse=True)
        print("%s %s mode: backward given the forward, all %d gradient tensors: worst %.2e (%s) "
              "median %.2e" % (label, dtype, len(ge), ge[0][0], ge[0][1], ge[len(ge) // 2][0]))
        if dtype == "fp32":
            assert ge[0][0] < TOL, ge[:5]
    return results


def test_c3_assemble_train_step_all_gradients():
    """BASELINE config 3: Assemble-ResNet-50 full training step, mixup type 1 + label smoothing,
    batch 8, 128 x 128."""
    ctor = dict(resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)
    _train_step_parity(ASSEMBLE, ctor, B=8, hw=128, label="C3")


def test_c5_assemble_r152_topology():
    """BASELINE config 5 topology: Assemble-ResNet-152 (bl_alpha=1, bl_beta=2), batch 8, 128 px."""
    ctor = dict(resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3, bl_alpha=1, bl_beta=2)
    _train_step_parity(R152, ctor, B=8, hw=128, label="C5")


def test_fp32_mode_two_runs_bit_identical():
    """All reductions are ordered (partial rows + fixed-order sums), wgrad / the small fc GEMMs run
    without split-K: the same step twice gives bit-identical loss, gradients and weights."""
    from assembled_cnn_b200.model_fns import Model, Trainer
    from assembled_cnn_b200.hparams import params_from_flags
    B, hw = 8, 128
    x, lab, g = _inputs(2 * B, hw, seed=4)
    lam = torch.rand(B, generator=g)
    outs = []
    for run in range(2):
        model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True,
                      anti_alias_type="sconv", anti_alias_filter_size=3, dtype="fp32", seed=42)
        params = params_from_flags(batch_size=B, mixup_type=1, label_smoothing=0.1,
                                   weight_decay=1e-4, base_learning_rate=0.05,
                                   learning_rate_decay_type="fixed", dtype="fp32", **ASSEMBLE)
        tr = Trainer(model, params, hw, hw, use_cuda_graph=(run == 1))
        l1 = tr.train_step(x, lab, lam1=lam).clone()
        l2 = tr.train_step(x, lab, lam1=lam).clone()
        torch.cuda.synchronize()
        outs.append((l1.cpu(), l2.cpu(), tr.rt.grads.cpu().clone(), tr.rt.params.cpu().clone(),
                     tr.rt.state.cpu().clone()))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)


def test_bf16_mode_forward_and_bn_reductions_bit_identical():
    """bf16 production mode (deterministic=None): every reduction is ordered -- the batch-norm
    partial rows, the split-K wgrad and the SK / SE GEMMs, whose partials are added in split order.
    Two eager steps and a CUDA-graph replay of the step give bit-identical loss, logits, BN
    statistics, gradients, weights and momentum."""
    _bf16_step_bit_identical(deterministic=None)


def test_bf16_mode_forward_and_bn_reductions_bit_identical_deterministic():
    """The same with deterministic=True (one split everywhere)."""
    _bf16_step_bit_identical(deterministic=True)


def _bf16_step_bit_identical(deterministic):
    import ctypes as C
    from assembled_cnn_b200.native import NativeModel, NativeRuntime
    from assembled_cnn_b200.plan import ModelConfig
    B, hw = 8, 128
    x, lab, g = _inputs(2 * B, hw, seed=4)
    lam = torch.rand(B, generator=g)
    outs = []
    for run in ("eager", "eager", "graph"):
        plan = NativeModel(ModelConfig(**ASSEMBLE), B, hw, hw, training=True, mixup_type=1,
                           label_smoothing=0.1, deterministic=deterministic)
        rt = NativeRuntime(plan)
        torch.manual_seed(0)
        rt.params.copy_(torch.randn(rt.params.shape, generator=torch.Generator().manual_seed(1)) * 0.05)
        for p in plan.params.values():
            if p.kind == "gamma":
                rt.pview(p.name).fill_(1.0)
        m = plan.meta
        rt.t[m["images"]].copy_(x)
        rt.t[m["labels"]].copy_(lab)
        rt.t[m["lam1"]].copy_(lam)
        rt.set_hparams(lr=0.05, momentum=0.9, weight_decay=1e-4, grad_scale=1.0)
        if run == "graph":
            rt.capture(train=True)
            rt.graph.replay()
        else:
            rt.run_step()
        torch.cuda.synchronize()
        outs.append((rt.slot_view(m["loss"]).cpu().clone(), rt.t[m["logits"]].cpu().clone(),
                     rt.state.cpu().clone(), rt.grads.cpu().clone(), rt.params.cpu().clone(),
                     rt.momentum.cpu().clone()))
    for other in outs[1:]:
        for a, b, what in zip(outs[0], other, ("loss", "logits", "moving statistics", "gradients",
                                                "weights", "momentum")):
            assert torch.equal(a, b), what
    # the default mode really ran split-K wgrads (acnn_conv_wgrad_plan: the layout the launcher uses)
    n_split = 0
    for op in plan.backward:
        if op.kind == "conv_wgrad":
            splits = C.c_int()
            assert rt.lib.acnn_conv_wgrad_plan(plan.conv_info(op)[0], 0, rt.det, None,
                                               C.byref(splits), None) == 0
            n_split += splits.value > 1
    assert (n_split > 0) == (not deterministic), n_split
