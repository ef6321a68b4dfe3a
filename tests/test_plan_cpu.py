"""CPU checks of the product's layer plan (no GPU, no kernels): the plan's topology, parameter
inventory / order / names, explicit backward emission and SGD are validated by running it through
the torch interpreter (oracle/plan_interp.py) and comparing logits, loss, every gradient and every
updated variable with the autograd oracle (oracle/model.py) in float64.

Tolerance 1e-6 relative (the only fp32 step is the reference's cast of the logits before the loss,
nets/run_loop_classification.py:123)."""
import pytest
import torch

from assembled_cnn_b200.plan import ModelConfig, build_plan
from oracle import model as M
from oracle import plan_interp as PI
from oracle import tf_ops as T

ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)

CASES = {
    # name: (model kwargs, use_resnet_d, mixup_type, input size)
    "vanilla_rv1": (dict(resnet_size=50, resnet_version=1), False, 0, 32),
    "assemble_rv2_mix1": (ASSEMBLE, False, 1, 64),
    "rv1_d_sk_sconv_mix2": (dict(resnet_size=50, resnet_version=1, use_sk_block=True,
                                 anti_alias_type="sconv", anti_alias_filter_size=3), True, 2, 32),
    "rv2_se_proj5": (dict(resnet_size=50, resnet_version=2, use_se_block=True,
                          anti_alias_type="proj", anti_alias_filter_size=5), False, 0, 32),
    "rv2_d_zero_gamma": (dict(zero_gamma=True, **ASSEMBLE), True, 0, 32),
}


def _setup(kw, d, mix, hw, B=4, dtype=torch.float64, training=True, plan_dtype="bf16"):
    cfg = ModelConfig(use_resnet_d=d, **kw)
    plan = build_plan(cfg, B, hw, hw, training=training, mixup_type=mix, label_smoothing=0.1,
                      dtype=plan_dtype)
    model, vs = M.build(seed=42, dtype=dtype, input_hw=hw, use_resnet_d=d, **kw)
    g = torch.Generator().manual_seed(1)
    for n in vs.vars:
        if n.endswith("gamma") and not kw.get("zero_gamma"):
            vs.vars[n] = (0.5 + torch.rand(vs.vars[n].shape, generator=g)).to(dtype)
        if n.endswith("beta"):
            vs.vars[n] = (0.1 * torch.randn(vs.vars[n].shape, generator=g)).to(dtype)
    it = PI.PlanInterpreter(plan, dtype=dtype)
    it.set_weights(vs.vars)
    Bin = plan.meta["input_batch"]
    x = (torch.randn(Bin, hw, hw, 3, generator=g) * 64).clamp(-124, 152).to(dtype)
    lab = torch.randint(1, 1001, (Bin,), generator=g).int()
    lam1 = torch.rand(Bin // 2, generator=g).to(dtype) if mix else None
    lam2 = torch.rand(Bin // 2, generator=g).to(dtype) if mix == 2 else None
    return plan, model, vs, it, x, lab, lam1, lam2


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("plan_dtype", ["bf16", "fp32"])
@pytest.mark.parametrize("name", list(CASES))
def test_plan_train_step_matches_autograd_oracle(name, plan_dtype):
    kw, d, mix, hw = CASES[name]
    if plan_dtype == "fp32" and name not in ("assemble_rv2_mix1", "rv1_d_sk_sconv_mix2",
                                             "rv2_se_proj5"):
        pytest.skip("fp32 plan: three configurations cover every op kind")
    _check_train_step(kw, d, mix, hw, 4, plan_dtype)


def _check_train_step(kw, d, mix, hw, B, plan_dtype):
    plan, model, vs, it, x, lab, lam1, lam2 = _setup(kw, d, mix, hw, B=B, plan_dtype=plan_dtype)
    if plan_dtype == "fp32":
        # the parity mode's plan: fp32 tensors, operand planes, two-pass statistics, unfused
        # dgrad epilogue -- same mathematics
        assert plan.meta["dtype"] == "fp32"
        assert any(o.kind == "split3" for o in plan.forward)
        assert any(o.kind == "bn_stats" for o in plan.forward)
        assert all(t.dtype != "bf16" or n.startswith("planes") for n, t in plan.tensors.items())
    names = [n for n in vs.vars if vs.trainable[n]]
    # same variables, same creation order, same TF-style names
    assert names == list(plan.params)
    assert [n for n in vs.vars if not vs.trainable[n]] == list(plan.state)
    for n, p in plan.params.items():
        assert tuple(vs.vars[n].shape) == p.tf_shape
        assert p.decay == M.decayed(n)
    hp = dict(lr=0.05, momentum=0.9, weight_decay=1e-4)
    it.hp.update(hp)
    logits, ce, l2 = it.train_step(x, lab, lam1, lam2)

    onehot = torch.nn.functional.one_hot(lab.long(), 1001).to(x.dtype)
    xo, yo = (x, onehot) if not mix else T.mixup(x, onehot, lam1, lam2, keep_batch_size=(mix == 2))
    mom = {n: torch.zeros_like(vs.vars[n]) for n in names}
    before = {n: vs.vars[n].clone() for n in vs.vars}
    out = M.train_step(model, vs, mom, xo, yo, lr=0.05, momentum=0.9, use_resnet_d=d,
                       label_smoothing=0.1, weight_decay=1e-4)
    assert _rel(logits, out["logits"]) < 1e-6
    assert abs(ce - out["cross_entropy"].item()) < 1e-6
    assert abs(l2 - out["l2_loss"].item()) < 1e-6
    for n in names:
        want = out["grads"][n] - (1e-4 * before[n] if M.decayed(n) else 0)
        got = it.get_tf(n, it.grads)
        err = ((got - want).norm() / want.norm().clamp_min(1e-30)).item()
        assert err < 1e-5 or (got - want).abs().max() < 1e-9, (n, err)
    for n in vs.vars:   # weights after the momentum step and BN moving statistics
        assert (it.get_tf(n) - vs.vars[n]).abs().max().item() <= 1e-6 * max(
            vs.vars[n].abs().max().item(), 1.0), n


def test_plan_eval_forward_matches_oracle():
    plan, model, vs, it, x, lab, _, _ = _setup(ASSEMBLE, False, 0, 64, B=2, training=False)
    g = torch.Generator().manual_seed(5)
    for n in vs.vars:       # make the moving statistics matter
        if n.endswith("moving_mean"):
            vs.vars[n] = 0.1 * torch.randn(vs.vars[n].shape, generator=g).double()
        if n.endswith("moving_variance"):
            vs.vars[n] = (0.5 + torch.rand(vs.vars[n].shape, generator=g)).double()
    it.set_weights(vs.vars)
    assert not plan.backward and not plan.update
    logits = it.forward(x, lab)
    want = M.forward(model, vs, x, training=False)
    assert _rel(logits, want) < 1e-9


def test_bench_model_inventory():
    """Assemble-ResNet-50 at the BASELINE shape: op counts, launch-relevant shapes, param totals."""
    cfg = ModelConfig(**ASSEMBLE)
    plan = build_plan(cfg, 8, 224, 224, training=True, mixup_type=1, label_smoothing=0.1)
    convs = [o for o in plan.forward if o.kind == "conv"]
    assert len(convs) == 76 + 1                       # 76 spatial convs + dense
    assert sum(1 for o in plan.forward if o.kind == "sk_fc") == 19
    assert sum(1 for o in plan.forward if o.kind == "blurpool") == 6
    assert sum(1 for o in plan.forward if o.kind == "avgpool") == 6
    assert len(plan.params) == 306
    n_tf = sum(torch.Size(p.tf_shape).numel() for p in plan.params.values())
    assert n_tf == 41_848_489
    assert plan.meta["input_batch"] == 16
    macs = sum(o.geom.B * o.geom.Ho * o.geom.Wo * o.geom.Cout * o.geom.kh * o.geom.kw * o.geom.Cin
               for o in convs)
    # stem runs as a 4x4x16 space-to-depth conv (256 instead of 147 MACs per output) -- a little
    # more than the reference's 5.726 GMAC/img
    assert 5.7e9 < macs / 8 < 5.9e9


def test_assemble_r152_inventory():
    """BASELINE config 5: Assemble-ResNet-152 (rv=2, bl_alpha=1, bl_beta=2)."""
    cfg = ModelConfig(resnet_size=152, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                      anti_alias_filter_size=3, bl_alpha=1, bl_beta=2)
    plan = build_plan(cfg, 2, 224, 224, training=True, mixup_type=1)
    assert len(plan.params) == 969
    assert sum(torch.Size(p.tf_shape).numel() for p in plan.params.values()) == 117_006_249
    assert sum(1 for o in plan.forward if o.kind == "conv") == 229 + 1
    assert sum(1 for o in plan.forward if o.kind == "sk_fc") == 70
    assert len(plan.bns) == 299


def test_flag_validation_errors_match_reference():
    with pytest.raises(ValueError):
        ModelConfig(resnet_version=3).validate()
    with pytest.raises(NotImplementedError):
        ModelConfig(resnet_size=18).validate()
    with pytest.raises(ValueError):
        ModelConfig(resnet_size=77).validate()
    with pytest.raises(NotImplementedError):
        ModelConfig(pool_type="max").validate()
    ModelConfig(pool_type="gem", embedding_size=256).validate()      # supported
    with pytest.raises(ValueError):
        ModelConfig(embedding_size=100).validate()


# --------------------------------------------------------------------------------------------------
# The same check over the flag space (hypothesis, derandomised): whatever combination of the reference's
# flags is requested, the plan's forward, EXPLICIT backward and SGD step agree with autograd through the
# oracle in float64 -- shortcut kinds x SK / SE x anti-alias variants and filter sizes x pooling / embedding
# heads x BigLittle widths x mixup types x storage modes.
# --------------------------------------------------------------------------------------------------
from hypothesis import given, settings, strategies as st, HealthCheck


@st.composite
def _train_flag_sets(draw):
    version = draw(st.sampled_from([1, 2]))
    kw = dict(resnet_size=50, resnet_version=version,
              use_sk_block=draw(st.booleans()), use_se_block=draw(st.booleans()),
              zero_gamma=draw(st.booleans()) and draw(st.booleans()),
              no_downsample=draw(st.booleans()),
              anti_alias_type=draw(st.sampled_from(["", "sconv", "proj", "sconv,proj"])),
              anti_alias_filter_size=draw(st.sampled_from([1, 2, 3, 4, 5, 7])),
              pool_type=draw(st.sampled_from(["gap", "gap", "gem", "flatten"])),
              embedding_size=draw(st.sampled_from([0, 0, 32, 64])),
              bl_alpha=draw(st.sampled_from([1, 2])), bl_beta=draw(st.sampled_from([1, 2, 4])))
    # 64 px: the stride-2 blur-pools of the last stage see 4x4 maps (REFLECT padding needs pad < size)
    return (kw, draw(st.booleans()), draw(st.sampled_from([0, 1, 2])), 64,
            # batch >= 4: with 2 samples and 1x1 stage-4 maps at 32 px the batch norms see two values per
            # channel (x-hat = +-1) and the gradients are ill-conditioned even in float64
            draw(st.sampled_from([4, 6])), draw(st.sampled_from(["bf16", "fp32"])))


@settings(max_examples=5, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(_train_flag_sets())
def test_plan_train_step_matches_autograd_oracle_over_the_flag_space(case):
    kw, d, mix, hw, B, plan_dtype = case
    if mix == 2 and B % 2:
        B += 1                      # mixup type 2 mixes the two halves of the batch
    _check_train_step(kw, d, mix, hw, B, plan_dtype)
