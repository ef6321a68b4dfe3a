"""CPU checks of the extra features (no GPU): the layer plan of DropBlock, the KD loss term, GeM /
flatten pooling and the embedding head against the autograd oracle (float64, 1e-6); the ECE metric;
checkpoint naming, the warm-start filter and the best-checkpoint keeper; the data-parallel bucket
schedule."""
import json
import os

import numpy as np
import pytest
import torch

from assembled_cnn_b200.plan import ModelConfig, build_plan
from oracle import model as M
from oracle import plan_interp as PI
from oracle import tf_ops as T

ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)


def _step_vs_autograd(kw, hw, B, mix=0, use_db=False, kd=0.0, plan_dtype="bf16", kp=0.9):
    dt = torch.float64
    plan = build_plan(ModelConfig(**kw), B, hw, hw, training=True, mixup_type=mix,
                      label_smoothing=0.1, dtype=plan_dtype, use_dropblock=use_db, kd_temp=kd)
    model, vs = M.build(seed=42, dtype=dt, input_hw=min(hw, 64), **kw)
    g = torch.Generator().manual_seed(1)
    for n in vs.vars:
        if n.endswith("gamma"):
            vs.vars[n] = (0.5 + torch.rand(vs.vars[n].shape, generator=g)).to(dt)
        if n.endswith("beta"):
            vs.vars[n] = (0.1 * torch.randn(vs.vars[n].shape, generator=g)).to(dt)
    it = PI.PlanInterpreter(plan, dtype=dt)
    it.set_weights(vs.vars)
    names = [n for n in vs.vars if vs.trainable[n]]
    assert names == list(plan.params)                 # same variables, same creation order
    assert [n for n in vs.vars if not vs.trainable[n]] == list(plan.state)
    Bin = plan.meta["input_batch"]
    x = (torch.randn(Bin, hw, hw, 3, generator=g) * 64).clamp(-124, 152).to(dt)
    lab = torch.randint(1, 1001, (Bin,), generator=g).int()
    lam1 = torch.rand(Bin // 2, generator=g).to(dt) if mix else None
    lam2 = torch.rand(Bin // 2, generator=g).to(dt) if mix == 2 else None
    us = []
    for name in plan.meta["dropblock_u"]:
        u = torch.rand(plan.tensors[name].shape, generator=g).to(dt)
        it.t[name] = u
        us.append(u[None])
    tl = None
    if kd > 0:
        tl = 3 * torch.randn(Bin, 1001, generator=g).to(dt)
        it.t[plan.meta["teacher_logits"]] = tl
    it.hp.update(lr=0.05, momentum=0.9, weight_decay=1e-4, keep_prob=kp)
    logits, ce, l2 = it.train_step(x, lab, lam1, lam2)
    kd_got = it.slot(plan.meta["loss"])[2].item()
    onehot = torch.nn.functional.one_hot(lab.long(), 1001).to(dt)
    teacher = torch.softmax(tl / kd, 1) if kd > 0 else None
    xo, yo = x, onehot
    if mix:
        r = T.mixup(x, onehot, lam1, lam2, keep_batch_size=(mix == 2), y_t=teacher)
        xo, yo = r[0], r[1]
        teacher = r[2] if kd > 0 else None
    mom = {n: torch.zeros_like(vs.vars[n]) for n in names}
    before = {n: vs.vars[n].clone() for n in vs.vars}
    out = M.train_step(model, vs, mom, xo, yo, lr=0.05, momentum=0.9, label_smoothing=0.1,
                       weight_decay=1e-4, teacher_labels=teacher, kd_temp=kd,
                       keep_prob=kp if use_db else 1.0, dropblock_u=list(us))
    assert ((logits - out["logits"]).abs().max() / out["logits"].abs().max()).item() < 1e-6
    assert abs(ce - out["cross_entropy"].item()) < 1e-6
    if kd > 0:
        assert abs(kd_got - float(out["kd_loss"])) < 1e-5 * abs(float(out["kd_loss"]))
    for n in names:
        want = out["grads"][n] - (1e-4 * before[n] if M.decayed(n) else 0)
        got = it.get_tf(n, it.grads)
        err = ((got - want).norm() / want.norm().clamp_min(1e-30)).item()
        assert err < 1e-5 or (got - want).abs().max() < 1e-9, (n, err)
    for n in vs.vars:
        assert (it.get_tf(n) - vs.vars[n]).abs().max().item() <= 1e-6 * max(
            vs.vars[n].abs().max().item(), 1.0), n
    return plan, len(us)


def test_gem_embedding_kd_mixup2_plan_matches_autograd():
    """GeM pooling (nets/blocks.py:22-42) + embedding head (resnet_model.py:575-593) + KD loss with
    type-2 mixup of the teacher labels (run_loop_classification.py:86-96,156-162)."""
    plan, _ = _step_vs_autograd(dict(pool_type="gem", embedding_size=64, **ASSEMBLE), 64, 4, mix=2,
                                kd=2.0)
    assert "resnet_model/embedding_dense/kernel" in plan.params
    assert "resnet_model/embedding_dense_batch_normalization/gamma" in plan.params
    assert plan.params["resnet_model/embedding_dense/kernel"].decay
    assert not plan.params["resnet_model/embedding_dense_batch_normalization/gamma"].decay
    assert plan.params["resnet_model/dense/kernel"].tf_shape == (64, 1001)


def test_flatten_kd_fp32_plan_matches_autograd():
    plan, _ = _step_vs_autograd(dict(resnet_size=50, resnet_version=1, pool_type="flatten"), 64, 4,
                                mix=1, kd=1.0, plan_dtype="fp32")
    assert plan.params["resnet_model/dense/kernel"].tf_shape == (2 * 2 * 2048, 1001)


def test_dropblock_plan_matches_autograd():
    """DropBlock on the Assemble topology at 224 px: 34 masks (stage 3: gamma_scale 0.25 on big3 /
    little3 / merge3, stage 4: 1.0), drawn in the reference's call order."""
    plan, n = _step_vs_autograd(ASSEMBLE, 224, 2, use_db=True)
    assert n == 34
    scales = [op.gamma_scale for op in plan.forward if op.kind == "dropblock_mask"]
    assert scales.count(1.0) == 3 * 3 + 1 and scales.count(0.25) == n - 10
    with pytest.raises(ValueError):          # 128 px: the stage-4 map (4x4) is smaller than the block
        build_plan(ModelConfig(**ASSEMBLE), 2, 128, 128, training=True, use_dropblock=True)
    # inference ignores DropBlock (nets/blocks.py:205)
    ev = build_plan(ModelConfig(**ASSEMBLE), 2, 128, 128, training=False, use_dropblock=True)
    assert not any(op.kind.startswith("dropblock") for op in ev.forward)


def test_dropblock_reference_semantics():
    """nets/blocks.py:191-251 on a hand-checkable case: one drawn centre zeroes a 3x3 block, the
    survivors are rescaled by size / kept."""
    x = torch.ones(2, 5, 5, 1)
    u = torch.ones(1, 3, 3, 1)
    u[0, 1, 1, 0] = 0.0                              # only the centre falls below gamma
    y = T.dropblock(x, 0.5, 3, 1.0, u)
    keep = torch.ones(5, 5)
    keep[1:4, 1:4] = 0
    assert torch.equal(y[0, :, :, 0] != 0, keep.bool()) and torch.equal(y[0], y[1])
    assert torch.allclose(y[0, 0, 0, 0], torch.tensor(25.0 / 16.0))
    assert T.dropblock(x, 1.0, 3, 1.0, u) is x       # keep_prob == 1.0 (float): identity


def test_ece_metric_matches_oracle():
    from assembled_cnn_b200.metrics import EvalMetrics
    g = torch.Generator().manual_seed(0)
    em = EvalMetrics()
    correct = csum = cnt = 0
    for _ in range(3):
        logits = 3 * torch.randn(64, 10, generator=g)
        lab = torch.randint(0, 10, (64,), generator=g)
        res = em.update(logits, lab)
        prob = torch.softmax(logits, 1)
        conf, pred = prob.max(1)
        _, c, s, n = T.ece(conf, pred, lab)
        correct, csum, cnt = correct + c, csum + s, cnt + n
    want = ((cnt / cnt.sum()) * (correct / (1e-7 + cnt) - csum / (1e-7 + cnt)).abs()).sum()
    assert abs(res["ece"] - float(want)) < 1e-6
    assert 0 <= res["accuracy"] <= res["accuracy_top_5"] <= 1


def test_warm_start_filter_and_checkpoint_keeper(tmp_path):
    from assembled_cnn_b200 import checkpoint as C
    plan = build_plan(ModelConfig(use_se_block=True, embedding_size=64, resnet_size=50,
                                  resnet_version=1), 2, 64, 64, training=True)
    names = list(plan.params)
    ws = C.warm_start_variables(names)
    # utils/hook_utils.py:36-44: classifier / embedding dense layers are NOT warm-started, the SE
    # block's dense layers are
    assert "resnet_model/dense/kernel" not in ws and "resnet_model/dense/bias" not in ws
    assert "resnet_model/embedding_dense/kernel" not in ws
    assert "resnet_model/embedding_dense_batch_normalization/gamma" not in ws
    assert any("se_block" in n and "seblock_dense_1" in n for n in ws)
    assert "resnet_model/conv2d/kernel" in ws and len(ws) == len(names) - 5
    # CheckpointKeeper (utils/checkpoint_utils.py): keep the 2 best by accuracy
    d = str(tmp_path)
    for step in (100, 200, 300, 400):
        np.savez(os.path.join(d, "model.ckpt-%d.npz" % step), x=np.zeros(1))
    keeper = C.CheckpointKeeper(d, num_to_keep=2, keep_epoch=True)
    for step, acc in ((100, 0.5), (200, 0.7), (300, 0.6), (400, 0.4)):
        keeper.save(acc, os.path.join(d, "model.ckpt-%d.npz" % step))
    best = json.load(open(keeper.best_checkpoints_file))
    assert best == {"model.ckpt-200": 0.7, "model.ckpt-300": 0.6}
    kept = sorted(os.listdir(os.path.join(d, "best")))
    assert kept == ["best_checkpoints", "model.ckpt-200.npz", "model.ckpt-300.npz"]
    assert len(os.listdir(os.path.join(d, "periodical"))) == 4
    assert C.latest_checkpoint(d).endswith("model.ckpt-400.npz")


def test_data_parallel_bucket_schedule():
    """assembled_cnn_b200/dp.py: the buckets tile the flat gradient buffer from its end, each is
    reduced only after its last writer, the final (un-overlappable) bucket is small."""
    from assembled_cnn_b200 import dp
    plan = build_plan(ModelConfig(**ASSEMBLE), 8, 224, 224, training=True, mixup_type=1)
    buckets = dp.grad_buckets(plan)
    segs = dp.backward_segments(plan, buckets)
    assert buckets[0][1] == plan.param_elems and buckets[-1][0] == 0
    assert all(a[0] == b[1] for a, b in zip(buckets[:-1], buckets[1:]))
    assert segs[0][0] == 0 and segs[-1][1] == len(plan.backward)
    assert all(a[1] == b[0] for a, b in zip(segs[:-1], segs[1:]))
    assert (buckets[-1][1] - buckets[-1][0]) < 0.05 * plan.param_elems
    writers = {}
    for i, op in enumerate(plan.backward):
        for key in ("w", "w1", "w2"):
            v = op.a.get(key)
            if op.kind in ("conv_wgrad", "sk_fc_bwd", "se_fc_bwd", "s2d_wgrad_unpack") \
                    and isinstance(v, str) and v in plan.params:
                writers[v] = i
    for (lo, hi, _), (a, b) in zip(buckets, segs):
        for n, i in writers.items():
            if lo <= plan.params[n].offset < hi:
                assert i < b, (n, i, b)        # written before the bucket's all-reduce
