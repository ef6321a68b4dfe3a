"""GPU checks of the extra features through the public surface (Model / Trainer / model_fn_cls):
DropBlock with the device RNG, the KD loss term, the embedding head, checkpoint round trips and the
EVAL-mode loss / metrics.  The kernels themselves are pinned op by op in tests/test_plan_gpu.py
(test_feature_rows_lockstep)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)


def _inputs(n, hw, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, hw, hw, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (n,), generator=g).int()
    return x, lab, g


def test_dropblock_device_rng(lib):
    """Philox masks: a pure function of (seed, step); ONE mask per call shared by the batch; the kept
    fraction follows gamma; keep_prob = 1 keeps everything; the renormalisation restores the mean."""
    from assembled_cnn_b200 import _lib
    H = W = 14
    C = 256
    dev = "cuda"
    n_scr = lib.acnn_dropblock_scratch_floats(H, W, C, 7)
    st = torch.cuda.current_stream().cuda_stream

    def mask(kp, step, seed=1234):
        hp = torch.zeros(8, device=dev)
        hp[4] = kp
        hp.view(torch.int32)[5] = step
        keep = torch.full((H, W, C), float("nan"), device=dev)
        scale = torch.zeros(1, device=dev)
        scratch = torch.zeros(n_scr, device=dev)
        _lib.check(lib.acnn_dropblock_mask(None, hp.data_ptr() + 16, hp.data_ptr() + 20, seed, 1.0, 7,
                                           keep.data_ptr(), scale.data_ptr(), scratch.data_ptr(),
                                           H, W, C, st), "dropblock_mask")
        torch.cuda.synchronize()
        return keep.cpu(), float(scale)

    k1, s1 = mask(0.9, 5)
    k2, s2 = mask(0.9, 5)
    k3, _ = mask(0.9, 6)
    k4, _ = mask(0.9, 5, seed=99)
    assert torch.equal(k1, k2) and s1 == s2                    # reproducible
    assert not torch.equal(k1, k3) and not torch.equal(k1, k4)   # step / seed change the mask
    assert set(k1.unique().tolist()) <= {0.0, 1.0}
    # every dropped cell lies in a full 7x7 block of zeros
    drop = (1 - k1).permute(2, 0, 1)[None]
    centres = torch.nn.functional.max_pool2d(-torch.nn.functional.max_pool2d(-drop, 7, 1), 1)
    assert (centres.sum() > 0)
    frac_dropped = 1 - k1.mean().item()
    gamma = 0.1 * (H * W) / 49 / ((H - 6) * (W - 6))
    expect = 1 - (1 - gamma) ** 49                              # interior cells: 49 candidate centres
    assert 0.3 * expect < frac_dropped < 1.2 * expect, (frac_dropped, expect)
    assert abs(s1 - k1.numel() / k1.sum().item()) < 1e-4 * s1
    k_all, s_all = mask(1.0, 5)
    assert k_all.min() == 1.0 and abs(s_all - 1.0) < 1e-6


def test_trainer_dropblock_kd_and_schedule():
    """One process, the reference's full regularisation recipe (scripts/train_assemble_from_scratch.sh:
    dropblock + KD T=1 + mixup 1 + label smoothing) at 224 px: finite 3-term loss, the keep_prob
    schedule of functions/model_fns.py:221-228 reaches the device, weights move."""
    from assembled_cnn_b200.model_fns import Model, Trainer, keep_prob_decay
    from assembled_cnn_b200.hparams import params_from_flags
    B = 4
    model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True,
                  anti_alias_type="sconv", anti_alias_filter_size=3)
    p = params_from_flags(batch_size=B, mixup_type=1, label_smoothing=0.1, weight_decay=1e-4,
                          base_learning_rate=0.01, learning_rate_decay_type="fixed",
                          use_dropblock=True, dropblock_kp=[1.0, 0.9], kd_temp=1, train_epochs=1,
                          **ASSEMBLE)
    tr = Trainer(model, p, 224, 224, use_cuda_graph=True)
    x, lab, g = _inputs(2 * B, 224)
    teacher = 2 * torch.randn(2 * B, 1001, generator=g)
    w0 = tr.rt.params.clone()
    losses = [tr.train_step(x, lab, teacher_logits=teacher).tolist() for _ in range(3)]
    assert all(len(l) == 3 and all(math.isfinite(v) for v in l) for l in losses)
    assert losses[0][2] > 0                                     # KD term present
    assert not torch.equal(w0, tr.rt.params)
    bpe = 1281167 / B
    want = keep_prob_decay(1.0, 0.9, int(1 * bpe))(2)
    assert abs(tr.last_keep_prob - want) < 1e-12
    assert abs(float(tr.rt.hp[4]) - want) < 1e-6
    assert int(tr.rt.hp.view(torch.int32)[5]) == 2
    # an explicit keep_prob makes the masks bite: compare the loss with DropBlock "off" (kp = 1)
    l_on = tr.train_step(x, lab, teacher_logits=teacher, keep_prob=0.5).tolist()
    assert math.isfinite(l_on[0])


def test_model_fn_cls_kd_labels_and_eval_loss():
    from assembled_cnn_b200 import model_fns as F
    from assembled_cnn_b200.hparams import params_from_flags
    params = params_from_flags(batch_size=4, label_smoothing=0.1, weight_decay=1e-4, kd_temp=2,
                               base_learning_rate=0.01, learning_rate_decay_type="fixed",
                               pool_type="gem", embedding_size=64, **ASSEMBLE)
    x, lab, g = _inputs(4, 64, seed=9)
    onehot = torch.nn.functional.one_hot(lab.long(), 1001).float()
    teacher = 2 * torch.randn(4, 1001, generator=g)
    kd_labels = torch.cat([onehot, teacher], 1)          # run_loop_classification.py:86-93
    spec = F.model_fn_cls({"image": x}, kd_labels, F.TRAIN, params)
    tr = spec.train_op
    ce, l2, kd = tr._loss_slot.tolist()
    assert abs(float(spec.loss) - (ce + l2 + kd)) < 1e-4 * abs(ce + l2 + kd)
    logits = spec.predictions["probabilities"].log()      # softmax is shift invariant
    t = torch.softmax(teacher.cuda() / 2, 1)
    want_kd = 4.0 * -(t * torch.log_softmax(tr.rt.t[tr.rt.plan.meta["logits"]][:, :1001] / 2, 1)
                      ).sum(1).mean()
    assert abs(kd - float(want_kd)) < 2e-3 * abs(float(want_kd))
    with pytest.raises(ValueError):
        F.model_fn_cls({"image": x}, lab, F.TRAIN, params)      # KD needs the 2*C label tensor
    # EVAL: loss = CE + L2 (+ KD), metrics carry 'ece'
    F.model_fn_cls.reset_metrics()
    ev = F.model_fn_cls({"image": x}, kd_labels, F.EVAL, params)
    assert set(ev.eval_metric_ops) == {"accuracy", "accuracy_top_5", "ece"}
    assert float(ev.loss) > l2 * 0.99
    emb = tr.model(x, training=False, return_embedding=True)
    assert emb.shape == (4, 64)


def test_checkpoint_round_trip_and_warm_start(tmp_path):
    from assembled_cnn_b200 import checkpoint as C
    from assembled_cnn_b200.model_fns import Model, Trainer
    from assembled_cnn_b200.hparams import params_from_flags
    kw = dict(resnet_size=50, resnet_version=1, use_se_block=True)
    p = params_from_flags(batch_size=4, weight_decay=1e-4, base_learning_rate=0.05,
                          learning_rate_decay_type="fixed", **kw)
    x, lab, _ = _inputs(4, 64, seed=3)
    # deterministic=True: no split-K atomics anywhere, so "same weights -> same step" is exact (tiny
    # batch-4 / 64 px networks amplify 1e-7 summation-order noise to 1e-4 in the loss)
    m1 = Model(50, resnet_version=1, use_se_block=True, seed=1, deterministic=True)
    t1 = Trainer(m1, p, 64, 64, use_cuda_graph=False)
    for _ in range(2):
        t1.train_step(x, lab)
    f = C.save_checkpoint(str(tmp_path / "model.ckpt-2"), m1, t1)
    ck = C.load_checkpoint(f)
    assert ck["resnet_model/conv2d/kernel"].shape == (7, 7, 3, 64)           # HWIO, TF naming
    assert "resnet_model/conv2d/kernel/Momentum" in ck and int(ck["global_step"]) == 2
    assert ck["resnet_model/dense/kernel"].shape == (2048, 1001)
    # full restore into a differently initialised model: the next step is bit-identical
    m2 = Model(50, resnet_version=1, use_se_block=True, seed=2, deterministic=True)
    t2 = Trainer(m2, p, 64, 64, use_cuda_graph=False)
    C.restore(m2, f, t2)
    assert t2.global_step == 2
    a = t1.train_step(x, lab).clone()
    b = t2.train_step(x, lab).clone()
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.equal(t1.rt.params, t2.rt.params) and torch.equal(t1.rt.momentum, t2.rt.momentum)
    # warm start: everything but the classifier (and not the BN moving statistics)
    m3 = Model(50, resnet_version=1, use_se_block=True, seed=3)
    m3(x, training=False)
    dense0 = m3.get_weights()["resnet_model/dense/kernel"].clone()
    names = C.warm_start(m3, f, global_step=0)
    w3, w1 = m3.get_weights(), C.load_checkpoint(f)
    assert "resnet_model/dense/kernel" not in names
    assert torch.equal(w3["resnet_model/dense/kernel"], dense0)
    assert torch.allclose(w3["resnet_model/conv2d/kernel"],
                          torch.as_tensor(w1["resnet_model/conv2d/kernel"]))
    assert C.warm_start(m3, f, global_step=5) == []


def test_sk_fc_fused_matches_multi_launch_path(lib):
    """The fused cooperative kernels of the SK attention chain (one launch per direction, K-split
    partials summed in split order) against the multi-launch split-K path (acnn_set_sk_fc_fused),
    forward and backward, at the Assemble-ResNet-50 shapes and at ragged batches; two fused runs are
    bit-identical (poisoned scratch: nothing needs zeroing)."""
    from assembled_cnn_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    for B, f in ((256, 64), (256, 512), (12, 128), (5, 256)):
        d = max(f // 2, 32)
        g = torch.Generator().manual_seed(f + B)
        rnd = lambda *s: torch.randn(*s, generator=g).cuda()
        s_, w1, w2 = rnd(B, f).abs(), rnd(d, f) * f ** -0.5, rnd(2 * f, d) * d ** -0.5
        gamma, beta = 0.5 + torch.rand(d, generator=g).cuda(), 0.1 * rnd(d)
        dA = rnd(B, f)
        outs = []
        for fused in (0, 1, 1):
            lib.acnn_set_sk_fc_fused(fused)
            mm, mv = torch.zeros(d, device="cuda"), torch.ones(d, device="cuda")
            zpre, z, att = (torch.full((B, n), float("nan"), device="cuda") for n in (d, d, f))
            bnstat = torch.zeros(2 * d, device="cuda")
            n_scr = lib.acnn_sk_fc_scratch_floats(B, f, d)
            assert n_scr >= B * (2 * f + d)
            scratch = (torch.zeros(n_scr, device="cuda") if fused == 0
                       else torch.full((n_scr,), float("nan"), device="cuda"))
            _lib.check(lib.acnn_sk_fc_fwd(s_.data_ptr(), w1.data_ptr(), gamma.data_ptr(),
                                          beta.data_ptr(), mm.data_ptr(), mv.data_ptr(), 0.997, 1e-5,
                                          1, w2.data_ptr(), zpre.data_ptr(), bnstat.data_ptr(),
                                          z.data_ptr(), att.data_ptr(), scratch.data_ptr(), B, f, d,
                                          0, st), "sk_fc_fwd")
            dw1, dw2 = 0.1 * torch.ones(d, f, device="cuda"), 0.2 * torch.ones(2 * f, d, device="cuda")
            dg, db = torch.zeros(d, device="cuda"), torch.zeros(d, device="cuda")
            ds = torch.full((B, f), float("nan"), device="cuda")
            _lib.check(lib.acnn_sk_fc_bwd(dA.data_ptr(), att.data_ptr(), z.data_ptr(),
                                          zpre.data_ptr(), bnstat.data_ptr(), gamma.data_ptr(),
                                          s_.data_ptr(), w1.data_ptr(), w2.data_ptr(),
                                          dw1.data_ptr(), dw2.data_ptr(), dg.data_ptr(),
                                          db.data_ptr(), ds.data_ptr(), scratch.data_ptr(), B, f, d,
                                          0, st), "sk_fc_bwd")
            torch.cuda.synchronize()
            outs.append([t.clone() for t in (zpre, z, att, bnstat, mm, mv, dw1, dw2, dg, db, ds)])
        lib.acnn_set_sk_fc_fused(-1)
        for a, b, c in zip(*outs):
            assert torch.isfinite(b).all()
            scale = a.abs().max().item() + 1e-12
            assert (a - b).abs().max().item() <= 2e-5 * scale, (B, f)
            assert torch.equal(b, c), (B, f)
