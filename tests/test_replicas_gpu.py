"""GPU checks of several data-parallel replicas per device: acnn_replica_accumulate bit for bit against a numpy
fp32 restatement of its phases (odd lengths, unaligned ranges and pointers, eager and graph replay); the
Trainer's replicas_per_device = R step bit for bit against a manual composition through the runtime (bf16 /
fp32, mixup type 1, DropBlock, KD, R = 2 and 3, graph and eager); the fp32 R = 2 step against the float64
oracle of two replicas; the c3 / c5 training plans at the recipes' per-replica batches; train_and_evaluate
with R = 2 (checkpoints, evaluation, resume); W = 2, R = 1 against W = 1, R = 2 with two GPUs."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SAVE, FIRST, MIDDLE, LAST = 0, 1, 2, 3
ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)


# ------------------------------------------------------------------------------------------ kernel
def _ref(phase, acc_g, g, base, acc_s, s, lo, hi, ns, scale):
    """The phases of acnn_replica_accumulate in numpy float32, in place."""
    if phase == SAVE:
        base[:ns] = s[:ns]
        return
    if phase == LAST:
        g[lo:hi] = acc_g[lo:hi] + g[lo:hi]
        s[:ns] = (acc_s[:ns] + s[:ns]) * np.float32(scale)
        return
    acc_g[lo:hi] = g[lo:hi] if phase == FIRST else acc_g[lo:hi] + g[lo:hi]
    acc_s[:ns] = s[:ns] if phase == FIRST else acc_s[:ns] + s[:ns]
    if base is not None:
        s[:ns] = base[:ns]


def _call(lib, phase, bufs, lo, hi, ns, scale):
    from assembled_cnn_b200 import _lib
    acc_g, g, base, acc_s, s = (None if b is None else b.data_ptr() for b in bufs)
    _lib.check(lib.acnn_replica_accumulate(phase, acc_g, g, base, acc_s, s, lo, hi, ns, scale,
                                           torch.cuda.current_stream().cuda_stream), "acnn_replica_accumulate")


@pytest.mark.parametrize("n,lo,hi,ns,offs", [
    (1003, 0, 1003, 130, (0, 0, 0, 0, 0)),       # odd length, aligned
    (1003, 1, 1002, 7, (1, 1, 1, 1, 1)),         # same misalignment everywhere: scalar head, float4 body
    (1003, 3, 7, 1, (0, 1, 2, 3, 0)),            # mixed alignments: scalars only
    (4096, 5, 5, 130, (2, 2, 0, 1, 3)),          # empty gradient range
    (257, 2, 255, 0, (0, 0, 0, 0, 0)),           # no state
    (1 << 20, 1, (1 << 20) - 3, 4099, (0, 0, 0, 0, 0)),   # multi-wave grid
])
def test_accumulate_phases_bit_exact(lib, n, lo, hi, ns, offs):
    rng = np.random.default_rng(n + lo + ns)
    sizes = (n, n, ns, ns, ns)
    host = [rng.standard_normal(sz + 4).astype(np.float32) * 100 for sz in sizes]
    dev = [torch.from_numpy(h).cuda() for h in host]
    views = [d[o:o + sz] for d, o, sz in zip(dev, offs, sizes)]
    hv = [h[o:o + sz] for h, o, sz in zip(host, offs, sizes)]
    for R in (2, 3):
        scale = 1.0 / R
        phases = [SAVE, FIRST] + [MIDDLE] * (R - 2) + [LAST]
        for ph in phases:
            # a new gradient and state per micro-step, as a forward + backward would leave them
            new_g = rng.standard_normal(n).astype(np.float32)
            new_s = rng.standard_normal(ns).astype(np.float32)
            if ph != SAVE:
                hv[1][:] = new_g
                hv[4][:] = new_s
                views[1].copy_(torch.from_numpy(new_g))
                views[4].copy_(torch.from_numpy(new_s))
            _ref(ph, hv[0], hv[1], hv[2], hv[3], hv[4], lo, hi, ns, scale)
            _call(lib, ph, views, lo, hi, ns, scale)
            torch.cuda.synchronize()
            for h, d in zip(host, dev):
                assert np.array_equal(d.cpu().numpy().view(np.uint32), h.view(np.uint32)), (R, ph)
    # state_base NULL leaves the state as it is (the loss slot)
    before = views[4].clone()
    _call(lib, FIRST, [views[0], views[1], None, views[3], views[4]], lo, hi, ns, 0.5)
    torch.cuda.synchronize()
    assert torch.equal(views[4], before) and torch.equal(views[3], before)


def test_accumulate_graph_replay(lib):
    n, ns = 100003, 517
    bufs = [torch.randn(n + 1, device="cuda")[1:], torch.randn(n, device="cuda"), torch.randn(ns, device="cuda"),
            torch.randn(ns + 3, device="cuda")[3:], torch.randn(ns, device="cuda")]
    init = [b.clone() for b in bufs]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graphs = []
    with torch.cuda.stream(s):
        for ph in (SAVE, FIRST, MIDDLE, LAST):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                _call(lib, ph, bufs, 3, n - 1, ns, 1.0 / 3)
            graphs.append(g)
    torch.cuda.current_stream().wait_stream(s)
    results = []
    for mode in ("graph", "eager"):
        for b, i in zip(bufs, init):
            b.copy_(i)
        for k, ph in enumerate((SAVE, FIRST, MIDDLE, LAST)):
            bufs[1].mul_(1.5)
            bufs[4].add_(0.25)
            if mode == "graph":
                graphs[k].replay()
            else:
                _call(lib, ph, bufs, 3, n - 1, ns, 1.0 / 3)
        torch.cuda.synchronize()
        results.append([b.clone() for b in bufs])
    assert all(torch.equal(a, b) for a, b in zip(*results))


def test_accumulate_argument_checks(lib):
    x = torch.zeros(16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert lib.acnn_replica_accumulate(4, x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                                       0, 4, 4, 0.5, st) != 0
    assert lib.acnn_replica_accumulate(FIRST, x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                                       4, 2, 4, 0.5, st) != 0
    assert lib.acnn_replica_accumulate(FIRST, None, x.data_ptr(), None, x.data_ptr(), x.data_ptr(), 0, 4, 4, 0.5,
                                       st) != 0
    assert lib.acnn_replica_accumulate(SAVE, None, None, None, None, x.data_ptr(), 0, 0, 4, 0.5, st) != 0


# ------------------------------------------------------------------------------------------ Trainer
B_REP, HW = 4, 224     # DropBlock needs a 7 x 7 map in group 4


def _params(dtype, R, mixup_type=1, kd=True, dropblock=True, batch=B_REP):
    from assembled_cnn_b200.hparams import params_from_flags
    return params_from_flags(batch_size=batch * R, mixup_type=mixup_type, label_smoothing=0.1, weight_decay=1e-4,
                             base_learning_rate=0.05, learning_rate_decay_type="fixed", dtype=dtype,
                             use_dropblock=dropblock, dropblock_kp=[1.0, 0.9], kd_temp=2.0 if kd else 0,
                             train_epochs=1, **ASSEMBLE)


def _model(dtype):
    from assembled_cnn_b200.model_fns import Model
    return Model(50, num_classes=1001, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                 anti_alias_filter_size=3, dtype=dtype, seed=5)


def _batches(R, steps, input_batch, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(steps):
        x = (torch.randn(R * input_batch, HW, HW, 3, generator=g) * 64).clamp(-124, 152)
        lab = torch.randint(1, 1001, (R * input_batch,), generator=g).int()
        lam = torch.rand(R, input_batch // 2, generator=g)
        teach = torch.randn(R * input_batch, 1001, generator=g) * 3
        out.append((x, lab, lam, teach))
    return out


def _manual(dtype, R, batches, keep_prob, lr):
    """The R-replica step composed by hand through a one-replica runtime: each replica's forward / backward from
    the same saved moving statistics, g = ((g0 + g1) + ...), state and loss = (sum in replica order) * (1/R) in
    fp32 torch ops, then the SGD update with grad_scale 1/R."""
    from assembled_cnn_b200.model_fns import Trainer
    model = _model(dtype)
    tr = Trainer(model, _params(dtype, 1, batch=B_REP), HW, HW, use_cuda_graph=False)
    rt, n = tr.rt, tr.input_batch
    m = rt.plan.meta
    loss_slot = rt.slot_view(m["loss"])
    losses = []
    for t, (x, lab, lam, teach) in enumerate(batches):
        rt.set_hparams(lr=lr, momentum=tr.p["momentum"], weight_decay=tr.p["weight_decay"], grad_scale=1.0 / R,
                       keep_prob=keep_prob, step=t)
        s0 = rt.state.clone()
        gsum = ssum = lsum = None
        for r in range(R):
            rt.state.copy_(s0)
            rt.t[m["images"]].copy_(x[r * n:(r + 1) * n])
            rt.t[m["labels"]].copy_(lab[r * n:(r + 1) * n])
            rt.t[m["lam1"]].copy_(lam[r])
            rt.t[m["teacher_logits"]].copy_(teach[r * n:(r + 1) * n])
            rt.run_forward()
            rt.run(rt.plan.backward)
            gsum = rt.grads.clone() if gsum is None else gsum + rt.grads
            ssum = rt.state.clone() if ssum is None else ssum + rt.state
            lsum = loss_slot.clone() if lsum is None else lsum + loss_slot
        rt.grads.copy_(gsum)
        rt.state.copy_(ssum * (1.0 / R))      # a float32 multiply by float32(1/R)
        loss_slot.copy_(lsum * (1.0 / R))
        rt.run(rt.plan.update)
        losses.append(loss_slot[:3].clone())
    torch.cuda.synchronize()
    return dict(params=rt.params.clone(), momentum=rt.momentum.clone(), state=rt.state.clone(),
                loss=torch.stack(losses))


def _trainer_run(dtype, R, batches, keep_prob, graph):
    from assembled_cnn_b200.model_fns import Trainer
    model = _model(dtype)
    tr = Trainer(model, _params(dtype, R), HW, HW, use_cuda_graph=graph, replicas_per_device=R)
    losses = []
    for x, lab, lam, teach in batches:
        losses.append(tr.train_step(x, lab, lam1=lam, teacher_logits=teach, keep_prob=keep_prob)[:3].clone())
    torch.cuda.synchronize()
    rt = tr.rt
    return tr, dict(params=rt.params.clone(), momentum=rt.momentum.clone(), state=rt.state.clone(),
                    loss=torch.stack(losses))


def _bits_equal(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)


@pytest.mark.parametrize("dtype,R", [("bf16", 2), ("fp32", 2), ("bf16", 3)])
def test_trainer_equals_manual_composition(dtype, R):
    batches = _batches(R, 3, 2 * B_REP, seed=R)
    tr, got = _trainer_run(dtype, R, batches, 0.9, graph=True)
    assert tr.local_batch == B_REP and tr.input_batch == 2 * B_REP
    want = _manual(dtype, R, batches, 0.9, tr.last_lr)
    assert _bits_equal(got, want), {k: (got[k] - want[k]).abs().max().item() for k in got}
    assert torch.isfinite(got["loss"]).all() and (got["loss"][:, 1] > 0).all()
    _, eager = _trainer_run(dtype, R, batches, 0.9, graph=False)
    assert _bits_equal(eager, got)


def test_parity_fp32_two_replicas_against_oracle():
    """An R = 2 fp32 step against the float64 oracle of two replicas (the MirroredStrategy semantics:
    per-replica BN, averaged gradients and moving statistics), within the parity suite's 1e-3."""
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    from oracle import model as M
    hw, b, R = 64, 4, 2
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(R * b, hw, hw, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (R * b,), generator=g).int()
    onehot = torch.nn.functional.one_hot(lab.long(), 1001)
    _, vs32 = M.build(seed=42, dtype=torch.float32, input_hw=hw, **ASSEMBLE)
    start = {n: v.clone() for n, v in vs32.vars.items()}
    ref = {}
    for dt in (torch.float32, torch.float64):
        omodel, vs = M.build(seed=42, dtype=torch.float32, input_hw=hw, **ASSEMBLE)
        for n in vs.vars:
            vs.vars[n] = vs.vars[n].to(dt)
        vs.dtype = dt
        mom = {n: torch.zeros_like(v) for n, v in vs.vars.items() if vs.trainable[n]}
        out = M.train_step(omodel, vs, mom, x.to(dt), onehot.to(dt), lr=0.05, momentum=0.9, label_smoothing=0.1,
                           weight_decay=1e-4, n_replicas=R)
        ref[dt] = (out, {n: v.clone() for n, v in vs.vars.items()})
    (out, r64), (_, r32) = ref[torch.float64], ref[torch.float32]
    model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                  anti_alias_filter_size=3, dtype="fp32")
    model.set_weights(start)
    p = params_from_flags(batch_size=R * b, label_smoothing=0.1, weight_decay=1e-4, base_learning_rate=0.05,
                          learning_rate_decay_type="fixed", dtype="fp32", **ASSEMBLE)
    tr = Trainer(model, p, hw, hw, use_cuda_graph=False, replicas_per_device=R)
    loss = tr.train_step(x, lab).tolist()
    got = model.get_weights()

    def nrel(a, b_):
        return ((a.double() - b_.double()).norm() / b_.double().norm().clamp_min(1e-30)).item()
    stats = [n for n in r64 if n.endswith("moving_mean") or n.endswith("moving_variance")]
    worst_stats = max(nrel(got[n], r64[n]) for n in stats)
    # trained variables: the fp32 oracle's own distance from the fp64 one is the yardstick (ReLU masks flip
    # under fp32 round-off, test_parity_fp32_gpu.py), as the one-replica parity test does
    bad = [(n, nrel(got[n], r64[n]), nrel(r32[n], r64[n])) for n in r64 if n not in stats]
    bad = [t for t in bad if not t[1] <= max(1e-3, 4.0 * t[2])]
    ce64, l264 = float(out["cross_entropy"]), float(out["l2_loss"])
    print("R = 2 fp32 step vs fp64 oracle of two replicas: moving statistics worst norm-rel %.2e, CE %.6f / %.6f"
          % (worst_stats, loss[0], ce64))
    assert worst_stats < 1e-3
    assert not bad, bad[:10]
    assert abs(loss[0] - ce64) < 1e-3 * abs(ce64)
    assert abs(loss[1] - l264) < 1e-3 * abs(l264)


@pytest.mark.parametrize("cfg", ["c3", "c5"])
@pytest.mark.parametrize("b", [128, 64])
def test_recipe_per_replica_batches_repeatable(cfg, b):
    """The c3 (Assemble-ResNet-50) and c5 (Assemble-ResNet-152) training plans at the recipes' per-replica
    batches, R = 2: two runs of the same step from the same start give identical bits."""
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    kw = dict(ASSEMBLE) if cfg == "c3" else dict(ASSEMBLE, resnet_size=152, bl_alpha=1, bl_beta=2)
    g = torch.Generator().manual_seed(b)
    R = 2
    x = (torch.randn(R * 2 * b, 224, 224, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (R * 2 * b,), generator=g).int()
    lam = torch.rand(R, b, generator=g)
    outs = []
    for _ in range(2):
        model = Model(num_classes=1001, dtype="bf16", seed=1, **kw)
        p = params_from_flags(batch_size=R * b, mixup_type=1, label_smoothing=0.1, weight_decay=1e-4,
                              base_learning_rate=0.1, dtype="bf16", **kw)
        tr = Trainer(model, p, 224, 224, use_cuda_graph=True, replicas_per_device=R)
        loss = tr.train_step(x.cuda(), lab.cuda(), lam1=lam).clone()
        torch.cuda.synchronize()
        outs.append((loss, tr.rt.params.clone(), tr.rt.state.clone()))
        del tr, model
        torch.cuda.empty_cache()
    assert torch.isfinite(outs[0][0]).all()
    assert all(torch.equal(a, b_) for a, b_ in zip(*outs))


# ------------------------------------------------------------------------------------------ loop
def test_train_and_evaluate_two_replicas_resumes(tmp_path):
    """The synthetic shards of test_train_input_gpu.py, global batch 32 as two replicas of 16."""
    import sys
    import test_train_input_gpu as T
    from assembled_cnn_b200.model_fns import train_and_evaluate
    sys.path.insert(0, os.path.join(T.ROOT, "golden"))
    import make_eval_preprocess_golden as mk
    Example = mk.example_class()
    shards = tmp_path / "data"
    shards.mkdir()
    rng = np.random.default_rng(0)
    for sh, n in enumerate((70, 70, 60)):
        T._write_shard(shards / ("train-%05d-of-00003" % sh), Example, mk, rng, n, kd=False)
    T._write_shard(shards / "validation-00000-of-00001", Example, mk, rng, 40, kd=False)
    flags = dict(T.FLAGS, replicas_per_device=2)
    run = tmp_path / "run"
    res = train_and_evaluate(str(shards), str(run), **flags)
    # 200 records, global batch 32 (two replicas of 16): 6 steps per cycle
    assert [r["global_step"] for r in res] == [6, 12]
    final = T._weights(str(run / "model.ckpt-12.npz"))
    resumed = tmp_path / "resumed"
    assert train_and_evaluate(str(shards), str(resumed), stop_threshold=0.0, **flags) == res[:1]
    assert train_and_evaluate(str(shards), str(resumed), **flags) == res[1:]
    got = T._weights(str(resumed / "model.ckpt-12.npz"))
    assert all(np.array_equal(got[n], final[n]) for n in final)
    assert all(np.isfinite(final[n]).all() for n in final)
    assert "model.ckpt-12.npz" in os.listdir(run) and os.listdir(run / "best")


# ------------------------------------------------------------------------------------------ two GPUs
def _w2_worker(rank, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=2)
    res = _two_way_run(rank, 2, 1)
    if rank == 0:
        torch.save(res, out)
    dist.barrier()
    dist.destroy_process_group()


def _two_way_run(rank, world, R):
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    b, hw = 8, 128
    g = torch.Generator().manual_seed(0)
    batches = [((torch.randn(2 * b, hw, hw, 3, generator=g) * 64).clamp(-124, 152),
                torch.randint(1, 1001, (2 * b,), generator=g).int()) for _ in range(2)]
    model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                  anti_alias_filter_size=3, dtype="bf16", seed=3, device="cuda:%d" % rank,
                  deterministic=True)
    p = params_from_flags(batch_size=2 * b, label_smoothing=0.1, weight_decay=1e-4, base_learning_rate=0.05,
                          dtype="bf16", **ASSEMBLE)
    tr = Trainer(model, p, hw, hw, use_cuda_graph=True, replicas_per_device=R)
    rows = slice(rank * b, (rank + 1) * b) if world == 2 else slice(0, 2 * b)
    losses = []
    for x, lab in batches:
        loss = tr.train_step(x[rows].cuda(), lab[rows].cuda())
        losses.append(loss.tolist())
    return dict(losses=losses, params=tr.rt.params.cpu(), state=tr.rt.state.cpu())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_equal_two_replicas_on_one(tmp_path):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "w2.pt")
    mp.spawn(_w2_worker, args=(port, out), nprocs=2, join=True)
    w2 = torch.load(out)
    r2 = _two_way_run(0, 1, 2)
    # rank 0's loss is its own replica's; the R = 2 loss is the mean of both replicas
    assert torch.allclose(w2["params"], r2["params"], rtol=1e-5, atol=1e-6)
    assert torch.allclose(w2["state"], r2["state"], rtol=1e-5, atol=1e-6)
    assert np.isfinite(np.array(r2["losses"])).all()
