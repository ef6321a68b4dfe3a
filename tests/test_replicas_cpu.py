"""Several data-parallel replicas per device, on the host: the input each replica reads does not depend on how
the replicas are split between processes; replicas_per_device and the batch's divisibility are checked before
any GPU work; and, in float64 with the Python plan, one R = 2 step on one process (the replicas in sequence,
then accumulated as acnn_replica_accumulate does) equals the two-rank gloo step of dp.py."""
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import test_dp_gloo_cpu as G

COUNTS = [23, 17, 31]          # records per file
SEED, SHUFFLE = 5, 40


def _replica_data(world, replicas, cycle, epochs, input_batch, steps):
    """{(q, t): (records, windows + flips, mixup lambdas)} of every replica q over `steps` steps."""
    from assembled_cnn_b200 import imagenet_train as it
    out = {}
    for rank in range(world):
        streams = it.replica_streams(COUNTS, SEED, cycle, epochs, SHUFFLE, input_batch, world, rank, replicas)
        assert len({s.steps for s in streams}) == 1
        for t in range(steps):
            lam = it.replica_mixup_lambdas(SEED, 100 + t, rank, replicas, input_batch)
            for r, s in enumerate(streams):
                recs = s.records(t)
                windows = [it.crop_window(50 + rec % 7, 60 + rec % 5, it.example_rng(SEED, cycle, pos))
                           for pos, rec in recs]
                out[(rank * replicas + r, t)] = (recs, windows, lam[r].tolist())
    return out


@pytest.mark.parametrize("input_batch", [4, 6])
def test_input_does_not_depend_on_the_split(input_batch):
    from assembled_cnn_b200 import imagenet_train as it
    total = sum(COUNTS)
    for cycle in (0, 1):
        steps = 2 * total // (4 * input_batch)
        runs = [_replica_data(w, r, cycle, 2, input_batch, steps) for w, r in ((1, 4), (2, 2), (4, 1))]
        assert runs[0] == runs[1] == runs[2]
        # one replica of a 4-rank run is what CycleStream(world=4, rank=q) and mixup_lambdas(rank=q) give
        s = it.CycleStream(COUNTS, SEED, cycle, 2, SHUFFLE, input_batch, 4, 3)
        assert runs[0][(3, 1)][0] == s.records(1)
        assert runs[0][(3, 1)][2] == it.mixup_lambdas(SEED, 101, 3, input_batch).tolist()
        # the replicas of one step read distinct records
        assert len({p for q in range(4) for p, _ in runs[0][(q, 0)][0]}) == 4 * input_batch
    # a run resumed at a cycle boundary builds the same streams: nothing carries over between cycles
    assert _replica_data(2, 2, 1, 2, 4, 3) == {k: v for k, v in _replica_data(2, 2, 1, 2, 4, 4).items() if k[1] < 3}


def test_replicas_argument_checks(monkeypatch):
    """R < 1 and a batch not divisible by world x R raise (the reference's text for the latter) before any GPU
    work: every CUDA entry point is made to fail, and the errors are still the argument errors."""
    from assembled_cnn_b200 import model_fns as F
    from assembled_cnn_b200.hparams import params_from_flags

    def no_gpu(*a, **k):
        raise AssertionError("GPU work before the argument checks")
    monkeypatch.setattr(torch.cuda, "current_device", no_gpu)
    monkeypatch.setattr(F.Model, "runtime", no_gpu)
    for bad in (0, -1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="replicas_per_device must be an integer >= 1"):
            F.check_replicas_per_device(bad)
        with pytest.raises(ValueError, match="replicas_per_device"):
            F.train_and_evaluate("/nonexistent", "/nonexistent", replicas_per_device=bad, batch_size=32)
    p = params_from_flags(batch_size=36)
    with pytest.raises(ValueError, match="Found 8 GPUs with a batch size of 36; try --batch_size=32 instead"):
        F.Trainer(object.__new__(F.Model), p, replicas_per_device=8)
    with pytest.raises(ValueError, match="Found 8 GPUs with a batch size of 36"):
        F.train_and_evaluate("/nonexistent", "/nonexistent", replicas_per_device=8, batch_size=36)
    with pytest.raises(ValueError, match="replicas_per_device"):
        F.Trainer(object.__new__(F.Model), p, replicas_per_device=0)


def _accumulate(phase, acc_g, g, base, acc_s, s, scale):
    """acnn_replica_accumulate's phases (acnn.h) on float64 torch tensors, in place."""
    if phase == "save":
        base.copy_(s)
    elif phase == "first":
        acc_g.copy_(g)
        acc_s.copy_(s)
        s.copy_(base)
    elif phase == "middle":
        acc_g.add_(g)
        acc_s.add_(s)
        s.copy_(base)
    else:
        g.copy_(acc_g + g)
        s.copy_((acc_s + s) * scale)


def test_two_replicas_on_one_process_equal_the_gloo_step(tmp_path):
    out = str(tmp_path / "dp.pt")
    mp.spawn(G._worker, args=(G._free_port(), out), nprocs=G.WORLD, join=True)
    want = torch.load(out)
    threads = torch.get_num_threads()
    torch.set_num_threads(4)          # as each gloo rank: the same summation order in the CPU convolutions
    try:
        _one_process_step(want)
    finally:
        torch.set_num_threads(threads)


def _one_process_step(want):
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from oracle import model as M, plan_interp as PI
    plan = build_plan(ModelConfig(**G.KW), G.B_LOCAL, G.HW, G.HW, training=True, mixup_type=0, label_smoothing=0.1)
    _, vs = M.build(seed=42, dtype=torch.float64, input_hw=G.HW, **G.KW)
    it = PI.PlanInterpreter(plan, dtype=torch.float64)
    it.set_weights(vs.vars)
    lr = 0.05
    it.hp.update(lr=lr, momentum=0.9, weight_decay=1e-4, sgd_grad_scale=1.0 / G.WORLD)
    start = {n: it.get_tf(n).clone() for n in plan.params}
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(G.B_LOCAL * G.WORLD, G.HW, G.HW, 3, generator=g) * 64).double()
    lab = torch.randint(1, 1001, (G.B_LOCAL * G.WORLD,), generator=g).int()
    acc_g, base, acc_s = torch.zeros_like(it.grads), torch.zeros_like(it.state), torch.zeros_like(it.state)
    _accumulate("save", acc_g, it.grads, base, acc_s, it.state, 0.5)
    for r, phase in enumerate(("first", "last")):
        sl = slice(r * G.B_LOCAL, (r + 1) * G.B_LOCAL)
        it.forward(x[sl], lab[sl])
        it.run(plan.backward)
        _accumulate(phase, acc_g, it.grads, base, acc_s, it.state, 0.5)
    it.run(plan.update)
    for n in list(plan.params) + list(plan.state):
        v = it.get_tf(n)
        assert (v - want[n]).abs().max().item() <= 1e-12 * max(want[n].abs().max().item(), 1.0), n
    # one step from zero momentum: momentum = (w0 - w1) / lr on both sides
    for n in plan.params:
        mom = it.get_tf(n, it.momentum)
        ref = (start[n] - want[n]) / lr
        assert (mom - ref).abs().max().item() <= 1e-10 * max(ref.abs().max().item(), 1.0), n
