"""Data parallelism on real GPUs: two processes, one per GPU, run Trainer.train_step under NCCL
(bucketed all-reduce overlapped with the backward, BN moving statistics mean-aggregated) and must
reproduce the oracle's MirroredStrategy semantics -- oracle.model.train_step(n_replicas=2): per-replica
BN statistics, averaged gradients, averaged moving statistics (official/utils/misc/
distribution_utils.py:24-76).  fp32 mode, so the comparison is tight.  With >= 2 GPUs
(two GPUs) the ranks sit on their own GPUs under NCCL; on a one-GPU box both ranks share
cuda:0 and the collectives go over gloo (CUDA tensors) -- the same Trainer schedule either way."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

KW = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
          anti_alias_filter_size=3)
HW, B_LOCAL, WORLD = 128, 8, 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _data():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(B_LOCAL * WORLD, HW, HW, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (B_LOCAL * WORLD,), generator=g).int()
    return x, lab


def _worker(rank, port, out_path, use_graph):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    # two GPUs: NCCL, one rank per GPU.  One GPU: the SAME Trainer code path
    # (bucketed, overlapped all-reduce between the backward segments / CUDA graphs, mean of the moving
    # statistics) with both ranks on cuda:0 over gloo, which accepts CUDA tensors
    two = torch.cuda.device_count() >= 2
    dev = rank if two else 0
    torch.cuda.set_device(dev)
    if two:
        dist.init_process_group("nccl", rank=rank, world_size=WORLD, device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    from assembled_cnn_b200.model_fns import Model, Trainer
    from assembled_cnn_b200.hparams import params_from_flags
    from oracle import model as M
    _, vs = M.build(seed=42, input_hw=64, **KW)
    model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True,
                  anti_alias_type="sconv", anti_alias_filter_size=3, dtype="fp32",
                  device="cuda:%d" % dev)
    model.set_weights(vs.vars)
    p = params_from_flags(batch_size=B_LOCAL * WORLD, label_smoothing=0.1, weight_decay=1e-4,
                          base_learning_rate=0.05, learning_rate_decay_type="fixed", dtype="fp32",
                          **KW)
    tr = Trainer(model, p, HW, HW, use_cuda_graph=use_graph)
    assert tr.world == WORLD and tr.local_batch == B_LOCAL and len(tr._buckets) >= 4
    x, lab = _data()
    sl = slice(rank * B_LOCAL, (rank + 1) * B_LOCAL)
    rt = tr.rt
    backup = (rt.params.clone(), rt.state.clone(), rt.momentum.clone())
    loss = tr.train_step(x[sl], lab[sl]).tolist()
    torch.cuda.synchronize()
    w = model.get_weights()
    # every replica holds the same variables after the step
    flat = torch.cat([rt.params, rt.state])
    other = flat.clone()
    dist.broadcast(other, src=0)
    same = bool(torch.equal(flat, other))
    # STRICT check of the bucketed, overlapped all-reduce (no ReLU-flip noise involved): the gradient
    # buffer the SGD step consumed must be bit-for-bit g_0 + g_1 of the replicas' local gradients
    # (fp32 mode is deterministic, and a two-term fp32 sum has one rounding whatever the order).
    reduced = rt.grads.clone()
    for buf, b in zip((rt.params, rt.state, rt.momentum), backup):
        buf.copy_(b)
    rt.run_forward()                       # inputs / labels / hyper-parameters are still staged
    rt.run(rt.plan.backward)
    torch.cuda.synchronize()
    local = [torch.empty_like(rt.grads) for _ in range(WORLD)]
    dist.all_gather(local, rt.grads)
    strict = bool(torch.equal(reduced, local[0] + local[1]))
    assert float(reduced.abs().max()) > 0
    if rank == 0:
        torch.save({"w": w, "loss": loss, "same": same, "strict": strict}, out_path)
    else:
        assert same and strict
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "cuda_graph"])
def test_two_gpu_trainer_matches_oracle_mirrored_strategy(tmp_path, use_graph):
    if torch.cuda.device_count() < 1:
        pytest.skip("needs a GPU")
    out = str(tmp_path / "dp.pt")
    mp.spawn(_worker, args=(_free_port(), out, use_graph), nprocs=WORLD, join=True)
    got = torch.load(out)
    assert got["same"] and got["strict"]
    from oracle import model as M
    x, lab = _data()

    def oracle(dt):
        model, vs = M.build(seed=42, dtype=torch.float32, input_hw=64, **KW)
        for n in vs.vars:
            vs.vars[n] = vs.vars[n].to(dt)
        vs.dtype = dt
        onehot = torch.nn.functional.one_hot(lab.long(), 1001).to(dt)
        mom = {n: torch.zeros_like(v) for n, v in vs.vars.items() if vs.trainable[n]}
        before = {n: v.clone() for n, v in vs.vars.items()}
        M.train_step(model, vs, mom, x.to(dt), onehot, lr=0.05, momentum=0.9, label_smoothing=0.1,
                     weight_decay=1e-4, n_replicas=WORLD)
        return vs, before

    vs, before = oracle(torch.float64)
    vs32, _ = oracle(torch.float32)
    nrel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()
    # moving statistics: the MEAN over the replicas' updates (forward quantities: tight)
    worst_state = max(nrel(got["w"][n], vs.vars[n]) for n in vs.vars if not vs.trainable[n])
    # weights after w - lr * (mean gradient + wd w): gradients of a ReLU network carry the mask-flip
    # noise of ANY fp32 evaluation (tests/test_parity_fp32_gpu.py), so the yardstick is the oracle's
    # own fp32-vs-fp64 difference on the same step
    worst = (0.0, 0.0, "")
    for n in vs.vars:
        if vs.trainable[n] and before[n].abs().max() > 0:
            err, yard = nrel(got["w"][n], vs.vars[n]), nrel(vs32.vars[n], vs.vars[n])
            assert err <= max(1e-3, 4 * yard), (n, err, yard)
            if err > worst[0]:
                worst = (err, yard, n)
    print("2-GPU DP vs oracle(n_replicas=2): moving stats worst %.2e, weights worst %.2e "
          "(oracle fp32-vs-fp64 on it %.2e, %s), rank-0 CE %.5f; reduced == g0 + g1 bitwise"
          % (worst_state, worst[0], worst[1], worst[2], got["loss"][0]))
    assert worst_state < 1e-3
