"""Data-parallel semantics on CPU with 2 gloo ranks: every rank runs the product's layer plan on
its shard (torch interpreter standing in for the kernels) and drives the SAME data-parallel code as
Trainer.train_step (assembled_cnn_b200/dp.py): the backward cut into segments, each followed by the
sum-all-reduce of its gradient bucket, the 1/N folded into the SGD step, and the mean aggregation of
the BN moving statistics.  The result must equal the oracle's MirroredStrategy semantics
(per-replica BN statistics, averaged gradients, averaged moving statistics;
official/utils/misc/distribution_utils.py:24-76)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

KW = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
          anti_alias_filter_size=3)
HW, B_LOCAL, WORLD = 64, 4, 2   # >= 4 samples per BN everywhere (B=2 degenerates)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    torch.set_num_threads(4)
    from assembled_cnn_b200 import dp
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from oracle import model as M, plan_interp as PI
    plan = build_plan(ModelConfig(**KW), B_LOCAL, HW, HW, training=True, mixup_type=0,
                      label_smoothing=0.1)
    _, vs = M.build(seed=42, dtype=torch.float64, input_hw=HW, **KW)
    it = PI.PlanInterpreter(plan, dtype=torch.float64)
    it.set_weights(vs.vars)
    it.hp.update(lr=0.05, momentum=0.9, weight_decay=1e-4, sgd_grad_scale=1.0 / WORLD)
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(B_LOCAL * WORLD, HW, HW, 3, generator=g) * 64).double()
    lab = torch.randint(1, 1001, (B_LOCAL * WORLD,), generator=g).int()
    sl = slice(rank * B_LOCAL, (rank + 1) * B_LOCAL)
    it.forward(x[sl], lab[sl])
    # the Trainer's schedule: backward segments interleaved with the bucket all-reduces
    buckets = dp.grad_buckets(plan)
    segments = dp.backward_segments(plan, buckets)
    assert len(buckets) >= 4 and segments[0][0] == 0 and segments[-1][1] == len(plan.backward)
    assert buckets[0][1] == plan.param_elems and buckets[-1][0] == 0
    reduced = torch.zeros(plan.param_elems, dtype=torch.bool)
    for ev in dp.schedule(buckets, segments):
        if ev[0] == "run":
            it.run(plan.backward[ev[1]:ev[2]])
        else:
            snapshot = it.grads[ev[1]:ev[2]].clone()
            dp.all_reduce_bucket(it.grads, ev[1], ev[2])
            reduced[ev[1]:ev[2]] = True
            it._bucket_check = getattr(it, "_bucket_check", []) + [(ev[1], ev[2], snapshot)]
    assert reduced.all()
    it.run(plan.update)
    # BN moving statistics are averaged across replicas (mirrored-variable mean aggregation)
    dp.average_moving_statistics(it.state, WORLD)
    if rank == 0:
        torch.save({n: it.get_tf(n).clone() for n in list(plan.params) + list(plan.state)}, out_path)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_data_parallel_matches_oracle(tmp_path):
    out = str(tmp_path / "dp.pt")
    mp.spawn(_worker, args=(_free_port(), out), nprocs=WORLD, join=True)
    got = torch.load(out)
    from oracle import model as M
    model, vs = M.build(seed=42, dtype=torch.float64, input_hw=HW, **KW)
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(B_LOCAL * WORLD, HW, HW, 3, generator=g) * 64).double()
    lab = torch.randint(1, 1001, (B_LOCAL * WORLD,), generator=g)
    onehot = torch.nn.functional.one_hot(lab, 1001).double()
    mom = {n: torch.zeros_like(v) for n, v in vs.vars.items() if vs.trainable[n]}
    M.train_step(model, vs, mom, x, onehot, lr=0.05, momentum=0.9, label_smoothing=0.1,
                 weight_decay=1e-4, n_replicas=WORLD)
    for n, v in vs.vars.items():
        assert (got[n] - v).abs().max().item() <= 1e-6 * max(v.abs().max().item(), 1.0), n


def test_per_device_batch_size_rule():
    """official/utils/misc/distribution_utils.py:48-76: the global batch must divide evenly."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    plan = build_plan(ModelConfig(**KW), 147 // 7, 32, 32, training=True)
    assert plan.meta["batch"] == 21
