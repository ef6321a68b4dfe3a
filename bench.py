#!/usr/bin/env python
"""Benchmark of the assembled-ResNet training step on one H100 (BASELINE.json's metric).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the reference's CPU path (oracle port) on host cores
    python bench.py --dump-outputs DIR ...    # + what the last timed step computed, as DIR/<name>.npy

One JSON line on stdout (rank 0).  A "step" = one full training step of Assemble-ResNet-50
(resnet_version=2, SK, anti-alias sconv/3) on one synthetic batch: mixup type 1 -> forward -> label-
smoothed softmax CE -> backward -> (NCCL all-reduce) -> weight-decay + momentum SGD, 256 images per
GPU at 224x224x3 (weak scaling).  `value` is timed on the device with inputs resident in HBM;
`e2e` goes through the public API (Trainer.train_step) from pinned host buffers, with the H2D copy
of every step's inputs and a D2H read of the loss inside the timed region.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "images/sec Assemble-ResNet-50 224^2 bf16 train step"
ASSEMBLE_FLAGS = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                      anti_alias_filter_size=3)
MODEL_FLAGS = ASSEMBLE_FLAGS
TRAIN_FLAGS = dict(mixup_type=1, label_smoothing=0.1, weight_decay=1e-4, momentum=0.9,
                   base_learning_rate=0.4, learning_rate_decay_type="cosine", lr_warmup_epochs=5,
                   train_epochs=600, bn_momentum=0.997)
PER_GPU_BATCH = 256
TRAIN_GFLOP_PER_IMG = 34.12      # BASELINE.md section 2 (2*MAC: fwd + dgrad + wgrad)

# BASELINE.json `configs` (c3 = the configuration the metric is quoted on = the default bench line;
# c4 is c3 under torchrun).  gflop = algorithmic 2*MAC per image (BASELINE.md section 2).
CONFIGS = {
    "c1": dict(kind="eval", model=dict(resnet_size=50, resnet_version=1), batch=1, gflop=8.18,
               metric="images/sec vanilla ResNet-50 224^2 bf16 eval forward (batch 1)",
               workload="vanilla ResNet-50 (resnet_version=1, no SK/SE/AA) eval-mode forward, "
                        "batch 1, 224x224x3, CUDA-graph replay"),
    "c2": dict(kind="fwd_loss", model=ASSEMBLE_FLAGS, batch=256, gflop=11.45,
               metric="images/sec Assemble-ResNet-50 224^2 bf16 forward+loss",
               workload="Assemble-ResNet-50 (resnet_version=2, use_sk_block, anti_alias sconv/3) "
                        "training-mode forward (batch statistics) + label-smoothed softmax CE, "
                        "224x224x3"),
    "c3": dict(kind="train", model=ASSEMBLE_FLAGS, batch=256, gflop=34.12, metric=METRIC,
               workload="Assemble-ResNet-50 (resnet_version=2, use_sk_block, anti_alias sconv/3) "
                        "full train step: mixup type 1 + label smoothing 0.1 + wd 1e-4 + momentum "
                        "SGD, 224x224x3"),
    "c5": dict(kind="train", model=dict(resnet_size=152, resnet_version=2, use_sk_block=True,
                                        anti_alias_type="sconv", anti_alias_filter_size=3,
                                        bl_alpha=1, bl_beta=2), batch=128, gflop=93.81,
               metric="images/sec Assemble-ResNet-152 (BigLittle alpha=1 beta=2) 224^2 bf16 train step",
               workload="Assemble-ResNet-152 (resnet_version=2, bl_alpha=1, bl_beta=2, use_sk_block, "
                        "anti_alias sconv/3) full train step: mixup type 1 + label smoothing 0.1 + "
                        "wd 1e-4 + momentum SGD, 224x224x3"),
}


def read_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as fh:
            d = json.load(fh)
        return dict(tflops=d["bf16_tflops_sustained"], hbm=d["hbm_gbs"], source="measured")
    # NVIDIA H100 SXM data sheet (dense BF16, HBM3; a 700 W card): an upper bound, not a measurement
    return dict(tflops=989.0, hbm=3350.0, source="H100 SXM data sheet (dense bf16 peak, not a measurement)")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region (profiling recipe)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                 "--format=csv,noheader,nounits", "-lms", "50"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, bufsize=1)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except OSError:
            self.proc = None

    def wait_first_sample(self, timeout=5.0):
        """nvidia-smi needs ~1 s to start sampling; call this (under load) before the timed
        region, then mark() so only samples taken during the region are kept."""
        t0 = time.time()
        while self.proc is not None and not self.lines and time.time() - t0 < timeout:
            time.sleep(0.02)

    def mark(self):
        self.lines = []

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
        sm, mx, reasons = [], 0, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1]))
                mx = max(mx, float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                "sw_power_cap"), f[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None,
                "reasons": sorted(reasons), "samples": len(sm)}


def synth_batch(n, hw, seed):
    """BASELINE.md section 3: images N(0, 64^2) clipped to [-124, 152], labels U{1..1000}."""
    import torch
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, hw, hw, 3, generator=g) * 64.0).clamp_(-124.0, 152.0)
    y = torch.randint(1, 1001, (n,), generator=g, dtype=torch.int32)
    return x, y


def effective_cores():
    """Host cores this process may really use: affinity mask capped by the cgroup CPU quota."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        with open("/sys/fs/cgroup/cpu.max") as fh:
            quota, period = fh.read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except (OSError, ValueError):
        pass
    return max(1, min(n, 64))


def _cpu_probe(cfg, model, vs, batch, hw):
    """Seconds of one CPU step of the configuration at `batch` (its second run: the first pays
    one-time initialisation)."""
    import torch
    from oracle import model as M, tf_ops as T
    x, lab = synth_batch(2 * batch if cfg["kind"] == "train" else batch, hw, 1234)
    onehot = torch.nn.functional.one_hot(lab.long(), 1001).float()
    t = 0.0
    for _ in range(2):
        t0 = time.perf_counter()
        if cfg["kind"] == "train":
            names = [n for n in vs.vars if vs.trainable[n]]
            mom = {n: torch.zeros_like(vs.vars[n]) for n in names}
            backup = {n: vs.vars[n].clone() for n in vs.vars}
            lam = torch.full((batch,), 0.5)
            xm, ym = T.mixup(x, onehot, lam, keep_batch_size=False)
            M.train_step(model, vs, mom, xm, ym, lr=0.0, momentum=0.9, label_smoothing=0.1,
                         weight_decay=1e-4)
            for n in backup:
                vs.vars[n] = backup[n]
        else:
            with torch.no_grad():
                if cfg["kind"] == "eval":
                    M.forward(model, vs, x, training=False)
                else:
                    M.loss_fn(model, vs, x, onehot, training=True, label_smoothing=0.1,
                              weight_decay=1e-4)
        t = time.perf_counter() - t0
    return t


def cpu_reference(cfg_name, steps, warmup, hw=224, budget_s=None):
    """The reference's TF1 CPU path, restated (oracle/model.py): same workload, host cores, on a
    bounded sample (small batch).  With `budget_s` a probe step picks the largest batch of
    8 / 4 / 2 / 1 for which warmup + steps steps fit the budget."""
    import torch
    from oracle import model as M, tf_ops as T
    cfg = CONFIGS[cfg_name]
    cores = effective_cores()
    torch.set_num_threads(cores)
    torch.set_flush_denormal(True)
    flags = cfg["model"]
    model, vs = M.build(seed=42, input_hw=64, **flags)
    batch = {"c1": 1, "c2": 8, "c3": 8, "c5": 4}[cfg_name]
    if budget_s is not None and batch > 1:
        t_probe = _cpu_probe(cfg, model, vs, batch, hw)      # also pages the code / weights in
        while batch > 1 and t_probe * (steps + warmup) > budget_s:
            batch //= 2
            t_probe /= 2.0
    times = []
    if cfg["kind"] == "train":
        names = [n for n in vs.vars if vs.trainable[n]]
        mom = {n: torch.zeros_like(vs.vars[n]) for n in names}
        x, lab = synth_batch(2 * batch, hw, 1234)
        onehot = torch.nn.functional.one_hot(lab.long(), 1001).float()
        for i in range(warmup + steps):
            lam = torch.distributions.Beta(0.2, 0.2).sample((batch,))
            t0 = time.perf_counter()
            xm, ym = T.mixup(x, onehot, lam, keep_batch_size=False)
            M.train_step(model, vs, mom, xm, ym, lr=1e-3, momentum=0.9, label_smoothing=0.1,
                         weight_decay=1e-4)
            if i >= warmup:
                times.append(time.perf_counter() - t0)
        what = "train step (mixup type 1 from %d inputs)" % (2 * batch)
    else:
        x, lab = synth_batch(batch, hw, 1234)
        onehot = torch.nn.functional.one_hot(lab.long(), 1001).float()
        with torch.no_grad():
            for i in range(warmup + steps):
                t0 = time.perf_counter()
                if cfg["kind"] == "eval":
                    M.forward(model, vs, x, training=False)
                else:
                    M.loss_fn(model, vs, x, onehot, training=True, label_smoothing=0.1,
                              weight_decay=1e-4)
                if i >= warmup:
                    times.append(time.perf_counter() - t0)
        what = "eval forward" if cfg["kind"] == "eval" else "training-mode forward + loss"
    sec = sum(times) / len(times)
    return dict(value=batch / sec, unit="images/sec", cores=cores, kind="port",
                sample="oracle/model.py %s (restatement of the reference TF1 CPU path; TF 1.14 not "
                       "installable), %s, 224x224, batch %d, %d timed step(s) after %d warm-up, "
                       "torch %d threads" % (what, cfg_name, batch, steps, warmup, cores)), sec, batch


def cpu_baseline_subprocess(cfg_name, timeout_s=240):
    """Times the oracle in a child process (bounded: the bench line must not hang on a slow host)."""
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--impl", "reference",
                            "--steps", "2", "--warmup", "1", "--config", cfg_name],
                           capture_output=True, text=True,
                           timeout=timeout_s)
        for ln in reversed(r.stdout.strip().splitlines()):
            if ln.startswith("{"):
                return json.loads(ln)["cpu_baseline"]
        return {"value": None, "unit": "images/sec", "cores": effective_cores(), "kind": "port",
                "sample": "failed: " + (r.stderr.strip().splitlines() or ["no output"])[-1][:200]}
    except subprocess.TimeoutExpired:
        return {"value": None, "unit": "images/sec", "cores": effective_cores(), "kind": "port",
                "sample": "timed out after %d s" % timeout_s}


def run_reference_arm(args):
    """`--impl reference`: the reference's CPU path (oracle port) on the host cores, EXACTLY
    --steps K timed steps after --warmup W, on the GPU arm's configuration / metric / unit; each
    step is a bounded sample of the workload (a small CPU batch, shrunk further if a probe step says
    K + W steps would not end within a few minutes).  Rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    steps, warmup = max(1, args.steps), max(0, args.warmup)
    cb, sec, batch = cpu_reference(args.config, steps, warmup, budget_s=150.0)
    cfg = CONFIGS[args.config]
    world = args.gpus
    B = args.batch or cfg["batch"]
    line = {
        "impl": "reference", "metric": cfg["metric"], "value": cb["value"], "unit": "images/sec",
        "n_gpus": args.gpus, "steps": steps, "warmup": warmup, "ms_per_step": sec * 1e3,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": {"workload": cfg["workload"], "name": args.config, "per_gpu_batch": B,
                   "global_batch": B * world, "parallelism": "dp%d" % world,
                   "sample": "CPU batch %d per step (bounded sample of the workload)" % batch},
        "cpu_baseline": cb,
        "e2e": {"value": cb["value"], "unit": "images/sec", "h2d_bytes_per_step": 0,
                "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


class ForwardRunner:
    """c1 / c2: one forward (eval, or training-mode forward + loss) of a Runtime as a CUDA graph,
    behind the same two entry points the Trainer offers (device-resident step, prefetch + step)."""

    def __init__(self, model, batch, hw, kind, dev):
        import torch
        self.torch = torch
        self.kind = kind
        if kind == "eval":
            self.rt = model.runtime(batch, hw, hw, training=False)
        else:
            self.rt = model.runtime(batch, hw, hw, training=True, label_smoothing=0.1)
        rt = self.rt
        m = rt.plan.meta
        self.images = rt.t[m["images"]]
        self.labels = rt.t[m["labels"]] if "labels" in m else None
        self.out = rt.t[m["logits"]] if kind == "eval" else rt.slot_view(m["loss"])[:1]
        self.input_batch = m["input_batch"]
        self.copy_stream = torch.cuda.Stream(dev)
        self.stage_x = torch.empty_like(self.images)
        self.stage_y = torch.empty_like(self.labels) if self.labels is not None else None
        self.staged = self.consumed = None
        self.use_graph = True
        self.world = 1
        self.graph = None

    def _run(self):
        rt = self.rt
        if self.kind == "eval":
            rt.run_forward()
        else:   # training-mode forward (batch statistics, moving-stat updates) + loss, no backward
            rt.zero_step_buffers()      # loss accumulator (+ the gradient buffer dbias lands in)
            rt.run(rt.plan.forward)

    def step(self, x=None, y=None):
        torch = self.torch
        if x is None:
            torch.cuda.current_stream().wait_event(self.staged)
            x, y = self.stage_x, self.stage_y
        self.images.copy_(x, non_blocking=True)
        if self.labels is not None:
            self.labels.copy_(y, non_blocking=True)
        if x is self.stage_x:
            self.consumed = torch.cuda.Event()
            self.consumed.record(torch.cuda.current_stream())
        if self.graph is None and self.use_graph:
            self._run()                       # warm-up outside capture
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, stream=s):
                    self._run()
            torch.cuda.current_stream().wait_stream(s)
        if self.use_graph:
            self.graph.replay()
        else:
            self._run()
        return self.out

    def prefetch(self, x, y):
        torch = self.torch
        if self.consumed is not None:
            self.copy_stream.wait_event(self.consumed)
        with torch.cuda.stream(self.copy_stream):
            self.stage_x.copy_(x, non_blocking=True)
            if self.stage_y is not None:
                self.stage_y.copy_(y, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.staged = ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default="c3", choices=sorted(CONFIGS),
                    help="BASELINE.json configuration (c3 = the headline metric; c4 = c3 under torchrun)")
    ap.add_argument("--batch", type=int, default=0, help="per-GPU batch (0 = the configuration's)")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"],
                    help="fp32 = the parity mode (not the metric's dtype; reported as such)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write what the last timed step computed as "
                         "DIR/<name>.npy (float32; fixed seeded samples of the large buffers)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference_arm(args)
    if args.warmup < 3:
        args.warmup = 3

    import torch
    import torch.distributed as dist
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer

    cfg = CONFIGS[args.config]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the GPU path has no CPU fallback "
                         "(use --impl reference for the CPU arm)")
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib = _lib.load()
    B = args.batch or cfg["batch"]
    flags = dict(cfg["model"])
    dev = torch.device("cuda", local)
    model = Model(flags.pop("resnet_size"), num_classes=1001, dtype=args.dtype,
                  device="cuda:%d" % local, **flags)
    is_train = cfg["kind"] == "train"
    if is_train:
        params = params_from_flags(batch_size=B * world, dtype=args.dtype, **cfg["model"],
                                   **TRAIN_FLAGS)
        tr = Trainer(model, params, 224, 224, use_cuda_graph=not args.no_graph)
        rt = tr.rt
        n_in = tr.input_batch
        dev_step_fn = lambda x, y: tr.train_step(x, y)
        prefetch = tr.prefetch
        result_read = lambda out: out.tolist()
        d2h = 8
    else:
        tr = ForwardRunner(model, B, 224, cfg["kind"], dev)
        tr.use_graph = not args.no_graph
        rt = tr.rt
        n_in = tr.input_batch
        dev_step_fn = lambda x, y: tr.step(x, y)
        prefetch = tr.prefetch
        if cfg["kind"] == "eval":       # the serving result: the predicted class of every image
            result_read = lambda out: out[:, :1001].argmax(dim=1).tolist()
            d2h = 8 * B
        else:
            result_read = lambda out: out.tolist()
            d2h = 4
    x_host, y_host = synth_batch(n_in, 224, 1234 + rank)
    x_host, y_host = x_host.pin_memory(), y_host.pin_memory()
    x_dev, y_dev = x_host.to(dev), y_host.to(dev)
    h2d = x_host.numel() * 4 + (y_host.numel() * 4 if cfg["kind"] != "eval" else 0) + \
        ((n_in // 2) * 4 + 32 if is_train else 0)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item()

    # launches of OUR kernels per step (counted on an eager step; graph replays re-issue them)
    was_graph = tr.use_graph
    tr.use_graph = False
    out_dev = dev_step_fn(x_dev, y_dev)       # first call: one-time setup launches excluded
                                              # (every step writes its result to this buffer)
    torch.cuda.synchronize()
    c0 = lib.acnn_launch_count()
    dev_step_fn(x_dev, y_dev)
    torch.cuda.synchronize()
    launches_per_step = lib.acnn_launch_count() - c0
    tr.use_graph = was_graph

    # ---- device-resident arm -------------------------------------------------------------
    dev_step = lambda: dev_step_fn(x_dev, y_dev)
    # a batch-1 forward touches ~100 MB (weights), comparable to the 50 MB L2: flush L2 between
    # iterations there
    flush = None
    if cfg["kind"] == "eval":
        flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        flush = lambda: flush_buf.fill_(1)
    sampler = ClockSampler(local)
    sampler.start()
    for _ in range(args.warmup):
        dev_step()
    if world == 1 and not args.dump_outputs:
        while sampler.proc is not None and not sampler.lines:  # keep the GPU loaded meanwhile
            dev_step()
            sampler.wait_first_sample(0.05)
    else:
        # every rank must issue the same number of collectives (and a dump must come from the same
        # step every run): no data-dependent extra steps
        sampler.wait_first_sample(3.0)
        for _ in range(args.warmup):
            dev_step()
    sampler.mark()
    if flush is None:
        ms_total = timed(dev_step, args.steps)
    else:
        # per-iteration events around the step only (the flush between them is not timed)
        evs = []
        barrier()
        for _ in range(args.steps):
            flush()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dev_step()
            b.record()
            evs.append((a, b))
        barrier()
        ms_total = sum(a.elapsed_time(b) for a, b in evs)
    clocks = sampler.stop()
    ms_step = ms_total / args.steps
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, cfg, rt, out_dev)
    value = B * world / (ms_step / 1e3)

    # ---- end-to-end arm: pinned host -> H2D -> step -> D2H result, every step -----------------
    # Every step's inputs are copied from pinned host memory inside the timed region; the copy of
    # step i+1 is issued (side stream) before step i is launched, so PCIe overlaps compute.
    def e2e_step():
        out = dev_step_fn(None, None)           # consumes the prefetched batch
        prefetch(x_host, y_host)                # next step's H2D, overlapped with this step
        return result_read(out)                 # D2H read of the step's result
    prefetch(x_host, y_host)
    for _ in range(3):
        e2e_step()
    ms_e2e = timed(e2e_step, args.steps) / args.steps
    e2e_value = B * world / (ms_e2e / 1e3)
    last = e2e_step()

    # ---- roofline of the wgmma conv GEMMs, timed live (CUDA events around every launch) -----
    peaks = read_peaks()
    roof = None
    if rank == 0:
        roof = conv_roofline(tr, rt, lambda: dev_step_fn(x_dev, y_dev), peaks, ms_step)
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu = cpu_baseline_subprocess(args.config)

    if rank == 0:
        gflop = cfg["gflop"]
        line = {
            "metric": cfg["metric"] if args.dtype == "bf16" else cfg["metric"].replace("bf16", "fp32-mode"),
            "value": value, "unit": "images/sec", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": args.dtype,
            "data": "synthetic",
            "config": {"workload": cfg["workload"], "name": args.config,
                       "per_gpu_batch": B, "global_batch": B * world, "parallelism": "dp%d" % world,
                       "l2": ("L2 flushed (256 MiB write) between timed iterations" if flush else
                              "per-step working set (activations + gradients, several GB) >> 50 MB L2"),
                       "cuda_graph": tr.use_graph,
                       "executor": ("libacnn model-level C ABI (acnn_create / acnn_bind / acnn_run_ops)"
                                    if hasattr(rt.plan, "conv_info") else "python plan + per-op ctypes"),
                       "result": last if not isinstance(last, list) or len(last) <= 4 else last[:4]},
            "clocks": clocks,
            "e2e": {"value": e2e_value, "unit": "images/sec", "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h},
            "gpu_launches": int(launches_per_step * args.steps),
            "launches_per_step": int(launches_per_step),
            "conv_flop_roofline": {"gflop_per_img": gflop,
                                   "achieved_tflops": gflop * value / 1e3,
                                   "peak_tflops": peaks["tflops"] * world,
                                   "frac": gflop * value / 1e3 / (peaks["tflops"] * world),
                                   "peak_source": peaks["source"] + (" bf16_tflops_sustained" if peaks["source"] == "measured" else "")},
            "roofline": roof,
            "cpu_baseline": cpu,
        }
        if cfg["kind"] == "eval":
            line["latency_ms"] = ms_step
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


DUMP_SAMPLE = 1 << 20      # elements of each sampled buffer (4 MiB of float32)


def dump_outputs(path, cfg, rt, out):
    """What the device-resident arm computed in its last timed step, as float32 .npy files: the
    step's result (logits of an eval forward; the loss vector of a training-mode step), the logits
    of a training-mode step, and for a training step fixed seeded samples of the updated parameters,
    the gradients and the momentum buffer.  The inputs and the number of steps before the dump are
    fixed by the arguments, so two builds can be compared file by file."""
    import numpy as np
    import torch
    torch.cuda.synchronize()
    os.makedirs(path, exist_ok=True)
    arrs = {}
    if cfg["kind"] == "eval":
        arrs["logits"] = out[:, :1001]
    else:
        arrs["loss"] = out
        m = rt.plan.meta
        if "logits" in m:
            arrs["logits"] = rt.t[m["logits"]][:, :1001]
    if cfg["kind"] == "train":
        for name in ("params", "grads", "momentum"):
            buf = getattr(rt, name, None)
            if buf is None:
                continue
            flat = buf.reshape(-1)
            g = torch.Generator().manual_seed(0)
            n = min(DUMP_SAMPLE, flat.numel())
            idx = torch.randperm(flat.numel(), generator=g)[:n].sort().values
            arrs[name + "_sample"] = flat[idx.to(flat.device)]
            arrs[name + "_sample_index"] = idx.double()
    for name, a in arrs.items():
        a = a.detach().float().cpu().numpy() if not name.endswith("_index") else a.numpy()
        np.save(os.path.join(path, name + ".npy"), a)


def conv_roofline(tr, rt, step_fn, peaks, ms_step):
    """Time every wgmma GEMM launch (fprop / dgrad / wgrad) of one eager step with CUDA events
    on the launching stream; achieved = ALGORITHMIC FLOPs of those launches / their summed time.
    Work the implementation adds on top (the stem's K padded 147 -> 256 by the space-to-depth
    form, the stride-2 dgrads run on zero-inserted gradients) is reported separately as
    `executed_gflop_per_step` and does not count as achieved."""
    import torch
    stream = torch.cuda.current_stream()
    evs = []
    GEMM = ("conv", "conv_dgrad", "conv_wgrad")
    native = hasattr(rt.plan, "conv_info")

    def work_of(op):
        """(algorithmic FLOPs, algorithmic HBM bytes, executed FLOPs) of one GEMM op."""
        if native:      # geometry from the library (acnn_op_conv_info)
            g, macs, aux = rt.plan.conv_info(op)
            Ho, Wo = g.out_hw()
        else:
            g, Ho, Wo = op.geom, op.geom.Ho, op.geom.Wo
            macs = op.a.get("alg_macs") or g.B * Ho * Wo * g.Cout * g.kh * g.kw * g.Cin
            aux = (op.a.get("add_src") is not None) + (op.a.get("mask_src") is not None)
        executed = 2.0 * g.B * Ho * Wo * g.Cout * g.kh * g.kw * g.Cin
        # algorithmic HBM bytes: both activation tensors once (bf16) + the filter (bf16, or the
        # fp32 gradient for wgrad) + the tiles the dgrad epilogue adds / masks with
        nin, nout = g.B * g.H * g.W * g.Cin, g.B * Ho * Wo * g.Cout
        nw = g.kh * g.kw * g.Cin * g.Cout
        byt = 2.0 * (nin + nout) + (4.0 if op.kind == "conv_wgrad" else 2.0) * nw
        if op.kind == "conv_dgrad":
            byt += 2.0 * nin * aux
        return 2.0 * macs, byt, executed

    orig_run = type(rt).run

    def run(ops, **kw):
        """rt.run with every GEMM op launched on its own between two events."""
        i = 0
        while i < len(ops):
            if ops[i].kind in GEMM:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                orig_run(rt, ops[i:i + 1])
                b.record(stream)
                evs.append((a, b) + work_of(ops[i]))
                i += 1
            else:
                j = i
                while j < len(ops) and ops[j].kind not in GEMM:
                    j += 1
                orig_run(rt, ops[i:j])
                i = j

    def run_forward():
        rt.zero_step_buffers()
        run(rt.plan.forward)

    rt.run, rt.run_forward = run, run_forward
    was, was_world = tr.use_graph, tr.world
    tr.use_graph = False
    tr.world = 1        # rank 0 only: no collective inside this instrumented step
    try:
        step_fn()          # warm
        evs.clear()
        step_fn()
        torch.cuda.synchronize()
    finally:
        tr.use_graph = was
        tr.world = was_world
        del rt.run, rt.run_forward
    t_ms = sum(e[0].elapsed_time(e[1]) for e in evs)
    fl = sum(e[2] for e in evs)
    alg_bytes = sum(e[3] for e in evs)
    executed = sum(e[4] for e in evs)
    achieved = fl / (t_ms / 1e3) / 1e12
    # DRAM traffic needs a hardware-counter profile of the same launches: not measured here
    traffic, traffic_src = None, None
    return {"bound": "tensor", "achieved": achieved, "peak": peaks["tflops"], "unit": "TFLOP/s",
            "frac": achieved / peaks["tflops"], "traffic": traffic, "traffic_unit": "bytes per step "
            "(DRAM reads + writes of the same launches; needs hardware counters: not measured)", "traffic_source": traffic_src,
            "algorithmic_bytes_per_step": alg_bytes,
            "kernel": "conv_gemm_kernel + conv_halo_kernel + wgrad_gemm_kernel (all %d wgmma launches of a step)" % len(evs),
            "launch_ms_sum": t_ms, "share_of_step": t_ms / ms_step,
            "algorithmic_gflop_per_step": fl / 1e9,
            "executed_gflop_per_step": executed / 1e9,
            "peak_source": peaks["source"] + (" bf16_tflops_sustained" if peaks["source"] == "measured" else "") +
                           " (kernel timed inside a long step)"}


if __name__ == "__main__":
    main()
