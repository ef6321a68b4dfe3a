#!/usr/bin/env python
"""The cost of AutoAugment on the device, on synthetic data: crop windows drawn by the training sampler from
500 x 375 sources, AutoAugment records drawn by autoaugment.resolve.

    python tools/bench_autoaugment.py [--iters 20] [--warmup 5]

CUDA-event times (median of --iters after --warmup):
  pass   acnn_crop_resize_autoaugment_u8 against acnn_crop_resize_u8 at B = 256 and 512, S = 224, with
         `imagenet` and `good` draws, alternated in one run
  step   the c3 training step (Assemble-ResNet-50: mixup type 1, label smoothing 0.1, bf16, 224 px, batch 256,
         so 512 examples per step) fed through Trainer.train_step_cropped(augment=) against the same step fed
         through train_step_cropped without it, alternated in one run
Prints the card name and power limit read in the same run and one JSON line per measurement."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from assembled_cnn_b200 import _lib  # noqa: E402
from assembled_cnn_b200 import autoaugment as A  # noqa: E402
from assembled_cnn_b200 import imagenet_train as it  # noqa: E402
from assembled_cnn_b200.hparams import params_from_flags  # noqa: E402
from assembled_cnn_b200.model_fns import Trainer, build_model  # noqa: E402
from assembled_cnn_b200.staging import pack_u8  # noqa: E402
from bench_train_input import FLAGS, card, event_ms, windows  # noqa: E402

SIZE, BATCH = 224, 256


def device_inputs(B, policy, seed):
    wins = windows(B, seed)
    hbuf, dbuf, addrs = pack_u8(None, None, [w for w, _ in wins], torch.device("cuda"))
    desc = np.zeros(B, it.CROP_DESC_DTYPE)
    for i, (w, f) in enumerate(wins):
        desc[i] = (addrs[i], w.shape[0], w.shape[1], int(f), (0, 0, 0))
    aug = np.array([A.resolve(policy, SIZE, np.random.default_rng([seed, i])) for i in range(B)],
                   A.AUTOAUG_DESC_DTYPE)
    A.check_autoaugment_descriptors(aug, SIZE)
    return (dbuf, torch.from_numpy(desc.view(np.uint8).copy()).cuda(),
            torch.from_numpy(aug.view(np.uint8).copy()).cuda(), int((aug["slot"]["op"] != 0).sum()))


def bench_pass(B, policy, a):
    lib = _lib.load()
    keep, desc, aug, applied = device_inputs(B, policy, B)
    out = torch.empty(B, SIZE, SIZE, 3, device="cuda")
    work = torch.empty(lib.acnn_autoaugment_work_bytes(B, SIZE), dtype=torch.uint8, device="cuda")
    mean = torch.tensor(it.CHANNEL_MEANS, device="cuda")
    st = lambda: torch.cuda.current_stream().cuda_stream
    plain = lambda: _lib.check(lib.acnn_crop_resize_u8(desc.data_ptr(), B, B, SIZE, mean.data_ptr(), out.data_ptr(),
                                                       st()), "crop")
    augd = lambda: _lib.check(lib.acnn_crop_resize_autoaugment_u8(desc.data_ptr(), aug.data_ptr(), B, B, SIZE,
                                                                  mean.data_ptr(), work.data_ptr(), out.data_ptr(),
                                                                  st()), "autoaugment")
    for _ in range(a.warmup):
        plain()
        augd()
    tp, ta = [], []
    for _ in range(a.iters):
        tp.append(event_ms(plain))
        ta.append(event_ms(augd))
    return {"batch": B, "policy": policy, "ops_applied": applied, "crop_resize_ms": round(statistics.median(tp), 4),
            "autoaugment_ms": round(statistics.median(ta), 4),
            "extra_ms": round(statistics.median(ta) - statistics.median(tp), 4)}


def bench_step(a):
    model = build_model(dtype="bf16", **FLAGS)
    p = params_from_flags(batch_size=BATCH, mixup_type=1, label_smoothing=0.1, dtype="bf16", **FLAGS)
    tr = Trainer(model, p, SIZE, SIZE)
    n = tr.input_batch
    keep, desc, aug, _ = device_inputs(n, "imagenet", 7)
    lab = torch.tensor(np.random.default_rng(0).integers(0, 1001, n), dtype=torch.int32, device="cuda")
    lam = it.mixup_lambdas(0, 0, 0, n // 2)
    mean = torch.tensor(it.CHANNEL_MEANS, device="cuda")
    plain = lambda: tr.train_step_cropped(desc, lab, mean, lam1=lam)
    augd = lambda: tr.train_step_cropped(desc, lab, mean, lam1=lam, augment=aug)
    for _ in range(a.warmup):            # the first step captures the graph
        plain()
        augd()
    torch.cuda.synchronize()
    tp, ta = [], []
    for _ in range(a.iters):
        tp.append(event_ms(plain))
        ta.append(event_ms(augd))
    out = {"input_batch": n, "policy": "imagenet", "cropped_step_ms": round(statistics.median(tp), 3),
           "augmented_step_ms": round(statistics.median(ta), 3)}
    out["extra_ms"] = round(out["augmented_step_ms"] - out["cropped_step_ms"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_autoaugment: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    for B in (256, 512):
        for policy in ("imagenet", "good"):
            print(json.dumps(bench_pass(B, policy, a)), flush=True)
    print(json.dumps(bench_step(a)), flush=True)


if __name__ == "__main__":
    main()
