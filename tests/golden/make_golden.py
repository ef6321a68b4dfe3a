#!/usr/bin/env python
"""Generates tests/golden/oracle_digests.json: digests of the oracle's outputs under fixed seeds.

The reference ships no golden vectors for this path and TensorFlow 1.14 cannot be run
here, so these fixtures pin the ORACLE (oracle/model.py) against silent change; they use the
reference's own digest convention (official/utils/testing/reference_data.py:105-124:
shape, first, last, sum).  Re-run only when the oracle is intentionally changed:

    python tests/golden/make_golden.py
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import model as M, tf_ops as T  # noqa: E402

ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)
CONFIGS = {
    # BASELINE configs at oracle-affordable sizes (seeds data=1234, weights=42, lam=7: BASELINE.md s.3)
    "C1_vanilla_r50_eval_b1_224": dict(kw=dict(resnet_size=50, resnet_version=1), d=False, B=1,
                                       hw=224, train=False, mix=0),
    "C2_assemble_r50_fwd_loss_b4_128": dict(kw=ASSEMBLE, d=False, B=4, hw=128, train=True, mix=0),
    "C3_assemble_r50_train_mixup_b4_128": dict(kw=ASSEMBLE, d=False, B=4, hw=128, train=True, mix=1),
    "alt_r50_d_sk_aa_train_b4_64": dict(kw=dict(resnet_size=50, resnet_version=1, use_sk_block=True,
                                                anti_alias_type="sconv", anti_alias_filter_size=3),
                                        d=True, B=4, hw=64, train=True, mix=0),
}


def digest(t):
    f = t.detach().double().flatten()
    return {"shape": list(t.shape), "first": f[0].item(), "last": f[-1].item(), "sum": f.sum().item(),
            "abs_sum": f.abs().sum().item()}


def run(cfg):
    model, vs = M.build(seed=42, input_hw=64, use_resnet_d=cfg["d"], **cfg["kw"])
    B, hw = cfg["B"], cfg["hw"]
    n_in = 2 * B if cfg["mix"] == 1 else B
    g = torch.Generator().manual_seed(1234)
    x = (torch.randn(n_in, hw, hw, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (n_in,), generator=g)
    onehot = torch.nn.functional.one_hot(lab, 1001).float()
    out = {}
    if cfg["mix"]:
        lam = torch.rand(B, generator=torch.Generator().manual_seed(7))
        x, onehot = T.mixup(x, onehot, lam, keep_batch_size=False)
    if not cfg["train"]:
        out["logits"] = digest(M.forward(model, vs, x, training=False, use_resnet_d=cfg["d"]))
        return out
    names = [n for n in vs.vars if vs.trainable[n]]
    mom = {n: torch.zeros_like(vs.vars[n]) for n in names}
    res = M.train_step(model, vs, mom, x, onehot, lr=0.1, momentum=0.9, use_resnet_d=cfg["d"],
                       label_smoothing=0.1, weight_decay=1e-4)
    out["logits"] = digest(res["logits"])
    out["loss"] = res["loss"].item()
    out["cross_entropy"] = res["cross_entropy"].item()
    out["l2_loss"] = res["l2_loss"].item()
    for n in (names[0], names[len(names) // 2], "resnet_model/dense/kernel", "resnet_model/dense/bias"):
        out["grad:" + n] = digest(res["grads"][n])
    return out


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 1)
    result = {name: run(cfg) for name, cfg in CONFIGS.items()}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_digests.json")
    with open(path, "w") as fh:
        json.dump(result, fh, indent=1, sort_keys=True)
    print("wrote", path)
