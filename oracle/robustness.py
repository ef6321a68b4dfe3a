"""Float64 CPU restatement of the reference's robustness evaluation (mce/eval_robustness.py,
--robustness_type ce), the yardstick of metrics.CorruptionError and model_fns.corruption_error.

  top1            tf.nn.top_k(tf.nn.softmax(logits), 1) (:186-187) in float64: the smallest index of the
                  largest probability
  errors          err = 1 - correct / num_of_images per distortion (:231-232), ce = err / ALEXNET_CE[d]
                  (:282-285)
  mce             np.mean of the 19 normalised CEs and of the 19 errors (:297-300)
  quota           process() (:249-278): the cumulative end indices, and distortions[start:end] per GPU
"""
from __future__ import annotations

import numpy as np

# mce/eval_robustness.py:91-97, in its order
ALEXNET_CE = {
    "gaussian_noise": 0.8864, "shot_noise": 0.8945, "impulse_noise": 0.9226,
    "defocus_blur": 0.8199, "glass_blur": 0.8263, "motion_blur": 0.7860, "zoom_blur": 0.7984,
    "snow": 0.8668, "frost": 0.8266, "fog": 0.8193, "brightness": 0.5646,
    "contrast": 0.8532, "elastic_transform": 0.6461, "pixelate": 0.7178, "jpeg_compression": 0.6065,
    "speckle_noise": 0.8454, "gaussian_blur": 0.7871, "spatter": 0.7175, "saturate": 0.6583,
}


def top1(logits):
    """Per row: the smallest index of the largest float64 softmax probability."""
    x = np.asarray(logits, dtype=np.float64)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return (e / e.sum(axis=1, keepdims=True)).argmax(axis=1)


def errors(correct, count, table=ALEXNET_CE):
    """{d: (err, ce)} from per-distortion counts; every distortion needs images (the reference asserts)."""
    out = {}
    for d, alex in table.items():
        assert count[d] > 0, d
        err = 1.0 - float(correct[d]) / float(count[d])
        out[d] = (err, err / alex)
    return out


def mce(correct, count, table=ALEXNET_CE):
    """(mCE, unnormalised mCE, per-distortion {d: (err, ce)})."""
    per = errors(correct, count, table)
    return (float(np.mean([per[d][1] for d in table])), float(np.mean([per[d][0] for d in table])), per)


def quota(num_gpus, distortions=tuple(ALEXNET_CE)):
    """The distortions of each GPU, statement for statement as process() computes its slice."""
    n = len(distortions)
    quota_base, overtime_task = n // num_gpus, n % num_gpus
    ends, base = [], 0
    for i in range(num_gpus):
        base += quota_base + 1 if i < overtime_task else quota_base
        ends.append(base)
    return [list(distortions[0 if i == 0 else ends[i - 1]:ends[i]]) for i in range(num_gpus)]
