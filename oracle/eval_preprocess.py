"""Restatement of the reference's ImageNet eval preprocessing and classification metrics, for the tests.

  geometry        preprocessing/imagenet_preprocessing.py:158-186 (_smallest_size_at_least, in float32 as
                  tf.float32), :100-119 (central_crop), :305-310 (resize_min per crop_type) and the
                  imagenet-family dispatch of utils/data_util.py:267-345
  resize_bilinear TF 1.14 resize_bilinear, align_corners = half_pixel_centers = False (the legacy
                  scaler), float32, every operation separately rounded (numpy never contracts to FMA)
  preprocess      resize, central crop, - CHANNEL_MEANS in float32
  argmax / in_top_k / softmax_conf / cross_entropy / ece: tf.argmax, tf.nn.in_top_k (fewer than k logits
                  strictly above the target's; out-of-range label or non-finite row -> False),
                  max softmax, tf.losses.softmax_cross_entropy(label_smoothing), metric/ece_metric.py,
                  in float64
"""
import re

import numpy as np

CHANNEL_MEANS = (123.68, 116.78, 103.94)


def eval_size(preprocessing_type, image_size=224):
    if preprocessing_type == "imagenet":
        return image_size, 0
    if preprocessing_type == "imagenet_224_256":
        return 256, 0
    if preprocessing_type == "imagenet_224_256a":
        return 256, 1
    if re.compile("imagenet_[0-9]{3}a").match(preprocessing_type):
        return int(preprocessing_type.split("_")[1][0:3]), 1
    if re.compile("imagenet_[0-9]{3}").match(preprocessing_type):
        return int(preprocessing_type.split("_")[1]), 0
    raise NotImplementedError(preprocessing_type)


def geometry(h, w, preprocessing_type="imagenet", image_size=224):
    """(S, rsz_h, rsz_w, crop_y, crop_x)."""
    s, crop_type = eval_size(preprocessing_type, image_size)
    resize_min = s + 1 if crop_type == 1 else int(s * (1.0 / 0.875))
    hf, wf = np.float32(h), np.float32(w)
    ratio = np.float32(resize_min) / np.minimum(hf, wf)
    rh, rw = int(np.int32(hf * ratio)), int(np.int32(wf * ratio))
    return s, rh, rw, (rh - s) // 2, (rw - s) // 2


def _weights(out_size, in_size, start=0, n=None):
    scale = np.float32(in_size) / np.float32(out_size)
    x = np.arange(start, start + (out_size if n is None else n), dtype=np.float32) * scale
    f = np.floor(x)
    lo = np.maximum(f.astype(np.int64), 0)
    hi = np.minimum(np.ceil(x).astype(np.int64), in_size - 1)
    return lo, hi, (x - f).astype(np.float32)


def resize_bilinear(img, out_h, out_w, window=None):
    """float32 [out_h, out_w, C] of an [H, W, C] image; window = (y0, x0, s): only its s x s pixels."""
    a = np.asarray(img).astype(np.float32)
    y0, x0, s = window if window is not None else (0, 0, None)
    ylo, yhi, yl = _weights(out_h, a.shape[0], y0, s)
    xlo, xhi, xl = _weights(out_w, a.shape[1], x0, s)
    xl = xl[None, :, None]
    top = a[ylo][:, xlo] + (a[ylo][:, xhi] - a[ylo][:, xlo]) * xl
    bot = a[yhi][:, xlo] + (a[yhi][:, xhi] - a[yhi][:, xlo]) * xl
    return (top + (bot - top) * yl[:, None, None]).astype(np.float32)


def preprocess(img, preprocessing_type="imagenet", image_size=224, means=CHANNEL_MEANS):
    """float32 [S, S, 3]: resize_bilinear to the eval geometry, central crop, - means."""
    s, rh, rw, cy, cx = geometry(img.shape[0], img.shape[1], preprocessing_type, image_size)
    r = resize_bilinear(img, rh, rw, (cy, cx, s))      # each pixel depends on its own coordinates only
    return r - np.asarray(means, dtype=np.float32)


def argmax(logits):
    x = np.asarray(logits, np.float64)
    out = x.argmax(1)
    out[~np.isfinite(x).all(1)] = -1
    return out


def in_top_k(logits, labels, k):
    x = np.asarray(logits, np.float64)
    labels = np.asarray(labels)
    out = np.zeros(len(x), dtype=bool)
    for r in range(len(x)):
        t = labels[r]
        if 0 <= t < x.shape[1] and np.isfinite(x[r]).all():
            out[r] = (x[r] > x[r, t]).sum() < k
    return out


def softmax_conf(logits):
    x = np.asarray(logits, np.float64)
    e = np.exp(x - x.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).max(1)


def cross_entropy(logits, labels, label_smoothing=0.0):
    x = np.asarray(logits, np.float64)
    nc = x.shape[1]
    m = x.max(1, keepdims=True)
    logp = x - m - np.log(np.exp(x - m).sum(1, keepdims=True))
    t = np.full(x.shape, label_smoothing / nc)
    t[np.arange(len(x)), np.asarray(labels)] += 1.0 - label_smoothing
    return -(t * logp).sum(1)


def ece(conf, pred, labels, num_thresholds=10):
    eps = 1e-7
    th = np.float32([0.0 - eps] + [(i + 1) * 1.0 / num_thresholds for i in range(num_thresholds - 1)]
                    + [1.0 + eps])
    c = np.asarray(conf, np.float32)
    ok = np.asarray(pred) == np.asarray(labels)
    acc_sum, conf_sum, cnt = np.zeros(num_thresholds), np.zeros(num_thresholds), np.zeros(num_thresholds)
    for i in range(num_thresholds):
        inb = (c > th[i]) & (c <= th[i + 1])
        cnt[i] = inb.sum()
        acc_sum[i] = (inb & ok).sum()
        conf_sum[i] = c[inb].astype(np.float64).sum()
    acc, avg = acc_sum / (eps + cnt), conf_sum / (eps + cnt)
    return float((cnt / cnt.sum() * np.abs(acc - avg)).sum())
