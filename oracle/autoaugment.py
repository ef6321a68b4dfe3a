"""Restatement of the reference's AutoAugment (preprocessing/autoaugment.py) in numpy, for the tests
(independent of assembled_cnn_b200).  Images are uint8 [S, S, 3]; every float step is a separately rounded
float32 operation (numpy never contracts to FMA).

  apply_op        one operation at a level, its argument negated or not, Cutout at a given centre:
    Invert        255 - x
    Posterize     (x >> s) << s, s = 8 - int(level / 10 * 4) clamped to [0, 7] (TF's uint8 shifts)
    Solarize      x < t ? x : 255 - x, t = int(level / 10 * 256) as a uint8 constant (256 wraps to 0)
    SolarizeAdd   x < 128 ? clip(x + int(level / 10 * 110)) : x
    AutoContrast  per channel, lo / hi its float min / max; hi > lo: x * (255 / (hi - lo)) + (-lo * scale)
    Equalize      PIL's ImageOps.equalize per channel in integers
    blend         img1 + f * (img2 - img1), clipped and truncated; f == 0: img1, f == 1: img2;
                  f = level / 10 * 1.8 + 0.1 (float64, then float32)
    Color         blend(grey, x), grey = trunc(((r/255 * .2989 + g/255 * .587) + b/255 * .114) * 255.5)
    Contrast      blend(min(trunc(S * S / 256), 255), x)   (sum(histogram) / 256, the reference's "mean")
    Brightness    blend(0, x)
    Sharpness     blend(smooth, x), smooth = 3x3 VALID [[1,1,1],[1,5,1],[1,1,1]] / 13 (taps left to right),
                  clipped, truncated, the border kept
    Rotate, ShearX/Y, TranslateX/Y  output (x, y) reads (round(t3 x + t4 y + t5), round(t0 x + t1 y + t2)),
                  round half away from zero; outside the image: (128, 128, 128)
    Cutout        rows [max(0, cy - p), min(S, cy + p)) x columns [max(0, cx - p), min(S, cx + p)) = 128,
                  p = int(level / 10 * 100)
  augment         a sub-policy's two operations in order, each applied or not
  preprocess      the training image with autoaugment_type set: the resize of oracle/train_preprocess.py,
                  clipped and truncated to uint8, augment, float32, - CHANNEL_MEANS
"""
import math

import numpy as np

from oracle.eval_preprocess import CHANNEL_MEANS, resize_bilinear

f32 = np.float32


def _trunc_u8(v):
    return np.clip(v, f32(0), f32(255)).astype(np.uint8)


def blend(img1, img2, factor):
    if factor == 0.0:
        return img1.copy()
    if factor == 1.0:
        return img2.copy()
    a, b = img1.astype(f32), img2.astype(f32)
    return _trunc_u8(a + f32(factor) * (b - a))


def grey(img):
    x = img.astype(f32) * f32(1.0 / 255.0)
    g = x[..., 0] * f32(0.2989) + x[..., 1] * f32(0.5870)
    g = g + x[..., 2] * f32(0.1140)
    return np.repeat((g * f32(255.5)).astype(np.uint8)[..., None], 3, axis=2)


def autocontrast(img):
    out = img.copy()
    for c in range(3):
        ch = img[..., c]
        lo, hi = f32(ch.min()), f32(ch.max())
        if hi > lo:
            scale = f32(255.0) / (hi - lo)
            offset = -lo * scale
            out[..., c] = _trunc_u8(ch.astype(f32) * scale + offset)
    return out


def equalize(img):
    out = img.copy()
    for c in range(3):
        ch = img[..., c]
        hist = np.bincount(ch.reshape(-1), minlength=256).astype(np.int64)
        nz = hist[hist != 0]
        step = (nz.sum() - nz[-1]) // 255
        if step == 0:
            continue
        lut = (np.cumsum(hist) + step // 2) // step
        lut = np.clip(np.concatenate([[0], lut[:-1]]), 0, 255)
        out[..., c] = lut[ch]
    return out


def sharpness(img, factor):
    S = img.shape[0]
    x = img.astype(f32)
    smooth = img.copy()
    if S >= 3 and img.shape[1] >= 3:
        w = np.full((3, 3), f32(1.0) / f32(13.0), f32)
        w[1, 1] = f32(5.0) / f32(13.0)
        acc = np.zeros((S - 2, img.shape[1] - 2, 3), f32)
        for ky in range(3):
            for kx in range(3):
                acc = acc + x[ky:ky + S - 2, kx:kx + img.shape[1] - 2] * w[ky, kx]
        smooth[1:-1, 1:-1] = _trunc_u8(acc)
    return blend(smooth, img, factor)


def _round_half_away(v):
    a = np.abs(v.astype(np.float64))
    return np.sign(v) * np.floor(a + 0.5)


def transform(img, t):
    """NEAREST projective transform with coefficients t0..t5 (float32), unwrap's grey outside."""
    H, W = img.shape[:2]
    t = [f32(v) for v in t]
    y, x = np.meshgrid(np.arange(H, dtype=f32), np.arange(W, dtype=f32), indexing="ij")
    ix = _round_half_away((t[0] * x + t[1] * y) + t[2])
    iy = _round_half_away((t[3] * x + t[4] * y) + t[5])
    inside = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    out = np.full_like(img, 128)
    out[inside] = img[iy[inside].astype(np.int64), ix[inside].astype(np.int64)]
    return out


def rotate_coeffs(degrees, H, W):
    rad = f32(f32(degrees) * f32(math.pi / 180.0))
    c, s = f32(math.cos(float(rad))), f32(math.sin(float(rad)))
    h1, w1 = f32(H - 1), f32(W - 1)
    xo = (w1 - (c * w1 - s * h1)) / f32(2.0)
    yo = (h1 - (s * w1 + c * h1)) / f32(2.0)
    return [c, -s, xo, s, c, yo]


def apply_op(img, name, level, negate=False, centre=(0, 0)):
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    sign = f32(-1.0) if negate else f32(1.0)
    if name == "Invert":
        return 255 - img
    if name == "AutoContrast":
        return autocontrast(img)
    if name == "Equalize":
        return equalize(img)
    if name == "Posterize":
        s = min(max(8 - int((level / 10.0) * 4), 0), 7)
        return ((img >> s) << s).astype(np.uint8)
    if name == "Solarize":
        t = int((level / 10.0) * 256) % 256
        return np.where(img < t, img, 255 - img).astype(np.uint8)
    if name == "SolarizeAdd":
        a = int((level / 10.0) * 110)
        return np.where(img < 128, np.clip(img.astype(np.int64) + a, 0, 255), img).astype(np.uint8)
    if name in ("Color", "Contrast", "Brightness", "Sharpness"):
        f = (level / 10.0) * 1.8 + 0.1
        if name == "Color":
            return blend(grey(img), img, f)
        if name == "Contrast":
            g = int(min(f32(f32(H * W) / f32(256.0)), f32(255.0)))
            return blend(np.full_like(img, g), img, f)
        if name == "Brightness":
            return blend(np.zeros_like(img), img, f)
        return sharpness(img, f)
    if name == "Rotate":
        return transform(img, rotate_coeffs(sign * f32((level / 10.0) * 30.0), H, W))
    if name in ("ShearX", "ShearY"):
        a = sign * f32((level / 10.0) * 0.3)
        return transform(img, [1, a, 0, 0, 1, 0] if name == "ShearX" else [1, 0, 0, a, 1, 0])
    if name in ("TranslateX", "TranslateY"):
        a = sign * f32((level / 10.0) * 250.0)
        return transform(img, [1, 0, a, 0, 1, 0] if name == "TranslateX" else [1, 0, 0, 0, 1, a])
    if name == "Cutout":
        p = int((level / 10.0) * 100)
        cy, cx = centre
        out = img.copy()
        out[max(0, cy - p):min(H, cy + p), max(0, cx - p):min(W, cx + p)] = 128
        return out
    raise ValueError(name)


def augment(img, subpolicy, applied, negated=(False, False), centres=((0, 0), (0, 0))):
    """subpolicy: ((name, prob, level), (name, prob, level)); slot j runs when applied[j]."""
    out = np.asarray(img, np.uint8)
    for j, (name, _, level) in enumerate(subpolicy):
        if applied[j]:
            out = apply_op(out, name, level, negated[j], centres[j])
    return out


def resized_u8(window, flip, S):
    a = np.asarray(window)
    if flip:
        a = a[:, ::-1]
    return _trunc_u8(resize_bilinear(a, S, S))


def preprocess(window, flip, S, subpolicy, applied, negated=(False, False), centres=((0, 0), (0, 0)),
               means=CHANNEL_MEANS):
    img = augment(resized_u8(window, flip, S), subpolicy, applied, negated, centres)
    return img.astype(f32) - np.asarray(means, dtype=f32)
