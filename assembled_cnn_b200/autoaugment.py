"""AutoAugment of the training input (preprocessing/autoaugment.py distort_image_with_autoaugment, applied by
preprocessing/imagenet_preprocessing.py:282-289 after the resize): the policies, the random draws of one image,
and the descriptor that tells the device (acnn_crop_resize_autoaugment_u8, include/acnn.h) what to do.

A policy is a list of sub-policies, each two operations (name, probability, level).  For one image:
  1. one sub-policy is drawn uniformly;
  2. each of its operations applies when floor(u + prob), in float32 and cast to bool, is true, u a uniform
     draw (u + 1.0 can round to 2.0);
  3. Rotate, ShearX/Y and TranslateX/Y negate their argument when floor(u' + 0.5) == 0 in float32;
  4. Cutout draws its centre row, then its centre column, each a uniform int in [0, S).
resolve() makes these draws from a numpy Generator in this fixed order: the sub-policy index, then per slot
the apply draw, then the sign draw (signed operations) or the two centre draws (Cutout).  The sign and centre
draws are made whether or not the operation applies, so the number of draws depends on the sub-policy only.
Uniforms are float32 on the 2^-24 grid of [0, 1): rng.integers(0, 2**24) * 2**-24.

The level of an operation becomes its argument in float64, as Python computes it in the reference
(_MAX_LEVEL = 10, translate_const = 250, cutout_const = 100), and then float32 or int.  Descriptor arguments
per operation are listed with acnn_autoaugment_desc in include/acnn.h.  Two corners of the v0 policy:
  * ('Posterize', 0.8, 2) gives bits = 0, a shift of 8; TF's shift ops clamp the shift to [0, 7] for uint8,
    so it is 7.
  * ('Solarize', 0.6, 10) gives the threshold 256.  `image < 256` converts 256 to a uint8 constant: TF 1.14's
    make_tensor_proto does np.array(256, dtype=np.uint8), which wraps to 0 with the numpy it was released
    with.  Nothing is below 0, so every pixel becomes 255 - x.
Rotate's projective transform is computed here: TF 1.14's angles_to_projective_transforms in float32, with
cos / sin of the float32 angle taken in float64 and rounded to float32 (equal to the C library's cosf / sinf
for every angle the tables produce; tests/test_autoaugment_cpu.py checks it).
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32

OPS = ("Identity", "AutoContrast", "Equalize", "Invert", "Rotate", "Posterize", "Solarize", "SolarizeAdd", "Color",
       "Contrast", "Brightness", "Sharpness", "ShearX", "ShearY", "TranslateX", "TranslateY", "Cutout")
OP_CODE = {n: i for i, n in enumerate(OPS)}          # include/acnn.h ACNN_AA_*
SIGNED = frozenset(("Rotate", "ShearX", "ShearY", "TranslateX", "TranslateY"))   # also the transforms
BLENDS = frozenset(("Color", "Contrast", "Brightness", "Sharpness"))
MAX_LEVEL, TRANSLATE_CONST, CUTOUT_CONST = 10.0, 250, 100

# include/acnn.h acnn_autoaugment_desc
AUTOAUG_OP_DTYPE = np.dtype([("op", "<i4"), ("i", "<i4", (3,)), ("f", "<f4", (6,))])
AUTOAUG_DESC_DTYPE = np.dtype([("subpolicy", "<i4"), ("reserved", "<i4"), ("slot", AUTOAUG_OP_DTYPE, (2,))])
assert AUTOAUG_OP_DTYPE.itemsize == 40 and AUTOAUG_DESC_DTYPE.itemsize == 88

# One sub-policy per line: "name probability level, name probability level".
_TABLES = {
    "v0": """
        Equalize 0.8 1, ShearY 0.8 4
        Color 0.4 9, Equalize 0.6 3
        Color 0.4 1, Rotate 0.6 8
        Solarize 0.8 3, Equalize 0.4 7
        Solarize 0.4 2, Solarize 0.6 2
        Color 0.2 0, Equalize 0.8 8
        Equalize 0.4 8, SolarizeAdd 0.8 3
        ShearX 0.2 9, Rotate 0.6 8
        Color 0.6 1, Equalize 1.0 2
        Invert 0.4 9, Rotate 0.6 0
        Equalize 1.0 9, ShearY 0.6 3
        Color 0.4 7, Equalize 0.6 0
        Posterize 0.4 6, AutoContrast 0.4 7
        Solarize 0.6 8, Color 0.6 9
        Solarize 0.2 4, Rotate 0.8 9
        Rotate 1.0 7, TranslateY 0.8 9
        ShearX 0.0 0, Solarize 0.8 4
        ShearY 0.8 0, Color 0.6 4
        Color 1.0 0, Rotate 0.6 2
        Equalize 0.8 4, Equalize 0.0 8
        Equalize 1.0 4, AutoContrast 0.6 2
        ShearY 0.4 7, SolarizeAdd 0.6 7
        Posterize 0.8 2, Solarize 0.6 10
        Solarize 0.6 8, Equalize 0.6 1
        Color 0.8 6, Rotate 0.4 5""",
    "imagenet": """
        Posterize 0.4 8, Rotate 0.6 9
        Solarize 0.6 5, AutoContrast 0.6 5
        Equalize 0.8 8, Equalize 0.6 3
        Posterize 0.6 7, Posterize 0.6 6
        Equalize 0.4 7, Solarize 0.2 4
        Equalize 0.4 4, Rotate 0.8 8
        Solarize 0.6 3, Equalize 0.6 7
        Posterize 0.8 5, Equalize 1.0 2
        Rotate 0.2 3, Solarize 0.6 8
        Equalize 0.6 8, Posterize 0.4 6
        Rotate 0.8 8, Color 0.4 0
        Rotate 0.4 9, Equalize 0.6 2
        Equalize 0.0 7, Equalize 0.8 8
        Invert 0.6 4, Equalize 1.0 8
        Color 0.6 4, Contrast 1.0 8
        Rotate 0.8 8, Color 1.0 2
        Color 0.8 8, Solarize 0.8 7
        Sharpness 0.4 7, Invert 0.6 8
        ShearX 0.6 5, Equalize 1.0 9
        Color 0.4 0, Equalize 0.6 3
        Equalize 0.4 7, Solarize 0.2 4
        Solarize 0.6 5, AutoContrast 0.6 5
        Invert 0.6 4, Equalize 1.0 8
        Color 0.6 4, Contrast 1.0 8
        Equalize 0.8 8, Equalize 0.6 3""",
    "good": """
        Invert 0.1 7, Contrast 0.2 6
        Rotate 0.7 2, TranslateX 0.3 9
        Sharpness 0.8 1, Sharpness 0.9 3
        ShearY 0.5 8, TranslateY 0.7 9
        AutoContrast 0.5 8, Equalize 0.9 2
        Solarize 0.4 5, AutoContrast 0.9 3
        TranslateY 0.9 9, TranslateY 0.7 9
        AutoContrast 0.9 2, Solarize 0.8 3
        Equalize 0.8 8, Invert 0.1 3
        TranslateY 0.7 9, AutoContrast 0.9 1
        Solarize 0.4 5, AutoContrast 0.0 2
        TranslateY 0.7 9, TranslateY 0.7 9
        AutoContrast 0.9 0, Solarize 0.4 3
        Equalize 0.7 5, Invert 0.1 3
        TranslateY 0.7 9, TranslateY 0.7 9
        Solarize 0.4 5, AutoContrast 0.9 1
        TranslateY 0.8 9, TranslateY 0.9 9
        AutoContrast 0.8 0, TranslateY 0.7 9
        TranslateY 0.2 7, Color 0.9 6
        Equalize 0.7 6, Color 0.4 9
        ShearY 0.2 7, Posterize 0.3 7
        Color 0.4 3, Brightness 0.6 7
        Sharpness 0.3 9, Brightness 0.7 9
        Equalize 0.6 5, Equalize 0.5 1
        Contrast 0.6 7, Sharpness 0.6 5
        Brightness 0.3 7, AutoContrast 0.5 8
        AutoContrast 0.9 4, AutoContrast 0.5 6
        Solarize 0.3 5, Equalize 0.6 5
        TranslateY 0.2 4, Sharpness 0.3 3
        Brightness 0.0 8, Color 0.8 8
        Solarize 0.2 6, Color 0.8 6
        Solarize 0.2 6, AutoContrast 0.8 1
        Solarize 0.4 1, Equalize 0.6 5
        Brightness 0.0 0, Solarize 0.5 2
        AutoContrast 0.9 5, Brightness 0.5 3
        Contrast 0.7 5, Brightness 0.0 2
        Solarize 0.2 8, Solarize 0.1 5
        Contrast 0.5 1, TranslateY 0.2 9
        AutoContrast 0.6 5, TranslateY 0.0 9
        AutoContrast 0.9 4, Equalize 0.8 4
        Brightness 0.0 7, Equalize 0.4 7
        Solarize 0.2 5, Equalize 0.7 5
        Equalize 0.6 8, Color 0.6 2
        Color 0.3 7, Color 0.2 4
        AutoContrast 0.5 2, Solarize 0.7 2
        AutoContrast 0.2 0, Equalize 0.1 0
        ShearY 0.6 5, Equalize 0.6 5
        Brightness 0.9 3, AutoContrast 0.4 1
        Equalize 0.8 8, Equalize 0.7 7
        Equalize 0.7 7, Solarize 0.5 0
        Equalize 0.8 4, TranslateY 0.8 9
        TranslateY 0.8 9, TranslateY 0.6 9
        TranslateY 0.9 0, TranslateY 0.5 9
        AutoContrast 0.5 3, Solarize 0.3 4
        Solarize 0.5 3, Equalize 0.4 4
        Color 0.7 7, TranslateX 0.5 8
        Equalize 0.3 7, AutoContrast 0.4 8
        TranslateY 0.4 3, Sharpness 0.2 6
        Brightness 0.9 6, Color 0.2 8
        Solarize 0.5 2, Invert 0.0 3
        AutoContrast 0.1 5, Brightness 0.0 0
        Cutout 0.2 4, Equalize 0.1 1
        Equalize 0.7 7, AutoContrast 0.6 4
        Color 0.1 8, ShearY 0.2 3
        ShearY 0.4 2, Rotate 0.7 0
        ShearY 0.1 3, AutoContrast 0.9 5
        TranslateY 0.3 6, Cutout 0.3 3
        Equalize 0.5 0, Solarize 0.6 6
        AutoContrast 0.3 5, Rotate 0.2 7
        Equalize 0.8 2, Invert 0.4 0
        Equalize 0.9 5, Color 0.7 0
        Equalize 0.1 1, ShearY 0.1 3
        AutoContrast 0.7 3, Equalize 0.7 0
        Brightness 0.5 1, Contrast 0.1 7
        Contrast 0.1 4, Solarize 0.6 5
        Solarize 0.2 3, ShearX 0.0 0
        TranslateX 0.3 0, TranslateX 0.6 0
        Equalize 0.5 9, TranslateY 0.6 7
        ShearX 0.1 0, Sharpness 0.5 1
        Equalize 0.8 6, Invert 0.3 6
        AutoContrast 0.3 9, Cutout 0.5 3
        ShearX 0.4 4, AutoContrast 0.9 2
        ShearX 0.0 3, Posterize 0.0 3
        Solarize 0.4 3, Color 0.2 4
        Equalize 0.1 4, Equalize 0.7 6
        Equalize 0.3 8, AutoContrast 0.4 3
        Solarize 0.6 4, AutoContrast 0.7 6
        AutoContrast 0.2 9, Brightness 0.4 8
        Equalize 0.1 0, Equalize 0.0 6
        Equalize 0.8 4, Equalize 0.0 4
        Equalize 0.5 5, AutoContrast 0.1 2
        Solarize 0.5 5, AutoContrast 0.9 5
        AutoContrast 0.6 1, AutoContrast 0.7 8
        Equalize 0.2 0, AutoContrast 0.1 2
        Equalize 0.6 9, Equalize 0.4 4""",
    "test": """
        TranslateX 1.0 4, Equalize 1.0 10""",
}


def _parse(text):
    subs = []
    for line in text.strip().splitlines():
        ops = []
        for part in line.split(","):
            name, prob, level = part.split()
            assert name in OP_CODE, name
            ops.append((name, float(prob), int(level)))
        assert len(ops) == 2, line
        subs.append(tuple(ops))
    return tuple(subs)


POLICIES = {name: _parse(text) for name, text in _TABLES.items()}
assert [len(POLICIES[n]) for n in ("v0", "imagenet", "good", "test")] == [25, 25, 95, 1]


def policy(name):
    """The sub-policies of `name` (v0, imagenet, good or test)."""
    if name not in POLICIES:
        raise ValueError("Invalid augmentation_name: {}".format(name))
    return POLICIES[name]


def level_to_arg(name, level):
    """The reference's argument of operation `name` at `level`, before any negation, in Python arithmetic:
    a float for Rotate (degrees), the blends, the shears and the translations; an int for Posterize (bits),
    Solarize (threshold), SolarizeAdd (addition) and Cutout (pad size); None for the rest."""
    if name == "Rotate":
        return (level / MAX_LEVEL) * 30.0
    if name == "Posterize":
        return int((level / MAX_LEVEL) * 4)
    if name == "Solarize":
        return int((level / MAX_LEVEL) * 256)
    if name == "SolarizeAdd":
        return int((level / MAX_LEVEL) * 110)
    if name in BLENDS:
        return (level / MAX_LEVEL) * 1.8 + 0.1
    if name in ("ShearX", "ShearY"):
        return (level / MAX_LEVEL) * 0.3
    if name in ("TranslateX", "TranslateY"):
        return (level / MAX_LEVEL) * float(TRANSLATE_CONST)
    if name == "Cutout":
        return int((level / MAX_LEVEL) * CUTOUT_CONST)
    return None


def rotate_transform(degrees, S):
    """float32 [t0..t5] of tf.contrib.image.rotate(S x S image, degrees * pi / 180) (TF 1.14
    angles_to_projective_transforms), degrees a float32."""
    rad = f32(f32(degrees) * f32(math.pi / 180.0))
    c, s = f32(math.cos(float(rad))), f32(math.sin(float(rad)))
    n = f32(S - 1)
    x_off = f32(f32(n - f32(f32(c * n) - f32(s * n))) / f32(2.0))
    y_off = f32(f32(n - f32(f32(s * n) + f32(c * n))) / f32(2.0))
    return [c, -s, x_off, s, c, y_off]


def op_record(name, level, S, negate=False, centre=(0, 0)):
    """One AUTOAUG_OP_DTYPE record: operation `name` at `level` applied to an S x S image, its argument
    negated when `negate` (signed operations), Cutout centred at `centre` = (row, column)."""
    r = np.zeros((), AUTOAUG_OP_DTYPE)
    r["op"] = OP_CODE[name]
    a = level_to_arg(name, level)
    if name in SIGNED:
        a = -f32(a) if negate else f32(a)
    if name == "Posterize":
        r["i"][0] = min(max(8 - a, 0), 7)
    elif name == "Solarize":
        r["i"][0] = a & 255                       # the uint8 constant of `image < threshold`
    elif name == "SolarizeAdd":
        r["i"][0] = a
    elif name in BLENDS:
        r["f"][0] = f32(a)
        if name == "Contrast":
            # the reference's "mean" is sum(histogram) / 256 = S * S / 256 in float32, clipped, truncated
            r["i"][0] = int(min(f32(f32(S * S) / f32(256.0)), f32(255.0)))
    elif name == "Rotate":
        r["f"] = rotate_transform(a, S)
    elif name == "ShearX":
        r["f"] = [1, a, 0, 0, 1, 0]
    elif name == "ShearY":
        r["f"] = [1, 0, 0, a, 1, 0]
    elif name == "TranslateX":                    # translate([-pixels, 0]): t2 = -dx = pixels
        r["f"] = [1, 0, a, 0, 1, 0]
    elif name == "TranslateY":
        r["f"] = [1, 0, 0, 0, 1, a]
    elif name == "Cutout":
        r["i"] = [int(centre[0]), int(centre[1]), a]
    return r


def subpolicy_record(name, k, S, applied, negated=(False, False), centres=((0, 0), (0, 0))):
    """The AUTOAUG_DESC_DTYPE record of sub-policy k of policy `name` on an S x S image with the outcome of
    its draws given: applied[j], negated[j] and centres[j] for slot j."""
    d = np.zeros((), AUTOAUG_DESC_DTYPE)
    d["subpolicy"] = k
    for j, (op, _, level) in enumerate(policy(name)[k]):
        if applied[j]:
            d["slot"][j] = op_record(op, level, S, negated[j], centres[j])
    return d


def uniform(rng):
    """One float32 uniform in [0, 1) on the 2^-24 grid."""
    return f32(int(rng.integers(0, 1 << 24)) * 2.0 ** -24)


def applies(u, prob):
    """floor(u + prob) in float32, cast to bool.  The sum can round up to 2.0 (prob 1.0, u near 1): that is
    true as well."""
    return bool(np.floor(f32(f32(u) + f32(prob))) != 0)


def resolve(name, S, rng):
    """The AUTOAUG_DESC_DTYPE record of one S x S image, its draws made from `rng` (a numpy Generator) in the
    order of the module docstring."""
    subs = policy(name)
    k = int(rng.integers(0, len(subs)))
    applied, negated, centres = [], [], []
    for op, prob, _ in subs[k]:
        applied.append(applies(uniform(rng), prob))
        negated.append(op in SIGNED and np.floor(f32(uniform(rng) + f32(0.5))) == 0)
        centres.append((int(rng.integers(0, S)), int(rng.integers(0, S))) if op == "Cutout" else (0, 0))
    return subpolicy_record(name, k, S, applied, negated, centres)


def check_autoaugment_descriptors(desc, S):
    """The host-side check of AutoAugment descriptors for S x S images before they go to the device
    (acnn_crop_resize_autoaugment_u8 does not read them on the host)."""
    desc = np.asarray(desc, AUTOAUG_DESC_DTYPE).reshape(-1)
    for b, d in enumerate(desc):
        for j in range(2):
            o = d["slot"][j]
            op, i, f = int(o["op"]), o["i"], o["f"]
            ok = 0 <= op < len(OPS)
            if ok:
                n = OPS[op]
                if n == "Posterize":
                    ok = 0 <= i[0] <= 7
                elif n in ("Solarize", "SolarizeAdd"):
                    ok = 0 <= i[0] <= 255
                elif n in BLENDS:
                    ok = bool(np.isfinite(f[0]) and f[0] >= 0) and (n != "Contrast" or 0 <= i[0] <= 255)
                elif n in SIGNED:
                    ok = bool(np.isfinite(f).all())
                elif n == "Cutout":
                    ok = 0 <= i[0] < S and 0 <= i[1] < S and i[2] >= 0
            if not ok:
                raise ValueError("autoaugment descriptor %d slot %d is invalid for S=%d: %s" % (b, j, S, o))
