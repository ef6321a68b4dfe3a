"""The JPEG test corpus, generated with PIL at test time (shared by test_jpeg_cpu.py and test_jpeg_gpu.py):
sizes from 1x1 to 2000x1500 (1xN, Nx1, not multiples of 8 or 16), 4:4:4 / 4:2:2 / 4:2:0 / grayscale,
quality 50-100, optimized Huffman tables, restart intervals in blocks and in rows, noise and smooth content,
and the JPEGs of tests/golden/eval_golden.tfrecord."""
import io
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def image(h, w, kind, rng, gray=False):
    if kind == "noise":
        a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        y, x = np.mgrid[0:h, 0:w].astype(np.float32)
        a = np.stack([127 + 120 * np.sin(x / 17.0 + c) * np.cos(y / 23.0 - c) for c in range(3)], -1)
        a = np.clip(a + rng.normal(0, 3, a.shape), 0, 255).astype(np.uint8)
    from PIL import Image
    im = Image.fromarray(a)
    return im.convert("L") if gray else im


def encode(im, **kw):
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def golden_jpegs():
    from assembled_cnn_b200 import imagenet_eval as E
    path = os.path.join(ROOT, "tests", "golden", "eval_golden.tfrecord")
    return [E.read_encoded(path, r[1], r[2]) for r in E.read_records(path)]


def corpus(big=True):
    """[(name, jpeg bytes)]."""
    rng = np.random.default_rng(1234)
    sizes = [(1, 1), (1, 37), (29, 1), (2, 2), (3, 5), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33), (33, 31),
             (61, 83), (100, 75), (375, 500), (500, 333)]
    if big:
        sizes += [(1500, 2000)]
    out = []
    for k, (h, w) in enumerate(sizes):
        for mode in ("444", "422", "420", "gray"):
            kind = "noise" if (k + len(mode)) % 2 else "smooth"
            if h * w > 10 ** 6 and mode in ("444", "gray"):
                continue
            q = int(rng.integers(50, 101))
            kw = dict(quality=q)
            if mode != "gray":
                kw["subsampling"] = {"444": 0, "422": 1, "420": 2}[mode]
            if k % 3 == 1:
                kw["optimize"] = True
            if k % 4 == 2:
                kw["restart_marker_blocks"] = int(rng.integers(1, 6))
            elif k % 4 == 3:
                kw["restart_marker_rows"] = int(rng.integers(1, 3))
            out.append(("%dx%d_%s_%s_%s" % (h, w, mode, kind, "_".join("%s%s" % i for i in sorted(kw.items()))),
                        encode(image(h, w, kind, rng, mode == "gray"), **kw)))
    im = image(64, 48, "smooth", rng)
    out.append(("q100", encode(im, quality=100)))
    out.append(("q100_opt_rst", encode(im, quality=100, optimize=True, restart_marker_blocks=1)))
    out += [("golden%d" % i, b) for i, b in enumerate(golden_jpegs())]
    return out


def pil_rgb(b):
    from PIL import Image
    with Image.open(io.BytesIO(b)) as im:
        return np.array(im.convert("RGB"), dtype=np.uint8)


def unsupported_samples():
    """[(name, bytes)] the device decoder must refuse: progressive, CMYK, PNG."""
    rng = np.random.default_rng(5)
    im = image(40, 56, "smooth", rng)
    b = io.BytesIO()
    im.save(b, "PNG")
    return [("progressive", encode(im, progressive=True)), ("cmyk", encode(im.convert("CMYK"))),
            ("png", b.getvalue())]
