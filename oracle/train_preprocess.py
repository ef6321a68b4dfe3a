"""Restatement of the reference's training input, for the tests (independent of assembled_cnn_b200).

  preprocess      preprocessing/imagenet_preprocessing.py:57-97,269-313 after the crop: the window mirrored
                  when flip, resize_bilinear (TF 1.14 legacy, float32, oracle/eval_preprocess.py) to S x S
                  with the scales h / S and w / S, - CHANNEL_MEANS, float32 throughout
  sample_box      TF 1.14's sample_distorted_bounding_box kernel (sample_distorted_bounding_box_op.cc:
                  GenerateRandomCrop + SatisfiesOverlapConstraints) with the whole image as the only object
                  box, float32 where the kernel computes in float; uniform [0, 1) draws from a callable
  interleave      interleave(cycle_length=20, block_length=1) over files of given record counts
  shuffle_buffer  dataset.shuffle(buffer): a buffer filled from the input, one uniformly chosen element out
                  and the next input element in its place; once the input ends, the last element fills the hole
  epoch / stream  file permutation -> interleave -> shuffle buffer, per epoch; repeat = concatenation
The draws follow the product's counter-based protocol (numpy default_rng keyed [seed, tag, ...]) so the
two can be compared example for example; the rules above are what the comparison checks.
"""
import numpy as np

from oracle.eval_preprocess import CHANNEL_MEANS, resize_bilinear

f32 = np.float32


def preprocess(window, flip, S, means=CHANNEL_MEANS):
    a = np.asarray(window)
    if flip:
        a = a[:, ::-1]
    return resize_bilinear(a, S, S) - np.asarray(means, dtype=np.float32)


def _round_even(x):
    return int(np.rint(f32(x)))


def _draw_int(draw, n):
    return min(int(draw() * n), n - 1)


def sample_box(h, w, draw, min_object_covered=0.1, aspect_range=(0.75, 1.33), area_range=(0.05, 1.0),
               max_attempts=100):
    """(y, x, crop_h, crop_w)."""
    amin, amax = f32(aspect_range[0]), f32(aspect_range[1])
    for _ in range(max_attempts):
        a = f32(f32(draw()) * f32(amax - amin)) + amin
        lo_area = f32(f32(area_range[0]) * f32(w)) * f32(h)
        hi_area = f32(f32(area_range[1]) * f32(w)) * f32(h)
        if not (area_range[1] > 0 and a > 0 and area_range[0] <= area_range[1]):
            continue
        ch = _round_even(np.sqrt(f32(lo_area / a)))
        ch_max = _round_even(np.sqrt(f32(hi_area / a)))
        if _round_even(f32(ch_max) * a) > w:
            ch_max = int((float(w) + 0.5 - float(f32(1e-7))) / float(a))
            if _round_even(f32(ch_max) * a) > w:
                ch_max = ch_max - 1
        if ch_max > h:
            ch_max = h
        if ch >= ch_max:
            ch = ch_max
        else:
            ch = ch + _draw_int(draw, ch_max - ch + 1)
        cw = _round_even(f32(ch) * a)
        if f32(cw * ch) < lo_area:
            ch += 1
            cw = _round_even(f32(ch) * a)
        if f32(cw * ch) > hi_area:
            ch -= 1
            cw = _round_even(f32(ch) * a)
        area = f32(cw * ch)
        if area < lo_area or area > hi_area or cw > w or ch > h or cw < 1 or ch < 1:
            continue
        y = _draw_int(draw, h - ch) if ch < h else 0
        x = _draw_int(draw, w - cw) if cw < w else 0
        if cw * ch >= 1 and h * w >= 1 and f32(f32(cw * ch) / f32(h * w)) >= f32(min_object_covered):
            return y, x, ch, cw
    return 0, 0, h, w


def example(h, w, seed, cycle, position, use_random_crop=True):
    """(y, x, crop_h, crop_w, flip) of the example at `position` of `cycle`."""
    rng = np.random.default_rng([seed, 2, cycle, position])
    flip = rng.random() < 0.5
    return sample_box(h, w, rng.random, 0.1 if use_random_crop else 1.0) + (bool(flip),)


def interleave(counts, files, cycle_length=20):
    """[(file, record)]."""
    iters = {}
    queue = list(files)
    slots = [None] * cycle_length
    out = []
    i = 0
    while queue or any(s is not None for s in slots):
        if slots[i] is None and queue:
            f = queue.pop(0)
            slots[i] = f
            iters[f] = iter(range(counts[f]))
        if slots[i] is not None:
            r = next(iters[slots[i]], None)
            if r is None:
                slots[i] = None
            else:
                out.append((slots[i], r))
        i = (i + 1) % cycle_length
    return out


def shuffle_buffer(items, size, u):
    """`u`: one uniform [0, 1) draw per emitted element."""
    src = iter(items)
    buf = []
    for x in src:
        buf.append(x)
        if len(buf) == size:
            break
    out = []
    k = 0
    while buf:
        j = min(int(u[k] * len(buf)), len(buf) - 1)
        k += 1
        out.append(buf[j])
        nxt = next(src, None)
        if nxt is not None:
            buf[j] = nxt
        else:
            buf[j] = buf[-1]
            buf.pop()
    return out


def epoch(counts, seed, cycle, e, buffer):
    rng = np.random.default_rng([seed, 1, cycle, e])
    files = [int(f) for f in rng.permutation(len(counts))]
    start = [sum(counts[:f]) for f in range(len(counts))]
    recs = [start[f] + r for f, r in interleave(counts, files)]
    return shuffle_buffer(recs, buffer, rng.random(len(recs)))


def stream(counts, seed, cycle, epochs, buffer):
    out = []
    for e in range(epochs):
        out += epoch(counts, seed, cycle, e, buffer)
    return out
