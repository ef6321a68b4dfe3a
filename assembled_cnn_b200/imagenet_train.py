"""The data side of training from TFRecord shards (input_fn_cls(is_training=True), functions/input_fns.py:
33-145, and utils/data_util.py:161-235,389-473): the training shards, the record stream, the crop window
sampler and the decoding of one crop window.  The device side is model_fns.Trainer.train_step_cropped and
model_fns.train_and_evaluate.

  train_files         utils/data_util.py:161-170       sorted(glob(data_dir/train_regex))
  read_train_records  utils/data_util.py:173-235       label, JPEG byte range, KD logits ('image/logit')
  train_size          utils/data_util.py:267-345       S of the imagenet-family dispatch, is_training=True
  sample_distorted_bounding_box                        TF 1.14's sample_distorted_bounding_box_op.cc kernel
                      (GenerateRandomCrop, SatisfiesOverlapConstraints), restated from its description
  crop_window         preprocessing/imagenet_preprocessing.py:57-97  the window of _decode_crop_and_flip
                      (no bounding boxes: the whole image is the object) and random_flip_left_right
  CycleStream         functions/input_fns.py:52-74 + utils/data_util.py:389-460: file shuffle, 20-way
                      round-robin interleave, shuffle buffer, repeat, batch, on record indices only

Randomness is counter-based, not TF's Philox stream: the order of cycle c is a function of (seed, c), the
window and flip of the example at position p of cycle c a function of (seed, c, p), the mixup lambdas of
global step t a function of (seed, t, rank).  So the batches do not depend on the number of decode threads
or of ranks, and a run resumed from a cycle's checkpoint replays the uninterrupted run's data.

Deviations from the reference: the partial last batch of a cycle is dropped (at most one batch per cycle;
the training step has a static shape).  The reference's `dataset.take(total_batches * batch_size)`
(utils/data_util.py:424) discards its result and so has no effect; nothing here imitates it.  The whole
image is decoded with PIL and the window sliced out of it; TF's fused decode_and_crop_jpeg has not been
compared with this.
"""
from __future__ import annotations

import glob
import io
import os

import numpy as np

from .imagenet_c import CHANNEL_MEANS, decode_rgb  # noqa: F401  (re-exported for the training input)
from .imagenet_eval import _OUT_OF_SCOPE, _TYPE_NNN, _TYPE_NNN_A, read_encoded, read_records

# include/acnn.h acnn_crop_desc
CROP_DESC_DTYPE = np.dtype([("src", "<u8"), ("h", "<i4"), ("w", "<i4"), ("flip", "<i4"),
                            ("reserved", "<i4", (3,))])
assert CROP_DESC_DTYPE.itemsize == 32

CYCLE_LENGTH = 20               # functions/input_fns.py:71-74 interleave(cycle_length=20), block_length 1
# functions/data_config.py: shuffle_buffer per dataset (Default: 1000)
SHUFFLE_BUFFER = {"imagenet": 10000, "food101": 1000, "cub_200_2011": 100, "SOP": 50000}
DEFAULT_SHUFFLE_BUFFER = 1000

# stream tags of the counter-based generators
_ORDER, _EXAMPLE, _MIXUP = 1, 2, 3


# ---------------------------------------------------------------------------------------- records
def train_files(data_dir, train_regex="train-*"):
    """get_filenames(is_training=True): the shards matching data_dir/train_regex, sorted (the order only
    seeds the per-epoch file permutation)."""
    files = sorted(glob.glob(os.path.join(data_dir, train_regex)))
    if not files:
        raise FileNotFoundError("training: no file matches %s" % os.path.join(data_dir, train_regex))
    return files


def read_train_records(files, num_classes, kd=False):
    """[(path, offset, length, label, logits or None)] of every record of `files`, file by file, and the
    record count of each file.  Every record is checked before any GPU work: a label outside
    [0, num_classes) or, with kd, an 'image/logit' list of other than num_classes values raises ValueError
    naming the file and the image's byte offset (parse_record_sup reshapes the logits to [num_classes])."""
    records, counts = [], []
    for path in files:
        recs = read_records(path, logits=kd)
        for r in recs:
            label, offset = r[0], r[1]
            if not 0 <= label < num_classes:
                raise ValueError("training: %s: label %d (image at byte offset %d) outside [0, %d)"
                                 % (path, label, offset, num_classes))
            if kd and len(r[3]) != num_classes:
                raise ValueError("training: %s: image/logit holds %d values (image at byte offset %d); "
                                 "kd_temp > 0 needs num_classes = %d" % (path, len(r[3]), offset, num_classes))
            records.append((path, offset, r[2], label, r[3] if kd else None))
        counts.append(len(recs))
    if not records:
        raise ValueError("training: the shards %s hold no record" % files)
    return records, counts


def train_size(preprocessing_type, image_size=224):
    """S of preprocess_image(is_training=True) for an imagenet-family preprocessing_type (utils/data_util.py:
    267-345, the same regular expressions in the same order).  S must be a multiple of 32 (the model's
    constraint): ValueError otherwise."""
    if preprocessing_type == "imagenet":
        s = image_size
    elif preprocessing_type in ("imagenet_224_256", "imagenet_224_256a"):
        s = 224
    elif _TYPE_NNN_A.match(preprocessing_type):
        s = int(preprocessing_type.split("_")[1][0:3])
    elif _TYPE_NNN.match(preprocessing_type):
        s = int(preprocessing_type.split("_")[1])
    elif preprocessing_type in _OUT_OF_SCOPE:
        raise NotImplementedError("preprocessing_type %r (reid / inception preprocessing) is not supported by "
                                  "training" % preprocessing_type)
    else:
        raise NotImplementedError("unknown preprocessing_type %r" % preprocessing_type)
    s = int(s)
    if s < 32 or s % 32:
        raise ValueError("preprocessing_type %r trains at %d px; the model needs a multiple of 32"
                         % (preprocessing_type, s))
    return s


# ---------------------------------------------------------------------------------------- sampler
_F = np.float32


def _lrintf(x):
    return int(np.rint(_F(x)))                     # round half to even, as lrintf in the default mode


def _uniform(draw, n):
    """random::SimplePhilox::Uniform(n), an integer in [0, n), from one uniform [0, 1) draw."""
    return min(int(draw() * n), n - 1)


def _generate_random_crop(W, H, min_rel, max_rel, aspect, draw):
    """GenerateRandomCrop (sample_distorted_bounding_box_op.cc): (x, y, w, h) or None, in float32."""
    if max_rel <= 0 or aspect <= 0 or W <= 0 or H <= 0 or min_rel > max_rel:
        return None
    min_area = _F(_F(min_rel) * _F(W)) * _F(H)
    max_area = _F(_F(max_rel) * _F(W)) * _F(H)
    height = _lrintf(np.sqrt(_F(min_area / aspect)))
    max_height = _lrintf(np.sqrt(_F(max_area / aspect)))
    if _lrintf(_F(max_height) * aspect) > W:
        # the smallest max_height with round(max_height * aspect) <= W; the expression is in double
        max_height = int((W + 0.5 - float(_F(1e-7))) / float(aspect))
        if _lrintf(_F(max_height) * aspect) > W:
            max_height -= 1
    max_height = min(max_height, H)
    height = min(height, max_height)
    if height < max_height:
        height += _uniform(draw, max_height - height + 1)
    width = _lrintf(_F(height) * aspect)
    area = _F(width * height)
    if area < min_area:
        height += 1
        width = _lrintf(_F(height) * aspect)
        area = _F(width * height)
    if area > max_area:
        height -= 1
        width = _lrintf(_F(height) * aspect)
        area = _F(width * height)
    if area < min_area or area > max_area or width > W or height > H or width <= 0 or height <= 0:
        return None
    y = _uniform(draw, H - height) if height < H else 0
    x = _uniform(draw, W - width) if width < W else 0
    return x, y, width, height


def sample_distorted_bounding_box(h, w, draw, min_object_covered=0.1, aspect_ratio_range=(0.75, 1.33),
                                  area_range=(0.05, 1.0), max_attempts=100):
    """(offset_y, offset_x, crop_h, crop_w) of tf.image.sample_distorted_bounding_box on an h x w image with
    no bounding boxes and use_image_if_no_bounding_boxes=True (the whole image is the object box), as
    TF 1.14's kernel computes it: up to max_attempts times, aspect = RandFloat() * (max - min) + min, a
    GenerateRandomCrop at that aspect, accepted when it covers >= min_object_covered of the object and its
    own area is >= 1; no accepted attempt gives the whole image.  `draw()` returns the uniform [0, 1) draws
    (the kernel's Philox stream cannot be reproduced; the rules are)."""
    lo, hi = _F(aspect_ratio_range[0]), _F(aspect_ratio_range[1])
    object_area = _F(h * w)
    for _ in range(max_attempts):
        aspect = _F(_F(_F(draw()) * _F(hi - lo)) + lo)
        r = _generate_random_crop(w, h, area_range[0], area_range[1], aspect, draw)
        if r is None:
            continue
        x, y, cw, ch = r
        if cw * ch < 1 or object_area < 1:
            continue
        # the crop lies inside the image: its intersection with the object box is the crop
        if _F(_F(cw * ch) / object_area) >= _F(min_object_covered):
            return y, x, ch, cw
    return 0, 0, h, w


def example_rng(seed, cycle, position):
    """The generator of the example at stream position `position` of cycle `cycle`."""
    return np.random.default_rng([seed, _EXAMPLE, cycle, position])


def crop_window(h, w, rng, use_random_crop=True):
    """(offset_y, offset_x, crop_h, crop_w, flip) of _decode_crop_and_flip for an h x w image:
    min_object_covered 0.1 (use_random_crop, the training_random_crop flag) or 1.0, and the
    random_flip_left_right draw (< 0.5 mirrors)."""
    flip = bool(rng.random() < 0.5)
    y, x, ch, cw = sample_distorted_bounding_box(h, w, rng.random, 0.1 if use_random_crop else 1.0)
    return y, x, ch, cw, flip


def jpeg_shape(buf):
    """(height, width) from the image header (tf.image.extract_jpeg_shape): the JPEG header parser of
    acnn_jpeg_parse, or PIL's lazy open for the images it does not accept; no decoding."""
    from .jpeg import jpeg_shape as shape
    return shape(buf)


def decode_window(path, offset, length, seed, cycle, position, use_random_crop=True):
    """(uint8 [crop_h, crop_w, 3] C-contiguous window, flip) of the record at path[offset:offset + length],
    the example at `position` of cycle `cycle`: its size from the header, the window and flip from
    crop_window, the whole image decoded (decode_rgb) and the window sliced out."""
    buf = read_encoded(path, offset, length)
    h, w = jpeg_shape(buf)
    y, x, ch, cw, flip = crop_window(h, w, example_rng(seed, cycle, position), use_random_crop)
    a = decode_rgb(io.BytesIO(buf))
    if a.shape[:2] != (h, w):
        raise ValueError("%s: the image at byte offset %d decodes to %s, its header says %dx%d"
                         % (path, offset, a.shape[:2], h, w))
    return np.ascontiguousarray(a[y:y + ch, x:x + cw]), flip


def encoded_window(path, offset, length, seed, cycle, position, use_random_crop=True):
    """(encoded bytes, (offset_y, offset_x, crop_h, crop_w), flip) of the record at path[offset:offset + length],
    the example at `position` of cycle `cycle`: the window and flip decode_window would cut, left for the
    device decoder (model_fns._TrainFeed.stage_encoded)."""
    buf = read_encoded(path, offset, length)
    h, w = jpeg_shape(buf)
    y, x, ch, cw, flip = crop_window(h, w, example_rng(seed, cycle, position), use_random_crop)
    return buf, (y, x, ch, cw), flip


def check_crop_descriptors(desc):
    """The host-side check of crop descriptors before they go to the device (acnn_crop_resize_u8 does not
    read them on the host): every row needs a source address and sizes >= 1."""
    bad = (desc["src"] == 0) | (desc["h"] < 1) | (desc["w"] < 1)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError("crop descriptor %d is invalid: %s" % (i, desc[i]))


# ---------------------------------------------------------------------------------------- stream
def mixup_lambdas(seed, global_step, rank, n):
    """float32 [n] Beta(0.2, 0.2) lambdas of one replica at one global step (utils/data_util.py:97-105)."""
    return np.random.default_rng([seed, _MIXUP, global_step, rank]).beta(0.2, 0.2, n).astype(np.float32)


def _interleave(counts, order):
    """(file, record) pairs of interleave(TFRecordDataset, cycle_length=20, block_length=1) over the files in
    `order`: round-robin over 20 slots; a slot whose file is exhausted takes the next file when the cycle
    comes back to it."""
    out = []
    pending = list(order)[::-1]
    slots = [None] * CYCLE_LENGTH           # [file, next record] or None
    k = 0
    while pending or any(s is not None for s in slots):
        s = slots[k]
        if s is None:
            if pending:
                f = pending.pop()
                slots[k] = s = [f, 0]
            else:
                k = (k + 1) % CYCLE_LENGTH
                continue
        if s[1] < counts[s[0]]:
            out.append((s[0], s[1]))
            s[1] += 1
        else:
            slots[k] = None
        k = (k + 1) % CYCLE_LENGTH
    return out


def epoch_order(counts, seed, cycle, epoch, shuffle_buffer):
    """Record indices (into the file-by-file record list) of one epoch of cycle `cycle`: the files in a
    random permutation (shuffle(buffer = number of files)), interleaved, then shuffle(shuffle_buffer):
    fill the buffer, then repeatedly emit a uniformly chosen element and refill from the input."""
    rng = np.random.default_rng([seed, _ORDER, cycle, epoch])
    perm = rng.permutation(len(counts))
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    src = [int(first[f]) + r for f, r in _interleave(counts, perm)]
    n = len(src)
    u = rng.random(n)
    size = np.minimum(shuffle_buffer, n - np.arange(n))          # buffer size at each emission
    pick = np.minimum((u * size).astype(np.int64), size - 1)
    buf = src[:min(shuffle_buffer, n)]
    nxt = len(buf)
    out = np.empty(n, dtype=np.int64)
    for i in range(n):
        j = int(pick[i])
        out[i] = buf[j]
        if nxt < n:
            buf[j] = src[nxt]
            nxt += 1
        else:
            buf[j] = buf[-1]
            buf.pop()
    return out


class CycleStream:
    """The examples of one training cycle (classifier.train(input_fn_train(epochs))): `epochs` repeats of
    epoch_order, batched into global steps of world x input_batch examples; at local step t replica r takes
    positions [(t * world + r) * input_batch, +input_batch) (MirroredStrategy hands consecutive batches to
    consecutive replicas).  The partial last batch is dropped.  Epoch orders are computed on demand."""

    def __init__(self, counts, seed, cycle, epochs, shuffle_buffer, input_batch, world=1, rank=0):
        self.counts, self.seed, self.cycle = list(counts), int(seed), int(cycle)
        self.n = int(sum(counts))
        self.shuffle_buffer, self.input_batch, self.world, self.rank = shuffle_buffer, input_batch, world, rank
        self.steps = int(epochs) * self.n // (world * input_batch)
        self._cache = {}

    def _epoch(self, e):
        if e not in self._cache:
            if len(self._cache) >= 2:
                self._cache.pop(min(self._cache))
            self._cache[e] = epoch_order(self.counts, self.seed, self.cycle, e, self.shuffle_buffer)
        return self._cache[e]

    def positions(self, t):
        a = (t * self.world + self.rank) * self.input_batch
        return range(a, a + self.input_batch)

    def records(self, t):
        """[(position, record index)] of this replica's batch at local step t."""
        if not 0 <= t < self.steps:
            raise IndexError("step %d outside the cycle's %d steps" % (t, self.steps))
        return [(p, int(self._epoch(p // self.n)[p % self.n])) for p in self.positions(t)]


def replica_streams(counts, seed, cycle, epochs, shuffle_buffer, input_batch, world=1, rank=0, replicas=1):
    """The CycleStreams of the `replicas` replicas q = rank * replicas + r of process `rank`: each gets what rank
    q of a world * replicas run gets, so the data does not depend on how the replicas are split over processes."""
    return [CycleStream(counts, seed, cycle, epochs, shuffle_buffer, input_batch, world * replicas, rank * replicas + r)
            for r in range(replicas)]


def replica_mixup_lambdas(seed, global_step, rank, replicas, n):
    """float32 [replicas, n]: row r holds mixup_lambdas of replica q = rank * replicas + r."""
    return np.stack([mixup_lambdas(seed, global_step, rank * replicas + r, n) for r in range(replicas)])


def epoch_schedule(train_epochs, epochs_between_evals, ratio_fine_eval, cur_epoch=0):
    """The epochs of each train-and-evaluate cycle (nets/run_loop_classification.py:453-467 and
    utils/config_utils.py:71-96 get_epoch_schedule): cycles of epochs_between_evals epochs, the last one
    shortened; cycles ending at or before cur_epoch are skipped; from train_epochs * ratio_fine_eval on a
    cycle is split into 1-epoch cycles.  train_epochs = 0 gives [0] (one evaluation)."""
    if not train_epochs:
        return [0]
    n = -(-train_epochs // epochs_between_evals)
    sched = [epochs_between_evals] * n
    sched[-1] = train_epochs - sum(sched[:-1])
    fine = int(train_epochs * ratio_fine_eval)
    out, acc = [], 0
    for e in sched:
        acc += e
        if acc <= cur_epoch:
            continue
        out += [1] * e if acc > fine else [e]
    return out
