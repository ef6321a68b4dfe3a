"""TensorBoard event files and the training loop's summaries (the outputs Estimator gives the reference's
run loop: `model_dir/events.out.tfevents.*`, `model_dir/eval/` and LoggingTensorHook's log lines).

An event file is a TFRecord file of `Event` protos (TensorFlow's public event.proto / summary.proto):
  Event    wall_time = 1 (double), step = 2 (int64), file_version = 3 (string), summary = 5 (Summary)
  Summary  value = 1 (repeated Value)
  Value    tag = 1 (string), simple_value = 2 (float)
The protos are encoded here by hand and framed with imagenet_eval.write_record (masked CRC-32C), so no
TensorFlow, TensorBoard or protobuf package is needed."""
from __future__ import annotations

import logging
import os
import socket
import struct
import time
from collections import deque

import numpy as np
import torch

from .imagenet_eval import write_record
from .metrics import TRAIN_METRICS_DTYPE, train_metric_values
from .native import decode_loss_scale_state

log = logging.getLogger("assembled_cnn_b200")


def _varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _bytes_field(field, payload):
    return _varint(field << 3 | 2) + _varint(len(payload)) + payload


def encode_event(wall_time, step=None, file_version=None, scalars=()):
    """The bytes of one Event: wall_time, step (when given), file_version (when given) and a Summary of the
    (tag, value) pairs `scalars`, each a simple_value (float32)."""
    out = bytearray(b"\x09" + struct.pack("<d", float(wall_time)))
    if step is not None:
        out += b"\x10" + _varint(int(step) & 0xFFFFFFFFFFFFFFFF)
    if file_version is not None:
        out += _bytes_field(3, file_version.encode())
    if scalars:
        values = b"".join(_bytes_field(1, _bytes_field(1, str(tag).encode()) + b"\x15" + struct.pack("<f", float(v)))
                          for tag, v in scalars)
        out += _bytes_field(5, values)
    return bytes(out)


class SummaryWriter:
    """Writes `logdir/events.out.tfevents.<10-digit unix time>.<hostname>`: first Event{wall_time,
    file_version "brain.Event:2"}, then one Event per scalar.  The directory is created.  When a file of that
    name exists (a second writer in the same second), the next free second names the new file, so a writer
    never appends to an older run's file."""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        host = socket.gethostname()
        t = int(time.time())
        while os.path.exists(os.path.join(logdir, "events.out.tfevents.%010d.%s" % (t, host))):
            t += 1
        self.path = os.path.join(logdir, "events.out.tfevents.%010d.%s" % (t, host))
        self._f = open(self.path, "xb")
        write_record(self._f, [encode_event(time.time(), file_version="brain.Event:2")])
        self._f.flush()

    def add_scalars(self, step, scalars, wall_time=None):
        """One Event per (tag, value) of `scalars` at `step`, then a flush."""
        wall_time = time.time() if wall_time is None else wall_time
        for tag, v in scalars:
            write_record(self._f, [encode_event(wall_time, step, scalars=[(tag, v)])])
        self._f.flush()

    def close(self):
        if self._f is not None:
            self._f.close()
            self._f = None


def check_save_summary_steps(n):
    """save_summary_steps: None (no summaries) or an integer >= 1 (ValueError otherwise); returns it."""
    if n is None:
        return None
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 1:
        raise ValueError("save_summary_steps must be None or an integer >= 1 (got %r)" % (n,))
    return int(n)


def check_summary_dir(summary_dir):
    """summary_dir: None, or a path that is a directory or can be made one; it is made here, so a bad one
    raises ValueError before any work.  Returns it."""
    if summary_dir is None:
        return None
    if not isinstance(summary_dir, (str, os.PathLike)) or not os.fspath(summary_dir):
        raise ValueError("summary_dir must be a path (got %r)" % (summary_dir,))
    try:
        os.makedirs(summary_dir, exist_ok=True)
    except OSError as e:
        raise ValueError("summary_dir %r is not a usable directory: %s" % (summary_dir, e)) from None
    return summary_dir


def is_summary_step(step, cycle_first_step, every):
    """Estimator's summary cadence inside one `classifier.train` call: the cycle's first step, then every
    `every`-th step after it (not the multiples of `every`: a cycle may start anywhere)."""
    return (step - cycle_first_step) % every == 0


def numeric_scalars(result):
    """The (tag, value) pairs of an evaluation result: every int or float entry except global_step."""
    return [(k, float(v)) for k, v in result.items()
            if k != "global_step" and not isinstance(v, bool) and isinstance(v, (int, float, np.integer, np.floating))]


class TrainSummaries:
    """The training summaries and log lines of rank 0 (nets/run_loop_classification.py:146-227 through
    Estimator's SummarySaverHook and LoggingTensorHook), without a host synchronisation per step.

    `record(loss, step, lr, keep_prob)` right after a summary step copies the step's loss slot and the Trainer's metric
    accumulator, on the current stream, into a slot of a pinned host ring and records an event; the host
    values (step, learning rate, keep prob, wall clock) are kept beside it.  `poll()` writes every slot whose
    event has completed (event.query(), no wait); `drain()` waits for the rest, and is called where the loop
    synchronises anyway (checkpoint, evaluation, end).  The ring is deeper than the steps the host can run
    ahead of the device (Trainer's hyper-parameter ring), so a full ring's oldest slot has completed."""

    RING = 8
    # dynamic loss scaling: per slot the state after the step (the scale it used, the steps skipped so far)
    _ls_host = None

    def __init__(self, model_dir, trainer):
        self.writer = SummaryWriter(model_dir)
        self.tr = trainer
        self.mixup = trainer.mixup_type > 0
        self.kd = trainer.kd_temp > 0
        self._host = [(torch.zeros(3, dtype=torch.float32).pin_memory(),
                       torch.zeros(TRAIN_METRICS_DTYPE.itemsize, dtype=torch.uint8).pin_memory())
                      for _ in range(self.RING)]
        if trainer.dynamic:
            self._ls_host = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(self.RING)]
        self._pending = deque()      # (slot, event, step, lr, keep_prob, wall time, steps/s or None)
        self._next = 0
        self._last = None            # (step, host clock) of the previous summary

    def record(self, loss, step, lr, keep_prob):
        if len(self._pending) == self.RING:
            self._write(self._pending.popleft(), wait=True)
        slot = self._next
        self._next = (slot + 1) % self.RING
        hloss, hacc = self._host[slot]
        hloss[:loss.numel()].copy_(loss, non_blocking=True)
        hacc.copy_(self.tr.train_metrics, non_blocking=True)
        if self._ls_host is not None:
            self._ls_host[slot].copy_(self.tr.rt.loss_scale_state_buf, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.tr.rt.dev))
        now = time.time()
        rate = None
        if self._last is not None and now > self._last[1]:
            rate = (step - self._last[0]) / (now - self._last[1])
        self._last = (step, now)
        self._pending.append((slot, ev, step, lr, keep_prob, now, rate))

    def poll(self):
        while self._pending and self._pending[0][1].query():
            self._write(self._pending.popleft())

    def drain(self):
        while self._pending:
            self._write(self._pending.popleft(), wait=True)

    def begin_cycle(self):
        """Each `classifier.train` call starts new metric variables and new hooks: the streaming metrics
        restart and the cycle's first summary has no global_step/sec."""
        self.tr.reset_train_metrics()
        self._last = None

    def _write(self, entry, wait=False):
        slot, ev, step, lr, keep_prob, wall, rate = entry
        if wait and not ev.query():
            ev.synchronize()
        hloss, hacc = self._host[slot]
        ce, l2, kd = (float(v) for v in hloss.tolist())
        rec = np.frombuffer(hacc.numpy().tobytes(), TRAIN_METRICS_DTYPE)[0]
        m = train_metric_values(rec, self.mixup)
        scalars = [("cross_entropy", ce), ("l2_loss", l2)]
        if self.kd:
            scalars.append(("cross_entropy_kd", kd))
        scalars += [("loss", ce + l2 + (kd if self.kd else 0.0)), ("sup/pred_prob", m["sup/pred_prob"]),
                    ("learning_rate", lr), ("dropblock_kp", keep_prob)]
        if not self.mixup:
            scalars += [(k, m[k]) for k in ("train_accuracy", "train_accuracy_top_5", "train_ece")]
        if rate is not None:
            scalars.append(("global_step/sec", rate))
        ls = ""
        if self._ls_host is not None:
            st = decode_loss_scale_state(self._ls_host[slot].numpy())
            scalars += [("loss_scale", st["last_scale"]), ("loss_scale/skipped_steps", st["skipped_steps"])]
            ls = ", loss_scale = %g, skipped_steps = %d" % (st["last_scale"], st["skipped_steps"])
        self.writer.add_scalars(step, scalars, wall)
        log.info("step %d: learning_rate = %.6g, cross_entropy = %.6g, train_accuracy = %.6g, train_ece = %.6g, "
                 "global_step/sec = %s%s", step, lr, ce, m.get("train_accuracy", 0), m.get("train_ece", 0),
                 "-" if rate is None else "%.4g" % rate, ls)

    def close(self):
        self.drain()
        self.writer.close()
