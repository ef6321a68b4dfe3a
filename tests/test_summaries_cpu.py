"""CPU checks of the training summaries: the hand-encoded event files against the protobuf runtime (through a
schema built here with TensorFlow's public event.proto / summary.proto field numbers) and the TFRecord frame
parser, the argument checks of save_summary_steps and summary_dir before any GPU work, the summary-step rule,
the ECE of binned counts against classification_result's, and the host-side checks of
acnn_train_metrics_accumulate."""
import glob
import logging
import os
import socket
import struct

import numpy as np
import pytest


def _event_class():
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="test_event.proto", package="tfev", syntax="proto3")
    opt, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED
    v = fd.message_type.add(name="Value")
    v.field.add(name="tag", number=1, type=F.TYPE_STRING, label=opt)
    v.field.add(name="simple_value", number=2, type=F.TYPE_FLOAT, label=opt)
    s = fd.message_type.add(name="Summary")
    s.field.add(name="value", number=1, type=F.TYPE_MESSAGE, label=rep, type_name=".tfev.Value")
    e = fd.message_type.add(name="Event")
    e.field.add(name="wall_time", number=1, type=F.TYPE_DOUBLE, label=opt)
    e.field.add(name="step", number=2, type=F.TYPE_INT64, label=opt)
    e.field.add(name="file_version", number=3, type=F.TYPE_STRING, label=opt)
    e.field.add(name="summary", number=5, type=F.TYPE_MESSAGE, label=opt, type_name=".tfev.Summary")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("tfev.Event"))


def read_events(path):
    """Every Event of an event file, after checking each frame's data CRC."""
    from assembled_cnn_b200.imagenet_eval import masked_crc32c, record_frames
    data = open(path, "rb").read()
    Event = _event_class()
    out = []
    for _, start, length in record_frames(data, path):
        body = data[start:start + length]
        assert struct.unpack("<I", data[start + length:start + length + 4])[0] == masked_crc32c(body)
        ev = Event()
        ev.ParseFromString(body)
        out.append(ev)
    return out


def test_event_file_parses_with_protobuf(tmp_path):
    from assembled_cnn_b200.summary import SummaryWriter
    w = SummaryWriter(str(tmp_path / "logs"))
    name = os.path.basename(w.path)
    prefix, t, host = name[:len("events.out.tfevents.")], name.split(".")[3], name.split(".", 4)[4]
    assert prefix == "events.out.tfevents." and len(t) == 10 and t.isdigit() and host == socket.gethostname()
    scalars = [("cross_entropy", 2.5), ("sup/pred_prob", 0.125), ("learning_rate", 1e-3), ("x", -7.0)]
    w.add_scalars(0, scalars[:2], wall_time=1234.5)
    w.add_scalars(2 ** 40 + 3, scalars[2:], wall_time=1700000000.25)
    w.close()
    ev = read_events(w.path)
    assert ev[0].file_version == "brain.Event:2" and ev[0].wall_time > 0 and not ev[0].HasField("summary")
    got = [(e.step, e.wall_time, v.tag, v.simple_value) for e in ev[1:] for v in e.summary.value]
    want = [(0, 1234.5, t, np.float32(x)) for t, x in scalars[:2]] + \
        [(2 ** 40 + 3, 1700000000.25, t, np.float32(x)) for t, x in scalars[2:]]
    assert got == want
    assert all(len(e.summary.value) == 1 for e in ev[1:])
    # a second writer in the same directory never appends to the first one's file
    w2 = SummaryWriter(str(tmp_path / "logs"))
    w2.close()
    assert w2.path != w.path and len(glob.glob(str(tmp_path / "logs" / "events.out.tfevents.*"))) == 2


def test_numeric_scalars():
    from assembled_cnn_b200.summary import numeric_scalars
    res = {"accuracy": 0.5, "accuracy_top_5": np.float64(0.75), "ece": 0.1, "loss": 3.0, "global_step": 12,
           "flag": True, "name": "x"}
    assert numeric_scalars(res) == [("accuracy", 0.5), ("accuracy_top_5", 0.75), ("ece", 0.1), ("loss", 3.0)]
    assert numeric_scalars({"recall_at_1": 0.25, "recall_at_5": 1, "global_step": 3}) == \
        [("recall_at_1", 0.25), ("recall_at_5", 1.0)]


@pytest.mark.parametrize("bad", [0, -1, 1.5, "100", True])
def test_save_summary_steps_refused_before_gpu_work(tmp_path, bad):
    from assembled_cnn_b200.model_fns import train_and_evaluate
    with pytest.raises(ValueError, match="save_summary_steps"):
        train_and_evaluate(str(tmp_path / "no-data"), str(tmp_path / "run"), save_summary_steps=bad)
    assert not (tmp_path / "run").exists()


def test_bad_summary_dir_refused_before_gpu_work(tmp_path):
    from assembled_cnn_b200.model_fns import corruption_error
    f = tmp_path / "file"
    f.write_bytes(b"")
    for bad in (str(f), str(f / "sub"), "", 3):
        with pytest.raises(ValueError, match="summary_dir"):
            corruption_error(None, str(tmp_path / "no-data"), str(tmp_path / "no-labels"), summary_dir=bad)


def test_summary_step_rule():
    from assembled_cnn_b200.summary import is_summary_step

    def steps(first, n, every):
        return [s for s in range(first, first + n) if is_summary_step(s, first, every)]
    assert steps(0, 250, 100) == [0, 100, 200]
    # a cycle that starts off a multiple of N counts from its own first step
    assert steps(6, 6, 4) == [6, 10]
    assert steps(37, 9, 100) == [37]
    assert steps(3, 5, 1) == [3, 4, 5, 6, 7]
    # a resumed run: the cycle restarts at the restored step
    assert steps(12510, 12510, 5000) == [12510, 17510, 22510]


def _old_ece(pred, conf, labels):
    """classification_result's ECE as it was written before the bins arithmetic was factored out."""
    pred, labels, conf = np.asarray(pred, np.int64), np.asarray(labels, np.int64), np.asarray(conf, np.float32)
    correct = pred == labels
    eps = 1e-7
    th = np.asarray([0.0 - eps] + [(i + 1) * 1.0 / 10 for i in range(9)] + [1.0 + eps], np.float32)
    inb = (conf[None, :] > th[:-1, None]) & (conf[None, :] <= th[1:, None])
    cnt = inb.sum(1).astype(np.float64)
    acc = (inb & correct[None, :]).sum(1) / (eps + cnt)
    avg = (np.where(inb, conf[None, :].astype(np.float64), 0.0)).sum(1) / (eps + cnt)
    with np.errstate(invalid="ignore"):
        return float((cnt / cnt.sum() * np.abs(acc - avg)).sum()), inb, correct


def test_ece_from_bins_equals_classification_result():
    from assembled_cnn_b200.metrics import classification_result, ece_from_bins
    rng = np.random.default_rng(3)
    th = np.asarray([0.0 - 1e-7] + [(i + 1) / 10 for i in range(9)] + [1.0 + 1e-7], np.float32)
    edges = np.concatenate([th, np.nextafter(th, np.float32(2)), np.nextafter(th, np.float32(-2)),
                            np.float32([0, -0.0, 1, np.nan, np.inf, -1])]).astype(np.float32)
    cases = [rng.random(n).astype(np.float32) for n in (1, 7, 256, 4097)] + [edges, np.float32([np.nan]),
                                                                              np.float32([0.05, 0.05])]
    for conf in cases:
        n = len(conf)
        labels = rng.integers(0, 5, n)
        pred = np.where(rng.random(n) < 0.5, labels, rng.integers(-1, 5, n))
        want, inb, correct = _old_ece(pred, conf, labels)
        res = classification_result(pred, conf, np.zeros(n), np.zeros(n), labels, [n])
        got = ece_from_bins(inb.sum(1), (inb & correct[None, :]).sum(1),
                            np.where(inb, conf[None, :].astype(np.float64), 0.0).sum(1))
        assert np.array_equal(np.float64(res["ece"]), np.float64(want), equal_nan=True)
        assert np.array_equal(np.float64(got), np.float64(want), equal_nan=True)


def test_train_metric_values():
    from assembled_cnn_b200.metrics import TRAIN_METRICS_DTYPE, ece_from_bins, train_metric_values
    assert TRAIN_METRICS_DTYPE.itemsize == 280
    rec = np.zeros((), TRAIN_METRICS_DTYPE)
    rec["rows"], rec["top1"], rec["top5"] = 8, 3, 6
    rec["bin_count"][9], rec["bin_correct"][9], rec["bin_conf"][9] = 8, 3, 7.5
    rec["step_rows"], rec["step_conf"] = 4, 3.0
    v = train_metric_values(rec)
    assert v == {"sup/pred_prob": 0.75, "train_accuracy": 3 / 8, "train_accuracy_top_5": 6 / 8,
                 "train_ece": ece_from_bins(rec["bin_count"], rec["bin_correct"], rec["bin_conf"])}
    assert train_metric_values(rec, mixup=True) == {"sup/pred_prob": 0.75}


def test_log_line_and_tags_without_gpu(tmp_path, caplog):
    """TrainSummaries._write turns a ring slot into the tags and the log line (mixup: 0 accuracy and ECE)."""
    import types
    import torch
    from assembled_cnn_b200.metrics import TRAIN_METRICS_DTYPE
    from assembled_cnn_b200.summary import SummaryWriter, TrainSummaries
    for mixup, kd in ((False, False), (True, True)):
        ts = TrainSummaries.__new__(TrainSummaries)
        ts.writer = SummaryWriter(str(tmp_path / ("m%d" % mixup)))
        ts.mixup, ts.kd = mixup, kd
        rec = np.zeros((), TRAIN_METRICS_DTYPE)
        rec["rows"], rec["top1"], rec["step_rows"], rec["step_conf"] = 4, 1, 4, 2.0
        ts._host = [(torch.tensor([2.0, 0.5, 0.25]), torch.from_numpy(np.frombuffer(rec.tobytes(), np.uint8).copy()))]
        done = types.SimpleNamespace(query=lambda: True)
        with caplog.at_level(logging.INFO, logger="assembled_cnn_b200"):
            ts._write((0, done, 7, 0.1, 0.9, 100.0, None))
            ts._write((0, done, 9, 0.1, 0.9, 101.0, 3.5))
        ts.writer.close()
        ev = read_events(ts.writer.path)
        tags = [v.tag for v in ev[1].summary.value] + [v.tag for e in ev[2:] for v in e.summary.value
                                                       if e.step == 7]
        want = ["cross_entropy", "l2_loss"] + (["cross_entropy_kd"] if kd else []) + \
            ["loss", "sup/pred_prob", "learning_rate", "dropblock_kp"] + \
            ([] if mixup else ["train_accuracy", "train_accuracy_top_5", "train_ece"])
        assert tags == want
        vals = {v.tag: v.simple_value for e in ev[1:] if e.step == 7 for v in e.summary.value}
        assert vals["loss"] == np.float32(2.5 + (0.25 if kd else 0)) and vals["sup/pred_prob"] == np.float32(0.5)
        assert "global_step/sec" not in vals
        assert [v.simple_value for e in ev[1:] if e.step == 9 for v in e.summary.value
                if v.tag == "global_step/sec"] == [np.float32(3.5)]
        line = [r.getMessage() for r in caplog.records if "step 7:" in r.getMessage()][-1]
        assert "cross_entropy = 2" in line and ("train_accuracy = 0," if mixup else "train_accuracy = 0.25,") in line
        caplog.clear()


def test_argument_errors_without_gpu():
    """The host-side checks of acnn_train_metrics_accumulate run before any CUDA call."""
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    INVALID, p = 1, 1 << 20

    def acc(pred=p, conf=p, hit=p, labels=p, n=4, step_begin=1, m=p):
        return lib.acnn_train_metrics_accumulate(pred, conf, hit, labels, n, step_begin, m, None)
    for kw in (dict(pred=None), dict(conf=None), dict(hit=None), dict(labels=None), dict(m=None), dict(n=0),
               dict(n=-3), dict(m=p + 4)):
        assert acc(**kw) == INVALID, kw
        assert lib.acnn_last_error()
