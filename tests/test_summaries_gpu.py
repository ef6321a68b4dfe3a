"""GPU checks of the training summaries: acnn_train_metrics_accumulate bit for bit against a numpy restatement of its
documented summation order (row counts around the CTA width, confidences on and next to every bin threshold,
NaN, pred = -1, step_begin on and off, graph replay, two streams); the Trainer's accumulator against
classification_result on the logits and labels read back after every micro-step (bf16 / fp32, R = 1 / 2, mixup +
KD), with the training bits unchanged; train_and_evaluate(save_summary_steps=2) over two cycles (tags, steps,
values, the eval file, a resumed run, the training bits) and the synchronisation calls it adds."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_summaries_cpu import read_events  # noqa: E402


# ------------------------------------------------------------------------------------------ kernel
def _tree(vals):
    """The kernel's fp64 sum: lane t adds rows t, t + 256, ... in order to 0.0, then p[i] += p[i + s]."""
    n = len(vals)
    k = -(-n // 256)
    pad = np.zeros(k * 256)
    pad[:n] = vals
    p = np.cumsum(pad.reshape(k, 256), axis=0)[-1].copy() if k else np.zeros(256)
    s = 128
    while s:
        p[:s] = p[:s] + p[s:2 * s]
        s //= 2
    return p[0]


def _ref(state, pred, conf, hit, labels, step_begin):
    from assembled_cnn_b200.metrics import ece_thresholds
    th = np.asarray(ece_thresholds(), np.float32)
    s = state.copy()
    ok = (pred >= 0) & (pred == labels)
    inb = (conf[None, :] > th[:-1, None]) & (conf[None, :] <= th[1:, None])
    c64 = conf.astype(np.float64)
    s["rows"] += len(pred)
    s["top1"] += ok.sum()
    s["top5"] += (hit != 0).sum()
    s["bin_count"] += inb.sum(1)
    s["bin_correct"] += (inb & ok[None, :]).sum(1)
    for b in range(10):
        s["bin_conf"][b] = s["bin_conf"][b] + _tree(np.where(inb[b], c64, 0.0))
    t = _tree(c64)
    s["step_rows"] = len(pred) if step_begin else s["step_rows"] + len(pred)
    s["step_conf"] = t if step_begin else s["step_conf"] + t
    return s


def _inputs(n, seed):
    from assembled_cnn_b200.metrics import ece_thresholds
    rng = np.random.default_rng(seed)
    th = np.asarray(ece_thresholds(), np.float32)
    special = np.concatenate([th, np.nextafter(th, np.float32(2)), np.nextafter(th, np.float32(-2)),
                              np.float32([np.nan, 0.0, 1.0])])
    conf = rng.random(n).astype(np.float32)
    k = min(n, len(special))
    conf[rng.permutation(n)[:k]] = special[:k]
    labels = rng.integers(0, 10, n).astype(np.int32)
    pred = np.where(rng.random(n) < 0.4, labels, rng.integers(-1, 10, n)).astype(np.int32)
    pred[rng.random(n) < 0.1] = -1
    hit = (rng.random(n) < 0.6).astype(np.int32)
    return pred, conf, hit, labels


def _dev(*arrays):
    return [torch.from_numpy(a).cuda() for a in arrays]


def _same(got, want):
    """Field by field: the same bits, except that a NaN equals a NaN of any payload."""
    for f in got.dtype.names:
        a, b = np.atleast_1d(got[f]), np.atleast_1d(want[f])
        if a.dtype.kind == "f":
            nan = np.isnan(a)
            if not (np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.int64), b[~nan].view(np.int64))):
                return False
        elif not np.array_equal(a, b):
            return False
    return True


def _host(acc):
    from assembled_cnn_b200.metrics import TRAIN_METRICS_DTYPE
    return np.frombuffer(acc.cpu().numpy().tobytes(), TRAIN_METRICS_DTYPE)[0]


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4096])
def test_kernel_bit_exact(n):
    from assembled_cnn_b200.metrics import TRAIN_METRICS_DTYPE, train_metrics_accumulate, train_metrics_buffer
    acc = train_metrics_buffer("cuda")
    want = np.zeros((), TRAIN_METRICS_DTYPE)
    for call, step_begin in enumerate((True, False, False, True)):
        pred, conf, hit, labels = _inputs(n, 10 * n + call)
        dp, dc, dh, dl = _dev(pred, conf, hit, labels)
        train_metrics_accumulate((dp, dc, dh), dl, acc, n, step_begin)
        want = _ref(want, pred, conf, hit, labels, step_begin)
        got = _host(acc)
        assert _same(got, want), (call, got, want)
    # NaN rows land in no bin but in the step's sum; they are counted as rows
    pred, conf, hit, labels = _inputs(n, 1)
    conf[:] = np.nan
    acc.zero_()
    train_metrics_accumulate(_dev(pred, conf, hit)[:3], _dev(labels)[0], acc, n, True)
    got = _host(acc)
    assert got["rows"] == n and got["bin_count"].sum() == 0 and np.isnan(got["step_conf"])


def test_kernel_graph_replay_and_streams():
    from assembled_cnn_b200.metrics import train_metrics_accumulate, train_metrics_buffer
    n = 1000
    pred, conf, hit, labels = _dev(*_inputs(n, 5))
    eager = train_metrics_buffer("cuda")
    for step_begin in (True, False, False):
        train_metrics_accumulate((pred, conf, hit), labels, eager, n, step_begin)
    graphed = train_metrics_buffer("cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graphs = []
    with torch.cuda.stream(s):
        for step_begin in (True, False):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                train_metrics_accumulate((pred, conf, hit), labels, graphed, n, step_begin)
            graphs.append(g)
    torch.cuda.current_stream().wait_stream(s)
    graphed.zero_()
    for g in (graphs[0], graphs[1], graphs[1]):
        g.replay()
    streams = [torch.cuda.Stream() for _ in range(2)]
    per = [train_metrics_buffer("cuda") for _ in streams]
    for st, a in zip(streams, per):
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            for step_begin in (True, False, False):
                train_metrics_accumulate((pred, conf, hit), labels, a, n, step_begin)
    torch.cuda.synchronize()
    assert torch.equal(graphed, eager) and all(torch.equal(a, eager) for a in per)


# ------------------------------------------------------------------------------------------ Trainer
NUM_CLASSES, SIZE, B = 37, 64, 8


def _run_trainer(dtype, R, graph, metrics, mixup_type=0, kd=False, steps=3):
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    p = params_from_flags(batch_size=B * R, dataset_name="oxford_iiit_pet", mixup_type=mixup_type,
                          kd_temp=2.0 if kd else 0, dtype=dtype, label_smoothing=0.1, base_learning_rate=0.1)
    tr = Trainer(Model(50, num_classes=NUM_CLASSES, dtype=dtype, seed=3), p, SIZE, SIZE, use_cuda_graph=graph,
                 replicas_per_device=R, train_metrics=metrics)
    seen = []
    if metrics:
        orig = tr._accumulate_metrics

        def hooked(r):
            logits = tr.rt.t[tr.rt.plan.meta["logits"]][:B, :NUM_CLASSES].clone()
            seen.append((tr.global_step, r, logits, tr.labels_buf[:B].clone()))
            orig(r)
        tr._accumulate_metrics = hooked
    g = torch.Generator().manual_seed(11)
    n = tr.input_batch
    losses, snaps = [], []
    for _ in range(steps):
        x = (torch.randn(R * n, SIZE, SIZE, 3, generator=g) * 64).clamp(-124, 152)
        lab = torch.randint(0, NUM_CLASSES, (R * n,), generator=g).int()
        teach = torch.randn(R * n, NUM_CLASSES, generator=g) * 3 if kd else None
        losses.append(tr.train_step(x, lab, teacher_logits=teach).clone())
        if metrics:
            snaps.append(tr.train_metrics.clone())
    torch.cuda.synchronize()
    rt = tr.rt
    bits = dict(params=rt.params.clone(), momentum=rt.momentum.clone(), state=rt.state.clone(),
                loss=torch.stack(losses))
    return tr, bits, seen, snaps


def _bits_equal(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)


@pytest.mark.parametrize("dtype,R", [("bf16", 1), ("fp32", 1), ("bf16", 2), ("fp32", 2)])
def test_trainer_metrics_equal_classification_result(dtype, R):
    from assembled_cnn_b200.metrics import (classification_result, classify_rows, ece_thresholds,
                                            train_metric_values)
    tr, on, seen, snaps = _run_trainer(dtype, R, graph=True, metrics=True)
    assert len(seen) == 3 * R and [(s, r) for s, r, _, _ in seen] == [(s, r) for s in range(3) for r in range(R)]
    th = np.asarray(ece_thresholds(), np.float32)
    rows = []
    for step in range(3):
        for _, r, logits, labels in seen[step * R:(step + 1) * R]:
            out = classify_rows(logits.contiguous(), labels.contiguous(), k=5, label_smoothing=0.1)
            rows.append([t.cpu().numpy() for t in out] + [labels.cpu().numpy()])
        got = _host(snaps[step])
        pred, conf, hit, ce, lab = (np.concatenate([rw[i] for rw in rows]) for i in range(5))
        want = classification_result(pred, conf, hit, ce, lab, [len(lab)])
        v = train_metric_values(got)
        assert got["rows"] == len(lab) and got["top1"] == int((pred == lab).sum()) and got["top5"] == int(hit.sum())
        assert v["train_accuracy"] == want["accuracy"] and v["train_accuracy_top_5"] == want["accuracy_top_5"]
        assert abs(v["train_ece"] - want["ece"]) <= 1e-12
        inb = (conf[None, :] > th[:-1, None]) & (conf[None, :] <= th[1:, None])
        assert np.array_equal(got["bin_count"], inb.sum(1))
        assert np.array_equal(got["bin_correct"], (inb & (pred == lab)[None, :]).sum(1))
        assert np.allclose(got["bin_conf"], np.where(inb, conf[None, :].astype(np.float64), 0).sum(1), rtol=0,
                           atol=1e-12)
        step_conf = np.concatenate([rw[1] for rw in rows[-R:]]).astype(np.float64)
        assert got["step_rows"] == B * R and abs(v["sup/pred_prob"] - step_conf.mean()) <= 1e-12
    # no effect on training: graph and eager, metrics on and off
    _, off, _, _ = _run_trainer(dtype, R, graph=True, metrics=False)
    assert _bits_equal(on, off)
    _, eager_on, _, eager_snaps = _run_trainer(dtype, R, graph=False, metrics=True)
    _, eager_off, _, _ = _run_trainer(dtype, R, graph=False, metrics=False)
    assert _bits_equal(eager_on, eager_off) and _bits_equal(eager_on, on)
    assert all(torch.equal(a, b) for a, b in zip(eager_snaps, snaps))
    assert tr.train_metrics is not None
    tr.reset_train_metrics()
    assert int(tr.train_metrics.sum()) == 0


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_trainer_metrics_with_mixup_and_kd(dtype):
    """With mixup the labels are mixed: the per-step fields are the ones the summaries read."""
    from assembled_cnn_b200.metrics import classify_rows
    tr, on, seen, snaps = _run_trainer(dtype, 2, graph=True, metrics=True, mixup_type=1, kd=True)
    assert tr.input_batch == 2 * B
    for step in range(3):
        confs = []
        for _, _, logits, labels in seen[2 * step:2 * step + 2]:
            confs.append(classify_rows(logits.contiguous(), labels.contiguous(), k=5)[1].cpu().numpy())
        got = _host(snaps[step])
        assert got["step_rows"] == 2 * B and got["rows"] == 2 * B * (step + 1)
        assert abs(got["step_conf"] - np.concatenate(confs).astype(np.float64).sum()) <= 1e-12
    _, off, _, _ = _run_trainer(dtype, 2, graph=True, metrics=False, mixup_type=1, kd=True)
    assert _bits_equal(on, off)


def test_trainer_without_metrics_has_no_buffer():
    tr, _, _, _ = _run_trainer("bf16", 1, graph=True, metrics=False, steps=1)
    assert tr.train_metrics is None


# ------------------------------------------------------------------------------- train_and_evaluate
sys.path.insert(0, os.path.join(HERE, "golden"))
DATASET = "oxford_iiit_pet"
FLAGS = dict(batch_size=32, dataset_name=DATASET, train_epochs=2, image_size=SIZE, seed=11, num_workers=4,
             dtype="bf16", label_smoothing=0.1, base_learning_rate=0.05, num_best_ckpt_to_keep=1,
             save_checkpoints_epochs=0.5, keep_checkpoint_max=3)


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    """200 training JPEGs in three train-* shards and 40 in one validation shard (the golden generator's
    writer, as tests/test_train_input_gpu.py writes them)."""
    import make_eval_preprocess_golden as mk
    from test_train_input_gpu import _write_shard
    Example = mk.example_class()
    root = tmp_path_factory.mktemp("data")
    rng = np.random.default_rng(0)
    for sh, n in enumerate((70, 70, 60)):
        _write_shard(root / ("train-%05d-of-00003" % sh), Example, mk, rng, n, kd=False)
    _write_shard(root / "validation-00000-of-00001", Example, mk, rng, 40, kd=False)
    return root


def _weights(path):
    with np.load(path) as z:
        return {n: z[n] for n in z.files}


def _scalars(path):
    """{step: {tag: value}} of the scalar events of a file (the file-version record first)."""
    ev = read_events(path)
    assert ev[0].file_version == "brain.Event:2"
    out = {}
    for e in ev[1:]:
        for v in e.summary.value:
            out.setdefault(e.step, {})[v.tag] = v.simple_value
    return out


def _counted_run(monkeypatch, *args, **kw):
    """train_and_evaluate with the device synchronisations counted and each step's loss recorded."""
    from assembled_cnn_b200 import model_fns
    count = {"n": 0}
    losses = {}
    orig_tsc = model_fns.Trainer.train_step_cropped

    def tsc(self, *a, **k):
        step = self.global_step
        loss = orig_tsc(self, *a, **k)
        losses[step] = loss.tolist()
        return loss

    def counting(fn):
        def f(*a, **k):
            count["n"] += 1
            return fn(*a, **k)
        return f
    with monkeypatch.context() as m:
        m.setattr(model_fns.Trainer, "train_step_cropped", tsc)
        m.setattr(torch.cuda, "synchronize", counting(torch.cuda.synchronize))
        m.setattr(torch.cuda.Event, "synchronize", counting(torch.cuda.Event.synchronize))
        res = model_fns.train_and_evaluate(*args, **kw)
    return res, losses, count["n"]


def test_train_and_evaluate_summaries(shards, tmp_path, monkeypatch):
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import learning_rate_with_decay
    run, plain = tmp_path / "run", tmp_path / "plain"
    res, losses, n_sync = _counted_run(monkeypatch, str(shards), str(run), save_summary_steps=2, **FLAGS)
    res0, losses0, n_sync0 = _counted_run(monkeypatch, str(shards), str(plain), **FLAGS)
    assert res == res0 and losses == losses0 and [r["global_step"] for r in res] == [6, 12]
    a, b = _weights(str(run / "model.ckpt-12.npz")), _weights(str(plain / "model.ckpt-12.npz"))
    assert all(np.array_equal(a[n], b[n]) for n in b)
    assert not glob.glob(str(plain / "events.*")) and not (plain / "eval").exists()
    # the step already waits on its hyper-parameter ring; the summaries add no wait per step (six summaries, four
    # checkpoints, two evaluations)
    assert n_sync - n_sync0 <= 4 + 2 + 1, (n_sync, n_sync0)

    files = glob.glob(str(run / "events.out.tfevents.*"))
    assert len(files) == 1
    got = _scalars(files[0])
    assert sorted(got) == [0, 2, 4, 6, 8, 10]     # each cycle's first step, then every second one
    p = params_from_flags(**{k: v for k, v in FLAGS.items() if k not in ("image_size", "seed", "num_workers")})
    lr_fn = learning_rate_with_decay(
        learning_rate_decay_type=p["learning_rate_decay_type"], batch_size=p["batch_size"],
        batch_denom=p["batch_size"], num_images=200, num_epochs_per_decay=p["num_epochs_per_decay"],
        learning_rate_decay_factor=p["learning_rate_decay_factor"], end_learning_rate=p["end_learning_rate"],
        piecewise_lr_boundary_epochs=p["piecewise_lr_boundary_epochs"],
        piecewise_lr_decay_rates=p["piecewise_lr_decay_rates"], base_lr=p["base_learning_rate"],
        train_epochs=p["train_epochs"], warmup_epochs=p["lr_warmup_epochs"])
    tags = {"cross_entropy", "l2_loss", "loss", "sup/pred_prob", "learning_rate", "dropblock_kp", "train_accuracy",
            "train_accuracy_top_5", "train_ece"}
    for step, vals in got.items():
        first = step in (0, 6)
        assert set(vals) == tags | (set() if first else {"global_step/sec"}), (step, sorted(vals))
        ce, l2 = losses[step][:2]
        assert vals["cross_entropy"] == np.float32(ce) and vals["l2_loss"] == np.float32(l2)
        assert vals["loss"] == np.float32(ce + l2)
        assert vals["learning_rate"] == np.float32(lr_fn(step)) and vals["dropblock_kp"] == 1.0
        assert 0 <= vals["train_accuracy"] <= vals["train_accuracy_top_5"] <= 1 and 0 < vals["sup/pred_prob"] <= 1
        assert first or vals["global_step/sec"] > 0
    ev = glob.glob(str(run / "eval" / "events.out.tfevents.*"))
    assert len(ev) == 1
    assert _scalars(ev[0]) == {r["global_step"]: {k: np.float32(v) for k, v in r.items() if k != "global_step"}
                               for r in res}

    # stopped after cycle 1, then resumed: a new file continues the steps
    resumed = tmp_path / "resumed"
    first = train_and_evaluate_kw(shards, resumed, stop_threshold=0.0)
    second = train_and_evaluate_kw(shards, resumed)
    assert first + second == res
    files = sorted(glob.glob(str(resumed / "events.out.tfevents.*")))
    assert len(files) == 2
    steps = sorted(sorted(_scalars(f)) for f in files)
    assert steps == [[0, 2, 4], [6, 8, 10]]
    c = _weights(str(resumed / "model.ckpt-12.npz"))
    assert all(np.array_equal(c[n], b[n]) for n in b)


def train_and_evaluate_kw(shards, model_dir, **kw):
    from assembled_cnn_b200.model_fns import train_and_evaluate
    return train_and_evaluate(str(shards), str(model_dir), save_summary_steps=2, **dict(FLAGS, **kw))
