"""Dynamic loss scaling on the H100: the finiteness check, the scale update and the skip-aware SGD against numpy
and the restatement of tests/test_dynamic_loss_scale_cpu.py, then the Trainer bit for bit against static runs
(constant scale, growth, overflow, replicas), train_and_evaluate with summaries and a resume, and acnn_step
through the model-level C ABI."""
import ctypes as C
import glob

import numpy as np
import pytest
import torch

from test_dynamic_loss_scale_cpu import update as ref_update

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
C3 = dict(resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what):
    from assembled_cnn_b200 import _lib
    _lib.check(rc, what)


def _c3_param_elems():
    from assembled_cnn_b200.native import NativeModel
    from assembled_cnn_b200.plan import ModelConfig
    return NativeModel(ModelConfig(resnet_size=50, **C3), 8, 64, 64, training=True).param_elems


# ------------------------------------------------------------------------------------ check kernel
def _flag_of(lib, x, flag):
    flag.zero_()
    _check(lib.acnn_grads_nonfinite(x.data_ptr(), x.numel(), flag.data_ptr(), _st()), "grads_nonfinite")
    return int(flag.item())


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 2 ** 20 + 3, "c3"])
def test_check_kernel(lib, n):
    n = _c3_param_elems() if n == "c3" else n
    g = torch.Generator(device="cuda").manual_seed(n % 1000)
    base = torch.randn(n + 1, device="cuda", generator=g)
    # finite extremes: -0, denormals, +-FLT_MAX
    special = torch.tensor([-0.0, 1e-45, -1e-40, FLT_MAX, -FLT_MAX], device="cuda")
    k = min(n, special.numel())
    base[n - k:n] = special[:k]
    base[0] = special[3] if n > 1 else base[0]
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    for off in (0, 1):                         # 16-byte aligned, and a scalar head before the first vector
        x = base[off:off + n]
        assert _flag_of(lib, x, flag) == int((~torch.isfinite(x)).any())
        assert _flag_of(lib, x, flag) == 0
        mid = min(n - 1, 4 * (n // 8) + 2)     # inside a float4 of the vector part
        tail = n - 1 - (n % 4) // 2            # among the last n % 4 elements (the tail when aligned)
        for pos in sorted({0, n - 1, mid, tail}):
            keep = x[pos].clone()
            for v in (float("inf"), float("-inf"), float("nan")):
                x[pos] = v
                assert _flag_of(lib, x, flag) == 1, (n, off, pos, v)
            x[pos] = keep
        assert _flag_of(lib, x, flag) == 0
    # the check never clears a set flag
    flag.fill_(1)
    _check(lib.acnn_grads_nonfinite(base.data_ptr(), n, flag.data_ptr(), _st()), "grads_nonfinite")
    assert int(flag.item()) == 1


def test_check_kernel_graph_replay_and_streams(lib):
    n = 2 ** 20 + 3
    x = torch.randn(n, device="cuda")
    x[n // 3] = float("nan")
    flags = torch.zeros(3, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _check(lib.acnn_grads_nonfinite(x.data_ptr(), n, flags[0:1].data_ptr(), s.cuda_stream), "grads_nonfinite")
    torch.cuda.current_stream().wait_stream(s)
    got = []
    for bad in (True, False, True):
        x[n // 3] = float("nan") if bad else 0.5
        flags.zero_()
        graph.replay()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        for st, i in ((s1, 1), (s2, 2)):
            st.wait_stream(torch.cuda.current_stream())
            _check(lib.acnn_grads_nonfinite(x.data_ptr(), n, flags[i:i + 1].data_ptr(), st.cuda_stream),
                   "grads_nonfinite")
            torch.cuda.current_stream().wait_stream(st)
        got.append(flags.tolist())
    assert got == [[1, 1, 1], [0, 0, 0], [1, 1, 1]]


# ------------------------------------------------------------------------------------ update kernel
def _state(scale, good=0, skipped=0, nonfinite=0):
    w = np.zeros(8, np.int32)
    w[[0, 4]] = np.array([scale, scale], np.float32).view(np.int32)
    w[1], w[2], w[3] = good, skipped, nonfinite
    return torch.from_numpy(w).cuda()


@pytest.mark.parametrize("start,growth", [(2.0 ** 15, 2000), (2.0, 3), (1.0, 1), (2.0 ** 126, 1), (0.5, 2)])
def test_update_kernel_equals_restatement(lib, start, growth):
    from assembled_cnn_b200.native import decode_loss_scale_state
    rng = np.random.default_rng(int(start) + growth)
    buf = _state(start)
    want = (np.float32(start), 0, 0)
    for p_bad in (0.0, 0.5, 0.1, 0.9):
        for bad in (rng.random(40) < p_bad).astype(int):
            buf[3] = int(bad)
            _check(lib.acnn_loss_scale_update(buf.data_ptr(), growth, _st()), "loss_scale_update")
            used, want = ref_update(want, bad, growth)
            got = decode_loss_scale_state(buf.cpu())
            assert (got["scale"], got["good_steps"], got["skipped_steps"]) == (float(want[0]), want[1], want[2])
            assert got["last_scale"] == float(used) and int(buf[3]) == 0


# ------------------------------------------------------------------------------------ skip-aware SGD
@pytest.mark.parametrize("divisor", [1, 3])
def test_sgd_skip_and_scale(lib, divisor):
    n = 256 * 1031
    g = torch.Generator(device="cuda").manual_seed(divisor)
    w0 = torch.randn(n, device="cuda", generator=g)
    grad = torch.randn(n, device="cuda", generator=g) * 300
    acc0 = torch.randn(n, device="cuda", generator=g)
    flags = (torch.rand(n // 256, device="cuda", generator=g) < 0.7).to(torch.uint8)
    scale = 512.0
    hp = torch.tensor([0.1, 0.9, 1e-4, 1.0 / (divisor * scale), 0, 0, 0, 0], device="cuda")
    assert float(hp[3]) == float(np.float32(1.0 / (divisor * scale)))
    nsc = lib.acnn_sgd_scratch_floats()

    def run(dyn, nonfinite):
        w, acc = w0.clone(), acc0.clone()
        l2 = torch.zeros(4, device="cuda")
        scratch = torch.zeros(nsc, device="cuda")
        if dyn:
            ls = _state(scale, nonfinite=nonfinite)
            _check(lib.acnn_sgd_momentum_loss_scaled(w.data_ptr(), grad.data_ptr(), acc.data_ptr(), n,
                                                     flags.data_ptr(), hp.data_ptr(), ls.data_ptr(), divisor,
                                                     l2.data_ptr(), scratch.data_ptr(), _st()), "sgd_loss_scaled")
        else:
            _check(lib.acnn_sgd_momentum(w.data_ptr(), grad.data_ptr(), acc.data_ptr(), n, flags.data_ptr(),
                                         hp.data_ptr(), l2.data_ptr(), scratch.data_ptr(), _st()), "sgd")
        return w, acc, l2

    ws, accs, l2s = run(False, 0)
    wd, accd, l2d = run(True, 0)
    assert torch.equal(ws.view(torch.int32), wd.view(torch.int32)) and torch.equal(accs, accd)
    assert torch.equal(l2s, l2d)
    wk, acck, l2k = run(True, 1)
    assert torch.equal(wk.view(torch.int32), w0.view(torch.int32))
    assert torch.equal(acck.view(torch.int32), acc0.view(torch.int32))
    assert torch.equal(l2k, l2s) and float(l2k[0]) > 0


def test_softmax_ce_scaled_equals_static(lib):
    B, NC, ld = 33, 1001, 1024
    g = torch.Generator(device="cuda").manual_seed(5)
    logits = torch.randn(B, ld, device="cuda", generator=g) * 4
    y = torch.softmax(torch.randn(B, NC, device="cuda", generator=g), 1).contiguous()
    scale = torch.tensor([128.0], device="cuda")
    outs = []
    for dev in (False, True):
        loss = torch.zeros(4, device="cuda")
        dl = torch.zeros(B, ld, dtype=torch.float16, device="cuda")
        dbias = torch.zeros(ld, device="cuda")
        work = torch.zeros(2 * 64 + B * ld, device="cuda")
        if dev:
            rc = lib.acnn_softmax_ce_scaled(logits.data_ptr(), y.data_ptr(), None, 0.0, B, NC, ld, 0.1,
                                            scale.data_ptr(), loss.data_ptr(), dl.data_ptr(), dbias.data_ptr(),
                                            work.data_ptr(), 3, _st())
        else:
            rc = lib.acnn_softmax_ce(logits.data_ptr(), y.data_ptr(), None, 0.0, B, NC, ld, 0.1, 128.0,
                                     loss.data_ptr(), dl.data_ptr(), dbias.data_ptr(), work.data_ptr(), 3, _st())
        _check(rc, "softmax_ce")
        outs.append((loss, dl, dbias))
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int16 if a.dtype == torch.float16 else torch.int32),
                           b.view(torch.int16 if b.dtype == torch.float16 else torch.int32))


# ------------------------------------------------------------------------------------ Trainer
NUM_CLASSES, SIZE, B = 37, 64, 8


def _trainer(dtype, loss_scale, graph, R=1, mixup_type=1, kd=True, **kw):
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    p = params_from_flags(batch_size=B * R, dataset_name="oxford_iiit_pet", mixup_type=mixup_type,
                          kd_temp=2.0 if kd else 0, dtype=dtype, label_smoothing=0.1, base_learning_rate=0.1,
                          loss_scale=loss_scale, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                          anti_alias_filter_size=3)
    model = Model(50, num_classes=NUM_CLASSES, dtype=dtype, seed=3, resnet_version=2, use_sk_block=True,
                  anti_alias_type="sconv", anti_alias_filter_size=3)
    return Trainer(model, p, SIZE, SIZE, use_cuda_graph=graph, replicas_per_device=R, **kw)


def _inputs(tr, steps, seed=11, kd=True):
    g = torch.Generator().manual_seed(seed)
    R, n = tr.replicas, tr.input_batch
    out = []
    for _ in range(steps):
        x = (torch.randn(R * n, SIZE, SIZE, 3, generator=g) * 64).clamp(-124, 152)
        lab = torch.randint(0, NUM_CLASSES, (R * n,), generator=g).int()
        teach = torch.randn(R * n, NUM_CLASSES, generator=g) * 3 if kd else None
        lam = torch.rand(R, n // 2, generator=g) if tr.mixup_type else None
        out.append((x, lab, teach, lam))
    return out


def _step(tr, inp):
    x, lab, teach, lam = inp
    return tr.train_step(x, lab, lam1=lam, teacher_logits=teach).clone()


def _bits(tr, losses=None):
    rt = tr.rt
    torch.cuda.synchronize()
    d = dict(params=rt.params.clone(), momentum=rt.momentum.clone(), state=rt.state.clone())
    if losses is not None:
        d["loss"] = torch.stack(losses)
    return d


def _same(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("dtype,init,static", [("fp16", 128.0, 128.0), ("bf16", 1.0, None)])
def test_dynamic_at_a_constant_scale_equals_static(graph, dtype, init, static):
    steps = 4
    dyn = _trainer(dtype, "dynamic", graph, initial_loss_scale=init, loss_scale_growth_interval=1000)
    ref = _trainer(dtype, static, graph)
    assert ref.loss_scale == (128.0 if dtype == "fp16" else 1.0) and dyn.loss_scale == "dynamic"
    inputs = _inputs(dyn, steps)
    ld = [_step(dyn, i) for i in inputs]
    ls = [_step(ref, i) for i in inputs]
    a, b = _bits(dyn, ld), _bits(ref, ls)
    assert torch.isfinite(a["params"]).all() and _same(a, b)
    assert dyn.loss_scale_state() == {"scale": init, "good_steps": steps, "skipped_steps": 0}
    assert ref.loss_scale_state() is None and dyn.global_step == ref.global_step == steps


def test_growth_equals_a_switched_static_run():
    steps, growth = 6, 2
    dyn = _trainer("fp16", "dynamic", True, initial_loss_scale=128.0, loss_scale_growth_interval=growth)
    ref = _trainer("fp16", 128.0, False)
    inputs = _inputs(dyn, steps)
    ld, ls, seen = [], [], []
    for t, inp in enumerate(inputs):
        s = 128.0 * 2 ** (t // growth)
        ref.loss_scale = s
        ref.rt.loss_scale = s
        ld.append(_step(dyn, inp))
        ls.append(_step(ref, inp))
        seen.append(dyn.loss_scale_state())
    assert [st["scale"] for st in seen] == [128, 256, 256, 512, 512, 1024]
    assert [st["good_steps"] for st in seen] == [1, 0, 1, 0, 1, 0]
    assert _same(_bits(dyn, ld), _bits(ref, ls))


def _load(tr, snap):
    rt = tr.rt
    rt.params.copy_(snap["params"])
    rt.momentum.copy_(snap["momentum"])
    rt.state.copy_(snap["state"])


def test_overflow_skips_then_equals_a_static_step():
    dyn = _trainer("fp16", "dynamic", True, initial_loss_scale=2.0 ** 24, loss_scale_growth_interval=1000)
    ref = _trainer("fp16", 128.0, False)
    inputs = _inputs(dyn, 24)
    skipped = 0
    for t, inp in enumerate(inputs):
        before = _bits(dyn)
        st0 = dyn.loss_scale_state()
        lr0 = dyn.learning_rate_fn(dyn.global_step)
        _step(dyn, inp)
        after = _bits(dyn)
        st1 = dyn.loss_scale_state()
        # the same step from the same state at the same scale, static
        _load(ref, before)
        ref.global_step = t
        ref.loss_scale = st0["scale"]
        ref.rt.loss_scale = st0["scale"]
        _step(ref, inp)
        other = _bits(ref)
        assert dyn.global_step == t + 1 and dyn.last_lr == lr0
        assert torch.equal(after["state"].view(torch.int32), other["state"].view(torch.int32))
        if st1["skipped_steps"] > st0["skipped_steps"]:
            skipped += 1
            assert st1 == {"scale": max(st0["scale"] / 2, 1.0), "good_steps": 0, "skipped_steps": skipped}
            assert torch.equal(after["params"].view(torch.int32), before["params"].view(torch.int32))
            assert torch.equal(after["momentum"].view(torch.int32), before["momentum"].view(torch.int32))
            assert not torch.isfinite(ref.rt.grads).all()
        else:
            assert skipped >= 1 and st1 == {"scale": st0["scale"], "good_steps": 1, "skipped_steps": skipped}
            assert _same(after, other) and torch.isfinite(after["params"]).all()
            break
    else:
        pytest.fail("no finite step after %d skips" % skipped)


def test_replicas_constant_scale_and_one_overflowing_micro_step():
    steps = 3
    dyn = _trainer("fp16", "dynamic", True, R=2, initial_loss_scale=128.0, loss_scale_growth_interval=1000)
    ref = _trainer("fp16", 128.0, True, R=2)
    inputs = _inputs(dyn, steps)
    ld = [_step(dyn, i) for i in inputs]
    ls = [_step(ref, i) for i in inputs]
    assert _same(_bits(dyn, ld), _bits(ref, ls))
    assert dyn.loss_scale_state() == {"scale": 128.0, "good_steps": steps, "skipped_steps": 0}
    # an inf pixel in the second micro-step's images: its gradients are not finite, the whole step is skipped
    x, lab, teach, lam = _inputs(dyn, 1, seed=12)[0]
    x[dyn.input_batch + 3, 5, 7, 1] = float("inf")
    before = _bits(dyn)
    _step(dyn, (x, lab, teach, lam))
    after = _bits(dyn)
    assert torch.equal(after["params"].view(torch.int32), before["params"].view(torch.int32))
    assert torch.equal(after["momentum"].view(torch.int32), before["momentum"].view(torch.int32))
    assert dyn.loss_scale_state() == {"scale": 64.0, "good_steps": 0, "skipped_steps": 1}


# ------------------------------------------------------------------------------------ train_and_evaluate
from test_summaries_gpu import FLAGS, _counted_run, _scalars, _weights, shards  # noqa: E402,F401


def _same_results(a, b):
    return len(a) == len(b) and all(x.keys() == y.keys() and all(np.array_equal(x[k], y[k], equal_nan=True) for k in x)
                                    for x, y in zip(a, b))


def test_train_and_evaluate_dynamic(shards, tmp_path, monkeypatch):  # noqa: F811
    from assembled_cnn_b200.checkpoint import LOSS_SCALE_KEYS
    from assembled_cnn_b200.model_fns import train_and_evaluate
    flags = dict(FLAGS, dtype="fp16", loss_scale="dynamic")
    run, quiet = tmp_path / "run", tmp_path / "quiet"
    res, losses, n_sync = _counted_run(monkeypatch, str(shards), str(run), save_summary_steps=1, **flags)
    res0, losses0, n_sync0 = _counted_run(monkeypatch, str(shards), str(quiet), **flags)
    _, _, n_sync_static = _counted_run(monkeypatch, str(shards), str(tmp_path / "static"), **dict(flags, loss_scale=None))
    # (the fp16 evaluation loss may be NaN: forward activations under barely-moved moving statistics)
    assert _same_results(res, res0) and [r["global_step"] for r in res] == [6, 12]
    assert sorted(losses) == sorted(losses0) == list(range(12))
    assert np.array_equal([losses[k] for k in range(12)], [losses0[k] for k in range(12)], equal_nan=True)
    # no wait per step: the summaries add at most one per checkpoint and evaluation, as for a static run, and
    # dynamic scaling itself adds none
    assert n_sync - n_sync0 <= 4 + 2 + 1 and n_sync0 == n_sync_static, (n_sync, n_sync0, n_sync_static)
    ck = _weights(str(run / "model.ckpt-12.npz"))
    assert set(LOSS_SCALE_KEYS) <= set(ck)
    got = _scalars(glob.glob(str(run / "events.out.tfevents.*"))[0])
    assert sorted(got) == list(range(12))
    scale, skipped = 2.0 ** 15, 0
    for step in range(12):
        vals = got[step]
        assert vals["loss_scale"] == scale, (step, vals["loss_scale"], scale)
        bad = vals["loss_scale/skipped_steps"] > skipped
        skipped = int(vals["loss_scale/skipped_steps"])
        scale = max(scale / 2, 1.0) if bad else scale
    assert float(ck[LOSS_SCALE_KEYS[0]]) == scale and int(ck[LOSS_SCALE_KEYS[2]]) == skipped
    # stopped after cycle 1, then resumed: the same weights and scale state
    resumed = tmp_path / "resumed"
    first = train_and_evaluate(str(shards), str(resumed), stop_threshold=0.0, **flags)
    second = train_and_evaluate(str(shards), str(resumed), **flags)
    assert _same_results(first + second, res)
    c = _weights(str(resumed / "model.ckpt-12.npz"))
    assert set(c) == set(ck) and all(np.array_equal(c[k], ck[k]) for k in ck)


# ------------------------------------------------------------------------------------ model-level C ABI
def test_acnn_step_equals_trainer():
    from assembled_cnn_b200 import native
    from assembled_cnn_b200.model_fns import Model
    steps = 6
    tr = _trainer("fp16", "dynamic", False, mixup_type=0, kd=False, initial_loss_scale=2.0 ** 24,
                  loss_scale_growth_interval=2)
    model = Model(50, num_classes=NUM_CLASSES, dtype="fp16", seed=3, resnet_version=2, use_sk_block=True,
                  anti_alias_type="sconv", anti_alias_filter_size=3)
    rt = model.runtime(B, SIZE, SIZE, training=True, mixup_type=0, label_smoothing=0.1)
    rt.enable_dynamic_loss_scale(2.0 ** 24, 2, 1)
    lib, h = rt.lib, rt.model.handle
    inputs = _inputs(tr, steps, kd=False)
    host = (C.c_int32 * 8)()
    la, lb = [], []
    for t, (x, lab, _, _) in enumerate(inputs):
        la.append(_step(tr, (x, lab, None, None)))
        hp = np.array([tr.learning_rate_fn(t), tr.p["momentum"], tr.p["weight_decay"], 0.0, 1.0, 0, 0, 0], np.float32)
        hp.view(np.int32)[5] = t
        xs, ls_ = x.contiguous(), lab.contiguous()
        _check(lib.acnn_set_inputs(h, xs.data_ptr(), ls_.data_ptr(), None, None, None, _st()), "acnn_set_inputs")
        _check(lib.acnn_set_hparams(h, hp.ctypes.data, _st()), "acnn_set_hparams")
        _check(lib.acnn_step(h, _st()), "acnn_step")
        torch.cuda.synchronize()
        lb.append(rt.slot_view(rt.plan.meta["loss"])[:2].clone())
        _check(lib.acnn_get_loss_scale_state(h, C.cast(host, C.c_void_p), _st()), "acnn_get_loss_scale_state")
        torch.cuda.synchronize()
        st = native.decode_loss_scale_state(np.frombuffer(host, np.int32))
        assert {k: st[k] for k in ("scale", "good_steps", "skipped_steps")} == tr.loss_scale_state()
    assert tr.loss_scale_state()["skipped_steps"] >= 1
    a = _bits(tr, la)
    b = dict(params=rt.params.clone(), momentum=rt.momentum.clone(), state=rt.state.clone(), loss=torch.stack(lb))
    assert _same(a, b)
