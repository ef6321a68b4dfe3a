"""GPU checks of AutoAugment on the device: acnn_crop_resize_autoaugment_u8 bit for bit against the numpy
oracle (every operation at every argument the tables produce, both signs, at S in {64, 224, 256, 320}, on
resized random windows and structured images; every sub-policy of every policy with its operations forced on
and off; images with no operation), graph replay and two streams, NativeRuntime.set_images_augmented against the
op-level call, and Trainer.train_step_cropped(augment=) against train_step fed the oracle's images."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MEAN = (123.68, 116.78, 103.94)


def _reference_tables():
    """The policy tables (tests/test_autoaugment_cpu.py pins them to the reference's)."""
    from assembled_cnn_b200.autoaugment import POLICIES
    return {n: [[list(o) for o in sub] for sub in subs] for n, subs in POLICIES.items()}


def _descs(windows, flips, recs, B=None):
    from assembled_cnn_b200.autoaugment import AUTOAUG_DESC_DTYPE
    from assembled_cnn_b200.imagenet_train import CROP_DESC_DTYPE, check_crop_descriptors
    B = B or len(windows)
    offs = np.cumsum([0] + [a.nbytes for a in windows])
    buf = torch.from_numpy(np.concatenate([a.reshape(-1) for a in windows])).cuda()
    desc = np.zeros(B, CROP_DESC_DTYPE)
    for i, (a, f) in enumerate(zip(windows, flips)):
        desc[i] = (buf.data_ptr() + int(offs[i]), a.shape[0], a.shape[1], int(f), (0, 0, 0))
    check_crop_descriptors(desc[:len(windows)])
    aug = np.zeros(B, AUTOAUG_DESC_DTYPE)
    aug[:len(recs)] = recs
    return (buf, torch.from_numpy(desc.view(np.uint8).copy()).cuda(),
            torch.from_numpy(aug.view(np.uint8).copy()).cuda())


def _run(desc, aug, B, n, S, out, mean, work=None):
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    if work is None:
        work = torch.empty(lib.acnn_autoaugment_work_bytes(B, S), dtype=torch.uint8, device="cuda")
    _lib.check(lib.acnn_crop_resize_autoaugment_u8(desc.data_ptr(), aug.data_ptr(), B, n, S, mean.data_ptr(),
                                                   work.data_ptr(), out.data_ptr(),
                                                   torch.cuda.current_stream().cuda_stream),
               "acnn_crop_resize_autoaugment_u8")
    return work


def _structured(S, rng):
    yy, xx = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    dominant = np.full((S, S, 3), 100, np.uint8)
    m = rng.random((S, S)) < 0.05
    dominant[m] = rng.integers(0, 256, (int(m.sum()), 3))
    return [np.full((S, S, 3), 77, np.uint8),                                       # hi == lo, step 0
            np.where(((yy // 3 + xx // 5) % 2 == 0)[..., None], 30, 200).repeat(3, -1).astype(np.uint8),
            dominant,
            np.stack([(yy * S + xx) * 255 // (S * S - 1), 255 - xx * 255 // (S - 1), yy * 255 // (S - 1)],
                     -1).astype(np.uint8)]


def _all_ops(tables):
    return sorted({(op, lv) for subs in tables.values() for sub in subs for op, _, lv in sub})


@pytest.mark.parametrize("S", [64, 224, 256, 320])
def test_every_operation_bit_identical_to_oracle(S):
    from assembled_cnn_b200 import autoaugment as A
    from oracle import autoaugment as O
    rng = np.random.default_rng(S)
    # S x S windows pass through the resize unchanged; the others are resized random windows
    images = _structured(S, rng) + [rng.integers(0, 256, (int(rng.integers(20, 500)), int(rng.integers(20, 500)), 3),
                                                 dtype=np.uint8) for _ in range(2)]
    flips = [False] * 4 + [False, True]
    windows, fl, recs, want = [], [], [], []
    for op, lv in _all_ops(_reference_tables()):
        for neg in ((False, True) if op in A.SIGNED else (False,)):
            for i, img in enumerate(images):
                slot = len(recs) % 2                       # the operation in slot 0 or in slot 1
                cen = (int(rng.integers(0, S)), int(rng.integers(0, S)))
                applied = (slot == 0, slot == 1)
                sub = ((op, 1.0, lv), ("Invert", 0.0, 0)) if slot == 0 else (("Invert", 0.0, 0), (op, 1.0, lv))
                d = np.zeros((), A.AUTOAUG_DESC_DTYPE)
                d["slot"][slot] = A.op_record(op, lv, S, neg, cen)
                recs.append(d)
                windows.append(img)
                fl.append(flips[i])
                negs = (neg, False) if slot == 0 else (False, neg)
                cens = (cen, (0, 0)) if slot == 0 else ((0, 0), cen)
                want.append((img, flips[i], sub, applied, negs, cens))
    A.check_autoaugment_descriptors(np.array(recs), S)
    buf, desc, aug = _descs(windows, fl, recs)
    B = len(windows)
    out = torch.full((B, S, S, 3), 12345.0, device="cuda")
    _run(desc, aug, B, B, S, out, torch.tensor(MEAN, device="cuda"))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for b, (img, f, sub, applied, negs, cens) in enumerate(want):
        ref = O.preprocess(img, f, S, sub, applied, negs, cens)
        assert np.array_equal(got[b], ref), (b, sub, applied, negs, cens, int((got[b] != ref).sum()))


def test_every_subpolicy_bit_identical_to_oracle():
    from assembled_cnn_b200 import autoaugment as A
    from oracle import autoaugment as O
    S = 64
    tables = _reference_tables()
    rng = np.random.default_rng(0)
    windows, fl, recs, want = [], [], [], []
    for name, subs in tables.items():
        for k, sub in enumerate(subs):
            for applied in ((False, False), (True, False), (False, True), (True, True)):
                negs = tuple(bool(x) for x in rng.random(2) < 0.5)
                cens = tuple((int(rng.integers(0, S)), int(rng.integers(0, S))) for _ in range(2))
                win = rng.integers(0, 256, (int(rng.integers(1, 300)), int(rng.integers(1, 300)), 3), dtype=np.uint8)
                flip = bool(rng.random() < 0.5)
                recs.append(A.subpolicy_record(name, k, S, applied, negs, cens))
                windows.append(win)
                fl.append(flip)
                want.append((win, flip, [tuple(o) for o in sub], applied, negs, cens))
    # two padding rows: rows >= n_valid are not written
    buf, desc, aug = _descs(windows, fl, recs, B=len(windows) + 2)
    B, n = len(windows) + 2, len(windows)
    out = torch.full((B, S, S, 3), 12345.0, device="cuda")
    for mean in (torch.tensor(MEAN, device="cuda"), torch.tensor(MEAN)):
        _run(desc, aug, B, n, S, out, mean)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        for b, (win, flip, sub, applied, negs, cens) in enumerate(want):
            assert np.array_equal(got[b], O.preprocess(win, flip, S, sub, applied, negs, cens)), (b, sub, applied)
        assert (got[n:] == 12345.0).all()


def test_no_operation_is_truncated_resize():
    from oracle import autoaugment as O
    from oracle import train_preprocess as T
    rng = np.random.default_rng(2)
    S = 224
    windows = [rng.integers(0, 256, (int(rng.integers(1, 600)), int(rng.integers(1, 600)), 3), dtype=np.uint8)
               for _ in range(16)]
    flips = [i % 2 == 1 for i in range(16)]
    buf, desc, aug = _descs(windows, flips, [])
    out = torch.empty(16, S, S, 3, device="cuda")
    _run(desc, aug, 16, 16, S, out, torch.tensor(MEAN, device="cuda"))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for b, (w, f) in enumerate(zip(windows, flips)):
        want = O.resized_u8(w, f, S).astype(np.float32) - np.float32(MEAN)
        assert np.array_equal(got[b], want)
        assert np.array_equal(want, np.trunc(T.preprocess(w, f, S, (0, 0, 0))) - np.float32(MEAN))


def test_graph_replay_and_streams():
    from assembled_cnn_b200 import autoaugment as A
    rng = np.random.default_rng(1)
    S, B = 224, 64
    windows = [rng.integers(0, 256, (int(rng.integers(1, 400)), int(rng.integers(1, 400)), 3), dtype=np.uint8)
               for _ in range(B)]
    flips = list(rng.random(B) < 0.5)
    recs = [A.resolve(("imagenet", "good")[i % 2], S, np.random.default_rng([9, i])) for i in range(B)]
    buf, desc, aug = _descs(windows, flips, recs)
    mean = torch.tensor(MEAN, device="cuda")
    ref = torch.empty(B, S, S, 3, device="cuda")
    _run(desc, aug, B, B, S, ref, mean)
    out = torch.zeros_like(ref)
    work = torch.empty(A_work(B, S), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _run(desc, aug, B, B, S, out, mean, work)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        out.zero_()
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    outs = [torch.empty_like(ref) for _ in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    for st, o in zip(streams, outs):
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            w = torch.empty(A_work(B, S), dtype=torch.uint8, device="cuda")
            for _ in range(3):
                _run(desc, aug, B, B, S, o, mean, w)
    torch.cuda.synchronize()
    assert all(torch.equal(o, ref) for o in outs)


def A_work(B, S):
    from assembled_cnn_b200 import _lib
    return _lib.load().acnn_autoaugment_work_bytes(B, S)


def test_native_runtime_set_images_augmented_equals_op_level():
    """NativeRuntime.set_images_augmented (acnn_set_images_augmented into the model's "images" buffer) writes
    what the op-level acnn_crop_resize_autoaugment_u8 writes into a buffer of its own; both refuse short
    tables and work buffers, the model level also host tables."""
    from assembled_cnn_b200 import autoaugment as A, native
    from assembled_cnn_b200.plan import ModelConfig
    B, S = 8, 64
    rt_nat = native.NativeRuntime(native.NativeModel(ModelConfig(resnet_size=50), B, S, S, training=False))
    rng = np.random.default_rng(4)
    windows = [rng.integers(0, 256, (int(rng.integers(1, 300)), int(rng.integers(1, 300)), 3), dtype=np.uint8)
               for _ in range(B)]
    recs = [A.resolve("good", S, np.random.default_rng([1, i])) for i in range(B)]
    buf, desc, aug = _descs(windows, [i % 2 == 0 for i in range(B)], recs)
    mean = torch.tensor(MEAN, device="cuda")
    work = torch.empty(A_work(B, S), dtype=torch.uint8, device="cuda")
    images = rt_nat.t[rt_nat.plan.meta["images"]]
    images.zero_()
    rt_nat.set_images_augmented(desc, aug, work, mean)
    op_level = torch.zeros_like(images)
    _run(desc, aug, B, B, S, op_level, mean, work)
    torch.cuda.synchronize()
    assert torch.equal(images, op_level) and op_level.abs().sum() > 0
    # host tables and a short work buffer are refused
    assert rt_nat.lib.acnn_set_images_augmented(rt_nat.model.handle, desc.data_ptr(), aug.cpu().pin_memory().data_ptr(),
                                                work.data_ptr(), mean.data_ptr(), rt_nat.stream) == 1
    with pytest.raises(ValueError):
        rt_nat.set_images_augmented(desc, aug[:88], work, mean)
    with pytest.raises(ValueError):
        rt_nat.set_images_augmented(desc, aug, work[:100], mean)


@pytest.mark.parametrize("dtype,mixup_type,kd_temp", [("bf16", 1, 0), ("fp32", 0, 0), ("bf16", 0, 2.0)])
def test_trainer_augment_equals_oracle_images(dtype, mixup_type, kd_temp):
    from assembled_cnn_b200 import autoaugment as A
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    from oracle import autoaugment as O
    NC, S = 37, 64
    tables = _reference_tables()
    p = params_from_flags(batch_size=8, dataset_name="oxford_iiit_pet", mixup_type=mixup_type, kd_temp=kd_temp,
                          dtype=dtype, label_smoothing=0.1, base_learning_rate=0.1)
    trainers = [Trainer(Model(50, num_classes=NC, dtype=dtype, seed=3), p, S, S, num_images=200) for _ in range(2)]
    ib = trainers[0].input_batch
    rng = np.random.default_rng(6)
    mean = torch.tensor(MEAN, device="cuda")
    losses = [[], []]
    for t in range(3):
        windows = [rng.integers(0, 256, (int(rng.integers(20, 200)), int(rng.integers(20, 200)), 3), dtype=np.uint8)
                   for _ in range(ib)]
        flips = [bool(x) for x in rng.random(ib) < 0.5]
        name = ("imagenet", "good", "v0")[t]
        recs = [A.resolve(name, S, np.random.default_rng([t, i])) for i in range(ib)]
        A.check_autoaugment_descriptors(np.array(recs), S)
        buf, desc, aug = _descs(windows, flips, recs)
        labels = torch.from_numpy(rng.integers(0, NC, ib).astype(np.int32))
        teacher = (rng.standard_normal((ib, NC)) * 2).astype(np.float32) if kd_temp else None
        lam = rng.beta(0.2, 0.2, ib // 2).astype(np.float32) if mixup_type else None
        losses[0].append(trainers[0].train_step_cropped(desc, labels.cuda(), mean, lam1=lam, teacher_logits=teacher,
                                                        augment=aug).tolist())
        x = []
        for w, f, r in zip(windows, flips, recs):
            sub = [tuple(o) for o in tables[name][int(r["subpolicy"])]]
            applied = tuple(bool(r["slot"][j]["op"]) for j in range(2))
            # the sign and the centre are read back from the record, the operations from the reference table
            negs, cens = [], []
            for j, (op, _, lv) in enumerate(sub):
                neg = applied[j] and op in A.SIGNED and \
                    A.op_record(op, lv, S, True).tobytes() == r["slot"][j].tobytes()
                negs.append(bool(neg))
                cens.append((int(r["slot"][j]["i"][0]), int(r["slot"][j]["i"][1])))
            x.append(O.preprocess(w, f, S, sub, applied, negs, cens))
        losses[1].append(trainers[1].train_step(torch.from_numpy(np.stack(x)).pin_memory(), labels, lam1=lam,
                                                teacher_logits=teacher).tolist())
    torch.cuda.synchronize()
    assert losses[0] == losses[1] and all(np.isfinite(l).all() for l in losses[0])
    wa, wb = trainers[0].model.get_weights(), trainers[1].model.get_weights()
    assert all(torch.equal(wa[n], wb[n]) for n in wa)
    assert torch.equal(trainers[0].rt.momentum, trainers[1].rt.momentum)
