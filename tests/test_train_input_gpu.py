"""GPU checks of training from TFRecord shards: acnn_crop_resize_u8 bit for bit against the float32 oracle
(random windows, both flips, down- and upscaling, 1-pixel windows, S in {64, 224, 256}, padding rows, graph
replay, two streams); Trainer steps fed through the staging ring and acnn_set_images_cropped against the
same steps fed the oracle's fp32 images (bf16 / fp32, mixup type 1, KD); model_fns.train_and_evaluate end to
end on synthetic shards (checkpoints, keeper, per-cycle evaluation, resume, graph vs eager, warm start)."""
import io
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.abspath(__file__))
MEAN = (123.68, 116.78, 103.94)


def _descs(windows, flips, B, device="cuda"):
    from assembled_cnn_b200.imagenet_train import CROP_DESC_DTYPE, check_crop_descriptors
    offs = np.cumsum([0] + [a.nbytes for a in windows])
    buf = torch.from_numpy(np.concatenate([a.reshape(-1) for a in windows])).to(device)
    desc = np.zeros(B, CROP_DESC_DTYPE)
    for i, (a, f) in enumerate(zip(windows, flips)):
        desc[i] = (buf.data_ptr() + int(offs[i]), a.shape[0], a.shape[1], int(f), (0, 0, 0))
    check_crop_descriptors(desc[:len(windows)])
    return buf, torch.from_numpy(desc.view(np.uint8).copy()).to(device)


def _crop_resize(desc, B, n, S, out, mean):
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    _lib.check(lib.acnn_crop_resize_u8(desc.data_ptr(), B, n, S, mean.data_ptr(), out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "acnn_crop_resize_u8")


SHAPES = [(1, 1), (1, 9), (9, 1), (500, 375), (375, 500), (33, 47), (224, 224), (300, 120), (2, 3), (64, 64),
          (700, 20), (17, 600)]


@pytest.mark.parametrize("S", [64, 224, 256])
def test_crop_resize_bit_identical_to_oracle(S):
    from oracle import train_preprocess as O
    rng = np.random.default_rng(S)
    windows = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in SHAPES for _ in range(2)]
    flips = [i % 2 == 1 for i in range(len(windows))]
    B = len(windows) + 3
    buf, desc = _descs(windows, flips, B)
    out = torch.full((B, S, S, 3), 12345.0, device="cuda")
    for mean in (torch.tensor(MEAN, device="cuda"), torch.tensor(MEAN)):
        _crop_resize(desc, B, len(windows), S, out, mean)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        for i, (a, f) in enumerate(zip(windows, flips)):
            assert np.array_equal(got[i], O.preprocess(a, f, S)), (a.shape, f, S)
        assert (got[len(windows):] == 12345.0).all()              # rows >= n_valid untouched
    # a 1 x 1 window is a constant image; flipping a window changes an asymmetric result
    assert np.array_equal(got[0], np.broadcast_to(windows[0][0, 0].astype(np.float32) - np.float32(MEAN), got[0].shape))
    assert not np.array_equal(O.preprocess(windows[6], False, S), O.preprocess(windows[6], True, S))


def test_crop_resize_graph_replay_and_streams():
    rng = np.random.default_rng(1)
    windows = [rng.integers(0, 256, (int(rng.integers(1, 400)), int(rng.integers(1, 400)), 3), dtype=np.uint8)
               for _ in range(32)]
    flips = list(rng.random(32) < 0.5)
    buf, desc = _descs(windows, flips, 32)
    mean = torch.tensor(MEAN, device="cuda")
    ref = torch.empty(32, 224, 224, 3, device="cuda")
    _crop_resize(desc, 32, 32, 224, ref, mean)
    out = torch.zeros_like(ref)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _crop_resize(desc, 32, 32, 224, out, mean)
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
            for _ in range(3):
                _crop_resize(desc, 32, 32, 224, o, mean)
    torch.cuda.synchronize()
    assert all(torch.equal(o, ref) for o in outs)


# ------------------------------------------------------------------------------------------ shards
NUM_CLASSES, SIZE, DATASET = 37, 64, "oxford_iiit_pet"


def _write_shard(path, Example, mk, rng, n, kd):
    from PIL import Image
    recs = []
    for _ in range(n):
        h, w = int(rng.integers(20, 150)), int(rng.integers(20, 150))
        base = rng.integers(0, 256, 3)
        img = np.clip(base + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        ex = Example()
        ex.features.feature["image/encoded"].bytes_list.value.append(buf.getvalue())
        ex.features.feature["image/class/label"].int64_list.value.append(int(rng.integers(0, NUM_CLASSES)))
        if kd:
            ex.features.feature["image/logit"].float_list.value.extend(
                (rng.standard_normal(NUM_CLASSES) * 2).astype(np.float32).tolist())
        data = ex.SerializeToString()
        head = len(data).to_bytes(8, "little")
        recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
    path.write_bytes(b"".join(recs))


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    """200 training JPEGs of mixed sizes in three train-* shards (with KD logits) and 40 in one validation
    shard, written with the golden generator's protobuf runtime and CRC."""
    sys.path.insert(0, os.path.join(ROOT, "golden"))
    import make_eval_preprocess_golden as mk
    Example = mk.example_class()
    root = tmp_path_factory.mktemp("data")
    rng = np.random.default_rng(0)
    for sh, n in enumerate((70, 70, 60)):
        _write_shard(root / ("train-%05d-of-00003" % sh), Example, mk, rng, n, kd=True)
    _write_shard(root / "validation-00000-of-00001", Example, mk, rng, 40, kd=False)
    return root


# ------------------------------------------------------------------------------- steps from records
@pytest.mark.parametrize("dtype,mixup_type,kd_temp", [("bf16", 0, 0), ("fp32", 0, 0), ("bf16", 1, 0),
                                                      ("fp32", 1, 0), ("bf16", 0, 2.0)])
def test_steps_from_records_equal_oracle_images(shards, dtype, mixup_type, kd_temp):
    from assembled_cnn_b200 import imagenet_train as it
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer, _TrainFeed
    from oracle import train_preprocess as O
    p = params_from_flags(batch_size=8, dataset_name=DATASET, mixup_type=mixup_type, kd_temp=kd_temp,
                          dtype=dtype, label_smoothing=0.1, base_learning_rate=0.1)
    kd = kd_temp > 0
    records, counts = it.read_train_records(it.train_files(str(shards)), NUM_CLASSES, kd)
    trainers = []
    for _ in range(2):
        m = Model(50, num_classes=NUM_CLASSES, dtype=dtype, seed=3)
        trainers.append(Trainer(m, p, SIZE, SIZE, num_images=len(records)))
    feed_tr, oracle_tr = trainers
    feed = _TrainFeed(feed_tr, kd)
    ib = feed_tr.input_batch
    stream = it.CycleStream(counts, 5, 0, 2 if mixup_type == 1 else 1, 100, ib)
    batches = []
    for t in range(3):
        recs = stream.records(t)
        wins = [it.decode_window(*records[r][:3], 5, 0, pos) for pos, r in recs]
        labels = [records[r][3] for _, r in recs]
        teacher = np.stack([records[r][4] for _, r in recs]) if kd else None
        lam = it.mixup_lambdas(5, t, 0, ib // 2) if mixup_type else None
        batches.append((wins, labels, teacher, lam))
    feed.stage(*batches[0][:3])
    losses = [[], []]
    for t, (wins, labels, teacher, lam) in enumerate(batches):
        losses[0].append(feed.step(lam).tolist())
        if t + 1 < len(batches):
            feed.stage(*batches[t + 1][:3])
        x = np.stack([O.preprocess(a, f, SIZE) for a, f in wins])
        losses[1].append(oracle_tr.train_step(torch.from_numpy(x).pin_memory(), torch.tensor(labels, dtype=torch.int32),
                                              lam1=lam, teacher_logits=teacher).tolist())
    torch.cuda.synchronize()
    assert losses[0] == losses[1] and all(np.isfinite(l).all() for l in losses[0])
    wa, wb = feed_tr.model.get_weights(), oracle_tr.model.get_weights()
    assert all(torch.equal(wa[n], wb[n]) for n in wa)
    assert torch.equal(feed_tr.rt.momentum, oracle_tr.rt.momentum)
    # a host descriptor table is refused
    rt = feed_tr.rt
    host = feed.slots[0][2].cpu().pin_memory()
    assert rt.lib.acnn_set_images_cropped(rt.model.handle, host.data_ptr(), feed.mean.data_ptr(), rt.stream) == 1
    with pytest.raises(ValueError):
        rt.set_images_cropped(feed.slots[0][2][:32], feed.mean)


# ------------------------------------------------------------------------------- train_and_evaluate
FLAGS = dict(batch_size=32, dataset_name=DATASET, train_epochs=2, image_size=SIZE, seed=11, num_workers=4,
             dtype="bf16", label_smoothing=0.1, base_learning_rate=0.05, num_best_ckpt_to_keep=1,
             save_checkpoints_epochs=0.5, keep_checkpoint_max=3)


def _weights(path):
    with np.load(path) as z:
        return {n: z[n] for n in z.files}


def _evaluate_checkpoint(path, root):
    from assembled_cnn_b200.model_fns import build_model, evaluate_classification
    w = _weights(path)
    model = build_model(resnet_size=50, num_classes=NUM_CLASSES, dtype="bf16")
    model.set_weights({n: torch.as_tensor(v) for n, v in w.items() if not n.endswith("/Momentum")
                       and n != "global_step"})
    return evaluate_classification(model, str(root), image_size=SIZE, batch_size=32, label_smoothing=0.1,
                                   global_step=int(w["global_step"]), num_workers=4)


def test_train_and_evaluate_end_to_end(shards, tmp_path):
    from assembled_cnn_b200.model_fns import train_and_evaluate
    run = tmp_path / "run"
    res = train_and_evaluate(str(shards), str(run), **FLAGS)
    # 200 records, batch 32: 6 steps per cycle (the partial batch dropped), a checkpoint every 3 steps
    assert [r["global_step"] for r in res] == [6, 12]
    assert sorted(os.listdir(run)) == ["best", "model.ckpt-12.npz", "model.ckpt-6.npz", "model.ckpt-9.npz",
                                       "periodical"]
    assert sorted(os.listdir(run / "periodical")) == ["model.ckpt-12.npz", "model.ckpt-6.npz"]
    assert len([f for f in os.listdir(run / "best") if f.endswith(".npz")]) == 1
    for r in res:
        assert r == _evaluate_checkpoint(str(run / ("model.ckpt-%d.npz" % r["global_step"])), shards)
    final = _weights(str(run / "model.ckpt-12.npz"))
    # stopped after cycle 1 (stop_threshold 0: any accuracy reaches it), then resumed
    resumed = tmp_path / "resumed"
    first = train_and_evaluate(str(shards), str(resumed), stop_threshold=0.0, **FLAGS)
    assert first == res[:1]
    second = train_and_evaluate(str(shards), str(resumed), **FLAGS)
    assert second == res[1:]
    got = _weights(str(resumed / "model.ckpt-12.npz"))
    assert all(np.array_equal(got[n], final[n]) for n in final)
    # eager launches give the same run
    eager = tmp_path / "eager"
    assert train_and_evaluate(str(shards), str(eager), use_cuda_graph=False, **FLAGS) == res
    got = _weights(str(eager / "model.ckpt-12.npz"))
    assert all(np.array_equal(got[n], final[n]) for n in final)


def test_train_and_evaluate_warm_start_other_num_classes(shards, tmp_path):
    from assembled_cnn_b200.checkpoint import save_checkpoint
    from assembled_cnn_b200.model_fns import build_model, train_and_evaluate
    src = build_model(resnet_size=50, num_classes=1001, dtype="bf16", seed=99)
    src.runtime(2, SIZE, SIZE, training=False)
    path = save_checkpoint(str(tmp_path / "pre" / "model.ckpt-500"), src)
    # max_train_steps 0: the checkpoint of the cycle holds the warm-started variables themselves
    res = train_and_evaluate(str(shards), str(tmp_path / "run"), pretrained_model_checkpoint_path=path,
                             max_train_steps=0, **dict(FLAGS, train_epochs=1))
    assert [r["global_step"] for r in res] == [0]
    pre, got = _weights(path), _weights(str(tmp_path / "run" / "model.ckpt-0.npz"))
    assert got["resnet_model/dense/kernel"].shape == (2048, NUM_CLASSES)
    restored = [n for n in pre if "dense" not in n and not n.endswith(("moving_mean", "moving_variance"))]
    assert len(restored) > 100 and all(np.array_equal(pre[n], got[n]) for n in restored)
    # and training goes on from there
    res = train_and_evaluate(str(shards), str(tmp_path / "run2"), pretrained_model_checkpoint_path=path,
                             max_train_steps=2, **dict(FLAGS, train_epochs=1))
    assert [r["global_step"] for r in res] == [2]


def _two_gpu_worker(rank, port, root, model_dir, out):
    import torch.distributed as dist
    from assembled_cnn_b200.model_fns import train_and_evaluate
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device("cuda", rank))
    res = train_and_evaluate(root, model_dir, max_train_steps=2, **dict(FLAGS, train_epochs=1))
    torch.save(res, "%s.%d" % (out, rank))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_train_and_evaluate_two_gpus(shards, tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "res")
    mp.spawn(_two_gpu_worker, args=(port, str(shards), str(tmp_path / "run"), out), nprocs=2, join=True)
    r0, r1 = torch.load(out + ".0"), torch.load(out + ".1")
    assert r0 == r1 and [r["global_step"] for r in r0] == [2]
    assert os.path.exists(tmp_path / "run" / "model.ckpt-2.npz")
