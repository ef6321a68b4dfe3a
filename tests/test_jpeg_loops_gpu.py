"""The input loops fed encoded JPEGs (the device decoder, PIL for what it does not decode) against the same loops
fed PIL-decoded pixels: training steps (_TrainFeed.stage_encoded vs stage: losses, weights and momentum, bit for
bit; bf16 / fp32, mixup type 1, KD), classification-evaluation rows (run_batch_encoded vs run_batch) and mCE
predictions and counts (run_batch_encoded vs run_batch), with progressive JPEGs mixed in for the PIL path."""
import io

import numpy as np
import pytest
import torch

from test_train_input_gpu import NUM_CLASSES, SIZE, DATASET, shards  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


def _progressive(rng, h, w):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(b, "JPEG", quality=85, progressive=True)
    return b.getvalue()


@pytest.mark.parametrize("dtype,mixup_type,kd_temp", [("bf16", 1, 0), ("fp32", 1, 0), ("bf16", 0, 2.0)])
def test_steps_from_encoded_records_equal_pil_windows(shards, dtype, mixup_type, kd_temp):  # noqa: F811
    from assembled_cnn_b200 import imagenet_train as it
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer, _TrainFeed
    p = params_from_flags(batch_size=8, dataset_name=DATASET, mixup_type=mixup_type, kd_temp=kd_temp,
                          dtype=dtype, label_smoothing=0.1, base_learning_rate=0.1)
    kd = kd_temp > 0
    records, counts = it.read_train_records(it.train_files(str(shards)), NUM_CLASSES, kd)
    trs = [Trainer(Model(50, num_classes=NUM_CLASSES, dtype=dtype, seed=3), p, SIZE, SIZE, num_images=len(records))
           for _ in range(2)]
    feeds = [_TrainFeed(tr, kd) for tr in trs]
    ib = trs[0].input_batch
    stream = it.CycleStream(counts, 5, 0, 2 if mixup_type == 1 else 1, 100, ib)
    losses = [[], []]
    for t in range(3):
        recs = stream.records(t)
        labels = [records[r][3] for _, r in recs]
        teacher = np.stack([records[r][4] for _, r in recs]) if kd else None
        lam = it.mixup_lambdas(5, t, 0, ib // 2) if mixup_type else None
        feeds[0].stage([it.decode_window(*records[r][:3], 5, 0, pos) for pos, r in recs], labels, teacher)
        feeds[1].stage_encoded([it.encoded_window(*records[r][:3], 5, 0, pos) for pos, r in recs], labels, teacher)
        for k in range(2):
            losses[k].append(feeds[k].step(lam).tolist())
    torch.cuda.synchronize()
    assert losses[0] == losses[1] and all(np.isfinite(l).all() for l in losses[0])
    wa, wb = trs[0].model.get_weights(), trs[1].model.get_weights()
    assert all(torch.equal(wa[n], wb[n]) for n in wa)
    assert torch.equal(trs[0].rt.momentum, trs[1].rt.momentum)


def test_classification_rows_from_encoded_equal_pil(shards):  # noqa: F811
    from assembled_cnn_b200 import imagenet_eval as E
    from assembled_cnn_b200.model_fns import Model, _ClassifyEvalDevice
    recs = [(str(shards / "validation-00000-of-00001"),) + r[1:3] + (r[0],)
            for r in E.read_records(str(shards / "validation-00000-of-00001"))][:16]
    bufs = [E.read_encoded(*r[:3]) for r in recs]
    bufs[5] = _progressive(np.random.default_rng(2), 90, 70)      # decoded by PIL on both paths
    labels = [r[3] for r in recs]
    model = Model(50, num_classes=NUM_CLASSES, dtype="bf16", seed=3)
    size, _ = E.eval_size("imagenet", SIZE)
    B = len(bufs)
    ev = _ClassifyEvalDevice(model, B, size, False, True, 0.1, 4 * B)
    geometry = lambda h, w: E.eval_geometry(h, w, "imagenet", SIZE)
    for _ in range(2):
        pil = []
        for b in bufs:
            a = E.decode_rgb(io.BytesIO(b))
            pil.append((a, geometry(*a.shape[:2])))
        ev.run_batch(pil, labels)
        ev.run_batch_encoded(bufs, labels, geometry)
    torch.cuda.synchronize()
    for rows in ev.rows:
        r = rows.cpu()
        assert torch.equal(r[:B], r[B:2 * B]) and torch.equal(r[:B], r[3 * B:])


def test_mce_from_encoded_files_equal_pil(tmp_path):
    from PIL import Image
    from assembled_cnn_b200 import imagenet_c
    from assembled_cnn_b200.model_fns import Model, _CorruptionEvalDevice
    rng = np.random.default_rng(4)
    files = []
    for i in range(12):
        a = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 40, (SIZE, SIZE, 3)), 0, 255).astype(np.uint8)
        f = tmp_path / ("img%d.JPEG" % i)
        Image.fromarray(a).save(f, "JPEG", quality=75 + i, progressive=(i == 7), subsampling=i % 3)
        files.append(str(f))
    labels = [int(v) for v in rng.integers(0, NUM_CLASSES, len(files))]
    model = Model(50, num_classes=NUM_CLASSES, dtype="bf16", seed=3)
    ev = _CorruptionEvalDevice(model, 16, SIZE, False, True)
    counts, preds = [], []
    for k in range(4):
        if k % 2 == 0:
            ev.run_batch([imagenet_c.decode_image(f, SIZE) for f in files], labels)
        else:
            ev.run_batch_encoded([open(f, "rb").read() for f in files], labels, files)
        preds.append(ev.pred[:len(files)].clone())
        counts.append(int(ev.take_count().item()))
    assert counts[0] == counts[1] == counts[2] == counts[3]
    assert all(torch.equal(preds[0], p) for p in preds[1:])
    # a file of the wrong size raises decode_image's error on the encoded path too
    bad = tmp_path / "small.JPEG"
    Image.fromarray(np.zeros((SIZE, SIZE + 8, 3), np.uint8)).save(bad, "JPEG")
    with pytest.raises(ValueError, match="expected"):
        ev.run_batch_encoded([bad.read_bytes()], [0], [str(bad)])
