"""GPU checks of the servable's batch ladder (1, 8, 64, 256): on every rung and for every request size, in
bf16, fp16 and fp32, each image's classes, probabilities, probabilities_sigmoid and embedding are bit for
bit those of the single-rung servable and of model(x, False) over max_batch rows, through predict_images
(eager launches) and predict (one CUDA graph per (slot, valid rows)).  The model has SK blocks, whose
attention GEMMs would otherwise split K differently below 65 rows than at 256; a model without SK / SE
blocks gives the same bits at any batch.  New weights loaded into the model reach every rung."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZE = 64
LADDER = (1, 8, 64, 256)
REQUESTS = (1, 2, 8, 9, 63, 64, 65, 255, 256, 257, 300)


def _jpegs(n, seed=5):
    from PIL import Image
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        h, w = int(rng.integers(40, 120)), int(rng.integers(40, 120))
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        out.append(buf.getvalue())
    return out


def _same(got, want, rows, what):
    assert set(got) == set(want), what
    for k, v in got.items():
        assert v.tobytes() == want[k][rows].tobytes(), (what, k)


@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32"])
def test_ladder_bits_equal_single_rung_and_model(dtype):
    from assembled_cnn_b200.metrics import predict_rows
    from assembled_cnn_b200.model_fns import Servable, build_model
    model = build_model(resnet_size=50, resnet_version=2, use_sk_block=True, embedding_size=32, dtype=dtype,
                        seed=21)
    single = Servable(model, image_size=SIZE, max_batch=256)
    ladder = Servable(model, image_size=SIZE, max_batch=256, batch_sizes=LADDER)
    x = (torch.randn(max(REQUESTS), SIZE, SIZE, 3, generator=torch.Generator().manual_seed(3)) * 60)
    want = single.predict_images(x)
    assert want["embedding"].shape == (len(x), 32)
    # model(x, False) over the max_batch rows: the same logits, so the same outputs
    logits = model(x[:256], False).float().clone()
    emb = model(x[:256], False, return_embedding=True).float().cpu().numpy()
    ref = [t.cpu().numpy() for t in predict_rows(logits)]
    assert np.array_equal(want["classes"][:256], ref[0].astype(np.int64))
    assert want["probabilities"][:256].tobytes() == ref[1].tobytes()
    assert want["probabilities_sigmoid"][:256].tobytes() == ref[2].tobytes()
    assert want["embedding"][:256].tobytes() == emb.tobytes()
    # eager launches (predict_images), every request size, each rung
    for n in REQUESTS:
        _same(ladder.predict_images(x[:n]), want, slice(0, n), ("images", n))
    assert sorted(ladder._pipes) == list(LADDER)
    # CUDA graphs (predict on JPEGs): the first call of a rung runs eagerly, the repeats replay graphs
    jp = _jpegs(max(REQUESTS))
    want_j = single.predict(jp)
    for n in REQUESTS:
        for _ in range(2):
            _same(ladder.predict(jp[:n]), want_j, slice(0, n), ("jpeg", n))
    assert all(len(p.graphs) > 0 for p in ladder._pipes.values())


def test_rows_without_attention_blocks_do_not_depend_on_batch():
    """Vanilla ResNet-50: model(x, False) at batch 1 and 8 gives each row the bits of batch 256."""
    from assembled_cnn_b200.model_fns import build_model
    model = build_model(resnet_size=50, dtype="bf16", seed=22)
    x = torch.randn(256, SIZE, SIZE, 3, generator=torch.Generator().manual_seed(4)) * 60
    full = model(x, False).float().cpu().numpy()
    for n in (1, 8, 64):
        assert model(x[:n], False).float().cpu().numpy().tobytes() == full[:n].tobytes(), n


def test_new_weights_reach_every_rung():
    from assembled_cnn_b200.model_fns import Servable, build_model
    model = build_model(resnet_size=50, resnet_version=2, use_sk_block=True, dtype="bf16", seed=23)
    ladder = Servable(model, image_size=SIZE, max_batch=256, batch_sizes=LADDER)
    x = torch.randn(200, SIZE, SIZE, 3, generator=torch.Generator().manual_seed(5)) * 60
    sizes = (1, 5, 40, 200)                       # one request per rung
    before = [ladder.predict_images(x[:n]) for n in sizes]
    w = model.get_weights()
    g = torch.Generator().manual_seed(6)
    model.set_weights({k: v * (1 + 0.1 * torch.rand(v.shape, generator=g)) if v.dim() > 1 else v
                       for k, v in w.items()})
    ref = Servable(model, image_size=SIZE, max_batch=256).predict_images(x)
    for n, old in zip(sizes, before):
        new = ladder.predict_images(x[:n])
        assert new["probabilities"].tobytes() != old["probabilities"].tobytes(), n
        _same(new, ref, slice(0, n), ("new weights", n))
