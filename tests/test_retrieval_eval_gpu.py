"""GPU checks of the zero-shot retrieval evaluation over TFRecord shards: model_fns.evaluate_retrieval against
model_fns.recall_at_k fed the PIL-decoded, float32-restated eval batches (the index rows bit for bit and the
recalls exactly; bf16 / fp32, cosine / euclidean, embedding / pooled features / logits), graph replay
against eager launches, the float64 oracle's recall on the returned index, and
train_and_evaluate(zeroshot_eval=True) end to end (recall dicts, the keeper's ranking, stop_threshold)."""
import io
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.abspath(__file__))
NUM_CLASSES, SIZE, BATCH = 10, 64, 16


def _jpeg(rng):
    from PIL import Image
    h, w = int(rng.integers(20, 150)), int(rng.integers(20, 150))
    base = rng.integers(0, 256, 3)
    img = np.clip(base + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="JPEG", quality=90)
    return buf.getvalue()


def _write_shard(path, items):
    """items: (JPEG bytes, label or None: no image/class/label) per record."""
    sys.path.insert(0, os.path.join(ROOT, "golden"))
    import make_eval_preprocess_golden as mk
    Example = mk.example_class()
    recs = []
    for jpeg, label in items:
        ex = Example()
        ex.features.feature["image/encoded"].bytes_list.value.append(jpeg)
        if label is not None:
            ex.features.feature["image/class/label"].int64_list.value.append(label)
        data = ex.SerializeToString()
        head = len(data).to_bytes(8, "little")
        recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
    path.write_bytes(b"".join(recs))


def _retrieval_items(rng):
    """45 records: 8 classes of three copies of one image (labels 100, 107, ... beyond num_classes), 10
    singletons (labels 3 and 2^40 among them) and 11 distractors, shuffled, then the first distractor moved
    to the front; with batches of 16 the last batch has 13 rows."""
    items = [(jpeg, 100 + 7 * c) for c, jpeg in enumerate([_jpeg(rng) for _ in range(8)]) for _ in range(3)]
    items += [(_jpeg(rng), lab) for lab in (3, 1 << 40, 5, 200, 201, 202, 203, 204, 205, 206)]
    items += [(_jpeg(rng), None) for _ in range(11)]
    order = rng.permutation(len(items))
    items = [items[i] for i in order]
    first = next(i for i, (_, lab) in enumerate(items) if lab is None)
    items[0], items[first] = items[first], items[0]
    return items


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    """{'front': the records with a distractor first, so that every query keeps its own row in its list (the
    reference's position rule), 'tail': the same records with every distractor after the last query (a
    query drops its own row; singletons miss)}: (directory, labels)."""
    items = _retrieval_items(np.random.default_rng(0))
    out = {}
    for name, recs in (("front", items), ("tail", [it for it in items if it[1] is not None]
                                          + [it for it in items if it[1] is None])):
        root = tmp_path_factory.mktemp(name)
        _write_shard(root / "validation-00000-of-00002", recs[:20])
        _write_shard(root / "validation-00001-of-00002", recs[20:])
        (root / "train-00000-of-00001").write_bytes(b"not a record")       # the glob skips it
        out[name] = root, [-1 if lab is None else lab for _, lab in recs]
    return out


def _pil_batches(root, ptype="imagenet"):
    """The evaluation's batches through the host path: PIL decode, the float32 restatement of the resize."""
    from assembled_cnn_b200 import imagenet_eval as ie
    from oracle import eval_preprocess as O
    recs = [(f, off, n, lab) for f in ie.validation_files(str(root))
            for lab, off, n in ie.read_records(f, missing_label=-1)]
    out = []
    for a in range(0, len(recs), BATCH):
        chunk = recs[a:a + BATCH]
        x = np.stack([O.preprocess(ie.decode_record(f, off, n, ptype, SIZE)[0], ptype, SIZE)
                      for f, off, n, _ in chunk])
        out.append((torch.from_numpy(x), torch.tensor([r[3] for r in chunk], dtype=torch.int64)))
    return out


def _index(model, root, return_embedding, use_cuda_graph=True):
    from assembled_cnn_b200 import imagenet_eval as ie
    from assembled_cnn_b200.model_fns import _retrieval_index
    recs = [(f, off, n, lab) for f in ie.validation_files(str(root))
            for lab, off, n in ie.read_records(f, missing_label=-1)]
    return _retrieval_index(model, recs, SIZE, BATCH, "imagenet", SIZE, return_embedding, False, use_cuda_graph, 4)


CASES = [("bf16", 32, True), ("bf16", 0, True), ("bf16", 32, False), ("fp32", 32, True), ("fp32", 0, False)]


@pytest.mark.parametrize("dtype,embedding_size,return_embedding", CASES)
def test_evaluate_retrieval_equals_recall_at_k_on_pil_batches(shards, dtype, embedding_size, return_embedding):
    from assembled_cnn_b200.model_fns import build_model
    model = build_model(resnet_size=50, num_classes=NUM_CLASSES, embedding_size=embedding_size, dtype=dtype)
    for root, labels in shards.values():
        _check_against_recall_at_k(model, root, labels, return_embedding)
    assert shards["front"][1][0] == -1 and shards["tail"][1][-11:] == [-1] * 11


def _check_against_recall_at_k(model, root, labels, return_embedding):
    from assembled_cnn_b200.model_fns import evaluate_retrieval, recall_at_k
    embedding_size = model.cfg_kwargs["embedding_size"]
    batches = _pil_batches(root)
    assert [len(y) for _, y in batches] == [16, 16, 13]
    # the index rows equal the host path's outputs bit for bit, graph replay or eager
    want = torch.cat([model(x, False, return_embedding=return_embedding).float().clone() for x, _ in batches])
    assert want.shape[1] == ((embedding_size or 2048) if return_embedding else NUM_CLASSES)
    for graph in (True, False):
        index, lab = _index(model, root, return_embedding, graph)
        assert torch.equal(index, want) and lab.tolist() == labels
    kw = dict(image_size=SIZE, batch_size=BATCH, return_embedding=return_embedding, num_workers=4)
    for similarity in ("cosine", "euclidean"):
        ref = recall_at_k(model, batches, len(labels), (1, 2, 5), similarity, return_embedding=return_embedding,
                          global_step=9)
        got = evaluate_retrieval(model, str(root), recall_at_k=(1, 2, 5), eval_similarity=similarity,
                                 global_step=9, **kw)
        assert got == ref and set(got) == {"recall_at_1", "recall_at_2", "recall_at_5", "global_step"}
        eager = evaluate_retrieval(model, str(root), recall_at_k=(1, 2, 5), eval_similarity=similarity,
                                   use_cuda_graph=False, **kw)
        assert eager == dict(got, global_step=None)


@pytest.mark.parametrize("similarity", ["cosine", "euclidean"])
def test_oracle_recall_on_the_returned_index(shards, similarity):
    """fp32 model (three-plane search): the float64 ranking of the index equals the device's."""
    from oracle import retrieval as R
    from assembled_cnn_b200.model_fns import build_model, evaluate_retrieval
    root, labels = shards["tail"]
    model = build_model(resnet_size=50, num_classes=NUM_CLASSES, embedding_size=32, dtype="fp32")
    index, lab = _index(model, root, True)
    want = R.recall_at_k(index.double().cpu().numpy(), lab.cpu().numpy(), (1, 5), similarity)
    got = evaluate_retrieval(model, str(root), image_size=SIZE, batch_size=BATCH, eval_similarity=similarity,
                             num_workers=4)
    assert got == {"recall_at_1": want[1], "recall_at_5": want[5], "global_step": None}
    assert lab.tolist() == labels
    assert 0 < want[1] < 1 and want[5] < 1      # the copies are found, the singletons are not


# ------------------------------------------------------------------------------- train_and_evaluate
DATASET = "cub_200_2011"            # 100 training classes; the test classes lie outside [0, 100)
FLAGS = dict(batch_size=16, dataset_name=DATASET, train_epochs=2, image_size=SIZE, seed=3, num_workers=4,
             dtype="bf16", embedding_size=32, base_learning_rate=0.05, num_best_ckpt_to_keep=2,
             val_batch_size=BATCH, zeroshot_eval=True, recall_at_k=[1, 5])


@pytest.fixture(scope="module")
def train_root(shards, tmp_path_factory):
    """The 'tail' retrieval shards plus 40 training records with labels in [0, 100)."""
    import shutil
    root = tmp_path_factory.mktemp("zeroshot")
    for f in ("validation-00000-of-00002", "validation-00001-of-00002"):
        shutil.copy(shards["tail"][0] / f, root / f)
    rng = np.random.default_rng(1)
    _write_shard(root / "train-00000-of-00001", [(_jpeg(rng), int(rng.integers(0, 100))) for _ in range(40)])
    return root


def test_train_and_evaluate_zeroshot(train_root, tmp_path):
    from assembled_cnn_b200.model_fns import build_model, evaluate_retrieval, train_and_evaluate
    run = tmp_path / "run"
    res = train_and_evaluate(str(train_root), str(run), **FLAGS)
    # 40 records, batch 16: 2 steps per cycle
    assert [r["global_step"] for r in res] == [2, 4]
    assert all(set(r) == {"recall_at_1", "recall_at_5", "global_step"} for r in res)
    best = json.loads((run / "best" / "best_checkpoints").read_text())
    assert best == {"model.ckpt-%d" % r["global_step"]: r["recall_at_1"] for r in res}
    # each result is the evaluation of its cycle's checkpoint
    for r in res:
        with np.load(run / ("model.ckpt-%d.npz" % r["global_step"])) as z:
            w = {n: torch.as_tensor(z[n]) for n in z.files if not n.endswith("/Momentum") and n != "global_step"}
        model = build_model(resnet_size=50, num_classes=100, embedding_size=32, dtype="bf16")
        model.set_weights(w)
        assert r == evaluate_retrieval(model, str(train_root), image_size=SIZE, batch_size=BATCH,
                                       global_step=r["global_step"], num_workers=4)
    # stop_threshold compares recall_at_1: 0 stops after the first cycle
    first = train_and_evaluate(str(train_root), str(tmp_path / "stopped"), stop_threshold=0.0, **FLAGS)
    assert first == res[:1]
