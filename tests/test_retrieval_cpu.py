"""CPU checks of the zero-shot retrieval evaluation (metric/recall_metric.py): the float64 oracle and the
product's post-top-k Recall@K bookkeeping against golden values of the reference's own `get_recall`
(tests/golden/make_recall_golden.py), the argument checks of acnn_knn_topk without a GPU, the SASS of
the fused kernel, and the new flags / dataset table against the reference."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "recall_golden.json")))
SHIM = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_shim_golden.json")))
CASES = sorted(GOLD["cases"])


def _case(name):
    c = GOLD["cases"][name]
    labels = np.array(c["labels"])
    return c, np.array(c["embeddings"]), labels, np.array(c["sorted_idx"]), labels[labels != -1]


def test_golden_covers_the_required_cases():
    k_lists = {tuple(GOLD["cases"][n]["k_list"]) for n in CASES}
    assert {(1, 5), (1, 10, 100), (4,)} <= k_lists
    layouts = set()
    for n in CASES:
        _, emb, labels, _, _ = _case(n)
        d = np.flatnonzero(labels == -1)
        q = np.flatnonzero(labels != -1)
        layouts.add("none" if d.size == 0 else ("after" if d.min() > q.max() else "interleaved"))
        if len({tuple(r) for r in emb.tolist()}) < len(emb):
            layouts.add("duplicates")
    assert layouts == {"none", "after", "interleaved", "duplicates"}


@pytest.mark.parametrize("name", CASES)
def test_oracle_get_recall_matches_reference(name):
    from oracle import retrieval as R
    c, _, labels, idx, qlab = _case(name)
    got = R.get_recall(idx, qlab, labels, c["k_list"])
    assert {str(k): v for k, v in got.items()} == c["recall"]


@pytest.mark.parametrize("name", CASES)
def test_product_recall_bookkeeping_matches_reference(name):
    """metrics.recall_from_sorted_idx -- what RecallAtK applies to the kernel's top-k on the GPU --
    run on CPU tensors reproduces the reference's numbers exactly."""
    from assembled_cnn_b200.metrics import recall_from_sorted_idx
    c, _, labels, idx, qlab = _case(name)
    got = recall_from_sorted_idx(torch.from_numpy(idx), torch.from_numpy(qlab), torch.from_numpy(labels),
                                 c["k_list"])
    assert {str(k): v for k, v in got.items()} == c["recall"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_top_k_order_matches_reference_ranking(name):
    """The oracle's similarity + top_k (value desc, lower index first) give the golden ranking,
    including the exact ties of duplicated rows."""
    from oracle import retrieval as R
    c, emb, labels, idx, _ = _case(name)
    sim = R.similarity(emb[labels != -1], emb, c["similarity"])
    vals, got = R.top_k(sim, idx.shape[1])
    assert (got == idx).all()
    assert (np.diff(vals, axis=1) <= 0).all()
    assert R.recall_at_k(emb, labels, c["k_list"], c["similarity"]) == \
        {int(k): v for k, v in c["recall"].items()}


def test_interleaved_distractors_exercise_the_position_quirk():
    """With a distractor before a query, dropping the query's position among the queries differs
    from dropping its own row; the golden recall is the former."""
    from oracle import retrieval as R
    differs = 0
    for name in CASES:
        c, _, labels, idx, qlab = _case(name)
        rows = np.flatnonzero(labels != -1)
        self_excluded = [[i for i in r if i != rows[q]] for q, r in enumerate(idx)]
        alt = {str(k): sum(qlab[q] in [labels[i] for i in r[:k]] for q, r in enumerate(self_excluded))
               / len(qlab) for k in c["k_list"]}
        differs += alt != c["recall"]
        if (labels == -1).sum() == 0 or np.flatnonzero(labels == -1).min() > rows.max():
            assert alt == c["recall"], name
    assert differs >= 2


def test_knn_argument_errors_without_gpu():
    """Every argument check of acnn_knn_topk runs on the host before any CUDA call."""
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    OK, INVALID, UNSUPPORTED = 0, 1, 3

    def call(nq=10, nx=20, d=16, k=5, metric=0, dtype=0, work=True, nbytes=1 << 30):
        dummy = 1 << 20 if work else None     # never dereferenced: the checks fail first
        return lib.acnn_knn_topk(dummy, dummy, nq, nx, d, k, metric, dtype, dummy, dummy,
                                 dummy if work else None, nbytes, None)

    assert call(k=129) == UNSUPPORTED and call(k=1000, nx=5000) == UNSUPPORTED
    assert call(k=21) == INVALID                       # k > nx (tf.nn.top_k fails too)
    for kw in (dict(nq=0), dict(nx=0), dict(d=0), dict(k=0), dict(nq=-3), dict(metric=2),
               dict(metric=-1), dict(dtype=2), dict(work=False), dict(nbytes=100)):
        assert call(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    assert lib.acnn_knn_work_bytes(10, 20, 16, 5, 0) > 0
    assert lib.acnn_knn_work_bytes(10, 20, 16, 129, 0) == -1
    assert lib.acnn_knn_work_bytes(0, 20, 16, 5, 0) == -1
    # the documented layout: Q', X' (K' = P * roundup(d, 64)), two norm vectors, 8 partial lists
    a = lambda b: (b + 255) // 256 * 256
    for nq, nx, d, k, dtype in ((1, 1, 1, 1, 0), (127, 129, 100, 101, 1), (5924, 5924, 512, 6, 0),
                                (60502, 60502, 2048, 128, 1)):
        kp = (6 if dtype else 1) * ((d + 63) // 64 * 64)
        total = a(a(a(a(a(nq * kp * 2) + nx * kp * 2) + nq * 4) + nx * 4) + 8 * nq * k * 4) + 8 * nq * k * 4
        assert lib.acnn_knn_work_bytes(nq, nx, d, k, dtype) == a(total)
    prev = lib.acnn_set_knn_splits(3)
    assert lib.acnn_set_knn_splits(prev) == 3


def test_knn_without_cuda_tensors_raises():
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.metrics import knn_topk
    with pytest.raises((_lib.AcnnError, ValueError)):
        knn_topk(torch.zeros(4, 8), torch.zeros(6, 8), 2)
    with pytest.raises(NotImplementedError):
        knn_topk(torch.zeros(4, 8), torch.zeros(6, 8), 2, similarity="dot")


def test_knn_sass_uses_wgmma_and_tma():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", os.path.join(ROOT, "assembled_cnn_b200", "build", "knn.o")],
                          capture_output=True, text=True).stdout
    assert "HGMMA" in sass and "UTMALDG" in sass


def test_retrieval_flags_and_datasets_match_reference():
    from assembled_cnn_b200.hparams import DATASETS, DEFAULTS
    ref = SHIM["train_pieces"]["flag_defaults"]
    for k in ("zeroshot_eval", "eval_similarity", "recall_at_k", "return_embedding", "val_batch_size"):
        assert DEFAULTS[k] == ref[k]["default"], k
    assert DATASETS == GOLD["datasets"]
    assert DATASETS["SOP"]["num_images"]["validation"] == 60502


def test_recall_update_copies_its_inputs():
    """A model's forward returns views of its runtime's buffers, rewritten by the next batch:
    RecallAtK keeps copies, as the reference copies every batch into np_features."""
    from assembled_cnn_b200.metrics import RecallAtK
    metric = RecallAtK((1,), device="cpu")
    buf, lab = torch.zeros(4, 8), torch.arange(4)
    for step in range(3):
        buf.fill_(step)
        lab.fill_(step)
        metric.update(buf, lab)
    assert [float(e[0, 0]) for e in metric.embeddings] == [0.0, 1.0, 2.0]
    assert [int(y[0]) for y in metric.labels] == [0, 1, 2]
    assert all(e.data_ptr() != buf.data_ptr() for e in metric.embeddings)
    assert metric.count == 12


def test_recall_rejects_non_finite_embeddings():
    from assembled_cnn_b200.metrics import RecallAtK
    for bad in (float("nan"), float("inf")):
        metric = RecallAtK((1,), device="cpu")
        e = torch.randn(6, 8)
        e[2, 3] = bad
        metric.update(e, torch.arange(6))
        with pytest.raises(ValueError):
            metric.result()
