#!/usr/bin/env python
"""Golden vectors of the zero-shot retrieval evaluation, produced by EXECUTING the reference's own
`get_recall` (metric/recall_metric.py:217-228) and its dataset table (functions/data_config.py) from a
checkout of the original project:

    python tests/golden/make_recall_golden.py REFERENCE_DIR      # rewrites recall_golden.json

Every case is a seeded set of integer-valued embeddings with labels (-1 = distractor).  The generator
ranks the index for every query in float64 (the reference's similarity formulas; ties by the lower
index, tf.nn.top_k's rule, through a stable sort) and records the resulting `sorted_idx` and the
recall the reference's `get_recall` computes from it.  tests/test_retrieval_cpu.py replays the oracle
and the product's recall bookkeeping on these data; it does not need the original project.
"""
import ast
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "recall_golden.json")
sys.path.insert(0, HERE)
import make_reference_shim_golden as mg  # noqa: E402  (reference_function: one function by its AST)

# name -> (rows, distractor layout, similarity, k_list, duplicated rows)
CASES = {
    "no_distractors_cosine": (120, "none", "cosine", [1, 5], 0),
    "distractors_after_euclidean": (160, "after", "euclidean", [1, 10, 100], 0),
    "distractors_interleaved_cosine": (140, "interleaved", "cosine", [1, 5], 0),
    "distractors_interleaved_euclidean": (160, "interleaved", "euclidean", [1, 10, 100], 0),
    "duplicate_rows_euclidean": (100, "none", "euclidean", [4], 30),
    "duplicate_rows_interleaved_cosine": (110, "interleaved", "cosine", [1, 5], 25),
}
NUM_CLASSES, DIM = 12, 8


def case_data(name):
    """(embeddings int [n][DIM], labels [n]) of a case, from its name's seed."""
    n, layout, _, _, dups = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    centers = rng.integers(-4, 5, (NUM_CLASSES, DIM))
    labels = rng.integers(0, NUM_CLASSES, n)
    emb = centers[labels] + rng.integers(-2, 3, (n, DIM))
    if layout == "after":
        labels[-n // 4:] = -1
    elif layout == "interleaved":
        labels[rng.choice(n, n // 5, replace=False)] = -1
    for dst in rng.choice(n, dups, replace=False):     # exact copies of other rows: exact ties
        emb[dst] = emb[rng.integers(0, n)]
    emb[(emb == 0).all(1), 0] = 1                       # no zero row (its cosine is undefined)
    return emb, labels


def sorted_idx_of(emb, labels, similarity, k):
    e = emb.astype(np.float64)
    q = e[labels != -1]
    if similarity == "cosine":
        qn = q / np.sqrt(np.maximum((q * q).sum(1, keepdims=True), 1e-12))
        en = e / np.sqrt(np.maximum((e * e).sum(1, keepdims=True), 1e-12))
        sim = qn @ en.T
    else:
        sim = -(((q * q).sum(1, keepdims=True) + (e * e).sum(1)[None, :]) - 2.0 * (q @ e.T))
    return np.argsort(-sim, axis=1, kind="stable")[:, :k]


def reference_datasets():
    """Every dataset functions/data_config.py:get_config knows: num_classes and image counts."""
    src = open(os.path.join(mg.REF_ROOT, "functions", "data_config.py")).read()
    ns = {}
    exec(compile(src, "functions/data_config.py", "exec"), ns)
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "get_config")
    names = [c.comparators[0].value for c in ast.walk(fn) if isinstance(c, ast.Compare)]
    out = {}
    for name in names:
        cfg = ns["get_config"](name)
        out[name] = {"num_classes": cfg.num_classes, "num_images": dict(cfg.num_images)}
    return out


def main():
    get_recall, _ = mg.reference_function("metric/recall_metric.py", "get_recall")
    gold = {"cases": {}, "datasets": reference_datasets()}
    for name, (_, _, similarity, k_list, _) in CASES.items():
        emb, labels = case_data(name)
        idx = sorted_idx_of(emb, labels, similarity, max(k_list) + 1)
        recall = get_recall(idx, labels[labels != -1], labels, list(k_list))
        gold["cases"][name] = {"similarity": similarity, "k_list": k_list,
                               "embeddings": emb.tolist(), "labels": labels.tolist(),
                               "sorted_idx": idx.tolist(),
                               "recall": {str(k): float(v) for k, v in recall.items()}}
        print(name, gold["cases"][name]["recall"])
    json.dump(gold, open(OUT, "w"), sort_keys=True, separators=(",", ":"))
    print("wrote", OUT)


if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isdir(os.path.join(sys.argv[1], "metric")):
        sys.exit("usage: python tests/golden/make_recall_golden.py REFERENCE_DIR\n"
                 "  REFERENCE_DIR: a checkout of clovaai/assembled-cnn (the directory holding metric/)")
    mg.REF_ROOT = os.path.abspath(sys.argv[1])
    main()
