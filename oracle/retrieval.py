"""Float64 CPU restatement of the reference's zero-shot retrieval evaluation (metric/recall_metric.py),
the yardstick of acnn_knn_topk and of the product's Recall@K bookkeeping.

  l2_normalize        tf.nn.l2_normalize(x, axis=1) (:99, :103): x * rsqrt(max(sum x^2, 1e-12))
  pairwise_distance   tf_simple_pairwise_distance (:207-215): (|q|^2 + |x|^2) - 2 q.x
  similarity          cosine = l2n(q) l2n(x)^T (:102-104); euclidean = -pairwise_distance (:105-106)
  top_k               tf.nn.top_k(sorted=True) (:110): values descending, and on equal values the lower
                      index first ("If two elements are equal, the lower-index element appears
                      first", tf.math.top_k documentation)
  get_recall          :217-228, statement for statement
"""
from __future__ import annotations

import numpy as np


def l2_normalize(x, eps=1e-12):
    x = np.asarray(x, dtype=np.float64)
    return x / np.sqrt(np.maximum((x * x).sum(axis=1, keepdims=True), eps))


def pairwise_distance(q, x):
    q = np.asarray(q, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    a = (q * q).sum(axis=1, keepdims=True)
    b = (x * x).sum(axis=1, keepdims=True).T
    return (a + b) - 2.0 * (q @ x.T)


def similarity(q, x, metric="cosine"):
    if metric == "cosine":
        return l2_normalize(q) @ l2_normalize(x).T
    if metric == "euclidean":
        return -pairwise_distance(q, x)
    raise NotImplementedError(metric)


def top_k(values, k):
    """(values, indices) [n][k] of every row: value descending, lower index first on ties."""
    values = np.asarray(values, dtype=np.float64)
    if k > values.shape[1]:
        raise ValueError("k=%d exceeds the row length %d" % (k, values.shape[1]))
    cols = np.broadcast_to(np.arange(values.shape[1]), values.shape)
    order = np.lexsort((cols, -values), axis=1)[:, :k]
    return np.take_along_axis(values, order, axis=1), order


def get_recall(sorted_idx, query_labels, labels, k_list=(1, 5)):
    """Recall@k of every k: query q's list drops the entries equal to q's POSITION among the queries
    (the reference's self-exclusion, which is self-exclusion only when no distractor comes before
    the query), then a hit is q's label among the first k labels that remain."""
    n = len(query_labels)
    count = {k: 0.0 for k in k_list}
    for qi, row in enumerate(sorted_idx):
        kept = [int(i) for i in row if int(i) != qi]
        got = [labels[i] for i in kept]
        for k in k_list:
            if query_labels[qi] in got[:k]:
                count[k] += 1.0
    return {k: v / n for k, v in count.items()}


def recall_at_k(embeddings, labels, k_list=(1, 5), metric="cosine"):
    """The whole evaluation of :150-161 on embeddings [N][d]: queries are the rows with label != -1,
    the index is every row."""
    labels = np.asarray(labels)
    feats = np.asarray(embeddings, dtype=np.float64)
    query = feats[labels != -1]
    _, idx = top_k(similarity(query, feats, metric), max(k_list) + 1)
    return get_recall(idx, labels[labels != -1], labels, k_list)
