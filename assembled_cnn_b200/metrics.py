"""Streaming evaluation metrics of the reference's EVAL mode (nets/run_loop_classification.py:
207-227): accuracy, top-5 accuracy (tf.metrics.accuracy / tf.metrics.mean(in_top_k)) and the
expected calibration error of metric/ece_metric.py:171-298 (10 confidence bins, per-bin running
sums).  They consume the logits the CUDA forward produced; a few tiny torch reductions per batch --
host-side bookkeeping, not part of the hot path."""
from __future__ import annotations

import torch


class EceMetric:
    """metric/ece_metric.py: accumulators accuracy_per_bin / confidence_per_bin / count_per_bin."""

    def __init__(self, num_thresholds=10, device="cpu"):
        eps = 1e-7
        th = [0.0 - eps] + [(i + 1) / num_thresholds for i in range(num_thresholds - 1)] + [1.0 + eps]
        self.eps = eps
        self.lo = torch.tensor(th[:num_thresholds], device=device).view(-1, 1)
        self.hi = torch.tensor(th[1:], device=device).view(-1, 1)
        self.correct = torch.zeros(num_thresholds, device=device)
        self.conf = torch.zeros(num_thresholds, device=device)
        self.cnt = torch.zeros(num_thresholds, device=device)

    def update(self, conf, pred, label):
        c = conf.float().view(1, -1)
        inb = (c > self.lo) & (c <= self.hi)
        ok = (pred.view(1, -1) == label.view(1, -1)) & inb
        self.correct += ok.float().sum(1)
        self.conf += (c * inb.float()).sum(1)
        self.cnt += inb.float().sum(1)
        return self.result()

    def result(self):
        acc = self.correct / (self.eps + self.cnt)
        avg = self.conf / (self.eps + self.cnt)
        return ((self.cnt / self.cnt.sum()) * (acc - avg).abs()).sum()


class EvalMetrics:
    """{'accuracy', 'accuracy_top_5', 'ece'} accumulated over the batches of an evaluation."""

    def __init__(self, device="cpu"):
        self.n = 0
        self.top1 = 0.0
        self.top5 = 0.0
        self.ece = EceMetric(device=device)

    def update(self, logits, labels):
        labels = labels.to(logits.device).long()
        prob = torch.softmax(logits.float(), dim=1)
        conf, pred = prob.max(dim=1)
        self.n += labels.numel()
        self.top1 += float((pred == labels).sum())
        self.top5 += float((logits.topk(5, dim=1).indices == labels[:, None]).any(1).sum())
        self.ece.update(conf, pred, labels)
        return self.result()

    def result(self):
        n = max(self.n, 1)
        return {"accuracy": self.top1 / n, "accuracy_top_5": self.top5 / n,
                "ece": float(self.ece.result())}


# --------------------------------------------------------------------------------------------------
# Zero-shot retrieval (metric/recall_metric.py:13-228)
# --------------------------------------------------------------------------------------------------
SIMILARITIES = {"cosine": 0, "euclidean": 1}
DTYPES = {"bf16": 0, "fp32": 1}


def knn_topk(query, index, k, similarity="cosine", dtype="bf16"):
    """acnn_knn_topk: for every row of `query` [nq, d] the k rows of `index` [nx, d] (CUDA tensors)
    with the largest similarity -- (indices int32 [nq, k], similarities fp32 [nq, k]) sorted by
    similarity descending, lower index first on ties (tf.nn.top_k's order).  'cosine' l2-normalises
    the rows, 'euclidean' is the negated squared distance; dtype 'bf16' runs bf16 operands, 'fp32'
    three bf16 planes per operand.  Enqueued on the current stream; no similarity matrix is stored."""
    from . import _lib
    lib = _lib.load()
    if similarity not in SIMILARITIES:
        raise NotImplementedError("eval_similarity must be one of %s" % sorted(SIMILARITIES))
    if dtype not in DTYPES:
        raise ValueError("dtype must be one of %s" % sorted(DTYPES))
    q = query.detach().to(torch.float32).contiguous()
    x = index.detach().to(torch.float32).contiguous()
    if q.dim() != 2 or x.dim() != 2 or q.shape[1] != x.shape[1]:
        raise ValueError("query [nq, d] and index [nx, d] must share d")
    if not (q.is_cuda and x.is_cuda and q.device == x.device):
        raise _lib.AcnnError("knn_topk runs on the GPU: query and index must be CUDA tensors on one device")
    (nq, d), nx = q.shape, x.shape[0]
    metric, dt = SIMILARITIES[similarity], DTYPES[dtype]
    nbytes = lib.acnn_knn_work_bytes(nq, nx, d, k, dt)
    if nbytes < 0:       # the library's argument check names the problem
        _lib.check(lib.acnn_knn_topk(None, None, nq, nx, d, k, metric, dt, None, None, None, 0, None),
                   "acnn_knn_topk")
    work = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    idx = torch.empty(nq, k, dtype=torch.int32, device=q.device)
    sim = torch.empty(nq, k, dtype=torch.float32, device=q.device)
    stream = torch.cuda.current_stream(q.device).cuda_stream
    _lib.check(lib.acnn_knn_topk(q.data_ptr(), x.data_ptr(), nq, nx, d, k, metric, dt, idx.data_ptr(),
                                 sim.data_ptr(), work.data_ptr(), nbytes, stream), "acnn_knn_topk")
    return idx, sim


def recall_from_sorted_idx(sorted_idx, query_labels, labels, k_list=(1, 5)):
    """get_recall (metric/recall_metric.py:217-228) as tensor ops on the device of `sorted_idx`:
    query q's list drops the entries equal to q's position among the queries, and a hit is q's label
    among the first k labels that remain.  Returns {k: recall} as Python floats."""
    sorted_idx = sorted_idx.long()
    labels = labels.to(sorted_idx.device).long()
    query_labels = query_labels.to(sorted_idx.device).long()
    n = sorted_idx.shape[0]
    keep = sorted_idx != torch.arange(n, device=sorted_idx.device)[:, None]
    rank = keep.long().cumsum(1) - 1                 # position among the entries that remain
    match = keep & (labels[sorted_idx] == query_labels[:, None])
    return {k: float(int((match & (rank < k)).any(1).sum())) / n for k in k_list}


class RecallAtK:
    """Streaming Recall@K of the reference's zero-shot evaluation (metric/recall_metric.py:150-161):
    `update(embeddings, labels)` appends a batch to device buffers; `result()` runs acnn_knn_topk with
    k = max(k_list) + 1 over queries = the rows whose label != -1 (distractors excluded) against the
    index = every row (distractors included), then get_recall's rules.

    As in the reference, query q drops the index entries equal to q's POSITION AMONG THE QUERIES, not
    to its own row: this is self-exclusion only when no distractor (label -1) comes before the query;
    otherwise the query's own row can remain (usually a hit) and an unrelated row is dropped.

    `update` copies its arguments: a model's forward returns views of its runtime's buffers, which the
    next batch overwrites (the reference copies every batch into np_features likewise).  `result`
    rejects non-finite embeddings, whose similarities cannot be ranked.

    Cost: the fused search is the faster path at small k (Recall@1/5, k = 6); at k = 101 (Recall@100)
    its per-row candidate merges make it slower than a chunked torch.mm + torch.topk (README)."""

    def __init__(self, k_list=(1, 5), similarity="cosine", dtype="bf16", device="cuda"):
        if similarity not in SIMILARITIES:
            raise NotImplementedError("eval_similarity must be one of %s" % sorted(SIMILARITIES))
        if dtype not in DTYPES:
            raise ValueError("dtype must be one of %s" % sorted(DTYPES))
        self.k_list = tuple(int(k) for k in k_list)
        self.similarity = similarity
        self.dtype = dtype
        self.device = torch.device(device)
        self.embeddings = []
        self.labels = []

    def update(self, embeddings, labels):
        self.embeddings.append(embeddings.detach().to(self.device, torch.float32, copy=True))
        self.labels.append(torch.as_tensor(labels).to(self.device, torch.int64, copy=True).flatten())

    @property
    def count(self):
        return sum(int(e.shape[0]) for e in self.embeddings)

    def result(self):
        feats = torch.cat(self.embeddings)
        labels = torch.cat(self.labels)
        if not bool(torch.isfinite(feats).all()):
            raise ValueError("RecallAtK: the embeddings contain NaN or infinite values")
        is_query = labels != -1
        idx, _ = knn_topk(feats[is_query], feats, max(self.k_list) + 1, self.similarity, self.dtype)
        if bool((idx >= feats.shape[0]).any()):
            # a row with fewer than k finite similarities (e.g. squared distances overflowing fp32)
            raise ValueError("RecallAtK: similarities are not finite; cannot rank the index")
        return recall_from_sorted_idx(idx, labels[is_query], labels, self.k_list)
