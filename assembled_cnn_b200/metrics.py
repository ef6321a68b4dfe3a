"""Streaming evaluation metrics of the reference's EVAL mode (nets/run_loop_classification.py:
207-227): accuracy, top-5 accuracy (tf.metrics.accuracy / tf.metrics.mean(in_top_k)) and the
expected calibration error of metric/ece_metric.py:171-298 (10 confidence bins, per-bin running
sums).  They consume the logits the CUDA forward produced; a few tiny torch reductions per batch --
host-side bookkeeping, not part of the hot path."""
from __future__ import annotations

import numpy as np
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
DTYPES = {"bf16": 0, "fp32": 1, "fp16": 3}     # acnn.h ACNN_BF16 / ACNN_F32 / ACNN_F16
KNN_MAX_K = 128      # the largest k of acnn_knn_topk's per-row candidate lists (include/acnn.h)


def knn_topk(query, index, k, similarity="cosine", dtype="bf16"):
    """acnn_knn_topk: for every row of `query` [nq, d] the k rows of `index` [nx, d] (CUDA tensors)
    with the largest similarity -- (indices int32 [nq, k], similarities fp32 [nq, k]) sorted by
    similarity descending, lower index first on ties (tf.nn.top_k's order).  'cosine' l2-normalises
    the rows, 'euclidean' is the negated squared distance; dtype 'bf16' runs bf16 operands, 'fp32'
    three bf16 planes per operand, 'fp16' fp16 operands (the reference's fp16 search).  Enqueued on the current stream; no similarity matrix is stored."""
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
        return recall_of_index(torch.cat(self.embeddings), torch.cat(self.labels), self.k_list, self.similarity,
                               self.dtype)


def recall_of_index(feats, labels, k_list=(1, 5), similarity="cosine", dtype="bf16"):
    """RecallAtK's result for a whole index already on the device: feats fp32 [N, d], labels int64 [N]
    (-1: a distractor).  One acnn_knn_topk with k = max(k_list) + 1 over queries = the rows whose label
    != -1 against every row, then get_recall's rules.  Non-finite embeddings raise ValueError."""
    if not bool(torch.isfinite(feats).all()):
        raise ValueError("RecallAtK: the embeddings contain NaN or infinite values")
    is_query = labels != -1
    idx, _ = knn_topk(feats[is_query], feats, max(k_list) + 1, similarity, dtype)
    if bool((idx >= feats.shape[0]).any()):
        # a row with fewer than k finite similarities (e.g. squared distances overflowing fp32)
        raise ValueError("RecallAtK: similarities are not finite; cannot rank the index")
    return recall_from_sorted_idx(idx, labels[is_query], labels, k_list)


# --------------------------------------------------------------------------------------------------
# ImageNet-C corruption error (mce/eval_robustness.py)
# --------------------------------------------------------------------------------------------------
# AlexNet's top-1 error on each corruption, pooled over the five severities (Hendrycks & Dietterich,
# "Benchmarking Neural Network Robustness to Common Corruptions and Perturbations", ICLR 2019): the
# normaliser of CE.  The 15 ImageNet-C corruptions, then the four extra ones, in the order of
# ALEXNET_CE in mce/eval_robustness.py:91-97 -- the order the distortions are split over GPUs.
ALEXNET_CE = {
    "gaussian_noise": 0.8864, "shot_noise": 0.8945, "impulse_noise": 0.9226,
    "defocus_blur": 0.8199, "glass_blur": 0.8263, "motion_blur": 0.7860, "zoom_blur": 0.7984,
    "snow": 0.8668, "frost": 0.8266, "fog": 0.8193, "brightness": 0.5646,
    "contrast": 0.8532, "elastic_transform": 0.6461, "pixelate": 0.7178, "jpeg_compression": 0.6065,
    "speckle_noise": 0.8454, "gaussian_blur": 0.7871, "spatter": 0.7175, "saturate": 0.6583,
}
DISTORTIONS = tuple(ALEXNET_CE)


def softmax_top1_count(logits, labels, correct, n_valid=None, pred=None):
    """acnn_softmax_top1_count on the current stream: pred = the smallest index of the largest fp32
    softmax probability of every row r < n_valid of `logits` (CUDA fp32 [B, NC], rows may be strided, as
    a model's logits view is), -1 for a row with a non-finite logit; adds the rows with pred == labels[r]
    to `correct` (a CUDA int64 tensor of one element).  Rows >= n_valid are not touched.  `pred` (int32
    [B]) is allocated unless given; returns it."""
    from . import _lib
    lib = _lib.load()
    if logits.dim() != 2 or logits.dtype != torch.float32 or logits.stride(1) != 1:
        raise ValueError("logits must be a float32 [B, NC] tensor with unit column stride")
    B, NC = logits.shape
    n_valid = B if n_valid is None else int(n_valid)
    if not (logits.is_cuda and labels.is_cuda and correct.is_cuda):
        raise _lib.AcnnError("softmax_top1_count runs on the GPU: logits, labels and correct must be CUDA tensors")
    if labels.dtype != torch.int32 or labels.numel() < B or not labels.is_contiguous():
        raise ValueError("labels must be a contiguous int32 tensor of at least B = %d values" % B)
    if correct.dtype != torch.int64 or correct.numel() != 1:
        raise ValueError("correct must be an int64 tensor of one element")
    if pred is None:
        pred = torch.empty(B, dtype=torch.int32, device=logits.device)
    stream = torch.cuda.current_stream(logits.device).cuda_stream
    _lib.check(lib.acnn_softmax_top1_count(logits.data_ptr(), B, logits.stride(0), NC, labels.data_ptr(), n_valid,
                                           pred.data_ptr(), correct.data_ptr(), stream), "acnn_softmax_top1_count")
    return pred


def corruption_error_result(correct, count):
    """show_corruption_error (mce/eval_robustness.py:231-232,287-300) from the per-distortion counts
    {distortion: int}: error = 1 - correct / count (pooled over the severities), ce = error /
    ALEXNET_CE[d], mCE = mean of the 19 ce, mCE_unnormalized = mean of the 19 errors."""
    out = {}
    for d in DISTORTIONS:
        if d not in count or count[d] <= 0:
            # the reference asserts num_of_images > 0 for every distortion (:231)
            raise ValueError("corruption error: no images evaluated for distortion %r" % d)
        err = 1 - 1. * correct[d] / count[d]
        out[d] = {"error": err, "ce": err / ALEXNET_CE[d]}
    out["mCE"] = float(np.mean([out[d]["ce"] for d in DISTORTIONS]))
    out["mCE_unnormalized"] = float(np.mean([out[d]["error"] for d in DISTORTIONS]))
    return out


class CorruptionError:
    """Streaming corruption error of the reference's robustness evaluation (mce/eval_robustness.py,
    --robustness_type ce).  `update(logits, labels, distortion, n_valid=None)` counts the correct top-1
    predictions of a batch into a per-distortion device counter (acnn_softmax_top1_count: no host
    synchronisation); `add_counts` takes counts made elsewhere (a captured CUDA graph, another device);
    `result()` reads the counters once and returns {'<distortion>': {'error', 'ce'}, ..., 'mCE',
    'mCE_unnormalized'}.  It refuses a result while a distortion has no images."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self.correct = torch.zeros(len(DISTORTIONS), dtype=torch.int64, device=self.device)
        self.count = [0] * len(DISTORTIONS)

    @staticmethod
    def index(distortion):
        if distortion not in ALEXNET_CE:
            raise ValueError("unknown distortion %r (one of %s)" % (distortion, list(DISTORTIONS)))
        return DISTORTIONS.index(distortion)

    def update(self, logits, labels, distortion, n_valid=None):
        k = self.index(distortion)
        n = logits.shape[0] if n_valid is None else int(n_valid)
        labels = torch.as_tensor(labels).to(self.device, torch.int32).contiguous()
        softmax_top1_count(logits, labels, self.correct[k:k + 1], n)
        self.count[k] += n

    def add_counts(self, distortion, correct, count):
        k = self.index(distortion)
        self.correct[k] += int(correct)
        self.count[k] += int(count)

    def result(self):
        correct = self.correct.tolist()
        return corruption_error_result({d: correct[k] for k, d in enumerate(DISTORTIONS)},
                                       {d: self.count[k] for k, d in enumerate(DISTORTIONS)})


# --------------------------------------------------------------------------------------------------
# ImageNet classification evaluation (classifier.evaluate(input_fn_eval), nets/run_loop_classification.py)
# --------------------------------------------------------------------------------------------------
def classify_rows(logits, labels, n_valid=None, k=5, label_smoothing=0.0, out=None):
    """acnn_classify_rows on the current stream, for the rows r < n_valid of `logits` (CUDA fp32 [B, NC],
    rows may be strided, as a model's logits view is) and `labels` (CUDA int32): pred = tf.argmax,
    conf = the largest softmax probability, hit_k = tf.nn.in_top_k(k), ce = the label-smoothed softmax
    cross-entropy.  Rows >= n_valid are not written.  `out` (pred int32, conf fp32, hit_k int32, ce fp32,
    each of at least B) is allocated unless given; returns it."""
    from . import _lib
    lib = _lib.load()
    if logits.dim() != 2 or logits.dtype != torch.float32 or logits.stride(1) != 1:
        raise ValueError("logits must be a float32 [B, NC] tensor with unit column stride")
    B, NC = logits.shape
    n_valid = B if n_valid is None else int(n_valid)
    if not (logits.is_cuda and labels.is_cuda):
        raise _lib.AcnnError("classify_rows runs on the GPU: logits and labels must be CUDA tensors")
    if labels.dtype != torch.int32 or labels.numel() < B or not labels.is_contiguous():
        raise ValueError("labels must be a contiguous int32 tensor of at least B = %d values" % B)
    if out is None:
        out = tuple(torch.empty(B, dtype=dt, device=logits.device)
                    for dt in (torch.int32, torch.float32, torch.int32, torch.float32))
    for t, dt in zip(out, (torch.int32, torch.float32, torch.int32, torch.float32)):
        if t.dtype != dt or t.numel() < B or not t.is_contiguous() or t.device != logits.device:
            raise ValueError("out must be contiguous (int32, float32, int32, float32) tensors of at least B = %d "
                             "values on %s" % (B, logits.device))
    pred, conf, hit, ce = out
    stream = torch.cuda.current_stream(logits.device).cuda_stream
    _lib.check(lib.acnn_classify_rows(logits.data_ptr(), B, logits.stride(0), NC, labels.data_ptr(), n_valid, int(k),
                                      float(label_smoothing), pred.data_ptr(), conf.data_ptr(), hit.data_ptr(),
                                      ce.data_ptr(), stream), "acnn_classify_rows")
    return out


# The layout of struct acnn_train_metrics (include/acnn.h).
TRAIN_METRICS_DTYPE = np.dtype([("rows", "<i8"), ("top1", "<i8"), ("top5", "<i8"), ("bin_count", "<i8", 10),
                                ("bin_correct", "<i8", 10), ("bin_conf", "<f8", 10), ("step_rows", "<i8"),
                                ("step_conf", "<f8")])


def train_metrics_buffer(device):
    """A zeroed device accumulator for train_metrics_accumulate (uint8, TRAIN_METRICS_DTYPE's size)."""
    return torch.zeros(TRAIN_METRICS_DTYPE.itemsize, dtype=torch.uint8, device=device)


def train_metrics_accumulate(rows, labels, acc, n=None, step_begin=True):
    """acnn_train_metrics_accumulate on the current stream: adds the rows r < n (default: all) of classify_rows'
    (pred, conf, hit_k, ce) `rows` (k = 5) and the CUDA int32 `labels` to the accumulator `acc`
    (train_metrics_buffer); step_begin clears its per-step fields first."""
    from . import _lib
    lib = _lib.load()
    pred, conf, hit = rows[:3]
    n = pred.numel() if n is None else int(n)
    for t, dt in ((pred, torch.int32), (conf, torch.float32), (hit, torch.int32), (labels, torch.int32)):
        if t.dtype != dt or t.numel() < n or not t.is_contiguous() or not t.is_cuda:
            raise ValueError("pred, conf, hit_k and labels must be contiguous CUDA (int32, float32, int32, int32) "
                             "tensors of at least n = %d values" % n)
    if acc.dtype != torch.uint8 or acc.numel() != TRAIN_METRICS_DTYPE.itemsize or not acc.is_cuda:
        raise ValueError("acc must be a CUDA uint8 tensor of %d bytes (train_metrics_buffer)" % TRAIN_METRICS_DTYPE.itemsize)
    stream = torch.cuda.current_stream(acc.device).cuda_stream
    _lib.check(lib.acnn_train_metrics_accumulate(pred.data_ptr(), conf.data_ptr(), hit.data_ptr(), labels.data_ptr(),
                                                 n, int(bool(step_begin)), acc.data_ptr(), stream),
               "acnn_train_metrics_accumulate")


def train_metric_values(record, mixup=False):
    """The training summaries of an accumulator read back to the host (a TRAIN_METRICS_DTYPE record):
    sup/pred_prob = the step's mean confidence and, without mixup, train_accuracy, train_accuracy_top_5 and
    train_ece over the rows since the last reset (with mixup the labels are mixed and they are not defined)."""
    out = {"sup/pred_prob": float(record["step_conf"]) / max(int(record["step_rows"]), 1)}
    if not mixup:
        rows = max(int(record["rows"]), 1)
        out["train_accuracy"] = int(record["top1"]) / rows
        out["train_accuracy_top_5"] = int(record["top5"]) / rows
        out["train_ece"] = ece_from_bins(record["bin_count"], record["bin_correct"], record["bin_conf"])
    return out


def predict_rows(logits, n_valid=None, out=None):
    """acnn_predict_rows on the current stream, for the rows r < n_valid of `logits` (CUDA fp32 [B, NC], rows
    may be strided, as a model's logits view is): the PREDICT dict of nets/run_loop_classification.py:126-130,
    classes = tf.argmax (-1 for a row holding a NaN), probabilities = the softmax, probabilities_sigmoid =
    the sigmoid.  Rows >= n_valid are not written.  `out` (classes int32 [>= B], probabilities and
    probabilities_sigmoid fp32 [>= B, NC], contiguous) is allocated unless given; returns it."""
    from . import _lib
    lib = _lib.load()
    if logits.dim() != 2 or logits.dtype != torch.float32 or logits.stride(1) != 1:
        raise ValueError("logits must be a float32 [B, NC] tensor with unit column stride")
    B, NC = logits.shape
    n_valid = B if n_valid is None else int(n_valid)
    if not logits.is_cuda:
        raise _lib.AcnnError("predict_rows runs on the GPU: logits must be a CUDA tensor")
    if out is None:
        out = (torch.empty(B, dtype=torch.int32, device=logits.device),
               torch.empty(B, NC, dtype=torch.float32, device=logits.device),
               torch.empty(B, NC, dtype=torch.float32, device=logits.device))
    classes, prob, sig = out
    if classes.dtype != torch.int32 or classes.numel() < B or not classes.is_contiguous() \
            or classes.device != logits.device:
        raise ValueError("classes must be a contiguous int32 tensor of at least B = %d values on %s"
                         % (B, logits.device))
    for t in (prob, sig):
        if t.dtype != torch.float32 or t.dim() != 2 or t.shape[0] < B or t.shape[1] != NC \
                or not t.is_contiguous() or t.device != logits.device:
            raise ValueError("probabilities must be contiguous float32 [>= %d, %d] tensors on %s"
                             % (B, NC, logits.device))
    stream = torch.cuda.current_stream(logits.device).cuda_stream
    _lib.check(lib.acnn_predict_rows(logits.data_ptr(), B, logits.stride(0), NC, n_valid, classes.data_ptr(),
                                     prob.data_ptr(), sig.data_ptr(), stream), "acnn_predict_rows")
    return out


ECE_EPS = 1e-7


def ece_thresholds(num_thresholds=10):
    """The bin thresholds of metric/ece_metric.py as Python floats: [-1e-7, 1/n, ..., (n-1)/n, 1 + 1e-7]
    (the bins compare float32 confidences with their float32 roundings)."""
    return [0.0 - ECE_EPS] + [(i + 1) * 1.0 / num_thresholds for i in range(num_thresholds - 1)] + [1.0 + ECE_EPS]


def ece_from_bins(count, correct, conf_sum):
    """metric/ece_metric.py's ECE from per-bin counts, correct counts and confidence sums, in float64: acc and
    confidence per bin over (1e-7 + count), weighted by count / total.  With no row in any bin it is 0 / 0,
    NaN as in the reference."""
    cnt = np.asarray(count).astype(np.float64)
    acc = np.asarray(correct) / (ECE_EPS + cnt)
    avg = np.asarray(conf_sum, np.float64) / (ECE_EPS + cnt)
    with np.errstate(invalid="ignore"):
        return float((cnt / cnt.sum() * np.abs(acc - avg)).sum())


def classification_result(pred, conf, hit_k, ce, labels, batch_sizes, num_thresholds=10):
    """The eval metrics of nets/run_loop_classification.py:141-234 from the per-row results of a whole
    evaluation (numpy arrays, rows in evaluation order), in float64:
      accuracy        tf.metrics.accuracy(labels, argmax)
      accuracy_top_5  tf.metrics.mean(in_top_k(5))
      ece             metric/ece_metric.py:171-298: bins (lo, hi] over the float32 thresholds
                      [-1e-7, 0.1, ..., 0.9, 1 + 1e-7], acc and confidence per bin over (1e-7 + count),
                      weighted by count / total; a NaN confidence falls in no bin
      cross_entropy   the mean over batches of each batch's mean `ce` -- tf.metrics.mean of the per-batch
                      loss, unweighted, so a short last batch counts as one batch."""
    pred, labels = np.asarray(pred, np.int64), np.asarray(labels, np.int64)
    conf, ce = np.asarray(conf, np.float32), np.asarray(ce, np.float64)
    hit = np.asarray(hit_k).astype(bool)
    sizes = [int(b) for b in batch_sizes]
    n = len(labels)
    if not (len(pred) == len(conf) == len(hit) == len(ce) == n) or sum(sizes) != n or n == 0 or min(sizes) < 1:
        raise ValueError("classification_result: per-row arrays of one length, batch sizes summing to it")
    correct = pred == labels
    th = np.asarray(ece_thresholds(num_thresholds), np.float32)
    inb = (conf[None, :] > th[:-1, None]) & (conf[None, :] <= th[1:, None])
    ece = ece_from_bins(inb.sum(1), (inb & correct[None, :]).sum(1),
                        (np.where(inb, conf[None, :].astype(np.float64), 0.0)).sum(1))
    bounds = np.cumsum([0] + sizes)
    batch_ce = [ce[a:b].mean() for a, b in zip(bounds[:-1], bounds[1:])]
    return {"accuracy": float(correct.mean()), "accuracy_top_5": float(hit.mean()), "ece": ece,
            "cross_entropy": float(np.mean(batch_ce))}
