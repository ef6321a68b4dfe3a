"""acnn_knn_topk (the fused wgmma similarity + top-k of the zero-shot retrieval evaluation) on the GPU:
against a float64 recomputation on the operands the kernel really used (read back from its work
buffer) with an element-wise rounding bound, exact indices on integer data with planted ties,
bit-identical results across column splits / CUDA-graph replay / concurrent streams, RecallAtK and
model_fns.recall_at_k on a small embedding model, and one Stanford-Online-Products-size search."""
import itertools

import numpy as np
import pytest
import torch

from assembled_cnn_b200 import _lib
from assembled_cnn_b200.metrics import DTYPES, RecallAtK, knn_topk

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -23       # fp32 unit roundoff, doubled: the tensor core truncates its addends
SPLITS_MAX = 8


def _a(b):
    return (b + 255) // 256 * 256


def _operands(work, nq, nx, d, k, dtype):
    """The rounded operands (float64, first d columns) and the fp32 squared norms the kernel used,
    from the work layout documented in include/acnn.h."""
    dp = (d + 63) // 64 * 64
    kp = (6 if dtype == "fp32" else 1) * dp
    oq, ox = 0, _a(nq * kp * 2)
    oqn = _a(ox + nx * kp * 2)
    oxn = _a(oqn + nq * 4)
    Q = work[oq:oq + nq * kp * 2].view(torch.bfloat16).view(nq, kp)
    X = work[ox:ox + nx * kp * 2].view(torch.bfloat16).view(nx, kp)
    if dtype == "fp32":      # Q' = (hi, mid, lo, ...), X' = (lo, mid, hi, ...)
        seg = lambda t, s: t[:, s * dp:s * dp + d].float()
        qr = (seg(Q, 0) + seg(Q, 1)) + seg(Q, 2)
        xr = (seg(X, 2) + seg(X, 1)) + seg(X, 0)
    else:
        qr, xr = Q[:, :d].float(), X[:, :d].float()
    qn = work[oqn:oqn + nq * 4].view(torch.float32)
    xn = work[oxn:oxn + nx * 4].view(torch.float32)
    return qr.double(), xr.double(), qn, xn, kp, Q, X


def _check_prep(q, x, work, k, metric, dtype):
    """The prep kernel's output against the inputs, independently of the kernel's arithmetic:
    cosine rows within bf16 (or 24-bit) rounding plus the fp32 normalisation error of the float64
    tf.nn.l2_normalize, euclidean rows exactly bf16(x) (or x itself from the three planes); zero
    padding; in the fp32 mode every segment in its place with the hi / mid / lo split of its row;
    the squared norms within fp32 summation error of the rounded rows'."""
    from oracle import retrieval as R
    (nq, d), nx = q.shape, x.shape[0]
    dp = (d + 63) // 64 * 64
    qr, xr, qn, xn, _, Q, X = _operands(work, nq, nx, d, k, dtype)
    for src, r, mat, nrm, pattern in ((q, qr, Q, qn, (0, 1, 2, 0, 1, 0)), (x, xr, X, xn, (2, 1, 0, 1, 0, 0))):
        s64 = src.double()
        if metric == "euclidean":
            assert torch.equal(r, s64 if dtype == "fp32" else src.bfloat16().double())
        else:
            ref = torch.from_numpy(R.l2_normalize(s64.cpu().numpy())).to(DEV)
            # unit roundoff of the stored value: 2^-8 for bf16 (8 significant bits), 2^-24 for the
            # 24 bits of three planes; plus the fp32 sum of squares and rsqrtf (2 ulp)
            eps = (d / 32 + 16) * 2.0 ** -24 + (2.0 ** -23 if dtype == "fp32" else 2.0 ** -8)
            err = (r - ref).abs() - eps * ref.abs()
            assert (err <= 0).all(), float(err.max())
        segs = [mat[:, i * dp:(i + 1) * dp] for i in range(mat.shape[1] // dp)]
        for sg in segs:
            assert not sg[:, d:].float().any()
        if dtype == "fp32":          # pattern: which of (hi, mid, lo) each segment holds
            v = r.float()
            hi = v.bfloat16()
            mid = (v - hi.float()).bfloat16()
            lo = (v - hi.float() - mid.float()).bfloat16()
            for sg, which in zip(segs, pattern):
                assert torch.equal(sg[:, :d], (hi, mid, lo)[which])
        ref_n = (r * r).sum(1)
        assert ((nrm.double() - ref_n).abs() <= (dp / 32 + 8) * 2.0 ** -23 * ref_n).all()


def _run(q, x, k, metric="cosine", dtype="bf16", splits=0):
    """knn_topk with a forced split count, returning the work buffer too."""
    lib = _lib.load()
    prev = lib.acnn_set_knn_splits(splits)
    try:
        nq, d = q.shape
        nbytes = lib.acnn_knn_work_bytes(nq, x.shape[0], d, k, DTYPES[dtype])
        work = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        idx = torch.empty(nq, k, dtype=torch.int32, device=DEV)
        sim = torch.empty(nq, k, dtype=torch.float32, device=DEV)
        _lib.check(lib.acnn_knn_topk(q.data_ptr(), x.data_ptr(), nq, x.shape[0], d, k,
                                     0 if metric == "cosine" else 1, DTYPES[dtype], idx.data_ptr(),
                                     sim.data_ptr(), work.data_ptr(), nbytes,
                                     torch.cuda.current_stream().cuda_stream), "acnn_knn_topk")
    finally:
        lib.acnn_set_knn_splits(prev)
    return idx, sim, work


def _check(qr, xr, idx, sim, metric, kp, rows=None):
    """Valid distinct indices in the total order; every returned similarity within the rounding
    bound of its float64 value; no omitted index beats the k-th returned one by more than the
    bounds of both."""
    if rows is not None:
        qr = qr[rows]
    nx, k = xr.shape[0], idx.shape[1]
    i = idx.long()
    assert ((i >= 0) & (i < nx)).all()
    assert (i.sort(1).values.diff(1) > 0).all(), "duplicate index"
    ds, di = sim.diff(1), i.diff(1)
    assert ((ds < 0) | ((ds == 0) & (di > 0))).all(), "not in (similarity desc, index asc) order"
    dot = qr @ xr.T
    adot = qr.abs() @ xr.abs().T
    bound = (kp + 16) * U * adot
    if metric == "cosine":
        s64 = dot
    else:
        a = (qr * qr).sum(1, keepdim=True)
        b = (xr * xr).sum(1)[None, :]
        s64 = -((a + b) - 2 * dot)
        bound = 2 * bound + (kp + 16) * U * (a + b) + 2 * U * (a + b + 2 * adot)
    got = s64.gather(1, i)
    eb = bound.gather(1, i)
    err = (sim.double() - got).abs()
    assert (err <= eb).all(), float((err - eb).max())
    kth = got[:, -1:] + eb[:, -1:]
    omitted = torch.ones_like(s64, dtype=torch.bool).scatter_(1, i, False)
    beat = omitted & (s64 > kth + bound)
    assert not beat.any(), int(beat.sum())


def _shape_cases():
    sizes, dims, ks = (1, 127, 129, 1000, 5924), (32, 100, 512, 2048), (1, 6, 64, 101, 128)
    out = []
    for m, (metric, dtype) in enumerate(itertools.product(("cosine", "euclidean"), ("bf16", "fp32"))):
        for n, (nq, nx) in enumerate(itertools.product(sizes, sizes)):
            fits = [kk for kk in ks if kk <= nx]          # k <= nx; every k in turn where all fit
            k = fits[(n + m) % len(fits)] if len(fits) < len(ks) else ks[(n // 5 + n + m) % 5]
            out.append((nq, nx, dims[(n + m) % 4], k, metric, dtype))
    return out


@pytest.mark.parametrize("nq,nx,d,k,metric,dtype", _shape_cases())
def test_knn_matches_float64_on_rounded_operands(nq, nx, d, k, metric, dtype):
    g = torch.Generator(device=DEV).manual_seed(nq * 7919 + nx * 31 + d + k)
    q = torch.randn(nq, d, device=DEV, generator=g)
    x = torch.randn(nx, d, device=DEV, generator=g)
    idx, sim, work = _run(q, x, k, metric, dtype)
    _check_prep(q, x, work, k, metric, dtype)
    qr, xr, _, _, kp, _, _ = _operands(work, nq, nx, d, k, dtype)
    _check(qr, xr, idx, sim, metric, kp)


def test_shape_cases_cover_every_value():
    cases = _shape_cases()
    for pos, values in ((0, (1, 127, 129, 1000, 5924)), (1, (1, 127, 129, 1000, 5924)),
                        (2, (32, 100, 512, 2048)), (3, (1, 6, 64, 101, 128))):
        for md in itertools.product(("cosine", "euclidean"), ("bf16", "fp32")):
            got = {c[pos] for c in cases if (c[4], c[5]) == md}
            assert set(values) <= got, (pos, md, set(values) - got)


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
@pytest.mark.parametrize("k", [6, 101, 128])
def test_planted_exact_ties_lower_index_wins(k, dtype):
    """Integer-valued euclidean data (exact in bf16 and fp32) with duplicated index rows: the result
    equals the exact integer ranking, the lower index first among equal similarities."""
    from oracle import retrieval as R
    g = torch.Generator().manual_seed(k)
    x = torch.randint(-6, 7, (1000, 32), generator=g)
    src = torch.randint(0, 1000, (300,), generator=g)
    dst = torch.randperm(1000, generator=g)[:300]
    x[dst] = x[src]
    q = torch.cat([x[torch.randint(0, 1000, (64,), generator=g)],
                   torch.randint(-6, 7, (65, 32), generator=g)])
    sim_exact = -((q * q).sum(1, keepdim=True) + (x * x).sum(1)[None] - 2 * q @ x.T)
    want_s, want_i = R.top_k(sim_exact.numpy(), k)
    qd, xd = q.float().to(DEV), x.float().to(DEV)
    for splits in (0, 1, 3, SPLITS_MAX):
        idx, sim, _ = _run(qd, xd, k, "euclidean", dtype, splits)
        assert (idx.cpu().numpy() == want_i).all()
        assert (sim.cpu().double().numpy() == want_s).all()
    # ties really occur among the returned lists
    assert (torch.from_numpy(want_s).diff(1) == 0).any()


@pytest.mark.parametrize("metric,dtype", [("cosine", "bf16"), ("euclidean", "bf16"),
                                          ("cosine", "fp32"), ("euclidean", "fp32")])
def test_bit_identical_across_splits(metric, dtype):
    g = torch.Generator(device=DEV).manual_seed(5)
    q = torch.randn(1000, 100, device=DEV, generator=g)
    x = torch.randn(5924, 100, device=DEV, generator=g)
    x[1000:1100] = x[:100]                      # exact ties across split boundaries too
    ref_i, ref_s, _ = _run(q, x, 64, metric, dtype, 1)
    for splits in (2, 3, SPLITS_MAX, 0):
        idx, sim, _ = _run(q, x, 64, metric, dtype, splits)
        assert torch.equal(idx, ref_i) and torch.equal(sim, ref_s), splits


def test_bit_identical_graph_replay_and_concurrent_streams():
    g = torch.Generator(device=DEV).manual_seed(6)
    qs = [torch.randn(700, 512, device=DEV, generator=g) for _ in range(2)]
    xs = [torch.randn(3000, 512, device=DEV, generator=g) for _ in range(2)]
    eager = [knn_topk(qs[i], xs[i], 101) for i in range(2)]
    torch.cuda.synchronize()
    # CUDA graph: captured once, replayed on new inputs written into the captured buffers
    qin, xin = qs[0].clone(), xs[0].clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gi, gs = knn_topk(qin, xin, 101)
    for i in (1, 0, 1):
        qin.copy_(qs[i])
        xin.copy_(xs[i])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(gi, eager[i][0]) and torch.equal(gs, eager[i][1])
    # two streams at once
    streams = [torch.cuda.Stream() for _ in range(2)]
    out = [None, None]
    for rep in range(3):
        for i in range(2):
            streams[i].wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(streams[i]):
                out[i] = knn_topk(qs[i], xs[i], 101)
        torch.cuda.synchronize()
        for i in range(2):
            assert torch.equal(out[i][0], eager[i][0]) and torch.equal(out[i][1], eager[i][1])


def _retrieval_batches():
    """8 classes of 4 identical images, 8 singletons and 8 distractors (label -1) interleaved, in
    batches of 12 (64 px).  A query's own copies rank first; a singleton is a hit only through the
    reference's position quirk.  The 24 distinct images have input scales 1.5 apart: with zero
    moving means and betas the network is positively homogeneous, so their embeddings' norms, and
    hence their euclidean distances, are well separated."""
    g = torch.Generator().manual_seed(11)
    scales = 1.5 ** torch.randperm(24, generator=g).double()
    distinct = [torch.randn(64, 64, 3, generator=g) * float(c) for c in scales]
    imgs = [distinct[c] for c in range(8) for _ in range(4)] + distinct[8:]
    labels = [c for c in range(8) for _ in range(4)] + list(range(8, 16)) + [-1] * 8
    perm = torch.randperm(len(imgs), generator=g)
    imgs = torch.stack(imgs)[perm]
    labels = torch.tensor(labels)[perm]
    return [(imgs[i:i + 12], labels[i:i + 12]) for i in range(0, len(imgs), 12)]


@pytest.mark.parametrize("similarity,dtype", [("cosine", "fp32"), ("euclidean", "bf16")])
def test_recall_at_k_on_an_embedding_model_matches_oracle(similarity, dtype):
    """The cosine case runs the fp32 model, whose search is on three bf16 planes: the embeddings of
    an untrained network are nearly parallel, and only fp32-level rounding is below their gaps."""
    from oracle import retrieval as R
    from assembled_cnn_b200.model_fns import build_model, recall_at_k
    model = build_model(resnet_size=50, resnet_version=1, embedding_size=32, num_classes=10, dtype=dtype)
    batches = _retrieval_batches()
    # clone: the forward returns a view of the runtime's buffer, which the next batch overwrites
    emb = torch.cat([model(x, False, return_embedding=True).float().clone() for x, _ in batches])
    labels = torch.cat([y for _, y in batches])
    e64 = emb.double().cpu().numpy()
    lab = labels.numpy()
    assert len({tuple(r) for r in e64.tolist()}) == 24          # the 24 distinct images
    # the margin: every different row is farther from a query than the rounding can reach
    s = R.similarity(e64, e64, similarity)
    same = (e64[:, None, :] == e64[None, :, :]).all(-1)
    gap = s.diagonal()[:, None] - s
    if similarity == "cosine":
        need = 1e-4 + 0 * gap
    else:
        norm = np.sqrt((e64 * e64).sum(1))
        need = 0.02 * (norm[:, None] + norm[None, :]) ** 2
    assert (gap > need)[~same].all(), float((gap - need)[~same].min())
    want = R.recall_at_k(e64, lab, (1, 5), similarity)
    assert 0 < want[1] < 1                       # singletons make it non-trivial
    metric = RecallAtK((1, 5), similarity=similarity, dtype=dtype, device=DEV)
    for (x, y) in batches:
        metric.update(model(x, False, return_embedding=True), y)
    assert metric.result() == want
    out = recall_at_k(model, batches, len(labels), (1, 5), similarity, global_step=7)
    assert out == {"recall_at_1": want[1], "recall_at_5": want[5], "global_step": 7}
    with pytest.raises(AssertionError):
        recall_at_k(model, batches, len(labels) + 1, (1, 5), similarity)


def test_sop_size_matches_chunked_fp32_reference():
    """60 502 x 60 502, d = 512, k = 6 (Stanford Online Products): 256 sampled query rows against a
    fp32 torch similarity + topk over the kernel's rounded operands."""
    n, d, k = 60502, 512, 6
    g = torch.Generator(device=DEV).manual_seed(12)
    feats = torch.randn(n, d, device=DEV, generator=g)
    idx, sim, work = _run(feats, feats, k, "cosine", "bf16")
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(3))[:256].to(DEV)
    qr, xr, _, _, kp, _, _ = _operands(work, n, n, d, k, "bf16")
    ref_s, ref_i = (qr[rows].float() @ xr.float().T).topk(k, dim=1)
    assert (idx[rows].long()[:, 0] == rows).all()          # itself first
    assert (sim[rows] - ref_s).abs().max() < 1e-3
    assert (idx[rows].long() == ref_i).float().mean() > 0.95
    _check(qr, xr, idx[rows], sim[rows], "cosine", kp, rows=rows)


def test_non_finite_rows_are_padded_and_refused_by_recall():
    """A query row whose similarities are all NaN gets the documented padding (-inf, 2147483647);
    RecallAtK refuses non-finite embeddings instead of indexing with it."""
    g = torch.Generator(device=DEV).manual_seed(13)
    q = torch.randn(5, 64, device=DEV, generator=g)
    x = torch.randn(300, 64, device=DEV, generator=g)
    q[2, 7] = float("nan")
    idx, sim = knn_topk(q, x, 6)
    assert (idx[2] == 2 ** 31 - 1).all() and (sim[2] == float("-inf")).all()
    good = torch.tensor([0, 1, 3, 4], device=DEV)
    assert torch.equal(idx[good], knn_topk(q[good], x, 6)[0])
    metric = RecallAtK((1, 5), device=DEV)
    metric.update(torch.cat([q, x]), torch.arange(305) % 7)
    with pytest.raises(ValueError):
        metric.result()
