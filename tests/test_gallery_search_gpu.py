"""GPU checks of image search.  Kernel: acnn_knn_search over an index prepared once by
acnn_knn_prepare_index equals acnn_knn_topk on the same Q and X bit for bit, in bf16, fp16 and fp32,
cosine and euclidean, over query counts from 1 to 1000, k up to 128, galleries up to 60 502 rows and d up to
2048; with exact ties across split boundaries at every forced split count up to one per SM, non-finite rows,
graph replay and two streams.  Servable: search equals metrics.knn_topk(predict(...)['embedding'], gallery)
bit for bit on every rung of (1, 8, 64, 256), for bf16 and fp32 models; a servable reloaded with the
gallery.npz that export_gallery wrote gives the same bits, and ranks each distinct image of the shards first."""
import io
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from assembled_cnn_b200 import _lib
from assembled_cnn_b200.metrics import DTYPES, KnnIndex, knn_topk

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.abspath(__file__))
SIZE = 64
LADDER = (1, 8, 64, 256)


def _splits(n):
    lib = _lib.load()
    return lib.acnn_set_knn_splits(n)


def _search(q, x, k, metric, dtype, splits=0, stream=None):
    """acnn_knn_search through the C ABI on a freshly prepared index, with a forced split count."""
    lib = _lib.load()
    (nq, d), nx = q.shape, x.shape[0]
    m, dt = (0 if metric == "cosine" else 1), DTYPES[dtype]
    st = (stream or torch.cuda.current_stream()).cuda_stream
    ib = lib.acnn_knn_index_bytes(nx, d, dt)
    index = torch.empty(ib, dtype=torch.uint8, device=DEV)
    _lib.check(lib.acnn_knn_prepare_index(x.data_ptr(), nx, d, m, dt, index.data_ptr(), ib, st), "prepare")
    wb = lib.acnn_knn_search_work_bytes(nq, nx, d, k, dt)
    work = torch.empty(wb, dtype=torch.uint8, device=DEV)
    idx = torch.empty(nq, k, dtype=torch.int32, device=DEV)
    sim = torch.empty(nq, k, dtype=torch.float32, device=DEV)
    prev = _splits(splits)
    try:
        _lib.check(lib.acnn_knn_search(q.data_ptr(), nq, index.data_ptr(), nx, d, k, m, dt, idx.data_ptr(),
                                       sim.data_ptr(), work.data_ptr(), wb, st), "acnn_knn_search")
    finally:
        _splits(prev)
    return idx, sim


def _same(a, b, what):
    assert torch.equal(a[0], b[0]) and a[1].view(torch.int32).equal(b[1].view(torch.int32)), what


def _cases():
    """Every (metric, dtype) runs every nq; nx, d and k cycle so that each value meets each pair."""
    nqs, nxs, ds, ks = (1, 7, 128, 129, 1000), (300, 5924, 60502), (100, 512, 2048), (1, 6, 101, 128)
    out = []
    for m, (metric, dtype) in enumerate(itertools.product(("cosine", "euclidean"), ("bf16", "fp16", "fp32"))):
        for i, nq in enumerate(nqs):
            out.append((nq, nxs[(i + m) % 3], ds[(i + 2 * m) % 3], ks[(i + m) % 4], metric, dtype))
    return out


@pytest.mark.parametrize("nq,nx,d,k,metric,dtype", _cases())
def test_search_equals_topk(nq, nx, d, k, metric, dtype):
    g = torch.Generator(device=DEV).manual_seed(nq * 131 + nx + d + k)
    q = torch.randn(nq, d, device=DEV, generator=g)
    x = torch.randn(nx, d, device=DEV, generator=g)
    x[nx // 2:nx // 2 + min(50, nx // 4)] = x[:min(50, nx // 4)]        # exact ties
    want = knn_topk(q, x, k, metric, dtype)
    _same(_search(q, x, k, metric, dtype), want, "default splits")
    # KnnIndex, the Python front of the same entry points
    _same(KnnIndex(x, metric, dtype).search(q, k), want, "KnnIndex")


def test_case_list_covers_every_value():
    cases = _cases()
    for pos, values in ((0, (1, 7, 128, 129, 1000)), (1, (300, 5924, 60502)), (2, (100, 512, 2048)),
                        (3, (1, 6, 101, 128))):
        for md in itertools.product(("cosine", "euclidean"), ("bf16", "fp16", "fp32")):
            assert set(values) <= {c[pos] for c in cases if (c[4], c[5]) == md}, (pos, md)


@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32"])
def test_ties_across_splits_at_every_split_count(dtype):
    """Integer rows (exact in every dtype) copied across many column tiles: every forced split count from 1
    to the cap (one per SM) gives acnn_knn_topk's bits, which are the exact integer ranking."""
    from oracle import retrieval as R
    g = torch.Generator().manual_seed(9)
    nx = 140 * 128 + 37
    x = torch.randint(-3, 4, (nx, 16), generator=g)
    src = torch.randint(0, nx, (3000,), generator=g)
    x[torch.randperm(nx, generator=g)[:3000]] = x[src]
    q = torch.cat([x[torch.randint(0, nx, (4,), generator=g)], torch.randint(-3, 4, (3, 16), generator=g)])
    want_s, want_i = R.top_k((-((q * q).sum(1, keepdim=True) + (x * x).sum(1)[None] - 2 * q @ x.T)).numpy(), 101)
    assert (np.diff(want_s, axis=1) == 0).any()
    qd, xd = q.float().to(DEV), x.float().to(DEV)
    want = knn_topk(qd, xd, 101, "euclidean", dtype)
    assert (want[0].cpu().numpy() == want_i).all() and (want[1].cpu().double().numpy() == want_s).all()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for s in range(1, min(sms, 132) + 1):
        _same(_search(qd, xd, 101, "euclidean", dtype, s), want, s)


def test_non_finite_rows():
    """A NaN query row gets the padding; NaN and inf index rows are never ranked -- as acnn_knn_topk."""
    g = torch.Generator(device=DEV).manual_seed(13)
    q = torch.randn(9, 64, device=DEV, generator=g)
    x = torch.randn(4000, 64, device=DEV, generator=g)
    q[2, 7] = float("nan")
    x[10, 3], x[3000, 0] = float("nan"), float("inf")
    for metric, dtype in itertools.product(("cosine", "euclidean"), ("bf16", "fp16", "fp32")):
        want = knn_topk(q, x, 6, metric, dtype)
        assert (want[0][2] == 2 ** 31 - 1).all() and (want[1][2] == float("-inf")).all()
        for s in (0, 1, 32):
            _same(_search(q, x, 6, metric, dtype, s), want, (metric, dtype, s))
    with pytest.raises(ValueError, match="NaN or infinite"):
        KnnIndex(x)


def test_graph_replay_and_two_streams():
    g = torch.Generator(device=DEV).manual_seed(6)
    x = torch.randn(20000, 512, device=DEV, generator=g)
    qs = [torch.randn(n, 512, device=DEV, generator=g) for n in (8, 8)]
    index = KnnIndex(x)
    eager = [knn_topk(q, x, 101) for q in qs]
    torch.cuda.synchronize()
    qin = qs[0].clone()
    out = (torch.empty(8, 101, dtype=torch.int32, device=DEV), torch.empty(8, 101, device=DEV))
    work = torch.empty(index.work_bytes(8, 101), dtype=torch.uint8, device=DEV)
    index.search(qin, 101, out, work)                 # loads the kernels before the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        index.search(qin, 101, out, work)
    for i in (1, 0, 1):
        qin.copy_(qs[i])
        graph.replay()
        torch.cuda.synchronize()
        _same(out, eager[i], ("graph", i))
    streams = [torch.cuda.Stream() for _ in range(2)]
    for _ in range(3):
        got = [None, None]
        for i in range(2):
            streams[i].wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(streams[i]):
                got[i] = index.search(qs[i], 101)
        torch.cuda.synchronize()
        for i in range(2):
            _same(got[i], eager[i], ("stream", i))


# ------------------------------------------------------------------------------------------ servable
def _jpeg(rng):
    from PIL import Image
    h, w = int(rng.integers(40, 120)), int(rng.integers(40, 120))
    img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="JPEG", quality=90)
    return buf.getvalue()


def _check_search(res, ref, gallery, k, dtype, labels=None):
    for name in ref:
        assert res[name].tobytes() == ref[name].tobytes(), name
    want_i, want_s = knn_topk(torch.from_numpy(ref["embedding"]).to(DEV), gallery, k, "cosine", dtype)
    assert res["neighbors"].dtype == np.int64 and res["neighbor_similarities"].dtype == np.float32
    assert np.array_equal(res["neighbors"], want_i.cpu().numpy().astype(np.int64))
    assert res["neighbor_similarities"].tobytes() == want_s.cpu().numpy().tobytes()
    if labels is not None:
        assert np.array_equal(res["neighbor_labels"], labels[res["neighbors"]])


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_servable_search_on_every_rung(dtype):
    from assembled_cnn_b200.model_fns import Servable, build_model
    model = build_model(resnet_size=50, embedding_size=32, dtype=dtype, seed=31)
    sv = Servable(model, image_size=SIZE, max_batch=256, batch_sizes=LADDER)
    rng = np.random.default_rng(7)
    jp = [_jpeg(rng) for _ in range(257)]
    ref = sv.predict(jp)
    g = torch.Generator().manual_seed(8)
    gal = torch.cat([torch.from_numpy(ref["embedding"][:40]), torch.randn(3000, 32, generator=g)]).to(DEV)
    labels = np.arange(len(gal)) % 17
    sv.set_gallery(gal, labels)
    for n in (1, 8, 64, 257):
        for k in (6, 101):
            for _ in range(2):        # the first call of a (rung, k) runs eagerly, the repeat replays graphs
                res = sv.search(jp[:n], k)
                _check_search(res, {key: v[:n] for key, v in ref.items()}, gal, k, dtype, labels)
    assert sorted(sv._pipes) == list(LADDER)
    # preprocessed images: eager launches
    x = torch.randn(70, SIZE, SIZE, 3, generator=torch.Generator().manual_seed(4)) * 60
    ref_x = sv.predict_images(x)
    _check_search(sv.search_images(x, 6), ref_x, gal, 6, dtype, labels)
    # predict is unchanged by the searches around it; a request of no image has empty neighbours
    assert all(sv.predict(jp[:9])[key].tobytes() == ref[key][:9].tobytes() for key in ref)
    empty = sv.search([], 6)
    assert empty["neighbors"].shape == (0, 6) and empty["neighbor_similarities"].shape == (0, 6)
    # a new gallery replaces the old one
    sv.set_gallery(gal.flip(0))
    _check_search(sv.search(jp[:8], 6), {key: v[:8] for key, v in ref.items()}, gal.flip(0), 6, dtype)


def test_search_graphs_survive_predict_and_k_changes():
    """A servable answering predict and search in turn replays the graphs it captured for both: no batch
    runs eagerly and no graph or search buffer is made again.  Each k has its own graphs, kept for the
    SEARCH_KS most recently used k, over one set of search buffers sized for the largest k."""
    from assembled_cnn_b200.model_fns import Servable, build_model
    model = build_model(resnet_size=50, embedding_size=32, dtype="bf16", seed=32)
    sv = Servable(model, image_size=SIZE, max_batch=256, batch_sizes=LADDER)
    rng = np.random.default_rng(9)
    jp = [_jpeg(rng) for _ in range(8)]
    ref = sv.predict(jp)
    gal = torch.randn(5000, 32, generator=torch.Generator().manual_seed(10)).to(DEV)
    sv.set_gallery(gal)
    # the first calls run eagerly, then each (k, staging slot) captures once: both orders cover both slots
    for order in ("sp", "sp", "ps", "ps"):
        for c in order:
            sv.search(jp, 6) if c == "s" else sv.predict(jp)
    pipe = sv._pipes[8]
    graphs, bufs = dict(pipe.graph_sets[6]), pipe.search_bufs
    predict_graphs = dict(pipe.graph_sets[0])
    assert sorted(graphs) == sorted(predict_graphs) == [(0, 8), (1, 8)]
    eager = []
    body = pipe._body
    pipe._body = lambda slot, n: (eager.append((pipe.k, slot, n, torch.cuda.is_current_stream_capturing())),
                                  body(slot, n))
    for _ in range(3):
        assert all(sv.predict(jp)[key].tobytes() == ref[key].tobytes() for key in ref)
        _check_search(sv.search(jp, 6), ref, gal, 6, "bf16")
    assert eager == [], eager             # every batch replayed a graph
    assert pipe.graph_sets[6] == graphs and pipe.graph_sets[0] == predict_graphs and pipe.search_bufs is bufs
    # many k: bounded graph sets, the buffers grow to the largest k only
    for k in (101, 7, 8, 9, 10, 6):
        _check_search(sv.search(jp, k), ref, gal, k, "bf16")
    assert pipe.k_cap == 101 and len(pipe.graph_sets) == 1 + pipe.SEARCH_KS
    assert list(pipe.graph_sets) == [0, 8, 9, 10, 6]


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


def test_export_gallery_reload_and_rank_itself_first(tmp_path):
    """Shards of 12 distinct images, 8 of them in three copies, 4 without a label.  The fp32 model's search
    (three bf16 planes) resolves the near-parallel embeddings of an untrained network."""
    from assembled_cnn_b200.model_fns import Servable, build_model, export_gallery, export_model, load_servable
    rng = np.random.default_rng(3)
    distinct = [_jpeg(rng) for _ in range(12)]
    items = [(distinct[c], 10 + c) for c in range(8) for _ in range(3)] + [(distinct[c], None) for c in range(8, 12)]
    items = [items[i] for i in rng.permutation(len(items))]
    data = tmp_path / "shards"
    data.mkdir()
    _write_shard(data / "validation-00000-of-00002", items[:15])
    _write_shard(data / "validation-00001-of-00002", items[15:])
    model = build_model(resnet_size=50, embedding_size=32, dtype="fp32", seed=41)
    binary, _ = export_model(model, str(tmp_path / "export"), preprocessing_type="imagenet", image_size=SIZE,
                             return_embedding=True)
    path = export_gallery(binary, str(data), batch_size=16)
    assert path == os.path.join(binary, "gallery.npz")
    assert sorted(os.listdir(binary)) == ["config.json", "gallery.npz", "variables.npz"]
    with pytest.raises(FileExistsError):
        export_gallery(binary, str(data))
    g = np.load(path)
    labels = np.array([-1 if lab is None else lab for _, lab in items])
    assert np.array_equal(g["label"], labels) and g["embedding"].dtype == np.float32
    assert list(g["shard_names"]) == ["validation-00000-of-00002", "validation-00001-of-00002"]
    assert np.array_equal(g["shard"], [0] * 15 + [1] * 13) and np.array_equal(g["record"], list(range(15)) + list(range(13)))
    jp = [b for b, _ in items]
    mem = Servable(model, image_size=SIZE, max_batch=16)
    ref = mem.predict(jp)
    assert g["embedding"].tobytes() == ref["embedding"].tobytes()      # the servable's own embedding
    mem.set_gallery(g["embedding"], g["label"])
    want = mem.search(jp, 5)
    loaded = load_servable(binary, max_batch=16, batch_sizes=(1, 8, 16))
    assert loaded.gallery_rows == len(items)
    for n in (1, 5, 28):
        got = loaded.search(jp[:n], 5)
        assert set(got) == set(want) and "neighbor_labels" in got
        for key in got:
            assert got[key].tobytes() == want[key][:n].tobytes(), (n, key)
    # each image's nearest rows are its own copies, the lowest row first
    first = want["neighbors"][:, 0]
    own = np.array([min(j for j, b in enumerate(jp) if b == q) for q in jp])
    assert np.array_equal(first, own)
    assert np.array_equal(want["neighbor_labels"][:, 0], labels[own])
