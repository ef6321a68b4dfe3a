"""GPU checks of the exported servables: acnn_predict_rows against float64 (ties, +-inf and NaN rows, graph
replay, two streams), Servable.predict on the golden TFRecord's JPEGs and generated images against
predictions_of(model(x, False)) on the PIL-decoded, float32-restated eval batches (bf16 / fp32), request sizes
around max_batch, a servable reloaded from disk, predict_images, export_test against evaluate_classification
and a numpy restatement of the reference's zero-shot Recall@1, and train_and_evaluate(export_dir=...,
export_only=...)."""
import glob
import io
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(ROOT, "golden", "eval_golden.tfrecord")
sys.path.insert(0, os.path.join(ROOT, "golden"))
import make_eval_preprocess_golden as mk  # noqa: E402

U = 2.0 ** -24          # fp32 unit roundoff
TINY = 2.0 ** -126      # subnormal results: an absolute slack of the smallest normal


# ---------------------------------------------------------------------------------- acnn_predict_rows
def _predict(logits, n_valid=None, out=None):
    from assembled_cnn_b200.metrics import predict_rows
    out = predict_rows(logits, n_valid, out)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def _first_max(x32):
    """tf.argmax of fp32 logits: the first index of the largest value, -1 for a row holding a NaN."""
    return np.where(np.isnan(x32).any(1), -1, np.argmax(np.where(np.isnan(x32), 0, x32), 1))


def _bounds(x32):
    """float64 probabilities and per-element bounds of the kernel's fp32 arithmetic.  Softmax: x_j - max
    rounds with a relative error u, which exp turns into |a_j| u; expf adds at most 2 ulp (4 u); the sum of
    NC terms in any fixed order adds (NC - 1) u to the terms' own max_k (|a_k| + 4) u; the division adds u:
    |p - p64| <= (|a_j| + max_k |a_k| + NC + 8) u p64.  Sigmoid: expf 4 u, the addition u, the division u:
    8 u relative.  Both plus the smallest normal for results in the subnormal range.  A -inf logit's
    probability is exactly 0 (expf(-inf)), so only the finite differences a_j enter the bound."""
    x = x32.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        a = x - x.max(1, keepdims=True)
        e = np.exp(a)
        p = e / e.sum(1, keepdims=True)
        af = np.where(np.isfinite(a), np.abs(a), 0.0)
        tol_p = (af + af.max(1, keepdims=True) + x.shape[1] + 8) * U * p + TINY
        s = 1.0 / (1.0 + np.exp(-x))
    return p, tol_p, s, 8 * U * s + TINY


def _check(x32, got):
    classes, prob, sig = got
    assert np.array_equal(classes, _first_max(x32))
    p, tol_p, s, tol_s = _bounds(x32)
    nan_p = np.isnan(p)
    assert np.array_equal(np.isnan(prob), nan_p)
    assert np.all(np.abs(prob[~nan_p] - p[~nan_p]) <= tol_p[~nan_p])
    assert np.array_equal(np.isnan(sig), np.isnan(s))
    ok = ~np.isnan(s)
    assert np.all(np.abs(sig[ok] - s[ok]) <= tol_s[ok])


def _special_rows(x):
    """Plants ties, +-inf and NaN rows in the float32 [B, NC] array x (rows 0..7 when B allows)."""
    B, NC = x.shape
    if NC >= 3:
        specials = [lambda r: r.__setitem__([1, NC - 1], r.max() + 1),        # a tie: the first index wins
                    lambda r: r.__setitem__(slice(None), 2.5),                 # all equal: 0
                    lambda r: r.__setitem__(NC // 2, np.inf),                  # +inf: its index, NaN softmax
                    lambda r: r.__setitem__([0, NC - 1], -np.inf),             # -inf at the ends
                    lambda r: r.__setitem__(slice(None), -np.inf),             # only -inf: 0
                    lambda r: r.__setitem__(NC - 1, np.nan),                   # NaN: -1
                    lambda r: r.__setitem__([0, 2], [np.inf, np.inf])]         # two +inf: the first
    else:
        specials = [lambda r: r.__setitem__(0, np.inf), lambda r: r.__setitem__(0, np.nan),
                    lambda r: r.__setitem__(0, -np.inf)]
    for i, f in enumerate(specials[:B - 1]):
        f(x[i + 1])
    return x


@pytest.mark.parametrize("B,NC,ld", [(1, 1, 32), (1, 1001, 1024), (256, 1001, 1024), (257, 37, 64)])
def test_predict_rows_matches_float64(B, NC, ld):
    rng = np.random.default_rng(B * 7 + NC)
    full = (rng.standard_normal((B, ld)) * 4).astype(np.float32)
    x = _special_rows(full[:, :NC].copy())
    full[:, :NC] = x
    full[:, NC:] = np.nan                     # columns >= NC are never read
    logits = torch.from_numpy(full).cuda()[:, :NC]
    _check(x, _predict(logits))
    # padding rows are not written
    if B > 1:
        out = (torch.full((B,), 77, dtype=torch.int32, device="cuda"),
               torch.full((B, NC), 77.0, device="cuda"), torch.full((B, NC), 77.0, device="cuda"))
        got = _predict(logits, B - 1, out)
        _check(x[:B - 1], [g[:B - 1] for g in got])
        assert got[0][B - 1] == 77 and (got[1][B - 1] == 77).all() and (got[2][B - 1] == 77).all()


def test_predict_rows_large_logits_and_single_column():
    x = np.array([[1e30, -1e30, 3e38], [-87.0, -104.0, 88.5], [0.0, -0.0, 1e-45]], np.float32)
    _check(x, _predict(torch.from_numpy(x).cuda()))
    one = np.array([[5.0], [-np.inf], [np.nan]], np.float32)
    got = _predict(torch.from_numpy(one).cuda())
    assert got[0].tolist() == [0, 0, -1]
    assert got[1][0, 0] == 1.0 and np.isnan(got[1][1:]).all()


def test_predict_rows_graph_replay_and_streams_bit_identical():
    from assembled_cnn_b200.metrics import predict_rows
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(256, 1024, generator=g) * 4).cuda()[:, :1001]
    ref = _predict(logits, 250)

    def outs(fill):
        return (torch.full((256,), fill, dtype=torch.int32, device="cuda"),
                torch.full((256, 1001), float(fill), device="cuda"), torch.full((256, 1001), float(fill), device="cuda"))

    outg = outs(-7)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            predict_rows(logits, 250, outg)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outg, ref):
        a = a.cpu().numpy()
        assert a[:250].tobytes() == b[:250].tobytes() and (a[250:] == -7).all()
    pairs = [(torch.cuda.Stream(), outs(0)) for _ in range(2)]
    for st, o in pairs:
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            for _ in range(4):
                predict_rows(logits, 250, o)
    torch.cuda.synchronize()
    for _, o in pairs:
        for a, b in zip(o, ref):
            assert a.cpu().numpy()[:250].tobytes() == b[:250].tobytes()


# ------------------------------------------------------------------------------------------- servable
def _jpeg(rng, h, w, gray=False, fmt="JPEG", **kw):
    from PIL import Image
    base = rng.integers(0, 256, 3)
    img = np.clip(base + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
    im = Image.fromarray(img).convert("L") if gray else Image.fromarray(img)
    buf = io.BytesIO()
    im.save(buf, format=fmt, **kw)
    return buf.getvalue()


@pytest.fixture(scope="module")
def images():
    """The golden TFRecord's six JPEGs, then generated ones of mixed sizes: grayscale, 4:2:0 and 4:4:4,
    progressive (decoded by PIL) and a PNG (PIL)."""
    from assembled_cnn_b200 import imagenet_eval as ie
    out = [ie.read_encoded(GOLDEN, off, n) for _, off, n in ie.read_records(GOLDEN)]
    rng = np.random.default_rng(3)
    for i in range(24):
        h, w = int(rng.integers(20, 160)), int(rng.integers(20, 160))
        kind = i % 6
        if kind == 0:
            out.append(_jpeg(rng, h, w, gray=True, quality=90))
        elif kind == 1:
            out.append(_jpeg(rng, h, w, quality=85, subsampling=0))
        elif kind == 2:
            out.append(_jpeg(rng, h, w, quality=95, progressive=True))
        elif kind == 3:
            out.append(_jpeg(rng, h, w, fmt="PNG"))
        else:
            out.append(_jpeg(rng, h, w, quality=90))
    return out


def _oracle_x(buffers, ptype, image_size):
    from assembled_cnn_b200 import imagenet_eval as ie
    from oracle import eval_preprocess as O
    return np.stack([O.preprocess(ie.decode_rgb(io.BytesIO(b)), ptype, image_size) for b in buffers])


SIZE = 64


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_predict_equals_model_on_pil_batches(images, dtype):
    from assembled_cnn_b200.metrics import predict_rows
    from assembled_cnn_b200.model_fns import Servable, build_model, predictions_of
    model = build_model(resnet_size=50, dtype=dtype, seed=11)
    n = len(images)
    sv = Servable(model, image_size=SIZE, max_batch=n)
    got = sv.predict(images)
    behind = sv._pipe.logits[:n].clone()          # the logits of the one chunk, before model() reuses buffers
    assert set(got) == {"classes", "probabilities", "probabilities_sigmoid"}
    assert got["classes"].dtype == np.int64 and got["probabilities"].shape == (n, 1001)
    x = _oracle_x(images, "imagenet", SIZE)
    logits = model(torch.from_numpy(x), False).float().clone()
    assert behind.cpu().numpy().tobytes() == logits.cpu().numpy().tobytes()
    want = predictions_of(logits)
    assert np.array_equal(got["classes"], want["classes"].cpu().numpy())
    # the kernel on the same logits: the same bits; torch's softmax / sigmoid within both their bounds
    same = [t.cpu().numpy() for t in predict_rows(logits)]
    assert got["probabilities"].tobytes() == same[1].tobytes()
    assert got["probabilities_sigmoid"].tobytes() == same[2].tobytes()
    x32 = logits.cpu().numpy()
    _check(x32, [got["classes"].astype(np.int32), got["probabilities"], got["probabilities_sigmoid"]])
    p, tol_p, s, tol_s = _bounds(x32)
    assert np.all(np.abs(got["probabilities"] - want["probabilities"].cpu().numpy()) <= 2 * tol_p)
    assert np.all(np.abs(got["probabilities_sigmoid"] - want["probabilities_sigmoid"].cpu().numpy()) <= 2 * tol_s)


def test_request_sizes_reload_and_preprocessed_input(images, tmp_path):
    from assembled_cnn_b200.model_fns import Servable, build_model, export_model, load_servable
    model = build_model(resnet_size=50, dtype="bf16", seed=12, embedding_size=64)
    B = 8
    sv = Servable(model, preprocessing_type="imagenet", image_size=SIZE, max_batch=B)
    pool = (images * 2)[:3 * B + 5]
    whole = sv.predict(pool)
    assert set(whole) == {"classes", "probabilities", "probabilities_sigmoid", "embedding"}
    assert whole["embedding"].shape == (len(pool), 64)
    for n in (1, B - 1, B, B + 1, 3 * B + 5):
        part = sv.predict(pool[:n])
        for k, v in part.items():
            assert v.tobytes() == whole[k][:n].tobytes(), (n, k)
    # preprocessed input: the same bits as the encoded images
    pre = sv.predict_images(_oracle_x(pool, "imagenet", SIZE))
    for k, v in pre.items():
        assert v.tobytes() == whole[k].tobytes(), k
    # reloaded from disk on a fresh Model: the same bits, through both signatures
    binary, prep = export_model(model, str(tmp_path / "export"), preprocessing_type="imagenet", image_size=SIZE)
    assert binary.startswith(str(tmp_path / "export" / "channels_last" / "binary_input"))
    for path in (binary, prep):
        sv2 = load_servable(path, max_batch=B)
        assert sv2.model is not model and sv2.outputs == sv.outputs
        got = sv2.predict(pool)
        for k, v in got.items():
            assert v.tobytes() == whole[k].tobytes(), (path, k)
    assert sv.predict([])["classes"].shape == (0,)


def _write_shard(path, rng, n, num_classes, distractors=False):
    Example = mk.example_class()
    recs, labels = [], []
    for i in range(n):
        ex = Example()
        ex.features.feature["image/encoded"].bytes_list.value.append(
            _jpeg(rng, int(rng.integers(20, 150)), int(rng.integers(20, 150)), quality=90))
        label = int(rng.integers(0, num_classes))
        if distractors and i % 5 == 4:
            label = -1                            # no image/class/label: a distractor
        else:
            ex.features.feature["image/class/label"].int64_list.value.append(label)
        labels.append(label)
        data = ex.SerializeToString()
        head = len(data).to_bytes(8, "little")
        recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
    path.write_bytes(b"".join(recs))
    return labels


def test_export_test_matches_evaluations(tmp_path):
    from assembled_cnn_b200.model_fns import build_model, evaluate_classification, export_model, export_test, \
        load_servable
    rng = np.random.default_rng(9)
    data = tmp_path / "data"
    data.mkdir()
    _write_shard(data / "validation-00000-of-00002", rng, 23, 10)
    _write_shard(data / "validation-00001-of-00002", rng, 19, 10)
    model = build_model(resnet_size=50, num_classes=10, dtype="bf16", seed=13)
    binary, _ = export_model(model, str(tmp_path / "cls"), preprocessing_type="imagenet", image_size=SIZE)
    acc = export_test(binary, str(data), batch_size=16)
    want = evaluate_classification(model, str(data), image_size=SIZE, batch_size=16)["accuracy"]
    assert acc == want
    text = open(os.path.join(binary, "model_performance.txt")).read()
    assert text == "IMPOTANT! Evaluation metric of exported saved_model.pb is {}".format(acc)
    # zero-shot: every row a query, distractors included, only the query itself excluded
    zs = tmp_path / "zs"
    zs.mkdir()
    labels = _write_shard(zs / "validation-00000-of-00001", rng, 40, 4, distractors=True)
    emb_model = build_model(resnet_size=50, num_classes=10, dtype="fp32", seed=14, embedding_size=32)
    binary, _ = export_model(emb_model, str(tmp_path / "emb"), preprocessing_type="imagenet", image_size=SIZE)
    got = export_test(binary, str(zs), batch_size=16, zeroshot=True)
    from assembled_cnn_b200 import imagenet_eval as ie
    path = str(zs / "validation-00000-of-00001")
    emb = load_servable(binary, max_batch=16).predict(
        [ie.read_encoded(path, off, n) for _, off, n in ie.read_records(path, missing_label=-1)])["embedding"]
    x = emb / np.maximum(np.linalg.norm(emb, axis=1, keepdims=True), 1e-12)        # sklearn's normalize
    sim = x.dot(x.T)
    np.fill_diagonal(sim, -10)
    lab = np.array(labels)
    want = sum(lab[np.argmax(sim[i])] == lab[i] for i in range(len(lab))) / len(lab)
    assert got == want
    with pytest.raises(ValueError, match="embedding"):
        export_test(export_model(model, str(tmp_path / "noemb"), preprocessing_type="imagenet",
                                 image_size=SIZE)[0], str(zs), zeroshot=True)


def test_train_and_evaluate_exports(tmp_path):
    from assembled_cnn_b200.checkpoint import latest_checkpoint, load_checkpoint, restore
    from assembled_cnn_b200.model_fns import Servable, build_model, load_servable, train_and_evaluate
    rng = np.random.default_rng(21)
    data = tmp_path / "data"
    data.mkdir()
    _write_shard(data / "train-00000-of-00001", rng, 24, 10)
    _write_shard(data / "validation-00000-of-00001", rng, 13, 10)
    kw = dict(batch_size=8, dataset_name="food101", train_epochs=1, image_size=SIZE, seed=3, num_workers=4,
              dtype="bf16", num_best_ckpt_to_keep=1)
    # food101 has 101 classes; the labels above are in [0, 10)
    run = tmp_path / "run"
    res = train_and_evaluate(str(data), str(run), max_train_steps=2, export_dir=str(tmp_path / "e1"), **kw)
    assert len(res) == 1 and res[0]["global_step"] == 2
    (binary,) = glob.glob(str(tmp_path / "e1" / "channels_last" / "binary_input" / "*"))
    (prep,) = glob.glob(str(tmp_path / "e1" / "channels_last" / "preprocessed_input" / "*"))
    assert sorted(os.listdir(binary)) == ["config.json", "model_performance.txt", "variables.npz"]
    assert sorted(os.listdir(prep)) == ["config.json", "variables.npz"]
    trained = build_model(resnet_size=50, num_classes=101, dtype="bf16")
    trained.runtime(1, SIZE, SIZE, training=False)
    restore(trained, latest_checkpoint(str(run)))
    imgs = [_jpeg(rng, 50, 70, quality=90) for _ in range(5)]
    want = Servable(trained, image_size=SIZE, max_batch=8).predict(imgs)
    got = load_servable(binary, max_batch=8).predict(imgs)
    for k in want:
        assert got[k].tobytes() == want[k].tobytes(), k
    # export_only: no cycle, the latest checkpoint's weights
    res2 = train_and_evaluate(str(data), str(run), export_only=True, export_dir=str(tmp_path / "e2"), **kw)
    assert res2 == []
    (binary2,) = glob.glob(str(tmp_path / "e2" / "channels_last" / "binary_input" / "*"))
    a, b = load_checkpoint(os.path.join(binary, "variables.npz")), load_checkpoint(os.path.join(binary2, "variables.npz"))
    assert sorted(a) == sorted(b) and all(np.array_equal(a[k], b[k]) for k in a)
    assert "global_step" not in a and not any(k.endswith("/Momentum") for k in a)
