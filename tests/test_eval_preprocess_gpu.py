"""GPU checks of the classification evaluation (classifier.evaluate(input_fn_eval)): acnn_resize_crop_u8
bit for bit against the float32 oracle over the golden size grid of every preprocessing type and a
mixed-size padded batch, whole-model logits through acnn_set_images_resized against the fp32 input path,
acnn_classify_rows against float64 (ties, non-finite rows, padding, graph replay, streams), and
model_fns.evaluate_classification end to end on synthetic TFRecord shards against an oracle pipeline."""
import io
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(ROOT, "golden", "eval_preprocess_golden.json")))
MEAN = (123.68, 116.78, 103.94)


def _mean(device="cuda"):
    return torch.tensor(MEAN, dtype=torch.float32, device=device)


def _descs(images, geoms, B, device="cuda"):
    """(device image bytes, device descriptor table of B rows) for uint8 [h, w, 3] arrays."""
    from assembled_cnn_b200.imagenet_eval import DESC_DTYPE, check_descriptors
    offs = np.cumsum([0] + [a.nbytes for a in images])
    buf = torch.from_numpy(np.concatenate([a.reshape(-1) for a in images])).to(device)
    desc = np.zeros(B, DESC_DTYPE)
    for i, (a, (s, rh, rw, cy, cx)) in enumerate(zip(images, geoms)):
        desc[i] = (buf.data_ptr() + int(offs[i]), a.shape[0], a.shape[1], rh, rw, cy, cx)
    check_descriptors(desc, len(images), geoms[0][0])
    return buf, torch.from_numpy(desc.view(np.uint8).copy()).to(device)


def _resize(images, geoms, B=None, out=None, mean=None):
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    n, S = len(images), geoms[0][0]
    B = B or n
    buf, desc = _descs(images, geoms, B)
    out = torch.full((B, S, S, 3), float("nan"), device="cuda") if out is None else out
    mean = _mean() if mean is None else mean
    _lib.check(lib.acnn_resize_crop_u8(desc.data_ptr(), B, n, S, mean.data_ptr(), out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "acnn_resize_crop_u8")
    torch.cuda.synchronize()
    return out


TYPES = sorted({(c["type"], c["image_size"]) for c in GOLD["cases"]})


@pytest.mark.parametrize("ptype,image_size", TYPES)
def test_resize_crop_bit_identical_to_oracle(ptype, image_size):
    from oracle import eval_preprocess as O
    cases = [c for c in GOLD["cases"] if (c["type"], c["image_size"]) == (ptype, image_size)]
    rng = np.random.default_rng(len(cases) + image_size)
    images = [rng.integers(0, 256, (c["h"], c["w"], 3), dtype=np.uint8) for c in cases]
    geoms = [(c["S"], c["rsz"][0], c["rsz"][1], c["crop"][0], c["crop"][1]) for c in cases]
    got = _resize(images, geoms).cpu().numpy()
    for i, a in enumerate(images):
        want = O.preprocess(a, ptype, image_size)
        assert np.array_equal(got[i], want), (ptype, a.shape)


def test_resize_mixed_batch_padding_and_host_mean():
    from assembled_cnn_b200.imagenet_eval import eval_geometry
    from oracle import eval_preprocess as O
    rng = np.random.default_rng(7)
    shapes = [(375, 500), (500, 333), (64, 64), (1, 300), (2592, 1944), (121, 400), (96, 80)]
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    geoms = [eval_geometry(h, w, "imagenet_224_256a") for h, w in shapes]
    out = torch.full((10, 256, 256, 3), 12345.0, device="cuda")
    for mean in (_mean("cuda"), _mean("cpu")):
        _resize(images, geoms, B=10, out=out, mean=mean)
        got = out.cpu().numpy()
        for i, a in enumerate(images):
            assert np.array_equal(got[i], O.preprocess(a, "imagenet_224_256a")), shapes[i]
        assert (got[7:] == 12345.0).all()            # rows >= n_valid untouched


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_model_logits_resized_path_bit_identical(dtype):
    from assembled_cnn_b200.model_fns import build_model
    from assembled_cnn_b200.imagenet_eval import eval_geometry
    from oracle import eval_preprocess as O
    model = build_model(resnet_size=50, num_classes=10, dtype=dtype)
    rng = np.random.default_rng(3)
    shapes = [(80, 60), (64, 64), (50, 120), (100, 75)]
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    geoms = [eval_geometry(h, w, "imagenet", 64) for h, w in shapes]
    x = np.stack([O.preprocess(a, "imagenet", 64) for a in images])
    want = model(torch.from_numpy(x), False).clone()
    rt = model.runtime(4, 64, 64, training=False)
    rt.t[rt.plan.meta["images"]].zero_()
    buf, desc = _descs(images, geoms, 4)
    rt.set_images_resized(desc, 4, _mean())
    rt.run_forward()
    assert torch.equal(rt.t[rt.plan.meta["logits"]][:, :10], want)
    # a host descriptor table is refused
    host = desc.cpu().pin_memory()
    assert rt.lib.acnn_set_images_resized(rt.model.handle, host.data_ptr(), 4, _mean().data_ptr(), rt.stream) == 1
    with pytest.raises(ValueError):
        rt.set_images_resized(desc[:64], 4, _mean())
    with pytest.raises(ValueError):
        rt.set_images_resized(desc, 5, _mean())


# ---------------------------------------------------------------------------- acnn_classify_rows
def _rows(logits, labels, n_valid=None, k=5, ls=0.0, out=None):
    from assembled_cnn_b200.metrics import classify_rows
    out = classify_rows(logits, labels, n_valid, k, ls, out)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def _check_rows(x, labels, got, ls, k=5):
    """pred and hit_k exact; conf and ce within an element-wise rounding bound of the fp32 evaluation
    (the sums run over NC terms: a relative bound of (NC + 8) fp32 ulps of the magnitudes involved)."""
    from oracle import eval_preprocess as O
    pred, conf, hit, ce = got
    x64 = x.double().cpu().numpy()
    lab = labels.cpu().numpy()
    assert (pred == O.argmax(x64)).all()
    assert (hit.astype(bool) == O.in_top_k(x64, lab, k)).all()
    ok = np.isfinite(x64).all(1)
    assert np.isnan(conf[~ok]).all() and np.isnan(ce[~ok]).all()
    nc = x64.shape[1]
    u = 2.0 ** -24 * (nc + 8)
    assert np.all(np.abs(conf[ok] - O.softmax_conf(x64[ok])) <= u * O.softmax_conf(x64[ok]))
    want = O.cross_entropy(x64[ok], lab[ok], ls)
    scale = np.abs(x64[ok] - x64[ok].max(1, keepdims=True)).max(1) + np.log(nc) + np.abs(want)
    assert np.all(np.abs(ce[ok] - want) <= 4 * u * scale)


@pytest.mark.parametrize("B,NC,ld,scale,ls", [(300, 1001, 1024, 3.0, 0.1), (64, 10, 128, 1.0, 0.0),
                                              (33, 1, 1, 1.0, 0.0), (257, 100, 100, 30.0, 0.2),
                                              (128, 1001, 1024, 0.01, 0.1)])
def test_classify_rows_matches_float64(B, NC, ld, scale, ls):
    g = torch.Generator().manual_seed(B * NC)
    full = (torch.randn(B, ld, generator=g) * scale).cuda()
    x = full[:, :NC]
    labels = torch.randint(0, NC, (B,), generator=g, dtype=torch.int32)
    labels[::3] = torch.from_numpy(x[::3].double().cpu().numpy().argmax(1)).int()
    labels = labels.cuda()
    _check_rows(x, labels, _rows(x, labels, ls=ls, k=min(5, NC)), ls, k=min(5, NC))


def test_classify_rows_ties_non_finite_and_padding():
    x = torch.full((12, 40), -3.0)
    x[0, [4, 9, 17]] = 2.0                          # argmax: the lowest index of equal logits
    x[1, :7] = torch.tensor([9., 8., 7., 6., 5., 5., 5.])   # label 6 ties at 5th place: in top 5
    x[2, :7] = torch.tensor([9., 8., 7., 6., 5.5, 5., 5.])  # label 6 ties below 5 others: out
    x[3, 5] = float("nan")
    x[4, 0] = float("inf")
    x[5, 39] = float("-inf")
    x[6, :] = 1.0                                   # all equal: pred 0, every label in top 1
    x[7, 2] = 4.0
    labels = torch.tensor([17, 6, 6, 5, 0, 1, 39, 2, 0, 1, 2, 3], dtype=torch.int32)
    out = [torch.full((12,), 77, dtype=dt, device="cuda") for dt in (torch.int32, torch.float32, torch.int32,
                                                                        torch.float32)]
    got = _rows(x.cuda(), labels.cuda(), n_valid=9, out=out, ls=0.1)
    assert got[0][:9].tolist() == [4, 0, 0, -1, -1, -1, 0, 2, 0]
    assert got[2][:9].tolist() == [1, 1, 0, 0, 0, 0, 1, 1, 1]
    for t in got:
        assert (t[9:] == 77).all()                  # padding rows: not written
    _check_rows(x[:9].cuda(), labels[:9].cuda(), [t[:9] for t in got], 0.1)
    # an out-of-range label: never in the top k, NaN loss
    lab = torch.tensor([40, -1], dtype=torch.int32, device="cuda")
    p, c, h, ce = _rows(x[6:8].cuda(), lab, k=40)
    assert h.tolist() == [0, 0] and np.isnan(ce).all() and p.tolist() == [0, 2]


def test_classify_rows_graph_replay_and_streams_bit_identical():
    from assembled_cnn_b200.metrics import classify_rows
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(256, 1024, generator=g) * 4).cuda()[:, :1001]
    labels = torch.randint(0, 1001, (256,), generator=g, dtype=torch.int32).cuda()
    ref = _rows(logits, labels, 250, ls=0.1)
    kinds = (torch.int32, torch.float32, torch.int32, torch.float32)
    outg = tuple(torch.full((256,), -7, dtype=dt, device="cuda") for dt in kinds)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            classify_rows(logits, labels, 250, 5, 0.1, outg)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outg, ref):
        a = a.cpu().numpy()
        assert np.array_equal(a[:250], b[:250]) and (a[250:] == -7).all()
    outs = [tuple(torch.empty(256, dtype=dt, device="cuda") for dt in kinds) for _ in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    for st, o in zip(streams, outs):
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            for _ in range(4):
                classify_rows(logits, labels, 250, 5, 0.1, o)
    torch.cuda.synchronize()
    for o in outs:
        for a, b in zip(o, ref):
            assert np.array_equal(a.cpu().numpy()[:250], b[:250])


# ------------------------------------------------------------------------------------ end to end
N_IMAGES, NUM_CLASSES, SIZE = 203, 10, 64


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    """Three validation shards (and one file the glob must skip) of N_IMAGES synthetic JPEGs of mixed
    sizes, written with the golden generator's protobuf runtime and CRC."""
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "golden"))
    import make_eval_preprocess_golden as mk
    Example = mk.example_class()
    root = tmp_path_factory.mktemp("val")
    rng = np.random.default_rng(0)
    labels = []
    for sh in range(3):
        recs = []
        for i in range(sh * 70, min((sh + 1) * 70, N_IMAGES)):
            h, w = int(rng.integers(20, 150)), int(rng.integers(20, 150))
            base = rng.integers(0, 256, 3)
            img = np.clip(base + rng.normal(0, 50, (h, w, 3)), 0, 255).astype(np.uint8)
            buf = io.BytesIO()
            Image.fromarray(img).save(buf, format="JPEG", quality=90)
            ex = Example()
            ex.features.feature["image/encoded"].bytes_list.value.append(buf.getvalue())
            label = int(rng.integers(0, NUM_CLASSES))
            ex.features.feature["image/class/label"].int64_list.value.append(label)
            labels.append(label)
            data = ex.SerializeToString()
            head = len(data).to_bytes(8, "little")
            recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
        (root / ("validation-%05d-of-00003" % sh)).write_bytes(b"".join(recs))
    (root / "train-00000-of-00001").write_bytes(b"not a record")
    return root, labels


def _oracle_eval(model, root, batch, ls, wd, ptype="imagenet"):
    from assembled_cnn_b200 import imagenet_eval as ie
    from assembled_cnn_b200.model_fns import l2_loss
    from oracle import eval_preprocess as O
    recs = [(f, off, n, lab) for f in ie.validation_files(str(root)) for lab, off, n in ie.read_records(f)]
    logits, labels, sizes = [], [], []
    for a in range(0, len(recs), batch):
        chunk = recs[a:a + batch]
        x = np.zeros((batch, SIZE, SIZE, 3), np.float32)
        for i, (f, off, n, _) in enumerate(chunk):
            x[i] = O.preprocess(ie.decode_rgb(io.BytesIO(ie.read_encoded(f, off, n))), ptype, SIZE)
        logits.append(model(torch.from_numpy(x), False)[:len(chunk)].double().cpu().numpy())
        labels += [r[3] for r in chunk]
        sizes.append(len(chunk))
    x, labels = np.concatenate(logits), np.array(labels)
    pred, hit = O.argmax(x), O.in_top_k(x, labels, 5)
    ce = O.cross_entropy(x, labels, ls)
    bounds = np.cumsum([0] + sizes)
    loss = np.mean([ce[a:b].mean() for a, b in zip(bounds[:-1], bounds[1:])])
    rt = model.runtime(batch, SIZE, SIZE, training=False)
    return {"accuracy": float((pred == labels).mean()), "accuracy_top_5": float(hit.mean()),
            "ece": O.ece(O.softmax_conf(x), pred, labels), "loss": loss + float(l2_loss(rt, wd))}, labels


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_evaluate_classification_end_to_end(shards, dtype):
    from assembled_cnn_b200.model_fns import build_model, evaluate_classification
    root, labels = shards
    model = build_model(resnet_size=50, num_classes=NUM_CLASSES, dtype=dtype)
    want, oracle_labels = _oracle_eval(model, root, 32, 0.1, 4e-5)
    assert oracle_labels.tolist() == labels
    kw = dict(image_size=SIZE, batch_size=32, label_smoothing=0.1, num_workers=4)
    got = evaluate_classification(model, str(root), global_step=77, **kw)
    assert set(got) == {"accuracy", "accuracy_top_5", "ece", "loss", "global_step"} and got["global_step"] == 77
    assert got["accuracy"] == want["accuracy"] and got["accuracy_top_5"] == want["accuracy_top_5"]
    assert abs(got["ece"] - want["ece"]) < 1e-6
    assert got["loss"] == pytest.approx(want["loss"], rel=1e-5)
    eager = evaluate_classification(model, str(root), use_cuda_graph=False, **kw)
    assert eager == dict(got, global_step=None)
