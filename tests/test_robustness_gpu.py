"""GPU checks of the robustness evaluation (mce/eval_robustness.py, --robustness_type ce): the uint8 input
conversion against torch bit for bit, whole-model logits through acnn_set_images_u8 against the fp32
input path, the softmax top-1 counter against float64 (ties, non-finite rows, padding, graph replay,
streams), a padded tail batch, and model_fns.corruption_error end to end on a synthetic ImageNet-C tree
against the float64 oracle."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MEAN = (123.68, 116.78, 103.94)


def _mean(device="cuda"):
    return torch.tensor(MEAN, dtype=torch.float32, device=device)


def _u8_ref(x, mean):
    return x.float() - mean.to(x.device)


def _images_from_u8(x, mean):
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    out = torch.full(x.shape, float("nan"), dtype=torch.float32, device=x.device)
    B, H, W, _ = x.shape
    _lib.check(lib.acnn_images_from_u8(x.data_ptr(), mean.data_ptr(), out.data_ptr(), B, H, W,
                                       torch.cuda.current_stream().cuda_stream), "acnn_images_from_u8")
    return out


def test_images_from_u8_every_byte_value():
    """Every byte value in every channel (both mean locations), against torch's x.float() - mean."""
    v = torch.arange(256, dtype=torch.uint8)
    x = torch.stack([v.roll(c) for c in range(3)], dim=1).reshape(1, 16, 16, 3).cuda()
    for mean in (_mean("cuda"), _mean("cpu"), _mean("cpu").pin_memory()):
        got = _images_from_u8(x, mean)
        assert torch.equal(got, _u8_ref(x, mean))
    # the three channels each saw all 256 values
    assert all(len(set(x[0, :, :, c].flatten().tolist())) == 256 for c in range(3))


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 5), (3, 7, 9), (4, 64, 64), (2, 224, 224), (5, 33, 31)])
def test_images_from_u8_random(shape):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randint(0, 256, shape + (3,), generator=g, dtype=torch.uint8).cuda()
    mean = torch.tensor([1.5, -2.25, 300.125]) if shape == (5, 33, 31) else _mean("cuda")
    assert torch.equal(_images_from_u8(x, mean.cuda() if shape[0] == 3 else mean), _u8_ref(x, mean))


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_model_logits_u8_path_bit_identical(dtype):
    from assembled_cnn_b200.model_fns import build_model
    model = build_model(resnet_size=50, num_classes=10, dtype=dtype)
    g = torch.Generator().manual_seed(11)
    x = torch.randint(0, 256, (4, 64, 64, 3), generator=g, dtype=torch.uint8).cuda()
    want = model(_u8_ref(x, _mean()), False).clone()
    rt = model.runtime(4, 64, 64, training=False)
    rt.t[rt.plan.meta["images"]].zero_()
    rt.set_images_u8(x, _mean())
    rt.run_forward()
    got = rt.t[rt.plan.meta["logits"]][:, :10]
    assert torch.equal(got, want)
    rt.set_images_u8(x, _mean("cpu"))          # host mean
    rt.run_forward()
    assert torch.equal(rt.t[rt.plan.meta["logits"]][:, :10], want)
    # a host image buffer is refused: the caller stages its own device buffer
    lib = rt.lib
    host = x.cpu().pin_memory()
    assert lib.acnn_set_images_u8(rt.model.handle, host.data_ptr(), _mean().data_ptr(),
                                  rt.stream) == 1
    with pytest.raises(ValueError):
        rt.set_images_u8(x[:3], _mean())
    with pytest.raises(ValueError):
        rt.set_images_u8(x.float(), _mean())


def _top1(logits, labels, n_valid=None, correct=None, pred=None):
    from assembled_cnn_b200.metrics import softmax_top1_count
    correct = torch.zeros(1, dtype=torch.int64, device="cuda") if correct is None else correct
    pred = softmax_top1_count(logits, labels, correct, n_valid, pred)
    return pred, correct


def _oracle_top1(x):
    """float64 softmax argmax, and a mask of rows whose top two float64 probabilities are within 8 fp32
    ulps (where the fp32 probabilities may round together)."""
    from oracle import robustness as R
    x64 = x.double().cpu().numpy()
    e = np.exp(x64 - x64.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True)
    if p.shape[1] == 1:
        return R.top1(x64), np.zeros(p.shape[0], dtype=bool)
    top2 = np.sort(p, axis=1)[:, -2:]
    close = (top2[:, 1] - top2[:, 0]) <= 8 * np.spacing(top2[:, 1].astype(np.float32)).astype(np.float64)
    return R.top1(x64), close


@pytest.mark.parametrize("B,NC,ld,scale", [(300, 1001, 1024, 3.0), (64, 10, 128, 1.0), (33, 1, 1, 1.0),
                                           (257, 100, 100, 30.0), (128, 1001, 1024, 0.01)])
def test_top1_matches_float64(B, NC, ld, scale):
    g = torch.Generator().manual_seed(B * NC)
    full = (torch.randn(B, ld, generator=g) * scale).cuda()
    logits = full[:, :NC]
    want, close = _oracle_top1(logits)
    labels = torch.from_numpy(want).int().cuda()
    labels[::3] = (labels[::3] + 1) % NC if NC > 1 else -5
    pred, correct = _top1(logits, labels)
    got = pred.cpu().numpy()
    assert close.sum() < B // 20 + 1
    assert (got[~close] == want[~close]).all()
    assert int(correct) == int((pred == labels).sum())


def test_top1_planted_ties():
    x = torch.full((6, 40), -10.0)
    x[0, 3] = x[0, 17] = 2.0                       # equal logits: the lower index
    x[1, 5] = x[1, 6] = x[1, 39] = 0.0
    a = np.float32(0.1)
    b = np.nextafter(a, np.float32(1))
    x[2, 8], x[2, 9] = float(a), float(b)         # exps both round to 1.0f: tie on the probabilities
    x[3, 30], x[3, 2] = float(b), float(a)         # the lower index is the smaller logit
    x[4, :] = 7.0                                  # all equal
    x[5, 21] = 1.0
    assert torch.argmax(x[2]).item() == 9          # an argmax over the logits would pick the higher index
    logits = x.cuda()
    labels = torch.tensor([3, 5, 8, 2, 0, 20], dtype=torch.int32, device="cuda")
    pred, correct = _top1(logits, labels)
    assert pred.tolist() == [3, 5, 8, 2, 0, 21]
    assert int(correct) == 5


def test_top1_non_finite_rows_and_padding():
    x = torch.randn(16, 50)
    x[1, 7] = float("nan")
    x[2, 0] = float("inf")
    x[3, 49] = float("-inf")
    x[4, :] = float("nan")
    logits = x.cuda()
    want, _ = _oracle_top1(x[5:])
    labels = torch.full((16,), -1, dtype=torch.int32)
    labels[5:] = torch.from_numpy(want).int()
    labels[0] = int(_oracle_top1(x[:1])[0][0])
    labels = labels.cuda()
    pred = torch.full((16,), 12345, dtype=torch.int32, device="cuda")
    correct = torch.full((1,), 100, dtype=torch.int64, device="cuda")
    _top1(logits, labels, n_valid=12, correct=correct, pred=pred)
    p = pred.tolist()
    assert p[1:5] == [-1, -1, -1, -1]              # non-finite: -1, not counted although labels are -1
    assert p[12:] == [12345] * 4                   # padding rows: never written
    assert int(correct) == 100 + 1 + 7             # row 0 and rows 5..11; padding rows 12..15 not counted
    _top1(logits, labels, n_valid=0, correct=correct, pred=pred)
    assert int(correct) == 108


def test_top1_graph_replay_and_streams_bit_identical():
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(256, 1024, generator=g) * 4).cuda()[:, :1001]
    labels = torch.randint(0, 1001, (256,), generator=g, dtype=torch.int32).cuda()
    labels[:128] = torch.from_numpy(_oracle_top1(logits[:128])[0]).int().cuda()
    pred0, c0 = _top1(logits, labels, n_valid=250)
    pred_g = torch.full((256,), -7, dtype=torch.int32, device="cuda")
    cg = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _top1(logits, labels, n_valid=250, correct=cg, pred=pred_g)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(pred_g[:250], pred0[:250]) and (pred_g[250:] == -7).all()
    assert int(cg) == 3 * int(c0)
    # two streams adding into one counter
    cs = torch.zeros(1, dtype=torch.int64, device="cuda")
    preds = [torch.empty(256, dtype=torch.int32, device="cuda") for _ in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    for st, pr in zip(streams, preds):
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            for _ in range(4):
                _top1(logits, labels, n_valid=250, correct=cs, pred=pr)
    torch.cuda.synchronize()
    assert int(cs) == 8 * int(c0)
    assert all(torch.equal(p[:250], pred0[:250]) for p in preds)


def test_tail_batch_padded_matches_exact_batch():
    from assembled_cnn_b200.model_fns import build_model
    model = build_model(resnet_size=50, num_classes=10)
    g = torch.Generator().manual_seed(37)
    x = torch.randint(0, 256, (37, 64, 64, 3), generator=g, dtype=torch.uint8).cuda()
    labels = torch.randint(0, 10, (37,), generator=g, dtype=torch.int32).cuda()
    rt37 = model.runtime(37, 64, 64, training=False)
    rt37.set_images_u8(x, _mean())
    rt37.run_forward()
    want, c37 = _top1(rt37.t[rt37.plan.meta["logits"]][:, :10], labels)
    rt64 = model.runtime(64, 64, 64, training=False)
    xp = torch.zeros(64, 64, 64, 3, dtype=torch.uint8, device="cuda")
    xp[:37] = x
    lp = torch.zeros(64, dtype=torch.int32, device="cuda")
    lp[:37] = labels
    lp[37:] = -3
    rt64.set_images_u8(xp, _mean())
    rt64.run_forward()
    pred = torch.full((64,), 999, dtype=torch.int32, device="cuda")
    _, c64 = _top1(rt64.t[rt64.plan.meta["logits"]][:, :10], lp, n_valid=37, pred=pred)
    assert torch.equal(pred[:37], want) and (pred[37:] == 999).all()
    assert int(c64) == int(c37)


# ------------------------------------------------------------------------------------ end to end
SYNSETS = ["n01440764", "n01443537", "n01484850"]


@pytest.fixture(scope="module")
def imagenet_c_tree(tmp_path_factory):
    from PIL import Image
    from assembled_cnn_b200.metrics import DISTORTIONS
    root = tmp_path_factory.mktemp("imagenet_c")
    (root / "labels.txt").write_text("background\n" + "\n".join(s.upper() for s in SYNSETS) + "\n")
    rng = np.random.default_rng(0)
    for d in DISTORTIONS:
        for s in range(1, 6):
            for k, syn in enumerate(SYNSETS):
                os.makedirs(root / "data" / d / str(s) / syn)
                for j in range(2):
                    base = rng.integers(0, 256, 3)
                    img = np.clip(base + rng.normal(0, 40 * s, (64, 64, 3)), 0, 255).astype(np.uint8)
                    Image.fromarray(img).save(root / "data" / d / str(s) / syn / ("%d.JPEG" % j), quality=90)
    return root


def _oracle_corruption_error(model, root, batch):
    """Per-distortion counts from Model(float images) logits (same runtime shape: batches padded to
    `batch`) and float64 softmax argmax; then the oracle's error / CE / mCE."""
    from assembled_cnn_b200 import imagenet_c
    from assembled_cnn_b200.metrics import DISTORTIONS
    from oracle import robustness as R
    syn = imagenet_c.get_synsets2idx(str(root / "labels.txt"))
    correct, count = {}, {}
    mean = _mean("cpu")
    for d in DISTORTIONS:
        files, labels = imagenet_c.distortion_images(str(root / "data"), d, syn, 1)
        c = 0
        for a in range(0, len(files), batch):
            u8 = torch.zeros(batch, 64, 64, 3, dtype=torch.uint8)
            n = len(files[a:a + batch])
            for i, f in enumerate(files[a:a + batch]):
                u8[i] = torch.from_numpy(imagenet_c.decode_image(f, 64))
            logits = model(u8.float() - mean, False)[:n].cpu()
            c += int((R.top1(logits.numpy()) == np.array(labels[a:a + batch])).sum())
        correct[d], count[d] = c, len(files)
    return R.mce(correct, count), correct


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_corruption_error_end_to_end(imagenet_c_tree, dtype):
    from assembled_cnn_b200.model_fns import build_model, corruption_error
    from assembled_cnn_b200.metrics import DISTORTIONS
    root = imagenet_c_tree
    model = build_model(resnet_size=50, num_classes=10, dtype=dtype)
    (m, mu, per), _ = _oracle_corruption_error(model, root, 8)
    kw = dict(batch_size=8, image_size=64, num_workers=4)
    got = corruption_error(model, str(root / "data"), str(root / "labels.txt"), global_step=1234, **kw)
    assert got["mCE"] == m and got["mCE_unnormalized"] == mu and got["global_step"] == 1234
    for d in DISTORTIONS:
        assert got[d] == {"error": per[d][0], "ce": per[d][1]}, d
    eager = corruption_error(model, str(root / "data"), str(root / "labels.txt"), use_cuda_graph=False, **kw)
    assert eager == {k: v for k, v in got.items() if k != "global_step"}


def test_corruption_error_two_devices(imagenet_c_tree):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from assembled_cnn_b200.model_fns import build_model, corruption_error
    root = imagenet_c_tree
    model = build_model(resnet_size=50, num_classes=10)
    kw = dict(batch_size=8, image_size=64)
    one = corruption_error(model, str(root / "data"), str(root / "labels.txt"), **kw)
    two = corruption_error(model, str(root / "data"), str(root / "labels.txt"), devices=["cuda:0", "cuda:1"], **kw)
    assert one == two
