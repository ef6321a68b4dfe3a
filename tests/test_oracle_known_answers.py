"""Known-answer micro-vectors that pin the oracle to the TF-1.14 semantics the reference relies on
.  The reference ships no tests for this path and TensorFlow 1.14 cannot be installed,
so these hand-computed vectors are one of three pins of the TF kernel semantics (see the header of
oracle/tf_ops.py): the others are third-party implementations rule by rule
(tests/test_oracle_independent_pins_cpu.py) and the reference's own model code executed on third-party
kernels in float64 (tests/test_reference_shim_golden_cpu.py)."""
import math

import torch

from oracle import model as M
from oracle import tf_ops as T


def test_strided_conv_uses_fixed_padding_not_tf_same():
    # 3x3 stride 2 on 4x4 ones, all-ones kernel: fixed_padding pads 1 before AND after
    # (nets/model_helper.py:53-63) -> windows start at -1 and 1.  TF-SAME would pad 0/1.
    x = torch.ones(1, 4, 4, 1)
    w = torch.ones(3, 3, 1, 1)
    y = T.conv2d_fixed_padding(x, w, 2)[0, :, :, 0]
    assert y.tolist() == [[4.0, 6.0], [6.0, 9.0]]
    # 1x1 stride 2 picks pixels 0, 2, ...
    x = torch.arange(16.0).view(1, 4, 4, 1)
    y = T.conv2d_fixed_padding(x, torch.ones(1, 1, 1, 1), 2)[0, :, :, 0]
    assert y.tolist() == [[0.0, 2.0], [8.0, 10.0]]


def test_stride1_conv_is_same():
    x = torch.ones(1, 3, 3, 1)
    y = T.conv2d_fixed_padding(x, torch.ones(3, 3, 1, 1), 1)[0, :, :, 0]
    assert y.tolist() == [[4.0, 6.0, 4.0], [6.0, 9.0, 6.0], [4.0, 6.0, 4.0]]


def test_kernel_layout_is_hwio():
    x = torch.zeros(1, 2, 2, 2)
    x[0, 0, 0, 1] = 1.0
    w = torch.zeros(1, 1, 2, 3)
    w[0, 0, 1, 2] = 5.0            # in-channel 1 -> out-channel 2
    y = T.conv2d_fixed_padding(x, w, 1)
    assert y[0, 0, 0].tolist() == [0.0, 0.0, 5.0]


def test_batch_norm_training_biased_norm_unbiased_moving():
    x = torch.tensor([1.0, 2.0, 3.0, 6.0]).view(4, 1, 1, 1)
    g, b = torch.tensor([2.0]), torch.tensor([0.5])
    mm, mv = torch.tensor([10.0]), torch.tensor([4.0])
    y, nmm, nmv = T.batch_norm(x, g, b, mm, mv, True, momentum=0.9, eps=1e-5)
    mean, var_b = 3.0, 3.5                    # biased variance: ((4+1+0+9)/4)
    want = [(v - mean) / math.sqrt(var_b + 1e-5) * 2 + 0.5 for v in (1, 2, 3, 6)]
    assert torch.allclose(y.flatten(), torch.tensor(want), atol=1e-6)
    assert abs(nmm.item() - (10 * 0.9 + 3.0 * 0.1)) < 1e-6
    var_u = 14.0 / 3.0                        # Bessel-corrected for the moving average
    assert abs(nmv.item() - (4 * 0.9 + var_u * 0.1)) < 1e-6
    y_eval, _, _ = T.batch_norm(x, g, b, mm, mv, False, eps=1e-5)
    assert abs(y_eval[0].item() - ((1 - 10) / math.sqrt(4 + 1e-5) * 2 + 0.5)) < 1e-6


def test_max_pool_same_pads_after():
    # 4x4, 3x3 s2 SAME -> 2x2; TF pads 0 before / 1 after: windows rows {0,1,2} and {2,3}
    x = torch.arange(16.0).view(1, 4, 4, 1)
    y = T.max_pool_same(x)[0, :, :, 0]
    assert y.tolist() == [[10.0, 11.0], [14.0, 15.0]]
    # a "pad 1 before" pool (PyTorch default) would have given [[5,7],[13,15]]
    x = -torch.ones(1, 4, 4, 1)               # padding is -inf, never wins
    assert T.max_pool_same(x).max().item() == -1.0


def test_avg_pool_variants():
    x = torch.arange(16.0).view(1, 4, 4, 1)
    # resnet-d, stride 2: plain 2x2 / 4
    y = T.avg_pool_resnet_d(x, 2)[0, :, :, 0]
    assert y.tolist() == [[2.5, 4.5], [10.5, 12.5]]
    # resnet-d, stride 1: 2x2 SAME, padded cells excluded from the divisor
    y = T.avg_pool_resnet_d(x, 1)[0, :, :, 0]
    assert y[0, 0].item() == 2.5 and y[0, 3].item() == (3 + 7) / 2 and y[3, 3].item() == 15.0
    assert y[3, 0].item() == (12 + 13) / 2
    # bl, stride 2: zero pad 1/1, 3x3 VALID, zeros COUNTED (always / 9)
    y = T.avg_pool_bl(x, 2)[0, :, :, 0]
    assert abs(y[0, 0].item() - (0 + 1 + 4 + 5) / 9) < 1e-6
    assert abs(y[1, 1].item() - (5 + 6 + 7 + 9 + 10 + 11 + 13 + 14 + 15) / 9) < 1e-6
    assert T.avg_pool_bl(x, 1) is x


def test_blur_pool_reflect():
    x = torch.arange(16.0).view(1, 4, 4, 1)
    y = T.anti_aliased_downsample(x, 3, 2)[0, :, :, 0]
    # row/col taps [1,2,1]/4 at input offsets (-1,0,1) with reflection: index -1 -> 1
    def tap(v):      # 1-D blur of a length-4 vector at output positions 0, 1
        return [(v[1] + 2 * v[0] + v[1]) / 4, (v[1] + 2 * v[2] + v[3]) / 4]
    rows = [tap([x[0, r, c, 0].item() for c in range(4)]) for r in range(4)]
    want = [tap([rows[r][c] for r in range(4)]) for c in range(2)]
    assert torch.allclose(y, torch.tensor(want).t(), atol=1e-6)
    assert y[0, 0].item() == 2.5             # (1+0+1)/.. worked by hand: rows->[0.5,2.25], ...


def test_upsample_nearest():
    x = torch.tensor([[1.0, 2.0], [3.0, 4.0]]).view(1, 2, 2, 1)
    y = T.upsample2x(x)[0, :, :, 0]
    assert y.tolist() == [[1, 1, 2, 2], [1, 1, 2, 2], [3, 3, 4, 4], [3, 3, 4, 4]]


def test_sk_attention_is_two_way_softmax_over_halves():
    torch.manual_seed(0)
    B, H, f, d = 4, 3, 4, 32
    u = torch.rand(B, H, H, 2 * f)
    w1, w2 = torch.randn(f, d), torch.randn(d, 2 * f)
    g, b, mm, mv = torch.ones(d), torch.zeros(d), torch.zeros(d), torch.ones(d)
    v, _, _ = T.sk_attention(u, w1, g, b, mm, mv, w2, True, 0.997)
    s = (u[..., :f] + u[..., f:]).mean((1, 2))
    z = s @ w1
    z = torch.relu((z - z.mean(0)) / torch.sqrt(z.var(0, unbiased=False) + 1e-5))
    a = z @ w2
    a0 = torch.sigmoid(a[:, :f] - a[:, f:])          # softmax over two == sigmoid of difference
    want = u[..., :f] * a0[:, None, None] + u[..., f:] * (1 - a0)[:, None, None]
    assert torch.allclose(v, want, atol=1e-5)


def test_se_block():
    x = torch.rand(2, 3, 3, 32)
    w1, w2 = torch.randn(32, 2), torch.randn(2, 32)
    e = torch.sigmoid(torch.relu(x.mean((1, 2)) @ w1) @ w2)
    assert torch.allclose(T.se_block(x, w1, w2), x * e[:, None, None])


def test_label_smoothing_divides_by_num_classes():
    logits = torch.tensor([[2.0, 0.0, -1.0]])
    onehot = torch.tensor([[1.0, 0.0, 0.0]])
    eps = 0.1
    lsm = torch.log_softmax(logits, 1)[0]
    yp = [1 - eps + eps / 3, eps / 3, eps / 3]
    want = -sum(y * l.item() for y, l in zip(yp, lsm))
    assert abs(T.softmax_cross_entropy(logits, onehot, eps).item() - want) < 1e-6
    # mean over the batch
    l2 = T.softmax_cross_entropy(torch.cat([logits, logits]), torch.cat([onehot, onehot]), eps)
    assert abs(l2.item() - want) < 1e-6


def test_mixup_types():
    x = torch.arange(4.0).view(4, 1, 1, 1)
    y = torch.eye(4)
    lam1 = torch.tensor([0.25, 1.0])
    mx, my = T.mixup(x, y, lam1, keep_batch_size=False)           # type 1: 2B -> B
    assert mx.flatten().tolist() == [0.25 * 0 + 0.75 * 2, 1.0]
    assert my[0].tolist() == [0.25, 0, 0.75, 0]
    lam2 = torch.tensor([0.5, 0.0])
    mx, my = T.mixup(x, y, lam1, lam2, keep_batch_size=True)      # type 2: second half vs reversed
    assert mx.flatten().tolist() == [1.5, 1.0, 0.5 * 0 + 0.5 * 3, 2.0]
    assert my[2].tolist() == [0.5, 0, 0, 0.5]


def test_momentum_and_l2():
    w, acc, g = torch.tensor([1.0]), torch.tensor([0.5]), torch.tensor([2.0])
    w2, acc2 = T.momentum_step(w, acc, g, lr=0.1, momentum=0.9)
    assert abs(acc2.item() - 2.45) < 1e-6 and abs(w2.item() - (1 - 0.245)) < 1e-6
    assert T.l2_loss(torch.tensor([3.0, 4.0])).item() == 12.5


def test_learning_rate_schedules():
    kw = dict(batch_size=256, num_images=1281167, base_lr=0.4)
    bpe = 1281167 / 256
    lr = T.learning_rate(100, decay_type="cosine", warmup_epochs=5, train_epochs=600, **kw)
    assert abs(lr - 0.4 * 100 / int(bpe * 5)) < 1e-9
    total = int(bpe * 600) - int(bpe * 5)
    lr = T.learning_rate(int(bpe * 5) + total // 2, decay_type="cosine", warmup_epochs=5,
                         train_epochs=600, **kw)
    assert abs(lr - 0.2) < 1e-4
    assert T.learning_rate(7, decay_type="fixed", **kw) == 0.4
    lr = T.learning_rate(int(bpe * 2) * 3 + 1, decay_type="exponential", **kw)
    assert abs(lr - 0.4 * 0.94 ** 3) < 1e-9


def test_parameter_inventory_matches_survey():
    """Totals: trainable tensors / parameters / BN layers per configuration."""
    cases = [
        (dict(resnet_size=50, resnet_version=1), False, 161, 25_559_081, 53),
        (dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
              anti_alias_filter_size=3), False, 306, 41_848_489, 95),
        (dict(resnet_size=50, resnet_version=1, use_sk_block=True, anti_alias_type="sconv",
              anti_alias_filter_size=3), True, 231, 38_793_097, 71),
    ]
    for kw, d, n_tr, n_par, n_bn in cases:
        _, vs = M.build(use_resnet_d=d, input_hw=64, **kw)
        tr = [n for n in vs.vars if vs.trainable[n]]
        assert len(tr) == n_tr
        assert sum(vs.vars[n].numel() for n in tr) == n_par
        assert sum(1 for n in vs.vars if n.endswith("moving_mean")) == n_bn
    # weight decay set: everything but BN gamma/beta (includes dense/bias and SK fc kernels)
    dec = [n for n in tr if M.decayed(n)]
    assert "resnet_model/dense/bias" in dec and not any(n.endswith("gamma") for n in dec)


def test_block_layer_ignores_last_relu_for_single_block():
    """nets/resnet_model.py:151-155: the first block call never receives last_relu=False."""
    m, vs = M.build(resnet_size=50, resnet_version=2, input_hw=64)
    x = torch.randn(2, 8, 8, 64)
    with torch.no_grad():
        with vs.scope("probe"):
            vs.creating = True
            y = m._block_layer(vs, x, 16, 1, 1, True, use_bl=True, last_relu=False)
    assert (y >= 0).all()
