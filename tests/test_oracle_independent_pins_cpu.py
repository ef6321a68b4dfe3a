"""Independent pins of the TF-1.14 KERNEL semantics the oracle restates.

TensorFlow is not installable here (no wheel for this interpreter, no network), so the oracle cannot be
run against the reference's own kernels.  Besides the hand-computed vectors of
test_oracle_known_answers.py, every rule that is a convention rather than arithmetic is checked here
against an implementation written by SOMEBODY ELSE and validated against TensorFlow by its authors:

  * TF 'SAME' padding (total = max((ceil(n/s)-1)*s + k - n, 0), the odd cell AFTER): Hugging Face's
    `DynamicPad2d` / `BitMaxPool2d` (transformers.models.bit -- the port of Google's TF BiT checkpoints,
    whose logits only reproduce with TF's padding);
  * fused batch norm (biased variance to normalise, UNBIASED variance into the moving average, eps
    inside the sqrt): ATen's `torch.nn.BatchNorm2d` kernel, which documents exactly this behaviour;
  * label smoothing y(1-eps) + eps/K and the batch-mean reduction: ATen's `cross_entropy(label_smoothing=)`;
  * MomentumOptimizer (acc = m*acc + g; w -= lr*acc, L2 as wd*w in the gradient): `torch.optim.SGD`;
  * average pooling that excludes padded cells from the divisor (TF SAME avg-pool): ATen's
    `avg_pool2d(count_include_pad=False)`;
  * REFLECT padding (no edge repeat) + binomial blur: `scipy.ndimage.correlate(mode='mirror')` (odd
    filters) / `numpy.pad(mode='reflect')` + explicit windows (even filters);
  * nearest 2x up-sampling: `torch.nn.Upsample(scale_factor=2, mode='nearest')`.
The oracle's own functions never call these (oracle/tf_ops.py pads and reduces by hand)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import tf_ops as T


def _rand(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


@pytest.mark.parametrize("size", [7, 8, 13, 14, 16, 17, 28, 56])
@pytest.mark.parametrize("k,s", [(3, 2), (3, 1), (2, 1), (2, 2), (5, 2), (7, 2), (1, 2)])
def test_same_padding_rule_vs_hf_bit_port(size, k, s):
    from transformers.models.bit.modeling_bit import DynamicPad2d
    x = torch.ones(1, 1, size, size + 3)
    padded = DynamicPad2d(k, s, 1, value=0)(x)
    (pt, pb), (pl, pr) = T._same_pads(size, k, s), T._same_pads(size + 3, k, s)
    assert padded.shape[-2:] == (size + pt + pb, size + 3 + pl + pr)
    # where the zeros went: before / after per axis
    rows = (padded[0, 0, :, pl] == 0).nonzero().flatten().tolist()
    cols = (padded[0, 0, pt, :] == 0).nonzero().flatten().tolist()
    assert rows == list(range(pt)) + list(range(size + pt, size + pt + pb))
    assert cols == list(range(pl)) + list(range(size + 3 + pl, size + 3 + pl + pr))
    assert pb - pt in (0, 1) and pr - pl in (0, 1)          # the odd cell goes AFTER


@pytest.mark.parametrize("hw", [(8, 8), (9, 12), (15, 7), (112, 112)])
def test_max_pool_same_vs_hf_bit_port(hw):
    from transformers.models.bit.modeling_bit import BitMaxPool2d
    x = _rand(2, hw[0], hw[1], 5, seed=hw[0])
    got = T.max_pool_same(x, 3, 2)
    ref = BitMaxPool2d(3, stride=2, padding_value=float("-inf"))(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    assert got.shape == ref.shape == (2, math.ceil(hw[0] / 2), math.ceil(hw[1] / 2), 5)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("k,s,hw", [(3, 1, (9, 9)), (1, 1, (6, 7)), (3, 2, (8, 8)), (3, 2, (9, 11)),
                                     (7, 2, (16, 16)), (5, 1, (7, 6))])
def test_conv_same_and_fixed_padding_vs_hf_bit_port(k, s, hw):
    """conv2d(padding='SAME') against DynamicPad2d + a plain VALID correlation; and the reference's
    fixed_padding (nets/model_helper.py:40-64) differs from SAME exactly for even inputs at stride 2."""
    from transformers.models.bit.modeling_bit import DynamicPad2d
    x, w = _rand(2, hw[0], hw[1], 3, seed=k), _rand(k, k, 3, 4, seed=s)
    got = T.conv2d(x, w, s, "SAME")
    xp = DynamicPad2d(k, s, 1, value=0)(x.permute(0, 3, 1, 2))
    ref = F.conv2d(xp, w.permute(3, 2, 0, 1), stride=s).permute(0, 2, 3, 1)
    assert torch.allclose(got, ref, rtol=0, atol=1e-12)
    fixed = T.conv2d_fixed_padding(x, w, s)
    same_as_fixed = torch.allclose(fixed, got, rtol=0, atol=1e-12) if fixed.shape == got.shape else False
    if s == 1 or k == 1:
        assert same_as_fixed
    elif hw[0] % 2 == 0 and hw[1] % 2 == 0 and k > 1:
        assert not same_as_fixed          # 'SAME' pads (k-2)/2 | k/2, fixed_padding (k-1)/2 | (k-1)/2


@pytest.mark.parametrize("n", [2, 4, 64])
def test_batch_norm_vs_aten_kernel(n):
    C, mom, eps = 6, 0.997, 1e-5
    x = _rand(n, 5, 3, C, seed=n) * 3 + 1.5
    gamma, beta = 0.5 + torch.rand(C, dtype=torch.float64), _rand(C, seed=1)
    mm, mv = _rand(C, seed=2), 0.5 + torch.rand(C, dtype=torch.float64)
    bn = torch.nn.BatchNorm2d(C, eps=eps, momentum=1 - mom).double()
    with torch.no_grad():
        bn.weight.copy_(gamma), bn.bias.copy_(beta), bn.running_mean.copy_(mm), bn.running_var.copy_(mv)
    bn.train()
    ref = bn(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    y, nmm, nmv = T.batch_norm(x, gamma, beta, mm, mv, True, mom, eps)
    assert torch.allclose(y, ref, rtol=1e-10, atol=1e-10)
    assert torch.allclose(nmm, bn.running_mean, rtol=1e-12, atol=1e-12)
    assert torch.allclose(nmv, bn.running_var, rtol=1e-12, atol=1e-12)     # UNBIASED batch variance
    bn.eval()
    ref_e = bn(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    y_e, _, _ = T.batch_norm(x, gamma, beta, bn.running_mean, bn.running_var, False, mom, eps)
    assert torch.allclose(y_e, ref_e, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("ls", [0.0, 0.1, 0.3])
def test_label_smoothed_cross_entropy_vs_aten_kernel(ls):
    logits = _rand(16, 1001, seed=3).float() * 3
    labels = torch.randint(0, 1001, (16,), generator=torch.Generator().manual_seed(4))
    got = T.softmax_cross_entropy(logits, F.one_hot(labels, 1001).float(), ls)
    ref = F.cross_entropy(logits, labels, label_smoothing=ls)
    assert abs(float(got) - float(ref)) < 2e-6 * abs(float(ref))
    # soft (mixup) targets
    soft = 0.3 * F.one_hot(labels, 1001).float() + 0.7 * F.one_hot(labels.flip(0), 1001).float()
    got = T.softmax_cross_entropy(logits, soft, ls)
    ref = F.cross_entropy(logits, soft, label_smoothing=ls)
    assert abs(float(got) - float(ref)) < 2e-6 * abs(float(ref))


def test_momentum_sgd_with_l2_vs_torch_optimizer():
    """acc = m*acc + (g + wd*w); w -= lr*acc: run_loop_classification.py:166-179 puts wd * l2_loss in the
    loss, so the decay reaches the optimizer as wd*w inside the gradient."""
    lr, m, wd = 0.4, 0.9, 1e-4
    w0 = _rand(50, seed=5)
    w, acc = w0.clone(), torch.zeros_like(w0)
    p = torch.nn.Parameter(w0.clone())
    opt = torch.optim.SGD([p], lr=lr, momentum=m, weight_decay=wd)
    for step in range(4):
        g = _rand(50, seed=10 + step)
        assert abs(float(wd * T.l2_loss(w)) - float(wd * 0.5 * (w ** 2).sum())) < 1e-6
        w, acc = T.momentum_step(w, acc, g + wd * w, lr, m)
        p.grad = g.clone()
        opt.step()
        assert torch.allclose(w, p.detach(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("hw", [(6, 6), (7, 9), (14, 14)])
def test_avg_pool_same_excludes_padding_vs_aten_kernel(hw):
    """resnet-D stride-1 shortcut (nets/resnet_model.py:126): 2x2 SAME average pool; TF divides by the
    number of in-image cells.  ATen pads symmetrically, so pad 1 on both sides and drop the first
    row / column: what is left are the windows [i, i+1] with the pad cell AFTER, divisor excluding it."""
    x = _rand(2, hw[0], hw[1], 3, seed=hw[1])
    got = T.avg_pool_resnet_d(x, 1)
    ref = F.avg_pool2d(x.permute(0, 3, 1, 2), 2, 1, padding=1, count_include_pad=False)[:, :, 1:, 1:]
    assert got.shape == x.shape
    assert torch.allclose(got, ref.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    # strided variants count the padded zeros (always /4, /9): plain VALID pooling of the padded image
    for fn, k in ((T.avg_pool_resnet_d, 2), (T.avg_pool_bl, 3)):
        lo = (k - 1) // 2
        xp = F.pad(x.permute(0, 3, 1, 2), (lo, k - 1 - lo, lo, k - 1 - lo))
        ref = F.avg_pool2d(xp, k, 2, count_include_pad=True).permute(0, 2, 3, 1)
        assert torch.allclose(fn(x, 2), ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("filt,stride", [(3, 2), (5, 2), (3, 1), (2, 2), (7, 2)])
def test_blur_pool_vs_scipy_mirror_correlate(filt, stride):
    """nets/blocks.py:45-107: tf.pad(mode='REFLECT') + binomial depthwise filter + stride.  scipy's
    'mirror' boundary is numpy 'reflect' (d c b | a b c d | c b a) = TF REFLECT."""
    from scipy import ndimage
    x = _rand(1, 10, 12, 2, seed=filt)
    got = T.anti_aliased_downsample(x, filt, stride)
    a = np.array(T._BINOMIAL[filt])
    f2 = np.outer(a, a) / np.outer(a, a).sum()
    p = int((filt - 1) / 2)
    for c in range(2):
        img = x[0, :, :, c].numpy()
        if filt % 2:
            # odd filter: centred correlation over the mirrored image, then the stride
            want = ndimage.correlate(img, f2, mode="mirror")[::stride, ::stride]
        else:
            # even filter (p before, p after: one cell short of 'same'): numpy's own reflect padding
            # + explicit VALID windows
            pad = np.pad(img, p, mode="reflect")
            full = np.array([[(pad[i:i + filt, j:j + filt] * f2).sum()
                              for j in range(pad.shape[1] - filt + 1)]
                             for i in range(pad.shape[0] - filt + 1)])
            want = full[::stride, ::stride]
        assert np.allclose(got[0, :, :, c].numpy(), want, rtol=1e-12, atol=1e-12), (filt, stride, c)


def test_upsample_nearest_vs_torch_module():
    x = _rand(2, 3, 5, 4, seed=9)
    ref = torch.nn.Upsample(scale_factor=2, mode="nearest")(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    assert torch.equal(T.upsample2x(x), ref)
