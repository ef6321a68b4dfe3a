"""The equivalence the shared resampling kernel rests on: acnn_crop_resize_u8 of a window without flip equals
acnn_resize_crop_u8 of the same pixels resized to S x S and cropped at (0, 0), bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MEAN = (123.68, 116.78, 103.94)
SHAPES = [(1, 1), (1, 9), (9, 1), (500, 375), (375, 500), (33, 47), (224, 224), (300, 120), (2, 3), (700, 20)]


@pytest.mark.parametrize("S", [64, 224])
def test_crop_resize_without_flip_equals_resize_crop_at_origin(S):
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.imagenet_eval import DESC_DTYPE
    from assembled_cnn_b200.imagenet_train import CROP_DESC_DTYPE
    lib = _lib.load()
    rng = np.random.default_rng(S)
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in SHAPES]
    B = len(images)
    offs = np.cumsum([0] + [a.nbytes for a in images])
    buf = torch.from_numpy(np.concatenate([a.reshape(-1) for a in images])).cuda()
    crop, resize = np.zeros(B, CROP_DESC_DTYPE), np.zeros(B, DESC_DTYPE)
    for i, a in enumerate(images):
        addr = buf.data_ptr() + int(offs[i])
        crop[i] = (addr, a.shape[0], a.shape[1], 0, (0, 0, 0))
        resize[i] = (addr, a.shape[0], a.shape[1], S, S, 0, 0)
    dcrop, dresize = (torch.from_numpy(d.view(np.uint8).copy()).cuda() for d in (crop, resize))
    mean = torch.tensor(MEAN, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    a_out = torch.full((B, S, S, 3), 1.0, device="cuda")
    b_out = torch.full((B, S, S, 3), 2.0, device="cuda")
    _lib.check(lib.acnn_crop_resize_u8(dcrop.data_ptr(), B, B, S, mean.data_ptr(), a_out.data_ptr(), stream),
               "acnn_crop_resize_u8")
    _lib.check(lib.acnn_resize_crop_u8(dresize.data_ptr(), B, B, S, mean.data_ptr(), b_out.data_ptr(), stream),
               "acnn_resize_crop_u8")
    torch.cuda.synchronize()
    assert torch.equal(a_out.view(torch.int32), b_out.view(torch.int32))
