"""CPU checks of the servable's batch ladder: every argument error of batch_sizes is raised before any GPU
work, a request of each size 0 .. 2 * max_batch + 1 is cut into the expected rung chunks, and the
acnn_set_fc_split_rows knob leaves the layer plans of the pinned configurations as they are."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LADDER = (1, 8, 64, 256)


@pytest.mark.parametrize("sizes, match", [
    ((), "positive ints"), ((0, 8), "positive ints"), ((-1, 8), "positive ints"), ((1.0, 8), "positive ints"),
    ((True, 8), "positive ints"), (("1", 8), "positive ints"), ((4, 2, 8), "strictly increasing"),
    ((4, 4, 8), "strictly increasing"), ((1, 4), "largest"), ((1, 16), "largest")])
def test_batch_sizes_errors_before_gpu(sizes, match, tmp_path):
    from assembled_cnn_b200.model_fns import Servable, build_model, load_servable
    model = build_model(resnet_size=50, num_classes=10)
    with pytest.raises(ValueError, match=match):
        Servable(model, image_size=64, max_batch=8, batch_sizes=sizes)
    # load_servable checks them before it reads the directory
    with pytest.raises(ValueError, match=match):
        load_servable(str(tmp_path / "missing"), max_batch=8, batch_sizes=sizes)
    assert model._runtimes == {} and model._primary == {}


def test_batch_sizes_accepted():
    from assembled_cnn_b200.model_fns import Servable, build_model
    model = build_model(resnet_size=50, num_classes=10)
    assert Servable(model, max_batch=256).batch_sizes == (256,)
    sv = Servable(model, max_batch=256, batch_sizes=[np.int64(1), 8, 64, 256])
    assert sv.batch_sizes == LADDER and all(type(b) is int for b in sv.batch_sizes)
    assert Servable(model, max_batch=5, batch_sizes=(5,)).batch_sizes == (5,)
    assert sv._pipe is None and model._runtimes == {}


@pytest.mark.parametrize("sizes", [LADDER, (256,), (3, 7, 10)])
def test_rung_of_every_request_size(sizes):
    from assembled_cnn_b200.model_fns import ladder_chunks
    top = sizes[-1]
    for n in range(0, 2 * top + 2):
        chunks = ladder_chunks(n, sizes)
        assert [a for _, a, _ in chunks] == list(range(0, n, top))
        assert all(b - a == (top if a + top <= n else n - a) for _, a, b in chunks)
        for rung, a, b in chunks:
            # the smallest rung that holds the chunk
            assert b - a <= rung and all(r < b - a for r in sizes if r < rung), (n, rung, a, b)
        if sizes == LADDER:
            tail = n % 256
            want_tail = 1 if tail == 1 else 8 if 2 <= tail <= 8 else 64 if 9 <= tail <= 64 else 256
            assert [r for r, _, _ in chunks] == [256] * (n // 256) + ([want_tail] if tail else [])


def test_fc_split_rows_knob_leaves_plans_unchanged():
    """The knob is read at acnn_bind: the layer plan text of the pinned configurations (eval at batch 1 and
    8, and the training plan) is the same with it set, those plans still resolve into launch records, and
    it defaults to 0 and returns the previous value."""
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.native import NativeModel
    from assembled_cnn_b200.plan import ModelConfig
    lib = _lib.load()
    c3 = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)
    configs = [(dict(resnet_size=50), B, dict(training=False)) for B in (1, 8)]
    configs += [(c3, B, dict(training=False)) for B in (1, 8)]
    configs += [(dict(resnet_size=50, use_se_block=True), 8, dict(training=False)),
                (c3, 4, dict(training=True, mixup_type=1, label_smoothing=0.1))]
    plain = [NativeModel(ModelConfig(**f), B, 224, 224, **kw).dump() for f, B, kw in configs]
    assert lib.acnn_set_fc_split_rows(256) == 0
    try:
        assert lib.acnn_set_fc_split_rows(256) == 256
        for (f, B, kw), text in zip(configs, plain):
            nm = NativeModel(ModelConfig(**f), B, 224, 224, **kw)
            assert nm.dump() == text
            nm.validate()
    finally:
        assert lib.acnn_set_fc_split_rows(-3) == 256
    assert lib.acnn_set_fc_split_rows(0) == 0
