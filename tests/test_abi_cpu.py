"""CPU checks of the boundary: the C-ABI library builds, loads and exports every symbol that
include/acnn.h declares (no compute calls without a GPU), the host logic (flags, LR schedule)
matches the reference, and the product path refuses to run without its CUDA library / device."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_build_and_symbols():
    import __graft_entry__ as ge
    ge.build()
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "acnn.h")).read()
    header = re.sub(r"/\*.*?\*/", " ", header, flags=re.S)
    declared = set(re.findall(r"\b(acnn_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 40
    assert declared == set(_lib.PROTOTYPES)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.acnn_version() >= 100
    assert lib.acnn_launch_count() == 0 or lib.acnn_launch_count() > 0
    # the library must not depend on libcuda at load time (driver entry points are fetched lazily)
    out = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out
    # struct layouts the ABI passes by pointer
    assert ctypes.sizeof(_lib.ConvGeom) == 64 and ctypes.sizeof(_lib.WeightDesc) == 40


def test_sass_uses_wgmma_and_tma():
    """The conv kernels really are wgmma/TMA code (sm_90a SASS mnemonics)."""
    from assembled_cnn_b200 import _lib
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", os.path.join(ROOT, "assembled_cnn_b200", "build",
                                                             "gemm.o")],
                          capture_output=True, text=True).stdout
    assert "HGMMA" in sass            # wgmma.mma_async (bf16 -> fp32)
    assert "UTMALDG" in sass          # TMA tensor loads (tiled + im2col)
    assert "UTMASTG" in sass          # TMA tensor stores of the staged epilogue tiles
    assert "HMMA.16816" not in sass   # no legacy (mma.sync) tensor path


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.model_fns import build_model
    m = build_model(resnet_size=50, resnet_version=1)
    with pytest.raises(_lib.AcnnError):
        m(torch.zeros(1, 64, 64, 3), training=False)


def test_model_argument_errors_match_reference():
    from assembled_cnn_b200.model_fns import Model, get_block_sizes, build_model
    with pytest.raises(ValueError):
        Model(50, resnet_version=3)
    with pytest.raises(NotImplementedError):
        Model(18)
    with pytest.raises(ValueError):
        Model(50, dtype="fp8")
    with pytest.raises(ValueError):
        get_block_sizes(51, 1)
    assert get_block_sizes(152, 2) == [5, 12, 30, 3] and get_block_sizes(200, 1) == [3, 24, 36, 3]
    with pytest.raises(TypeError):
        build_model(resnet_size=50, not_a_flag=1)
    m = build_model(resnet_size=50, use_sk_block=True, use_resnet_d=True, anti_alias_type="sconv",
                    anti_alias_filter_size=3)
    assert m.use_resnet_d and m.cfg_kwargs["use_sk_block"]


def test_flag_defaults_match_reference():
    from assembled_cnn_b200.hparams import DEFAULTS, params_from_flags
    # nets/hparams_config.py / official/utils/flags defaults
    assert DEFAULTS["resnet_version"] == 1 and DEFAULTS["bl_alpha"] == 2 and DEFAULTS["bl_beta"] == 4
    assert DEFAULTS["weight_decay"] == 4e-5 and DEFAULTS["momentum"] == 0.9
    assert DEFAULTS["bn_momentum"] == 0.997 and DEFAULTS["label_smoothing"] == 0.0
    assert DEFAULTS["learning_rate_decay_type"] == "exponential" and DEFAULTS["base_learning_rate"] == 0.01
    p = params_from_flags(use_sk_block=True)
    assert p["use_sk_block"] and not p["use_se_block"]
    with pytest.raises(KeyError):
        params_from_flags(bogus=1)


def test_learning_rate_schedule_matches_oracle():
    from assembled_cnn_b200.model_fns import learning_rate_with_decay, keep_prob_decay
    from oracle import tf_ops as T
    for decay in ("exponential", "fixed", "polynomial", "piecewise", "cosine"):
        fn = learning_rate_with_decay(decay, 1024, 1024, 1281167, 2.0, 0.94, 1e-4, [30, 60, 80, 90],
                                      [1, 0.1, 0.01, 0.001, 1e-4], 0.4, warmup_epochs=5,
                                      train_epochs=600)
        for step in (0, 10, 6254, 6255, 50000, 400000, 750000):
            want = T.learning_rate(step, decay_type=decay, batch_size=1024, num_images=1281167,
                                   base_lr=0.4, warmup_epochs=5, train_epochs=600)
            assert abs(fn(step) - want) < 1e-12, (decay, step)
    kp = keep_prob_decay(1.0, 0.9, 1000)
    assert kp(0) == 1.0 and abs(kp(500) - 0.95) < 1e-12 and abs(kp(5000) - 0.9) < 1e-12


def test_sk_fc_scratch_formula_matches_library():
    """plan.py sizes the scratch of the fused SK attention chains with a Python mirror of
    acnn_sk_fc_scratch_floats (a pure host function: no GPU needed)."""
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.plan import sk_fc_scratch_floats
    lib = _lib.load()
    for B in (1, 2, 5, 12, 64, 128, 256, 300):
        for f in (64, 128, 256, 512, 96):
            d = max(f // 2, 32)
            assert lib.acnn_sk_fc_scratch_floats(B, f, d) == sk_fc_scratch_floats(B, f, d), (B, f)


def test_conv_wgrad_plan_properties():
    """acnn_conv_wgrad_plan (host only: the SM count is the H100's 132 without a device) against
    the rules include/acnn.h states, over a grid of geometries and both precisions: one split when
    deterministic, a stage partition whose last split is non-empty, the partial tiles within 64 MiB,
    the documented pixels per stage, and a forced split count honoured within the capacity caps."""
    import ctypes as C
    from assembled_cnn_b200 import _lib
    lib = _lib.load()

    def plan(g, precision, det):
        pix, splits, sps = C.c_int(), C.c_int(), C.c_int()
        _lib.check(lib.acnn_conv_wgrad_plan(g, precision, det, C.byref(pix), C.byref(splits),
                                            C.byref(sps)), "acnn_conv_wgrad_plan")
        return pix.value, splits.value, sps.value

    geoms = []
    for B in (1, 3, 32, 256):
        for H in (7, 14, 56):
            for Cin, Cout in ((16, 32), (64, 64), (32, 128), (64, 256), (256, 512), (2048, 1024)):
                for k, stride in ((1, 1), (3, 1), (3, 2), (1, 2)):
                    p = (k - 1) // 2
                    geoms.append(_lib.ConvGeom(B, H, H, Cin, Cout, k, k, stride, p, k - 1 - p, p,
                                               k - 1 - p))
    n_split = 0
    prev_s, prev_p = lib.acnn_set_wgrad_splits(0), lib.acnn_set_wgrad_pixels(0)
    try:
        for g in geoms:
            Ho, Wo = g.out_hw()
            P = g.B * Ho * Wo
            # the partial tiles of one split: ceil(Ktot / 128) x 128 rows by Cout columns (fp32)
            split_bytes = -(-g.kh * g.kw * g.Cin // 128) * 128 * g.Cout * 4
            for precision in (0, 1):
                pix, splits, sps = plan(g, precision, 0)
                assert pix == (128 if precision == 0 and g.Cout < 256 and P >= 4096 else 64)
                stages = -(-P // pix)
                assert splits * sps >= stages > (splits - 1) * sps >= 0
                assert splits == 1 or splits * split_bytes <= 64 << 20
                n_split += splits > 1
                assert plan(g, precision, 1) == (pix, 1, stages)
                lib.acnn_set_wgrad_pixels(64)
                assert plan(g, precision, 0)[0] == 64
                lib.acnn_set_wgrad_pixels(0)
                for n in (1, 2, 3, 7, 1000):
                    lib.acnn_set_wgrad_splits(n)
                    want = max(min(n, stages, (64 << 20) // split_bytes), 1)
                    want = -(-stages // -(-stages // want))      # re-normalised: no empty split
                    assert plan(g, precision, 0) == (pix, want, -(-stages // want)), (n, P)
                    assert plan(g, precision, 1) == (pix, 1, stages)
                lib.acnn_set_wgrad_splits(0)
    finally:
        lib.acnn_set_wgrad_splits(prev_s)
        lib.acnn_set_wgrad_pixels(prev_p)
    assert n_split > len(geoms) // 4          # the default cost model does split
    assert lib.acnn_set_wgrad_splits(0) == 0
