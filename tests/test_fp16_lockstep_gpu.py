"""GPU parity of the fp16 mode, op by op: test_plan_gpu.lockstep on fp16 plans (dtype='fp16': fp16
activation / gradient storage, f16 wgmma GEMMs) against the float64 plan interpreter that rounds every
stored fp16 tensor and every GEMM weight to fp16 (round to nearest even, overflow to inf).  After every op
its outputs are compared and then overwritten with the interpreter's, so each kernel is checked on
identical inputs -- including the op kinds no op-level test covers in fp16 (SE, KD teacher labels,
grad_combine, DropBlock masks, the space-to-depth stem and the dgrad add / mask epilogue).

Tolerances relative to each output's largest magnitude: fp16 tensors 2^-10 (one fp16 ulp at the top of
the range: an fp32 summation-order difference can flip one rounding); fp32 slots, gradients and partial
rows test_plan_gpu.F32_TOL, fp32 tensors and moving statistics 1e-4 -- the bf16 lock-step's bounds.

The backward runs at the reference's static loss scale of 128 (its fp16 recipes' scale), once at scale 1.
`python tests/test_fp16_lockstep_gpu.py [run ...]` prints the worst error per op kind and output of each
run in fp16 next to the same run in bf16.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import pytest

import test_plan_gpu as P

pytestmark = pytest.mark.gpu

_ASSEMBLE = P.CONFIGS["assemble_rv2_sk_sconv_mix1"][0]

# name -> (model flags, use_resnet_d, lockstep keyword arguments)
RUNS = {
    **{name + "_ls128": (kw, d, dict(mix=mix, loss_scale=128.0))
       for name, (kw, d, mix) in P.CONFIGS.items()},
    # the unscaled backward (a power-of-two scale is exact only where no fp16 value overflows or is
    # subnormal)
    "assemble_rv2_sk_sconv_mix1_ls1": (_ASSEMBLE, False, dict(mix=1, loss_scale=1.0)),
    # gem, gem_bwd, kd_teacher (mixup 2: the teacher-label quirk)
    "gem_embedding_kd_mix2": (P.FEATURE_CONFIGS["gem_embedding_kd_mix2"]["cfg"], False,
                              dict(mix=2, kd_temp=2.0, loss_scale=128.0)),
    # grad_combine (the flatten head's gradient is a view)
    "flatten_kd_rv1": (dict(resnet_size=50, resnet_version=1, pool_type="flatten"), False,
                       dict(mix=1, kd_temp=1.0, loss_scale=128.0)),
    # dropblock_mask / _apply; at 224 px the 56 x 56 stage, where the default conv settings pick the
    # halo kernel
    "dropblock_assemble_224": (_ASSEMBLE, False, dict(use_dropblock=True, B=4, HW=224, loss_scale=128.0)),
    # ragged tiles: batch 3, 64 x 96
    "assemble_b3_64x96": (_ASSEMBLE, False, dict(B=3, HW=(64, 96), mix=0, loss_scale=128.0)),
    # the inference path
    "assemble_eval": (_ASSEMBLE, False, dict(B=2, mix=0, training=False)),
}


def build_run_plan(name, dtype="fp16"):
    """The plan lockstep() builds for run `name` (no GPU needed)."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    kw, d, ls = RUNS[name]
    HW = ls.get("HW", 64)
    H, W = (HW, HW) if isinstance(HW, int) else HW
    return build_plan(ModelConfig(use_resnet_d=d, **kw), ls.get("B", 4), H, W,
                      training=ls.get("training", True), mixup_type=ls.get("mix", 0), label_smoothing=0.1,
                      dtype=dtype, use_dropblock=ls.get("use_dropblock", False), kd_temp=ls.get("kd_temp", 0.0))


def run(name, dtype="fp16", **extra):
    kw, d, ls = RUNS[name]
    args = dict(ls, **extra)
    if dtype != "fp16":
        args.pop("loss_scale", None)
    return P.lockstep(kw, d, dtype=dtype, **args)


def _report(name, worst):
    print("fp16 lock-step %s: worst rel err per op kind:output" % name)
    for k, v in sorted(worst.items()):
        print("  %-28s %.3e" % (k, v))


@pytest.mark.parametrize("name", [n for n in RUNS if n != "dropblock_assemble_224"])
def test_fp16_lockstep(name):
    failures, worst = run(name)
    _report(name, worst)
    assert not failures, "\n".join(failures[:20])


def test_fp16_lockstep_dropblock_224_on_the_halo_kernel(lib):
    """DropBlock at 224 px, and at least one fp16 conv of the run on the halo kernel: its partial-statistics
    row count (a function of the kernel the launcher picks) differs from the im2col kernel's."""
    halo = []

    def hook(plan, rt):
        for op, native_op in zip(plan.forward, rt.plan.forward):
            g = op.a.get("geom")
            if op.kind != "conv" or op.a.get("x_wpad") or g.kh != 3 or g.stride != 1:
                continue
            geom = rt.plan.conv_info(native_op)[0]
            prev = lib.acnn_set_conv_halo(0)
            try:
                n_im2col = lib.acnn_conv_stats_parts(geom)
            finally:
                lib.acnn_set_conv_halo(prev)
            if lib.acnn_conv_stats_parts(geom) != n_im2col:
                halo.append(g.astuple())

    failures, worst = run("dropblock_assemble_224", plan_hook=hook)
    _report("dropblock_assemble_224", worst)
    assert halo, "no 3x3 conv of the 224 px plan runs on the halo kernel"
    assert not failures, "\n".join(failures[:20])


if __name__ == "__main__":
    # --bf16 / --fp16: only that mode's column
    names = [a for a in sys.argv[1:] if not a.startswith("--")] or list(RUNS)
    for n in names:
        w16 = run(n, "fp16")[1] if "--bf16" not in sys.argv else {}
        wbf = run(n, "bf16")[1] if "--fp16" not in sys.argv else {}
        print("===== %s: worst rel err, fp16 (bound 2^-10 = %.2e on fp16 tensors) vs bf16 (2^-7 = %.2e)"
              % (n, P.F16_TOL, P.BF16_TOL), flush=True)
        for k in sorted(set(w16) | set(wbf)):
            a, b = w16.get(k), wbf.get(k)
            print("  %-28s %10s %10s" % (k, "%.3e" % a if a is not None else "-",
                                         "%.3e" % b if b is not None else "-"), flush=True)
