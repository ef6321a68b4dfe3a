"""Dynamic loss scaling without a GPU: the "dynamic" spelling of loss_scale and the errors raised before any GPU
work, a numpy restatement of the scale's state machine (TF 2 Keras' LossScaleOptimizer) against hand-worked
sequences, the new entry points in the headers and their ctypes declarations, and the checkpoint keys."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------ the state machine
def update(state, nonfinite, growth_interval):
    """One step of the rules of include/acnn.h (acnn_loss_scale_state) on (scale, good_steps, skipped_steps),
    the scale as float32: the scale the step used and the new state."""
    scale, good, skipped = np.float32(state[0]), int(state[1]), int(state[2])
    if nonfinite:
        return scale, (max(scale / np.float32(2), np.float32(1)), 0, skipped + 1)
    good += 1
    if good >= growth_interval:
        with np.errstate(over="ignore"):
            up = scale * np.float32(2)
        if np.isfinite(up):
            scale = up
        good = 0
    return state[0], (np.float32(scale), good, skipped)


def run(state, flags, growth_interval):
    out = []
    for f in flags:
        _, state = update(state, f, growth_interval)
        out.append((float(state[0]), state[1], state[2]))
    return out


def test_growth_every_interval():
    assert run((1.0, 0, 0), [0, 0, 0, 0, 0], 2) == [(1, 1, 0), (2, 0, 0), (2, 1, 0), (4, 0, 0), (4, 1, 0)]
    assert run((128.0, 0, 0), [0] * 3, 1) == [(256, 0, 0), (512, 0, 0), (1024, 0, 0)]


def test_skip_halves_and_resets_the_run_of_good_steps():
    assert run((2.0 ** 15, 0, 0), [0, 1, 0, 0, 1], 3) == [
        (2.0 ** 15, 1, 0), (2.0 ** 14, 0, 1), (2.0 ** 14, 1, 1), (2.0 ** 14, 2, 1), (2.0 ** 13, 0, 2)]


def test_floor_at_one():
    assert run((4.0, 0, 0), [1, 1, 1, 1], 2) == [(2, 0, 1), (1, 0, 2), (1, 0, 3), (1, 0, 4)]
    # a scale below 1 (an explicit initial scale) is raised to the floor by the first skip
    assert run((0.25, 0, 0), [1], 2) == [(1, 0, 1)]


def test_growth_to_a_non_finite_scale_is_not_kept():
    top = float(np.float32(2.0 ** 127))
    assert run((top, 0, 0), [0, 0, 0], 1) == [(top, 0, 0)] * 3
    # the interval still restarts
    assert run((top, 0, 0), [0, 0, 0], 2) == [(top, 1, 0), (top, 0, 0), (top, 1, 0)]
    big = float(np.float32(3.0 * 2.0 ** 126))            # 2 * big > FLT_MAX
    assert run((big, 0, 0), [0, 1], 1) == [(big, 0, 0), (big / 2, 0, 1)]


def test_the_scale_a_step_used():
    used, state = update((64.0, 1, 0), 0, 2)
    assert used == 64.0 and state == (128.0, 0, 0)
    used, state = update(state, 1, 2)
    assert used == 128.0 and state == (64.0, 0, 1)


# ------------------------------------------------------------------------------------ flags
def test_dynamic_is_accepted_and_other_strings_raise():
    from assembled_cnn_b200.hparams import DEFAULTS, get_loss_scale, params_from_flags
    assert "loss_scale" in DEFAULTS and DEFAULTS["loss_scale"] is None
    assert params_from_flags(loss_scale="dynamic")["loss_scale"] == "dynamic"
    for dt in ("fp16", "bf16", "fp32"):
        assert get_loss_scale("dynamic", dt) == "dynamic"
    for bad in ("Dynamic", "static", "", "128"):
        with pytest.raises(ValueError):
            params_from_flags(loss_scale=bad)
        with pytest.raises(ValueError):
            get_loss_scale(bad, "fp16")


def test_numeric_and_none_resolution_unchanged():
    from assembled_cnn_b200.hparams import get_loss_scale
    assert get_loss_scale(None, "fp16") == 128.0 and get_loss_scale(None, "bf16") == 1.0
    assert get_loss_scale(None, "fp32") == 1.0
    assert get_loss_scale(0, "fp16") == 1.0 and get_loss_scale(256, "bf16") == 256.0
    assert isinstance(get_loss_scale(512, "fp16"), float)


def test_errors_before_any_gpu_work(tmp_path):
    """A bad string, initial scale or growth interval raises ValueError where a GPU would be needed next (this
    machine has none: the runtime would raise AcnnError)."""
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer, train_and_evaluate
    model = Model(50, num_classes=10, dtype="fp16")
    with pytest.raises(ValueError, match="loss_scale"):
        Trainer(model, dict(params_from_flags(batch_size=8), loss_scale="auto"), 64, 64)
    p = params_from_flags(batch_size=8, loss_scale="dynamic")
    for kw in (dict(initial_loss_scale=0.0), dict(initial_loss_scale=float("inf")),
               dict(initial_loss_scale=1e39), dict(loss_scale_growth_interval=0),
               dict(loss_scale_growth_interval=2.5)):
        with pytest.raises(ValueError):
            Trainer(model, p, 64, 64, **kw)
    with pytest.raises(ValueError, match="loss_scale"):
        train_and_evaluate(str(tmp_path / "no-data"), str(tmp_path / "run"), loss_scale="on")


# ------------------------------------------------------------------------------------ the ABI
def test_entry_points_declared_and_bound():
    from assembled_cnn_b200 import _lib, native
    protos = _lib.PROTOTYPES
    v, i, i64 = C.c_void_p, C.c_int, C.c_int64
    assert protos["acnn_grads_nonfinite"] == (i, [v, i64, v, v])
    assert protos["acnn_loss_scale_update"] == (i, [v, i, v])
    assert protos["acnn_sgd_momentum_loss_scaled"] == (i, [v, v, v, i64, v, v, v, i, v, v, v])
    assert protos["acnn_softmax_ce_scaled"] == (i, [v, v, v, C.c_float, i, i, i, C.c_float, v, v, v, v, v, i, v])
    # the existing entry points keep their signatures
    assert protos["acnn_sgd_momentum"] == (i, [v, v, v, i64, v, v, v, v, v])
    assert protos["acnn_softmax_ce"][1][8] is C.c_float
    header = open(native.MODEL_HEADER).read()
    for name in ("acnn_set_dynamic_loss_scale", "acnn_get_loss_scale_state"):
        assert re.search(r"\bint %s\(" % name, header) and name in native.PROTOTYPES
    assert native.PROTOTYPES["acnn_set_dynamic_loss_scale"] == (i, [v, v, C.c_double, i, i, v])


def test_state_struct_layout():
    """acnn_loss_scale_state is 32 bytes with the fields native.decode_loss_scale_state reads."""
    from assembled_cnn_b200.native import decode_loss_scale_state
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "acnn.h"\nint main(void) {\n'
           '  printf("%d %d %d %d %d %d\\n", (int)sizeof(acnn_loss_scale_state),'
           ' (int)offsetof(acnn_loss_scale_state, scale), (int)offsetof(acnn_loss_scale_state, good_steps),'
           ' (int)offsetof(acnn_loss_scale_state, skipped_steps), (int)offsetof(acnn_loss_scale_state, nonfinite),'
           ' (int)offsetof(acnn_loss_scale_state, last_scale));\n  return 0;\n}\n')
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "probe.c"), "w") as f:
            f.write(src)
        exe = os.path.join(d, "probe")
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(d, "probe.c")], check=True)
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in out] == [32, 0, 4, 8, 12, 16]
    words = np.zeros(8, np.int32)
    words[[0, 4]] = np.array([512.0, 1024.0], np.float32).view(np.int32)
    words[1], words[2], words[3] = 7, 3, 1
    assert decode_loss_scale_state(words) == {"scale": 512.0, "good_steps": 7, "skipped_steps": 3,
                                              "last_scale": 1024.0}


# ------------------------------------------------------------------------------------ checkpoints
class _Rt:
    plan = type("P", (), {"params": {}})()


class _Model:
    def __init__(self):
        self.w = {"resnet_model/conv2d/kernel": np.arange(6, dtype=np.float32).reshape(1, 1, 2, 3)}

    def get_weights(self, use_resnet_d=None):
        import torch
        return {n: torch.as_tensor(v) for n, v in self.w.items()}

    def set_weights(self, w):
        self.w = {n: np.asarray(v) for n, v in w.items()}


class _Trainer:
    def __init__(self, dynamic, state=None):
        self.rt, self.dynamic, self.global_step, self.state = _Rt(), dynamic, 0, state

    def loss_scale_state(self):
        return self.state if self.dynamic else None

    def set_loss_scale_state(self, scale, good_steps=0, skipped_steps=0):
        self.state = {"scale": scale, "good_steps": good_steps, "skipped_steps": skipped_steps}


def test_checkpoint_keys_round_trip(tmp_path):
    from assembled_cnn_b200.checkpoint import LOSS_SCALE_KEYS, load_checkpoint, restore, save_checkpoint, warm_start
    st = {"scale": 2048.0, "good_steps": 17, "skipped_steps": 4}
    tr = _Trainer(True, dict(st))
    tr.global_step = 21
    f = save_checkpoint(str(tmp_path / "dyn"), _Model(), tr)
    ck = load_checkpoint(f)
    assert LOSS_SCALE_KEYS == ("loss_scale/current_loss_scale", "loss_scale/good_steps", "loss_scale/skipped_steps")
    assert ck[LOSS_SCALE_KEYS[0]].dtype == np.float32 and float(ck[LOSS_SCALE_KEYS[0]]) == 2048.0
    assert int(ck[LOSS_SCALE_KEYS[1]]) == 17 and int(ck[LOSS_SCALE_KEYS[2]]) == 4
    # a resumed dynamic run restores them
    back = _Trainer(True, {"scale": 32768.0, "good_steps": 0, "skipped_steps": 0})
    restore(_Model(), f, back)
    assert back.state == st and back.global_step == 21
    # a static Trainer ignores them, and a static run writes none
    static = _Trainer(False)
    restore(_Model(), f, static)
    assert static.state is None
    f2 = save_checkpoint(str(tmp_path / "static"), _Model(), _Trainer(False))
    assert not set(LOSS_SCALE_KEYS) & set(load_checkpoint(f2))
    # a checkpoint without them leaves a dynamic run at its initial scale
    fresh = _Trainer(True, {"scale": 32768.0, "good_steps": 0, "skipped_steps": 0})
    restore(_Model(), f2, fresh)
    assert fresh.state == {"scale": 32768.0, "good_steps": 0, "skipped_steps": 0}
    # extra keys are harmless to a full restore of the weights
    m = _Model()
    m.w["resnet_model/conv2d/kernel"] = m.w["resnet_model/conv2d/kernel"] * 0
    assert restore(m, f) == [] and np.array_equal(m.w["resnet_model/conv2d/kernel"], _Model().w[
        "resnet_model/conv2d/kernel"])
    assert warm_start(m, f, global_step=5) == []
