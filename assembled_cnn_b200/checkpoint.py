"""Checkpoint import / export in the reference's TF variable naming, the warm-start filter and the
best-checkpoint keeper (utils/hook_utils.py:29-56, utils/checkpoint_utils.py:24-137).

File format: one `.npz` per checkpoint (TensorFlow's tensor-bundle format cannot be written without
TensorFlow).  Keys are the reference's variable names -- `resnet_model/conv2d/kernel`,
`.../batch_normalization_3/moving_mean`, ... -- with values in the reference's layouts (HWIO conv
kernels, [in, out] dense kernel), the MomentumOptimizer slots as `<var>/Momentum`, `global_step` and,
for a run with dynamic loss scaling, its state as `loss_scale/current_loss_scale`, `loss_scale/good_steps`
and `loss_scale/skipped_steps`,
i.e. exactly what `tf.train.load_checkpoint(path).get_tensor(name)` returns for a TF-1.14 checkpoint
of the reference.  A released checkpoint converts with four lines run where TensorFlow exists:

    r = tf.train.load_checkpoint(ckpt)
    np.savez(out, **{n: r.get_tensor(n) for n in r.get_variable_to_shape_map()})
"""
from __future__ import annotations

import glob
import json
import os
from shutil import copyfile

import numpy as np
import torch


# the dynamic loss scale's state (TF 2 Keras' LossScaleOptimizer keeps current_loss_scale and good_steps)
LOSS_SCALE_KEYS = ("loss_scale/current_loss_scale", "loss_scale/good_steps", "loss_scale/skipped_steps")


def save_checkpoint(path, model, trainer=None, use_resnet_d=None):
    """Write `<path>.npz` with every variable of the model (trainables + BN moving statistics) and,
    when a Trainer is given, the momentum slots, global_step and, with dynamic loss scaling, its state.
    Returns the file name."""
    if use_resnet_d is None:
        use_resnet_d = getattr(model, "use_resnet_d", False)
    arrays = {n: v.numpy() for n, v in model.get_weights(use_resnet_d).items()}
    if trainer is not None:
        rt = trainer.rt
        for n in rt.plan.params:
            arrays[n + "/Momentum"] = rt.get_tf(n, rt.momentum).detach().float().cpu().numpy().copy()
        arrays["global_step"] = np.asarray(trainer.global_step, dtype=np.int64)
        ls = trainer.loss_scale_state() if getattr(trainer, "dynamic", False) else None
        if ls is not None:
            arrays[LOSS_SCALE_KEYS[0]] = np.asarray(ls["scale"], dtype=np.float32)
            arrays[LOSS_SCALE_KEYS[1]] = np.asarray(ls["good_steps"], dtype=np.int64)
            arrays[LOSS_SCALE_KEYS[2]] = np.asarray(ls["skipped_steps"], dtype=np.int64)
    fname = path if path.endswith(".npz") else path + ".npz"
    os.makedirs(os.path.dirname(os.path.abspath(fname)), exist_ok=True)
    np.savez(fname, **arrays)
    return fname


def load_checkpoint(path):
    """name -> numpy array of a checkpoint written by save_checkpoint (or converted from TF)."""
    fname = path if path.endswith(".npz") else path + ".npz"
    with np.load(fname) as z:
        return {n: z[n] for n in z.files}


def latest_checkpoint(directory):
    """tf.train.latest_checkpoint for a directory of `model.ckpt-<step>.npz` files."""
    best, best_step = None, -1
    for f in glob.glob(os.path.join(directory, "*.npz")):
        stem = os.path.basename(f)[:-4]
        try:
            step = int(stem.rsplit("-", 1)[1])
        except (IndexError, ValueError):
            step = 0
        if step > best_step:
            best, best_step = f, step
    return best


def restore(model, ckpt, trainer=None, strict=True):
    """Full restore (every variable; momentum + global_step into the Trainer if present, and the dynamic loss
    scale's state into a Trainer with dynamic loss scaling: without it that run keeps its initial scale; a
    static Trainer ignores it)."""
    if isinstance(ckpt, str):
        ckpt = load_checkpoint(ckpt)
    cur = model.get_weights()
    missing = [n for n in cur if n not in ckpt]
    if missing and strict:
        raise KeyError("checkpoint lacks %d variable(s), e.g. %s" % (len(missing), missing[:3]))
    cur.update({n: torch.as_tensor(ckpt[n]) for n in cur if n in ckpt})
    model.set_weights(cur)
    if trainer is not None:
        rt = trainer.rt
        for n in rt.plan.params:
            key = n + "/Momentum"
            if key in ckpt:
                rt.set_tf(n, torch.as_tensor(ckpt[key]), rt.momentum)
        if "global_step" in ckpt:
            trainer.global_step = int(ckpt["global_step"])
        if getattr(trainer, "dynamic", False) and LOSS_SCALE_KEYS[0] in ckpt:
            trainer.set_loss_scale_state(float(ckpt[LOSS_SCALE_KEYS[0]]), int(ckpt.get(LOSS_SCALE_KEYS[1], 0)),
                                         int(ckpt.get(LOSS_SCALE_KEYS[2], 0)))
    return missing


def warm_start_variables(names):
    """utils/hook_utils.py:36-44: the TRAINABLE variables restored for fine-tuning -- everything
    except names containing 'dense' (the classifier `dense/*` and `embedding_dense/*`), unless they
    belong to an SE block (`se_block*/seblock_dense_*`).  `names` must be the trainable variables
    (tf.contrib.framework.get_trainable_variables): BN moving statistics are NOT warm-started."""
    return [n for n in names if not ("dense" in n and "se_block" not in n)]


def warm_start(model, ckpt, global_step=0):
    """WarmStartHook.after_create_session: only when global_step == 0; directories resolve to
    their latest checkpoint.  Returns the list of restored variable names."""
    if global_step != 0 or ckpt is None:
        return []
    if isinstance(ckpt, str):
        if os.path.isdir(ckpt):
            ckpt = latest_checkpoint(ckpt)
        ckpt = load_checkpoint(ckpt)
    rt = next(iter(model._primary.values())) if model._primary else None
    if rt is None:
        raise ValueError("warm_start: build a runtime first (call the model or create a Trainer)")
    names = warm_start_variables(list(rt.plan.params))
    cur = model.get_weights()
    for n in names:
        if n not in ckpt:
            raise KeyError("warm start: %s not in the checkpoint" % n)
        cur[n] = torch.as_tensor(ckpt[n])
    model.set_weights(cur)
    return names


class CheckpointKeeper:
    """utils/checkpoint_utils.py:24-137: keeps the `num_to_keep` best checkpoints (by an evaluation
    value) under <save_dir>/best and, optionally, every evaluated one under <save_dir>/periodical;
    the ranking lives in <save_dir>/best/best_checkpoints (json)."""

    def __init__(self, save_dir, num_to_keep=1, keep_epoch=False, maximize=True):
        self._num_to_keep = num_to_keep
        self._save_dir = save_dir
        self._best_save_path = os.path.join(save_dir, "best")
        self._periodical_save_path = os.path.join(save_dir, "periodical")
        self._maximize = maximize
        self._keep_epoch = keep_epoch
        os.makedirs(self._best_save_path, exist_ok=True)
        if keep_epoch:
            os.makedirs(self._periodical_save_path, exist_ok=True)
        self.best_checkpoints_file = os.path.join(self._best_save_path, "best_checkpoints")

    def _keep_ckpt(self, name, mode="best"):
        dst = self._best_save_path if mode == "best" else self._periodical_save_path
        for f in glob.glob(os.path.join(self._save_dir, name) + "*"):
            if os.path.isfile(f):
                copyfile(f, os.path.join(dst, os.path.basename(f)))

    def _load(self):
        with open(self.best_checkpoints_file) as fh:
            return json.load(fh)

    def _store(self, d):
        with open(self.best_checkpoints_file, "w") as fh:
            json.dump(d, fh, indent=3)

    def save(self, value, current_ckpt):
        if os.path.isdir(current_ckpt):
            current_ckpt = latest_checkpoint(current_ckpt)
        name = os.path.basename(current_ckpt)
        if name.endswith(".npz"):
            name = name[:-4]
        value = float(value)
        if not os.path.exists(self.best_checkpoints_file):
            self._store({name: value})
            self._keep_ckpt(name)
        else:
            best = self._load()
            if len(best) < self._num_to_keep:
                best[name] = value
                self._store(best)
                self._keep_ckpt(name)
            else:
                if self._maximize:
                    should = not all(v >= value for v in best.values())
                else:
                    should = not all(v <= value for v in best.values())
                if should:
                    ranked = sorted(best, key=best.get, reverse=self._maximize)
                    worst = ranked.pop(-1)
                    for f in glob.glob(os.path.join(self._best_save_path, worst) + ".*"):
                        os.remove(f)
                    best = {k: best[k] for k in ranked}
                    best[name] = value
                    self._store(best)
                    self._keep_ckpt(name)
        if self._keep_epoch:
            self._keep_ckpt(name, mode="periodical")
