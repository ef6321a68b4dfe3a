"""The workflows of an fp16 model (dtype='fp16') on the GPU:

  * train_and_evaluate on the synthetic shards of test_train_input_gpu.py with the c3 model flags, mixup type
    1, DropBlock and knowledge distillation, at replicas_per_device 1 and 2: it trains, checkpoints and
    evaluates, every variable stays finite, and a resumed run reproduces the uninterrupted run's bits;
  * the reference's from-scratch recipe (scripts/train_assemble_from_scratch.sh) with --dtype=fp16 and
    without AutoAugment, scaled down to these shards: finite losses through train_and_evaluate;
  * an fp16 servable: predictions equal the model's own logits, and the servable reloaded from disk (its
    config.json carries the dtype) gives the in-memory servable's bits.
"""
import json
import logging
import math
import os
import re

import numpy as np
import pytest
import torch

import test_serving_gpu as SV
import test_train_input_gpu as T
from test_serving_gpu import images  # noqa: F401  (fixture)
from test_train_input_gpu import shards  # noqa: F401  (fixture: training shards with KD logits)

pytestmark = pytest.mark.gpu

C3 = dict(resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)


def _finite(path):
    w = T._weights(path)
    return all(np.isfinite(v).all() for v in w.values())


def _same(a, b):
    """Evaluation result lists equal value for value (a NaN equals a NaN)."""
    return len(a) == len(b) and all(
        ra.keys() == rb.keys() and all(x == y or (isinstance(x, float) and math.isnan(x) and math.isnan(y))
                                       for x, y in ((ra[k], rb[k]) for k in ra))
        for ra, rb in zip(a, b))


def _train_losses(caplog):
    """The cross-entropy of every training step, from train_and_evaluate's log lines (save_summary_steps=1)."""
    return [float(m.group(1)) for r in caplog.records
            for m in [re.search(r"cross_entropy = (\S+),", r.getMessage())] if m]


@pytest.mark.parametrize("replicas", [1, 2])
def test_train_and_evaluate_fp16_c3_mixup_dropblock_kd_resumes(shards, tmp_path, replicas, caplog):  # noqa: F811
    """The fp16 workflow end to end: every training step's loss is finite, the checkpoints hold finite weights,
    both evaluations run, and the resumed run reproduces the checkpoint and the evaluation results bit for
    bit.  The evaluation values are reported, not asserted finite: after 6 and 12 steps from a random
    initialisation the eval-mode activations are far outside fp16's range (measured in bf16 on these flags:
    logits of 1.8e9 after 6 steps), and fp16 turns them into inf, as the reference's fp16 casts do."""
    from assembled_cnn_b200.model_fns import train_and_evaluate
    caplog.set_level(logging.INFO, logger="assembled_cnn_b200")
    flags = dict(T.FLAGS, dtype="fp16", image_size=224, mixup_type=1, use_dropblock=True, kd_temp=1.0,
                 replicas_per_device=replicas, **C3)
    run = tmp_path / "run"
    res = train_and_evaluate(str(shards), str(run), save_summary_steps=1, **flags)
    steps = [r["global_step"] for r in res]
    assert len(res) == 2 and 0 < steps[0] < steps[1]
    losses = _train_losses(caplog)
    assert len(losses) == steps[1] and all(math.isfinite(v) for v in losses), losses
    print("fp16 c3 workflow, %d replica(s): training cross-entropy per step %s, evaluations %s"
          % (replicas, losses, res))
    last = "model.ckpt-%d.npz" % steps[1]
    final = T._weights(str(run / last))
    assert _finite(str(run / last))
    resumed = tmp_path / "resumed"
    assert _same(train_and_evaluate(str(shards), str(resumed), stop_threshold=0.0, **flags), res[:1])
    assert _same(train_and_evaluate(str(shards), str(resumed), **flags), res[1:])
    got = T._weights(str(resumed / last))
    assert all(np.array_equal(got[n], final[n]) for n in final)


def test_reference_from_scratch_recipe_in_fp16(shards, tmp_path, caplog):  # noqa: F811
    """scripts/train_assemble_from_scratch.sh with --dtype=fp16, without --autoaugment_type, on these shards:
    batch 1024 over 8 GPUs becomes batch 32 over 2 replicas of 16 (a per-replica batch normalisation, as the
    reference's 128 per GPU), 600 epochs become 2 and the 5 warm-up epochs 1; every other flag is the
    recipe's.  The loss scale is the fp16 default, 128.  Every training step's loss is finite and so are the
    trained weights.  (The evaluations after 6 and 12 steps normalise with moving statistics that have barely
    left their initial values at the recipe's bn_momentum 0.997, so their activations overflow fp16; they are
    reported, not asserted -- see the test above for evaluations with converged statistics.)"""
    from assembled_cnn_b200.model_fns import train_and_evaluate
    caplog.set_level(logging.INFO, logger="assembled_cnn_b200")
    flags = dict(dataset_name=T.DATASET, preprocessing_type="imagenet_224_256", batch_size=32, mixup_type=1,
                 resnet_version=2, resnet_size=50, use_sk_block=True, anti_alias_type="sconv",
                 anti_alias_filter_size=3, use_dropblock=True, learning_rate_decay_type="cosine", weight_decay=1e-4,
                 base_learning_rate=0.4, momentum=0.9, lr_warmup_epochs=1, zero_gamma=True, label_smoothing=0.1,
                 kd_temp=1, dtype="fp16", train_epochs=2, seed=5, num_workers=4, num_best_ckpt_to_keep=1)
    run = tmp_path / "recipe"
    res = train_and_evaluate(str(shards), str(run), epochs_between_evals=1, image_size=224,
                             replicas_per_device=2, save_summary_steps=1, **flags)
    losses = _train_losses(caplog)
    print("from-scratch recipe in fp16: training cross-entropy per step", losses, "evaluations", res)
    assert len(res) == 2 and len(losses) == res[-1]["global_step"] > 0
    assert all(math.isfinite(v) for v in losses), losses
    assert _finite(str(run / ("model.ckpt-%d.npz" % res[-1]["global_step"])))


def test_fp16_servable_round_trip(images, tmp_path):  # noqa: F811
    from assembled_cnn_b200.model_fns import Servable, build_model, export_model, load_servable
    SV.test_predict_equals_model_on_pil_batches(images, "fp16")
    model = build_model(resnet_size=50, dtype="fp16", seed=12, embedding_size=64)
    B = 8
    sv = Servable(model, preprocessing_type="imagenet", image_size=SV.SIZE, max_batch=B)
    pool = (images * 2)[:3 * B + 5]
    whole = sv.predict(pool)
    assert all(np.isfinite(v).all() for k, v in whole.items() if k != "classes")
    binary, prep = export_model(model, str(tmp_path / "export"), preprocessing_type="imagenet",
                                image_size=SV.SIZE)
    for path in (binary, prep):
        with open(os.path.join(path, "config.json")) as fh:
            assert json.load(fh)["dtype"] == "fp16"
        sv2 = load_servable(path, max_batch=B)
        assert sv2.model is not model and sv2.model.dtype == "fp16"
        got = sv2.predict(pool)
        for k, v in got.items():
            assert v.tobytes() == whole[k].tobytes(), (path, k)
    x = torch.from_numpy(SV._oracle_x(pool[:B], "imagenet", SV.SIZE))
    assert sv.predict_images(x.numpy())["probabilities"].tobytes() == whole["probabilities"][:B].tobytes()
