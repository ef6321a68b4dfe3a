"""Flag names and defaults of the reference's model / training surface, as a plain dict.

Only the flags the hot path consumes; each entry cites where the reference defines it.
`params_from_flags(**overrides)` builds the `params` dict that `model_fn_cls` receives from
`nets/run_loop_classification.py:322-366`.
"""
from __future__ import annotations

DEFAULTS = {
    # nets/run_loop_classification.py:507-514, nets/hparams_config.py
    "resnet_size": 50,                    # run_loop_classification.py:507-514 ('50')
    "resnet_version": 1,                  # hparams_config.py:170
    "use_sk_block": False,                # :157
    "use_se_block": False,                # :153
    "use_resnet_d": False,                # :149
    "anti_alias_type": "",                # :164
    "anti_alias_filter_size": 0,          # :160
    "bl_alpha": 2,                        # :177
    "bl_beta": 4,                         # :182
    "mixup_type": 0,                      # :137
    "label_smoothing": 0.0,               # :200
    "weight_decay": 4e-5,                 # :187
    "momentum": 0.9,                      # :68
    "bn_momentum": 0.997,                 # :72
    "zero_gamma": False,                  # :214
    "base_learning_rate": 0.01,           # :55
    "learning_rate_decay_type": "exponential",   # :63
    "learning_rate_decay_factor": 0.94,
    "num_epochs_per_decay": 2.0,
    "end_learning_rate": 0.0001,
    "piecewise_lr_boundary_epochs": [30, 60, 80, 90],
    "piecewise_lr_decay_rates": [1, 0.1, 0.01, 0.001, 1e-4],
    "lr_warmup_epochs": 0,                # :211
    "use_dropblock": False,               # :191
    "dropblock_kp": [1.0, 0.9],           # :195 (inactive unless use_dropblock)
    "kd_temp": 0,                         # :204
    "pool_type": "gap",                   # :116
    "embedding_size": 0,                  # :76
    "no_downsample": False,
    "cls_loss_type": "softmax",
    "dataset_name": None,                 # :31 (None -> the ImageNet constants, as data_config)
    # zero-shot retrieval evaluation (metric/recall_metric.py; model_fns.evaluate_retrieval, recall_at_k)
    "zeroshot_eval": False,               # :273 (train_and_evaluate: evaluate_retrieval, keep by recall_at_1)
    "eval_similarity": "cosine",          # :91 ('cosine' | 'euclidean')
    "recall_at_k": [1, 5],                # :288 (max + 1 <= 128; train_and_evaluate needs 1 in it)
    "return_embedding": False,            # :27 (train_and_evaluate embeds with True, as the reference's loop)
    "val_batch_size": 256,                # :39 (the retrieval evaluation's batch)
    # classification and retrieval evaluation (model_fns.evaluate_classification, evaluate_retrieval)
    "preprocessing_type": "imagenet",     # :128
    "val_regex": "validation-*",          # :284
    # training from TFRecord shards (model_fns.train_and_evaluate)
    "train_regex": "train-*",             # :280
    "training_random_crop": True,         # :256
    "autoaugment_type": None,             # :132 (only None in train_and_evaluate, which does not draw AutoAugment
                                          # records yet; Trainer.train_step_cropped(augment=) runs it)
    "num_best_ckpt_to_keep": 3,           # :242
    "keep_ckpt_every_eval": True,         # :246
    "keep_checkpoint_max": 20,            # :249
    "eval_only": False,                   # :252
    # export (model_fns.export_model, train_and_evaluate(export_dir=...)); export_dir itself is a keyword of
    # train_and_evaluate, as official/utils/flags/_base.py defines it outside hparams_config.py
    "export_only": False,                 # :259 (no cycle: export the latest checkpoint)
    "export_decoder_type": "jpeg",        # :262 ('jpeg': export_test runs after the export)
    "save_checkpoints_epochs": 1.0,       # :266
    "ratio_fine_eval": 1.0,               # :269
    "pretrained_model_checkpoint_path": None,   # :43
    # official/utils/flags/_base.py:50-105, _performance.py:74-137
    "batch_size": 32,
    "train_epochs": 90,                   # main_classification.py:38
    "dtype": "bf16",                      # reference enum is fp32|fp16; bf16 added (the default here)
    "loss_scale": None,                   # None: the dtype's default, get_loss_scale (fp16: 128, else 1);
                                          # "dynamic": dynamic loss scaling (model_fns.Trainer)
    "data_format": "channels_last",       # NHWC is the only layout of this implementation
    "num_gpus": 1,
}

# functions/data_config.py:22-148, keyed by get_config's names; the *_zeroshot / SOP / CUB entries
# are the retrieval datasets of the zero-shot evaluation
DATASETS = {
    "food101": dict(num_classes=101, num_images={"train": 75750, "validation": 25250}),
    "imagenet": dict(num_classes=1001, num_images={"train": 1281167, "validation": 50000}),
    "cub_200_2011": dict(num_classes=100, num_images={"train": 5864, "validation": 5924}),
    "iFood2019": dict(num_classes=251, num_images={"train": 118475, "validation": 11994}),
    "SOP": dict(num_classes=11318, num_images={"train": 59551, "validation": 60502}),
    "oxford_flowers102": dict(num_classes=102, num_images={"train": 2040, "validation": 6149}),
    "cars196": dict(num_classes=196, num_images={"train": 8144, "validation": 8041}),
    "cars196_zeroshot": dict(num_classes=196, num_images={"train": 8054, "validation": 8131}),
    "oxford_iiit_pet": dict(num_classes=37, num_images={"train": 3680, "validation": 3669}),
    "fgvc_aircraft": dict(num_classes=100, num_images={"train": 6667, "validation": 3333}),
}


def params_from_flags(**overrides) -> dict:
    unknown = set(overrides) - set(DEFAULTS)
    if unknown:
        raise KeyError("unknown flag(s): %s" % ", ".join(sorted(unknown)))
    check_loss_scale(overrides.get("loss_scale"))
    p = dict(DEFAULTS)
    p.update(overrides)
    return p


# official/utils/flags/_performance.py:28-44 DTYPE_MAP: the static loss scale of a dtype when --loss_scale is
# not given (bf16 keeps the full fp32 exponent range and needs none)
DEFAULT_LOSS_SCALE = {"fp16": 128, "fp32": 1, "bf16": 1}


def check_loss_scale(loss_scale):
    """loss_scale: None, a number, or the string "dynamic" (the spelling later versions of the reference's
    official/utils/flags/_performance.py accept); any other string raises ValueError."""
    if isinstance(loss_scale, str) and loss_scale != "dynamic":
        raise ValueError('loss_scale must be None, a number or "dynamic" (got %r)' % (loss_scale,))
    return loss_scale


def get_loss_scale(loss_scale, dtype):
    """official/utils/flags/_performance.py:39-42 get_loss_scale: an explicit loss_scale wins, otherwise the
    dtype's default (fp16: 128; bf16 / fp32: 1).  0 counts as 1 (no scaling).  "dynamic" is returned as it
    is, for every dtype; any other string raises ValueError."""
    if dtype not in DEFAULT_LOSS_SCALE:
        raise ValueError("dtype must be one of: {}".format(tuple(DEFAULT_LOSS_SCALE)))
    if check_loss_scale(loss_scale) == "dynamic":
        return "dynamic"
    if loss_scale is None:
        return float(DEFAULT_LOSS_SCALE[dtype])
    return float(loss_scale or 1)
