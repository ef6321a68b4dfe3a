#!/usr/bin/env python
"""Golden data of the training input, produced by EXECUTING the reference's own code (by its AST) from a
checkout of the original project:

    python tests/golden/make_train_preprocess_golden.py REFERENCE_DIR
        # rewrites train_preprocess_golden.json

It runs, against a stand-in `tf` whose sample_distorted_bounding_box and random_uniform return scripted
values and record their arguments,
  * utils/data_util.py preprocess_image (the preprocessing_type dispatch, is_training=True) ->
    preprocessing/imagenet_preprocessing.py preprocess_image(is_training=True) -> _decode_crop_and_flip,
    _resize_image, mean_image_subtraction, for every imagenet-family type, both use_random_crop values and a
    grid of image sizes: the sampler's arguments, the crop window given to decode_and_crop_jpeg, the order
    of the operations and S;
  * functions/input_fns.py input_fn_cls: the batch size and epoch count it hands to input_fn, with and
    without mixup type 1;
  * nets/run_loop_classification.py's schedule statement with utils/config_utils.py get_epoch_schedule, for
    a grid of (train_epochs, epochs_between_evals, ratio_fine_eval, resume step).
tests/test_train_input_cpu.py checks the product against this file; it does not need the original project.
"""
import ast
import json
import math
import os
import re
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "train_preprocess_golden.json")
PRE = os.path.join("preprocessing", "imagenet_preprocessing.py")
DATA = os.path.join("utils", "data_util.py")
INPUT = os.path.join("functions", "input_fns.py")
CONFIG = os.path.join("utils", "config_utils.py")
RUN_LOOP = os.path.join("nets", "run_loop_classification.py")

TYPES = [("imagenet", 224), ("imagenet", 160), ("imagenet", 64), ("imagenet_224_256", 224),
         ("imagenet_224_256a", 224), ("imagenet_256", 224), ("imagenet_320", 224), ("imagenet_256a", 224),
         ("imagenet_288a", 224)]
SIZES = [(500, 375), (375, 500), (2592, 1944), (224, 224), (100, 100), (50, 80), (1, 500), (500, 1), (1, 1),
         (2, 3)]
# (train_epochs, epochs_between_evals, ratio_fine_eval, resume global step); num_images 1000, batch 32
SCHEDULES = [(90, 1, 1.0, 0), (90, 5, 1.0, 0), (90, 4, 1.0, 0), (10, 3, 0.5, 0), (10, 3, 0.5, 93),
             (10, 3, 0.5, 186), (10, 3, 0.5, 279), (7, 7, 0.9, 0), (7, 2, 0.0, 31), (5, 10, 1.0, 0),
             (0, 1, 1.0, 0), (12, 4, 0.7, 124), (12, 4, 0.7, 250), (3, 1, 1.0, 62)]
SCHED_IMAGES, SCHED_BATCH = 1000, 32


class FakeImage:
    def __init__(self, h, w, log):
        self.h, self.w, self.log = int(h), int(w), log

    def set_shape(self, shape):
        assert [self.h, self.w] == [int(shape[0]), int(shape[1])], (self.h, self.w, shape)
        self.log["set_shape"] = [int(s) for s in shape]

    def get_shape(self):
        return types.SimpleNamespace(ndims=3)

    def __sub__(self, other):
        self.log["ops"].append("mean")
        self.log["mean"] = [float(v) for v in other]
        return self


def stub_tf(log, box, u_flip):
    """`box` = (y, x, h, w) the scripted sampler returns; `u_flip` the scripted random_uniform value."""
    def sample_distorted_bounding_box(image_size, bounding_boxes, min_object_covered, aspect_ratio_range,
                                      area_range, max_attempts, use_image_if_no_bounding_boxes):
        log["ops"].append("sample")
        log["sampler"] = {"image_size": [int(v) for v in image_size], "bounding_boxes": bounding_boxes,
                          "min_object_covered": float(min_object_covered),
                          "aspect_ratio_range": [float(v) for v in aspect_ratio_range],
                          "area_range": [float(v) for v in area_range], "max_attempts": int(max_attempts),
                          "use_image_if_no_bounding_boxes": bool(use_image_if_no_bounding_boxes)}
        y, x, h, w = box
        return [y, x, 0], [h, w, -1], None

    def decode_and_crop_jpeg(buf, crop_window, channels, dct_method=""):
        log["ops"].append("decode_and_crop")
        log["crop_window"] = [int(v) for v in crop_window]
        return FakeImage(crop_window[2], crop_window[3], log)

    def random_uniform(shape, minval=0.0, maxval=1.0, dtype=None, seed=None):
        log["random_uniform"] = {"shape": list(shape), "minval": float(minval), "maxval": float(maxval)}
        return u_flip

    def random_flip_left_right(image, seed=None):
        # image_ops_impl.random_flip_left_right (TF 1.14): mirror_cond = random_uniform([], 0, 1.0) < 0.5
        log["ops"].append("flip")
        log["flipped"] = bool(random_uniform([], 0, 1.0, seed=seed) < 0.5)
        return image

    def resize_images(image, size, method, align_corners):
        assert method == "BILINEAR" and align_corners is False
        log["ops"].append("resize")
        log["resize"] = [int(size[0]), int(size[1])]
        return FakeImage(size[0], size[1], log)

    def zeros(shape, dtype=None):
        log["bbox_zeros"] = [int(s) for s in shape]
        return "zeros%s" % list(shape)

    image = types.SimpleNamespace(
        extract_jpeg_shape=lambda buf: [buf[0], buf[1], 3],
        sample_distorted_bounding_box=sample_distorted_bounding_box, decode_and_crop_jpeg=decode_and_crop_jpeg,
        random_flip_left_right=random_flip_left_right, resize_images=resize_images,
        ResizeMethod=types.SimpleNamespace(BILINEAR="BILINEAR"))
    return types.SimpleNamespace(
        float32=np.float32, int32=np.int32, cast=lambda x, dt: x, image=image, zeros=zeros,
        unstack=lambda t: list(t), stack=lambda t: list(t), random_uniform=random_uniform,
        shape=lambda img: [np.int32(img.h), np.int32(img.w), np.int32(3)],
        broadcast_to=lambda means, shape: means, logging=types.SimpleNamespace(info=lambda *a, **k: None))


def module_nodes(path, names):
    tree = ast.parse(open(path).read())
    keep = []
    for n in tree.body:
        if isinstance(n, ast.FunctionDef) and n.name in names:
            keep.append(n)
        elif isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id in names for t in n.targets):
            keep.append(n)
    return ast.Module(body=keep, type_ignores=[])


def reference_train_preprocess(ref_root, h, w, preprocessing_type, image_size, use_random_crop, box, u_flip):
    log = {"ops": []}
    tf = stub_tf(log, box, u_flip)
    pre = {"tf": tf}
    exec(compile(module_nodes(os.path.join(ref_root, PRE),
                              {"_R_MEAN", "_G_MEAN", "_B_MEAN", "CHANNEL_MEANS", "_decode_crop_and_flip",
                               "mean_image_subtraction", "_resize_image", "preprocess_image"}), PRE, "exec"), pre)
    data = {"tf": tf, "re": re, "imagenet_preprocessing": types.SimpleNamespace(**pre)}
    exec(compile(module_nodes(os.path.join(ref_root, DATA), {"preprocess_image"}), DATA, "exec"), data)
    out = data["preprocess_image"](image_buffer=(h, w), is_training=True, num_channels=3, dtype=np.float32,
                                   use_random_crop=use_random_crop, image_size=image_size,
                                   preprocessing_type=preprocessing_type)
    assert isinstance(out, FakeImage)
    s = log["set_shape"][0]
    assert log["resize"] == [s, s]
    return {"type": preprocessing_type, "image_size": image_size, "h": h, "w": w,
            "use_random_crop": use_random_crop, "box": list(box), "u_flip": u_flip, "S": s,
            "sampler": log["sampler"], "crop_window": log["crop_window"], "ops": log["ops"],
            "flipped": log["flipped"], "random_uniform": log["random_uniform"], "bbox_zeros": log["bbox_zeros"],
            "mean": log["mean"]}


def reference_input_fn_cls(ref_root, mixup_type, batch_size, num_epochs, num_gpus):
    calls = []

    def input_fn(is_training, filenames, use_random_crop, batch_size, num_train_files, num_images,
                 shuffle_buffer, num_channels, num_epochs=1, num_gpus=None, dtype=None, **kw):
        calls.append({"batch_size": batch_size, "num_epochs": num_epochs, "shuffle_buffer": shuffle_buffer,
                      "return_logits": kw.get("return_logits")})
        return "dataset"

    ds = types.SimpleNamespace(map=lambda fn: ds)
    tf = types.SimpleNamespace(logging=types.SimpleNamespace(info=lambda *a, **k: None),
                               data=types.SimpleNamespace(Dataset=types.SimpleNamespace(zip=lambda t: ds)))
    flags = types.SimpleNamespace(mixup_type=mixup_type, batch_size=batch_size, data_dir="d", train_regex="train-*",
                                  val_regex="validation-*", dataset_name="imagenet", autoaugment_type=None,
                                  with_drawing_bbox=False, preprocessing_type="imagenet", kd_temp=0,
                                  dct_method="INTEGER_ACCURATE")
    g = {"tf": tf, "input_fn": input_fn,
         "distribution_utils": types.SimpleNamespace(per_device_batch_size=lambda b, n: b // max(n, 1)),
         "flags_core": types.SimpleNamespace(get_num_gpus=lambda f: num_gpus, get_tf_dtype=lambda f: "float32"),
         "data_util": types.SimpleNamespace(get_filenames=lambda *a, **k: ["f"], parse_record_sup=None),
         "data_config": types.SimpleNamespace(get_config=lambda n: types.SimpleNamespace(
             num_train_files=1024, num_images={"train": 1281167}, shuffle_buffer=10000, num_channels=3))}
    exec(compile(module_nodes(os.path.join(ref_root, INPUT), {"input_fn_cls"}), INPUT, "exec"), g)
    g["input_fn_cls"](True, True, num_epochs, flags)
    g["input_fn_cls"](False, False, 1, flags)
    return {"mixup_type": mixup_type, "batch_size": batch_size, "num_epochs": num_epochs, "num_gpus": num_gpus,
            "train": calls[0], "eval": calls[1]}


def reference_schedule(ref_root, train_epochs, ebe, ratio, resume_step):
    ckpt = None if resume_step == 0 else "/m/model.ckpt-%d" % resume_step
    tf = types.SimpleNamespace(gfile=types.SimpleNamespace(Exists=lambda d: True),
                               train=types.SimpleNamespace(latest_checkpoint=lambda d: ckpt),
                               logging=types.SimpleNamespace(info=lambda *a, **k: None))
    cfg = {"tf": tf}
    exec(compile(module_nodes(os.path.join(ref_root, CONFIG), {"get_epoch_schedule"}), CONFIG, "exec"), cfg)
    # the schedule statement of resnet_main (`if flags_obj.eval_only or not flags_obj.train_epochs: ...`)
    src = open(os.path.join(ref_root, RUN_LOOP)).read()
    main = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "resnet_main")
    stmt = next(n for n in main.body if isinstance(n, ast.If) and "eval_only" in ast.unparse(n.test))
    flags = types.SimpleNamespace(eval_only=False, export_only=False, train_epochs=train_epochs,
                                  epochs_between_evals=ebe, ratio_fine_eval=ratio, model_dir="/m",
                                  batch_size=SCHED_BATCH)
    g = {"flags_obj": flags, "math": math, "tf": tf, "num_images": {"train": SCHED_IMAGES},
         "config_utils": types.SimpleNamespace(get_epoch_schedule=cfg["get_epoch_schedule"])}
    exec(compile(ast.Module(body=[stmt], type_ignores=[]), RUN_LOOP, "exec"), g)
    return {"train_epochs": train_epochs, "epochs_between_evals": ebe, "ratio_fine_eval": ratio,
            "resume_step": resume_step, "num_images": SCHED_IMAGES, "batch_size": SCHED_BATCH,
            "schedule": [int(e) for e in g["schedule"]]}


def main(ref_root):
    rng = np.random.default_rng(11)
    cases = []
    for t, s in TYPES:
        for h, w in SIZES:
            for use_random_crop in (True, False):
                ch, cw = int(rng.integers(1, h + 1)), int(rng.integers(1, w + 1))
                box = (int(rng.integers(0, h - ch + 1)), int(rng.integers(0, w - cw + 1)), ch, cw)
                u = float(rng.choice([0.0, 0.25, 0.4999, 0.5, 0.75]))
                cases.append(reference_train_preprocess(ref_root, h, w, t, s, use_random_crop, box, u))
    inputs = [reference_input_fn_cls(ref_root, m, b, e, g) for m in (0, 1, 2) for b, e, g in
              ((256, 1, 1), (256, 3, 1), (512, 2, 8))]
    schedules = [reference_schedule(ref_root, *a) for a in SCHEDULES]
    json.dump({"cases": cases, "input_fn_cls": inputs, "schedules": schedules}, open(OUT, "w"), sort_keys=True,
              indent=0)
    print("wrote", OUT)


if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isfile(os.path.join(sys.argv[1], PRE)):
        sys.exit("usage: python tests/golden/make_train_preprocess_golden.py REFERENCE_DIR\n"
                 "  REFERENCE_DIR: a checkout of clovaai/assembled-cnn (the directory holding preprocessing/)")
    main(os.path.abspath(sys.argv[1]))
