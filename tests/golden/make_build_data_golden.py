#!/usr/bin/env python
"""Golden records of the dataset builders, produced by EXECUTING the reference's own builder code
(datasets/build_imagenet_data.py, build_ethz_food101.py, build_cub_bird200_zeroshot.py,
build_cars196_zeroshot.py, build_sop.py with datasets/dataset_utils.py and utils/data_util.py of a checkout
of the original project) through the TF-1.14 stand-in in tests/golden/tf1_shim/:

    python tests/golden/make_build_data_golden.py REFERENCE_DIR   # rewrites build_data_golden.json

The builders run on a small raw tree that make_tree generates from SEED: every dataset's annotation
format, an ImageNet PNG and CMYK JPEG under the reference's file names, a grayscale and a progressive JPEG,
bbox and logit files, and an undecodable image in the Food-101 and SOP lists (skipped by those scripts).
The reference's listing, shuffles, shard layout and Example construction run unchanged; the TF pieces they
call are recorded instead of run:
  * tf.gfile.Glob returns sorted matches (TF 1.14 returns the file system's readdir order);
  * the image coders decode with PIL (for the height, width and decodability); a PNG -> JPEG or CMYK -> RGB
    conversion and a crop + encode_jpeg return a marker naming the source file (and the crop window)
    instead of TF's JPEG bytes;
  * tf.train.Example records its feature map, tf.python_io.TFRecordWriter the Examples of each file.
The JSON holds, per dataset, every record's features (image/encoded as {'file': path in the tree} for the
file's own bytes, {'png_to_jpeg' | 'cmyk_to_rgb': path} or {'crop': [y, x, h, w], 'file': path}; float
lists longer than 8 as their float32 sha256) and, per num_threads, the shard names with their record ids
in order.  tests/test_build_data_cpu.py regenerates the tree and compares the product's shards with it; it
does not need the original project.
"""
import hashlib
import io
import json
import os
import sys
import tarfile
import tempfile
import threading
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "build_data_golden.json")
SEED = 20261017
THREADS = (1, 2, 8)
SHARDS = 8                    # train_shards / validation_shards where the script has the flags

IMAGENET_SYNSETS = ["n01739381", "n02105855", "n03000001"]
IMAGENET_PNG = "n02105855_2933.JPEG"
IMAGENET_CMYK = "n01739381_1309.JPEG"


# -------------------------------------------------------------------------------------------- tree
def _image(rng, h, w, mode="RGB", fmt="JPEG", **kw):
    from PIL import Image
    base = rng.randint(0, 256, size=(4, 4, 3)).astype(np.uint8)
    a = np.array(Image.fromarray(base).resize((w, h), Image.BILINEAR))
    a = np.clip(a.astype(np.int16) + rng.randint(-20, 21, size=a.shape), 0, 255).astype(np.uint8)
    im = Image.fromarray(a).convert(mode)
    b = io.BytesIO()
    im.save(b, fmt, **({"quality": 90} if fmt == "JPEG" else {}), **kw)
    return b.getvalue()


def _put(root, rel, data):
    path = os.path.join(root, rel)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(data)


def _size(rng, lo=17, hi=48):
    return int(rng.randint(lo, hi)), int(rng.randint(lo, hi))


def make_tree(root, seed=SEED):
    """Writes the raw tree of every dataset under root (imagenet/, food101/, cub/, cars196/, sop/)."""
    rng = np.random.RandomState(seed)
    # ImageNet: train/<synset>/*.JPEG, validation/<synset>/ILSVRC2012_val_*.JPEG and the flat validation
    # labels, label / metadata / bbox files, logits/<split>_<k>.csv
    im = os.path.join(root, "imagenet")
    _put(im, "synsets.txt", ("\n".join(IMAGENET_SYNSETS) + "\n").encode())
    _put(im, "metadata.txt", b"n00004475\torganism, being\nn01739381\tvine snake\n"
                             b"n02105855\tShetland sheepdog, Shetland sheep dog, Shetland\nn03000001\tthing\n")
    names = {"train": [], "validation": []}
    for k, s in enumerate(IMAGENET_SYNSETS):
        for j in range(4 + k):
            name = "%s_%d.JPEG" % (s, 100 + j)
            if s == "n01739381" and j == 0:
                name, data = IMAGENET_CMYK, _image(rng, *_size(rng), mode="CMYK")
            elif s == "n02105855" and j == 0:
                name, data = IMAGENET_PNG, _image(rng, *_size(rng), fmt="PNG")
            elif s == "n02105855" and j == 1:
                data = _image(rng, *_size(rng), mode="L")
            elif s == "n03000001" and j == 1:
                data = _image(rng, *_size(rng), progressive=True)
            else:
                data = _image(rng, *_size(rng))
            _put(im, "train/%s/%s" % (s, name), data)
            names["train"].append(name)
        _put(im, "train/%s/notes.txt" % s, b"not an image\n")          # outside the *.JPEG glob
    _put(im, "train/n03000001/lower.jpeg", _image(rng, 20, 20))         # the glob is case-sensitive
    val_labels = [IMAGENET_SYNSETS[int(v)] for v in rng.randint(0, 3, size=9)]
    for i, s in enumerate(val_labels):
        name = "ILSVRC2012_val_%08d.JPEG" % (i + 1)
        _put(im, "validation/%s/%s" % (s, name), _image(rng, *_size(rng)))
        names["validation"].append(name)
    _put(im, "val_labels.txt", ("\n".join(val_labels) + "\n").encode())
    lines = []
    for n in names["train"][::2] + names["validation"][::3]:
        for _ in range(1 + (len(lines) % 3 == 0)):
            lines.append("%s,%.4f,%.4f,%.4f,%.4f\n" % ((n,) + tuple(np.round(rng.rand(4), 4))))
    _put(im, "bboxes.csv", "".join(lines).encode())
    for split in ("train", "validation"):
        half = (len(names[split]) + 1) // 2
        for k, part in enumerate((names[split][:half], names[split][half:])):
            rows = ["%s,%s\n" % (n, ",".join("%.6f" % v for v in rng.randn(1001))) for n in part]
            _put(im, "logits/%s_%d.csv" % (split, k), "".join(rows).encode())
    # Food-101: images/<label>/<id>.jpg, meta/labels.txt (display names), meta/train.txt, meta/test.txt
    fd = os.path.join(root, "food101")
    labels = ["Apple pie", "Baby back ribs", "Beef tartare"]
    _put(fd, "meta/labels.txt", ("\n".join(labels) + "\n").encode())
    lists = {"train": [], "test": []}
    for k, lab in enumerate(labels):
        d = lab.lower().replace(" ", "_")
        for j in range(6):
            rel = "%s/%d" % (d, 1000 + 7 * j + k)
            data = _image(rng, *_size(rng))
            if k == 1 and j == 2:
                data = data[:len(data) // 2]                                # undecodable: skipped
            _put(fd, "images/%s.jpg" % rel, data)
            lists["train" if j < 4 else "test"].append(rel)
    for split in lists:
        _put(fd, "meta/%s.txt" % split, ("\n".join(lists[split]) + "\n").encode())
    # CUB-200-2011: images/<NNN.name>/<file>.jpg over 102 class directories (a stray file among them),
    # images.txt and bounding_boxes.txt
    cub = os.path.join(root, "cub")
    _put(cub, "images/000.readme", b"not a class\n")
    rows_img, rows_box, iid = [], [], 1
    for c in range(102):
        d = "%03d.Bird_%d" % (c + 1, c)
        os.makedirs(os.path.join(cub, "images", d), exist_ok=True)
        if c not in (0, 1, 2, 100, 101):
            continue
        for j in range(2 + (c % 2)):
            rel = "%s/Bird_%d_%04d_%d.jpg" % (d, c, j, 10 + j)
            h, w = _size(rng, 24, 48)
            _put(cub, "images/" + rel, _image(rng, h, w))
            x, y = float(rng.randint(0, w // 2)), float(rng.randint(0, h // 2))
            bw = float(rng.randint(4, w)) + 0.5                               # may reach past the edge
            bh = float(rng.randint(4, h)) + 0.5
            rows_img.append("%d %s\n" % (iid, rel))
            rows_box.append("%d %.1f %.1f %.1f %.1f\n" % (iid, x, y, bw, bh))
            iid += 1
    _put(cub, "images.txt", "".join(rows_img).encode())
    _put(cub, "bounding_boxes.txt", "".join(rows_box).encode())
    # Cars196: car_ims.tgz (+ extracted car_ims/), cars_annos.mat; classes 1..99 so both label ranges are hit
    from scipy.io import savemat
    cars = os.path.join(root, "cars196")
    classes = list(range(1, 100)) + [1, 99, 50]
    order = rng.permutation(len(classes))
    ann = []
    for i, c in enumerate(classes[k] for k in order):
        rel = "car_ims/%06d.jpg" % (i + 1)
        h, w = _size(rng, 16, 32)
        _put(cars, rel, _image(rng, h, w))
        x1, y1 = int(rng.randint(0, w // 2)), int(rng.randint(0, h // 2))
        ann.append((rel, x1, y1, x1 + int(rng.randint(3, w)), y1 + int(rng.randint(3, h)), c, i % 2))
    rec = np.zeros(len(ann), dtype=[("relative_im_path", object), ("bbox_x1", object), ("bbox_y1", object),
                                     ("bbox_x2", object), ("bbox_y2", object), ("class", object), ("test", object)])
    for i, a in enumerate(ann):
        rec[i] = (a[0],) + tuple(np.array([[v]], dtype=np.uint8 if k == 5 else np.uint16)
                                 for k, v in enumerate(a[1:], start=1))
    savemat(os.path.join(cars, "cars_annos.mat"), {"annotations": rec.reshape(1, -1)})
    with tarfile.open(os.path.join(cars, "car_ims.tgz"), "w:gz") as t:
        for a in sorted(ann, key=lambda a: a[0]):
            t.add(os.path.join(cars, a[0]), arcname=a[0])
    # SOP: Ebay_train.txt / Ebay_test.txt ('image_id class_id super_class_id path' after a header)
    sop = os.path.join(root, "sop")
    rows = {"train": ["image_id class_id super_class_id path\n"], "test": ["image_id class_id super_class_id path\n"]}
    for i in range(16):
        split = "train" if i < 10 else "test"
        cls = 1 + i // 2
        rel = "%s_final/%d_%d.JPG" % (("bicycle", "chair")[i % 2], 111 + cls, i)
        data = _image(rng, *_size(rng))
        if i == 3:
            data = data[:len(data) // 3]                                    # undecodable: skipped
        _put(sop, rel, data)
        rows[split].append("%d %d %d %s\n" % (i + 1, cls, 1 + i % 2, rel))
    for split in rows:
        _put(sop, "Ebay_%s.txt" % split, "".join(rows[split]).encode())


# ----------------------------------------------------------------------------- the recording stand-in
class _Img:
    def __init__(self, rel, shape, window=None):
        self.rel, self.shape, self.window = rel, shape, window


def _install(tf, files):
    """Adds what the builders touch to the stand-in; `files` maps sha256 of a file's bytes to its path in
    the tree.  Returns the dict the writers record into: file name -> [Example feature maps]."""
    from PIL import Image
    written, lock = {}, threading.Lock()

    def rel_of(data):
        return files[hashlib.sha256(data).hexdigest()]

    def pil(data):
        with Image.open(io.BytesIO(data)) as im:
            return np.array(im.convert("RGB"))

    class InvalidArgumentError(Exception):
        pass

    def glob(pattern):
        import fnmatch
        d, pat = os.path.split(pattern)
        if not os.path.isdir(d):
            return []
        return [os.path.join(d, f) for f in sorted(os.listdir(d)) if fnmatch.fnmatchcase(f, pat)]

    class Flags:
        def __getattr__(self, name):
            if name.startswith("DEFINE_"):
                return lambda n, default, *a, **k: setattr(self, n, default)
            raise AttributeError(name)

    flags = Flags()
    tf.app = types.SimpleNamespace(flags=types.SimpleNamespace(FLAGS=flags, **{
        "DEFINE_" + k: getattr(flags, "DEFINE_" + k) for k in ("string", "integer", "boolean")}))
    tf.gfile = types.SimpleNamespace(FastGFile=open, GFile=open, Glob=glob)
    tf.errors = types.SimpleNamespace(InvalidArgumentError=InvalidArgumentError)

    def feature(**kw):
        (kind, lst), = kw.items()
        return (kind.split("_")[0], list(lst))

    tf.train.Int64List = tf.train.FloatList = tf.train.BytesList = lambda value: value
    tf.train.Feature = feature
    tf.train.Features = lambda feature: feature
    tf.train.Example = lambda features: _Example(features)
    tf.train.Coordinator = lambda: types.SimpleNamespace(join=lambda threads: [t.join() for t in threads])

    class Writer:
        def __init__(self, path):
            self.name, self.records = os.path.basename(path), []

        def write(self, ex):
            self.records.append(ex)

        def close(self):
            with lock:
                assert self.name not in written, self.name
                written[self.name] = self.records

    tf.python_io = types.SimpleNamespace(TFRecordWriter=Writer)

    class ImageCoder:                                 # build_imagenet_data.ImageCoder
        def png_to_jpeg(self, data):
            return b"@png_to_jpeg:" + rel_of(data).encode()

        def cmyk_to_rgb(self, data):
            return b"@cmyk_to_rgb:" + rel_of(data).encode()

        def decode_jpeg(self, data):
            if data.startswith(b"@"):
                data = open(os.path.join(files["root"], data.split(b":", 1)[1].decode()), "rb").read()
            return pil(data)

    coder = types.ModuleType("datasets.image_coder")  # datasets/image_coder.py

    def decode_jpg(data):
        try:
            return _Img(rel_of(data), pil(data).shape)
        except (OSError, SyntaxError, ValueError) as e:
            raise InvalidArgumentError(str(e))

    def crop_bbox(image, bbox=None):
        oh, ow, ch, cw = bbox
        assert oh >= 0 and ow >= 0 and ch > 0 and cw > 0
        assert oh + ch <= image.shape[0] and ow + cw <= image.shape[1]
        return _Img(image.rel, (ch, cw, 3), [int(v) for v in bbox])

    coder.decode_jpg = decode_jpg
    coder.crop_bbox = crop_bbox
    coder.encode_jpg = lambda image: b"@crop:" + json.dumps({"file": image.rel, "crop": image.window}).encode()
    return written, ImageCoder, coder


class _Example:
    def __init__(self, features):
        self.features = features

    def SerializeToString(self):
        return self.features


def _value(kind, values):
    if kind == "bytes":
        return [v.decode() if isinstance(v, bytes) else v for v in values]
    if kind == "float":
        vals = [float(np.float32(v)) for v in values]
        if len(vals) > 8:
            return {"sha256": hashlib.sha256(np.asarray(vals, dtype="<f4").tobytes()).hexdigest(), "n": len(vals)}
        return vals
    return [int(v) for v in values]


def _record(features):
    """(record id, JSON features) of a recorded Example."""
    out = {}
    for key, (kind, values) in features.items():
        if key == "image/encoded":
            (data,) = values
            if data.startswith(b"@crop:"):
                desc = json.loads(data[len(b"@crop:"):].decode())
            elif data.startswith(b"@"):
                op, rel = data[1:].decode().split(":", 1)
                desc = {op: rel}
            else:
                desc = {"file": FILES[hashlib.sha256(data).hexdigest()]}
            out[key] = ["image", desc]
        else:
            out[key] = [kind, _value(kind, values)]
    rid = json.dumps(out["image/encoded"][1], sort_keys=True)
    return rid, out


FILES = {}


def main(ref_root):
    global FILES
    sys.path[:0] = [os.path.join(HERE, "tf1_shim"), ref_root]
    np.int = int                                      # the reference's np.int (removed from numpy)
    import tensorflow as tf
    for m in ("preprocessing", "preprocessing.imagenet_preprocessing", "preprocessing.inception_preprocessing",
              "preprocessing.reid_preprocessing"):
        sys.modules[m] = types.ModuleType(m)
    work = tempfile.mkdtemp(prefix="build_data_golden_")
    tree = os.path.join(work, "tree")
    make_tree(tree)
    for dp, _, fs in os.walk(tree):
        for f in fs:
            p = os.path.join(dp, f)
            FILES[hashlib.sha256(open(p, "rb").read()).hexdigest()] = os.path.relpath(p, tree)
    FILES["root"] = tree
    written, ImageCoder, coder = _install(tf, FILES)
    sys.modules["datasets.image_coder"] = coder
    import datasets
    datasets.image_coder = coder
    import importlib
    mods = {n: importlib.import_module("datasets." + n) for n in
            ("build_imagenet_data", "build_ethz_food101", "build_cub_bird200_zeroshot", "build_cars196_zeroshot",
             "build_sop")}
    mods["build_imagenet_data"].ImageCoder = ImageCoder
    out_dir = os.path.join(work, "out")
    im = os.path.join(tree, "imagenet")

    def imagenet(t, logits=True):
        m = mods["build_imagenet_data"]
        f = tf.app.flags.FLAGS
        for k, v in dict(train_directory=im + "/train", validation_directory=im + "/validation", output_directory=out_dir,
                         train_shards=SHARDS, validation_shards=SHARDS, num_threads=t, make_val=True,
                         make_train=True, labels_file=im + "/synsets.txt", imagenet_metadata_file=im + "/metadata.txt",
                         bounding_box_file=im + "/bboxes.csv", logits_file_path=im + "/logits").items():
            setattr(f, k, v)
        saved = m._find_image_teacher_logits, m._convert_to_example
        if not logits:                                # the product's logits_file_path=None: no image/logit
            m._find_image_teacher_logits = lambda filenames, lookup: [[] for _ in filenames]

            def without_logit(*args):
                ex = saved[1](*args)
                del ex.features["image/logit"]
                return ex
            m._convert_to_example = without_logit
        try:
            m.main(None)
        finally:
            m._find_image_teacher_logits, m._convert_to_example = saved

    def argparse_main(name, **flags):
        def run(t):
            m = mods[name]
            m.FLAGS = types.SimpleNamespace(output_dir=out_dir, num_threads=t, **flags)
            m.main(None)
        return run

    def cars(t):
        cwd = os.getcwd()
        os.chdir(tree)                                # _get_bbox_info() reads ./cars196 whatever data_dir is
        try:
            argparse_main("build_cars196_zeroshot", data_dir="cars196", use_bbox=True)(t)
        finally:
            os.chdir(cwd)

    configs = {
        "imagenet": (imagenet, THREADS),
        "imagenet_no_logits": (lambda t: imagenet(t, logits=False), (2,)),
        "food101": (argparse_main("build_ethz_food101", data_dir=os.path.join(tree, "food101"),
                                  train_shards=SHARDS, validation_shards=SHARDS), THREADS),
        "cub_200_2011": (argparse_main("build_cub_bird200_zeroshot", data_dir=os.path.join(tree, "cub"),
                                       use_bbox=True), THREADS),
        "cub_200_2011_no_bbox": (argparse_main("build_cub_bird200_zeroshot", data_dir=os.path.join(tree, "cub"),
                                               use_bbox=False), (8,)),
        "cars196_zeroshot": (cars, THREADS),
        "SOP": (argparse_main("build_sop", input_dir=os.path.join(tree, "sop"), train_shards=SHARDS,
                              validation_shards=SHARDS), THREADS),
    }
    golden = {"seed": SEED, "shards": SHARDS, "datasets": {}}
    for name, (run, threads) in configs.items():
        records, layouts = {}, {}
        for t in threads:
            written.clear()
            run(t)
            layout = []
            for fname in sorted(written):
                ids = []
                for ex in written[fname]:
                    rid, rec = _record(ex.features if isinstance(ex, _Example) else ex)
                    assert records.setdefault(rid, rec) == rec, (name, rid)
                    ids.append(rid)
                layout.append([fname, ids])
            layouts[str(t)] = layout
        golden["datasets"][name] = {"records": records, "layouts": layouts}
        print(name, len(records), "records", {t: len(l) for t, l in layouts.items()}, "shards")
    with open(OUT, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(os.path.abspath(sys.argv[1]))
