"""CPU checks of the zero-shot retrieval evaluation over TFRecord shards (model_fns.evaluate_retrieval and
train_and_evaluate(zeroshot_eval=True)): the reader's opt-in label for records without one, labels outside
[0, num_classes) kept, and every argument and data error raised before any GPU work."""
import io
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
SHARD = os.path.join(ROOT, "golden", "eval_golden.tfrecord")


def _write_shard(path, labels, seed=0):
    """One JPEG record per entry of `labels`; None writes an Example without image/class/label."""
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "golden"))
    import make_eval_preprocess_golden as mk
    Example = mk.example_class()
    rng = np.random.default_rng(seed)
    recs = []
    for label in labels:
        buf = io.BytesIO()
        Image.fromarray(rng.integers(0, 256, (12, 17, 3), dtype=np.uint8)).save(buf, format="JPEG", quality=90)
        ex = Example()
        ex.features.feature["image/encoded"].bytes_list.value.append(buf.getvalue())
        if label is not None:
            ex.features.feature["image/class/label"].int64_list.value.append(label)
        data = ex.SerializeToString()
        head = len(data).to_bytes(8, "little")
        recs.append(head + mk.masked(head).to_bytes(4, "little") + data + mk.masked(data).to_bytes(4, "little"))
    path.write_bytes(b"".join(recs))
    return path


LABELS = [3, None, 150, 1 << 40, None, 7, 3, 0]


def test_reader_missing_label_only_when_asked(tmp_path):
    from assembled_cnn_b200.imagenet_eval import parse_example, read_records
    path = str(_write_shard(tmp_path / "validation-00000-of-00001", LABELS))
    recs = read_records(path, missing_label=-1)
    assert [r[0] for r in recs] == [-1 if lab is None else lab for lab in LABELS]
    assert [r[0] for r in read_records(path, missing_label=-7)][1] == -7
    data = open(path, "rb").read()
    n0 = int.from_bytes(data[:8], "little")
    second = data[12 + n0 + 4:]
    n1 = int.from_bytes(second[:8], "little")
    # the default still refuses the record, naming its byte offset
    with pytest.raises(ValueError, match="record at byte offset %d: Example without image/encoded or "
                                         "image/class/label" % (12 + n0 + 4)):
        read_records(path)
    with pytest.raises(ValueError, match="without image/encoded or image/class/label"):
        parse_example(memoryview(second[12:12 + n1]))
    label, (a, b) = parse_example(memoryview(second[12:12 + n1]), missing_label=-1)
    assert label == -1 and second[12 + a:12 + b] == data[recs[1][1]:recs[1][1] + recs[1][2]]
    # a record with a label keeps it whatever missing_label says; existing callers see the same records
    assert read_records(SHARD, missing_label=-1) == read_records(SHARD)
    assert read_records(SHARD, logits=True, missing_label=-1)[0][:3] == read_records(SHARD)[0]


def _retrieval_dir(tmp_path):
    d = tmp_path / "data"
    d.mkdir()
    _write_shard(d / "validation-00000-of-00002", LABELS[:5])
    _write_shard(d / "validation-00001-of-00002", LABELS[5:], seed=1)
    return d


@pytest.fixture
def no_gpu_work(monkeypatch):
    """Any attempt to start the device loop fails the test."""
    from assembled_cnn_b200 import model_fns

    def refuse(*a, **k):
        raise AssertionError("the device loop started")
    monkeypatch.setattr(model_fns, "_RetrievalEvalDevice", refuse)
    monkeypatch.setattr(model_fns, "_retrieval_index", refuse)


def test_evaluate_retrieval_checks_before_any_gpu_work(tmp_path, no_gpu_work):
    from assembled_cnn_b200.model_fns import build_model, evaluate_retrieval
    model = build_model(resnet_size=50, num_classes=100)
    d = _retrieval_dir(tmp_path)
    with pytest.raises(FileNotFoundError):
        evaluate_retrieval(model, str(tmp_path / "empty"))
    with pytest.raises(FileNotFoundError):
        evaluate_retrieval(model, str(d), val_regex="test-*")
    with pytest.raises(NotImplementedError, match="eval_similarity"):
        evaluate_retrieval(model, str(d), eval_similarity="dot")
    with pytest.raises(ValueError, match="recall_at_k"):
        evaluate_retrieval(model, str(d), recall_at_k=[])
    with pytest.raises(ValueError, match="recall_at_k"):
        evaluate_retrieval(model, str(d), recall_at_k=[0, 1])
    with pytest.raises(ValueError, match="129 exceeds 128, the largest k of the fused top-k search"):
        evaluate_retrieval(model, str(d), recall_at_k=[1, 128])
    with pytest.raises(ValueError, match="hold 8 records"):   # k = 128 is in the search's range
        evaluate_retrieval(model, str(d), recall_at_k=[1, 127])
    with pytest.raises(NotImplementedError, match="reid / inception"):
        evaluate_retrieval(model, str(d), preprocessing_type="reid_224")
    with pytest.raises(NotImplementedError):
        evaluate_retrieval(model, str(d), preprocessing_type="inception_331")
    with pytest.raises(ValueError, match="multiple of 32"):
        evaluate_retrieval(model, str(d), preprocessing_type="imagenet_300")
    # 8 records: k = max + 1 = 9 cannot be ranked
    with pytest.raises(ValueError, match="hold 8 records, 6 of them queries"):
        evaluate_retrieval(model, str(d), recall_at_k=[1, 8])
    only_distractors = tmp_path / "distractors"
    only_distractors.mkdir()
    _write_shard(only_distractors / "validation-00000-of-00001", [None] * 10)
    with pytest.raises(ValueError, match="0 of them queries"):
        evaluate_retrieval(model, str(only_distractors))
    corrupt = tmp_path / "corrupt"
    shutil.copytree(d, corrupt)
    data = (corrupt / "validation-00001-of-00002").read_bytes()
    (corrupt / "validation-00001-of-00002").write_bytes(data[:-3])
    with pytest.raises(ValueError, match="validation-00001-of-00002: truncated record at byte offset"):
        evaluate_retrieval(model, str(corrupt))
    # the classification evaluation still refuses what the retrieval evaluation reads
    from assembled_cnn_b200.model_fns import evaluate_classification
    with pytest.raises(ValueError, match="byte offset"):
        evaluate_classification(model, str(d))


def test_train_and_evaluate_zeroshot_checks_first(tmp_path, no_gpu_work):
    from assembled_cnn_b200.model_fns import train_and_evaluate
    m = str(tmp_path / "m")
    with pytest.raises(FileNotFoundError):              # the shards are read before any GPU work
        train_and_evaluate(str(tmp_path), m, zeroshot_eval=True, dataset_name="cub_200_2011")
    with pytest.raises(NotImplementedError, match="eval_similarity"):
        train_and_evaluate(str(tmp_path), m, zeroshot_eval=True, eval_similarity="dot")
    with pytest.raises(ValueError, match="must hold 1"):
        train_and_evaluate(str(tmp_path), m, zeroshot_eval=True, recall_at_k=[2, 4])
    with pytest.raises(ValueError, match="fused top-k search"):
        train_and_evaluate(str(tmp_path), m, zeroshot_eval=True, recall_at_k=[1, 200])
    # without zeroshot_eval the retrieval flags are not read
    with pytest.raises(FileNotFoundError):
        train_and_evaluate(str(tmp_path), m, eval_similarity="dot", recall_at_k=[])
    assert not os.path.exists(m)
