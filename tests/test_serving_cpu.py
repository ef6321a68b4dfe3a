"""CPU checks of the export path (no GPU): the servable layout and its config.json / variables.npz round trip
for a model whose weights were given to set_weights, every argument error of export_model, load_servable,
Servable and train_and_evaluate's export flags raised before anything is written and before any GPU work,
the export_only schedule, and acnn_predict_rows' host-side checks.  (The export flags' defaults are checked
against the reference's with every other flag, in test_reference_shim_golden_cpu.)"""
import json
import os
import subprocess

import numpy as np
import pytest
import torch


def _model_with_weights(**flags):
    from assembled_cnn_b200.model_fns import build_model
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    model = build_model(resnet_size=50, num_classes=10, **flags)
    plan = build_plan(ModelConfig(use_resnet_d=model.use_resnet_d, **model.cfg_kwargs), 1, 64, 64, training=False)
    g = torch.Generator().manual_seed(0)
    weights = {n: torch.randn(p.tf_shape, generator=g) for n, p in list(plan.params.items()) + list(plan.state.items())}
    model.set_weights(weights)
    return model, weights


def test_export_layout_and_round_trip(tmp_path):
    from assembled_cnn_b200.checkpoint import load_checkpoint
    from assembled_cnn_b200.model_fns import SIGNATURES, export_model, load_servable, read_servable_config
    model, weights = _model_with_weights(dtype="fp32", use_resnet_d=True, use_sk_block=True, embedding_size=64)
    out = tmp_path / "export"
    paths = export_model(model, str(out), preprocessing_type="imagenet_128a", image_size=224,
                         return_embedding=True, decoder_type="webp")
    assert model._runtimes == {}                      # no GPU work
    stamp = os.path.basename(paths[0])
    assert paths == tuple(str(out / "channels_last" / s / stamp) for s in SIGNATURES) and stamp.isdigit()
    assert sorted(os.listdir(out / "channels_last")) == sorted(SIGNATURES)
    for sig, path in zip(SIGNATURES, paths):
        assert sorted(os.listdir(os.path.dirname(path))) == [stamp]          # no hidden directory left
        assert sorted(os.listdir(path)) == ["config.json", "variables.npz"]
        cfg = read_servable_config(path)
        assert cfg == json.load(open(os.path.join(path, "config.json")))
        assert cfg["signature"] == sig and cfg["dtype"] == "fp32" and cfg["use_resnet_d"] is True
        assert cfg["model"] == model.cfg_kwargs
        assert (cfg["preprocessing_type"], cfg["image_size"], cfg["eval_size"]) == ("imagenet_128a", 224, 128)
        assert cfg["decoder_type"] == "webp" and cfg["return_embedding"] is True
        assert sorted(cfg["outputs"]) == ["classes", "embedding", "probabilities", "probabilities_sigmoid"]
        saved = load_checkpoint(os.path.join(path, "variables.npz"))
        assert sorted(saved) == sorted(weights)
        assert all(saved[n].dtype == np.float32 and np.array_equal(saved[n], weights[n].numpy()) for n in weights)
        sv = load_servable(path, device="cuda:0", max_batch=7)       # host work only
        assert sv.signature == sig and sv.max_batch == 7 and sv.size == 128 and sv.use_resnet_d
        assert sv.outputs == ("classes", "probabilities", "probabilities_sigmoid", "embedding")
        assert sv.model.dtype == "fp32" and sv.model.cfg_kwargs == model.cfg_kwargs and sv.model._runtimes == {}
        assert all(np.array_equal(np.asarray(sv.model._pending_weights[n]), weights[n].numpy()) for n in weights)


def test_export_argument_errors_write_nothing(tmp_path, monkeypatch):
    from assembled_cnn_b200.model_fns import build_model, export_model
    model = build_model(resnet_size=50, num_classes=10)             # no weights yet: exporting would need the GPU
    out = tmp_path / "export"
    cases = [(NotImplementedError, dict(preprocessing_type="bogus", image_size=224)),
             (NotImplementedError, dict(preprocessing_type="inception_331", image_size=224)),
             (ValueError, dict(preprocessing_type="imagenet", image_size=100)),
             (ValueError, dict(preprocessing_type="imagenet", image_size=0)),
             (ValueError, dict(preprocessing_type="imagenet", image_size="224")),
             (ValueError, dict(preprocessing_type="imagenet_224_256", image_size=-1)),
             (ValueError, dict(preprocessing_type="imagenet", image_size=224, decoder_type="png"))]
    for exc, kw in cases:
        with pytest.raises(exc):
            export_model(model, str(out), **kw)
        assert not out.exists() and model._runtimes == {}, kw
    with pytest.raises(TypeError):
        export_model(model, str(out), image_size=224)             # preprocessing_type has no default
    # an existing target, of either signature
    import time
    monkeypatch.setattr(time, "time", lambda: 1700000000.5)
    for sig in ("binary_input", "preprocessed_input"):
        target = out / "channels_last" / sig / "1700000000"
        target.mkdir(parents=True)
        with pytest.raises(FileExistsError):
            export_model(model, str(out), preprocessing_type="imagenet", image_size=224)
        target.rmdir()
        assert [p for p in out.rglob("*") if p.is_file()] == [] and model._runtimes == {}


def test_load_servable_and_servable_errors(tmp_path):
    from assembled_cnn_b200.model_fns import Servable, build_model, export_model, load_servable
    with pytest.raises(ValueError, match="not an exported servable"):
        load_servable(str(tmp_path))
    model, _ = _model_with_weights()
    binary, _ = export_model(model, str(tmp_path / "e"), preprocessing_type="imagenet", image_size=64)
    cfg = json.load(open(os.path.join(binary, "config.json")))
    json.dump(dict(cfg, format="something else"), open(os.path.join(binary, "config.json"), "w"))
    with pytest.raises(ValueError, match="format"):
        load_servable(binary, device="cuda:0")
    json.dump(dict(cfg, model=dict(cfg["model"], use_se_block=True)), open(os.path.join(binary, "config.json"), "w"))
    with pytest.raises(ValueError, match="lacks"):
        load_servable(binary, device="cuda:0")
    sv = Servable(build_model(resnet_size=50, num_classes=10), image_size=64, max_batch=4)
    with pytest.raises(TypeError):
        sv.predict([b"\xff\xd8", "not bytes"])
    with pytest.raises(ValueError, match="64, 64, 3"):
        sv.predict_images(np.zeros((2, 32, 32, 3), np.float32))
    with pytest.raises(ValueError):
        Servable(model, image_size=64, max_batch=0)
    assert sv._pipe is None and sv.model._runtimes == {}          # nothing reached the GPU


def test_export_only_schedule():
    from assembled_cnn_b200 import imagenet_train as it
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import cycle_schedule
    assert cycle_schedule(params_from_flags(export_only=True), 1, 0) == ([], 0)
    assert cycle_schedule(params_from_flags(export_only=True, train_epochs=5), 2, 3) == ([], 0)
    # the reference checks eval_only / train_epochs = 0 first
    assert cycle_schedule(params_from_flags(export_only=True, eval_only=True), 1, 0) == ([0], 0)
    assert cycle_schedule(params_from_flags(export_only=True, train_epochs=0), 1, 0) == ([0], 0)
    p = params_from_flags(train_epochs=5)
    assert cycle_schedule(p, 2, 0) == (it.epoch_schedule(5, 2, 1.0), 0)


def test_train_and_evaluate_export_errors_before_gpu(tmp_path):
    from assembled_cnn_b200.model_fns import train_and_evaluate
    data, run = str(tmp_path / "data"), str(tmp_path / "run")
    with pytest.raises(ValueError, match="export_dir"):
        train_and_evaluate(data, run, export_only=True)
    with pytest.raises(ValueError, match="no checkpoint"):
        train_and_evaluate(data, run, export_only=True, export_dir=str(tmp_path / "e"))
    with pytest.raises(ValueError, match="export_decoder_type"):
        train_and_evaluate(data, run, export_dir=str(tmp_path / "e"), export_decoder_type="gif")
    assert not (tmp_path / "e").exists() and not (tmp_path / "run").exists()


def test_predict_rows_argument_errors_without_gpu():
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    INVALID, p = 1, 1 << 20          # p is never dereferenced: the checks fail first

    def rows(logits=p, B=4, ld=16, NC=10, n_valid=4, classes=p, prob=p, sig=p):
        return lib.acnn_predict_rows(logits, B, ld, NC, n_valid, classes, prob, sig, None)

    for kw in (dict(logits=None), dict(classes=None), dict(prob=None), dict(sig=None), dict(B=0), dict(NC=0),
               dict(ld=9), dict(n_valid=5), dict(n_valid=-1)):
        assert rows(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    assert rows(n_valid=0) == 0


def test_predict_rows_kernel_in_sass():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from assembled_cnn_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "predict_rows_kernel" in sass
