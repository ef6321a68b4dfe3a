"""CPU checks of image search (no GPU): the argument checks and byte counts of acnn_knn_prepare_index /
acnn_knn_search, the gallery.npz round trip through load_servable, every refusal of set_gallery, search and
export_gallery raised before any GPU work, and the new merge kernel in the library's SASS."""
import os
import subprocess

import numpy as np
import pytest
import torch

OK, INVALID, UNSUPPORTED = 0, 1, 3


def _a(b):
    return (b + 255) // 256 * 256


def test_search_argument_errors_without_gpu():
    """Every argument check of acnn_knn_prepare_index and acnn_knn_search runs on the host before any CUDA
    call, with acnn_knn_topk's rules."""
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    dummy = 1 << 20                  # never dereferenced: the checks fail first

    def search(nq=10, nx=20, d=16, k=5, metric=0, dtype=0, work=True, nbytes=1 << 30, index=dummy):
        return lib.acnn_knn_search(dummy, nq, index, nx, d, k, metric, dtype, dummy, dummy,
                                   dummy if work else None, nbytes, None)

    def prepare(nx=20, d=16, metric=0, dtype=0, index=dummy, nbytes=1 << 30):
        return lib.acnn_knn_prepare_index(dummy, nx, d, metric, dtype, index, nbytes, None)

    assert search(k=129) == UNSUPPORTED and search(k=1000, nx=5000) == UNSUPPORTED
    for kw in (dict(k=21), dict(nq=0), dict(nx=0), dict(d=0), dict(k=0), dict(nq=-3), dict(metric=2),
               dict(dtype=2), dict(work=False), dict(index=None), dict(nbytes=100), dict(index=dummy + 16)):
        assert search(**kw) == INVALID, kw
        assert lib.acnn_last_error()
    for kw in (dict(nx=0), dict(d=0), dict(metric=-1), dict(dtype=2), dict(index=None), dict(nbytes=100),
               dict(index=dummy + 64)):
        assert prepare(**kw) == INVALID, kw
    assert lib.acnn_knn_index_bytes(0, 16, 0) == -1 and lib.acnn_knn_index_bytes(20, 16, 2) == -1
    assert lib.acnn_knn_search_work_bytes(10, 20, 16, 129, 0) == -1
    assert lib.acnn_knn_search_work_bytes(10, 20, 16, 21, 0) == -1


@pytest.mark.parametrize("nq,nx,d,k,dtype", [(1, 1, 1, 1, 0), (7, 129, 100, 101, 1), (128, 5924, 512, 6, 3),
                                             (1, 60502, 2048, 128, 0), (1000, 60502, 512, 6, 1),
                                             (64, 2048, 64, 16, 0), (64, 2176, 64, 16, 0)])
def test_search_byte_counts_follow_the_documented_layout(nq, nx, d, k, dtype):
    """include/acnn.h: the index is X' then |x|^2; the work is Q', |q|^2, S = min(132, ceil(nx / 128))
    per-split lists and, when S > 16, ceil(S / 16) lists of the first merge pass."""
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    kp = (6 if dtype == 1 else 1) * ((d + 63) // 64 * 64)
    assert lib.acnn_knn_index_bytes(nx, d, dtype) == _a(_a(nx * kp * 2) + nx * 4)
    s = min(132, -(-nx // 128))
    m = -(-s // 16) if s > 16 else 0
    lists = _a(_a(_a(_a(nq * kp * 2) + nq * 4) + s * nq * k * 4) + s * nq * k * 4)
    assert lib.acnn_knn_search_work_bytes(nq, nx, d, k, dtype) == _a(_a(lists + m * nq * k * 4) + m * nq * k * 4)


def test_new_kernel_in_sass():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from assembled_cnn_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "knn_merge_kernelILi16E" in sass and "knn_merge_kernelILi8E" in sass


def _export(tmp_path, embedding_size=32, return_embedding=False):
    from assembled_cnn_b200.model_fns import build_model, export_model
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    model = build_model(resnet_size=50, num_classes=10, embedding_size=embedding_size, dtype="bf16")
    plan = build_plan(ModelConfig(use_resnet_d=model.use_resnet_d, **model.cfg_kwargs), 1, 64, 64, training=False)
    g = torch.Generator().manual_seed(0)
    model.set_weights({n: torch.randn(p.tf_shape, generator=g)
                       for n, p in list(plan.params.items()) + list(plan.state.items())})
    binary, _ = export_model(model, str(tmp_path / "export"), preprocessing_type="imagenet_128a", image_size=224,
                             return_embedding=return_embedding)
    return binary


def _gallery(n, d, seed=0):
    g = np.random.default_rng(seed)
    return {"embedding": g.standard_normal((n, d)).astype(np.float32),
            "label": g.integers(-1, 5, n).astype(np.int64), "shard": np.zeros(n, np.int32),
            "record": np.arange(n, dtype=np.int64), "shard_names": np.asarray(["validation-00000-of-00001"])}


def test_gallery_npz_round_trip_is_host_work(tmp_path):
    from assembled_cnn_b200.model_fns import load_servable
    binary = _export(tmp_path)
    sv = load_servable(binary, device="cuda:0")
    assert sv.gallery_rows == 0 and sv.embedding_width == 32
    gal = _gallery(300, 32)
    np.savez(os.path.join(binary, "gallery.npz"), **gal)
    sv = load_servable(binary, device="cuda:0", batch_sizes=(1, 8, 64, 256))
    assert sv.gallery_rows == 300 and sv._index is None and sv.model._runtimes == {}
    emb, similarity = sv._gallery
    assert similarity == "cosine" and emb.dtype == torch.float32 and np.array_equal(emb.numpy(), gal["embedding"])
    assert np.array_equal(sv.gallery_labels, gal["label"])


def test_refusals_before_gpu_work(tmp_path, monkeypatch):
    from assembled_cnn_b200.model_fns import export_gallery, load_servable
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    # a servable without an embedding output
    plain = _export(tmp_path / "plain", embedding_size=0)
    sv = load_servable(plain, device="cuda:0")
    with pytest.raises(ValueError, match="embedding"):
        sv.set_gallery(np.zeros((4, 2048), np.float32))
    with pytest.raises(ValueError, match="embedding"):
        export_gallery(plain, str(tmp_path))
    assert sorted(os.listdir(plain)) == ["config.json", "variables.npz"]
    # with the pooled features as its embedding (return_embedding, no embedding layer): width 2048
    pooled = load_servable(_export(tmp_path / "pooled", embedding_size=0, return_embedding=True), device="cuda:0")
    assert pooled.embedding_width == 2048
    pooled.set_gallery(np.ones((3, 2048), np.float32))
    # the gallery's width, labels, values and similarity
    sv = load_servable(_export(tmp_path / "emb"), device="cuda:0")
    for bad in (np.zeros((4, 31), np.float32), np.zeros((0, 32), np.float32), np.zeros(32, np.float32)):
        with pytest.raises(ValueError):
            sv.set_gallery(bad)
    with pytest.raises(ValueError):
        sv.set_gallery(np.zeros((4, 32), np.float32), labels=[1, 2, 3])
    for v in (np.nan, np.inf):
        e = np.ones((4, 32), np.float32)
        e[2, 5] = v
        with pytest.raises(ValueError, match="NaN or infinite"):
            sv.set_gallery(e)
    with pytest.raises(NotImplementedError):
        sv.set_gallery(np.ones((4, 32), np.float32), similarity="dot")
    # search before a gallery, then k outside [1, min(128, rows)]
    with pytest.raises(ValueError, match="no gallery"):
        sv.search([b"x"], 1)
    with pytest.raises(ValueError, match="no gallery"):
        sv.search_images(np.zeros((1, 128, 128, 3), np.float32), 1)
    sv.set_gallery(np.ones((100, 32), np.float32))
    for k in (0, -1, 101, 129, 2.0, True, None):
        with pytest.raises(ValueError, match="k must be"):
            sv.search([b"x"], k)
    sv.set_gallery(np.ones((300, 32), np.float32), labels=np.arange(300))
    with pytest.raises(ValueError, match=r"\[1, 128\]"):
        sv.search_images(np.zeros((1, 128, 128, 3), np.float32), 129)
    assert sv.model._runtimes == {} and sv._pipes == {}
    # an existing gallery.npz (or a partial one) is never overwritten
    binary = _export(tmp_path / "exists")
    for name in ("gallery.npz", ".gallery.npz.partial"):
        open(os.path.join(binary, name), "wb").close()
        with pytest.raises(FileExistsError):
            export_gallery(binary, str(tmp_path / "no-such-dir"))
        os.remove(os.path.join(binary, name))
    with pytest.raises(FileNotFoundError):            # an empty glob
        export_gallery(binary, str(tmp_path / "no-such-dir"))
    assert sorted(os.listdir(binary)) == ["config.json", "variables.npz"]
