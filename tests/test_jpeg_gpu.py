"""The device JPEG decoder against PIL bit for bit: whole images and windows of the corpus, mixed
supported / unsupported batches, CUDA-graph replay and concurrent streams, and damaged scans (status set,
the other images and the bytes around every output untouched, PIL's result at the wrapper)."""
import io

import numpy as np
import pytest
import torch

import jpeg_corpus as JC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    return JC.corpus()


def test_device_decode_equals_pil(corpus):
    from assembled_cnn_b200 import jpeg
    dec = jpeg.JpegDecoder("cuda")
    bufs = [b for _, b in corpus]
    desc, jobs, out, status = dec.enqueue(bufs)
    assert status.cpu().tolist() == [0] * len(bufs)
    for (name, b), j in zip(corpus, jobs):
        want = JC.pil_rgb(b)
        o = int(j["out"])
        got = out[o:o + want.size].view(want.shape).cpu().numpy()
        assert np.array_equal(got, want), (name, int((got != want).sum()))


def test_device_windows_equal_pil_slices(corpus):
    from assembled_cnn_b200 import jpeg
    rng = np.random.default_rng(3)
    bufs, wins, wants = [], [], []
    for name, b in corpus:
        a = JC.pil_rgb(b)
        H, W = a.shape[:2]
        cand = [(0, 0, 1, 1), (H - 1, W - 1, 1, 1), (0, W - 1, H, 1), (H - 1, 0, 1, W)]
        for _ in range(3):
            h, w = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
            cand.append((int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w))
        for y, x, h, w in cand:
            bufs.append(b)
            wins.append((y, x, h, w))
            wants.append((name, a[y:y + h, x:x + w]))
    got = jpeg.decode_jpegs(bufs, np.array(wins, np.int32))
    for g, (name, want), w in zip(got, wants, wins):
        assert g.is_cuda and g.dtype == torch.uint8
        assert np.array_equal(g.cpu().numpy(), want), (name, w)


def test_mixed_supported_and_unsupported_batch(corpus):
    from assembled_cnn_b200 import jpeg
    odd = JC.unsupported_samples()
    bufs = [corpus[3][1], odd[0][1], corpus[20][1], odd[1][1], odd[2][1], corpus[-1][1]]
    desc = jpeg.parse(bufs)
    assert desc["supported"].tolist() == [1, 0, 1, 0, 0, 1]
    got = jpeg.decode_jpegs(bufs)
    for b, g in zip(bufs, got):
        assert np.array_equal(g.cpu().numpy(), JC.pil_rgb(b))


def _prepared(bufs, windows=None, gap=0):
    """Device copies of a planned batch; with gap > 0, every output is placed `gap` guard bytes after the
    previous one."""
    from assembled_cnn_b200 import jpeg
    data, offsets, lengths = jpeg.pack(bufs)
    desc = jpeg.parse_packed(data, offsets, lengths)
    jobs, batch = jpeg.plan(desc, offsets, windows)
    if gap:
        o = gap
        for j in jobs:
            j["out"] = o
            o += int(j["win_h"]) * int(j["win_w"]) * 3 * bool(j["active"]) + gap
        batch.out_bytes = o
    d = dict(desc=desc, jobs=jobs, batch=batch,
             data=torch.from_numpy(data.copy()).cuda(),
             ddesc=torch.from_numpy(desc.view(np.uint8).copy()).cuda(),
             djobs=torch.from_numpy(jobs.view(np.uint8).copy()).cuda(),
             work=torch.empty(batch.work_bytes, dtype=torch.uint8, device="cuda"),
             out=torch.full((batch.out_bytes,), 0xA5, dtype=torch.uint8, device="cuda"),
             status=torch.full((len(bufs),), -1, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    return d


def _launch(d, stream):
    from assembled_cnn_b200 import _lib, jpeg
    _lib.check(_lib.load().acnn_jpeg_decode(d["ddesc"].data_ptr(), d["djobs"].data_ptr(),
                                            jpeg.C.addressof(d["batch"]), d["data"].data_ptr(),
                                            d["out"].data_ptr(), d["work"].data_ptr(), d["work"].numel(),
                                            d["status"].data_ptr(), stream.cuda_stream), "acnn_jpeg_decode")


def test_graph_replay_and_concurrent_streams(corpus):
    bufs = [b for _, b in corpus]
    ref = _prepared(bufs)
    _launch(ref, torch.cuda.current_stream())
    torch.cuda.synchronize()
    want = ref["out"].clone()
    assert ref["status"].cpu().tolist() == [0] * len(bufs)
    # CUDA graph: capture once, replay twice
    g_in = _prepared(bufs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        graph.capture_begin()
        _launch(g_in, s)
        graph.capture_end()
    for _ in range(2):
        g_in["out"].fill_(0xA5)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(g_in["out"], want) and g_in["status"].cpu().tolist() == [0] * len(bufs)
    # two streams at once, each with its own workspace
    a, b = _prepared(bufs), _prepared(bufs)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    _launch(a, sa)
    _launch(b, sb)
    torch.cuda.synchronize()
    assert torch.equal(a["out"], want) and torch.equal(b["out"], want)


def _damaged(rng):
    from assembled_cnn_b200 import jpeg
    out = []
    for kw in (dict(quality=90), dict(quality=80, restart_marker_blocks=3), dict(quality=95, optimize=True)):
        b = JC.encode(JC.image(96, 136, "noise", rng), **kw)
        d = jpeg.parse([b])[0]
        start, n = int(d["ecs_offset"]), int(d["ecs_length"])
        out.append(b[:start + n // 3])                          # truncated scan
        for _ in range(8):                                      # bit flips the scan checks catch
            bad = bytearray(b)
            pos = start + int(rng.integers(0, n))
            bad[pos] ^= 1 << int(rng.integers(0, 8))
            if bad[pos] == 0xFF or bad[pos - 1] == 0xFF:
                continue
            out.append(bytes(bad))
    return out


def test_damaged_scans_set_status_and_touch_nothing_else(corpus):
    from assembled_cnn_b200 import jpeg
    rng = np.random.default_rng(21)
    good = [b for _, b in corpus[:24]]
    bad = _damaged(rng)
    bufs = []
    for i in range(max(len(good), len(bad))):
        if i < len(good):
            bufs.append(good[i])
        if i < len(bad):
            bufs.append(bad[i])
    gap = 64
    d = _prepared(bufs, gap=gap)
    _launch(d, torch.cuda.current_stream())
    torch.cuda.synchronize()
    st = d["status"].cpu().numpy()
    out = d["out"].cpu().numpy()
    covered = np.zeros(out.size, bool)
    n_flagged = 0
    for b, j, s in zip(bufs, d["jobs"], st):
        o, size = int(j["out"]), int(j["win_h"]) * int(j["win_w"]) * 3
        covered[o:o + size] = True
        if b in good:
            assert s == 0
            assert np.array_equal(out[o:o + size].reshape(int(j["win_h"]), int(j["win_w"]), 3), JC.pil_rgb(b))
        elif s:
            n_flagged += 1
            assert s & (jpeg.ST_BAD_CODE | jpeg.ST_OUT_OF_BITS | jpeg.ST_MCU_COUNT)
            assert (out[o:o + size] == 0xA5).all()    # a failed image's window is not written
        else:
            # a flip the checks cannot see is a valid scan: it decodes as PIL decodes it
            assert np.array_equal(out[o:o + size].reshape(int(j["win_h"]), int(j["win_w"]), 3), JC.pil_rgb(b))
    assert n_flagged >= 3
    assert (out[~covered] == 0xA5).all()              # guard bytes between and around the outputs
    # at the wrapper level a damaged image takes the PIL path: PIL's pixels, or PIL's error
    for b in bad:
        try:
            want = JC.pil_rgb(b)
        except OSError:
            with pytest.raises(OSError):
                jpeg.decode_jpegs([b])
            continue
        assert np.array_equal(jpeg.decode_jpegs([b])[0].cpu().numpy(), want)


def test_long_synchronisation_chains():
    """Large 4:4:4 noise images without restart markers (Cb and Cr share their tables, so subsequences take
    long to synchronise and many neighbours are re-decoded in the same pass): still PIL bit for bit."""
    from assembled_cnn_b200 import jpeg
    rng = np.random.default_rng(8)
    bufs = [JC.encode(JC.image(h, w, "noise", rng), quality=q, subsampling=0)
            for h, w, q in ((1200, 1600, 97), (900, 700, 100), (640, 1400, 92), (2000, 1000, 99))]
    got = jpeg.decode_jpegs(bufs)
    for b, g in zip(bufs, got):
        assert np.array_equal(g.cpu().numpy(), JC.pil_rgb(b))
