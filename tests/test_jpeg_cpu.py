"""CPU checks of the JPEG decoder: the header parser of libjpeg (dimensions, the supported flag, rejected
headers), and the __host__ __device__ stage functions of csrc/jpeg_stages.cuh, built for the host with
g++ and run serially in the order of the device kernels (tests/c_host/jpeg_host.cpp), against PIL bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_corpus as JC

ROOT = JC.ROOT


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("jpeg_host") / "jpeg_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "c_host", "jpeg_host.cpp")], check=True)
    lib = C.CDLL(so)
    lib.jpeg_host_decode.restype = C.c_int
    lib.jpeg_host_decode.argtypes = [C.c_void_p] * 4
    return lib


@pytest.fixture(scope="module")
def corpus():
    return JC.corpus()


def host_decode(host, b, window=None):
    from assembled_cnn_b200 import jpeg
    desc = jpeg.parse([b])
    jobs, _ = jpeg.plan(desc, np.zeros(1, np.int64), None if window is None else np.array([window], np.int32))
    j = jobs[0]
    out = np.zeros((max(int(j["win_h"]), 1), max(int(j["win_w"]), 1), 3), np.uint8)
    buf = np.frombuffer(b, np.uint8)
    st = host.jpeg_host_decode(desc.ctypes.data, jobs.ctypes.data, buf.ctypes.data, out.ctypes.data)
    return st, out


def test_parser_dimensions_and_flags(corpus):
    from PIL import Image
    import io
    from assembled_cnn_b200 import jpeg
    desc = jpeg.parse([b for _, b in corpus])
    for (name, b), d in zip(corpus, desc):
        with Image.open(io.BytesIO(b)) as im:
            assert (int(d["height"]), int(d["width"])) == (im.size[1], im.size[0]), name
        assert d["supported"] == 1, (name, jpeg.reason_text(d["reason"]))
        assert jpeg.jpeg_shape(b) == (im.size[1], im.size[0])
        assert d["ncomp"] == (1 if "gray" in name else 3) or name.startswith("golden")


def test_parser_refuses_unsupported():
    from assembled_cnn_b200 import jpeg
    samples = JC.unsupported_samples()
    desc = jpeg.parse([b for _, b in samples])
    want = {"progressive": "progressive", "cmyk": "colour space", "png": "not a JPEG"}
    for (name, b), d in zip(samples, desc):
        assert d["supported"] == 0, name
        assert want[name] in jpeg.reason_text(d["reason"]), (name, jpeg.reason_text(d["reason"]))
    # progressive and CMYK still give their size (tf.image.extract_jpeg_shape reads any JPEG)
    assert tuple(desc[0][["height", "width"]]) == (40, 56) and tuple(desc[1][["height", "width"]]) == (40, 56)
    for name, b in samples:
        assert jpeg.jpeg_shape(b) == (40, 56)


def _segments(b):
    """[(marker, start of the segment's length field)] up to SOS."""
    out, p = [], 2
    while True:
        m = b[p + 1]
        out.append((m, p + 2))
        if m == 0xDA:
            return out
        p += 2 + (b[p + 2] << 8 | b[p + 3])


def test_malformed_headers_are_rejected_with_a_message():
    from assembled_cnn_b200 import jpeg
    b = JC.encode(JC.image(24, 40, "smooth", np.random.default_rng(3)), quality=85)
    seg = dict(_segments(b))
    cases = {}
    cases["truncated header"] = b[:seg[0xDB] + 10]
    bad = bytearray(b)
    bad[seg[0xDB]:seg[0xDB] + 2] = b"\xff\xf0"            # DQT length past the end of the buffer
    cases["dqt length"] = bytes(bad)
    bad = bytearray(b)
    bad[seg[0xC4] + 2] = 0x27                             # DHT table class 2
    cases["dht class"] = bytes(bad)
    bad = bytearray(b)
    bad[seg[0xC4] + 3:seg[0xC4] + 19] = bytes([3] * 16)   # more codes of length 1..2 than exist
    cases["dht overfull"] = bytes(bad)
    bad = bytearray(b)
    bad[seg[0xC0] + 9] = 9                                # SOF: 9 components in a 3-component segment
    cases["sof count"] = bytes(bad)
    bad = bytearray(b)
    bad[seg[0xDA] + 2] = 2                                # SOS: fewer components than the frame
    cases["sos count"] = bytes(bad)
    cases["no scan"] = b[:seg[0xDA] - 2] + b"\xff\xd9"
    desc = jpeg.parse(list(cases.values()))
    for (name, _), d in zip(cases.items(), desc):
        assert d["supported"] == 0, name
        msg = jpeg.reason_text(d["reason"])
        assert msg and msg != "supported", name
    assert jpeg.reason_text(desc[0]["reason"]).startswith("the buffer ends inside")
    assert jpeg.reason_text(desc[1]["reason"]).startswith("the buffer ends inside")
    assert "malformed" in jpeg.reason_text(desc[2]["reason"]) and "malformed" in jpeg.reason_text(desc[3]["reason"])


def test_stage_functions_equal_pil(host, corpus):
    for name, b in corpus:
        st, out = host_decode(host, b)
        assert st == 0, (name, st)
        want = JC.pil_rgb(b)
        assert out.shape == want.shape and np.array_equal(out, want), (name, int((out != want).sum()))


def test_stage_functions_windows(host, corpus):
    rng = np.random.default_rng(7)
    for name, b in corpus:
        want = JC.pil_rgb(b)
        H, W = want.shape[:2]
        wins = [(0, 0, 1, 1), (H - 1, W - 1, 1, 1), (0, 0, H, W)]
        for _ in range(3):
            h, w = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
            wins.append((int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w))
        for y, x, h, w in wins:
            st, out = host_decode(host, b, (y, x, h, w))
            assert st == 0 and np.array_equal(out, want[y:y + h, x:x + w]), (name, (y, x, h, w))


def test_stage_functions_report_damaged_scans(host):
    """Truncated and bit-flipped scans: the status says so (and PIL decides what the image is)."""
    from assembled_cnn_b200 import jpeg
    rng = np.random.default_rng(11)
    for kw in (dict(quality=90), dict(quality=75, restart_marker_blocks=2), dict(quality=95, optimize=True)):
        b = JC.encode(JC.image(120, 88, "noise", rng), **kw)
        d = jpeg.parse([b])[0]
        start, n = int(d["ecs_offset"]), int(d["ecs_length"])
        st, _ = host_decode(host, b[:start + n // 2])
        assert st & (jpeg.ST_OUT_OF_BITS | jpeg.ST_MCU_COUNT | jpeg.ST_BAD_CODE), st
        flagged = 0
        for k in range(20):
            bad = bytearray(b)
            pos = start + int(rng.integers(0, n))
            bad[pos] ^= 1 << int(rng.integers(0, 8))
            if bad[pos] == 0xFF or (pos > 0 and bad[pos - 1] == 0xFF):
                continue
            st, out = host_decode(host, bytes(bad))
            if st:
                flagged += 1
            else:   # a flip that still decodes cleanly must decode as PIL does
                assert np.array_equal(out, JC.pil_rgb(bytes(bad)))
        assert flagged > 0
