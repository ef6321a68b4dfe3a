"""The input loops' staging helpers without a GPU: read_ahead's order, its bound on the batches in flight and
its error propagation; the 16-byte aligned offsets pack_u8 places arrays at."""
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from assembled_cnn_b200.staging import aligned_offsets, read_ahead


@pytest.mark.parametrize("ahead", [1, 2, 4])
def test_read_ahead_order_and_bound(ahead):
    batches = [[(j, i) for i in range(j % 3 + 1)] for j in range(11)]
    read = []                # the batches the generator has taken from `batches`
    lock = threading.Lock()

    def source():
        for b in batches:
            read.append(b[0][0])
            yield b

    def work(item):
        with lock:
            return item[0] * 100 + item[1]

    with ThreadPoolExecutor(max_workers=3) as pool:
        for j, (b, results) in enumerate(read_ahead(pool, source(), work, ahead=ahead)):
            assert b == batches[j]
            assert results == [j * 100 + i for i in range(len(b))]
            # batches j+1 .. j+ahead are submitted, and nothing beyond
            assert read == list(range(min(j + ahead, len(batches) - 1) + 1))


def test_read_ahead_raises_worker_error_at_its_batch():
    def work(x):
        if x == 5:
            raise KeyError("bad record")
        return x

    seen = []
    with ThreadPoolExecutor(max_workers=2) as pool:
        with pytest.raises(KeyError, match="bad record"):
            for b, results in read_ahead(pool, [[0, 1], [2, 3], [4, 5], [6, 7]], work):
                seen.append(results)
    assert seen == [[0, 1], [2, 3]]


def test_read_ahead_empty():
    with ThreadPoolExecutor(max_workers=1) as pool:
        assert list(read_ahead(pool, [], lambda x: x)) == []


def test_pack_u8_aligned_offsets():
    arrays = [np.zeros(n, np.uint8) for n in (1, 16, 17, 3 * 5 * 7, 0, 32)]
    offs = aligned_offsets(arrays)
    assert offs == [0, 16, 32, 64, 176, 176, 208]
    assert all(o % 16 == 0 for o in offs)
    for a, o, nxt in zip(arrays, offs, offs[1:]):
        assert o + a.nbytes <= nxt < o + a.nbytes + 16
