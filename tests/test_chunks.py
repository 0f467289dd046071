"""The chunk rule of option "chunk_atoms" (the reference's --chunk-size), on the CPU.

The engine's own rule (vb_chunk_fragments of the C library, through ctypes, and its wrapper
ai2bmd_b200.parallel.chunk_fragments) against tests/golden/reference_chunks.json, which the reference's own
DeviceStrategy._set_combined_work_partitions wrote (tests/golden/make_reference_chunks.py): blocks per device first, then chunks
inside each block.  Then the cases where this rule departs from the reference on purpose: chunks smaller than a
fragment, fragments without atoms, and a negative chunk size.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def lib():
    from ai2bmd_b200 import engine as vengine
    return vengine.load_library()


def lib_chunks(lib, offsets, chunk):
    """[(lo, hi)] from vb_chunk_fragments on fragment atom offsets [G + 1]; a negative status as is."""
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    out = np.full(len(offsets), -7, dtype=np.int64)
    n = lib.vb_chunk_fragments(len(offsets) - 1, offsets.ctypes.data_as(C.c_void_p), int(chunk),
                               out.ctypes.data_as(C.c_void_p))
    if n < 0:
        return n
    return [(int(out[c]), int(out[c + 1])) for c in range(n)]


def _golden():
    return json.load(open(os.path.join(GOLDEN, "reference_chunks.json")))


@pytest.mark.parametrize("key", sorted(_golden()))
def test_chunks_equal_the_reference_function(lib, key):
    from ai2bmd_b200.fixtures import load_fragments
    from ai2bmd_b200.parallel import chunk_fragments, partition_fragments
    name, n_dev, chunk = key.split(":")
    n_dev, chunk = int(n_dev), int(chunk)
    fd, _ = load_fragments(name)
    start, end = np.asarray(fd.start), np.asarray(fd.end)
    want = [tuple(x) for x in _golden()[key]]
    blocks = partition_fragments(start, end, n_dev) if n_dev > 1 else [(0, len(start))]
    got_lib, got_py = [], []
    for dev, (lo, hi) in enumerate(blocks):
        if hi <= lo:
            continue
        offsets = np.append(start[lo:hi], end[hi - 1]) - start[lo]
        got_lib += [(dev, lo + a, lo + b) for a, b in lib_chunks(lib, offsets, chunk)]
        got_py += [(dev, lo + a, lo + b) for a, b in chunk_fragments(start[lo:hi], end[lo:hi], chunk)]
    assert got_lib == want
    assert got_py == want


def test_every_golden_chunk_size_cuts_the_batch(lib):
    """The golden cases are not all one chunk per block: the rule is exercised, not bypassed."""
    g = _golden()
    assert any(len(v) > 4 * int(k.split(":")[1]) for k, v in g.items())
    assert all(v[0][1] == 0 for v in g.values())


def test_chunk_below_every_fragment_takes_one_fragment_each(lib):
    from ai2bmd_b200.fixtures import load_fragments
    from ai2bmd_b200.parallel import chunk_fragments
    fd, _ = load_fragments("chig")
    start, end = np.asarray(fd.start), np.asarray(fd.end)
    sizes = end - start
    for chunk in (1, 5, int(sizes.min()) // 2, int(sizes.min()) - 1):   # the reference's loop never ends on the first three
        assert chunk_fragments(start, end, chunk) == [(g, g + 1) for g in range(len(start))]
    # 100 atoms on Chignolin: whole fragments, contiguous, each chunk within a fragment of the target
    ch = chunk_fragments(start, end, 100)
    assert ch[0][0] == 0 and ch[-1][1] == len(start) and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
    assert all(abs(int(end[hi - 1] - start[lo]) - 100) <= sizes.max() for lo, hi in ch[:-1])


def test_zero_chunk_is_one_chunk(lib):
    assert lib_chunks(lib, [0, 10, 25, 31], 0) == [(0, 3)]


def test_fragments_without_atoms_join_the_chunk_they_fall_in(lib):
    # sizes 10, 0, 10, 0, 0, 10, 0: the empty fragments (CYX partner slots) never form a chunk of their own
    sizes = [10, 0, 10, 0, 0, 10, 0]
    offsets = np.concatenate([[0], np.cumsum(sizes)])
    for chunk in (1, 4, 10, 15, 20, 1000):
        ch = lib_chunks(lib, offsets, chunk)
        assert ch[0][0] == 0 and ch[-1][1] == len(sizes) and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
        assert all(offsets[hi] > offsets[lo] for lo, hi in ch), (chunk, ch)
    # an empty fragment at a cut opens the next chunk; trailing ones close the last chunk
    assert lib_chunks(lib, offsets, 1) == [(0, 1), (1, 3), (3, 7)]
    assert lib_chunks(lib, offsets, 1000) == [(0, 7)]
    # leading empty fragments join the first chunk that has atoms
    assert lib_chunks(lib, [0, 0, 0, 5, 10], 1) == [(0, 3), (3, 4)]
    # a batch whose fragments are all empty is one chunk
    assert lib_chunks(lib, [0, 0, 0], 3) == [(0, 2)]


def test_bad_input_is_rejected(lib):
    from ai2bmd_b200.parallel import chunk_fragments
    assert lib_chunks(lib, [0, 10, 20], -1) < 0
    assert lib_chunks(lib, [0, 10, 5], 10) < 0                      # offsets that decrease
    with pytest.raises(ValueError):
        chunk_fragments([0, 10], [10, 20], -1)
    with pytest.raises(ValueError):
        chunk_fragments([0, 12], [10, 20], 10)                       # not packed
