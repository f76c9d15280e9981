"""The z pass's warp-local record test against the candidate scatter + pixel test, on the CPU
(tests/warp_test/harness.cpp drives the phase functions of phases.h in `for (tid ...)` loops).

For random chunks of 1 to 128 pre-masked records - one to four 32-record groups of the warp test, on either side of
the size where the kernel switches between the two paths - each pixel's candidate set and its final (z, own, bown)
must be the ones the scatter + pixel test give, bit for bit: small-triangle-like masks, dense masks (pixels with more than PIX_SLOTS
candidates), exact z ties between distinct triangles, and perspective-correct (1/z) planes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

_HERE = os.path.dirname(os.path.abspath(__file__))
PRE_DTYPE = np.dtype([("mask", "<u4", 8), ("zp", "<f8", 3), ("id", "<i4"), ("pad", "<i4")])
assert PRE_DTYPE.itemsize == 64
SMALL_FLAG = 0x40000000
PIX_SLOTS = 8


@pytest.fixture(scope="module")
def lib():
    d = os.path.join(_HERE, "warp_test")
    subprocess.run(["make", "-C", d, "libwarptest.so"], check=True, capture_output=True)
    L = C.CDLL(os.path.join(d, "libwarptest.so"))
    L.wt_run_chunk.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 4
    L.wt_run_chunk.restype = C.c_int
    return L


def small_mask(rng):
    """Coverage of a micro-triangle-like blob: a few rows of short spans, anywhere in the 16x16 tile."""
    m = np.zeros(16, np.uint32)  # row masks
    y0 = rng.integers(0, 16)
    h = rng.integers(1, 5)
    x0 = rng.integers(0, 16)
    for y in range(y0, min(16, y0 + h)):
        xb = max(0, x0 + rng.integers(-2, 2))
        xe = min(15, xb + rng.integers(0, 6))
        m[y] = ((1 << (xe - xb + 1)) - 1) << xb
    return (m[0::2] | (m[1::2] << 16)).astype(np.uint32)


def make_chunk(rng, n, dense=0.0, tie_frac=0.2, persp=False):
    recs = np.zeros(n, PRE_DTYPE)
    for t in range(n):
        if rng.random() < dense:
            recs[t]["mask"] = rng.integers(0, 2 ** 32, size=8, dtype=np.uint64).astype(np.uint32)
        else:
            recs[t]["mask"] = small_mask(rng)
        if persp:  # 1/z plane, positive over the tile
            recs[t]["zp"] = [rng.uniform(-1e-4, 1e-4), rng.uniform(-1e-4, 1e-4), rng.uniform(0.05, 1.0)]
        else:
            recs[t]["zp"] = [rng.uniform(-0.01, 0.01), rng.uniform(-0.01, 0.01), rng.uniform(1.0, 10.0)]
        recs[t]["id"] = int(rng.integers(0, 1 << 20)) | (SMALL_FLAG if rng.random() < 0.7 else 0)
    # exact ties: copies of another record's plane under a different triangle id
    for t in range(n):
        if n > 1 and rng.random() < tie_frac:
            src = int(rng.integers(0, n))
            recs[t]["zp"] = recs[src]["zp"]
    # exact ties on a constant plane: every such pixel ties
    if n >= 4 and rng.random() < 0.5:
        for t in rng.choice(n, size=3, replace=False):
            recs[t]["zp"] = [0.0, 0.0, 2.0 if not persp else 0.5]
    return recs


def run(lib, recs, persp, x0=32, y0=48):
    n = len(recs)
    recs = np.ascontiguousarray(recs)
    mism = np.zeros(4, np.int32)
    z = np.zeros(256)
    own = np.zeros(256, np.int32)
    bown = np.zeros(256, np.int32)
    rc = lib.wt_run_chunk(recs.ctypes.data, n, x0, y0, int(persp), mism.ctypes.data, z.ctypes.data, own.ctypes.data,
                          bown.ctypes.data)
    assert rc == 0
    return mism, z, own, bown


NAMES = ["scattered candidate lists", "warp candidate sets", "warp test states", "candidate counters left"]


@pytest.mark.parametrize("persp", [False, True])
def test_every_chunk_size(lib, persp):
    rng = np.random.default_rng(7 + persp)
    for n in range(1, 129):
        for rep in range(3):
            recs = make_chunk(rng, n, dense=0.05 if rep == 2 else 0.0, persp=persp)
            mism, *_ = run(lib, recs, persp)
            bad = {NAMES[k]: int(mism[k]) for k in range(4) if mism[k]}
            assert not bad, f"n={n} rep={rep}: {bad}"


@pytest.mark.parametrize("n", [1, 31, 32, 33, 64, 65, 127, 128])
def test_crowded_pixels_and_ties(lib, n):
    """Dense masks: many pixels with more than PIX_SLOTS candidates (the scan fall-back of phase_pix_test); every
    record on one of two planes so that most covered pixels end in an exact tie."""
    rng = np.random.default_rng(100 + n)
    recs = make_chunk(rng, n, dense=0.6, tie_frac=0.0)
    planes = np.array([[0.0, 0.0, 3.0], [0.001, -0.002, 3.0]])
    for t in range(n):
        recs[t]["zp"] = planes[t % 2]
    mism, z, own, bown = run(lib, recs, False)
    assert not mism.any(), {NAMES[k]: int(mism[k]) for k in range(4) if mism[k]}
    counts = np.zeros(256, int)
    for t in range(n):
        for p in range(8):
            w = int(recs[t]["mask"][p])
            for lane in range(32):
                counts[p * 32 + lane] += (w >> lane) & 1
    if n > PIX_SLOTS:
        assert (counts > PIX_SLOTS).any()
    if n > 2:
        assert (own != bown).any()  # exact ties between distinct triangles were exercised


def test_empty_words_and_single_pixels(lib):
    """Records covering one pixel each, most row pairs empty: the warps that find no candidate do nothing."""
    rng = np.random.default_rng(3)
    for n in (1, 2, 17, 32, 33, 96, 128):
        recs = make_chunk(rng, n)
        for t in range(n):
            recs[t]["mask"] = 0
            px = int(rng.integers(0, 256))
            recs[t]["mask"][px // 32] = np.uint32(1 << (px % 32))
        mism, *_ = run(lib, recs, False)
        assert not mism.any(), (n, mism)
