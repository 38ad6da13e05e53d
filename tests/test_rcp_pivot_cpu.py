"""The reciprocal the chain eliminations use for their pivots (csrc/trl_rcp.cuh: rcp_pivot) against 1.0 / x.

The device seed (MUFU.RCP64H) is not available on the CPU, so the five FMAs after it are run from seeds whose high word is that of
the rounded reciprocal moved up to 2 units either way, with the device's low word: the result must be 1.0 / x, bit for bit, for every
such seed -- for an x whose significand is all ones only from seeds at or above the power of two 1 / x lies just above (from
below, Markstein's final correction cannot round up across the power of two; the device seed is the one the compiler's own `1.0 / x`
uses, which rounds correctly there).  Operands: the pivots of real trajectories (tests/golden/rcp_pivots.npy: 20,000 of the distinct
pivots the kernel source met in 3 envs each of dog / slopes_mixed, raptor / narrow_gaps and goat / cliffs, 100-140 env-steps, on
the SIMT emulator), dense samples of [2^-40, 2^40], and both sides of every exponent boundary in that range, including the
all-ones significands just below each power of two."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deepterrainrl_b200", "csrc")
OFFSETS = (-2, -1, 0, 1, 2)

DRIVER = r"""
#define __device__
#define __forceinline__ inline
#include "trl_rcp.cuh"
extern "C" void rcp_refine_seeded(const double* x, long n, int hi_offset, double* out) {
    for (long i = 0; i < n; ++i) out[i] = trl::rcp_refine(x[i], trl::rcp_seed_emu(x[i], hi_offset));
}
extern "C" void rcp_pivot_cpu(const double* x, long n, double* out) {
    for (long i = 0; i < n; ++i) out[i] = trl::rcp_pivot(x[i]);
}
"""


@pytest.fixture(scope="module")
def lib():
    with tempfile.TemporaryDirectory() as d:
        src, so = os.path.join(d, "rcp.cpp"), os.path.join(d, "librcp.so")
        with open(src, "w") as f:
            f.write(DRIVER)
        subprocess.run([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-DTRL_SIMT_EMU=1",
                        "-I", CSRC, src, "-o", so], check=True)
        L = C.CDLL(so)
        for fn in (L.rcp_refine_seeded, L.rcp_pivot_cpu):
            fn.restype = None
        yield L


def _check(L, x):
    x = np.ascontiguousarray(x, np.float64)
    want = 1.0 / x
    out = np.empty_like(x)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    all_ones = (x.view(np.uint64) & np.uint64((1 << 52) - 1)) == np.uint64((1 << 52) - 1)
    for off in OFFSETS:
        L.rcp_refine_seeded(ptr(x), C.c_long(len(x)), off, ptr(out))
        bad = np.flatnonzero((out.view(np.uint64) != want.view(np.uint64)) & ~(all_ones & (off < 0)))
        assert len(bad) == 0, (off, x[bad[:5]], out[bad[:5]], want[bad[:5]])
    L.rcp_pivot_cpu(ptr(x), C.c_long(len(x)), ptr(out))
    assert out.tobytes() == want.tobytes()


def test_recorded_pivots(lib):
    piv = np.load(os.path.join(ROOT, "tests", "golden", "rcp_pivots.npy"))
    assert len(piv) > 1000 and (piv > 0).all()
    _check(lib, piv)


def test_dense_samples(lib):
    rng = np.random.default_rng(7)
    _check(lib, np.exp2(rng.uniform(-40.0, 40.0, 2_000_000)))
    # every significand pattern of the seed's 20 leading fraction bits, near 1
    _check(lib, 1.0 + (np.arange(1 << 20) + rng.uniform(0.0, 1.0, 1 << 20)) * 2.0 ** -20)


def test_exponent_boundaries(lib):
    p = np.exp2(np.arange(-40, 41, dtype=np.float64))
    below = np.nextafter(p, 0.0)                     # all-ones significands
    xs = [p, below, np.nextafter(p, np.inf), np.nextafter(below, 0.0)]
    for k in range(1, 64):                           # a run of neighbours on both sides
        xs += [p * (1.0 + k * 2.0 ** -52), p * (1.0 - k * 2.0 ** -53)]
    _check(lib, np.concatenate(xs))
