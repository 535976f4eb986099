"""The work split of the four-step row pass (k_fs_rows in reevr_b200/csrc/kernels_fourstep.cuh) on the CPU: every
persistent CTA walks item_range(items, ctas, b), and those ranges must cover each item (a row of the column spectra)
exactly once, in order, with no range longer than ceil(items / ctas).  The function is the header's own, compiled by g++
through tests/cpp/fourstep_range_shim.cpp; the kernel itself is covered on the GPU (tests/test_fourstep.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fsr") / "libfourstep_range.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, os.path.join(ROOT, "tests", "cpp", "fourstep_range_shim.cpp"), "-o", so]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lib = C.CDLL(so)
    lib.fsr_ranges.argtypes = [C.c_uint, C.c_uint, np.ctypeslib.ndpointer(np.uint32), np.ctypeslib.ndpointer(np.uint32)]
    return lib


def ranges(lib, items, ctas):
    b, e = np.zeros(ctas, np.uint32), np.zeros(ctas, np.uint32)
    lib.fsr_ranges(items, ctas, b, e)
    return b.astype(np.int64), e.astype(np.int64)


# the IR-spectrum build (nseg = 1) at C = 1 ... 8, short and long groups, and the metric's stereo group (nseg = 36)
ITEMS = sorted({c * 257 for c in range(1, 9)} | {c * 257 * q for c in (1, 2, 4, 8) for q in (2, 3, 7, 17)} | {18504, 1, 299})


@pytest.mark.parametrize("items", ITEMS)
def test_every_item_once(shim, items):
    assert shim.fsr_rows() == 257
    for ctas in range(1, 301):
        b, e = ranges(shim, items, ctas)
        assert b[0] == 0 and e[-1] == items
        assert np.all(b[1:] == e[:-1])                       # contiguous, in order: each item exactly once
        assert np.all(e >= b)
        assert (e - b).max() <= -(-items // ctas)
        if items >= ctas:
            assert (e - b).min() >= items // ctas           # balanced: lengths differ by at most one


def test_metric_ranges_cross_few_rows(shim):
    # stereo, 36 segments per row: 264 resident CTAs (132 SMs x 2) each cross at most two row boundaries, so a CTA
    # fetches at most three spectrum rows
    nseg, items = 36, 18504
    b, e = ranges(shim, items, 264)
    rows = (e - 1) // nseg - b // nseg + 1
    assert rows.max() <= 3
