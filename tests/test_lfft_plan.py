"""The segment plan of the line-FFT sweep (reevr_b200/csrc/kernels_lfft.cuh, cmac_variant 41) on the CPU: a float64
model of overlap-save along the block index — window starts, the valid outputs of each segment, zeros past the line's
Lt samples, the DC / Nyquist entry's two real convolutions and the one-block-early start of a time-slice rank (extra)
— against direct convolution.  The plan's functions are the header's own, compiled by g++ through
tests/cpp/lfft_plan_shim.cpp; the kernels are covered on the GPU (tests/test_lfft_sweep.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lfp") / "liblfft_plan.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, os.path.join(ROOT, "tests", "cpp", "lfft_plan_shim.cpp"), "-o", so]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lib = C.CDLL(so)
    lib.lfp_window_start.restype = C.c_longlong
    lib.lfp_window_start.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.lfp_output_of.restype = C.c_longlong
    lib.lfp_output_of.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    lib.lfp_spectra_bytes.restype = C.c_ulonglong
    lib.lfp_spectra_bytes.argtypes = [C.c_ulonglong, C.c_int]
    return lib


def plan(lib, P, nb):
    out = (C.c_longlong * 6)()
    lib.lfp_plan(P, nb, out)
    return dict(zip(("P", "Q", "L", "nseg", "Lt", "Lty"), out))


def sweep_model(lib, P, nb, x, h):
    """float64 overlap-save of the complex line x (Lt samples) with the P values h, segment by segment as the kernel
    plans it; returns the Lty outputs and how often each was written"""
    N = lib.lfp_n()
    p = plan(lib, P, nb)
    y = np.zeros(p["Lty"], np.complex128)
    hits = np.zeros(p["Lty"], np.int64)
    Hf = np.fft.fft(h, N)
    for q in range(p["nseg"]):
        w0 = lib.lfp_window_start(P, nb, q)
        win = np.zeros(N, np.complex128)
        n = max(0, min(N, p["Lt"] - w0))                     # past Lt: zeros
        win[:n] = x[w0:w0 + n]
        c = np.fft.ifft(np.fft.fft(win) * Hf)
        for m in range(N):
            s = lib.lfp_output_of(P, nb, q, m)
            if s >= 0:
                y[s] = c[m]
                hits[s] += 1
    return y, hits, p


def direct(x, h, Q, Lty):
    """y[s] = sum_p h[p] x[s + Q - p], x zero past its end"""
    P = h.size
    xp = np.concatenate([x, np.zeros(Lty + Q + 1, x.dtype)])
    y = np.zeros(Lty, np.complex128)
    for p in range(P):
        y += h[p] * xp[Q - p:Q - p + Lty]
    return y


@pytest.mark.parametrize("P,nb", [(1, 1), (2, 100), (64, 4097), (65, 300), (938, 16384), (961, 16385), (961, 3 * 4096 + 7)])
def test_segment_plan_against_direct_convolution(shim, P, nb):
    rng = np.random.default_rng(P * 7919 + nb)
    p = plan(shim, P, nb)
    N = shim.lfp_n()
    assert p["L"] == N - (P - 1) and p["nseg"] * p["L"] >= p["Lty"] > (p["nseg"] - 1) * p["L"]
    assert shim.lfp_window_start(P, nb, 0) == p["Q"] - (P - 1) >= 0
    x = rng.standard_normal(p["Lt"]) + 1j * rng.standard_normal(p["Lt"])
    h = rng.standard_normal(P) + 1j * rng.standard_normal(P)
    y, hits, _ = sweep_model(shim, P, nb, x, h)
    assert np.all(hits == 1)                                  # every output slot written once
    ref = direct(x, h, p["Q"], p["Lty"])
    assert np.max(np.abs(y - ref)) <= 1e-9 * np.max(np.abs(ref))
    # the last segment's window runs past Lt (it reads zeros there) unless the outputs end just inside it
    assert shim.lfp_window_start(P, nb, p["nseg"] - 1) + N >= p["Lty"] + p["Q"]


def test_dc_nyquist_entry_as_two_real_convolutions(shim):
    """entry 0: Z = FFT(xr + i xi), FFT(y) = Z (HR + HI) / 2 + conj(Z[-f]) (HR - HI) / 2 gives (hr * xr, hi * xi)"""
    N = shim.lfp_n()
    rng = np.random.default_rng(5)
    P = 961
    xr, xi = rng.standard_normal(N), rng.standard_normal(N)
    hr, hi = rng.standard_normal(P), rng.standard_normal(P)
    Z = np.fft.fft(xr + 1j * xi)
    HR, HI = np.fft.fft(hr, N), np.fft.fft(hi, N)
    Zm = np.conj(Z[(-np.arange(N)) % N])
    y = np.fft.ifft(Z * (HR + HI) / 2 + Zm * (HR - HI) / 2)
    ref_r = np.real(np.fft.ifft(np.fft.fft(xr) * HR))
    ref_i = np.real(np.fft.ifft(np.fft.fft(xi) * HI))
    assert np.max(np.abs(y.real - ref_r)) <= 1e-9 * np.max(np.abs(ref_r))
    assert np.max(np.abs(y.imag - ref_i)) <= 1e-9 * np.max(np.abs(ref_i))


@pytest.mark.parametrize("extra", [0, 1])
def test_extra_block_in_front(shim, extra):
    """block t of the group sits at tau = Q + extra + t and comes out at slot extra + t; with extra = 1, slot 0 is block
    -1, the overlap state sum_p H[p] X[-1 - p]"""
    P, nb = 938, 5000
    p = plan(shim, P, nb + extra)
    rng = np.random.default_rng(11 + extra)
    hist = P + 2                                              # blocks in front of the group
    X = rng.standard_normal(hist + nb) + 1j * rng.standard_normal(hist + nb)   # X[hist + t] = block t
    h = rng.standard_normal(P) + 1j * rng.standard_normal(P)
    x = np.zeros(p["Lt"], np.complex128)
    for tau in range(p["Lt"]):
        b = tau - p["Q"] - extra                              # group block at tau
        if -hist <= b < nb:
            x[tau] = X[hist + b]
    y, _, _ = sweep_model(shim, P, nb + extra, x, h)
    for t in (-extra, 0, 1, P, nb - 1):
        want = sum(h[q] * X[hist + t - q] for q in range(P) if t - q >= -hist)
        assert abs(y[extra + t] - want) <= 1e-9 * np.sum(np.abs(h)) * np.max(np.abs(X))


def test_spectra_bytes(shim):
    N = shim.lfp_n()
    assert shim.lfp_spectra_bytes(1024, 2) == (1024 + 2) * N * 8
    assert (1024 + 2) * N * 8 <= 64 << 20                     # the metric shape: stereo, B = 512
