"""The four-step sweep (reevr_b200/csrc/kernels_fourstep.cuh, cmac_variant 42) on the CPU: a float64 numpy model of
exactly its factorisation — two real columns packed per complex 512-point DFT and separated by Z[k] +- conj Z[-k],
the Hermitian half k1 = 0 ... 256 with rows 0 and 256 as ordinary complex rows, the twiddles W_M^{n2 k1}, the
4096-point row transforms with the spectrum and the conjugate inverse, the rebuilt full column spectrum of the
inverse — over the header's segment plan (history in front of the group, the partial last segment), against direct
convolution.  The plan's functions are the header's own, compiled by g++ through tests/cpp/fourstep_plan_shim.cpp; the
kernels are covered on the GPU (tests/test_fourstep.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 512


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fsp") / "libfourstep_plan.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, os.path.join(ROOT, "tests", "cpp", "fourstep_plan_shim.cpp"), "-o", so]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lib = C.CDLL(so)
    lib.fsp_m.restype = C.c_longlong
    lib.fsp_window_start.restype = C.c_longlong
    lib.fsp_window_start.argtypes = [C.c_int, C.c_longlong, C.c_int]
    lib.fsp_output_of.restype = C.c_longlong
    lib.fsp_output_of.argtypes = [C.c_int, C.c_longlong, C.c_int, C.c_longlong]
    lib.fsp_plan.argtypes = [C.c_int, C.c_longlong, C.POINTER(C.c_longlong)]
    lib.fsp_work_bytes.restype = C.c_ulonglong
    lib.fsp_work_bytes.argtypes = [C.c_int, C.c_longlong, C.c_int]
    lib.fsp_spectrum_bytes.restype = C.c_ulonglong
    lib.fsp_hist_bytes.restype = C.c_ulonglong
    return lib


def plan(lib, P, n):
    out = (C.c_longlong * 5)()
    lib.fsp_plan(P, n, out)
    return dict(zip(("P", "nseg", "Lh", "L", "n"), out))


class Model:
    """float64 four-step overlap-save, pass by pass as the kernels compute it"""

    def __init__(self, lib):
        self.N1, self.N2, self.M, self.R = lib.fsp_n1(), lib.fsp_n2(), lib.fsp_m(), lib.fsp_rows()
        k1 = np.arange(self.R)[:, None]
        n2 = np.arange(self.N2)[None, :]
        self.tw = np.exp(-2j * np.pi * (n2 * k1) / self.M)           # W_M^{n2 k1}, k1 = 0 ... 256

    def cols(self, win):
        """pass 1: window of M real samples -> [257][4096] twiddled column spectra"""
        x = win.reshape(self.N1, self.N2)                            # x[n1][n2] = win[N2 n1 + n2]
        Z = np.fft.fft(x[:, 0::2] + 1j * x[:, 1::2], axis=0)         # two real columns per complex transform
        Zm = np.conj(Z[(-np.arange(self.N1)) % self.N1])             # conj Z[-k1]: in the same lane
        A = np.empty((self.R, self.N2), np.complex128)
        A[:, 0::2] = ((Z + Zm) / 2)[:self.R]
        A[:, 1::2] = ((Z - Zm) / 2j)[:self.R]
        return A * self.tw

    def spectrum(self, h):
        """the IR spectrum: passes 1 and 2 of the taps, times 1 / M"""
        win = np.zeros(self.M)
        win[:h.size] = h
        return np.fft.fft(self.cols(win), axis=1) / self.M

    def rows(self, A, S):
        """pass 2: row FFT, product, inverse as conj(FFT(conj(.)))"""
        return np.conj(np.fft.fft(np.conj(np.fft.fft(A, axis=1) * S), axis=1))

    def cols_inv(self, Cr):
        """pass 3: undo the twiddle, rebuild the full column spectra from the half, inverse 512-point DFTs"""
        D = Cr * np.conj(self.tw)
        D[0] = D[0].real                                             # real bins of a real column
        D[self.R - 1] = D[self.R - 1].real
        full = np.empty((self.N1, self.N2), np.complex128)
        full[:self.R] = D
        full[self.R:] = np.conj(D[1:self.R - 1][::-1])               # D[512 - k1] = conj D[k1]
        Z = full[:, 0::2] + 1j * full[:, 1::2]
        z = np.fft.ifft(Z, axis=0) * self.N1                         # unscaled: 1 / M is in the spectrum
        y = np.empty((self.N1, self.N2))
        y[:, 0::2] = z.real
        y[:, 1::2] = z.imag
        return y.reshape(-1)

    def run(self, lib, P, hist, x, h):
        """the group's outputs and how often each was written"""
        p = plan(lib, P, x.size)
        S = self.spectrum(h)
        y = np.full(x.size, np.nan)
        hits = np.zeros(x.size, np.int64)
        for q in range(p["nseg"]):
            w0 = lib.fsp_window_start(P, x.size, q)
            pos = w0 + np.arange(self.M)
            win = np.zeros(self.M)
            neg = pos < 0
            win[neg] = hist[hist.size + pos[neg]]
            ok = (pos >= 0) & (pos < x.size)
            win[ok] = x[pos[ok]]
            c = self.cols_inv(self.rows(self.cols(win), S))
            m = np.arange(self.M)
            t = q * p["L"] + m - (p["Lh"] - 1)
            valid = (m >= p["Lh"] - 1) & (t < x.size)
            for mm in (0, p["Lh"] - 2, p["Lh"] - 1, self.M - 1):     # the header's output_of
                want = int(t[mm]) if valid[mm] else -1
                assert lib.fsp_output_of(P, x.size, q, mm) == want
            y[t[valid]] = c[valid]
            hits[t[valid]] += 1
        return y, hits, p


@pytest.fixture(scope="module")
def model(shim):
    return Model(shim)


def group(lib, P, n, seed):
    rng = np.random.default_rng(seed)
    Lh = P * B
    h = rng.standard_normal(Lh) * np.exp(-np.arange(Lh) / (0.3 * Lh))
    return rng.standard_normal(Lh - 1), rng.standard_normal(n), h


@pytest.mark.parametrize("P,extra", [(1, 1), (3, 4095)])
def test_against_np_convolve(shim, model, P, extra):
    """short IRs: the whole group against np.convolve of history and samples (two segments, the last one partial)"""
    p0 = plan(shim, P, 1)
    n = p0["L"] + extra
    hist, x, h = group(shim, P, n, 17 + P)
    y, hits, p = model.run(shim, P, hist, x, h)
    assert p["nseg"] == 2
    assert np.all(hits == 1)
    ref = np.convolve(np.concatenate([hist, x]), h)[hist.size:hist.size + n]
    assert np.max(np.abs(y - ref)) <= 1e-11 * np.max(np.abs(ref))


@pytest.mark.parametrize("P", [938, 961])
def test_long_ir_at_the_segment_edges(shim, model, P):
    """the metric's IR lengths, three segments and one block: outputs at the start (history), at both edges of every
    segment and at the end, each against its direct sum"""
    p0 = plan(shim, P, 1)
    n = 3 * p0["L"] + B
    hist, x, h = group(shim, P, n, P)
    y, hits, p = model.run(shim, P, hist, x, h)
    assert p["nseg"] == 4 and np.all(hits == 1)
    xx = np.concatenate([hist, x])
    hr = h[::-1]
    ts = [0, 1, 100, h.size - 2, n - 1]
    for q in range(1, p["nseg"]):
        ts += [q * p["L"] - 1, q * p["L"]]
    for t in ts:
        want = float(np.dot(hr, xx[t:t + h.size]))
        assert abs(y[t] - want) <= 1e-11 * np.sum(np.abs(h)) * np.max(np.abs(xx)), t


def test_column_pairing_and_hermitian_half(model):
    """pass 1 of a window equals the M-point FFT rows k1 = 0 ... 256 before the row transform: X[k1 + 512 k2]"""
    rng = np.random.default_rng(3)
    win = rng.standard_normal(model.M)
    X = np.fft.fft(win)
    got = np.fft.fft(model.cols(win), axis=1)
    want = X.reshape(model.N2, model.N1).T[:model.R]                  # [k1][k2] = X[k1 + N1 k2]
    assert np.max(np.abs(got - want)) <= 1e-9 * np.max(np.abs(X))
    # rows 0 and 256 are complex between the passes
    assert np.max(np.abs(model.cols(win)[[0, model.R - 1]].imag)) > 1.0


def test_plan_and_scratch(shim):
    M = shim.fsp_m()
    assert M == 1 << 21 and shim.fsp_rows() == 257
    assert shim.fsp_plan_ok(1) and shim.fsp_plan_ok(961) and not shim.fsp_plan_ok(962) and not shim.fsp_plan_ok(0)
    p = plan(shim, 938, 112608 * B)                                   # the metric step
    assert p["L"] == M - (938 * B - 1) and p["nseg"] == 36
    assert shim.fsp_window_start(938, p["n"], 0) == -(938 * B - 1)
    assert shim.fsp_window_start(938, p["n"], 1) == p["L"] - (938 * B - 1)
    assert shim.fsp_work_bytes(938, p["n"], 2) == 2 * 36 * 257 * 4096 * 8
    assert shim.fsp_spectrum_bytes(2) == 2 * 257 * 4096 * 8
    assert shim.fsp_hist_bytes(938, 2) == 2 * 938 * B * 4
