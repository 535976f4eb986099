"""The FP16 tensor-core sweep (reevr_b200/csrc/kernels_tc.cuh, cmac_variant 40) on the CPU: geometry, shared-memory
budget, the 16-bit SWIZZLE_128B offsets, the power-of-two exponent choice and a float64 model of the whole
arithmetic — k_tc_build_a (2^eh H split into FP16 hi / lo), k_tc_split_x (FP32 time lines, rows outside the history
read as zero), the sweep's producer (2^ex per tile and time line, FP16 hi / lo strips), the tiled Toeplitz products
hi*hi + hi*lo + lo*hi, the 2^-(ex + eh) epilogue and k_tc_merge_y — against a direct complex convolution, within the
bound DESIGN.md section 5 states.  The header's own inline functions are compiled by g++ through
tests/cpp/tc_f16_layout_shim.cpp; the kernels themselves are covered on the GPU (tests/test_tc_f16_range.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("tc16") / "libtc_f16_layout.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, os.path.join(ROOT, "tests", "cpp", "tc_f16_layout_shim.cpp"), "-o", so]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lib = C.CDLL(so)
    lib.tc16_sw128_h.restype = C.c_uint
    lib.tc16_sw128_h.argtypes = [C.c_uint, C.c_uint]
    lib.tc16_xf_index.restype = C.c_ulonglong
    lib.tc16_xf_index.argtypes = [C.c_longlong, C.c_int, C.c_longlong, C.c_int]
    lib.tc16_a_image_bytes.restype = C.c_ulonglong
    lib.tc16_a_image_bytes.argtypes = [C.c_ulonglong, C.c_int]
    lib.tc16_scale_exp.restype = C.c_int
    lib.tc16_scale_exp.argtypes = [C.c_uint]
    return lib


def geom(lib, P, nb):
    out = (C.c_int * 5)()
    lib.tc16_geom(P, nb, out)
    return dict(zip(("Q", "nchunk", "nseg", "ntile", "rows"), out))


def consts(lib):
    out = (C.c_int * 12)()
    lib.tc16_consts(out)
    return dict(zip(("R", "N", "strip_rows", "strip_bytes", "a_tile_bytes", "chunk_k", "max_chunks", "stage_bytes", "smem",
                     "flush", "a_stages", "strip_threads"), out))


def scale_exp(lib, values):
    """The kernels' exponent of a window: largest magnitude as float32 bits -> scale_exp."""
    v = np.asarray(values, np.float32)
    m = int(np.max(np.abs(v).view(np.uint32))) if v.size else 0      # integer max: NaN bits sort above Inf
    return lib.tc16_scale_exp(m)


def test_geometry_limits_and_shared_memory(shim):
    k = consts(shim)
    assert (k["R"], k["N"], k["strip_rows"], k["strip_bytes"], k["a_tile_bytes"], k["chunk_k"]) == (64, 64, 80, 80 * 128, 16384, 64)
    assert k["a_tile_bytes"] == 128 * k["chunk_k"] * 2                   # 128 rows [Hr ; Hi] x 64 halves
    assert k["stage_bytes"] == 2 * k["strip_rows"] * 64 * 4              # FP32 re / im rows of one tile
    # two FP16 buffers x (re, im) x (hi, lo) strips, the image ring, the FP32 staging rows, 1 KB of alignment slack
    assert k["smem"] == 8 * k["strip_bytes"] + k["a_stages"] * k["a_tile_bytes"] + k["stage_bytes"] + 1024
    assert k["smem"] + 1024 <= 227 * 1024                                # + the static barriers / exponents
    assert k["strip_bytes"] % 1024 == 0 and (k["a_stages"] * k["a_tile_bytes"]) % 1024 == 0
    assert k["strip_threads"] == 96
    g = geom(shim, 938, 112608)                                          # the metric shape
    assert g == dict(Q=960, nchunk=16, nseg=1760, ntile=28, rows=28 * 64 + 16)
    assert shim.tc16_a_image_bytes(1, g["nchunk"]) == 512 * 1024         # per line: half the tf32 images' 1 MB
    assert shim.tc16_geom_ok(961, 5000, 512) == 1 and shim.tc16_geom_ok(962, 5000, 512) == 0
    assert geom(shim, 961, 5000)["nchunk"] == k["max_chunks"] == 16
    assert shim.tc16_geom_ok(100, 5000, 48) == 0 and shim.tc16_geom_ok(1, 1, 32) == 1
    assert geom(shim, 1, 1) == dict(Q=0, nchunk=1, nseg=1, ntile=1, rows=80)
    for P in (1, 2, 65, 100, 938, 961):
        g = geom(shim, P, 9000)
        assert g["nchunk"] * 64 == g["Q"] + 64                            # K = Q + 64 in chunks of 64
        assert (g["nchunk"] - 1) + k["N"] <= k["strip_rows"]             # the largest row shift stays inside the strip


def test_f16_swizzle_is_a_permutation_of_each_row(shim):
    for r in range(16):
        offs = [shim.tc16_sw128_h(r, e) for e in range(64)]
        assert sorted(offs) == [r * 128 + 2 * e for e in range(64)]
        for q in range(8):                                                # 8 halves = one 16-byte unit, kept together
            assert offs[8 * q + 1:8 * q + 8] == [offs[8 * q] + 2 * i for i in range(1, 8)]
            assert offs[8 * q] - r * 128 == 16 * (q ^ (r % 8))           # the 128-byte swizzle: unit q ^ (row % 8)
    # the strip of tile nt is one contiguous piece of the FP32 time line
    rows = 3 * 64 + 16
    for line, comp, nt in [(0, 0, 0), (5, 1, 2), (7, 0, 1)]:
        base = shim.tc16_xf_index(line, comp, nt * 64 * 64, rows)
        assert shim.tc16_xf_index(line, comp, nt * 64 * 64 + 80 * 64 - 1, rows) == base + 80 * 64 - 1
        assert base == ((line * 2 + comp) * rows + nt * 64) * 64


def test_exponent_selection(shim):
    assert scale_exp(shim, [0.0, -0.0]) == 0                              # silence: exact zeros
    for bad in (np.inf, -np.inf, np.nan):                                 # non-finite windows stay unscaled
        assert scale_exp(shim, [1.0, bad, 3.0]) == 0
    assert scale_exp(shim, [1.0]) == 14 and scale_exp(shim, [32768.0]) == -1 and scale_exp(shim, [-1.5]) == 14
    rng = np.random.default_rng(7)
    u = rng.integers(1, 0x7f800000, 20000, dtype=np.uint64).astype(np.uint32)   # every finite magnitude, subnormals too
    u = np.concatenate([u, np.array([1, 0x007fffff, 0x00800000, 0x7f7fffff], np.uint32)])
    for m in u:
        v = float(np.uint32(m).view(np.float32))
        e = shim.tc16_scale_exp(int(m))
        assert 2.0 ** 14 <= v * 2.0 ** e < 2.0 ** 15, (hex(int(m)), e)
        assert -126 <= e // 2 and e - e // 2 <= 127                      # the producer's two factors are normal floats
    # scaling a window by 2^k moves its exponent by exactly -k
    w = rng.standard_normal(64).astype(np.float32)
    for k in (-100, -20, 0, 37, 100):
        assert scale_exp(shim, np.ldexp(w, k)) == scale_exp(shim, w) - k


def f16_split(v32):
    """The kernels' split of an FP32 value: FP16 hi (round to nearest even), FP16 rounding of the FP32 residual."""
    hi = v32.astype(np.float16)
    lo = (v32 - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def model(shim, H, x, P, nb, xrow0):
    """float64 model of build + split + sweep + merge; H [lines][P] complex64, x [lines][xrow0 + nb] complex64.
    Returns y [lines][nb] and, per line, the (tile, comp) exponents and eh."""
    g = geom(shim, P, nb)
    Q, rows, nchunk, ntile = g["Q"], g["rows"], g["nchunk"], g["ntile"]
    lines = H.shape[0]
    # k_tc_split_x: tau = row - (xrow0 - Q); rows outside [xrow0 - (P - 1), xrow0 + nb) read as zero
    Xt = np.full(lines * 2 * rows * 64, np.nan, np.float32)
    tau = np.arange(rows * 64)
    row = xrow0 - Q + tau
    inside = (row >= xrow0 - (P - 1)) & (row < xrow0 + nb)
    for line in range(lines):
        v = np.zeros(rows * 64, np.complex64)
        v[inside] = x[line, row[inside]]
        for comp in range(2):
            base = shim.tc16_xf_index(line, comp, 0, rows)
            Xt[base:base + rows * 64] = v.real if comp == 0 else v.imag
    assert not np.isnan(Xt).any()                                         # the poisoned history never reaches the strips
    y = np.zeros((lines, nb), complex)
    exps = []
    for line in range(lines):
        # k_tc_build_a: eh from the bin's P values, images of 2^eh H
        eh = scale_exp(shim, np.concatenate([H[line].real, H[line].imag]))
        Hs = [np.ldexp(H[line].real.astype(np.float32), eh), np.ldexp(H[line].imag.astype(np.float32), eh)]
        imgs = []
        i = np.arange(64)[:, None]
        jj = np.arange(64)[None, :]
        for c in range(nchunk):
            pp = i + Q - (64 * c + jj)
            ok = (pp >= 0) & (pp < P)
            A = np.zeros((128, 64), np.float32)
            for part in range(2):
                A[part * 64:part * 64 + 64][ok] = Hs[part][pp[ok]]
            imgs.append(f16_split(A))
        line_exps = []
        for nt in range(ntile):
            D = np.zeros((2, 128, 64))
            ex = [0, 0]
            for comp in range(2):
                base = shim.tc16_xf_index(line, comp, nt * 64 * 64, rows)
                strip = Xt[base:base + 80 * 64].reshape(80, 64)
                ex[comp] = scale_exp(shim, strip)
                s1, s2 = np.float32(2.0 ** (ex[comp] // 2)), np.float32(2.0 ** (ex[comp] - ex[comp] // 2))
                xh, xl = f16_split(strip * s1 * s2)
                for c in range(nchunk):
                    Ah, Al = imgs[c]
                    Bh, Bl = xh[c:c + 64], xl[c:c + 64]                    # row shift c: [n][jj]
                    D[comp] += Ah @ Bh.T + Ah @ Bl.T + Al @ Bh.T
                D[comp] = np.ldexp(D[comp], -(ex[comp] + eh))
            line_exps.append(ex)
            for n in range(64):                                           # k_tc_merge_y
                t0 = 64 * (nt * 64 + n)
                if t0 >= nb:
                    break
                cnt = min(64, nb - t0)
                d0, d1, e0, e1 = D[0, :cnt, n], D[0, 64:64 + cnt, n], D[1, :cnt, n], D[1, 64:64 + cnt, n]
                y[line, t0:t0 + cnt] = (d0 + 1j * e1) if line == 0 else (d0 - e1) + 1j * (d1 + e0)
        exps.append((eh, line_exps))
    return y, exps


def direct(H, x, P, nb, xrow0):
    lines = H.shape[0]
    ref = np.zeros((lines, nb), complex)
    absref = np.zeros((lines, nb))
    sum_h = np.zeros(lines)
    for line in range(lines):
        h = H[line].astype(complex)
        xs = np.stack([x[line, xrow0 + t - np.arange(P)] for t in range(nb)]).astype(complex)     # [t][p]
        if line == 0:
            ref[line] = xs.real @ h.real + 1j * (xs.imag @ h.imag)
        else:
            ref[line] = xs @ h
        ha, xa = np.maximum(abs(h.real), abs(h.imag)), np.maximum(abs(xs.real), abs(xs.imag))
        absref[line] = xa @ ha
        sum_h[line] = ha.sum()
    return ref, absref, sum_h


def bound(absref, sum_h, xsum, exps, nb):
    """DESIGN.md section 5: per real product |err| <= 3 * 2^-22 |h||x| + 2^-25 (2^-ex |h| + 2^-eh |x|); two real
    products per output component."""
    out = np.zeros_like(absref)
    for line, (eh, line_exps) in enumerate(exps):
        for t in range(nb):
            ex = min(line_exps[t // 4096])
            out[line, t] = 2 * (3 * 2.0 ** -22 * absref[line, t] + 2.0 ** -25 * (2.0 ** -ex * sum_h[line] + 2.0 ** -eh * xsum[line, t]))
    return out


@pytest.mark.parametrize("P,nb,quiet_db", [(100, 300, 0), (938, 200, 0), (1, 70, 0), (65, 4100, 0), (100, 300, 120), (65, 4100, 80)])
def test_float64_model_of_the_scaled_f16_sweep(shim, P, nb, quiet_db):
    rng = np.random.default_rng(P * 1000 + nb + quiet_db)
    g = geom(shim, P, nb)
    Q = g["Q"]
    lines = 2                                                             # line 0 is the packed DC / Nyquist entry
    H = (rng.standard_normal((lines, P)) + 1j * rng.standard_normal((lines, P))) * np.exp(-np.arange(P) / 40.0)
    H = H.astype(np.complex64)
    xrow0 = Q + 2
    x = (rng.standard_normal((lines, xrow0 + nb)) + 1j * rng.standard_normal((lines, xrow0 + nb))).astype(np.complex64)
    if quiet_db:                                                          # a step inside one tile window
        x[:, xrow0 + nb // 2:] *= np.float32(10.0 ** (-quiet_db / 20))
    x[:, :xrow0 - (P - 1)] = np.nan                                       # rows no sweep reads: must not leak in
    y, exps = model(shim, H, x, P, nb, xrow0)
    assert np.isfinite(y).all()
    ref, absref, sum_h = direct(H, x, P, nb, xrow0)
    xsum = np.zeros((lines, nb))
    for line in range(lines):
        xa = np.maximum(abs(x[line].real), abs(x[line].imag)).astype(np.float64)
        xsum[line] = [np.sum(xa[xrow0 + t - np.arange(P)]) for t in range(nb)]
    b = bound(absref, sum_h, xsum, exps, nb)
    err = np.maximum(abs(y.real - ref.real), abs(y.imag - ref.imag))
    assert (err <= b * (1 + 1e-9) + 1e-300).all(), float(np.max(err / b))
    # the quiet part keeps ~2^-22 relative precision within ~100 dB of its window's peak
    if quiet_db and quiet_db <= 100:
        t = np.arange(nb // 2 + P, nb)
        assert np.max(err[:, t] / absref[:, t]) <= 2.0 ** -19
    # exact power-of-two invariance: only the exponents move (while every scaled sample stays a normal float)
    if not quiet_db:
        for k in (100, -100):
            xk = (x * np.float32(2.0 ** k)).astype(np.complex64)
            xv = np.abs(np.concatenate([xk.real.ravel(), xk.imag.ravel()]))
            assert np.all((xv[np.isfinite(xv)] >= 2.0 ** -126) | (xv[np.isfinite(xv)] == 0))
            ys, _ = model(shim, H, xk, P, nb, xrow0)
            assert np.array_equal(ys, y * 2.0 ** k)                             # exact in float64


def test_flop_model_matches_the_f16_kernel(shim):
    """bench.py and tools/tc_sweep_bench.py count (Q/32 + 2) K chunks x 24 MMAs of 2*128*64*8 flop per tile; the FP16
    kernel executes nchunk_f16 = Q/64 + 1 chunks x 12 m64n128k16 MMAs (4 k-steps: hi*hi, lo*hi against the hi image,
    hi*lo against the lo image) x 2 warpgroups.  The two counts are the same arithmetic."""
    for P, nb, Cc, B in [(938, 112608, 2, 512), (938, 14077, 2, 512), (100, 4608, 2, 64), (961, 8192, 4, 256), (1, 4096, 1, 32)]:
        g = geom(shim, P, nb)
        q = (max(P - 1, 0) + 63) // 64 * 64
        ntile = -(-(-(-nb // 64)) // 64)
        assert (q, ntile) == (g["Q"], g["ntile"])
        bench_flop = Cc * B * ntile * (q // 32 + 2) * 24 * 2.0 * 128 * 64 * 8
        kernel_flop = Cc * B * g["ntile"] * g["nchunk"] * (4 * 3) * 2 * (2.0 * 64 * 128 * 16)
        assert bench_flop == kernel_flop
