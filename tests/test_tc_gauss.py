"""The three-product (Gauss) form of the tensor-core sweep (reevr_b200/csrc/kernels_tc.cuh, k_tc_sweep) on the CPU:
shared-memory budget, the 192-row image and its slices, the pair walk, the executed flop count, and a float64 model of
the whole arithmetic — k_tc_build_a (2^eh Hr, 2^eh Hi, 2^eh' (Hr + Hi) split into FP16 hi / lo), the strips of the re,
im and re + im time lines (2^ex per tile and line), the products hi*hi + hi*lo + lo*hi, the per-product 2^-(ex + eh)
descale and y = (D1 - D2, D3 - (D1 + D2)) — against a direct complex convolution, within the bound DESIGN.md section 5
states.  The header's inline functions are compiled by g++ through tests/cpp/tc_gauss_shim.cpp; the kernel itself is
covered on the GPU (tests/test_tc_sweep.py, tests/test_tc_pairs.py, tests/test_tc_f16_range.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.test_tc_f16_layout import direct, f16_split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("tcg") / "libtc_gauss.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", cuda_inc, os.path.join(ROOT, "tests", "cpp", "tc_gauss_shim.cpp"), "-o", so]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lib = C.CDLL(so)
    lib.tcg_a_image_bytes.restype = C.c_ulonglong
    lib.tcg_a_image_bytes.argtypes = [C.c_ulonglong, C.c_int]
    lib.tcg_sw128_h.restype = C.c_uint
    lib.tcg_sw128_h.argtypes = [C.c_uint, C.c_uint]
    lib.tcg_xf_index.restype = C.c_ulonglong
    lib.tcg_xf_index.argtypes = [C.c_longlong, C.c_int, C.c_longlong, C.c_int]
    lib.tcg_scale_exp.restype = C.c_int
    lib.tcg_scale_exp.argtypes = [C.c_uint]
    return lib


def consts(lib):
    out = (C.c_int * 10)()
    lib.tcg_consts(out)
    return dict(zip(("rows", "slice", "image", "stages", "wg_strips", "smem", "strip", "products", "flush", "strip_rows"), out))


def geom(lib, P, nb):
    out = (C.c_int * 5)()
    lib.tcg_geom(P, nb, out)
    return dict(zip(("Q", "nchunk", "ntile", "rows", "npair"), out))


def scale_exp(lib, values):
    v = np.asarray(values, np.float32)
    m = int(np.max(np.abs(v).view(np.uint32))) if v.size else 0
    return lib.tcg_scale_exp(m)


def test_shared_memory_and_image_layout(shim):
    k = consts(shim)
    assert (k["rows"], k["slice"], k["image"], k["products"]) == (192, 8192, 192 * 128, 3)
    assert k["wg_strips"] == 3 * 2 * k["strip"]                        # re, im, re + im x hi, lo
    assert k["smem"] == 2 * k["wg_strips"] + k["stages"] * k["image"] + 1024
    assert k["smem"] + 1024 <= 227 * 1024                              # + the static barriers and per-warp maxima
    # every wgmma operand base sits on a 1024-byte swizzle atom: strips, ring stages and the image slices inside them
    for off in [i * k["strip"] for i in range(12)] + [2 * k["wg_strips"] + s * k["image"] + p * k["slice"]
                                                       for s in range(k["stages"]) for p in range(3)]:
        assert off % 1024 == 0
    assert k["slice"] * 3 == k["image"]
    assert k["flush"] == 2                                             # chains of two chunks (TC_BIAS)
    g = geom(shim, 938, 112608)                                        # the metric shape
    assert (g["nchunk"], g["ntile"], g["npair"]) == (16, 28, 14)
    assert shim.tcg_a_image_bytes(1, g["nchunk"]) == 768 * 1024
    assert shim.tcg_a_image_bytes(1024, g["nchunk"]) + 1024 * 2 * 4 <= 806 * 1024 * 1024


def test_swizzle_covers_the_192_row_image(shim):
    offs = {shim.tcg_sw128_h(r, e) for r in range(192) for e in range(0, 64, 8)}
    assert offs == set(range(0, 192 * 128, 16))                        # every 16-byte unit exactly once
    for r in (0, 63, 64, 127, 128, 191):                              # slice p reads rows 64 p ... with its own row phase
        assert sorted(shim.tcg_sw128_h(r, e) for e in range(64)) == [r * 128 + 2 * i for i in range(64)]


@pytest.mark.parametrize("P,nb", [(1, 1), (100, 4096), (100, 4097), (938, 112608), (961, 3 * 4096 + 5), (65, 4 * 4096)])
def test_pair_walk_covers_every_tile_and_stays_in_the_time_lines(shim, P, nb):
    g = geom(shim, P, nb)
    assert g["npair"] == (g["ntile"] + 1) // 2
    tiles = []
    for m in range(g["npair"]):
        rows = shim.tcg_pair_rows(g["ntile"], m)
        own = [nt for nt in (2 * m, 2 * m + 1) if nt < g["ntile"]]
        tiles += own
        assert rows == 64 * (len(own) - 1) + 80                        # the rows the pair's strips read, prefetched to L2
        assert 2 * m * 64 + rows <= g["rows"]
    assert tiles == list(range(g["ntile"]))


def test_executed_flops_are_three_quarters_of_the_four_product_count(shim):
    """bench.py counts (Q/32 + 2) x 24 MMAs of 2*128*64*8 flop per tile (four real products).  The kernel executes, per
    K chunk and tile, 3 products x 4 k-steps x (hi*hi, lo*hi, hi*lo) m64n64k16 = 18 m64n128k16-equivalents."""
    for P, nb, Cc, B in [(938, 112608, 2, 512), (100, 4608, 2, 64), (961, 8192, 4, 256), (1, 4096, 1, 32)]:
        g = geom(shim, P, nb)
        four = Cc * B * g["ntile"] * (g["Q"] // 32 + 2) * 24 * 2.0 * 128 * 64 * 8
        executed = Cc * B * g["ntile"] * g["nchunk"] * 3 * 4 * 3 * (2.0 * 64 * 64 * 16)
        assert executed == 18 * Cc * B * g["ntile"] * g["nchunk"] * (2.0 * 64 * 128 * 16)
        assert executed * 4 == four * 3


def model(shim, H, x, P, nb, xrow0):
    """float64 model of build + strips + three products + descale + combine; returns y [lines][nb] and per line
    (eh, eh', [per tile (ex_re, ex_im, ex_sum)])."""
    g = geom(shim, P, nb)
    Q, rows, nchunk, ntile = g["Q"], g["rows"], g["nchunk"], g["ntile"]
    lines = H.shape[0]
    tau = np.arange(rows * 64)
    row = xrow0 - Q + tau
    inside = (row >= xrow0 - (P - 1)) & (row < xrow0 + nb)
    y = np.zeros((lines, nb), complex)
    exps = []
    i = np.arange(64)[:, None]
    jj = np.arange(64)[None, :]
    for line in range(lines):
        v = np.zeros(rows * 64, np.complex64)
        v[inside] = x[line, row[inside]]
        xl = [v.real.astype(np.float32), v.imag.astype(np.float32)]
        xl.append(xl[0] + xl[1])                                       # one FP32 add (round to nearest)
        hr, hi = H[line].real.astype(np.float32), H[line].imag.astype(np.float32)
        hs = hr + hi
        eh, ehs = scale_exp(shim, np.concatenate([hr, hi])), scale_exp(shim, hs)
        hp = [np.ldexp(hr, eh), np.ldexp(hi, eh), np.ldexp(hs, ehs)]
        ehp = [eh, eh, ehs]
        imgs = []
        for c in range(nchunk):
            pp = i + Q - (64 * c + jj)
            ok = (pp >= 0) & (pp < P)
            A = np.zeros((192, 64), np.float32)
            for part in range(3):
                A[part * 64:part * 64 + 64][ok] = hp[part][pp[ok]]
            imgs.append(f16_split(A))
        line_exps = []
        for nt in range(ntile):
            D = np.zeros((3, 64, 64))
            ex = []
            for p in range(3):
                strip = xl[p][nt * 4096:nt * 4096 + 80 * 64].reshape(80, 64)
                e = scale_exp(shim, strip)
                ex.append(e)
                s1, s2 = np.float32(2.0 ** (e // 2)), np.float32(2.0 ** (e - e // 2))
                xh, xlo = f16_split(strip * s1 * s2)
                for c in range(nchunk):
                    Ah, Al = imgs[c][0][64 * p:64 * p + 64], imgs[c][1][64 * p:64 * p + 64]
                    Bh, Bl = xh[c:c + 64], xlo[c:c + 64]
                    D[p] += Ah @ Bh.T + Ah @ Bl.T + Al @ Bh.T
                D[p] = np.ldexp(D[p], -(e + ehp[p]))
            line_exps.append(ex)
            for n in range(64):
                t0 = 64 * (nt * 64 + n)
                if t0 >= nb:
                    break
                cnt = min(64, nb - t0)
                d1, d2, d3 = D[0, :cnt, n], D[1, :cnt, n], D[2, :cnt, n]
                y[line, t0:t0 + cnt] = (d1 + 1j * d2) if line == 0 else (d1 - d2) + 1j * (d3 - (d1 + d2))
        exps.append((eh, ehs, line_exps))
    return y, exps


def bound(absref, sum_h, xsum, exps, nb):
    """DESIGN.md section 5, with |h| = max(|Hr|, |Hi|) and |x| = max(|xr|, |xi|) per term: y.re as the four-product
    form (two real products), y.im from three products whose sum operands are up to 2|h| and 2|x| plus the FP32
    rounding of both sums:  20 * 2^-22 |h||x| + 2^-23 (2^-ex |h| + 2^-eh |x|), ex / eh the smallest of the tile's."""
    b_re, b_im = np.zeros_like(absref), np.zeros_like(absref)
    for line, (eh, ehs, line_exps) in enumerate(exps):
        for t in range(nb):
            ex = min(line_exps[t // 4096])
            e_h = min(eh, ehs)
            sub = 2.0 ** -ex * sum_h[line] + 2.0 ** -e_h * xsum[line, t]
            b_re[line, t] = 6 * 2.0 ** -22 * absref[line, t] + 2.0 ** -24 * sub
            b_im[line, t] = 20 * 2.0 ** -22 * absref[line, t] + 2.0 ** -23 * sub
    return b_re, b_im


def run_case(shim, H, x, P, nb, xrow0):
    y, exps = model(shim, H, x, P, nb, xrow0)
    assert np.isfinite(y).all()
    ref, absref, sum_h = direct(H, x, P, nb, xrow0)
    lines = H.shape[0]
    xsum = np.zeros((lines, nb))
    for line in range(lines):
        xa = np.maximum(abs(x[line].real), abs(x[line].imag)).astype(np.float64)
        xsum[line] = [np.sum(xa[xrow0 + t - np.arange(P)]) for t in range(nb)]
    b_re, b_im = bound(absref, sum_h, xsum, exps, nb)
    assert (abs(y.real - ref.real) <= b_re * (1 + 1e-9) + 1e-300).all(), float(np.max(abs(y.real - ref.real) / b_re))
    assert (abs(y.imag - ref.imag) <= b_im * (1 + 1e-9) + 1e-300).all(), float(np.max(abs(y.imag - ref.imag) / b_im))
    return y, ref, absref


@pytest.mark.parametrize("P,nb,quiet_db,cancel", [(100, 300, 0, False), (938, 200, 0, False), (1, 70, 0, False), (65, 4100, 0, False),
                                                   (100, 300, 120, False), (65, 4100, 80, False), (100, 300, 0, True), (65, 4100, 0, True)])
def test_float64_model_of_the_three_product_sweep(shim, P, nb, quiet_db, cancel):
    rng = np.random.default_rng(P * 1000 + nb + quiet_db + 7 * cancel)
    Q = geom(shim, P, nb)["Q"]
    lines = 3                                                          # line 0 is the packed DC / Nyquist entry
    H = (rng.standard_normal((lines, P)) + 1j * rng.standard_normal((lines, P))) * np.exp(-np.arange(P) / 40.0)
    xrow0 = Q + 2
    x = rng.standard_normal((lines, xrow0 + nb)) + 1j * rng.standard_normal((lines, xrow0 + nb))
    if cancel:                                                         # Hr ~ -Hi and xr ~ -xi: the sum operands nearly cancel
        H = H.real - 1j * H.real * (1 + 1e-3 * rng.standard_normal(H.shape))
        x = x.real - 1j * (x.real + 1e-4 * rng.standard_normal(x.shape))
    H = H.astype(np.complex64)
    x = x.astype(np.complex64)
    if quiet_db:
        x[:, xrow0 + nb // 2:] *= np.float32(10.0 ** (-quiet_db / 20))
    x[:, :xrow0 - (P - 1)] = np.nan                                    # rows no sweep reads: must not leak in
    y, ref, absref = run_case(shim, H, x, P, nb, xrow0)
    if quiet_db and quiet_db <= 100:                                   # full relative precision within ~100 dB
        t = np.arange(nb // 2 + P, nb)
        err = np.maximum(abs(y.real - ref.real), abs(y.imag - ref.imag))
        assert np.max(err[:, t] / absref[:, t]) <= 2.0 ** -17
    if not quiet_db:                                                   # exact power-of-two invariance
        for k in (100, -100):
            xk = (x * np.float32(2.0 ** k)).astype(np.complex64)
            ys, _ = model(shim, H, xk, P, nb, xrow0)
            assert np.array_equal(ys, y * 2.0 ** k)
