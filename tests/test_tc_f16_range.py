"""Range and edge cases of the FP16 tensor-core sweep (cmac_variant 40, reevr_b200/csrc/kernels_tc.cuh) on the GPU,
forced and chosen automatically (launch groups >= 4096 blocks), against the float64 convolution of
tests/test_conv_precision.py: level steps inside one tile window of 4096 blocks (the quiet part shares the window's
power-of-two scale with the loud part), an IR whose per-bin range exceeds 100 dB, exact power-of-two scale
invariance, silence, a NaN sample confined to the tile windows that contain it, and the tile-count / channel /
partition-count geometries against the FFMA sweep (variant 22) and the float64 truth."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests.backends import get_lib
from tests.test_conv_precision import FLOOR, K_FORM, Form, _variant_is, run_engine, run_oracle, truth

pytestmark = pytest.mark.gpu

TILE = 64 * 64                          # output blocks per tile window


def tc_form(B, P, C, groups, variant, name="k2x"):
    return Form(f"{name}-B{B}-P{P}-C{C}-v{variant}", "k2x", B, P, C=C, groups=groups, batch=sum(groups) + 8, variant=variant,
                expect=_variant_is(40))


def errors(form, lib, xs, irs, segs):
    """engine outputs and, per channel and segment, (e64(oracle), e64(engine), peak64)"""
    ys, calls, stages, ir_lens = run_engine(form, lib, xs, irs)
    form.check_selection(calls, stages)
    yo = run_oracle(form, xs, irs)
    rows = []
    for c in range(form.C):
        r = truth(xs[c], irs[c][:ir_lens[c]])
        for lo, hi in segs:
            t = r[lo:hi]
            pk = float(np.max(np.abs(t)))
            rows.append((float(np.max(np.abs(yo[c][lo:hi] - t))) / pk, float(np.max(np.abs(ys[c][lo:hi] - t))) / pk, pk))
    return ys, rows


@pytest.mark.parametrize("variant", [40, 0])
@pytest.mark.parametrize("db", [60, 80, 100, 120, 140])
def test_level_step_inside_one_tile_window(variant, db):
    """loud noise for 512 blocks, then the same noise db lower with no gap: the quiet outputs of tile 0 (after the loud
    rows have left the IR) are computed with the loud part's scale.  Within ~100 dB of the window peak they keep full
    precision; beyond, the error is absolute, at most ~2^-39 of the window peak per product (DESIGN.md section 5),
    which the output shows far below 2^-30 of the loud peak."""
    lib = get_lib("cuda")
    B, P = 32, 100
    f = tc_form(B, P, 1, [TILE], variant)
    n = TILE * B
    a = 512 * B
    x = orc.synth_input(n, 0)
    x[a:] *= np.float32(10.0 ** (-db / 20))
    h = orc.synth_ir(f.ir_len, 0)
    q0 = a + f.ir_len + 2 * B
    _, rows = errors(f, lib, [x], [h], [(0, a), (q0, n)])
    (_, _, pk_loud), (e_o, e_e, pk_q) = rows
    if db <= 100:
        assert e_e <= max(K_FORM["k2x"] * e_o, FLOOR), (db, e_o, e_e)
    else:
        assert e_e * pk_q <= max(K_FORM["k2x"] * e_o * pk_q, 2.0 ** -30 * pk_loud), (db, e_o, e_e, e_e * pk_q / pk_loud)


@pytest.mark.parametrize("variant", [40, 0])
def test_ir_with_more_than_100_db_per_bin(variant):
    """partition-probe deltas of amplitudes 1, 2^-7, 2^-14 and 2^-20: every bin holds a 120 dB range of H, all of it
    under one exponent eh"""
    lib = get_lib("cuda")
    B, P = 32, 300
    f = tc_form(B, P, 2, [TILE, TILE + 1], variant)
    n = f.round_n(0)
    irs = []
    for c in range(2):
        h = np.zeros(f.ir_len, np.float32)
        for i, t in enumerate([0, B - 1, B, 77 * B + 5, 150 * B, 220 * B + 31, f.ir_len - 1]):
            h[t] = 2.0 ** -[0, 7, 14, 20][(i + c) % 4]
        irs.append(h)
    xs = [orc.synth_input(n, c) for c in range(2)]
    _, rows = errors(f, lib, xs, irs, [(0, n)])
    for e_o, e_e, _ in rows:
        assert e_e <= max(K_FORM["k2x"] * e_o, FLOOR), (e_o, e_e)


def test_power_of_two_scale_invariance():
    lib = get_lib("cuda")
    B, P = 64, 200
    f = tc_form(B, P, 2, [TILE + 1], 40)
    n = f.round_n(0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(2)]
    xs = [orc.synth_input(n, c) for c in range(2)]
    y0 = run_engine(f, lib, xs, irs)[0]
    for k in (100, -100):
        yk = run_engine(f, lib, [np.ldexp(x, k).astype(np.float32) for x in xs], irs)[0]
        for c in range(2):
            back = np.ldexp(yk[c].astype(np.float64), -k)
            if k > 0:
                assert np.array_equal(back, y0[c].astype(np.float64))
            else:          # x * 2^-100 puts a few FFT intermediates near zero crossings into FP32's subnormal range
                assert np.max(np.abs(back - y0[c])) <= 2.0 ** -60 * np.max(np.abs(y0[c]))


@pytest.mark.parametrize("variant", [40, 0])
def test_silence_gives_exact_zeros(variant):
    lib = get_lib("cuda")
    f = tc_form(32, 961, 2, [TILE, TILE + 1], variant)
    n = f.round_n(0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(2)]
    ys = run_engine(f, lib, [np.zeros(n, np.float32) for _ in range(2)], irs)[0]
    for y in ys:
        assert not np.any(y)


def test_nan_sample_stays_in_its_tile_windows():
    """A NaN in block 1000 makes the outputs that depend on it non-finite.  Tile 0's window (4096 output blocks plus
    Q blocks of history, 5120 time-line rows) is left unscaled; inside it the NaN reaches every 64-block segment whose
    K window holds it (the Toeplitz image's structural zeros multiply it too).  Tile 1's window starts at block
    4096 - Q and does not reach block 1001, so its partial products are those of the clean run; output block 4096 still
    takes the overlap-add tail of block 4095 (tile 0), and every output from block 4097 on is bit-equal."""
    lib = get_lib("cuda")
    B, P = 32, 100
    f = tc_form(B, P, 1, [2 * TILE], 40)
    n = f.round_n(0)
    h = orc.synth_ir(f.ir_len, 0)
    x = orc.synth_input(n, 0)
    clean = run_engine(f, lib, [x], [h])[0][0]
    xn = x.copy()
    b = 1000
    xn[b * B + 7] = np.nan
    dirty = run_engine(f, lib, [xn], [h])[0][0]
    assert np.all(np.isfinite(clean))
    assert not np.any(np.isfinite(dirty[(b + 1) * B:(b + P - 1) * B]))
    assert np.all(np.isfinite(dirty[(TILE + 1) * B:]))
    assert np.array_equal(dirty[(TILE + 1) * B:], clean[(TILE + 1) * B:])


@pytest.mark.parametrize("B,P,C,groups", [(32, 961, 1, [4096, 4097, 8193]), (512, 1, 4, [4096, 8193]), (32, 1, 4, [4097, 8193]),
                                          (512, 938, 1, [4097])])
def test_geometries_against_float64_and_the_ffma_sweep(B, P, C, groups):
    lib = get_lib("cuda")
    f = tc_form(B, P, C, groups, 40)
    n = f.round_n(0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(C)]
    xs = [orc.synth_input(n, c) for c in range(C)]
    ys, rows = errors(f, lib, xs, irs, [(0, n)])
    for e_o, e_e, _ in rows:
        assert e_e <= max(K_FORM["k2x"] * e_o, FLOOR), (e_o, e_e)
    ffma = Form("k2", "k2", B, P, C=C, groups=groups, batch=sum(groups) + 8, variant=22, expect=_variant_is(22))
    y22 = run_engine(ffma, lib, xs, irs)[0]
    for c in range(C):
        assert np.max(np.abs(ys[c].astype(np.float64) - y22[c])) <= 4e-6 * np.max(np.abs(y22[c]))
