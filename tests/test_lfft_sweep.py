"""The line-FFT sweep (cmac_variant 41, reevr_b200/csrc/kernels_lfft.cuh) on the GPU, forced and chosen automatically
(launch groups >= 16384 blocks, P <= 961): geometries against the float64 convolution and the FFMA sweep (variant
22), the selection threshold, the B = 512 direct-form schedules (ragged groups behind an open block, a time-slice rank
whose sweep starts one block early, real-time calls and an FFMA group after a line-FFT group), the DC / Nyquist entry,
silence, NaN locality per overlap-save segment and an IR re-init between groups.

The CPU oracle takes about a second per thousand blocks and channel, so it is run on the first ORACLE_BLOCKS blocks of
each channel (a whole segment and the start of the next); the FFMA sweep is compared over the whole output."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests.backends import get_lib
from tests.test_conv_precision import FLOOR, K_FORM, Form, _variant_is, run_engine, truth
from tests.test_tc_direct import on_device, peak_err

pytestmark = pytest.mark.gpu

KN = 4096                   # transform size of the line FFTs
LFFT_MIN = 16384            # shortest launch group that selects variant 41 by itself
ORACLE_BLOCKS = 4500
TOL = 1e-5                  # against the oracle (parity)
TOL_FFMA = 4e-6             # against the FFMA sweep
# The FFT form's error is relative to the line's energy, about log2 kN roundings per transform and two transforms
# (DESIGN.md section 5).  It only shows above K_FORM x the oracle's error where the oracle's own is one rounding per
# output: P = 1.
LFFT_FLOOR = 2 * 12 * 2.0 ** -24


def lfft_form(B, P, C, groups, variant):
    return Form(f"k2f-B{B}-P{P}-C{C}-v{variant}", "k2x", B, P, C=C, groups=groups, batch=max(groups) + 8, variant=variant,
                expect=_variant_is(41))


def oracle_prefix(B, h, x, blocks):
    o = orc.OracleUniform()
    assert o.init(B, h)
    return o.process(np.ascontiguousarray(x[:blocks * B]))


def check_against_oracle_and_ffma(f, lib, xs, irs, ys):
    m = min(ORACLE_BLOCKS, f.round_n(0) // f.B) * f.B
    for c in range(f.C):
        r = truth(xs[c][:m], irs[c])
        pk = float(np.max(np.abs(r)))
        e_o = float(np.max(np.abs(oracle_prefix(f.B, irs[c], xs[c], m // f.B) - r))) / pk
        e_e = float(np.max(np.abs(ys[c][:m] - r))) / pk
        assert e_e <= max(K_FORM["k2x"] * e_o, FLOOR if f.P > 1 else LFFT_FLOOR), (c, e_o, e_e)
    ffma = Form("k2", "k2", f.B, f.P, C=f.C, groups=f.groups, batch=f.batch, variant=22, expect=_variant_is(22))
    y22 = run_engine(ffma, lib, xs, irs)[0]
    for c in range(f.C):
        assert np.isfinite(ys[c]).all()
        assert np.max(np.abs(ys[c].astype(np.float64) - y22[c])) <= TOL_FFMA * np.max(np.abs(y22[c])), c


@pytest.mark.parametrize("B,P,C,groups,variant", [
    (512, 938, 1, [LFFT_MIN, LFFT_MIN + 1], 0), (512, 938, 2, [LFFT_MIN + 1, 3 * KN + 7], 41),
    (512, 961, 1, [3 * KN + 7, LFFT_MIN], 41), (512, 961, 2, [LFFT_MIN], 0),
    (32, 961, 4, [LFFT_MIN, LFFT_MIN + 1], 0), (512, 1, 2, [LFFT_MIN], 0), (32, 1, 1, [3 * KN + 7], 41)])
def test_geometries_against_float64_and_the_ffma_sweep(B, P, C, groups, variant):
    lib = get_lib("cuda")
    f = lfft_form(B, P, C, groups, variant)
    n = f.round_n(0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(C)]
    xs = [orc.synth_input(n, c) for c in range(C)]
    ys, calls, stages, _ = run_engine(f, lib, xs, irs)
    f.check_selection(calls, stages)
    check_against_oracle_and_ffma(f, lib, xs, irs, ys)


def test_selection_threshold():
    lib = get_lib("cuda")
    B, P = 32, 100
    irs = [orc.synth_ir(P * B - 3, 0)]
    for groups, tc, want in (([LFFT_MIN - 1], 1, 40), ([LFFT_MIN], 1, 41), ([LFFT_MIN], 0, 22)):
        f = Form("sel", "k2x", B, P, groups=groups, batch=LFFT_MIN + 8, options={"tc": tc}, expect=_variant_is(want))
        xs = [orc.synth_input(f.round_n(0), 0)]
        _, calls, stages, _ = run_engine(f, lib, xs, irs)
        f.check_selection(calls, stages)


def test_dc_and_nyquist_on_entry_zero():
    """DC plus an alternating +-1 input lives in entry 0 alone (DC in its real part, Nyquist in its imaginary part)"""
    lib = get_lib("cuda")
    B, P, C = 32, 100, 2
    f = lfft_form(B, P, C, [LFFT_MIN], 0)
    t = np.arange(f.round_n(0))
    xs = [(0.5 + (0.25 + 0.1 * c) * (1 - 2 * (t % 2))).astype(np.float32) for c in range(C)]
    irs = [orc.synth_ir(f.ir_len, c) for c in range(C)]
    ys, calls, stages, _ = run_engine(f, lib, xs, irs)
    f.check_selection(calls, stages)
    check_against_oracle_and_ffma(f, lib, xs, irs, ys)


def test_silence_gives_exact_zeros():
    lib = get_lib("cuda")
    f = lfft_form(32, 961, 2, [LFFT_MIN, LFFT_MIN + 1], 0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(2)]
    ys, calls, stages, _ = run_engine(f, lib, [np.zeros(f.round_n(0), np.float32) for _ in range(2)], irs)
    f.check_selection(calls, stages)
    for y in ys:
        assert not np.any(y)


def test_nan_sample_stays_in_its_segments():
    """A NaN in block 1000 sits at tau = Q + 1000 of the time line, inside segment 0's window only (segment 1's starts
    at tau = L + Q - (P - 1)).  Segment 0's outputs (sweep outputs 0 ... L - 1) are non-finite, the ones that depend on
    the sample included; from output block L + 1 on (block L takes the overlap-add tail of block L - 1) every sample is
    bit-equal to the clean run's."""
    lib = get_lib("cuda")
    B, P = 32, 100
    L = KN - (P - 1)
    f = lfft_form(B, P, 1, [LFFT_MIN], 0)
    h = orc.synth_ir(f.ir_len, 0)
    x = orc.synth_input(f.round_n(0), 0)
    clean = run_engine(f, lib, [x], [h])[0][0]
    xn = x.copy()
    b = 1000
    xn[b * B + 7] = np.nan
    dirty = run_engine(f, lib, [xn], [h])[0][0]
    assert np.all(np.isfinite(clean))
    assert not np.any(np.isfinite(dirty[(b + 1) * B:(b + P - 1) * B]))
    assert np.array_equal(dirty[(L + 1) * B:], clean[(L + 1) * B:])


def test_ir_reinit_between_groups_rebuilds_the_spectra():
    lib = get_lib("cuda")
    B, P, C = 32, 300, 2
    n = LFFT_MIN * B
    irs1 = [orc.synth_ir(P * B - 3, c) for c in range(C)]
    irs2 = [orc.synth_ir(P * B - 3, c + 5) for c in range(C)]
    x1 = [orc.synth_input(n, c) for c in range(C)]
    x2 = [orc.synth_input(n, c + 3) for c in range(C)]
    e = Engine(C, max_batch_blocks=LFFT_MIN + 8, lib=lib)
    assert e.init_uniform(B, irs1)
    on_device(e, x1)
    assert e.last_sweep_variant() == 41
    assert e.init_uniform(B, irs2)
    got = on_device(e, x2)
    assert e.last_sweep_variant() == 41
    e.close()
    fresh = Engine(C, max_batch_blocks=LFFT_MIN + 8, lib=lib)
    assert fresh.init_uniform(B, irs2)
    want = on_device(fresh, x2)
    fresh.close()
    for c in range(C):
        assert np.array_equal(got[c], want[c])
        r = truth(x2[c], irs2[c])
        assert peak_err(got[c], r) <= TOL


# ---- B = 512 direct form: the forward FFT writes the time lines, the inverse reads the result lines ----------------
B512 = 512


def run_schedule(C, irs, xs, calls, batch, tc):
    """calls: samples per call; device-resident calls for groups of >= 4096 blocks, host calls otherwise"""
    e = Engine(C, max_batch_blocks=batch, lib=get_lib("cuda"))
    assert e.init_uniform(B512, irs)
    e.set_option("tc", tc)
    outs, variants, pos = [[] for _ in range(C)], [], 0
    for k in calls:
        seg = [np.ascontiguousarray(x[pos:pos + k]) for x in xs]
        ys = on_device(e, seg) if k >= 4096 * B512 else e.process(seg)
        variants.append(e.last_sweep_variant())
        for c in range(C):
            outs[c].append(ys[c])
        pos += k
    e.close()
    return [np.concatenate(o) for o in outs], variants


def check_direct(irs, xs, got, ffma):
    for c in range(len(xs)):
        assert np.isfinite(got[c]).all()
        assert peak_err(got[c], ffma[c]) <= TOL_FFMA
        m = ORACLE_BLOCKS * B512
        assert peak_err(got[c][:m], oracle_prefix(B512, irs[c], xs[c], ORACLE_BLOCKS)) <= TOL


@pytest.mark.parametrize("P", [938, 961])
def test_ragged_groups_behind_an_open_block(P):
    C = 1
    irs = [orc.synth_ir(P * B512 - 7, c) for c in range(C)]
    calls = [3 * B512 + 100, 16387 * B512 + 300, 16390 * B512 + 13 * B512 - 5]
    xs = [orc.synth_input(sum(calls), c) for c in range(C)]
    got, variants = run_schedule(C, irs, xs, calls, 16420, 1)
    assert variants[1:] == [41, 41], variants
    ffma, _ = run_schedule(C, irs, xs, calls, 16420, 0)
    check_direct(irs, xs, got, ffma)


def test_line_fft_group_then_real_time_calls_then_ffma_group():
    C, P = 2, 938
    irs = [orc.synth_ir(P * B512 - 3, c) for c in range(C)]
    calls = [(16390 * B512, 1, 41)] + [(B512, 1, None)] * 5 + [(200, 1, None), (B512 - 200, 1, None),
                                                                 (4100 * B512, 0, 22), (16385 * B512, 1, 41)]
    xs = [orc.synth_input(sum(k for k, _, _ in calls), c) for c in range(C)]
    e = Engine(C, max_batch_blocks=16400, lib=get_lib("cuda"))
    assert e.init_uniform(B512, irs)
    outs, pos = [[] for _ in range(C)], 0
    for k, tc, variant in calls:
        e.set_option("tc", tc)
        seg = [np.ascontiguousarray(x[pos:pos + k]) for x in xs]
        ys = on_device(e, seg) if k >= 4096 * B512 else e.process(seg)
        if variant is not None:
            assert e.last_sweep_variant() == variant
        for c in range(C):
            outs[c].append(ys[c])
        pos += k
    e.close()
    got = [np.concatenate(o) for o in outs]
    ffma, _ = run_schedule(C, irs, xs, [k for k, _, _ in calls], 16400, 0)
    check_direct(irs, xs, got, ffma)


def test_sliced_rank_with_an_early_block():
    # rank 1's slice starts behind a forward-FFT-only advance: its sweep starts one block early (extra = 1)
    G, T, C, P = 2, 2 * LFFT_MIN + 20, 1, 938
    irs = [orc.synth_ir(P * B512 - 5, c) for c in range(C)]
    xs = [orc.synth_input(T * B512, c) for c in range(C)]
    import torch
    x = torch.from_numpy(np.stack(xs)).cuda()
    y = torch.full_like(x, float("nan"))
    for g in range(G):
        e = Engine(C, max_batch_blocks=T // G + 1, lib=get_lib("cuda"))
        assert e.init_uniform(B512, irs)
        e.process_device_sliced(x.data_ptr(), T * B512, y.data_ptr(), T * B512, T * B512, g, G, sync=True)
        assert e.last_sweep_variant() == 41
        e.close()
    got = list(y.cpu().numpy())
    whole = Engine(C, max_batch_blocks=T + 1, lib=get_lib("cuda"))
    assert whole.init_uniform(B512, irs)
    whole.set_option("tc", 0)
    ref = on_device(whole, xs)
    whole.close()
    assert not np.isnan(got[0]).any()
    assert peak_err(got[0], ref[0]) <= TOL_FFMA
    # rank 1's first blocks, where the early block enters, against the oracle
    lo, hi = (T // G - 10) * B512, (T // G + ORACLE_BLOCKS // 4) * B512
    o = orc.OracleUniform()
    o.init(B512, irs[0])
    assert peak_err(got[0][lo:hi], o.process(xs[0][:hi])[lo:]) <= TOL
