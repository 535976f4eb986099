"""The four-step sweep (cmac_variant 42, reevr_b200/csrc/kernels_fourstep.cuh) on the GPU, forced and chosen
automatically (B = 512 groups of >= 32768 whole blocks, P <= 961): geometries against the float64 convolution, the
oracle and the FFMA sweep (variant 22); call sequences that mix four-step groups with real-time calls, FFMA and
line-FFT groups (the history, X-row and overlap-row hand-off); silence, NaN locality per segment, an IR re-init between
groups and the selection threshold."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests.backends import get_lib
from tests.test_conv_precision import Form, _variant_is, run_engine
from tests.test_lfft_sweep import TOL, TOL_FFMA, check_against_oracle_and_ffma, check_direct
from tests.test_tc_direct import on_device, peak_err

pytestmark = pytest.mark.gpu

B = 512
M = 1 << 21
FS_MIN = 32768              # shortest launch group that selects variant 42 by itself


def seg_len(P):
    return M - (P * B - 1)


def three_segments_and_a_block(P):
    return -(-3 * seg_len(P) // B) + 1


def fs_form(P, C, groups, variant):
    return Form(f"k2s-P{P}-C{C}-v{variant}", "k2x", B, P, C=C, groups=groups, batch=max(groups) + 8, variant=variant,
                expect=_variant_is(42))


@pytest.mark.parametrize("P,C,groups,variant", [
    (938, 1, [FS_MIN], 0), (961, 2, [FS_MIN + 4095], 0), (1, 2, [three_segments_and_a_block(1)], 42),
    (20, 2, [FS_MIN, three_segments_and_a_block(20)], 42), (938, 1, [three_segments_and_a_block(938)], 42)])
def test_geometries_against_float64_the_oracle_and_the_ffma_sweep(P, C, groups, variant):
    lib = get_lib("cuda")
    f = fs_form(P, C, groups, variant)
    n = f.round_n(0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(C)]
    xs = [orc.synth_input(n, c) for c in range(C)]
    ys, calls, stages, _ = run_engine(f, lib, xs, irs)
    f.check_selection(calls, stages)
    check_against_oracle_and_ffma(f, lib, xs, irs, ys)


def run_calls(C, irs, xs, calls, batch):
    """calls: (samples, tc, expected variant or None); device-resident calls for groups of >= 4096 blocks"""
    e = Engine(C, max_batch_blocks=batch, lib=get_lib("cuda"))
    assert e.init_uniform(B, irs)
    outs, pos = [[] for _ in range(C)], 0
    for k, tc, variant in calls:
        e.set_option("tc", tc)
        seg = [np.ascontiguousarray(x[pos:pos + k]) for x in xs]
        ys = on_device(e, seg) if k >= 4096 * B else e.process(seg)
        if variant is not None:
            assert e.last_sweep_variant() == variant, (k, e.last_sweep_variant())
        for c in range(C):
            outs[c].append(ys[c])
        pos += k
    e.close()
    return [np.concatenate(o) for o in outs]


def test_four_step_groups_between_real_time_ffma_and_line_fft_calls():
    C, P = 2, 938
    irs = [orc.synth_ir(P * B - 3, c) for c in range(C)]
    calls = ([(B, 1, None), (FS_MIN * B, 1, 42)] + [(B, 1, None)] * 5 +
             [(4100 * B, 0, 22), ((FS_MIN + 9) * B, 1, 42), (20000 * B, 1, 41), (FS_MIN * B, 1, 42)])
    xs = [orc.synth_input(sum(k for k, _, _ in calls), c) for c in range(C)]
    got = run_calls(C, irs, xs, calls, FS_MIN + 16)
    ffma = run_calls(C, irs, xs, [(k, 0, None) for k, _, _ in calls], FS_MIN + 16)
    check_direct(irs, xs, got, ffma)


def test_silence_gives_exact_zeros():
    lib = get_lib("cuda")
    f = fs_form(938, 2, [FS_MIN], 0)
    irs = [orc.synth_ir(f.ir_len, c) for c in range(2)]
    ys, calls, stages, _ = run_engine(f, lib, [np.zeros(f.round_n(0), np.float32) for _ in range(2)], irs)
    f.check_selection(calls, stages)
    for y in ys:
        assert not np.any(y)


def test_nan_sample_stays_in_its_segments():
    """A NaN at sample 1000 B + 7 is inside segment 0's window only (segment 1's starts at L - (Lh - 1)): segment 0's
    outputs are not finite, every later output is bit-equal to the clean run's."""
    lib = get_lib("cuda")
    P = 938
    L = seg_len(P)
    f = fs_form(P, 1, [FS_MIN], 0)
    h = orc.synth_ir(f.ir_len, 0)
    x = orc.synth_input(f.round_n(0), 0)
    clean = run_engine(f, lib, [x], [h])[0][0]
    xn = x.copy()
    xn[1000 * B + 7] = np.nan
    dirty = run_engine(f, lib, [xn], [h])[0][0]
    assert np.all(np.isfinite(clean))
    assert not np.any(np.isfinite(dirty[1000 * B + 7:L]))
    assert np.array_equal(dirty[L:], clean[L:])


def test_ir_reinit_between_groups_rebuilds_the_spectrum():
    lib = get_lib("cuda")
    P, C = 300, 2
    n = FS_MIN * B
    irs1 = [orc.synth_ir(P * B - 3, c) for c in range(C)]
    irs2 = [orc.synth_ir(P * B - 3, c + 5) for c in range(C)]
    x1 = [orc.synth_input(n, c) for c in range(C)]
    x2 = [orc.synth_input(n, c + 3) for c in range(C)]
    e = Engine(C, max_batch_blocks=FS_MIN + 8, lib=lib)
    assert e.init_uniform(B, irs1)
    on_device(e, x1)
    assert e.last_sweep_variant() == 42
    assert e.init_uniform(B, irs2)
    got = on_device(e, x2)
    assert e.last_sweep_variant() == 42
    e.close()
    fresh = Engine(C, max_batch_blocks=FS_MIN + 8, lib=lib)
    assert fresh.init_uniform(B, irs2)
    fresh.set_option("tc", 0)
    want = on_device(fresh, x2)
    fresh.close()
    for c in range(C):
        assert peak_err(got[c], want[c]) <= TOL_FFMA


def test_selection_threshold_and_forced_shapes():
    lib = get_lib("cuda")
    P = 100
    irs = [orc.synth_ir(P * B - 3, 0)]
    x = [orc.synth_input(FS_MIN * B, 0)]
    for blocks, tc, want in ((FS_MIN - 1, 1, 41), (FS_MIN, 1, 42), (FS_MIN, 0, 22)):
        e = Engine(1, max_batch_blocks=FS_MIN + 8, lib=lib)
        assert e.init_uniform(B, irs)
        e.set_option("tc", tc)
        on_device(e, [x[0][:blocks * B]])
        assert e.last_sweep_variant() == want, (blocks, tc)
        e.close()
    # forced on a group that does not start on a block boundary: refused
    e = Engine(1, max_batch_blocks=FS_MIN + 8, cmac_variant=42, lib=lib)
    assert e.init_uniform(B, irs)
    with pytest.raises(Exception):
        e.process([x[0][:100]])
        on_device(e, [x[0][100:100 + 8 * B]])
    e.close()
