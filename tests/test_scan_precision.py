"""The chunked scans of the recursive filters against serial float64 filters, over REEV-R's full parameter ranges.

The device runs every recursive filter as a chunked scan (irshape.cu k_scan2, kernels_chain.cuh k_chain_send): T chunks
run from a zero state, A^L from L zero-input steps, one thread scans S_{t+1} = A^L S_t + Z_t, the chunks re-run from
their true states.  With poles within ~1e-4 of the unit circle (20 Hz at 96 or 192 kHz, Q 8) an error in S_t persists
for tens of chunks, so these tests go where the mild cases of test_ir_recalc.py / test_chain.py do not: EQ bands
20 Hz - 20 kHz, Q 0.707 - 8, +-24 dB (src/Globals.h EQ_MAX_GAIN, src/PluginProcessor.cpp:86-105), cuts 20 Hz - 20 kHz
(:58-59), inverted cuts, 44.1 - 192 kHz, ragged and empty last chunks.

References: tests/cpp/scan_f64.c runs the exact recurrences serially in double from the oracle's float32 coefficients;
run in float it reproduces the oracle bit for bit (checked below), so its float run is the serial FP32 restatement.

Criterion, for every output, with e64(y) = max |y - float64 serial run| and peak64 = max |float64 serial run|:
    e64(device) <= max(TOL * peak64, FACTOR * e64(serial FP32 restatement))
and, where the restatement itself is accurate (e64(restatement) <= WELL * peak64), the project's bar against it:
    max |device - restatement| <= TOL * peak(restatement).
The first line stays meaningful where the output is nearly silent (inverted cuts): there the FP32 filter itself is far
from float64 and the device only has to be as good as it, within FACTOR.  FACTOR = 4: the chunk interiors run the
reference's FP32 recurrence, so a chunk's own rounding error is that of the serial FP32 filter; with the scan in
float64 the initial states it hands over are the float64 ones rounded to float, which adds one more rounding of the
state per chunk that then decays like the serial filter's own errors.  Measured over this file's cases, wherever the
1e-5 term does not cover it, the device's e64 is at most 1.7x the restatement's on the emulation build and 1.5x on the
H100 (-fmad=true); 4 leaves more than 2x of headroom over that and stays far below what the FP32 scan gave (up to 32x
the restatement's error, 5e-5 of peak for a 20 Hz, Q 8, +24 dB low shelf at 96 kHz).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import recalc as rc
from reevr_b200.convolver import Engine, ir_recalc
from reevr_b200.synth import synth_ir
from tests.backends import get_lib, lib  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5
FACTOR = 4.0
WELL = 1e-6
SCAN_T = 1024                       # chunks of k_scan2 (irshape.cu kScanThreads)
DB24_UP, DB24_DOWN = 15.85, 0.063   # +-24 dB (EQ_MAX_GAIN)

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")


@pytest.fixture(scope="module")
def f64(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("scan") / "libscan_f64.so")
    srcs = [os.path.join(ROOT, "tests", "cpp", "scan_f64.c"), os.path.join(ROOT, "oracle", "chain_oracle.c"),
            os.path.join(ROOT, "oracle", "partconv_oracle.c")]
    cmd = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", *srcs, "-o", so, "-lm"]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    h = C.CDLL(so)
    h.sf_svf_coeffs.restype = C.c_int
    h.sf_svf_coeffs.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, _f32p]
    h.sf_svf_run64.argtypes = [C.c_int, _f32p, _f64p, _f64p, C.c_size_t]
    h.sf_svf_run32.argtypes = [C.c_int, _f32p, _f32p, _f32p, C.c_size_t]
    h.sf_svf_oracle.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, _f32p, C.c_size_t]
    h.sf_filter_coeffs.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, _f32p]
    h.sf_filter_run64.argtypes = [C.c_int, C.c_int, _f32p, _f64p, _f64p, _f64p, C.c_size_t]
    h.sf_filter_run32.argtypes = [C.c_int, C.c_int, _f32p, _f32p, _f32p, _f32p, C.c_size_t]
    h.sf_filter_oracle.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, _f32p, _f32p, C.c_size_t]
    h.sf_rs_lowpass64.argtypes = [C.c_double, _f64p, _f64p, C.c_size_t, C.c_int]
    h.sf_rs_feedback_l1.restype = C.c_double
    h.sf_rs_feedback_l1.argtypes = [C.c_double, C.c_size_t]
    return h


def _check(got, r32, r64, what):
    """the criterion of the module docstring for one output"""
    got, r32, r64 = (np.asarray(a, np.float64) for a in (got, r32, r64))
    assert got.shape == r32.shape == r64.shape, what
    peak64 = float(np.max(np.abs(r64), initial=0.0))
    e_dev = float(np.max(np.abs(got - r64), initial=0.0))
    e_32 = float(np.max(np.abs(r32 - r64), initial=0.0))
    assert e_dev <= max(TOL * peak64, FACTOR * e_32), (what, e_dev / max(peak64, 1e-300), e_32 / max(peak64, 1e-300))
    if e_32 <= WELL * peak64:
        peak32 = float(np.max(np.abs(r32), initial=0.0))
        assert float(np.max(np.abs(got - r32), initial=0.0)) <= TOL * peak32, (what, "against the restatement")


# ---- the helper is the oracle's arithmetic -------------------------------------------------------------------------
def test_helper_reproduces_the_oracle_svf(f64):
    x = (synth_ir(20000, 0) + np.float32(0.3)).astype(np.float32)
    for mode in range(10):
        for freq, q, gain, sr in ((20.0, 8.0, DB24_UP, 96000.0), (20000.0, 0.707, DB24_DOWN, 44100.0),
                                  (1000.0, 2.0, 1.5, 48000.0), (90000.0, 0.707, DB24_UP, 192000.0)):
            c = np.empty(8, np.float32)
            m = f64.sf_svf_coeffs(mode, freq, q, gain, sr, c)
            want = x.copy()
            f64.sf_svf_oracle(mode, freq, q, gain, sr, want, want.size)
            got = np.empty_like(x)
            f64.sf_svf_run32(m, c, x, got, x.size)
            assert np.array_equal(got, want), (mode, freq, q, gain, sr)


def test_helper_reproduces_the_oracle_filter(f64):
    x = (orc.synth_input(20000, 0) + np.float32(0.4)).astype(np.float32)
    for slope in (0, 1, 2):
        for mode in (0, 1, 2):
            for freq, sr in ((20.0, 96000.0), (1000.0, 44100.0), (20000.0, 44100.0), (20000.0, 192000.0)):
                c = np.empty(9, np.float32)
                f64.sf_filter_coeffs(slope, mode, sr, freq, c)
                want = np.empty_like(x)
                f64.sf_filter_oracle(slope, mode, sr, freq, x, want, x.size)
                got = np.empty_like(x)
                f64.sf_filter_run32(slope, mode, c, np.zeros(5, np.float32), x, got, x.size)
                assert np.array_equal(got, want), (slope, mode, freq, sr)
                q = 0.0765 if slope == 2 else 0.2929
                assert np.array_equal(got, orc.OracleFilter(slope, mode, sr, freq, q).run(x))


# ---- parametric EQ: k_scan2<SvfRec> through b200conv_ir_recalc -----------------------------------------------------
def _svf_refs(f64, bands, srate, raws):
    """(FP32 serial restatement, float64 serial run) of the band cascade over every channel"""
    r32, r64 = [], []
    for x in raws:
        a, b = x.astype(np.float32), x.astype(np.float64)
        for mode, freq, q, gain in bands:
            c = np.empty(8, np.float32)
            m = f64.sf_svf_coeffs(mode, freq, q, gain, srate, c)
            a2, b2 = np.empty_like(a), np.empty_like(b)
            f64.sf_svf_run32(m, c, a, a2, a.size)
            f64.sf_svf_run64(m, c, b, b2, b.size)
            a, b = a2, b2
        r32.append(a)
        r64.append(b)
    return r32, r64


def _run_param_eq(l, f64, bands, srate, n, restated=True):
    raws = [synth_ir(n, c) for c in range(2)]
    kw = dict(ir_srate=srate, srate=srate, stretch=0.0, autogain=False, gain=1.0, clip=False, param_eq=bands)
    got = ir_recalc(raws, lib=l, **kw)
    r32, r64 = _svf_refs(f64, bands, srate, raws)
    if restated:                       # the helper's FP32 run is the restatement of the whole recalculation
        want = rc.ir_recalc(raws, **kw)
        assert all(np.array_equal(a, b) for a, b in zip(r32, want))
    for c in range(2):
        _check(got[c], r32[c], r64[c], (bands, srate, n, c))


def _gain_modes():
    """(mode, freq, q, gain) of single bands at the edges: every mode, 20 Hz and 20 kHz, Q 0.707 and 8, +-24 dB where the
    mode has a gain (LS, HS, PK, Off); HP6 / LP6 have no Q"""
    out = []
    for mode in range(10):
        for freq in (20.0, 20000.0):
            for q in ((0.707,) if mode in (7, 8) else (0.707, 8.0)):
                for gain in ((DB24_UP, DB24_DOWN) if mode in (3, 4, 5, 9) else (1.0,)):
                    out.append((mode, freq, q, gain))
    return out


BANDS = _gain_modes()
STACKS = {
    "issue4": ((7, 20.0, 0.707, 1.0), (5, 20.0, 8.0, DB24_UP), (5, 40.0, 8.0, DB24_UP), (8, 20000.0, 0.707, 1.0)),
    "lows_up": ((3, 20.0, 8.0, DB24_UP), (5, 25.0, 8.0, DB24_UP), (9, 31.5, 8.0, DB24_UP), (4, 20000.0, 8.0, DB24_UP)),
    "cuts_down": ((2, 20.0, 8.0, 1.0), (3, 20.0, 0.707, DB24_DOWN), (5, 20000.0, 8.0, DB24_DOWN), (0, 20000.0, 8.0, 1.0)),
    "mixed": ((2, 20.0, 0.707, 1.0), (6, 20.0, 8.0, 1.0), (1, 20.0, 8.0, 1.0), (4, 20.0, 0.707, DB24_DOWN)),
}


@pytest.mark.parametrize("band", BANDS, ids=[f"m{b[0]}-{b[1]:g}Hz-q{b[2]:g}-g{b[3]:g}" for b in BANDS])
def test_param_eq_band_edges(lib, f64, band):
    _run_param_eq(lib, f64, (band,), 96000.0, 96000)


@pytest.mark.parametrize("srate", [44100.0, 96000.0, 192000.0])
@pytest.mark.parametrize("stack", sorted(STACKS))
def test_param_eq_stacks(lib, f64, stack, srate):
    _run_param_eq(lib, f64, STACKS[stack], srate, 96000)


@pytest.mark.parametrize("srate", [44100.0, 192000.0])
@pytest.mark.parametrize("mode", [3, 5, 9])
def test_param_eq_sessions(lib, f64, mode, srate):
    _run_param_eq(lib, f64, ((mode, 20.0, 8.0, DB24_UP),), srate, int(srate))


LOW_SHELF = ((3, 20.0, 8.0, DB24_UP),)


@pytest.mark.parametrize("n", [1, 2, 1023, 1024, 1025, 1024 * 94 - 1, 1024 * 94, 1024 * 94 + 1, 96000, 480000])
def test_scan_geometry(lib, f64, n):
    """one sample, fewer samples than chunks, one sample per chunk, ragged / full / one-sample last chunks (the `full`
    test of scan_states: L = 94 and 95), the 1 s and 5 s IRs at 96 kHz"""
    _run_param_eq(lib, f64, LOW_SHELF, 96000.0, n)


@pytest.mark.gpu
@pytest.mark.parametrize("stack", ["issue4", "lows_up"])
def test_scan_geometry_30s_ir_96k(f64, stack):
    """a 30 s IR at 96 kHz: 2.88 M taps, L = 2813 samples per chunk"""
    _run_param_eq(get_lib("cuda"), f64, STACKS[stack], 96000.0, 2880000, restated=False)


@pytest.mark.gpu
@pytest.mark.parametrize("band", BANDS, ids=[f"m{b[0]}-{b[1]:g}Hz-q{b[2]:g}-g{b[3]:g}" for b in BANDS])
def test_param_eq_band_edges_5s_192k(f64, band):
    _run_param_eq(get_lib("cuda"), f64, (band,), 192000.0, 960000, restated=False)


# ---- resampler low pass: k_scan2<RsFilterRec> (FP64 scan) ------------------------------------------------------------
def _interp64(x, ratio, M):
    """rs_interp in float64: output m at input position m * ratio, zero beyond the input"""
    pos = np.arange(M, dtype=np.float64) * ratio
    i = pos.astype(np.int64)
    a = np.where(i < x.size, x[np.minimum(i, x.size - 1)], 0.0)
    b = np.where(i + 1 < x.size, x[np.minimum(i + 1, x.size - 1)], 0.0)
    return a + (pos - i) * (b - a)


def _rs_stage64(f64, x, ratio, M, scale, flush):
    """one ResamplingAudioSource pass as ir_pipeline runs it (irshape.cu rs_stage), in float64"""
    if ratio > 1.0001:
        ls = int((M - 1) * ratio) + 2
        s = np.zeros(ls, np.float64)
        s[:min(ls, x.size)] = x[:ls]
        y = np.empty_like(s)
        f64.sf_rs_lowpass64(ratio, s, y, ls, flush)
        return _interp64(y, ratio, M) * scale
    t = _interp64(x, ratio, M)
    y = np.empty_like(t)
    f64.sf_rs_lowpass64(ratio, t, y, M, flush)
    return y * scale


RESAMPLE = {
    "192k_to_44k1_stretch-1": (192000.0, 44100.0, -1.0, 192000),
    "44k1_to_192k_stretch+1": (44100.0, 192000.0, 1.0, 44100),
}


@pytest.mark.parametrize("case", sorted(RESAMPLE))
def test_resampler_low_pass(lib, f64, case):
    """The low pass runs in double everywhere, so the device, the restatement and the float64 pipeline agree near float
    rounding.  The one non-linear step is JUCE's flush of |y| <= 1e-8 to zero, which the chunks apply to their own
    zero-state runs as well: per sample it moves the filter's state by at most 1e-8, so it can move an output by at most
    1e-8 times the l1 norm of the recursive part's impulse response, per stage, times the stage's output scale."""
    ir_sr, sr, stretch, n = RESAMPLE[case]
    raws = [synth_ir(n, c) for c in range(2)]
    kw = dict(ir_srate=ir_sr, srate=sr, stretch=stretch, autogain=False, gain=1.0, clip=False)
    got = ir_recalc(raws, lib=lib, **kw)
    r32 = rc.ir_recalc(raws, **kw)
    rs = ir_sr / sr
    n1 = int(np.ceil(n / rs))
    ss = 2.0 ** stretch * sr
    st = sr / ss
    n2 = int(np.ceil(n1 * ss / sr))
    assert got[0].size == r32[0].size == n2
    flush_bound = 1e-8 * (f64.sf_rs_feedback_l1(rs, 1 << 20) * float(np.float32(rs)) * 2.0
                          + f64.sf_rs_feedback_l1(st, 1 << 20))
    for c in range(2):
        x = raws[c].astype(np.float64)
        r64 = _rs_stage64(f64, _rs_stage64(f64, x, rs, n1, float(np.float32(rs)), 1), st, n2, 1.0, 1)
        r64_noflush = _rs_stage64(f64, _rs_stage64(f64, x, rs, n1, float(np.float32(rs)), 0), st, n2, 1.0, 0)
        assert np.max(np.abs(r64 - r64_noflush)) <= flush_bound, case
        peak = float(np.max(np.abs(r64)))
        e_dev = float(np.max(np.abs(got[c] - r64)))
        e_32 = float(np.max(np.abs(r32[c] - r64)))
        # float rounding of the stages' outputs (~6e-8 of peak each, three roundings) plus the flush's reach
        assert e_dev <= max(1e-6 * peak, FACTOR * e_32) + flush_bound, (case, c, e_dev / peak, e_32 / peak)
        assert e_32 <= 1e-6 * peak + flush_bound, (case, c)
        assert np.max(np.abs(got[c] - r32[c])) <= TOL * peak


# ---- send chain: k_chain_send through b200conv_chain_process -----------------------------------------------------------
class F64Chain:
    """the send path's low cut (HP) and high cut (LP) per channel, serially in float64 and in float32 (the restatement),
    filter state carried across calls and slope switches as Filter keeps it (ic1..ic4 and the 6 dB `state`)"""

    def __init__(self, f64, srate):
        self.f, self.sr = f64, srate
        self.st64 = [[np.zeros(5, np.float64) for _ in range(2)] for _ in range(2)]
        self.st32 = [[np.zeros(5, np.float32) for _ in range(2)] for _ in range(2)]

    def set(self, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope):
        self.filters = []                                  # (index, slope, mode, coefficients) of the filters that are on
        for k, (on, slope, mode, fr) in enumerate(((lowcut_hz > 20.0, lowcut_slope, 2, lowcut_hz),
                                                   (highcut_hz < 20000.0, highcut_slope, 0, highcut_hz))):
            c = np.empty(9, np.float32)
            self.f.sf_filter_coeffs(slope, mode, self.sr, fr, c)
            if on:
                self.filters.append((k, slope, mode, c))

    def process(self, xs):
        out32, out64 = [], []
        for ch, x in enumerate(xs):
            a, b = x.astype(np.float32), x.astype(np.float64)
            for k, slope, mode, c in self.filters:
                a2, b2 = np.empty_like(a), np.empty_like(b)
                self.f.sf_filter_run32(slope, mode, c, self.st32[ch][k], a, a2, a.size)
                self.f.sf_filter_run64(slope, mode, c, self.st64[ch][k], b, b2, b.size)
                a, b = a2, b2
            out32.append(a)
            out64.append(b)
        return out32, out64


ONE_TAP = np.ones(1, np.float32)


def _chain_engine(l, srate, cuts):
    """a stereo handle whose wet output is the filtered send times 0.5: IR [1], no predelay, dry 0, wet 1, width 1
    (mid + side = L, times the normalisation 1 / (1 + width))"""
    e = Engine(2, lib=l)
    assert e.init_uniform(64, [ONE_TAP, ONE_TAP])
    e.chain_configure(srate=srate, predelay=0, width=1.0, drygain=0.0, wetgain=1.0, **cuts)
    return e


def _dc_noise(n, seed):
    rng = np.random.default_rng(seed)
    return [(0.6 - 0.3 * ch + 0.25 * rng.standard_normal(n)).astype(np.float32) for ch in range(2)]


def test_chain_output_scale_is_one_half():
    """the wet mixdown of the restatement (chain_oracle.c::oc_chain_wet) at width 1, dry 0, wet 1 is 0.5 * L / 0.5 * R
    to float rounding, for any L, R: what _chain_engine relies on"""
    a, b = _dc_noise(5000, 1)
    ch = orc.OracleChain(48000.0, 20.0, 0, 20000.0, 0, 0, 1.0, 0.0, 1.0, delay_size=4096)
    z = np.zeros_like(a)
    oL, oR = ch.wet(z, z, a, b, None, None, np.ones_like(a))
    peak = max(np.max(np.abs(a)), np.max(np.abs(b)))
    assert np.max(np.abs(oL - 0.5 * a)) <= 1.2e-7 * peak and np.max(np.abs(oR - 0.5 * b)) <= 1.2e-7 * peak


def _run_chain(l, f64, srate, cuts, calls, seed=5, updates=None):
    """the calls through the device chain and the two serial references; updates: {call index: new cuts}"""
    n = sum(calls)
    x = _dc_noise(n, seed)
    e = _chain_engine(l, srate, cuts)
    ref = F64Chain(f64, srate)
    ref.set(**cuts)
    got, r32, r64 = [[], []], [[], []], [[], []]
    pos = 0
    for k, m in enumerate(calls):
        if updates and k in updates:
            e.chain_update(srate=srate, predelay=0, width=1.0, drygain=0.0, wetgain=1.0, **updates[k])
            ref.set(**updates[k])
        sl = slice(pos, pos + m)
        a, b = e.chain_process(x[0][sl], x[1][sl])
        o32, o64 = ref.process([x[0][sl], x[1][sl]])
        for ch, y in enumerate((a, b)):
            got[ch].append(np.asarray(y, np.float64) * 2.0)
            r32[ch].append(o32[ch])
            r64[ch].append(o64[ch])
        pos += m
    e.close()
    for ch in range(2):
        _check(np.concatenate(got[ch]), np.concatenate(r32[ch]), np.concatenate(r64[ch]), (srate, cuts, ch))


def _cuts(lc, lcs, hc, hcs):
    return dict(lowcut_hz=lc, lowcut_slope=lcs, highcut_hz=hc, highcut_slope=hcs)


# low cut 20 Hz and high cut 20 kHz are the off positions (src/PluginProcessor.cpp:1643, :1647); 20.5 Hz is the lowest
# low cut that runs.  20 Hz / 40 Hz at 12 / 24 dB is the case the FP32 scan failed at 96 kHz.
CHAIN_CUTS = [_cuts(lc, s, 20000.0, 0) for lc in (20.5, 1000.0, 20000.0) for s in (0, 1, 2)] + \
             [_cuts(20.0, 0, hc, s) for hc in (20.0, 1000.0, 19999.0) for s in (0, 1, 2)] + \
             [_cuts(20.5, 1, 40.0, 2), _cuts(20.5, 2, 20.0, 2), _cuts(20.0, 0, 20000.0, 0),
              _cuts(20000.0, 2, 20.0, 2), _cuts(20000.0, 0, 20.0, 0), _cuts(1000.0, 1, 1000.0, 1)]
CHAIN_IDS = [f"lc{c['lowcut_hz']:g}x{c['lowcut_slope']}-hc{c['highcut_hz']:g}x{c['highcut_slope']}" for c in CHAIN_CUTS]
RT_CALLS = [1, 63, 64, 65, 128] * 4                 # real-time calls (the pinned zero-copy path)
BATCH_CALLS = [1023, 1024, 1025, 48000]


@pytest.mark.parametrize("srate", [44100.0, 96000.0, 192000.0])
@pytest.mark.parametrize("cuts", CHAIN_CUTS, ids=CHAIN_IDS)
def test_chain_cuts(lib, f64, cuts, srate):
    """every cut position and slope, inverted cuts, a stream of real-time and batch calls over DC plus noise"""
    _run_chain(lib, f64, srate, cuts, RT_CALLS + BATCH_CALLS + RT_CALLS)


@pytest.mark.parametrize("srate", [44100.0, 96000.0, 192000.0])
def test_chain_one_long_call(lib, f64, srate):
    """low cut 20 Hz 12 dB, high cut 40 Hz 24 dB in one 96 000-sample call: 1024 chunks of 94"""
    _run_chain(lib, f64, srate, _cuts(20.5, 1, 40.0, 2), [96000])


@pytest.mark.gpu
@pytest.mark.parametrize("srate", [44100.0, 96000.0, 192000.0])
@pytest.mark.parametrize("cuts", CHAIN_CUTS, ids=CHAIN_IDS)
def test_chain_cuts_long_calls(f64, cuts, srate):
    _run_chain(get_lib("cuda"), f64, srate, cuts, [192000, 128, 192000, 48000] + RT_CALLS * 10)


@pytest.mark.parametrize("cuts", [_cuts(20.5, 2, 40.0, 2), _cuts(20.5, 1, 20000.0, 0)], ids=["lc20.5x2-hc40x2", "lc20.5x1"])
def test_chain_swap_warm_up_replay(lib, f64, cuts):
    """The hot swap's warm-up (b200conv_chain_swap, host block 128 at 96 kHz) replays numBlocks * 128 = 23 936 samples
    of the filtered send history through fresh filters in one chunked-scan launch (src/PluginProcessor.cpp:1694-1756).
    The incoming IR is a delta at tap D, so once the 50 ms fade has completed the output is 0.5 * the replayed, refiltered
    history for the first D samples after the swap, and the current send after that."""
    sr, hb, D = 96000.0, 128, 20000
    W = int(np.ceil(sr)) // 4
    N = W // hb * hb
    pre = [hb] * 20 + [24000] + [hb] * 20
    post = [hb] * ((D + 3000) // hb)
    calls = pre + post
    x = _dc_noise(sum(calls), 7)
    live = _chain_engine(lib, sr, cuts)
    inc = Engine(2, lib=lib)
    h = np.zeros(D + 1, np.float32)
    h[D] = 1.0
    assert inc.init_uniform(64, [h, h])
    ref = F64Chain(f64, sr)
    ref.set(**cuts)
    sends32, sends64 = ref.process(x)                        # the live chain's filtered send, all calls
    got = [[], []]
    pos = 0
    swap_at = sum(pre)
    done_at = None
    for k, m in enumerate(calls):
        if k == len(pre):
            live.chain_swap(inc, hb)
        sl = slice(pos, pos + m)
        a, b = live.chain_process(x[0][sl], x[1][sl])
        if k >= len(pre):
            got[0].append(a)
            got[1].append(b)
        pos += m
        if k >= len(pre) and live.chain_swap_state() == 3:
            live, inc = inc, live
            done_at = pos - swap_at                          # samples after the swap from which alpha = 1
    assert done_at is not None and done_at < D
    live.close()
    inc.close()
    # the replay: index j reads the sample W - 1 - j back from the end of the swap call (one piece)
    end = swap_at + post[0]
    idx = end - (W - 1 - np.arange(N))
    rep32, rep64 = F64Chain(f64, sr), F64Chain(f64, sr)    # fresh filters; float history into float, double into double
    rep32.set(**cuts)
    rep64.set(**cuts)
    r32 = rep32.process([sends32[ch][idx] for ch in range(2)])[0]
    r64 = rep64.process([sends64[ch][idx] for ch in range(2)])[1]
    for ch in range(2):
        y = np.concatenate(got[ch])[done_at:].astype(np.float64) * 2.0
        i = np.arange(done_at, done_at + y.size)
        s32 = np.concatenate([r32[ch], sends32[ch][swap_at:]])
        s64 = np.concatenate([r64[ch], sends64[ch][swap_at:]])
        _check(y, s32[N + i - D], s64[N + i - D], ("swap", cuts, ch))


@pytest.mark.parametrize("srate", [48000.0, 96000.0])
def test_chain_slope_switch_low_cut(lib, f64, srate):
    """b200conv_chain_update 6 -> 24 -> 6 -> 12 dB at a 20.5 Hz low cut mid-stream: the stash exchange of slot 0 feeds
    the scan's initial state, whose error a 20 Hz pole keeps for seconds"""
    base = _cuts(20.5, 0, 20000.0, 0)
    calls = [128] * 20 + [48000] + [128] * 20 + [96000] + [65] * 30 + [48000] + [128] * 10 + [20000]
    ups = {21: _cuts(20.5, 2, 20000.0, 0), 42: _cuts(20.5, 0, 20000.0, 0), 73: _cuts(20.5, 1, 20000.0, 0),
           84: _cuts(20.5, 2, 40.0, 2)}
    _run_chain(lib, f64, srate, base, calls, updates=ups)
