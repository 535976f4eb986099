"""The whole of Impulse::recalcImpulse (src/dsp/Impulse.cpp:299-360) through b200conv_ir_recalc / b200conv_init_*_recalc:
resampling to the project rate and stretch (JUCE ResamplingAudioSource), the parametric EQ (SVF sections) and the decay
EQ with its table built from bands, around the steps b200conv_ir_shape already covers.

The C restatement (recalc_oracle.c::oc_ir_recalc) is pinned to the reference's own compiled Impulse.cpp
(oracle/_ref/librefimpulse.so) when it is present, else to tests/golden/pins/impulse_pins.npz; the emulation build and the
H100 build are checked against the restatement."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import recalc as rc
from reevr_b200 import _lib
from reevr_b200.convolver import B200ConvError, Engine, ir_recalc, ir_recalc_len, ir_shape
from tests import ircases
from tests.backends import get_lib, lib  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = os.path.join(ROOT, "tests", "golden", "pins", "impulse_pins.npz")
CASES = ircases.cases()
IDS = [c[0] for c in CASES]


def _peak(chans):
    return max((float(np.max(np.abs(c))) for c in chans if c.size), default=0.0)


def _digest(chans):
    return hashlib.sha256(b"".join(np.ascontiguousarray(c, np.float32).tobytes() for c in chans)).hexdigest()


@pytest.fixture(scope="module")
def pins():
    return np.load(PINS)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_matches_reference(case, pins):
    """oc_ir_recalc == the compiled Impulse::recalcImpulse: bit-identical without the decay EQ (serial, same arithmetic),
    within 1e-6 of peak with it (its FFT is not the reference's AudioFFT)"""
    name, n, nch, kw = case
    raws = ircases.raw(n, nch)
    got = rc.ir_recalc(raws, **kw)
    exact = not kw.get("decay_eq")
    if rc.ref_impulse_available():
        want = rc.ref_ir_recalc(raws, **kw)
        assert got[0].size == want[0].size
        if exact:
            assert all(np.array_equal(g, w) for g, w in zip(got, want))
        for g, w in zip(got, want):
            assert np.max(np.abs(g - w), initial=0.0) <= 1e-6 * _peak(want)
    assert got[0].size == int(pins[f"{name}/len"])
    if exact:
        assert _digest(got) == str(pins[f"{name}/sha256"])
    idx = pins[f"{name}/index"]
    for c in range(nch):
        assert np.max(np.abs(got[c][idx] - pins[f"{name}/value"][c]), initial=0.0) <= 1e-6 * float(pins[f"{name}/peak"])


@pytest.mark.parametrize("which", ["emu", "product"])
def test_lengths(which, pins):
    """b200conv_ir_recalc_len (host arithmetic, no device needed) == the reference's output length, every case"""
    l = get_lib("emu") if which == "emu" else _lib.load()
    for name, n, nch, kw in CASES:
        assert ir_recalc_len(n, lib=l, **kw) == int(pins[f"{name}/len"]), name
        assert ir_recalc_len(n, lib=l, **kw) == rc.ir_recalc_len(n, **kw), name


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_device_matches_restatement(lib, case, pins):
    name, n, nch, kw = case
    raws = ircases.raw(n, nch)
    want = rc.ir_recalc(raws, **kw)
    got = ir_recalc(raws, lib=lib, **kw)
    assert got[0].size == want[0].size == int(pins[f"{name}/len"])
    # the first STFT hop is ill-conditioned in the reference itself when the decay EQ is on (window starts at 0)
    lo = 1024 if kw.get("decay_eq") else 0
    peak = _peak(want)
    for c in range(nch):
        assert np.max(np.abs(got[c][lo:] - want[c][lo:]), initial=0.0) <= 1e-5 * peak, (name, c)


@pytest.mark.gpu
def test_device_full_size():
    """10 s quad IR recorded at 44.1 kHz in a 48 kHz session, stretch 1: about 1 M output taps per channel, so the chunked
    scans run chunks of ~1000 samples"""
    kw = dict(ir_srate=44100.0, srate=48000.0, stretch=1.0, param_eq=ircases.PARAM_EQS[1], decay_eq=ircases.DECAY_EQS[1][0],
              decay_rate=0.5)
    raws = ircases.raw(441000, 4)
    want = rc.ir_recalc(raws, **kw)
    got = ir_recalc(raws, lib=get_lib("cuda"), **kw)
    assert got[0].size == want[0].size > 950000
    peak = _peak(want)
    for c in range(4):
        assert np.max(np.abs(got[c][1024:] - want[c][1024:])) <= 1e-5 * peak, c


@pytest.mark.parametrize("kind", ["twostage", "uniform"])
def test_recalc_init_equals_recalc_then_init(lib, kind):
    """b200conv_init_*_recalc (taps never leave the device) == recalculating with the restatement, then a plain init.
    (No decay EQ here: its first STFT hop is ill-conditioned in the reference itself and would leak into every output.)"""
    kw = dict(ir_srate=44100.0, srate=48000.0, stretch=0.25, reverse=True, trim_left=0.02, gain=2.0,
              param_eq=ircases.PARAM_EQS[2], decay=0.1)
    raws = ircases.raw(12000, 4)
    shaped = rc.ir_recalc(raws, **kw)
    x = [orc.synth_input(128 * 60, c) for c in range(4)]
    e, o = Engine(4, lib=lib), Engine(4, lib=lib)
    if kind == "twostage":
        assert e.init_twostage_recalc(128, 1024, raws, **kw)
        assert o.init_twostage(128, 1024, shaped)
    else:
        assert e.init_uniform_recalc(256, raws, **kw)
        assert o.init_uniform(256, shaped)
    ys, ref = e.process(x), o.process(x)
    for c in range(4):
        assert np.max(np.abs(ys[c] - ref[c])) <= 2e-5 * np.max(np.abs(ref[c]))
    e.close()
    o.close()


def test_decay_table_from_bands(lib):
    """the library's decay table from bands == the restatement's (bit for bit)"""
    for bands, rate in ircases.DECAY_EQS[1:]:
        for sr in (44100.0, 48000.0, 96000.0):
            arr = (_lib.EqBand * len(bands))(*[_lib.EqBand(*b) for b in bands])
            got = np.empty(2049, np.float64)
            lib.pc_ir_decay_lut(arr, len(bands), C.c_double(sr), C.c_float(rate), got.ctypes.data_as(C.c_void_p))
            assert np.array_equal(got, rc.decay_lut(bands, sr, rate))


def test_shape_path_unchanged(lib):
    """without resampling, stretch and the parametric EQ, b200conv_ir_recalc is b200conv_ir_shape with the table built from
    the bands: bit-identical"""
    bands, rate = ircases.DECAY_EQS[1]
    arr = (_lib.EqBand * len(bands))(*[_lib.EqBand(*b) for b in bands])
    lut = np.empty(2049, np.float64)
    lib.pc_ir_decay_lut(arr, len(bands), C.c_double(48000.0), C.c_float(rate), lut.ctypes.data_as(C.c_void_p))
    common = dict(autogain=True, reverse=True, trim_left=0.1, trim_right=0.05, gain=40.0, clip=True, attack=0.02, decay=0.3)
    for nch in (2, 4):
        raws = ircases.raw(21000, nch)
        for with_decay in (False, True):
            got = ir_recalc(raws, lib=lib, ir_srate=48000.0, srate=48000.0, stretch=0.0,
                            decay_eq=bands if with_decay else (), decay_rate=rate, **common)
            want = ir_shape(raws, lib=lib, lut=lut if with_decay else None, srate=48000.0, **common)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), (nch, with_decay)


def _call(l, raws, p, out_cap=None, out_len=True, outs=True, device=0):
    n = raws[0].size
    bufs = [np.zeros(max(out_cap or 1, 1), np.float32) for _ in raws]
    rp = (C.c_void_p * len(raws))(*[a.ctypes.data for a in raws])
    op = (C.c_void_p * len(raws))(*[b.ctypes.data for b in bufs]) if outs else None
    m = C.c_size_t(0)
    cap = out_cap if out_cap is not None else l.b200conv_ir_recalc_len(n, C.byref(p) if p is not None else None)
    return l.b200conv_ir_recalc(device, rp, len(raws), n, C.byref(p) if p is not None else None, op, cap,
                                C.byref(m) if out_len else None)


def test_error_paths():
    l = get_lib("emu")
    raws = ircases.raw(2000, 2)

    def params(**kw):
        return Engine._recalc_params(**kw)

    good, keep = params(ir_srate=44100.0, srate=48000.0, stretch=0.5, param_eq=ircases.PARAM_EQS[1])
    need = l.b200conv_ir_recalc_len(2000, C.byref(good))
    assert need > 2000
    assert _call(l, raws, good, out_cap=need) == 0
    assert _call(l, raws, good, out_cap=need - 1) == -1                      # out_cap smaller than the output
    assert _call(l, raws, None, out_cap=need) == -1                          # NULL parameters
    assert _call(l, raws, good, out_cap=need, out_len=False) == -1           # NULL out_len
    assert _call(l, raws, good, out_cap=need, outs=False) == -1              # NULL out
    assert l.b200conv_ir_recalc(0, None, 2, 2000, C.byref(good), None, need, None) == -1
    assert l.b200conv_ir_recalc_len(2000, None) == 0
    for bad in (dict(srate=0.0), dict(srate=-48000.0), dict(ir_srate=0.0), dict(ir_srate=-1.0),
                dict(param_eq=[(5, 1000.0, 0.7, 2.0)] * 9), dict(decay_eq=[(5, 1000.0, 0.7, 2.0)] * 9),
                dict(param_eq=[(10, 1000.0, 0.7, 2.0)]), dict(decay_eq=[(-1, 1000.0, 0.7, 2.0)])):
        kw = dict(ir_srate=44100.0, srate=48000.0)
        kw.update(bad)
        p, keep2 = params(**kw)
        assert _call(l, raws, p, out_cap=10 ** 6) == -1, bad
    e = Engine(2, lib=l)
    assert not e.init_twostage_recalc(64, 512, raws, srate=0.0)              # B200CONV_EINVAL, handle still usable
    assert e.init_twostage_recalc(64, 512, raws, ir_srate=44100.0, srate=48000.0)
    e.close()


def test_no_device_is_ecuda():
    """the product library reports B200CONV_ECUDA for a device it cannot select (no GPU, or no such ordinal)"""
    l = _lib.load()
    raws = ircases.raw(2000, 2)
    p, keep = Engine._recalc_params(ir_srate=44100.0, srate=48000.0)
    assert _call(l, raws, p, device=4096) == -2
    with pytest.raises(B200ConvError):
        ir_recalc(raws, device=4096, lib=l, ir_srate=44100.0, srate=48000.0)


def test_reference_build_skips_without_sources(tmp_path):
    """oracle/recalc.mk's `ref` target is a no-op where the reference sources are absent"""
    out = subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "recalc.mk", "ref", f"REF={tmp_path}/absent"],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "reference sources absent; librefimpulse.so not rebuilt"


@pytest.mark.skipif(not os.path.isfile("/root/reference/src/dsp/Impulse.cpp"), reason="reference sources absent")
def test_reference_build_makes_librefimpulse():
    rc.build()
    assert os.path.exists(os.path.join(ROOT, "oracle", "_ref", "librefimpulse.so"))


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="no nvcc")
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "reevr_b200", "csrc", "irshape.cu")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", src,
                          "-o", str(tmp_path / "irshape.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stderr.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Compiling entry function" in line and ("k_scan2" in line or "k_rs_interp" in line):
            props = lines[i + 2]
            assert "0 bytes spill stores, 0 bytes spill loads" in props, (line, props)
            seen += 1
    assert seen == 3
