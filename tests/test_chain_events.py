"""Chain parameter changes at sample offsets inside one device call (b200conv_chain_process_device_events).

The contract: an events call equals the call cut at every event offset into b200conv_chain_process_device calls with
b200conv_chain_update just before each, within float rounding (here 1e-5 of peak), and leaves the handle as those
calls leave it.  Short pieces run k_chain_send once per segment; long pieces over several segments run the segmented
whole-GPU send form (kernels_chain.cuh k_chain_seg_*), which is also held to the float64 criterion of
tests/test_scan_precision.py.  On the emulation build "device" buffers are host arrays; under -m gpu they are CUDA
tensors.
"""
import ctypes as C

import numpy as np
import pytest

from reevr_b200 import _lib
from reevr_b200.convolver import Engine
from tests import backends
from tests.backends import lib  # noqa: F401
from tests.test_chain_device import Dev, _cfg, _engine, _irs, _signals
from tests.test_scan_precision import ONE_TAP, F64Chain, _check, _dc_noise, f64  # noqa: F401

ESTATE, EINVAL = -3, -1
LONG = 524288
MBB = LONG // 64 + 2                   # uniform 64 handles: Lmax = MBB * 64, pieces of Lmax - 64 samples
PIECE = MBB * 64 - 64
CTA = 8192                             # samples per CTA of the whole-GPU forms (kWideLc * kWideT)
TOL = 1e-5


def _gpu(l):
    return backends._cache.get("emu") is not l


def _every(l):
    """event spacing of the dense sweeps: one per 64-sample chunk on the emulation build, 512 on the GPU"""
    return 512 if _gpu(l) else 64


def _cut_run(l, e, d, X, O, YS, YR, n, events, stride):
    """the cut-call sequence on e: chain_update just before the call that starts at each event offset"""
    pos = 0
    for off, cfg in events:
        if off > pos:
            e.chain_process_device(d.ptr(X, pos), stride, d.ptr(O, pos), stride, off - pos, d.ptr(YS, pos),
                                   d.ptr(YR, pos), sync=True)
            pos = off
        e.chain_update(**cfg)
    e.chain_process_device(d.ptr(X, pos), stride, d.ptr(O, pos), stride, n - pos, d.ptr(YS, pos), d.ptr(YR, pos),
                           sync=True)


def _pair(l, C_, cfg0, events, n, seed=3, irs=None, env=True, mbb=0, after=None):
    """(events call, cut calls) outputs on twin handles; after(e, d): more calls on each handle, outputs appended"""
    d = Dev(l)
    L, R, ys, yr = _signals(n, seed, env)
    outs = []
    for mode in ("events", "cuts"):
        e = _engine(l, C_, cfg0, irs, max_batch_blocks=mbb)
        X = d.put(np.stack([L, R]))
        O = d.put(np.zeros((2, n), np.float32))
        YS, YR = (d.put(a) if a is not None else None for a in (ys, yr))
        if mode == "events":
            e.chain_process_device_events(d.ptr(X), n, d.ptr(O), n, n, events, d.ptr(YS), d.ptr(YR), sync=True)
        else:
            _cut_run(l, e, d, X, O, YS, YR, n, events, n)
        got = [d.get(O)]
        if after:
            got += after(e, d)
        e.close()
        outs.append(got)
    return outs


def _close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    peak = float(np.max(np.abs(b)))
    err = float(np.max(np.abs(a - b)))
    assert err <= TOL * max(peak, 1e-30), (what, err / max(peak, 1e-30))


def _assert_pairs(outs, what):
    for k, (a, b) in enumerate(zip(*outs)):
        _close(a, b, (what, k))


# ---- 1. no events is the device call --------------------------------------------------------------------------------
FULL = _cfg(lc=150.0, lcs=1, hc=9000.0, hcs=2, predelay=700, drygain=0.6, wetgain=0.8, width=0.5)


@pytest.mark.parametrize("C_", [2, 4])
@pytest.mark.parametrize("length", ["short", "long"])
def test_no_events_is_the_device_call(lib, C_, length):
    n, mbb = (4096, 0) if length == "short" else (LONG + 999, MBB)
    d = Dev(lib)
    L, R, ys, yr = _signals(n, 4)
    outs = []
    for mode in ("device", "events"):
        e = _engine(lib, C_, FULL, _irs(C_, 20) if C_ == 4 else None, max_batch_blocks=mbb)
        X = d.put(np.stack([L, R]))
        O = d.put(np.zeros((2, n), np.float32))
        YS, YR = d.put(ys), d.put(yr)
        for k in range(2):                     # the second call continues from the state the first left
            if mode == "device":
                e.chain_process_device(d.ptr(X), n, d.ptr(O), n, n, d.ptr(YS), d.ptr(YR), sync=True)
            else:
                e.chain_process_device_events(d.ptr(X), n, d.ptr(O), n, n, [], d.ptr(YS), d.ptr(YR), sync=True)
            outs.append((mode, k, d.get(O)))
        e.close()
    for k in range(2):
        assert np.array_equal(outs[k][2], outs[2 + k][2])


# ---- 2. events equal cut calls --------------------------------------------------------------------------------------
def _ev(off, srate=48000.0, **kw):
    return off, _cfg(srate=srate, **kw)


def _sweep(n, step, first=0):
    out = []
    for k, off in enumerate(range(first, n, step)):
        f = 20.5 * (1.0 + 0.37 * (k % 97)) ** 1.5
        out.append(_ev(off, lc=min(f, 5000.0), lcs=(k // 7) % 3, hc=max(20000.0 - 13.0 * k, 3000.0), hcs=2 - (k // 11) % 3,
                       predelay=300, drygain=0.5, wetgain=0.7, width=0.6))
    return out


@pytest.mark.parametrize("length", ["short", "long"])
def test_cut_frequency_sweep(lib, length):
    n, mbb = (4096 * 3 + 5, 0) if length == "short" else (LONG + 77, MBB)
    ev = _sweep(n, _every(lib))
    _assert_pairs(_pair(lib, 2, _cfg(lc=100.0, lcs=1, predelay=300), ev, n, mbb=mbb), "sweep")


def test_slope_switches(lib):
    """6 <-> 12 <-> 24 dB on both cuts: inside a 64-sample chunk, on a CTA boundary, on a piece boundary"""
    n = PIECE + 3 * CTA + 100
    offs = [3 * 64 + 37, 5 * CTA, 5 * CTA + 64 * 7 + 1, 9 * CTA - 1, PIECE, PIECE + 13, PIECE + 2 * CTA]
    slopes = [(0, 1), (2, 0), (1, 2), (0, 0), (2, 1), (1, 0), (0, 2)]
    ev = [_ev(o, lc=40.0 + 10 * k, lcs=a, hc=9000.0 - 100 * k, hcs=b, predelay=64)
          for k, (o, (a, b)) in enumerate(zip(offs, slopes))]
    _assert_pairs(_pair(lib, 2, _cfg(lc=30.0, lcs=1, hc=12000.0, hcs=1, predelay=64), ev, n, mbb=MBB), "slopes")


def test_filters_off_and_on(lib):
    n = LONG + 4321
    ev = []
    for k, off in enumerate(range(1000, n, 37 * 211)):
        lc = 20.0 if k % 3 == 0 else 200.0 + k           # 20 Hz: the low cut is off
        hc = 20000.0 if k % 4 == 1 else 7000.0 - k      # 20 kHz: the high cut is off
        ev.append(_ev(off, lc=lc, lcs=k % 3, hc=hc, hcs=(k + 1) % 3))
    _assert_pairs(_pair(lib, 2, _cfg(lc=20.0, hc=20000.0), ev, n, mbb=MBB), "on/off")


def test_predelay_changes_and_growth(lib):
    """up and down, and beyond D = 2 s: the delay line grows, the history reads zero from that event's sample"""
    n = PIECE + 200000
    pds = [(3000, 100), (CTA * 3 + 5, 3000), (60000, 50), (200000, 100000), (PIECE + 17, 120000), (PIECE + 90000, 7)]
    ev = [_ev(o, lc=90.0, lcs=1, predelay=p, drygain=0.3) for o, p in pds]
    for length, mbb in (("long", MBB), ("short", 0)):
        _assert_pairs(_pair(lib, 2, _cfg(lc=90.0, lcs=1, predelay=500, drygain=0.3), ev, n, mbb=mbb),
                      ("predelay", length))


def test_wet_parameters_on_quad(lib):
    n = LONG + 3000
    ev = [_ev(o, lc=80.0, lcs=2, hc=11000.0, hcs=1, predelay=200 + k, width=(k % 5) * 0.4, drygain=0.1 * (k % 7),
              wetgain=1.0 - 0.05 * (k % 9), ts=bool(k % 2))
          for k, o in enumerate(range(0, n, 4099))]
    cfg0 = _cfg(lc=80.0, lcs=2, hc=11000.0, hcs=1, predelay=200)
    _assert_pairs(_pair(lib, 4, cfg0, ev, n, irs=_irs(4, 40), mbb=MBB), "quad")
    short = [(o, c) for o, c in ev if o < 4096 * 2] + [_ev(4096 * 2 + 1, ts=False, width=1.3)]
    _assert_pairs(_pair(lib, 4, cfg0, short, 4096 * 3, irs=_irs(4, 40)), "quad short")


@pytest.mark.parametrize("length", ["short", "long"])
def test_events_at_first_and_last_sample(lib, length):
    n, mbb = (3000, 0) if length == "short" else (LONG + 11, MBB)
    ev = [_ev(0, lc=300.0, lcs=0, predelay=10, width=0.2), _ev(n - 1, lc=900.0, lcs=2, hc=5000.0, hcs=0, predelay=9,
                                                                width=1.5, drygain=0.9)]
    _assert_pairs(_pair(lib, 2, FULL, ev, n, mbb=mbb), "first / last")


def test_consecutive_events(lib):
    n = LONG + 500
    ev = [_ev(o, lc=50.0 + 3 * k, lcs=k % 3, hc=8000.0 - k, hcs=(k // 2) % 3, predelay=100 + (k % 5), width=0.1 * (k % 11))
          for k, o in enumerate(range(CTA * 2 + 40, CTA * 2 + 340))]
    _assert_pairs(_pair(lib, 2, _cfg(lc=50.0, lcs=1, predelay=100), ev, n, mbb=MBB), "consecutive")


# ---- 3. precision against float64 -----------------------------------------------------------------------------------
@pytest.mark.parametrize("srate", [96000.0, 192000.0])
@pytest.mark.parametrize("step", [256, 4096])
def test_segmented_scan_against_float64(lib, f64, srate, step):
    """a ONE_TAP handle (the mix is 0.5 * the filtered send) over long pieces with thousands of segments near the unit
    circle (20.5 Hz .. 60 Hz low cuts), against the serial float64 filter with set() at each event"""
    n = LONG + 4096
    x = _dc_noise(n, 7)
    cuts = []
    for k in range(0, n, step):
        cuts.append((k, dict(lowcut_hz=20.5 + (k // step % 13) * 3.0, lowcut_slope=(k // step // 5) % 3,
                             highcut_hz=20000.0 if (k // step) % 4 else 15000.0, highcut_slope=(k // step) % 3)))
    base = dict(srate=srate, predelay=0, width=1.0, drygain=0.0, wetgain=1.0)
    ev = [(o, dict(base, **c)) for o, c in cuts]
    d = Dev(lib)
    e = _engine(lib, 2, dict(base, **cuts[0][1]), max_batch_blocks=MBB)
    X = d.put(np.stack(x))
    O = d.put(np.zeros((2, n), np.float32))
    e.chain_process_device_events(d.ptr(X), n, d.ptr(O), n, n, ev, sync=True)
    got = d.get(O)
    e.close()
    ref = F64Chain(f64, srate)
    r32, r64 = [[], []], [[], []]
    bounds = [o for o, _ in cuts] + [n]
    for k, (o, c) in enumerate(cuts):
        ref.set(**c)
        o32, o64 = ref.process([x[0][o:bounds[k + 1]], x[1][o:bounds[k + 1]]])
        for ch in range(2):
            r32[ch].append(o32[ch])
            r64[ch].append(o64[ch])
    for ch in range(2):
        _check(got[ch].astype(np.float64) * 2.0, np.concatenate(r32[ch]), np.concatenate(r64[ch]), (srate, step, ch))


# ---- 4. continuation ------------------------------------------------------------------------------------------------
def test_continuation_after_events(lib):
    """after the events call: a host call, an update and a device call, and an IR hot swap behave as after cut calls"""
    n = LONG + 2000
    ev = [_ev(o, lc=60.0 + k, lcs=(k + 1) % 3, hc=9000.0, hcs=k % 3, predelay=150 + 1000 * (k % 3), width=0.7,
              drygain=0.4) for k, o in enumerate(range(100, n, 9001))]
    ev.append(_ev(n - 500, lc=70.0, lcs=0, hc=8000.0, hcs=2, predelay=100000, width=0.9, drygain=0.2))

    def after(e, d):
        got = []
        L, R, ys, yr = _signals(4096, 11)
        a, b = e.chain_process(L, R, ys, yr)                    # the last event's configuration, the same ring
        got.append(np.stack([a, b]))
        e.chain_update(**_cfg(lc=500.0, lcs=1, predelay=40000, drygain=0.25))
        X = d.put(np.stack([L, R]))
        O = d.put(np.zeros((2, 4096), np.float32))
        e.chain_process_device(d.ptr(X), 4096, d.ptr(O), 4096, 4096, sync=True)
        got.append(d.get(O))
        inc = Engine(2, lib=e._l, max_batch_blocks=MBB)
        assert inc.init_twostage(64, 512, _irs(2, 70))
        e.chain_swap(inc, 512)                                  # warm-up replays the ring the events call wrote
        outs = []
        for k in range(30):
            a, b = (e if e.chain_swap_state() != 3 else inc).chain_process(L[:512], R[:512])
            outs.append(np.stack([a, b]))
        assert e.chain_swap_state() == 3
        got.append(np.concatenate(outs, axis=1))
        inc.close()
        return got

    outs = _pair(lib, 2, _cfg(lc=60.0, lcs=1, predelay=150), ev, n, irs=_irs(2, 60), mbb=MBB, after=after)
    _assert_pairs(outs, "continuation")


# ---- 5. refusals ----------------------------------------------------------------------------------------------------
def _raw(e, dry, out, n, events, n_events):
    arr = (_lib.ChainEvent * max(len(events or []), 1))()
    for k, (off, c) in enumerate(events or []):
        arr[k].offset = off
        arr[k].cfg = _lib.ChainConfig(c["srate"], c["lowcut_hz"], c["lowcut_slope"], c["highcut_hz"], c["highcut_slope"],
                                      c["predelay"], c["width"], c["drygain"], c["wetgain"], int(c["true_stereo"]))
    p = C.cast(arr, C.c_void_p) if events is not None else None
    return e._l.b200conv_chain_process_device_events(e._h, dry, 64, None, None, out, 64, n, p, n_events, 1)


def test_refusals(lib):
    d = Dev(lib)
    n = 64
    sig = _signals(n, 12)
    ok = [_ev(0, lc=100.0), _ev(10, predelay=200000)]        # valid, and the second would grow the delay line
    bad = {
        "slope": [_ev(0, lc=100.0), _ev(5, lcs=3)],
        "predelay": [_ev(0), _ev(5, predelay=-1)],
        "srate": [_ev(0), _ev(5, srate=44100.0)],
        "order": [_ev(10), _ev(5)],
        "equal": [_ev(5), _ev(5)],
        "beyond": ok[:1] + [_ev(64)],
        "grow-then-bad": [_ev(0, predelay=300000), _ev(5, hcs=-1)],
    }
    e = _engine(lib, 2, _cfg(lc=80.0, lcs=1))
    twin = _engine(lib, 2, _cfg(lc=80.0, lcs=1))
    X = d.put(np.stack(sig[:2]))
    O = d.put(np.zeros((2, n), np.float32))
    p, q = d.ptr(X), d.ptr(O)
    for what, evs in bad.items():
        assert _raw(e, p, q, n, evs, len(evs)) == EINVAL, what
    assert _raw(e, None, q, n, ok, 2) == EINVAL
    assert _raw(e, p, None, n, ok, 2) == EINVAL
    assert _raw(e, p, q, n, None, 2) == EINVAL
    assert _raw(e, p, q, 0, ok, 2) == EINVAL                  # offsets must lie below len
    outs = []
    for h in (e, twin):                                       # nothing changed: the next call matches the twin's
        O2 = d.put(np.zeros((2, n), np.float32))
        assert _raw(h, p, d.ptr(O2), n, ok, 2) == 0
        outs.append(d.get(O2))
    assert np.array_equal(outs[0], outs[1])
    e.close()
    twin.close()
    # no chain, fixed-latency handle, pending swap (armed, then fading)
    e = Engine(2, lib=lib)
    assert e.init_uniform(64, [ONE_TAP, ONE_TAP])
    assert _raw(e, p, q, n, ok, 2) == ESTATE
    e.chain_configure(**_cfg())
    e.set_latency(64)
    assert _raw(e, p, q, n, ok, 2) == ESTATE
    e.close()
    e = _engine(lib, 2, _cfg(), _irs(2, 80))
    twin = _engine(lib, 2, _cfg(), _irs(2, 80))
    incs = []
    for h in (e, twin):
        inc = Engine(2, lib=lib)
        assert inc.init_twostage(64, 512, _irs(2, 90))
        h.chain_swap(inc, 64)
        incs.append(inc)
    assert _raw(e, p, q, n, ok, 2) == ESTATE
    assert _raw(incs[0], p, q, n, ok, 2) == ESTATE             # the incoming handle owns no chain
    outs = []
    for h in (e, twin):
        O2 = d.put(np.zeros((2, n), np.float32))
        h.chain_process_device(p, 64, d.ptr(O2), 64, n, sync=True)
        outs.append(d.get(O2))
    assert np.array_equal(outs[0], outs[1])
    assert e.chain_swap_state() == 2
    assert _raw(e, p, q, n, ok, 2) == ESTATE
    for h in (e, twin, *incs):
        h.close()


# ---- 6. real size on the GPU ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_metric_shape_every_512():
    """the offline benchmark's metric shape (stereo, uniform 512, 2 s IR at 48 kHz) over 2 M samples, an event every
    512 samples, against the cut calls"""
    import torch
    from reevr_b200.synth import synth_input, synth_ir
    l = backends.get_lib("cuda")
    n = 2 * 1024 * 1024 + 512 * 37
    cfg0 = _cfg(lc=20.5, lcs=1, hc=16000.0, hcs=2, predelay=2400, width=0.8, drygain=0.7, wetgain=0.5)
    ev = []
    for k, off in enumerate(range(0, n, 512)):
        ev.append(_ev(off, lc=20.5 + (k % 50) * 4.0, lcs=1 + (k // 300) % 2, hc=16000.0 - (k % 40) * 100.0, hcs=2,
                      predelay=2400 + (k % 8) * 16, width=0.8 + 0.01 * (k % 20), drygain=0.7, wetgain=0.5))
    X = torch.from_numpy(np.stack([synth_input(n, 0), synth_input(n, 1)])).cuda()
    outs = []
    for mode in ("events", "cuts"):
        e = Engine(2, lib=l)
        assert e.init_uniform(512, [synth_ir(96000, c) for c in range(2)])
        e.chain_configure(**cfg0)
        O = torch.zeros_like(X)
        if mode == "events":
            e.chain_process_device_events(X.data_ptr(), n, O.data_ptr(), n, n, ev, sync=True)
        else:
            pos = 0
            for off, c in ev:
                if off > pos:
                    e.chain_process_device(X.data_ptr() + 4 * pos, n, O.data_ptr() + 4 * pos, n, off - pos)
                    pos = off
                e.chain_update(**c)
            e.chain_process_device(X.data_ptr() + 4 * pos, n, O.data_ptr() + 4 * pos, n, n - pos, sync=True)
        outs.append(O.cpu().numpy())
        e.close()
    _close(outs[0], outs[1], "metric")
