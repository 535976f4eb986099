"""The send / wet chain on device buffers (b200conv_chain_process_device).

Pieces shorter than the whole-GPU threshold run k_chain_send as the host entry does: device calls made of them are
bit for bit b200conv_chain_process.  Longer pieces run the whole-GPU send form (kernels_chain.cuh k_chain_wide_*): they
are held to the float64 criterion of tests/test_scan_precision.py and to 1e-5 of peak against the host entry.  The
tests use pieces of at most 4 096 or at least 524 288 samples, so they do not depend on where the threshold lies.
On the emulation build "device" buffers are host arrays; under -m gpu they are CUDA tensors.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests import backends
from tests.backends import lib  # noqa: F401
from tests.test_scan_precision import CHAIN_CUTS, CHAIN_IDS, ONE_TAP, RT_CALLS, F64Chain, _check, _cuts, _dc_noise, f64  # noqa: F401

ESTATE, EINVAL = -3, -1
LONG = 524288                          # a long piece
WIDE_LC = 64                           # chunk length of the whole-GPU form (kernels_chain.cuh kWideLc)
HEAD, TAIL = 64, 512
IR_LEN = 2 * TAIL + 3 * TAIL + 31


class Dev:
    """device buffers of the backend: numpy arrays on the emulation build, CUDA tensors on the GPU"""

    def __init__(self, l):
        self.gpu = backends._cache.get("emu") is not l

    def put(self, a):
        a = np.ascontiguousarray(a, np.float32)
        if self.gpu:
            import torch
            return torch.from_numpy(a.copy()).cuda()
        return a.copy()

    def ptr(self, b, off=0):
        if b is None:
            return 0
        return (b.data_ptr() if self.gpu else b.ctypes.data) + 4 * off

    def get(self, b):
        return b.cpu().numpy() if self.gpu else b.copy()


def _engine(l, C_, cfg, irs=None, max_batch_blocks=0):
    e = Engine(C_, lib=l, max_batch_blocks=max_batch_blocks)
    if irs is None:
        assert e.init_uniform(64, [ONE_TAP] * C_)
    else:
        assert e.init_twostage(HEAD, TAIL, irs)
    e.chain_configure(**cfg)
    return e


def _signals(n, seed, env=True):
    rng = np.random.default_rng(seed)
    L, R = orc.synth_input(n, seed), orc.synth_input(n, seed + 1)
    if not env:
        return L, R, None, None
    ysend = (0.5 + 0.5 * np.abs(np.sin(np.arange(n) * 1e-3))).astype(np.float32)
    yrev = (0.25 + 0.75 * rng.random(n)).astype(np.float32)
    return L, R, ysend, yrev


def _run(l, e, sig, sched, inplace=False, between=None):
    """sched: ("dev" | "host", length) calls; the device calls read / write one device buffer per signal at the call's
    offset.  between: {call index: f(engine)} run before that call.  Returns the [2, n] mix."""
    d = Dev(l)
    L, R, ys, yr = sig
    n = L.size
    X = d.put(np.stack([L, R]))
    O = X if inplace else d.put(np.zeros((2, n), np.float32))
    YS, YR = (d.put(a) if a is not None else None for a in (ys, yr))
    host = np.zeros((2, n), np.float32)
    on_dev = np.zeros(n, bool)
    pos = 0
    for k, (kind, m) in enumerate(sched):
        if between and k in between:
            e = between[k](e) or e
        sl = slice(pos, pos + m)
        if kind == "dev":
            e.chain_process_device(d.ptr(X, pos), n, d.ptr(O, pos), n, m, d.ptr(YS, pos), d.ptr(YR, pos), sync=True)
            on_dev[sl] = True
        else:
            a, b = e.chain_process(L[sl], R[sl], None if ys is None else ys[sl], None if yr is None else yr[sl])
            host[0, sl], host[1, sl] = a, b
        pos += m
    return np.where(on_dev, d.get(O), host)


def _cfg(srate=48000.0, lc=20.0, lcs=0, hc=20000.0, hcs=0, predelay=0, width=1.0, drygain=0.0, wetgain=1.0, ts=True):
    return dict(srate=srate, lowcut_hz=lc, lowcut_slope=lcs, highcut_hz=hc, highcut_slope=hcs, predelay=predelay,
                width=width, drygain=drygain, wetgain=wetgain, true_stereo=ts)


def _irs(nconv, seed):
    return [orc.synth_ir(IR_LEN, seed + c) * (1.0 + 0.25 * c) for c in range(nconv)]


# ---- 1. short pieces are the host path ------------------------------------------------------------------------------
SHORT = {
    "stereo-off-pd0-noenv": (2, _cfg(predelay=0, drygain=0.7, wetgain=0.5, width=0.3), False, False),
    "stereo-6-12-pd100": (2, _cfg(lc=180.0, lcs=0, hc=6000.0, hcs=1, predelay=100, drygain=0.8, wetgain=0.6, width=0.4),
                          True, True),
    "stereo-12-6-44k": (2, _cfg(44100.0, lc=400.0, lcs=1, hc=9000.0, hcs=0, predelay=50, width=1.7), True, False),
    "quad-ts-24-24-pd5000": (4, _cfg(lc=60.0, lcs=2, hc=12000.0, hcs=2, predelay=5000, drygain=0.5, wetgain=0.9,
                                     width=0.0), True, True),
    "quad-nots-6-24-pd0": (4, _cfg(lc=20.5, lcs=0, hc=16000.0, hcs=2, predelay=0, ts=False, drygain=1.0, width=1.0),
                           False, True),
}
SHORT_CALLS = [64, 1, 63, 128, 4096, 1000, 4096, 3000, 17, 4096, 2048]


@pytest.mark.parametrize("case", sorted(SHORT))
def test_short_pieces_are_the_host_call(lib, case):
    nconv, cfg, real_ir, env = SHORT[case]
    n = sum(SHORT_CALLS)
    sig = _signals(n, 3, env)
    irs = _irs(nconv, 10) if real_ir else None
    outs = []
    for kind in ("host", "dev"):
        e = _engine(lib, nconv, cfg, irs)
        outs.append(_run(lib, e, sig, [(kind, m) for m in SHORT_CALLS]))
        e.close()
    assert np.array_equal(outs[0], outs[1])


# ---- 2. long pieces against float64 ---------------------------------------------------------------------------------
def _long_engine(l, srate, cuts, predelay=0, calls_max=LONG + 8192):
    """_chain_engine's handle (IR [1], dry 0, wet 1, width 1: the mix is 0.5 * the filtered, delayed send) with a launch
    group that takes a whole long call as one piece"""
    return _engine(l, 2, _cfg(srate, predelay=predelay, **_short_cuts(cuts)), max_batch_blocks=calls_max // 64 + 2)


def _short_cuts(cuts):
    return dict(lc=cuts["lowcut_hz"], lcs=cuts["lowcut_slope"], hc=cuts["highcut_hz"], hcs=cuts["highcut_slope"])


def _run_f64(l, f64, srate, cuts, sched, updates=None, seed=5):
    """sched through the device and host entries against the serial float32 / float64 filters, state carried;
    updates: {call index: new cuts}"""
    n = sum(m for _, m in sched)
    x = _dc_noise(n, seed)
    e = _long_engine(l, srate, cuts)
    ref = F64Chain(f64, srate)
    ref.set(**cuts)
    between = {}
    for k, c in (updates or {}).items():
        between[k] = (lambda c: lambda e: e.chain_update(srate=srate, predelay=0, width=1.0, drygain=0.0, wetgain=1.0,
                                                        **c))(c)
    got = _run(l, e, (x[0], x[1], None, None), sched, between=between)
    e.close()
    r32, r64 = [[], []], [[], []]
    pos = 0
    for k, (_, m) in enumerate(sched):
        if updates and k in updates:
            ref.set(**updates[k])
        o32, o64 = ref.process([x[0][pos:pos + m], x[1][pos:pos + m]])
        for ch in range(2):
            r32[ch].append(o32[ch])
            r64[ch].append(o64[ch])
        pos += m
    for ch in range(2):
        _check(got[ch].astype(np.float64) * 2.0, np.concatenate(r32[ch]), np.concatenate(r64[ch]), (srate, cuts, ch))


LONG_SCHED = [("host", m) for m in RT_CALLS] + [("dev", LONG + 77)] + [("host", m) for m in RT_CALLS] + \
             [("dev", LONG)] + [("host", 4096)]


@pytest.mark.parametrize("srate", [44100.0, 96000.0, 192000.0])
@pytest.mark.parametrize("cuts", CHAIN_CUTS, ids=CHAIN_IDS)
def test_long_pieces_against_float64(lib, f64, cuts, srate):
    _run_f64(lib, f64, srate, cuts, LONG_SCHED)


# ---- 3. continuity across updates -----------------------------------------------------------------------------------
@pytest.mark.parametrize("srate", [48000.0, 96000.0])
def test_slope_switch_between_long_calls(lib, f64, srate):
    """6 -> 24 -> 6 dB at a 20.5 Hz low cut between long device calls: the stash exchange feeds the carry scan"""
    base = _cuts(20.5, 0, 20000.0, 0)
    sched = [("host", 128)] * 4 + [("dev", LONG)] + [("dev", LONG + 1000)] + [("host", 128)] * 4 + [("dev", LONG)] + \
            [("dev", 4096)]
    ups = {5: _cuts(20.5, 2, 20000.0, 0), 6: _cuts(20.5, 2, 40.0, 2), 10: _cuts(20.5, 0, 20000.0, 0)}
    _run_f64(lib, f64, srate, base, sched, updates=ups)


def test_predelay_growth_between_long_calls(lib, f64):
    """a predelay beyond the delay line (2 s) grows it: reads below the floor are zeros, later ones the delayed send"""
    sr, cuts, pd0, pd1 = 48000.0, _cuts(100.0, 1, 9000.0, 2), 3000, 100000
    sched = [("dev", LONG), ("host", 512), ("dev", LONG), ("dev", LONG + 333)]
    n = sum(m for _, m in sched)
    x = _dc_noise(n, 9)
    e = _long_engine(lib, sr, cuts, predelay=pd0)
    at = LONG + 512                          # the update before the third call: floor = its first sample
    grow = {2: lambda e: e.chain_update(srate=sr, predelay=pd1, width=1.0, drygain=0.0, wetgain=1.0, **cuts)}
    got = _run(lib, e, (x[0], x[1], None, None), sched, between=grow)
    e.close()
    ref = F64Chain(f64, sr)
    ref.set(**cuts)
    s32, s64 = ref.process(x)
    i = np.arange(n)
    for ch in range(2):
        want = []
        for s in (s32[ch], s64[ch]):
            w = np.zeros(n, np.float64)
            early = i < at
            w[early] = np.where(i[early] >= pd0, s[np.maximum(i[early] - pd0, 0)], 0.0)
            late = (i >= at) & (i - pd1 >= at)
            w[late] = s[i[late] - pd1]
            want.append(w)
        # below the floor: the convolver's FFT round-off of earlier blocks only
        assert float(np.max(np.abs(got[ch][(i >= at) & (i - pd1 < at)]))) <= 1e-6 * float(np.max(np.abs(want[1])))
        _check(got[ch].astype(np.float64) * 2.0, want[0], want[1], ("growth", ch))


# ---- 4. the full chain ----------------------------------------------------------------------------------------------
FULL = _cfg(48000.0, lc=20.5, lcs=1, hc=16000.0, hcs=2, predelay=2400, width=0.6, drygain=0.7, wetgain=0.8, ts=True)


def test_full_chain_long_calls(lib):
    """quad true stereo with a real IR, predelay, envelopes, width and dry / wet: device vs host entry on the same long
    calls; two device runs bit-identical; in place equal to out of place"""
    calls = [LONG + 100, 300, LONG]
    n = sum(calls)
    sig = _signals(n, 4)
    irs = _irs(4, 30)
    runs = {}
    for name, kind, inplace in (("host", "host", False), ("dev", "dev", False), ("dev2", "dev", False),
                                ("inplace", "dev", True)):
        e = _engine(lib, 4, FULL, irs, max_batch_blocks=(LONG + 8192) // 64 + 2)
        runs[name] = _run(lib, e, sig, [(kind, m) for m in calls], inplace=inplace)
        e.close()
    peak = float(np.max(np.abs(runs["host"])))
    assert float(np.max(np.abs(runs["dev"] - runs["host"]))) <= 1e-5 * peak
    assert np.array_equal(runs["dev"], runs["dev2"])
    assert np.array_equal(runs["dev"], runs["inplace"])


# ---- 5. hot swap over device calls ----------------------------------------------------------------------------------
def _swap_run(l, kind, post, irs_old, irs_new, cfg, sig, hb=128):
    """chain calls of `kind` through a swap (stereo -> quad) armed after 20 host blocks; returns (mix, the live
    handle's swap state after arming and after every later call)"""
    mb = (LONG + 8192) // 64 + 2
    live = _engine(l, 2, cfg, irs_old, max_batch_blocks=mb)
    inc = Engine(4, lib=l, max_batch_blocks=mb)
    assert inc.init_twostage(HEAD, TAIL, irs_new)
    pre = [hb] * 20
    first = live
    states = []
    out = []
    pos = 0
    for k, m in enumerate(pre + post):
        if k == len(pre):
            live.chain_swap(inc, hb)
            states.append(first.chain_swap_state())
        part = tuple(a[pos:pos + m] if a is not None else None for a in sig)
        out.append(_run(l, live, part, [(kind, m)]))
        if k >= len(pre):
            states.append(first.chain_swap_state())
            if live is first and first.chain_swap_state() == 3:
                live = inc                                   # std::swap(loadConvolver, convolver)
        pos += m
    first.close()
    inc.close()
    return np.concatenate(out, axis=1), states


@pytest.mark.parametrize("long", [False, True], ids=["short", "long"])
def test_hot_swap_over_device_calls(lib, long):
    cfg = _cfg(48000.0, lc=180.0, lcs=1, hc=6000.0, hcs=2, predelay=777, width=0.4, drygain=0.8, wetgain=0.6)
    post = [128, LONG] if long else [128] + [1024] * 4
    n = 20 * 128 + sum(post)
    sig = _signals(n, 6)
    irs_old, irs_new = _irs(2, 10), _irs(4, 20)
    host, st_h = _swap_run(lib, "host", post, irs_old, irs_new, cfg, sig)
    dev, st_d = _swap_run(lib, "dev", post, irs_old, irs_new, cfg, sig)
    assert st_d == st_h
    assert st_d[0] == 1 and st_d[1] == 2 and st_d[-1] == 3
    if long:
        peak = float(np.max(np.abs(host)))
        assert float(np.max(np.abs(dev - host))) <= 1e-5 * peak
    else:
        assert np.array_equal(dev, host)


# ---- 6. ragged lengths ----------------------------------------------------------------------------------------------
def test_ragged_lengths(lib, f64):
    """len 1; whole-GPU pieces whose last chunk is Lc - 1, 1 and Lc samples; calls one sample either side of the
    launch-group size (chunk = Lmax - B0), which leave a 1-sample piece after a long one"""
    sr, cuts = 96000.0, _cuts(20.5, 1, 40.0, 2)
    chunk = LONG
    sched = [("dev", 1), ("dev", LONG - 1), ("dev", LONG - WIDE_LC + 1), ("dev", LONG - WIDE_LC - 1), ("dev", 1),
             ("dev", chunk + 1), ("dev", chunk - 1), ("dev", LONG), ("host", 1)]
    n = sum(m for _, m in sched)
    x = _dc_noise(n, 11)
    e = _engine(lib, 2, _cfg(sr, **_short_cuts(cuts)), max_batch_blocks=chunk // 64 + 1)
    got = _run(lib, e, (x[0], x[1], None, None), sched)
    e.close()
    ref = F64Chain(f64, sr)
    ref.set(**cuts)
    r32, r64 = ref.process(x)
    for ch in range(2):
        _check(got[ch].astype(np.float64) * 2.0, r32[ch], r64[ch], ("ragged", ch))


# ---- 7. errors and async --------------------------------------------------------------------------------------------
def _raw(e, dry, out, n, sync=1):
    return e._l.b200conv_chain_process_device(e._h, dry, 8, None, None, out, 8, n, sync)


def test_errors(lib):
    d = Dev(lib)
    buf = d.put(np.zeros((2, 8), np.float32))
    p = d.ptr(buf)
    e = Engine(2, lib=lib)
    assert e.init_uniform(64, [ONE_TAP, ONE_TAP])
    assert _raw(e, p, p, 8) == ESTATE                      # no chain
    e.chain_configure(**_cfg())
    assert _raw(e, None, p, 8) == EINVAL
    assert _raw(e, p, None, 8) == EINVAL
    assert _raw(e, None, None, 0) == 0                     # len 0: nothing to do
    assert _raw(e, p, p, 8) == 0
    e.set_latency(64)
    assert _raw(e, p, p, 8) == ESTATE                      # fixed-latency handle
    e.close()


@pytest.mark.gpu
def test_async_equals_sync():
    import torch
    l = backends.get_lib("cuda")
    calls = [4096, LONG, 777]
    n = sum(calls)
    L, R, ys, yr = _signals(n, 8)
    outs = []
    for sync in (True, False):
        e = _engine(l, 4, FULL, _irs(4, 30), max_batch_blocks=(LONG + 8192) // 64 + 2)
        X = torch.from_numpy(np.stack([L, R])).cuda()
        YS, YR = torch.from_numpy(ys).cuda(), torch.from_numpy(yr).cuda()
        O = torch.zeros_like(X)
        torch.cuda.synchronize()
        pos = 0
        for m in calls:
            e.chain_process_device(X.data_ptr() + 4 * pos, n, O.data_ptr() + 4 * pos, n, m, YS.data_ptr() + 4 * pos,
                                   YR.data_ptr() + 4 * pos, sync=sync)
            pos += m
        if not sync:
            torch.cuda.ExternalStream(e.stream).synchronize()
        outs.append(O.cpu().numpy())
        e.close()
    assert np.array_equal(outs[0], outs[1])
