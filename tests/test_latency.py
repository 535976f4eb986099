"""Fixed-latency mode (b200conv_set_latency): the output of every entry point that supports it is the zero-latency
output delayed by exactly D samples, whatever the call lengths; refused states and entry points; the drop-in classes."""
import ctypes as C
import os
import time

import numpy as np
import pytest

from oracle import oracle as orc
from oracle.hotswap import HotSwapChain
from reevr_b200.convolver import B200ConvError, Engine
from tests.backends import get_lib, lib  # noqa: F401

TOL = 1e-5
ESTATE, EINVAL = -3, -1


def _irs(n, length, seed):
    return [orc.synth_ir(length, seed + c) * (1.0 + 0.25 * c) for c in range(n)]


def _make(lib, shape, irs, **kw):
    e = Engine(len(irs), lib=lib, **kw)
    if shape[0] == "uniform":
        assert e.init_uniform(shape[1], irs)
    else:
        assert e.init_twostage(shape[1], shape[2], irs)
    return e


def _ragged(B0, D, total):
    """call lengths that complete no block, one block, several blocks, and calls longer than D"""
    pat = [B0 // 3, B0 - B0 // 3, 1, 2 * B0 + 5, B0 - 6, 5 * D + 7, B0, 3]
    out, i = [], 0
    while sum(out) < total:
        out.append(min(pat[i % len(pat)], total - sum(out)))
        i += 1
    return out


def _feed(e, xs, calls):
    ys, pos = [[] for _ in range(len(e.process([x[:0] for x in xs])))], 0
    for m in calls:
        for c, y in enumerate(e.process([x[pos:pos + m] for x in xs])):
            ys[c].append(y)
        pos += m
    return [np.concatenate(y) for y in ys]


def _oracle(shape, irs, xs):
    out = []
    for ir, x in zip(irs, xs):
        o = orc.OracleUniform() if shape[0] == "uniform" else orc.OracleTwoStage()
        assert o.init(shape[1], ir) if shape[0] == "uniform" else o.init(shape[1], shape[2], ir)
        out.append(o.process(x))
    return out


def _check_shifted(got, want, D):
    """the first D samples exactly 0, the rest within TOL of peak of `want` shifted by D"""
    n = got.size
    assert np.all(got[:D] == 0.0)
    ref = want[:n - D]
    scale = max(np.max(np.abs(ref)), 1e-30)
    err = np.max(np.abs(got[D:] - ref)) / scale
    assert err <= TOL, err


# (id, shape, channels, IR taps, samples); the GPU adds REEV-R's quad 128 / 8192 with a 10 s IR
SHAPES = [
    ("uniform64", ("uniform", 64), 2, 3000, 9000),
    ("uniform512", ("uniform", 512), 1, 6000, 20000),
    ("twostage64-256-quad", ("twostage", 64, 256), 4, 3000, 9000),
]
GPU_SHAPES = [
    ("uniform512-long", ("uniform", 512), 2, 48000, 60000),
    ("twostage128-8192-quad-10s", ("twostage", 128, 8192), 4, 480000, 96000),
]


def _shifted_equality(lib, shape, nch, taps, n, mult):
    B0 = shape[1]
    D = mult * B0
    irs = _irs(nch, taps, 10)
    xs = [orc.synth_input(n, 40 + c) for c in range(nch)]
    e = _make(lib, shape, irs)
    e.set_latency(D)
    assert e.latency == D
    got = _feed(e, xs, _ragged(B0, D, n))
    want = _oracle(shape, irs, xs)
    for c in range(nch):
        _check_shifted(got[c], want[c], D)
    # calls of exactly B0: bitwise the zero-latency handle fed the same calls
    z, f = _make(lib, shape, irs), _make(lib, shape, irs)
    f.set_latency(D)
    calls = [B0] * (n // B0)
    yz, yf = _feed(z, xs, calls), _feed(f, xs, calls)
    for c in range(nch):
        assert np.all(yf[c][:D] == 0.0)
        assert np.array_equal(yf[c][D:], yz[c][:-D])


@pytest.mark.parametrize("mult", [1, 2, 4])
@pytest.mark.parametrize("case", SHAPES, ids=[s[0] for s in SHAPES])
def test_shifted_equality(lib, case, mult):
    _shifted_equality(lib, *case[1:], mult)


@pytest.mark.gpu
@pytest.mark.parametrize("mult", [1, 2, 4])
@pytest.mark.parametrize("case", GPU_SHAPES, ids=[s[0] for s in GPU_SHAPES])
def test_shifted_equality_long_irs_on_gpu(case, mult):
    _shifted_equality(get_lib("cuda"), *case[1:], mult)


@pytest.mark.parametrize("mult", [1, 4])
def test_calls_longer_than_one_pass(lib, mult):
    """max_batch_blocks = 8 makes a pass 8 head blocks (512 samples): calls of several passes, with the input slots
    reused within a call and output offsets carried across passes; process and chain"""
    B0, n = 64, 12000
    D = mult * B0
    shape = ("twostage", B0, 256)
    irs = _irs(2, 3000, 90)
    xs = [orc.synth_input(n, 95 + c) for c in range(2)]
    calls = _ragged(B0, D, 3000) + [4001, 37, 2 * 512 + 64] + _ragged(B0, D, n)
    calls = calls[:next(i for i in range(len(calls)) if sum(calls[:i + 1]) >= n) + 1]
    calls[-1] -= sum(calls) - n
    assert max(calls) > 4 * 512
    e = _make(lib, shape, irs, max_batch_blocks=8)
    e.set_latency(D)
    got = _feed(e, xs, calls)
    want = _oracle(shape, irs, xs)
    z = _make(lib, shape, irs, max_batch_blocks=8)
    yz = _feed(z, xs, [B0] * (n // B0))
    for c in range(2):
        _check_shifted(got[c], want[c], D)
        m = yz[c].size
        assert np.array_equal(got[c][D:m], yz[c][:m - D])
    # the chain through the same passes, against the zero-latency chain in head-block calls
    sig = _signals(n, 7)
    cz, cf = _make(lib, shape, irs, max_batch_blocks=8), _make(lib, shape, irs, max_batch_blocks=8)
    cz.chain_configure(**CFG)
    cf.chain_configure(**CFG)
    cf.set_latency(D)
    gz = _chain_run(cz, sig, [B0] * (n // B0), {})
    gf = _chain_run(cf, sig, calls, {})
    for c in range(2):
        assert np.all(gf[c][:D] == 0.0)
        m = gz[c].size
        assert np.array_equal(gf[c][D:m], gz[c][:m - D])


@pytest.mark.parametrize("mult", [1, 2])
def test_routing_quad_mixdown(lib, mult):
    B0, n = 64, 8000
    D = mult * B0
    irs = _irs(4, 3000, 20)
    L, R = orc.synth_input(n, 1), orc.synth_input(n, 2)
    mix = [[1, 0, 0, 1], [0, 1, 1, 0]]
    z, f, g = (_make(lib, ("twostage", B0, 256), irs) for _ in range(3))
    for e in (z, f, g):
        e.set_routing([0, 1, 0, 1], mix)
    f.set_latency(D)
    g.set_latency(D)
    calls = [B0] * (n // B0)
    yz, yf = _feed(z, [L, R], calls), _feed(f, [L, R], calls)
    yg = _feed(g, [L, R], _ragged(B0, D, n))
    for c in range(2):
        assert np.all(yf[c][:D] == 0.0)
        assert np.array_equal(yf[c][D:], yz[c][:-D])
        _check_shifted(yg[c][:yz[c].size], yz[c], D)


# ---- send / wet chain ---------------------------------------------------------------------------------------------
CFG = dict(srate=48000.0, lowcut_hz=180.0, lowcut_slope=1, highcut_hz=6000.0, highcut_slope=2, predelay=777,
           width=0.4, drygain=0.8, wetgain=0.6, true_stereo=True)
UPDATES = {   # input position (a multiple of the head block) -> chain_update arguments
    1024: dict(CFG, lowcut_hz=400.0, lowcut_slope=0),
    2560: dict(CFG, lowcut_hz=400.0, lowcut_slope=2, highcut_hz=9000.0, highcut_slope=1, predelay=100),
    4096: dict(CFG, lowcut_hz=60.0, lowcut_slope=2, highcut_hz=20000.0, predelay=1500, width=1.5),
}


def _signals(n, seed=0):
    rng = np.random.default_rng(seed)
    L, R = orc.synth_input(n, seed), orc.synth_input(n, seed + 1)
    ysend = (0.5 + 0.5 * np.abs(np.sin(np.arange(n) * 1e-3))).astype(np.float32)
    yrev = (0.25 + 0.75 * rng.random(n)).astype(np.float32)
    return L, R, ysend, yrev


def _split_at(calls, marks):
    """cuts the call lengths so that every mark is a call boundary"""
    out, pos = [], 0
    for m in calls:
        cuts = sorted(k - pos for k in marks if pos < k < pos + m)
        prev = 0
        for c in cuts + [m]:
            out.append(c - prev)
            prev = c
        pos += m
    return out


def _chain_run(e, sig, calls, updates, env=True):
    L, R, ys, yr = sig
    got, pos = [[], []], 0
    for m in calls:
        if pos in updates:
            e.chain_update(**updates[pos])
        sl = slice(pos, pos + m)
        a, b = e.chain_process(L[sl], R[sl], ys[sl] if env else None, yr[sl] if env else None)
        got[0].append(a)
        got[1].append(b)
        pos += m
    return [np.concatenate(g) for g in got]


@pytest.mark.parametrize("quad", [False, True])
@pytest.mark.parametrize("env", [True, False])
def test_chain_with_updates(lib, quad, env):
    B0, n = 64, 6000
    D = 2 * B0
    irs = _irs(4 if quad else 2, 3000, 30)
    sig = _signals(n, 5)
    z, f = _make(lib, ("twostage", B0, 256), irs), _make(lib, ("twostage", B0, 256), irs)
    z.chain_configure(**CFG)
    f.chain_configure(**CFG)
    f.set_latency(D)
    yz = _chain_run(z, sig, [B0] * (n // B0), UPDATES, env)
    yf = _chain_run(f, sig, _split_at(_ragged(B0, D, n), UPDATES), UPDATES, env)
    for c in range(2):
        assert np.all(yf[c][:D] == 0.0)
        assert np.array_equal(yf[c][D:yz[c].size], yz[c][:yz[c].size - D])


@pytest.mark.parametrize("n_old,n_new", [(2, 2), (2, 4), (4, 4)])
def test_chain_hot_swap_against_oracle(lib, n_old, n_new):
    """warm-up in the first step after arming, the fade counted per head-block step, the hand-over mid-call; against
    processBlock's restatement fed head-block callbacks, shifted by D"""
    B0, TAIL, D = 64, 512, 128
    ir_len = 5 * TAIL + 31
    cfg = dict(CFG, true_stereo=True)
    fade = int(np.ceil(cfg["srate"] * 50 / 1000.0))
    arm_at = 40 * B0
    n = arm_at + fade + ir_len + 4000
    n -= n % B0
    sig = _signals(n, 3)
    irs_old, irs_new = _irs(n_old, ir_len, 10), _irs(n_new, ir_len, 20)
    live, inc = _make(lib, ("twostage", B0, TAIL), irs_old), _make(lib, ("twostage", B0, TAIL), irs_new)
    live.chain_configure(**cfg)
    live.set_latency(D)
    with pytest.raises(B200ConvError):          # unequal latencies
        live.chain_swap(inc, B0)
    inc.set_latency(D)
    ora = HotSwapChain(**cfg)
    ora.set_live(B0, TAIL, irs_old)
    want, pos = [[], []], 0
    while pos < n:
        if pos == arm_at:
            ora.arm(B0, TAIL, irs_new, B0)
        a, b = ora.process(*[s[pos:pos + B0] for s in sig])
        want[0].append(a)
        want[1].append(b)
        pos += B0
    want = [np.concatenate(w) for w in want]
    calls = _split_at(_ragged(B0, D, n), [arm_at])
    got, pos, swapped = [[], []], 0, None
    for k, m in enumerate(calls):
        if pos == arm_at:
            live.chain_swap(inc, B0)
            assert live.chain_swap_state() == 1
        a, b = live.chain_process(*[s[pos:pos + m] for s in sig])
        got[0].append(a)
        got[1].append(b)
        pos += m
        if swapped is None and live.chain_swap_state() == 3:
            # the call that enqueued the step completing the fade
            assert pos >= arm_at + fade and pos - m < arm_at + fade + B0
            swapped = k
            live, inc = inc, live
    assert swapped is not None
    assert live.chain_swap_state() == 0 and inc.chain_swap_state() == 3
    for c in range(2):
        _check_shifted(np.concatenate(got[c]), want[c], D)


# ---- clear, reset, init ---------------------------------------------------------------------------------------------
def test_clear_reset_init(lib):
    B0, D, n = 64, 192, 5000
    irs = _irs(2, 3000, 50)
    xs = [orc.synth_input(n, 60 + c) for c in range(2)]
    e = _make(lib, ("twostage", B0, 256), irs)
    e.set_latency(D)
    e.process([x[:1234] for x in xs])
    e.clear()
    assert e.latency == D
    fresh = _make(lib, ("twostage", B0, 256), irs)
    fresh.set_latency(D)
    calls = _ragged(B0, D, n - 1234)
    rest = [x[1234:] for x in xs]
    got, want = _feed(e, rest, calls), _feed(fresh, rest, calls)
    for c in range(2):
        assert np.all(got[c][:D] == 0.0)
        assert np.array_equal(got[c], want[c])
    e.reset()
    assert e.latency == 0
    e2 = _make(lib, ("uniform", B0), irs)
    e2.set_latency(B0)
    assert e2.init_uniform(B0, irs) and e2.latency == 0


# ---- validation ---------------------------------------------------------------------------------------------------
def _rc(e, name, *args):
    return getattr(e._l, name)(e._h, *args)


def test_validation(lib):
    B0 = 64
    irs = _irs(2, 3000, 70)
    e = Engine(2, lib=lib)
    assert _rc(e, "b200conv_set_latency", B0) == ESTATE             # no IR
    assert e.init_twostage(B0, 256, irs)
    for bad in (B0 // 2, B0 + 1, 3 * B0 // 2, 17 * B0):
        assert _rc(e, "b200conv_set_latency", bad) == EINVAL, bad
        assert e.latency == 0
    e.set_latency(16 * B0)
    assert e.latency == 16 * B0 and e.latency_waits == 0
    x = np.zeros(4 * B0, np.float32)
    y = np.zeros(4 * B0, np.float32)
    ptrs = (C.c_void_p * 2)(x.ctypes.data, x.ctypes.data)
    outs = (C.c_void_p * 2)(y.ctypes.data, y.ctypes.data)
    assert _rc(e, "b200conv_process_device", x.ctypes.data, B0, y.ctypes.data, B0, B0, 1) == ESTATE
    assert _rc(e, "b200conv_process_device_sliced", x.ctypes.data, B0, y.ctypes.data, B0, B0, 0, 1, 1) == ESTATE
    assert _rc(e, "b200conv_process_sliced", ptrs, outs, B0, 0, 1) == ESTATE
    assert _rc(e, "b200conv_prime", ptrs, B0) == ESTATE
    other = _make(lib, ("twostage", B0, 256), irs)
    assert e._l.b200conv_process_xfade(other._h, e._h, ptrs, outs, B0, 0.0, 0.01) == ESTATE
    assert e._l.b200conv_process_xfade(e._h, other._h, ptrs, outs, B0, 0.0, 0.01) == ESTATE
    e.set_latency(0)
    assert e.latency == 0
    assert _rc(e, "b200conv_prime", ptrs, B0) == 0
    # a pending hot swap and a sharded handle
    live, inc = _make(lib, ("twostage", B0, 256), irs), _make(lib, ("twostage", B0, 256), irs)
    live.chain_configure(srate=48000.0)
    live.chain_swap(inc, B0)
    assert _rc(live, "b200conv_set_latency", B0) == ESTATE
    assert _rc(inc, "b200conv_set_latency", B0) == ESTATE
    sh = Engine(2, lib=lib, shard_rank=0, shard_count=2)
    assert sh.init_twostage(B0, 256, irs)
    assert _rc(sh, "b200conv_set_latency", B0) == ESTATE


# ---- on the H100 --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_launch_per_call_on_gpu():
    B0 = 128
    e = _make(get_lib("cuda"), ("uniform", B0), _irs(2, 24000, 80))
    e.set_latency(B0)
    xs = [orc.synth_input(B0, 90 + c) for c in range(2)]
    for _ in range(50):
        e.process(xs)
    for _ in range(200):
        n0 = e.launch_count
        e.process(xs)
        assert e.launch_count == n0 + 1


@pytest.mark.gpu
def test_no_waits_at_the_callback_pace_on_gpu():
    """REEV-R's quad two-stage 128 / 8192 with a 10 s IR, host block 128 at 48 kHz: 2000 calls with a full callback
    period (2.67 ms) of sleep after each.  No catch-up schedule: after a host stall the next call would follow its
    predecessor back to back and wait for a step enqueued microseconds earlier, which says nothing about the device."""
    B0 = 128
    period = B0 / 48000.0
    e = _make(get_lib("cuda"), ("twostage", B0, 8192), _irs(4, 480000, 100))
    e.set_routing([0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]])
    e.set_latency(B0)
    xs = [orc.synth_input(B0, 110 + c) for c in range(2)]
    for _ in range(200):
        e.process(xs)
        time.sleep(period)
    e.set_latency(B0)                            # resets the count
    for _ in range(2000):
        e.process(xs)
        time.sleep(period)
    assert e.latency_waits == 0


def _dropin(libpath, exe):
    from tests.test_cpp_dropin import _build_and_run
    _build_and_run(os.path.dirname(libpath), os.path.basename(libpath), exe,
                   src=os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "latency_dropin_test.cpp"))


def test_dropin_set_latency_on_emulation(tmp_path):
    from tests.emu.build_emu import build
    _dropin(build(), str(tmp_path / "latency_dropin_emu"))


@pytest.mark.gpu
def test_dropin_set_latency_on_gpu(tmp_path):
    from reevr_b200 import _lib
    _dropin(_lib.LIB_PATH, str(tmp_path / "latency_dropin_gpu"))
