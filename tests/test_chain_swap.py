"""IR hot swap inside the device chain (b200conv_chain_swap): warmer history, warm-up replay, 50 ms crossfade and the
hand-over of the chain, against the call-by-call restatement of processBlock (oracle/hotswap_oracle.c)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from oracle.hotswap import HotSwapChain
from reevr_b200.convolver import B200ConvError, Engine
from tests.backends import get_lib, lib  # noqa: F401

TOL = 1e-5
ESTATE, EINVAL = -3, -1
HEAD, TAIL = 64, 512
IR_LEN = 2 * TAIL + 3 * TAIL + 31

CFGS = {
    "neutral48": dict(srate=48000.0, lowcut_hz=20.0, lowcut_slope=0, highcut_hz=20000.0, highcut_slope=0, predelay=0,
                      width=1.0, drygain=1.0, wetgain=1.0, true_stereo=True),
    "f12_24_48": dict(srate=48000.0, lowcut_hz=180.0, lowcut_slope=1, highcut_hz=6000.0, highcut_slope=2, predelay=777,
                      width=0.4, drygain=0.8, wetgain=0.6, true_stereo=True),
    "f24_6_44": dict(srate=44100.0, lowcut_hz=60.0, lowcut_slope=2, highcut_hz=12000.0, highcut_slope=0, predelay=50,
                     width=1.7, drygain=0.0, wetgain=1.0, true_stereo=False),
    "f6_12_44": dict(srate=44100.0, lowcut_hz=400.0, lowcut_slope=0, highcut_hz=9000.0, highcut_slope=1, predelay=0,
                     width=0.0, drygain=0.5, wetgain=0.5, true_stereo=True),
}


def _irs(nconv, seed):
    return [orc.synth_ir(IR_LEN, seed + c) * (1.0 + 0.25 * c) for c in range(nconv)]


def _signals(n, seed=0):
    rng = np.random.default_rng(seed)
    L, R = orc.synth_input(n, seed), orc.synth_input(n, seed + 1)
    ysend = (0.5 + 0.5 * np.abs(np.sin(np.arange(n) * 1e-3))).astype(np.float32)
    yrev = (0.25 + 0.75 * rng.random(n)).astype(np.float32)
    return L, R, ysend, yrev


def _calls(kind, host_block, total):
    """call lengths of a host: real-time calls, ragged pairs around the host block, or real-time calls with one long
    call where the swap is armed"""
    out = []
    while sum(out) < total:
        if kind == "ragged":
            out += [host_block - 28, 28] if len(out) % 4 == 0 else [host_block // 2 + 3, host_block - host_block // 2 - 3]
        else:
            out.append(host_block)
    return out


def _run(lib, cfg, n_old, n_new, host_block, kind, arm_after, after=IR_LEN + 1500, rt=True):
    """Device chain through a swap old -> new, against the oracle; returns (device states per call, oracle swap call)."""
    fade = int(np.ceil(cfg["srate"] * 50 / 1000.0))
    pre = _calls("rt" if kind == "long" else kind, host_block, arm_after)
    post = [max(4096, fade + 300)] if kind == "long" else []
    post += _calls("rt" if kind == "long" else kind, host_block, fade + after)
    calls = pre + post
    n = sum(calls)
    L, R, ys, yr = _signals(n, 3)
    irs_old, irs_new = _irs(n_old, 10), _irs(n_new, 20)
    live, inc = Engine(n_old, lib=lib), Engine(n_new, lib=lib)
    for e in (live, inc):
        e.set_option("rt", int(rt))
    assert live.init_twostage(HEAD, TAIL, irs_old) and inc.init_twostage(HEAD, TAIL, irs_new)
    live.chain_configure(**cfg)
    ora = HotSwapChain(**cfg)
    ora.set_live(HEAD, TAIL, irs_old)
    got, want, pos = [[], []], [[], []], 0
    states, swap_call, ora_swap_call = [], None, None
    for k, m in enumerate(calls):
        if k == len(pre):
            live.chain_swap(inc, host_block)
            assert live.chain_swap_state() == 1 and inc.chain_swap_state() == 1
            ora.arm(HEAD, TAIL, irs_new, host_block)
        sl = slice(pos, pos + m)
        a, b = live.chain_process(L[sl], R[sl], ys[sl], yr[sl])
        c, d = ora.process(L[sl], R[sl], ys[sl], yr[sl])
        got[0].append(a); got[1].append(b); want[0].append(c); want[1].append(d)
        if ora.swapped:
            ora_swap_call = k
        if k >= len(pre) and swap_call is None:
            states.append((live.chain_swap_state(), inc.chain_swap_state()))
            if live.chain_swap_state() == 3:
                swap_call = k
                live, inc = inc, live              # std::swap(loadConvolver, convolver)
        pos += m
    gl, gr = np.concatenate(got[0]), np.concatenate(got[1])
    wl, wr = np.concatenate(want[0]), np.concatenate(want[1])
    scale = max(np.max(np.abs(wl)), np.max(np.abs(wr)))
    err = max(np.max(np.abs(gl - wl)), np.max(np.abs(gr - wr))) / scale
    assert err <= TOL, err
    assert swap_call is not None and swap_call == ora_swap_call, (swap_call, ora_swap_call)
    # the completing call is the first whose samples reach the fade length; at least one IR length follows it
    lens = np.cumsum(calls[len(pre):])
    assert swap_call - len(pre) == int(np.argmax(lens >= fade))
    assert sum(calls[swap_call + 1:]) >= IR_LEN
    assert live.chain_swap_state() == 0 and inc.chain_swap_state() == 3
    return states, calls, pre


CASES = [
    # id, cfg, n_old, n_new, host_block, call kind, samples before the swap is armed
    ("st-st-rt-wrapped", "neutral48", 2, 2, 128, "rt", 20000),
    ("quad-ts-ragged-early", "f12_24_48", 4, 4, 256, "ragged", 5000),
    ("quad-nots-rt-wrapped", "f24_6_44", 4, 4, 128, "rt", 15000),
    ("st-quad-long", "f6_12_44", 2, 4, 256, "long", 14000),
    ("quad-st-Wdiv", "f12_24_48", 4, 2, 96, "rt", 13000),          # W = 12000 = 125 * 96
    ("quad-ts-st-ragged-44", "f6_12_44", 4, 2, 128, "ragged", 3000),
    ("st-st-filters-long-early", "f24_6_44", 2, 2, 128, "long", 2000),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_chain_swap_against_oracle(lib, case):
    _, cfg, n_old, n_new, hb, kind, arm_after = case
    states, calls, pre = _run(lib, CFGS[cfg], n_old, n_new, hb, kind, arm_after)
    assert states[-1] == (3, 0) and all(s == (2, 2) for s in states[:-1])     # fading after the warm-up call
    if kind == "long":
        assert len(states) == 1                     # warm-up, the whole fade and the hand-over in one call


@pytest.mark.gpu
@pytest.mark.parametrize("rt", [1, 0])
def test_chain_swap_both_realtime_paths(rt):
    _run(get_lib("cuda"), CFGS["f12_24_48"], 4, 4, 128, "rt", 14000, rt=bool(rt))


def test_chain_swap_double_buffering(lib):
    """A -> B, then A re-initialised as the next incoming handle, then B -> A: both swaps against the oracle"""
    cfg = CFGS["f12_24_48"]
    irs = [_irs(2, 10), _irs(4, 20), _irs(2, 30)]
    hb = 128
    fade = int(np.ceil(cfg["srate"] * 0.05))
    calls = [hb] * 300
    L, R, ys, yr = _signals(sum(calls), 5)
    A, B = Engine(2, lib=lib), Engine(4, lib=lib)
    assert A.init_twostage(HEAD, TAIL, irs[0]) and B.init_twostage(HEAD, TAIL, irs[1])
    A.chain_configure(**cfg)
    ora = HotSwapChain(**cfg)
    ora.set_live(HEAD, TAIL, irs[0])
    live, spare = A, B
    arm_at = {60: 1, 60 + fade // hb + 40: 2}
    got, want = [[], []], [[], []]
    swaps = 0
    for k, m in enumerate(calls):
        if k in arm_at:
            which = arm_at[k]
            if which == 2:                          # the handle that gave its chain away is loaded with the next IR
                assert spare.chain_swap_state() == 3
                assert spare.init_twostage(HEAD, TAIL, irs[2])
                assert spare.chain_swap_state() == 0
            live.chain_swap(spare, hb)
            ora.arm(HEAD, TAIL, irs[which], hb)
        sl = slice(k * hb, (k + 1) * hb)
        a, b = live.chain_process(L[sl], R[sl], ys[sl], yr[sl])
        c, d = ora.process(L[sl], R[sl], ys[sl], yr[sl])
        got[0].append(a); got[1].append(b); want[0].append(c); want[1].append(d)
        if live.chain_swap_state() == 3:
            assert ora.swapped
            live, spare = spare, live
            swaps += 1
    assert swaps == 2 and live is A
    gl, gr = np.concatenate(got[0]), np.concatenate(got[1])
    wl, wr = np.concatenate(want[0]), np.concatenate(want[1])
    scale = max(np.max(np.abs(wl)), np.max(np.abs(wr)))
    assert max(np.max(np.abs(gl - wl)), np.max(np.abs(gr - wr))) <= TOL * scale


def test_chain_swap_warm_up_launches_do_not_grow_with_the_block_count(lib):
    """the replay of numBlocks host blocks is ONE batched call: same launch count for host blocks 64 and 512"""
    cfg = CFGS["f12_24_48"]
    counts = []
    for hb in (64, 512):
        L, R, ys, yr = _signals(128 * 120, 1)
        live, inc = Engine(4, lib=lib), Engine(4, lib=lib)
        assert live.init_twostage(HEAD, TAIL, _irs(4, 10)) and inc.init_twostage(HEAD, TAIL, _irs(4, 20))
        live.chain_configure(**cfg)
        for k in range(110):
            live.chain_process(L[k * 128:(k + 1) * 128], R[k * 128:(k + 1) * 128], ys[:128], yr[:128])
        live.chain_swap(inc, hb)
        before = live.launch_count + inc.launch_count
        live.chain_process(L[-128:], R[-128:], ys[:128], yr[:128])
        counts.append(live.launch_count + inc.launch_count - before)
        assert live.chain_swap_state() == 2
    assert counts[0] == counts[1], counts


def _rc(lib, live, inc, hb=128):
    return lib.b200conv_chain_swap(live._h, inc._h, hb)


def test_chain_swap_errors_and_cancellation(lib):
    cfg = CFGS["neutral48"]
    irs2, irs4 = _irs(2, 10), _irs(4, 20)

    def handle(nconv=2, chain=False, head=HEAD, **kw):
        e = Engine(nconv, lib=lib, **kw)
        assert e.init_twostage(head, TAIL, irs2 if nconv == 2 else irs4)
        if chain:
            e.chain_configure(**cfg)
        return e

    a, b = handle(), handle()
    assert _rc(lib, a, b) == ESTATE                                   # live has no chain
    a.chain_configure(**cfg)
    empty = Engine(2, lib=lib)
    assert _rc(lib, a, empty) == ESTATE                               # incoming has no IR
    assert _rc(lib, a, handle(chain=True)) == ESTATE                  # incoming already owns a chain
    assert _rc(lib, a, a) == EINVAL                                   # same handle twice
    assert _rc(lib, a, b, hb=0) == EINVAL                             # host_block 0
    assert _rc(lib, a, handle(head=32)) == EINVAL                     # unequal staging sizes
    routed = handle()
    routed.set_routing([0, 1], [[1, 0], [0, 1]])
    assert _rc(lib, a, routed) == EINVAL                              # routed
    assert _rc(lib, a, handle(shard_count=2)) == EINVAL               # sharded
    emu = get_lib("emu")                                              # (one device is enough for the emulation)
    if lib is emu:
        assert _rc(lib, a, handle(device=1)) == EINVAL                # different devices
    assert a.chain_swap_state() == 0 and b.chain_swap_state() == 0
    # pending: a second swap, configure on either handle, init on either handle
    assert _rc(lib, a, b) == 0
    c = handle()
    assert _rc(lib, a, c) == ESTATE and _rc(lib, c, b) == ESTATE
    for e in (a, b):
        with pytest.raises(B200ConvError, match=r"\(-3\)"):
            e.chain_configure(**cfg)
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        b.init_twostage(HEAD, TAIL, irs2)
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        b.init_twostage_recalc(HEAD, TAIL, irs2)
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        b.chain_process(np.zeros(128), np.zeros(128))                 # the incoming handle has no chain yet
    # cancellation by reset of the incoming handle: the live one continues alone, exactly like a chain without a swap
    L, R, ys, yr = _signals(128 * 40, 2)
    ref = handle(chain=True)
    want = [ref.chain_process(L[k * 128:(k + 1) * 128], R[k * 128:(k + 1) * 128]) for k in range(40)]
    b.reset()
    assert a.chain_swap_state() == 0 and b.chain_swap_state() == 0
    got = [a.chain_process(L[k * 128:(k + 1) * 128], R[k * 128:(k + 1) * 128]) for k in range(40)]
    assert all(np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]) for g, w in zip(got, want))
    # cancellation by destroying the incoming handle in the middle of the fade
    assert b.init_twostage(HEAD, TAIL, irs2)
    a.chain_swap(b, 128)
    a.chain_process(L[:128], R[:128])
    assert a.chain_swap_state() == 2
    b.close()
    assert a.chain_swap_state() == 0
    a.chain_process(L[:128], R[:128])
    # cancellation by destroying / resetting the live handle: the incoming one is free again
    d, e = handle(chain=True), handle()
    d.chain_swap(e, 128)
    d.close()
    assert e.chain_swap_state() == 0
    e.chain_configure(**cfg)
    e.chain_process(L[:128], R[:128])
    f = handle()
    e.chain_swap(f, 128)
    e.reset()
    assert f.chain_swap_state() == 0 and e.chain_swap_state() == 0
    assert f.init_twostage(HEAD, TAIL, irs2)
    # clear(live) during the fade: the chain's history starts over, the incoming handle is untouched, the fade goes on
    g, h = handle(chain=True), handle()
    g.chain_swap(h, 128)
    g.chain_process(L[:128], R[:128])
    g.clear()
    assert g.chain_swap_state() == 2 and h.chain_swap_state() == 2
    for k in range(30):
        g.chain_process(L[k * 128:(k + 1) * 128], R[k * 128:(k + 1) * 128])
        if g.chain_swap_state() == 3:
            break
    assert g.chain_swap_state() == 3 and h.chain_swap_state() == 0
    h.chain_process(L[:128], R[:128])


def test_chain_swap_kernels_do_not_spill():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reevr_b200", "csrc", "kernels_chain.cuh")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        cu = os.path.join(d, "k.cu")
        with open(cu, "w") as f:
            f.write(f'#include "{src}"\n'
                    "void launch(pc::ChainSendParams s, pc::ChainWetParams w) {\n"
                    "  pc::k_chain_send<<<2, 64>>>(s); pc::k_chain_wet<<<1, 256>>>(w); pc::k_chain_wet_xfade<<<1, 256>>>(w); }\n")
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-std=c++17", "-c", cu,
                              "-o", os.path.join(d, "k.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    log = out.stdout + out.stderr
    # the warm-up replay is a mode of k_chain_send, whose stack frame (the filter cascade's state arrays) it leaves as it was
    for name in ("k_chain_wet_xfade",):
        blk = re.search(r"Compiling entry function '[^']*" + name + r"[^']*'.*?Used \d+ registers", log, re.S)
        assert blk, name
        spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk.group(0))
        assert spills and all(s == ("0", "0") for s in spills), (name, spills)
