"""Chain parameter changes while playing (b200conv_chain_update): new cut frequencies / slopes, predelay, width,
dry / wet and true stereo from the next call on, with the filter states and the delay history kept — against the
call-by-call restatement of processBlock's onSlider and per-block reads (oracle/params_oracle.c), whose filter re-init
is pinned against the reference's own Filter.cpp."""
import hashlib

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import params
from reevr_b200.convolver import B200ConvError, Engine
from tests.backends import lib  # noqa: F401
from tests.golden import make_filter_switch_pins as pins

TOL = 1e-5
ESTATE, EINVAL = -3, -1
HEAD, TAIL = 64, 512
IR_LEN = 2 * TAIL + 3 * TAIL + 31
LONG = 5000

# handle width, rate, call kind: every scenario covers stereo and quad, 48 and 44.1 kHz, real-time, ragged and long calls
COMBOS = [(2, 48000.0, "rt"), (4, 44100.0, "ragged"), (4, 48000.0, "long"), (2, 44100.0, "long")]
COMBO_IDS = ["st-48-rt", "quad-44-ragged", "quad-48-long", "st-44-long"]


def _cfg(srate, **kw):
    c = dict(srate=srate, lowcut_hz=180.0, lowcut_slope=1, highcut_hz=9000.0, highcut_slope=2, predelay=300,
             width=0.8, drygain=0.7, wetgain=0.6, true_stereo=True)
    c.update(kw)
    return c


def _call_len(kind, k):
    if kind == "ragged":
        return (100, 28, 61, 67)[k % 4]
    if kind == "long":
        return LONG if k % 10 == 9 else 128
    return 128


def _irs(nconv, seed):
    return [orc.synth_ir(IR_LEN, seed + c) * (1.0 + 0.25 * c) for c in range(nconv)]


class Rig:
    """The device chain and its oracle driven call by call with the same updates and swaps."""

    def __init__(self, lib, nconv, cfg, rt=True):
        self.lib, self.cfg, self.rt = lib, dict(cfg), rt
        self.live = self._engine(nconv, 10)
        self.live.chain_configure(**self.cfg)
        self.ora = params.ParamHotSwapChain(**self.cfg)
        self.ora.set_live(HEAD, TAIL, _irs(nconv, 10))
        self.inc = None
        self.got, self.want = [[], []], [[], []]
        self.pos, self.calls, self.swaps = 0, 0, 0
        n = 1 << 18
        rng = np.random.default_rng(int(cfg["srate"]) + nconv)
        self.L, self.R = orc.synth_input(n, 3), orc.synth_input(n, 4)
        self.ys = (0.5 + 0.5 * np.abs(np.sin(np.arange(n) * 1e-3))).astype(np.float32)
        self.yr = (0.25 + 0.75 * rng.random(n)).astype(np.float32)

    def _engine(self, nconv, seed):
        e = Engine(nconv, lib=self.lib)
        e.set_option("rt", int(self.rt))
        assert e.init_twostage(HEAD, TAIL, _irs(nconv, seed))
        return e

    def update(self, **changes):
        self.cfg.update(changes)
        self.live.chain_update(**self.cfg)
        self.ora.set(**self.cfg)

    def swap(self, nconv, host_block=128):
        self.inc = self._engine(nconv, 20 + 10 * self.swaps)
        self.live.chain_swap(self.inc, host_block)
        self.ora.arm(HEAD, TAIL, _irs(nconv, 20 + 10 * self.swaps), host_block)

    def call(self, m):
        sl = slice(self.pos % (self.L.size - LONG), self.pos % (self.L.size - LONG) + m)
        a, b = self.live.chain_process(self.L[sl], self.R[sl], self.ys[sl], self.yr[sl])
        c, d = self.ora.process(self.L[sl], self.R[sl], self.ys[sl], self.yr[sl])
        self.got[0].append(a); self.got[1].append(b); self.want[0].append(c); self.want[1].append(d)
        self.pos += m
        self.calls += 1
        if self.live.chain_swap_state() == 3:
            assert self.ora.swapped
            self.live, self.inc = self.inc, self.live          # std::swap(loadConvolver, convolver)
            self.swaps += 1
        else:
            assert not self.ora.swapped

    def check(self):
        gl, gr = np.concatenate(self.got[0]), np.concatenate(self.got[1])
        wl, wr = np.concatenate(self.want[0]), np.concatenate(self.want[1])
        scale = max(np.max(np.abs(wl)), np.max(np.abs(wr)))
        err = max(np.max(np.abs(gl - wl)), np.max(np.abs(gr - wr))) / scale
        assert err <= TOL, err


@pytest.mark.parametrize("combo", COMBOS, ids=COMBO_IDS)
def test_automation_ramp(lib, combo):
    """cut frequencies, width and dry / wet move on every callback"""
    nconv, sr, kind = combo
    rig = Rig(lib, nconv, _cfg(sr))
    for k in range(300):
        u = k / 299.0
        theta = u * np.pi / 2
        rig.update(lowcut_hz=30.0 + 770.0 * u, highcut_hz=15000.0 - 12000.0 * u, width=2.0 * u,
                   drygain=float(np.cos(theta)), wetgain=float(np.sin(theta)))
        rig.call(_call_len(kind, k))
    rig.check()


# (lowcut_hz, lowcut_slope, highcut_hz, highcut_slope): low cut 6 -> 12 -> 24 -> 6 dB, then off, 24 -> 6 (-> off) -> 12;
# high cut 24 -> 12 -> 6 dB, off, 24 -> 12, off, 6 -> 24 -> 6; 20 Hz and 20 kHz exactly are off (> 20, < 20000)
SLOPES = [(150.0, 0, 8000.0, 2), (150.0, 1, 8000.0, 2), (150.0, 2, 8000.0, 1), (150.0, 0, 8000.0, 0),
          (15.0, 0, 25000.0, 0), (300.0, 2, 6000.0, 2), (300.0, 0, 6000.0, 1), (20.0, 0, 20000.0, 1),
          (400.0, 1, 5000.0, 0), (400.0, 2, 5000.0, 2), (1000.0, 0, 3000.0, 0), (10.0, 1, 19999.0, 1)]


@pytest.mark.parametrize("combo", COMBOS, ids=COMBO_IDS)
def test_slope_switches_and_on_off(lib, combo):
    nconv, sr, kind = combo
    rig = Rig(lib, nconv, _cfg(sr, lowcut_hz=150.0, lowcut_slope=0, highcut_hz=8000.0, highcut_slope=2))
    for k in range(12 * len(SLOPES)):
        if k % 12 == 0:
            lc, lcs, hc, hcs = SLOPES[k // 12]
            rig.update(lowcut_hz=lc, lowcut_slope=lcs, highcut_hz=hc, highcut_slope=hcs)
        rig.call(_call_len(kind, k))
    rig.check()


@pytest.mark.parametrize("combo", COMBOS, ids=COMBO_IDS)
def test_predelay_changes_growth_and_swap_after_growth(lib, combo):
    """predelay up, down, to 0 and close to D - call length reads the history in the line; a predelay beyond D grows
    the line and clears its history (zeros), while the warmer survives: a swap right after the growth replays it"""
    nconv, sr, kind = combo
    D = int(2.0 * sr)
    big = D - LONG - 1
    rig = Rig(lib, nconv, _cfg(sr))
    plan = [(2000, 2000), (6000, 0), (9000, 777), (big + 4000, big), (big + 12000, 100)]
    k = 0
    for at, pd in plan:
        while rig.pos < at:
            rig.call(_call_len(kind, k)); k += 1
        rig.update(predelay=pd)
    for _ in range(20):
        rig.call(_call_len(kind, k)); k += 1
    assert rig.ora.delay_size == D
    rig.update(predelay=D + 500)                     # growth: D = 2 * predelay, the delay history reads zero
    assert rig.ora.delay_size == 2 * (D + 500)
    rig.call(_call_len(kind, k)); k += 1
    rig.swap(6 - nconv)
    start = rig.pos
    while rig.swaps == 0 or rig.pos < start + 4000 + IR_LEN:
        rig.call(_call_len(kind, k)); k += 1
    rig.update(predelay=300)                         # back below D: the history since the growth is there
    for _ in range(30):
        rig.call(_call_len(kind, k)); k += 1
    rig.check()


@pytest.mark.parametrize("combo", [c for c in COMBOS if c[0] == 4] + [(4, 44100.0, "rt")],
                         ids=[i for c, i in zip(COMBOS, COMBO_IDS) if c[0] == 4] + ["quad-44-rt"])
def test_true_stereo_toggle_outside_and_during_a_fade(lib, combo):
    _, sr, kind = combo
    rig = Rig(lib, 4, _cfg(sr))
    k = 0
    for k in range(60):
        if k % 20 == 10:
            rig.update(true_stereo=not rig.cfg["true_stereo"])
        rig.call(_call_len(kind, k))
    rig.swap(4)
    while rig.swaps == 0:
        rig.update(true_stereo=not rig.cfg["true_stereo"])
        rig.call(_call_len(kind, k)); k += 1
    for j in range(60):
        if j % 20 == 5:
            rig.update(true_stereo=not rig.cfg["true_stereo"])
        rig.call(_call_len(kind, k)); k += 1
    rig.check()


@pytest.mark.parametrize("combo", COMBOS, ids=COMBO_IDS)
def test_updates_during_a_swap(lib, combo):
    """between chain_swap and the warm-up call (the replay runs through the new filters), during the fade, in the
    completing call and on the new live handle after the hand-over"""
    nconv, sr, kind = combo
    rig = Rig(lib, nconv, _cfg(sr))
    fade = int(np.ceil(sr * 50 / 1000.0))
    k = 0
    for k in range(120):
        rig.call(_call_len(kind, k))
    rig.swap(6 - nconv)
    old, new = rig.live, rig.inc
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        new.chain_update(**rig.cfg)                      # the incoming handle owns no chain yet
    rig.update(lowcut_hz=400.0, lowcut_slope=2, highcut_hz=5000.0, highcut_slope=0, predelay=900)
    done = 0
    while rig.swaps == 0:
        m = _call_len(kind, k)
        if done + m >= fade:                             # the call that completes the fade
            rig.update(width=1.6, drygain=0.2, wetgain=0.9, highcut_slope=1, lowcut_hz=250.0)
        elif k % 3 == 0:
            rig.update(lowcut_hz=rig.cfg["lowcut_hz"] * 0.9, width=rig.cfg["width"] * 0.8, predelay=rig.cfg["predelay"] + 40)
        rig.call(m); k += 1
        done += m
    assert rig.live is new and old.chain_swap_state() == 3
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        old.chain_update(**rig.cfg)                      # gave its chain away
    for j in range(100):
        if j % 7 == 0:
            rig.update(lowcut_hz=100.0 + 13.0 * j, lowcut_slope=j % 3, width=0.3 + 0.01 * j, predelay=50 + 11 * j)
        rig.call(_call_len(kind, k)); k += 1
    rig.check()


def _pair(lib, nconv, cfg):
    a, b = Engine(nconv, lib=lib), Engine(nconv, lib=lib)
    for e in (a, b):
        assert e.init_twostage(HEAD, TAIL, _irs(nconv, 10))
        e.chain_configure(**cfg)
    return a, b


@pytest.mark.parametrize("nconv", [2, 4])
def test_same_configuration_is_bit_identical_and_launches_nothing(lib, nconv):
    cfg = _cfg(48000.0)
    a, b = _pair(lib, nconv, cfg)
    L, R = orc.synth_input(128 * 80, 0), orc.synth_input(128 * 80, 1)
    for k in range(80):
        sl = slice(k * 128, (k + 1) * 128)
        before = b.launch_count
        b.chain_update(**cfg)
        assert b.launch_count == before
        x, y = a.chain_process(L[sl], R[sl]), b.chain_process(L[sl], R[sl])
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
    before = b.launch_count
    b.chain_update(**_cfg(48000.0, lowcut_hz=500.0, lowcut_slope=0, width=0.1, predelay=4000))
    assert b.launch_count == before


def test_update_errors_change_nothing(lib):
    cfg = _cfg(44100.0)
    ref, e = _pair(lib, 2, cfg)
    bad = [dict(lowcut_slope=3), dict(highcut_slope=-1), dict(predelay=-1), dict(srate=48000.0)]
    L, R = orc.synth_input(128 * 40, 0), orc.synth_input(128 * 40, 1)
    for k in range(40):
        sl = slice(k * 128, (k + 1) * 128)
        if k < len(bad):
            with pytest.raises(B200ConvError, match=r"\(-1\)"):
                e.chain_update(**dict(cfg, **bad[k]))
        if k == len(bad):
            assert lib.b200conv_chain_update(e._h, None) == EINVAL
        x, y = ref.chain_process(L[sl], R[sl]), e.chain_process(L[sl], R[sl])
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
    fresh = Engine(2, lib=lib)
    assert fresh.init_twostage(HEAD, TAIL, _irs(2, 10))
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        fresh.chain_update(**cfg)                        # never configured
    # the incoming handle of a pending swap and the handle that gave its chain away: see test_updates_during_a_swap;
    # an error during a pending swap leaves the swap and the chain as they were
    inc = Engine(2, lib=lib)
    assert inc.init_twostage(HEAD, TAIL, _irs(2, 20))
    ref2, live = _pair(lib, 2, cfg)
    inc2 = Engine(2, lib=lib)
    assert inc2.init_twostage(HEAD, TAIL, _irs(2, 20))
    ref2.chain_swap(inc2, 128)
    live.chain_swap(inc, 128)
    assert lib.b200conv_chain_update(inc._h, None) == ESTATE
    with pytest.raises(B200ConvError, match=r"\(-1\)"):
        live.chain_update(**dict(cfg, predelay=-5))
    swapped = False
    for k in range(30):
        sl = slice(k * 128, (k + 1) * 128)
        x, y = ref2.chain_process(L[sl], R[sl]), live.chain_process(L[sl], R[sl])
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
        assert ref2.chain_swap_state() == live.chain_swap_state()
        if live.chain_swap_state() == 3:
            assert lib.b200conv_chain_update(live._h, None) == ESTATE       # gave its chain away
            ref2, live, swapped = inc2, inc, True
    assert swapped


def test_filter_switch_restatement_is_bit_identical_to_the_reference_filter():
    stored = iter(np.load(pins.PATH, allow_pickle=False)["sha256"])
    live = params.ref_switch_filter_available()
    for sr, mode, j, sched in pins.cases():
        a = pins.run(params.SwitchFilter, mode, sr, sched)
        assert hashlib.sha256(a.tobytes()).hexdigest() == next(stored), (sr, mode, j)
        if live:
            assert np.array_equal(a, pins.run(params.RefSwitchFilter, mode, sr, sched)), (sr, mode, j)
