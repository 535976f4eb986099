"""Send / wet chain calls of a group (b200conv_chain_group_process): the qualifying members' chain calls as one send
launch, one k_rt_group launch per shape class and one wet launch, with one wait on the group's completion word.  Every
member has a twin built by the same recipe and driven by b200conv_chain_process with the same call lengths, envelopes
and parameter changes: on the CPU emulation the group's outputs equal the twins' bit for bit, on the H100 to the
tolerance of tests/test_group.py (1e-6 absolute up to 1, 1e-6 of peak above), and both stay within 1e-5 of peak of the
float64 oracle chain (oracle chain + oracle two-stage convolvers)."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import B200ConvError, Engine, Group
from tests.backends import get_lib
from tests.test_chain import _reference_chain
from tests.test_conv_precision import rt_cluster_ctas
from tests.test_group import TWIN_TOL, irs_for, twostage, uniform
from tests.test_rt_cross import variable_calls

BACKENDS = ["emu", pytest.param("cuda", marks=pytest.mark.gpu)]
TOL = 1e-5
EINVAL, ESTATE = -1, -3

CFGS = [
    dict(srate=48000.0, lowcut_hz=180.0, lowcut_slope=1, highcut_hz=6000.0, highcut_slope=2, predelay=777,
         width=0.4, drygain=0.8, wetgain=0.6, true_stereo=True),
    dict(srate=48000.0, lowcut_hz=60.0, lowcut_slope=2, highcut_hz=12000.0, highcut_slope=0, predelay=50,
         width=1.7, drygain=0.0, wetgain=1.0, true_stereo=False),
    dict(srate=48000.0, lowcut_hz=400.0, lowcut_slope=0, highcut_hz=20000.0, highcut_slope=1, predelay=4000,
         width=0.0, drygain=0.5, wetgain=0.5, true_stereo=True),
    dict(srate=48000.0, lowcut_hz=20.0, lowcut_slope=0, highcut_hz=20000.0, highcut_slope=0, predelay=0,
         width=1.0, drygain=1.0, wetgain=1.0, true_stereo=True),
]


class ChainMember:
    """a chained member and its twin, built by the same recipe; ysend / yrev None: the envelope is 1 (NULL)"""

    def __init__(self, lib, nch, setup, irs, cfg, n, seed, send=True, rev=True, latency=0):
        self.lib, self.nch, self.setup, self.irs, self.cfg, self.latency = lib, nch, setup, irs, cfg, latency
        rng = np.random.default_rng(seed)
        self.L, self.R = orc.synth_input(n, 100 * seed), orc.synth_input(n, 100 * seed + 1)
        self.ysend = (0.5 + 0.5 * np.abs(np.sin(np.arange(n) * 1e-3 * (seed + 1)))).astype(np.float32) if send else None
        self.yrev = (0.25 + 0.75 * rng.random(n)).astype(np.float32) if rev else None
        self.h, self.twin = self.make(), self.make()
        self.got, self.want, self.calls = [], [], []
        self.pos = 0

    def make(self, chain=True):
        e = Engine(self.nch, lib=self.lib)
        self.setup(e, self.irs)
        if self.latency:
            e.set_latency(self.latency)
        if chain:
            e.chain_configure(**self.cfg)
        return e

    def take(self, k):
        """the member's next k samples: (dry L, dry R), ysend, yrev"""
        s = slice(self.pos, self.pos + k)
        self.pos += k
        self.calls.append(k)
        env = [None if e is None else e[s] for e in (self.ysend, self.yrev)]
        return (self.L[s], self.R[s]), env[0], env[1]

    def single(self, k):
        """one call of the member's own b200conv_chain_process next to the twin's"""
        d, ys, yr = self.take(k)
        self.record(self.h.chain_process(*d, ys, yr), self.twin.chain_process(*d, ys, yr))

    def record(self, got, want):
        self.got.append(got)
        self.want.append(want)

    def outputs(self):
        return ([np.concatenate([g[c] for g in self.got]) for c in range(2)],
                [np.concatenate([w[c] for w in self.want]) for c in range(2)])

    def oracle(self, head, tail):
        n = self.pos
        ones = np.ones(n, np.float32)
        return _reference_chain(self.cfg, self.irs, head, tail, self.L[:n], self.R[:n],
                                ones if self.ysend is None else self.ysend[:n],
                                ones if self.yrev is None else self.yrev[:n], self.calls)


def group_call(g, ms, k):
    ins = [m.take(k) for m in ms]
    ys = g.chain_process([x[0] for x in ins], [x[1] for x in ins], [x[2] for x in ins])
    for m, x, y in zip(ms, ins, ys):
        m.record(y, m.twin.chain_process(*x[0], x[1], x[2]))


def check_twins(ms, backend, oracle=None):
    """oracle: (head, tail) of the members' two-stage convolvers, to check against the float64 chain as well"""
    for m in ms:
        got, want = m.outputs()
        for a, b in zip(got, want):
            if backend == "emu":
                assert np.array_equal(a, b)
            else:
                assert float(np.max(np.abs(a - b))) <= TWIN_TOL[backend] * max(1.0, float(np.max(np.abs(b))))
        if oracle:
            ref = m.oracle(*oracle)
            scale = max(float(np.max(np.abs(r))) for r in ref)
            for a, r in zip(got, ref):
                assert float(np.max(np.abs(a - r))) <= TOL * scale


def close(g, ms):
    g.close()
    for m in ms:
        m.h.close()
        m.twin.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_four_quads(backend):
    """4 quad two-stage members with different filters, predelays, widths, gains and true stereo on / off, envelopes
    per sample or NULL: three launches per call; the members count launches only when a tail block completes"""
    lib = get_lib(backend)
    head, tail, L = (16, 256, 3000) if backend == "emu" else (128, 8192, 480000)
    calls = [head] * 200
    n = sum(calls)
    ms = [ChainMember(lib, 4, twostage(head, tail), irs_for(4, L, i), CFGS[i], n, i, send=i != 1, rev=i != 2)
          for i in range(4)]
    g = Group([m.h for m in ms])
    pos, tails = 0, 0
    for k in calls:
        g0, m0 = g.launch_count, [m.h.launch_count for m in ms]
        group_call(g, ms, k)
        assert g.launch_count - g0 == 3
        if (pos + k) // tail > pos // tail:
            tails += 1
            assert all(m.h.launch_count > c for m, c in zip(ms, m0))
        else:
            assert [m.h.launch_count for m in ms] == m0
        pos += k
    assert tails >= 2
    check_twins(ms, backend, (head, tail))
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_crossing_calls(backend):
    """host block 480 on head 512 (30 on 32 on the emulation), then seeded lengths in [1, head]: two stereo members and
    a quad, one send, one wet and one cluster launch per shape class"""
    lib = get_lib(backend)
    emu = backend == "emu"
    M, T, L = (32, 256, 3000) if emu else (512, 8192, 100000)
    calls = [M - M // 16] * 40 + variable_calls((1 if emu else 4) * T, 1, M, 31)
    n = sum(calls)
    ms = [ChainMember(lib, nch, twostage(M, T), irs_for(nch, L, i), CFGS[i], n, i)
          for i, nch in enumerate([2, 2, 4])]
    classes = {(m.nch, rt_cluster_ctas(M, m.nch, int(m.h.stages()[0]["partitions"]))) for m in ms}
    assert all(w > 0 for _, w in classes)
    g = Group([m.h for m in ms])
    for k in calls:
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == 2 + len(classes)
    check_twins(ms, backend, (M, T))
    close(g, ms)


def swap_through(g, i, m, incoming):
    """member i's pending hot swap has completed: the group and the twin go on with the incoming handles; returns the
    outgoing pair"""
    assert m.h.chain_swap_state() == 3 and m.twin.chain_swap_state() == 3
    g.set_member(i, incoming[0])
    out = (m.h, m.twin)
    m.h, m.twin = incoming
    return out


@pytest.mark.parametrize("backend", BACKENDS)
def test_mixed_group(backend):
    """two shape classes (stereo and quad members: four launches per call) next to members that run alone: a split-mode
    uniform member, a fixed-latency member and a member with a pending hot swap; and one call longer than the head
    block, which no member shares.  The swapping member's incoming handle takes its place once the swap completes."""
    lib = get_lib(backend)
    emu = backend == "emu"
    head, tail, L = (32, 256, 3000) if emu else (128, 8192, 100000)
    calls = variable_calls(12 * tail // 4, 1, head, 41)
    calls = calls[:len(calls) // 2] + [3 * head + 5] + calls[len(calls) // 2:]
    n = sum(calls)
    ms = [ChainMember(lib, 4, twostage(head, tail), irs_for(4, L, 0), CFGS[0], n, 0),
          ChainMember(lib, 2, twostage(head, tail), irs_for(2, L, 1), CFGS[1], n, 1),
          ChainMember(lib, 2, uniform(256), irs_for(2, 256 * 1100 - 9, 2), CFGS[2], n, 2),       # split mode
          ChainMember(lib, 2, twostage(head, tail), irs_for(2, L, 3), CFGS[3], n, 3, latency=head),
          ChainMember(lib, 2, twostage(head, tail), irs_for(2, L, 4), CFGS[1], n, 4)]
    assert rt_cluster_ctas(256, 2, int(ms[2].h.stages()[0]["partitions"])) == -1
    swapper = ms[4]
    new_irs = irs_for(2, L // 2, 7)
    incoming = []
    for e in (swapper.h, swapper.twin):
        x = Engine(2, lib=lib)
        assert x.init_twostage(head, tail, new_irs)
        e.chain_swap(x, head)
        incoming.append(x)
    g = Group([m.h for m in ms])
    outgoing = ()
    for k in calls:
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == (4 if k <= head else 0)
        if not outgoing and swapper.h.chain_swap_state() == 3:
            outgoing = swap_through(g, 4, swapper, incoming)
    assert bool(outgoing) == (not emu)             # the emulation's calls end before the 50 ms fade does
    check_twins(ms, backend)
    check_twins(ms[:2], backend, (head, tail))
    close(g, ms)
    for e in outgoing:
        e.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_chain_updates_between_group_calls(backend):
    """b200conv_chain_update on some members between group calls: 6 <-> 12 / 24 dB slope switches, a filter switched off
    and on again, width / gain / true-stereo changes and a predelay that grows past the delay line"""
    lib = get_lib(backend)
    emu = backend == "emu"
    head, tail, L = (16, 256, 3000) if emu else (128, 8192, 100000)
    calls = variable_calls(8 * tail, 1, head, 5)
    n = sum(calls)
    ms = [ChainMember(lib, 4 if i % 2 else 2, twostage(head, tail), irs_for(4 if i % 2 else 2, L, i), CFGS[i], n, i)
          for i in range(3)]
    updates = [
        (0, dict(CFGS[0], lowcut_slope=0, highcut_slope=0)),               # 12 / 24 dB -> 6 dB
        (1, dict(CFGS[1], lowcut_hz=20.0, true_stereo=True, width=0.7)),  # low cut off
        (0, dict(CFGS[0], lowcut_slope=2, highcut_slope=1)),               # 6 dB -> 24 / 12 dB
        (2, dict(CFGS[2], predelay=2 * 48000 + 1234)),                     # beyond D = 2 * srate: the line grows
        (1, dict(CFGS[1], lowcut_hz=90.0, lowcut_slope=0, drygain=0.3)),   # low cut back on, at 6 dB
        (2, dict(CFGS[2], lowcut_slope=1, highcut_hz=20000.0, wetgain=0.9)),
    ]
    every = len(calls) // (len(updates) + 1)
    g = Group([m.h for m in ms])
    for j, k in enumerate(calls):
        if j and j % every == 0 and j // every <= len(updates):
            i, cfg = updates[j // every - 1]
            for e in (ms[i].h, ms[i].twin):
                e.chain_update(**cfg)
        group_call(g, ms, k)
    check_twins(ms, backend)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_hot_swap_inside_a_group(backend):
    """chain_swap armed on one member: it runs alone until the swap completes (state 3); then a group call refuses the
    outgoing handle, which owns no chain any more, and set_member puts the incoming handle in its place"""
    lib = get_lib(backend)
    emu = backend == "emu"
    head, tail, L = (16, 256, 3000) if emu else (128, 8192, 100000)
    calls = variable_calls(3 * 2400 + 4 * tail, 1, head, 17)
    n = sum(calls)
    ms = [ChainMember(lib, 4, twostage(head, tail), irs_for(4, L, i), CFGS[i], n, i) for i in range(3)]
    new_irs = irs_for(4, L // 2, 8)
    incoming = []
    for e in (ms[1].h, ms[1].twin):
        x = Engine(4, lib=lib)
        assert x.init_twostage(head, tail, new_irs)
        incoming.append(x)
    g = Group([m.h for m in ms])
    for j, k in enumerate(calls):
        if j == 20:
            for e, x in zip((ms[1].h, ms[1].twin), incoming):
                e.chain_swap(x, head)
        if ms[1].h.chain_swap_state() == 3:
            g0 = g.launch_count
            with pytest.raises(B200ConvError, match="member 1 owns no send / wet chain"):
                g.chain_process([(np.zeros(k, np.float32),) * 2] * 3)
            assert g.launch_count == g0
            for e in swap_through(g, 1, ms[1], incoming):
                e.close()
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == 3        # the swapping member runs alone, the other two share the launches
    assert ms[1].h is incoming[0]
    check_twins(ms, backend)
    close(g, ms)


def _device_chain_call(e, d, ys, yr, sync):
    """b200conv_chain_process_device of one call on torch buffers; returns a function that yields (L, R) once the call
    has completed"""
    import torch
    x = torch.from_numpy(np.ascontiguousarray(np.stack(d))).cuda()
    y = torch.empty_like(x)
    env = [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (ys, yr)]
    e.chain_process_device(x.data_ptr(), x.shape[1], y.data_ptr(), x.shape[1], x.shape[1],
                           *[0 if a is None else a.data_ptr() for a in env], sync=sync)

    def result():
        torch.cuda.synchronize()
        keep = env                                           # noqa: F841  the envelopes live until the call is done
        return tuple(y.cpu().numpy())
    return result


@pytest.mark.parametrize("backend", BACKENDS)
def test_interleaved_with_own_calls(backend):
    """group calls between the members' own chain_process calls, and (on the GPU) an unsynchronised
    chain_process_device right before a group call"""
    lib = get_lib(backend)
    head, tail, L = (16, 128, 1500) if backend == "emu" else (128, 8192, 30000)
    calls = variable_calls(6 * tail, 1, head, 13)
    ms = [ChainMember(lib, 2 + 2 * (i % 2), twostage(head, tail), irs_for(2 + 2 * (i % 2), L, i), CFGS[i], 7 * tail, i)
          for i in range(4)]
    g = Group([m.h for m in ms])
    for i, k in enumerate(calls):
        if i % 7 == 3:
            for m in ms:
                m.single(k)
        elif i % 11 == 5 and backend == "cuda":
            m = ms[1]
            d, ys, yr = m.take(head)
            got = _device_chain_call(m.h, d, ys, yr, False)
            want = _device_chain_call(m.twin, d, ys, yr, True)
            group_call(g, ms, k)
            m.got.insert(-1, got())
            m.want.insert(-1, want())
        else:
            group_call(g, ms, k)
    check_twins(ms, backend)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_forty_members(backend):
    """40 members of one shape class: two launches of each kind per call"""
    lib = get_lib(backend)
    head, L = (16, 300) if backend == "emu" else (128, 3000)
    calls = variable_calls(12 * head, 1, head, 7)
    n = sum(calls)
    ms = [ChainMember(lib, 2, uniform(head), irs_for(2, L, i), CFGS[i % 4], n, i) for i in range(40)]
    g = Group([m.h for m in ms])
    for k in calls:
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == 6
    check_twins(ms, backend)
    close(g, ms)


def _raw_call(lib, g, drys, outs, n):
    """b200conv_chain_group_process with hand-built tables (entries None: NULL)"""
    m = len(drys)
    keep = [None if d is None else (C.c_void_p * 2)(*[None if a is None else a.ctypes.data for a in d]) for d in drys]
    keep_o = [(C.c_void_p * 2)(*[a.ctypes.data for a in o]) for o in outs]
    dt = (C.c_void_p * m)(*[None if k is None else C.cast(k, C.c_void_p) for k in keep])
    ot = (C.c_void_p * m)(*[C.cast(k, C.c_void_p) for k in keep_o])
    return lib.b200conv_chain_group_process(g._g, C.cast(dt, C.POINTER(C.c_void_p)), None, None,
                                            C.cast(ot, C.POINTER(C.c_void_p)), n)


@pytest.mark.parametrize("backend", BACKENDS)
def test_refusals(backend):
    """a member without a chain, NULL buffers and every set_member error: refused before anything is enqueued, so
    the members go on exactly as their twins"""
    lib = get_lib(backend)
    head, tail, L = (16, 128, 1000) if backend == "emu" else (128, 8192, 20000)
    n = 20 * head
    ms = [ChainMember(lib, 2, twostage(head, tail), irs_for(2, L, i), CFGS[i], n, i) for i in range(3)]
    plain = ms[2].make(chain=False)
    g = Group([ms[0].h, ms[1].h, plain])
    zeros = [np.zeros(head, np.float32) for _ in range(2)]
    outs = [[np.zeros(head, np.float32) for _ in range(2)] for _ in range(3)]
    l0 = g.launch_count
    assert _raw_call(lib, g, [zeros] * 3, outs, head) == ESTATE                     # member 2 owns no chain
    assert b"member 2" in lib.b200conv_group_last_error(g._g)
    g.set_member(2, ms[2].h)
    assert _raw_call(lib, g, [zeros, None, zeros], outs, head) == EINVAL            # a NULL table entry
    assert _raw_call(lib, g, [zeros, [zeros[0], None], zeros], outs, head) == EINVAL   # a NULL channel
    assert lib.b200conv_chain_group_process(g._g, None, None, None, None, head) == EINVAL
    assert _raw_call(lib, g, [zeros] * 3, outs, 0) == 0                              # len == 0 does nothing
    assert g.launch_count == l0
    for index, h in [(3, ms[0].h._h), (-1, ms[0].h._h), (0, None), (1, ms[0].h._h)]:
        assert lib.b200conv_group_set_member(g._g, index, h) == EINVAL
    assert lib.b200conv_group_set_member(None, 0, ms[0].h._h) == EINVAL
    if backend == "emu":                                                             # a handle on another device
        other = Engine(2, device=1, lib=lib)
        assert lib.b200conv_group_set_member(g._g, 0, other._h) == EINVAL
        other.close()
    assert lib.b200conv_group_set_member(g._g, 1, ms[1].h._h) == 0                  # the member already there
    assert [e._h for e in g.engines] == [m.h._h for m in ms]
    for k in variable_calls(n, 1, head, 3):
        group_call(g, ms, k)
    check_twins(ms, backend, (head, tail))
    plain.close()
    close(g, ms)
