"""Fixed-latency groups (b200conv_group_set_latency): the members at the group's latency run the head-block steps of a
group call in shared launches, one k_rt_group launch per round and shape class (the chain form adds one send and one
wet launch per round).  Every member has a twin built by the same recipe, given the same latency by its own
b200conv_set_latency (in the same order relative to chain_configure) and driven by its own process / chain_process with
the same call lengths: equal bit for bit on the CPU emulation, within the twin tolerance of tests/test_group.py on the
H100, and the output is the float64 oracle's delayed by the latency."""
import time

import numpy as np
import pytest

from reevr_b200.convolver import Engine, Group
from tests.backends import get_lib
from tests.test_chain_group import CFGS, ChainMember
from tests.test_chain_group import check_twins as check_chain_twins
from tests.test_chain_group import group_call as chain_group_call
from tests.test_chain_group import swap_through
from tests.test_group import (TOL, Member, check_twins, close, group_call, irs_for, peak_err, stages, twostage,
                              uniform)
from tests.test_rt_cross import variable_calls

BACKENDS = ["emu", pytest.param("cuda", marks=pytest.mark.gpu)]
EINVAL, ESTATE = -1, -3
QUAD_MAP, QUAD_MIX = [0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]]


class BatchMember(Member):
    """a Member whose engines take max_batch_blocks (a small staging size, so a small ring piece)"""

    def __init__(self, *args, batch=0, **kw):
        self.batch = batch
        super().__init__(*args, **kw)

    def make(self):
        e = Engine(self.nch, lib=self.lib, max_batch_blocks=self.batch)
        self.setup(e, self.irs)
        if self.in_map:
            e.set_routing(self.in_map, self.mix)
        return e


def set_group_latency(g, ms, D):
    """the group's latency on the members, the same latency on each twin on its own"""
    for m in ms:
        m.twin.set_latency(D)
    g.set_latency(D)
    assert g.latency == D and all(m.h.latency == D for m in ms)


def blocks(pos, k, B):
    return (pos + k) // B - pos // B


@pytest.mark.parametrize("backend", BACKENDS)
def test_four_routed_quads(backend):
    """REEV-R's quad two-stage members with routing and the quad mixdown, D = 2 head blocks, host block head / 4"""
    lib = get_lib(backend)
    head, tail, L = (16, 256, 3000) if backend == "emu" else (128, 8192, 100000)
    D = 2 * head
    calls = [head // 4] * (12 * tail // head)
    n = sum(calls)
    ms = [Member(lib, 4, twostage(head, tail), irs_for(4, L, i), n, i, QUAD_MAP, QUAD_MIX) for i in range(4)]
    g = Group([m.h for m in ms])
    set_group_latency(g, ms, D)
    for k in calls:
        group_call(g, ms, k)
    check_twins(ms, backend)
    for m in ms:
        got, _ = m.outputs()
        for a, ref in zip(got, m.oracle(n)):
            assert not np.any(a[:D]) and peak_err(a[D:], ref[:n - D]) <= TOL
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_mixed_shapes_and_lengths(backend):
    """head blocks 64 and 128 at D = 256 (two shape classes), a three-stage and a uniform member, one member with a ring
    piece of 1024 samples, next to members that cannot share (C = 9, split mode); calls up to 1300 samples"""
    lib = get_lib(backend)
    emu = backend == "emu"
    L = 3000 if emu else 60000
    calls = variable_calls(6000 if emu else 40000, 1, 1300, 23)
    n = sum(calls)
    ms = [BatchMember(lib, 2, twostage(64, 512), irs_for(2, L, 0), n, 0, batch=8),
          Member(lib, 4, twostage(128, 1024), irs_for(4, L, 1), n, 1, QUAD_MAP, QUAD_MIX),
          Member(lib, 2, stages([64, 256, 1024], [0, 512, 2048]), irs_for(2, L, 2), n, 2),
          Member(lib, 2, uniform(128), irs_for(2, 40 * 128 - 5, 3), n, 3),
          Member(lib, 9, uniform(64), irs_for(9, 20 * 64, 4), n, 4),                      # C = 9
          Member(lib, 2, uniform(256), irs_for(2, 256 * 1100 - 9, 5), n, 5)]             # split mode
    g = Group([m.h for m in ms])
    set_group_latency(g, ms, 256)
    pos = 0
    for k in calls:
        g0, m4, m5 = g.launch_count, ms[4].h.launch_count, ms[5].h.launch_count
        group_call(g, ms, k)
        if k >= 256:                             # the members that cannot share run every step of their own
            assert ms[4].h.launch_count > m4 and ms[5].h.launch_count > m5
        assert (g.launch_count > g0) == (blocks(pos, k, 64) > 0)
        pos += k
    check_twins(ms, backend)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("chain", [False, True])
def test_launch_counts(backend, chain):
    """one shape class: a call that completes no head block adds no group launch, one that completes one on every
    member adds one (chain: three), a call of 3 head blocks three (chain: nine); members count only tail blocks"""
    lib = get_lib(backend)
    head, tail, L = (16, 256, 2000) if backend == "emu" else (128, 8192, 30000)
    D = 2 * head
    calls = ([head // 4] * 8 + [3 * head] + [head] * 3 + [head // 2] * 3) * (3 * tail // head // 8)
    n = sum(calls)
    if chain:
        ms = [ChainMember(lib, 2, twostage(head, tail), irs_for(2, L, i), CFGS[i], n, i) for i in range(4)]
    else:
        ms = [Member(lib, 2, twostage(head, tail), irs_for(2, L, i), n, i) for i in range(4)]
    g = Group([m.h for m in ms])
    set_group_latency(g, ms, D)
    per = 3 if chain else 1
    pos, tails = 0, 0
    for k in calls:
        g0, m0 = g.launch_count, [m.h.launch_count for m in ms]
        (chain_group_call if chain else group_call)(g, ms, k)
        assert g.launch_count - g0 == per * blocks(pos, k, head)
        if blocks(pos, k, tail):
            tails += 1
            assert all(m.h.launch_count > c for m, c in zip(ms, m0))
        else:
            assert [m.h.launch_count for m in ms] == m0
        pos += k
    assert tails >= 2
    (check_chain_twins if chain else check_twins)(ms, backend)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_interleaved(backend):
    """own process calls between group calls, clear() on one member, another latency on one member (it then runs
    alone), and Group.set_latency(0): the launch counts of a zero-latency group from then on"""
    lib = get_lib(backend)
    head, tail, L = (16, 128, 1500) if backend == "emu" else (128, 8192, 30000)
    calls = variable_calls(8 * tail, 1, head, 13)
    ms = [Member(lib, 2, twostage(head, tail), irs_for(2, L, i), 9 * tail, i) for i in range(4)]
    g = Group([m.h for m in ms])
    set_group_latency(g, ms, 2 * head)
    third = len(calls) // 3
    p1 = 0                                                    # member 1's samples since its own set_latency
    for i, k in enumerate(calls):
        if i == third // 2:
            for e in (ms[2].h, ms[2].twin):
                e.clear()
        if i == third:
            for e in (ms[1].h, ms[1].twin):
                e.set_latency(3 * head)
            p1 = 0
        if i == 2 * third:
            for m in ms:
                if m.twin.latency:
                    m.twin.set_latency(0)
            g.set_latency(0)
            assert g.latency == 0 and all(m.h.latency == 0 for m in ms)
        if i % 7 == 3:
            for m in ms:
                x = m.take(k)
                m.record(m.h.process(x), m.twin.process(x))
            p1 += k
            continue
        g0, own = g.launch_count, ms[1].h.launch_count
        group_call(g, ms, k)
        if third <= i < 2 * third and blocks(p1, k, head):
            assert ms[1].h.launch_count > own                 # member 1 no longer shares
        p1 += k
        if i > 2 * third:
            assert g.launch_count - g0 == 1                   # one zero-latency launch per call
    check_twins(ms, backend)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_chain_updates_and_hot_swap(backend):
    """chain_update between group calls, own chain_process calls, and a hot swap on one member: it runs alone while the
    swap is pending, then its incoming handle shares the steps again once set_member puts it in place"""
    lib = get_lib(backend)
    emu = backend == "emu"
    head, tail, L = (16, 256, 3000) if emu else (128, 8192, 60000)
    D = 2 * head
    calls = variable_calls(3 * 2400 + 4 * tail, 1, head, 17)
    n = sum(calls)
    ms = [ChainMember(lib, 4, twostage(head, tail), irs_for(4, L, i), CFGS[i], n, i) for i in range(3)]
    g = Group([m.h for m in ms])
    set_group_latency(g, ms, D)
    incoming = []
    for _ in range(2):
        x = Engine(4, lib=lib)
        assert x.init_twostage(head, tail, irs_for(4, L // 2, 8))
        x.set_latency(D)
        incoming.append(x)
    outgoing, shares_again = (), 0
    for j, k in enumerate(calls):
        if j == 10:
            for e in (ms[0].h, ms[0].twin):
                e.chain_update(**dict(CFGS[0], lowcut_slope=0, highcut_slope=0, width=0.7))
        if j == 15:
            for m in ms:
                m.single(k)
            continue
        if j == 20:
            for e, x in zip((ms[1].h, ms[1].twin), incoming):
                e.chain_swap(x, head)
        if not outgoing and ms[1].h.chain_swap_state() == 3:
            outgoing = swap_through(g, 1, ms[1], incoming)
        own = ms[1].h.launch_count
        pos = sum(ms[1].calls)
        chain_group_call(g, ms, k)
        stepped = blocks(pos, k, head) and not blocks(pos, k, tail)
        if stepped and 20 <= j and not outgoing:
            assert ms[1].h.launch_count > own                 # alone while the swap is pending
        if stepped and outgoing and ms[1].h.launch_count == own:     # its steps went into the group's launches
            shares_again += 1
    assert outgoing and shares_again
    check_chain_twins(ms, backend)
    close(g, ms)
    for e in outgoing:
        e.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_refusals(backend):
    """a latency that is not a multiple of one member's head block, above 16 of one member's head blocks, a member
    without an IR, a sharded member and a member with a pending hot swap: refused, no member changes or is cleared"""
    lib = get_lib(backend)
    head, tail, L = (16, 128, 1000) if backend == "emu" else (128, 8192, 20000)
    n = 24 * head
    ms = [Member(lib, 2, twostage(head, tail), irs_for(2, L, 0), n, 0),
          Member(lib, 2, twostage(head, tail), irs_for(2, L, 1), n, 1),
          Member(lib, 2, twostage(2 * head, tail), irs_for(2, L, 2), n, 2)]
    g = Group([m.h for m in ms])
    set_group_latency(g, ms, 2 * head)
    calls = iter(variable_calls(n, 1, head, 3))
    for _ in range(6):
        group_call(g, ms, next(calls))

    def refused(grp, D, code, member):
        l0 = grp.launch_count
        assert lib.b200conv_group_set_latency(grp._g, D) == code
        assert f"member {member}".encode() in lib.b200conv_group_last_error(grp._g)
        assert grp.launch_count == l0

    refused(g, 3 * head, EINVAL, 2)                      # not a multiple of member 2's head block
    refused(g, 17 * head, EINVAL, 0)                     # above 16 of member 0's head blocks
    noir = Engine(2, lib=lib)
    sharded = Engine(2, lib=lib, shard_rank=0, shard_count=2)
    assert sharded.init_twostage(head, tail, irs_for(2, L, 5))
    live, nxt = Engine(2, lib=lib), Engine(2, lib=lib)
    for e in (live, nxt):
        assert e.init_twostage(head, tail, irs_for(2, L, 6))
    live.chain_configure(**CFGS[0])
    live.chain_swap(nxt, head)
    for bad, code in ((noir, ESTATE), (sharded, ESTATE), (live, ESTATE)):
        g2 = Group([ms[0].h, bad])
        refused(g2, 2 * head, code, 1)
        assert g2.latency == 0
        g2.close()
    assert g.latency == 2 * head and all(m.h.latency == 2 * head for m in ms)
    for k in calls:
        group_call(g, ms, k)
    check_twins(ms, backend)
    for e in (noir, sharded, live, nxt):
        e.close()
    close(g, ms)


@pytest.mark.gpu
def test_no_waits_at_the_callback_pace_on_gpu():
    """four of REEV-R's quad two-stage 128 / 8192 members with a 10 s IR, group latency 128, host block 128 at 48 kHz,
    paced as tests/test_latency.py paces one handle: no member waits"""
    B0 = 128
    period = B0 / 48000.0
    lib = get_lib("cuda")
    ms = [Member(lib, 4, twostage(B0, 8192), irs_for(4, 480000, 100 + i), B0, i, QUAD_MAP, QUAD_MIX) for i in range(4)]
    g = Group([m.h for m in ms])
    xs = [[m.xs[0], m.xs[1]] for m in ms]
    g.set_latency(B0)
    for _ in range(200):
        g.process(xs)
        time.sleep(period)
    g.set_latency(B0)                            # resets the counts
    for _ in range(2000):
        g.process(xs)
        time.sleep(period)
    assert [m.h.latency_waits for m in ms] == [0] * 4
    close(g, ms)
