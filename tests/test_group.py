"""Groups of handles (b200conv_group_process): the real-time calls of several handles as one k_rt_group launch per shape
class.  Every member has a twin handle with the same IR and routing driven by b200conv_process with the same call
lengths: on the CPU emulation the group's outputs equal the twins' bit for bit, on the H100 to 1e-6 absolute (the
tolerance of the one-launch real-time tests) for outputs up to 1, and to 1e-6 of the twin's peak above that, and both
stay within 1e-5 of peak of the float64-accumulating oracle.  The relative part is needed because two handles driven
identically do not give bitwise equal outputs on the GPU. Tail blocks, and the heads of split-mode handles, run the
streaming sweep, which adds partial sums with float atomics in whatever order its CTAs finish. With 10 s IRs the
outputs reach about 100, where that order changes the last bit or two (7.6e-6 and more)."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine, Group
from tests.backends import get_lib
from tests.test_conv_precision import rt_cluster_ctas
from tests.test_rt_cross import variable_calls

BACKENDS = ["emu", pytest.param("cuda", marks=pytest.mark.gpu)]
TOL = 1e-5
TWIN_TOL = {"emu": 0.0, "cuda": 1e-6}


def peak_err(y, ref):
    return float(np.max(np.abs(np.asarray(y, np.float64) - ref)) / max(np.max(np.abs(ref)), 1e-30))


def conv(ir, x):
    o = orc.OracleUniform()
    assert o.init(256, ir)
    return o.process(x)


class Member:
    """a member and its twin, built by the same recipe; `irs` per convolver, `xs` per (routed) input, `mix` or None"""

    def __init__(self, lib, nch, setup, irs, n, seed, in_map=None, mix=None):
        self.lib, self.nch, self.setup, self.irs, self.in_map, self.mix = lib, nch, setup, irs, in_map, mix
        n_in = max(in_map) + 1 if in_map else nch
        self.xs = [orc.synth_input(n, 100 * seed + c) for c in range(n_in)]
        self.h, self.twin = self.make(), self.make()
        self.got, self.want = [], []
        self.pos = 0

    def make(self):
        e = Engine(self.nch, lib=self.lib)
        self.setup(e, self.irs)
        if self.in_map:
            e.set_routing(self.in_map, self.mix)
        return e

    def take(self, k):
        """the member's next k input samples"""
        self.pos += k
        return [x[self.pos - k:self.pos] for x in self.xs]

    def oracle(self, n):
        """what the member must produce for the first n samples"""
        ys = [conv(ir, self.xs[self.in_map[c] if self.in_map else c][:n]) for c, ir in enumerate(self.irs)]
        if self.mix is None:
            return ys
        return [sum(m * y for m, y in zip(row, ys)) for row in np.asarray(self.mix, np.float64)]

    def record(self, got, want):
        self.got.append(got)
        self.want.append(want)

    def outputs(self):
        return ([np.concatenate([g[c] for g in self.got]) for c in range(len(self.got[0]))],
                [np.concatenate([w[c] for w in self.want]) for c in range(len(self.want[0]))])


def group_call(g, ms, k):
    ins = [m.take(k) for m in ms]
    ys = g.process(ins)
    for m, x, y in zip(ms, ins, ys):
        m.record(y, m.twin.process(x))


def check_twins(ms, backend, oracle_n=None):
    for m in ms:
        got, want = m.outputs()
        for a, b in zip(got, want):
            if backend == "emu":
                assert np.array_equal(a, b)
            else:
                assert float(np.max(np.abs(a - b))) <= TWIN_TOL[backend] * max(1.0, float(np.max(np.abs(b))))
        if oracle_n:
            for a, ref in zip(got, m.oracle(oracle_n)):
                assert peak_err(a[:oracle_n], ref) <= TOL


def twostage(head, tail):
    return lambda e, irs: e.init_twostage(head, tail, irs)


def uniform(block):
    return lambda e, irs: e.init_uniform(block, irs)


def stages(blocks, offsets):
    return lambda e, irs: e.init_stages(blocks, offsets, irs)


def irs_for(nch, L, seed):
    return [orc.synth_ir(L, 10 * seed + c) for c in range(nch)]


def close(g, ms):
    g.close()
    for m in ms:
        m.h.close()
        m.twin.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_one_class_of_four_quads(backend):
    """4 quad two-stage members: one launch per call; the calls that complete a tail block complete it on every member
    at once, and only then do the members count launches (their tail blocks)"""
    lib = get_lib(backend)
    head, tail, L = (16, 256, 3000) if backend == "emu" else (128, 8192, 480000)
    calls = [head] * 200
    n = sum(calls)
    ms = [Member(lib, 4, twostage(head, tail), irs_for(4, L, i), n, i) for i in range(4)]
    g = Group([m.h for m in ms])
    pos, tails = 0, 0
    for k in calls:
        g0, m0 = g.launch_count, [m.h.launch_count for m in ms]
        group_call(g, ms, k)
        completes = (pos + k) // tail > pos // tail
        assert g.launch_count - g0 == 1
        if completes:
            tails += 1
            assert all(m.h.launch_count > c for m, c in zip(ms, m0))
        else:
            assert [m.h.launch_count for m in ms] == m0
        pos += k
    assert tails >= 2
    check_twins(ms, backend, n)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_crossing_calls_with_different_stages(backend):
    """480-sample calls on head 512 (30 on 32 on the emulation), then seeded lengths in [1, head]; a two-stage, a
    3-stage init_stages and a uniform member: one launch per distinct cluster width per call"""
    lib = get_lib(backend)
    emu = backend == "emu"
    M = 32 if emu else 512
    T = 256 if emu else 8192
    recipes = [(twostage(M, T), 3000 if emu else 100000),
               (stages([M, 4 * M, 16 * M], [0, 8 * M, 32 * M]), 3000 if emu else 60000),
               (uniform(M), 40 * M - 5 if emu else 100 * M - 7)]
    calls = [M - M // 16] * 40
    calls += variable_calls((1 if emu else 4) * T, 1, M, 31)
    n = sum(calls)
    ms = [Member(lib, 2, setup, irs_for(2, L, i), n, i) for i, (setup, L) in enumerate(recipes)]
    widths = {rt_cluster_ctas(M, 2, int(m.h.stages()[0]["partitions"])) for m in ms}
    assert all(w > 0 for w in widths)
    g = Group([m.h for m in ms])
    for k in calls:
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == len(widths)
    check_twins(ms, backend, n)
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_mixed_group(backend):
    """two shape classes (a routed quad with device mixdown; two stereo two-stage members) next to members that run on
    their own: split mode, C = 9, fixed latency; and one call longer than the head block, which no member shares"""
    lib = get_lib(backend)
    emu = backend == "emu"
    head, tail, L = (32, 256, 3000) if emu else (128, 8192, 100000)
    quad_map, quad_mix = [0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]]
    calls = variable_calls(12 * tail // 4, 1, head, 41)
    calls = calls[:len(calls) // 2] + [3 * head + 5] + calls[len(calls) // 2:]
    n = sum(calls)
    ms = [Member(lib, 4, twostage(head, tail), irs_for(4, L, 0), n, 0, quad_map, quad_mix),
          Member(lib, 2, twostage(head, tail), irs_for(2, L, 1), n, 1),
          Member(lib, 2, uniform(256), irs_for(2, 256 * 1100 - 9, 2), n, 2),            # split mode
          Member(lib, 9, uniform(head), irs_for(9, 20 * head, 3), n, 3),               # C = 9
          Member(lib, 2, twostage(head, tail), irs_for(2, L, 4), n, 4),
          Member(lib, 2, twostage(head, tail), irs_for(2, L, 5), n, 5)]
    assert rt_cluster_ctas(256, 2, int(ms[2].h.stages()[0]["partitions"])) == -1
    for e in (ms[5].h, ms[5].twin):
        e.set_latency(head)
    g = Group([m.h for m in ms])
    for k in calls:
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == (2 if k <= head else 0)
    check_twins(ms, backend)
    for m in ms[:5]:
        got, _ = m.outputs()
        for a, ref in zip(got, m.oracle(n)):
            assert peak_err(a, ref) <= TOL
    got, _ = ms[5].outputs()                                  # the latency member: its output `head` samples later
    for a, ref in zip(got, ms[5].oracle(n)):
        assert not np.any(a[:head]) and peak_err(a[head:], ref[:n - head]) <= TOL
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_forty_members_two_launches(backend):
    lib = get_lib(backend)
    head, L = (16, 300) if backend == "emu" else (128, 3000)
    calls = variable_calls(12 * head, 1, head, 7)
    n = sum(calls)
    ms = [Member(lib, 2, uniform(head), irs_for(2, L, i), n, i) for i in range(40)]
    g = Group([m.h for m in ms])
    for k in calls:
        g0 = g.launch_count
        group_call(g, ms, k)
        assert g.launch_count - g0 == 2
    check_twins(ms, backend, n)
    close(g, ms)


def _device_call(backend, e, xs, sync):
    """b200conv_process_device of one call; returns a function that yields the outputs once the call has completed"""
    if backend == "emu":
        x = np.ascontiguousarray(np.stack(xs))
        y = np.empty_like(x)
        e.process_device(x.ctypes.data, x.shape[1], y.ctypes.data, x.shape[1], x.shape[1], sync=sync)
        return lambda: list(y)
    import torch
    x = torch.from_numpy(np.ascontiguousarray(np.stack(xs))).cuda()
    y = torch.empty_like(x)
    e.process_device(x.data_ptr(), x.shape[1], y.data_ptr(), x.shape[1], x.shape[1], sync=sync)

    def result():
        torch.cuda.synchronize()
        return list(y.cpu().numpy())
    return result


@pytest.mark.parametrize("backend", BACKENDS)
def test_interleaved_with_single_calls(backend):
    """group calls between single b200conv_process calls, an unsynchronised process_device right before a group call,
    clear (the member then matches a fresh twin), reset (zeros from then on) and init_* with a new IR"""
    lib = get_lib(backend)
    head, tail, L = (16, 128, 1500) if backend == "emu" else (128, 8192, 30000)
    calls = variable_calls(6 * tail, 1, head, 13)
    ms = [Member(lib, 2, twostage(head, tail), irs_for(2, L, i), 7 * tail, i) for i in range(4)]
    g = Group([m.h for m in ms])
    new_irs = irs_for(2, L // 2, 9)
    zeros_from = None
    for i, k in enumerate(calls):
        if i % 7 == 3:                                        # single calls on the members
            for m in ms:
                x = m.take(k)
                m.record(m.h.process(x), m.twin.process(x))
        elif i % 11 == 5:                                     # an unsynchronised device call on member 1, then the group
            x = ms[1].take(head)
            got = _device_call(backend, ms[1].h, x, False)
            want = _device_call(backend, ms[1].twin, x, True)
            group_call(g, ms, k)
            ms[1].got.insert(-1, got())
            ms[1].want.insert(-1, want())
        else:
            group_call(g, ms, k)
        if i == len(calls) // 3:
            ms[2].h.clear()
            ms[2].twin.close()
            ms[2].twin = ms[2].make()
        if i == len(calls) // 2:
            ms[3].h.reset()
            ms[3].twin.reset()
            zeros_from = len(ms[3].got)
        if i == 2 * len(calls) // 3:
            for e in (ms[0].h, ms[0].twin):
                assert e.init_twostage(head, tail, new_irs)
    check_twins(ms, backend)
    after = np.concatenate([y[0] for y in ms[3].got[zeros_from:]])
    assert after.size and not np.any(after) and np.any(ms[3].got[0][0])
    close(g, ms)


@pytest.mark.parametrize("backend", BACKENDS)
def test_refusals(backend):
    lib = get_lib(backend)
    head, tail, L = (16, 128, 1000) if backend == "emu" else (128, 8192, 20000)
    n = 20 * head
    ms = [Member(lib, 2, twostage(head, tail), irs_for(2, L, i), n, i) for i in range(3)]
    hs = [m.h._h for m in ms]
    assert not lib.b200conv_group_create((C.c_void_p * 1)(hs[0]), 0)
    assert not lib.b200conv_group_create((C.c_void_p * 2)(hs[0], hs[0]), 2)
    assert not lib.b200conv_group_create((C.c_void_p * 2)(hs[0], None), 2)
    g = Group([m.h for m in ms])
    group_call(g, ms, head)
    # a NULL input table of member 1: B200CONV_EINVAL before anything is enqueued
    keep = [[np.zeros(head, np.float32) for _ in range(2)] for _ in ms]
    ptrs = [(C.c_void_p * 2)(*[a.ctypes.data for a in x]) for x in keep]
    ins = (C.c_void_p * 3)(C.cast(ptrs[0], C.c_void_p), None, C.cast(ptrs[2], C.c_void_p))
    outs = (C.c_void_p * 3)(*[C.cast(p, C.c_void_p) for p in ptrs])
    l0 = g.launch_count
    assert lib.b200conv_group_process(g._g, C.cast(ins, C.POINTER(C.c_void_p)), C.cast(outs, C.POINTER(C.c_void_p)),
                                      head) == -1
    assert b"null buffer" in lib.b200conv_group_last_error(g._g)
    # len == 0 does nothing
    assert lib.b200conv_group_process(g._g, C.cast(ins, C.POINTER(C.c_void_p)), C.cast(outs, C.POINTER(C.c_void_p)),
                                      0) == 0
    assert g.launch_count == l0
    for k in variable_calls(n - head, 1, head, 3):
        group_call(g, ms, k)
    check_twins(ms, backend, n)
    close(g, ms)
