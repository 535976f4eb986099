"""Group calls on device buffers (b200conv_group_process_device, b200conv_chain_group_process_device): the members that
share run their whole call of up to 16 head blocks as one k_rt_group_steps cluster per member, one launch per shape
class.  Every member has two twins built by the same recipe:
- the DEVICE twin, driven by b200conv_process_device / b200conv_chain_process_device with the same call lengths: the
  group's outputs stay within 1e-5 of its peak (a call over one head block runs its multi-kernel path there);
- the CUT twin, driven with the same samples cut at the member's head-block boundaries, so that every piece is one
  launch: a sharing member equals it bit for bit on the CPU emulation and to tests/test_group.py's TWIN_TOL on the
  H100 (a member that runs its own call equals its device twin instead).
Plain members also stay within 1e-5 of peak of the float64 oracle, chain members of the float64 oracle chain."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import B200ConvError, Engine, Group
from tests import backends
from tests.backends import get_lib
from tests.test_chain_group import ChainMember
from tests.test_group import TWIN_TOL, conv, irs_for, peak_err, twostage, uniform
from tests.test_rt_cross import variable_calls

BACKENDS = ["emu", pytest.param("cuda", marks=pytest.mark.gpu)]
TOL = 1e-5
EINVAL, ESTATE = -1, -3


class Dev:
    """device buffers of the backend: numpy arrays on the emulation build, CUDA tensors on the GPU"""

    def __init__(self, lib):
        self.gpu = backends._cache.get("emu") is not lib

    def put(self, a):
        a = np.ascontiguousarray(a, np.float32)
        if self.gpu:
            import torch
            return torch.from_numpy(a.copy()).cuda()
        return a.copy()

    def empty(self, rows, n):
        return self.put(np.full((rows, max(n, 1)), np.nan, np.float32))

    def ptr(self, b, off=0):
        if b is None:
            return 0
        return (b.data_ptr() if self.gpu else b.ctypes.data) + 4 * off

    def get(self, b):
        if self.gpu:
            import torch
            torch.cuda.synchronize()
            return b.cpu().numpy()
        return b.copy()


def steps_of(M, pos, k):
    """head blocks a call of k samples touches from stream position pos"""
    len1 = min(k, M - pos % M)
    return 1 + -(-(k - len1) // M)


def cuts(M, pos, k):
    """a call cut at the head-block boundaries"""
    out = []
    while k:
        n = min(k, M - pos % M)
        out.append(n)
        pos, k = pos + n, k - n
    return out


class DevMember:
    """a member, its device twin and its cut twin; `shares(pos, k)`: whether a group call of k samples at pos shares"""

    def __init__(self, lib, nch, setup, irs, n, seed, M, in_map=None, mix=None, shares=None):
        self.lib, self.nch, self.setup, self.irs, self.in_map, self.mix, self.M = lib, nch, setup, irs, in_map, mix, M
        self.n_in = max(in_map) + 1 if in_map else nch
        self.n_out = len(mix) if mix else nch
        self.xs = np.stack([orc.synth_input(n, 100 * seed + c) for c in range(self.n_in)]).astype(np.float32)
        self.shares = shares or (lambda pos, k: steps_of(M, pos, k) <= 16)
        self.h, self.dev, self.cut = self.make(), self.make(), self.make()
        self.got, self.want_dev, self.want_cut, self.shared = [], [], [], []
        self.pos = 0
        self.zero = 0           # input position of the last clear(): the handles' block boundaries count from there

    def make(self):
        e = Engine(self.nch, lib=self.lib)
        assert self.setup(e, self.irs) is not False
        if self.in_map:
            e.set_routing(self.in_map, self.mix)
        return e

    def oracle(self, n):
        ys = [conv(ir, self.xs[self.in_map[c] if self.in_map else c][:n]) for c, ir in enumerate(self.irs)]
        if self.mix is None:
            return ys
        return [sum(m * y for m, y in zip(row, ys)) for row in np.asarray(self.mix, np.float64)]

    def twins(self, d, x, k):
        """the twins' outputs for input x (n_in x k)"""
        xi, yo = d.put(x), d.empty(self.n_out, k)
        self.dev.process_device(d.ptr(xi), xi.shape[1], d.ptr(yo), yo.shape[1], k)
        want_dev = d.get(yo)[:, :k]
        parts, a = [], 0
        for n in cuts(self.M, self.pos - self.zero, k):
            xc, yc = d.put(x[:, a:a + n]), d.empty(self.n_out, n)
            self.cut.process_device(d.ptr(xc), n, d.ptr(yc), n, n)
            parts.append(d.get(yc)[:, :n])
            a += n
        return want_dev, np.concatenate(parts, axis=1)

    def close(self):
        for e in (self.h, self.dev, self.cut):
            e.close()


def group_call(g, d, ms, k, sync=False):
    """one b200conv_group_process_device call of k samples on every member, and the twins' calls"""
    ins = [m.xs[:, m.pos:m.pos + k] for m in ms]
    bi = [d.put(x) for x in ins]
    bo = [d.empty(m.n_out, k) for m in ms]
    g.process_device([d.ptr(b) for b in bi], [b.shape[1] for b in bi], [d.ptr(b) for b in bo],
                     [b.shape[1] for b in bo], k, sync=sync)
    for m, x, b in zip(ms, ins, bo):
        m.got.append(d.get(b)[:, :k])
        m.shared.append(m.shares(m.pos - m.zero, k))
        wd, wc = m.twins(d, x, k)
        m.want_dev.append(wd)
        m.want_cut.append(wc)
        m.pos += k


def twin_close(a, b, backend):
    if backend == "emu":
        return np.array_equal(a, b)
    return float(np.max(np.abs(a - b))) <= TWIN_TOL[backend] * max(1.0, float(np.max(np.abs(b))))


def check(ms, backend, oracle=True):
    """a member that never shares equals its device twin; one that shares equals its cut twin up to its first call
    that does not share: from there on its history rows come from the multi-kernel path, the cut twin's from the
    one-launch path, and the two agree to rounding only"""
    for m in ms:
        own_only, parted = not any(m.shared), False
        for got, wd, wc, sh in zip(m.got, m.want_dev, m.want_cut, m.shared):
            parted |= not sh
            if own_only or not parted:
                assert twin_close(got, wd if own_only else wc, backend)
        got = np.concatenate(m.got, axis=1)
        wd = np.concatenate(m.want_dev, axis=1)
        for a, b in zip(got, wd):
            assert peak_err(a, b.astype(np.float64)) <= TOL
        if oracle:
            for a, ref in zip(got, m.oracle(m.pos)):
                assert peak_err(a, ref) <= TOL


def lengths(M, n, seed):
    """1, 37, M, M + 1, 5M + 17, the 16-block bound from the current fill and one sample past it, then seeded lengths
    up to 17 head blocks"""
    out, pos = [], 0
    for k in (1, 37, M, M + 1, 5 * M + 17, None, None, 3, None):
        if k is None:
            k = 16 * M - pos % M + (1 if len(out) % 2 else 0)
        out.append(k)
        pos += k
    return out + variable_calls(n - pos, 1, 17 * M, seed)


def plain_members(lib, emu, n):
    head, tail, L = (16, 256, 3000) if emu else (128, 8192, 480000)
    head2, tail2 = (32, 512) if emu else (512, 8192)
    never = lambda pos, k: False
    return [DevMember(lib, 4, twostage(head, tail), irs_for(4, L, 0), n, 0, head),
            DevMember(lib, 2, twostage(head2, tail2), irs_for(2, L, 1), n, 1, head2),
            DevMember(lib, 4, twostage(head, tail), irs_for(4, L, 2), n, 2, head, [0, 1, 0, 1],
                      [[1, 0, 0.5, 1], [0, 1, 1, -0.25]]),
            DevMember(lib, 2, uniform(head if emu else 256), irs_for(2, 20 * (head if emu else 256) - 3, 3), n, 3,
                      head if emu else 256),
            DevMember(lib, 2, uniform(256), irs_for(2, 256 * 1100 - 9, 4), n, 4, 256, shares=never),      # split mode
            DevMember(lib, 16, uniform(head), irs_for(16, 20 * head, 5), n, 5, head, shares=never)]       # C = 16


@pytest.mark.parametrize("backend", BACKENDS)
def test_plain_members(backend):
    """two-stage quads and stereo, a routed quad, a uniform handle next to a split-mode and a C = 16 member, at every
    call length from 1 to one sample past 16 head blocks, across tail-block boundaries"""
    lib = get_lib(backend)
    emu = backend == "emu"
    d = Dev(lib)
    n = 3000 if emu else 60000
    ms = plain_members(lib, emu, n)
    calls = lengths(ms[0].M, n, 7)
    g = Group([m.h for m in ms])
    for k in calls:
        g0 = g.launch_count
        group_call(g, d, ms, k)
        classes = {(m.M, m.nch) for m in ms if m.shares(m.pos - k, k)}
        assert g.launch_count - g0 == len(classes)
    assert any(not m.shared[i] for m in ms[:4] for i in range(len(calls)))      # the length rule was met
    check(ms, backend)
    g.close()
    for m in ms:
        m.close()


def chain_cfgs():
    base = dict(srate=48000.0, width=0.8, drygain=0.7, wetgain=0.6)
    return [dict(base, lowcut_hz=150.0, lowcut_slope=1, highcut_hz=20000.0, highcut_slope=0, predelay=0,
                 true_stereo=True),
            dict(base, lowcut_hz=20.0, lowcut_slope=0, highcut_hz=5000.0, highcut_slope=2, predelay=0,
                 true_stereo=False),
            dict(base, lowcut_hz=20.0, lowcut_slope=0, highcut_hz=20000.0, highcut_slope=0, predelay=480,
                 true_stereo=True)]


class DevChain(ChainMember):
    """a chain member with a device twin and a cut twin (ChainMember's twin is the device twin).  The send filters
    run a chunked scan whose rounding depends on the call length: a group call's send is its device twin's, its
    convolvers are its cut twin's, so after the first call of several pieces both agree within rounding only."""

    def __init__(self, lib, nch, setup, irs, cfg, n, seed, M, send, rev):
        super().__init__(lib, nch, setup, irs, cfg, n, seed, send, rev)
        self.M, self.cut = M, self.make()
        self.want_cut, self.shared = [], []

    def run(self, e, d, dry, ys, yr, k, inplace=False):
        bd = d.put(np.stack(dry))
        bs, br = (None if a is None else d.put(a) for a in (ys, yr))
        bo = bd if inplace else d.empty(2, k)
        e.chain_process_device(d.ptr(bd), bd.shape[1], d.ptr(bo), bo.shape[1], k, d.ptr(bs), d.ptr(br))
        return d.get(bo)[:, :k]


def chain_group_call(g, d, ms, k, inplace=False):
    pos = [m.pos for m in ms]
    ins = [m.take(k) for m in ms]
    bd = [d.put(np.stack(x[0])) for x in ins]
    bs = [None if x[1] is None else d.put(x[1]) for x in ins]
    br = [None if x[2] is None else d.put(x[2]) for x in ins]
    bo = bd if inplace else [d.empty(2, k) for _ in ms]
    g.chain_process_device([d.ptr(b) for b in bd], [b.shape[1] for b in bd], [d.ptr(b) for b in bo],
                           [b.shape[1] for b in bo], k, [d.ptr(b) for b in bs], [d.ptr(b) for b in br])
    for m, p, x, b in zip(ms, pos, ins, bo):
        got = d.get(b)[:, :k]
        # the send's chunked scan rounds by call length: the cut twin is exact only while every call was one piece
        m.shared.append(len(cuts(m.M, p, k)) == 1)
        want_dev = m.run(m.twin, d, x[0], x[1], x[2], k)
        parts, a = [], 0
        for n in cuts(m.M, p, k):
            sl = slice(a, a + n)
            parts.append(m.run(m.cut, d, [c[sl] for c in x[0]], None if x[1] is None else x[1][sl],
                               None if x[2] is None else x[2][sl], n))
            a += n
        m.record(got, want_dev)
        m.want_cut.append(np.concatenate(parts, axis=1))


def chain_check(ms, backend, head, tail):
    for m in ms:
        parted = False
        for j, (got, wc, sh) in enumerate(zip(m.got, m.want_cut, m.shared)):
            parted |= not sh
            if not parted:
                assert twin_close(got, wc, backend), j
        got = np.concatenate(m.got, axis=1)
        wd = np.concatenate(m.want, axis=1)
        ref = m.oracle(head, tail)
        scale = max(float(np.max(np.abs(r))) for r in ref)
        wc = np.concatenate(m.want_cut, axis=1)
        for a, b, c, r in zip(got, wd, wc, ref):
            assert float(np.max(np.abs(a - b))) <= TOL * max(float(np.max(np.abs(b))), 1e-30)
            assert float(np.max(np.abs(a - c))) <= TOL * max(float(np.max(np.abs(c))), 1e-30)
            assert float(np.max(np.abs(a - r))) <= TOL * scale


@pytest.mark.parametrize("backend", BACKENDS)
def test_chain_members(backend):
    """12 dB low cut, 24 dB high cut, 480-sample predelay, both envelopes or none, quad true stereo; in place"""
    lib = get_lib(backend)
    emu = backend == "emu"
    d = Dev(lib)
    head, tail, L = (16, 256, 3000) if emu else (128, 8192, 480000)
    n = 2500 if emu else 40000
    cfgs = chain_cfgs()
    ms = [DevChain(lib, 4, twostage(head, tail), irs_for(4, L, i), cfgs[i], n, i, head, i != 1, i != 2)
          for i in range(3)]
    g = Group([m.h for m in ms])
    calls = lengths(head, n, 11)
    for j, k in enumerate(calls):
        g0 = g.launch_count
        chain_group_call(g, d, ms, k, inplace=j % 3 == 2)
        if steps_of(head, ms[0].pos - k, k) <= 16:
            assert g.launch_count - g0 == 3              # one send width, one shape class, one wet launch
        else:
            assert g.launch_count == g0
    chain_check(ms, backend, head, tail)
    g.close()
    for m in ms:
        for e in (m.h, m.twin, m.cut):
            e.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_interleaved_calls(backend):
    """device group calls between each member's own device and host calls, clear() and host group calls: the states
    carry across them as across the twins' own calls"""
    lib = get_lib(backend)
    emu = backend == "emu"
    d = Dev(lib)
    head, tail, L = (16, 256, 3000) if emu else (128, 8192, 100000)
    n = 4000 if emu else 60000
    ms = [DevMember(lib, 2, twostage(head, tail), irs_for(2, L, i), n, i, head) for i in range(3)]
    g = Group([m.h for m in ms])

    def own(m, k, host):
        x = m.xs[:, m.pos:m.pos + k]
        if host:
            got = np.stack(m.h.process(list(x)))
        else:
            xi, yo = d.put(x), d.empty(m.n_out, k)
            m.h.process_device(d.ptr(xi), k, d.ptr(yo), k, k)
            got = d.get(yo)[:, :k]
        wd, wc = m.twins(d, x, k)
        m.got.append(got)
        m.want_dev.append(wd)
        m.want_cut.append(wc)
        m.shared.append(False)
        m.pos += k

    rng = np.random.default_rng(5)
    for j in range(60 if emu else 120):
        what = j % 5
        k = int(rng.integers(1, 10 * head))
        if what == 0:
            own(ms[j % 3], min(k, head), host=True)
            for m in ms[:j % 3] + ms[j % 3 + 1:]:
                own(m, min(k, head), host=False)
        elif what == 1 and j % 15 == 1:
            for m in ms:
                for e in (m.h, m.dev, m.cut):
                    e.clear()
                m.zero = m.pos
        elif what == 2:
            kk = min(k, head)
            ins = [list(m.xs[:, m.pos:m.pos + kk]) for m in ms]
            ys = g.process(ins)
            for m, x, y in zip(ms, ins, ys):
                wd, wc = m.twins(d, np.stack(x), kk)
                m.got.append(np.stack(y))
                m.want_dev.append(wd)
                m.want_cut.append(wc)
                m.shared.append(True)
                m.pos += kk
        else:
            group_call(g, d, ms, k)
    for m in ms:            # the own calls of one head block or less run one launch: the cut twin's path too
        m.shared = [True] * len(m.got)
    check(ms, backend, oracle=False)
    g.close()
    for m in ms:
        m.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_errors_advance_nothing(backend):
    lib = get_lib(backend)
    emu = backend == "emu"
    d = Dev(lib)
    head, tail, L = (16, 256, 2000) if emu else (128, 8192, 50000)
    n = 2000
    ms = [DevMember(lib, 2, twostage(head, tail), irs_for(2, L, i), n, i, head) for i in range(2)]
    for m in ms:
        for e in (m.h, m.dev, m.cut):
            e.chain_configure(**chain_cfgs()[0])
    g = Group([m.h for m in ms])
    l_ = g._l
    group_call(g, d, ms, 3 * head + 5)
    x, y = d.put(np.zeros((2, 64))), d.empty(2, 64)
    P = lambda v: (np.ctypeslib.ctypes.c_void_p * 2)(*v)
    S = lambda v: (np.ctypeslib.ctypes.c_size_t * 2)(*v)
    ok_p, ok_s = P([d.ptr(x)] * 2), S([64, 64])
    assert l_.b200conv_group_process_device(g._g, None, ok_s, ok_p, ok_s, 64, 0) == EINVAL
    assert l_.b200conv_group_process_device(g._g, ok_p, ok_s, ok_p, None, 64, 0) == EINVAL
    assert l_.b200conv_group_process_device(g._g, P([d.ptr(x), 0]), ok_s, ok_p, ok_s, 64, 0) == EINVAL
    assert l_.b200conv_group_process_device(g._g, P([d.ptr(x), 0]), ok_s, ok_p, ok_s, 0, 0) == 0
    assert l_.b200conv_chain_group_process_device(g._g, ok_p, ok_s, None, None, P([0, d.ptr(y)]), ok_s, 64, 0) == EINVAL
    bare = Engine(2, lib=lib)
    assert bare.init_twostage(head, tail, irs_for(2, L, 9))
    g2 = Group([ms[0].h, bare])
    assert l_.b200conv_chain_group_process_device(g2._g, ok_p, ok_s, None, None, ok_p, ok_s, 64, 0) == ESTATE
    bare.set_latency(head)
    assert l_.b200conv_group_process_device(g2._g, ok_p, ok_s, ok_p, ok_s, 64, 0) == ESTATE
    g2.close()
    bare.close()
    g3 = Group([Engine(2, lib=lib)])
    g3.engines[0].init_twostage(head, tail, irs_for(2, L, 8))
    g3.set_latency(head)
    assert l_.b200conv_group_process_device(g3._g, P([d.ptr(x)] * 1), S([64]), P([d.ptr(y)] * 1), S([64]), 64, 0) == ESTATE
    g3.close()
    g3.engines[0].close()
    with pytest.raises(B200ConvError):
        g.process_device([d.ptr(x), 0], [64, 64], [d.ptr(y)] * 2, [64, 64], 64)
    group_call(g, d, ms, 5 * head + 1)                   # nothing advanced: the twins still agree
    check(ms, backend, oracle=False)
    g.close()
    for m in ms:
        m.close()


@pytest.mark.gpu
def test_stream_ordering_on_the_gpu():
    """inputs produced on a torch stream the group stream waits on, outputs consumed on a torch stream after waiting
    on the group stream, and sync = 1"""
    import torch
    lib = get_lib("cuda")
    head, tail, L = 128, 8192, 480000
    ms = [DevMember(lib, 4, twostage(head, tail), irs_for(4, L, i), 20000, i, head) for i in range(4)]
    ms.append(DevMember(lib, 2, uniform(256), irs_for(2, 256 * 1100 - 9, 9), 20000, 9, 256))       # its own call
    g = Group([m.h for m in ms])
    gs = torch.cuda.ExternalStream(g.stream)
    prod, cons = torch.cuda.Stream(), torch.cuda.Stream()
    d = Dev(lib)
    for j, k in enumerate([2048, 480, 2048, 1000, 2048]):
        src = [torch.from_numpy(np.ascontiguousarray(m.xs[:, m.pos:m.pos + k])).pin_memory() for m in ms]
        with torch.cuda.stream(prod):
            torch.cuda._sleep(2_000_000)                  # the inputs land late: the group must wait for them
            bi = [s.cuda(non_blocking=True) for s in src]
            bo = [torch.full((m.n_out, k), float("nan"), device="cuda") for m in ms]
        gs.wait_stream(prod)
        g.process_device([b.data_ptr() for b in bi], [k] * len(ms), [b.data_ptr() for b in bo], [k] * len(ms), k,
                         sync=j == 4)
        cons.wait_stream(gs)
        with torch.cuda.stream(cons):
            outs = [b.clone() for b in bo]
        torch.cuda.synchronize()
        for m, x, o in zip(ms, src, outs):
            m.got.append(o.cpu().numpy())
            m.shared.append(m.shares(m.pos, k))
            wd, wc = m.twins(d, x.numpy(), k)
            m.want_dev.append(wd)
            m.want_cut.append(wc)
            m.pos += k
    ms[-1].shared = [False] * len(ms[-1].got)
    check(ms, "cuda", oracle=False)
    g.close()
    for m in ms:
        m.close()
