"""Real-time calls that cross a head-block boundary: k_rt_block runs the rest of the open block and the start of the
next one as two segments of one cluster launch (FFTConvolver.cpp:164-208 as two loop iterations).  Host blocks that
are not a power of two (480 samples at 48 kHz on head 512) and variable host blocks cross on most calls."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine, StereoConvolver
from tests import test_chain_swap as tcs
from tests.backends import lib  # noqa: F401
from tests.test_conv_precision import rt_cluster_ctas
from tests.test_tail_shards import _run_shards, _unsharded

TOL = 1e-5


def peak_err(y, ref):
    return float(np.max(np.abs(np.asarray(y, np.float64) - ref)) / max(np.max(np.abs(ref)), 1e-30))


def variable_calls(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    out = []
    while sum(out) < n:
        out.append(int(rng.integers(lo, hi + 1)))
    out[-1] -= sum(out) - n
    return [k for k in out if k]


def edge_calls(B, n, seed):
    """crossings by 1 and by B - 1 samples, calls that start and calls that end exactly at a boundary, full-block
    crossings, then seeded lengths in [1, B]"""
    b3 = B // 3
    out = [B - 1, 2, B - 2, b3, B, B - b3 - 1, B, 1, B - 1, B // 2, B // 2 + 1, B - 1]
    return out + variable_calls(n - sum(out), 1, B, seed)


def run(e, xs, chunks, clear_at=None):
    """outputs per channel and launches per call"""
    outs, launches, pos = [[] for _ in xs], [], 0
    for i, k in enumerate(chunks):
        if i == clear_at:
            e.clear()
        l0 = e.launch_count
        ys = e.process([x[pos:pos + k] for x in xs])
        launches.append(e.launch_count - l0)
        for c, y in enumerate(ys):
            outs[c].append(y)
        pos += k
    return [np.concatenate(o) for o in outs], launches


def crosses(chunks, B, start=0):
    """per call: does it cross a boundary of blocks of B (complete one block and start the next)"""
    pos, out = start, []
    for k in chunks:
        out.append((pos % B) + k > B)
        pos += k
    return out


def completes(chunks, B):
    """per call: does it complete a block of B"""
    pos, out = 0, []
    for k in chunks:
        out.append((pos + k) // B > pos // B)
        pos += k
    return out


@pytest.mark.parametrize("host", [37, 48, 60, 63, "var"])
def test_one_launch_per_crossing_call(lib, host):
    head, tail = 64, 256
    irs = [orc.synth_ir(2 * tail + 4 * tail + 77, c) for c in range(2)]
    n = 64 * 120
    xs = [orc.synth_input(n, c) for c in range(2)]
    chunks = variable_calls(n, 1, 64, 11) if host == "var" else [host] * (n // host)
    n = sum(chunks)
    # k: launches of the tail block an inside call enqueues on the same shape
    e = Engine(2, lib=lib)
    assert e.init_twostage(head, tail, irs)
    _, l64 = run(e, xs, [64] * 8)
    k = l64[3] - 1
    assert k >= 1 and l64[:3] == [1, 1, 1]
    e = Engine(2, lib=lib)
    assert e.init_twostage(head, tail, irs)
    ys, launches = run(e, xs, chunks)
    tail_done = completes(chunks, tail)
    assert any(c and not t for c, t in zip(crosses(chunks, head), tail_done))
    assert all(l == 1 for l, t in zip(launches, tail_done) if not t), launches
    assert sum(launches) <= len(chunks) + k * sum(tail_done) + 2
    for c in range(2):
        o = orc.OracleTwoStage()
        o.init(head, tail, irs[c])
        assert peak_err(ys[c], o.process(xs[c][:n])) <= TOL


# the K0 forms of test_conv_precision: every template M, cluster geometries C x NC = 1x1 ... 8x2
K0_SHAPES = [(16, 1, 40), (32, 1, 40), (64, 8, 100), (128, 4, 100), (256, 2, 100), (512, 1, 100), (1024, 1, 60),
             (1024, 2, 9)]


@pytest.mark.parametrize("M,C,P", K0_SHAPES, ids=[f"M{M}-C{C}x{rt_cluster_ctas(M, C, P)}" for M, C, P in K0_SHAPES])
def test_uniform_parity_every_template(lib, M, C, P):
    assert rt_cluster_ctas(M, C, P) > 0
    irs = [orc.synth_ir(P * M - 3, c) for c in range(C)]
    n = P * M + 6 * M
    xs = [orc.synth_input(n, c) for c in range(C)]
    chunks = edge_calls(M, n, M + C)
    e = Engine(C, lib=lib)
    assert e.init_uniform(M, irs)
    ys, launches = run(e, xs, chunks)
    cross = crosses(chunks, M)
    assert sum(cross) >= 5 and chunks[1] == 2 and cross[1] and cross[4] and cross[8]
    assert all(l == 1 for l in launches), sorted(set(launches))
    for c in range(C):
        o = orc.OracleUniform()
        o.init(M, irs[c])
        assert peak_err(ys[c], o.process(xs[c])) <= TOL


@pytest.mark.parametrize("kind", ["twostage", "stages-q4", "stages-q1"])
def test_staged_parity(lib, kind):
    """crossings that complete a tail block, clear() in the middle of a block, long (multi-kernel) calls in between;
    init_stages with stage delays of 4 blocks (q = 4) and of 1 block (q = 1: a crossing that completes such a stage's
    block needs its output inside the call and keeps the multi-kernel path)"""
    head = 16 if kind.startswith("stages") else 64
    if kind == "twostage":
        L = 2 * 256 + 5 * 256 + 9
    elif kind == "stages-q4":
        blocks, offsets, L = [16, 64, 256], [0, 256, 1024], 1024 + 4 * 256 + 5
    else:
        blocks, offsets, L = [16, 64], [0, 64], 64 * 9 + 5
    irs = [orc.synth_ir(L, c) for c in range(2)]
    calls = [head - 1, 2] + variable_calls(6 * head, 1, head, 3) + [5 * head + 7] + variable_calls(L, 1, head, 4)
    calls += [head * 30] + variable_calls(L + 7, 1, head, 5)
    clear_at, n = len(calls), sum(calls)
    xs = [orc.synth_input(n + 3000, c) for c in range(2)]
    calls += [head // 2 + 1] + variable_calls(3000 - head // 2 - 1, 1, head, 6)

    def oracle(c):
        o = orc.OracleTwoStage() if kind == "twostage" else orc.OracleUniform()
        assert o.init(head, 256, irs[c]) if kind == "twostage" else o.init(head, irs[c])
        return o

    e = Engine(2, lib=lib)
    assert e.init_twostage(head, 256, irs) if kind == "twostage" else e.init_stages(blocks, offsets, irs)
    ys, launches = run(e, xs, calls, clear_at=clear_at)
    before = calls[:clear_at]
    tail_b = 256 if kind == "twostage" else 64
    tail_done = completes(before, tail_b)
    assert any(c and t for c, t in zip(crosses(before, head), tail_done))
    for c in range(2):
        assert peak_err(ys[c][:n], oracle(c).process(xs[c][:n])) <= TOL
        # after clear() the stream starts afresh, here with crossing calls
        assert peak_err(ys[c][n:], oracle(c).process(xs[c][n:n + 3000])) <= TOL
    # every call of at most one head block that completes no later-stage block is one launch
    assert all(l == 1 for l, t, k in zip(launches, tail_done, before) if not t and k <= head)


def test_quad_device_mixdown_host_block_100(lib):
    sc = StereoConvolver(lib=lib)
    sc.prepare(100)                                        # head 128, tail 8192
    irs = [orc.synth_ir(30000, c) for c in range(4)]      # LL, RR, LR, RL
    sc.loadImpulse(*irs)
    sc.enable_device_mixdown(true_stereo=True)
    n = 100 * 300
    L, R = orc.synth_input(n, 0), orc.synth_input(n, 1)
    wl, wr = np.empty_like(L), np.empty_like(R)
    for i in range(300):
        seg = slice(100 * i, 100 * (i + 1))
        wl[seg], wr[seg] = sc.process_mixed(L[seg], R[seg])
    outs = []
    for ir, src in zip(irs, (L, R, L, R)):
        o = orc.OracleTwoStage()
        o.init(128, 8192, ir)
        outs.append(o.process(src))
    LL, RR, LR, RL = outs
    assert peak_err(wl, LL + RL) <= TOL and peak_err(wr, RR + LR) <= TOL


@pytest.mark.parametrize("kind", ["rt", "var"])
def test_chain_with_swap_at_host_block_100(lib, kind, monkeypatch):
    """the device chain and an IR hot swap armed with host_block = 100 on head 128 (most live, warm-up and fade calls
    cross a boundary), against the hot-swap oracle (oracle/hotswap.py's HotSwapChain) fed the same call lengths"""
    monkeypatch.setattr(tcs, "HEAD", 128)
    if kind == "var":
        monkeypatch.setattr(tcs, "_calls", lambda _kind, hb, total: variable_calls(total, 1, 128, 9))
    tcs._run(lib, tcs.CFGS["f12_24_48"], 2, 4, 100, "rt", 3000)


def test_split_mode_shape_keeps_the_multi_kernel_path(lib):
    """uniform 256 x 1100 partitions: too large for one cluster, so crossing calls do not qualify"""
    irs = [orc.synth_ir(256 * 1100 - 9, c) for c in range(2)]
    chunks = [200] * 40
    xs = [orc.synth_input(sum(chunks), c) for c in range(2)]
    e = Engine(2, lib=lib)
    assert e.init_uniform(256, irs)
    ys, launches = run(e, xs, chunks)
    cross = crosses(chunks, 256)
    assert all(l > 1 for l, c in zip(launches, cross) if c)
    assert all(l == 3 for l, c in zip(launches, cross) if not c)      # front + sweep + back
    for c in range(2):
        o = orc.OracleUniform()
        o.init(256, irs[c])
        assert peak_err(ys[c], o.process(xs[c])) <= TOL


@pytest.mark.parametrize("backend", ["emu", pytest.param("cuda", marks=pytest.mark.gpu)])
def test_tail_shards_rank0_crossing_calls(backend):
    from tests.backends import get_lib
    lib_ = get_lib(backend)
    head, tail = (16, 256) if backend == "emu" else (128, 8192)
    irs = [orc.synth_ir(2 * tail + 5 * tail + 41, c) for c in range(2)]
    chunks = variable_calls(8 * tail + 123, 1, head, 21)
    xs = [orc.synth_input(sum(chunks), c) for c in range(2)]

    def init(e):
        return e.init_twostage(head, tail, irs)
    got, _ = _run_shards(lib_, 2, 2, init, xs, chunks)
    want = _unsharded(lib_, 2, init, xs, chunks)
    assert sum(crosses(chunks, head)) > len(chunks) // 4
    for c in range(2):
        assert peak_err(got[c], want[c]) <= TOL


@pytest.mark.gpu
def test_reevr_quad_480_at_512_8192():
    """REEV-R's quad handle at 48 kHz, 10 ms host blocks: head 512, tail 8192, 10 s IRs, 480-sample calls"""
    from tests.backends import get_lib
    lib_ = get_lib("cuda")
    irs = [orc.synth_ir(480000, c) for c in range(4)]      # LL, RR, LR, RL
    n = 96000
    L, R = orc.synth_input(n, 0), orc.synth_input(n, 1)
    e = Engine(4, lib=lib_)
    assert e.init_twostage(512, 8192, irs)
    e.set_routing([0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]])
    chunks = [480] * (n // 480)
    ys, launches = run(e, [L, R], chunks)
    tail_done = completes(chunks, 8192)
    assert all(l == 1 for l, t in zip(launches, tail_done) if not t), sorted(set(launches))
    outs = []
    for ir, src in zip(irs, (L, R, L, R)):
        o = orc.OracleTwoStage()
        o.init(512, 8192, ir)
        outs.append(o.process(src))
    LL, RR, LR, RL = outs
    assert peak_err(ys[0], LL + RL) <= TOL and peak_err(ys[1], RR + LR) <= TOL
