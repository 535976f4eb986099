"""Tail-stage sharding (Engine(..., shard_head=False)): rank 0 keeps the head stage whole, the stages >= 1 are
partition-range sharded, and their partial spectra reach rank 0 through the tail slot exchange or the reduce hook.
G shards of one convolver run in G threads of this process (raw-pointer exchange, host barrier) or one after the
other (sequential stand-in for the reduce), on the emulation build and on the GPU."""
import threading

import numpy as np
import pytest
import scipy.signal

from oracle import oracle as orc
from reevr_b200.convolver import B200ConvError, Engine
from reevr_b200.synth import synth_input, synth_ir
from tests.backends import get_lib

TOL = 1e-5

# (head, tail, IR taps, channels, input samples) per backend: REEV-R's quad two-stage handle on the GPU
TWO_STAGE = {"emu": (16, 256, 5000, 1, 4000), "cuda": (128, 8192, 480000, 4, 8192 * 7 + 300)}
# three stages through init_stages: (blocks, offsets, IR taps, input samples)
THREE_STAGE = {"emu": ([16, 64, 256], [0, 128, 1024], 5000, 4000),
               "cuda": ([128, 1024, 8192], [0, 2048, 16384], 144000, 8192 * 6 + 77)}

# (head, tail, input samples) of the short-IR cases
SHORT = {"emu": (16, 256, 4000), "cuda": (128, 8192, 8192 * 6 + 100)}

BACKENDS = ["emu", pytest.param("cuda", marks=pytest.mark.gpu)]
BACKEND_G = [("emu", 2), ("emu", 4), pytest.param("cuda", 2, marks=pytest.mark.gpu),
             pytest.param("cuda", 4, marks=pytest.mark.gpu)]


def _ragged(n, head, seed=7):
    """Call lengths: mostly single head blocks (the real-time path on rank 0), some odd and some long calls."""
    rng = np.random.default_rng(seed)
    out, pos = [], 0
    while pos < n:
        r = rng.random()
        k = head if r < 0.6 else (int(rng.integers(1, head)) if r < 0.8 else int(rng.integers(head, 40 * head)))
        k = min(k, n - pos)
        out.append(k)
        pos += k
    return out


def _err(y, ref):
    return float(np.max(np.abs(np.asarray(y, np.float64) - ref)) / np.max(np.abs(ref)))


def _run_shards(lib_, G, C, init, xs, chunks, clear_at=None):
    """G tail-sharded shards in G threads; returns (rank 0's outputs per channel, every rank's stage ranges)."""
    gather_box, gather_bar, host_bar = [None] * G, threading.Barrier(G), threading.Barrier(G)
    outs, stages, errs = [None] * G, [None] * G, []

    def worker(rank):
        try:
            e = Engine(C, shard_rank=rank, shard_count=G, shard_head=False, lib=lib_)
            assert init(e)
            stages[rank] = e.stages()

            def allgather(blob):
                gather_box[rank] = blob
                gather_bar.wait(120)
                res = list(gather_box)
                gather_bar.wait(120)
                return res
            e.p2p_attach(allgather, mode=1, host_barrier=lambda: (host_bar.wait(300), 0)[1])
            ys, pos = [], 0
            for i, k in enumerate(chunks):
                if i == clear_at:
                    e.clear()
                ys.append(e.process([x[pos:pos + k] for x in xs]))
                pos += k
            outs[rank] = [np.concatenate([y[c] for y in ys]) for c in range(C)]
            gather_bar.wait(300)          # nobody frees exchange buffers while a peer may still touch them
            e.close()
        except Exception as ex:           # pragma: no cover
            errs.append(ex)
            gather_bar.abort()
            host_bar.abort()

    ths = [threading.Thread(target=worker, args=(r,)) for r in range(G)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(900)
    assert not errs, errs
    return outs[0], stages


def _unsharded(lib_, C, init, xs, chunks, clear_at=None):
    e = Engine(C, lib=lib_)
    assert init(e)
    ys, pos = [], 0
    for i, k in enumerate(chunks):
        if i == clear_at:
            e.clear()
        ys.append(e.process([x[pos:pos + k] for x in xs]))
        pos += k
    e.close()
    return [np.concatenate([y[c] for y in ys]) for c in range(C)]


def _check_ranges(stages, G):
    """Rank 0 holds stage 0 whole, the other ranks none of it; the tail ranges partition every tail stage."""
    full = stages[0][0]["partitions"]
    assert (stages[0][0]["p_begin"], stages[0][0]["p_end"]) == (0, full)
    for r in range(1, G):
        assert stages[r][0]["p_end"] == stages[r][0]["p_begin"]
    for s in range(1, len(stages[0])):
        P = stages[0][s]["partitions"]
        spans = sorted((stages[r][s]["p_begin"], stages[r][s]["p_end"]) for r in range(G))
        covered = 0
        for b, e in spans:
            assert b == covered or b == e
            covered = max(covered, e)
        assert covered == P and sum(e - b for b, e in spans) == P


@pytest.mark.parametrize("backend,G", BACKEND_G)
def test_two_stage_tail_exchange(backend, G):
    lib_ = get_lib(backend)
    head, tail, n_ir, C, n = TWO_STAGE[backend]
    irs = [synth_ir(n_ir, c) for c in range(C)]
    xs = [synth_input(n, c) for c in range(C)]
    chunks = _ragged(n, head)
    init = lambda e: e.init_twostage(head, tail, irs)       # noqa: E731
    y, stages = _run_shards(lib_, G, C, init, xs, chunks)
    _check_ranges(stages, G)
    assert len(stages[0]) == 2 and stages[1][1]["p_end"] > stages[1][1]["p_begin"]
    ref = _unsharded(lib_, C, init, xs, chunks)
    for c in range(C):
        o = orc.OracleTwoStage()
        o.init(head, tail, irs[c])
        assert _err(y[c], o.process(xs[c])) <= TOL, c
        assert _err(y[c], ref[c]) <= TOL, c


@pytest.mark.parametrize("backend,G", BACKEND_G)
def test_three_stage_tail_exchange(backend, G):
    lib_ = get_lib(backend)
    blocks, offsets, n_ir, n = THREE_STAGE[backend]
    h, x = synth_ir(n_ir), synth_input(n)
    chunks = _ragged(n, blocks[0], seed=11)
    init = lambda e: e.init_stages(blocks, offsets, [h])    # noqa: E731
    y, stages = _run_shards(lib_, G, 1, init, [x], chunks)
    assert len(stages[0]) == 3
    _check_ranges(stages, G)
    truth = scipy.signal.fftconvolve(x.astype(np.float64), h.astype(np.float64))[:n]
    assert _err(y[0], truth) <= TOL
    assert _err(y[0], _unsharded(lib_, 1, init, [x], chunks)[0]) <= TOL


@pytest.mark.parametrize("backend", BACKENDS)
def test_clear_mid_stream_matches_a_fresh_handle(backend):
    lib_ = get_lib(backend)
    head, tail, n_ir, C, n = TWO_STAGE[backend]
    irs = [synth_ir(n_ir, c) for c in range(C)]
    xs = [synth_input(n, c) for c in range(C)]
    chunks = _ragged(n, head, seed=3)
    cut = len(chunks) // 2
    init = lambda e: e.init_twostage(head, tail, irs)       # noqa: E731
    y, _ = _run_shards(lib_, 2, C, init, xs, chunks, clear_at=cut)
    start = sum(chunks[:cut])
    fresh = _unsharded(lib_, C, init, [x[start:] for x in xs], chunks[cut:])
    for c in range(C):
        assert _err(y[c][start:], fresh[c]) <= TOL, c


@pytest.mark.parametrize("backend", BACKENDS)
def test_tail_with_fewer_partitions_than_ranks(backend):
    """Two tail partitions over four ranks: ranks 2 and 3 own none and still publish zero slots (the exchange sweep with
    an empty partition range)."""
    lib_ = get_lib(backend)
    head, tail, n = SHORT[backend]
    h = synth_ir(4 * tail - 10)
    x = synth_input(n)
    chunks = _ragged(n, head, seed=5)
    init = lambda e: e.init_twostage(head, tail, [h])       # noqa: E731
    y, stages = _run_shards(lib_, 4, 1, init, [x], chunks)
    assert stages[0][1]["partitions"] == 2
    assert [st[1]["p_end"] - st[1]["p_begin"] for st in stages] == [1, 1, 0, 0]
    o = orc.OracleTwoStage()
    o.init(head, tail, h)
    assert _err(y[0], o.process(x)) <= TOL


@pytest.mark.parametrize("backend", BACKENDS)
def test_ir_without_a_tail_stage(backend):
    """An IR shorter than the tail offset: one stage, whole on rank 0; the other ranks own nothing."""
    lib_ = get_lib(backend)
    head, tail, n = SHORT[backend]
    h = synth_ir(2 * tail - 100)
    x = synth_input(n)
    chunks = _ragged(n, head, seed=9)
    init = lambda e: e.init_twostage(head, tail, [h])       # noqa: E731
    y, stages = _run_shards(lib_, 3, 1, init, [x], chunks)
    assert [len(st) for st in stages] == [1, 1, 1]
    _check_ranges(stages, 3)
    o = orc.OracleTwoStage()
    o.init(head, tail, h)
    assert _err(y[0], o.process(x)) <= TOL


@pytest.mark.parametrize("backend", BACKENDS)
def test_many_channels_through_the_exchange(backend):
    """17 convolvers with 8192-sample tail blocks: 17 x 16 (channel, bin tile) tickets in the exchange sweep, more than
    a handle of up to 8 channels needs."""
    lib_ = get_lib(backend)
    C, head, tail = 17, 512, 8192
    n = tail * 5 + 300
    irs = [synth_ir(5 * tail - 77, c) for c in range(C)]
    xs = [synth_input(n, c) for c in range(C)]
    chunks = _ragged(n, head, seed=21)
    init = lambda e: e.init_twostage(head, tail, irs)       # noqa: E731
    y, stages = _run_shards(lib_, 2, C, init, xs, chunks)
    _check_ranges(stages, 2)
    ref = _unsharded(lib_, C, init, xs, chunks)
    for c in range(C):
        o = orc.OracleTwoStage()
        o.init(head, tail, irs[c])
        assert _err(y[c], o.process(xs[c])) <= TOL, c
        assert _err(y[c], ref[c]) <= TOL, c


@pytest.mark.parametrize("G", [2, 3])
@pytest.mark.parametrize("backend", BACKENDS)
def test_reduce_hook_runs_once_per_tail_block(backend, G):
    """Sequential stand-in for the reduce: ranks 1..G-1 run first and park their partial spectra, rank 0's hook adds
    them.  The hook sees one tail block at a time (the head is never reduced), in the same order on every rank."""
    from tests.test_distributed import _add, _read
    lib_ = get_lib(backend)
    blocks, offsets, n_ir, n = THREE_STAGE[backend]
    h, x = synth_ir(n_ir), synth_input(n)
    chunks = _ragged(n, blocks[0], seed=13)
    parked, sizes = {}, {}

    def make_hook(rank):
        state = {"i": 0}

        def hook(ptr, nf, stream):
            if backend == "cuda":
                import torch
                torch.cuda.synchronize()
            i = state["i"]
            state["i"] += 1
            sizes.setdefault(rank, []).append(nf)
            if rank != 0:
                parked.setdefault(i, []).append(_read(backend, ptr, nf))
            else:
                for v in parked.get(i, []):
                    _add(backend, ptr, nf, v)
            return 0
        return hook

    y = None
    for rank in list(range(1, G)) + [0]:
        e = Engine(1, shard_rank=rank, shard_count=G, shard_head=False, lib=lib_)
        assert e.init_stages(blocks, offsets, [h])
        e.set_reduce(make_hook(rank))
        ys, pos = [], 0
        for k in chunks:
            ys.append(e.process([x[pos:pos + k]])[0])
            pos += k
        if rank == 0:
            y = np.concatenate(ys)
        e.close()
    # one call per completed tail block, each one row of its stage (C * B float2), never a head row
    assert sorted(set(sizes[0])) == sorted(2 * B for B in blocks[1:])
    for B in blocks[1:]:
        assert sizes[0].count(2 * B) == n // B
    assert all(sizes[r] == sizes[0] for r in range(1, G))
    truth = scipy.signal.fftconvolve(x.astype(np.float64), h.astype(np.float64))[:n]
    assert _err(y, truth) <= TOL


def test_refusals():
    lib_ = get_lib("emu")
    h = synth_ir(5000)
    # the layout is chosen before the IR is loaded
    e = Engine(2, shard_rank=0, shard_count=2, lib=lib_)
    assert e.init_twostage(16, 256, [h, h])
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        e.set_option("shard_head", 0)
    # the slot exchange still refuses a staged handle whose head is sharded
    with pytest.raises(B200ConvError, match="single-stage"):
        e.p2p_export(mode=1)
    e.close()
    # the send / wet chain stays refused on sharded handles, the tail layout included
    t = Engine(2, shard_rank=0, shard_count=2, shard_head=False, lib=lib_)
    assert t.init_twostage(16, 256, [h, h])
    with pytest.raises(B200ConvError, match=r"\(-3\)"):
        t.chain_configure(48000.0)
    t.reset()
    t.set_option("shard_head", 1)        # after a reset the layout can change again
    t.close()


@pytest.mark.gpu
def test_rank0_real_time_call_is_one_launch():
    """Rank 0 of a tail-sharded quad handle: a 128-sample call that completes no tail block is one launch, as on an
    unsharded handle, and its output matches the unsharded engine."""
    lib_ = get_lib("cuda")
    head, tail, n_ir, C, _ = TWO_STAGE["cuda"]
    irs = [synth_ir(n_ir, c) for c in range(C)]
    xs = [synth_input(head * 8, c) for c in range(C)]
    e = Engine(C, shard_rank=0, shard_count=4, shard_head=False, lib=lib_)
    u = Engine(C, lib=lib_)
    assert e.init_twostage(head, tail, irs) and u.init_twostage(head, tail, irs)
    for i in range(8):
        blk = [x[i * head:(i + 1) * head] for x in xs]
        l0, m0 = e.launch_count, u.launch_count
        ye, yu = e.process(blk), u.process(blk)
        assert e.launch_count - l0 == 1 and u.launch_count - m0 == 1
        for c in range(C):
            np.testing.assert_allclose(ye[c], yu[c], rtol=0, atol=1e-6)
    e.close()
    u.close()
