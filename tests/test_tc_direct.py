"""B = 512 launch groups on the tensor-core sweep take the direct form: the sweep stores its complex result bin-major and
the inverse FFT reads it there (the overlap state of the next group is gathered from it), with no transpose into Y
rows.  Checked across launch sequences that hand state from one form to the other, and on a time-slice rank whose
sweep starts one block early.  GPU only (the CPU emulation has no tensor-core sweep)."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests.backends import get_lib

pytestmark = pytest.mark.gpu
B = 512
TOL = 1e-5


def on_device(e, xs):
    """one device-resident call (a single launch group when the handle's batch holds it)"""
    import torch
    x = torch.from_numpy(np.stack(xs)).cuda()
    y = torch.zeros_like(x)
    n = x.shape[1]
    e.process_device(x.data_ptr(), n, y.data_ptr(), n, n, sync=True)
    return list(y.cpu().numpy())


def peak_err(y, ref):
    y = np.asarray(y, np.float64)
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(y - ref)) / max(np.max(np.abs(ref)), 1e-30))


def test_stale_time_line_past_the_group_end_is_zeroed():
    # The long call leaves huge samples (blocks 5000-5099) in the time-line scratch, where the shorter call's tiles read
    # past its own end.  They leave the history 100 blocks later and share no tile window with the long call's last
    # block (its tile starts at block 8192), so the short call's result is normal.
    lib = get_lib("cuda")
    nparts, long_t, short_t = 100, 8500, 4100
    irs = [orc.synth_ir(nparts * B - 3, c) for c in range(2)]
    x1 = [orc.synth_input(long_t * B, c) for c in range(2)]
    for x in x1:
        x[5000 * B:5100 * B] *= np.float32(1e30)
    x2 = [orc.synth_input(short_t * B, c + 2) for c in range(2)]
    ys = {}
    for tc in (1, 0):
        e = Engine(2, max_batch_blocks=long_t + 1, lib=lib)
        assert e.init_uniform(B, irs)
        e.set_option("tc", tc)
        on_device(e, x1)
        assert e.last_sweep_variant() == (40 if tc else 22)
        ys[tc] = on_device(e, x2)
        assert e.last_sweep_variant() == (40 if tc else 22)
        e.close()
    for c in range(2):
        assert np.isfinite(ys[1][c]).all()
        assert peak_err(ys[1][c], ys[0][c]) <= 4e-6


def test_mixed_launch_sequence_on_one_handle():
    # tensor-core group, real-time calls, tensor-core group (ragged), FFMA group, tensor-core group: each one reads the
    # history the one before left in the X rows and the overlap state in Y row 0
    lib = get_lib("cuda")
    nparts, C = 100, 2
    irs = [orc.synth_ir(nparts * B - 11, c) for c in range(C)]
    calls = [(4200 * B, 1, 40)] + [(B, 1, None)] * 12 + [(4300 * B + 37, 1, 40), (4100 * B - 37, 0, 22), (4096 * B, 1, 40)]
    n = sum(k for k, _, _ in calls)
    xs = [orc.synth_input(n, c) for c in range(C)]
    e = Engine(C, max_batch_blocks=4400, lib=lib)
    assert e.init_uniform(B, irs)
    outs = [[] for _ in range(C)]
    pos = 0
    for k, tc, variant in calls:
        e.set_option("tc", tc)
        seg = [np.ascontiguousarray(x[pos:pos + k]) for x in xs]
        ys = on_device(e, seg) if variant is not None else e.process(seg)
        if variant is not None:
            assert e.last_sweep_variant() == variant
        for c in range(C):
            outs[c].append(ys[c])
        pos += k
    e.close()
    for c in range(C):
        o = orc.OracleUniform()
        o.init(B, irs[c])
        assert peak_err(np.concatenate(outs[c]), o.process(xs[c])) <= TOL


def test_sliced_rank_with_an_early_block():
    # rank 1's slice of 4200 blocks starts behind a forward-FFT-only advance: its sweep starts one block early and
    # computes the overlap state itself
    lib = get_lib("cuda")
    G, nparts, T, C = 2, 100, 8400, 2
    irs = [orc.synth_ir(nparts * B - 5, c) for c in range(C)]
    n = 2 * T * B
    xs = [orc.synth_input(n, c) for c in range(C)]
    engs = [Engine(C, max_batch_blocks=T // G + 1, lib=lib) for _ in range(G)]
    for e in engs:
        assert e.init_uniform(B, irs)
    import torch
    outs = [np.full(n, np.nan, np.float32) for _ in range(C)]
    for call in range(2):
        x = torch.from_numpy(np.stack([xx[call * T * B:(call + 1) * T * B] for xx in xs])).cuda()
        y = torch.full_like(x, float("nan"))
        for g in range(G):
            engs[g].process_device_sliced(x.data_ptr(), T * B, y.data_ptr(), T * B, T * B, g, G, sync=True)
            assert engs[g].last_sweep_variant() == 40
        for c in range(C):
            outs[c][call * T * B:(call + 1) * T * B] = y[c].cpu().numpy()
    for e in engs:
        e.close()
    whole = Engine(C, max_batch_blocks=T + 1, lib=lib)
    assert whole.init_uniform(B, irs)
    ref = [np.concatenate(p) for p in zip(*[on_device(whole, [x[i * T * B:(i + 1) * T * B] for x in xs]) for i in range(2)])]
    whole.close()
    for c in range(C):
        assert not np.isnan(outs[c]).any()
        assert peak_err(outs[c], ref[c]) <= 4e-6
        o = orc.OracleUniform()
        o.init(B, irs[c])
        assert peak_err(outs[c], o.process(xs[c])) <= TOL
