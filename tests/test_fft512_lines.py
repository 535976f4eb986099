"""B = 512 launch groups on the tensor-core sweep: the forward FFT writes the group's blocks straight into the sweep's
time lines in 16-sample tiles (X rows only for the history later calls read), k_tc_split_x fills only the history in
front of the group and the zero tail behind it.  Checked over call schedules whose groups end at many residues mod 16,
with an open partial block in front of a group, on a
time-slice rank whose sweep starts one block early, across real-time calls and an FFMA group that read the X rows the
fused forward FFT left out, and across timeline compactions.  Each result against the oracle and against the same
schedule with the tensor-core sweep off.  GPU only."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests.backends import get_lib
from tests.test_tc_direct import on_device, peak_err

pytestmark = pytest.mark.gpu
B = 512
TOL = 1e-5          # against the oracle
TOL_FFMA = 4e-6     # against the FFMA sweep of the same engine


def run_schedule(C, irs, xs, calls, batch, tc):
    """calls: samples per call; device-resident calls for groups of >= 4096 blocks, host calls otherwise"""
    e = Engine(C, max_batch_blocks=batch, lib=get_lib("cuda"))
    assert e.init_uniform(B, irs)
    e.set_option("tc", tc)
    outs, variants, pos = [[] for _ in range(C)], [], 0
    for k in calls:
        seg = [np.ascontiguousarray(x[pos:pos + k]) for x in xs]
        ys = on_device(e, seg) if k >= 4096 * B else e.process(seg)
        variants.append(e.last_sweep_variant())
        for c in range(C):
            outs[c].append(ys[c])
        pos += k
    e.close()
    return [np.concatenate(o) for o in outs], variants


def check(C, irs, xs, calls, batch, fused_calls):
    got, variants = run_schedule(C, irs, xs, calls, batch, 1)
    for i in fused_calls:
        assert variants[i] == 40, (i, variants)
    ffma, _ = run_schedule(C, irs, xs, calls, batch, 0)
    for c in range(C):
        assert np.isfinite(got[c]).all()
        assert peak_err(got[c], ffma[c]) <= TOL_FFMA
        o = orc.OracleUniform()
        o.init(B, irs[c])
        assert peak_err(got[c], o.process(xs[c])) <= TOL


@pytest.mark.parametrize("P", [938, 961])
@pytest.mark.parametrize("C", [1, 2])
def test_ragged_groups_behind_an_open_block(P, C):
    # an open partial block (3 blocks + 100 samples), then groups that start inside it and end on different residues
    # of the 16-block tiles, the last one with a partial block of its own
    irs = [orc.synth_ir(P * B - 7, c) for c in range(C)]
    calls = [3 * B + 100, 4099 * B + 300, 4101 * B - 400, 4109 * B + 5, 4096 * B + 13 * B - 5]
    xs = [orc.synth_input(sum(calls), c) for c in range(C)]
    check(C, irs, xs, calls, 4200, fused_calls=[1, 2, 3, 4])


def test_fused_group_then_real_time_calls_then_ffma_group():
    # the real-time calls and the FFMA group read their history from the X rows the fused forward FFT wrote for the
    # last blocks of its group only
    C, P = 2, 938
    irs = [orc.synth_ir(P * B - 3, c) for c in range(C)]
    calls = [4203 * B] + [B] * 5 + [200, B - 200]
    xs = [orc.synth_input(sum(calls) + 4100 * B + 4097 * B, c) for c in range(C)]
    lib = get_lib("cuda")
    e = Engine(C, max_batch_blocks=4300, lib=lib)
    assert e.init_uniform(B, irs)
    outs, pos = [[] for _ in range(C)], 0
    for k, tc, variant in [(k, 1, 40 if k >= 4096 * B else None) for k in calls] + [(4100 * B, 0, 22), (4097 * B, 1, 40)]:
        e.set_option("tc", tc)
        seg = [np.ascontiguousarray(x[pos:pos + k]) for x in xs]
        ys = on_device(e, seg) if k >= 4096 * B else e.process(seg)
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


def test_groups_across_timeline_compactions():
    # a batch of 4110 blocks: the X ring holds two histories and one batch, so it is compacted in front of every group
    # after the first
    C, P = 2, 961
    irs = [orc.synth_ir(P * B - 1, c) for c in range(C)]
    calls = [4100 * B, 4099 * B + 17, 4100 * B - 17, 4098 * B]
    xs = [orc.synth_input(sum(calls), c) for c in range(C)]
    check(C, irs, xs, calls, 4110, fused_calls=[0, 1, 2, 3])


@pytest.mark.parametrize("P", [938, 961])
def test_sliced_pair_with_an_early_block(P):
    # rank 1's slice starts behind a forward-FFT-only advance: its sweep starts one block early (tau = Q + 1 ...), so
    # its tiles and runs sit one sample off those of rank 0
    G, T, C = 2, 8210, 1
    irs = [orc.synth_ir(P * B - 5, c) for c in range(C)]
    xs = [orc.synth_input(T * B, c) for c in range(C)]
    import torch
    x = torch.from_numpy(np.stack(xs)).cuda()
    y = torch.full_like(x, float("nan"))
    for g in range(G):
        e = Engine(C, max_batch_blocks=T // G + 1, lib=get_lib("cuda"))
        assert e.init_uniform(B, irs)
        e.process_device_sliced(x.data_ptr(), T * B, y.data_ptr(), T * B, T * B, g, G, sync=True)
        assert e.last_sweep_variant() == 40
        e.close()
    got = list(y.cpu().numpy())
    whole = Engine(C, max_batch_blocks=T + 1, lib=get_lib("cuda"))
    assert whole.init_uniform(B, irs)
    whole.set_option("tc", 0)
    ref = on_device(whole, xs)
    whole.close()
    for c in range(C):
        assert not np.isnan(got[c]).any()
        assert peak_err(got[c], ref[c]) <= TOL_FFMA
        o = orc.OracleUniform()
        o.init(B, irs[c])
        assert peak_err(got[c], o.process(xs[c])) <= TOL
