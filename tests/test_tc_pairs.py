"""Tensor-core sweep (cmac_variant 40) at every tile count a launch group can end on: launch groups of exactly and one
past a multiple of 4096 blocks (1 to 4 tiles of 64 segments x 64 blocks per bin, the last one full or holding a single
block), one and four channels, a single partition and the largest supported count, bins of 32 and 512.  Each case makes
two calls of the group, so the second sweep starts from the history the first left.  Checked against the FFMA sweep of
the same engine (4e-6 of peak) and the oracle (FFTConvolver.cpp:176-187 restated, 1e-5).  GPU only."""
import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests.backends import get_lib

pytestmark = pytest.mark.gpu


def peak_err(y, ref):
    y = np.asarray(y, np.float64)
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(y - ref)) / max(np.max(np.abs(ref)), 1e-30))


@pytest.mark.parametrize("B,nparts,C,nb", [
    (32, 961, 1, 4096), (32, 961, 1, 4097), (32, 961, 1, 8192), (32, 961, 1, 8193), (32, 961, 1, 12288), (32, 961, 1, 12289),
    (512, 1, 4, 4096), (512, 1, 4, 8193), (32, 1, 4, 12289), (512, 961, 1, 4097), (32, 961, 4, 8192),
])
def test_tc_sweep_tile_counts(B, nparts, C, nb):
    lib = get_lib("cuda")
    irs = [orc.synth_ir(nparts * B - (3 if nparts > 1 else 0), c) for c in range(C)]
    xs = [orc.synth_input(2 * nb * B, c) for c in range(C)]
    ys = {}
    for variant in (40, 22):
        e = Engine(C, cmac_variant=variant, max_batch_blocks=nb + 1, lib=lib)
        assert e.init_uniform(B, irs)
        outs = [[] for _ in range(C)]
        for call in range(2):
            part = e.process([x[call * nb * B:(call + 1) * nb * B] for x in xs])
            assert e.last_sweep_variant() == variant
            for c in range(C):
                outs[c].append(part[c])
        ys[variant] = [np.concatenate(o) for o in outs]
        e.close()
    for c in range(C):
        o = orc.OracleUniform()
        o.init(B, irs[c])
        ref = o.process(xs[c])
        assert peak_err(ys[40][c], ref) <= 1e-5
        assert peak_err(ys[40][c], ys[22][c]) <= 4e-6
