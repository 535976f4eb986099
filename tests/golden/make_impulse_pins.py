"""Generates tests/golden/pins/impulse_pins.npz: what tests/test_ir_recalc.py compares the restatement of
Impulse::recalcImpulse (oracle/recalc_oracle.c) against where the reference sources are absent, computed by the UNMODIFIED
reference compiled into oracle/_ref/librefimpulse.so (oracle/recalc.mk).

  python -m tests.golden.make_impulse_pins

For every case of tests/ircases.py: the output length, peak and SHA-256 of the float32 output (all channels), and a
seeded sample (positions + values) of it.
"""
import hashlib
import os

import numpy as np

from oracle import recalc
from tests import ircases

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "pins", "impulse_pins.npz")      # outside the glob of the replayable fixtures (golden/*.npz)
SAMPLES = 512


def sample_index(n):
    if n <= SAMPLES:
        return np.arange(n, dtype=np.int32)
    return np.unique(np.random.default_rng(n).integers(0, n, SAMPLES)).astype(np.int32)


def digest(chans):
    return hashlib.sha256(b"".join(np.ascontiguousarray(c, np.float32).tobytes() for c in chans)).hexdigest()


def main():
    assert recalc.ref_impulse_available(), "needs oracle/_ref/librefimpulse.so (the compiled reference)"
    out = {}
    for name, n, C, kw in ircases.cases():
        y = recalc.ref_ir_recalc(ircases.raw(n, C), **kw)
        m = y[0].size
        out[f"{name}/len"] = np.int64(m)
        out[f"{name}/sha256"] = np.array(digest(y))
        out[f"{name}/peak"] = np.float64(max(np.max(np.abs(c.astype(np.float64))) for c in y) if m else 0.0)
        idx = sample_index(m)
        out[f"{name}/index"] = idx
        out[f"{name}/value"] = np.stack([c[idx] for c in y]) if m else np.zeros((C, 0), np.float32)
    np.savez_compressed(PATH, **out)
    print(PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
