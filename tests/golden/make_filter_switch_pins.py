"""Generates tests/golden/pins/filter_switch_pins.npz: the SHA-256 of the reference Filter's float32 output while its
slope and frequency are switched mid-stream the way onSlider does it (setSlope + init, no reset;
src/PluginProcessor.cpp:837-848), computed by the UNMODIFIED reference compiled into oracle/_ref, so that the pin of
the restatement (oracle/params_oracle.c) also runs where the reference sources are absent.

  python -m tests.golden.make_filter_switch_pins
"""
import hashlib
import os

import numpy as np

from oracle import params

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "pins", "filter_switch_pins.npz")
RATES = (44100.0, 48000.0, 96000.0)
MODES = (0, 2)                          # LP (high cut), HP (low cut)
SEGMENT = 700
# (slope, frequency) per segment: every slope transition 6 -> 12 -> 24 -> 6 -> 24 -> 12 -> 6 dB, with frequency moves
# inside a slope and across it, up to the clamps of getCoeff (20 Hz, 0.48 srate)
SCHEDULES = (
    ((0, 300.0), (1, 300.0), (2, 1200.0), (0, 90.0), (2, 90.0), (1, 5000.0), (0, 5000.0), (0, 40.0)),
    ((2, 8000.0), (2, 180.0), (1, 15.0), (0, 19999.0), (1, 30000.0), (2, 55.5), (0, 1234.0), (1, 1234.0)),
)


def q_for(slope):
    return 0.0765 if slope == 2 else 0.2929


def signal():
    return np.random.default_rng(11).standard_normal(SEGMENT * max(len(s) for s in SCHEDULES)).astype(np.float32)


def run(cls, mode, srate, schedule):
    x = signal()
    slope, freq = schedule[0]
    f = cls(slope, mode, srate, freq, q_for(slope))
    out = []
    for k, (slope, freq) in enumerate(schedule):
        if k:
            f.set(slope, srate, freq, q_for(slope))
        out.append(f.run(x[k * SEGMENT:(k + 1) * SEGMENT]))
    return np.concatenate(out).astype(np.float32)


def digest(y):
    return hashlib.sha256(np.ascontiguousarray(y, np.float32).tobytes()).hexdigest()


def cases():
    for sr in RATES:
        for mode in MODES:
            for j, sched in enumerate(SCHEDULES):
                yield sr, mode, j, sched


def main():
    assert params.ref_switch_filter_available(), "needs oracle/_ref (the compiled reference)"
    np.savez_compressed(PATH, sha256=np.array([digest(run(params.RefSwitchFilter, m, sr, s)) for sr, m, _, s in cases()]))
    print(PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
