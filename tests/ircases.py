"""The case matrix of tests/test_ir_recalc.py and of tests/golden/pins/impulse_pins.npz: Impulse::recalcImpulse
(src/dsp/Impulse.cpp:299-360) with resampling to the project rate, stretch, the parametric EQ and the decay EQ."""
import itertools

import numpy as np

from reevr_b200.synth import synth_ir

# (ir_srate, srate): equal, 48k -> 44.1k, 44.1k -> 48k, 96k -> 44.1k, 44.1k -> 96k, and a ratio inside (0.9999, 1.0001)
# that is still resampled (|ir_srate - srate| > 1e-6): linear interpolation without the low pass
RATES = ((48000.0, 48000.0), (48000.0, 44100.0), (44100.0, 48000.0), (96000.0, 44100.0), (44100.0, 96000.0),
         (48000.5, 48000.0))
STRETCHES = (-1.0, -0.3, 0.0, 0.25, 1.0)
# bands (mode, freq, q, gain) in REEV-R's order (src/PluginProcessor.cpp:225-233): HP / LS / HP6 first, BP / PK / Off in the
# middle, LP / HS / LP6 last.  Modes: 0 LP, 1 BP, 2 HP, 3 LS, 4 HS, 5 PK, 6 BS, 7 HP6, 8 LP6, 9 Off (run as PK).
PARAM_EQS = (
    (),
    ((7, 80.0, 0.7, 1.0), (5, 400.0, 0.9, 0.5), (5, 2500.0, 1.4, 2.0), (8, 12000.0, 0.7, 1.0)),
    ((3, 250.0, 0.7, 1.6), (9, 700.0, 0.7, 1.8), (9, 3000.0, 1.1, 0.6), (4, 6000.0, 0.7, 0.5)),
    ((2, 120.0, 0.9, 1.0), (1, 900.0, 0.8, 1.0), (1, 3000.0, 2.0, 1.0), (0, 12000.0, 0.8, 1.0)),
    ((2, 60.0, 0.7, 1.0), (6, 1000.0, 1.5, 1.0), (5, 5000.0, 0.7, 1.3), (0, 15000.0, 0.7, 1.0)),
)
DECAY_EQS = (
    ((), 1.0),
    (((3, 400.0, 0.7, 2.0), (5, 2500.0, 0.8, 0.4), (9, 1000.0, 0.7, 1.5), (4, 8000.0, 0.7, 0.25)), 0.5),
    (((7, 200.0, 0.7, 1.0), (8, 5000.0, 0.7, 1.0)), 2.0),
)


def cases():
    """(name, n, C, recalc keywords) of every case; the raw taps come from raw(n, C)."""
    out = []
    for i, ((ir_sr, sr), st) in enumerate(itertools.product(RATES, STRETCHES)):
        deq, rate = DECAY_EQS[i % 3]
        kw = dict(ir_srate=ir_sr, srate=sr, stretch=st, reverse=i % 4 == 1, trim_left=0.05 if i % 3 == 0 else 0.0,
                  trim_right=0.1 if i % 3 == 0 else 0.0, gain=1.5 if i % 2 else 1.0, param_eq=PARAM_EQS[i % 5],
                  decay_eq=deq, decay_rate=rate, attack=0.01 if i % 5 == 2 else 0.0, decay=0.2 if i % 5 == 3 else 0.0)
        out.append((f"m{i:02d}", 6000, 2 if i % 2 == 0 else 4, kw))
    out += [
        ("one_tap_up", 1, 2, dict(ir_srate=44100.0, srate=48000.0, stretch=0.25, param_eq=PARAM_EQS[1])),
        ("one_tap_quad", 1, 4, dict(ir_srate=48000.0, srate=48000.0, stretch=-0.3, param_eq=PARAM_EQS[2])),
        ("short_quad", 3000, 4, dict(ir_srate=96000.0, srate=44100.0, stretch=-0.3, param_eq=PARAM_EQS[3],
                                     decay_eq=DECAY_EQS[1][0], decay_rate=2.0)),
        ("long_down", 20000, 2, dict(ir_srate=48000.0, srate=44100.0, stretch=1.0, param_eq=PARAM_EQS[2],
                                     decay_eq=DECAY_EQS[2][0], decay_rate=0.5, reverse=True)),
        ("long_up_quad", 20000, 4, dict(ir_srate=44100.0, srate=96000.0, stretch=-1.0, param_eq=PARAM_EQS[4])),
        ("trim_empty", 5000, 2, dict(ir_srate=48000.0, srate=44100.0, stretch=0.25, trim_left=0.6, trim_right=0.5)),
    ]
    return out


def raw(n, C):
    """C raw channels {LL, RR[, LR, RL]} of n taps, with different levels so that the auto gain matters."""
    return [synth_ir(n, c) * np.float32(1.0 + 0.5 * c) for c in range(C)]
