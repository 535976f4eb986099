"""Times chain parameter changes while playing (b200conv_chain_update) at REEV-R's shape.

  python tools/chain_params_bench.py [--calls 2000] [--growths 8]

Workload: a quad two-stage handle (head 128, tail 8192) holding a 10 s IR at 48 kHz, the send / wet chain with both
cut filters on and a 10 ms predelay, host calls of 128 samples (one callback period = 2.67 ms).  Every call is timed on
the host clock around b200conv_chain_process, which returns after its final synchronise.  Three kinds of call:
  steady      no parameter change;
  automation  b200conv_chain_update before every call (low cut sweep, width and dry / wet ramps); the call is timed
              with the update in front of it, and the update alone is reported too;
  growth      the call after an update whose predelay exceeds the delay line (D = 2 s at 48 kHz): the update grows the
              line (one synchronise and a reallocation of the ring) and is timed separately.  The chain is configured
              again before each growth so that every growth starts from the same D.
Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SRATE, HEAD, TAIL, BLOCK, IR_SECONDS = 48000.0, 128, 8192, 128, 10.0
CHAIN = dict(srate=SRATE, lowcut_hz=120.0, lowcut_slope=1, highcut_hz=12000.0, highcut_slope=2, predelay=480,
             width=0.8, drygain=0.7, wetgain=0.5, true_stereo=True)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": round(float(np.median(a)), 4), "min_ms": round(float(a.min()), 4),
            "max_ms": round(float(a.max()), 4), "n": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--growths", type=int, default=8)
    a = ap.parse_args()

    import torch
    from reevr_b200 import Engine
    from reevr_b200.synth import synth_input, synth_ir

    assert torch.cuda.is_available(), "the measurement needs a CUDA device"
    n_ir = int(IR_SECONDS * SRATE)
    e = Engine(4, device=0)
    assert e.init_twostage(HEAD, TAIL, [synth_ir(n_ir, c) for c in range(4)])
    e.chain_configure(**CHAIN)
    L, R = synth_input(BLOCK * 4096, 0), synth_input(BLOCK * 4096, 1)
    ysend, yrev = np.ones(BLOCK, np.float32), np.ones(BLOCK, np.float32)
    pos = 0

    def call():
        nonlocal pos
        k = pos % (L.size // BLOCK)
        t = time.perf_counter()
        e.chain_process(L[k * BLOCK:(k + 1) * BLOCK], R[k * BLOCK:(k + 1) * BLOCK], ysend, yrev)
        pos += 1
        return (time.perf_counter() - t) * 1e3

    for _ in range(300):
        call()
    steady, auto, upd = [], [], []
    for i in range(a.calls):                      # alternate the two kinds so that both see the same host noise
        steady.append(call())
        u = (i % 400) / 399.0
        cfg = dict(CHAIN, lowcut_hz=60.0 + 400.0 * u, width=2.0 * u, drygain=float(np.cos(u * np.pi / 2)),
                   wetgain=float(np.sin(u * np.pi / 2)))
        t = time.perf_counter()
        e.chain_update(**cfg)
        t1 = time.perf_counter()
        auto.append(call() + (t1 - t) * 1e3)
        upd.append((t1 - t) * 1e3)
    grow_update, grow_call = [], []
    for _ in range(a.growths):
        e.chain_configure(**CHAIN)
        for _ in range(200):
            call()
        t = time.perf_counter()
        e.chain_update(**dict(CHAIN, predelay=int(2.0 * SRATE) + 480))
        grow_update.append((time.perf_counter() - t) * 1e3)
        grow_call.append(call())
    e.close()
    res = {"workload": f"quad two-stage head {HEAD} tail {TAIL}, {IR_SECONDS:g} s IR at {SRATE / 1000:g} kHz, host block {BLOCK}",
           "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "callback_period_ms": round(BLOCK / SRATE * 1e3, 4),
           "steady_call": stats(steady), "automation_update_plus_call": stats(auto), "automation_update_alone": stats(upd),
           "growth_update": stats(grow_update), "call_after_growth": stats(grow_call)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
