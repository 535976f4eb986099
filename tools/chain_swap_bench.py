"""Times an IR hot swap inside the device chain (b200conv_chain_swap) at REEV-R's shape.

  python tools/chain_swap_bench.py [--swaps 8] [--steady 200] [--no-reference]

Workload: quad two-stage handles (head 128, tail 8192) holding 10 s IRs at 48 kHz, the send / wet chain with both cut
filters on and a 10 ms predelay, host calls of 128 samples (one callback period = 2.67 ms).  Every call is timed on the
host clock around b200conv_chain_process, which returns after its final synchronise.  One swap = the warm-up call (replay
of 93 host blocks of history plus the call's own audio), the fading calls and the call that completes the 50 ms fade;
the handles then trade places (double buffering) and the next swap follows after `--steady` plain calls.  The first
swap is a warm-up of the measurement and is not counted.

The host leg replays the same sequence through the reference's own TwoStageFFTConvolver (compiled into oracle/_ref):
93 x 2 warm-up process() calls of 128 samples (LL and RR of the incoming IR), then per fading callback the incoming
LL / RR plus the four outgoing convolvers.  Prints one JSON line with the card's name and power limit read in the same run.
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
    if not ms:
        return None
    a = np.asarray(ms)
    return {"median_ms": round(float(np.median(a)), 4), "min_ms": round(float(a.min()), 4),
            "p90_ms": round(float(np.percentile(a, 90)), 4), "max_ms": round(float(a.max()), 4), "n": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--swaps", type=int, default=8)
    ap.add_argument("--steady", type=int, default=200)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()

    import torch
    from reevr_b200 import Engine
    from reevr_b200.synth import synth_input, synth_ir

    n_ir = int(IR_SECONDS * SRATE)
    irsets = [[synth_ir(n_ir, 4 * k + c) for c in range(4)] for k in range(2)]
    L, R = synth_input(BLOCK * 4096, 0), synth_input(BLOCK * 4096, 1)
    ysend = np.ones(BLOCK, np.float32)
    yrev = np.ones(BLOCK, np.float32)
    live, inc = Engine(4, device=0), Engine(4, device=0)
    assert live.init_twostage(HEAD, TAIL, irsets[0]) and inc.init_twostage(HEAD, TAIL, irsets[1])
    live.chain_configure(**CHAIN)
    pos = 0

    def call():
        nonlocal pos
        k = pos % (L.size // BLOCK)
        t = time.perf_counter()
        live.chain_process(L[k * BLOCK:(k + 1) * BLOCK], R[k * BLOCK:(k + 1) * BLOCK], ysend, yrev)
        pos += 1
        return (time.perf_counter() - t) * 1e3

    steady, warm, fading, completing, fade_calls = [], [], [], [], []
    for s in range(a.swaps + 1):
        st = [call() for _ in range(a.steady)]
        live.chain_swap(inc, BLOCK)
        w = call()
        fd, nf = [], 1
        while live.chain_swap_state() != 3:
            fd.append(call())
            nf += 1
        comp = fd.pop()
        if s > 0:
            steady += st; warm.append(w); fading += fd; completing.append(comp); fade_calls.append(nf)
        live, inc = inc, live                          # std::swap(loadConvolver, convolver)
        assert inc.init_twostage(HEAD, TAIL, irsets[s % 2])
    period_ms = BLOCK / SRATE * 1e3
    res = {"workload": f"quad two-stage head {HEAD} tail {TAIL}, {IR_SECONDS:g} s IR at {SRATE / 1000:g} kHz, host block {BLOCK}",
           "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "callback_period_ms": round(period_ms, 4), "calls_per_swap": int(np.median(fade_calls)) if fade_calls else None,
           "gpu_steady_call": stats(steady), "gpu_warm_up_call": stats(warm), "gpu_fading_call": stats(fading),
           "gpu_completing_call": stats(completing)}
    res["warm_up_call_exceeds_period"] = bool(warm) and float(np.median(warm)) > period_ms
    live.close(); inc.close()

    ref = None
    if not a.no_reference:
        from oracle import oracle as orc
        if orc.ref_available():
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
            W = int(np.ceil(SRATE)) // 4
            nblocks = W // BLOCK
            fade = int(np.ceil(SRATE * 50 / 1000.0))
            warm_ms, fade_ms = [], []
            outgoing = []
            for c in range(4):
                o = orc.RefTwoStage()
                assert o.init(HEAD, TAIL, irsets[0][c])
                outgoing.append(o)
            for rep in range(3):
                incoming = []
                for c in range(2):
                    o = orc.RefTwoStage()
                    assert o.init(HEAD, TAIL, irsets[1][c])
                    incoming.append(o)
                x = L[:BLOCK]
                t = time.perf_counter()
                for _ in range(nblocks):
                    for o in incoming:
                        o.process(x)
                warm_ms.append((time.perf_counter() - t) * 1e3)
                for _ in range((fade + BLOCK - 1) // BLOCK):
                    t = time.perf_counter()
                    for o in outgoing + incoming:
                        o.process(x)
                    fade_ms.append((time.perf_counter() - t) * 1e3)
            ref = {"cpu_reference_warm_up": stats(warm_ms), "cpu_reference_fading_callback": stats(fade_ms),
                   "warm_up_process_calls": 2 * nblocks}
    res["cpu_reference"] = ref if ref is not None else "not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
