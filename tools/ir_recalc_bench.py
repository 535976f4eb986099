"""Times the whole IR recalculation (Impulse::recalcImpulse) on the device against the reference on one CPU core.

  python tools/ir_recalc_bench.py [--seconds 120] [--reps 5] [--no-reference]

Workload: a quad IR of `seconds` recorded at 44.1 kHz loaded into a 48 kHz session, stretch 0.5, four parametric-EQ bands
and four decay-EQ bands.  The device leg is b200conv_init_twostage_recalc (head 512, tail 8192: upload, recalculation and
the partition spectra, taps never return to the host), timed with CUDA events around the call plus a synchronise, after
one warm-up call.  The CPU leg is the reference's own Impulse::recalcImpulse compiled into oracle/_ref/librefimpulse.so,
pinned to one core.  Prints one JSON line, with the card's name and power limit read in the same run.
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

PARAM_EQ = ((3, 200.0, 0.7, 1.5), (5, 800.0, 1.0, 0.6), (5, 3000.0, 1.2, 1.8), (4, 9000.0, 0.7, 0.7))
DECAY_EQ = ((3, 300.0, 0.7, 2.0), (5, 1500.0, 0.8, 0.5), (9, 4000.0, 0.7, 1.4), (4, 10000.0, 0.7, 0.3))


def recalc_params(seconds):
    return dict(ir_srate=44100.0, srate=48000.0, stretch=0.5, param_eq=PARAM_EQ, decay_eq=DECAY_EQ, decay_rate=1.0)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()

    import torch
    from reevr_b200 import Engine
    from reevr_b200.synth import synth_ir

    n = int(a.seconds * 44100)
    raws = [synth_ir(n, c) for c in range(4)]
    kw = recalc_params(a.seconds)
    e = Engine(4, device=0)
    assert e.init_twostage_recalc(512, 8192, raws, **kw)          # warm-up: context, modules, allocator
    times = []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        assert e.init_twostage_recalc(512, 8192, raws, **kw)
        t1.record()
        torch.cuda.synchronize()
        times.append(t0.elapsed_time(t1))
    taps = e.ir_len(0)
    e.close()
    res = {"workload": f"{a.seconds:g} s quad IR, 44.1 kHz -> 48 kHz, stretch 0.5, 4 param-EQ + 4 decay-EQ bands",
           "raw_taps": n, "taps_after_trim": int(taps), "device": torch.cuda.get_device_name(0),
           "power_limit_w": power_limit_w(), "gpu_init_twostage_recalc_ms_median": float(np.median(times)),
           "gpu_ms_all": [round(t, 3) for t in times]}
    if not a.no_reference:
        from oracle import recalc as rc
        if rc.ref_impulse_available():
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
            t = time.perf_counter()
            ref = rc.ref_ir_recalc(raws, **{k: v for k, v in kw.items()})
            res["cpu_reference_recalc_ms"] = (time.perf_counter() - t) * 1e3
            res["cpu_reference_taps"] = int(ref[0].size)
            res["speedup"] = res["cpu_reference_recalc_ms"] / res["gpu_init_twostage_recalc_ms_median"]
        else:
            res["cpu_reference_recalc_ms"] = None
    print(json.dumps(res))


if __name__ == "__main__":
    main()
