"""Host-clock time of a real-time call at zero latency and in fixed-latency mode (b200conv_set_latency).

  python tools/latency_bench.py [--warmup 200] [--calls 2000] [--out result.json]

Workload: REEV-R's quad two-stage handle (head 128, tail 8192) holding 10 s IRs at 48 kHz, host calls of 128 samples
paced by a full callback period of sleep after every call (2.67 ms, not timed; no catch-up after a host stall, which
would make calls follow each other back to back).  Two entry points:
  process  b200conv_process with the quad mixdown routing ({L, R} in, {L, R} out)
  chain    b200conv_chain_process: send filters, 10 ms predelay, the four convolvers, width and dry / wet mix
each at D = 0 (synchronous), 128 and 256 samples.  Every leg has its own handle; `warmup` untimed calls, then `calls`
timed ones.  Reports the median, p99 and maximum per call, the waits the latency mode counted (latency_waits), and the
card's name and power limit read in the same run, and the host-clock floor of a ctypes call into the library that does
no CUDA work (b200conv_latency), paced the same way.  Prints one JSON line.
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


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 2), "p99_us": round(float(np.percentile(a, 99)), 2),
            "max_us": round(float(a.max()), 2), "n": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from reevr_b200 import Engine
    from reevr_b200.convolver import _ptr_array
    from reevr_b200.synth import synth_input, synth_ir

    n_ir = int(IR_SECONDS * SRATE)
    irs = [synth_ir(n_ir, 7 + c) for c in range(4)]
    total = a.warmup + a.calls
    L, R = synth_input(total * BLOCK, 1), synth_input(total * BLOCK, 2)
    ys = np.full(total * BLOCK, 0.9, np.float32)
    yr = np.full(total * BLOCK, 0.8, np.float32)
    period = BLOCK / SRATE
    legs = {}
    for kind in ("process", "chain"):
        for D in (0, HEAD, 2 * HEAD):
            e = Engine(4)
            assert e.init_twostage(HEAD, TAIL, irs)
            if kind == "chain":
                e.chain_configure(**CHAIN)
            else:
                e.set_routing([0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]])
            e.set_latency(D)
            # host buffers of one call, reused: the timed region is the C call alone
            ins, outs, ev = ([np.zeros(BLOCK, np.float32) for _ in range(2)] for _ in range(3))
            pin, pout = _ptr_array(ins), _ptr_array(outs)
            lib, h = e._l, e._h
            times = []
            waits0 = 0
            for i in range(total):
                sl = slice(i * BLOCK, (i + 1) * BLOCK)
                ins[0][:] = L[sl]
                ins[1][:] = R[sl]
                ev[0][:] = ys[sl]
                ev[1][:] = yr[sl]
                if i == a.warmup:
                    waits0 = e.latency_waits
                t0 = time.perf_counter()
                if kind == "chain":
                    rc = lib.b200conv_chain_process(h, pin, ev[0].ctypes.data, ev[1].ctypes.data, pout, BLOCK)
                else:
                    rc = lib.b200conv_process(h, pin, pout, BLOCK)
                t1 = time.perf_counter()
                assert rc == 0, lib.b200conv_last_error(h)
                if i >= a.warmup:
                    times.append((t1 - t0) * 1e6)
                time.sleep(period)
            legs[f"{kind}_D{D}"] = dict(stats(times), latency_waits=int(e.latency_waits - waits0))
            e.close()
    floor = []
    e = Engine(1)
    for _ in range(a.calls):
        t0 = time.perf_counter()
        e._l.b200conv_latency(e._h)
        floor.append((time.perf_counter() - t0) * 1e6)
        time.sleep(period)
    e.close()
    legs["ctypes_floor"] = stats(floor)
    res = {"metric": "latency_call_host_us", "shape": "quad two-stage 128/8192, 10 s IRs, 48 kHz, host block 128, paced",
           "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "legs": legs}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
