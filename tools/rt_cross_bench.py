"""A / B timing of real-time calls that cross a head-block boundary, between builds of libb200conv.so.

  python tools/rt_cross_bench.py --lib base=path/to/old/libb200conv.so --lib new=reevr_b200/libb200conv.so [--out DIR]

Host blocks that are not a power of two (480 samples at 48 kHz and 441 at 44.1 kHz both give head 512) cross a
head-block boundary on most calls.  Every library is loaded by path and drives its own handle over the same input; the
libraries take turns, round by round, each continuing its own stream.  Calls are paced like an audio callback: call k
starts no earlier than its samples' real-time deadline.  Legs:
  quad512            REEV-R's quad two-stage 512 / 8192, 10 s IRs, device mixdown (LL + RL, RR + LR), 512-sample
                     calls: none crosses, both builds run one launch per call (the cost of the two-segment kernel form
                     for calls that stay inside the open block);
  quad480 / quad441  the same handle at 480 samples (48 kHz) and 441 samples (44.1 kHz);
  chain480           the same handle through b200conv_chain_process (send / wet chain, true stereo);
  quadvar            the quad handle with seeded call lengths in [32, 512];
  uni256x600         uniform 256 with 600 partitions, C = 2, 200-sample calls (two serial sweeps in a crossing launch
                     stream 1.2 MB of spectra per convolver each).
Reported per leg and library: host-clock time per call (median / p99 / max, microseconds), launches per call, and the
output's max |y - y_first| / peak against the first library over the whole stream.  The card's name and power limit are
read in the same run.  Needs a GPU; there is no CPU path."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from reevr_b200 import _lib  # noqa: E402
from reevr_b200.convolver import Engine  # noqa: E402
from reevr_b200.synth import synth_input, synth_ir  # noqa: E402


def card_info() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, sm, smax = [v.strip() for v in out.split(",")]
        info.update(power_limit_w=float(pl), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(smax))
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"not available: {e}"
    return info


def quad_engine(lib, irs, chain=False):
    e = Engine(4, lib=lib)
    assert e.init_twostage(512, 8192, irs)
    if chain:
        e.chain_configure(srate=48000.0, lowcut_hz=80.0, lowcut_slope=1, highcut_hz=12000.0, highcut_slope=1,
                          predelay=240, width=1.0, drygain=0.7, wetgain=0.5, true_stereo=True)
    else:
        e.set_routing([0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]])
    return e


def legs(calls_per_leg: int):
    quad_irs = [synth_ir(480000, c) for c in range(4)]          # 10 s at 48 kHz: LL, RR, LR, RL
    uni_irs = [synth_ir(256 * 600 - 5, c) for c in range(2)]
    rng = np.random.default_rng(2026)
    var = [int(v) for v in rng.integers(32, 513, calls_per_leg)]
    return [
        ("quad512", lambda lib: quad_engine(lib, quad_irs), "process", [512] * calls_per_leg, 48000),
        ("quad480", lambda lib: quad_engine(lib, quad_irs), "process", [480] * calls_per_leg, 48000),
        ("quad441", lambda lib: quad_engine(lib, quad_irs), "process", [441] * calls_per_leg, 44100),
        ("chain480", lambda lib: quad_engine(lib, quad_irs, chain=True), "chain", [480] * calls_per_leg, 48000),
        ("quadvar", lambda lib: quad_engine(lib, quad_irs), "process", var, 48000),
        ("uni256x600", lambda lib: _uniform(lib, uni_irs), "process", [200] * calls_per_leg, 48000),
    ]


def _uniform(lib, irs):
    e = Engine(2, lib=lib)
    assert e.init_uniform(256, irs)
    return e


def run_leg(libs, make, kind, calls, sr, rounds, warmup):
    n = sum(calls)
    xs = [synth_input(n, c) for c in range(2)]
    env = [np.full(n, 0.8, np.float32), np.full(n, 0.9, np.float32)]
    engines = {name: make(lib) for name, lib in libs}
    outs = {name: [[], []] for name, _ in libs}
    times = {name: [] for name, _ in libs}
    launches = {name: [] for name, _ in libs}
    starts = np.concatenate([[0], np.cumsum(calls)])
    per_round = -(-len(calls) // rounds)
    for r0 in range(0, len(calls), per_round):
        for name, _ in libs:
            e = engines[name]
            t_next = time.perf_counter()
            for i in range(r0, min(r0 + per_round, len(calls))):
                sl = slice(int(starts[i]), int(starts[i + 1]))
                while time.perf_counter() < t_next:          # pace like an audio callback
                    pass
                t_next += calls[i] / sr
                l0 = e.launch_count
                t0 = time.perf_counter()
                if kind == "chain":
                    ys = e.chain_process(xs[0][sl], xs[1][sl], env[0][sl], env[1][sl])
                else:
                    ys = e.process([xs[0][sl], xs[1][sl]])
                dt = time.perf_counter() - t0
                if i >= warmup:
                    times[name].append(dt * 1e6)
                    launches[name].append(e.launch_count - l0)
                for c in range(2):
                    outs[name][c].append(ys[c])
    first = libs[0][0]
    ref = np.stack([np.concatenate(o) for o in outs[first]])
    peak = float(np.max(np.abs(ref)))
    res = {"calls": len(calls), "timed_calls": len(times[first]), "samples": n, "rate": sr, "libs": {}}
    for name, _ in libs:
        y = np.stack([np.concatenate(o) for o in outs[name]])
        t = np.array(times[name])
        res["libs"][name] = {
            "median_us": round(float(np.median(t)), 1), "p99_us": round(float(np.percentile(t, 99)), 1),
            "max_us": round(float(np.max(t)), 1), "launches_per_call": round(float(np.mean(launches[name])), 3),
            "max_diff_vs_" + first: float(np.max(np.abs(y - ref))) / peak,
        }
        engines[name].close()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, metavar="NAME=PATH", help="a build of libb200conv.so (repeat)")
    ap.add_argument("--calls", type=int, default=600, help="calls per leg and library")
    ap.add_argument("--rounds", type=int, default=4, help="turns each library takes per leg")
    ap.add_argument("--warmup", type=int, default=40, help="untimed calls at the start of each leg")
    ap.add_argument("--legs", default=None, help="comma-separated subset of the legs")
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rt_cross_bench needs a CUDA device")
    libs = []
    for spec in args.lib:
        name, path = spec.split("=", 1)
        libs.append((name, _lib.load(os.path.abspath(path))))
    res = {"card_before": card_info(), "legs": {}}
    for name, make, kind, calls, sr in legs(args.calls):
        if args.legs and name not in args.legs.split(","):
            continue
        res["legs"][name] = run_leg(libs, make, kind, calls, sr, args.rounds, args.warmup)
    res["card_after"] = card_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rt_cross_bench.json"), "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
