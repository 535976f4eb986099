"""A / B timing of the tensor-core sweep (cmac_variant 40) between builds of libb200conv.so, at the metric shape.

  python tools/tc_sweep_bench.py --lib base=path/to/old/libb200conv.so --lib new=reevr_b200/libb200conv.so [--out DIR]

Every library is loaded by path (several builds of the same C ABI live side by side in one process) and drives its own
engine over the same device-resident input: stereo, 10 s IR at 48 kHz, block 512 (P = 938), 112 608 blocks per step, the
shape and batch of bench.py's headline.  Reported per library:
  * step time: CUDA events around one process_device call, L2 flushed before each, the libraries alternated round by
    round (`--rounds` rounds of `--steps` steps each), median and min - max;
  * per-kernel device time per step from torch.profiler (a separate pass after the timed one);
  * k_tc_sweep's executed tensor rate: tiles x (Q/64 + 1) K chunks x 18 m64n128k16-equivalents (3 products x
    4 k-steps x the 3xFP16 split, as m64n64k16) over its profiled time, and that rate over the data sheet's dense FP16
    rate (989 TFLOP/s, H100 SXM at 700 W).  `k_tc_sweep_tflops_four_product` counts the four real products of the
    earlier form (24 equivalents per chunk and tile, what bench.py's roofline counts): the executed rate of a build of
    that form, 4/3 of the executed rate of this one;
  * max |y - y_first| / peak against the first library's output of the same step (a build of the earlier tf32 form as
    the first library shows how far the FP16 form moved the outputs).
The card's name, power limit and SM clocks are read in the same run.  Needs a GPU; there is no CPU path."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from reevr_b200 import _lib  # noqa: E402
from reevr_b200.convolver import Engine  # noqa: E402
from reevr_b200.synth import synth_input, synth_ir  # noqa: E402

C, SR, IR_S, BLOCK, T = 2, 48000, 10, 512, 112608
FP16_DENSE_TFLOPS = 989.0               # H100 SXM data sheet, dense FP16 / BF16 with FP32 accumulate


def card_info() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm,temperature.gpu",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, sm, smax, temp = [v.strip() for v in out.split(",")]
        info.update(power_limit_w=float(pl), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(smax), temperature_c=float(temp))
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"not available: {e}"
    return info


def tc_flop(P: int, nb: int, products: int = 3) -> float:
    q = (max(P - 1, 0) + 63) // 64 * 64
    nchunk = q // 64 + 1
    ntile = -(-(-(-nb // 64)) // 64)
    return float(C * BLOCK * ntile * nchunk * 6 * products) * 2.0 * 128 * 64 * 16


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, metavar="NAME=PATH", help="a build of libb200conv.so (repeat)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4, help="timed steps per library per round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tc_sweep_bench needs a CUDA device")
    libs = []
    for spec in args.lib:
        name, path = spec.split("=", 1)
        libs.append((name, _lib.load(os.path.abspath(path))))

    n = T * BLOCK
    irs = [synth_ir(IR_S * SR, c) for c in range(C)]
    x = torch.from_numpy(np.stack([synth_input(n, c) for c in range(C)])).cuda()
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")    # > 50 MB L2
    engines, ys = {}, {}
    for name, lib in libs:
        e = Engine(C, max_batch_blocks=T + 1, lib=lib)
        assert e.init_uniform(BLOCK, irs)
        engines[name] = e
        ys[name] = torch.empty_like(x)
    P = int(engines[libs[0][0]].stages()[0]["partitions"])

    def step(name):
        engines[name].process_device(x.data_ptr(), n, ys[name].data_ptr(), n, n, sync=False)

    for name, _ in libs:
        engines[name].clear()
        for _ in range(args.warmup):
            step(name)
        torch.cuda.synchronize()
        assert engines[name].last_sweep_variant() == 40, f"{name}: the metric shape did not run the tensor-core sweep"

    # same input from a cleared state: every library computes the same step
    out = {}
    for name, _ in libs:
        engines[name].clear()
        step(name)
        torch.cuda.synchronize()
        out[name] = ys[name].clone()
    first = libs[0][0]
    peak = float(out[first].abs().max())
    parity = {name: float((out[name] - out[first]).abs().max()) / peak for name, _ in libs}
    del out

    times = {name: [] for name, _ in libs}
    card_before = card_info()
    for _ in range(args.rounds):
        for name, _ in libs:
            stream = torch.cuda.ExternalStream(engines[name].stream)
            for _ in range(args.steps):
                flush.zero_()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                step(name)
                b.record(stream)
                b.synchronize()
                times[name].append(a.elapsed_time(b))
    card_after = card_info()

    kernels = {}
    from torch.profiler import ProfilerActivity, profile
    for name, _ in libs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                flush.zero_()
                step(name)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0 and not ev.key.startswith(("void at::", "Memset", "Memcpy")):
                per[ev.key] = per.get(ev.key, 0.0) + t / 1e3 / args.profile_steps
        kernels[name] = dict(sorted(per.items(), key=lambda kv: -kv[1]))

    flop, flop4 = tc_flop(P, T), tc_flop(P, T, products=4)
    res = {"shape": {"C": C, "block": BLOCK, "partitions": P, "blocks_per_step": T}, "card_before": card_before,
           "card_after": card_after, "libs": {}}
    for name, _ in libs:
        ts = times[name]
        sweep_ms = sum(v for k, v in kernels[name].items() if "k_tc_sweep" in k)
        res["libs"][name] = {
            "step_ms_median": statistics.median(ts), "step_ms_min": min(ts), "step_ms_max": max(ts), "steps": len(ts),
            "k_tc_sweep_ms": sweep_ms, "k_tc_sweep_tflops": flop / (sweep_ms * 1e-3) / 1e12 if sweep_ms > 0 else None,
            "k_tc_sweep_frac_of_fp16_dense": flop / (sweep_ms * 1e-3) / 1e12 / FP16_DENSE_TFLOPS if sweep_ms > 0 else None,
            "k_tc_sweep_tflops_four_product": flop4 / (sweep_ms * 1e-3) / 1e12 if sweep_ms > 0 else None,
            "max_err_vs_" + first: parity[name],
            "kernels_ms_per_step": {k: round(v, 4) for k, v in kernels[name].items()},
        }
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tc_sweep_bench.json"), "w") as f:
            f.write(line)
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
