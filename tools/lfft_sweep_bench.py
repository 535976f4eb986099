"""A / B timing of the two sweep forms of long launch groups in one process: the tensor-core Toeplitz sweep (cmac_variant
40, k_tc_sweep) against the line-FFT sweep (41, k_lfft_sweep), both forced, on one build of libb200conv.so.

  python tools/lfft_sweep_bench.py [--lib reevr_b200/libb200conv.so] [--groups 4224,16384,112608] [--out DIR]

Shape: stereo, 10 s IR at 48 kHz, block 512 (P = 938), device-resident input, one process_device call per step of
`group` blocks (112 608 is bench.py's headline group, 4 224 the default launch group).  Reported per group length:
  * step time of each form: CUDA events around one call, L2 flushed before each, the forms alternated round by round,
    median and min - max;
  * per-kernel device time per step from torch.profiler (a separate pass after the timed one);
  * for 41: k_lfft_sweep's bytes and FP32 flops per step from the shape, and the achieved GB/s (against 3.35 TB/s,
    H100 SXM data sheet) and TFLOP/s (against 67 TFLOP/s FP32).  Bytes: every segment's kN-sample window of the re and
    im planes, the Lty result slots written, the line spectra read once.  Flops: 5 kN log2 kN per complex transform
    (two per segment) plus 6 kN for the spectrum product.  k_lfft_build_h runs once per IR and is listed apart.
bench.py --dump-outputs compares the outputs of two builds.
The card's name, power limit and SM clocks are read in the same run.  Needs a GPU; there is no CPU path."""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from reevr_b200 import _lib  # noqa: E402
from reevr_b200.convolver import Engine  # noqa: E402
from reevr_b200.synth import synth_input, synth_ir  # noqa: E402
from tools.tc_sweep_bench import card_info  # noqa: E402

C, SR, IR_S, BLOCK = 2, 48000, 10, 512
KN = 4096                               # kernels_lfft.cuh kN
HBM_TBS, FP32_TFLOPS = 3.35, 67.0       # H100 SXM data sheet, 700 W


def lfft_counts(P: int, nb: int) -> tuple[float, float]:
    """(bytes, flops) of one k_lfft_sweep launch: kernels_lfft.cuh make_plan over kernels_tc.cuh make_geom"""
    ntile = -(-(-(-nb // 64)) // 64)
    lty = ntile * 64 * 64
    L = KN - (P - 1)
    nseg = -(-lty // L)
    lines = C * BLOCK
    nbytes = lines * nseg * KN * 8 + lines * lty * 8 + (lines + C) * KN * 8
    flops = lines * nseg * (2 * 5 * KN * math.log2(KN) + 6 * KN)
    return float(nbytes), float(flops)


def profile_kernels(step, flush, steps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            flush.zero_()
            step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0 and not ev.key.startswith(("void at::", "Memset", "Memcpy")):
            per[ev.key] = per.get(ev.key, 0.0) + t / 1e3 / steps
    return dict(sorted(per.items(), key=lambda kv: -kv[1]))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "reevr_b200", "libb200conv.so"))
    ap.add_argument("--groups", default="4224,16384,112608", help="blocks per step, comma separated")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3, help="timed steps per form per round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lfft_sweep_bench needs a CUDA device")
    lib = _lib.load(os.path.abspath(args.lib))
    irs = [synth_ir(IR_S * SR, c) for c in range(C)]
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")    # > 50 MB L2
    res = {"card_before": card_info(), "groups": {}}
    for T in [int(g) for g in args.groups.split(",")]:
        n = T * BLOCK
        x = torch.from_numpy(np.stack([synth_input(n, c) for c in range(C)])).cuda()
        engines, ys = {}, {}
        for v in (40, 41):
            e = Engine(C, max_batch_blocks=T + 1, cmac_variant=v, lib=lib)
            assert e.init_uniform(BLOCK, irs)
            engines[v], ys[v] = e, torch.empty_like(x)
        P = int(engines[40].stages()[0]["partitions"])

        def step(v):
            engines[v].process_device(x.data_ptr(), n, ys[v].data_ptr(), n, n, sync=False)

        for v in (40, 41):
            for _ in range(args.warmup):
                step(v)
            torch.cuda.synchronize()
            assert engines[v].last_sweep_variant() == v
        times = {40: [], 41: []}
        for _ in range(args.rounds):
            for v in (40, 41):
                stream = torch.cuda.ExternalStream(engines[v].stream)
                for _ in range(args.steps):
                    flush.zero_()
                    torch.cuda.synchronize()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    step(v)
                    b.record(stream)
                    b.synchronize()
                    times[v].append(a.elapsed_time(b))
        kernels = {v: profile_kernels(lambda v=v: step(v), flush, args.profile_steps) for v in (40, 41)}
        nbytes, flops = lfft_counts(P, T)
        sweep_ms = sum(t for k, t in kernels[41].items() if "k_lfft_sweep" in k)
        res["groups"][str(T)] = {
            "partitions": P,
            "step_ms": {str(v): {"median": statistics.median(times[v]), "min": min(times[v]), "max": max(times[v])} for v in (40, 41)},
            "speedup_41_over_40": statistics.median(times[40]) / statistics.median(times[41]),
            "k_tc_sweep_ms": sum(t for k, t in kernels[40].items() if "k_tc_sweep" in k),
            "k_lfft_sweep_ms": sweep_ms,
            "k_lfft_sweep_gbytes": nbytes / 1e9, "k_lfft_sweep_gflop": flops / 1e9,
            "k_lfft_sweep_gbs": nbytes / (sweep_ms * 1e-3) / 1e9 if sweep_ms > 0 else None,
            "k_lfft_sweep_frac_of_hbm": nbytes / (sweep_ms * 1e-3) / 1e12 / HBM_TBS if sweep_ms > 0 else None,
            "k_lfft_sweep_tflops": flops / (sweep_ms * 1e-3) / 1e12 if sweep_ms > 0 else None,
            "k_lfft_sweep_frac_of_fp32": flops / (sweep_ms * 1e-3) / 1e12 / FP32_TFLOPS if sweep_ms > 0 else None,
            "kernels_ms_per_step": {str(v): {k: round(t, 4) for k, t in kernels[v].items()} for v in (40, 41)},
        }
        # k_lfft_build_h: once per IR, timed on a fresh handle's first call
        e = Engine(C, max_batch_blocks=T + 1, cmac_variant=41, lib=lib)
        assert e.init_uniform(BLOCK, irs)
        k1 = profile_kernels(lambda: e.process_device(x.data_ptr(), n, ys[41].data_ptr(), n, n, sync=False), flush, 1)
        res["groups"][str(T)]["k_lfft_build_h_ms_once"] = sum(t for k, t in k1.items() if "k_lfft_build_h" in k)
        e.close()
        for e in engines.values():
            e.close()
        del x, ys
    res["card_after"] = card_info()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lfft_sweep_bench.json"), "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
