"""A / B timing of the two sweep forms of long B = 512 launch groups in one process: the line-FFT sweep (cmac_variant
41: k_fwd_fft512_lines, k_lfft_sweep, k_inv_fft512) against the four-step sweep (42: k_fs_cols, k_fs_rows,
k_fs_cols_inv), both forced, on one build of libb200conv.so.

  python tools/fourstep_bench.py [--lib reevr_b200/libb200conv.so] [--groups 32768,112608] [--out DIR]

Shape: stereo, 10 s IR at 48 kHz, block 512 (P = 938), device-resident input, one process_device call per step of
`group` blocks (112 608 is bench.py's headline group).  Reported per group length:
  * step time of each form: CUDA events around one call, L2 flushed before each, the forms alternated round by round,
    median and min - max;
  * per-kernel device time per step from torch.profiler (a separate pass after the timed one);
  * for 42, per pass: the bytes the pass must move (kernels_fourstep.cuh's plan: pass 1 reads every segment's M-sample
    window and writes its 257 x 4096 column spectra, pass 2 reads and rewrites them and reads the IR spectrum, pass 3
    reads them and writes the group's samples) and the achieved GB/s against 3.35 TB/s (H100 SXM data sheet).
The card's name, power limit and SM clocks are read in the same run.  Needs a GPU; there is no CPU path."""
from __future__ import annotations

import argparse
import json
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
from tools.lfft_sweep_bench import profile_kernels  # noqa: E402
from tools.tc_sweep_bench import card_info  # noqa: E402

C, SR, IR_S, BLOCK = 2, 48000, 10, 512
M, ROWS, N2 = 1 << 21, 257, 4096        # kernels_fourstep.cuh kM, kRows, kN2
HBM_TBS = 3.35                          # H100 SXM data sheet, 700 W
FORMS = (41, 42)


def pass_bytes(P: int, nb: int) -> dict:
    """bytes each pass of a four-step group must move (kernels_fourstep.cuh make_plan)"""
    n = nb * BLOCK
    L = M - (P * BLOCK - 1)
    nseg = -(-n // L)
    work = C * nseg * ROWS * N2 * 8
    return {"k_fs_cols": C * nseg * M * 4 + work, "k_fs_rows": 2 * work + C * ROWS * N2 * 8, "k_fs_cols_inv": work + C * n * 4}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "reevr_b200", "libb200conv.so"))
    ap.add_argument("--groups", default="32768,112608", help="blocks per step, comma separated")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3, help="timed steps per form per round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fourstep_bench needs a CUDA device")
    lib = _lib.load(os.path.abspath(args.lib))
    irs = [synth_ir(IR_S * SR, c) for c in range(C)]
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")    # > 50 MB L2
    res = {"card_before": card_info(), "groups": {}}
    for T in [int(g) for g in args.groups.split(",")]:
        n = T * BLOCK
        x = torch.from_numpy(np.stack([synth_input(n, c) for c in range(C)])).cuda()
        engines, ys = {}, {}
        for v in FORMS:
            e = Engine(C, max_batch_blocks=T + 1, cmac_variant=v, lib=lib)
            assert e.init_uniform(BLOCK, irs)
            engines[v], ys[v] = e, torch.empty_like(x)
        P = int(engines[41].stages()[0]["partitions"])

        def step(v):
            engines[v].process_device(x.data_ptr(), n, ys[v].data_ptr(), n, n, sync=False)

        for v in FORMS:
            for _ in range(args.warmup):
                step(v)
            torch.cuda.synchronize()
            assert engines[v].last_sweep_variant() == v
        times = {v: [] for v in FORMS}
        for _ in range(args.rounds):
            for v in FORMS:
                stream = torch.cuda.ExternalStream(engines[v].stream)
                for _ in range(args.steps):
                    flush.zero_()
                    torch.cuda.synchronize()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    step(v)
                    b.record(stream)
                    torch.cuda.synchronize()
                    times[v].append(a.elapsed_time(b))
        kernels = {v: profile_kernels(lambda v=v: step(v), flush, args.profile_steps) for v in FORMS}
        passes = {}
        for name, nbytes in pass_bytes(P, T).items():
            ms = sum(t for k, t in kernels[42].items() if k.split("(")[0].endswith(name) or f"{name}<" in k)
            passes[name] = {"ms": round(ms, 4), "gbytes": round(nbytes / 1e9, 4),
                            "gbs": nbytes / (ms * 1e-3) / 1e9 if ms > 0 else None,
                            "frac_of_hbm": nbytes / (ms * 1e-3) / 1e12 / HBM_TBS if ms > 0 else None}
        out_diff = float((ys[41] - ys[42]).abs().max() / ys[41].abs().max())
        res["groups"][str(T)] = {
            "partitions": P,
            "step_ms": {str(v): {"median": statistics.median(times[v]), "min": min(times[v]), "max": max(times[v])} for v in FORMS},
            "speedup_42_over_41": statistics.median(times[41]) / statistics.median(times[42]),
            "passes_42": passes,
            "max_diff_42_vs_41_of_peak": out_diff,
            "kernels_ms_per_step": {str(v): {k: round(t, 4) for k, t in kernels[v].items()} for v in FORMS},
        }
        for e in engines.values():
            e.close()
        del x, ys
    res["card_after"] = card_info()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fourstep_bench.json"), "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
