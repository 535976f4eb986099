"""Times chain parameter events inside one device call (b200conv_chain_process_device_events) against the same
automation as cut calls.

  python tools/chain_events_bench.py [--rounds 2] [--steps 1] [--blocks 112608] [--workload metric|quad|both]
                                     [--every 512,4096,65536]

Workloads and chain: tools/chain_offline_bench.py's ("metric" = stereo, 10 s IR at 48 kHz, uniform block 512; "quad" =
REEV-R's quad two-stage 128 / 8192 with true stereo), a step of --blocks blocks of 512 frames.  The automation moves
the low cut (20.5 .. 220 Hz), the high cut (16 .. 12 kHz) and the width every P samples.  Legs, alternated over the
rounds after one warm-up step each, timed with CUDA events on the handle's stream:
  none        b200conv_chain_process_device, no events
  events_P    b200conv_chain_process_device_events with an event every P samples (the event array built beforehand)
  cuts_P      the same automation as b200conv_chain_update + b200conv_chain_process_device per P samples
Then: a window of events_512 against cuts_512 on fresh handles (<= 1e-5 of peak) and a torch.profiler run of one
events_512 step (per-kernel time).  Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from chain_offline_bench import CHAIN, make_engine, power_limit_w  # noqa: E402


def automation(n, every):
    ev = []
    for k, off in enumerate(range(0, n, every)):
        c = dict(CHAIN)
        c.update(lowcut_hz=20.5 + 10.0 * (k % 21), highcut_hz=16000.0 - 200.0 * (k % 21), width=0.5 + 0.05 * (k % 11))
        ev.append((off, c))
    return ev


def run_workload(wl, a, torch, Engine, synth_ir, synth_input, chain_event_array):
    n = a.blocks * 512
    x = torch.from_numpy(np.stack([synth_input(n, 0), synth_input(n, 1)])).cuda()
    t = np.arange(n, dtype=np.float64)
    env = torch.from_numpy(np.stack([(0.5 + 0.5 * np.abs(np.sin(t * 1e-4))).astype(np.float32),
                                     (0.25 + 0.75 * np.abs(np.cos(t * 3e-5))).astype(np.float32)])).cuda()
    out = torch.empty_like(x)
    ys, yr = env[0].data_ptr(), env[1].data_ptr()
    autos = {p: automation(n, p) for p in a.every}
    arrays = {p: chain_event_array(ev) for p, ev in autos.items()}     # built once, outside the timed legs

    def timed(e, fn):
        s = torch.cuda.ExternalStream(e.stream)
        a0, b0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record(s)
        fn()
        b0.record(s)
        b0.synchronize()
        return a0.elapsed_time(b0)

    def cut_calls(e, ev, m):
        pos = 0
        for off, c in ev:
            if off >= m:
                break
            if off > pos:
                e.chain_process_device(x.data_ptr() + 4 * pos, n, out.data_ptr() + 4 * pos, n, off - pos, ys + 4 * pos,
                                       yr + 4 * pos)
                pos = off
            e.chain_update(**c)
        e.chain_process_device(x.data_ptr() + 4 * pos, n, out.data_ptr() + 4 * pos, n, m - pos, ys + 4 * pos,
                               yr + 4 * pos)

    engines = {"none": make_engine(Engine, synth_ir, wl, True)}
    legs = {"none": lambda: timed(engines["none"], lambda: engines["none"].chain_process_device(
        x.data_ptr(), n, out.data_ptr(), n, n, ys, yr))}
    for p, ev in autos.items():
        for kind in ("events", "cuts"):
            k = f"{kind}_{p}"
            e = engines[k] = make_engine(Engine, synth_ir, wl, True)
            if kind == "events":
                legs[k] = (lambda e, arr: lambda: timed(e, lambda: e.chain_process_device_events(
                    x.data_ptr(), n, out.data_ptr(), n, n, arr, ys, yr)))(e, arrays[p])
            else:
                legs[k] = (lambda e, ev: lambda: timed(e, lambda: cut_calls(e, ev, n)))(e, ev)
    for f in legs.values():
        f()                                   # warm-up step
    ms = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, f in legs.items():
            for _ in range(a.steps):
                ms[k].append(f())
    for e in engines.values():
        e.close()
    res = {"frames_per_step": n}
    for k, v in ms.items():
        med = float(np.median(v))
        res[k] = {"ms_per_step": round(med, 3), "min_ms": round(float(np.min(v)), 3), "max_ms": round(float(np.max(v)), 3),
                  "M_stereo_frames_per_s": round(n / med / 1e3, 1), "n": len(v)}

    # parity: a window of the events call against the cut calls at the densest automation, fresh handles
    p0 = min(a.every)
    m = min(n, 2 * 2160000 + 12345)
    ev = [(o, c) for o, c in autos[p0] if o < m]
    e_ev, e_cut = make_engine(Engine, synth_ir, wl, True), make_engine(Engine, synth_ir, wl, True)
    e_ev.chain_process_device_events(x.data_ptr(), n, out.data_ptr(), n, m, ev, ys, yr, sync=True)
    got = out[:, :m].cpu().numpy()
    cut_calls(e_cut, ev, m)
    torch.cuda.ExternalStream(e_cut.stream).synchronize()
    ref = out[:, :m].cpu().numpy()
    peak = float(np.max(np.abs(ref)))
    err = float(np.max(np.abs(got - ref)))
    res["check_every"] = p0
    res["check_window_samples"] = m
    res["check_max_err_over_peak"] = err / peak
    assert err <= 1e-5 * peak, (wl, err / peak)
    e_ev.close()
    e_cut.close()

    # kernels of one events step at the densest automation
    from torch.profiler import ProfilerActivity, profile
    e = make_engine(Engine, synth_ir, wl, True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.chain_process_device_events(x.data_ptr(), n, out.data_ptr(), n, n, arrays[p0], ys, yr, sync=True)
        torch.cuda.synchronize()
    ker = {}
    for kev in prof.key_averages():
        if "chain" in kev.key:
            us = getattr(kev, "device_time_total", None) or kev.cuda_time_total
            ker[kev.key.split("(")[0].replace("pc::", "")] = round(us / 1e3, 3)
    res["kernels_ms_per_events_step"] = ker
    res["segmented_send_ms_per_step"] = round(sum(v for k, v in ker.items() if "chain_seg" in k), 3)
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--blocks", type=int, default=112608)
    ap.add_argument("--workload", default="both", choices=["metric", "quad", "both"])
    ap.add_argument("--every", default="512,4096,65536")
    a = ap.parse_args()
    a.every = [int(v) for v in a.every.split(",")]

    import torch
    from reevr_b200 import Engine
    from reevr_b200.convolver import chain_event_array
    from reevr_b200.synth import synth_input, synth_ir

    assert torch.cuda.is_available(), "the measurement needs a CUDA device"
    out = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "chain": CHAIN,
           "blocks_per_step": a.blocks, "every": a.every}
    for wl in (("metric", "quad") if a.workload == "both" else (a.workload,)):
        out[wl] = run_workload(wl, a, torch, Engine, synth_ir, synth_input, chain_event_array)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
