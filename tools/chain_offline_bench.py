"""Times the send / wet chain on device buffers (b200conv_chain_process_device) against the bare convolver.

  python tools/chain_offline_bench.py [--rounds 3] [--steps 2] [--blocks 112608] [--workload metric|quad|both]

Workloads: "metric" = stereo, 10 s IR at 48 kHz, uniform block 512 (bench.py's shape), "quad" = REEV-R's quad
two-stage 128 / 8192 with true stereo, same IR length.  A step is --blocks blocks of 512 frames (112 608: 57.7 M stereo
frames), on handles with the default launch-group size.  Chain: low cut 20.5 Hz 12 dB, high cut 16 kHz 24 dB, 50 ms
predelay, send and reverb envelopes.  Legs, alternated over the rounds after one warm-up step each, all in this process:
  conv        b200conv_process_device on the dry signal (quad: L, R, L, R), CUDA events on the handle's stream
  chain_dev   b200conv_chain_process_device, CUDA events on the handle's stream
  chain_host  b200conv_chain_process from pinned host arrays, host clock (the call synchronises)
Then: a window of chain_dev against chain_host on fresh handles (<= 1e-5 of peak); a torch.profiler run of one step of
chain_dev (per-kernel time and bytes/s against the byte floor); the send forms against each other at equal piece
lengths (k_chain_send through host calls, the whole-GPU form through device calls).  Prints one JSON line with the
card's name and power limit read in the same run.
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

SRATE, IR_SECONDS = 48000.0, 10.0
CHAIN = dict(srate=SRATE, lowcut_hz=20.5, lowcut_slope=1, highcut_hz=16000.0, highcut_slope=2, predelay=2400,
             width=0.8, drygain=0.7, wetgain=0.5, true_stereo=True)
HBM_TBS = 3.35                       # H100 SXM data-sheet HBM3 bandwidth


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def floor_bytes(frames, quad_ts):
    """bytes the chain must move per step: send passes 1 + 2 read dry + ysend (24 B), ring + convolver input (16 B);
    wet reads dry, LL / RR (+ LR / RL) and yrev, writes the mix (28 B, +8 quad true stereo)"""
    return frames * (24 + 16), frames * (28 + (8 if quad_ts else 0))


def make_engine(Engine, synth_ir, wl, chain):
    C = 4 if wl == "quad" else 2
    e = Engine(C, device=0)
    irs = [synth_ir(int(IR_SECONDS * SRATE), c) for c in range(C)]
    assert (e.init_twostage(128, 8192, irs) if wl == "quad" else e.init_uniform(512, irs))
    if chain:
        e.chain_configure(**CHAIN)
    return e


def run_workload(wl, a, torch, Engine, synth_ir, synth_input):
    n = a.blocks * 512
    x = torch.empty((2, n), dtype=torch.float32).pin_memory()
    env = torch.empty((2, n), dtype=torch.float32).pin_memory()
    xh, eh = x.numpy(), env.numpy()
    xh[0], xh[1] = synth_input(n, 0), synth_input(n, 1)
    t = np.arange(n, dtype=np.float64)
    eh[0] = (0.5 + 0.5 * np.abs(np.sin(t * 1e-4))).astype(np.float32)
    eh[1] = (0.25 + 0.75 * np.abs(np.cos(t * 3e-5))).astype(np.float32)
    outh = torch.empty((2, n), dtype=torch.float32).pin_memory().numpy()
    xd, envd = x.cuda(), env.cuda()
    outd = torch.empty_like(xd)
    C = 4 if wl == "quad" else 2
    xc = torch.cat([xd, xd]) if C == 4 else xd
    yc = torch.empty_like(xc)
    e_conv = make_engine(Engine, synth_ir, wl, False)
    e_dev = make_engine(Engine, synth_ir, wl, True)
    e_host = make_engine(Engine, synth_ir, wl, True)

    def timed_dev(e, fn):
        s = torch.cuda.ExternalStream(e.stream)
        a0, b0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record(s)
        fn()
        b0.record(s)
        b0.synchronize()
        return a0.elapsed_time(b0)

    legs = {
        "conv": lambda: timed_dev(e_conv, lambda: e_conv.process_device(xc.data_ptr(), n, yc.data_ptr(), n, n)),
        "chain_dev": lambda: timed_dev(e_dev, lambda: e_dev.chain_process_device(
            xd.data_ptr(), n, outd.data_ptr(), n, n, envd[0].data_ptr(), envd[1].data_ptr())),
    }

    def host_leg():
        t0 = time.perf_counter()
        e_host.chain_process(xh[0], xh[1], eh[0], eh[1])
        return (time.perf_counter() - t0) * 1e3
    legs["chain_host"] = host_leg
    for f in legs.values():
        f()                                   # warm-up step
    ms = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, f in legs.items():
            for _ in range(a.steps):
                ms[k].append(f())
    for e in (e_conv, e_dev, e_host):
        e.close()
    res = {"frames_per_step": n}
    for k, v in ms.items():
        med = float(np.median(v))
        res[k] = {"ms_per_step": round(med, 3), "min_ms": round(float(np.min(v)), 3), "max_ms": round(float(np.max(v)), 3),
                  "M_stereo_frames_per_s": round(n / med / 1e3, 1), "n": len(v)}

    # accuracy: a window of the device leg against the host leg, fresh handles, three launch groups
    e_dev, e_host = make_engine(Engine, synth_ir, wl, True), make_engine(Engine, synth_ir, wl, True)
    m = min(n, 3 * 2160000 + 12345)
    e_dev.chain_process_device(xd.data_ptr(), n, outd.data_ptr(), n, m, envd[0].data_ptr(), envd[1].data_ptr(), sync=True)
    hl, hr = e_host.chain_process(xh[0][:m], xh[1][:m], eh[0][:m], eh[1][:m])
    dv = outd[:, :m].cpu().numpy()
    peak = max(float(np.max(np.abs(hl))), float(np.max(np.abs(hr))))
    err = max(float(np.max(np.abs(dv[0] - hl))), float(np.max(np.abs(dv[1] - hr))))
    res["check_window_samples"] = m
    res["check_max_err_over_peak"] = err / peak
    assert err <= 1e-5 * peak, (wl, err / peak)

    # kernels of one device step
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e_dev.chain_process_device(xd.data_ptr(), n, outd.data_ptr(), n, n, envd[0].data_ptr(), envd[1].data_ptr(), sync=True)
        torch.cuda.synchronize()
    ker = {}
    for ev in prof.key_averages():
        if "chain" in ev.key:
            us = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            ker[ev.key.split("(")[0].replace("pc::", "")] = round(us / 1e3, 3)
    send_ms = sum(v for k, v in ker.items() if "wide" in k or "chain_send" in k)
    wet_ms = sum(v for k, v in ker.items() if "wet" in k)
    fs, fw = floor_bytes(n, wl == "quad")
    res["kernels_ms_per_step"] = ker
    res["send_GBps_vs_floor"] = round(fs / (send_ms * 1e-3) / 1e9, 1) if send_ms else None
    res["wet_GBps_vs_floor"] = round(fw / (wet_ms * 1e-3) / 1e9, 1) if wet_ms else None
    res["floor_ms_at_datasheet"] = round((fs + fw) / (HBM_TBS * 1e12) * 1e3, 3)
    e_dev.close()
    e_host.close()

    # the send forms at equal piece lengths: k_chain_send (host calls) against the whole-GPU form (device calls)
    forms = {}
    for piece in (16384, 32768, 65536, 262144, 2097152):
        if piece > n:
            continue
        row = {}
        for kind in ("host", "dev"):
            e = make_engine(Engine, synth_ir, wl, True)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for k in range(4):
                    o = k * piece
                    if kind == "dev":
                        e.chain_process_device(xd.data_ptr() + 4 * o, n, outd.data_ptr() + 4 * o, n, piece,
                                               envd[0].data_ptr() + 4 * o, envd[1].data_ptr() + 4 * o, sync=True)
                    else:
                        e.chain_process(xh[0][o:o + piece], xh[1][o:o + piece], eh[0][o:o + piece], eh[1][o:o + piece])
                torch.cuda.synchronize()
            tot = 0.0
            for ev in prof.key_averages():
                if "chain_send" in ev.key or "chain_wide" in ev.key:
                    tot += getattr(ev, "device_time_total", None) or ev.cuda_time_total
            row["k_chain_send_us" if kind == "host" else "wide_us"] = round(tot / 4, 1)
            e.close()
        forms[str(piece)] = row
    res["send_form_per_piece"] = forms
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--blocks", type=int, default=112608)
    ap.add_argument("--workload", default="both", choices=["metric", "quad", "both"])
    a = ap.parse_args()

    import torch
    from reevr_b200 import Engine
    from reevr_b200.synth import synth_input, synth_ir

    assert torch.cuda.is_available(), "the measurement needs a CUDA device"
    out = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "chain": CHAIN, "blocks_per_step": a.blocks}
    for wl in (("metric", "quad") if a.workload == "both" else (a.workload,)):
        out[wl] = run_workload(wl, a, torch, Engine, synth_ir, synth_input)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
