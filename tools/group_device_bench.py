"""Device-buffer calls of N handles: N own b200conv_process_device / b200conv_chain_process_device calls against one
b200conv_group_process_device / b200conv_chain_group_process_device, for chunks longer than one head block.

For each shape (quad 128 / 8192 and quad 512 / 8192, 10 s IRs) and N in --sizes, two sets of handles with the same IRs,
chain configuration and input: the twins make N own device calls per chunk, the members one group call.  Each chunk is
timed with the host clock from the first call to the end of a device synchronise.  Both sets are cleared before each
chunk length; the first `--warm` chunks are untimed.  Reported per leg: median / p99 microseconds per chunk, launches
per chunk (the group's shared launches plus the members' own, tail blocks included) and the largest difference between
the two outputs.  The card's name and power limit are read in the same run.

  python tools/group_device_bench.py [--warm 20] [--calls 200] [--sizes 1,2,4,8,16] [--chunks 128,480,2048,8192]
                                     [--out FILE]
"""
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

from reevr_b200.convolver import Engine, Group  # noqa: E402
from reevr_b200.synth import synth_input, synth_ir  # noqa: E402

SR = 48000
IR_10S = 480000
CFG = dict(srate=float(SR), lowcut_hz=120.0, lowcut_slope=1, highcut_hz=9000.0, highcut_slope=2, predelay=480,
           width=0.8, drygain=0.7, wetgain=0.5, true_stereo=True)


def build(head, seed):
    e = Engine(4)
    assert e.init_twostage(head, 8192, [synth_ir(IR_10S, 4 * seed + c) for c in range(4)])
    e.chain_configure(**CFG)
    return e


class Set:
    """N members in a group and N twins; device input, envelopes and outputs of up to `cap` samples per chunk"""

    def __init__(self, head, n, cap):
        self.members = [build(head, i) for i in range(n)]
        self.twins = [build(head, i) for i in range(n)]
        self.group = Group(self.members)
        self.cap = cap
        src = np.stack([np.stack([synth_input(cap * 8, 7 * i + c) for c in range(4)]) for i in range(n)])
        self.src = torch.from_numpy(src.astype(np.float32)).cuda()                 # [n][4][8 cap]
        t = torch.arange(cap * 8, device="cuda", dtype=torch.float32)
        self.env = [0.5 + 0.5 * torch.sin(t * 1e-3).abs(), 0.25 + 0.75 * torch.cos(t * 7e-4).abs()]
        self.y_own = torch.zeros(n, 4, cap, device="cuda")
        self.y_grp = torch.zeros(n, 4, cap, device="cuda")

    def launches(self):
        return self.group.launch_count + sum(e.launch_count for e in self.members + self.twins)

    def clear(self):
        for e in self.members + self.twins:
            e.clear()

    def close(self):
        self.group.close()
        for e in self.members + self.twins:
            e.close()


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 1), "p99_us": round(float(np.percentile(a, 99)), 1)}


def run_leg(s, chain, k, warm, calls):
    n = len(s.members)
    s.clear()
    torch.cuda.synchronize()
    L = s.cap * 8
    t_own, t_grp, l_own, l_grp, dmax = [], [], [], [], 0.0
    for j in range(warm + calls):
        off = (j * k) % (L - k)
        x = s.src[:, :, off:off + k].contiguous()
        es = [e[off:off + k].contiguous() for e in s.env]
        yo, yg = s.y_own[:, :, :k].contiguous(), s.y_grp[:, :, :k].contiguous()
        torch.cuda.synchronize()
        l0 = s.launches()
        t0 = time.perf_counter()
        for i, e in enumerate(s.twins):
            if chain:
                e.chain_process_device(x[i].data_ptr(), k, yo[i].data_ptr(), k, k, es[0].data_ptr(), es[1].data_ptr())
            else:
                e.process_device(x[i].data_ptr(), k, yo[i].data_ptr(), k, k)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        l1 = s.launches()
        if chain:
            s.group.chain_process_device([x[i].data_ptr() for i in range(n)], [k] * n, [yg[i].data_ptr() for i in range(n)],
                                         [k] * n, k, [es[0].data_ptr()] * n, [es[1].data_ptr()] * n)
        else:
            s.group.process_device([x[i].data_ptr() for i in range(n)], [k] * n, [yg[i].data_ptr() for i in range(n)],
                                   [k] * n, k)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if j >= warm:
            t_own.append((t1 - t0) * 1e6)
            t_grp.append((t2 - t1) * 1e6)
            l_own.append(l1 - l0)
            l_grp.append(s.launches() - l1)
            rows = 2 if chain else 4
            dmax = max(dmax, float((yo[:, :rows] - yg[:, :rows]).abs().max()))
    return {"chain": chain, "chunk": k, "own": stats(t_own), "group": stats(t_grp),
            "own_launches_per_chunk": round(float(np.mean(l_own)), 2),
            "group_launches_per_chunk": round(float(np.mean(l_grp)), 2), "max_abs_diff": dmax}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        return f"unavailable: {ex}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warm", type=int, default=20)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--sizes", default="1,2,4,8,16")
    ap.add_argument("--chunks", default="128,480,2048,8192")
    ap.add_argument("--heads", default="128,512")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("group_device_bench needs a CUDA device")
    chunks = [int(c) for c in a.chunks.split(",")]
    results = [{"card": card()}]
    print(json.dumps(results[0]), flush=True)
    for head in [int(h) for h in a.heads.split(",")]:
        for n in [int(v) for v in a.sizes.split(",")]:
            s = Set(head, n, max(chunks))
            for chain in (False, True):
                for k in chunks:
                    r = {"shape": f"quad {head}/8192, 10 s IRs", "handles": n, **run_leg(s, chain, k, a.warm, a.calls)}
                    results.append(r)
                    print(json.dumps(r), flush=True)
            s.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
