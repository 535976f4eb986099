"""Real-time calls of N handles per audio callback: N single b200conv_process calls against one b200conv_group_process.

Every callback is paced at the audio rate (host block / 48 kHz) and does both, on two sets of handles with the same IRs
fed the same input: first the N single calls on the twins, then the group call on the members, each timed with the
host clock (the call returns with its output complete).  The first `--warm` callbacks are untimed.  Reported per leg:
median / p99 / max microseconds per callback, group launches per callback, and the largest difference between the
group's and the single calls' outputs.

  python tools/group_bench.py [--warm 200] [--calls 2000] [--legs quad128,quad480,mixed] [--occupancy] [--out FILE]

--occupancy also builds tools/rt_occupancy.cu (nvcc, into a temporary directory) and prints how many k_rt_group
clusters the GPU keeps resident per cluster size.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from reevr_b200.convolver import Engine, Group  # noqa: E402
from reevr_b200.synth import synth_input, synth_ir  # noqa: E402

SR = 48000
IR_10S = 480000


def quad(head, tail, seed):
    return lambda: (Engine(4), lambda e: e.init_twostage(head, tail, [synth_ir(IR_10S, 4 * seed + c) for c in range(4)]))


def stereo_uniform(block, parts, seed):
    return lambda: (Engine(2), lambda e: e.init_uniform(block, [synth_ir(block * parts - 3, 2 * seed + c) for c in range(2)]))


def build(recipe):
    e, init = recipe()
    assert init(e)
    return e


class Leg:
    def __init__(self, recipes, block):
        self.block = block
        self.members = [build(r) for r in recipes]
        self.twins = [build(r) for r in recipes]
        self.group = Group(self.members)
        self.lib = self.members[0]._l
        n = block
        self.xin = [[np.zeros(n, np.float32) for _ in range(e.n_channels)] for e in self.members]
        self.y_single = [[np.zeros(n, np.float32) for _ in range(e.n_channels)] for e in self.members]
        self.y_group = [[np.zeros(n, np.float32) for _ in range(e.n_channels)] for e in self.members]

        def table(arrs):
            return (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        self.p_in = [table(x) for x in self.xin]
        self.p_single = [table(y) for y in self.y_single]
        self.p_group = [table(y) for y in self.y_group]
        self.g_in = (C.c_void_p * len(self.members))(*[C.cast(p, C.c_void_p) for p in self.p_in])
        self.g_out = (C.c_void_p * len(self.members))(*[C.cast(p, C.c_void_p) for p in self.p_group])
        self.src = [[synth_input(block * 64, 7 * i + c) for c in range(e.n_channels)] for i, e in enumerate(self.members)]

    def feed(self, k):
        off = (k % 63) * self.block
        for x, s in zip(self.xin, self.src):
            for a, b in zip(x, s):
                a[:] = b[off:off + self.block]

    def single(self):
        for e, pi, po in zip(self.twins, self.p_in, self.p_single):
            if self.lib.b200conv_process(e._h, pi, po, self.block):
                raise RuntimeError(self.lib.b200conv_last_error(e._h).decode())

    def grouped(self):
        if self.lib.b200conv_group_process(self.group._g, C.cast(self.g_in, C.POINTER(C.c_void_p)),
                                           C.cast(self.g_out, C.POINTER(C.c_void_p)), self.block):
            raise RuntimeError(self.lib.b200conv_group_last_error(self.group._g).decode())

    def diff(self):
        return max(float(np.max(np.abs(a - b))) for ys, yg in zip(self.y_single, self.y_group) for a, b in zip(ys, yg))

    def close(self):
        self.group.close()
        for e in self.members + self.twins:
            e.close()


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 1), "p99_us": round(float(np.percentile(a, 99)), 1),
            "max_us": round(float(np.max(a)), 1)}


def run_leg(name, recipes, block, warm, calls):
    leg = Leg(recipes, block)
    period = block / SR
    t_single, t_group, launches, dmax = [], [], [], 0.0
    t_next = time.perf_counter()
    for k in range(warm + calls):
        while time.perf_counter() < t_next:
            pass
        leg.feed(k)
        l0 = leg.group.launch_count
        t0 = time.perf_counter()
        leg.single()
        t1 = time.perf_counter()
        leg.grouped()
        t2 = time.perf_counter()
        if k >= warm:
            t_single.append((t1 - t0) * 1e6)
            t_group.append((t2 - t1) * 1e6)
            launches.append(leg.group.launch_count - l0)
            dmax = max(dmax, leg.diff())
        t_next += period
        t_next = max(t_next, time.perf_counter())       # a late callback does not start a burst of catch-up calls
    leg.close()
    return {"leg": name, "handles": len(recipes), "host_block": block, "calls": calls, "single": stats(t_single),
            "group": stats(t_group), "group_launches_per_callback": round(float(np.mean(launches)), 3),
            "max_abs_diff_vs_single": dmax}


def occupancy():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "rt_occupancy")
        subprocess.run([nvcc, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(ROOT, "tools", "rt_occupancy.cu")], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    return [json.loads(line) for line in out.splitlines() if line.strip()]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        q = f"unavailable: {ex}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warm", type=int, default=200)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--legs", default="quad128,quad480,mixed")
    ap.add_argument("--sizes", default="1,2,4,8,16")
    ap.add_argument("--occupancy", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    results = [{"card": card()}]
    if a.occupancy:
        results += occupancy()
    sizes = [int(s) for s in a.sizes.split(",")]
    legs = a.legs.split(",")
    for n in sizes:
        if "quad128" in legs:
            results.append(run_leg("quad 128/8192, 10 s IRs", [quad(128, 8192, i) for i in range(n)], 128, a.warm, a.calls))
        if "quad480" in legs:
            results.append(run_leg("quad 512/8192, 10 s IRs, 480-sample calls", [quad(512, 8192, i) for i in range(n)], 480,
                                   a.warm, a.calls))
    if "mixed" in legs:
        results.append(run_leg("mixed: quad 128/8192, stereo uniform 256 x 600, stereo split-mode uniform 256 x 1100",
                               [quad(128, 8192, 0), stereo_uniform(256, 600, 1), stereo_uniform(256, 1100, 2)], 128,
                               a.warm, a.calls))
    for r in results:
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
