"""Every sweep and FFT form of the convolver against a float64 convolution, bounded by the oracle's own error.

The parity tests compare the engine with the FP32 oracle (oracle/partconv_oracle.c: float64 FFT, float32 CMAC, like the
reference) at 1e-5 of peak, about 30x the error either of them has against the true convolution, and with white noise
through a noise IR, which spreads the energy evenly over bins and partitions.  Here the truth is the float64 linear
convolution of the same float32 input and trimmed IR (FFTConvolver::init's 1e-6 threshold, e.ir_len(c)), and the
engine must stay within a small factor of the oracle's error, for every output channel and segment:

    e64(engine) <= max(K_FORM[form] * e64(oracle), 2^-23 * peak64)

with e64(y) = max |y - truth| / peak64, peak64 = max |truth| over the segment, and the oracle run on the same input
with the same call schedule; the 1e-5 bar against the oracle stays as a second assertion.  Signal classes beyond
noise x noise IR (signals()): DC against an all-positive IR (same-sign products turn a truncating accumulate into a
bias), the Nyquist tone and DC alone (all the energy in entry 0, which packs DC and Nyquist), tones on the last bin and
on the first bin of the last tile of each kernel, a sparse partition-probe IR (a misplaced or dropped partition shows
far above the oracle's error) and a level step, whose quiet part is checked against its own peak.

Every form is forced and its selection asserted per call (last_sweep_variant, launch_count, or the fft512 switch
changing / not changing the output): K2 FFMA batch, K2x tensor-core sweep (GPU), K2t streaming sweep, K0 k_rt_block
over every template M and cluster geometry, the register-resident FFT512 and the generic Stockham FFTs, and REEV-R's
stage schedules.  K_FORM comes from DESIGN.md section 5's table (tools/conv_precision_table.py prints it).  The
tensor-core sweep's DC + noise case also bounds its mean signed error (TC_BIAS): its truncating accumulate is a bias
that a max-error bound against an oracle with a long float32 accumulation chain of its own does not see.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import oracle as orc
from reevr_b200.convolver import Engine
from tests.backends import get_lib

TOL = 1e-5
FLOOR = 2.0 ** -23
# about 1.5x the largest e64(engine) / e64(oracle) per form family in DESIGN.md section 5's table, H100 and emulation
# build (worst seen: K2 3.2, K2x 4.6, K2t 4.0, K0 3.5, FFTs 4.3, stage schedules 3.5)
K_FORM = {"k2": 5.0, "k2x": 7.0, "k2t": 6.0, "k0": 5.5, "fft": 6.5, "stages": 5.5}
# The tensor core's accumulate truncates, so same-sign products (DC + noise through the all-positive IR) give the
# tensor-core sweep a mean signed error the FFMA sweep does not have: 8.1e-7 - 8.7e-7 of peak measured on the H100
# (FFMA sweep <= 3.2e-7, the oracle's own).  Folding the accumulators into FP32 registers every 4 chunks keeps it there;
# one chain per K range gave 2.3e-6 - 2.8e-6.  Bound: 1.5x the measured bias.
TC_BIAS = 1.3e-6


# ---- forms ----------------------------------------------------------------------------------------------------------
def rt_cluster_ctas(M: int, C: int, P: int) -> int:
    """engine.cu rt_cluster_ctas for a one-stage handle: CTAs per convolver of k_rt_block, -1 = split mode"""
    max_nc = 1
    while max_nc * 2 * C <= 16 and max_nc * 2 <= M // 32:
        max_nc *= 2
    nc = 1
    while M // nc // 2 > 256:
        nc *= 2
    nbytes = P * M * 16
    while nc < max_nc and nbytes // nc > 64 * 1024:
        nc *= 2
    if nc > max_nc or nbytes // nc > 384 * 1024:
        return -1 if (C <= 8 and M >= 64) else 0
    return nc


class Form:
    """one engine configuration, its call schedule and what must have run"""

    def __init__(self, name, family, B, P=None, C=1, kind="uniform", tail=None, blocks=None, offsets=None, ir_len=None,
                 sched="long", host=None, variant=0, batch=0, options=None, expect=None, groups=None):
        self.name, self.family, self.B, self.C, self.kind = name, family, B, C, kind
        self.tail, self.blocks, self.offsets = tail, blocks, offsets
        self.ir_len = ir_len if ir_len is not None else P * B - 3
        self.P = P
        self.sched, self.host, self.variant, self.batch = sched, host, variant, batch
        self.options = options or {}
        self.expect, self.groups = expect, groups

    @property
    def stage_blocks(self):
        if self.kind == "uniform":
            return [self.B]
        if self.kind == "twostage":
            return [self.B, self.tail]
        return list(self.blocks)

    def engine(self, lib, irs, **options):
        e = Engine(self.C, cmac_variant=self.variant, max_batch_blocks=self.batch, lib=lib)
        for k, v in {**self.options, **options}.items():
            e.set_option(k, v)
        if self.kind == "uniform":
            assert e.init_uniform(self.B, irs)
        elif self.kind == "twostage":
            assert e.init_twostage(self.B, self.tail, irs)
        else:
            assert e.init_stages(self.blocks, self.offsets, irs)
        return e

    def oracle(self, ir):
        if self.kind == "twostage":
            o = orc.OracleTwoStage()
            assert o.init(self.B, self.tail, ir)
        else:                           # init_stages: the same linear convolution as a uniform convolver of the head block
            o = orc.OracleUniform()
            assert o.init(self.B, ir)
        return o

    def chunks(self, n):
        B = self.B
        if self.groups:
            out = [g * B for g in self.groups]
        elif self.sched == "long":
            out = [n]
        elif self.sched == "blocks":
            out = [B] * (n // B)
        elif self.sched == "inside":         # every call inside the open block, none a power of two (B >= 16)
            out = [B // 3, B - B // 3] * (n // B)
        elif self.sched == "host":
            out = [self.host] * (n // self.host)
        else:
            raise ValueError(self.sched)
        rest = n - sum(out)
        assert rest >= 0
        return out + ([rest] if rest else [])

    def round_n(self, n):
        if self.groups:
            return sum(self.groups) * self.B
        q = self.host or self.B
        return -(-n // q) * q

    def check_selection(self, calls, stages):
        """calls: (length, last_sweep_variant, launches) per call; stages: Engine.stages()"""
        if self.kind == "uniform":
            assert [s["block"] for s in stages] == [self.B] and stages[0]["partitions"] == self.P
        else:
            assert [s["block"] for s in stages] == self.stage_blocks
        self.expect(calls)


def _variant_is(*vs):
    def check(calls):
        assert all(v in vs for n, v, l in calls if n), [v for n, v, l in calls]
    return check


def _k2_groups(group_blocks, B):
    def check(calls):
        _variant_is(22)(calls)
        for n, v, l in calls:            # a forward FFT, sweep and inverse FFT per launch group (at least)
            assert l >= 3 * -(-n // (group_blocks * B)), (n, l)
    return check


def _launches_per_call(k):
    def check(calls):
        assert all(l == k for n, v, l in calls), sorted({l for n, v, l in calls})
    return check


def _any(calls):
    pass


FORMS = [
    # K2: packed-FMA batched sweep (variant 22, the default below 4096 blocks per group); small groups split the calls
    # and make the timeline compact (hist rows moved to the front) many times
    Form("k2-B512-P60", "k2", 512, 60, C=2, variant=22, expect=_variant_is(22)),
    Form("k2-B64-P200-batch16", "k2", 64, 200, C=2, variant=22, batch=16, expect=_k2_groups(16, 64)),
    Form("k2-B256-P33-batch5", "k2", 256, 33, C=1, variant=22, batch=5, sched="host", host=700, expect=_k2_groups(5, 256)),
    # K2t: streaming sweep, one block per launch (real-time path off): automatic choice and the dynamic-ticket / skewed
    # forms, partition counts that leave ragged ring stages
    *[Form(f"k2t-{'auto' if v == 0 else v}-B{B}-P{P}", "k2t", B, P, C=2, variant=v, sched="blocks", options={"rt": 0},
           expect=_variant_is(*((103, 104) if v == 0 else (v,))))
      for v in (0, 106, 107, 108) for B, P in ((512, 21), (128, 37))],
    # K0: k_rt_block, every template M, cluster geometries C x NC = 1x1, 1x16, 2x8, 4x4, 8x2 and the split mode
    *[Form(f"k0-M{M}-C{C}x{rt_cluster_ctas(M, C, P)}", "k0", M, P, C=C, sched="inside",
           expect=_launches_per_call(1 if rt_cluster_ctas(M, C, P) > 0 else 3))
      for M, C, P in ((16, 1, 40), (32, 1, 40), (64, 8, 100), (128, 4, 100), (256, 2, 100), (512, 1, 100),
                      (1024, 1, 60), (1024, 2, 9), (64, 2, 800))],
    # FFTs: register-resident FFT512 (launches of >= 32 transforms), generic Stockham kernels (B 512 in short launches,
    # B 16 and 2048; B 8192 is the tail of the 128 / 8192 schedule below)
    Form("fft512-B512-P9", "fft", 512, 9, C=2, expect=_any),
    Form("stockham-B512-P9-short", "fft", 512, 9, C=2, sched="host", host=1024, options={"rt": 0}, expect=_any),
    Form("stockham-B16-P300", "fft", 16, 300, C=1, expect=_any),
    Form("stockham-B2048-P6", "fft", 2048, 6, C=1, expect=_any),
    # stage schedules: REEV-R's quad head 128 / tail 8192 (host block 100), heads 16 / 32 / 1024 with tail 8192,
    # and a 4-stage schedule
    Form("quad-128-8192-host100", "stages", 128, C=4, kind="twostage", tail=8192, ir_len=16384 + 3 * 8192 - 5,
         sched="host", host=100, expect=_any),
    Form("twostage-16-8192-host16", "stages", 16, C=2, kind="twostage", tail=8192, ir_len=16384 + 2 * 8192 - 5,
         sched="host", host=16, expect=_any),
    Form("twostage-32-8192-host24", "stages", 32, C=2, kind="twostage", tail=8192, ir_len=16384 + 2 * 8192 - 5,
         sched="host", host=24, expect=_any),
    Form("twostage-1024-8192-host1000", "stages", 1024, C=2, kind="twostage", tail=8192, ir_len=16384 + 3 * 8192 - 5,
         sched="host", host=1000, expect=_any),
    Form("stages4-16-64-512-4096", "stages", 16, C=1, kind="stages", blocks=[16, 64, 512, 4096],
         offsets=[0, 128, 1024, 8192], ir_len=8192 + 3 * 4096 - 7, sched="host", host=300, expect=_any),
]
# K2x: tensor-core sweep (GPU only), launch groups of exactly 4096, 4097 and 8193 blocks through process_device, the
# later groups starting from the history of the earlier ones; chosen automatically (>= 4096 blocks, P <= 961)
FORMS_TC = [
    Form("k2x-B32-P961-C4", "k2x", 32, 961, C=4, groups=[4096, 4097, 8193], batch=8200, expect=_variant_is(40)),
    Form("k2x-B512-P938-C1", "k2x", 512, 938, C=1, groups=[4096, 4097], batch=8200, expect=_variant_is(40)),
]
FORM_BY_NAME = {f.name: f for f in FORMS + FORMS_TC}


# ---- signal classes -------------------------------------------------------------------------------------------------
def positive_ir(n, seed):
    """all-positive, decaying to -60 dB at the last tap"""
    rng = np.random.default_rng(99 + seed)
    h = (0.5 + 0.5 * rng.random(n)) * np.exp(-np.arange(n) * np.log(1000.0) / n)
    return (h / h.max()).astype(np.float32)


def probe_ir(form):
    """deltas at taps 0, B - 1, B, a middle partition, the stage boundaries and the last tap, amplitudes 1 / 2^-7 / 2^-14"""
    L, B = form.ir_len, form.B
    taps = [0, B - 1, B, (L // B // 2) * B + B // 3, L - 1]
    if form.kind != "uniform":
        offs = form.offsets if form.kind == "stages" else [0, 2 * form.tail]
        taps += [t + d for t in offs[1:] for d in (-1, 0) if t + d < L]
    h = np.zeros(L, np.float32)
    for i, t in enumerate(sorted(set(taps))):
        h[t] = 2.0 ** (-7 * (i % 3))
    h[L - 1] = 2.0 ** -14
    return h


def tone_bins(form):
    """bins at tile edges: the last bin, one in the last 32-bin column of K2, the first bin of k_rt_block's last tile"""
    B = form.B
    out = {"tone-last": B - 1, "tone-col": B - 17 if B >= 32 else B // 2}
    if form.family == "k0":
        nc = abs(rt_cluster_ctas(B, form.C, form.P))
        if nc > 1:
            out["tone-tile"] = (nc - 1) * B // nc
    return out


def signals(form):
    return ["noise", "dc", "nyquist", "dc-only", *tone_bins(form), "probe", "step"]


def make_case(form, signal):
    """(inputs per channel, IRs per channel, segments [(lo, hi)])"""
    L, B, C = form.ir_len, form.B, form.C
    bmax = max(form.stage_blocks)
    irs = [orc.synth_ir(L, c) for c in range(C)]
    if signal == "step":
        quiet = L + 2 * bmax                      # the loud rows have left every stage's delay line after this
        if form.groups:
            n = form.round_n(0)
            a = (n - quiet - L) // 2
            assert a >= 4 * B
        else:
            a = max(4 * B, L // 4)
            n = form.round_n(a + quiet + L + 4 * B)
        xs = []
        for c in range(C):
            x = orc.synth_input(n, c)
            x[a:a + quiet] = 0.0
            x[a + quiet:] *= np.float32(1e-4)
            xs.append(x)
        return xs, irs, [(0, a + quiet), (a + quiet, n)]
    n = form.round_n(max(L + 8 * B, 4 * bmax)) if not form.groups else form.round_n(0)
    t = np.arange(n)
    if signal == "noise":
        xs = [orc.synth_input(n, c) for c in range(C)]
    elif signal == "dc":
        irs = [positive_ir(L, c) for c in range(C)]
        xs = [(0.5 + 0.02 * orc.synth_input(n, c)).astype(np.float32) for c in range(C)]
    elif signal == "nyquist":
        xs = [(0.5 * (1 - 2 * (t % 2))).astype(np.float32) for c in range(C)]
    elif signal == "dc-only":
        xs = [np.full(n, 0.5, np.float32) for c in range(C)]
    elif signal.startswith("tone-"):
        k = tone_bins(form)[signal]
        xs = [(0.5 * np.cos(np.pi * k * t / B + 0.3 * c)).astype(np.float32) for c in range(C)]
    elif signal == "probe":
        irs = [probe_ir(form) for c in range(C)]
        xs = [orc.synth_input(n, c) for c in range(C)]
    else:
        raise ValueError(signal)
    return xs, irs, [(0, n)]


def truth(x, h):
    """float64 linear convolution, first x.size samples"""
    n = x.size + h.size - 1
    m = 1 << (n - 1).bit_length()
    y = np.fft.irfft(np.fft.rfft(x.astype(np.float64), m) * np.fft.rfft(h.astype(np.float64), m), m)
    return y[:x.size]


# ---- running --------------------------------------------------------------------------------------------------------
def run_engine(form, lib, xs, irs, **options):
    """outputs, (length, last_sweep_variant, launches) per call, stages, trimmed IR lengths"""
    e = form.engine(lib, irs, **options)
    chunks = form.chunks(xs[0].size)
    calls, outs, pos = [], [[] for _ in xs], 0
    if form.groups:
        import torch
        xd = torch.from_numpy(np.stack(xs)).cuda()
        yd = torch.zeros_like(xd)
        stride = xd.shape[1]
    for k in chunks:
        l0 = e.launch_count
        if form.groups:
            e.process_device(xd.data_ptr() + 4 * pos, stride, yd.data_ptr() + 4 * pos, stride, k, sync=True)
        else:
            for c, y in enumerate(e.process([x[pos:pos + k] for x in xs])):
                outs[c].append(y)
        calls.append((k, e.last_sweep_variant(), e.launch_count - l0))
        pos += k
    stages, ir_lens = e.stages(), [e.ir_len(c) for c in range(form.C)]
    e.close()
    ys = list(yd.cpu().numpy()) if form.groups else [np.concatenate(o) for o in outs]
    return ys, calls, stages, ir_lens


def run_oracle(form, xs, irs):
    chunks = form.chunks(xs[0].size)
    ys = []
    for x, h in zip(xs, irs):
        o = form.oracle(h)
        pos, out = 0, []
        for k in chunks:
            out.append(o.process(x[pos:pos + k]))
            pos += k
        ys.append(np.concatenate(out))
    return ys


def measure(form, signal, lib):
    """[(channel, segment, e64(oracle), e64(engine), error against the oracle / oracle peak, |mean signed error| / peak64
    of the oracle and of the engine)], calls, stages"""
    xs, irs, segs = make_case(form, signal)
    ys, calls, stages, ir_lens = run_engine(form, lib, xs, irs)
    yo = run_oracle(form, xs, irs)
    rows = []
    for c in range(form.C):
        r = truth(xs[c], irs[c][:ir_lens[c]])
        for s, (lo, hi) in enumerate(segs):
            t = r[lo:hi]
            pk = float(np.max(np.abs(t)))
            e_o = float(np.max(np.abs(yo[c][lo:hi] - t))) / pk
            e_e = float(np.max(np.abs(ys[c][lo:hi] - t))) / pk
            vs = float(np.max(np.abs(ys[c][lo:hi].astype(np.float64) - yo[c][lo:hi])) /
                       np.max(np.abs(yo[c][lo:hi].astype(np.float64))))
            b_o = abs(float(np.mean(yo[c][lo:hi] - t))) / pk
            b_e = abs(float(np.mean(ys[c][lo:hi] - t))) / pk
            rows.append((c, s, e_o, e_e, vs, b_o, b_e))
    return rows, calls, stages


def check(form, signal, lib):
    rows, calls, stages = measure(form, signal, lib)
    form.check_selection(calls, stages)
    k = K_FORM[form.family]
    for c, s, e_o, e_e, vs, b_o, b_e in rows:
        what = (form.name, signal, c, s, e_o, e_e, b_e)
        assert e_e <= max(k * e_o, FLOOR), what
        assert vs <= TOL, what
        if form.family == "k2x" and signal == "dc":
            assert b_e <= TC_BIAS, what
    return rows


def _cases(forms):
    return [pytest.param(f.name, s, id=f"{f.name}-{s}") for f in forms for s in signals(f)]


@pytest.fixture(params=["emu", pytest.param("cuda", marks=pytest.mark.gpu)])
def backend(request):
    return request.param


@pytest.mark.parametrize("form,signal", _cases(FORMS))
def test_conv_precision(backend, form, signal):
    check(FORM_BY_NAME[form], signal, get_lib(backend))


@pytest.mark.gpu
@pytest.mark.parametrize("form,signal", _cases(FORMS_TC))
def test_tc_sweep_precision(form, signal):
    check(FORM_BY_NAME[form], signal, get_lib("cuda"))


@pytest.mark.parametrize("backend_", ["emu", pytest.param("cuda", marks=pytest.mark.gpu)])
def test_fft512_selection(backend_):
    """the fft512 switch changes the output of a long B = 512 launch (the register-resident kernels ran) and leaves
    the short launches alone (the Stockham kernels ran with or without it)"""
    lib = get_lib(backend_)
    for name, differs in (("fft512-B512-P9", True), ("stockham-B512-P9-short", False)):
        f = FORM_BY_NAME[name]
        xs, irs, _ = make_case(f, "noise")
        ys = {on: run_engine(f, lib, xs, irs, fft512=on)[0] for on in (1, 0)}
        assert any(not np.array_equal(a, b) for a, b in zip(ys[0], ys[1])) == differs, name


def test_rt_geometries_are_the_listed_ones():
    """the K0 forms above cover every template M and the cluster geometries C x NC of the real-time kernel"""
    geo = {(f.B, f.C, rt_cluster_ctas(f.B, f.C, f.P)) for f in FORMS if f.family == "k0"}
    assert {m for m, _, _ in geo} == {16, 32, 64, 128, 256, 512, 1024}
    assert {(c, nc) for _, c, nc in geo} >= {(1, 1), (1, 16), (2, 8), (4, 4), (8, 2), (2, -1)}
