"""The streaming sweep and the long-IR paths against float64 at steady state: every partition holding signal, the TMA
ring wrapping.

tests/test_conv_precision.py runs the streaming sweep (K2t, k_cmac_stream_tma / _dyn) only at P <= 37, where no CTA
walks more than three ring stages, and the shapes at which the engine selects it for long IRs only with most of the
history zero.  Here the history is full: a long batched call of more than P blocks fills every FDL row, then a window
of single-block calls runs the streaming form (both walk directions, since stream_alternate flips the walk per launch,
and many ticket bases of the dynamic forms).  Each GPU case asserts the sweep form it means to test and that its ring
wraps at least twice (ring_geometry() restates launch_cmac_stream_tma's slice rule with the card's SM count).

Replaying the FP32 oracle from the start costs P x (P + n) block-partitions, minutes per channel at P = 11 250, so the
yardstick is oracle_window(): a vectorised restatement of oc_uniform_process (oracle/partconv_oracle.c) for a window of
output blocks of block-aligned calls, with the oracle's float32 accumulation order.  It is pinned against the C oracle
on the CPU (test_model_matches_the_oracle).  Two-stage handles use the float64 sum of three such models (head, first
tail block, remaining tail), pinned against OracleTwoStage.  The truth is the float64 convolution of the float32 input
and the trimmed IR over the window only.  The criterion is test_conv_precision's:

    e64(engine) <= max(K_FORM[family] * e64(yardstick), 2^-23 * peak64),   |engine - yardstick| <= 1e-5 of peak

and, for DC + noise through an all-positive IR, |mean signed error| <= max(2 * the yardstick's, 2^-23 * peak64): the
streaming form sums its slices with RED.ADD, which must not add a bias.

The emulation build runs a reduced set (B 512, C 8, P 231: 33 slices of 7 partitions with 132 SMs, so either walk
has a partial last stage).  It runs the same slice and stage arithmetic without the ring, so there
it checks the slicing and the model, not the barriers.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import refcheck
from reevr_b200.convolver import Engine
from tests.backends import BACKENDS, get_lib
from tests.test_conv_precision import FLOOR, K_FORM, TOL, positive_ir, truth

STAGE_BYTES = 16384
# variant -> (ring stages S, CTAs per SM), launch_cmac_as
RING = {103: (6, 2), 104: (12, 1), 106: (6, 2), 107: (12, 1), 108: (6, 2)}
SKEW = 0.08                     # variant 108's default slice skew (B200CONV_STREAM_SKEW unset)
N_SM_EMU = 132                  # the emulation build's SM count
WINDOW = 32                     # single-block calls checked after the prefill


# ---- geometry of the streaming sweep ----------------------------------------------------------------------------------
def stream_w(B):
    return min(B, 512)


def stream_pp(B):
    return STAGE_BYTES // (16 * stream_w(B))


def n_sm(backend):
    if backend == "emu":
        return N_SM_EMU
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def auto_variant(B, P, C):
    """select_cmac for a single-block sweep"""
    return 104 if B < 512 or (B == 512 and P * B * 16 * C <= 32 << 20) else 103


def ring_geometry(B, P, C, variant, sms):
    """(nsplit, stages of a full slice, ring wraps of that slice) of launch_cmac_stream_tma.  The dynamic forms
    (106 / 107) count the stages per CTA on average; the skewed form (108) its lightest slice."""
    S, per_sm = RING[variant]
    PP = stream_pp(B)
    nsplit = max(1, min(per_sm * sms // ((B // stream_w(B)) * C), max(1, P // (2 * PP))))
    if variant in (106, 107):
        nst = -(-P // PP) // nsplit
    else:
        per = -(-P // nsplit)
        if variant == 108:
            per = int(per * (1 - SKEW)) - PP
        nst = per // PP
    return nsplit, nst, nst // S


# ---- yardstick: the oracle's arithmetic for a window of output blocks ------------------------------------------------
def _spectra(blocks, B):
    """float64 FFT of [block ; 0] rounded to float32 (oc_rfft), re and im rows"""
    F = np.fft.rfft(blocks.astype(np.float64), 2 * B, axis=1)
    re, im = F.real.astype(np.float32), F.imag.astype(np.float32)
    im[:, 0] = 0.0
    im[:, -1] = 0.0
    return re, im


def _blocks(x, b0, b1, B):
    return refcheck._blocks(x, b0, b1, B).reshape(b1 - b0, B)


def oracle_window(B, h, x, w0, n):
    """Output blocks [w0, w0 + n) of oc_uniform_process (block-aligned calls) for the trimmed IR h, float32: the
    pre-multiplied sum over partitions 1 .. P-1 in the oracle's order and float32 evaluation order (oc_cmac), then
    partition 0 with the current block, the float64 inverse rounded to float32, plus the previous block's overlap.
    X rows of blocks before the window come straight from the input; nothing before w0 is replayed."""
    h = np.asarray(h, np.float32)
    P = -(-h.size // B)
    Hr, Hi = _spectra(np.pad(h, (0, P * B - h.size)).reshape(P, B), B)
    lo = w0 - 1 - (P - 1)                 # oldest block read (the overlap needs block w0 - 1 as well)
    Xr, Xi = _spectra(_blocks(x, lo, w0 + n, B), B)
    m = n + 1                            # blocks w0 - 1 .. w0 + n - 1
    pr = np.zeros((m, B + 1), np.float32)
    pi = np.zeros((m, B + 1), np.float32)
    for i in range(1, P):                # row of block b - i: (b - i) - lo, b from w0 - 1
        xr, xi = Xr[P - 1 - i:P - 1 - i + m], Xi[P - 1 - i:P - 1 - i + m]
        pr = (pr + Hr[i] * xr) - Hi[i] * xi
        pi = (pi + Hr[i] * xi) + Hi[i] * xr
    xr, xi = Xr[P - 1:], Xi[P - 1:]      # the current block (cmac(cv, cur, ir0): X is the first operand)
    pr = (pr + xr * Hr[0]) - xi * Hi[0]
    pi = (pi + xr * Hi[0]) + xi * Hr[0]
    pi[:, 0] = 0.0
    pi[:, -1] = 0.0
    y = np.fft.irfft(pr.astype(np.float64) + 1j * pi.astype(np.float64), 2 * B, axis=1).astype(np.float32)
    ov = y[:-1, B:] if w0 >= 1 else np.vstack([np.zeros((1, B), np.float32), y[1:-1, B:]])
    return (y[1:, :B] + ov).reshape(-1)


def twostage_window(head, T, h, x, s0, s1):
    """samples [s0, s1) (multiples of T) of a head / T two-stage handle: the float64 sum of the head model over h[:T],
    block T over h[T:2T] delayed by T and block T over h[2T:] delayed by 2T"""
    y = oracle_window(head, h[:T], x, s0 // head, (s1 - s0) // head).astype(np.float64)
    for k in (1, 2):
        part = h[k * T:(k + 1) * T] if k == 1 else h[2 * T:]
        if part.size:
            y += oracle_window(T, part, x, (s0 - k * T) // T, (s1 - s0) // T)
    return y


def truth_window(h, x, s0, s1):
    """float64 linear convolution of x and h, samples [s0, s1)"""
    lo = s0 - h.size
    seg = x[max(lo, 0):s1].astype(np.float64)
    if lo < 0:
        seg = np.concatenate([np.zeros(-lo), seg])
    return truth(seg, h)[-(s1 - s0):]


# ---- signals ----------------------------------------------------------------------------------------------------------
def probe_taps(B, L, P, C, variant, sms):
    """a delta at the first and the last partition of every CTA slice, at the first slice's stage boundary PP * S
    (where its ring first wraps) and at the last tap"""
    S, _ = RING[variant]
    nsplit, _, _ = ring_geometry(B, P, C, variant, sms)
    per = -(-P // nsplit)
    parts = {0, stream_pp(B) * S}
    for y in range(nsplit):
        if y * per < P:
            parts |= {y * per, min(P, (y + 1) * per) - 1}
    return sorted({p * B + (p * 37) % B for p in parts if p < P} | {L - 1})


def make_irs(signal, L, C, probe=None):
    if signal == "dc":
        return [positive_ir(L, c) for c in range(C)]
    if signal == "probe":
        h = np.zeros(L, np.float32)
        for i, t in enumerate(probe):
            h[t] = 2.0 ** (-7 * (i % 3))
        h[L - 1] = 2.0 ** -14
        return [h.copy() for _ in range(C)]
    return [orc.synth_ir(L, c) for c in range(C)]


def make_inputs(signal, n, C, quiet_from=None):
    if signal == "dc":
        return [(0.5 + 0.02 * orc.synth_input(n, c)).astype(np.float32) for c in range(C)]
    xs = [orc.synth_input(n, c) for c in range(C)]
    if quiet_from is not None:            # the level step: silence, then the input 80 dB down
        a, q = quiet_from
        for x in xs:
            x[a:a + q] = 0.0
            x[a + q:] *= np.float32(1e-4)
    return xs


_cache: dict = {}


def reference(key, h, x, s0, s1, model):
    """(yardstick, truth) for samples [s0, s1), cached per (IR, input, window): several forms share them"""
    if key not in _cache:
        _cache[key] = (model(h, x, s0, s1), truth_window(h, x, s0, s1))
    return _cache[key]


# ---- running and checking -----------------------------------------------------------------------------------------------
def run(lib, C, init, xs, chunks, variant=0, batch=0, options=None, engine=None):
    """outputs per channel over all chunks and (length, last_sweep_variant, launches) per call"""
    e = engine or Engine(C, cmac_variant=variant, max_batch_blocks=batch, lib=lib)
    for k, v in (options or {}).items():
        e.set_option(k, v)
    if init is not None:
        init(e)
    outs, calls, pos = [[] for _ in range(C)], [], 0
    for k in chunks:
        l0 = e.launch_count
        for c, y in enumerate(e.process([x[pos:pos + k] for x in xs])):
            outs[c].append(y)
        calls.append((k, e.last_sweep_variant(), e.launch_count - l0))
        pos += k
    return [np.concatenate(o) for o in outs], calls, e


def check(ys, yard, tru, family, signal, what):
    """the criterion of tests/test_conv_precision.py for one channel and window; returns (e64 yard, e64 engine)"""
    pk = float(np.max(np.abs(tru)))
    e_y = float(np.max(np.abs(yard - tru))) / pk
    e_e = float(np.max(np.abs(ys - tru))) / pk
    vs = float(np.max(np.abs(ys.astype(np.float64) - yard)) / np.max(np.abs(yard)))
    info = (what, signal, e_y, e_e, vs)
    assert e_e <= max(K_FORM[family] * e_y, FLOOR), info
    assert vs <= TOL, info
    if signal == "dc":
        b_y = abs(float(np.mean(yard - tru))) / pk
        b_e = abs(float(np.mean(ys - tru))) / pk
        assert b_e <= max(2 * b_y, FLOOR), info + (b_y, b_e)
    return e_y, e_e


def check_uniform(ys, irs, xs, B, s0, s1, key, family, signal, what, ir_lens):
    out = []
    for c in range(len(xs)):
        h = irs[c][:ir_lens[c]]
        yard, tru = reference(key + (c,), h, xs[c], s0, s1,
                              lambda h_, x_, a, b: oracle_window(B, h_, x_, a // B, (b - a) // B))
        out.append(check(ys[c][s0:s1], yard, tru, family, signal, what + (c,)))
    return out


# ---- the model against the oracle (CPU) ---------------------------------------------------------------------------
def test_model_matches_the_oracle():
    """oracle_window reproduces the C oracle's window within 1e-6 of peak, at the oracle's own error level"""
    B, P, w0, n = 512, 1000, 1010, 8
    h = orc.synth_ir(P * B - 3, 0)
    x = orc.synth_input((w0 + n) * B, 0)
    ref = refcheck.ref_window(B, h, x, w0, n).astype(np.float64)
    mod = oracle_window(B, refcheck.trimmed(h), x, w0, n).astype(np.float64)
    tru = truth_window(refcheck.trimmed(h), x, w0 * B, (w0 + n) * B)
    pk = np.max(np.abs(tru))
    assert np.max(np.abs(mod - ref)) <= 1e-6 * np.max(np.abs(ref))
    e_ref, e_mod = np.max(np.abs(ref - tru)) / pk, np.max(np.abs(mod - tru)) / pk
    assert 0.5 * e_ref <= e_mod <= 2.0 * e_ref, (e_ref, e_mod)


def test_model_matches_the_oracle_from_a_cold_start():
    """the window that starts at block 0 (no overlap, no history) and ragged last partition"""
    B, L, n = 64, 64 * 20 - 17, 30
    h = orc.synth_ir(L, 1)
    x = orc.synth_input(n * B, 1)
    o = orc.OracleUniform()
    assert o.init(B, h)
    ref = o.run(x, B).astype(np.float64)
    mod = oracle_window(B, refcheck.trimmed(h), x, 0, n)
    assert np.max(np.abs(mod - ref)) <= 1e-6 * np.max(np.abs(ref))


def test_twostage_model_matches_the_oracle():
    """the sum of three uniform models against OracleTwoStage run whole (head 64 / tail 256, three tail stages used)"""
    head, T = 64, 256
    h = orc.synth_ir(5 * T - 11, 2)
    n = 12 * T
    x = orc.synth_input(n, 2)
    o = orc.OracleTwoStage()
    assert o.init(head, T, h)
    ref = o.run(x, head).astype(np.float64)
    ht = refcheck.trimmed(h)
    tru = truth(x, ht)
    for s0, s1 in ((0, n), (4 * T, 9 * T)):
        mod = twostage_window(head, T, ht, x, s0, s1)
        r = ref[s0:s1]
        assert np.max(np.abs(mod - r)) <= 1e-6 * np.max(np.abs(r)), (s0, s1)
        pk = np.max(np.abs(tru[s0:s1]))
        e_ref, e_mod = np.max(np.abs(r - tru[s0:s1])) / pk, np.max(np.abs(mod - tru[s0:s1])) / pk
        assert 0.5 * e_ref <= e_mod <= 2.0 * e_ref, (e_ref, e_mod)


# ---- the streaming sweep at steady state -------------------------------------------------------------------------------
class Shape:
    def __init__(self, B, P, C, pre=None):
        self.B, self.P, self.C = B, P, C
        self.L = P * B - 3
        self.pre = pre if pre is not None else P + 8          # prefill blocks: every partition holds signal

    @property
    def key(self):
        return (self.B, self.P, self.C)


EMU_SHAPE = Shape(512, 231, 8)
LONG = Shape(512, 11250, 2)             # 120 s at 48 kHz, bench.py's roofline_stream / ir120 shape
LONG1 = Shape(512, 11250, 1)
CFG4 = Shape(512, 938, 8)               # 8-channel 10 s IR
B128 = Shape(128, 3200, 8)
B256 = Shape(256, 2000, 8)
COLD = Shape(512, 3200, 2)


def stream_case(backend, shape, variant, signal="noise", options=None, expect=None):
    """WINDOW single-block calls of `variant` at steady state, checked against the yardstick.  Automatic selection
    (variant 0, expect = what it must select): the history comes from one call of shape.pre blocks (the batched FFMA
    sweep).  A forced variant also runs the history, as shape.pre single-block calls."""
    lib = get_lib(backend)
    B, P, C, L = shape.B, shape.P, shape.C, shape.L
    sms = n_sm(backend)
    want = expect or variant
    _, nst, wraps = ring_geometry(B, P, C, want, sms)
    if backend == "cuda":
        assert wraps >= 2, (shape.key, want, nst)
    probe = probe_taps(B, L, P, C, want, sms) if signal == "probe" else None
    irs = make_irs(signal, L, C, probe)
    n = (shape.pre + WINDOW) * B
    xs = make_inputs(signal, n, C)
    chunks = [shape.pre * B] + [B] * WINDOW if variant == 0 else [B] * (shape.pre + WINDOW)
    ys, calls, e = run(lib, C, lambda e: e.init_uniform(B, irs), xs, chunks, variant=variant,
                       options={"rt": 0, **(options or {})})
    ir_lens = [e.ir_len(c) for c in range(C)]
    assert e.stages()[0]["partitions"] == P
    e.close()
    if variant == 0:
        assert calls[0][1] == 22, calls[0]
        calls = calls[1:]
    assert all(v == want and l == 3 for k, v, l in calls), sorted({(v, l) for k, v, l in calls})
    key = (shape.key, signal, tuple(probe) if probe else None)
    return check_uniform(ys, irs, xs, B, shape.pre * B, n, key, "k2t", signal,
                         (shape.key, variant, options), ir_lens)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("variant", [103, 104, 106, 107, 108])
def test_stream_steady_state_forced(backend, variant):
    """every streaming form, both walk directions, history from single-block calls.  Emulation: B 512, C 8, P 231
    (103: 33 slices of 7 partitions, a partial last stage in either walk).  H100: cfg4's B 512, C 8, P 938, where
    every form wraps its ring twice"""
    stream_case(backend, EMU_SHAPE if backend == "emu" else CFG4, variant)


@pytest.mark.parametrize("backend", BACKENDS)
def test_stream_steady_state_probe(backend):
    """deltas at both ends of every slice and at the first stage boundary that wraps the ring (variant 103)"""
    stream_case(backend, EMU_SHAPE if backend == "emu" else CFG4, 103, signal="probe")


@pytest.mark.gpu
@pytest.mark.parametrize("variant,options", [(0, None), (104, None), (106, None), (107, None), (108, None),
                                             (103, {"stream_alternate": 0})],
                         ids=["auto", "104", "106", "107", "108", "103-ascending"])
def test_stream_120s(variant, options):
    """B 512, P 11 250, C 2: 132 slices of ~86 partitions, ~43 stages each (seven wraps of the 6-stage ring)"""
    stream_case("cuda", LONG, variant, options=options, expect=103 if variant == 0 else None)


@pytest.mark.gpu
@pytest.mark.parametrize("signal", ["dc", "probe"])
def test_stream_120s_signals(signal):
    stream_case("cuda", LONG, 0, signal=signal, expect=103)


@pytest.mark.gpu
def test_stream_120s_mono():
    """C 1: 264 slices"""
    stream_case("cuda", LONG1, 0, expect=103)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [CFG4, B128, B256], ids=["cfg4-B512-P938-C8", "B128-P3200-C8", "B256-P2000-C8"])
def test_stream_other_shapes(shape):
    """cfg4 (automatic 103), and whole-row copies with several partition groups per stage at B 128 / 256 (104)"""
    stream_case("cuda", shape, 0, expect=auto_variant(shape.B, shape.P, shape.C))


@pytest.mark.gpu
def test_stream_level_step():
    """80 dB step at P 3200: the window lies in the quiet part once the loud rows have left the delay line, and is
    checked against its own peak"""
    s = COLD
    B, P, C, L = s.B, s.P, s.C, s.L
    lib = get_lib("cuda")
    a, q = 64 * B, L + 2 * B
    pre = -(-(a + q) // B) + 8
    n = (pre + WINDOW) * B
    irs = make_irs("noise", L, C)
    xs = make_inputs("noise", n, C, quiet_from=(a, q))
    ys, calls, e = run(lib, C, lambda e: e.init_uniform(B, irs), xs, [pre * B] + [B] * WINDOW, options={"rt": 0})
    ir_lens = [e.ir_len(c) for c in range(C)]
    e.close()
    assert ring_geometry(B, P, C, 103, n_sm("cuda"))[2] >= 2
    assert all(v == 103 and l == 3 for k, v, l in calls[1:]), calls[1:3]
    check_uniform(ys, irs, xs, B, pre * B, n, ("step",) + s.key, "k2t", "step", ("step",), ir_lens)


@pytest.mark.gpu
def test_stream_cold_start():
    """pure streaming from the first sample (single-block calls only): the window around block P, where the last
    partition first receives signal"""
    s = COLD
    B, P, C, L = s.B, s.P, s.C, s.L
    lib = get_lib("cuda")
    assert ring_geometry(B, P, C, 103, n_sm("cuda"))[2] >= 2
    nblk = P + 16
    irs = make_irs("noise", L, C)
    xs = make_inputs("noise", nblk * B, C)
    ys, calls, e = run(lib, C, lambda e: e.init_uniform(B, irs), xs, [B] * nblk, options={"rt": 0})
    ir_lens = [e.ir_len(c) for c in range(C)]
    e.close()
    assert all(v == 103 and l == 3 for k, v, l in calls), sorted({(v, l) for k, v, l in calls})
    check_uniform(ys, irs, xs, B, (P - 16) * B, nblk * B, ("cold",) + s.key, "k2t", "noise", ("cold",), ir_lens)


@pytest.mark.gpu
def test_k2_batched_120s():
    """the FFMA batched sweep at P 11 250 (beyond the tensor-core forms): one long call in launch groups of 1000
    blocks, so that the timeline is compacted a dozen times with 11 250 history rows"""
    s = LONG
    B, P, C = s.B, s.P, s.C
    lib = get_lib("cuda")
    irs = make_irs("noise", s.L, C)
    n = (s.pre + WINDOW) * B
    xs = make_inputs("noise", n, C)
    ys, calls, e = run(lib, C, lambda e: e.init_uniform(B, irs), xs, [n], batch=1000)
    ir_lens = [e.ir_len(c) for c in range(C)]
    e.close()
    (k, v, l), = calls
    assert v == 22 and l >= 3 * -(-n // (1000 * B)), calls
    check_uniform(ys, irs, xs, B, s.pre * B, n, (s.key, "noise", None), "k2", "noise", ("k2-batched",), ir_lens)


# ---- the real-time split mode (front kernel, all-SM streaming sweep, back kernel) --------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("host", [512, 480, 128])
def test_rt_split_mode_120s(host):
    """rt on (the default) on the 120 s uniform handle: host blocks of 512 (split mode on every call), 480 (calls that
    cross a block boundary take the multi-kernel path, the others split mode) and 128 (calls inside the open block)"""
    s = LONG
    B, P, C = s.B, s.P, s.C
    lib = get_lib("cuda")
    assert ring_geometry(B, P, C, 103, n_sm("cuda"))[2] >= 2
    irs = make_irs("noise", s.L, C)
    ncalls = -(-WINDOW * B // host)
    n = s.pre * B + ncalls * host
    xs = make_inputs("noise", n, C)
    ys, calls, e = run(lib, C, lambda e: e.init_uniform(B, irs), xs, [s.pre * B] + [host] * ncalls)
    ir_lens = [e.ir_len(c) for c in range(C)]
    e.close()
    fill, split = 0, 0
    for k, v, l in calls[1:]:
        if fill + k <= B:                 # inside the open block or completing it: front, sweep, back
            assert (v, l) == (103, 3), (fill, k, v, l)
            split += 1
        fill = (fill + k) % B
    if host == 480:                       # only calls that start at fill <= 32 stay inside the block
        assert 2 <= split < ncalls, (split, ncalls)
    else:
        assert split == ncalls, (split, ncalls)
    check_uniform(ys, irs, xs, B, s.pre * B, (s.pre + WINDOW) * B, (s.key, "noise", None), "k0", "noise",
                  ("rt", host), ir_lens)


# ---- REEV-R's two-stage layouts at real lengths --------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("head,C,L,host,min_wraps", [(128, 4, 480000, 100, 1), (128, 4, 480000, 128, 1),
                                                     (64, 2, 2880000, 100, 2), (64, 2, 2880000, 64, 2)],
                         ids=["128-8192-C4-10s-host100", "128-8192-C4-10s-host128",
                              "64-8192-C2-30s96k-host100", "64-8192-C2-30s96k-host64"])
def test_twostage_long(head, C, L, host, min_wraps):
    """tail 8192: at 10 s / 48 kHz the tail stage has ~57 partitions in 4 slices (one wrap of the ring at most); at
    30 s / 96 kHz ~350 partitions in 8 slices of segment copies (W = 512 < B, 16 bin tiles), three wraps"""
    T = 8192
    lib = get_lib("cuda")
    irs = make_irs("noise", L, C)
    pre = -(-(L + 2 * T) // T) * T         # the window starts on a tail-block boundary
    s0, s1 = pre, pre + 4 * T
    ncalls = -(-(s1 - s0) // host)
    n = pre + ncalls * host
    xs = make_inputs("noise", n, C)
    ys, calls, e = run(lib, C, lambda e: e.init_twostage(head, T, irs), xs, [pre] + [host] * ncalls)
    ir_lens = [e.ir_len(c) for c in range(C)]
    stages = e.stages()
    e.close()
    assert [st["block"] for st in stages] == [head, T]
    Pt = stages[1]["partitions"]
    assert ring_geometry(T, Pt, C, 103, n_sm("cuda"))[2] >= min_wraps, Pt
    if host <= head:      # a longer call sweeps the head with launch_cmac last, which last_sweep_variant then reports
        assert 103 in {v for k, v, l in calls[1:]}, sorted({v for k, v, l in calls[1:]})
    for c in range(C):
        h = irs[c][:ir_lens[c]]
        yard, tru = reference(("twostage", head, L, C, c), h, xs[c], s0, s1,
                              lambda h_, x_, a, b: twostage_window(head, T, h_, x_, a, b))
        check(ys[c][s0:s1], yard, tru, "stages", "noise", (head, L, host, c))


# ---- state across the long history -------------------------------------------------------------------------------------
def _clear_case(backend, shape):
    """clear() at steady state (prefill + an even number of streaming calls): the first P blocks after it match a fresh
    handle (bit for bit on the emulation; on the GPU RED.ADD sums the slices in any order) and the truth of the
    post-clear input alone"""
    B, P, C, L = shape.B, shape.P, shape.C, shape.L
    lib = get_lib(backend)
    irs = make_irs("noise", L, C)
    before = shape.pre * B + 8 * B
    after = (P + 8) * B
    xs = make_inputs("noise", before + after, C)
    x2 = [x[before:] for x in xs]
    if backend == "cuda":
        assert ring_geometry(B, P, C, auto_variant(B, P, C), n_sm(backend))[2] >= 2
    e = Engine(C, lib=lib)
    e.set_option("rt", 0)
    assert e.init_uniform(B, irs)
    run(lib, C, None, xs, [shape.pre * B] + [B] * 8, engine=e)
    e.clear()
    ys, calls, _ = run(lib, C, None, x2, [B] * (P + 8), engine=e)
    ir_lens = [e.ir_len(c) for c in range(C)]
    e.close()
    want = auto_variant(B, P, C)
    assert all(v == want for k, v, l in calls)
    yf, _, f = run(lib, C, lambda f: f.init_uniform(B, irs), x2, [B] * (P + 8), options={"rt": 0})
    f.close()
    for c in range(C):
        if backend == "emu":
            assert np.array_equal(ys[c], yf[c]), c
        else:
            assert np.max(np.abs(ys[c] - yf[c])) <= 2.0 ** -20 * np.max(np.abs(yf[c])), c
    check_uniform(ys, irs, x2, B, (P - 16) * B, after, ("clear",) + shape.key, "k2t", "noise", ("clear",), ir_lens)


def _reinit_case(backend, shape, P2):
    """an IR re-init to a different P between calls of the dynamic form (106): its ticket counters carry on across the
    re-init, and the output after it matches a fresh handle and the truth"""
    B, P, C = shape.B, shape.P, shape.C
    lib = get_lib(backend)
    irs1 = make_irs("noise", shape.L, C)
    L2 = P2 * B - 5
    irs2 = [orc.synth_ir(L2, c + 10) for c in range(C)]
    n1, n2 = 8 * B, (P2 + 8) * B
    xs = make_inputs("noise", n1 + n2, C)
    x2 = [x[n1:] for x in xs]
    if backend == "cuda":
        assert ring_geometry(B, P2, C, 106, n_sm(backend))[2] >= 2
    e = Engine(C, cmac_variant=106, lib=lib)
    e.set_option("rt", 0)
    assert e.init_uniform(B, irs1)
    _, c1, _ = run(lib, C, None, xs, [B] * 8, engine=e)
    assert e.init_uniform(B, irs2)
    ys, c2, _ = run(lib, C, None, x2, [B] * (P2 + 8), engine=e)
    ir_lens = [e.ir_len(c) for c in range(C)]
    assert e.stages()[0]["partitions"] == P2
    e.close()
    assert all(v == 106 for k, v, l in c1 + c2)
    yf, _, f = run(lib, C, lambda f: f.init_uniform(B, irs2), x2, [B] * (P2 + 8), variant=106, options={"rt": 0})
    f.close()
    for c in range(C):
        assert np.max(np.abs(ys[c] - yf[c])) <= 2.0 ** -20 * np.max(np.abs(yf[c])), c
    check_uniform(ys, irs2, x2, B, (P2 - 16) * B, n2, ("reinit", P2) + shape.key, "k2t", "noise", ("reinit",), ir_lens)


@pytest.mark.parametrize("backend", BACKENDS)
def test_clear_at_steady_state(backend):
    _clear_case(backend, EMU_SHAPE if backend == "emu" else COLD)


@pytest.mark.parametrize("backend", BACKENDS)
def test_reinit_between_streaming_calls(backend):
    if backend == "emu":
        _reinit_case(backend, EMU_SHAPE, 150)
    else:
        _reinit_case(backend, COLD, 3500)
