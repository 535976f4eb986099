"""Python mirror of the reference's convolver surface on top of the C ABI (tests / bench glue).

Class and method names follow the reference:
  FFTConvolver          libs/FFTConvolver/FFTConvolver.h:62-80         init / process / clear / reset
  TwoStageFFTConvolver  libs/FFTConvolver/TwoStageFFTConvolver.h:65-83 init / process / reset / clear
  StereoConvolver       src/dsp/StereoConvolver.h:20-30                prepare / loadImpulse / process / reset / clear
`Engine` is the multi-channel handle underneath (one launch set for C channels).
The C++ drop-in classes for the JUCE host live in include/FFTConvolver.h and
include/TwoStageFFTConvolver.h; this module exists because the test-suite and bench are Python.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from . import _lib


class B200ConvError(RuntimeError):
    pass


def _ptr_array(arrs: Sequence[np.ndarray]):
    arr = (C.c_void_p * len(arrs))()
    for i, a in enumerate(arrs):
        arr[i] = a.ctypes.data
    return arr


def chain_event_array(events):
    """[(offset, dict of chain_update's keywords), ...] as the b200conv_chain_event array Engine.chain_process_device_events
    passes to the library"""
    arr = (_lib.ChainEvent * len(events))()
    for k, (off, kw) in enumerate(events):
        kw = dict(kw)
        ts = int(kw.pop("true_stereo", True))
        arr[k].offset = int(off)
        arr[k].cfg = _lib.ChainConfig(kw.pop("srate"), kw.pop("lowcut_hz", 20.0), kw.pop("lowcut_slope", 0),
                                      kw.pop("highcut_hz", 20000.0), kw.pop("highcut_slope", 0), kw.pop("predelay", 0),
                                      kw.pop("width", 1.0), kw.pop("drygain", 1.0), kw.pop("wetgain", 1.0), ts)
        if kw:
            raise TypeError(f"unknown chain parameters {sorted(kw)}")
    return arr


class Engine:
    """C mono convolvers in one handle (b200conv_t)."""

    def __init__(self, n_channels: int = 1, device: int = 0, max_batch_blocks: int = 0,
                 shard_rank: int = 0, shard_count: int = 1, cmac_variant: int = 0, lib=None, shard_head: bool = True):
        """shard_head=False (sharded handles): rank 0 keeps the head stage whole and only the stages >= 1 are split
        over the ranks — the real-time call stays one launch on rank 0 and no collective runs per call."""
        self._l = lib or _lib.default()
        cfg = _lib.Config(n_channels, device, max_batch_blocks, shard_rank, shard_count, cmac_variant)
        self._h = self._l.b200conv_create(C.byref(cfg))
        if not self._h:
            raise B200ConvError("b200conv_create failed")
        self.n_channels = n_channels
        self._reduce_cb = None
        if not shard_head:
            self.set_option("shard_head", 0)

    # -- helpers ---------------------------------------------------------------------------
    def _check(self, rc: int, what: str, allow_einval: bool = False) -> int:
        if rc == 0 or (allow_einval and rc == -1):
            return rc
        raise B200ConvError(f"{what} failed ({rc}): {self._l.b200conv_last_error(self._h).decode()}")

    def _irs(self, irs):
        irs = [np.ascontiguousarray(a, dtype=np.float32) for a in irs]
        if len(irs) != self.n_channels:
            raise ValueError("need one IR per channel")
        keep = [a if a.size else np.zeros(1, np.float32) for a in irs]
        lens = (C.c_size_t * len(irs))(*[a.size for a in irs])
        return keep, _ptr_array(keep), lens

    # -- IR load ---------------------------------------------------------------------------
    def init_uniform(self, block: int, irs) -> bool:
        keep, ptrs, lens = self._irs(irs)
        return self._check(self._l.b200conv_init_uniform(self._h, block, ptrs, lens), "init_uniform", True) == 0

    def init_twostage(self, head: int, tail: int, irs) -> bool:
        keep, ptrs, lens = self._irs(irs)
        return self._check(self._l.b200conv_init_twostage(self._h, head, tail, ptrs, lens), "init_twostage", True) == 0

    @staticmethod
    def _shape_params(autogain=True, reverse=False, trim_left=0.0, trim_right=0.0, gain=1.0, lut=None, srate=48000.0,
                      clip=True, attack=0.0, decay=0.0):
        keep = None if lut is None else np.ascontiguousarray(lut, dtype=np.float64)
        sp = _lib.IrShapeParams(int(autogain), int(reverse), trim_left, trim_right, gain,
                                keep.ctypes.data if keep is not None else None, float(srate), int(clip), attack, decay)
        return sp, keep

    def init_twostage_shaped(self, head: int, tail: int, raw_irs, **shape) -> bool:
        """IR shaping (Impulse::recalcImpulse subset) on the device, partition spectra built from the device-resident
        taps (b200conv_init_twostage_shaped); raw_irs: equally long raw channels."""
        keep, ptrs, lens = self._irs(raw_irs)
        sp, lut = self._shape_params(**shape)
        return self._check(self._l.b200conv_init_twostage_shaped(self._h, head, tail, ptrs, keep[0].size, C.byref(sp)),
                           "init_twostage_shaped", True) == 0

    def init_uniform_shaped(self, block: int, raw_irs, **shape) -> bool:
        keep, ptrs, lens = self._irs(raw_irs)
        sp, lut = self._shape_params(**shape)
        return self._check(self._l.b200conv_init_uniform_shaped(self._h, block, ptrs, keep[0].size, C.byref(sp)),
                           "init_uniform_shaped", True) == 0

    @staticmethod
    def _recalc_params(ir_srate=48000.0, srate=48000.0, stretch=0.0, autogain=True, reverse=False, trim_left=0.0,
                       trim_right=0.0, gain=1.0, param_eq=(), decay_eq=(), decay_rate=1.0, clip=True, attack=0.0, decay=0.0):
        """b200conv_ir_recalc_params; bands: (mode, freq, q, gain) tuples (mode = SVF::Mode 0..9).  Returns the struct and
        the band arrays it points to (keep them alive for the call)."""
        def bands(bs):
            bs = list(bs or [])
            arr = (_lib.EqBand * max(len(bs), 1))(*[_lib.EqBand(int(m), f, q, g) for m, f, q, g in bs])
            return len(bs), arr
        npq, pq = bands(param_eq)
        ndc, dc = bands(decay_eq)
        rp = _lib.IrRecalcParams(float(ir_srate), float(srate), stretch, int(autogain), int(reverse), trim_left, trim_right,
                                 gain, npq, C.cast(pq, C.POINTER(_lib.EqBand)), ndc, C.cast(dc, C.POINTER(_lib.EqBand)),
                                 decay_rate, int(clip), attack, decay)
        return rp, (pq, dc)

    def init_twostage_recalc(self, head: int, tail: int, raw_irs, **recalc) -> bool:
        """The whole Impulse::recalcImpulse on the device (resampling, stretch, parametric and decay EQ included), partition
        spectra built from the device-resident taps (b200conv_init_twostage_recalc); raw_irs: equally long raw channels."""
        keep, ptrs, lens = self._irs(raw_irs)
        rp, bands = self._recalc_params(**recalc)
        return self._check(self._l.b200conv_init_twostage_recalc(self._h, head, tail, ptrs, keep[0].size, C.byref(rp)),
                           "init_twostage_recalc", True) == 0

    def init_uniform_recalc(self, block: int, raw_irs, **recalc) -> bool:
        keep, ptrs, lens = self._irs(raw_irs)
        rp, bands = self._recalc_params(**recalc)
        return self._check(self._l.b200conv_init_uniform_recalc(self._h, block, ptrs, keep[0].size, C.byref(rp)),
                           "init_uniform_recalc", True) == 0

    def init_stages(self, blocks, offsets, irs) -> bool:
        keep, ptrs, lens = self._irs(irs)
        b = (C.c_size_t * len(blocks))(*blocks)
        o = (C.c_size_t * len(offsets))(*offsets)
        return self._check(self._l.b200conv_init_stages(self._h, len(blocks), b, o, ptrs, lens), "init_stages", True) == 0

    # -- processing ------------------------------------------------------------------------
    def process(self, xs) -> list:
        """xs: C arrays of equal length (host). Returns C float32 arrays."""
        xs = [np.ascontiguousarray(a, dtype=np.float32) for a in xs]
        n = xs[0].size
        n_in = getattr(self, "_n_in", None) or self.n_channels
        n_out = getattr(self, "_n_out", None) or self.n_channels
        if any(a.size != n for a in xs) or len(xs) != n_in:
            raise ValueError("need one equally long input per (routed) input channel")
        ys = [np.empty(max(n, 1), np.float32)[:n] for _ in range(n_out)]
        if n:
            self._check(self._l.b200conv_process(self._h, _ptr_array(xs), _ptr_array(ys), n), "process")
        return ys

    def prime(self, xs) -> None:
        """Feeds history through the convolver in one batched call without producing output
        (IR hot-swap warm-up, src/PluginProcessor.cpp:1695-1750)."""
        xs = [np.ascontiguousarray(a, dtype=np.float32) for a in xs]
        if xs[0].size:
            self._check(self._l.b200conv_prime(self._h, _ptr_array(xs), xs[0].size), "prime")

    def process_xfade(self, new: "Engine", xs, alpha0: float, alpha_step: float) -> list:
        """self = outgoing convolver, `new` = incoming one: device-side crossfade of both outputs
        (src/PluginProcessor.cpp:1800-1830)."""
        xs = [np.ascontiguousarray(a, dtype=np.float32) for a in xs]
        n = xs[0].size
        n_out = getattr(self, "_n_out", None) or self.n_channels
        ys = [np.empty(max(n, 1), np.float32)[:n] for _ in range(n_out)]
        if n:
            self._check(self._l.b200conv_process_xfade(self._h, new._h, _ptr_array(xs), _ptr_array(ys), n,
                                                       alpha0, alpha_step), "process_xfade")
        return ys

    def process_into(self, in_ptrs, out_ptrs, n: int) -> None:
        """Raw host pointers (ctypes arrays of void*), e.g. pinned staging buffers."""
        self._check(self._l.b200conv_process(self._h, in_ptrs, out_ptrs, n), "process")

    def process_device(self, in_ptr: int, in_stride: int, out_ptr: int, out_stride: int, n: int, sync: bool = False):
        self._check(self._l.b200conv_process_device(self._h, in_ptr, in_stride, out_ptr, out_stride, n, int(sync)),
                    "process_device")

    def process_sliced(self, xs, ys, slice_rank: int, slice_count: int) -> None:
        """Time-slice sharding (b200conv_process_sliced): xs / ys are the WHOLE call's host arrays; only this
        rank's slice of every ys[c] is written."""
        n = xs[0].size
        self._check(self._l.b200conv_process_sliced(self._h, _ptr_array(xs), _ptr_array(ys), n, slice_rank, slice_count),
                    "process_sliced")

    def process_sliced_into(self, in_ptrs, out_ptrs, n: int, slice_rank: int, slice_count: int) -> None:
        self._check(self._l.b200conv_process_sliced(self._h, in_ptrs, out_ptrs, n, slice_rank, slice_count), "process_sliced")

    def process_device_sliced(self, in_ptr: int, in_stride: int, out_ptr: int, out_stride: int, n: int,
                              slice_rank: int, slice_count: int, sync: bool = False):
        self._check(self._l.b200conv_process_device_sliced(self._h, in_ptr, in_stride, out_ptr, out_stride, n,
                                                           slice_rank, slice_count, int(sync)), "process_device_sliced")

    def chain_configure(self, srate: float, lowcut_hz: float = 20.0, lowcut_slope: int = 0, highcut_hz: float = 20000.0,
                        highcut_slope: int = 0, predelay: int = 0, width: float = 1.0, drygain: float = 1.0,
                        wetgain: float = 1.0, true_stereo: bool = True) -> None:
        """The send / wet chain of REEVRAudioProcessor::processBlock on the device (b200conv_chain_configure)."""
        cfg = _lib.ChainConfig(srate, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, predelay, width, drygain, wetgain,
                               int(true_stereo))
        self._check(self._l.b200conv_chain_configure(self._h, C.byref(cfg)), "chain_configure")

    def chain_update(self, srate: float, lowcut_hz: float = 20.0, lowcut_slope: int = 0, highcut_hz: float = 20000.0,
                     highcut_slope: int = 0, predelay: int = 0, width: float = 1.0, drygain: float = 1.0,
                     wetgain: float = 1.0, true_stereo: bool = True) -> None:
        """New chain parameters from the next chain_process call on, keeping the filter states and the delay history
        (b200conv_chain_update; what the reference's onSlider and per-block parameter reads do).  srate must be the
        configured rate."""
        cfg = _lib.ChainConfig(srate, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, predelay, width, drygain, wetgain,
                               int(true_stereo))
        self._check(self._l.b200conv_chain_update(self._h, C.byref(cfg)), "chain_update")

    def chain_process(self, dryL, dryR, ysend=None, yrev=None):
        """(outL, outR) = drygain * dry + wetgain * width(yrev * mixdown(convolvers(predelay(filters(dry * ysend)))))"""
        xs = [np.ascontiguousarray(a, dtype=np.float32) for a in (dryL, dryR)]
        n = xs[0].size
        env = [None if e is None else np.ascontiguousarray(e, dtype=np.float32) for e in (ysend, yrev)]
        ys = [np.empty(max(n, 1), np.float32)[:n] for _ in range(2)]
        if n:
            self._check(self._l.b200conv_chain_process(
                self._h, _ptr_array(xs), env[0].ctypes.data if env[0] is not None else None,
                env[1].ctypes.data if env[1] is not None else None, _ptr_array(ys), n), "chain_process")
        return ys[0], ys[1]

    def chain_process_device(self, dry_ptr: int, dry_stride: int, out_ptr: int, out_stride: int, n: int,
                             ysend_ptr: int = 0, yrev_ptr: int = 0, sync: bool = False):
        """chain_process on device buffers (b200conv_chain_process_device): dry L / R rows dry_stride floats apart, the
        mix into out L / R rows out_stride apart (out_ptr == dry_ptr with equal strides: in place); envelope pointers 0
        mean 1.  Asynchronous on the handle's stream unless sync."""
        self._check(self._l.b200conv_chain_process_device(self._h, dry_ptr, dry_stride, ysend_ptr or None, yrev_ptr or None,
                                                          out_ptr, out_stride, n, int(sync)), "chain_process_device")

    def chain_process_device_events(self, dry_ptr: int, dry_stride: int, out_ptr: int, out_stride: int, n: int, events,
                                    ysend_ptr: int = 0, yrev_ptr: int = 0, sync: bool = False):
        """chain_process_device with parameter changes inside the call (b200conv_chain_process_device_events):
        events = [(offset, dict of chain_update's keywords), ...], offsets strictly increasing and below n, or an
        array from chain_event_array (built once, reused by calls with the same automation); each configuration takes
        effect at its sample, as chain_update before a call cut there would."""
        arr = events if isinstance(events, C.Array) else chain_event_array(events)
        self._check(self._l.b200conv_chain_process_device_events(
            self._h, dry_ptr, dry_stride, ysend_ptr or None, yrev_ptr or None, out_ptr, out_stride, n,
            C.cast(arr, C.c_void_p) if len(arr) else None, len(arr), int(sync)), "chain_process_device_events")

    def chain_swap(self, incoming: "Engine", host_block: int) -> None:
        """IR hot swap inside the chain (b200conv_chain_swap): the next chain_process call replays the send history
        through `incoming` and starts the 50 ms crossfade; when chain_swap_state() becomes 3 the chain has moved to
        `incoming`, which the caller uses from then on (std::swap(loadConvolver, convolver))."""
        self._check(self._l.b200conv_chain_swap(self._h, incoming._h, host_block), "chain_swap")

    def chain_swap_state(self) -> int:
        """0 no swap pending, 1 armed, 2 fading, 3 this handle gave its chain away."""
        return int(self._l.b200conv_chain_swap_state(self._h))

    def clear(self):
        self._check(self._l.b200conv_clear(self._h), "clear")

    def reset(self):
        self._check(self._l.b200conv_reset(self._h), "reset")

    def set_latency(self, samples: int) -> None:
        """Fixed-latency mode (b200conv_set_latency): process / chain_process return their output `samples` later
        (0 = zero latency, else a multiple of the head block up to 16 head blocks).  Clears the handle."""
        self._check(self._l.b200conv_set_latency(self._h, samples), "set_latency")

    @property
    def latency(self) -> int:
        return int(self._l.b200conv_latency(self._h))

    @property
    def latency_waits(self) -> int:
        """Calls in fixed-latency mode that had to wait for the device (an underrun indicator)."""
        return int(self._l.b200conv_latency_waits(self._h))

    # -- introspection ---------------------------------------------------------------------
    def stages(self) -> list:
        out = []
        for s in range(self._l.b200conv_num_stages(self._h)):
            info = _lib.StageInfo()
            self._l.b200conv_stage(self._h, s, C.byref(info))
            out.append(dict(block=info.block, partitions=info.partitions, tap_offset=info.tap_offset,
                            p_begin=info.p_begin, p_end=info.p_end))
        return out

    def ir_len(self, c: int = 0) -> int:
        return int(self._l.b200conv_ir_len(self._h, c))

    @property
    def launch_count(self) -> int:
        return int(self._l.b200conv_launch_count(self._h))

    def last_sweep_variant(self) -> int:
        """22 / 26 packed-FMA batched sweep, 40 tensor-core sweep, 100..108 streaming forms."""
        return int(self._l.b200conv_last_sweep_variant(self._h))

    @property
    def stream(self) -> int:
        return int(self._l.b200conv_stream(self._h) or 0)

    def set_option(self, name: str, value: int):
        """A/B switches of the engine: "rt" (one-launch real-time path), "fft512" (register-resident B = 512 FFTs), "tc" (tensor-core sweep for long launch groups);
        "shard_head" (layout of a sharded handle, before the IR is loaded)."""
        self._check(self._l.b200conv_set_option(self._h, name.encode(), int(value)), "set_option")

    def set_timing(self, on: bool):
        self._l.b200conv_set_timing(self._h, int(on))

    def last_timing(self) -> dict:
        a, b, c, n = C.c_float(), C.c_float(), C.c_float(), C.c_int()
        self._l.b200conv_last_timing(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(n))
        return dict(cmac_ms=a.value, fft_ms=b.value, ifft_ms=c.value, cmac_launches=n.value)

    def set_reduce(self, fn):
        """fn(dev_ptr:int, n_floats:int, stream:int) -> int (0 = ok); sums the buffer into shard 0."""
        def tramp(_user, ptr, n, stream):
            try:
                return int(fn(int(ptr), int(n), int(stream or 0)) or 0)
            except Exception:  # never raise through the C ABI
                import traceback
                traceback.print_exc()
                return -1
        self._reduce_cb = _lib.REDUCE_FN(tramp)
        self._l.b200conv_set_reduce(self._h, self._reduce_cb, None)

    def set_routing(self, in_map, mix):
        """Convolver c reads input in_map[c]; output o = sum_c mix[o][c] * y_c (computed on the device).
        `mix` is an (n_out, C) array.  set_routing(None, None) removes the routing."""
        if in_map is None:
            self._check(self._l.b200conv_set_routing(self._h, 0, None, 0, None), "set_routing")
            self._n_in = self._n_out = None
            return
        mix = np.ascontiguousarray(mix, dtype=np.float32)
        n_out, Cc = mix.shape
        assert Cc == self.n_channels and len(in_map) == self.n_channels
        n_in = max(in_map) + 1
        im = (C.c_int * Cc)(*in_map)
        self._check(self._l.b200conv_set_routing(self._h, n_in, im, n_out,
                                                 mix.ctypes.data_as(C.POINTER(C.c_float))), "set_routing")
        self._n_in, self._n_out = n_in, n_out

    def p2p_attach(self, allgather, mode: int = 0, host_barrier=None):
        """Enables the fused multi-GPU path (slot exchange over peer memory, see b200conv.h).
        `allgather(blob: bytes) -> list[bytes]` must return every shard's blob in rank order.
        mode 0 = CUDA IPC (one process per GPU), 1 = raw pointers (all shards in this process).
        `host_barrier` (callable -> 0) replaces the flag kernel in the CPU emulation build."""
        if host_barrier is not None:
            def tramp(_user):
                try:
                    return int(host_barrier() or 0)
                except Exception:
                    import traceback
                    traceback.print_exc()
                    return -1
            self._barrier_cb = _lib.BARRIER_FN(tramp)
            self._l.b200conv_p2p_set_host_barrier(self._h, self._barrier_cb, None)
        blobs = allgather(self.p2p_export(mode))
        self.p2p_import(blobs)

    def p2p_export(self, mode: int = 0) -> bytes:
        n = self._l.b200conv_p2p_blob_size(self._h)
        blob = C.create_string_buffer(n)
        self._check(self._l.b200conv_p2p_export(self._h, blob, mode), "p2p_export")
        return blob.raw

    def p2p_import(self, blobs) -> None:
        """blobs: every shard's exported blob, in rank order."""
        data = b"".join(blobs)
        joined = C.create_string_buffer(data, len(data))
        self._check(self._l.b200conv_p2p_import(self._h, joined), "p2p_import")

    def p2p_detach(self):
        """Leave the slot-exchange path (every shard must do the same); the reduce hook takes over again."""
        self._check(self._l.b200conv_p2p_detach(self._h), "p2p_detach")

    def p2p_set_input_broadcast(self, on: bool = True):
        """Host-pointer calls: only shard 0 uploads the input; the peers receive it over NVLink."""
        self._check(self._l.b200conv_p2p_set_input_broadcast(self._h, int(on)), "p2p_set_input_broadcast")

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200conv_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Group:
    """Several Engines whose real-time calls run together (b200conv_group_process): process(inputs) is
    engines[i].process(inputs[i]) for every i, with the calls that fit one cluster launch sharing one launch per
    shape class.  Keeps references to its engines, which must stay open while the group is."""

    def __init__(self, engines: Sequence[Engine], lib=None):
        self._l = lib or engines[0]._l
        self.engines = list(engines)
        hs = (C.c_void_p * len(self.engines))(*[e._h for e in self.engines])
        self._g = self._l.b200conv_group_create(hs, len(self.engines))
        if not self._g:
            raise B200ConvError("b200conv_group_create failed")

    def process(self, inputs) -> list:
        """inputs[i]: what engines[i].process takes (equally long calls); returns the list of their outputs."""
        xs = [[np.ascontiguousarray(a, dtype=np.float32) for a in x] for x in inputs]
        if len(xs) != len(self.engines):
            raise ValueError("need one input list per engine")
        n = xs[0][0].size
        ys, ins, outs = [], (C.c_void_p * len(xs))(), (C.c_void_p * len(xs))()
        keep = []
        for i, (e, x) in enumerate(zip(self.engines, xs)):
            n_in = getattr(e, "_n_in", None) or e.n_channels
            n_out = getattr(e, "_n_out", None) or e.n_channels
            if len(x) != n_in or any(a.size != n for a in x):
                raise ValueError("need one equally long input per (routed) input channel of every engine")
            y = [np.empty(max(n, 1), np.float32)[:n] for _ in range(n_out)]
            pi, po = _ptr_array(x), _ptr_array(y)
            keep += [pi, po]
            ins[i], outs[i] = C.cast(pi, C.c_void_p), C.cast(po, C.c_void_p)
            ys.append(y)
        if n:
            self._check(self._l.b200conv_group_process(self._g, C.cast(ins, C.POINTER(C.c_void_p)),
                                                       C.cast(outs, C.POINTER(C.c_void_p)), n))
        return ys

    def chain_process(self, drys, ysends=None, yrevs=None) -> list:
        """drys[i] = (dryL, dryR) of engines[i] (equally long calls), ysends / yrevs: per-engine envelopes (an entry or
        the whole list None: 1); returns [(outL, outR), ...] = engines[i].chain_process(...) for every i, with the
        calls that fit one cluster launch sharing the send, convolver and wet launches (b200conv_chain_group_process)."""
        m = len(self.engines)
        if len(drys) != m or any(len(d) != 2 for d in drys):
            raise ValueError("need (dryL, dryR) per engine")
        xs = [[np.ascontiguousarray(a, dtype=np.float32) for a in d] for d in drys]
        n = xs[0][0].size
        envs = []
        for es in (ysends, yrevs):
            if es is not None and len(es) != m:
                raise ValueError("need one envelope (or None) per engine")
            envs.append(None if es is None else [None if e is None else np.ascontiguousarray(e, dtype=np.float32)
                                                  for e in es])
        if any(a.size != n for x in xs for a in x) or any(e is not None and e.size != n for es in envs if es for e in es):
            raise ValueError("every buffer of a group call has the same length")
        ys = [[np.empty(max(n, 1), np.float32)[:n] for _ in range(2)] for _ in range(m)]
        keep = [[_ptr_array(x), _ptr_array(y)] for x, y in zip(xs, ys)]
        drs = (C.c_void_p * m)(*[C.cast(k[0], C.c_void_p) for k in keep])
        outs = (C.c_void_p * m)(*[C.cast(k[1], C.c_void_p) for k in keep])
        tabs = [None if es is None else (C.c_void_p * m)(*[None if e is None else e.ctypes.data for e in es])
                for es in envs]
        if n:
            self._check(self._l.b200conv_chain_group_process(
                self._g, C.cast(drs, C.POINTER(C.c_void_p)),
                *[None if t is None else C.cast(t, C.POINTER(C.c_void_p)) for t in tabs],
                C.cast(outs, C.POINTER(C.c_void_p)), n))
        return [(y[0], y[1]) for y in ys]

    def process_device(self, in_ptrs, in_strides, out_ptrs, out_strides, n: int, sync: bool = False) -> None:
        """engines[i].process_device(in_ptrs[i], in_strides[i], out_ptrs[i], out_strides[i], n) for every i, on the
        group's stream (b200conv_group_process_device): device addresses (ints), strides in samples.  The members that
        fit share one cluster launch per shape class for calls of up to 16 head blocks.  Order other streams with
        `stream`; sync=True returns once the call has completed."""
        m = len(self.engines)
        if any(len(t) != m for t in (in_ptrs, in_strides, out_ptrs, out_strides)):
            raise ValueError("need one buffer and stride per engine")
        pp = lambda t: (C.c_void_p * m)(*[int(a) for a in t])
        ss = lambda t: (C.c_size_t * m)(*[int(a) for a in t])
        self._check(self._l.b200conv_group_process_device(
            self._g, C.cast(pp(in_ptrs), C.POINTER(C.c_void_p)), ss(in_strides),
            C.cast(pp(out_ptrs), C.POINTER(C.c_void_p)), ss(out_strides), n, int(sync)))

    def chain_process_device(self, dry_ptrs, dry_strides, out_ptrs, out_strides, n: int, ysend_ptrs=None,
                             yrev_ptrs=None, sync: bool = False) -> None:
        """engines[i].chain_process_device(...) for every i on the group's stream (b200conv_chain_group_process_device):
        dry_ptrs[i] / out_ptrs[i] address L with R one stride later; ysend_ptrs / yrev_ptrs: per-engine envelope
        addresses (an entry 0 / None, or the whole list None: envelope 1)."""
        m = len(self.engines)
        if any(len(t) != m for t in (dry_ptrs, dry_strides, out_ptrs, out_strides)):
            raise ValueError("need one buffer and stride per engine")
        if any(t is not None and len(t) != m for t in (ysend_ptrs, yrev_ptrs)):
            raise ValueError("need one envelope (or None) per engine")
        pp = lambda t: None if t is None else C.cast((C.c_void_p * m)(*[int(a or 0) for a in t]), C.POINTER(C.c_void_p))
        ss = lambda t: (C.c_size_t * m)(*[int(a) for a in t])
        self._check(self._l.b200conv_chain_group_process_device(
            self._g, pp(dry_ptrs), ss(dry_strides), pp(ysend_ptrs), pp(yrev_ptrs), pp(out_ptrs), ss(out_strides), n,
            int(sync)))

    @property
    def stream(self) -> int:
        """the cudaStream_t of the group's calls, e.g. for torch.cuda.ExternalStream"""
        return int(self._l.b200conv_group_stream(self._g) or 0)

    def set_member(self, i: int, engine: Engine) -> None:
        """engines[i] = engine (b200conv_group_set_member), e.g. the incoming engine of a completed chain_swap"""
        self._check(self._l.b200conv_group_set_member(self._g, i, engine._h))
        self.engines[i] = engine

    def set_latency(self, samples: int) -> None:
        """One fixed latency for every engine (b200conv_group_set_latency): each engine's set_latency(samples), after
        all of them were checked; the engines at the group's latency then share their head-block steps in group calls.
        0: the engines in fixed-latency mode go back to zero latency."""
        self._check(self._l.b200conv_group_set_latency(self._g, samples))

    @property
    def latency(self) -> int:
        return int(self._l.b200conv_group_latency(self._g))

    def _check(self, rc: int) -> None:
        if rc != 0:
            raise B200ConvError(f"group process failed ({rc}): {self._l.b200conv_group_last_error(self._g).decode()}")

    @property
    def launch_count(self) -> int:
        return int(self._l.b200conv_group_launch_count(self._g))

    def close(self):
        if getattr(self, "_g", None):
            self._l.b200conv_group_destroy(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ir_decay_eq(ir, lut, srate: float, device: int = 0, lib=None) -> np.ndarray:
    """Device version of Impulse::applyDecay (src/dsp/Impulse.cpp:602-648): returns the shaped IR."""
    lib = lib or _lib.default()
    buf = np.array(ir, dtype=np.float32, copy=True)
    lut = np.ascontiguousarray(lut, dtype=np.float64)
    if lut.size != 2049:
        raise ValueError("lut needs 2049 entries (4096-point STFT)")
    rc = lib.b200conv_ir_decay_eq(device, buf.ctypes.data, buf.size, lut.ctypes.data, float(srate))
    if rc != 0:
        raise B200ConvError(f"b200conv_ir_decay_eq failed ({rc})")
    return buf


def ir_shape(raw_irs, device: int = 0, lib=None, **shape):
    """Device version of the Impulse::recalcImpulse subset (b200conv_ir_shape); returns the shaped channels."""
    lib = lib or _lib.default()
    raws = [np.ascontiguousarray(a, dtype=np.float32) for a in raw_irs]
    n = raws[0].size
    outs = [np.empty(max(n, 1), np.float32) for _ in raws]
    sp, lut = Engine._shape_params(**shape)
    m = C.c_size_t(0)
    rc = lib.b200conv_ir_shape(device, _ptr_array(raws), len(raws), n, C.byref(sp), _ptr_array(outs), C.byref(m))
    if rc != 0:
        raise B200ConvError(f"b200conv_ir_shape failed ({rc})")
    return [o[:m.value].copy() for o in outs]


def ir_recalc_len(n: int, lib=None, **recalc) -> int:
    """Taps per channel that ir_recalc returns for n raw taps (b200conv_ir_recalc_len)."""
    lib = lib or _lib.default()
    rp, bands = Engine._recalc_params(**recalc)
    return int(lib.b200conv_ir_recalc_len(n, C.byref(rp)))


def ir_recalc(raw_irs, device: int = 0, lib=None, **recalc):
    """Device version of the whole Impulse::recalcImpulse (b200conv_ir_recalc); raw_irs = {LL, RR[, LR, RL]}, equally long.
    Keywords: ir_srate, srate, stretch, autogain, reverse, trim_left, trim_right, gain, param_eq, decay_eq (lists of
    (mode, freq, q, gain)), decay_rate, clip, attack, decay.  Returns the recalculated channels."""
    lib = lib or _lib.default()
    raws = [np.ascontiguousarray(a, dtype=np.float32) for a in raw_irs]
    n = raws[0].size
    if any(a.size != n for a in raws):
        raise ValueError("raw channels must be equally long")
    rp, bands = Engine._recalc_params(**recalc)
    cap = int(lib.b200conv_ir_recalc_len(n, C.byref(rp)))
    outs = [np.empty(max(cap, 1), np.float32) for _ in raws]
    m = C.c_size_t(0)
    rc = lib.b200conv_ir_recalc(device, _ptr_array(raws), len(raws), n, C.byref(rp), _ptr_array(outs), cap, C.byref(m))
    if rc != 0:
        raise B200ConvError(f"b200conv_ir_recalc failed ({rc})")
    return [o[:m.value].copy() for o in outs]


class FFTConvolver:
    """Uniform partitioned convolver, one channel (reference: FFTConvolver.h:62-80)."""

    def __init__(self, **kw):
        self._e = Engine(1, **kw)

    def init(self, blockSize: int, ir) -> bool:
        return self._e.init_uniform(blockSize, [ir])

    def process(self, x) -> np.ndarray:
        return self._e.process([x])[0]

    def clear(self):
        self._e.clear()

    def reset(self):
        self._e.reset()


class TwoStageFFTConvolver(FFTConvolver):
    """Head/tail convolver, one channel (reference: TwoStageFFTConvolver.h:65-83)."""

    def init(self, headBlockSize: int, tailBlockSize: int, ir) -> bool:  # type: ignore[override]
        return self._e.init_twostage(headBlockSize, tailBlockSize, [ir])


class StereoConvolver:
    """LL/RR (+LR/RL in quad mode) convolvers of src/dsp/StereoConvolver.{h,cpp} as ONE handle."""

    def __init__(self, **kw):
        self._kw = kw
        self._e = None
        self.isQuad = False
        self.headBlockSize = 0
        self.tailBlockSize = 0
        self.size = 0

    def prepare(self, samplesPerBlock: int):          # StereoConvolver.cpp:8-20
        self.size = samplesPerBlock
        h = 1
        while h < samplesPerBlock:
            h *= 2
        self.headBlockSize = h
        self.tailBlockSize = max(8192, 2 * h)

    def loadImpulse(self, irLL, irRR, irLR=None, irRL=None):   # StereoConvolver.cpp:22-31
        self.isQuad = irLR is not None and irRL is not None
        irs = [irLL, irRR] + ([irLR, irRL] if self.isQuad else [])
        if self._e is None or self._e.n_channels != len(irs):
            self._e = Engine(len(irs), **self._kw)
        return self._e.init_twostage(self.headBlockSize, self.tailBlockSize, irs)

    def process(self, dataL, dataR):                   # StereoConvolver.cpp:33-42
        """Returns (bufferLL, bufferRR[, bufferLR, bufferRL])."""
        xs = [dataL, dataR] + ([dataL, dataR] if self.isQuad else [])
        return tuple(self._e.process(xs))

    def enable_device_mixdown(self, true_stereo: bool = True):
        """SURVEY 8f-1: feed {L, R} once and get the wet {L, R} back, mixed on the device as
        src/PluginProcessor.cpp:1833-1838 does on the host (L = LL + RL, R = RR + LR when quad & true stereo)."""
        if self.isQuad:
            ts = 1.0 if true_stereo else 0.0
            self._e.set_routing([0, 1, 0, 1], [[1, 0, 0, ts], [0, 1, ts, 0]])
        else:
            self._e.set_routing([0, 1], [[1, 0], [0, 1]])

    def process_mixed(self, dataL, dataR):
        """(wetL, wetR) after enable_device_mixdown()."""
        return tuple(self._e.process([dataL, dataR]))

    def clear(self):
        if self._e:
            self._e.clear()

    def reset(self):
        if self._e:
            self._e.reset()
