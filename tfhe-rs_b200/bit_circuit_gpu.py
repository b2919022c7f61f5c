"""GPU executor of compiled bit circuits (`bit_circuit.Schedule`): the wire
pool is one int64 tensor of LWEs, a schedule's tables are uploaded once per
(circuit, instance count) and kept for the few most recent ones, and a whole
schedule runs in one `b200_bit_circuit_64_async` call (per layer: linear
kernel, keyswitch, PBS scattering into the pool).

Streams: the work runs on `streams.streams[0]`, after the caller's current
stream (inputs may be produced there).  The inputs stay reserved for that
stream until the work has read them, so the caller may drop them at once; the
caller's current stream waits for the result before anything enqueued on it
later, and the result may be freed from it."""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict
from typing import Optional

import numpy as np
import torch

from . import _lib, bit_circuit as bc, gpu

DELTA = (1 << 63) // bc.TOTAL_MOD


def _u32(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32))


def _u64(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64))


def body_words(sched: bc.Schedule, iconst_bits: Optional[np.ndarray]) -> np.ndarray:
    """body constants [R, instances] as torus words (value * delta mod 2^64)"""
    body = sched.body(iconst_bits) if sched.num_iconsts else np.repeat(sched.body_base[:, None],
                                                                       sched.num_instances, axis=1)
    with np.errstate(over="ignore"):
        return body.astype(np.uint64) * np.uint64(DELTA)


class _DeviceSchedule:
    def __init__(self, sched: bc.Schedule, device, stream, luts: gpu.CudaGlweCiphertextList):
        self.luts = luts  # accumulators of sched.lut_tables()
        luts, dests = sched.gpu_tables()
        widest = max([sched.layer_outputs(L) for L in range(sched.num_layers)], default=0)
        with torch.cuda.stream(stream):
            def up(t):
                return t.to(device, non_blocking=True)

            self.row_offsets = up(_u32(sched.row_offsets))
            self.term_slots = up(_u32(sched.term_slots if len(sched.term_slots) else np.zeros(1, np.uint32)))
            self.term_coefs = up(torch.from_numpy(np.ascontiguousarray(
                sched.term_coefs if len(sched.term_coefs) else np.zeros(1, np.int64))))
            self.lut_idx = up(_u64(luts))
            self.out_idx = up(_u64(dests))
            self.in_idx = torch.arange(max(widest, 1), dtype=torch.int64, device=device)
            self.body = None if sched.num_iconsts else up(_u64(body_words(sched, None)))
            # pool rows of the inputs and outputs: no pageable copy (which waits
            # for the stream) inside a call
            I = sched.num_instances
            self.shared_in_rows = up(torch.from_numpy(sched.addr(sched.shared_input_slots, 0)))
            self.inst_in_rows = up(torch.from_numpy(
                sched.addr(sched.instance_input_slots[None, :], np.arange(I)[:, None]).reshape(-1)))
            self.out_rows = up(torch.from_numpy(sched.output_rows()))
        self.layer_rows = np.ascontiguousarray(sched.layer_rows, dtype=np.uint32)
        self.layer_shared_rows = np.ascontiguousarray(sched.layer_shared_rows, dtype=np.uint32)
        self.widest = widest


class CudaBitCircuitRunner:
    """Runs bit circuits with one `server_key.CudaServerKey` (2_2 blocks)."""

    # device tables kept for this many (circuit, instance count) pairs: a full
    # chunk, a last chunk and a few message lengths
    MAX_TABLES = 4
    # allocator rounding and fragmentation (torch's caching allocator and the
    # library's stream-ordered pool) on top of the counted bytes
    SLACK = 256 << 20

    def __init__(self, server_key):
        self.skey = server_key
        self.streams = server_key.streams
        bsk = server_key.bsk
        self.luts = gpu.CudaGlweCiphertextList.from_glwe_ciphertext_list(
            bc.lut_glwes(bsk.polynomial_size, bsk.glwe_dimension), bsk.glwe_dimension, bsk.polynomial_size,
            self.streams)
        self._tables: "OrderedDict[tuple, _DeviceSchedule]" = OrderedDict()
        self._scratch: Optional[gpu.PbsScratch] = None
        self._scratch_samples = 0

    @property
    def device(self):
        return self.streams.device(0)

    def _scratch_for(self, samples: int) -> gpu.PbsScratch:
        if self._scratch is None or samples > self._scratch_samples:
            if self._scratch is not None:
                self._scratch.close()
            bsk = self.skey.bsk
            self._scratch = gpu.PbsScratch(
                self.streams, bsk.input_lwe_dimension, bsk.glwe_dimension, bsk.polynomial_size,
                bsk.decomp_level_count, samples,
                centered=not self.skey.multi_bit and bsk.ms_noise_reduction_configuration is not None,
                multi_bit=self.skey.multi_bit)
            self._scratch_samples = samples
        return self._scratch

    def close(self):
        if self._scratch is not None:
            self._scratch.close()
            self._scratch = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def device_tables(self, circuit: bc.Circuit, sched: bc.Schedule) -> _DeviceSchedule:
        """The schedule's device tables, uploaded on first use; the least
        recently used pair beyond MAX_TABLES is dropped (its tensors were
        allocated on the work stream, so queued work that reads them is safe).
        A circuit with LUTs of its own gets its own accumulators (the fixed
        set, then its tables); the others share the runner's."""
        key = (circuit, sched.num_instances)
        if key in self._tables:
            self._tables.move_to_end(key)
        else:
            luts = self.luts
            if sched.extra_luts:
                bsk = self.skey.bsk
                luts = gpu.CudaGlweCiphertextList.from_glwe_ciphertext_list(
                    bc.lut_glwes(bsk.polynomial_size, bsk.glwe_dimension, sched.lut_tables()), bsk.glwe_dimension,
                    bsk.polynomial_size, self.streams)
            self._tables[key] = _DeviceSchedule(sched, self.device, self.streams.streams[0], luts)
            while len(self._tables) > self.MAX_TABLES:
                self._tables.popitem(last=False)
        return self._tables[key]

    def pbs_workspace_bytes(self) -> int:
        """Largest stream-ordered workspace one PBS launch of a layer takes:
        the multi-bit low-latency path's key bundle, (n / g) * l * 4 spectra of
        N / 2 complex doubles per sample, for up to one sample per SM (larger
        launches take the fused kernel, which has none); the classic N = 2048
        kernel has none; any other shape may take the generic kernel's
        workspace, at most two CTAs per SM of one SM's shared memory each."""
        bsk = self.skey.bsk
        props = torch.cuda.get_device_properties(self.device)
        sms = props.multi_processor_count
        if self.skey.multi_bit:
            steps = bsk.input_lwe_dimension // bsk.grouping_factor
            return sms * steps * bsk.decomp_level_count * 4 * (bsk.polynomial_size // 2) * 16
        return 2 * sms * props.shared_memory_per_multiprocessor

    def chunk_size(self, circuit: bc.Circuit, num_instances: int) -> int:
        """Instances per call that fit in free device memory, from the bytes a
        call allocates: per instance, its pool slots, its rows of the widest
        layer's staging (big and small LWEs, and the int8 keyswitch's digit
        matrix of big_dim * ks_level bytes per row), its output LWEs, its
        entries of the LUT / destination / body tables; once, the shared slots
        and shared rows and one PBS launch's workspace (pbs_workspace_bytes),
        plus SLACK."""
        one = bc.schedule(circuit, 1)
        big, small = self.skey.big_dim, self.skey.small_dim
        ks_digits = -(-big * self.skey.ksk.decomp_level_count // 64) * 64
        row_bytes = 8 * (big + 1) + 8 * (small + 1) + ks_digits
        per_rows = max([int(one.layer_rows[L + 1] - one.layer_rows[L] - one.layer_shared_rows[L])
                        for L in range(one.num_layers)], default=0)
        per_inst = (8 * (one.num_instance_slots + len(one.output_slots)) * (big + 1) + per_rows * row_bytes
                    + 16 * one.pbs_per_instance_rows + 8 * len(one.row_lut))
        shared_rows = max([int(x) for x in one.layer_shared_rows], default=0)
        fixed = (8 * one.num_shared_slots * (big + 1) + (shared_rows + 128) * row_bytes
                 + self.pbs_workspace_bytes() + self.SLACK)
        free, _ = torch.cuda.mem_get_info(self.device)
        fit = (free - fixed) // max(per_inst, 1)
        return int(max(1, min(num_instances, fit)))

    def run(self, circuit: bc.Circuit, shared, instance=None, iconsts=None, num_instances: int = 1) -> torch.Tensor:
        """shared: [num_shared_inputs, big + 1] int64 blocks; instance:
        [num_instances * num_instance_inputs, big + 1] (instance-major);
        iconsts: [num_instances, num_iconsts] bits.  Returns the outputs
        [num_instances * outputs, big + 1], instance-major."""
        chunk = self.chunk_size(circuit, num_instances)
        outs = []
        for first in range(0, num_instances, chunk):
            n = min(chunk, num_instances - first)
            ni = circuit.num_instance_inputs
            outs.append(self._run_chunk(
                circuit, bc.schedule(circuit, n), shared,
                None if instance is None else instance[first * ni:(first + n) * ni],
                None if iconsts is None else np.asarray(iconsts)[first:first + n]))
        st = self.streams.streams[0]
        with torch.cuda.stream(st):
            out = outs[0] if len(outs) == 1 else torch.cat(outs)
        caller = torch.cuda.current_stream(self.device)
        caller.wait_stream(st)
        out.record_stream(caller)
        return out

    def run_schedule(self, key, sched: bc.Schedule, instance) -> torch.Tensor:
        """A schedule laid out as tables rather than compiled from a circuit
        (`radix_find`'s cross-candidate trees: one instance, inputs at pool
        rows 0 ..), in one call; `key` (hashable) names its device tables.
        instance: [num_instance_inputs, big + 1].  Returns the outputs, with
        the stream rules of `run`."""
        st = self.streams.streams[0]
        out = self._run_chunk(key, sched, None, instance, None)
        caller = torch.cuda.current_stream(self.device)
        caller.wait_stream(st)
        out.record_stream(caller)
        return out

    def trivial(self, digits) -> torch.Tensor:
        """noiseless blocks of the given messages (mask 0, body m * delta),
        [len(digits), big + 1] on the caller's current stream"""
        big = self.skey.big_dim
        out = torch.zeros((len(digits), big + 1), dtype=torch.int64, device=self.device)
        out[:, big] = torch.tensor([int(d) * DELTA for d in digits], dtype=torch.int64)
        return out

    def _run_chunk(self, circuit: bc.Circuit, sched: bc.Schedule, shared, instance, iconsts) -> torch.Tensor:
        L = _lib.lib()
        skey, bsk, ksk = self.skey, self.skey.bsk, self.skey.ksk
        big = skey.big_dim
        st = self.streams.streams[0]
        dev = self.device
        T = self.device_tables(circuit, sched)
        scratch = self._scratch_for(max(T.widest, 1))
        st.wait_stream(torch.cuda.current_stream(dev))  # inputs made on the caller's stream
        with torch.cuda.stream(st):
            pool = torch.empty((sched.pool_rows, big + 1), dtype=torch.int64, device=dev)
            # the inputs are read on st: reserve them for it, so that a caller
            # dropping them right after the call cannot have their memory reused
            # by its own stream before st has read them
            for rows, x in ((T.shared_in_rows, shared), (T.inst_in_rows, instance)):
                if len(rows):
                    x = x.to(dev)
                    pool.index_copy_(0, rows, x)
                    x.record_stream(st)
            body = T.body if T.body is not None else _u64(body_words(sched, iconsts)).to(dev, non_blocking=True)
        sp = self.streams.ptr(0)
        gi = self.streams.gpu_indexes[0]
        L.b200_bit_circuit_64_async(
            sp, gi, pool.data_ptr(), sched.num_shared_slots, sched.num_instances, sched.num_layers,
            T.layer_rows.ctypes.data_as(C.POINTER(C.c_uint32)),
            T.layer_shared_rows.ctypes.data_as(C.POINTER(C.c_uint32)),
            T.row_offsets.data_ptr(), T.term_slots.data_ptr(), T.term_coefs.data_ptr(), body.data_ptr(),
            T.lut_idx.data_ptr(), T.out_idx.data_ptr(), T.in_idx.data_ptr(), ksk.d_vec.as_c_ptr(),
            ksk.decomp_base_log, ksk.decomp_level_count, T.luts.d_vec.as_c_ptr(), bsk.d_vec.as_c_ptr(),
            scratch.buf, big, bsk.input_lwe_dimension, bsk.glwe_dimension, bsk.polynomial_size,
            bsk.decomp_base_log, bsk.decomp_level_count, bsk.grouping_factor if skey.multi_bit else 1)
        with torch.cuda.stream(st):
            return pool.index_select(0, T.out_rows)
