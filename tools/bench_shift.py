#!/usr/bin/env python
"""Cost of radix shifts, rotations and bit counts on one GPU (CUDA events, L2
flushed before every timed step, after one warm-up call), FheUint64 (32
blocks of 2_2), classic PARAM_MESSAGE_2_CARRY_2 and multi-bit
PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2:

  * left_shift and signed right_shift by an FheUint64 amount, rotate_left,
    scalar_left_shift by an odd clear amount (13), leading_zeros, count_ones
    and ilog2 (CudaRadixServerKey methods), at 1 input and at 256 inputs
    (one call, bit-sliced), in ms, operations/s and PBS/s;
  * every call's PBS count and PBS layers;
  * plain KS + PBS of a batch the size of the call's widest layer, for scale.

Every call runs with the key's work stream as the caller's stream.
Synthetic (random) keys and ciphertexts: the kernels' work does not depend on
their values.  Correctness is covered by tests/test_radix_bits.py.  Prints one
JSON line per measurement, then the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SCALAR_AMOUNT = 13


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--throughput-inputs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    from bench import gpu_identity
    from bench_trivium import plain_ks_pbs
    from tfhe_rs_b200 import bit_circuit as bc, gpu, integer, lib, radix_bits as RB, server_key

    L = lib()
    streams = gpu.CudaStreams.new_single_gpu(0)
    st, sp, dev = streams.streams[0], streams.ptr(0), streams.device(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2
    rng = np.random.default_rng(64)
    k, N, n_blocks = 1, 2048, 32
    W = k * N + 1

    def timed(fn, reps):
        """mean device ms of `reps` steps after one warm-up, on stream st"""
        with torch.cuda.stream(st):
            fn()
            st.synchronize()
            ms = 0.0
            for _ in range(reps):
                flush_buf.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                fn()
                b.record(st)
                b.synchronize()
                ms += a.elapsed_time(b)
        return ms / reps

    def rand_blocks(rows):
        with torch.cuda.stream(st):
            return torch.from_numpy(rng.integers(0, 1 << 63, (rows, W))).to(dev)

    for name, n, g, pbs_base_log, ks_base_log, ks_level in (("classic P22", 918, 1, 23, 4, 4),
                                                           ("multi-bit g=4", 920, 4, 22, 3, 5)):
        num_ggsw = n if g == 1 else (n // g) << g
        h_bsk = rng.integers(0, 1 << 64, size=num_ggsw * 4 * N, dtype=np.uint64)
        h_ksk = rng.integers(0, 1 << 64, size=k * N * ks_level * (n + 1), dtype=np.uint64)
        skey = server_key.upload_server_key(h_bsk, h_ksk, n=n, k=k, N=N, pbs_base_log=pbs_base_log, pbs_level=1,
                                            ks_base_log=ks_base_log, ks_level=ks_level, grouping_factor=g,
                                            centered_ms=g == 1, streams=streams)
        rk = integer.CudaRadixServerKey(skey, None, k, N)

        def operands(inputs, signed=False):
            kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
            return kind(rand_blocks(n_blocks * inputs), inputs)

        for mode, inputs in (("latency", 1), ("throughput", args.throughput_inputs)):
            a, amount, sa = operands(inputs), operands(inputs), operands(inputs, True)
            calls = (
                ("left_shift", ("left_shift", False, n_blocks), lambda: rk.left_shift(a, amount)),
                ("signed right_shift", ("right_shift", True, n_blocks), lambda: rk.right_shift(sa, amount)),
                ("rotate_left", ("rotate_left", False, n_blocks), lambda: rk.rotate_left(a, amount)),
                (f"scalar_left_shift by {SCALAR_AMOUNT}", ("scalar_left_shift", False, SCALAR_AMOUNT),
                 lambda: rk.scalar_left_shift(a, SCALAR_AMOUNT)),
                ("leading_zeros", ("leading_zeros", False, None), lambda: rk.leading_zeros(a)),
                ("count_ones", ("count_ones", False, None), lambda: rk.count_ones(a)),
                ("ilog2", ("ilog2", False, None), lambda: rk.ilog2(a)),
            )
            for what, (op, signed, arg), fn in calls:
                circ = RB.circuit(op, n_blocks, signed, arg)
                s = bc.schedule(circ, inputs)
                assert rk.runner.chunk_size(circ, inputs) == inputs
                t = timed(fn, args.reps)
                widest = max(s.layer_outputs(i) for i in range(s.num_layers))
                rec = {"what": f"{what} FheUint64, {name}", "mode": mode, "num_inputs": inputs, "ms": t,
                       "ops_per_s": inputs / t * 1e3, "pbs": s.pbs_count(), "pbs_layers": s.num_layers,
                       "pbs_per_s": s.pbs_count() / t * 1e3, "widest_layer": widest,
                       "plain_ks_pbs_widest_layer_ms": plain_ks_pbs(
                           L, torch, gpu, streams, sp, skey, rk, timed, args.reps, rng, n, k, N, g,
                           pbs_base_log, ks_base_log, ks_level, widest)}
                print(json.dumps(rec), flush=True)
        rk.runner.close()
    print(json.dumps({"gpu": gpu_identity(0), "torch_device": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
