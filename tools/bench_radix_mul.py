#!/usr/bin/env python
"""Cost of radix products and sums on one GPU (CUDA events, L2 flushed before
every timed step, after one warm-up call), FheUint64 (32 blocks of 2_2),
classic PARAM_MESSAGE_2_CARRY_2 and multi-bit
PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2:

  * mul, signed_overflowing_mul, scalar_mul and a 4-operand sum_ciphertexts
    (CudaRadixServerKey methods) at 1 input and at 64 inputs (one call,
    bit-sliced), in ms, operations/s and PBS/s;
  * unchecked_mul (the host-orchestrated BlockEngine path, one integer per
    call) in the same process, at 1 input;
  * every call's PBS count, PBS layers and the CPU time to build and compile
    its circuit (once per circuit; the schedule is cached after that);
  * plain KS + PBS of a batch the size of the call's widest layer, for scale.

Every call runs with the key's work stream as the caller's stream.
Synthetic (random) keys and ciphertexts: the kernels' work does not depend on
their values.  Correctness is covered by tests/test_radix_mul.py.  Prints one
JSON line per measurement, then the card's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--throughput-inputs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5, help="timed steps at one input")
    ap.add_argument("--throughput-reps", type=int, default=2, help="timed steps at --throughput-inputs")
    args = ap.parse_args()
    import torch

    from bench import gpu_identity
    from bench_trivium import plain_ks_pbs
    from tfhe_rs_b200 import bit_circuit as bc, gpu, integer, lib, radix_mul as RM, server_key

    L = lib()
    streams = gpu.CudaStreams.new_single_gpu(0)
    st, sp, dev = streams.streams[0], streams.ptr(0), streams.device(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2
    rng = np.random.default_rng(64)
    k, N, n_blocks = 1, 2048, 32
    W = k * N + 1
    circuits = {"mul": ("mul", None), "signed_overflowing_mul": ("signed_overflowing_mul", None),
                "scalar_mul": ("scalar_mul", None), "sum_ciphertexts (4 operands)": ("sum", 4)}

    compile_s = {}
    for what, (op, count) in circuits.items():
        t0 = time.perf_counter()
        bc.schedule(RM.circuit(op, n_blocks, count), 1)
        compile_s[what] = time.perf_counter() - t0

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

        for mode, inputs, reps in (("latency", 1, args.reps),
                                   ("throughput", args.throughput_inputs, args.throughput_reps)):
            a, b, c, d = (operands(inputs) for _ in range(4))
            sa, sb = operands(inputs, True), operands(inputs, True)
            scalars = [int(x) for x in rng.integers(1, 1 << 63, inputs)]
            for what, fn in (("mul", lambda: rk.mul(a, b)),
                             ("signed_overflowing_mul", lambda: rk.signed_overflowing_mul(sa, sb)),
                             ("scalar_mul", lambda: rk.scalar_mul(a, scalars)),
                             ("sum_ciphertexts (4 operands)", lambda: rk.sum_ciphertexts([a, b, c, d]))):
                op, count = circuits[what]
                circ = RM.circuit(op, n_blocks, count)
                s = bc.schedule(circ, inputs)
                assert rk.runner.chunk_size(circ, inputs) == inputs
                t = timed(fn, reps)
                widest = max(s.layer_outputs(i) for i in range(s.num_layers))
                rec = {"what": f"{what} FheUint64, {name}", "mode": mode, "num_inputs": inputs, "ms": t,
                       "ops_per_s": inputs / t * 1e3, "pbs": s.pbs_count(), "pbs_layers": s.num_layers,
                       "pbs_per_s": s.pbs_count() / t * 1e3, "widest_layer": widest,
                       "cpu_compile_s": compile_s[what],
                       "plain_ks_pbs_widest_layer_ms": plain_ks_pbs(
                           L, torch, gpu, streams, sp, skey, rk, timed, args.reps, rng, n, k, N, g,
                           pbs_base_log, ks_base_log, ks_level, widest)}
                print(json.dumps(rec), flush=True)
        a, b = operands(1), operands(1)
        t = timed(lambda: rk.unchecked_mul(a, b), args.reps)
        rk.engine.pbs_count = 0
        rk.unchecked_mul(a, b)
        print(json.dumps({"what": f"unchecked_mul FheUint64, {name}", "mode": "latency", "num_inputs": 1, "ms": t,
                          "ops_per_s": 1 / t * 1e3, "pbs": rk.engine.pbs_count,
                          "pbs_per_s": rk.engine.pbs_count / t * 1e3}), flush=True)
        streams.synchronize()
        rk.runner.close()
    print(json.dumps({"gpu": gpu_identity(0), "torch_device": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
