#!/usr/bin/env python
"""Cost of vector find and the encrypted key-value store on one GPU (CUDA
events, L2 flushed before every timed call, after one warm-up call),
FheUint64 (32 blocks of 2_2), classic PARAM_MESSAGE_2_CARRY_2 and multi-bit
PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2:

  * kv_store_get and kv_store_update on stores of 64 and 1024 entries
    (FheUint64 keys and values), match_value with 16 and 256 entries
    (FheUint64 in and out) and contains over 64 encrypted FheUint64;
  * per call: PBS count and PBS layers (the per-candidate call then the
    cross-candidate tree), ms and PBS/s, and a plain KS + PBS of a batch the
    size of the call's widest layer, for scale;
  * the host time to build the M = 1024 trees and compile the per-candidate
    circuits (cold caches).

Synthetic (random) keys and ciphertexts: the kernels' work does not depend
on their values.  Correctness is covered by tests/test_radix_find.py and
tests/test_kv_store.py.  Prints one JSON line per measurement, then the
card's name, power limit and SM clocks."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def sm_clocks(gpu_index=0):
    r = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    cur, top = [x.strip() for x in r.stdout.strip().split(",")[:2]]
    return {"sm_clock_mhz": float(cur), "max_sm_clock_mhz": float(top)}


def widest_layer(sched):
    return max([sched.layer_outputs(i) for i in range(sched.num_layers)], default=0)


def host_build_times():
    """seconds to build the M = 1024 trees and compile the per-candidate
    circuits of get and update, from cold caches"""
    from tfhe_rs_b200 import bit_circuit as bc, radix_find as F

    F.tree.cache_clear()
    F._circuit.cache_clear()
    t0 = time.perf_counter()
    F.tree("select", 1024, 33)
    F.tree("any", 1024)
    t1 = time.perf_counter()
    bc.schedule(F.circuit("select", 32, 32), 1024)
    bc.schedule(F.circuit("update", 32, 32), 1024)
    t2 = time.perf_counter()
    return {"what": "host build, M = 1024, FheUint64 get + update", "trees_s": t1 - t0, "circuits_s": t2 - t1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    from bench import gpu_identity
    from bench_trivium import plain_ks_pbs
    from tfhe_rs_b200 import bit_circuit as bc, gpu, integer, kv_store, lib, radix_find as F, server_key

    print(json.dumps(host_build_times()), flush=True)
    L = lib()
    streams = gpu.CudaStreams.new_single_gpu(0)
    st, sp, dev = streams.streams[0], streams.ptr(0), streams.device(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2
    rng = np.random.default_rng(64)
    k, N, nb = 1, 2048, 32
    W = k * N + 1

    def timed(fn, reps):
        """mean device ms of `reps` calls after one warm-up, on stream st"""
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

    def ct():
        with torch.cuda.stream(st):
            return integer.CudaUnsignedRadixCiphertext(
                torch.from_numpy(rng.integers(0, 1 << 63, (nb, W))).to(dev), 1)

    for name, n, g, pbs_base_log, ks_base_log, ks_level in (("classic P22", 918, 1, 23, 4, 4),
                                                           ("multi-bit g=4", 920, 4, 22, 3, 5)):
        num_ggsw = n if g == 1 else (n // g) << g
        h_bsk = rng.integers(0, 1 << 64, size=num_ggsw * 4 * N, dtype=np.uint64)
        h_ksk = rng.integers(0, 1 << 64, size=k * N * ks_level * (n + 1), dtype=np.uint64)
        skey = server_key.upload_server_key(h_bsk, h_ksk, n=n, k=k, N=N, pbs_base_log=pbs_base_log, pbs_level=1,
                                            ks_base_log=ks_base_log, ks_level=ks_level, grouping_factor=g,
                                            centered_ms=g == 1, streams=streams)
        rk = integer.CudaRadixServerKey(skey, None, k, N)
        calls = []
        for M in (64, 1024):
            store = kv_store.CudaKVStore()
            for key in rng.choice(1 << 62, M, replace=False):
                store.insert(int(key), ct())
            q, new = ct(), ct()
            calls.append((f"kv_store_get, {M} entries", "select", M, F.tree("select", M, 1 + nb),
                          lambda store=store, q=q: rk.kv_store_get(store, q)))
            calls.append((f"kv_store_update, {M} entries", "update", M, F.tree("any", M),
                          lambda store=store, q=q, new=new: rk.kv_store_update(store, q, new)))
        for M in (16, 256):
            matches = [(int(a), int(b)) for a, b in zip(rng.choice(1 << 62, M, replace=False),
                                                        rng.integers(0, 1 << 63, M))]
            width = F.num_blocks_for(max(b for _, b in matches))
            q = ct()
            calls.append((f"match_value, {M} entries", "eq_clear", M,
                          F.tree("dot", M, 1, width, tuple(b for _, b in matches)),
                          lambda q=q, matches=matches: rk.match_value(q, matches)))
        cts, q = [ct() for _ in range(64)], ct()
        calls.append(("contains, 64 encrypted", "eq", 64, F.tree("any", 64), lambda: rk.contains(cts, q)))
        for what, op, M, tree, fn in calls:
            per = bc.schedule(F.circuit(op, nb, nb if op in ("select", "update") else 0), M)
            pbs = per.pbs_count() + tree.pbs_count()
            widest = max(widest_layer(per), widest_layer(tree))
            t = timed(fn, args.reps)
            rec = {"what": f"{what} FheUint64, {name}", "ms": t, "pbs": pbs,
                   "pbs_layers": per.num_layers + tree.num_layers, "pbs_per_s": pbs / t * 1e3,
                   "widest_layer": widest,
                   "plain_ks_pbs_widest_layer_ms": plain_ks_pbs(
                       L, torch, gpu, streams, sp, skey, rk, timed, args.reps, rng, n, k, N, g,
                       pbs_base_log, ks_base_log, ks_level, widest)}
            print(json.dumps(rec), flush=True)
        rk.runner.close()
    print(json.dumps({"gpu": gpu_identity(0), **sm_clocks(0), "torch_device": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
