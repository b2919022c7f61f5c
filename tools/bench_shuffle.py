#!/usr/bin/env python
"""Cost of the oblivious bitonic shuffle on one GPU (CUDA events, L2 flushed
before every timed call), FheUint64 data (32 blocks of 2_2), classic
PARAM_MESSAGE_2_CARRY_2 and multi-bit PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2,
lists of 8, 52, 64, 256 and 1024 elements, sort keys by
collision_probability(2^-40) and by num_bits(8):

  * PBS, PBS layers and stages of a shuffle (`radix_shuffle.cost`);
  * ms of a `bitonic_shuffle` call (OPRF sort keys, then the network), and
    its PBS/s against a plain KS + PBS batch the size of its widest layer;
  * the share of the call taken by drawing the sort keys (OPRF), and by
    drawing and re-randomizing them (`bitonic_shuffle_and_re_randomize`);
  * the share taken by the index gathers that build each stage's inputs,
    replayed alone at the same shapes.

Lists up to 256 get one warm-up call at their shape first; a 1024-element
call runs for minutes, so it is timed once, cold (its first stage uploads
its tables).  Synthetic (random) keys and ciphertexts: the kernels' work does
not depend on their values; correctness is covered by
tests/test_radix_shuffle.py.  Prints one JSON line per case, then the card's
name, power limit and SM clocks."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lens", type=int, nargs="+", default=[8, 52, 64, 256, 1024])
    ap.add_argument("--kinds", nargs="+", default=["classic", "multi_bit_g4"])
    args = ap.parse_args()
    import torch

    from bench import gpu_identity
    from bench_find import sm_clocks, widest_layer
    from bench_trivium import plain_ks_pbs
    from tfhe_rs_b200 import bit_circuit as bc, gpu, integer, lib, oprf, radix_shuffle as S, rerand, server_key

    sizes = (("collision_probability(2^-40)", S.BitonicShuffleKeySize.collision_probability(2.0 ** -40)),
             ("num_bits(8)", S.BitonicShuffleKeySize.num_bits(8)))
    if not torch.cuda.is_available():   # the counts only: every time is a GPU's
        for length in args.lens:
            for size_name, size in sizes:
                nk = size.num_blocks(length)
                pbs, layers, stages = S.cost(length, nk, 32)
                print(json.dumps({"what": f"bitonic_shuffle, {length} x FheUint64, keys {size_name}",
                                  "key_blocks": nk, "pbs": pbs * stages, "pbs_per_stage": pbs,
                                  "pbs_layers_per_stage": layers, "stages": stages, "ms": "not measured"}))
        return
    L = lib()
    streams = gpu.CudaStreams.new_single_gpu(0)
    st, sp, dev = streams.streams[0], streams.ptr(0), streams.device(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2
    rng = np.random.default_rng(1024)
    k, N, nb = 1, 2048, 32
    W = k * N + 1

    def timed(fn, reps=1, warm=True):
        """mean device ms of `reps` calls (after one warm-up call when `warm`), on stream st"""
        with torch.cuda.stream(st):
            if warm:
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

    def gathers_ms(length, nk, nd):
        """the stage gathers of one shuffle alone: an index_select of the
        n (nk + nd) input blocks per stage, then the final pick"""
        n = S.next_power_of_two(length)
        E = nk + nd
        with torch.cuda.stream(st):
            store = torch.empty((n * E, W), dtype=torch.int64, device=dev)
            row = np.arange(n, dtype=np.int64)
            srcs = []
            for stage in S.network(n):
                pairs, _ = S.stage_inputs(stage)
                srcs.append(torch.as_tensor((row[pairs.reshape(-1)][:, None] * E + np.arange(E)).reshape(-1),
                                            device=dev))
                row[pairs.reshape(-1)] = np.arange(n)
            keep = torch.as_tensor(row[:length], device=dev)

        def run():
            for src in srcs:
                store.index_select(0, src)
            store.view(n, E, W).index_select(0, keep)
        return timed(run, reps=3)

    for kind in args.kinds:
        g, n, pbs_base_log, ks_base_log, ks_level = (1, 918, 23, 4, 4) if kind == "classic" else (4, 920, 22, 3, 5)
        name = "classic P22" if kind == "classic" else "multi-bit g=4"
        num_ggsw = n if g == 1 else (n // g) << g
        h_bsk = rng.integers(0, 1 << 64, size=num_ggsw * 4 * N, dtype=np.uint64)
        h_ksk = rng.integers(0, 1 << 64, size=k * N * ks_level * (n + 1), dtype=np.uint64)
        skey = server_key.upload_server_key(h_bsk, h_ksk, n=n, k=k, N=N, pbs_base_log=pbs_base_log, pbs_level=1,
                                            ks_base_log=ks_base_log, ks_level=ks_level, grouping_factor=g,
                                            centered_ms=g == 1, streams=streams)
        rk = integer.CudaRadixServerKey(skey, None, k, N)
        okey = oprf.CudaOprfServerKey(skey.bsk, streams)
        cpk = rerand.CudaCompactPublicKey.from_compact_public_key(
            rng.integers(0, 1 << 64, N, dtype=np.uint64), rng.integers(0, 1 << 64, N, dtype=np.uint64), 17, streams)
        rr_key = rerand.CudaReRandomizationKey.derived(cpk)
        ctx = rerand.ReRandomizationContext(b"TFHE_Rrd", b"TFHE_Enc")
        for length in args.lens:
            with torch.cuda.stream(st):
                data = [integer.CudaUnsignedRadixCiphertext(torch.from_numpy(
                    rng.integers(0, 1 << 63, (nb, W))).to(dev), 1) for _ in range(length)]
            for size_name, size in sizes:
                nk = size.num_blocks(length)
                pbs, layers, stages = S.cost(length, nk, nb)
                nkp = nk + (S.next_power_of_two(length) != length)
                widest = widest_layer(bc.schedule(S.circuit(nkp, nb), S.next_power_of_two(length) // 2))
                warm = length <= 256
                call = timed(lambda: rk.bitonic_shuffle(okey, data, size, 7), warm=warm)
                chunks = [2 * nk] * length
                t_oprf = timed(lambda: okey.generate_oblivious_pseudo_random_bits_chunks(7, chunks), reps=3)
                t_rr = timed(lambda: okey.generate_oblivious_pseudo_random_bits_chunks_and_re_randomize(
                    7, chunks, rr_key, ctx), reps=3)
                t_gather = gathers_ms(length, nkp, nb)
                total = pbs * stages
                rec = {"what": f"bitonic_shuffle, {length} x FheUint64, keys {size_name}, {name}",
                       "key_blocks": nk, "pbs": total, "pbs_per_stage": pbs, "pbs_layers_per_stage": layers,
                       "stages": stages, "ms": call, "warm": warm, "pbs_per_s": total / call * 1e3,
                       "widest_layer": widest,
                       "plain_ks_pbs_widest_layer_pbs_per_s": widest / plain_ks_pbs(
                           L, torch, gpu, streams, sp, skey, rk, timed, 3, rng, n, k, N, g, pbs_base_log,
                           ks_base_log, ks_level, widest) * 1e3,
                       "oprf_ms": t_oprf, "oprf_share": t_oprf / call,
                       "oprf_rerand_ms": t_rr, "oprf_rerand_share": t_rr / call,
                       "gather_ms": t_gather, "gather_share": t_gather / call}
                print(json.dumps(rec), flush=True)
            del data
        rk.runner.close()
    print(json.dumps({"gpu": gpu_identity(0), **sm_clocks(0), "torch_device": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
