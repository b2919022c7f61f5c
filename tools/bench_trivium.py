#!/usr/bin/env python
"""Cost of homomorphic Trivium and Kreyvium on one GPU (CUDA events, L2
flushed before every timed step), classic PARAM_MESSAGE_2_CARRY_2 and
multi-bit PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2:

  * CudaTriviumServerKey.{trivium,kreyvium}_{init, next(64), next(512),
    generate_keystream(512)} at num_inputs in {1, 16, 64}: ms per call, PBS
    count and PBS layers per call;
  * apply_keystream of 1 KiB and 64 KiB streams (one PBS per 2 bits).  A
    1 MiB stream is not timed: its 8,388,608 keystream LWEs alone take 137 GB
    at this LWE size (2,049 words), more than the card holds;
  * plain KS + PBS (cuda_keyswitch_lwe_ciphertext_vector_64_64_async +
    cuda_[multi_bit_]programmable_bootstrap_64_async) of a batch the size of
    generate_keystream(512)'s widest layer, for scale.

Every call runs with the key's work stream as the caller's stream, so the
events cover the host-side register shifts too.  Synthetic (random) keys and
ciphertexts: the kernels' work does not depend on their values.  Correctness
is covered by tests/test_trivium.py.  Prints one JSON line per measurement,
then the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", default="1,16,64")
    ap.add_argument("--stream-kib", default="1,64")
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch

    from bench import gpu_identity
    from tfhe_rs_b200 import bit_circuit as bc, gpu, lib, server_key, trivium as T

    L = lib()
    streams = gpu.CudaStreams.new_single_gpu(0)
    st, sp, dev = streams.streams[0], streams.ptr(0), streams.device(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2
    rng = np.random.default_rng(7)
    k, N = 1, 2048
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
        tk = T.CudaTriviumServerKey(skey)
        for cipher in ("trivium", "kreyvium"):
            kb = T.KEY_BITS[cipher]
            init, nxt = getattr(tk, f"{cipher}_init"), getattr(tk, f"{cipher}_next")
            gen = getattr(tk, f"{cipher}_generate_keystream")
            for inputs in [int(x) for x in args.inputs.split(",")]:
                key, iv = rand_blocks(kb * inputs), rand_blocks(kb * inputs)
                with torch.cuda.stream(st):
                    state = init(key, iv, inputs)
                calls = [("init", 0, lambda: init(key, iv, inputs)),
                         ("next", 64, lambda: nxt(state, 64)),
                         ("next", 512, lambda: nxt(state, 512)),
                         ("generate_keystream", 512, lambda: gen(key, iv, 512, inputs))]
                for what, steps, fn in calls:
                    kind = {"init": f"{cipher}_init", "next": f"{cipher}_next",
                            "generate_keystream": f"{cipher}_keystream"}[what]
                    s = bc.schedule(T.circuit(kind, steps), inputs)
                    assert tk.runner.chunk_size(T.circuit(kind, steps), inputs) == inputs
                    t = timed(fn, args.reps)
                    rec = {"what": f"{cipher} {what}" + (f"({steps})" if steps else "") + ", " + name,
                           "num_inputs": inputs, "ms": t, "ms_per_input": t / inputs, "pbs": s.pbs_count(),
                           "pbs_layers": s.num_layers, "pbs_per_s": s.pbs_count() / t * 1e3}
                    if what == "generate_keystream":
                        widest = max(s.layer_outputs(i) for i in range(s.num_layers))
                        rec["widest_layer"] = widest
                        rec["plain_ks_pbs_widest_layer_ms"] = plain_ks_pbs(
                            L, torch, gpu, streams, sp, skey, tk, timed, args.reps, rng, n, k, N, g, pbs_base_log,
                            ks_base_log, ks_level, widest)
                    print(json.dumps(rec), flush=True)
                del key, iv, state
        for kib in [int(x) for x in args.stream_kib.split(",")]:
            n_bits = 8192 * kib
            ks = rand_blocks(n_bits)
            data = rng.integers(0, 256, n_bits // 8, dtype=np.uint8).tobytes()
            blocks = n_bits // 2
            assert tk.runner.chunk_size(T.circuit("apply_keystream"), blocks) == blocks
            t = timed(lambda: T.apply_keystream(tk, ks, data, n_bits), args.reps)
            print(json.dumps({"what": "apply_keystream, " + name, "stream_bytes": n_bits // 8, "ms": t,
                              "pbs": blocks, "pbs_layers": 1, "pbs_per_s": blocks / t * 1e3,
                              "MB_per_s": n_bits / 8 / t / 1e3}), flush=True)
            del ks
        tk.runner.close()
    print(json.dumps({"gpu": gpu_identity(0), "torch_device": torch.cuda.get_device_name(0)}))


def plain_ks_pbs(L, torch, gpu, streams, sp, skey, tk, timed, reps, rng, n, k, N, g, pbs_base_log, ks_base_log,
                 ks_level, rows):
    """ms of one keyswitch + PBS batch of `rows` LWEs on the same keys"""
    big = gpu.CudaLweCiphertextList.from_lwe_ciphertext_list(
        rng.integers(0, 1 << 63, (rows, k * N + 1)).astype(np.uint64), streams)
    small = gpu.CudaLweCiphertextList.new(n, rows, streams)
    out = gpu.CudaLweCiphertextList.new(k * N, rows, streams)
    lut_idx = gpu.CudaVec.new(rows, streams)
    triv = gpu.trivial_indexes(rows, streams)
    scratch = gpu.PbsScratch(streams, n, k, N, 1, rows, centered=g == 1, multi_bit=g > 1)
    bsk, ksk = skey.bsk, skey.ksk

    def ks_pbs():
        L.cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
            sp, 0, small.d_vec.as_c_ptr(), triv.as_c_ptr(), big.d_vec.as_c_ptr(), triv.as_c_ptr(),
            ksk.d_vec.as_c_ptr(), k * N, n, ks_base_log, ks_level, rows)
        a = (sp, 0, out.d_vec.as_c_ptr(), triv.as_c_ptr(), tk.runner.luts.d_vec.as_c_ptr(),
             lut_idx.as_c_ptr(), small.d_vec.as_c_ptr(), triv.as_c_ptr(), bsk.d_vec.as_c_ptr(), scratch.buf,
             n, k, N)
        if g == 1:
            L.cuda_programmable_bootstrap_64_async(*a, pbs_base_log, 1, rows, 1, 0)
        else:
            L.cuda_multi_bit_programmable_bootstrap_64_async(*a, g, pbs_base_log, 1, rows, 1, 0)

    t = timed(ks_pbs, reps)
    scratch.close()
    return t


if __name__ == "__main__":
    main()
