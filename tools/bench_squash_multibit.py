"""Time the multi-bit 128-bit PBS of noise squashing
(cuda_multi_bit_programmable_bootstrap_128_async) at the squash shape of
tfhe-rs' GPU parameters, n = 920, k = 2, N = 2048, l = 4, base_log 18,
grouping factor 4, with synthetic keys (uniform u128 words): 16 PBS (one
FheUint64: 32 blocks packed two per LWE) and 2048 (128 FheUint64).  CUDA
events around each call, L2 flushed before every call.

--lib ref runs the same inputs through the reference's own CUDA backend
(oracle/_ref/libtfhe_cuda_backend_ref.so with its multi-bit 128-bit PBS,
built by oracle/build_ref_cuda.sh and oracle/build_ref_pbs128_mb.sh) through the
same C-ABI calls: its key conversion, scratch and bootstrap.

Prints the card's name and power limit with the times, as one JSON line."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMALL_N, K_, N_, L_, BL_, G_ = 920, 2, 2048, 4, 18, 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lib", choices=["ours", "ref"], default="ours")
    ap.add_argument("--counts", type=int, nargs="+", default=[16, 2048])
    args = ap.parse_args()
    if args.lib == "ref":
        ref_so = os.path.join(ROOT, "oracle", "_ref", "libtfhe_cuda_backend_ref.so")
        if not os.path.exists(ref_so):
            raise SystemExit(f"{ref_so} is not built (oracle/build_ref_cuda.sh, oracle/build_ref_pbs128_mb.sh)")
        os.environ["B200_LIB_PATH"] = ref_so
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_squash_multibit.py needs a CUDA device")
    import tfhe_rs_b200

    L = tfhe_rs_b200.lib()
    if not hasattr(L, "cuda_multi_bit_programmable_bootstrap_128_async"):
        raise SystemExit("the library has no cuda_multi_bit_programmable_bootstrap_128_async "
                         "(oracle/build_ref_pbs128_mb.sh)")
    from tfhe_rs_b200 import gpu

    dev = torch.device("cuda:0")
    st = gpu.CudaStreams.new_single_gpu(0)
    torch.cuda.set_stream(st.streams[0])  # the events and every launch on one stream
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(1)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.steps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(torch.cuda.current_stream())
            fn()
            b.record(torch.cuda.current_stream())
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        return float(np.median(ms)), [round(x, 3) for x in ms]

    words = (SMALL_N // G_ << G_) * L_ * (K_ + 1) ** 2 * N_  # u128 words of the key
    h_bsk = rng.integers(0, 2**64, 2 * words, dtype=np.uint64)
    d_bsk = torch.zeros(2 * words, dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    L.cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async(st.ptr(0), 0, d_bsk.data_ptr(),
                                                                      h_bsk.ctypes.data, SMALL_N, K_, L_, N_, G_)
    st.synchronize()
    del h_bsk
    lut = torch.from_numpy(rng.integers(0, 2**63, 2 * (K_ + 1) * N_, dtype=np.uint64).view(np.int64)).to(dev)
    results = {"card": smi, "lib": args.lib,
               "shape": dict(n=SMALL_N, k=K_, N=N_, l=L_, base_log=BL_, grouping_factor=G_),
               "fourier_key_bytes": 2 * words * 8}
    for count in args.counts:
        cts = torch.from_numpy(rng.integers(0, 2**63, count * (SMALL_N + 1), dtype=np.uint64).view(np.int64)).to(dev)
        idx = torch.arange(count, dtype=torch.int64, device=dev)
        out = torch.empty(count * (K_ * N_ + 1) * 2, dtype=torch.int64, device=dev)
        buf = C.POINTER(C.c_int8)()
        sp = st.ptr(0)
        L.scratch_cuda_multi_bit_programmable_bootstrap_128_async(sp, 0, C.byref(buf), K_, N_, L_, count, True)

        def run():
            L.cuda_multi_bit_programmable_bootstrap_128_async(sp, 0, out.data_ptr(), idx.data_ptr(), lut.data_ptr(),
                                                              cts.data_ptr(), idx.data_ptr(), d_bsk.data_ptr(), buf,
                                                              SMALL_N, K_, N_, G_, BL_, L_, count, 1, 0)

        med, all_ms = timed(run)
        L.cleanup_cuda_multi_bit_programmable_bootstrap_128(sp, 0, C.byref(buf))
        kernel = L.b200_last_pbs_kernel().decode() if args.lib == "ours" else "reference (its own dispatch)"
        results[f"pbs128_mb_x{count}"] = dict(ms=med, all_ms=all_ms, kernel=kernel, pbs_per_s=count / (med * 1e-3))
    print(json.dumps(results))


if __name__ == "__main__":
    main()
