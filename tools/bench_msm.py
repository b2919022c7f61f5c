#!/usr/bin/env python
"""Latency of the BLS12-446 G1 / G2 multi-scalar multiplications of
include/tfhe_b200_zk.h on one GPU, at the sizes of tfhe-zk-pok's PKE v2
verify (about 128 to 4,100 points per call with the compact-key parameters)
and above:

  * the device-resident call (g{1,2}_msm_unmanaged_wrapper_async, caller
    scratch): CUDA events around the call, mean over --reps after a warm-up;
  * the managed host-array call (g{1,2}_msm_managed_wrapper, points in normal
    form as tfhe-zk-pok passes them): host wall time of the synchronous call;
  * the per-phase split of one device call (torch.profiler kernel times:
    digits, sort, accumulation, reduction, window sums) and the host Horner
    combination (b200_last_msm_combine_us), with its share of the call;
  * an IMAD bound computed from the shapes: the field multiplications the
    algorithm needs at the chosen window size (mixed additions 10 M, XYZZ
    additions 14 M, doublings 9 M; an Fp2 product is 3 M) times the 784
    IMADs of one 14-limb Montgomery product, over 64 IMAD/clk/SM at the
    card's maximum SM clock.  The host combination is not in it.

With --lib ref the reference's zk-cuda-backend (oracle/_ref/
libzk_cuda_backend_ref.so, oracle/build_ref_zk.sh) runs the same inputs in the
same session, and its normalized results must equal this library's word for
word.  Points are known multiples of the generators (tests/bls12_446_model.py),
4,096 distinct ones tiled up to n; scalars are uniform below r.  Prints one
JSON line per (group, n, library), then the card's name and power limit."""
import argparse
import ctypes as C
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = (("digits", ("msm_digits",)), ("sort", ("RadixSort", "Onesweep")),
          ("accumulation", ("bucket_bounds", "task_count", "DeviceScan", "ScanKernel", "InitKernel",
                            "msm_accumulate", "bucket_tree")),
          ("reduction", ("bucket_reduce",)), ("window_sums", ("window_sum",)))


def _inputs(name, n, seed):
    from tests import bls12_446_model as M
    from tfhe_rs_b200 import zk

    curve, g = (M.G1, zk.G1) if name == "g1" else (M.G2, zk.G2)
    base = min(n, 4096)
    logs, pts = M.known_multiples(curve, base, random.Random(seed))
    rng = random.Random(seed + n)
    ks = [rng.randrange(M.R_ORDER) for _ in range(n)]
    normal = zk.points(g, pts)
    idx = np.arange(n) % base
    return curve, g, [logs[i] for i in idx], normal[idx], ks


def _to_mont(L, g, normal):
    """Montgomery-form copy of ABI points through fp_to_montgomery_wrapper."""
    out = normal.copy()
    src, dst = np.zeros(7, np.uint64), np.zeros(7, np.uint64)
    for i in range(len(normal)):
        for f in ("x", "y"):
            for c in (out[i][f].reshape(-1, 7)):
                src[:] = c
                L.fp_to_montgomery_wrapper(dst.ctypes.data, src.ctypes.data)
                c[:] = dst
    return out


def _imad_bound_ms(name, n, cfg, sms, clock_mhz):
    c, W = (int(cfg[k]) for k in ("c", "windows"))
    S = int(cfg["segments"])
    B = 1 << (c - 1)
    madds = n * -(-299 // c)  # scalars below r: about 299 / c nonzero digits each
    adds = 2 * W * B + 3 * W * S
    dbls = W * (B // S).bit_length()
    muls = 10 * madds + 14 * adds + 9 * dbls
    muls *= 3 if name == "g2" else 1
    return muls * 784 / (64 * sms * clock_mhz * 1e3)


def _max_sm_clock_mhz():
    import subprocess

    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    return float(r.stdout.strip())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="128,2048,4100,16384,65536")
    ap.add_argument("--groups", default="g1,g2")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--lib", choices=("b200", "ref"), default="b200")
    args = ap.parse_args()

    import torch

    from bench import gpu_identity
    from tfhe_rs_b200 import _lib, gpu, zk

    assert torch.cuda.is_available(), "bench_msm needs a CUDA device"
    L = _lib.lib()
    R = _lib.load_zk() if args.lib == "ref" else None
    ident = gpu_identity(0)
    props = torch.cuda.get_device_properties(0)
    clock_mhz = _max_sm_clock_mhz()
    streams = gpu.CudaStreams.new_single_gpu(0)
    st = streams.streams[0]
    for name in args.groups.split(","):
        for n in (int(s) for s in args.sizes.split(",")):
            curve, g, logs, normal, ks_int = _inputs(name, n, 1)
            ks = zk.scalars(ks_int)
            montp = _to_mont(L, g, normal)
            d_pts, d_ks = zk.to_device(montp, streams), zk.to_device(ks, streams)
            rows = [("b200", L)] + ([("ref", R)] if R is not None else [])
            results = {}
            for lib_name, lib in rows:
                scratch_bytes = int(getattr(lib, f"pippenger_scratch_size_{name}_wrapper")(n, 0))
                with torch.cuda.stream(st):
                    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device="cuda:0")
                raw = np.zeros(g.proj_shape, np.uint64)
                unmanaged = getattr(lib, f"{name}_msm_unmanaged_wrapper_async")

                def dev_call():
                    unmanaged(streams.ptr(0), 0, raw.ctypes.data, d_pts.data_ptr(), d_ks.data_ptr(), n,
                              scratch.data_ptr())

                managed = getattr(lib, f"{name}_msm_managed_wrapper")
                mraw = np.zeros(g.proj_shape, np.uint64)
                tracker = C.c_uint64(0)

                def host_call():
                    managed(streams.ptr(0), 0, mraw.ctypes.data, normal.ctypes.data, ks.ctypes.data, n, False,
                            C.byref(tracker))

                for _ in range(2):
                    dev_call(), host_call()
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                combine = 0.0
                start.record(st)
                for _ in range(args.reps):
                    dev_call()
                    if lib is L:
                        combine += L.b200_last_msm_combine_us()
                stop.record(st)
                stop.synchronize()
                dev_ms = start.elapsed_time(stop) / args.reps
                t0 = time.perf_counter()
                for _ in range(args.reps):
                    host_call()
                managed_ms = (time.perf_counter() - t0) * 1e3 / args.reps
                norm = zk.normalize(g, raw)
                assert norm.tobytes() == zk.normalize(g, mraw).tobytes(), "managed and unmanaged calls differ"
                results[lib_name] = norm
                row = {"group": name.upper(), "n": n, "lib": lib_name, "device_call_ms": round(dev_ms, 4),
                       "managed_call_ms": round(managed_ms, 4)}
                if lib is L:
                    cfg = dict(kv.split("=", 1) for kv in L.b200_last_msm_config().decode().split())
                    row["config"] = {k: cfg[k] for k in ("c", "windows", "task", "segments")}
                    row["host_combine_ms"] = round(combine / args.reps / 1e3, 4)
                    row["host_combine_share"] = round(combine / args.reps / 1e3 / dev_ms, 3)
                    from torch.profiler import ProfilerActivity, profile

                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        dev_call()
                    split = {k: 0.0 for k, _ in PHASES}
                    for ev in prof.key_averages():
                        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / 1e3
                        for phase, keys in PHASES:
                            if any(k in ev.key for k in keys):
                                split[phase] += t
                                break
                    row["phase_ms"] = {k: round(v, 4) for k, v in split.items()}
                    row["phase_ms"]["host_combination"] = row["host_combine_ms"]
                    gpu_ms = sum(split.values())
                    row["imad_bound_ms"] = round(_imad_bound_ms(name, n, cfg, props.multi_processor_count,
                                                                clock_mhz), 4)
                    row["imad_bound_share_of_kernels"] = round(row["imad_bound_ms"] / gpu_ms, 3) if gpu_ms else None
                print(json.dumps(row), flush=True)
                del scratch
            if "ref" in results:
                assert results["ref"].tobytes() == results["b200"].tobytes(), f"{name} n={n}: results differ"
            from tests import bls12_446_model as M

            want = M.msm_by_logs(curve, ks_int, logs)
            assert zk.normalized_to_affine(g, results["b200"]) == want, f"{name} n={n}: wrong result"
    print(json.dumps({"gpu": ident, "torch_device": torch.cuda.get_device_name(0),
                      "sms": props.multi_processor_count, "clocks_max_sm_mhz": clock_mhz}))


if __name__ == "__main__":
    main()
