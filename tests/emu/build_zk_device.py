"""Builds the device side of the BLS12-446 field and curve tests with the
library's nvcc and flags: tfhe-rs_b200/csrc/bls12_446.cuh's sm_90a path behind
the batched C interface of tests/emu/zk_device.cu (tests/emu/libzk_device.so)."""
import os
import subprocess

from tests.emu.build_pbs128 import CSRC, HERE

LIB = os.path.join(HERE, "libzk_device.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-shared",
         "-Xcompiler", "-fPIC"]


def build() -> str:
    src = os.path.join(HERE, "zk_device.cu")
    deps = [src, os.path.join(CSRC, "bls12_446.cuh"),
            os.path.join(os.path.dirname(os.path.dirname(CSRC)), "include", "tfhe_b200_zk.h")]
    if os.path.exists(LIB) and os.path.getmtime(LIB) >= max(os.path.getmtime(d) for d in deps):
        return LIB
    subprocess.check_call([NVCC] + FLAGS + [src, "-o", LIB + ".tmp"])
    os.replace(LIB + ".tmp", LIB)
    return LIB
