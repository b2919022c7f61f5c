"""Builds the CPU side of the BLS12-446 MSM tests with g++: tfhe-rs_b200/csrc/
bls12_446.cuh's host path behind the small C interface of tests/emu/zk_host.cpp
(tests/emu/libzk_host.so)."""
import os

from tests.emu.build_pbs128 import CSRC, HERE, _compile

LIB = os.path.join(HERE, "libzk_host.so")


def build() -> str:
    root = os.path.dirname(CSRC)
    deps = [os.path.join(CSRC, "bls12_446.cuh"), os.path.join(os.path.dirname(root), "include", "tfhe_b200_zk.h")]
    return _compile(os.path.join(HERE, "zk_host.cpp"), LIB, deps)
