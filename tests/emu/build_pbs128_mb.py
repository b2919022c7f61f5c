"""Builds the CPU side of the multi-bit 128-bit PBS tests with g++: the exact
multi-bit u128 blind rotation (tests/emu/libpbs128_mb_exact.so, no kernel
source) and the model of the kernel's folded MAC (tests/emu/
libemu_pbs128_mb.so)."""
import os

from tests.emu.build_pbs128 import CSRC, HERE, _compile

EXACT = os.path.join(HERE, "libpbs128_mb_exact.so")
MODEL = os.path.join(HERE, "libemu_pbs128_mb.so")


def build() -> tuple:
    """(exact library, model library)."""
    kernel_headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    return (_compile(os.path.join(HERE, "pbs128_mb_exact.cpp"), EXACT, [os.path.join(HERE, "pbs128_exact.cpp")]),
            _compile(os.path.join(HERE, "emu_pbs128_mb.cpp"), MODEL, kernel_headers))
