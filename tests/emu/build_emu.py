"""Builds the CPU CTA emulator (tests/emu/libemu_p22.so) with g++."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "libemu_p22.so")
SRC = os.path.join(HERE, "emu_p22.cpp")
CSRC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "tfhe-rs_b200", "csrc")


def build_no_contract(dest: str) -> dict:
    """emu_p22.cpp, emu_lanepair.cpp and emu_pbs128.cpp built into `dest`
    without floating-point contraction, {source name: library path}.  g++ would otherwise fuse
    multiplies and adds wherever the shape of the surrounding code lets it,
    differently in the two files and differently from the kernels; without it
    both replays evaluate the kernels' expressions in source order, which is
    what nvcc -fmad=false does on the device (tests/emu/build_nofma.py).  The
    explicit fma calls of the double-double arithmetic (dd.cuh) stay fused on
    both sides, and are correctly rounded on both."""
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    out = {}
    for src in ("emu_p22.cpp", "emu_lanepair.cpp", "emu_pbs128.cpp"):
        lib = os.path.join(dest, src.replace(".cpp", "_nocontract.so"))
        subprocess.check_call([gxx, "-O2", "-mavx2", "-mfma", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
                               "-w", "-x", "c++", os.path.join(HERE, src), "-o", lib])
        out[src] = lib
    return out


def build() -> str:
    deps = [SRC] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    if os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(d) for d in deps):
        return OUT
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-O2", "-mavx2", "-mfma", "-std=c++17", "-fPIC", "-shared", "-x", "c++", SRC,
                           "-o", OUT])
    return OUT
