"""Builds a test copy of the library without floating-point contraction:
tfhe-rs_b200/csrc/b200_backend.cu with csrc/Makefile's NVFLAGS plus
-fmad=false, into tests/emu/libtfhe_cuda_backend_b200_nofma.so.

nvcc otherwise fuses `a*b + c` into DFMAs wherever the expression allows it,
and the CPU replays of the PBS kernels (emu_p22.cpp, emu_lanepair.cpp, built
with -ffp-contract=off) do not.  Without contraction the kernels evaluate the
same expressions in the same order with the same IEEE rounding as the replays,
so the two can be compared word for word (tests/test_gpu_replay_words.py).
The library exports the same C ABI; tests load it with tfhe_rs_b200._lib.load.
It is never the product library."""
import os
import re
import subprocess

from tests.emu.build_emu import CSRC, HERE

LIB = os.path.join(HERE, "libtfhe_cuda_backend_b200_nofma.so")
MAKEFILE = os.path.join(CSRC, "Makefile")
EXTRA = ["-fmad=false"]


def makefile_vars(path: str = MAKEFILE) -> dict:
    """The `NAME ?= value` / `NAME := value` assignments of the Makefile, line
    continuations joined and $(NAME) references to earlier ones expanded."""
    with open(path) as f:
        text = f.read().replace("\\\n", " ")
    out = {}
    for line in text.splitlines():
        m = re.match(r"^([A-Z_]+)\s*[:?]?=\s*(.*)$", line)
        if m:
            out[m.group(1)] = re.sub(r"\$\((\w+)\)", lambda r: out.get(r.group(1), ""), m.group(2)).strip()
    return out


def flags() -> list:
    """csrc/Makefile's NVFLAGS, then -fmad=false: nothing else differs."""
    return makefile_vars()["NVFLAGS"].split() + EXTRA


def command(out: str) -> list:
    v = makefile_vars()
    nvcc = os.environ.get("NVCC", v["NVCC"])
    return [nvcc] + flags() + ["-shared", "-o", out, v["SRCS"]]


def build() -> str:
    v = makefile_vars()
    deps = [MAKEFILE, os.path.join(CSRC, v["SRCS"])] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)
                                                        if f.endswith(".cuh")]
    inc = os.path.join(os.path.dirname(os.path.dirname(CSRC)), "include")
    deps += [os.path.join(inc, f) for f in os.listdir(inc) if f.endswith(".h")]
    if os.path.exists(LIB) and os.path.getmtime(LIB) >= max(os.path.getmtime(d) for d in deps):
        return LIB
    r = subprocess.run(command(LIB + ".tmp"), cwd=CSRC, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc build of %s failed:\n%s" % (os.path.basename(LIB), r.stderr[-4000:]))
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build())
