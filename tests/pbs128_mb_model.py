"""CPU side of the multi-bit 128-bit PBS tests: the exact multi-bit u128 blind
rotation (tests/emu/pbs128_mb_exact.cpp) and the kernel's folded MAC
(tests/emu/emu_pbs128_mb.cpp).  u128 arrays are numpy (..., 2) uint64, low
word then high word, as in tests/pbs128_model.py."""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass

import numpy as np

from tests import pbs128_model as P
from tests.pbs128_model import Params128, zeros128

vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64


@functools.lru_cache(maxsize=1)
def _libs():
    from tests.emu.build_pbs128_mb import build

    exact_path, model_path = build()
    exact, model = C.CDLL(exact_path), C.CDLL(model_path)
    sigs = {
        exact: {
            "p128mb_gen_bsk": [u64, vp, u32, vp, u32, u32, u32, u32, u32, u32, vp],
            "p128mb_degrees": [vp, u32, u32, vp],
            "p128mb_pbs_exact": [vp, vp, vp, u32, u32, u32, u32, u32, u32, u32, vp],
        },
        model: {
            "emu128_mb_product": [vp, vp, vp, u32, u32, vp],
            "emu128_mb_degrees": [vp, u32, u32, vp],
            "emu128_mb_pbs": [vp, vp, vp, u32, u32, u32, u32, u32, u32, vp],
        },
    }
    for dll, table in sigs.items():
        for name, args in table.items():
            getattr(dll, name).argtypes = args
            getattr(dll, name).restype = None
    return exact, model


def lib() -> C.CDLL:
    """The exact multi-bit u128 blind rotation (shares no code with the kernel)."""
    return _libs()[0]


def model() -> C.CDLL:
    """The kernel's folded MAC compiled for the CPU."""
    return _libs()[1]


def _p(a: np.ndarray):
    assert a.flags.c_contiguous
    return a.ctypes.data_as(vp)


@dataclass
class KeysMb:
    params: Params128
    grouping: int
    lwe_sk: np.ndarray  # n u64 bits
    glwe_sk: np.ndarray  # k*N u64 bits
    bsk: np.ndarray  # [n/g][2^g][l][k+1][k+1][N] u128


def ggsw_words(p: Params128) -> int:
    return p.level * (p.k + 1) ** 2 * p.N


def keygen(p: Params128, g: int, seed: int, lwe_sk: np.ndarray | None = None,
           glwe_sk: np.ndarray | None = None) -> KeysMb:
    rng = np.random.default_rng(seed)
    if lwe_sk is None:
        lwe_sk = rng.integers(0, 2, p.n, dtype=np.uint64)
    if glwe_sk is None:
        glwe_sk = rng.integers(0, 2, p.k * p.N, dtype=np.uint64)
    lwe_sk, glwe_sk = np.ascontiguousarray(lwe_sk, dtype=np.uint64), np.ascontiguousarray(glwe_sk, dtype=np.uint64)
    bsk = zeros128((p.n // g << g) * ggsw_words(p))
    lib().p128mb_gen_bsk(C.c_uint64(seed), _p(lwe_sk), p.n, _p(glwe_sk), p.k, p.N, p.base_log, p.level, g,
                         p.glwe_noise_log2, _p(bsk))
    return KeysMb(p, g, lwe_sk, glwe_sk, bsk)


def pooled_keygen(p: Params128, g: int, seed: int, lwe_sk: np.ndarray, glwe_sk: np.ndarray | None = None) -> KeysMb:
    """A key for any n (a multiple of g) from 2^g generated groups, one per
    pattern of g key bits: group j of the key is the pool group of its bits.
    Key generation then costs 2^g groups whatever n is."""
    patterns = np.array([(b >> (g - 1 - u)) & 1 for b in range(1 << g) for u in range(g)], dtype=np.uint64)
    pool = keygen(Params128(n=g << g, k=p.k, N=p.N, base_log=p.base_log, level=p.level,
                            glwe_noise_log2=p.glwe_noise_log2), g, seed, patterns, glwe_sk)
    lwe_sk = np.ascontiguousarray(lwe_sk, dtype=np.uint64)
    bits = lwe_sk.reshape(-1, g).astype(np.int64)
    pick = (bits << np.arange(g - 1, -1, -1)).sum(axis=1)
    group = (1 << g) * ggsw_words(p)
    bsk = np.ascontiguousarray(pool.bsk.reshape(1 << g, group, 2)[pick].reshape(-1, 2))
    return KeysMb(p, g, lwe_sk, pool.glwe_sk, bsk)


def degrees(mask, g: int, log_mod: int) -> list:
    """The exact model's degrees of GGSWs 1..2^g-1 of one group."""
    m = np.ascontiguousarray(mask, dtype=np.uint64)
    out = np.zeros((1 << g) - 1, dtype=np.uint32)
    lib().p128mb_degrees(_p(m), g, log_mod, _p(out))
    return [int(x) for x in out]


def kernel_degrees(mask, g: int, log_mod: int) -> list:
    """The kernel's degrees of GGSWs 0..2^g-1 (p128_mb_degree)."""
    m = np.ascontiguousarray(mask, dtype=np.uint64)
    out = np.zeros(1 << g, dtype=np.uint32)
    model().emu128_mb_degrees(_p(m), g, log_mod, _p(out))
    return [int(x) for x in out]


def replay_pbs(keys: KeysMb, lut: np.ndarray, cts: np.ndarray) -> np.ndarray:
    """The kernel replayed on the CPU (emu128_mb_pbs) on the key as the kernel
    converts it (emu128_bsk_convert of the classic model): (count, k*N + 1, 2)."""
    p = keys.params
    bskf = np.zeros(keys.bsk.size, dtype=np.float64)
    emu = P.model()
    emu.emu128_bsk_convert.argtypes = [vp, u64, u32, vp]
    emu.emu128_bsk_convert(_p(keys.bsk), C.c_uint64(keys.bsk.shape[0] // p.N), p.N, _p(bskf))
    cts = np.ascontiguousarray(cts, dtype=np.uint64).reshape(-1, p.n + 1)
    out = zeros128(cts.shape[0], p.k * p.N + 1)
    lut = np.ascontiguousarray(lut)
    for s in range(cts.shape[0]):
        model().emu128_mb_pbs(_p(bskf), _p(lut), _p(cts[s]), p.n, p.k, p.N, keys.grouping, p.base_log, p.level,
                              _p(out[s]))
    return out


def pbs_exact(keys: KeysMb, lut: np.ndarray, cts: np.ndarray) -> np.ndarray:
    """cts: (count, n + 1) u64 LWEs -> (count, k*N + 1, 2) u128 LWEs."""
    p = keys.params
    cts = np.ascontiguousarray(cts, dtype=np.uint64).reshape(-1, p.n + 1)
    out = zeros128(cts.shape[0], p.k * p.N + 1)
    lib().p128mb_pbs_exact(_p(keys.bsk), _p(np.ascontiguousarray(lut)), _p(cts), cts.shape[0], p.n, p.k, p.N,
                           keys.grouping, p.base_log, p.level, _p(out))
    return out
