"""The PBS kernels on the GPU against their CPU replays, word for word.

The replays (tests/emu/emu_p22.cpp, emu_lanepair.cpp, emu_pbs128.cpp) run the
kernels' own B200_HD phase functions with g++; built without floating-point
contraction they
evaluate every expression in source order with IEEE round-to-nearest.  The
library built by tests/emu/build_nofma.py (csrc/Makefile's NVFLAGS plus
-fmad=false) does the same on the device: explicit fma calls stay fused on both
sides, nothing else is.  So each output word of that library must equal the
replay's, and a difference is a fault of the kernel's synchronisation, rings,
exchanges, indexing or key layout -- a fault the phase criterion of
tests/test_pbs_routes.py cannot see when it stays under the f64 floor or hits
every instance alike.  The shipped library's contraction is not covered here:
its outputs differ from the replays' in the last bits and stay judged
statistically by the route tests (the first control below asserts both).

Per table row: one kernel instance, pinned by its switches, run at batch 1, at
one wave at one and at two resident CTAs per SM (SMs, 2 SMs) and one past each,
and at 4096 on the automatic route.  Inputs come from a pool of uniform
LWEs and crafted words (zero masks, mask words that switch to N and
2N - 1, exact ties of the modulus switch in mask and body); in_idx repeats them,
lut_idx picks one of 3 LUTs (two many-LUT accumulators, one of random words),
out_idx scatters into a sentinel-filled output.  Every output of every launch
is compared with the replay of its (input, LUT) pair, and every row no sample
addresses must keep the sentinel.  Keys are uniform words at the shipped n
(n = 918 classic and multi-bit g = 3, n = 920 multi-bit g = 4): no GGSW repeats,
so a key block read from the wrong step changes the words.

The multi-bit rows pin each mode at every batch size: the fused kernel
(ll_max = 0, replay emu_pbs_mb) and the low-latency bundle + sequential pair
(ll_max large, replay emu_pbs_mb_ll).

The any-(N, k, l) kernel (pbs_generic.cuh, replay emu_pbs_generic) runs classic
shapes with k > 1 or l > 1, N = 512 and 8192 with the register kernels off,
the u32 torus entry point and every multi-bit shape off N = 2048.  Its
shared-memory rows run at batch 1 and one past a wave; its global-workspace
rows at 2 SMs, 2 SMs + 1 and 4 SMs + 3, where each CTA of the persistent grid
(2 SMs wide) reuses its workspace slice for a second and a third sample.  The
128-bit kernel (pbs128.cuh, replay emu128_pbs) runs one CTA per SM striding
over the samples, with the accumulator and output spectra in a reused global
workspace; its rows cover every instance, pbs128<256> to pbs128<4096>."""
import concurrent.futures as cf
import ctypes as C
import dataclasses
import os
import re
import subprocess

import numpy as np
import pytest

from tests.emu import build_nofma

SENTINEL = np.uint64(0xDEADBEEFCAFEF00D)


def test_nofma_library_flags_are_the_makefile_flags_plus_fmad_false():
    """The test library differs from the product build by -fmad=false alone:
    the flags are the ones `make` would pass to nvcc for the product library."""
    assert build_nofma.flags() == build_nofma.makefile_vars()["NVFLAGS"].split() + ["-fmad=false"]
    r = subprocess.run(["make", "-n", "-B", "-C", build_nofma.CSRC, "all"], capture_output=True, text=True, check=True)
    line = next(x for x in r.stdout.splitlines() if "nvcc" in x and "-shared" in x)
    product = line.split("2>")[0].split()
    ours = build_nofma.command(product[product.index("-o") + 1])
    at = product.index("-shared")
    assert ours == product[:at] + ["-fmad=false"] + product[at:]
    assert "-fmad=false" not in product and "arch=compute_90a,code=sm_90a" in ours


# ----------------------------------------------------------------------------
# replays
# ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    from tests.emu.build_emu import build_no_contract

    libs = build_no_contract(str(tmp_path_factory.mktemp("emu_nocontract")))
    return C.CDLL(libs["emu_p22.cpp"]), C.CDLL(libs["emu_lanepair.cpp"]), C.CDLL(libs["emu_pbs128.cpp"])


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _pool():
    return cf.ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1)))  # ctypes calls release the GIL


@dataclasses.dataclass
class Shape:
    """One key and parameter set: family p22 (N = 2048 classic), mb (multi-bit
    N = 2048), n8192 (N = 8192, l = 2), n512 (N = 512, l = 1, k <= 4), gen (the any-(N, k, l) kernel, classic
    or multi-bit, `torus` 64 or 32) or p128 (the 128-bit PBS: u64 inputs, u128
    LUTs, keys and outputs, each u128 word two u64, low then high).  `mask` is
    the b200_set_register_kernels value the key is converted under: it fixes the
    key layout."""
    name: str
    family: str
    n: int
    base_log: int
    l: int = 1
    g: int = 1
    k: int = 1
    N: int = 2048
    torus: int = 64
    mask: int = 3
    pool: int = 8  # uniform inputs of the pool (the crafted ones come on top)

    @property
    def log_mod(self):
        return (self.N * 2).bit_length() - 1

    @property
    def num_ggsw(self):
        return (self.n // self.g) << self.g if self.g > 1 else self.n

    @property
    def u64_per_word(self):
        return 2 if self.family == "p128" else 1

    @property
    def key_words(self):
        """f64 words of the Fourier key = u64 words of the standard-domain key"""
        return self.num_ggsw * self.l * (self.k + 1) ** 2 * self.N * self.u64_per_word

    @property
    def width(self):
        """u64 words of one output LWE (u32 outputs are widened to one u64 each)"""
        return (self.k * self.N + 1) * self.u64_per_word

    @property
    def sentinel(self):
        return SENTINEL & np.uint64(0xFFFFFFFF) if self.torus == 32 else SENTINEL


def emu_convert(emus, S, bsk):
    """the replay's Fourier key (float64 words) of the standard-domain key `bsk`"""
    emu = emus[0]
    out = np.empty(S.key_words, dtype=np.float64)
    if S.family in ("gen", "p128"):  # polynomials are independent and contiguous: convert them in parallel
        per = S.N * S.u64_per_word
        polys = S.key_words // per
        chunks = [(a, min(polys, a + 64)) for a in range(0, polys, 64)]
        if S.family == "gen":
            conv = lambda c: emu.emu_bsk_convert_generic(_vp(bsk[c[0] * S.N:]), C.c_uint64(c[1] - c[0]), S.N,
                                                         S.torus, _vp(out[c[0] * S.N:]))
        else:
            conv = lambda c: emus[2].emu128_bsk_convert(_vp(bsk[c[0] * per:]), C.c_uint64(c[1] - c[0]), S.N,
                                                        _vp(out[c[0] * per:]))
        with _pool() as ex:
            list(ex.map(conv, chunks))
    elif S.family == "n512":
        polys = S.key_words // S.N
        with _pool() as ex:
            list(ex.map(lambda a: emu.emu_bsk_convert_n512(_vp(bsk), S.k, C.c_uint64(a), C.c_uint64(min(64, polys - a)),
                                                           _vp(out)), range(0, polys, 64)))
    elif S.family == "p22":
        emu.emu_bsk_convert_p22(_vp(bsk), S.n, _vp(out))
    elif S.family == "n8192":
        emu.emu_bsk_convert_n8192(_vp(bsk), S.n, _vp(out))
    else:  # groups are independent and contiguous on both sides: convert them in parallel
        groups, per = S.n // S.g, S.key_words // (S.n // S.g)
        chunks = [(a, min(groups, a + 16)) for a in range(0, groups, 16)]
        with _pool() as ex:
            list(ex.map(lambda c: emu.emu_bsk_convert_mb(_vp(bsk[c[0] * per:]), (c[1] - c[0]) * S.g, S.l, S.g,
                                                         _vp(out[c[0] * per:])), chunks))
    return out


def emu_pbs(emus, replay, S, bskf, lut, ct, centered, ties_even, stride):
    """one sample, num_many_lut = 2 (its first output is the num_many_lut = 1
    output; the 128-bit PBS has one output), as [output][u64 word]"""
    emu, emu_lp = emus[:2]
    out = np.zeros((2, S.N + 1), dtype=np.uint64)
    lut, ct = np.ascontiguousarray(lut), np.ascontiguousarray(ct)
    if replay == "emu_pbs_generic":
        out = np.zeros((2, S.k * S.N + 1), dtype=np.uint32 if S.torus == 32 else np.uint64)
        emu.emu_pbs_generic(_vp(bskf), _vp(lut), _vp(ct), S.n, S.k, S.N, S.base_log, S.l, S.g, int(centered),
                            int(ties_even), 2, stride, 1, S.torus, _vp(out))
        return out.astype(np.uint64)
    if replay.startswith("emu_pbs_n512"):
        out = np.zeros((2, S.k * S.N + 1), dtype=np.uint64)
        emu.emu_pbs_n512(_vp(bskf), _vp(lut), _vp(ct), S.n, S.k, S.base_log, int(centered), int(replay.endswith("ring")),
                         2, stride, 1, _vp(out))
        return out
    if replay == "emu128_pbs":
        out = np.zeros((1, S.width), dtype=np.uint64)
        emus[2].emu128_pbs(_vp(bskf), _vp(lut), _vp(ct), S.n, S.k, S.N, S.base_log, S.l, int(centered), _vp(out))
        return out
    if replay in ("emu_pbs_mb", "emu_pbs_mb_ll"):
        getattr(emu, replay)(_vp(bskf), _vp(lut), _vp(ct), S.n, S.base_log, S.l, S.g, 2, stride, 1, _vp(out))
    elif replay == "emu_pbs_n8192":
        emu.emu_pbs_n8192(_vp(bskf), _vp(lut), _vp(ct), S.n, S.base_log, int(centered), int(ties_even), 2, stride, 1,
                          _vp(out))
    else:
        lib = emu_lp if "lanepair" in replay else emu
        getattr(lib, replay)(_vp(bskf), _vp(lut), _vp(ct), S.n, S.base_log, int(centered), 2, stride, 1, _vp(out))
    return out


@pytest.mark.parametrize("g,l", [(2, 2), (3, 1), (4, 2)])
def test_low_latency_multibit_replay_decrypts(oracle, keyset, emus, g, l):
    """The replay of the low-latency multi-bit mode bootstraps: on a real key it
    decrypts to f(m), like the fused kernel's replay (whose words it need not
    equal: the bundle is summed before the MAC, not inside it)."""
    n = 4 * g
    P = oracle.Params("MB_LL_g%d_l%d" % (g, l), n=n, k=1, N=2048, pbs_base_log=22 if l == 1 else 15, pbs_level=l,
                      ks_base_log=4, ks_level=4, lwe_noise_log2=45, glwe_noise_log2=17, grouping_factor=g,
                      centered_ms=False)
    keys = keyset(P, seed=5 + g, with_ksk=False)
    S = Shape("mb", "mb", n, P.pbs_base_log, l, g)
    bskf = emu_convert(emus, S, keys.bsk)
    msgs = np.arange(6) % 16
    cts = oracle.lwe_encrypt_batch(oracle.Rng(g), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    f = [(5 * x + 3) % 16 for x in range(16)]
    lut = oracle.make_lut(P, f)
    for replay in ("emu_pbs_mb", "emu_pbs_mb_ll"):
        out = np.stack([emu_pbs(emus, replay, S, bskf, lut, ct, False, 1, 0)[0] for ct in cts])
        dec = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, out), P.delta, 16)
        assert np.array_equal(dec, np.array([f[m] for m in msgs])), replay


def test_replays_called_from_many_threads_give_the_serial_words(emus, tmp_path):
    """The replays run in a thread pool.  A fresh copy of the library, first
    used by 16 threads at once, must give the words of serial calls: its
    transform tables are filled once, before any thread reads them."""
    import shutil

    lib = str(tmp_path / "emu_copy.so")
    shutil.copy(emus[0]._name, lib)
    lib128 = str(tmp_path / "emu128_copy.so")
    shutil.copy(emus[2]._name, lib128)
    fresh = (C.CDLL(lib), emus[1], C.CDLL(lib128))
    for S, replay in ((Shape("n8192_n16", "n8192", 16, 15, 2, N=8192), "emu_pbs_n8192"),
                      (Shape("gen_mb_n16", "gen", 16, 12, 2, 4, k=2, N=1024), "emu_pbs_generic"),
                      (Shape("gen_u32_n16", "gen", 16, 8, 2, k=2, N=512, torus=32), "emu_pbs_generic"),
                      (Shape("p128_n8", "p128", 8, 24, 3, k=2, N=512), "emu128_pbs")):
        bskf = emu_convert(emus, S, fresh_key(S, 3))
        cts, (luts, stride) = input_pool(S, 4), luts_of(S, 5)
        args = [(i % len(cts), i % 3) for i in range(16)]
        with cf.ThreadPoolExecutor(16) as ex:
            got = list(ex.map(lambda a: emu_pbs(fresh, replay, S, bskf, luts[a[1]], cts[a[0]], True, 1, stride),
                              args))
        for a, g in zip(args, got):
            assert np.array_equal(g, emu_pbs(emus, replay, S, bskf, luts[a[1]], cts[a[0]], True, 1, stride)), (S, a)


# ----------------------------------------------------------------------------
# keys and inputs
# ----------------------------------------------------------------------------
def fresh_key(S, seed):
    """uniform key words: every GGSW distinct (a real key's masks are uniform
    too, and the kernels' arithmetic does not depend on the bodies' structure)"""
    key = np.random.default_rng(seed).integers(0, 2 ** 64, S.key_words, dtype=np.uint64)
    return key.astype(np.uint32) if S.torus == 32 else key


def _top(S):
    """the largest word of the shape's torus"""
    return np.uint64((1 << S.torus) - 1)


def crafted_inputs(S, rng):
    """mask words of the modulus switch's edges (log_mod = log2(2N)), as u64
    words below 2^torus"""
    n, sh, top = S.n, S.torus - S.log_mod, _top(S)
    two_n = np.uint64(1 << S.log_mod)
    rnd = lambda: rng.integers(0, 2 ** 64, n + 1, dtype=np.uint64) & top
    out = []
    zero = rnd()
    zero[:n] = 0  # every step skipped (classic), every degree 0 (multi-bit)
    out.append(zero)
    edge = rnd()  # a_hat = N and a_hat = 2N - 1
    edge[0:n:3] = np.uint64(1 << (S.torus - 1))
    edge[1:n:3] = (two_n - np.uint64(1)) << np.uint64(sh)
    out.append(edge)
    tie = rnd()  # exact ties: (j + 1/2) 2^(64 - log_mod) in the mask and the body
    tie = ((tie >> np.uint64(sh)) << np.uint64(sh)) | np.uint64(1 << (sh - 1))
    tie[5:n:7] = 0
    out.append(tie)
    near = rnd()  # one below and one above the tie, and a tie that wraps to 0
    base = (near >> np.uint64(sh)) << np.uint64(sh)
    near = base | np.uint64(1 << (sh - 1))
    near[0::3] -= np.uint64(1)
    near[1::3] += np.uint64(1)
    near[2:n:11] = top - np.uint64((1 << (sh - 1)) - 1)
    out.append(near)
    return np.stack(out)


def input_pool(S, seed):
    """S.pool uniform LWEs (what a fresh encryption's mask is) and the crafted
    ones, in the shape's torus (the 128-bit PBS takes u64 LWEs)"""
    rng = np.random.default_rng(seed)
    uni = rng.integers(0, 2 ** 64, (S.pool, S.n + 1), dtype=np.uint64) & _top(S)
    pool = np.ascontiguousarray(np.concatenate([uni, crafted_inputs(S, rng)]))
    return pool.astype(np.uint32) if S.torus == 32 else pool


def luts_of(S, seed):
    """3 LUTs of k + 1 polynomials: two many-LUT accumulators (num_many_lut = 2,
    stride `stride`) and one of random words (exercises the u64 -> u32 rounding
    of the rotation); for the 128-bit PBS three of random u128 words"""
    from tfhe_rs_b200 import algorithms

    rng = np.random.default_rng(seed)
    if S.family == "p128":
        return np.ascontiguousarray(rng.integers(0, 2 ** 64, (3, (S.k + 1) * S.N * 2), dtype=np.uint64)), 0
    p = 64 if S.family == "n8192" else 16
    delta = (1 << 63) // p
    fns = [[(a * x + b) % p for x in range(p)] for a, b in ((1, 0), (3, 1), (5, 2))]
    built = [algorithms.generate_many_lut_accumulator(S.N, S.k + 1, p, delta, [fns[j], fns[j + 1]])
             for j in range(2)]
    rnd = rng.integers(0, 2 ** 64, (S.k + 1) * S.N, dtype=np.uint64)
    luts = np.ascontiguousarray(np.stack([built[0][0].reshape(-1), built[1][0].reshape(-1), rnd]))
    if S.torus == 32:  # the top halves: the accumulators' words are multiples of 2^32
        luts = (luts >> np.uint64(32)).astype(np.uint32)
    return luts, int(built[0][1])


# ----------------------------------------------------------------------------
# the library without contraction (and the shipped one) on the GPU
# ----------------------------------------------------------------------------
class Lib:
    """Drives one library through the C ABI on its own stream; device buffers
    are torch tensors."""

    def __init__(self, L, torch):
        self.L, self.torch = L, torch
        self.stream = L.cuda_create_stream_ffi(0)

    def sync(self):
        self.L.cuda_synchronize_stream(self.stream, 0)

    def dev(self, a):
        a = np.ascontiguousarray(a)
        signed = {8: np.int64, 4: np.int32}[a.dtype.itemsize] if a.dtype.kind == "u" else a.dtype
        t = self.torch.from_numpy(a.view(signed).reshape(-1)).cuda()
        self.torch.cuda.synchronize()
        return t

    def host(self, t):
        self.sync()
        unsigned = {self.torch.int64: np.uint64, self.torch.int32: np.uint32}.get(t.dtype)
        return t.cpu().numpy().view(unsigned) if unsigned else t.cpu().numpy()

    def switches(self, sw):
        L = self.L
        L.b200_set_pbs_variant(sw.get("variant", 0))
        L.b200_set_register_kernels(sw.get("mask", 3))
        L.b200_set_multibit_ll_max(sw.get("ll_max", -1))
        L.b200_set_multibit_tie_rule(sw.get("ties", 0))
        L.b200_set_n512_mode(sw.get("n512", 0))

    def convert(self, S, bsk):
        """the device key, converted under the shape's register-kernel mask"""
        d = self.torch.zeros(S.key_words, dtype=self.torch.float64, device="cuda")
        self.torch.cuda.synchronize()
        h = np.ascontiguousarray(bsk)
        L, args = self.L, (self.stream, 0, d.data_ptr(), h.ctypes.data, S.n, S.k, S.l, S.N)
        L.b200_set_register_kernels(S.mask)
        try:
            if S.family == "p128":
                L.cuda_convert_lwe_programmable_bootstrap_key_128_async(*args)
            elif S.g > 1:
                L.cuda_convert_lwe_multi_bit_programmable_bootstrap_key_64_async(*args, S.g)
            elif S.torus == 32:
                L.cuda_convert_lwe_programmable_bootstrap_key_32_async(*args)
            else:
                L.cuda_convert_lwe_programmable_bootstrap_key_64_async(*args)
            self.sync()
        finally:
            L.b200_set_register_kernels(3)
        return d

    def convert_seeded(self, S, bodies, seed):
        d = self.torch.zeros(S.key_words, dtype=self.torch.float64, device="cuda")
        self.torch.cuda.synchronize()
        key = (seed & (2 ** 128 - 1)).to_bytes(16, "little")
        self.L.b200_set_register_kernels(S.mask)
        try:
            self.L.b200_convert_seeded_lwe_programmable_bootstrap_key_64_async(
                self.stream, 0, d.data_ptr(), np.ascontiguousarray(bodies).ctypes.data, key, 0, 0, 0, S.n, S.k, S.l,
                S.N, S.g)
            self.sync()
        finally:
            self.L.b200_set_register_kernels(3)
        return d

    def pbs(self, S, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride, centered):
        """one launch into a sentinel-filled output; (output words as u64, kernel)"""
        word = np.uint32 if S.torus == 32 else np.uint64
        d_out = self.dev(np.full(rows * S.width, S.sentinel, dtype=word))
        count = len(in_idx)
        buf = C.POINTER(C.c_int8)()
        L, st = self.L, self.stream
        if S.family == "p128":
            # one LUT per launch, inputs and outputs in order: the samples are gathered on the host
            assert len(set(lut_idx)) == 1 and np.array_equal(out_idx, np.arange(count))
            d_lut, d_cts = self.dev(luts[lut_idx[0]]), self.dev(cts[in_idx])
            L.scratch_cuda_programmable_bootstrap_128_async(st, 0, C.byref(buf), S.n, S.k, S.N, S.l, count, True,
                                                            int(centered))
            L.cuda_programmable_bootstrap_128_async(st, 0, d_out.data_ptr(), d_lut.data_ptr(), d_cts.data_ptr(),
                                                    d_bsk.data_ptr(), buf, S.n, S.k, S.N, S.base_log, S.l, count)
            kernel = L.b200_last_pbs_kernel().decode()
            L.cleanup_cuda_programmable_bootstrap_128(st, 0, C.byref(buf))
            return self.host(d_out).reshape(rows, S.width), kernel
        d_lut, d_cts = self.dev(luts), self.dev(cts)
        d_oi, d_li, d_ii = (self.dev(np.asarray(a, dtype=word)) for a in (out_idx, lut_idx, in_idx))
        args = (d_out.data_ptr(), d_oi.data_ptr(), d_lut.data_ptr(), d_li.data_ptr(), d_cts.data_ptr(),
                d_ii.data_ptr(), d_bsk.data_ptr(), buf)
        if S.g > 1:
            L.scratch_cuda_multi_bit_programmable_bootstrap_64_async(st, 0, C.byref(buf), S.k, S.N, S.l, count, True)
            L.cuda_multi_bit_programmable_bootstrap_64_async(st, 0, *args, S.n, S.k, S.N, S.g, S.base_log, S.l, count,
                                                             many, stride)
            kernel = L.b200_last_pbs_kernel().decode()
            L.cleanup_cuda_multi_bit_programmable_bootstrap_64(st, 0, C.byref(buf))
        else:
            L.scratch_cuda_programmable_bootstrap_64_async(st, 0, C.byref(buf), S.n, S.k, S.N, S.l, count, True,
                                                           int(centered))
            run = (L.cuda_programmable_bootstrap_lwe_ciphertext_vector_32_async if S.torus == 32
                   else L.cuda_programmable_bootstrap_64_async)
            run(st, 0, *args, S.n, S.k, S.N, S.base_log, S.l, count, many, stride)
            kernel = L.b200_last_pbs_kernel().decode()
            L.cleanup_cuda_programmable_bootstrap_64(st, 0, C.byref(buf))
        return self.host(d_out).astype(np.uint64).reshape(rows, S.width), kernel


@pytest.fixture(scope="module")
def G():
    import torch

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import tfhe_rs_b200
    from tfhe_rs_b200 import _lib

    assert os.path.exists(build_nofma.LIB), "build() makes %s" % build_nofma.LIB
    nofma = Lib(_lib.load(build_nofma.LIB), torch)
    shipped = Lib(tfhe_rs_b200.lib(), torch)
    yield type("G", (), dict(nofma=nofma, shipped=shipped, torch=torch, sms=nofma.L.cuda_get_number_of_sms()))
    for lib in (nofma, shipped):
        lib.switches({})


# ----------------------------------------------------------------------------
# the table
# ----------------------------------------------------------------------------
@dataclasses.dataclass
class Run:
    batch: object  # a size, or (m, a): m * SM count + a
    kernel: str


@dataclasses.dataclass
class Row:
    id: str
    shape: str
    replay: str
    switches: dict
    runs: list
    centered: tuple = (True, False)  # the modulus switch of each config (classic routes)
    ties_even: tuple = (1,)  # tie rule of the decomposition: 1 ties to even, 0 the reference's (switch ties = 1)
    many: tuple = (1, 2)  # num_many_lut of the configs (the 128-bit PBS has one output)


SHAPES = {
    "p22": Shape("p22_n918", "p22", 918, 23),
    "mb2_l1": Shape("mb_g2_l1", "mb", 48, 22, 1, 2),
    "mb2_l2": Shape("mb_g2_l2", "mb", 48, 15, 2, 2),
    "mb3_l1": Shape("mb_g3_l1", "mb", 48, 22, 1, 3),
    "mb3_l2": Shape("mb_g3_l2_n918", "mb", 918, 15, 2, 3),
    "mb4_l1": Shape("mb_g4_l1_n920", "mb", 920, 22, 1, 4),
    "mb4_l2": Shape("mb_g4_l2", "mb", 48, 15, 2, 4),
    "n8192": Shape("n8192_n64", "n8192", 64, 15, 2, N=8192),
    # N = 512 register kernel: k = 1..4, base_log 31, n = 1024 (its a_hat limit), the shipped 1_1 set (n = 879, k = 4)
    **{"n512_k%d" % k: Shape("n512_k%d" % k, "n512", 24, 23, k=k, N=512) for k in (1, 2, 3, 4)},
    "n512_bl31": Shape("n512_k2_bl31", "n512", 24, 31, k=2, N=512),
    "n512_n1024": Shape("n512_k1_n1024", "n512", 1024, 23, k=1, N=512, pool=4),
    "n512_n879": Shape("n512_k4_n879", "n512", 879, 23, k=4, N=512, pool=4),
    # any-(N, k, l) kernel, classic: k > 1, l > 1, N off 2048, and N = 512 / 8192 with the register kernels off
    "gen_k3_l3": Shape("gen_k3_l3_n512", "gen", 16, 7, 3, k=3, N=512),
    "gen_k1_l3": Shape("gen_k1_l3_n512", "gen", 16, 7, 3, k=1, N=512),
    "gen_n1024": Shape("gen_k1_l2_n1024", "gen", 16, 15, 2, k=1, N=1024),
    "gen_n4096": Shape("gen_k1_l1_n4096", "gen", 16, 20, 1, k=1, N=4096),
    "gen_n512_off": Shape("gen_k2_l1_n512_off", "gen", 16, 23, 1, k=2, N=512, mask=0),
    "gen_n8192_off": Shape("gen_k1_l2_n8192_off", "gen", 16, 15, 2, k=1, N=8192, mask=0),
    "gen_n16384": Shape("gen_k1_l1_n16384", "gen", 8, 20, 1, k=1, N=16384, pool=4),
    "gen_u32": Shape("gen_u32_k2_l2_n512", "gen", 16, 8, 2, k=2, N=512, torus=32),
    "gen_u32_n16384": Shape("gen_u32_k1_l2_n16384", "gen", 8, 8, 2, k=1, N=16384, torus=32, pool=4),
    # any-(N, k, l) kernel, multi-bit: the 1_1 sets (g = 4 at its shipped n = 800), k = 2, and the 3_3 shapes
    "gen_mb2_k4": Shape("gen_mb_g2_k4_n512", "gen", 24, 22, 1, 2, k=4, N=512),
    "gen_mb3_k4": Shape("gen_mb_g3_k4_n512", "gen", 24, 22, 1, 3, k=4, N=512),
    "gen_mb4_k4": Shape("gen_mb_g4_k4_n512_n800", "gen", 800, 22, 1, 4, k=4, N=512, pool=4),
    "gen_mb2_k2": Shape("gen_mb_g2_k2_n1024", "gen", 24, 22, 1, 2, k=2, N=1024),
    "gen_mb4_n8192": Shape("gen_mb_g4_l2_n8192", "gen", 12, 14, 2, 4, k=1, N=8192),
    "gen_mb3_n16384": Shape("gen_mb_g3_l2_n16384", "gen", 9, 14, 2, 3, k=1, N=16384, pool=4),
    # 128-bit PBS: every instance, k = 1..3, base_log * l = 128, and the squash shape at its shipped n
    "p128_n256": Shape("p128_k1_24x3_n256", "p128", 16, 24, 3, k=1, N=256),
    "p128_n256_r128": Shape("p128_k2_64x2_n256", "p128", 16, 64, 2, k=2, N=256),
    "p128_n512": Shape("p128_k2_18x4_n512", "p128", 16, 18, 4, k=2, N=512),
    "p128_n1024": Shape("p128_k3_24x3_n1024", "p128", 8, 24, 3, k=3, N=1024),
    "p128_n2048": Shape("p128_k1_32x4_n2048", "p128", 8, 32, 4, k=1, N=2048),
    "p128_squash": Shape("p128_k2_24x3_n2048_n918", "p128", 918, 24, 3, k=2, N=2048, pool=2),
    "p128_n4096": Shape("p128_k1_24x3_n4096", "p128", 8, 24, 3, k=1, N=4096),
}
WAVES = [1, (1, 0), (1, 1), (2, 0), (2, 1)]  # batch 1, one wave at 1 and 2 CTAs / SM, and one past each
GEN_SMEM = [1, (1, 1)]  # one CTA per sample: batch 1 and one past a wave
GEN_WS = [(2, 0), (2, 1), (4, 3)]  # persistent grid of 2 SMs CTAs: one, two and three samples per slice
P128 = [1, (1, 0), (1, 1), (2, 1)]
# N = 512: one wave at 1, 2 and 3 LWEs per CTA; 3 SMs + 1 leaves a partial last group at G = 2 and 3, and
# gives each persistent CTA a second group
N512_WAVES = WAVES + [(3, 1)]
N512_MODES = ((3, 1, "true"), (2, 2, "true"), (4, 3, "true"), (1, 2, "false"))  # (b200_set_n512_mode, G, ring)  # one CTA per SM: one and two samples per CTA


def _rows():
    from tests.test_pbs_routes import FAST_VARIANTS, V6_LARGE, V6_SMALL

    rows = [Row("n2048_auto", "p22", "emu_pbs_p22_v3", {},
                [Run(1, V6_SMALL), Run((1, 0), V6_SMALL), Run((1, 1), V6_LARGE), Run((2, 0), V6_LARGE),
                 Run((2, 1), V6_LARGE), Run(4096, V6_LARGE)])]
    rows.append(Row("n2048_v1", "p22", "emu_pbs_p22", {"variant": 1}, [Run(b, "n2048_v1") for b in WAVES]))
    for v, name in FAST_VARIANTS.items():
        rows.append(Row("n2048_variant%d" % v, "p22", "emu_pbs_p22_v3", {"variant": v}, [Run(b, name) for b in WAVES]))
    # the shipped two-CTA instance with exchange 2 through half-warp shuffles (x2_shfl.cuh), its A/B partner
    rows.append(Row("n2048_variant23", "p22", "emu_pbs_p22_v3", {"variant": 23},
                    [Run(b, "n2048_v6<2,true,2,1,0>") for b in WAVES]))
    for g in (2, 3, 4):
        for l in (1, 2):
            name = "multibit_fused<%d,%d>" % (g, l)
            rows.append(Row("mb_g%d_l%d" % (g, l), "mb%d_l%d" % (g, l), "emu_pbs_mb", {"ll_max": 0},
                            [Run(b, name) for b in WAVES], centered=(False,)))
            ll = "multibit_ll<%d,%d,%s>" % (g, l, "tma" if l == 1 else "regs")
            rows.append(Row("mb_ll_g%d_l%d" % (g, l), "mb%d_l%d" % (g, l), "emu_pbs_mb_ll", {"ll_max": 1 << 20},
                            [Run(b, ll) for b in WAVES], centered=(False,)))
    for sw, name in (({}, "n8192_v2<false>"), ({"mask": 11}, "n8192_v2<true>"), ({"mask": 7}, "n8192_v1")):
        for ties in (1, 0):
            rows.append(Row("n8192_%s_ties%s" % (re.sub(r"\W", "", name), "even" if ties else "ref"), "n8192",
                            "emu_pbs_n8192", dict(sw, ties=1 - ties), [Run(1, name), Run((1, 0), name), Run((1, 1), name)],
                            ties_even=(ties,)))
    for k in (1, 2, 3, 4):
        for mode, g, ring in N512_MODES:
            name = "n512<%d,%d,%s>" % (k, g, ring)
            rows.append(Row("n512_k%d_G%d_%s" % (k, g, "ring" if ring == "true" else "regs"), "n512_k%d" % k,
                            "emu_pbs_n512_" + ("ring" if ring == "true" else "regs"), {"n512": mode},
                            [Run(b, name) for b in N512_WAVES]))
    for k in (1, 4):
        ring = lambda G: "n512<%d,%d,true>" % (k, G)
        rows.append(Row("n512_k%d_auto" % k, "n512_k%d" % k, "emu_pbs_n512_ring", {},
                        [Run(1, ring(1)), Run((1, 0), ring(1)), Run((1, 1), ring(2)), Run((2, 0), ring(2)),
                         Run((2, 1), ring(3)), Run(4096, ring(3))]))
    for key in ("n512_bl31", "n512_n1024", "n512_n879"):
        S = SHAPES[key]
        rows.append(Row(key, key, "emu_pbs_n512_ring", {}, [Run(1, "n512<%d,1,true>" % S.k),
                                                            Run((1, 1), "n512<%d,2,true>" % S.k),
                                                            Run((2, 1), "n512<%d,3,true>" % S.k)]))
        rows.append(Row(key + "_regs", key, "emu_pbs_n512_regs", {"n512": 1},
                        [Run(b, "n512<%d,2,false>" % S.k) for b in (1, (2, 1))]))
    for key in ("gen_k3_l3", "gen_k1_l3", "gen_n1024", "gen_n4096", "gen_n512_off", "gen_u32", "gen_mb2_k4",
                "gen_mb3_k4", "gen_mb4_k4", "gen_mb2_k2"):
        S = SHAPES[key]
        name = "generic_smem_u32" if S.torus == 32 else "generic_smem"
        rows.append(Row(key, key, "emu_pbs_generic", {"mask": S.mask}, [Run(b, name) for b in GEN_SMEM],
                        centered=(False,) if S.g > 1 else (True, False)))
    for key in ("gen_n8192_off", "gen_n16384", "gen_u32_n16384"):
        S = SHAPES[key]
        name = "generic_workspace_u32" if S.torus == 32 else "generic_workspace"
        rows.append(Row(key, key, "emu_pbs_generic", {"mask": S.mask}, [Run(b, name) for b in GEN_WS]))
    for key in ("gen_mb4_n8192", "gen_mb3_n16384"):
        for ties in (1, 0):
            rows.append(Row("%s_ties%s" % (key, "even" if ties else "ref"), key, "emu_pbs_generic", {"ties": 1 - ties},
                            [Run(b, "generic_workspace") for b in GEN_WS], centered=(False,), ties_even=(ties,)))
    for key in sorted(k for k in SHAPES if k.startswith("p128")):
        name = "pbs128<%d>" % SHAPES[key].N
        rows.append(Row(key, key, "emu128_pbs", {}, [Run(b, name) for b in P128], many=(1,)))
    return rows


ROWS = _rows()


class Shapes:
    """per shape: host key, device key of the no-FMA library, inputs, LUTs and
    the replay tables [config][input][lut] -> (2, N + 1) words, made on first use"""

    def __init__(self, G, emus):
        self.G, self.emus, self.cache, self.tables = G, emus, {}, {}

    def get(self, key):
        if key not in self.cache:
            S = SHAPES[key]
            seed = sum(map(ord, S.name))
            bsk = fresh_key(S, seed)
            d_bsk = self.G.nofma.convert(S, bsk)
            self.cache[key] = dict(S=S, bsk=bsk, d_bsk=d_bsk, bskf=self.G.nofma.host(d_bsk), cts=input_pool(S, seed + 1),
                                   luts=luts_of(S, seed + 2))
        return self.cache[key]

    def table(self, key, replay, centered, ties_even, bskf=None):
        """replays of every (input, LUT) pair"""
        tk = (key, replay, centered, ties_even, bskf is None)
        if bskf is None and tk in self.tables:
            return self.tables[tk]
        d = self.get(key)
        S, (luts, stride), cts = d["S"], d["luts"], d["cts"]
        bskf = d["bskf"] if bskf is None else bskf
        pairs = [(i, j) for i in range(len(cts)) for j in range(len(luts))]
        with _pool() as ex:
            outs = list(ex.map(lambda p: emu_pbs(self.emus, replay, S, bskf, luts[p[1]], cts[p[0]], centered,
                                                 ties_even, stride), pairs))
        t = np.stack(outs).reshape(len(cts), len(luts), *outs[0].shape)
        if tk[-1]:
            self.tables[tk] = t
        return t


@pytest.fixture(scope="module")
def shapes(G, emus):
    return Shapes(G, emus)


def launch_plan(batch, many, pool, seed, one_lut=False):
    """one_lut: the 128-bit PBS's launch (one LUT, outputs in input order, 3
    sentinel rows past them)"""
    rng = np.random.default_rng(seed)
    in_idx = rng.integers(0, pool, batch)
    in_idx[: min(batch, pool)] = np.arange(min(batch, pool))  # every input at least once where the batch allows
    lut_idx = rng.integers(0, 3, batch)
    if one_lut:
        return in_idx, np.full(batch, seed % 3), np.arange(batch), batch + 3
    if many == 1:
        rows = batch + batch // 2 + 3
        out_idx = rng.permutation(rows)[:batch]
    else:
        rows = many * batch + 5
        out_idx = rng.permutation(batch)
    return in_idx, lut_idx, out_idx, rows


def run_and_compare(lib, d, d_bsk, batch, many, centered, table, seed, where):
    """one launch; returns (kernel, samples, words compared, the first mismatch or
    None, the fraction of differing words)"""
    S, (luts, stride), cts = d["S"], d["luts"], d["cts"]
    in_idx, lut_idx, out_idx, rows = launch_plan(batch, many, len(cts), seed, S.family == "p128")
    out, kernel = lib.pbs(S, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride, centered)
    hit = np.concatenate([m * batch + out_idx for m in range(many)])
    addressed = np.zeros(rows, dtype=bool)
    addressed[hit] = True
    assert (out[~addressed] == S.sentinel).all(), ("stray write outside the addressed rows", where)
    got = np.stack([out[m * batch + out_idx] for m in range(many)], axis=1)  # [batch][many][width]
    want = table[in_idx, lut_idx, :many]
    diff = got != want
    first = None
    if diff.any():
        s, m, w = (int(x[0]) for x in np.nonzero(diff))
        first = "sample %d (input %d, lut %d), output %d, word %d: got %#x want %#x" % (
            s, in_idx[s], lut_idx[s], m, w, int(got[s, m, w]), int(want[s, m, w]))
    return kernel, batch, got.size, first, float(diff.mean())


CONFIGS = [(1, True), (2, False), (2, True), (1, False)]  # (num_many_lut, centered) by run, cycled


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=[r.id for r in ROWS])
def test_gpu_words_equal_the_replay(G, shapes, row):
    d = shapes.get(row.shape)
    lib = G.nofma
    try:
        lib.switches(row.switches)
        configs = [(m, c) for m, c in CONFIGS if c in row.centered and m in row.many]
        for k, run in enumerate(row.runs):
            batch = run.batch if isinstance(run.batch, int) else run.batch[0] * G.sms + run.batch[1]
            many, centered = configs[k % len(configs)]
            table = shapes.table(row.shape, row.replay, centered, row.ties_even[0])
            where = (row.id, batch)
            kernel, samples, words, first, frac = run_and_compare(lib, d, d["d_bsk"], batch, many, centered, table,
                                                                  k * 7919 + batch, where)
            print("REPLAY %-24s %-24s batch %5d  many %d  centered %d  samples %5d  words %9d  %s" % (
                row.id, kernel, batch, many, int(centered), samples, words, "ok" if first is None else first))
            assert kernel == run.kernel, (where, kernel)
            assert first is None, "%s batch %d: %s" % (row.id, batch, first)
    finally:
        lib.switches({})


# ----------------------------------------------------------------------------
# replays agree with each other (the lane-pair replay of the shipped instance)
# ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_lane_pair_replay_equals_the_replay_of_the_table(G, shapes):
    """the pool replayed through the shipped instance's lane-pair replay (x2m)
    gives the words every p22 row was compared with"""
    want = shapes.table("p22", "emu_pbs_p22_v3", True, 1)
    got = shapes.table("p22", "emu_pbs_p22_lanepair_x2m", True, 1)
    assert np.array_equal(got, want)


# ----------------------------------------------------------------------------
# key conversion
# ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(SHAPES))
def test_device_key_equals_the_replay_conversion(G, emus, shapes, key):
    d = shapes.get(key)
    S = d["S"]
    want = emu_convert(emus, S, d["bsk"])
    got = d["bskf"]
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    print("KEY %-16s words %9d  differing %d" % (S.name, got.size, bad.size))
    assert bad.size == 0, "%s: first differing word %d: %r != %r" % (S.name, bad[0], got[bad[0]], want[bad[0]])


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["p22", "mb3_l2", "gen_k3_l3", "gen_n512_off", "gen_mb3_k4", "gen_mb4_n8192"])
def test_seeded_key_ingest_gives_the_same_device_words(G, shapes, key):
    """masks regenerated on the GPU from the seed: the same device key as the
    standard-domain key with those masks converted"""
    from tests.test_multibit_generic_routes import _seeded_host_key

    d = shapes.get(key)
    S = d["S"]
    P = type("P", (), dict(N=S.N, k=S.k))
    bodies = np.ascontiguousarray(d["bsk"].reshape(-1, S.k + 1, S.N)[:, S.k, :])
    seed = 0x5EED_2048_0918_0000_1111_2222_3333_4444
    host = _seeded_host_key(P, seed, 0, 0, bodies)
    full = G.nofma.host(G.nofma.convert(S, host))
    seeded = G.nofma.host(G.nofma.convert_seeded(S, bodies, seed))
    assert np.array_equal(full.view(np.uint64), seeded.view(np.uint64))


# ----------------------------------------------------------------------------
# controls: the comparison is sharp
# ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_control_shipped_library_differs_from_the_replay(G, oracle, keyset, shapes, emus):
    """The shipped library (nvcc contraction on), on the same launch, differs
    from the replay in some words; its phase against the no-FMA library's output
    still passes the route tests' criterion (real keys and encryptions, n = 64)."""
    from tests.test_pbs_routes import acc32_tau, phase_criterion, phase_error

    d = shapes.get("p22")
    table = shapes.table("p22", "emu_pbs_p22_v3", True, 1)
    d_bsk = G.shipped.convert(d["S"], d["bsk"])
    kernel, samples, words, first, frac = run_and_compare(G.shipped, d, d_bsk, 4096, 2, True, table, 5, "shipped")
    print("CONTROL shipped library %s batch %d: %.4f of %d words differ from the replay" % (kernel, samples, frac,
                                                                                        words))
    assert first is not None and frac > 0
    P = oracle.Params("P22_n64", n=64, k=1, N=2048, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=45, glwe_noise_log2=17)
    shipped_phase_against_nofma(G, oracle, keyset, P, Shape("p22_n64", "p22", 64, 23), acc32_tau(1, 2048, 32 - 23, 64))


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["generic", "n512"])
def test_control_shipped_library_differs_from_the_replay_off_n2048(G, oracle, keyset, shapes, family):
    """The same control on the any-(N, k, l) kernel (k = 1, N = 1024, l = 2,
    64-bit accumulator: no rounding term) and on the N = 512 kernel (k = 4,
    32-bit accumulator)."""
    from tests.test_pbs_routes import acc32_tau

    key, replay, name = {"generic": ("gen_n1024", "emu_pbs_generic", "generic_smem"),
                         "n512": ("n512_k4", "emu_pbs_n512_ring", "n512<4,3,true>")}[family]
    d = shapes.get(key)
    table = shapes.table(key, replay, True, 1)
    d_bsk = G.shipped.convert(d["S"], d["bsk"])
    kernel, samples, words, first, frac = run_and_compare(G.shipped, d, d_bsk, 2 * G.sms + 1, 2, True, table, 5,
                                                          "shipped")
    print("CONTROL shipped library %s batch %d: %.4f of %d words differ from the replay" % (kernel, samples, frac,
                                                                                        words))
    assert kernel == name and first is not None and frac > 0
    if family == "generic":
        P = oracle.Params("GEN_K2_L2_N1024_n64", n=64, k=2, N=1024, pbs_base_log=15, pbs_level=2, ks_base_log=4,
                          ks_level=4, lwe_noise_log2=45, glwe_noise_log2=17)
        S, tau = Shape("gen_k2_n64", "gen", 64, 15, 2, k=2, N=1024), 0.0
    else:
        P = oracle.Params("N512_K4_n64", n=64, k=4, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                          lwe_noise_log2=45, glwe_noise_log2=17)
        S, tau = Shape("n512_k4_n64", "n512", 64, 23, k=4, N=512), acc32_tau(4, 512, 32 - 23, 64)
    shipped_phase_against_nofma(G, oracle, keyset, P, S, tau)


def shipped_phase_against_nofma(G, oracle, keyset, P, S, tau):
    """real keys and encryptions: the shipped library's phase against the no-FMA
    library's output passes the route tests' criterion"""
    from tests.test_pbs_routes import phase_criterion, phase_error

    keys = keyset(P, seed=0xB200F00D, with_ksk=False)
    msgs = np.arange(24) % 16
    cts = oracle.lwe_encrypt_batch(oracle.Rng(7), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    lut = oracle.make_lut(P, [(3 * x + 1) % 16 for x in range(16)])
    idx = np.arange(len(cts))
    outs = []
    for lib in (G.nofma, G.shipped):
        out, _ = lib.pbs(S, lib.convert(S, keys.bsk), lut, cts, np.zeros_like(idx), idx, idx, len(cts), 1, 0, True)
        outs.append(out)
    fft = oracle.pbs_batch(keys, lut, cts, exact=False)
    exact = oracle.pbs_batch(keys, lut, cts, exact=True)
    e_fft = phase_error(keys.glwe_sk, fft, exact)
    e = phase_error(keys.glwe_sk, outs[1], outs[0])
    stats, failures = phase_criterion(e, e_fft, tau)
    print("CONTROL %s shipped vs no-FMA phase: rms/floor %.3f, %d/%d words differ, %s" % (
        S.name, stats["ratio"], int((outs[0] != outs[1]).sum()), outs[0].size, failures or "ok"))
    assert not failures, stats


@pytest.mark.gpu
def test_control_one_ulp_in_the_key_is_seen(G, shapes):
    """One ulp added to one Fourier coefficient of one GGSW of the device key:
    some replayed sample differs."""
    d = shapes.get("p22")
    S = d["S"]
    table = shapes.table("p22", "emu_pbs_p22_v3", True, 1)
    d_bsk = d["d_bsk"].clone()
    G.torch.cuda.synchronize()
    pos = (S.n // 2) * 4 * 1024 * 2 + 2 * 1024 * 2 + 2 * 777  # GGSW n / 2, its third block, one real part
    bits = d_bsk.view(G.torch.int64)
    bits[pos] += 1
    G.torch.cuda.synchronize()
    kernel, samples, words, first, frac = run_and_compare(G.nofma, d, d_bsk, 2 * G.sms + 1, 2, True, table, 9, "ulp")
    print("CONTROL one ulp in GGSW %d (%s, batch %d): %.5f of %d words differ; first: %s" % (
        S.n // 2, kernel, samples, frac, words, first))
    assert first is not None


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["n512_k2", "gen_n1024", "gen_mb2_k2", "p128_n512"])
def test_control_one_ulp_in_an_n512_generic_or_128_bit_key_is_seen(G, shapes, key):
    """One ulp added to one real part (the high double of a double-double) of
    the third key block of GGSW n / 2 (of group n / 2g, multi-bit): the
    replayed words differ.  Measured on an H100: 12.8 % of the words at
    gen_n1024, 9.0 % at gen_mb2_k2 and 90.2 % at p128_n512."""
    d = shapes.get(key)
    S = d["S"]
    replay = {"p128": "emu128_pbs", "n512": "emu_pbs_n512_ring"}.get(S.family, "emu_pbs_generic")
    table = shapes.table(key, replay, S.g == 1, 1)
    M, per = S.N // 2, 2 * S.u64_per_word  # f64 words per frequency
    block = M * per
    step = (S.n // S.g) // 2  # a classic GGSW, or the first GGSW of a multi-bit group
    pos = step * (1 << S.g if S.g > 1 else 1) * S.l * (S.k + 1) ** 2 * block + 2 * block + per * 77
    d_bsk = d["d_bsk"].clone()
    G.torch.cuda.synchronize()
    d_bsk.view(G.torch.int64)[pos] += 1
    G.torch.cuda.synchronize()
    many = 1 if S.family == "p128" else 2
    kernel, samples, words, first, frac = run_and_compare(G.nofma, d, d_bsk, G.sms + 1, many, S.g == 1, table, 9,
                                                          "ulp")
    print("CONTROL one ulp in %s step %d (%s, batch %d): %.5f of %d words differ; first: %s" % (
        S.name, step, kernel, samples, frac, words, first))
    assert first is not None and frac > 0.05, frac


# ----------------------------------------------------------------------------
# the table covers every instance
# ----------------------------------------------------------------------------
# instances the backend can report that no row runs, and why
NOT_REPLAYED = {
    "multibit_ll<2,1,regs>": "register-prefetch sequential kernel of l = 1: B200_MULTIBIT_SEQ_TMA=0, read once per "
                             "process",
    "multibit_ll<3,1,regs>": "same",
    "multibit_ll<4,1,regs>": "same",
}


# kernel names of b200_backend.cu that b200_last_keyswitch_kernel reports (tests/test_keyswitch_routes.py
# covers them); every other kernel name there is a PBS instance
KEYSWITCH_NAMES = {"ks_imma<1>", "ks_imma<2>", "ks_f64", "ks_int", "ks_int_wide", "ks_64_32", "ks128"}


def backend_kernel_names():
    """every kernel instance name in csrc/b200_backend.cu: its `name<args>`
    string literals, and the `name` literals of its kernel tables (lines naming
    a *_kernel) and of its t_last_pbs_kernel assignments"""
    from tests.emu.build_emu import CSRC

    with open(os.path.join(CSRC, "b200_backend.cu")) as f:
        src = f.read()
    literal = re.compile(r'"([A-Za-z]\w*(?:<[\w,]*>)?)"')
    names = set(re.findall(r'"([A-Za-z]\w*<[\w,]*>)"', src))
    for stmt in re.findall(r"t_last_pbs_kernel\s*=([^;]*);", src):
        names |= set(literal.findall(stmt))
    for line in src.splitlines():
        if re.search(r"\w_kernel\b", line):
            names |= set(literal.findall(line))
    return names


def test_replay_table_covers_every_pbs_instance():
    """Every PBS instance name the backend can report appears in a row of the
    table (the names not replayed are listed above, with the reason).  A kernel
    name of a new family fails here until a row runs it."""
    names = backend_kernel_names() - KEYSWITCH_NAMES
    assert {"n2048_v1", "generic_smem", "generic_workspace_u32", "pbs128<256>", "pbs128<4096>", "n8192_v1",
            "n512<4,3,true>", "multibit_ll<2,1,regs>"} <= names
    rows = {run.kernel for row in ROWS for run in row.runs}
    assert rows <= names, sorted(rows - names)
    assert names - set(NOT_REPLAYED) <= rows, sorted(names - set(NOT_REPLAYED) - rows)


# ----------------------------------------------------------------------------
# the new replays on real keys (CPU)
# ----------------------------------------------------------------------------
@pytest.mark.parametrize("k,N,bl,l,g,torus", [(2, 1024, 15, 2, 1, 64), (1, 512, 7, 3, 1, 64), (2, 512, 22, 1, 3, 64),
                                             (1, 1024, 12, 2, 4, 64), (2, 512, 8, 2, 1, 32)],
                         ids=["k2_l2_n1024", "k1_l3_n512", "mb_g3_k2_n512", "mb_g4_l2_n1024", "u32_k2_l2_n512"])
def test_generic_replay_decrypts_and_meets_the_exact_criterion(oracle, keyset, emus, k, N, bl, l, g, torus):
    """On oracle keys the replay of the any-(N, k, l) kernel decrypts to f(m),
    and its phase error against the exact blind rotation passes the route
    tests' criterion against the oracle's own f64 error (64-bit accumulator:
    tau = 0; the u32 torus rounds its outputs to 32 bits, so its criterion
    holds the rounded exact output too)."""
    from tests.test_pbs_routes import phase_criterion, phase_error

    n = 24
    P = oracle.Params("GEN_REPLAY_k%d_N%d_%dx%d_g%d" % (k, N, bl, l, g), n=n, k=k, N=N, pbs_base_log=bl,
                      pbs_level=l, ks_base_log=4, ks_level=4, lwe_noise_log2=45, glwe_noise_log2=17,
                      grouping_factor=g, centered_ms=g == 1)
    keys = keyset(P, seed=77 + N + k + g, with_ksk=False)
    if torus == 32:  # the oracle bootstraps with the key the u32 entry point sees: its words' top halves
        keys = dataclasses.replace(keys, bsk=keys.bsk & ~np.uint64(0xFFFFFFFF), _fourier=None)
    S = Shape("gen_replay", "gen", n, bl, l, g, k=k, N=N, torus=torus)
    bsk = (keys.bsk >> np.uint64(32)).astype(np.uint32) if torus == 32 else keys.bsk
    bskf = emu_convert(emus, S, bsk)
    msgs = np.arange(32) % 16
    cts = oracle.lwe_encrypt_batch(oracle.Rng(5 + g), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    f = [(3 * x + 5) % 16 for x in range(16)]
    lut = oracle.make_lut(P, f)
    centered = g == 1
    if torus == 32:  # the u32 entry point reads the top halves (the oracle's inputs and LUT keep them exactly)
        cts = cts & ~np.uint64(0xFFFFFFFF)
        lut = lut & ~np.uint64(0xFFFFFFFF)
        run_cts, run_lut = (cts >> np.uint64(32)).astype(np.uint32), (lut >> np.uint64(32)).astype(np.uint32)
    else:
        run_cts, run_lut = cts, lut
    with _pool() as ex:
        out = np.stack(list(ex.map(lambda ct: emu_pbs(emus, "emu_pbs_generic", S, bskf, run_lut, ct, centered, 1,
                                                      0)[0], run_cts)))
    if torus == 32:
        out = out << np.uint64(32)
    dec = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, out), P.delta, 16)
    assert np.array_equal(dec, np.array([f[m] for m in msgs]))
    exact = oracle.pbs_batch(keys, lut, cts, exact=True, centered_ms=centered)
    fft = oracle.pbs_batch(keys, lut, cts, exact=False, centered_ms=centered)
    e_fft = phase_error(keys.glwe_sk, fft, exact)
    e = phase_error(keys.glwe_sk, out, exact)
    tau = 0.0 if torus == 64 else float(np.sqrt((k * N / 2 + 1) / 12.0)) * 2.0 ** -32
    stats, failures = phase_criterion(e, e_fft, tau)
    print("REPLAY generic %s: rms/floor %.3f %s" % (P.name, stats["ratio"], failures or "ok"))
    assert not failures, stats


@pytest.mark.parametrize("N,k,base_log,level,centered", [(256, 1, 24, 3, True), (512, 2, 18, 4, False),
                                                          (256, 2, 64, 2, True)])
def test_128_bit_replay_decrypts_and_stays_within_the_transform_bound(emus, N, k, base_log, level, centered):
    """On model keys the replay of the 128-bit kernel decrypts to f(m), and its
    rms phase error against the exact u128 blind rotation stays within the
    bound test_noise_squashing.py holds the GPU to."""
    import math

    from tests import pbs128_model as P128
    from tests.test_noise_squashing import (_encrypt_small, _signed, _switch, fft_term_variance,
                                            rounding_term_variance)

    n, p_msg = 16, 16
    prm = P128.Params128(n=n, k=k, N=N, base_log=base_log, level=level, glwe_noise_log2=2)
    keys = P128.keygen(prm, 300 + N + k)
    S = Shape("p128_replay", "p128", n, base_log, level, k=k, N=N)
    bskf = emu_convert(emus, S, np.ascontiguousarray(keys.bsk).reshape(-1))
    rng = np.random.default_rng(N + k)
    msgs = [int(x) for x in rng.integers(0, p_msg, 12)]
    cts = _encrypt_small(rng, keys.lwe_sk, msgs, (1 << 63) // p_msg, 30)
    f = [(7 * m + 2) % p_msg for m in range(p_msg)]
    delta = (1 << 127) // p_msg
    lut = np.ascontiguousarray(P128.make_lut(k, N, f, delta)).reshape(-1)
    with _pool() as ex:
        out = np.stack(list(ex.map(lambda ct: emu_pbs(emus, "emu128_pbs", S, bskf, lut, ct, centered, 1, 0)[0],
                                   cts))).reshape(len(cts), -1, 2)
    phase = P128.decrypt(keys.glwe_sk, out)
    assert P128.decode(phase, delta, p_msg) == [f[m] for m in msgs]
    exact = P128.decrypt(keys.glwe_sk, P128.pbs_exact(keys, lut.reshape(-1, 2), _switch(cts, N, centered)))
    err = [_signed(x - y) / 2.0 ** 128 for x, y in zip(phase, exact)]
    rms = math.sqrt(sum(e * e for e in err) / len(err))
    bound = 2 * math.sqrt(fft_term_variance(n, k, N, base_log, level)
                          + 2 * rounding_term_variance(n, k, N, base_log, level))
    print("REPLAY 128-bit N=%d k=%d %dx%d: rms %.3g, bound %.3g" % (N, k, base_log, level, rms, bound))
    assert rms <= bound, (rms, bound)


@pytest.mark.parametrize("k", [1, 4])
def test_n512_replay_decrypts_and_meets_the_exact_criterion(oracle, keyset, emus, k):
    """On oracle keys both key modes of the N = 512 replay decrypt to f(m), and
    their phase error against the exact blind rotation passes the route tests'
    criterion (32-bit accumulator: acc32_tau)."""
    from tests.test_pbs_routes import acc32_tau, phase_criterion, phase_error

    n = 24
    P = oracle.Params("N512_REPLAY_k%d" % k, n=n, k=k, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4,
                      ks_level=4, lwe_noise_log2=45, glwe_noise_log2=17, message_bits=1, carry_bits=1)
    keys = keyset(P, seed=512 + k, with_ksk=False)
    S = Shape("n512_replay", "n512", n, 23, k=k, N=512)
    bskf = emu_convert(emus, S, keys.bsk)
    msgs = np.arange(32) % 4
    cts = oracle.lwe_encrypt_batch(oracle.Rng(9 + k), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    f = [(3 * x + 1) % 4 for x in range(4)]
    lut = oracle.make_lut(P, f)
    exact = oracle.pbs_batch(keys, lut, cts, exact=True, centered_ms=True)
    e_fft = phase_error(keys.glwe_sk, oracle.pbs_batch(keys, lut, cts, exact=False, centered_ms=True), exact)
    for replay in ("emu_pbs_n512_ring", "emu_pbs_n512_regs"):
        with _pool() as ex:
            out = np.stack(list(ex.map(lambda ct: emu_pbs(emus, replay, S, bskf, lut, ct, True, 1, 0)[0], cts)))
        dec = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, out), P.delta, 4)
        assert np.array_equal(dec, np.array([f[m] for m in msgs])), replay
        stats, failures = phase_criterion(phase_error(keys.glwe_sk, out, exact), e_fft,
                                          acc32_tau(k, 512, 32 - 23, n))
        print("REPLAY %s k=%d: rms/floor %.3f %s" % (replay, k, stats["ratio"], failures or "ok"))
        assert not failures, (replay, stats)
