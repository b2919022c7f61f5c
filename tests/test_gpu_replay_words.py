"""The PBS kernels on the GPU against their CPU replays, word for word.

The replays (tests/emu/emu_p22.cpp, emu_lanepair.cpp) run the kernels' own
B200_HD phase functions with g++; built without floating-point contraction they
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
(ll_max large, replay emu_pbs_mb_ll)."""
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
    return C.CDLL(libs["emu_p22.cpp"]), C.CDLL(libs["emu_lanepair.cpp"])


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _pool():
    return cf.ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1)))  # ctypes calls release the GIL


@dataclasses.dataclass
class Shape:
    """One key and parameter set: family p22 (N = 2048 classic), mb (multi-bit
    N = 2048) or n8192 (N = 8192, l = 2)."""
    name: str
    family: str
    n: int
    base_log: int
    l: int = 1
    g: int = 1

    @property
    def N(self):
        return 8192 if self.family == "n8192" else 2048

    @property
    def log_mod(self):
        return (self.N * 2).bit_length() - 1

    @property
    def num_ggsw(self):
        return (self.n // self.g) << self.g if self.g > 1 else self.n

    @property
    def key_words(self):
        return self.num_ggsw * self.l * 4 * self.N


def emu_convert(emu, S, bsk):
    """the replay's Fourier key (float64 words) of the standard-domain key `bsk`"""
    out = np.empty(S.key_words, dtype=np.float64)
    if S.family == "p22":
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
    """one sample, num_many_lut = 2 (its first output is the num_many_lut = 1 output)"""
    emu, emu_lp = emus
    out = np.zeros((2, S.N + 1), dtype=np.uint64)
    lut, ct = np.ascontiguousarray(lut), np.ascontiguousarray(ct)
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
    bskf = emu_convert(emus[0], S, keys.bsk)
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
    fresh = (C.CDLL(lib), emus[1])
    S = Shape("n8192_n16", "n8192", 16, 15, 2)
    bskf = emu_convert(emus[0], S, fresh_key(S, 3))
    cts, (luts, stride) = input_pool(S, 4), luts_of(S, 5)
    args = [(i % len(cts), i % 3) for i in range(16)]
    with cf.ThreadPoolExecutor(16) as ex:
        got = list(ex.map(lambda a: emu_pbs(fresh, "emu_pbs_n8192", S, bskf, luts[a[1]], cts[a[0]], True, 1, stride),
                          args))
    for a, g in zip(args, got):
        assert np.array_equal(g, emu_pbs(emus, "emu_pbs_n8192", S, bskf, luts[a[1]], cts[a[0]], True, 1, stride)), a


# ----------------------------------------------------------------------------
# keys and inputs
# ----------------------------------------------------------------------------
def fresh_key(S, seed):
    """uniform key words: every GGSW distinct (a real key's masks are uniform
    too, and the kernels' arithmetic does not depend on the bodies' structure)"""
    return np.random.default_rng(seed).integers(0, 2 ** 64, S.key_words, dtype=np.uint64)


def crafted_inputs(S, rng):
    """mask words of the modulus switch's edges (log_mod = log2(2N))"""
    n, sh = S.n, 64 - S.log_mod
    two_n = np.uint64(1 << S.log_mod)
    rnd = lambda: rng.integers(0, 2 ** 64, n + 1, dtype=np.uint64)
    out = []
    zero = rnd()
    zero[:n] = 0  # every step skipped (classic), every degree 0 (multi-bit)
    out.append(zero)
    edge = rnd()  # a_hat = N and a_hat = 2N - 1
    edge[0:n:3] = np.uint64(1 << 63)
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
    near[2:n:11] = ~np.uint64(0) - np.uint64((1 << (sh - 1)) - 1)
    out.append(near)
    return np.stack(out)


def input_pool(S, seed):
    """8 uniform LWEs (what a fresh encryption's mask is) and the crafted ones"""
    rng = np.random.default_rng(seed)
    uni = rng.integers(0, 2 ** 64, (8, S.n + 1), dtype=np.uint64)
    return np.ascontiguousarray(np.concatenate([uni, crafted_inputs(S, rng)]))


def luts_of(S, seed):
    """3 LUTs: two many-LUT accumulators (num_many_lut = 2, stride `stride`) and
    one of random words (exercises the u64 -> u32 rounding of the rotation)"""
    from tfhe_rs_b200 import algorithms

    p = 64 if S.family == "n8192" else 16
    delta = (1 << 63) // p
    fns = [[(a * x + b) % p for x in range(p)] for a, b in ((1, 0), (3, 1), (5, 2))]
    built = [algorithms.generate_many_lut_accumulator(S.N, 2, p, delta, [fns[j], fns[j + 1]]) for j in range(2)]
    rnd = np.random.default_rng(seed).integers(0, 2 ** 64, 2 * S.N, dtype=np.uint64)
    luts = np.stack([built[0][0].reshape(-1), built[1][0].reshape(-1), rnd])
    return np.ascontiguousarray(luts), int(built[0][1])


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
        t = self.torch.from_numpy(np.ascontiguousarray(a).view(np.int64).reshape(-1)).cuda()
        self.torch.cuda.synchronize()
        return t

    def host(self, t):
        self.sync()
        return t.cpu().numpy().view(np.uint64) if t.dtype == self.torch.int64 else t.cpu().numpy()

    def switches(self, sw):
        L = self.L
        L.b200_set_pbs_variant(sw.get("variant", 0))
        L.b200_set_register_kernels(sw.get("mask", 3))
        L.b200_set_multibit_ll_max(sw.get("ll_max", -1))
        L.b200_set_multibit_tie_rule(sw.get("ties", 0))

    def convert(self, S, bsk):
        d = self.torch.zeros(S.key_words, dtype=self.torch.float64, device="cuda")
        self.torch.cuda.synchronize()
        h = np.ascontiguousarray(bsk)
        if S.g > 1:
            self.L.cuda_convert_lwe_multi_bit_programmable_bootstrap_key_64_async(
                self.stream, 0, d.data_ptr(), h.ctypes.data, S.n, 1, S.l, S.N, S.g)
        else:
            self.L.cuda_convert_lwe_programmable_bootstrap_key_64_async(self.stream, 0, d.data_ptr(), h.ctypes.data,
                                                                        S.n, 1, S.l, S.N)
        self.sync()
        return d

    def convert_seeded(self, S, bodies, seed):
        d = self.torch.zeros(S.key_words, dtype=self.torch.float64, device="cuda")
        self.torch.cuda.synchronize()
        key = (seed & (2 ** 128 - 1)).to_bytes(16, "little")
        self.L.b200_convert_seeded_lwe_programmable_bootstrap_key_64_async(
            self.stream, 0, d.data_ptr(), np.ascontiguousarray(bodies).ctypes.data, key, 0, 0, 0, S.n, 1, S.l, S.N,
            S.g)
        self.sync()
        return d

    def pbs(self, S, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride, centered):
        """one launch into a sentinel-filled output; (output words, kernel)"""
        width = S.N + 1
        d_out = self.dev(np.full(rows * width, SENTINEL, dtype=np.uint64))
        d_lut, d_cts = self.dev(luts), self.dev(cts)
        d_oi, d_li, d_ii = (self.dev(np.asarray(a, dtype=np.uint64)) for a in (out_idx, lut_idx, in_idx))
        count = len(in_idx)
        buf = C.POINTER(C.c_int8)()
        L, st = self.L, self.stream
        if S.g > 1:
            L.scratch_cuda_multi_bit_programmable_bootstrap_64_async(st, 0, C.byref(buf), 1, S.N, S.l, count, True)
            L.cuda_multi_bit_programmable_bootstrap_64_async(
                st, 0, d_out.data_ptr(), d_oi.data_ptr(), d_lut.data_ptr(), d_li.data_ptr(), d_cts.data_ptr(),
                d_ii.data_ptr(), d_bsk.data_ptr(), buf, S.n, 1, S.N, S.g, S.base_log, S.l, count, many, stride)
            kernel = L.b200_last_pbs_kernel().decode()
            L.cleanup_cuda_multi_bit_programmable_bootstrap_64(st, 0, C.byref(buf))
        else:
            L.scratch_cuda_programmable_bootstrap_64_async(st, 0, C.byref(buf), S.n, 1, S.N, S.l, count, True,
                                                           int(centered))
            L.cuda_programmable_bootstrap_64_async(
                st, 0, d_out.data_ptr(), d_oi.data_ptr(), d_lut.data_ptr(), d_li.data_ptr(), d_cts.data_ptr(),
                d_ii.data_ptr(), d_bsk.data_ptr(), buf, S.n, 1, S.N, S.base_log, S.l, count, many, stride)
            kernel = L.b200_last_pbs_kernel().decode()
            L.cleanup_cuda_programmable_bootstrap_64(st, 0, C.byref(buf))
        return self.host(d_out).reshape(rows, width), kernel


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


SHAPES = {
    "p22": Shape("p22_n918", "p22", 918, 23),
    "mb2_l1": Shape("mb_g2_l1", "mb", 48, 22, 1, 2),
    "mb2_l2": Shape("mb_g2_l2", "mb", 48, 15, 2, 2),
    "mb3_l1": Shape("mb_g3_l1", "mb", 48, 22, 1, 3),
    "mb3_l2": Shape("mb_g3_l2_n918", "mb", 918, 15, 2, 3),
    "mb4_l1": Shape("mb_g4_l1_n920", "mb", 920, 22, 1, 4),
    "mb4_l2": Shape("mb_g4_l2", "mb", 48, 15, 2, 4),
    "n8192": Shape("n8192_n64", "n8192", 64, 15, 2),
}
WAVES = [1, (1, 0), (1, 1), (2, 0), (2, 1)]  # batch 1, one wave at 1 and 2 CTAs / SM, and one past each


def _rows():
    from tests.test_pbs_routes import FAST_VARIANTS, V6_LARGE, V6_SMALL

    rows = [Row("n2048_auto", "p22", "emu_pbs_p22_v3", {},
                [Run(1, V6_SMALL), Run((1, 0), V6_SMALL), Run((1, 1), V6_LARGE), Run((2, 0), V6_LARGE),
                 Run((2, 1), V6_LARGE), Run(4096, V6_LARGE)])]
    rows.append(Row("n2048_v1", "p22", "emu_pbs_p22", {"variant": 1}, [Run(b, "n2048_v1") for b in WAVES]))
    for v, name in FAST_VARIANTS.items():
        rows.append(Row("n2048_variant%d" % v, "p22", "emu_pbs_p22_v3", {"variant": v}, [Run(b, name) for b in WAVES]))
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
        t = np.stack(outs).reshape(len(cts), len(luts), 2, S.N + 1)
        if tk[-1]:
            self.tables[tk] = t
        return t


@pytest.fixture(scope="module")
def shapes(G, emus):
    return Shapes(G, emus)


def launch_plan(batch, many, pool, seed):
    rng = np.random.default_rng(seed)
    in_idx = rng.integers(0, pool, batch)
    in_idx[: min(batch, pool)] = np.arange(min(batch, pool))  # every input at least once where the batch allows
    lut_idx = rng.integers(0, 3, batch)
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
    in_idx, lut_idx, out_idx, rows = launch_plan(batch, many, len(cts), seed)
    out, kernel = lib.pbs(S, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride, centered)
    hit = np.concatenate([m * batch + out_idx for m in range(many)])
    addressed = np.zeros(rows, dtype=bool)
    addressed[hit] = True
    assert (out[~addressed] == SENTINEL).all(), ("stray write outside the addressed rows", where)
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
        configs = [(m, c) for m, c in CONFIGS if c in row.centered]
        for k, run in enumerate(row.runs):
            batch = run.batch if isinstance(run.batch, int) else run.batch[0] * G.sms + run.batch[1]
            many, centered = configs[k % len(configs)]
            table = shapes.table(row.shape, row.replay, centered, row.ties_even[0])
            where = (row.id, batch)
            kernel, samples, words, first, frac = run_and_compare(lib, d, d["d_bsk"], batch, many, centered, table,
                                                                  k * 7919 + batch, where)
            print("REPLAY %-22s %-24s batch %5d  many %d  centered %d  samples %5d  words %9d  %s" % (
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
    want = emu_convert(emus[0], S, d["bsk"])
    got = d["bskf"]
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    print("KEY %-16s words %9d  differing %d" % (S.name, got.size, bad.size))
    assert bad.size == 0, "%s: first differing word %d: %r != %r" % (S.name, bad[0], got[bad[0]], want[bad[0]])


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["p22", "mb3_l2"])
def test_seeded_key_ingest_gives_the_same_device_words(G, shapes, key):
    """masks regenerated on the GPU from the seed: the same device key as the
    standard-domain key with those masks converted"""
    from tests.test_multibit_generic_routes import _seeded_host_key

    d = shapes.get(key)
    S = d["S"]
    P = type("P", (), dict(N=S.N, k=1))
    bodies = np.ascontiguousarray(d["bsk"].reshape(-1, 2, S.N)[:, 1, :])
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
    keys = keyset(P, seed=0xB200F00D, with_ksk=False)
    S = Shape("p22_n64", "p22", 64, 23)
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
    stats, failures = phase_criterion(e, e_fft, acc32_tau(1, 2048, 32 - 23, 64))
    print("CONTROL shipped vs no-FMA phase: rms/floor %.3f, %d/%d words differ, %s" % (
        stats["ratio"], int((outs[0] != outs[1]).sum()), outs[0].size, failures or "ok"))
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
