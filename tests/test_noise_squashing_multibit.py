"""The multi-bit 128-bit PBS (noise squashing with grouped squashing keys)
against the exact multi-bit u128 blind rotation.

CPU: the exact model (tests/emu/pbs128_mb_exact.cpp, no kernel code) is pinned
against a Python big-integer restatement of tfhe-rs' multi-bit algorithm --
key generation's combined key bits, the degrees of the summed u64 mask words
and the selection-bit order, one bundle per group -- and decrypts a toy
squash; the kernel's folded MAC (compiled by g++) stays within a derived bound
of the exact product of a digit polynomial with sum_b X^{deg_b} B_b.

GPU: cuda_multi_bit_programmable_bootstrap_128_async across shapes, batches
and indexes against the exact model; the full squash shape; the Python API
end to end on tfhe-rs' GPU multi-bit parameters, through compression; and the
reference backend on the same keys and inputs when it is built."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests import pbs128_mb_model as MB
from tests import pbs128_model as P
from tests.noise_formula import multi_bit_pbs_fft_variance, multi_bit_pbs_variance_tuniform_fft
from tests.test_noise_squashing import _encrypt_small, _rand128, _signed, product_bound, py_decompose, py_negacyclic

MASK = P.MASK128
SENTINEL = 0xDEADBEEFCAFEF00D


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


# ----------------------------------------------------------------------------
# restatements (Python integers)
# ----------------------------------------------------------------------------
def py_switch(x, log_mod):
    return (((x >> (63 - log_mod)) + 1) >> 1) % (1 << log_mod)


def py_degrees(mask, g, log_mod):
    """modulus_switch_multi_bit: GGSW b (b >= 1) selects mask word u when bit
    g - 1 - u of b is set (selection_bit); the selected u64 words are summed
    with wrapping, then switched once."""
    return [py_switch(sum(int(mask[u]) for u in range(g) if (b >> (g - 1 - u)) & 1) % 2**64, log_mod)
            for b in range(1, 1 << g)]


def py_combined_bit(bits, b):
    """combine_key_bits: prod_u (s_u if bit g-1-u of b is set else 1 - s_u)."""
    g, m = len(bits), 1
    for u, s in enumerate(bits):
        m *= int(s) if (b >> (g - 1 - u)) & 1 else 1 - int(s)
    return m


def py_rotate(p, e):
    """p * X^e mod X^N + 1, e in [0, 2N)."""
    N = len(p)
    out = [0] * N
    for j, x in enumerate(p):
        t, neg = j + e, False
        while t >= N:
            t, neg = t - N, not neg
        out[t] = (-x if neg else x) & MASK
    return out


def py_pbs_multibit(bsk, lut, ct, n, k, N, g, base_log, level):
    """tfhe-rs' multi-bit blind rotation on Python integers: one bundle
    sum_b X^{deg_b} GGSW_b per group, acc <- bundle (x) acc, then sample
    extraction of coefficient 0."""
    log_mod = int(math.log2(N)) + 1
    words = P.to_int(bsk)
    polys = level * (k + 1) * (k + 1)
    acc = [py_rotate(lut[r * N:(r + 1) * N], (2 * N - py_switch(int(ct[n]), log_mod)) % (2 * N)) for r in range(k + 1)]
    for j in range(n // g):
        degs = [0] + py_degrees(ct[j * g:(j + 1) * g], g, log_mod)
        base = j * (1 << g) * polys * N
        bundle = [[0] * N for _ in range(polys)]
        for b in range(1 << g):
            for q in range(polys):
                off = base + (b * polys + q) * N
                rot = py_rotate(words[off:off + N], degs[b])
                bundle[q] = [(x + y) & MASK for x, y in zip(bundle[q], rot)]
        digits = [[py_decompose(x, base_log, level) for x in acc[r]] for r in range(k + 1)]
        new = [[0] * N for _ in range(k + 1)]
        for t in range(level):
            for r in range(k + 1):
                d = [digits[r][i][t] for i in range(N)]
                for c in range(k + 1):
                    prod = py_negacyclic(d, [_signed(x) for x in bundle[(t * (k + 1) + r) * (k + 1) + c]])
                    new[c] = [(x + y) & MASK for x, y in zip(new[c], prod)]
        acc = new
    out = []
    for r in range(k):
        out += [acc[r][0]] + [(-acc[r][N - t]) & MASK for t in range(1, N)]
    return out + [acc[k][0]]


def fft_term(n, k, N, base_log, level, g):
    """tfhe-rs' multi-bit FFT variance at mantissa 104 on the 2^128 torus."""
    return multi_bit_pbs_fft_variance(n, k, N, base_log, level, g, mantissa=104, modulus=2.0 ** 128)


def rounding_term(n, k, N, base_log, level, g):
    """The rounding term of the multi-bit formula: the bits the decomposition
    drops, over n / g steps."""
    q2, b2l = 2.0 ** -256, 2.0 ** (-2.0 * base_log * level)
    return n / g * (-q2 / 12 + k * N * (q2 / 48 + b2l / 24) + b2l / 12)


def _lut(k, N, f, p_msg):
    return P.make_lut(k, N, f, (1 << 127) // p_msg)


# ----------------------------------------------------------------------------
# CPU
# ----------------------------------------------------------------------------
def _crafted_mask(g):
    """Group words whose switched sum differs from the sum of the switched
    words (each is exactly half a step: it rounds up alone, and two of them
    make one step), and distinct words so that a reversed selection order
    changes the degrees."""
    half = 1 << (63 - 9)  # log_mod 9 (N = 256)
    return np.array([half, half + 3 * (half << 1), half + 17 * (half << 1), (1 << 63) + half][:g], dtype=np.uint64)


@pytest.mark.parametrize("g", [2, 3, 4])
def test_degrees_sum_words_before_switching(g):
    rng = np.random.default_rng(g)
    masks = [_crafted_mask(g)] + [rng.integers(0, 2**64, g, dtype=np.uint64, endpoint=False) for _ in range(50)]
    for mask in masks:
        want = py_degrees(mask, g, 9)
        assert MB.degrees(mask, g, 9) == want
        assert MB.kernel_degrees(mask, g, 9) == [0] + want
    crafted = _crafted_mask(g)
    # the rule matters on the crafted mask: switching each word first differs
    each = [py_switch(int(a), 9) for a in crafted]
    assert py_degrees(crafted, g, 9)[2] != (each[g - 2] + each[g - 1]) % 512
    # and the selection order: the reversed order gives other degrees
    assert py_degrees(crafted, g, 9) != py_degrees(crafted[::-1], g, 9)


@pytest.mark.parametrize("g", [2, 4])
def test_keygen_encrypts_combined_key_bits(g):
    prm = P.Params128(n=8, k=1, N=256, base_log=24, level=2, glwe_noise_log2=30)
    keys = MB.keygen(prm, g, 5 + g)
    words = MB.ggsw_words(prm)
    N, k, l = prm.N, prm.k, prm.level
    for j in range(prm.n // g):
        bits = keys.lwe_sk[j * g:(j + 1) * g]
        for b in range(1 << g):
            ggsw = keys.bsk[(j * (1 << g) + b) * words:(j * (1 << g) + b + 1) * words]
            # row r = k of level index l - 1 (level 1): phase m * 2^(128 - base_log) in coefficient 0
            row = ggsw[((l - 1) * (k + 1) + k) * (k + 1) * N:((l - 1) * (k + 1) + k + 1) * (k + 1) * N]
            mask, body = P.to_int(row[:k * N]), P.to_int(row[k * N:])
            s = [int(x) for x in keys.glwe_sk]
            prod = py_negacyclic(s, [_signed(x) for x in mask])
            phase = _signed(body[0] - prod[0]) / 2.0 ** (128 - prm.base_log)
            assert round(phase) == py_combined_bit(bits, b), (j, b, phase)


@pytest.mark.parametrize("g", [2, 4])
def test_exact_model_matches_python(g):
    prm = P.Params128(n=8, k=1, N=256, base_log=24, level=2, glwe_noise_log2=30)
    keys = MB.keygen(prm, g, 21 + g)
    rng = np.random.default_rng(g)
    cts = _encrypt_small(rng, keys.lwe_sk, [3, 11], (1 << 63) // 16, 30)
    cts[0, :g] = _crafted_mask(g)
    lut = _lut(prm.k, prm.N, [(5 * m + 1) % 16 for m in range(16)], 16)
    out = MB.pbs_exact(keys, lut, cts)
    for s in range(len(cts)):
        want = py_pbs_multibit(keys.bsk, P.to_int(lut), [int(x) for x in cts[s]], prm.n, prm.k, prm.N, g,
                               prm.base_log, prm.level)
        assert P.to_int(out[s]) == want


@pytest.mark.parametrize("g", [2, 3, 4])
def test_exact_squash_decrypts_toy(g):
    p = 16
    prm = P.Params128(n=12, k=1, N=256, base_log=24, level=3, glwe_noise_log2=30)
    keys = MB.keygen(prm, g, 40 + g)
    msgs = list(range(p))
    cts = _encrypt_small(np.random.default_rng(3), keys.lwe_sk, msgs, (1 << 63) // p, 20)
    f = [(5 * m + 3) % p for m in msgs]
    out = MB.pbs_exact(keys, _lut(prm.k, prm.N, f, p), cts)
    assert P.decode(P.decrypt(keys.glwe_sk, out), (1 << 127) // p, p) == f


@pytest.mark.parametrize("N", [256, 1024, 2048, 4096])
@pytest.mark.parametrize("g", [2, 4])
def test_folded_mac_within_bound(N, g):
    """The kernel's fold, d * sum_b X^{deg_b} B_b through its transforms,
    against the exact product.  Each term is a transform-based product of d
    with B_b whose spectrum is multiplied once more by a double-double root,
    so the bound is the sum over b of product_bound at one more level."""
    rng = np.random.default_rng(N + g)
    nggsw = 1 << g
    d = [int(x) for x in rng.integers(-2**17, 2**17 + 1, N)]
    Gs = [_rand128(rng, N) for _ in range(nggsw)]
    degs = [0] + [int(x) for x in rng.integers(0, 2 * N, nggsw - 1)]
    D = P.to_u128(d)
    exact = P.zeros128(N)
    for b in range(nggsw):
        rot = P.to_u128(py_rotate(Gs[b], degs[b]))
        P.lib().p128_negacyclic_mul_add(_vp(exact), _vp(D), _vp(rot), N)
    got = P.zeros128(N)
    MB.model().emu128_mb_product(_vp(D), _vp(P.to_u128([x for G in Gs for x in G])),
                                 _vp(np.array(degs, dtype=np.uint32)), nggsw, N, _vp(got))
    err = max(abs(_signed(a - b)) for a, b in zip(P.to_int(got), P.to_int(exact)))
    logM = int(math.log2(N)) - 1
    bound = sum(product_bound(d, G, logM + 1) for G in Gs)
    assert err <= bound, (math.log2(max(err, 1)), math.log2(bound))


# ----------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def G():
    import torch

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import tfhe_rs_b200
    from tfhe_rs_b200 import gpu

    L = tfhe_rs_b200.lib()
    return type("G", (), dict(gpu=gpu, lib=L, st=gpu.CudaStreams.new_single_gpu(0), torch=torch,
                              sms=L.cuda_get_number_of_sms()))


def upload_bsk_mb(G, keys, lib=None):
    lib = lib or G.lib
    p = keys.params
    d = G.torch.zeros(keys.bsk.size, dtype=G.torch.float64, device=G.st.device(0))
    G.torch.cuda.synchronize()
    lib.cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async(G.st.ptr(0), 0, d.data_ptr(),
                                                                        keys.bsk.ctypes.data, p.n, p.k, p.level, p.N,
                                                                        keys.grouping)
    G.torch.cuda.synchronize()
    return d


def gpu_pbs_mb(G, keys, d_bsk, lut, cts, in_idx=None, out_idx=None, rows=None, lib=None):
    """One call into a sentinel-filled output of `rows` LWEs; returns the
    output words, the kernel name and the launch count."""
    lib = lib or G.lib
    torch, p = G.torch, keys.params
    dev = G.st.device(0)
    width = p.k * p.N + 1
    count = len(in_idx) if in_idx is not None else len(cts)
    in_idx = np.arange(count, dtype=np.uint64) if in_idx is None else np.asarray(in_idx, dtype=np.uint64)
    out_idx = np.arange(count, dtype=np.uint64) if out_idx is None else np.asarray(out_idx, dtype=np.uint64)
    rows = rows or count
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).to(dev)
    d_out = t(np.full((rows, width, 2), SENTINEL, dtype=np.uint64))
    d_lut, d_in, d_ii, d_oi = t(lut), t(cts), t(in_idx), t(out_idx)
    buf = C.POINTER(C.c_int8)()
    torch.cuda.synchronize()
    lib.scratch_cuda_multi_bit_programmable_bootstrap_128_async(G.st.ptr(0), 0, C.byref(buf), p.k, p.N, p.level,
                                                                count, True)
    counter = lib if hasattr(lib, "b200_kernel_launch_count") else G.lib  # the reference has no counter
    before = counter.b200_kernel_launch_count()
    lib.cuda_multi_bit_programmable_bootstrap_128_async(G.st.ptr(0), 0, d_out.data_ptr(), d_oi.data_ptr(),
                                                        d_lut.data_ptr(), d_in.data_ptr(), d_ii.data_ptr(),
                                                        d_bsk.data_ptr(), buf, p.n, p.k, p.N, keys.grouping,
                                                        p.base_log, p.level, count, 1, 0)
    launches = counter.b200_kernel_launch_count() - before
    kernel = counter.b200_last_pbs_kernel().decode()
    lib.cleanup_cuda_multi_bit_programmable_bootstrap_128(G.st.ptr(0), 0, C.byref(buf))
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64).reshape(rows, width, 2), kernel, launches


def _route_world(N, k, g, base_log, level, n, seed):
    p_msg = 16
    prm = P.Params128(n=n, k=k, N=N, base_log=base_log, level=level, glwe_noise_log2=2)
    keys = MB.keygen(prm, g, seed)
    rng = np.random.default_rng(seed)
    pool = 4  # distinct inputs; the exact model runs on these
    msgs = [int(x) for x in rng.integers(0, p_msg, pool)]
    cts = _encrypt_small(rng, keys.lwe_sk, msgs, (1 << 63) // p_msg, 30)
    f = [(7 * m + 2) % p_msg for m in range(p_msg)]
    lut = _lut(k, N, f, p_msg)
    exact_phase = P.decrypt(keys.glwe_sk, MB.pbs_exact(keys, lut, cts))
    assert P.decode(exact_phase, (1 << 127) // p_msg, p_msg) == [f[m] for m in msgs]
    return keys, cts, lut, msgs, f, exact_phase


# (N, k, g, base_log, level, n, batches); "sms-1" etc. resolved at run time
ROUTES = [
    (256, 1, 2, 18, 4, 8, [1, "sms-1", "sms+1", "4sms+5"]),
    (256, 2, 3, 24, 3, 6, [1, 33]),
    (512, 1, 4, 32, 4, 8, [1, "sms+1"]),
    (512, 2, 2, 24, 3, 4, [7]),
    (2048, 2, 4, 18, 4, 8, [1, "sms-1", "sms+1"]),
    (2048, 1, 3, 24, 3, 6, [5]),
    (2048, 2, 2, 32, 4, 4, [3]),
    (4096, 1, 2, 32, 4, 4, [1, "sms+1"]),
    (4096, 2, 4, 18, 4, 4, [2]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("N,k,g,base_log,level,n,batches", ROUTES,
                         ids=["N%d_k%d_g%d_%dx%d_n%d" % r[:6] for r in ROUTES])
def test_pbs128_mb_route_against_exact(G, N, k, g, base_log, level, n, batches):
    keys, cts, lut, msgs, f, exact_phase = _route_world(N, k, g, base_log, level, n, 3000 + N + k + g)
    d_bsk = upload_bsk_mb(G, keys)
    p_msg, delta = 16, (1 << 127) // 16
    sigma = math.sqrt(fft_term(n, k, N, base_log, level, g))
    bound = 2 * math.sqrt(fft_term(n, k, N, base_log, level, g) + 2 * rounding_term(n, k, N, base_log, level, g))
    for b in batches:
        b = {"sms-1": G.sms - 1, "sms+1": G.sms + 1, "4sms+5": 4 * G.sms + 5}.get(b, b)
        idx = np.arange(b) % len(cts)
        out, kernel, launches = gpu_pbs_mb(G, keys, d_bsk, lut, cts[idx], rows=b + 3)
        assert kernel == "pbs128_mb<%d>" % N
        assert launches == 1
        assert (out[b:] == SENTINEL).all(), "rows past num_samples were written"
        phase = P.decrypt(keys.glwe_sk, out[:b])
        assert P.decode(phase, delta, p_msg) == [f[msgs[i]] for i in idx]
        err = [_signed(x - exact_phase[i]) / 2.0 ** 128 for x, i in zip(phase, idx)]
        rms = math.sqrt(sum(e * e for e in err) / len(err))
        print(f"N={N} k={k} g={g} {base_log}x{level} batch {b}: rms {rms:.3g}, / fft-term sigma {rms / sigma:.3g}, "
              f"/ bound {rms / bound:.3g}")
        assert rms <= bound, (rms, bound)
        if (N, k, base_log, level, g) == (2048, 2, 18, 4, 4):
            assert rms <= 2 * sigma, (rms, sigma)


@pytest.mark.gpu
def test_pbs128_mb_indexes(G):
    keys, cts, lut, msgs, f, exact_phase = _route_world(512, 1, 2, 24, 3, 4, 77)
    d_bsk = upload_bsk_mb(G, keys)
    count, rows = G.sms + 1, 3 * G.sms
    rng = np.random.default_rng(5)
    in_idx = rng.integers(0, len(cts), count)  # repeated rows
    out_idx = rng.permutation(rows)[:count]  # scattered rows
    out, kernel, launches = gpu_pbs_mb(G, keys, d_bsk, lut, cts, in_idx, out_idx, rows=rows)
    assert kernel == "pbs128_mb<512>" and launches == 1
    untouched = np.setdiff1d(np.arange(rows), out_idx)
    assert (out[untouched] == SENTINEL).all()
    phase = P.decrypt(keys.glwe_sk, out[out_idx])
    assert P.decode(phase, (1 << 127) // 16, 16) == [f[msgs[i]] for i in in_idx]


@pytest.fixture(scope="module")
def nofma(G):
    """The library built with -fmad=false (tests/emu/build_nofma.py): its
    kernels compute the CPU replay's words exactly."""
    from tests.emu.build_nofma import LIB
    from tfhe_rs_b200 import _lib

    return _lib.load(LIB)


@pytest.mark.gpu
def test_pbs128_mb_words_equal_the_replay(G, nofma):
    """Every output word of the -fmad=false kernel equals the CPU replay of
    its own phases, on a key of uniform words at n = 920: a key block read
    from the wrong group or GGSW changes the output."""
    prm = P.Params128(n=920, k=1, N=256, base_log=18, level=4, glwe_noise_log2=2)
    g = 4
    rng = np.random.default_rng(920)
    words = (prm.n // g << g) * MB.ggsw_words(prm)
    keys = MB.KeysMb(prm, g, np.zeros(prm.n, dtype=np.uint64), np.zeros(prm.N, dtype=np.uint64),
                     rng.integers(0, 2**64, (words, 2), dtype=np.uint64))
    pool = rng.integers(0, 2**64, (3, prm.n + 1), dtype=np.uint64)
    lut = P.to_u128(_rand128(rng, (prm.k + 1) * prm.N))
    want = MB.replay_pbs(keys, lut, pool)
    d_bsk = upload_bsk_mb(G, keys, nofma)
    for b in (1, G.sms, G.sms + 1):
        idx = np.arange(b) % len(pool)
        out, kernel, launches = gpu_pbs_mb(G, keys, d_bsk, lut, pool, in_idx=idx, rows=b + 2, lib=nofma)
        assert launches == 1 and kernel == "pbs128_mb<256>"
        assert (out[b:] == SENTINEL).all()
        assert np.array_equal(out[:b], want[idx]), f"batch {b}"


SQUASH = dict(n=920, k=2, N=2048, base_log=18, level=4, g=4)


@pytest.fixture(scope="module")
def mb4_world(G, oracle, keyset):
    """tfhe-rs' GPU multi-bit g = 4 server keys and a multi-bit squashing key
    (k = 2, N = 2048, 18 x 4, g = 4, TUniform(30)) on their small key, built
    from one generated group per pattern of 4 key bits."""
    from oracle import csprng
    from tfhe_rs_b200 import noise_squashing, server_key

    Pp = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(Pp, seed=0x5A4)
    s = SQUASH
    prm = P.Params128(n=s["n"], k=s["k"], N=s["N"], base_log=s["base_log"], level=s["level"], glwe_noise_log2=30)
    sq = MB.pooled_keygen(prm, s["g"], 920, keys.lwe_sk)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=Pp.n, k=Pp.k, N=Pp.N, pbs_base_log=Pp.pbs_base_log,
                                        pbs_level=Pp.pbs_level, ks_base_log=Pp.ks_base_log, ks_level=Pp.ks_level,
                                        grouping_factor=Pp.grouping_factor, centered_ms=False, streams=G.st)
    nsk = noise_squashing.CudaNoiseSquashingKey.from_multi_bit_bootstrap_key_128(
        sq.bsk, s["n"], s["k"], s["N"], s["base_log"], s["level"], s["g"], 4, 4, G.st)
    return Pp, keys, sq, skey, nsk


@pytest.mark.gpu
def test_pbs128_mb_full_squash_parameters(G, mb4_world):
    _, _, sq, _, nsk = mb4_world
    s = SQUASH
    p_msg, count = 16, 4096
    rng = np.random.default_rng(4096)
    msgs = [int(x) for x in rng.integers(0, p_msg, count)]
    cts = _encrypt_small(rng, sq.lwe_sk, msgs, (1 << 63) // p_msg, 45)
    delta = (1 << 127) // p_msg
    lut = _lut(s["k"], s["N"], list(range(p_msg)), p_msg)
    out, kernel, _ = gpu_pbs_mb(G, sq, _Ptr(nsk.d_bsk.as_c_ptr()), lut, cts)
    assert kernel == "pbs128_mb<2048>"
    phase = P.decrypt(sq.glwe_sk, out)
    assert P.decode(phase, delta, p_msg) == msgs
    err = P.centered_error(phase, msgs, delta)
    var = sum(e * e for e in err) / count
    formula = multi_bit_pbs_variance_tuniform_fft(s["n"], s["k"], s["N"], s["base_log"], s["level"], s["g"],
                                                  mantissa=104, modulus=2.0 ** 128)
    print(f"full multi-bit squash parameters: measured variance / formula = {var / formula:.3f}")
    assert var <= 1.1 * formula, (var, formula)


class _Ptr:
    """A device pointer passed where a tensor's data_ptr() is read."""

    def __init__(self, ptr):
        self.ptr = ptr

    def data_ptr(self):
        return self.ptr


def _mb4_item(G, oracle, Pp, keys, kind, count, seed):
    from tfhe_rs_b200 import compact_list, integer

    rng = np.random.default_rng(seed)
    if kind == "boolean":
        digits = [1]
    elif kind == "signed":
        value = -123456789012345 % 2**64
        digits = [(value >> (2 * i)) & 3 for i in range(count)]
    else:
        digits = [int(x) for x in rng.integers(0, 4, count)]
    cts = oracle.lwe_encrypt_batch(oracle.Rng(seed), keys.glwe_sk,
                                   np.asarray(digits, dtype=np.uint64) * np.uint64(Pp.delta), Pp.lwe_noise_log2)
    blocks = G.torch.from_numpy(cts.view(np.int64)).to(G.st.device(0))
    ct = {"unsigned": integer.CudaUnsignedRadixCiphertext, "signed": compact_list.CudaSignedRadixCiphertext,
          "boolean": compact_list.CudaBooleanBlock}[kind](blocks)
    pairs = [digits[2 * i] + 4 * (digits[2 * i + 1] if 2 * i + 1 < count else 0) for i in range((count + 1) // 2)]
    return ct, pairs


@pytest.mark.gpu
def test_squash_multi_bit_end_to_end_and_compress(G, oracle, mb4_world):
    from tests import pks128_model as M
    from tfhe_rs_b200 import squashed_compression as SC

    Pp, keys, sq, skey, nsk = mb4_world
    assert nsk.grouping_factor == 4
    r = M.REAL_MB
    assert r["n"] == SQUASH["k"] * SQUASH["N"]
    comp_sk = np.random.default_rng(9).integers(0, 2, r["k"] * r["N"], dtype=np.uint64)
    ckey_words = M.gen_key(33, sq.glwe_sk, comp_sk, r["k"], r["N"], r["base_log"], r["level"])
    ckey = SC.CudaNoiseSquashingCompressionKey(ckey_words, r["n"], r["k"], r["N"], r["base_log"], r["level"], r["L"],
                                               G.st)
    b = SC.CudaCompressedSquashedNoiseCiphertextListBuilder()
    want = []
    for i, (kind, count) in enumerate([("unsigned", 32), ("unsigned", 7), ("signed", 32), ("boolean", 1)]):
        ct, pairs = _mb4_item(G, oracle, Pp, keys, kind, count, 50 + i)
        before = G.lib.b200_kernel_launch_count()
        res = nsk.squash_radix_ciphertext_noise(skey, ct)
        launches = G.lib.b200_kernel_launch_count() - before
        ks_launches = 2 if G.lib.b200_last_keyswitch_kernel().decode().startswith("ks_imma") else 1
        assert launches == 2 + ks_launches  # packing, keyswitch, PBS
        assert G.lib.b200_last_pbs_kernel().decode() == "pbs128_mb<2048>"
        assert res.kind == kind and res.original_block_count == count
        host = res.to_host()
        assert host.shape == ((count + 1) // 2, r["n"] + 1, 2)
        assert M.decode(sq.glwe_sk, host) == pairs
        b.push(res)
        want.append(pairs)
    lst = b.build(ckey, G.st)
    for i, pairs in enumerate(want):
        assert M.decode(comp_sk, lst.get(i, G.st).to_host()) == pairs


@pytest.mark.gpu
def test_squash_multi_bit_rejects_bad_arguments(G, oracle, mb4_world):
    import dataclasses

    from tfhe_rs_b200 import integer, noise_squashing

    Pp, keys, sq, skey, nsk = mb4_world
    s = SQUASH
    ctor = noise_squashing.CudaNoiseSquashingKey.from_multi_bit_bootstrap_key_128
    before = G.lib.b200_kernel_launch_count()
    for args in [(sq.bsk, 920, 2, 2048, 18, 4, 5, 4, 4),  # grouping factor
                 (sq.bsk, 918, 2, 2048, 18, 4, 4, 4, 4),  # n not a multiple of g
                 (sq.bsk[:-1], 920, 2, 2048, 18, 4, 4, 4, 4),  # key size
                 (sq.bsk, 920, 2, 8192, 18, 4, 4, 4, 4),  # polynomial size
                 (sq.bsk, 920, 2, 2048, 18, 4, 4, 8, 4)]:  # moduli
        with pytest.raises(ValueError):
            ctor(*args, G.st)
    wrong = G.torch.zeros((2, 100), dtype=G.torch.int64, device=G.st.device(0))
    with pytest.raises(ValueError):
        nsk.squash_radix_ciphertext_noise(skey, integer.CudaUnsignedRadixCiphertext(wrong))
    other = dataclasses.replace(skey, message_modulus=8, carry_modulus=8)
    ct, _ = _mb4_item(G, oracle, Pp, keys, "unsigned", 2, 5)
    with pytest.raises(ValueError):
        nsk.squash_radix_ciphertext_noise(other, ct)
    assert G.lib.b200_kernel_launch_count() == before
    assert s["g"] == nsk.grouping_factor


REF_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                       "libtfhe_cuda_backend_ref.so")


@pytest.mark.gpu
@pytest.mark.parametrize("N,k,g,base_log,level,n", [(2048, 2, 4, 18, 4, 8), (512, 1, 2, 24, 3, 4)])
def test_pbs128_mb_matches_reference_backend(G, N, k, g, base_log, level, n):
    if not os.path.exists(REF_LIB):
        pytest.skip("the reference CUDA backend is not built (oracle/_ref/libtfhe_cuda_backend_ref.so)")
    from tfhe_rs_b200 import _lib

    ref = _lib.load(REF_LIB, strict=False)
    try:
        getattr(ref, "cuda_multi_bit_programmable_bootstrap_128_async")
    except AttributeError:
        pytest.skip("the reference build lacks cuda_multi_bit_programmable_bootstrap_128_async")
    keys, cts, lut, msgs, f, exact_phase = _route_world(N, k, g, base_log, level, n, 555 + N)
    bound = 2 * math.sqrt(fft_term(n, k, N, base_log, level, g) + 2 * rounding_term(n, k, N, base_log, level, g))
    idx = np.arange(G.sms + 1) % len(cts)
    results = []
    for lib in (G.lib, ref):
        d_bsk = upload_bsk_mb(G, keys, lib)
        out, _, _ = gpu_pbs_mb(G, keys, d_bsk, lut, cts[idx], lib=lib)
        phase = P.decrypt(keys.glwe_sk, out)
        dec = P.decode(phase, (1 << 127) // 16, 16)
        assert dec == [f[msgs[i]] for i in idx]
        err = [_signed(x - exact_phase[i]) / 2.0 ** 128 for x, i in zip(phase, idx)]
        rms = math.sqrt(sum(e * e for e in err) / len(err))
        print(f"{'b200' if lib is G.lib else 'reference'} N={N} g={g}: rms against exact {rms:.3g}, bound {bound:.3g}")
        assert rms <= bound, (rms, bound)
        results.append(dec)
    assert results[0] == results[1]
