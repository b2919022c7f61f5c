"""Exchange 2 of the lane-pair N = 2048 classic PBS through the warp's own rows
of the exchange-1 buffer (x2m_*, csrc/x2_smem.cuh) instead of half-warp
shuffles (x2h_*, csrc/x2_shfl.cuh).

CPU (tests/emu/emu_lanepair.cpp): x2m_* leaves exactly the registers x2h_*
leaves on all 32 lanes, every quarter-warp access of its slot map is
bank-conflict free, and a whole PBS replayed with it is word-identical to the
lane-pair replay with shuffles.
GPU: the two lane-pair instances and the round-1 kernel agree word for word on
a PARAM_MESSAGE_2_CARRY_2 key, and the automatic two-CTA route runs the
instance with exchange 2 through shared memory."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
# variant id -> instance name (b200_backend.cu, N2048_INSTANCES)
X2M, X2H, ROUND1 = 20, 23, 5
NAMES = {X2M: "n2048_v6<2,true,2,1>", X2H: "n2048_v6<2,true,2,1,0>", ROUND1: "n2048_v3<0,1>"}


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    """(lane-pair replay with either exchange 2, emulator of the other layouts
    for the key conversion), both built without floating-point contraction so
    that word identity is a question of which operations run in which order."""
    d = tmp_path_factory.mktemp("emu_x2m")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    libs = []
    for src in ("emu_lanepair.cpp", "emu_p22.cpp"):
        out = str(d / src.replace(".cpp", ".so"))
        subprocess.check_call([gxx, "-O2", "-mavx2", "-mfma", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
                               "-w", "-x", "c++", os.path.join(HERE, "emu", src), "-o", out])
        libs.append(C.CDLL(out))
    libs[0].emu_x2m_register_check.argtypes = [C.c_uint64]
    return libs


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _p22(oracle, n):
    return oracle.Params("P22_n%d" % n, n=n, k=1, N=2048, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                         lwe_noise_log2=45, glwe_noise_log2=17)


@pytest.mark.parametrize("seed", [1, 2, 0xC0FFEE])
def test_x2m_reproduces_x2h_register_for_register(emus, seed):
    """Forward and inverse, all 32 lanes x 16 registers, bit for bit."""
    assert emus[0].emu_x2m_register_check(seed) == 0


def test_x2m_slot_map_is_bank_conflict_free(emus):
    """Both access sides of both directions hit 8 distinct 16-byte bank groups
    per quarter-warp; the unswizzled map 16 i + b would be an 8-way conflict on
    the pass-3 side, which the audit sees."""
    assert emus[0].emu_x2m_conflict_audit(1) == 1
    assert emus[0].emu_x2m_conflict_audit(0) == 8


@pytest.mark.parametrize("n,centered,many", [(1, True, 1), (16, True, 2), (48, False, 2)])
def test_x2m_replay_is_word_identical(oracle, keyset, emus, n, centered, many):
    """A whole PBS with exchange 2 through the warps' rows (run warp after warp
    inside the pass-2 window) against the lane-pair replay with shuffles."""
    P = _p22(oracle, n)
    keys = keyset(P, seed=31 + n, with_ksk=False)
    bskf = np.empty(P.n * 4 * 1024 * 2)
    lp, emu = emus
    emu.emu_bsk_convert_p22(_vp(keys.bsk), P.n, _vp(bskf))
    msgs = np.arange(6) % 16
    cts = oracle.lwe_encrypt_batch(oracle.Rng(5 + n), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    if n > 1:  # a zero mask word: a step that adds exactly nothing
        with np.errstate(over="ignore"):
            cts[1, -1] -= cts[1, 3] * keys.lwe_sk[3]
        cts[1, 3] = 0
    lut = oracle.make_lut(P, [(7 * i + 2) % 16 for i in range(16)])
    outs = []
    for fn in (lp.emu_pbs_p22_lanepair, lp.emu_pbs_p22_lanepair_x2m):
        out = np.zeros((many, len(cts), 2049), dtype=np.uint64)
        for s in range(len(cts)):
            fn(_vp(bskf), _vp(lut), _vp(np.ascontiguousarray(cts[s])), P.n, P.pbs_base_log, int(centered), many, 3,
               len(cts), _vp(out[0, s]))
        outs.append(out)
    assert np.array_equal(outs[1], outs[0])
    dec = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, outs[1][0]), P.delta, 16)
    assert np.array_equal(dec, np.array([(7 * m + 2) % 16 for m in msgs]))


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
    return type("G", (), dict(gpu=gpu, lib=L, streams=gpu.CudaStreams.new_single_gpu(0), sms=L.cuda_get_number_of_sms()))


@pytest.fixture(scope="module")
def p22(oracle, keyset, G):
    P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0xB2000023, with_ksk=False)
    d_bsk = G.gpu.CudaLweBootstrapKey.from_lwe_bootstrap_key(
        keys.bsk, P.n, P.k, P.N, P.pbs_base_log, P.pbs_level,
        G.gpu.CudaModulusSwitchNoiseReductionConfiguration.CENTERED, G.streams)
    return P, keys, d_bsk


def _launch(G, P, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride, variant):
    gpu, st = G.gpu, G.streams
    G.lib.b200_set_pbs_variant(variant)
    try:
        d_out = gpu.CudaLweCiphertextList.from_lwe_ciphertext_list(
            np.full((rows, P.N + 1), 0xDEADBEEFCAFEF00D, dtype=np.uint64), st)
        v = lambda a: gpu.CudaVec.from_cpu_async(np.ascontiguousarray(a, dtype=np.uint64).reshape(-1), st)
        gpu.programmable_bootstrap(st, d_out.d_vec, v(out_idx), v(luts), v(lut_idx), v(cts), v(in_idx), d_bsk.d_vec,
                                   P.n, P.k, P.N, P.pbs_base_log, P.pbs_level, len(in_idx),
                                   d_bsk.ms_noise_reduction_configuration, many, stride)
        kernel = G.lib.b200_last_pbs_kernel().decode()
        st.synchronize()
        return d_out.to_lwe_ciphertext_list(st), kernel
    finally:
        G.lib.b200_set_pbs_variant(0)


def _case(oracle, P, keys, count, many):
    from tfhe_rs_b200 import algorithms

    rng = np.random.default_rng(count * 7 + many)
    pool = 64
    msgs = rng.integers(0, 4, pool)
    cts = oracle.lwe_encrypt_batch(oracle.Rng(count + many), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta),
                                   P.lwe_noise_log2)
    fns = [[(a * x + b) % 16 for x in range(16)] for a, b in ((1, 0), (3, 1), (5, 2))]
    in_idx = rng.integers(0, pool, count)
    lut_idx = rng.integers(0, 3, count)
    if many == 1:
        luts, stride = np.stack([oracle.make_lut(P, f) for f in fns]), 0
        rows = count + 3
        out_idx = rng.permutation(rows)[:count]
        want = [[fns[lut_idx[s]][msgs[in_idx[s]]] for s in range(count)]]
    else:
        built = [algorithms.generate_many_lut_accumulator(P.N, P.k + 1, P.p, P.delta, [fns[j], fns[(j + 1) % 3]])
                 for j in range(3)]
        luts, stride = np.stack([b[0] for b in built]), built[0][1]
        rows = many * count
        out_idx = rng.permutation(count)
        want = [[fns[(lut_idx[s] + m) % 3][msgs[in_idx[s]]] for s in range(count)] for m in range(many)]
    return (luts, cts, lut_idx, in_idx, out_idx, rows, many, stride), want


@pytest.mark.gpu
@pytest.mark.parametrize("count", [300, 4096])
@pytest.mark.parametrize("many", [1, 2])
def test_x2m_instance_matches_shuffle_and_round1(oracle, G, p22, count, many):
    """300 is more than one wave of 264 resident CTAs; 4096 the bench batch."""
    P, keys, d_bsk = p22
    args, want = _case(oracle, P, keys, count, many)
    luts, cts, lut_idx, in_idx, out_idx, rows, many, stride = args
    outs = {}
    for variant in (X2M, X2H, ROUND1):
        outs[variant], kernel = _launch(G, P, d_bsk, *args, variant=variant)
        assert kernel == NAMES[variant]
    assert np.array_equal(outs[X2M], outs[X2H])
    assert np.array_equal(outs[X2M], outs[ROUND1])
    for m in range(many):
        got = outs[X2M][m * count + out_idx] if many > 1 else outs[X2M][out_idx]
        dec = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, got), P.delta, 16)
        assert np.array_equal(dec, np.array(want[m]))


@pytest.mark.gpu
def test_automatic_two_cta_route_runs_the_x2m_instance(oracle, G, p22):
    P, keys, d_bsk = p22
    count = 2 * G.sms + 7  # past one CTA per SM: the two-CTA route
    args, _ = _case(oracle, P, keys, count, 1)
    got, kernel = _launch(G, P, d_bsk, *args, variant=0)
    assert kernel == NAMES[X2M]
    want, _ = _launch(G, P, d_bsk, *args, variant=X2M)
    assert np.array_equal(got, want)
