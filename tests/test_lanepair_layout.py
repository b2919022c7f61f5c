"""The lane-pair layout of the shipped two-CTA N = 2048 classic PBS instance
(`n2048_v6<2,true,2,1>`, csrc/pbs_n2048.cuh): each warp holds 16 threads of
polynomial 0 on lanes 0-15 and the same 16 threads of polynomial 1 on lanes
16-31, exchange 2 runs inside each half-warp (x2h_*), exchange 1 through the
x1h_* swizzle, and the MAC takes the other polynomial's spectrum from lane
l ^ 16.

CPU: a replay of that lane map (tests/emu/emu_lanepair.cpp) is word-identical
to the emulated kernel of the other layouts, and its exchange-1 and accumulator
address patterns are bank-conflict free.  GPU: the instance is word-identical
to the two-CTA instance of the other layout (variant 17, `n2048_v6<2,true,2>`)
on the same keys and inputs."""
import ctypes as C

import numpy as np
import pytest

LANE_PAIR, OTHER_LAYOUT = "n2048_v6<2,true,2,1>", "n2048_v6<2,true,2>"


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    """(emulator of the other layouts, lane-pair replay), both built without
    floating-point contraction: the host compiler would otherwise fuse
    multiplies and adds differently in the two files, and word identity is a
    question of which operations run in which order."""
    from tests.emu.build_emu import build_no_contract

    libs = build_no_contract(str(tmp_path_factory.mktemp("emu_lanepair")))
    return [C.CDLL(libs["emu_p22.cpp"]), C.CDLL(libs["emu_lanepair.cpp"])]


@pytest.fixture(scope="module")
def emu(emus):
    return emus[0]


@pytest.fixture(scope="module")
def emu_lp(emus):
    return emus[1]


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _p22(oracle, n):
    return oracle.Params("P22_n%d" % n, n=n, k=1, N=2048, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                         lwe_noise_log2=45, glwe_noise_log2=17)


def _run(fn, bskf, P, lut, cts, centered, many, stride):
    out = np.zeros((many, len(cts), 2049), dtype=np.uint64)
    for s in range(len(cts)):
        fn(_vp(bskf), _vp(lut), _vp(np.ascontiguousarray(cts[s])), P.n, P.pbs_base_log, int(centered), many, stride,
           len(cts), _vp(out[0, s]))
    return out


def test_exchange1_layout_is_bank_conflict_free(emu_lp):
    assert emu_lp.emu_lanepair_conflict_audit(0, 0) == 1


def test_accumulator_rows_are_bank_conflict_free(emu_lp):
    """The two halves of a warp touch the same 16 coefficients of both
    accumulator rows; 16 words of row offset put them on disjoint banks, which
    the audit sees (and without the offset every access is a 2-way conflict)."""
    assert emu_lp.emu_lanepair_conflict_audit(1, 2048 + 16) == 1
    assert emu_lp.emu_lanepair_conflict_audit(1, 2048) == 2


@pytest.mark.parametrize("n,centered,many", [(1, True, 1), (16, True, 2), (16, False, 1), (48, True, 2)])
def test_lane_pair_replay_is_word_identical(oracle, keyset, emu, emu_lp, n, centered, many):
    """n = 1 is one CMUX; n = 16 and 48 a full PBS, with many-LUT outputs.  The
    masks include a zero word (a step that adds exactly nothing)."""
    P = _p22(oracle, n)
    keys = keyset(P, seed=11 + n, with_ksk=False)
    bskf = np.empty(P.n * 4 * 1024 * 2)
    emu.emu_bsk_convert_p22(_vp(keys.bsk), P.n, _vp(bskf))
    msgs = np.arange(6) % 16
    cts = oracle.lwe_encrypt_batch(oracle.Rng(3 + n), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    if n > 1:  # same message: the zeroed word's share comes out of the body
        with np.errstate(over="ignore"):
            cts[1, -1] -= cts[1, 3] * keys.lwe_sk[3]
        cts[1, 3] = 0
    lut = oracle.make_lut(P, [(5 * i + 3) % 16 for i in range(16)])
    want = _run(emu.emu_pbs_p22_v3, bskf, P, lut, cts, centered, many, 3)
    got = _run(emu_lp.emu_pbs_p22_lanepair, bskf, P, lut, cts, centered, many, 3)
    assert np.array_equal(got, want)
    dec = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, got[0]), P.delta, 16)
    assert np.array_equal(dec, np.array([(5 * m + 3) % 16 for m in msgs]))


# ----------------------------------------------------------------------------
# GPU: the shipped instance against the other layout, word for word
# ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def G():
    import torch

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import tfhe_rs_b200
    from tfhe_rs_b200 import gpu

    L = tfhe_rs_b200.lib()
    return type("G", (), dict(gpu=gpu, lib=L, streams=gpu.CudaStreams.new_single_gpu(0), sms=L.cuda_get_number_of_sms()))


def _launch(G, keys, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride, variant):
    P, gpu, st = keys.params, G.gpu, G.streams
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


@pytest.mark.gpu
@pytest.mark.parametrize("batch", ["sms+1", "ragged", 4096])
@pytest.mark.parametrize("many", [1, 2])
def test_lane_pair_instance_matches_other_layout(oracle, keyset, G, batch, many):
    from tfhe_rs_b200 import algorithms

    P = _p22(oracle, 64)
    keys = keyset(P, seed=0x1A9E, with_ksk=False)
    d_bsk = G.gpu.CudaLweBootstrapKey.from_lwe_bootstrap_key(
        keys.bsk, P.n, P.k, P.N, P.pbs_base_log, P.pbs_level,
        G.gpu.CudaModulusSwitchNoiseReductionConfiguration.CENTERED, G.streams)
    count = {"sms+1": G.sms + 1, "ragged": 3 * G.sms + 37}.get(batch, batch)
    rng = np.random.default_rng(count * 3 + many)
    pool = 64
    msgs = rng.integers(0, 4, pool)
    cts = oracle.lwe_encrypt_batch(oracle.Rng(count), keys.lwe_sk, msgs.astype(np.uint64) * np.uint64(P.delta), 45)
    fns = [[(a * x + b) % 16 for x in range(16)] for a, b in ((1, 0), (3, 1), (5, 2))]
    if many == 1:
        luts, stride = np.stack([oracle.make_lut(P, f) for f in fns]), 0
        rows = count + count // 2 + 3
        out_idx = rng.permutation(rows)[:count]
    else:
        built = [algorithms.generate_many_lut_accumulator(P.N, P.k + 1, P.p, P.delta, [fns[j], fns[(j + 1) % 3]])
                 for j in range(3)]
        luts, stride = np.stack([b[0] for b in built]), built[0][1]
        rows = many * count + 5
        out_idx = rng.permutation(count)
    in_idx = rng.integers(0, pool, count)
    lut_idx = rng.integers(0, 3, count)
    args = (G, keys, d_bsk, luts, cts, lut_idx, in_idx, out_idx, rows, many, stride)
    got, k_auto = _launch(*args, variant=0)
    want, k_other = _launch(*args, variant=17)
    assert (k_auto, k_other) == (LANE_PAIR, OTHER_LAYOUT)
    assert np.array_equal(got, want)
    written = np.zeros(rows, dtype=bool)
    for m in range(many):
        written[m * count + out_idx] = True
    assert np.all(got[~written] == np.uint64(0xDEADBEEFCAFEF00D))
    assert not np.any(got[written] == np.uint64(0xDEADBEEFCAFEF00D))
