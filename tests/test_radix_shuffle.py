"""Oblivious bitonic shuffle of radix integers (tfhe-rs_b200/radix_shuffle.py,
the shuffle methods of integer.CudaRadixServerKey, and
CudaOprfServerKey.generate_oblivious_pseudo_random_bits_chunks_and_re_randomize).

CPU: the network against the reference's own n = 8 table and the 0-1
principle; the key-size rule; the compare-and-swap schedule on
`bit_circuit.run_cleartext` (which asserts the noise budget and the value
range on every row), exhaustively over the keys at 1 and 2 blocks in both
directions and on random FheUint64 / FheInt64 data; whole shuffles through
the server key's host code on a cleartext runner against
`tests/shuffle_model.py`, with heavy ties; one pair through real keyswitches
and PBS on the oracle; the re-randomization seed against an independent
SHAKE256 composition; argument checks; pinned counts.

GPU: classic P22 and multi-bit g = 4 compute keys (the OPRF key on the same
bootstrapping key): shuffles by encrypted keys, by OPRF keys (against the
exact OPRF model of tests/test_oprf.py), with re-randomized keys (word for
word against tests/rerand_model.py), and shuffled outputs into add and gt."""
import hashlib
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import bit_circuit as bc, integer, radix as R, radix_shuffle as S

from tests import shuffle_model as SM
from tests import trivium_model as M
from tests.test_radix import ct, ints
from tests.test_radix_find import cleartext_key, run_oracle_shared

SEP_ENC, SEP_RRD = b"TFHE_Enc", b"TFHE_Rrd"
KS = S.BitonicShuffleKeySize


def one(v, n, signed=False):
    return ct([v], n, signed)


def lst(values, n, signed=False):
    return [one(v, n, signed) for v in values]


def values_of(cts, signed=False):
    return [ints(c, signed)[0] for c in cts]


# ---------------------------------------------------------------------------
# the network
# ---------------------------------------------------------------------------
def test_network_matches_the_reference_table():
    assert SM.network(8) == SM.NETWORK_8
    assert [list(s) for s in S.network(8)] == SM.NETWORK_8
    for n in (2, 4, 16, 64, 1024):
        stages = S.network(n)
        log_n = n.bit_length() - 1
        assert len(stages) == log_n * (log_n + 1) // 2
        assert [list(s) for s in stages] == SM.network(n)
        for s in stages:   # every element once per stage
            assert sorted(x for i, j, _ in s for x in (i, j)) == list(range(n))
    for bad in (0, 1, 3, 12):
        with pytest.raises(ValueError):
            S.network(bad)


@pytest.mark.parametrize("n", [2, 4, 8, 16])
def test_network_sorts_every_0_1_input(n):
    """the 0-1 principle: a comparator network that sorts all 2^n inputs of
    0s and 1s sorts every input"""
    x = (np.arange(2 ** n)[:, None] >> np.arange(n)[None, :]) & 1
    for stage in S.network(n):
        for i, j, asc in stage:
            lo, hi = np.minimum(x[:, i], x[:, j]), np.maximum(x[:, i], x[:, j])
            x[:, i], x[:, j] = (lo, hi) if asc else (hi, lo)
    assert np.all(np.diff(x, axis=1) >= 0)


# ---------------------------------------------------------------------------
# the key size
# ---------------------------------------------------------------------------
def test_key_size_blocks():
    for length in (0, 1, 2, 3, 8, 13, 52, 64, 256, 1024, 10 ** 6):
        for p in (2.0 ** -80, 2.0 ** -40, 1e-9, 0.01, 0.25, 0.5, 0.75, 0.999999, 1 - 2 ** -52):
            assert KS.collision_probability(p).num_blocks(length) == SM.key_blocks_for_probability(length, p), \
                (length, p)
    # hand-worked: 1024^2 / 2^-39 = 2^59 -> 30 blocks; 52^2 / 2^-39 -> 51 bits, 26 blocks
    assert KS.collision_probability(2.0 ** -40).num_blocks(1024) == 30
    assert KS.collision_probability(2.0 ** -40).num_blocks(52) == 26
    # the empty list (log2(0) = -inf) and p close to 1 at one element: 0 blocks
    assert KS.collision_probability(0.5).num_blocks(0) == 0
    assert KS.collision_probability(0.9).num_blocks(1) == 0
    assert KS.collision_probability(0.4).num_blocks(1) == 1
    assert [KS.num_bits(b).num_blocks(100) for b in (0, 1, 2, 3, 8, 63, 64)] == [0, 1, 1, 2, 4, 32, 32]
    for p in (0, 1, 0.0, 1.0, -0.5, 2, float("nan"), float("inf"), "0.5", None, True):
        with pytest.raises(ValueError):
            KS.collision_probability(p)
    for b in (-1, 2 ** 32, 1.5, None, True):
        with pytest.raises(ValueError):
            KS.num_bits(b)


# ---------------------------------------------------------------------------
# the compare-and-swap schedule
# ---------------------------------------------------------------------------
def swap_model(ki, kj, di, dj, asc):
    swap = ki > kj if asc else ki <= kj
    return (kj, ki, dj, di) if swap else (ki, kj, di, dj)


def run_pairs(nk, nd, pairs, signed=False):
    """pairs of (k_i, k_j, d_i, d_j, ascending) on the cleartext executor:
    the outputs as (k_i', k_j', d_i', d_j')"""
    s = bc.schedule(S.circuit(nk, nd), len(pairs))
    ins = np.array([R.to_digits(ki, nk) + R.to_digits(di, nd) + R.to_digits(kj, nk) + R.to_digits(dj, nd)
                    for ki, kj, di, dj, _ in pairs], dtype=np.int64)
    desc = np.array([[0 if asc else 1] for *_, asc in pairs], dtype=np.int64)
    out = bc.run_cleartext(s, [], ins, desc)
    assert out.min() >= 0 and out.max() <= bc.MAX_BLOCK_VALUE
    E = nk + nd
    return [(R.from_digits(o[:nk]), R.from_digits(o[E:E + nk]), R.from_digits(o[nk:E], signed),
             R.from_digits(o[E + nk:], signed)) for o in out]


@pytest.mark.parametrize("nk", [1, 2])
def test_compare_and_swap_exhaustive_over_keys(nk):
    rng = np.random.default_rng(nk)
    dom = range(4 ** nk)
    pairs = [(ki, kj, int(rng.integers(0, 16)), int(rng.integers(0, 16)), asc)
             for ki in dom for kj in dom for asc in (True, False)]
    assert run_pairs(nk, 2, pairs) == [swap_model(*p) for p in pairs]


@pytest.mark.parametrize("signed", [False, True])
def test_compare_and_swap_fheuint64_data(signed):
    rng = np.random.default_rng(64 + signed)
    lo, hi = R.scalar_range(32, signed)
    pairs = []
    for asc in (True, False):
        for _ in range(20):
            ki = int(rng.integers(0, 2 ** 32, dtype=np.uint64))
            kj = ki if rng.random() < 0.3 else int(rng.integers(0, 2 ** 32, dtype=np.uint64))
            di, dj = (int(v) for v in rng.integers(lo, hi, 2, dtype=np.int64 if signed else np.uint64))
            pairs.append((ki, kj, di, dj, asc))
    assert run_pairs(16, 32, pairs, signed) == [swap_model(*p) for p in pairs]


def test_every_output_is_a_stored_pbs_output():
    """outputs are PBS rows (level 1, value <= 3): no input passes through"""
    for nk, nd in ((1, 1), (3, 5), (17, 32)):
        c = S.circuit(nk, nd)
        assert len(c.outputs) == 2 * (nk + nd)
        assert all(c.gates[w][0] == "lut" and c.vmax[w] <= bc.MAX_BLOCK_VALUE for w in c.outputs)
        s = bc.schedule(c, 1)
        last = set(s.row_dest[int(s.layer_rows[-2]):].tolist())
        assert set(s.output_slots.tolist()) <= set(s.row_dest.tolist())
        assert last <= set(s.output_slots.tolist())


# (PBS per stage, PBS layers per stage, stages) of an FheUint64 shuffle:
# 2K - 1 compare + 4 (K + D) swap PBS per pair, K with the padding block
PINNED = {
    (2, 1, 32): (1 * (1 + 4 * 33), 3, 1),
    (8, 1, 32): (4 * (1 + 4 * 33), 3, 6),
    (8, 4, 32): (4 * (7 + 4 * 36), 5, 6),
    (52, 26, 32): (32 * (53 + 4 * 59), 8, 21),
    (64, 4, 32): (32 * (7 + 4 * 36), 5, 21),
    (64, 27, 32): (32 * (53 + 4 * 59), 8, 21),
    (1024, 30, 32): (512 * (59 + 4 * 62), 8, 55),
    (13, 1, 1): (8 * (3 + 4 * 3), 4, 10),
}


def test_pinned_counts():
    got = {k: S.cost(*k) for k in PINNED}
    assert got == PINNED, got
    assert S.cost(1, 4, 32) == S.cost(0, 4, 32) == (0, 0, 0)


def test_circuit_cache_is_bounded():
    assert S._circuit.cache_info().maxsize == R.CIRCUIT_CACHE_SIZE
    assert S.circuit(4, 32) is S.circuit(4, 32)


# ---------------------------------------------------------------------------
# whole shuffles on the cleartext runner
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("length", [2, 3, 5, 8, 13, 64])
@pytest.mark.parametrize("nk", [1, 3])
def test_shuffle_with_keys_equals_the_model(length, nk):
    key = cleartext_key()
    rng = np.random.default_rng(zlib.crc32(f"shuffle{length}_{nk}".encode()))
    for signed, nd in ((False, 2), (True, 3)):
        lo, hi = R.scalar_range(nd, signed)
        data = [int(v) for v in rng.integers(lo, hi, length)]
        for keys in ([int(v) for v in rng.integers(0, 4 ** nk, length)],      # ties at nk = 1
                     [4 ** nk - 1] * length, [0] * length,                    # all equal, at both ends
                     list(range(length)), list(range(length))[::-1]):
            keys = [k % 4 ** nk for k in keys]
            before = key.runner.calls
            out = key.bitonic_shuffle_with_keys(lst(data, nd, signed), lst(keys, nk))
            assert all(type(o) is type(one(0, nd, signed)) and o.num_inputs == 1 for o in out)
            assert values_of(out, signed) == SM.shuffle(data, keys, nk), (data, keys)
            n = 1 << (length - 1).bit_length()
            log_n = n.bit_length() - 1
            assert key.runner.calls - before == log_n * (log_n + 1) // 2


def test_shuffle_ties_follow_the_asymmetric_rule():
    """equal keys: the ascending pair keeps its order, the descending one swaps"""
    assert SM.shuffle([10, 20], [1, 1], 1) == [10, 20]
    key = cleartext_key()
    assert values_of(key.bitonic_shuffle_with_keys(lst([10, 20], 5), lst([1, 1], 1))) == [10, 20]
    # n = 4, all equal: (0, 1) asc, (2, 3) desc -> 10 20 40 30; then (0, 2) (1, 3) asc, ...
    got = values_of(key.bitonic_shuffle_with_keys(lst([10, 20, 30, 40], 5), lst([2, 2, 2, 2], 1)))
    assert got == SM.shuffle([10, 20, 30, 40], [2, 2, 2, 2], 1) and got != [10, 20, 30, 40]


def test_short_lists_come_back_unchanged():
    key = cleartext_key()
    x = one(7, 2)
    assert key.bitonic_shuffle_with_keys([], []) == []
    assert key.bitonic_shuffle_with_keys([x], [one(1, 1)]) == [x]
    assert key.bitonic_shuffle(_FakeOprf(), [x], KS.num_bits(8), 1) == [x]
    assert key.bitonic_shuffle(_FakeOprf(), [], KS.num_bits(8), 1) == []
    assert key.runner.calls == 0


# ---------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------
class _FakeOprf:
    """an OPRF key that fails if it is ever asked for sort keys"""

    def __new__(cls):
        from tfhe_rs_b200 import oprf

        k = oprf.CudaOprfServerKey.__new__(oprf.CudaOprfServerKey)
        k.message_bits, k.streams = 2, None
        k.generate_oblivious_pseudo_random_bits_chunks = _no_gpu
        k.generate_oblivious_pseudo_random_bits_chunks_and_re_randomize = _no_gpu
        return k


def _no_gpu(*args, **kwargs):
    raise AssertionError("GPU work before the argument checks")


def test_argument_checks_raise_before_any_call():
    from tfhe_rs_b200 import rerand

    key = cleartext_key()
    ok = KS.num_bits(8)
    rr_key = rerand.CudaReRandomizationKey.__new__(rerand.CudaReRandomizationKey)
    ctx = rerand.ReRandomizationContext(SEP_RRD, SEP_ENC)
    u2, u3, s2 = lst([1, 2], 2), lst([1, 2], 3), lst([1, 2], 2, True)
    two = ct([1, 2], 2)
    o = _FakeOprf()
    bad = [
        lambda: key.bitonic_shuffle(o, [u2[0], u3[0]], ok, 1),                 # block counts
        lambda: key.bitonic_shuffle(o, [u2[0], s2[0]], ok, 1),                 # kinds
        lambda: key.bitonic_shuffle(o, [two, two], ok, 1),                     # num_inputs
        lambda: key.bitonic_shuffle(o, u2, KS.num_bits(0), 1),                 # 0 key blocks
        lambda: key.bitonic_shuffle(o, [u2[0]], KS.num_bits(0), 1),            # ... before the len <= 1 return
        lambda: key.bitonic_shuffle(o, [], KS.collision_probability(0.5), 1),  # log2(0)
        lambda: key.bitonic_shuffle(o, [u2[0]], KS.collision_probability(0.9), 1),
        lambda: key.bitonic_shuffle(o, u2, 8, 1),                              # not a key size
        lambda: key.bitonic_shuffle("oprf", u2, ok, 1),
        lambda: key.bitonic_shuffle(o, u2, KS.num_bits(130), 1),               # 65 blocks
        lambda: key.bitonic_shuffle_and_re_randomize(o, u2, ok, 1, "key", ctx),
        lambda: key.bitonic_shuffle_and_re_randomize(o, u2, ok, 1, rr_key, "ctx"),
        lambda: key.bitonic_shuffle_and_re_randomize(o, u2, KS.num_bits(0), 1, rr_key, ctx),
        lambda: key.bitonic_shuffle_with_keys(u2, lst([1], 1)),                # lengths
        lambda: key.bitonic_shuffle_with_keys(u2, lst([1, 2], 1, True)),       # signed keys
        lambda: key.bitonic_shuffle_with_keys(u2, [one(1, 1), one(1, 2)]),     # key block counts
        lambda: key.bitonic_shuffle_with_keys([u2[0], u3[0]], lst([1, 2], 1)),
        lambda: key.bitonic_shuffle_with_keys(u2, [two, two]),
        lambda: key.bitonic_shuffle_with_keys(u2 + u2[:1], lst([1, 2, 3], 64)),  # 64 + 1 blocks
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert key.runner.calls == 0


def test_a_non_2_2_key_is_rejected_before_any_call():
    class _SKey:
        message_modulus, carry_modulus = 8, 8

    class _Engine:
        skey = _SKey()

    key = integer.CudaRadixServerKey.__new__(integer.CudaRadixServerKey)
    key.engine = _Engine()
    u2 = lst([1, 2], 2)
    for f in (lambda: key.bitonic_shuffle_with_keys(u2, lst([1, 2], 1)),
              lambda: key.bitonic_shuffle(_FakeOprf(), u2, KS.num_bits(8), 1)):
        with pytest.raises(ValueError, match="2_2"):
            f()
    assert key._runner is None


# ---------------------------------------------------------------------------
# the re-randomization seed of the sort keys
# ---------------------------------------------------------------------------
def test_prf_rerand_seed_is_the_shake256_composition():
    from tfhe_rs_b200 import oprf, rerand

    ctx = rerand.ReRandomizationContext(SEP_RRD, SEP_ENC)
    ctx.add_bytes(b"shuffle context")
    rle = oprf.rle_bytes([16] * 5, 2, 5)
    for seed, seed_bytes in ((0xC0FFEE, (0xC0FFEE).to_bytes(16, "little")), (b"any bytes", b"any bytes")):
        got = rerand.new_prf_rerand_seed(ctx, seed, rle)
        h = hashlib.shake_256(SEP_RRD + b"shuffle context" + seed_bytes + rle + (0).to_bytes(8, "little"))
        assert got.data == SEP_ENC + h.digest(32)
        assert rerand.new_prf_rerand_seed(ctx, seed, rle).data == got.data   # the context is unchanged
    # the copy is independent of the context it was taken from
    cp = ctx.copy()
    cp.add_bytes(b"more")
    assert ctx.finalize().next_seed().data == SEP_ENC + hashlib.shake_256(
        SEP_RRD + b"shuffle context" + (0).to_bytes(8, "little")).digest(32)
    assert cp.finalize().next_seed().data != ctx.finalize().next_seed().data
    assert rerand.new_prf_rerand_seed(ctx, 1, oprf.rle_bytes([16] * 5, 2, 5)).data != \
        rerand.new_prf_rerand_seed(ctx, 1, oprf.rle_bytes([16] * 4, 2, 5)).data
    with pytest.raises(ValueError):
        rerand.new_prf_rerand_seed("ctx", 1, rle)


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def test_one_pair_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy 2_2
    parameters of test_radix: equal keys in both directions, and unequal
    keys, 2-block keys and data"""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=62)
    rng = oracle.Rng(0x5AFF)
    pairs = [(9, 9, 3, 12, True), (9, 9, 3, 12, False), (14, 2, 5, 7, True), (14, 2, 5, 7, False)]
    s = bc.schedule(S.circuit(2, 2), len(pairs))
    digits = [d for ki, kj, di, dj, _ in pairs
              for d in R.to_digits(ki, 2) + R.to_digits(di, 2) + R.to_digits(kj, 2) + R.to_digits(dj, 2)]
    inst = M.encrypt_bits(oracle, keys, rng, digits)
    desc = np.array([[0 if p[4] else 1] for p in pairs], dtype=np.int64)
    out = run_oracle_shared(oracle, keys, s, np.zeros((0, P.big_n + 1), np.uint64), inst, desc)
    got = M.decrypt_messages(oracle, keys, out, vmax=3).reshape(len(pairs), 8)
    for g, p in zip(got, pairs):
        assert (R.from_digits(g[0:2]), R.from_digits(g[4:6]), R.from_digits(g[2:4]), R.from_digits(g[6:8])) == \
            swap_model(*p), p


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
B = 17   # TUniform bound of the P22 compact public keys (tests/test_rerand.py)


@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_shuffle(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, oprf, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0x5F00 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    rk = integer.CudaRadixServerKey(skey, glwe_dimension=P.k, polynomial_size=P.N)
    okey = oprf.CudaOprfServerKey(skey.bsk, streams)
    rng = oracle.Rng(0x5F02)

    def enc_list(values, n, signed=False):
        digits = [d for v in values for d in R.to_digits(int(v), n)]
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, digits).view(np.int64)).to(streams.device(0))
        kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
        return [kind(t[i * n:(i + 1) * n], 1) for i in range(len(values))]

    def dec(x, signed=False):
        d = M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64), vmax=3)
        return R.from_digits(d, signed)

    yield type("G", (), dict(rk=rk, okey=okey, keys=keys, P=P, streams=streams, enc_list=enc_list, dec=dec,
                             oracle=oracle))
    rk.runner.close()


def oprf_sort_keys(G, seed, length, nk):
    """the sort keys the OPRF draws for `seed`: tests/test_oprf.py's exact model"""
    from tests.test_oprf import _model
    from tfhe_rs_b200 import oprf

    _, bits, msgs = _model(oprf, seed, [2 * nk] * length, G.keys.lwe_sk, G.P.N)
    assert bits == [2] * (length * nk)
    return [R.from_digits(msgs[e * nk:(e + 1) * nk]) for e in range(length)]


def data_values(length, signed, tag):
    rng = np.random.default_rng(zlib.crc32(tag.encode()))
    lo, hi = R.scalar_range(32, signed)
    return [int(v) for v in rng.integers(lo, hi, length, dtype=np.int64 if signed else np.uint64)]


@pytest.mark.gpu
@pytest.mark.parametrize("nk,signed", [(1, False), (1, True), (16, False), (16, True)])
def test_gpu_shuffle_with_keys(gpu_shuffle, nk, signed):
    G = gpu_shuffle
    rng = np.random.default_rng(nk + 2 * signed)
    for length in (2, 3, 8, 13, 64):
        data = data_values(length, signed, f"with_keys{nk}{signed}{length}")
        keys = [int(v) for v in rng.integers(0, 4 ** nk, length, dtype=np.uint64)]
        out = G.rk.bitonic_shuffle_with_keys(G.enc_list(data, 32, signed), G.enc_list(keys, nk))
        assert [G.dec(o, signed) for o in out] == SM.shuffle(data, keys, nk), (length, keys)


@pytest.mark.gpu
def test_gpu_bitonic_shuffle_is_the_oprf_permutation(gpu_shuffle):
    G = gpu_shuffle
    data = data_values(13, False, "oprf13")
    cts = G.enc_list(data, 32)
    size = KS.collision_probability(2.0 ** -40)
    nk = size.num_blocks(13)
    assert nk == 24
    want = SM.shuffle(data, oprf_sort_keys(G, 0x5EED, 13, nk), nk)
    assert sorted(want) == sorted(data)
    out = G.rk.bitonic_shuffle(G.okey, cts, size, 0x5EED)
    assert [G.dec(o) for o in out] == want
    assert [G.dec(o) for o in G.rk.bitonic_shuffle(G.okey, cts, size, 0x5EED)] == want
    # two seeds at 16 elements: two permutations, each the model's
    data16 = list(range(100, 116))
    cts16 = G.enc_list(data16, 32)
    perms = []
    for seed in (1, 2):
        got = [G.dec(o) for o in G.rk.bitonic_shuffle(G.okey, cts16, KS.num_bits(8), seed)]
        assert got == SM.shuffle(data16, oprf_sort_keys(G, seed, 16, 4), 4)
        perms.append(got)
    assert perms[0] != perms[1]


@pytest.mark.gpu
def test_gpu_re_randomized_keys(gpu_shuffle):
    from tests import compact_pke as CP
    from tests import rerand_model as RM
    from tfhe_rs_b200 import oprf, rerand

    G = gpu_shuffle
    pk = CP.compact_pk_gen(np.random.default_rng(0x5F5F), G.keys.glwe_sk, B)
    cpk = rerand.CudaCompactPublicKey.from_compact_public_key(pk[0], pk[1], B, G.streams)
    rr_key = rerand.CudaReRandomizationKey.derived(cpk)
    ctx = rerand.ReRandomizationContext(SEP_RRD, SEP_ENC)
    ctx.add_bytes(b"test_radix_shuffle")
    data = data_values(8, True, "rerand8")
    cts = G.enc_list(data, 32, True)
    size = KS.num_bits(6)
    plain = [G.dec(o, True) for o in G.rk.bitonic_shuffle(G.okey, cts, size, 77)]
    got = [G.dec(o, True) for o in G.rk.bitonic_shuffle_and_re_randomize(G.okey, cts, size, 77, rr_key, ctx)]
    assert got == plain == SM.shuffle(data, oprf_sort_keys(G, 77, 8, 3), 3)
    # the re-randomized key words: the plain OPRF words plus one list of zeros
    # drawn from SHAKE256(context || seed || RLE || index 0)
    chunks = [6] * 8
    words = lambda cs: np.concatenate([c.d_vec.t.cpu().numpy().view(np.uint64) for c in cs]).reshape(  # noqa: E731
        -1, G.P.k * G.P.N + 1)
    base = words(G.okey.generate_oblivious_pseudo_random_bits_chunks(77, chunks))
    rr = words(G.okey.generate_oblivious_pseudo_random_bits_chunks_and_re_randomize(77, chunks, rr_key, ctx))
    seed = SEP_ENC + hashlib.shake_256(SEP_RRD + b"test_radix_shuffle" + (77).to_bytes(16, "little")
                                       + oprf.rle_bytes(chunks, 2, 5) + (0).to_bytes(8, "little")).digest(32)
    assert np.array_equal(rr, RM.rerand_without_keyswitch(base, pk, seed, B))
    assert not np.array_equal(rr, base)


@pytest.mark.gpu
def test_gpu_shuffled_outputs_feed_add_and_gt(gpu_shuffle):
    """shuffled blocks are clean PBS outputs: into add and gt"""
    G = gpu_shuffle
    data = [5, 17, 40, 2 ** 63, 8]
    out = G.rk.bitonic_shuffle(G.okey, G.enc_list(data, 32), KS.num_bits(16), 9)
    vals = [G.dec(o) for o in out]
    assert sorted(vals) == sorted(data)
    s = G.rk.add(out[0], out[1])
    assert G.dec(s) == (vals[0] + vals[1]) % 2 ** 64
    gt = G.rk.gt(out[2], out[3])
    assert int(M.decrypt_messages(G.oracle, G.keys, gt.blocks.cpu().numpy().view(np.uint64))[0]) == \
        int(vals[2] > vals[3])
