"""Vector find and compare on radix integers (tfhe-rs_b200/radix_find.py and
the matching methods of integer.CudaRadixServerKey).

CPU: every operation through the server key's host code on a cleartext runner
(the per-candidate schedules and the cross-candidate trees on
`bit_circuit.run_cleartext`, which asserts the noise budget and the value
range on every row), exhaustively over the query at 1 and 2 blocks, unsigned
and signed where tfhe-rs allows it, on lists of length 0 to 6 with and
without duplicates, against `tests/find_model.py`; pinned PBS and layer
counts at FheUint64; argument checks; `first_index_of` through real LWE
keyswitches and PBS on the oracle.

GPU: every method at FheUint64 on classic P22 and multi-bit g = 4, found and
not found, signed where allowed, and a result chained into add and gt."""
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import bit_circuit as bc, integer, radix as R, radix_find as F

from tests import find_model as FM
from tests import trivium_model as M
from tests.test_radix import bools, ct, ints
from tests.test_trivium import CleartextRunner, run_oracle


class FindCleartextRunner(CleartextRunner):
    """the cleartext runner with the table-built trees and trivial blocks"""

    def run_schedule(self, key, sched, instance):
        import torch

        self.calls += 1
        out = bc.run_cleartext(sched, [], instance[:, 0].numpy().reshape(1, -1))
        return torch.from_numpy(out.reshape(-1, 1).astype(np.int64))

    def trivial(self, digits):
        import torch

        return torch.tensor([[int(d)] for d in digits], dtype=torch.int64)


def cleartext_key():
    k = integer.CudaRadixServerKey.__new__(integer.CudaRadixServerKey)
    k._runner = FindCleartextRunner()
    return k


def one(v, n, signed=False):
    return ct([v], n, signed)


def lst(values, n, signed=False):
    return [one(v, n, signed) for v in values]


def radix_of(x, signed=False):
    """(value, num_blocks) of a single-integer cleartext result"""
    return ints(x, signed)[0], x.num_blocks


def flag(b):
    return bools(b)[0]


def domain(n, signed):
    lo, hi = R.scalar_range(n, signed)
    return list(range(lo, hi))


def lists(n, signed, seed):
    """per length 0..6: a list without duplicates (when the domain allows)
    and one with"""
    rng = np.random.default_rng(seed)
    dom = domain(n, signed)
    out = [[]]
    for L in range(1, 7):
        if L <= len(dom):
            out.append([dom[int(i)] for i in rng.permutation(len(dom))[:L]])
        if L >= 2:
            v = [dom[int(i)] for i in rng.integers(0, len(dom), L)]
            v[-1] = v[0]   # the first value repeated at the end
            out.append(v)
    return out


def queries(values, n, signed):
    """every value at 1 block; at 2 the list's values and absent ones"""
    dom = domain(n, signed)
    if n == 1:
        return dom
    absent = [v for v in dom if v not in values][:3]
    return sorted(set(values)) + absent


# ---------------------------------------------------------------------------
# the plain model
# ---------------------------------------------------------------------------
def test_model():
    assert [FM.num_blocks_for(v) for v in (0, 1, 3, 4, 15, 16, 2 ** 64 - 1)] == [1, 1, 1, 2, 2, 3, 32]
    assert FM.match_value(5, []) == ((0, 1), 0)
    assert FM.match_value(5, [(5, 0), (6, 0)]) == ((0, 1), 1)
    assert FM.match_value(6, [(5, 300), (6, 17)]) == ((17, 5), 1)
    assert FM.match_value_or(7, [(5, 3)], 70) == (70, 4) and FM.match_value_or(7, [], 70) == (70, 4)
    assert FM.index_in_clears(3, [], 4) == ((0, 4), 0)
    # duplicates: digit-wise sums mod 4 of the matching indices (1 + 2 = 3, 1 + 3 = 4 -> 0)
    assert FM.index_in_clears(9, [1, 9, 9, 2], 2) == ((3, 1), 1)
    assert FM.index_in_clears(9, [1, 9, 2, 9], 2) == ((0, 1), 1)
    assert FM.first_index_in_clears(9, [9, 9, 1, 1, 1, 1, 2], 2) == ((0, 2), 1)
    assert FM.first_index_in_clears(2, [9, 9, 2, 2], 2) == ((2, 1), 1)
    assert FM.first_index_of([4, 9, 9], 9, 3) == ((1, 1), 1) and FM.first_index_of([], 9, 3) == ((0, 3), 0)
    assert FM.all_eq_slices([], []) == 1 and FM.all_eq_slices([1], []) == 0
    assert FM.contains_sub_slice([1, 2, 3], [2, 3]) == 1 and FM.contains_sub_slice([1], [1, 1]) == 0


# ---------------------------------------------------------------------------
# exhaustive at 1 and 2 blocks
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_searches(n, signed):
    key = cleartext_key()
    for values in lists(n, signed, zlib.crc32(f"find{n}{signed}".encode())):
        cts = lst(values, n, signed)
        for x in queries(values, n, signed):
            q = one(x, n, signed)
            assert flag(key.contains(cts, q)) == FM.contains(values, x)
            assert flag(key.contains_clear(cts, x)) == FM.contains(values, x)
            assert flag(key.is_in_clears(q, values)) == FM.is_in_clears(x, values)
            for name, got, want in (
                    ("index_in_clears", key.index_in_clears(q, values), FM.index_in_clears(x, values, n)),
                    ("first_index_in_clears", key.first_index_in_clears(q, values),
                     FM.first_index_in_clears(x, values, n)),
                    ("index_of", key.index_of(cts, q), FM.index_of(values, x, n)),
                    ("index_of_clear", key.index_of_clear(cts, x), FM.index_of(values, x, 1)),
                    ("first_index_of", key.first_index_of(cts, q), FM.first_index_of(values, x, n)),
                    ("first_index_of_clear", key.first_index_of_clear(cts, x), FM.first_index_of(values, x, 1))):
                assert type(got[0]) is integer.CudaUnsignedRadixCiphertext
                assert (radix_of(got[0]), flag(got[1])) == want, (name, values, x)


@pytest.mark.parametrize("n", [1, 2])
def test_exhaustive_match_value(n):
    """unsigned only, as tfhe-rs types it: tables of 0 to 6 unique inputs,
    outputs of 1 to 5 blocks, a zero-only table, and every or_value width"""
    key = cleartext_key()
    rng = np.random.default_rng(zlib.crc32(f"match{n}".encode()))
    dom = domain(n, False)
    for L in range(0, 7):
        ins = [dom[int(i)] for i in rng.permutation(len(dom))[:min(L, len(dom))]]
        for outs in ([int(rng.integers(0, 4)) for _ in ins], [int(rng.integers(0, 1 << 20)) for _ in ins],
                     [0] * len(ins)):
            matches = list(zip(ins, outs))
            for x in dom:
                q = one(x, n)
                v, found = key.match_value(q, matches)
                assert (radix_of(v), flag(found)) == FM.match_value(x, matches), (matches, x)
                for or_value in (0, 5, 1 << 30):
                    got = key.match_value_or(q, matches, or_value)
                    assert radix_of(got) == FM.match_value_or(x, matches, or_value), (matches, x, or_value)


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_slices(n, signed):
    key = cleartext_key()
    dom = domain(n, signed)
    rng = np.random.default_rng(zlib.crc32(f"slices{n}{signed}".encode()))
    for L in range(0, 5):
        for _ in range(3):
            a = [dom[int(i)] for i in rng.integers(0, len(dom), L)]
            for b in (list(a), [dom[int(i)] for i in rng.integers(0, len(dom), L)], a[:-1],
                      a[:-1] + [dom[(dom.index(a[-1]) + 1) % len(dom)]] if a else [dom[0]]):
                assert flag(key.all_eq_slices(lst(a, n, signed), lst(b, n, signed))) == FM.all_eq_slices(a, b)
    for L in range(0, 7):
        a = [dom[int(i)] for i in rng.integers(0, min(len(dom), 3), L)]
        for P in range(1, 4):
            for p in ([a[i:i + P] for i in range(L - P + 1)][:2]
                      + [[dom[int(i)] for i in rng.integers(0, min(len(dom), 3), P)] for _ in range(2)]):
                got = flag(key.contains_sub_slice(lst(a, n, signed), lst(p, n, signed)))
                assert got == FM.contains_sub_slice(a, p), (a, p)
    # a pair of different block counts is unequal, as tfhe-rs has it
    assert flag(key.all_eq_slices([one(1, 1)], [one(1, 2)])) == 0


def test_wide_operands():
    """FheUint64 searches and a 100-entry list: the trees at several levels"""
    key = cleartext_key()
    n = 32
    rng = np.random.default_rng(7)
    values = [int(v) for v in rng.integers(0, 2 ** 63, 100, dtype=np.uint64)]
    values[60] = values[17]
    cts = lst(values, n)
    for x in (values[0], values[17], values[99], 12345):
        q = one(x, n)
        assert flag(key.contains(cts, q)) == FM.contains(values, x)
        assert (radix_of(key.first_index_of(cts, q)[0]), flag(key.first_index_of(cts, q)[1])) == \
            FM.first_index_of(values, x, n)
        got = key.index_in_clears(q, values)
        assert (radix_of(got[0]), flag(got[1])) == FM.index_in_clears(x, values, n)
    matches = [(v, (v * 7919) % (1 << 64)) for v in sorted(set(values))[:16]]
    for x in (matches[3][0], 5):
        v, found = key.match_value(one(x, n), matches)
        assert (radix_of(v), flag(found)) == FM.match_value(x, matches)


# ---------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------
# (PBS, PBS layers) of one FheUint64 call, the per-candidate call then the
# tree; recorded in DESIGN §8o
PINNED = {
    ("kv_store_get", 1): (74, 5), ("kv_store_get", 2): (181, 6),
    ("kv_store_get", 64): (5297, 8), ("kv_store_get", 1024): (84257, 10),
    ("kv_store_update", 1): (138, 6), ("kv_store_update", 2): (277, 7),
    ("kv_store_update", 64): (8849, 9), ("kv_store_update", 1024): (141569, 11),
    ("match_value", 16): (1294, 7), ("contains", 64): (2705, 7),
}


def test_pinned_counts():
    got = {(op, M): F.cost(op, M, 32, 32) for op, M in PINNED}
    assert got == PINNED, got


def test_layers_grow_with_log_m():
    for op in ("kv_store_get", "kv_store_update"):
        assert F.cost(op, 1024, 32, 32)[1] - F.cost(op, 64, 32, 32)[1] <= 3
    assert F.cost("contains", 1024, 32)[1] - F.cost("contains", 64, 32)[1] <= 3
    # the first-match scan: ceil(log5 (M - 1)) + 1 layers
    for M, want in ((2, 1), (6, 2), (7, 3), (26, 3), (27, 4), (1024, 6)):
        args = ("dot", M, 1, F.num_blocks_for(M - 1), tuple(range(M)), 0)
        assert F.tree(*args, True).num_layers - F.tree(*args).num_layers == want, M


def test_trees_pass_the_budget_at_1024():
    """every row of the M = 1024 trees on the cleartext executor, with one
    selector set: its value comes out"""
    M, nv = 1024, 4
    for hot in (0, 517, 1023):
        sel = np.zeros((M, 1 + nv), dtype=np.int64)
        sel[:, 1:] = 0
        sel[hot] = [1, 3, 2, 1, 0]
        out = bc.run_cleartext(F.tree("select", M, 1 + nv), [], sel.reshape(1, -1))[0]
        assert list(out) == [3, 2, 1, 0, 1]
        s = np.zeros(M, dtype=np.int64)
        s[hot] = 1
        s[1000] = 1
        first = bc.run_cleartext(F.tree("dot", M, 1, 5, tuple(range(M)), 0, True), [], s.reshape(1, -1))[0]
        assert R.from_digits(first[:5]) == min(hot, 1000) and first[5] == 1


def test_circuit_cache_is_bounded():
    assert F._circuit.cache_info().maxsize == R.CIRCUIT_CACHE_SIZE
    assert F.tree.cache_info().maxsize == R.CIRCUIT_CACHE_SIZE
    assert F.circuit("select", 32, 32) is F.circuit("select", 32, 32)


# ---------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------
def test_argument_checks_raise_before_any_call():
    key = cleartext_key()
    u2, s2 = one(1, 2), one(1, 2, True)
    two = ct([1, 2], 2)
    bad = [
        lambda: key.contains(lst([1, 2], 2), one(1, 3)),           # widths
        lambda: key.contains(lst([1], 2) + lst([1], 3), u2),
        lambda: key.contains(lst([1], 2), s2),                      # signedness
        lambda: key.index_of(lst([1, 2], 2), two),                  # num_inputs
        lambda: key.is_in_clears(two, [1]),
        lambda: key.contains([two], u2),
        lambda: key.is_in_clears(u2, [16]),                         # clears that do not fit
        lambda: key.is_in_clears(s2, [8]),
        lambda: key.index_in_clears(u2, [-1]),
        lambda: key.contains_clear(lst([1], 2), 16),
        lambda: key.first_index_of_clear(lst([1], 2, True), -9),
        lambda: key.match_value(u2, [(1, 2), (1, 3)]),              # duplicate inputs
        lambda: key.match_value(u2, [(16, 2)]),
        lambda: key.match_value(s2, [(1, 2)]),                      # unsigned only
        lambda: key.match_value(u2, [(1, -2)]),
        lambda: key.match_value_or(u2, [(1, 2)], -1),
        lambda: key.all_eq_slices(lst([1], 2), lst([1], 2, True)),
        lambda: key.contains_sub_slice(lst([1], 2), []),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert key.runner.calls == 0


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def test_first_index_of_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_radix: first_index_of over 5 encrypted 2-block
    candidates (the query twice in the list), the per-candidate schedule and
    the tree each on the oracle."""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=61)
    rng = oracle.Rng(0xF1D0)
    n, values = 2, [3, 9, 14, 9, 0]
    for x in (9, 5):
        digits = [d for v in values for d in R.to_digits(v, n)]
        s = bc.schedule(F.circuit("eq", n), len(values))
        query = M.encrypt_bits(oracle, keys, rng, R.to_digits(x, n))
        inst = M.encrypt_bits(oracle, keys, rng, digits)
        sels = run_oracle_shared(oracle, keys, s, query, inst)
        t = F.tree("dot", len(values), 1, 2, tuple(range(len(values))), 0, True)
        out = M.decrypt_messages(oracle, keys, run_oracle(oracle, keys, t, sels), vmax=3)
        want, found = FM.first_index_of(values, x, n)
        assert (R.from_digits(out[:2]), 2, int(out[2])) == want + (found,)


def run_oracle_shared(oracle, keys, sched, shared_blocks, instance_blocks, iconst_bits=None):
    """`run_oracle` for a schedule with shared inputs: the shared slots
    filled, then the same layers"""
    P = keys.params
    luts = np.stack([oracle.make_lut(P, f) for f in sched.lut_tables()])
    pool = np.zeros((sched.pool_rows, P.big_n + 1), dtype=np.uint64)
    I = sched.num_instances
    pool[sched.addr(sched.shared_input_slots, 0)] = shared_blocks
    pool[sched.addr(sched.instance_input_slots[None, :], np.arange(I)[:, None]).reshape(-1)] = instance_blocks
    body = sched.body(iconst_bits)
    lut_rows, dests = sched.gpu_tables()
    o = 0
    for L in range(sched.num_layers):
        r0, r1 = int(sched.layer_rows[L]), int(sched.layer_rows[L + 1])
        sh = int(sched.layer_shared_rows[L])
        staged = []
        for r in range(r0, r1):
            t0, t1 = int(sched.row_offsets[r]), int(sched.row_offsets[r + 1])
            for i in ([0] if r - r0 < sh else range(I)):
                acc = np.zeros(P.big_n + 1, dtype=np.uint64)
                with np.errstate(over="ignore"):
                    acc[-1] = np.uint64(int(body[r, i]) * P.delta % 2 ** 64)
                    for t in range(t0, t1):
                        acc += np.uint64(int(sched.term_coefs[t]) % 2 ** 64) * pool[sched.addr(int(sched.term_slots[t]), i)]
                staged.append(acc)
        small = oracle.keyswitch_batch(keys, np.stack(staged))
        pool[dests[o:o + len(staged)].astype(np.int64)] = oracle.pbs_batch(keys, luts, small,
                                                                           lut_idx=lut_rows[o:o + len(staged)])
        o += len(staged)
    return pool[sched.output_rows()]


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_find(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0xF100 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    rk = integer.CudaRadixServerKey(skey, glwe_dimension=P.k, polynomial_size=P.N)
    rng = oracle.Rng(0xF102)

    def enc_list(values, n, signed=False):
        """one single-integer ciphertext per value (one encryption call)"""
        digits = [d for v in values for d in R.to_digits(int(v), n)]
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, digits).view(np.int64)).to(streams.device(0))
        kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
        return [kind(t[i * n:(i + 1) * n], 1) for i in range(len(values))]

    def enc(v, n, signed=False):
        return enc_list([v], n, signed)[0]

    def dec(x, signed=False):
        """an int, or (value, num_blocks) of a radix; copies on the caller's
        current stream, which waits for the work stream"""
        if isinstance(x, integer.CudaBooleanBlock):
            assert x.blocks.shape[0] == 1
            return int(M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64))[0])
        d = M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64), vmax=3)
        return R.from_digits(d, signed), x.num_blocks

    yield rk, enc, enc_list, dec
    rk.runner.close()


def _pair(dec, got, signed=False):
    return dec(got[0], signed), dec(got[1])


@pytest.mark.gpu
@pytest.mark.parametrize("signed", [False, True])
def test_gpu_every_search_fheuint64(gpu_find, signed):
    rk, enc, enc_list, dec = gpu_find
    n = 32
    rng = np.random.default_rng(zlib.crc32(f"gpufind{signed}".encode()))
    lo, hi = R.scalar_range(n, signed)
    values = [int(v) for v in rng.integers(lo, hi, 7, dtype=np.int64 if signed else np.uint64)]
    values[5] = values[2]   # a duplicate
    cts = enc_list(values, n, signed)
    absent = next(v for v in (0, 1, 2, 3) if v not in values)
    for x in (values[2], values[6], absent):
        q = enc(x, n, signed)
        assert dec(rk.contains(cts, q)) == FM.contains(values, x)
        assert dec(rk.contains_clear(cts, x)) == FM.contains(values, x)
        assert dec(rk.is_in_clears(q, values)) == FM.is_in_clears(x, values)
        assert _pair(dec, rk.index_in_clears(q, values)) == FM.index_in_clears(x, values, n)
        assert _pair(dec, rk.first_index_in_clears(q, values)) == FM.first_index_in_clears(x, values, n)
        assert _pair(dec, rk.index_of(cts, q)) == FM.index_of(values, x, n)
        assert _pair(dec, rk.index_of_clear(cts, x)) == FM.index_of(values, x, 1)
        assert _pair(dec, rk.first_index_of(cts, q)) == FM.first_index_of(values, x, n)
        assert _pair(dec, rk.first_index_of_clear(cts, x)) == FM.first_index_of(values, x, 1)
    assert dec(rk.all_eq_slices(cts[:3], enc_list(values[:3], n, signed))) == 1
    assert dec(rk.all_eq_slices(cts[:3], enc_list(values[:2] + [values[6]], n, signed))) == 0
    assert dec(rk.contains_sub_slice(cts, enc_list(values[4:6], n, signed))) == 1
    assert dec(rk.contains_sub_slice(cts, enc_list([values[6], values[0]], n, signed))) == \
        FM.contains_sub_slice(values, [values[6], values[0]])


@pytest.mark.gpu
def test_gpu_match_value_fheuint64(gpu_find):
    rk, enc, _, dec = gpu_find
    n = 32
    matches = [(3, 1 << 40), (2 ** 63 + 9, 77), (12, 0), (99, 2 ** 64 - 1)]
    for x in (2 ** 63 + 9, 99, 5):
        q = enc(x, n)
        v, found = rk.match_value(q, matches)
        assert (dec(v), dec(found)) == FM.match_value(x, matches), x
        assert dec(rk.match_value_or(q, matches, 1234)) == FM.match_value_or(x, matches, 1234), x


@pytest.mark.gpu
def test_gpu_index_into_add_and_gt(gpu_find):
    """an index is clean blocks: fed into add and gt"""
    rk, enc, enc_list, dec = gpu_find
    values = [5, 17, 40, 17, 8]
    (idx, found) = rk.first_index_of(enc_list(values, 32), enc(17, 32))
    assert (dec(idx), dec(found)) == ((1, 2), 1)
    two = enc(2, 2)
    assert dec(rk.add(idx, two)) == (3, 2)
    assert dec(rk.gt(idx, two)) == 0 and dec(rk.gt(two, idx)) == 1
