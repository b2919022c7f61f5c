"""Products, sums, clear-operand arithmetic, signed overflow flags and abs of
radix integers (tfhe-rs_b200/radix_mul.py, the `ARITH_OPERATIONS` of
tfhe-rs_b200/radix.py and their integer.CudaRadixServerKey methods).

CPU: every method through the server key's host code on a cleartext runner
(the compiled schedules on `bit_circuit.run_cleartext`, which asserts the
noise budget and the value range on every row): every operand pair and every
clear scalar at 1, 2 and 3 blocks, unsigned and signed; abs of every value;
sums of 1 to 7 operands at 1 and 2 blocks; edge values at 32 and 64 blocks;
against the plain models.  Also the pinned FheUint64 schedule counts, argument
checks, and 3-block mul and signed_overflowing_mul through real LWE
keyswitches and PBS on the oracle.

GPU: `CudaRadixServerKey` on classic P22 and multi-bit g = 4: every new
method at FheUint64 with 1 and 7 inputs, unsigned and signed; FheUint128
mul and unsigned_overflowing_mul; mul against unchecked_mul; a product
chained into add, gt and div_rem."""
import itertools
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import bit_circuit as bc, integer, radix as R, radix_div as D, radix_mul as RM

from tests import trivium_model as M
from tests.test_radix import bools, cleartext_key, ct, ints, rand_int, wrap
from tests.test_trivium import run_oracle


def domain(n, signed):
    lo, hi = R.scalar_range(n, signed)
    return list(range(lo, hi))


def overflowing(v, n, signed):
    lo, hi = R.scalar_range(n, signed)
    return wrap(v, n, signed), int(not lo <= v < hi)


# the clear-operand and signed-overflow methods: name -> model(a, b, n, signed)
SCALAR = {
    "scalar_add": lambda a, b, n, s: wrap(a + b, n, s),
    "scalar_sub": lambda a, b, n, s: wrap(a - b, n, s),
    "scalar_bitand": lambda a, b, n, s: wrap(a & b, n, s),
    "scalar_bitor": lambda a, b, n, s: wrap(a | b, n, s),
    "scalar_bitxor": lambda a, b, n, s: wrap(a ^ b, n, s),
    "scalar_mul": lambda a, b, n, s: RM.model("scalar_mul", (a, b), n, s),
}
UNSIGNED_SCALAR = {"unsigned_overflowing_scalar_add": lambda a, b, n, s: overflowing(a + b, n, False)}
SIGNED_SCALAR = {"signed_overflowing_scalar_add": lambda a, b, n, s: overflowing(a + b, n, True),
                 "signed_overflowing_scalar_sub": lambda a, b, n, s: overflowing(a - b, n, True)}


def results(out, signed):
    """ints, or (ints, bools) pairs for a (radix, flag) result"""
    if isinstance(out, tuple):
        return list(zip(ints(out[0], signed), bools(out[1])))
    return ints(out, signed)


def binary(key, op, a, b, n, signed):
    return results(getattr(key, op)(ct(a, n, signed), ct(b, n, signed)), signed)


def binary_ops(signed):
    """the encrypted binary methods of a signedness: name -> model"""
    ops = {"mul": lambda a, b, n: RM.model("mul", (a, b), n, signed)}
    if signed:
        ops["signed_overflowing_mul"] = lambda a, b, n: RM.model("signed_overflowing_mul", (a, b), n, True)
        ops["signed_overflowing_add"] = lambda a, b, n: overflowing(a + b, n, True)
        ops["signed_overflowing_sub"] = lambda a, b, n: overflowing(a - b, n, True)
    else:
        ops["unsigned_overflowing_mul"] = lambda a, b, n: RM.model("unsigned_overflowing_mul", (a, b), n)
    return ops


def scalar_ops(signed):
    return {**SCALAR, **(SIGNED_SCALAR if signed else UNSIGNED_SCALAR)}


# ---------------------------------------------------------------------------
# the plain model
# ---------------------------------------------------------------------------
def test_model():
    assert RM.model("mul", (7, 3), 2) == 5 and RM.model("mul", (-3, 3), 2, True) == 7
    assert RM.model("unsigned_overflowing_mul", (5, 3), 2) == (15, 0)
    assert RM.model("unsigned_overflowing_mul", (4, 4), 2) == (0, 1)
    assert RM.model("signed_overflowing_mul", (-8, 1), 2, True) == (-8, 0)
    assert RM.model("signed_overflowing_mul", (-8, -1), 2, True) == (-8, 1)
    assert RM.model("signed_overflowing_mul", (-4, 2), 2, True) == (-8, 0)
    assert RM.model("signed_overflowing_mul", (4, 2), 2, True) == (-8, 1)
    assert RM.model("sum", (), 2) is None and RM.model("sum", (15, 1, 3), 2) == 3
    assert overflowing(7 + 1, 2, True) == (-8, 1) and overflowing(-8 - 1, 2, True) == (7, 1)


# ---------------------------------------------------------------------------
# exhaustive at 1, 2 and 3 blocks
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_binary(n, signed):
    """every operand pair as instances of one call (3 blocks: 4,096 pairs)"""
    key = cleartext_key()
    vals = domain(n, signed)
    a, b = map(list, zip(*itertools.product(vals, vals)))
    for op, f in binary_ops(signed).items():
        assert binary(key, op, a, b, n, signed) == [f(x, y, n) for x, y in zip(a, b)], op


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_scalars(n, signed):
    """every value with every in-range clear scalar, one per input; and one
    scalar given once for every input"""
    key = cleartext_key()
    vals = domain(n, signed)
    a, b = map(list, zip(*itertools.product(vals, vals)))
    for op, f in scalar_ops(signed).items():
        got = results(getattr(key, op)(ct(a, n, signed), b), signed)
        assert got == [f(x, y, n, signed) for x, y in zip(a, b)], op
        for s in (vals[0], vals[-1]):
            got = results(getattr(key, op)(ct(vals, n, signed), s), signed)
            assert got == [f(x, s, n, signed) for x in vals], (op, s)


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_abs(n, signed):
    key = cleartext_key()
    vals = domain(n, signed)
    calls = key.runner.calls
    assert ints(key.abs(ct(vals, n, signed)), signed) == [wrap(abs(v), n, signed) for v in vals]
    assert key.runner.calls == calls + int(signed)   # an unsigned abs is a copy


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("count", range(1, 8))
def test_sum_ciphertexts(n, count):
    """every tuple while there are <= 4,096, else 4,096 seeded ones with the
    all-maximum and all-minimum tuples; unsigned and signed"""
    key = cleartext_key()
    rng = np.random.default_rng(zlib.crc32(f"sum{n}{count}".encode()))
    for signed in (False, True):
        vals = domain(n, signed)
        if len(vals) ** count <= 4096:
            tuples = list(itertools.product(vals, repeat=count))
        else:
            tuples = [tuple(int(v) for v in rng.choice(vals, count)) for _ in range(4094)]
            tuples += [(vals[-1],) * count, (vals[0],) * count]
        cols = [list(col) for col in zip(*tuples)]
        out = key.sum_ciphertexts([ct(col, n, signed) for col in cols])
        assert ints(out, signed) == [RM.model("sum", t, n, signed) for t in tuples]
    assert key.sum_ciphertexts([]) is None


# ---------------------------------------------------------------------------
# edge values at 32 and 64 blocks
# ---------------------------------------------------------------------------
def edge_values(n, signed, rng):
    lo, hi = R.scalar_range(n, signed)
    rand = [rand_int(rng, n, signed) for _ in range(3)]
    return sorted({0, 1, 2, 3, hi - 1, lo, wrap(-1, n, signed), 1 << (n - 1), 1 << (2 * n - 2),
                   wrap(1 << (2 * n - 1), n, signed), 1 << n} | set(rand))


def edge_pairs(n, signed, rng):
    """every pair of edge values, and powers of two whose product is one past
    the range (2^bits unsigned, MAX + 1 signed) or at its end (2^bits - 2^k,
    MIN)"""
    vals = edge_values(n, signed, rng)
    pairs = list(itertools.product(vals, vals))
    bits = 2 * n
    for k in (1, n, bits - 2):
        if signed:
            x, y = 1 << k, 1 << (bits - 1 - k)
            pairs += [(x, y), (-x, -y), (-x, y), (x, -y)]
        else:
            x, y = 1 << k, 1 << (bits - k)
            pairs += [(x, y), (x, y - 1)]
    return pairs


@pytest.mark.parametrize("n", [32, 64])
@pytest.mark.parametrize("signed", [False, True])
def test_edges_at_wide_integers(n, signed):
    rng = np.random.default_rng(zlib.crc32(f"mul{n}{signed}".encode()))
    key = cleartext_key()
    a, b = map(list, zip(*edge_pairs(n, signed, rng)))
    ops = binary_ops(signed) if n == 32 else {k: v for k, v in binary_ops(signed).items() if "mul" in k}
    for op, f in ops.items():
        want = [f(x, y, n) for x, y in zip(a, b)]
        assert binary(key, op, a, b, n, signed) == want, op
        if "overflowing_mul" in op:
            assert any(w[1] for w in want) and not all(w[1] for w in want)
    sops = scalar_ops(signed) if n == 32 else {"scalar_mul": SCALAR["scalar_mul"]}
    for op, f in sops.items():
        got = results(getattr(key, op)(ct(a, n, signed), b), signed)
        assert got == [f(x, y, n, signed) for x, y in zip(a, b)], op
    vals = edge_values(n, signed, rng)
    assert ints(key.abs(ct(vals, n, signed)), signed) == [wrap(abs(v), n, signed) for v in vals]
    cols = [vals, vals[::-1], [wrap(-1, n, signed)] * len(vals), vals[1:] + vals[:1]]
    out = key.sum_ciphertexts([ct(col, n, signed) for col in cols])
    assert ints(out, signed) == [RM.model("sum", t, n, signed) for t in zip(*cols)]


def test_products_that_overflow_by_one():
    """the exact product one past the range: flag set; one below: clear"""
    key = cleartext_key()
    n, bits = 32, 64
    a, b = [1 << 32, 1 << 31, 3, 5], [1 << 32, 1 << 33, 6148914691236517206, 3689348814741910324]
    # (2^64, 2^64, 2^64 + 2, 2^64 + 4) overflow; each with b - 1 does not
    want = [(x * y % (1 << bits), int(x * y >= 1 << bits)) for x, y in zip(a + a, b + [y - 1 for y in b])]
    assert [w[1] for w in want] == [1] * 4 + [0] * 4
    assert binary(key, "unsigned_overflowing_mul", a + a, b + [y - 1 for y in b], n, False) == want
    # signed: MAX + 1 = 2^31 * 2^32 and MIN - 1 = -(3 * 3074457345618258603)
    a, b = [1 << 31, -3, 1 << 31, -3], [1 << 32, 3074457345618258603, (1 << 32) - 1, 3074457345618258602]
    want = [RM.model("signed_overflowing_mul", (x, y), n, True) for x, y in zip(a, b)]
    assert [w[1] for w in want] == [1, 1, 0, 0]
    assert binary(key, "signed_overflowing_mul", a, b, n, True) == want


# ---------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------
# (PBS count, PBS layers, peak slots) of one FheUint64 (32 blocks) instance;
# recorded in DESIGN §8n
PINNED_MUL = {
    ("mul", None): (1883, 13, 1024), ("scalar_mul", None): (1883, 13, 1024),
    ("unsigned_overflowing_mul", None): (2088, 13, 1118), ("signed_overflowing_mul", None): (2786, 27, 849),
    ("sum", 2): (218, 7, 64), ("sum", 4): (281, 8, 128), ("sum", 7): (344, 9, 224),
}
PINNED_ARITH = {
    "signed_overflowing_add": (220, 7, 64), "signed_overflowing_sub": (220, 7, 64), "abs": (218, 7, 63),
    "scalar_add": (218, 7, 63), "scalar_sub": (218, 7, 63), "scalar_overflowing_add": (224, 7, 64),
    "scalar_signed_overflowing_add": (220, 7, 64), "scalar_signed_overflowing_sub": (220, 7, 64),
    "scalar_bitand": (32, 1, 32), "scalar_bitor": (32, 1, 32), "scalar_bitxor": (32, 1, 32),
}


def test_every_circuit_is_pinned():
    assert {op for op, _ in PINNED_MUL} == set(RM.OPERATIONS)
    assert set(PINNED_ARITH) == set(R.ARITH_OPERATIONS)


@pytest.mark.parametrize("op,count", sorted(PINNED_MUL, key=str))
def test_pinned_product_schedules(op, count):
    s = bc.schedule(RM.circuit(op, 32, count), 1)
    assert (s.pbs_count(), s.num_layers, s.peak_slots) == PINNED_MUL[(op, count)]
    assert s.pbs_shared_rows == 0


@pytest.mark.parametrize("op", sorted(PINNED_ARITH))
def test_pinned_arith_schedules(op):
    """the same counts unsigned and signed (abs: signed; unsigned abs never
    runs a circuit)"""
    s = bc.schedule(R.circuit(op, 32, True), 1)
    assert (s.pbs_count(), s.num_layers, s.peak_slots) == PINNED_ARITH[op]
    if op != "abs":
        assert R.circuit(op, 32, False) is R.circuit(op, 32, True)


def test_schedule_bounds():
    """FheUint64 mul: <= 1,904 PBS (unchecked_mul's count) and <= 13 layers;
    scalar_mul costs no more than mul; the signed overflow flags add no layer
    to add / sub; the §8j schedules are unchanged; one compile serves every
    instance count"""
    s = bc.schedule(RM.circuit("mul", 32), 1)
    assert s.pbs_count() <= 1904 and s.num_layers <= 13
    assert bc.schedule(RM.circuit("scalar_mul", 32), 1).pbs_count() <= s.pbs_count()
    assert bc.schedule(RM.circuit("mul", 32), 7).pbs_count() == 7 * s.pbs_count()
    add = bc.schedule(R.circuit("add", 32), 1)
    for op in ("signed_overflowing_add", "signed_overflowing_sub", "scalar_signed_overflowing_add"):
        assert bc.schedule(R.circuit(op, 32), 1).num_layers == add.num_layers == 7
    assert (add.pbs_count(), add.peak_slots) == (218, 64)
    assert RM.circuit("mul", 32) is RM.circuit("mul", 32)
    assert RM.circuit("sum", 32, 3) is not RM.circuit("sum", 32, 4)
    assert bc.NUM_FIXED_LUTS == 11


# ---------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------
def test_argument_checks_raise_before_any_call():
    key = cleartext_key()
    u2, u3, s2 = ct([1, 2], 2), ct([1, 2], 3), ct([1, 2], 2, signed=True)
    bad = [
        lambda: key.mul(u2, u3),                          # block counts
        lambda: key.mul(u2, s2),                          # signedness
        lambda: key.mul(u2, ct([5], 2)),                  # num_inputs
        lambda: key.mul(u2, u2.blocks),
        lambda: key.unsigned_overflowing_mul(s2, s2),     # kind of the operation
        lambda: key.signed_overflowing_mul(u2, u2),
        lambda: key.signed_overflowing_add(u2, u2),
        lambda: key.signed_overflowing_sub(u2, u2),
        lambda: key.signed_overflowing_scalar_add(u2, 1),
        lambda: key.signed_overflowing_scalar_sub(u2, 1),
        lambda: key.unsigned_overflowing_scalar_add(s2, 1),
        lambda: key.sum_ciphertexts([u2, u3]),
        lambda: key.sum_ciphertexts([u2, s2]),
        lambda: key.sum_ciphertexts([u2, ct([5], 2)]),
        lambda: key.scalar_mul(u2, 16),                   # out of [0, 16)
        lambda: key.scalar_add(u2, -1),
        lambda: key.scalar_sub(s2, 8),                    # out of [-8, 8)
        lambda: key.scalar_bitand(s2, -9),
        lambda: key.scalar_bitor(u2, [1, 2, 3]),
        lambda: key.scalar_bitxor(u2, 1.5),
        lambda: key.unsigned_overflowing_scalar_add(u2, True),
        lambda: key.abs(u2.blocks),
        lambda: key.mul(ct([0], 65), ct([1], 65)),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert key.runner.calls == 0
    for args in (("mul", 0), ("mul", 65), ("div", 4), ("sum", 4, 0), ("sum", 4, None), ("sum", 4, True)):
        with pytest.raises(ValueError):
            RM.circuit(*args)
    with pytest.raises(ValueError):
        R.circuit("scalar_mul", 4)


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def test_three_block_products_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_radix: mul and signed_overflowing_mul; every block
    decrypts exactly and holds <= 3"""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=53)
    rng = oracle.Rng(0x3A1)
    n = 3

    def run(op, signed, a, b):
        s = bc.schedule(RM.circuit(op, n), len(a))
        digits = [d for x, y in zip(a, b) for v in (x, y) for d in R.to_digits(v, n)]
        out = run_oracle(oracle, keys, s, M.encrypt_bits(oracle, keys, rng, digits))
        rows = M.decrypt_messages(oracle, keys, out, vmax=3).reshape(len(a), -1)
        return [(R.from_digits(r[:n], signed),) + tuple(int(v) for v in r[n:]) for r in rows]

    a, b = [63, 50, 7, 0], [63, 5, 9, 41]
    assert run("mul", False, a, b) == [(x * y % 64,) for x, y in zip(a, b)]
    a, b = [-32, -32, 31, -7, 5], [-1, 1, 2, -4, -6]
    assert run("signed_overflowing_mul", True, a, b) == [RM.model("signed_overflowing_mul", (x, y), n, True)
                                                         for x, y in zip(a, b)]


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_mul(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0x3A00 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    rk = integer.CudaRadixServerKey(skey, glwe_dimension=P.k, polynomial_size=P.N)
    rng = oracle.Rng(0x3A02)

    def enc(values, n, signed=False):
        digits = [d for v in values for d in R.to_digits(int(v), n)]
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, digits).view(np.int64)).to(streams.device(0))
        kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
        return kind(t, len(values))

    def dec(x, signed=False):
        """copy on the caller's current stream, which waits for the work stream"""
        if isinstance(x, tuple):
            return list(zip(dec(x[0], signed), dec(x[1])))
        if isinstance(x, integer.CudaBooleanBlock):
            return [int(v) for v in M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64))]
        d = M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64), vmax=3)
        return [R.from_digits(r, signed) for r in d.reshape(x.num_inputs, -1)]

    yield rk, enc, dec
    rk.runner.close()


def gpu_pairs(n, signed, num_inputs, rng):
    """at one input a random pair, else random pairs then edge pairs"""
    rand = [(rand_int(rng, n, signed), rand_int(rng, n, signed)), (rand_int(rng, n, signed),
                                                                   wrap(int(rng.integers(1, 1 << 30)), n, signed))]
    if num_inputs == 1:
        return rand[:1]
    pairs = edge_pairs(n, signed, rng)
    return (rand + [pairs[int(i)] for i in rng.permutation(len(pairs))])[:num_inputs]


@pytest.mark.gpu
@pytest.mark.parametrize("num_inputs", [1, 7])
@pytest.mark.parametrize("signed", [False, True])
def test_gpu_fheuint64(gpu_mul, num_inputs, signed):
    rk, enc, dec = gpu_mul
    n = 32
    rng = np.random.default_rng(zlib.crc32(f"gpumul{num_inputs}{signed}".encode()))
    a, b = map(list, zip(*gpu_pairs(n, signed, num_inputs, rng)))
    A, B = enc(a, n, signed), enc(b, n, signed)
    for op, f in binary_ops(signed).items():
        assert dec(getattr(rk, op)(A, B), signed) == [f(x, y, n) for x, y in zip(a, b)], op
    for op, f in scalar_ops(signed).items():
        assert dec(getattr(rk, op)(A, b), signed) == [f(x, y, n, signed) for x, y in zip(a, b)], op
    assert dec(rk.scalar_mul(A, b[0]), signed) == [RM.model("mul", (x, b[0]), n, signed) for x in a]
    assert dec(rk.abs(A), signed) == [wrap(abs(x), n, signed) for x in a]
    C = enc(b[::-1], n, signed)
    assert dec(rk.sum_ciphertexts([A, B, C, A]), signed) == [RM.model("sum", (x, y, z, x), n, signed)
                                                             for x, y, z in zip(a, b, b[::-1])]


@pytest.mark.gpu
def test_gpu_fheuint128(gpu_mul):
    rk, enc, dec = gpu_mul
    n = 64
    a, b = [(0xDEADBEEF << 96) + 0x1234567, 0xFFFF << 50], [(0xCAFE << 40) + 99, 0x1234 << 60]
    A, B = enc(a, n), enc(b, n)
    want = [x * y % (1 << 128) for x, y in zip(a, b)]
    assert dec(rk.mul(A, B)) == want
    assert dec(rk.unsigned_overflowing_mul(A, B)) == [(w, int(x * y >> 128 != 0)) for w, x, y in zip(want, a, b)]


@pytest.mark.gpu
def test_gpu_mul_matches_unchecked_mul(gpu_mul):
    """mul and unchecked_mul on the same operands decrypt to the same value"""
    rk, enc, dec = gpu_mul
    n = 32
    a, b = [0xFEDCBA9876543210], [0x0123456789ABCDEF]
    A, B = enc(a, n), enc(b, n)
    want = [a[0] * b[0] % (1 << 64)]
    assert dec(rk.mul(A, B)) == dec(rk.unchecked_mul(A, B)) == want


@pytest.mark.gpu
def test_gpu_product_into_add_gt_and_div_rem(gpu_mul):
    """a product is clean blocks: fed into add, gt and div_rem"""
    rk, enc, dec = gpu_mul
    n = 32
    a, b, c = [123456789, 1 << 40], [987654321, 3], [10 ** 17, 7]
    p = rk.mul(enc(a, n), enc(b, n))
    C = enc(c, n)
    prod = [x * y % (1 << 64) for x, y in zip(a, b)]
    assert dec(rk.add(p, C)) == [(x + z) % (1 << 64) for x, z in zip(prod, c)]
    assert dec(rk.gt(p, C)) == [int(x > z) for x, z in zip(prod, c)]
    q, r = rk.div_rem(p, C)
    assert list(zip(dec(q), dec(r))) == [D.model(x, z, n) for x, z in zip(prod, c)]
