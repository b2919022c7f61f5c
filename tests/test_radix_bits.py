"""Shifts, rotations and bit counts of radix integers (tfhe-rs_b200/radix_bits.py
and the matching methods of integer.CudaRadixServerKey).

CPU: every operation through the server key's host code on a cleartext runner
(the compiled schedules on `bit_circuit.run_cleartext`, which asserts the
noise budget and the value range on every row), exhaustively at 1, 2 and 3
blocks, unsigned and signed, with every amount of 1- and 2-block amounts and
every clear amount in [0, 2 bits], and on edge values at 32 and 64 blocks,
against the plain model `radix_bits.model`; the pinned FheUint64 schedule
counts and layer bounds; argument checks; left_shift, signed right_shift,
rotate_right and leading_zeros through real LWE keyswitches and PBS on the
oracle.

GPU: `CudaRadixServerKey` on classic P22 and multi-bit g = 4: every new
method at FheUint64 with 1 and 7 inputs, unsigned and signed, one FheUint128
shift by an FheUint8 amount, and a right_shift chained into add and gt; every
output block decrypts to the model's value."""
import itertools
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import bit_circuit as bc, integer, radix as R, radix_bits as RB

from tests import trivium_model as M
from tests.test_radix import bools, cleartext_key, ct, ints, rand_int, wrap
from tests.test_trivium import run_oracle

SHIFTS = RB.SHIFTS
SCALARS = tuple(f"scalar_{o}" for o in SHIFTS)
COUNTS = RB.COUNTS


def run(key, op, values, n, signed, amount=None, amount_blocks=None):
    """op on a list of integers through the server key: a list of ints, or of
    (ilog2, flag) for checked_ilog2"""
    A = ct(values, n, signed)
    if op in SHIFTS:
        return ints(getattr(key, op)(A, ct(amount, amount_blocks)), signed)
    if op in SCALARS:
        return ints(getattr(key, op)(A, amount), signed)
    out = getattr(key, op)(A)
    if op == "checked_ilog2":
        assert out[0].num_blocks == RB.ilog2_blocks(n)
        return list(zip(ints(out[0]), bools(out[1])))
    assert type(out) is integer.CudaUnsignedRadixCiphertext and out.num_blocks == RB.result_blocks(op, n)
    return ints(out)


def want(op, values, n, signed, amount=None):
    amounts = amount if isinstance(amount, (list, tuple)) else [amount] * len(values)
    return [RB.model(op, v, n, signed, a) for v, a in zip(values, amounts)]


# ---------------------------------------------------------------------------
# the plain model
# ---------------------------------------------------------------------------
def test_model():
    assert RB.model("left_shift", 3, 2, amount=1) == 6 and RB.model("left_shift", 3, 2, amount=4) == 0
    assert RB.model("right_shift", -8, 2, True, 1) == -4 and RB.model("right_shift", -8, 2, True, 99) == -1
    assert RB.model("right_shift", 7, 2, True, 4) == 0 and RB.model("right_shift", 8, 2, False, 3) == 1
    # 6 bits read m = 3 amount bits: 8 rotates by 0, 7 by 1; a clear 8 by 2
    assert RB.rotation_bits(3) == 3 and RB.rotation_bits(32) == 6 and RB.rotation_bits(1) == 1
    assert RB.model("rotate_left", 0b000011, 3, amount=8) == 0b000011
    assert RB.model("rotate_left", 0b000011, 3, amount=7) == 0b000110
    assert RB.model("scalar_rotate_left", 0b000011, 3, amount=8) == 0b001100
    assert RB.model("rotate_right", 1, 2, amount=1) == 8 and RB.model("rotate_right", -8, 2, True, 3) == 1
    assert RB.model("leading_zeros", 1, 32) == 63 and RB.model("trailing_ones", -1, 32, True) == 64
    assert RB.model("count_ones", -1, 4, True) == 8 and RB.model("count_zeros", 1, 4) == 7
    # ilog2(0) = (bits - 1) - bits cast to ilog2_blocks: all ones
    assert RB.model("ilog2", 0, 32) == 255 and RB.model("ilog2", 1 << 63, 32) == 63
    assert RB.model("checked_ilog2", -1, 2, True) == (3, 0) and RB.model("checked_ilog2", 5, 2) == (2, 1)
    assert [RB.count_blocks(n) for n in (1, 2, 3, 4, 32, 64)] == [1, 2, 2, 2, 4, 4]
    assert [RB.ilog2_blocks(n) for n in (1, 2, 3, 4, 32, 64)] == [1, 2, 2, 2, 4, 4]


# ---------------------------------------------------------------------------
# exhaustive at 1, 2 and 3 blocks
# ---------------------------------------------------------------------------
def domain(n, signed):
    lo, hi = R.scalar_range(n, signed)
    return list(range(lo, hi))


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_shifts_and_rotations(n, signed):
    """every (value, amount) pair with 1- and 2-block amounts, as instances of
    one call: overshifts and, at 3 blocks, the 6-bit rotation read of m = 3
    amount bits are among them"""
    key = cleartext_key()
    vals = domain(n, signed)
    for amount_blocks in (1, 2):
        a, b = map(list, zip(*itertools.product(vals, range(4 ** amount_blocks))))
        for op in SHIFTS:
            assert run(key, op, a, n, signed, b, amount_blocks) == want(op, a, n, signed, b), (op, amount_blocks)


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_scalar_shifts_and_rotations(n, signed):
    key = cleartext_key()
    vals = domain(n, signed)
    for op in SCALARS:
        for amount in range(0, 4 * n + 1):
            assert run(key, op, vals, n, signed, amount) == want(op, vals, n, signed, amount), (op, amount)


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_bit_counts(n, signed):
    key = cleartext_key()
    vals = domain(n, signed)
    for op in COUNTS:
        assert run(key, op, vals, n, signed) == want(op, vals, n, signed), op


# ---------------------------------------------------------------------------
# edge values at 32 and 64 blocks
# ---------------------------------------------------------------------------
def edge_values(n, signed, rng):
    """0, 1, MIN, MAX, -1, single-bit patterns, their complements and random
    values"""
    lo, hi = R.scalar_range(n, signed)
    bits = 2 * n
    single = [wrap(1 << i, n, signed) for i in sorted({0, 1, 2, 3, bits // 2, bits - 2, bits - 1}
                                                        | {int(i) for i in rng.integers(0, bits, 3)})]
    return sorted({0, 1, lo, hi - 1, wrap(-1, n, signed)} | set(single) | {wrap(~v, n, signed) for v in single}
                  | {rand_int(rng, n, signed) for _ in range(3)})


def edge_amounts(n, amount_blocks):
    bits = 2 * n
    top = 4 ** amount_blocks - 1
    return sorted({a for a in (0, 1, 2, 3, 7, bits // 2 + 1, bits - 1, bits, bits + 1, 2 * bits, top)
                   if a <= top})


@pytest.mark.parametrize("n", [32, 64])
@pytest.mark.parametrize("signed", [False, True])
def test_edges_at_wide_integers(n, signed):
    rng = np.random.default_rng(zlib.crc32(f"bits{n}{signed}".encode()))
    key = cleartext_key()
    vals = edge_values(n, signed, rng)
    for amount_blocks in (n, 4, 1):
        a, b = map(list, zip(*itertools.product(vals, edge_amounts(n, amount_blocks))))
        for op in SHIFTS:
            assert run(key, op, a, n, signed, b, amount_blocks) == want(op, a, n, signed, b), (op, amount_blocks)
    for op in SCALARS:
        for amount in edge_amounts(n, n) + [4 ** 40 + 3]:
            assert run(key, op, vals, n, signed, amount) == want(op, vals, n, signed, amount), (op, amount)
    for op in COUNTS:
        assert run(key, op, vals, n, signed) == want(op, vals, n, signed), op


# ---------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------
# (PBS count, PBS layers, peak slots) of one FheUint64 (32 blocks) instance:
# shifts by an FheUint64 amount, clear shifts by 13; recorded in DESIGN §8m
PINNED = {
    ("left_shift", False): (653, 6, 166), ("right_shift", False): (653, 6, 166),
    ("right_shift", True): (653, 6, 167),
    ("rotate_left", False): (708, 6, 193), ("rotate_right", False): (708, 6, 193),
    ("scalar_left_shift", False): (27, 1, 33), ("scalar_right_shift", False): (27, 1, 32),
    ("scalar_right_shift", True): (26, 1, 32),
    ("scalar_rotate_left", False): (32, 1, 32), ("scalar_rotate_right", False): (32, 1, 32),
    ("leading_zeros", False): (163, 7, 68), ("leading_ones", False): (163, 7, 68),
    ("trailing_zeros", False): (163, 7, 68), ("trailing_ones", False): (163, 7, 68),
    ("count_ones", False): (50, 8, 32), ("count_zeros", False): (50, 8, 32),
    ("ilog2", False): (163, 7, 74), ("checked_ilog2", False): (164, 7, 74), ("checked_ilog2", True): (165, 7, 75),
}
LAYER_BOUNDS = {**{op: 10 for op in SHIFTS}, **{op: 1 for op in SCALARS},
                **{op: 16 for op in COUNTS}, "ilog2": 18, "checked_ilog2": 18}


def pinned_circuit(op, signed, n=32):
    arg = n if op in SHIFTS else (13 if op in SCALARS else None)
    return RB.circuit(op, n, signed, arg)


def test_every_operation_is_pinned():
    assert {op for op, _ in PINNED} == set(RB.OPERATIONS)
    assert {op for op, signed in PINNED if signed} == set(RB.SIGNED_OPS)


@pytest.mark.parametrize("op,signed", sorted(PINNED))
def test_pinned_schedule_counts(op, signed):
    s = bc.schedule(pinned_circuit(op, signed), 1)
    assert (s.pbs_count(), s.num_layers, s.peak_slots) == PINNED[(op, signed)]
    assert s.pbs_shared_rows == 0


def test_schedule_bounds():
    """FheUint64 layer bounds whatever the signedness: <= 10 for a shift or
    rotation by an encrypted amount, exactly 1 by a clear one (every amount),
    <= 16 for the counts and <= 18 for ilog2; one compile serves every
    instance count; circuits are cached per (op, blocks, amount, signed), a
    clear amount in its canonical form"""
    for op in RB.OPERATIONS:
        for signed in (False, True):
            n = bc.schedule(pinned_circuit(op, signed), 1).num_layers
            assert n <= LAYER_BOUNDS[op] and (op not in SCALARS or n == 1), (op, signed)
    for op in SCALARS:
        for amount in range(0, 65):
            assert bc.schedule(RB.circuit(op, 32, False, amount), 1).num_layers == 1
    for amount_blocks in (1, 4, 64):
        assert bc.schedule(RB.circuit("left_shift", 32, False, amount_blocks), 1).num_layers <= 10
    s = bc.schedule(RB.circuit("left_shift", 32, False, 32), 1)
    assert bc.schedule(RB.circuit("left_shift", 32, False, 32), 7).pbs_count() == 7 * s.pbs_count()
    assert RB.circuit("left_shift", 32, False, 32) is RB.circuit("left_shift", 32, True, 32)
    assert RB.circuit("right_shift", 32, False, 32) is not RB.circuit("right_shift", 32, True, 32)
    assert RB.circuit("left_shift", 32, False, 32) is not RB.circuit("left_shift", 32, False, 4)
    assert RB.circuit("scalar_rotate_left", 32, False, 5) is RB.circuit("scalar_rotate_left", 32, False, 69)
    assert RB.circuit("scalar_left_shift", 32, False, 64) is RB.circuit("scalar_left_shift", 32, False, 10 ** 30)
    assert RB.circuit("scalar_left_shift", 32, False, 63) is not RB.circuit("scalar_left_shift", 32, False, 64)
    assert bc.NUM_FIXED_LUTS == 11 and len(s.extra_luts) > 0


# ---------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------
def test_argument_checks_raise_before_any_call():
    key = cleartext_key()
    u2, s2 = ct([1, 2], 2), ct([1, 2], 2, signed=True)
    bad = [
        lambda: key.left_shift(u2, ct([1, 2], 2, signed=True)),   # signed amount
        lambda: key.right_shift(u2, ct([1], 2)),                  # num_inputs
        lambda: key.rotate_left(u2, u2.blocks),
        lambda: key.left_shift(ct([0], 65), ct([1], 1)),          # 65 blocks
        lambda: key.left_shift(u2, ct([0, 1], 65)),
        lambda: key.rotate_right(u2, integer.CudaUnsignedRadixCiphertext(u2.blocks[:0], 2)),   # 0 blocks
        lambda: key.leading_zeros(ct([0], 65)),
        lambda: key.count_ones(integer.CudaUnsignedRadixCiphertext(u2.blocks[:0], 1)),
        lambda: key.scalar_left_shift(u2, -1),                    # negative, bool, not an int
        lambda: key.scalar_right_shift(s2, True),
        lambda: key.scalar_rotate_left(u2, 1.0),
        lambda: key.scalar_rotate_right(u2, [1, 2]),
        lambda: key.scalar_left_shift(ct([0], 65), 1),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert key.runner.calls == 0
    for args in (("left_shift", 0, False, 1), ("left_shift", 4, False, 0), ("left_shift", 4, False, 65),
                 ("scalar_left_shift", 4, False, -2), ("shl", 4, False, 1)):
        with pytest.raises(ValueError):
            RB.circuit(*args)
    # a signed integer shifted by a 1-block amount; numpy ints are amounts too
    assert ints(key.right_shift(s2, ct([1, 3], 1)), True) == [0, 0]
    assert ints(key.scalar_left_shift(u2, np.int64(1))) == [2, 4]


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def test_three_block_shifts_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_radix: left_shift, signed right_shift and
    rotate_right by 2-block amounts (overshifts and the 6-bit rotation among
    them), and leading_zeros; every block decrypts exactly and holds <= 3."""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=53)
    rng = oracle.Rng(0xB175)
    n, ab = 3, 2

    def go(op, signed, a, b=None):
        s = bc.schedule(RB.circuit(op, n, signed, ab if b is not None else None), len(a))
        digits = [d for i, v in enumerate(a) for d in R.to_digits(v, n) + (R.to_digits(b[i], ab) if b else [])]
        out = run_oracle(oracle, keys, s, M.encrypt_bits(oracle, keys, rng, digits))
        return [R.from_digits(r, signed and op != "leading_zeros")
                for r in M.decrypt_messages(oracle, keys, out, vmax=3).reshape(len(a), -1)]

    a, b = [0b101101, 63, 1, 22], [1, 5, 6, 15]
    assert go("left_shift", False, a, b) == want("left_shift", a, n, False, b)
    a, b = [-32, -3, 31, -1], [3, 7, 2, 6]
    assert go("right_shift", True, a, b) == want("right_shift", a, n, True, b)
    a, b = [0b000011, 0b100001, 42], [8, 7, 13]
    assert go("rotate_right", False, a, b) == want("rotate_right", a, n, False, b)
    a = [0, 1, 2, 7, 32, 63]
    assert go("leading_zeros", False, a) == want("leading_zeros", a, n, False)


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_bits(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0xB100 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    rk = integer.CudaRadixServerKey(skey, glwe_dimension=P.k, polynomial_size=P.N)
    rng = oracle.Rng(0xB102)

    def enc(values, n, signed=False):
        digits = [d for v in values for d in R.to_digits(int(v), n)]
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, digits).view(np.int64)).to(streams.device(0))
        kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
        return kind(t, len(values))

    def dec(x, signed=False):
        """copy on the caller's current stream, which waits for the work stream"""
        if isinstance(x, integer.CudaBooleanBlock):
            assert x.blocks.shape[0] == x.num_inputs
            return [int(v) for v in M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64))]
        d = M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64), vmax=3)
        return [R.from_digits(r, signed) for r in d.reshape(x.num_inputs, -1)]

    yield rk, enc, dec
    rk.runner.close()


@pytest.mark.gpu
@pytest.mark.parametrize("num_inputs", [1, 7])
@pytest.mark.parametrize("signed", [False, True])
def test_gpu_every_operation_fheuint64(gpu_bits, num_inputs, signed):
    rk, enc, dec = gpu_bits
    n = 32
    rng = np.random.default_rng(zlib.crc32(f"gpubits{num_inputs}{signed}".encode()))
    vals = edge_values(n, signed, rng)
    a = [rand_int(rng, n, signed)] + [vals[int(i)] for i in rng.permutation(len(vals))[:num_inputs - 1]]
    # one overshift at one input; at 7: in range, bits - 1, bits, a large amount
    b = [64] if num_inputs == 1 else [0, 1, 13, 63, 64, 65, 4 ** 31 + 5]
    A, B = enc(a, n, signed), enc(b, n)
    for op in SHIFTS:
        assert dec(getattr(rk, op)(A, B), signed) == want(op, a, n, signed, b), op
    for op, amount in itertools.product(SCALARS, (13, 64 if num_inputs == 1 else 70)):
        assert dec(getattr(rk, op)(A, amount), signed) == want(op, a, n, signed, amount), (op, amount)
    for op in COUNTS:
        out = getattr(rk, op)(A)
        got = list(zip(dec(out[0]), dec(out[1]))) if op == "checked_ilog2" else dec(out)
        assert got == want(op, a, n, signed), op


@pytest.mark.gpu
def test_gpu_fheuint128_shift_by_fheuint8(gpu_bits):
    rk, enc, dec = gpu_bits
    n = 64
    a, b = [(0xDEADBEEF << 96) + 0x1234567, (1 << 127) + 5], [77, 200]
    assert dec(rk.left_shift(enc(a, n), enc(b, 4))) == want("left_shift", a, n, False, b)


@pytest.mark.gpu
def test_gpu_right_shift_into_add_and_gt(gpu_bits):
    """a right_shift result is clean blocks: fed into add and gt"""
    rk, enc, dec = gpu_bits
    n = 32
    a, b, c = [10 ** 18, -(1 << 62), 12345], [3, 60, 64], [999, 7, -1]
    shifted = rk.right_shift(enc(a, n, True), enc(b, n))
    want_s = want("right_shift", a, n, True, b)
    assert dec(shifted, True) == want_s
    C = enc(c, n, True)
    assert dec(rk.add(shifted, C), True) == [wrap(x + z, n, True) for x, z in zip(want_s, c)]
    assert dec(rk.gt(shifted, C)) == [int(x > z) for x, z in zip(want_s, c)]
