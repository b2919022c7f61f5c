"""Radix-integer operations on 2_2 blocks (tfhe-rs_b200/radix.py and the
methods of integer.CudaRadixServerKey).

CPU: the compiler's block inputs; every operation through the server key's
host code on a cleartext runner (the compiled schedules on
`bit_circuit.run_cleartext`, which asserts the noise budget and the value
range on every row), exhaustively at 1, 2 and 3 blocks and on edge values at
5, 32 and 64 blocks, against Python integers; the pinned schedule counts and
layer bounds; argument checks; gt, signed lt, add and transfer through real
LWE keyswitches and PBS on the oracle.

GPU: `CudaRadixServerKey` on classic P22 and multi-bit g = 4: every output
block decrypts to the model's value and holds <= 3, booleans decrypt to 0 or
1."""
import itertools
import types
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import aes, bit_circuit as bc, integer, radix as R, trivium as T

from tests import trivium_model as M
from tests.test_trivium import CleartextRunner, run_oracle

CMP = {"eq": lambda a, b: a == b, "ne": lambda a, b: a != b, "gt": lambda a, b: a > b,
       "ge": lambda a, b: a >= b, "lt": lambda a, b: a < b, "le": lambda a, b: a <= b}


# ---------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------
def wrap(v, n, signed=False):
    """v as an n-block integer: mod 4^n, two's complement when signed"""
    return R.from_digits(R.to_digits(v, n), signed)


def model(op, n, signed, a, b=None, cond=None):
    """expected result of op: an int, a bool, or a tuple"""
    if op in CMP:
        return int(CMP[op](a, b))
    if op == "min":
        return min(a, b)
    if op == "max":
        return max(a, b)
    if op == "if_then_else":
        return a if cond else b
    if op == "add":
        return wrap(a + b, n, signed)
    if op == "sub":
        return wrap(a - b, n, signed)
    if op == "neg":
        return wrap(-a, n, signed)
    if op == "overflowing_add":
        return wrap(a + b, n), int(a + b >= 4 ** n)
    if op == "overflowing_sub":
        return wrap(a - b, n), int(a < b)
    if op == "bitand":
        return wrap(a & b, n, signed)
    if op == "bitor":
        return wrap(a | b, n, signed)
    if op == "bitxor":
        return wrap(a ^ b, n, signed)
    if op == "bitnot":
        return wrap(~a, n, signed)
    raise AssertionError(op)


def transfer_model(frm, to, amount, n):
    sent = amount if frm >= amount else 0
    return wrap(frm - sent, n), wrap(to + sent, n)


# ---------------------------------------------------------------------------
# the server key's host code on a cleartext runner
# ---------------------------------------------------------------------------
def cleartext_key():
    k = integer.CudaRadixServerKey.__new__(integer.CudaRadixServerKey)
    k._runner = CleartextRunner()
    return k


def ct(values, n, signed=False):
    """cleartext radix ciphertext of `values` (one integer per input)"""
    import torch

    digits = np.array([R.to_digits(int(v), n) for v in values], dtype=np.int64)
    kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
    return kind(torch.from_numpy(digits.reshape(-1, 1)), len(values))


def boolean(values):
    import torch

    return integer.CudaBooleanBlock(torch.tensor(np.asarray(values, dtype=np.int64).reshape(-1, 1)), len(values))


def ints(x, signed=False):
    """integers of a cleartext result (checking every block is <= 3)"""
    d = x.blocks[:, 0].numpy().reshape(x.num_inputs, -1)
    assert d.min() >= 0 and d.max() <= 3
    return [R.from_digits(row, signed) for row in d]


def bools(x):
    d = [int(v) for v in x.blocks.reshape(x.num_inputs, -1)[:, 0]]
    assert x.blocks.shape[0] == x.num_inputs and set(d) <= {0, 1}
    return d


def run_op(key, op, n, signed, a, b=None, cond=None):
    """op on lists of integers through the server key: results as ints / bools"""
    A = ct(a, n, signed)
    if op in CMP:
        return bools(getattr(key, op)(A, ct(b, n, signed)))
    if op in ("neg", "bitnot"):
        return ints(getattr(key, op)(A), signed)
    if op == "if_then_else":
        return ints(key.if_then_else(boolean(cond), A, ct(b, n, signed)), signed)
    if op.startswith("overflowing"):
        out, flag = getattr(key, f"unsigned_{op}")(A, ct(b, n))
        return list(zip(ints(out), bools(flag)))
    return ints(getattr(key, op)(A, ct(b, n, signed)), signed)


BINARY = ["eq", "ne", "gt", "ge", "lt", "le", "min", "max", "add", "sub", "bitand", "bitor", "bitxor"]


def domain(n, signed):
    lo, hi = R.scalar_range(n, signed)
    return list(range(lo, hi))


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_binary_operations(n, signed):
    """every (a, b) pair as instances of one call (3 blocks: 4,096 pairs)"""
    key = cleartext_key()
    vals = domain(n, signed)
    a, b = zip(*itertools.product(vals, vals))
    ops = BINARY + (["overflowing_add", "overflowing_sub"] if not signed else [])
    for op in ops:
        got = run_op(key, op, n, signed, a, b)
        assert got == [model(op, n, signed, x, y) for x, y in zip(a, b)], (op, n, signed)


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_unary_and_select(n, signed):
    key = cleartext_key()
    vals = domain(n, signed)
    for op in ("neg", "bitnot"):
        assert run_op(key, op, n, signed, vals) == [model(op, n, signed, x) for x in vals]
    cond, a, b = zip(*itertools.product((0, 1), vals, vals))
    assert run_op(key, "if_then_else", n, signed, a, b, cond) == [x if c else y for c, x, y in zip(cond, a, b)]


@pytest.mark.parametrize("n", [1, 2, 3])
def test_exhaustive_transfer(n):
    """every (from, to, amount) at 1 and 2 blocks; every (from, amount) pair
    at 3 blocks, `to` random"""
    key = cleartext_key()
    vals = domain(n, False)
    if n < 3:
        frm, to, amt = zip(*itertools.product(vals, vals, vals))
    else:
        rng = np.random.default_rng(3)
        frm, amt = zip(*itertools.product(vals, vals))
        to = [int(x) for x in rng.integers(0, 4 ** n, len(frm))]
    new_from, new_to = key.transfer(ct(frm, n), ct(to, n), ct(amt, n))
    assert list(zip(ints(new_from), ints(new_to))) == [transfer_model(f, t, x, n) for f, t, x in zip(frm, to, amt)]


@pytest.mark.parametrize("signed", [False, True])
def test_every_scalar_at_two_blocks(signed):
    """every (a, scalar) at 2 blocks, one scalar per input; and a scalar
    given once for every input"""
    key = cleartext_key()
    vals = domain(2, signed)
    a, s = zip(*itertools.product(vals, vals))
    for op in CMP:
        got = bools(getattr(key, f"scalar_{op}")(ct(a, 2, signed), list(s)))
        assert got == [int(CMP[op](x, y)) for x, y in zip(a, s)], op
        got = bools(getattr(key, f"scalar_{op}")(ct(vals, 2, signed), vals[3]))
        assert got == [int(CMP[op](x, vals[3])) for x in vals], op


def rand_int(rng, n, signed):
    return wrap(int.from_bytes(rng.bytes(16), "little"), n, signed)


def edge_values(n, signed, rng):
    """0, the maximum, the signed minimum, -1, 1 and random values"""
    lo, hi = R.scalar_range(n, signed)
    return [0, hi - 1, lo, wrap(-1, n, signed), 1] + [rand_int(rng, n, signed) for _ in range(4)]


def edge_pairs(n, signed, rng):
    """pairs of edge values, equal operands, operands differing only in block
    0 or only in the top block, and full carry chains"""
    vals = edge_values(n, signed, rng)
    pairs = [(x, y) for x in vals for y in vals]
    top = 4 ** (n - 1)
    for x in vals:
        pairs += [(x, x), (x, wrap(x ^ 1, n, signed)), (x, wrap(x ^ 2, n, signed)), (x, wrap(x ^ top, n, signed)),
                  (x, wrap(x ^ (2 * top), n, signed))]
    # 0x5555.. + 0xAAAA.. + 1: block 0 generates, every other block propagates
    fives, tens = R.from_digits([1] * n, signed), R.from_digits([2] * n, signed)
    pairs += [(fives, tens), (fives, wrap(tens + 1, n, signed)), (wrap(tens + 1, n, signed), fives)]
    return pairs


@pytest.mark.parametrize("n", [5, 32, 64])
@pytest.mark.parametrize("signed", [False, True])
def test_edges_at_wide_integers(n, signed):
    rng = np.random.default_rng(zlib.crc32(f"edges{n}{signed}".encode()))
    key = cleartext_key()
    a, b = zip(*edge_pairs(n, signed, rng))
    ops = BINARY + (["overflowing_add", "overflowing_sub"] if not signed else [])
    for op in ops:
        assert run_op(key, op, n, signed, a, b) == [model(op, n, signed, x, y) for x, y in zip(a, b)], (op, n)
    for op in ("neg", "bitnot"):
        assert run_op(key, op, n, signed, a) == [model(op, n, signed, x) for x in a]
    cond = [int(x) for x in rng.integers(0, 2, len(a))]
    assert run_op(key, "if_then_else", n, signed, a, b, cond) == [x if c else y for c, x, y in zip(cond, a, b)]
    for op in CMP:
        got = bools(getattr(key, f"scalar_{op}")(ct(a, n, signed), list(b)))
        assert got == [int(CMP[op](x, y)) for x, y in zip(a, b)], op
    if not signed:
        # transfer: amount > from, amount == from, amount == 0, and the pairs
        frm, amt = [5, 5, 5, 0, 4 ** n - 1] + list(a), [6, 5, 0, 0, 4 ** n - 1] + list(b)
        to = [4 ** n - 1, 7, 3, 0, 1] + [rand_int(rng, n, False) for _ in a]
        new_from, new_to = key.transfer(ct(frm, n), ct(to, n), ct(amt, n))
        assert list(zip(ints(new_from), ints(new_to))) == [transfer_model(f, t, x, n)
                                                           for f, t, x in zip(frm, to, amt)]


# ---------------------------------------------------------------------------
# the compiler's block inputs
# ---------------------------------------------------------------------------
def test_block_inputs_in_the_compiler():
    c = bc.Circuit("blocks")
    x, y = c.inputs_block(2, False)
    bit = c.input(False)
    assert c.vmax[x] == bc.MAX_BLOCK_VALUE and c.vmax[bit] == 1
    for bad in (lambda: c.xor(x, bit), lambda: c.not_(x), lambda: c.and_(bit, x), lambda: c.mat(x),
                lambda: c.output([x])):
        with pytest.raises(ValueError):
            bad()
    s = c.lut([(x, 4), (y, 1)], 0, R.table(c, lambda v: (v // 4 + v % 4) % 4))
    # a block input passed straight through is refreshed by the identity, not parity
    c.output_blocks([s, y, bit])
    sched = bc.compile_circuit(c)
    assert sched.extra_luts[1] == (0, 1, 2, 3) + (0,) * 12
    ins = np.array([[u, v, w] for u in range(4) for v in range(4) for w in (0, 1)])
    got = bc.run_cleartext(sched.for_instances(len(ins)), [], ins)
    assert np.array_equal(got, np.array([c.evaluate([], i, []) for i in ins]))
    assert [list(r) for r in got] == [[(u + v) % 4, v, w] for u, v, w in ins]
    assert list(sched.row_lut).count(bc.LUT_PARITY) == 1      # only the bit's refresh
    # the compiler refuses a parity refresh of a block input
    d = bc.Circuit("raw")
    d.outputs.append(d.input_block(False))
    with pytest.raises(ValueError):
        bc.compile_circuit(d)


def test_existing_schedules_compile_to_identical_tables():
    """the fixed LUT set is unchanged: AES and Trivium circuits keep their
    pins and carry no tables of their own (but apply_keystream's)"""
    from tests import test_aes, test_trivium

    assert len(bc.lut_functions()) == bc.NUM_FIXED_LUTS == 11
    for kind in ("sbox", "counter_add"):
        s = bc.schedule(aes.circuit(kind), 1)
        assert (s.pbs_count(), s.num_layers, s.peak_slots) == test_aes.PINNED[kind] and s.extra_luts == ()
    for kind, n in (("trivium_next", 64), ("kreyvium_next", 64), ("apply_keystream", 0)):
        s = bc.schedule(T.circuit(kind, n), 1)
        assert (s.pbs_count(), s.num_layers, s.peak_slots) == test_trivium.PINNED[(kind, n)]


# ---------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------
# (PBS count, PBS layers, peak slots) of one FheUint64 (32 blocks) instance;
# recorded in DESIGN §8j
PINNED = {
    ("eq", False): (42, 4, 64), ("ne", False): (42, 4, 64),
    ("gt", False): (63, 6, 64), ("gt", True): (63, 6, 64),
    ("ge", False): (63, 6, 64), ("ge", True): (63, 6, 64),
    ("lt", False): (63, 6, 64), ("lt", True): (63, 6, 64),
    ("le", False): (63, 6, 64), ("le", True): (63, 6, 64),
    ("scalar_eq", False): (42, 4, 32), ("scalar_ne", False): (42, 4, 32),
    ("scalar_gt", False): (63, 6, 32), ("scalar_gt", True): (63, 6, 32),
    ("scalar_ge", False): (63, 6, 32), ("scalar_ge", True): (63, 6, 32),
    ("scalar_lt", False): (63, 6, 32), ("scalar_lt", True): (63, 6, 32),
    ("scalar_le", False): (63, 6, 32), ("scalar_le", True): (63, 6, 32),
    ("min", False): (159, 8, 96), ("min", True): (159, 8, 96),
    ("max", False): (159, 8, 96), ("max", True): (159, 8, 96),
    ("if_then_else", False): (96, 2, 65),
    ("add", False): (218, 7, 64), ("sub", False): (218, 7, 64), ("neg", False): (218, 7, 63),
    ("overflowing_add", False): (224, 7, 64), ("overflowing_sub", False): (224, 7, 64),
    ("bitand", False): (32, 1, 64), ("bitor", False): (32, 1, 64), ("bitxor", False): (32, 1, 64),
    ("bitnot", False): (32, 1, 32),
    ("transfer", False): (531, 14, 128),
}

LAYER_BOUNDS = {"eq": 4, "ne": 4, "gt": 6, "ge": 6, "lt": 6, "le": 6, "min": 8, "max": 8, "if_then_else": 2,
                "add": 7, "sub": 7, "neg": 7, "overflowing_add": 7, "overflowing_sub": 7, "bitand": 1,
                "bitor": 1, "bitxor": 1, "bitnot": 1, "transfer": 14}


def test_every_operation_is_pinned():
    assert {op for op, _ in PINNED} == set(R.OPERATIONS)


@pytest.mark.parametrize("op,signed", sorted(PINNED))
def test_pinned_schedule_counts(op, signed):
    s = bc.schedule(R.circuit(op, 32, signed), 1)
    assert (s.pbs_count(), s.num_layers, s.peak_slots) == PINNED[(op, signed)]


def test_schedule_depth_targets():
    """FheUint64 layer bounds: comparisons <= 6 (eq / ne <= 4), min / max <= 8,
    add / sub <= 7, transfer <= 14, whatever the signedness; the schedule
    serves any instance count with one compile"""
    for op in R.OPERATIONS:
        base = op[len("scalar_"):] if op.startswith("scalar_") else op
        for signed in (False, True):
            assert bc.schedule(R.circuit(op, 32, signed), 1).num_layers <= LAYER_BOUNDS[base], (op, signed)
    assert R.circuit("add", 32) is R.circuit("add", 32) is R.circuit("add", 32, True)
    s1, s7 = bc.schedule(R.circuit("transfer", 32), 1), bc.schedule(R.circuit("transfer", 32), 7)
    assert s7.pbs_count() == 7 * s1.pbs_count() and s1.pbs_shared_rows == 0
    # 64 blocks: one more scan / tree level
    assert bc.schedule(R.circuit("add", 64), 1).num_layers == 8
    assert bc.schedule(R.circuit("gt", 64), 1).num_layers == 7


# ---------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------
def test_argument_checks_raise_before_any_call():
    key = cleartext_key()
    u2, u3, s2 = ct([1, 2], 2), ct([1, 2], 3), ct([1, 2], 2, signed=True)
    u2_one = ct([5], 2)
    bad = [
        lambda: key.add(u2, u3),                   # block counts
        lambda: key.gt(u2, s2),                    # signedness
        lambda: key.eq(u2, u2_one),                # num_inputs
        lambda: key.if_then_else(boolean([1]), u2, u2),
        lambda: key.if_then_else(u2, u2, u2),
        lambda: key.transfer(s2, s2, s2),
        lambda: key.unsigned_overflowing_add(s2, s2),
        lambda: key.scalar_gt(u2, 16),             # out of [0, 16)
        lambda: key.scalar_gt(u2, -1),
        lambda: key.scalar_lt(s2, 8),              # out of [-8, 8)
        lambda: key.scalar_lt(s2, -9),
        lambda: key.scalar_eq(u2, [1, 2, 3]),
        lambda: key.scalar_eq(u2, 1.5),
        lambda: key.add(ct([0], 65), ct([0], 65)),
        lambda: key.add(integer.CudaUnsignedRadixCiphertext(u2.blocks, 3), integer.CudaUnsignedRadixCiphertext(
            u2.blocks, 3)),
        lambda: key.bitnot(u2.blocks),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert key.runner.calls == 0
    assert bools(key.scalar_lt(s2, -8)) == [0, 0] and bools(key.scalar_gt(u2, 15)) == [0, 0]
    for args in (("add", 0), ("add", 65), ("mul", 4)):
        with pytest.raises(ValueError):
            R.circuit(*args)
    # the radix runner needs a 2_2 key
    k = integer.CudaRadixServerKey.__new__(integer.CudaRadixServerKey)
    k.engine = types.SimpleNamespace(skey=types.SimpleNamespace(message_modulus=8, carry_modulus=8))
    with pytest.raises(ValueError, match="2_2"):
        k.add(u2, u2)


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def test_four_block_operations_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_aes: gt, signed lt, add and transfer on 4 blocks;
    every block decrypts exactly and holds <= 3."""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=43)
    rng = oracle.Rng(0x4AD1)
    n = 4

    def enc(*operands):
        digits = [d for vals in zip(*operands) for v in vals for d in R.to_digits(v, n)]
        return M.encrypt_bits(oracle, keys, rng, digits)

    def run(op, signed, *operands):
        s = bc.schedule(R.circuit(op, n, signed), len(operands[0]))
        out = run_oracle(oracle, keys, s, enc(*operands))
        return M.decrypt_messages(oracle, keys, out, vmax=3).reshape(len(operands[0]), -1)

    a, b = [200, 7, 99], [13, 7, 100]
    assert list(run("gt", False, a, b)[:, 0]) == [1, 0, 0]
    sa, sb = [-128, 5, -1], [127, -3, -1]
    assert list(run("lt", True, sa, sb)[:, 0]) == [1, 0, 0]
    assert [R.from_digits(r) for r in run("add", False, [250, 85], [9, 170])] == [3, 255]
    frm, to, amt = [100, 10], [5, 250], [40, 11]
    out = run("transfer", False, frm, to, amt)
    assert [(R.from_digits(r[:n]), R.from_digits(r[n:])) for r in out] == [(60, 45), (10, 250)]


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_radix(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0x4AD0 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    rk = integer.CudaRadixServerKey(skey, glwe_dimension=P.k, polynomial_size=P.N)
    rng = oracle.Rng(0x4AD2)

    def enc(values, n, signed=False):
        digits = [d for v in values for d in R.to_digits(int(v), n)]
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, digits).view(np.int64)).to(streams.device(0))
        kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
        return kind(t, len(values))

    def enc_bool(values):
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, values).view(np.int64)).to(streams.device(0))
        return integer.CudaBooleanBlock(t, len(values))

    def dec(x, signed=False):
        """copy on the caller's current stream, which waits for the work stream"""
        if isinstance(x, integer.CudaBooleanBlock):
            assert x.blocks.shape[0] == x.num_inputs
            return [int(v) for v in M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64))]
        d = M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64), vmax=3)
        return [R.from_digits(r, signed) for r in d.reshape(x.num_inputs, -1)]

    yield rk, enc, enc_bool, dec
    rk.runner.close()


def gpu_operands(n, signed, num_inputs, rng):
    """num_inputs (a, b) pairs: edge pairs first, then random ones"""
    pairs = edge_pairs(n, signed, rng)
    rand = [(rand_int(rng, n, signed), rand_int(rng, n, signed)) for _ in range(num_inputs)]
    if num_inputs == 1:
        return rand
    return rand[:2] + [pairs[int(i)] for i in rng.permutation(len(pairs))[:num_inputs - 2]]


@pytest.mark.gpu
@pytest.mark.parametrize("num_inputs", [1, 7])
@pytest.mark.parametrize("signed", [False, True])
def test_gpu_every_operation_fheuint64(gpu_radix, num_inputs, signed):
    rk, enc, enc_bool, dec = gpu_radix
    n = 32
    rng = np.random.default_rng(zlib.crc32(f"gpu{num_inputs}{signed}".encode()))
    a, b = map(list, zip(*gpu_operands(n, signed, num_inputs, rng)))
    A, B = enc(a, n, signed), enc(b, n, signed)
    for op in BINARY:
        out = getattr(rk, op)(A, B)
        got = dec(out) if op in CMP else dec(out, signed)
        assert got == [model(op, n, signed, x, y) for x, y in zip(a, b)], op
        if op in CMP:
            got = dec(getattr(rk, f"scalar_{op}")(A, b))
            assert got == [model(op, n, signed, x, y) for x, y in zip(a, b)], f"scalar_{op}"
    for op in ("neg", "bitnot"):
        assert dec(getattr(rk, op)(A), signed) == [model(op, n, signed, x) for x in a], op
    cond = [int(x) for x in rng.integers(0, 2, num_inputs)]
    assert dec(rk.if_then_else(enc_bool(cond), A, B), signed) == [x if c else y for c, x, y in zip(cond, a, b)]
    if not signed:
        for op in ("overflowing_add", "overflowing_sub"):
            out, flag = getattr(rk, f"unsigned_{op}")(A, B)
            assert list(zip(dec(out), dec(flag))) == [model(op, n, False, x, y) for x, y in zip(a, b)], op


@pytest.mark.gpu
def test_gpu_transfer_64_inputs(gpu_radix):
    """64 random transfers, with amount > from, amount == from and amount == 0
    among them"""
    rk, enc, _, dec = gpu_radix
    n = 32
    rng = np.random.default_rng(7984)
    frm = [int(x) for x in rng.integers(0, 1 << 62, 64)]
    to = [int(x) for x in rng.integers(0, 1 << 62, 64)]
    amt = [int(x) for x in rng.integers(0, 1 << 62, 64)]
    amt[0], amt[1], amt[2] = frm[0] + 1, frm[1], 0
    to[3] = 4 ** n - 1
    new_from, new_to = rk.transfer(enc(frm, n), enc(to, n), enc(amt, n))
    assert list(zip(dec(new_from), dec(new_to))) == [transfer_model(f, t, x, n) for f, t, x in zip(frm, to, amt)]


@pytest.mark.gpu
def test_gpu_64_block_add_and_gt(gpu_radix):
    rk, enc, _, dec = gpu_radix
    n = 64
    top = 4 ** n
    a = [R.from_digits([1] * n), top - 1, 12345 << 100]
    b = [R.from_digits([2] * n) + 1, 1, (12345 << 100) + (1 << 126)]
    A, B = enc(a, n), enc(b, n)
    assert dec(rk.add(A, B)) == [(x + y) % top for x, y in zip(a, b)]
    assert dec(rk.gt(A, B)) == [int(x > y) for x, y in zip(a, b)]


@pytest.mark.gpu
def test_gpu_unchecked_mul_into_gt(gpu_radix):
    """the products of unchecked_mul (one FheUint64 each) compared by gt"""
    rk, enc, _, dec = gpu_radix
    n = 32
    x, y, z = 0xDEADBEEF, 0x12345678, 0xFFFFFFFF
    prod_xy = rk.unchecked_mul(enc([x], n), enc([y], n))
    prod_zz = rk.unchecked_mul(enc([z], n), enc([z], n))
    assert dec(prod_xy) == [x * y % 4 ** n] and dec(prod_zz) == [z * z % 4 ** n]
    assert dec(rk.gt(prod_xy, prod_zz)) == [int(x * y > z * z)]
    assert dec(rk.gt(prod_zz, prod_xy)) == [int(z * z > x * y)]
