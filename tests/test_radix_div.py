"""Division and remainder of radix integers (tfhe-rs_b200/radix_div.py and the
division methods of integer.CudaRadixServerKey).

CPU: every division through the server key's host code on a cleartext runner
(the compiled schedules on `bit_circuit.run_cleartext`, which asserts the
noise budget and the value range on every row), exhaustively at 1, 2 and 3
blocks, unsigned and signed, by encrypted and by every clear divisor, and on
edge values at 32 and 64 blocks, against the plain model
`radix_div.model`; the pinned FheUint64 schedule counts; argument checks;
unsigned and signed div_rem through real LWE keyswitches and PBS on the
oracle.

GPU: `CudaRadixServerKey` on classic P22 and multi-bit g = 4: FheUint64
divisions at 1 and 7 inputs, one FheUint128 div_rem, and a quotient chained
into add and gt; every output block decrypts to the model's value."""
import itertools
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import bit_circuit as bc, integer, radix as R, radix_div as D

from tests import trivium_model as M
from tests.test_radix import cleartext_key, ct, ints, rand_int, wrap
from tests.test_trivium import run_oracle


def div_ops(key, op, a, b, n, signed, scalar):
    """(quotients, remainders) of op on lists of integers through the server
    key (None for the half op does not output)"""
    A = ct(a, n, signed)
    if scalar:
        out = getattr(key, f"scalar_{op}")(A, list(b))
    else:
        out = getattr(key, op)(A, ct(b, n, signed))
    if op == "div_rem":
        return ints(out[0], signed), ints(out[1], signed)
    return (ints(out, signed), None) if op == "div" else (None, ints(out, signed))


def check_all(key, a, b, n, signed, scalar):
    want = [D.model(x, y, n, signed) for x, y in zip(a, b)]
    q, r = div_ops(key, "div_rem", a, b, n, signed, scalar)
    assert list(zip(q, r)) == want, (n, signed, scalar)
    assert div_ops(key, "div", a, b, n, signed, scalar)[0] == q
    assert div_ops(key, "rem", a, b, n, signed, scalar)[1] == r


# ---------------------------------------------------------------------------
# the plain model
# ---------------------------------------------------------------------------
def test_model():
    assert D.model(7, 2, 2) == (3, 1) and D.model(7, 0, 2) == (15, 7)
    assert D.model(-7, 2, 2, True) == (-3, -1) and D.model(7, -2, 2, True) == (-3, 1)
    assert D.model(-8, -1, 2, True) == (-8, 0)                       # MIN / -1 wraps
    assert D.model(5, 0, 2, True) == (-1, 5) and D.model(0, 0, 2, True) == (-1, 0)
    assert D.model(-5, 0, 2, True) == (1, -5)


# ---------------------------------------------------------------------------
# exhaustive at 1, 2 and 3 blocks
# ---------------------------------------------------------------------------
def domain(n, signed):
    lo, hi = R.scalar_range(n, signed)
    return list(range(lo, hi))


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_division(n, signed):
    """every (n, d) pair, d = 0 included, as instances of one call (3 blocks:
    4,096 pairs)"""
    key = cleartext_key()
    vals = domain(n, signed)
    a, b = zip(*itertools.product(vals, vals))
    check_all(key, a, b, n, signed, scalar=False)


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("signed", [False, True])
def test_exhaustive_scalar_division(n, signed):
    """every numerator by every in-range non-zero clear divisor, one divisor
    per input; and one divisor given once for every input"""
    key = cleartext_key()
    vals = domain(n, signed)
    a, b = zip(*itertools.product(vals, [v for v in vals if v]))
    check_all(key, a, b, n, signed, scalar=True)
    d = vals[-1]
    q, r = key.scalar_div_rem(ct(vals, n, signed), d)
    assert list(zip(ints(q, signed), ints(r, signed))) == [D.model(x, d, n, signed) for x in vals]


# ---------------------------------------------------------------------------
# edge values at 32 and 64 blocks
# ---------------------------------------------------------------------------
def edge_pairs(n, signed, rng):
    """0, 1, max, MIN, -1, powers of two and random values, each divided by
    0, 1, -1, max, MIN, itself, a larger value, powers of two and random
    values"""
    lo, hi = R.scalar_range(n, signed)
    rand = [rand_int(rng, n, signed) for _ in range(3)]
    small = [wrap(int(x), n, signed) for x in rng.integers(1, 1 << 20, 2)]
    nums = sorted({0, 1, hi - 1, lo, wrap(-1, n, signed), 1 << (n - 1), 1 << (2 * n - 3)} | set(rand))
    dens = sorted({0, 1, wrap(-1, n, signed), hi - 1, lo, 2, 1 << n, 1 << (2 * n - 2)} | set(rand) | set(small))
    pairs = [(x, y) for x in nums for y in dens]
    pairs += [(x, x) for x in nums]                                          # d == n
    pairs += [(x, wrap(x + 1, n, signed)) for x in rand + small if x + 1 < hi]   # d > n
    return pairs


@pytest.mark.parametrize("n", [32, 64])
@pytest.mark.parametrize("signed", [False, True])
def test_edges_at_wide_integers(n, signed):
    rng = np.random.default_rng(zlib.crc32(f"div{n}{signed}".encode()))
    key = cleartext_key()
    a, b = zip(*edge_pairs(n, signed, rng))
    want = [D.model(x, y, n, signed) for x, y in zip(a, b)]
    q, r = div_ops(key, "div_rem", a, b, n, signed, False)
    assert list(zip(q, r)) == want
    nz = [(x, y) for x, y in zip(a, b) if y]
    sa, sb = zip(*nz)
    q, r = div_ops(key, "div_rem", sa, sb, n, signed, True)
    assert list(zip(q, r)) == [D.model(x, y, n, signed) for x, y in nz]
    if n == 32:
        assert div_ops(key, "div", a, b, n, signed, False)[0] == [w[0] for w in want]
        assert div_ops(key, "rem", a, b, n, signed, False)[1] == [w[1] for w in want]
        assert div_ops(key, "div", sa, sb, n, signed, True)[0] == [D.model(x, y, n, signed)[0] for x, y in nz]
        assert div_ops(key, "rem", sa, sb, n, signed, True)[1] == [D.model(x, y, n, signed)[1] for x, y in nz]


# ---------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------
# (PBS count, PBS layers, peak slots) of one FheUint64 (32 blocks) instance;
# recorded in DESIGN §8l
PINNED = {
    ("div_rem", False): (13378, 236, 415), ("div", False): (13346, 235, 415), ("rem", False): (13346, 236, 415),
    ("scalar_div_rem", False): (12832, 226, 255), ("scalar_div", False): (12800, 225, 255),
    ("scalar_rem", False): (12800, 226, 224),
    ("div_rem", True): (14251, 250, 431), ("div", True): (14001, 248, 430), ("rem", True): (14000, 250, 430),
    ("scalar_div_rem", True): (13487, 240, 287), ("scalar_div", True): (13237, 238, 286),
    ("scalar_rem", True): (13236, 240, 225),
}


def test_every_division_is_pinned():
    assert {op for op, _ in PINNED} == set(D.OPERATIONS)


@pytest.mark.parametrize("op,signed", sorted(PINNED))
def test_pinned_schedule_counts(op, signed):
    s = bc.schedule(D.circuit(op, 32, signed), 1)
    assert (s.pbs_count(), s.num_layers, s.peak_slots) == PINNED[(op, signed)]
    assert s.pbs_shared_rows == 0


def test_schedule_bounds():
    """FheUint64 unsigned div_rem: <= 13,592 PBS and <= 274 layers (tfhe-rs'
    algorithm restated without folding); signed <= 300 layers; one compile
    serves every instance count; the circuits are cached per (op, blocks,
    signed)"""
    s = bc.schedule(D.circuit("div_rem", 32), 1)
    assert s.pbs_count() <= 13592 and s.num_layers <= 274
    assert bc.schedule(D.circuit("div_rem", 32, True), 1).num_layers <= 300
    assert bc.schedule(D.circuit("div_rem", 32), 7).pbs_count() == 7 * s.pbs_count()
    assert D.circuit("div_rem", 32) is D.circuit("div_rem", 32)
    assert D.circuit("div_rem", 32) is not D.circuit("div_rem", 32, True)
    # the fixed LUT set is unchanged: division tables are circuit-local
    assert bc.NUM_FIXED_LUTS == 11 and len(s.extra_luts) > 0


# ---------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------
def test_argument_checks_raise_before_any_call():
    key = cleartext_key()
    u2, u3, s2 = ct([1, 2], 2), ct([1, 2], 3), ct([1, 2], 2, signed=True)
    bad = [
        lambda: key.div_rem(u2, u3),               # block counts
        lambda: key.div(u2, s2),                   # signedness
        lambda: key.rem(u2, ct([5], 2)),           # num_inputs
        lambda: key.div_rem(u2, u2.blocks),
        lambda: key.scalar_div_rem(u2, 0),         # attempt to divide by 0
        lambda: key.scalar_div(s2, [1, 0]),
        lambda: key.scalar_rem(u2, 16),            # out of [0, 16)
        lambda: key.scalar_rem(u2, -1),
        lambda: key.scalar_div(s2, 8),             # out of [-8, 8)
        lambda: key.scalar_div(s2, -9),
        lambda: key.scalar_div_rem(u2, [1, 2, 3]),
        lambda: key.scalar_div_rem(u2, 1.5),
        lambda: key.scalar_div_rem(u2, True),
        lambda: key.div_rem(ct([0], 65), ct([1], 65)),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert key.runner.calls == 0
    with pytest.raises(ValueError, match="divide by 0"):
        key.scalar_div_rem(u2, 0)
    for args in (("div_rem", 0), ("div_rem", 65), ("mod", 4)):
        with pytest.raises(ValueError):
            D.circuit(*args)
    q, r = key.scalar_div_rem(s2, -8)
    assert ints(q, True) == [0, 0] and ints(r, True) == [1, 2]


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def test_three_block_division_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_radix: unsigned and signed div_rem, /0 and
    MIN / -1 among the cases; every block decrypts exactly and holds <= 3."""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=47)
    rng = oracle.Rng(0xD1F)
    n = 3

    def run(op, signed, a, b):
        s = bc.schedule(D.circuit(op, n, signed), len(a))
        if op.startswith("scalar_"):
            digits, iconsts = [d for v in a for d in R.to_digits(v, n)], D.scalar_iconsts(b, n, signed)
        else:
            digits = [d for x, y in zip(a, b) for v in (x, y) for d in R.to_digits(v, n)]
            iconsts = None
        out = run_oracle(oracle, keys, s, M.encrypt_bits(oracle, keys, rng, digits), iconsts)
        rows = M.decrypt_messages(oracle, keys, out, vmax=3).reshape(len(a), -1)
        return [(R.from_digits(r[:n], signed), R.from_digits(r[n:], signed)) for r in rows]

    a, b = [63, 50, 7], [5, 0, 63]
    assert run("div_rem", False, a, b) == [D.model(x, y, n) for x, y in zip(a, b)]
    a, b = [-32, -32, 31, -7], [-1, 0, 0, 2]
    assert run("div_rem", True, a, b) == [D.model(x, y, n, True) for x, y in zip(a, b)]
    a, b = [-32, 29], [-1, -4]
    assert run("scalar_div_rem", True, a, b) == [D.model(x, y, n, True) for x, y in zip(a, b)]


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_div(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0xD100 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    rk = integer.CudaRadixServerKey(skey, glwe_dimension=P.k, polynomial_size=P.N)
    rng = oracle.Rng(0xD102)

    def enc(values, n, signed=False):
        digits = [d for v in values for d in R.to_digits(int(v), n)]
        t = torch.from_numpy(M.encrypt_bits(oracle, keys, rng, digits).view(np.int64)).to(streams.device(0))
        kind = integer.CudaSignedRadixCiphertext if signed else integer.CudaUnsignedRadixCiphertext
        return kind(t, len(values))

    def dec(x, signed=False):
        """copy on the caller's current stream, which waits for the work stream"""
        if isinstance(x, integer.CudaBooleanBlock):
            return [int(v) for v in M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64))]
        d = M.decrypt_messages(oracle, keys, x.blocks.cpu().numpy().view(np.uint64), vmax=3)
        return [R.from_digits(r, signed) for r in d.reshape(x.num_inputs, -1)]

    yield rk, enc, dec
    rk.runner.close()


def gpu_pairs(n, signed, num_inputs, rng):
    """num_inputs (numerator, divisor) pairs: at one input a random pair;
    else random pairs, /0, d == n, d > n, and (signed) MIN / -1, then edge
    pairs"""
    rand = [(rand_int(rng, n, signed), wrap(int(rng.integers(1, 1 << 40)), n, signed)) for _ in range(2)]
    if num_inputs == 1:
        return rand[:1]
    lo, hi = R.scalar_range(n, signed)
    fixed = [(12345, 0), (hi - 1, hi - 1), (77, 78), (lo, wrap(-1, n, signed)) if signed else (hi - 1, 1)]
    pairs = [p for p in edge_pairs(n, signed, rng) if p[1]]
    return (rand + fixed + [pairs[int(i)] for i in rng.permutation(len(pairs))])[:num_inputs]


@pytest.mark.gpu
@pytest.mark.parametrize("num_inputs", [1, 7])
@pytest.mark.parametrize("signed", [False, True])
def test_gpu_division_fheuint64(gpu_div, num_inputs, signed):
    rk, enc, dec = gpu_div
    n = 32
    rng = np.random.default_rng(zlib.crc32(f"gpudiv{num_inputs}{signed}".encode()))
    a, b = map(list, zip(*gpu_pairs(n, signed, num_inputs, rng)))
    A, B = enc(a, n, signed), enc(b, n, signed)
    want = [D.model(x, y, n, signed) for x, y in zip(a, b)]
    q, r = rk.div_rem(A, B)
    assert list(zip(dec(q, signed), dec(r, signed))) == want
    assert dec(rk.div(A, B), signed) == [w[0] for w in want]
    assert dec(rk.rem(A, B), signed) == [w[1] for w in want]
    # clear divisors: the zero divisor replaced by 3
    s = [y if y else 3 for y in b]
    want = [D.model(x, y, n, signed) for x, y in zip(a, s)]
    q, r = rk.scalar_div_rem(A, s)
    assert list(zip(dec(q, signed), dec(r, signed))) == want
    assert dec(rk.scalar_div(A, s), signed) == [w[0] for w in want]
    assert dec(rk.scalar_rem(A, s), signed) == [w[1] for w in want]


@pytest.mark.gpu
def test_gpu_fheuint128_div_rem(gpu_div):
    rk, enc, dec = gpu_div
    n = 64
    a, b = [(0xDEADBEEF << 96) + 0x1234567], [(0xCAFE << 40) + 99]
    q, r = rk.div_rem(enc(a, n), enc(b, n))
    assert (dec(q), dec(r)) == ([a[0] // b[0]], [a[0] % b[0]])


@pytest.mark.gpu
def test_gpu_quotient_into_add_and_gt(gpu_div):
    """a quotient and a remainder are clean blocks: fed into add and gt"""
    rk, enc, dec = gpu_div
    n = 32
    a, b, c = [10 ** 18, 999], [7, 1000], [142857142857142857, 5]
    q, r = rk.div_rem(enc(a, n), enc(b, n))
    C = enc(c, n)
    assert dec(rk.add(q, r)) == [(x // y + x % y) % 4 ** n for x, y in zip(a, b)]
    assert dec(rk.gt(q, C)) == [int(x // y > z) for x, y, z in zip(a, b, c)]
