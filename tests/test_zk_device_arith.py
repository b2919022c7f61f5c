"""BLS12-446 field and curve arithmetic of csrc/bls12_446.cuh's device branch
(14 x u32 limbs, PTX carry chains) op by op against the plain-integer model.

The device code is not the code tests/test_zk_msm.py checks op by op: that
file runs the header's host branch (7 x u64 limbs, unsigned __int128) through
g++.  Here tests/emu/zk_device.cu includes the header unmodified, builds it
for sm_90a and exports batched field, point and window-digit calls.

CPU: a Python restatement of the device's CIOS rows, add, sub and final
subtraction, used only to prove that the crafted operand set reaches every
carry, borrow and final-subtraction edge listed in EDGES; the crafted set
also goes through the host build (tests/emu/libzk_host.so).
GPU: every Fp and Fp2 op on the crafted set and on 10^5 random pairs, the
XYZZ group law of G1 and G2 from normalised and non-normalised inputs, and
the window digits, all against the model.  Field elements are compared as
raw Montgomery words (the model computes a b R^-1 mod p and so on), so every
output word must match and every output must be fully reduced."""
import ctypes as C
import random

import numpy as np
import pytest

from tests import bls12_446_model as M
from tests.test_zk_msm import host  # noqa: F401  (the g++ build's fixture)

P = M.P
R = M.MONT_R
RINV = pow(R, -1, P)
M32 = (1 << 32) - 1
P32 = [(P >> (32 * j)) & M32 for j in range(14)]
PINV32 = M.PINV & M32
# the largest unreduced CIOS result (a b + m p) / R for a, b < p, m < R
T_MAX = ((P - 1) ** 2 + (R - 1) * P) // R
NEG_PINV_R = -pow(P, -1, R) % R  # -p^-1 mod R


def cios_t(a, b):
    """the unreduced CIOS result T = (a b + m p) / R, m = -a b p^-1 mod R"""
    return (a * b + (a * b * NEG_PINV_R % R) * P) // R


ADD, SUB, MUL, SQR, NEG, TO_MONT, FROM_MONT = 0, 1, 2, 3, 4, 6, 7


def model_fp(op, a, b):
    return {ADD: (a + b) % P, SUB: (a - b) % P, MUL: a * b * RINV % P, SQR: a * a * RINV % P, NEG: -a % P,
            TO_MONT: a * R % P, FROM_MONT: a * RINV % P}[op]


def model_fp2(op, a, b):
    if op == SQR:
        op, b = MUL, a
    if op == MUL:
        return ((a[0] * b[0] - a[1] * b[1]) * RINV % P, (a[0] * b[1] + a[1] * b[0]) * RINV % P)
    if op == NEG:
        return (-a[0] % P, -a[1] % P)
    return (model_fp(op, a[0], b[0]), model_fp(op, a[1], b[1]))


# ------------------------------------------- the device chains, restated ---

def _words(v):
    return [(v >> (32 * j)) & M32 for j in range(14)]


def _value(w):
    return sum(x << (32 * j) for j, x in enumerate(w))


class Edges:
    """The conditions a run reached: named events, and per chain the longest
    run of words a carry (or borrow) crossed on its own, i.e. carry in 1, the
    word's own sum 0xFFFFFFFF (its own difference 0), carry out 1."""

    def __init__(self):
        self.events, self.runs = set(), {}

    def run(self, chain, length):
        self.runs[chain] = max(self.runs.get(chain, 0), length)


def _add_chain(x, y, cin, ev, chain):
    out, c, run = [], cin, 0
    for xj, yj in zip(x, y):
        run = run + 1 if c and xj + yj == M32 else 0
        ev.run(chain, run)
        s = xj + yj + c
        out.append(s & M32)
        c = s >> 32
    return out, c


def _sub_chain(x, y, ev, chain):
    out, b, run = [], 0, 0
    for xj, yj in zip(x, y):
        run = run + 1 if b and xj == yj else 0
        ev.run(chain, run)
        d = xj - yj - b
        out.append(d & M32)
        b = 1 if d < 0 else 0
    return out, b


def _reduce_once(t, ev, tag):
    """reduce_once: t - p unless that borrows; also where the comparison with
    p was decided (the highest word where t and p differ)"""
    d, borrow = _sub_chain(t, P32, ev, f"{tag}_reduce")
    diff = [j for j in range(14) if t[j] != P32[j]]
    if diff and diff[-1] == 0:
        ev.events.add(f"{tag}_reduce_decided_at_word_0")
    ev.events.add(f"{tag}_reduce_{'kept' if borrow else 'subtracted'}")
    return t if borrow else d


def _mac_row(t, a, b, ev, tag):
    """mac_row / mac_row_p: t[0..14] += a[0..13] * b, a mad.lo chain ending in
    an addc into word 14, then a mad.hi chain ending in a madc.hi into word 14"""
    lo, c = _add_chain(t[:14], [(aj * b) & M32 for aj in a], 0, ev, f"mul_{tag}_lo")
    if c:
        ev.events.add(f"mul_{tag}_lo_carries_into_word_14")
    t[:14], t[14] = lo, t[14] + c
    assert t[14] <= M32
    hi, c = _add_chain(t[1:14], [(aj * b) >> 32 for aj in a[:13]], 0, ev, f"mul_{tag}_hi")
    if c:
        ev.events.add(f"mul_{tag}_hi_carries_into_word_14")
    t[1:14] = hi
    t[14] += ((a[13] * b) >> 32) + c
    assert t[14] <= M32, "a CIOS row overflowed 15 words"


def dev_mul(a, b, ev):
    x, y, t = _words(a), _words(b), [0] * 15
    for i in range(14):
        _mac_row(t, x, y[i], ev, "row")
        _mac_row(t, P32, (t[0] * PINV32) & M32, ev, "rowp")
        assert t[0] == 0
        t = t[1:] + [0]
        if i < 13 and _value(t) >= P:
            ev.events.add("mul_between_rows_t_at_least_p")
    T = _value(t)
    assert T == cios_t(a, b) and T < 2 * P
    if P - (1 << 32) <= T < P:
        ev.events.add("mul_T_just_below_p")
    if P <= T < P + (1 << 32):
        ev.events.add("mul_T_just_above_p")
    if T >= T_MAX - (T_MAX - P) // 64:
        ev.events.add("mul_T_near_its_largest")
    return _value(_reduce_once(t[:14], ev, "mul"))


def dev_add(a, b, ev):
    s, c = _add_chain(_words(a), _words(b), 0, ev, "add")
    assert c == 0
    for name, v in (("p-1", P - 1), ("p", P), ("p+1", P + 1), ("2p-2", 2 * P - 2)):
        if a + b == v:
            ev.events.add(f"add_sum_{name}")
    return _value(_reduce_once(s, ev, "add"))


def dev_sub(a, b, ev):
    d, borrow = _sub_chain(_words(a), _words(b), ev, "sub")
    s, _ = _add_chain(d, [pj if borrow else 0 for pj in P32], 0, ev, "sub_add_p")
    for name, v in (("0", 0), ("-1", -1), ("-(p-1)", -(P - 1))):
        if a - b == v:
            ev.events.add(f"sub_diff_{name}")
    return _value(s)


# every condition the crafted set must reach, and the longest carry run each
# chain must see (13 is a carry or borrow crossing every word above word 0)
EDGES = {"add_sum_p-1", "add_sum_p", "add_sum_p+1", "add_sum_2p-2", "add_reduce_kept", "add_reduce_subtracted",
         "add_reduce_decided_at_word_0", "sub_diff_0", "sub_diff_-1", "sub_diff_-(p-1)",
         "mul_row_lo_carries_into_word_14", "mul_row_hi_carries_into_word_14", "mul_rowp_lo_carries_into_word_14",
         "mul_rowp_hi_carries_into_word_14", "mul_between_rows_t_at_least_p", "mul_T_just_below_p",
         "mul_T_just_above_p", "mul_T_near_its_largest", "mul_reduce_kept", "mul_reduce_subtracted",
         "mul_reduce_decided_at_word_0"}
RUNS = {"add": 12, "add_reduce": 13, "sub": 13, "sub_add_p": 13, "mul_reduce": 13, "mul_row_lo": 1,
        "mul_rowp_lo": 2, "mul_rowp_hi": 12}


# ------------------------------------------------------ the crafted set ---

def crafted_values():
    """Raw Montgomery words: 0, 1, p - 1, p - 2, R mod p and, for every limb
    boundary j, 2^(32j) - 1, 2^(32j), p - 2^(32j), p with the words below j
    cleared, and p in every word above j with word j one less and all ones
    below."""
    v = {0, 1, 2, P - 1, P - 2, R % P, (R - 1) % P, P // 2, 1 << 445}
    for j in range(1, 14):
        v |= {(1 << (32 * j)) - 1, 1 << (32 * j), P - (1 << (32 * j)), P - 1 - ((1 << (32 * j)) - 1)}
    for j in range(14):
        high = P >> (32 * (j + 1)) << (32 * (j + 1))
        v |= {high, high + ((P32[j] - 1) << (32 * j)) + (1 << (32 * j)) - 1}
    return sorted(x for x in v if 0 <= x < P)


def _mul_search_pairs():
    """Mul pairs placing the unreduced CIOS result T = (a b + m p) / R just
    below p, just above p, and near its largest value T_MAX."""
    rng = random.Random(0x446)
    pairs = []
    # T = a b R^-1 mod p when that is the result just below p (T < p always
    # holds there: T - p would be > T_MAX - p)
    for r in (P - 1, P - 2, P - 0xaab0aaab):
        a = rng.randrange(1, P)
        pairs.append((a, r * R * pow(a, -1, P) % P))
    # a small result r is almost always reached as T = p + r
    for r in (1, 2, 0x554f5553):
        found = 0
        while found < 2:
            a = rng.randrange(1, P)
            b = r * R * pow(a, -1, P) % P
            if cios_t(a, b) >= P:
                pairs.append((a, b))
                found += 1
    # m = -a b p^-1 mod R close to R and a, b close to p: for a large odd a,
    # b = -m p a^-1 mod R, kept when it lands just below p
    found = 0
    for a in (P - 2, P - 0x10, P - (1 << 32)):
        ainv = pow(a, -1, R)
        for delta in range(1, 1 << 16, 2):
            b = (-(R - delta) * P * ainv) % R
            if P - P // 64 <= b < P:
                pairs.append((a, b))
                found += 1
                break
    assert found == 3
    return pairs


def crafted_pairs():
    """{op: [(a, b)]} for add, sub and mul."""
    vals = crafted_values()
    cross = [(a, b) for a in vals for b in vals]
    add = list(cross)
    for s in (P - 1, P, P + 1, 2 * P - 2):
        add += [(a, s - a) for a in vals if 0 <= s - a < P]
    sub = list(cross)
    for d in (0, -1, -(P - 1)):
        sub += [(a, a - d) for a in vals if 0 <= a - d < P]
    return {ADD: add, SUB: sub, MUL: cross + _mul_search_pairs()}


def crafted_fp2():
    """Fp2 elements from the crafted values, plus a0 + a1 = p (the Karatsuba
    sum wraps to 0), a0 = a1 (the squaring's a0 - a1 is 0) and a0 + a1 = p +- 1."""
    vals = crafted_values()
    picks = vals[::3] + [P - 1, 1, 0]
    elems = [(a, b) for a in picks for b in picks]
    for a in vals:
        elems += [(a, a)] + [(a, s - a) for s in (P - 1, P, P + 1) if 0 <= s - a < P]
    return elems


def _emulate(pairs):
    ev = Edges()
    for op, lst in pairs.items():
        fn = {ADD: dev_add, SUB: dev_sub, MUL: dev_mul}[op]
        for a, b in lst:
            assert fn(a, b, ev) == model_fp(op, a, b), (op, hex(a), hex(b))
    return ev


# ------------------------------------------------------------------ CPU ---

def test_the_restated_chains_compute_the_model():
    rng = random.Random(9)
    pairs = [(rng.randrange(P), rng.randrange(P)) for _ in range(300)]
    _emulate({ADD: pairs, SUB: pairs, MUL: pairs})


def test_crafted_set_reaches_every_carry_edge():
    """If the crafted set is trimmed, an edge of the device chains goes
    untested on the GPU; this names it."""
    ev = _emulate(crafted_pairs())
    assert EDGES <= ev.events, sorted(EDGES - ev.events)
    short = {k: (ev.runs.get(k, 0), need) for k, need in RUNS.items() if ev.runs.get(k, 0) < need}
    assert not short, short


def test_random_pairs_rarely_reach_the_edges():
    """The edges are not what random operands give: 300 random pairs miss the
    value edges and every long carry run."""
    rng = random.Random(10)
    pairs = [(rng.randrange(P), rng.randrange(P)) for _ in range(300)]
    ev = _emulate({ADD: pairs, SUB: pairs, MUL: pairs})
    rare = {e for e in EDGES if "sum_" in e or "diff_" in e or "T_just" in e or "decided" in e}
    assert not rare & ev.events, sorted(rare & ev.events)
    assert all(ev.runs.get(k, 0) < 4 for k in ("add", "sub", "sub_add_p", "add_reduce", "mul_reduce"))


def _enc(vals):
    """uint64 limbs of a sequence of ints (Fp) or of (c0, c1) tuples (Fp2)"""
    flat = [x for v in vals for x in (v if isinstance(v, tuple) else (v,))]
    return np.frombuffer(b"".join(x.to_bytes(56, "little") for x in flat), dtype=np.uint64).copy()


def _dec(arr, degree=1):
    raw = np.ascontiguousarray(arr, dtype=np.uint64).tobytes()
    flat = [int.from_bytes(raw[i:i + 56], "little") for i in range(0, len(raw), 56)]
    return flat if degree == 1 else [tuple(flat[i:i + degree]) for i in range(0, len(flat), degree)]


def test_host_build_on_the_crafted_set(host):
    out = np.zeros(7, np.uint64)
    pairs = crafted_pairs()
    for op, lst in pairs.items():
        for a, b in lst:
            ea, eb = _enc([a]), _enc([b])
            host.zk_fp_op(op, out.ctypes.data, ea.ctypes.data, eb.ctypes.data)
            assert _dec(out)[0] == model_fp(op, a, b), (op, hex(a), hex(b))
    for a in crafted_values():
        for op in (SQR, NEG, TO_MONT, FROM_MONT):
            ea = _enc([a])
            host.zk_fp_op(op, out.ctypes.data, ea.ctypes.data, ea.ctypes.data)
            assert _dec(out)[0] == model_fp(op, a, a), (op, hex(a))
    out2 = np.zeros(14, np.uint64)
    elems = crafted_fp2()
    rng = random.Random(12)
    for a in elems:
        b = rng.choice(elems)
        for op in (ADD, SUB, MUL, SQR, NEG):
            ea, eb = _enc([a]), _enc([b])
            host.zk_fp2_op(op, out2.ctypes.data, ea.ctypes.data, eb.ctypes.data)
            assert tuple(_dec(out2)) == model_fp2(op, a, b), (op, a, b)


# ------------------------------------------------------------------ GPU ---

@pytest.fixture(scope="module")
def dev():
    """tests/emu/libzk_device.so, built by __graft_entry__.build() (rebuilt
    here when a source is newer); a missing library fails the tests."""
    from tests.emu.build_zk_device import build

    lib = C.CDLL(build())
    vp, i, u = C.c_void_p, C.c_int, C.c_uint32
    for name in ("zk_dev_fp_op", "zk_dev_fp2_op", "zk_dev_g1_op", "zk_dev_g2_op"):
        getattr(lib, name).argtypes = [i, u, vp, vp, vp]
        getattr(lib, name).restype = i
    lib.zk_dev_signed_digits.argtypes = [u, vp, vp, i]
    lib.zk_dev_signed_digits.restype = i
    return lib


def _dev_field(dev, degree, op, a, b):
    n = len(a)
    ea, eb = _enc(a), _enc(b)
    out = np.zeros_like(ea)
    fn = dev.zk_dev_fp_op if degree == 1 else dev.zk_dev_fp2_op
    assert fn(op, n, out.ctypes.data, ea.ctypes.data, eb.ctypes.data) == 0
    return _dec(out, degree)


def _check_field(dev, degree, op, a, b):
    got = _dev_field(dev, degree, op, a, b)
    model = model_fp if degree == 1 else model_fp2
    bad = [(x, y, g) for x, y, g in zip(a, b, got) if g != model(op, x, y)]
    assert not bad, (op, len(bad), bad[:3])


@pytest.mark.gpu
def test_fp_crafted_operands(dev):
    for op, lst in crafted_pairs().items():
        _check_field(dev, 1, op, [a for a, _ in lst], [b for _, b in lst])
    vals = crafted_values()
    for op in (SQR, NEG, TO_MONT, FROM_MONT):
        _check_field(dev, 1, op, vals, vals)


@pytest.mark.gpu
@pytest.mark.parametrize("op", [ADD, SUB, MUL, SQR, NEG, TO_MONT, FROM_MONT])
def test_fp_random_operands(dev, op):
    rng = random.Random(100 + op)
    n = 100_000
    a = [rng.randrange(P) for _ in range(n)]
    b = [rng.randrange(P) for _ in range(n)]
    _check_field(dev, 1, op, a, b)


@pytest.mark.gpu
def test_fp_rejects_the_host_only_inverse(dev):
    z = _enc([1])
    assert dev.zk_dev_fp_op(5, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data) != 0


@pytest.mark.gpu
@pytest.mark.parametrize("op", [ADD, SUB, MUL, SQR, NEG])
def test_fp2_crafted_and_random_operands(dev, op):
    rng = random.Random(200 + op)
    elems = crafted_fp2()
    a = elems + [(rng.randrange(P), rng.randrange(P)) for _ in range(20_000)]
    b = [rng.choice(elems) for _ in elems] + [(rng.randrange(P), rng.randrange(P)) for _ in range(20_000)]
    # every crafted element against every crafted special case, too
    specials = [e for e in elems if e[0] == e[1] or e[0] + e[1] in (P - 1, P, P + 1)]
    a += [x for x in specials for _ in range(3)]
    b += [y for _ in specials for y in rng.sample(specials, 3)]
    _check_field(dev, 2, op, a, b)


# ---- points: raw XYZZ (X, Y, ZZ, ZZZ) in Montgomery form ----

def _mont(v, degree):
    return v * R % P if degree == 1 else (v[0] * R % P, v[1] * R % P)


def _unmont(v, degree):
    return v * RINV % P if degree == 1 else (v[0] * RINV % P, v[1] * RINV % P)


def _xyzz(curve, pt, t):
    """pt (affine, or None for the identity) as XYZZ (x t^2, y t^3, t^2, t^3)"""
    F, degree = curve.F, 1 if curve is M.G1 else 2
    if pt is None:
        return (F.zero,) * 4 if degree == 1 else ((0, 0),) * 4
    t2 = F.mul(t, t)
    t3 = F.mul(t2, t)
    return tuple(_mont(v, degree) for v in (F.mul(pt[0], t2), F.mul(pt[1], t3), t2, t3))


def _affine(curve, raw):
    """(x, y) of a raw XYZZ output, None for the identity; checks that ZZ^3 =
    ZZZ^2 and that every coordinate is fully reduced"""
    F, degree = curve.F, 1 if curve is M.G1 else 2
    flat = [x for v in raw for x in (v if degree == 2 else (v,))]
    assert all(x < P for x in flat), "an output coordinate is not fully reduced"
    X, Y, ZZ, ZZZ = (_unmont(v, degree) for v in raw)
    if ZZ == F.zero:
        assert ZZZ == F.zero
        return None
    assert F.mul(F.mul(ZZ, ZZ), ZZ) == F.mul(ZZZ, ZZZ), "ZZ^3 != ZZZ^2"
    return F.mul(X, F.inv(ZZ)), F.mul(Y, F.inv(ZZZ))


def _point_cases(curve, rng):
    """[(p as XYZZ, q as XYZZ, p affine, q affine)]: generic sums, the same
    point in two XYZZ representations added to itself and to its negation
    (the doubling and identity branches of xyzz_add from non-normalised
    inputs), against its own affine form, and the identity on either side"""
    F = curve.F
    one = F.one

    def scale():
        return rng.randrange(2, P) if curve is M.G1 else (rng.randrange(P), rng.randrange(1, P))

    Pp = curve.mul(rng.randrange(1, M.R_ORDER), curve.gen)
    Q = curve.mul(rng.randrange(1, M.R_ORDER), curve.gen)
    cases = []
    for p, q in [(Pp, Q), (Pp, Pp), (Pp, curve.neg(Pp)), (None, Pp), (Pp, None), (None, None), (Q, Pp)]:
        cases.append((_xyzz(curve, p, one), _xyzz(curve, q, one), p, q))  # the cases of the host test
        cases.append((_xyzz(curve, p, scale()), _xyzz(curve, q, scale()), p, q))
        cases.append((_xyzz(curve, p, scale()), _xyzz(curve, q, one), p, q))
    if curve is M.G1:
        # (-1, 0) has order 2: its doubling, and T + T, are the identity
        T2 = (P - 1, 0)
        assert curve.on_curve(T2)
        cases.append((_xyzz(curve, T2, scale()), _xyzz(curve, T2, one), T2, T2))
        cases.append((_xyzz(curve, T2, one), _xyzz(curve, T2, scale()), T2, T2))
    return cases


def _dev_points(dev, curve, mode, ps, qs):
    degree = 1 if curve is M.G1 else 2
    ea, eb = _enc([x for p in ps for x in p]), _enc([x for q in qs for x in q])
    out = np.zeros_like(ea)
    fn = dev.zk_dev_g1_op if curve is M.G1 else dev.zk_dev_g2_op
    assert fn(mode, len(ps), out.ctypes.data, ea.ctypes.data, eb.ctypes.data) == 0
    flat = _dec(out, degree)
    return [tuple(flat[4 * i:4 * i + 4]) for i in range(len(ps))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
def test_group_law_on_the_device(dev, name):
    curve = M.G1 if name == "g1" else M.G2
    F = curve.F
    cases = _point_cases(curve, random.Random(30))
    ps, qs = [c[0] for c in cases], [c[1] for c in cases]
    # 1: XYZZ + XYZZ, 2: doubling
    for mode, expect in ((1, [curve.add(c[2], c[3]) for c in cases]), (2, [curve.add(c[2], c[2]) for c in cases])):
        got = _dev_points(dev, curve, mode, ps, qs)
        for i, (g, e) in enumerate(zip(got, expect)):
            assert _affine(curve, g) == e, (mode, i)
    # 0: mixed addition of q's affine form (never the identity)
    mixed = [c for c in cases if c[3] is not None]
    got = _dev_points(dev, curve, 0, [c[0] for c in mixed], [_xyzz(curve, c[3], F.one) for c in mixed])
    for i, (g, c) in enumerate(zip(got, mixed)):
        assert _affine(curve, g) == curve.add(c[2], c[3]), (0, i)
    # 3: (X ZZZ, Y ZZ, ZZ ZZZ), the identity (0, 0, 0)
    degree = 1 if name == "g1" else 2
    got = _dev_points(dev, curve, 3, ps, qs)
    for i, (g, c) in enumerate(zip(got, cases)):
        X, Y, Z, rest = (_unmont(v, degree) for v in g)
        assert rest == F.zero and all(x < P for v in g for x in (v if degree == 2 else (v,)))
        if c[2] is None:
            assert X == Y == Z == F.zero, i
        else:
            zi = F.inv(Z)
            assert (F.mul(X, zi), F.mul(Y, zi)) == c[2], (3, i)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
def test_chained_additions_on_the_device(dev, name):
    """Non-normalised accumulators as the bucket kernels build them: k P by
    repeated mixed additions, then added to j P (the doubling branch when j = k)
    and to -j P (the identity)."""
    curve = M.G1 if name == "g1" else M.G2
    F = curve.F
    rng = random.Random(31)
    G = curve.mul(rng.randrange(1, M.R_ORDER), curve.gen)
    ks = [2, 3, 5, 8]
    acc = [_xyzz(curve, G, F.one) for _ in ks]
    for step in range(1, max(ks)):
        live = [i for i, k in enumerate(ks) if step < k]
        got = _dev_points(dev, curve, 0, [acc[i] for i in live], [_xyzz(curve, G, F.one)] * len(live))
        for i, g in zip(live, got):
            acc[i] = g
    for k, a in zip(ks, acc):
        assert _affine(curve, a) == curve.mul(k, G)
    for other in ks:
        got = _dev_points(dev, curve, 1, acc, [acc[ks.index(other)]] * len(ks))
        for k, g in zip(ks, got):
            assert _affine(curve, g) == curve.mul(k + other, G), (k, other)
    neg = [(a[0], _mont(F.neg(_unmont(a[1], 1 if name == "g1" else 2)), 1 if name == "g1" else 2), a[2], a[3])
           for a in acc]
    got = _dev_points(dev, curve, 1, acc, neg)
    assert all(_affine(curve, g) is None for g in got)


@pytest.mark.gpu
@pytest.mark.parametrize("c", range(4, 17))
def test_signed_digits_on_the_device(dev, host, c):
    r, top = M.R_ORDER, (1 << 320) - 1
    rng = random.Random(40 + c)
    ks = [0, 1, 2, r - 1, r, r + 1, top, top - 1, 1 << 319, (1 << 320) - (1 << 300), 0x80 << 312,
          sum(((1 << (c - 1)) + 1) << (c * w) for w in range(320 // c))] + [rng.getrandbits(320) for _ in range(500)]
    ks = [k % (1 << 320) for k in ks]
    W = 320 // c + 1
    scal = np.frombuffer(b"".join(k.to_bytes(40, "little") for k in ks), dtype=np.uint64).copy()
    out = np.zeros(len(ks) * W, np.int32)
    assert dev.zk_dev_signed_digits(len(ks), out.ctypes.data, scal.ctypes.data, c) == 0
    out = out.reshape(len(ks), W)
    expect = np.zeros(W, np.int32)
    half = 1 << (c - 1)
    for i, k in enumerate(ks):
        host.zk_signed_digits(expect.ctypes.data, scal[5 * i:5 * i + 5].ctypes.data, c)
        assert np.array_equal(out[i], expect), (c, i)
        assert sum(int(d) << (c * w) for w, d in enumerate(out[i])) == k
        assert all(-half < int(d) <= half for d in out[i])
