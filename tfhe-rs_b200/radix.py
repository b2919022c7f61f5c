"""Radix-integer circuits on 2_2 message blocks, compiled to batched KS -> PBS
layers by `bit_circuit`: comparisons, selects, additions, subtractions and
bitwise operations, and erc7984's confidential-token transfer.  Host code
only: the GPU runs them with `b200_bit_circuit_64_async` through
`integer.CudaRadixServerKey`.

Blocks are 2_2 message blocks (values 0..3), least significant first (tfhe-rs
radix order).  A signed integer is two's complement over all its blocks, the
sign being bit 1 of the top block.  Every PBS input is a linear step inside
the 2_2 noise budget (sum |c_i| <= 5, value in [0, 15], `bit_circuit`), and
every output block is a PBS output holding a value <= 3, so results chain into
any operation here and into `integer.unchecked_mul`.

The builders add gates to a `bit_circuit.Circuit` and return wire lists, so
they compose; an operand block is a list of (wire, coef) terms giving its
value (one client block, or the two bits of a clear digit entering as
per-instance body constants).  Circuits:

  * block sign {INFERIOR, EQUAL, SUPERIOR} = one PBS on 4 l + r (noise 5,
    value <= 15); the top block of a signed integer compares its 2-bit
    two's-complement digits (tfhe-rs `compare_blocks_with_sign_bit`);
  * ordering: a binary tree of PBS on 4 msb + lsb (value <= 10, tfhe-rs
    `reduce_two_orderings_function`), the final boolean folded into the last
    reduction's table;
  * equality: block equality bits on 4 l + r, then sums of <= 5 bits reduced
    by [x == count] (32 -> 7 -> 2 -> 1 blocks);
  * select: 4 cond + x -> x or 0 (noise 5), and the two halves of
    `if_then_else` summed by one identity PBS (noise 2);
  * add / sub: the message (a + b) mod 4 and the carry state of a + b
    (sub: a + 3 - b, + 1 into block 0), a Hillis-Steele scan of the states
    with `integer`'s combine table on 4 cur + prev, and one PBS per block on
    m_i + 4 state_{i-1} (noise 5, value <= 11); the carry out is folded into
    the scan's last combine of the top block;
  * signed overflow of add / sub: one PBS on 4 a_top + b_top (sub: 3 - b_top)
    gives a code {never, iff carry, iff no carry, always}, and one PBS on
    4 code + state_{n-2}, beside the last layer, the flag;
  * abs: `radix_div.cond_negate` on the sign block.
"""
from __future__ import annotations

import functools
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import bit_circuit as bc
from . import integer

MSG_MOD = integer.MSG_MOD
INFERIOR, EQUAL, SUPERIOR = 0, 1, 2   # tfhe-rs' block orderings
MAX_BLOCKS = 64
CIRCUIT_CACHE_SIZE = 32               # compiled (operation, num_blocks, signed) circuits kept

_INT_LUTS = integer.lut_functions()
MSG_TABLE = _INT_LUTS[integer.LUT_MSG]            # x mod 4
STATE_TABLE = _INT_LUTS[integer.LUT_STATE]        # carry state of a block sum
COMBINE_TABLE = _INT_LUTS[integer.LUT_COMBINE]    # prefix operator on 4 cur + prev
CARRY_TABLE = _INT_LUTS[integer.LUT_CARRY_BIT]    # [state == GENERATE]

COMPARISONS = ("eq", "ne", "gt", "ge", "lt", "le")
ORDER_FINAL = {"gt": lambda s: s == SUPERIOR, "ge": lambda s: s != INFERIOR,
               "lt": lambda s: s == INFERIOR, "le": lambda s: s != SUPERIOR}
BITOPS = {"bitand": lambda l, r: l & r, "bitor": lambda l, r: l | r, "bitxor": lambda l, r: l ^ r}
# operations whose circuit depends on the signedness of the operands
SIGNED_OPS = ("gt", "ge", "lt", "le", "min", "max", "abs") + tuple(f"scalar_{o}" for o in ("gt", "ge", "lt", "le"))
# additions with a flag: (flag, signed flag) by base operation
ADDS = {"add": (False, False), "sub": (False, False), "overflowing_add": (True, False),
        "overflowing_sub": (True, False), "signed_overflowing_add": (True, True),
        "signed_overflowing_sub": (True, True)}
OPERATIONS = (COMPARISONS + tuple(f"scalar_{o}" for o in COMPARISONS) + ("min", "max", "if_then_else", "add",
              "sub", "neg", "overflowing_add", "overflowing_sub", "bitnot", "transfer") + tuple(BITOPS))
# clear-operand arithmetic, signed overflow flags and abs: circuits of this
# module too, kept apart from OPERATIONS, whose every schedule is pinned as is
ARITH_OPERATIONS = (("signed_overflowing_add", "signed_overflowing_sub", "abs")
                    + tuple(f"scalar_{o}" for o in ("add", "sub", "overflowing_add", "signed_overflowing_add",
                                                    "signed_overflowing_sub") + tuple(BITOPS)))

Block = List[Tuple[int, int]]   # (wire, coef) terms of one operand block's value


def table(c: bc.Circuit, f) -> int:
    """LUT index of f over the 16 values of the padded message space in
    circuit `c`, a circuit-local table added once per circuit"""
    t = tuple(int(f(x)) for x in range(bc.TOTAL_MOD))
    if t in c.extra_luts:
        return bc.NUM_FIXED_LUTS + c.extra_luts.index(t)
    return c.add_lut(t)


def _pbs(c: bc.Circuit, terms: Block, body: int, f) -> int:
    return c.lut(terms, body, table(c, f))


def _scaled(x: Block, k: int) -> Block:
    return [(w, k * coef) for w, coef in x]


def blocks_of(wires: Sequence[int]) -> List[Block]:
    return [[(w, 1)] for w in wires]


def scalar_blocks(c: bc.Circuit, num_blocks: int) -> List[Block]:
    """a clear operand: per block the two bits of its digit as per-instance
    constants (`scalar_iconsts`)"""
    return [[(c.iconst(), 1), (c.iconst(), 2)] for _ in range(num_blocks)]


def _signed_digit(v: int) -> int:
    return v - MSG_MOD if v >= MSG_MOD // 2 else v


def _sign(l: int, r: int) -> int:
    return INFERIOR if l < r else (EQUAL if l == r else SUPERIOR)


# ---------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------
def _pair(x: int, f) -> int:
    """f(hi, lo) of the packed value 4 hi + lo (0 past the operands' range)"""
    return int(f(x // MSG_MOD, x % MSG_MOD)) if x < MSG_MOD * MSG_MOD else 0


def compare(c: bc.Circuit, lhs: Sequence[Block], rhs: Sequence[Block], op: str, signed: bool = False) -> int:
    """The boolean `lhs op rhs`, op in COMPARISONS: one wire holding 0 or 1."""
    n = len(lhs)
    assert len(rhs) == n >= 1 and op in COMPARISONS
    packed = [_scaled(l, MSG_MOD) + list(r) for l, r in zip(lhs, rhs)]
    if op in ("eq", "ne"):
        want = op == "eq"
        if n == 1:
            return _pbs(c, packed[0], 0, lambda x: _pair(x, lambda l, r: (l == r) == want))
        bits = [_pbs(c, p, 0, lambda x: _pair(x, lambda l, r: l == r)) for p in packed]
        while True:
            groups = [bits[i:i + bc.MAX_TERMS] for i in range(0, len(bits), bc.MAX_TERMS)]
            last = len(groups) == 1
            bits = []
            for g in groups:
                k = len(g)
                if k == 1 and not last:
                    bits.append(g[0])
                    continue
                f = (lambda x, k=k: (x == k) == want) if last else (lambda x, k=k: x == k)
                bits.append(_pbs(c, [(w, 1) for w in g], 0, f))
            if last:
                return bits[0]
    final = ORDER_FINAL[op]

    def sign_of(i):
        top = signed and i == n - 1
        return lambda l, r: _sign(_signed_digit(l), _signed_digit(r)) if top else _sign(l, r)

    if n == 1:
        s = sign_of(0)
        return _pbs(c, packed[0], 0, lambda x: _pair(x, lambda l, r: final(s(l, r))))
    signs = [_pbs(c, p, 0, lambda x, s=sign_of(i): _pair(x, s)) for i, p in enumerate(packed)]

    def reduce(msb, lsb):   # reduce_two_orderings_function
        return lsb if msb == EQUAL else msb

    while True:
        last = len(signs) == 2
        out = (lambda m, l: final(reduce(m, l))) if last else reduce
        nxt = []
        for i in range(0, len(signs) - 1, 2):
            lsb, msb = signs[i], signs[i + 1]
            nxt.append(_pbs(c, [(msb, MSG_MOD), (lsb, 1)], 0,
                            lambda x: _pair(x, lambda m, l: out(m, l) if m <= SUPERIOR and l <= SUPERIOR else 0)))
        if len(signs) % 2:
            nxt.append(signs[-1])
        if last:
            return nxt[0]
        signs = nxt


# ---------------------------------------------------------------------------
# selects
# ---------------------------------------------------------------------------
def keep_if(c: bc.Circuit, cond: int, x: Sequence[Block], when: int = 1, flip: Optional[int] = None) -> List[int]:
    """x where cond == when, else 0: one PBS per block on 4 cond + x.  With
    `flip` (an `iconst` bit), x where cond XOR flip == when: the bit enters
    the same PBS as the body constant 8 flip (value <= 15, no noise)."""
    if flip is None:
        f = lambda v: (v % MSG_MOD) if v // MSG_MOD == when else 0  # noqa: E731
        return [_pbs(c, [(cond, MSG_MOD)] + list(b), 0, f) for b in x]
    f = lambda v: (v % MSG_MOD) if ((v // MSG_MOD) & 1) ^ (v // (2 * MSG_MOD)) == when else 0  # noqa: E731
    return [_pbs(c, [(cond, MSG_MOD), (flip, 2 * MSG_MOD)] + list(b), 0, f) for b in x]


def if_then_else(c: bc.Circuit, cond: int, a: Sequence[Block], b: Sequence[Block]) -> List[int]:
    """a where cond else b: keep_if both halves, then one identity PBS on their
    sum (noise 2, value <= 3)"""
    ka, kb = keep_if(c, cond, a, 1), keep_if(c, cond, b, 0)
    return [_pbs(c, [(x, 1), (y, 1)], 0, lambda v: MSG_TABLE[v]) for x, y in zip(ka, kb)]


# ---------------------------------------------------------------------------
# additions
# ---------------------------------------------------------------------------
def _signed_overflow(top: int, carry: int) -> bool:
    """whether a signed sum leaves [MIN, MAX], from 4 a_top + b_top (b_top the
    top digit of ~b for a subtraction) and the carry into the top block"""
    t = _signed_digit(top // MSG_MOD) + _signed_digit(top % MSG_MOD) + carry
    return not -MSG_MOD // 2 <= t < MSG_MOD // 2


def add(c: bc.Circuit, a: Optional[Sequence[Block]], b: Sequence[Block], sub: bool = False,
        flag: bool = False, signed: bool = False) -> Tuple[List[int], Optional[int]]:
    """a + b, or a - b (a + ~b + 1; a None is 0: the negation of b), wrapping
    mod 4^blocks.  With `flag`, also the carry out of a + b, or for a - b the
    borrow [a < b] (tfhe-rs' unsigned overflow flags); with `flag` and
    `signed`, [the exact two's-complement result is outside [MIN, MAX]].
    Returns (blocks, flag wire or None)."""
    n = len(b)
    sums: List[Tuple[Block, int]] = []
    for i in range(n):
        terms = [] if a is None else list(a[i])
        if sub:
            terms += _scaled(b[i], -1)
            sums.append((terms, MSG_MOD - 1 + (i == 0)))
        else:
            sums.append((terms + list(b[i]), 0))
    flag_f = (lambda s: s != integer.ST_GENERATE) if sub else (lambda s: s == integer.ST_GENERATE)
    msgs = [_pbs(c, t, body, lambda v: MSG_TABLE[v]) for t, body in sums]
    code = None
    if flag and signed:
        # 4 a_top + b_top (sub: 3 - b_top), noise 5: with the carry into the
        # top block known (n == 1) the flag, else a code read with the carry
        # state: 0 never, 1 iff carry, 2 iff no carry, 3 always
        top = (_scaled(a[n - 1], MSG_MOD) + (_scaled(b[n - 1], -1) if sub else list(b[n - 1])),
               MSG_MOD - 1 if sub else 0)
        if n == 1:
            return msgs, _pbs(c, *top, lambda v: int(_signed_overflow(v, int(sub))))
        code = _pbs(c, *top, lambda v: int(_signed_overflow(v, 1)) + 2 * int(_signed_overflow(v, 0)))
        flag = False
    if flag and n == 1:
        return msgs, _pbs(c, *sums[0], lambda v: flag_f(STATE_TABLE[v]))
    # inclusive prefix states of blocks 0..i: the state feeding block i + 1,
    # and for the flag the whole integer's, folded into its last combine
    need = n if flag else n - 1
    out_flag = None
    states = [_pbs(c, *sums[i], lambda v: STATE_TABLE[v]) for i in range(need)]
    d = 1
    while d < need:
        nxt = list(states)
        for i in range(d, need):
            if flag and i == n - 1 and 2 * d > i:   # the top block's last combine: the flag itself
                out_flag = _pbs(c, [(states[i], MSG_MOD), (states[i - d], 1)], 0,
                                lambda v: int(flag_f(COMBINE_TABLE[v])) if v <= 10 else 0)
            else:
                nxt[i] = _pbs(c, [(states[i], MSG_MOD), (states[i - d], 1)], 0,
                              lambda v: COMBINE_TABLE[v] if v <= 10 else 0)
        states = nxt
        d *= 2
    if code is not None:   # one PBS on 4 code + state_{n-2}, beside the last layer
        out_flag = _pbs(c, [(code, MSG_MOD), (states[n - 2], 1)], 0,
                        lambda v: (v // MSG_MOD >> int(v % MSG_MOD != integer.ST_GENERATE)) & 1)
    out = [msgs[0]] + [_pbs(c, [(msgs[i], 1), (states[i - 1], MSG_MOD)], 0,
                            lambda v: (v % MSG_MOD + CARRY_TABLE[v // MSG_MOD]) % MSG_MOD if v < 12 else 0)
                       for i in range(1, n)]
    return out, out_flag


def bitop(c: bc.Circuit, a: Sequence[Block], b: Sequence[Block], op: str) -> List[int]:
    f = BITOPS[op]
    return [_pbs(c, _scaled(x, MSG_MOD) + list(y), 0, lambda v: _pair(v, f)) for x, y in zip(a, b)]


def bitnot(c: bc.Circuit, a: Sequence[Block]) -> List[int]:
    return [_pbs(c, list(x), 0, lambda v: MSG_MOD - 1 - v if v < MSG_MOD else 0) for x in a]


def transfer(c: bc.Circuit, frm: Sequence[Block], to: Sequence[Block], amount: Sequence[Block]
             ) -> Tuple[List[int], List[int]]:
    """erc7984's `transfer_whitepaper`: has_enough = from >= amount; sent =
    has_enough ? amount : 0; returns (from - sent, to + sent)."""
    has_enough = compare(c, frm, amount, "ge")
    sent = blocks_of(keep_if(c, has_enough, amount))
    new_to, _ = add(c, to, sent)
    new_from, _ = add(c, frm, sent, sub=True)
    return new_from, new_to


# ---------------------------------------------------------------------------
# compiled circuits
# ---------------------------------------------------------------------------
def check_num_blocks(num_blocks) -> int:
    if isinstance(num_blocks, bool) or not isinstance(num_blocks, (int, np.integer)) \
            or not 1 <= num_blocks <= MAX_BLOCKS:
        raise ValueError(f"num_blocks must be an integer in [1, {MAX_BLOCKS}], got {num_blocks!r}")
    return int(num_blocks)


def circuit(op: str, num_blocks: int, signed: bool = False) -> bc.Circuit:
    """The circuit of one operation on `num_blocks`-block integers.  Per
    instance, inputs are the operands' blocks in argument order
    (`if_then_else`: the condition block first) and the outputs are the
    result's blocks: a boolean is one block; the `overflowing_*` operations
    output the blocks then the flag; `transfer` new_from then new_to.
    `scalar_*` read the clear rhs as 2 * num_blocks per-instance bits
    (`scalar_iconsts`).  `op` is one of OPERATIONS or ARITH_OPERATIONS.
    The CIRCUIT_CACHE_SIZE most recent (op, num_blocks, signed) are kept (an
    operation that does not depend on the signedness has one circuit); the
    schedule of each is compiled once (`bit_circuit.schedule`)."""
    n = check_num_blocks(num_blocks)
    if op not in OPERATIONS + ARITH_OPERATIONS:
        raise ValueError(f"unknown radix operation {op!r}")
    return _circuit(op, n, bool(signed) and op in SIGNED_OPS)


@functools.lru_cache(maxsize=CIRCUIT_CACHE_SIZE)
def _circuit(op: str, n: int, signed: bool) -> bc.Circuit:
    c = bc.Circuit(f"{'signed' if signed else 'unsigned'}_{op}_{n}")
    if op == "if_then_else":
        cond = c.input(False)
        a, b = blocks_of(c.inputs_block(n, False)), blocks_of(c.inputs_block(n, False))
        c.output_blocks(if_then_else(c, cond, a, b))
        return c
    if op == "transfer":
        frm, to, amount = (blocks_of(c.inputs_block(n, False)) for _ in range(3))
        new_from, new_to = transfer(c, frm, to, amount)
        c.output_blocks(new_from + new_to)
        return c
    if op == "abs":   # unsigned: the identity
        from . import radix_div

        x = c.inputs_block(n, False)
        c.output_blocks(radix_div.cond_negate(c, x, x[-1], lambda v: v >= MSG_MOD // 2) if signed else x)
        return c
    a = blocks_of(c.inputs_block(n, False))
    if op in ("neg", "bitnot"):
        c.output_blocks(add(c, None, a, sub=True)[0] if op == "neg" else bitnot(c, a))
        return c
    b = scalar_blocks(c, n) if op.startswith("scalar_") else blocks_of(c.inputs_block(n, False))
    base = op[len("scalar_"):] if op.startswith("scalar_") else op
    if base in COMPARISONS:
        c.output_blocks([compare(c, a, b, base, signed)])
    elif base in ("min", "max"):
        gt = compare(c, a, b, "gt", signed)
        c.output_blocks(if_then_else(c, gt, b, a) if base == "min" else if_then_else(c, gt, a, b))
    elif base in ADDS:
        out, flag = add(c, a, b, sub=base.endswith("sub"), flag=ADDS[base][0], signed=ADDS[base][1])
        c.output_blocks(out + ([flag] if flag is not None else []))
    else:
        c.output_blocks(bitop(c, a, b, base))
    return c


def scalar_range(num_blocks: int, signed: bool) -> Tuple[int, int]:
    """[lo, hi) of the integers a num_blocks-block radix holds"""
    bits = 2 * num_blocks
    return (-(1 << (bits - 1)), 1 << (bits - 1)) if signed else (0, 1 << bits)


def scalar_iconsts(scalars: Sequence[int], num_blocks: int, signed: bool) -> np.ndarray:
    """The per-instance constants of a `scalar_*` circuit: [instances,
    2 * num_blocks] bits, the two's-complement digits of each scalar, LSB
    first.  Scalars outside the integer's range raise ValueError."""
    lo, hi = scalar_range(num_blocks, signed)
    out = np.zeros((len(scalars), 2 * num_blocks), dtype=np.int64)
    for i, s in enumerate(scalars):
        if isinstance(s, bool) or not isinstance(s, (int, np.integer)) or not lo <= int(s) < hi:
            raise ValueError(f"scalar {s!r} is outside the range [{lo}, {hi}) of a {num_blocks}-block "
                             f"{'signed' if signed else 'unsigned'} integer")
        v = int(s) % (1 << (2 * num_blocks))
        out[i] = [(v >> j) & 1 for j in range(2 * num_blocks)]
    return out


# ---------------------------------------------------------------------------
# plain model (the semantics the circuits implement)
# ---------------------------------------------------------------------------
def to_digits(v: int, num_blocks: int) -> List[int]:
    """two's-complement 2-bit digits of v, least significant first"""
    v %= 1 << (2 * num_blocks)
    return [(v >> (2 * i)) & 3 for i in range(num_blocks)]


def from_digits(digits: Sequence[int], signed: bool = False) -> int:
    v = sum(int(d) << (2 * i) for i, d in enumerate(digits))
    bits = 2 * len(digits)
    return v - (1 << bits) if signed and v >> (bits - 1) else v
