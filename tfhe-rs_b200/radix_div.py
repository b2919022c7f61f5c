"""Division and remainder of radix integers on 2_2 blocks, compiled to batched
KS -> PBS layers by `bit_circuit`: `div_rem`, `div`, `rem` by an encrypted
divisor and their `scalar_*` forms by a clear one, unsigned and signed.  Host
code only: the GPU runs them with `b200_bit_circuit_64_async` through
`integer.CudaRadixServerKey`, like the circuits of `radix`.

The unsigned core is tfhe-rs' `unsigned_div_rem_block_by_block_2_2`: the
remainder starts as the numerator and one iteration per block, from the top
block down, computes one quotient digit.  With L the live length (the
remainder's blocks from the current one up) an iteration

  * subtracts d, 2d and 3d (their low L blocks) from the live remainder with
    `radix.add(sub=True, flag=True)`; the borrow of k·d is OR-ed with "k·d has a
    non-zero block at or above L" (precomputed once per multiple and L), one
    PBS: o_k = [remainder < k·d], monotone in k;
  * keeps exactly one of r - 3d, r - 2d, r - d and r by the zero-out tables on
    2 x + c (c in {0, 1}: keep when c == 1) and 3 x + c (c in {0, 1, 2}: keep
    when c == 2), with c3 = 1 - o3, c2 = 1 - o2 + o3, c1 = 1 - o1 + o2,
    c0 = o1 (noise <= 5, value <= 11);
  * makes the quotient digit with one PBS on 3 - (o1 + o2 + o3);
  * leaves the new remainder blocks as the sum of the four selected wires (at
    most one non-zero): the next iteration's subtractions read that sum
    directly (noise 4 + 1 for the divisor's block, value <= 15), and a message
    extraction of it, off the critical path, feeds the next zero-out.

2d is one PBS per block on 4 d_i + d_(i-1) and 3d = 4d - d one subtraction,
both on n + 1 blocks; the "non-zero above" flags are a radix-5 suffix OR of
per-block non-zero bits.  For a clear divisor the digits of d, 2d and 3d,
the flags and the divisor's sign are per-instance constants (`scalar_iconsts`),
so the divisor side costs no PBS.

Signed operands (tfhe-rs `signed_unchecked_div_rem_parallelized`): |n| and |d|
by a conditional negation (one PBS per block on 4 sign_block + x, then the
carry scan of `radix.add`), the unsigned core, then the quotient negated when
the sign bits differ and the remainder when n < 0.  Division by an encrypted
zero gives, unsigned, q = 2^b - 1 and r = n; signed, r = n and q = -1 when
n >= 0, else 1 (what tfhe-rs computes).
"""
from __future__ import annotations

import functools
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import bit_circuit as bc
from . import integer
from . import radix
from .radix import MSG_MOD, Block, _pbs, blocks_of

OPERATIONS = ("div_rem", "div", "rem", "scalar_div_rem", "scalar_div", "scalar_rem")
# (quotient, remainder) each operation outputs, in that order
OUTPUTS = {"div_rem": (True, True), "div": (True, False), "rem": (False, True)}


def _zero_out(c: bc.Circuit, x: int, factor: int, cond: Block, body: int, keep: int) -> int:
    """x where the condition's value (body + cond, in [0, factor)) is `keep`,
    else 0: one PBS on factor * x + cond"""
    return _pbs(c, [(x, factor)] + list(cond), body,
                lambda v: v // factor if v % factor == keep and v // factor < MSG_MOD else 0)


def _suffix_any(c: bc.Circuit, bits: Sequence[int]) -> List[int]:
    """out[i] = OR of bits[i:]: a radix-5 Hillis-Steele suffix scan"""
    cur, s = list(bits), 1
    while s < len(cur):
        nxt = list(cur)
        for i in range(len(cur) - s):
            grp = [cur[j] for j in range(i, min(len(cur), i + bc.MAX_TERMS * s), s)]
            nxt[i] = _pbs(c, [(w, 1) for w in grp], 0, lambda v: int(v > 0))
        cur, s = nxt, s * bc.MAX_TERMS
    return cur


def _carry_out(c: bc.Circuit, msgs: List[int], states: List[int]) -> List[int]:
    """the blocks of a sum from its per-block messages and carry states: the
    prefix scan and final step of `radix.add`"""
    n = len(msgs)
    states = states[:n - 1]
    d = 1
    while d < n - 1:
        states = states[:d] + [_pbs(c, [(states[i], MSG_MOD), (states[i - d], 1)], 0,
                                    lambda v: radix.COMBINE_TABLE[v] if v <= 10 else 0)
                               for i in range(d, n - 1)]
        d *= 2
    return [msgs[0]] + [_pbs(c, [(msgs[i], 1), (states[i - 1], MSG_MOD)], 0,
                             lambda v: (v % MSG_MOD + radix.CARRY_TABLE[v // MSG_MOD]) % MSG_MOD if v < 12 else 0)
                        for i in range(1, n)]


def cond_negate(c: bc.Circuit, x: Sequence[int], sel: int, pred) -> List[int]:
    """-x (mod 4^blocks) where pred(value of `sel`) holds, else x: per block one
    PBS on 4 sel + x_i for its message and one for its carry state (~x + 1),
    then the carry scan.  `sel` may be one of x's wires (noise 5, value 15)."""
    def total(v, i):
        cond = pred(v // MSG_MOD)
        return (MSG_MOD - 1 - v % MSG_MOD + (i == 0)) if cond else v % MSG_MOD

    def state(t):
        return integer.ST_GENERATE if t >= MSG_MOD else (integer.ST_PROPAGATE if t == MSG_MOD - 1
                                                         else integer.ST_NONE)

    terms = [[(sel, MSG_MOD + 1)] if w == sel else [(sel, MSG_MOD), (w, 1)] for w in x]
    msgs = [_pbs(c, t, 0, lambda v, i=i: total(v, i) % MSG_MOD) for i, t in enumerate(terms)]
    states = [_pbs(c, t, 0, lambda v, i=i: state(total(v, i))) for i, t in enumerate(terms[:-1])]
    return _carry_out(c, msgs, states)


def multiples(c: bc.Circuit, d: Sequence[int]) -> Tuple[Dict[int, List[Block]], Dict[int, List[Optional[Block]]]]:
    """d, 2d and 3d of an encrypted divisor on n + 1 blocks, and per multiple k
    and live length L in [1, n] the flag "k d >= 4^L" (None: always 0)"""
    n = len(d)
    two = [_pbs(c, [(d[0], 1)], 0, lambda v: 2 * v % MSG_MOD)]
    nz2 = []
    for i in range(1, n + 1):
        t = [(d[i], MSG_MOD), (d[i - 1], 1)] if i < n else [(d[n - 1], 1)]
        f = (lambda v: (2 * (v // MSG_MOD) + v % MSG_MOD // 2) % MSG_MOD) if i < n else (lambda v: v // 2)
        two.append(_pbs(c, t, 0, f))
        nz2.append(_pbs(c, t, 0, lambda v, f=f: int(f(v) != 0)))
    ds = blocks_of(d)
    three, _ = radix.add(c, [[]] + ds, ds + [[]], sub=True)   # 4d - d
    nz1 = [_pbs(c, [(w, 1)], 0, lambda v: int(v != 0)) for w in d[1:]]
    nz3 = [_pbs(c, [(w, 1)], 0, lambda v: int(v != 0)) for w in three[1:]]
    mults = {1: ds + [[]], 2: blocks_of(two), 3: blocks_of(three)}
    flags = {k: [None] + [[(w, 1)] for w in _suffix_any(c, nz)] for k, nz in ((1, nz1), (2, nz2), (3, nz3))}
    flags[1].append(None)   # d has no block at or above n
    return mults, flags


def scalar_divisor(c: bc.Circuit, n: int, signed: bool):
    """a clear divisor as per-instance constants, in the order of
    `scalar_iconsts`: the digits of |d|, 2|d| and 3|d| (low n blocks), the
    flags "k |d| >= 4^L" for k = 1..3 and L = 1..n, and the sign of d.
    Returns (multiples, flags, sign constant or None)."""
    mults = {k: radix.scalar_blocks(c, n) for k in (1, 2, 3)}
    flags = {k: [None] + [[(c.iconst(), 1)] for _ in range(n)] for k in (1, 2, 3)}
    flags[1][n] = None   # never set: |d| < 4^n
    return mults, flags, (c.iconst() if signed else None)


def unsigned_div_rem(c: bc.Circuit, num: Sequence[int], mults, flags, want_q: bool = True,
                     want_r: bool = True) -> Tuple[List[int], List[int]]:
    """(quotient, remainder) blocks of num / d, d given by its multiples and
    flags (`multiples` or `scalar_divisor`); num's blocks are single wires"""
    n = len(num)
    form: List[Block] = []     # the remainder's blocks above the live one, as sums of 4 wires
    clean: List[int] = []      # the same blocks extracted to single wires
    q: List[int] = []
    for j in reversed(range(n)):
        L = n - j
        live = [[(num[j], 1)]] + form
        o = {}
        diff = {}
        for k in (3, 2, 1):
            diff[k], borrow = radix.add(c, live, mults[k][:L], sub=True, flag=True)
            f = flags[k][L]
            o[k] = borrow if f is None else _pbs(c, [(borrow, 1)] + f, 0, lambda v: int(v > 0))
        keep = [
            [_zero_out(c, w, 2, [(o[3], -1)], 1, 1) for w in diff[3]],
            [_zero_out(c, w, 3, [(o[2], -1), (o[3], 1)], 1, 2) for w in diff[2]],
            [_zero_out(c, w, 3, [(o[1], -1), (o[2], 1)], 1, 2) for w in diff[1]],
            [_zero_out(c, w, 2, [(o[1], 1)], 0, 1) for w in [num[j]] + clean],
        ]
        if want_q:
            q.append(_pbs(c, [(o[1], -1), (o[2], -1), (o[3], -1)], MSG_MOD - 1, lambda v: v if v < MSG_MOD else 0))
        form = [[(w, 1) for w in ws] for ws in zip(*keep)]
        if j > 0 or want_r:
            clean = [_pbs(c, t, 0, lambda v: radix.MSG_TABLE[v]) for t in form]
    return q[::-1], clean


def _sign(v: int) -> int:
    return int(v >= MSG_MOD // 2)


def div_rem(c: bc.Circuit, num: Sequence[int], d: Optional[Sequence[int]], signed: bool, want_q: bool = True,
            want_r: bool = True) -> List[int]:
    """the quotient's blocks (if want_q) then the remainder's (if want_r) of
    num / d; d None is a clear divisor (`scalar_divisor`)"""
    n = len(num)
    top = num[-1]
    if signed:
        num = cond_negate(c, num, top, _sign)
    if d is None:
        mults, flags, d_sign = scalar_divisor(c, n, signed)
    else:
        d_top = d[-1]
        mults, flags = multiples(c, cond_negate(c, d, d_top, _sign) if signed else d)
    q, r = unsigned_div_rem(c, num, mults, flags, want_q, want_r)
    if signed and want_q:
        if d is None:
            differ = _pbs(c, [(top, 1), (d_sign, MSG_MOD)], 0, lambda v: int(_sign(v % MSG_MOD) != v // MSG_MOD))
        else:
            differ = _pbs(c, [(top, MSG_MOD), (d_top, 1)], 0, lambda v: int(_sign(v // MSG_MOD) != _sign(v % MSG_MOD)))
        q = cond_negate(c, q, differ, lambda s: s == 1)
    if signed and want_r:
        r = cond_negate(c, r, top, _sign)
    return (q if want_q else []) + (r if want_r else [])


# ---------------------------------------------------------------------------
# compiled circuits
# ---------------------------------------------------------------------------
def circuit(op: str, num_blocks: int, signed: bool = False) -> bc.Circuit:
    """The circuit of one division on `num_blocks`-block integers.  Per
    instance, the inputs are the numerator's blocks then (not `scalar_*`) the
    divisor's; the outputs are the quotient's blocks then the remainder's
    (`div_rem`) or one of them.  `scalar_*` read the clear divisor as
    `scalar_iconsts`.  The radix.CIRCUIT_CACHE_SIZE most recent (op,
    num_blocks, signed) are kept; each schedule is compiled once."""
    n = radix.check_num_blocks(num_blocks)
    if op not in OPERATIONS:
        raise ValueError(f"unknown radix division {op!r}")
    return _circuit(op, n, bool(signed))


@functools.lru_cache(maxsize=radix.CIRCUIT_CACHE_SIZE)
def _circuit(op: str, n: int, signed: bool) -> bc.Circuit:
    c = bc.Circuit(f"{'signed' if signed else 'unsigned'}_{op}_{n}")
    scalar = op.startswith("scalar_")
    num = c.inputs_block(n, False)
    d = None if scalar else c.inputs_block(n, False)
    c.output_blocks(div_rem(c, num, d, signed, *OUTPUTS[op[len("scalar_"):] if scalar else op]))
    return c


def scalar_iconsts(scalars: Sequence[int], num_blocks: int, signed: bool) -> np.ndarray:
    """The per-instance constants of a `scalar_*` division: [instances, 9 n
    (+ 1 signed)] bits: the two bits of each of the low n digits of |d|, 2|d|
    and 3|d|; the flags [k |d| >= 4^L] for k = 1..3, L = 1..n; and [d < 0]
    when signed.  A zero divisor, or one outside the integer's range, raises
    ValueError."""
    lo, hi = radix.scalar_range(num_blocks, signed)
    n = num_blocks
    out = np.zeros((len(scalars), 9 * n + int(signed)), dtype=np.int64)
    for i, s in enumerate(scalars):
        if isinstance(s, bool) or not isinstance(s, (int, np.integer)) or not lo <= int(s) < hi:
            raise ValueError(f"divisor {s!r} is outside the range [{lo}, {hi}) of a {n}-block "
                             f"{'signed' if signed else 'unsigned'} integer")
        if int(s) == 0:
            raise ValueError("attempt to divide by 0")
        a = abs(int(s))
        row = []
        for k in (1, 2, 3):
            v = k * a
            row += [(v >> j) & 1 for j in range(2 * n)]
        for k in (1, 2, 3):
            row += [int(k * a >= 4 ** L) for L in range(1, n + 1)]
        if signed:
            row.append(int(int(s) < 0))
        out[i] = row
    return out


# ---------------------------------------------------------------------------
# plain model (the semantics the circuits implement)
# ---------------------------------------------------------------------------
def model(n: int, d: int, num_blocks: int, signed: bool = False) -> Tuple[int, int]:
    """(quotient, remainder) of n / d on num_blocks-block integers"""
    bits = 2 * num_blocks
    if not signed:
        return ((1 << bits) - 1, n) if d == 0 else (n // d, n % d)
    if d == 0:
        return (-1 if n >= 0 else 1), n
    q = abs(n) // abs(d)
    q = -q if (n < 0) != (d < 0) else q
    r = n - q * d
    q = radix.from_digits(radix.to_digits(q, num_blocks), True)   # MIN / -1 wraps to MIN
    return q, r
