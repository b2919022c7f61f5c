"""Shifts, rotations and bit counts of radix integers on 2_2 blocks, compiled
to batched KS -> PBS layers by `bit_circuit`: `left_shift`, `right_shift`,
`rotate_left`, `rotate_right` by an encrypted amount and their `scalar_*`
forms by a clear one; `leading_zeros`, `leading_ones`, `trailing_zeros`,
`trailing_ones`, `count_ones`, `count_zeros`, `ilog2` and `checked_ilog2`.
Host code only: the GPU runs them with `b200_bit_circuit_64_async` through
`integer.CudaRadixServerKey`, like the circuits of `radix`.

Semantics are tfhe-rs' (bits = 2 * num_blocks, signed integers read as their
two's-complement bit pattern except where stated):

  * a shift by an encrypted amount < bits is exact, right shifts of signed
    integers arithmetic; by amount >= bits the result is 0, or -1 for a
    signed right shift of a negative value (`shift.rs` `overshift_predicate`,
    `apply_arithmetic_right_shift_overshift`).  A clear amount follows the
    same rule (`scalar_shift.rs:170-184`);
  * the barrel shifter of a rotation reads m = floor(log2 bits) + [bits is
    not a power of 2] bits of the amount (`shift.rs:351-360`,
    `unchecked_shift_rotate_bits_assign`), each stage rotating modulo bits,
    so an encrypted rotation is by (amount mod 2^m) mod bits: at 6 bits an
    amount of 8 rotates by 0.  A clear rotation is by n mod bits
    (`scalar_rotate.rs:612`);
  * leading / trailing counts have ceil((floor(log2 bits) + 1) / 2) blocks
    (`ilog2.rs:161-162`), `count_*` 16 blocks, enough for 32 bits
    (`count_zeros_ones.rs:140`); `ilog2` is (bits - 1) - leading_zeros on
    ceil((floor(log2(bits - 1)) + 2) / 2) blocks (`ilog2.rs:247-248`), so
    ilog2(0) is all ones after the cast to unsigned (`ilog2.rs:345`), and
    `checked_ilog2`'s flag is `ct > 0` compared with the integer's own
    signedness (`ilog2.rs:694`): 0 for a negative signed value.

Circuits (every PBS input within the 2_2 budget, sum |c_i| <= 5, value <= 15):

  * encrypted shift / rotation, a bit-level barrel shifter.  Stage 0 reads
    the whole amount block 0 (shift by t in 0..3 bits): output bit i is the
    sum, over the <= 3 blocks holding its candidate source bits, of one PBS
    on 4 a_0 + x_B (noise 5) that yields the bit if block B holds the source
    for t = a_0, else 0.  Stage k >= 2 (shift by 2^k) reads amount bit k, s,
    extracted in layer 1: bit i = t1 + t2 with t1 = PBS(2 s + d_src) = s ∧
    d_src and t2 = PBS(2 s + d_i) = ¬s ∧ d_i, where d is the previous
    stage's unmaterialised sum (level <= 3, noise <= 5).  A shift's last
    stage reads, instead of s, a mode wire in {0: keep, 1: take, 2: zero,
    3: ones} that folds in the overshift predicate (and for a signed right
    shift the sign); its outputs carry the bit's weight (1 or 2) and one
    identity PBS per block on the 4 summed terms packs them (noise 4).  The
    overshift predicate, off the critical path: `radix.compare(low amount,
    bits, "ge")` when the low amount blocks can reach bits, and [sum of <= 5
    high amount blocks != 0], OR-ed down to <= 2 wires.
  * clear shift / rotation: one PBS per output block on 4 x_hi + x_lo of the
    <= 2 source blocks (noise 5, value 15); vacated blocks are one zero PBS,
    or the sign block; exactly one layer.
  * leading / trailing counts and ilog2: F_k = "every block beyond k holds
    the neutral pattern (0, or 3 for ones)" by a radix-5 scan of [sum of <= 5
    blocks (or of 3 - x) == 0] then [sum of flags == count]; the first
    non-neutral block k contributes its count, one PBS per output digit on
    4 F_k + x_k; only one k contributes, so each output digit is the sum of
    its column, reduced by identity PBS on sums of <= 5 (value <= 15).
  * count_ones / count_zeros: one PBS per block pair on 4 x_a + x_b gives
    their popcount (<= 4); columns are compressed by message / carry PBS on
    sums of <= 5 wires (value <= 15) to <= 2 wires of value <= 3 each, then
    one `radix.add`.
"""
from __future__ import annotations

import functools
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import bit_circuit as bc
from . import radix
from .radix import MSG_MOD, _pbs, blocks_of

SHIFTS = ("left_shift", "right_shift", "rotate_left", "rotate_right")
COUNTS = ("leading_zeros", "leading_ones", "trailing_zeros", "trailing_ones", "count_ones", "count_zeros",
          "ilog2", "checked_ilog2")
OPERATIONS = SHIFTS + tuple(f"scalar_{o}" for o in SHIFTS) + COUNTS
# operations whose circuit depends on the signedness of the operand
SIGNED_OPS = ("right_shift", "scalar_right_shift", "checked_ilog2")
COUNT_ONES_BLOCKS = 16    # tfhe-rs: "enough to hold 32 bits"


def count_blocks(num_blocks: int) -> int:
    """blocks of a leading / trailing count: enough to hold bits"""
    return (2 * num_blocks).bit_length() + 1 >> 1


def ilog2_blocks(num_blocks: int) -> int:
    """blocks of ilog2: ceil((floor(log2(bits - 1)) + 2) / 2)"""
    return ((2 * num_blocks - 1).bit_length() + 1 + 1) // 2


def rotation_bits(num_blocks: int) -> int:
    """m: amount bits the barrel shifter reads"""
    bits = 2 * num_blocks
    return bits.bit_length() - 1 + (bits & (bits - 1) != 0)


def result_blocks(op: str, num_blocks: int) -> int:
    if op in ("count_ones", "count_zeros"):
        return COUNT_ONES_BLOCKS
    if op in ("ilog2", "checked_ilog2"):
        return ilog2_blocks(num_blocks)
    if op in COUNTS:
        return count_blocks(num_blocks)
    return num_blocks


def _src(op: str, signed: bool, bits: int, i: int, t: int) -> Optional[int]:
    """the source bit of output bit i in a shift / rotation by t bits (None: 0)"""
    if op == "left_shift":
        return i - t if i >= t else None
    if op == "right_shift":
        return i + t if i + t < bits else (bits - 1 if signed else None)
    if op == "rotate_left":
        return (i - t) % bits
    return (i + t) % bits


def _zero(c: bc.Circuit, x: Sequence[int]) -> int:
    """a wire holding 0 (one PBS per instance, shared by every reader)"""
    return _pbs(c, [(x[0], 1)], 0, lambda v: 0)


def _bits_of(v: int, unit: Sequence[Tuple[int, int]], src, block: int) -> int:
    """sum of weight * source bit over the unit's (bit, weight), for the
    source bits that block `block` (value v) holds"""
    out = 0
    for i, w in unit:
        j = src(i)
        if j is not None and j // 2 == block:
            out += w * ((v >> (j % 2)) & 1)
    return out


# ---------------------------------------------------------------------------
# shifts and rotations by an encrypted amount
# ---------------------------------------------------------------------------
def _stage0(c: bc.Circuit, x: Sequence[int], a0: int, op: str, signed: bool, units) -> List[List[Tuple[int, int]]]:
    """shift by t = a_0 in 0..3 bits: per unit (a list of (bit, weight)) the
    terms of its value, one PBS on 4 a_0 + x_B per source block B"""
    bits = 2 * len(x)
    out = []
    for unit in units:
        blocks = sorted({j // 2 for i, _ in unit for t in range(MSG_MOD)
                         for j in [_src(op, signed, bits, i, t)] if j is not None})
        terms = []
        for B in blocks:
            f = (lambda v, B=B, unit=unit: _bits_of(v % MSG_MOD, unit,
                                                     lambda i: _src(op, signed, bits, i, v // MSG_MOD), B))
            terms.append((_pbs(c, [(a0, MSG_MOD), (x[B], 1)], 0, f), 1))
        out.append(terms)
    return out


def _mux(c: bc.Circuit, sel: List[Tuple[int, int]], d_src, d_cur, weight: int, modes: bool):
    """the terms of `sel ? d_src : d_cur` (two PBS on 2 sel + d, d a bit of
    level <= 3); with `modes` sel is a mode wire: 0 keep d_cur, 1 take d_src,
    2 zero, 3 ones"""
    sel2 = [(w, 2 * k) for w, k in sel]
    terms = []
    if d_src is not None:
        terms.append((_pbs(c, sel2 + list(d_src), 0, lambda v: weight * (v // 2 == 1 and v % 2)), 1))
    f = (lambda v: weight * ((v // 2 == 0 and v % 2) or v // 2 == 3)) if modes else \
        (lambda v: weight * (v // 2 == 0 and v % 2))
    terms.append((_pbs(c, sel2 + list(d_cur), 0, f), 1))
    return terms


def _or_down(c: bc.Circuit, flags: List[int], keep: int) -> List[int]:
    """OR groups of <= 5 flags until at most `keep` remain"""
    while len(flags) > keep:
        flags = [_pbs(c, [(w, 1) for w in flags[i:i + bc.MAX_TERMS]], 0, lambda v: int(v > 0))
                 for i in range(0, len(flags), bc.MAX_TERMS)]
    return flags


def _overshift(c: bc.Circuit, amount: Sequence[int], bits: int) -> List[int]:
    """<= 2 wires whose OR is [amount >= bits] ([] when it cannot be)"""
    split = min((rotation_bits(bits // 2) + 1) // 2, len(amount))
    flags = []
    if MSG_MOD ** split > bits:
        digits = radix.to_digits(bits, split)
        const = [[(c.const(d & 1), 1), (c.const(d >> 1), 2)] for d in digits]
        flags.append(radix.compare(c, blocks_of(amount[:split]), const, "ge"))
    high = amount[split:]
    flags += [_pbs(c, [(w, 1) for w in high[i:i + bc.MAX_TERMS]], 0, lambda v: int(v > 0))
              for i in range(0, len(high), bc.MAX_TERMS)]
    return _or_down(c, flags, 2)


def shift(c: bc.Circuit, x: Sequence[int], amount: Sequence[int], op: str, signed: bool) -> List[int]:
    """the blocks of x shifted or rotated (op in SHIFTS) by the encrypted
    amount's value"""
    n = len(x)
    bits = 2 * n
    m = rotation_bits(n)
    stages = [k for k in range(2, m) if k // 2 < len(amount)]
    rotate = op.startswith("rotate")
    over = [] if rotate else _overshift(c, amount, bits)
    if over:
        if signed and op == "right_shift":   # 0: in range, 1: overshift of x >= 0, 2: of x < 0
            neg = _pbs(c, [(x[-1], 1)], 0, lambda v: (v >> 1) & 1)
            over = [_pbs(c, [(neg, 1)] + [(w, 2) for w in over], 0, lambda v: (v // 2 > 0) * (1 + v % 2))]

        def mode_of(s):
            terms = ([(s, 1)] if s is not None else []) + [(w, 2) for w in over]
            return _pbs(c, terms, 0, lambda v: v % 2 if v // 2 == 0 else
                        (min(1 + v // 2, 3) if signed and op == "right_shift" else 2))
    final_units = [[(2 * j, 1), (2 * j + 1, 2)] for j in range(n)]
    if not stages and not over:   # stage 0 is the last: its PBS make whole blocks
        forms = _stage0(c, x, amount[0], op, signed, final_units)
        return [t[0][0] if len(t) == 1 else _pbs(c, t, 0, lambda v: v if v < MSG_MOD else 0) for t in forms]
    d = _stage0(c, x, amount[0], op, signed, [[(i, 1)] for i in range(bits)])
    if over and not stages:
        stages = [None]   # a masking stage of its own
    for idx, k in enumerate(stages):
        last = idx == len(stages) - 1
        s = None if k is None else _pbs(c, [(amount[k // 2], 1)], 0, lambda v, k=k: (v >> (k % 2)) & 1)
        if last and over:
            sel, modes = [(mode_of(s), 1)], True
        else:
            sel, modes = [(s, 1)], False
        t = 0 if k is None else 1 << k
        nd = []
        for i in range(bits):
            j = _src(op, signed, bits, i, t) if k is not None else None
            if not last and j == i:
                nd.append(d[i])
                continue
            nd.append(_mux(c, sel, None if j is None else d[j], d[i], 1 + (last and i % 2), modes))
        d = nd
    return [_pbs(c, d[2 * j] + d[2 * j + 1], 0, lambda v: v if v < MSG_MOD else 0) for j in range(n)]


# ---------------------------------------------------------------------------
# shifts and rotations by a clear amount
# ---------------------------------------------------------------------------
def canonical_amount(op: str, num_blocks: int, amount: int) -> int:
    """the clear amount giving the same result in [0, bits]: n mod bits for a
    rotation, min(n, bits) for a shift"""
    bits = 2 * num_blocks
    return amount % bits if op.startswith("scalar_rotate") else min(amount, bits)


def scalar_shift(c: bc.Circuit, x: Sequence[int], amount: int, op: str, signed: bool) -> List[int]:
    """x shifted or rotated by the clear `amount` (op in SHIFTS): one PBS per
    block on its <= 2 source blocks"""
    n = len(x)
    bits = 2 * n
    out = []
    for j in range(n):
        unit = [(2 * j, 1), (2 * j + 1, 2)]

        def src(i):
            return _src(op, signed, bits, i, amount)
        blocks = sorted({src(i) // 2 for i, _ in unit if src(i) is not None})
        if not blocks:
            out.append(_zero(c, x))
        elif len(blocks) == 1:
            B = blocks[0]
            out.append(_pbs(c, [(x[B], 1)], 0, lambda v, B=B, src=src, unit=unit:
                            _bits_of(v, unit, src, B) if v < MSG_MOD else 0))
        else:
            lo, hi = blocks
            out.append(_pbs(c, [(x[hi], MSG_MOD), (x[lo], 1)], 0, lambda v, lo=lo, hi=hi, src=src, unit=unit:
                            _bits_of(v // MSG_MOD, unit, src, hi) + _bits_of(v % MSG_MOD, unit, src, lo)))
    return out


# ---------------------------------------------------------------------------
# bit counts
# ---------------------------------------------------------------------------
def _neutral_terms(x: int, ones: bool):
    """(terms, body) of a block's distance from the neutral pattern: x, or 3 - x"""
    return ([(x, -1)], MSG_MOD - 1) if ones else ([(x, 1)], 0)


def _suffix_neutral(c: bc.Circuit, x: Sequence[int], ones: bool) -> List[int]:
    """S[k] = every block k.. is neutral: a radix-5 Hillis-Steele scan, first
    [sum of <= 5 distances == 0], then [sum of <= 5 flags == count]"""
    n = len(x)
    cur = []
    for k in range(n):
        terms, body = [], 0
        for w in x[k:k + bc.MAX_TERMS]:
            t, b = _neutral_terms(w, ones)
            terms += t
            body += b
        cur.append(_pbs(c, terms, body, lambda v: int(v == 0)))
    s = bc.MAX_TERMS
    while s < n:
        nxt = list(cur)
        for k in range(n - s):
            grp = cur[k:n:s][:bc.MAX_TERMS]
            nxt[k] = _pbs(c, [(w, 1) for w in grp], 0, lambda v, g=len(grp): int(v == g))
        cur, s = nxt, s * bc.MAX_TERMS
    return cur


def _sum_one_hot(c: bc.Circuit, x: Sequence[int], columns: List[List[int]]) -> List[int]:
    """per column the sum of its wires, at most one of them non-zero: identity
    PBS on sums of <= 5 (values <= 3 each)"""
    out = []
    for col in columns:
        while len(col) > 1:
            col = [_pbs(c, [(w, 1) for w in col[i:i + bc.MAX_TERMS]], 0, lambda v: v if v < MSG_MOD else 0)
                   for i in range(0, len(col), bc.MAX_TERMS)]
        out.append(col[0] if col else _zero(c, x))
    return out


def first_block_count(c: bc.Circuit, x: Sequence[int], op: str) -> List[int]:
    """leading / trailing zeros / ones, or ilog2, of the bit pattern of x: the
    first non-neutral block from the far end contributes its count"""
    n = len(x)
    bits = 2 * n
    leading = op.startswith("leading") or op == "ilog2"
    ones = op.endswith("ones")
    width = ilog2_blocks(n) if op == "ilog2" else count_blocks(n)
    order = list(reversed(range(n))) if leading else list(range(n))   # far end first
    # flags[q]: the n - q blocks farthest from the near end are neutral, so
    # flags[n - p] covers order[:p], the blocks before order[p], and flags[0] all
    flags = _suffix_neutral(c, [x[k] for k in reversed(order)], ones)
    neutral = MSG_MOD - 1 if ones else 0

    def within(v):   # neutral bits of a non-neutral block from the far end
        far = (v >> 1) & 1 if leading else v & 1
        return int(far == (1 if ones else 0))

    def value(k, v):   # the result when block k (value v) is the first non-neutral one
        if op == "ilog2":
            return 2 * k + (v >> 1)
        before = n - 1 - k if leading else k
        return 2 * before + within(v)

    all_value = (MSG_MOD ** width - 1) if op == "ilog2" else bits
    columns: List[List[int]] = [[] for _ in range(width)]
    for p, k in enumerate(order):
        for j in range(width):
            def f(v, k=k, j=j):
                fl, xv = (v // MSG_MOD, v % MSG_MOD) if p else (1, v)
                if not fl or xv == neutral or xv >= MSG_MOD:
                    return 0
                return (value(k, xv) >> (2 * j)) & (MSG_MOD - 1)
            if not any(f(v) for v in range(bc.TOTAL_MOD)):
                continue
            terms = [(flags[n - p], MSG_MOD), (x[k], 1)] if p else [(x[k], 1)]
            columns[j].append(_pbs(c, terms, 0, f))
    for j in range(width):
        dig = (all_value >> (2 * j)) & (MSG_MOD - 1)
        if dig:
            columns[j].append(_pbs(c, [(flags[0], 1)], 0, lambda v, dig=dig: dig * (v == 1)))
    return _sum_one_hot(c, x, columns)


def count_bits(c: bc.Circuit, x: Sequence[int], ones: bool) -> List[int]:
    """count_ones / count_zeros on COUNT_ONES_BLOCKS blocks"""
    n = len(x)
    pc = [bin(v).count("1") if ones else 2 - bin(v).count("1") for v in range(MSG_MOD)]
    col0 = []
    for i in range(0, n - 1, 2):
        col0.append(_pbs(c, [(x[i + 1], MSG_MOD), (x[i], 1)], 0,
                         lambda v: pc[v // MSG_MOD] + pc[v % MSG_MOD]))
    if n % 2:
        col0.append(_pbs(c, [(x[-1], 1)], 0, lambda v: pc[v] if v < MSG_MOD else 0))
    ncols = count_blocks(n)   # blocks that can hold bits
    columns = [col0] + [[] for _ in range(ncols - 1)]
    vmax = c.vmax

    def done(col):
        return len(col) <= 2 and all(vmax[w] < MSG_MOD for w in col)

    while not all(done(col) for col in columns):
        new: List[List[int]] = [[] for _ in range(ncols)]
        for j, col in enumerate(columns):
            if done(col):
                new[j] += col
                continue
            groups, cur = [], []
            for w in sorted(col, key=lambda w: vmax[w]):
                if cur and (len(cur) == bc.MAX_TERMS or sum(vmax[u] for u in cur) + vmax[w] > bc.MAX_VALUE):
                    groups.append(cur)
                    cur = []
                cur.append(w)
            groups.append(cur)
            for g in groups:
                terms = [(w, 1) for w in g]
                new[j].append(_pbs(c, terms, 0, lambda v: v % MSG_MOD))
                if sum(vmax[w] for w in g) >= MSG_MOD and j + 1 < ncols:
                    new[j + 1].append(_pbs(c, terms, 0, lambda v: v // MSG_MOD))
        columns = new
    top = max(j for j, col in enumerate(columns) if col)
    if all(len(col) <= 1 for col in columns):
        out = [col[0] if col else _zero(c, x) for col in columns[:top + 1]]
    else:
        live = min(ncols, top + 2)   # the add may carry one column up
        a = [[(col[0], 1)] if col else [(_zero(c, x), 1)] for col in columns[:live]]
        b = [[(col[1], 1)] if len(col) > 1 else [] for col in columns[:live]]
        out, _ = radix.add(c, a, b)
    return out + [_zero(c, x)] * (COUNT_ONES_BLOCKS - len(out))


# ---------------------------------------------------------------------------
# compiled circuits
# ---------------------------------------------------------------------------
def check_amount(op: str, amount) -> int:
    if isinstance(amount, bool) or not isinstance(amount, (int, np.integer)) or amount < 0:
        raise ValueError(f"{op} takes a non-negative integer amount, got {amount!r}")
    return int(amount)


def circuit(op: str, num_blocks: int, signed: bool = False, arg: Optional[int] = None) -> bc.Circuit:
    """The circuit of one operation on `num_blocks`-block integers.  Per
    instance, the inputs are the integer's blocks then, for an encrypted
    shift or rotation, the amount's `arg` blocks; a `scalar_*` circuit is
    compiled for the clear amount `arg` (in its canonical form,
    `canonical_amount`).  Outputs are the result's blocks (`result_blocks`),
    for `checked_ilog2` followed by the flag.  The radix.CIRCUIT_CACHE_SIZE
    most recent (op, num_blocks, arg, signed) are kept (an operation that
    does not depend on the signedness has one circuit)."""
    n = radix.check_num_blocks(num_blocks)
    if op not in OPERATIONS:
        raise ValueError(f"unknown radix bit operation {op!r}")
    if op in SHIFTS:
        arg = radix.check_num_blocks(arg)
    elif op.startswith("scalar_"):
        arg = canonical_amount(op, n, check_amount(op, arg))
    else:
        arg = None
    return _circuit(op, n, arg, bool(signed) and op in SIGNED_OPS)


@functools.lru_cache(maxsize=radix.CIRCUIT_CACHE_SIZE)
def _circuit(op: str, n: int, arg: Optional[int], signed: bool) -> bc.Circuit:
    c = bc.Circuit(f"{'signed' if signed else 'unsigned'}_{op}_{n}" + ("" if arg is None else f"_{arg}"))
    x = c.inputs_block(n, False)
    if op in SHIFTS:
        c.output_blocks(shift(c, x, c.inputs_block(arg, False), op, signed))
    elif op.startswith("scalar_"):
        c.output_blocks(scalar_shift(c, x, arg, op[len("scalar_"):], signed))
    elif op in ("count_ones", "count_zeros"):
        c.output_blocks(count_bits(c, x, op == "count_ones"))
    elif op == "checked_ilog2":
        out = first_block_count(c, x, "ilog2")
        nonzero = _suffix_neutral(c, x, False)[0]   # shared with ilog2's flags when the order matches
        if signed:
            neg = _pbs(c, [(x[-1], 1)], 0, lambda v: (v >> 1) & 1)
            flag = _pbs(c, [(nonzero, 2), (neg, 1)], 0, lambda v: int(v == 0))
        else:
            flag = _pbs(c, [(nonzero, 1)], 0, lambda v: int(v == 0))
        c.output_blocks(out + [flag])
    else:
        c.output_blocks(first_block_count(c, x, op))
    return c


# ---------------------------------------------------------------------------
# plain model (the semantics the circuits implement)
# ---------------------------------------------------------------------------
def model(op: str, value: int, num_blocks: int, signed: bool = False, amount: Optional[int] = None):
    """the result of op on the num_blocks-block integer `value`: an int (of
    the operand's signedness for a shift or rotation, unsigned for a count),
    or (ilog2, flag) for checked_ilog2"""
    bits = 2 * num_blocks
    mask = (1 << bits) - 1
    u = value & mask
    base = op[len("scalar_"):] if op.startswith("scalar_") else op
    if base in SHIFTS:
        if base == "left_shift":
            r = (u << amount) & mask if amount < bits else 0
        elif base == "right_shift":
            r = (radix.from_digits(radix.to_digits(u, num_blocks), signed) >> min(amount, bits)) & mask
        else:
            t = (amount % bits) if op.startswith("scalar_") else (amount % (1 << rotation_bits(num_blocks))) % bits
            if base == "rotate_right":
                t = (bits - t) % bits
            r = ((u << t) | (u >> (bits - t))) & mask
        return radix.from_digits(radix.to_digits(r, num_blocks), signed)
    if op in ("count_ones", "count_zeros"):
        ones = bin(u).count("1")
        return ones if op == "count_ones" else bits - ones
    lz = bits - u.bit_length()
    if op in ("ilog2", "checked_ilog2"):
        r = (bits - 1 - lz) % MSG_MOD ** ilog2_blocks(num_blocks)
        return (r, int(value > 0)) if op == "checked_ilog2" else r
    if op == "leading_zeros":
        return lz
    if op == "leading_ones":
        return bits - (u ^ mask).bit_length()
    tz = bits if u == 0 else (u & -u).bit_length() - 1
    if op == "trailing_zeros":
        return tz
    v = u ^ mask
    return bits if v == 0 else (v & -v).bit_length() - 1
