"""Products and sums of radix integers on 2_2 blocks, compiled to batched
KS -> PBS layers by `bit_circuit`: `mul`, `scalar_mul`,
`unsigned_overflowing_mul`, `signed_overflowing_mul` and `sum_ciphertexts`.
Host code only: the GPU runs them with `b200_bit_circuit_64_async` through
`integer.CudaRadixServerKey`, like the circuits of `radix`.

The product restates tfhe-rs' `unchecked_mul_parallelized`
(`integer/server_key/radix_parallel/mul.rs:333-470`, `sum.rs`) as one circuit:

  * partial products: for rhs block i and lhs block j with i + j < n, one PBS
    on 4 y_i + x_j for (x y) mod 4 into column i + j and, when i + j + 1 < n,
    one for (x y) / 4 into column i + j + 1 (noise 5, value 15).  A clear rhs
    (`scalar_mul`) enters as per-instance body constants, so the same rows run
    at noise 1 and one circuit serves every scalar;
  * column compression (`sum.rs`): while a column holds more than 5 terms,
    every full chunk of 5 is summed (value <= 15) and split into its message
    (staying) and carry (one column up) by two PBS;
  * a last split of every column of >= 2 terms into message and carry, whose
    carry moves one column up (each column then holds <= 2 wires of value
    <= 3), and `radix.add`'s carry scan, whose last layer adds the carry bit
    and extracts the message.

Overflow flags:

  * unsigned (`mul.rs:638-713`): [exact product >= 4^n] is the OR of "some
    x_j y_i != 0 with i + j >= n", "some x_j y_i >= 4 with i + j = n - 1" and
    every carry that leaves column n - 1 (in the compression, the last split
    and the scan).  The first is computed with a suffix OR of [x_j != 0]: per
    i one PBS on 4 [some x_j != 0, j >= n - i] + y_i, not one per block pair;
  * signed: tfhe-rs multiplies sign-extended 2n-block operands
    (`mul.rs:824-878`).  Here |x| and |y| come from `radix_div.cond_negate`,
    their unsigned product P and flag U from the circuit above, and the result
    is P negated when the signs differ.  The flag is U or [P >= 2^(b-1)],
    except for P = 2^(b-1) with differing signs (the product MIN).

`sum_ciphertexts` puts block i of every operand in column i and runs the same
compression and carry scan; two operands are one `radix.add`.
"""
from __future__ import annotations

import functools
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import bit_circuit as bc
from . import radix
from . import radix_div
from .radix import MSG_MOD, Block, _pbs, _scaled, blocks_of

OPERATIONS = ("mul", "scalar_mul", "unsigned_overflowing_mul", "signed_overflowing_mul", "sum")


def _or(c: bc.Circuit, bits: List[int]) -> int:
    """one wire holding the OR of `bits`: sums of <= 5 reduced by [v > 0]"""
    while len(bits) > 1:
        bits = [_pbs(c, [(w, 1) for w in bits[i:i + bc.MAX_TERMS]], 0, lambda v: int(v > 0))
                for i in range(0, len(bits), bc.MAX_TERMS)]
    return bits[0]


def products(c: bc.Circuit, x: Sequence[Block], y: Sequence[Block], flags: Optional[List[int]] = None
             ) -> List[List[int]]:
    """the partial-product columns of x * y mod 4^n (`compute_terms_for_mul_low`);
    with `flags`, appends the unsigned overflow bits of the pairs with
    i + j >= n - 1"""
    n = len(x)
    lsb = lambda v: (v // MSG_MOD) * (v % MSG_MOD) % MSG_MOD    # noqa: E731
    msb = lambda v: (v // MSG_MOD) * (v % MSG_MOD) // MSG_MOD   # noqa: E731
    columns: List[List[int]] = [[] for _ in range(n)]
    for i in range(n):
        for j in range(n - i):
            t = _scaled(y[i], MSG_MOD) + list(x[j])
            columns[i + j].append(_pbs(c, t, 0, lsb))
            if i + j + 1 < n:
                columns[i + j + 1].append(_pbs(c, t, 0, msb))
            elif flags is not None:   # i + j = n - 1: the (x y) / 4 that would leave the integer
                flags.append(_pbs(c, t, 0, lambda v: int(v // MSG_MOD * (v % MSG_MOD) >= MSG_MOD)))
    if flags is not None and n > 1:
        # some pair with i + j >= n: y_i != 0 and some x_j != 0 with j >= n - i
        nz = [_pbs(c, list(b), 0, lambda v: int(v != 0)) for b in x[1:]]
        above = radix_div._suffix_any(c, nz)   # above[k - 1] = OR of [x_j != 0], j >= k
        for i in range(1, n):
            flags.append(_pbs(c, [(above[n - i - 1], MSG_MOD)] + list(y[i]), 0,
                              lambda v: int(v // MSG_MOD == 1 and v % MSG_MOD != 0)))
    return columns


def sum_columns(c: bc.Circuit, columns: List[List[int]], flags: Optional[List[int]] = None
                ) -> Tuple[List[int], Optional[int]]:
    """the blocks of sum_i 4^i (sum of column i) mod 4^n, columns holding wires
    of value <= 3; with `flags`, also the flag [the sum >= 4^n] OR-ed with
    `flags`.  Returns (blocks, flag wire or None)."""
    n = len(columns)
    out_flags = None if flags is None else list(flags)

    def split(terms, i, nxt):
        """message of a column chunk stays, its carry goes one column up"""
        t = [(w, 1) for w in terms]
        m = _pbs(c, t, 0, lambda v: v % MSG_MOD)
        if i + 1 < n:
            nxt[i + 1].append(_pbs(c, t, 0, lambda v: v // MSG_MOD))
        elif out_flags is not None:   # a carry out of the top column
            out_flags.append(_pbs(c, t, 0, lambda v: int(v >= MSG_MOD)))
        return m

    while any(len(col) > bc.MAX_TERMS for col in columns):
        new: List[List[int]] = [[] for _ in range(n)]
        for i, col in enumerate(columns):   # the oldest terms first
            new[i] += col[len(col) // bc.MAX_TERMS * bc.MAX_TERMS:] if len(col) >= bc.MAX_TERMS else col
        for i, col in enumerate(columns):
            if len(col) >= bc.MAX_TERMS:
                for k in range(0, len(col) // bc.MAX_TERMS * bc.MAX_TERMS, bc.MAX_TERMS):
                    new[i].append(split(col[k:k + bc.MAX_TERMS], i, new))
        columns = new
    if any(len(col) > 2 for col in columns):
        new = [[] for _ in range(n)]
        msgs = [col[0] if len(col) == 1 else split(col, i, new) for i, col in enumerate(columns)]
        columns = [[m] + extra for m, extra in zip(msgs, new)]
    assert all(1 <= len(col) <= 2 for col in columns)
    if all(len(col) == 1 for col in columns):
        out, carry = [col[0] for col in columns], None
    else:
        a = [[(col[0], 1)] for col in columns]
        b = [[(col[1], 1)] if len(col) > 1 else [] for col in columns]
        out, carry = radix.add(c, a, b, flag=out_flags is not None)
    if out_flags is None:
        return out, None
    last = [] if carry is None else [carry]
    rest = out_flags
    while len(rest) + len(last) > bc.MAX_TERMS:   # OR the early flags down, off the critical path
        rest = [_or(c, rest[i:i + bc.MAX_TERMS]) for i in range(0, len(rest), bc.MAX_TERMS)]
    return out, _or(c, rest + last)


def mul(c: bc.Circuit, x: Sequence[Block], y: Sequence[Block], flag: bool = False
        ) -> Tuple[List[int], Optional[int]]:
    """x * y mod 4^n; with `flag`, also [x * y >= 4^n] (unsigned operands)"""
    flags: Optional[List[int]] = [] if flag else None
    return sum_columns(c, products(c, x, y, flags), flags)


def signed_overflowing_mul(c: bc.Circuit, x: Sequence[int], y: Sequence[int]) -> Tuple[List[int], int]:
    """x * y mod 4^n and [x * y outside [MIN, MAX]] for two's-complement x, y"""
    n = len(x)
    neg = lambda v: v >= MSG_MOD // 2   # noqa: E731
    differ = _pbs(c, [(x[-1], MSG_MOD), (y[-1], 1)], 0, lambda v: int(neg(v // MSG_MOD) != neg(v % MSG_MOD)))
    ax, ay = radix_div.cond_negate(c, x, x[-1], neg), radix_div.cond_negate(c, y, y[-1], neg)
    p, u = mul(c, blocks_of(ax), blocks_of(ay), flag=True)
    # low = [P mod 4^(n-1) == 0]; exact = low and the signs differ, where P = 2^(b-1) is allowed
    if n > 1:
        low = radix.compare(c, blocks_of(p[:-1]), [[] for _ in p[:-1]], "eq")
        exact = _pbs(c, [(low, 1), (differ, 1)], 0, lambda v: int(v == 2))
    else:
        exact = differ
    big = _pbs(c, [(exact, MSG_MOD), (p[-1], 1)], 0,
               lambda v: int(v % MSG_MOD >= 2 and not (v // MSG_MOD == 1 and v % MSG_MOD == 2)))
    flag = _pbs(c, [(big, 1), (u, 1)], 0, lambda v: int(v > 0))
    return radix_div.cond_negate(c, p, differ, lambda s: s == 1), flag


# ---------------------------------------------------------------------------
# compiled circuits
# ---------------------------------------------------------------------------
def check_count(count) -> int:
    if isinstance(count, bool) or not isinstance(count, (int, np.integer)) or count < 1:
        raise ValueError(f"a sum takes a positive integer count of operands, got {count!r}")
    return int(count)


def circuit(op: str, num_blocks: int, count: Optional[int] = None) -> bc.Circuit:
    """The circuit of one operation on `num_blocks`-block integers.  Per
    instance, the inputs are the operands' blocks in argument order (`sum`:
    `count` operands); `scalar_mul` reads the clear rhs as
    `radix.scalar_iconsts`.  The outputs are the result's blocks, followed by
    the flag for the overflowing products.  Signed and unsigned integers share
    every circuit but `signed_overflowing_mul`'s.  The
    radix.CIRCUIT_CACHE_SIZE most recent (op, num_blocks, count) are kept; each
    schedule is compiled once."""
    n = radix.check_num_blocks(num_blocks)
    if op not in OPERATIONS:
        raise ValueError(f"unknown radix product {op!r}")
    return _circuit(op, n, check_count(count) if op == "sum" else None)


@functools.lru_cache(maxsize=radix.CIRCUIT_CACHE_SIZE)
def _circuit(op: str, n: int, count: Optional[int]) -> bc.Circuit:
    c = bc.Circuit(f"{op}_{n}" + ("" if count is None else f"_{count}"))
    if op == "sum":
        xs = [c.inputs_block(n, False) for _ in range(count)]
        if count == 1:
            c.output_blocks(xs[0])
        else:
            c.output_blocks(sum_columns(c, [list(col) for col in zip(*xs)])[0])
        return c
    x = c.inputs_block(n, False)
    if op == "signed_overflowing_mul":
        out, flag = signed_overflowing_mul(c, x, c.inputs_block(n, False))
        c.output_blocks(out + [flag])
        return c
    y = radix.scalar_blocks(c, n) if op == "scalar_mul" else blocks_of(c.inputs_block(n, False))
    out, flag = mul(c, blocks_of(x), y, flag=op == "unsigned_overflowing_mul")
    c.output_blocks(out + ([flag] if flag is not None else []))
    return c


# ---------------------------------------------------------------------------
# plain model (the semantics the circuits implement)
# ---------------------------------------------------------------------------
def model(op: str, operands: Sequence[int], num_blocks: int, signed: bool = False):
    """the result of op on num_blocks-block integers of the given signedness:
    `mul` / `scalar_mul` the wrapping product (`mul.rs:472`), `sum` the
    wrapping sum of every operand (`gpu/server_key/radix/add.rs:405`, None
    for no operand), the overflowing products (product, flag) with the flag
    set when the exact product is >= 2^bits (`mul.rs:638`, unsigned) or
    outside [MIN, MAX] (`mul.rs:824`, signed)"""
    def wrap(v):
        return radix.from_digits(radix.to_digits(v, num_blocks), signed)

    if op == "sum":
        return wrap(sum(operands)) if operands else None
    a, b = operands
    p = a * b
    if op in ("mul", "scalar_mul"):
        return wrap(p)
    lo, hi = radix.scalar_range(num_blocks, signed)
    return wrap(p), int(not lo <= p < hi)
