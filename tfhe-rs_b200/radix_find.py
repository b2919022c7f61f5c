"""Vector find and compare on radix integers, and the encrypted-key
operations of the key-value store (`kv_store.CudaKVStore`), as batched
KS -> PBS layers: `match_value`, `match_value_or`, `contains`,
`contains_clear`, `is_in_clears`, `index_in_clears`, `first_index_in_clears`,
`index_of`, `index_of_clear`, `first_index_of`, `first_index_of_clear`,
`all_eq_slices`, `contains_sub_slice` and `kv_store_get` / `update` / `map` /
`contains_*`.  Host code only: the GPU runs both halves with
`b200_bit_circuit_64_async` through `integer.CudaRadixServerKey`.

Semantics are tfhe-rs' (`vector_find.rs`, `vector_comparisons.rs`,
`kv_store.rs`); `tests/find_model.py` restates them on Python integers.

Every call is two executor calls on 2_2 blocks (sum |c_i| <= 5, value <= 15
on every PBS input, `bit_circuit`):

  * a per-candidate circuit, compiled once per (operation, key blocks, value
    blocks) with the candidates (list entries, clears, store entries) as its
    instance axis.  The query is a shared input; a clear candidate enters as
    per-instance body constants (`radix.scalar_blocks`), an encrypted one as
    per-instance blocks.  The selector sel_i = [query == candidate_i] is
    `radix.compare`'s equality (block equality on 4 q + c, then [sum == k]
    on groups of <= 5); a store read also keeps the entry's value under its
    selector (`radix.keep_if`), a store write selects sel_i ? new : v_i
    (`radix.if_then_else`).  Equality does not depend on the signedness, so
    these circuits do not either.
  * a cross-candidate tree (`Tree`), generated for each candidate count M
    directly as schedule tables for one instance, reading the first call's
    outputs as its inputs at absolute pool rows.  Each step reduces groups of
    <= 5 wires per PBS, so the PBS depth grows with log5 M:
      - OR of the selectors, [sum > 0] (found / contains);
      - AND, [sum == k] (`all_eq_slices`);
      - one-hot sum of selected encrypted blocks, (sum mod 4) on <= 5
        blocks of value <= 3;
      - clear outputs as a dot product: output digit j is
        (sum_i d_ij sel_i) mod 4, the digits as coefficients grouped so that
        their sum stays <= 5, then one-hot sums.  `match_value_or` adds its
        default digit o_j to the body and uses d_ij - o_j mod 4: with at
        most one selector set the digit is d_ij, or o_j when none is;
      - first match only: inclusive prefix ORs P_i by a radix-5
        Hillis-Steele scan, then first_i = [2 sel_i + P_{i-1} == 2];
      - the index: the dot product with the digits of i.
    On duplicate matches the non-`first` index variants give, per output
    digit, the sum mod 4 of the matching indices' digits (tfhe-rs leaves the
    result unspecified; its one-hot aggregation adds blocks without
    carries).
"""
from __future__ import annotations

import functools
from typing import Callable, List, Sequence, Tuple

import numpy as np

from . import bit_circuit as bc
from . import radix
from .radix import MSG_MOD, blocks_of

CANDIDATE_OPS = ("eq_clear", "eq", "select", "apply", "update")


# ---------------------------------------------------------------------------
# per-candidate circuits
# ---------------------------------------------------------------------------
def circuit(op: str, key_blocks: int, value_blocks: int = 0) -> bc.Circuit:
    """The per-candidate circuit of `op` (one of CANDIDATE_OPS); candidates
    are its instances.  Shared inputs, in order: the query's `key_blocks`
    blocks (`apply`: none), then for `update` / `apply` the new value's
    `value_blocks` blocks.  Per instance:
      eq_clear: the candidate's 2 * key_blocks digit bits as constants
                -> [sel];
      eq:       the candidate's blocks -> [sel];
      select:   key digits as constants, the entry's value -> [sel] + (sel ? v : 0);
      apply:    the entry's selector, its value -> (sel ? new : v);
      update:   key digits as constants, the entry's value -> [sel] + (sel ? new : v).
    The radix.CIRCUIT_CACHE_SIZE most recent circuits are kept."""
    if op not in CANDIDATE_OPS:
        raise ValueError(f"unknown per-candidate operation {op!r}")
    nk = radix.check_num_blocks(key_blocks) if op != "apply" else 0
    nv = radix.check_num_blocks(value_blocks) if op in ("select", "apply", "update") else 0
    return _circuit(op, nk, nv)


@functools.lru_cache(maxsize=radix.CIRCUIT_CACHE_SIZE)
def _circuit(op: str, nk: int, nv: int) -> bc.Circuit:
    c = bc.Circuit(f"find_{op}_{nk}_{nv}")
    query = blocks_of(c.inputs_block(nk, True))
    new = blocks_of(c.inputs_block(nv, True)) if op in ("apply", "update") else None
    if op == "apply":
        sel = c.input(False)
        c.output_blocks(radix.if_then_else(c, sel, new, blocks_of(c.inputs_block(nv, False))))
        return c
    cand = blocks_of(c.inputs_block(nk, False)) if op == "eq" else radix.scalar_blocks(c, nk)
    sel = radix.compare(c, query, cand, "eq")
    if op in ("eq", "eq_clear"):
        c.output_blocks([sel])
        return c
    value = blocks_of(c.inputs_block(nv, False))
    kept = radix.keep_if(c, sel, value) if op == "select" else radix.if_then_else(c, sel, new, value)
    c.output_blocks([sel] + kept)
    return c


# ---------------------------------------------------------------------------
# cross-candidate trees
# ---------------------------------------------------------------------------
class Tree:
    """PBS rows over the outputs of a per-candidate call (the tree's inputs,
    pool rows 0 .. num_inputs - 1), laid out as a `bit_circuit.Schedule` for
    one instance: every slot is a pool row, none is reused, each row goes to
    the layer after its latest input."""

    def __init__(self, name: str, input_vmax: Sequence[int]):
        self.name = name
        self.num_inputs = len(input_vmax)
        self.vmax = [int(v) for v in input_vmax]
        self.layer = [0] * self.num_inputs
        self.rows: List[Tuple[Tuple[Tuple[int, int], ...], int, int, int]] = []   # (terms, body, table, out)
        self.tables: List[Tuple[int, ...]] = []

    def pbs(self, terms: Sequence[Tuple[int, int]], body: int, f: Callable[[int], int]) -> int:
        terms = tuple((int(w), int(k)) for w, k in terms)
        noise = sum(abs(k) for _, k in terms)
        lo = body + sum(min(0, k) * self.vmax[w] for w, k in terms)
        hi = body + sum(max(0, k) * self.vmax[w] for w, k in terms)
        assert noise <= bc.MAX_NOISE_LEVEL and 0 <= lo and hi <= bc.MAX_VALUE, (self.name, terms, body)
        t = tuple(int(f(v)) for v in range(bc.TOTAL_MOD))
        if t not in self.tables:
            self.tables.append(t)
        out = len(self.vmax)
        self.vmax.append(max(t))
        self.layer.append(1 + max(self.layer[w] for w, _ in terms))
        self.rows.append((terms, int(body), self.tables.index(t), out))
        return out

    def _reduce(self, wires: Sequence[int], f_of_count) -> int:
        wires = list(wires)
        while len(wires) > 1:
            wires = [self.pbs([(w, 1) for w in g], 0, f_of_count(len(g))) if len(g) > 1 else g[0]
                     for g in (wires[i:i + bc.MAX_TERMS] for i in range(0, len(wires), bc.MAX_TERMS))]
        return wires[0]

    def any(self, bits: Sequence[int]) -> int:
        """OR of >= 1 bits: [sum > 0] on groups of <= 5"""
        return self._reduce(bits, lambda k: (lambda v: int(v > 0)))

    def all(self, bits: Sequence[int]) -> int:
        """AND of >= 1 bits: [sum == k] on groups of k <= 5"""
        return self._reduce(bits, lambda k: (lambda v, k=k: int(v == k)))

    def sum(self, blocks: Sequence[int]) -> int:
        """(sum mod 4) of >= 1 blocks of value <= 3: at most one is non-zero
        when the blocks were kept under one-hot selectors"""
        return self._reduce(blocks, lambda k: (lambda v: v % MSG_MOD))

    def dot(self, sels: Sequence[int], clears: Sequence[int], width: int, default: int = 0) -> List[int]:
        """the `width` blocks of sum_i sel_i * clears[i] (one-hot sels), or of
        `default` when no selector is set"""
        out = []
        for j in range(width):
            dj = (default >> (2 * j)) & (MSG_MOD - 1)
            coefs = [((int(v) >> (2 * j)) - dj) % MSG_MOD for v in clears]
            groups, cur = [], []
            for s, k in zip(sels, coefs):
                if not k:
                    continue
                if sum(kk for _, kk in cur) + k > bc.MAX_NOISE_LEVEL:
                    groups.append(cur)
                    cur = []
                cur.append((s, k))
            if cur or not groups:
                groups.append(cur)
            firsts = []
            for gi, g in enumerate(groups):
                body = dj if gi == 0 else 0
                if not g:   # no selector changes this digit: a PBS making the constant
                    firsts.append(self.pbs([(sels[0], 1)], 0, lambda v, dj=dj: dj))
                else:
                    firsts.append(self.pbs(g, body, lambda v: v % MSG_MOD))
            out.append(self.sum(firsts))
        return out

    def first(self, sels: Sequence[int]) -> List[int]:
        """only the first set selector: first_i = sel_i and not P_{i-1}, P_i
        the inclusive prefix OR, by a radix-5 Hillis-Steele scan"""
        M = len(sels)
        if M <= 1:
            return list(sels)
        P, span = list(sels), 1
        while span < M - 1:   # P[i] covers sels[i - span + 1 .. i]; P[i] for i <= M - 2 is read
            nxt = []
            for i in range(M - 1):
                g = [P[j] for j in range(i, i - bc.MAX_TERMS * span, -span) if j >= 0]
                nxt.append(g[0] if len(g) == 1 else self.pbs([(w, 1) for w in g], 0, lambda v: int(v > 0)))
            P, span = nxt, span * bc.MAX_TERMS
        return [sels[0]] + [self.pbs([(sels[i], 2), (P[i - 1], 1)], 0, lambda v: int(v == 2)) for i in range(1, M)]

    def schedule(self, outputs: Sequence[int]) -> bc.Schedule:
        rows = sorted(self.rows, key=lambda r: (self.layer[r[3]], r[3]))
        num_layers = max([self.layer[r[3]] for r in rows], default=0)
        layer_rows = np.searchsorted(np.array([self.layer[r[3]] for r in rows], dtype=np.int64),
                                     np.arange(1, num_layers + 2), side="left")
        offs = np.cumsum([0] + [len(r[0]) for r in rows])
        return bc.Schedule(
            circuit_name=self.name, num_instances=1, num_shared_slots=0, num_instance_slots=len(self.vmax),
            layer_rows=layer_rows.astype(np.uint32), layer_shared_rows=np.zeros(num_layers, dtype=np.uint32),
            row_offsets=offs.astype(np.uint32),
            term_slots=np.array([w for r in rows for w, _ in r[0]], dtype=np.uint32),
            term_coefs=np.array([k for r in rows for _, k in r[0]], dtype=np.int64),
            body_base=np.array([r[1] for r in rows], dtype=np.int64),
            iterm_rows=np.zeros(0, dtype=np.int64), iterm_index=np.zeros(0, dtype=np.int64),
            iterm_coefs=np.zeros(0, dtype=np.int64),
            row_lut=np.array([bc.NUM_FIXED_LUTS + r[2] for r in rows], dtype=np.uint32),
            row_dest=np.array([r[3] for r in rows], dtype=np.uint32),
            frees=[np.zeros(0, dtype=np.int64) for _ in range(num_layers + 1)],
            shared_input_slots=np.zeros(0, dtype=np.int64),
            instance_input_slots=np.arange(self.num_inputs, dtype=np.int64),
            output_slots=np.array(outputs, dtype=np.int64), num_iconsts=0,
            pbs_per_instance_rows=len(rows), pbs_shared_rows=0, extra_luts=tuple(self.tables))


@functools.lru_cache(maxsize=radix.CIRCUIT_CACHE_SIZE)
def tree(kind: str, M: int, per: int = 1, width: int = 0, clears: Tuple[int, ...] = (), default: int = 0,
         first: bool = False) -> bc.Schedule:
    """The cross-candidate schedule of one call over M candidates, each
    giving `per` outputs of the per-candidate call (its selector first).
    Outputs, by kind:
      any:     [OR of sels];
      all:     [AND of sels];
      windows: M = windows * per selectors, window-major: [OR over windows of the AND of each];
      dot:     `width` blocks of the clears selected (the first match only with
               `first`; `default` where none matches), then [OR of sels];
      dot_or:  the `width` blocks of `dot` alone;
      select:  the one-hot sum of each of the per - 1 value columns, then [OR of sels];
    The radix.CIRCUIT_CACHE_SIZE most recent trees are kept."""
    t = Tree(f"find_tree_{kind}_{M}", [1 if k == 0 or kind == "windows" else MSG_MOD - 1
                                       for _ in range(M) for k in range(per)])
    sels = [i * per for i in range(M)]
    if kind == "any":
        return t.schedule([t.any(sels)])
    if kind == "all":
        return t.schedule([t.all(sels)])
    if kind == "windows":
        return t.schedule([t.any([t.all(list(range(w * per, (w + 1) * per))) for w in range(M)])])
    if kind in ("dot", "dot_or"):
        picked = t.first(sels) if first else sels
        out = t.dot(picked, clears, width, default)
        return t.schedule(out if kind == "dot_or" else out + [t.any(sels)])
    assert kind == "select"
    cols = [t.sum([i * per + k for i in range(M)]) for k in range(1, per)]
    return t.schedule(cols + [t.any(sels)])


def num_blocks_for(value: int) -> int:
    """tfhe-rs `num_blocks_to_represent_unsigned_value`: blocks of the bits of
    an unsigned value (at least one bit)"""
    return (max(int(value).bit_length(), 1) + 1) // 2


# ---------------------------------------------------------------------------
# PBS and layer counts of the store operations and the searches (per call)
# ---------------------------------------------------------------------------
def cost(op: str, M: int, key_blocks: int, value_blocks: int = 0) -> Tuple[int, int]:
    """(PBS, PBS layers) of one call of `op` over M candidates:
    `kv_store_get` / `kv_store_update` on a store of M entries,
    `match_value` with M matches of outputs < 4^value_blocks, `contains` over
    M encrypted integers; the per-candidate call then the tree."""
    if M == 0:
        return 0, 0
    if op == "kv_store_get":
        s, t = circuit("select", key_blocks, value_blocks), tree("select", M, 1 + value_blocks)
    elif op == "kv_store_update":
        s, t = circuit("update", key_blocks, value_blocks), tree("any", M)
    elif op == "match_value":
        s = circuit("eq_clear", key_blocks)
        t = tree("dot", M, 1, value_blocks, tuple(MSG_MOD ** value_blocks - 1 - i for i in range(M)))
    elif op == "contains":
        s, t = circuit("eq", key_blocks), tree("any", M)
    else:
        raise ValueError(f"no cost model for {op!r}")
    one = bc.schedule(s, M)
    return one.pbs_count() + t.pbs_count(), one.num_layers + t.num_layers


# ---------------------------------------------------------------------------
# the operations on `integer.CudaRadixServerKey` (argument checks first, then
# the per-candidate call and the tree)
# ---------------------------------------------------------------------------
def _one(key, ct, what: str):
    """(kind, num_blocks) of a single-integer operand"""
    kind, n, I = key._operands(ct)
    if I != 1:
        raise ValueError(f"{what} must hold one integer (num_inputs = 1), got {I}")
    return kind, n


def _stack(key, cts, what: str):
    """(kind, num_blocks, blocks [M * num_blocks, W]) of a non-empty list of
    single-integer ciphertexts of one kind and block count"""
    import torch

    kind, n, I = key._operands(*cts)
    if I != 1:
        raise ValueError(f"every entry of {what} must hold one integer (num_inputs = 1), got {I}")
    return kind, n, torch.cat([ct.blocks for ct in cts])


def _same(kind, n, other_kind, other_n, what: str):
    if other_kind is not kind:
        raise ValueError(f"{what} differs in signedness: {kind.__name__} and {other_kind.__name__}")
    if other_n != n:
        raise ValueError(f"{what} differs in block count: {n} and {other_n}")


def _clears(values, n: int, signed: bool) -> np.ndarray:
    """per-candidate digit bits of clear values (ValueError outside the range
    of an n-block integer of that signedness)"""
    return radix.scalar_iconsts(list(values), n, signed)


def _check_outputs(values, what: str) -> List[int]:
    out = []
    for v in values:
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 0 \
                or num_blocks_for(v) > radix.MAX_BLOCKS:
            raise ValueError(f"{what} must be unsigned integers of at most {2 * radix.MAX_BLOCKS} bits, got {v!r}")
        out.append(int(v))
    return out


def _trivial(key, value: int, n: int, kind=None):
    from . import integer

    blocks = key.runner.trivial(radix.to_digits(value, n))
    return integer.CudaBooleanBlock(blocks, 1) if kind is None else kind(blocks, 1)


def _find(key, circ: bc.Circuit, M: int, shared, instance, iconsts, tree_args: tuple, take=None):
    """the per-candidate call over M candidates, then the tree `tree(*tree_args)`
    on its outputs (columns `take` of each candidate's, all by default).
    Returns (per-candidate outputs [M, outs, W], tree outputs [outs, W])."""
    import torch

    out = key.runner.run(circ, shared, instance, iconsts, M)
    W = out.shape[-1]
    per = out.reshape(M, -1, W)
    inputs = (per if take is None else per[:, list(take)]).reshape(-1, W)
    sched = tree(*tree_args)
    if sched.num_layers == 0:   # one candidate: its outputs are the result
        return per, inputs[torch.as_tensor(sched.output_slots, device=inputs.device)]
    return per, key.runner.run_schedule(("find_tree",) + tree_args, sched, inputs)


def _bool(out):
    from . import integer

    return integer.CudaBooleanBlock(out, 1)


def _index_result(out, width):
    """(the unsigned radix of the first `width` output blocks, the flag after them)"""
    from . import integer

    return integer.CudaUnsignedRadixCiphertext(out[:width], 1), _bool(out[width:])


def _matches(matches) -> Tuple[List[int], List[int]]:
    pairs = list(matches.items()) if isinstance(matches, dict) else [tuple(p) for p in matches]
    if any(len(p) != 2 for p in pairs):
        raise ValueError("matches must be (input, output) pairs")
    ins, outs = [p[0] for p in pairs], [p[1] for p in pairs]
    return ins, outs


def match_value(key, ct, matches):
    """tfhe-rs `match_value`: (the output of the match whose input equals ct,
    or 0; [a match was found]) on num_blocks_for(largest output) blocks"""
    from . import integer

    kind, n = _one(key, ct, "the matched integer")
    if kind.signed:
        raise ValueError("match_value takes an unsigned integer")
    ins, outs = _matches(matches)
    if len(set(ins)) != len(ins):
        raise ValueError("the inputs of match_value must be unique")
    iconsts = _clears(ins, n, False)
    outs = _check_outputs(outs, "match outputs")
    if not ins:
        return _trivial(key, 0, 1, integer.CudaUnsignedRadixCiphertext), _trivial(key, 0, 1)
    width = num_blocks_for(max(outs))
    M = len(ins)
    if max(outs) == 0:   # 0 is the only output: only the flag is computed
        _, t = _find(key, circuit("eq_clear", n), M, ct.blocks, None, iconsts, ("any", M))
        return _trivial(key, 0, width, integer.CudaUnsignedRadixCiphertext), _bool(t)
    _, t = _find(key, circuit("eq_clear", n), M, ct.blocks, None, iconsts, ("dot", M, 1, width, tuple(outs)))
    return _index_result(t, width)


def match_value_or(key, ct, matches, or_value):
    """tfhe-rs `match_value_or`: the matched output, or `or_value` when no
    input matches, on enough blocks for both"""
    from . import integer

    kind, n = _one(key, ct, "the matched integer")
    if kind.signed:
        raise ValueError("match_value_or takes an unsigned integer")
    ins, outs = _matches(matches)
    if len(set(ins)) != len(ins):
        raise ValueError("the inputs of match_value_or must be unique")
    iconsts = _clears(ins, n, False)
    outs = _check_outputs(outs, "match outputs")
    (or_value,) = _check_outputs([or_value], "or_value")
    if not ins:
        return _trivial(key, or_value, num_blocks_for(or_value), integer.CudaUnsignedRadixCiphertext)
    width = max(num_blocks_for(max(outs)), num_blocks_for(or_value))
    M = len(ins)
    _, t = _find(key, circuit("eq_clear", n), M, ct.blocks, None, iconsts,
                 ("dot_or", M, 1, width, tuple(outs), or_value))
    return integer.CudaUnsignedRadixCiphertext(t, 1)


def _selectors(key, cts, value=None, clear=None):
    """(kind, n, M, circuit, shared, instance, iconsts) of the equality of
    each entry of `cts` with an encrypted `value` or a `clear` one"""
    kind, n, stacked = _stack(key, cts, "the list")
    M = len(cts)
    if value is not None:
        _same(kind, n, *_one(key, value, "the searched value"), "the searched value")
        return kind, n, M, circuit("eq", n), value.blocks, stacked, None
    iconsts = _clears([clear] * M, n, kind.signed)
    return kind, n, M, radix.circuit("scalar_eq", n), None, stacked, iconsts


def contains(key, cts, value):
    """[value is in cts]"""
    cts = list(cts)
    if not cts:
        _one(key, value, "the searched value")
        return _trivial(key, 0, 1)
    _, _, M, circ, shared, inst, iconsts = _selectors(key, cts, value=value)
    return _bool(_find(key, circ, M, shared, inst, iconsts, ("any", M))[1])


def contains_clear(key, cts, clear):
    """[clear is in cts]"""
    cts = list(cts)
    if not cts:
        return _trivial(key, 0, 1)
    _, _, M, circ, shared, inst, iconsts = _selectors(key, cts, clear=clear)
    return _bool(_find(key, circ, M, shared, inst, iconsts, ("any", M))[1])


def is_in_clears(key, ct, clears):
    """[ct is one of the clears]"""
    kind, n = _one(key, ct, "the searched integer")
    iconsts = _clears(clears, n, kind.signed)
    M = len(iconsts)
    if not M:
        return _trivial(key, 0, 1)
    return _bool(_find(key, circuit("eq_clear", n), M, ct.blocks, None, iconsts, ("any", M))[1])


def index_in_clears(key, ct, clears, first: bool = False):
    """(index of ct in clears, found); `first`: of its first occurrence, the
    later duplicates dropped before the search as tfhe-rs does"""
    from . import integer

    kind, n = _one(key, ct, "the searched integer")
    clears = list(clears)
    iconsts = _clears(clears, n, kind.signed)
    if not clears:
        return _trivial(key, 0, n, integer.CudaUnsignedRadixCiphertext), _trivial(key, 0, 1)
    idx = list(range(len(clears)))
    if first:
        seen = {}
        for i, v in enumerate(clears):
            seen.setdefault(int(v), i)
        idx = sorted(seen.values())
        iconsts = iconsts[idx]
    M, width = len(idx), num_blocks_for(max(idx))
    _, t = _find(key, circuit("eq_clear", n), M, ct.blocks, None, iconsts, ("dot", M, 1, width, tuple(idx)))
    return _index_result(t, width)


def index_of(key, cts, value=None, clear=None, first: bool = False):
    """(index of the encrypted `value` or the `clear` in cts, found);
    `first`: of its first occurrence"""
    from . import integer

    cts = list(cts)
    if not cts:
        n = _one(key, value, "the searched value")[1] if value is not None else 1
        return _trivial(key, 0, n, integer.CudaUnsignedRadixCiphertext), _trivial(key, 0, 1)
    _, _, M, circ, shared, inst, iconsts = _selectors(key, cts, value=value, clear=clear)
    width = num_blocks_for(M - 1)
    _, t = _find(key, circ, M, shared, inst, iconsts, ("dot", M, 1, width, tuple(range(M)), 0, first))
    return _index_result(t, width)


def all_eq_slices(key, lhs, rhs):
    """[lhs and rhs have the same length and are equal entry by entry]; a
    pair of different block counts is unequal"""
    import torch

    lhs, rhs = list(lhs), list(rhs)
    if len(lhs) != len(rhs):
        return _trivial(key, 0, 1)
    if not lhs:
        return _trivial(key, 1, 1)
    if any(_one(key, a, "an entry")[1] != _one(key, b, "an entry")[1] for a, b in zip(lhs, rhs)):
        return _trivial(key, 0, 1)
    kind, n, _ = key._operands(*lhs, *rhs)
    M = len(lhs)
    W = lhs[0].blocks.shape[-1]
    inst = torch.cat([torch.cat([a.blocks, b.blocks]) for a, b in zip(lhs, rhs)]).reshape(-1, W)
    return _bool(_find(key, radix.circuit("eq", n), M, None, inst, None, ("all", M))[1])


def contains_sub_slice(key, lhs, pattern):
    """[pattern occurs in lhs as a contiguous run]"""
    import torch

    lhs, pattern = list(lhs), list(pattern)
    if not pattern:
        raise ValueError("contains_sub_slice needs a non-empty pattern")
    for ct in lhs + pattern:
        _one(key, ct, "an entry")
    kind, n, _ = key._operands(*lhs, *pattern)
    if len(pattern) > len(lhs):
        return _trivial(key, 0, 1)
    P, windows = len(pattern), len(lhs) - len(pattern) + 1
    inst = torch.cat([torch.cat([lhs[w + j].blocks, pattern[j].blocks]) for w in range(windows) for j in range(P)])
    return _bool(_find(key, radix.circuit("eq", n), windows * P, None, inst, None, ("windows", windows, P))[1])


# -- the key-value store --------------------------------------------------------
def _store_key(key, store, enc_key):
    kind, nk = _one(key, enc_key, "the encrypted key")
    iconsts = _clears(store.keys(), nk, kind.signed)
    return kind, nk, iconsts


def _store_value(store, value, what: str):
    from . import integer

    if not isinstance(value, integer.CudaUnsignedRadixCiphertext) or value.num_inputs != 1:
        raise ValueError(f"{what} must be a radix ciphertext holding one integer")
    _same(store.kind, store.num_blocks, type(value), value.num_blocks, what)


def kv_store_get(key, store, enc_key, _selectors_too: bool = False):
    """(the value stored under the key equal to enc_key, or 0 on the key's
    block count for an empty store; found)"""
    kind, nk, iconsts = _store_key(key, store, enc_key)
    M = len(store)
    if not M:
        res = (_trivial(key, 0, nk, kind), _trivial(key, 0, 1))
        return res + (None,) if _selectors_too else res
    nv = store.num_blocks
    per, t = _find(key, circuit("select", nk, nv), M, enc_key.blocks, store.stacked(), iconsts,
                   ("select", M, 1 + nv))
    res = (store.kind(t[:nv], 1), _bool(t[nv:]))
    return res + (per[:, :1],) if _selectors_too else res


def kv_store_update(key, store, enc_key, new_value):
    """every entry v_i becomes sel_i ? new_value : v_i; returns found"""
    import torch

    kind, nk, iconsts = _store_key(key, store, enc_key)
    M = len(store)
    if not M:
        return _trivial(key, 0, 1)
    _store_value(store, new_value, "the new value")
    nv = store.num_blocks
    shared = torch.cat([enc_key.blocks, new_value.blocks])
    per, t = _find(key, circuit("update", nk, nv), M, shared, store.stacked(), iconsts, ("any", M), take=[0])
    store._set_values(per[:, 1:])
    return _bool(t)


def kv_store_map(key, store, enc_key, func):
    """(old, new, found): old as `kv_store_get`, new = func(old), and every
    entry v_i becomes sel_i ? new : v_i (the selectors of the read reused)"""
    import torch

    old, found, sels = kv_store_get(key, store, enc_key, _selectors_too=True)
    new = func(old)
    M = len(store)
    if M:
        _store_value(store, new, "the mapped value")
        nv = store.num_blocks
        W = new.blocks.shape[-1]
        inst = torch.cat([sels, store.stacked().reshape(M, nv, W)], 1).reshape(-1, W)
        out = key.runner.run(circuit("apply", 0, nv), new.blocks, inst, None, M)
        store._set_values(out.reshape(M, nv, W))
    return old, new, found


def kv_store_contains_key(key, store, enc_key):
    kind, nk, iconsts = _store_key(key, store, enc_key)
    M = len(store)
    if not M:
        return _trivial(key, 0, 1)
    return _bool(_find(key, circuit("eq_clear", nk), M, enc_key.blocks, None, iconsts, ("any", M))[1])


def kv_store_contains_value(key, store, value):
    return contains(key, store.values(), value)


def kv_store_contains_clear_value(key, store, clear):
    return contains_clear(key, store.values(), clear)
