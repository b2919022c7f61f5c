"""Boolean circuits on encrypted bits, compiled to batched KS -> PBS layers.

A bit is a shortint block holding 0 or 1 at delta = 2^63 / 16.  Every
ciphertext the engine bootstraps is a *linear step*

    sum_i c_i * w_i + c_0

over wires w_i that are fresh client bits or PBS outputs, followed by one
keyswitch and one PBS with a LUT of the fixed set `lut_functions()` (or of the
circuit's own tables, `Circuit.add_lut`, indexed after it).  The compiler keeps
every such input inside the noise contract of the 2_2 parameter sets
(tfhe-rs `MaxNoiseLevel` 5, scalar multiplication multiplying the noise level):

    sum_i |c_i| * level(w_i) <= 5    and    value in [0, 15],

with level 1 for every wire the engine stores.  XOR / NOT are free: a wire is
kept as a parity *form* (a set of stored wires plus constants) and folded into
its consumers' linear steps; a form is only bootstrapped when a consumer could
not take it within the budget.  An AND is one PBS on `w * a + b` (w > max b)
when `w * |a| + |b| <= 5`; otherwise its operands are first reduced by parity
PBS, earliest-ready wires first.  Rows go to the earliest layer their inputs
allow (as soon as possible), and stored wires share slots once their last
reader has run.

A circuit is compiled once, and its schedule is laid out for any instance
count, bit-sliced: slots are wire-major, instance-minor, and wires that
depend only on shared inputs (keys, an IV) are stored and computed once.
Per-instance plaintext bits (a counter) enter as per-instance body constants.

The schedule's tables are consumed by three executors: `run_cleartext` below
(values and noise levels, asserting the budget on every row), an oracle-backed
one in the tests, and the GPU's `b200_bit_circuit_64_async`.
"""
from __future__ import annotations

import dataclasses
import weakref
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

MAX_NOISE_LEVEL = 5   # MaxNoiseLevel of the 2_2 parameter sets
MAX_VALUE = 15        # message * carry modulus - 1
TOTAL_MOD = 16
MAX_TERMS = 5         # a parity PBS folds at most 5 level-1 wires

# ---------------------------------------------------------------------------
# LUT set (index order of the accumulators uploaded by the executors)
# ---------------------------------------------------------------------------
LUT_PARITY = 0                      # x mod 2
LUT_AND_BASE = 1                    # 1 + 4 * (w - 2) + 2 * fa + fb, w in {2, 3}
LUT_COMBINE = 9                     # carry state 3 * cur + prev -> prev if cur == P else cur
LUT_SUM_BIT = 10                    # 3 * (bit + k) + prev -> (bit ^ k) ^ [prev == G]
ST_KILL, ST_PROPAGATE, ST_GENERATE = 0, 1, 2


def lut_and(w: int, fa: int, fb: int) -> int:
    return LUT_AND_BASE + 4 * (w - 2) + 2 * fa + fb


def lut_functions() -> List[List[int]]:
    """f tables over the 16 values of the padded message space, by LUT index."""
    parity = [x & 1 for x in range(TOTAL_MOD)]
    ands = [[(((x // w) & 1) ^ fa) & (((x % w) & 1) ^ fb) for x in range(TOTAL_MOD)]
            for w in (2, 3) for fa in (0, 1) for fb in (0, 1)]
    combine = [((x % 3) if x // 3 == ST_PROPAGATE else x // 3) if x < 9 else 0 for x in range(TOTAL_MOD)]
    sum_bit = [((x // 3) & 1) ^ (1 if x % 3 == ST_GENERATE else 0) for x in range(TOTAL_MOD)]
    return [parity] + ands + [combine, sum_bit]


# largest value each LUT can output (the value range of the wire it makes)
LUT_VMAX = [1] * 9 + [2, 1]
NUM_FIXED_LUTS = len(LUT_VMAX)
MAX_BLOCK_VALUE = 3   # message modulus - 1: the largest value an output block may hold


def lut_glwes(polynomial_size: int, glwe_dimension: int, tables: Optional[Sequence[Sequence[int]]] = None
              ) -> np.ndarray:
    """The accumulators of `tables` (default `lut_functions()`) for the 2_2 encoding."""
    from . import algorithms

    delta = (1 << 63) // TOTAL_MOD
    return np.stack([algorithms.generate_programmable_bootstrap_glwe_lut(
        polynomial_size, glwe_dimension + 1, TOTAL_MOD, delta, f)
        for f in (lut_functions() if tables is None else tables)])


# ---------------------------------------------------------------------------
# circuits
# ---------------------------------------------------------------------------
class Circuit:
    """A DAG of gates on wire ids.  Gates:
      ('in', shared, index)        fresh client bit (shared or per instance),
                                   or message block (`input_block`, vmax 3)
      ('const', b)                 shared constant bit
      ('iconst', index)            per-instance plaintext bit (given per call)
      ('xor', a, b), ('not', a), ('and', a, b)
      ('lut', ((wire, coef), ...), c0, lut)   one PBS on an explicit linear step
      ('mat', a)                   store `a` as a PBS output (a refresh point)
    `lut` terms read the wire's *value* (a bit, or a carry state in {0, 1, 2});
    a term on an XOR form of several wires is stored first.  Only `lut` gates
    may read a wire whose values exceed 1 (a carry state, or a client message
    block made by `input_block`): the bit gates and `output` raise
    ValueError on one.  `output_blocks` is the explicit opt-in for outputs
    that are 2_2 message blocks (values up to MAX_BLOCK_VALUE).

    A circuit may carry LUT tables of its own (`add_lut`): they take the
    indexes after the fixed set, and the executors upload their accumulators
    with it."""

    def __init__(self, name: str):
        self.name = name
        self.gates: List[tuple] = []
        self.num_shared_inputs = 0
        self.num_instance_inputs = 0
        self.num_iconsts = 0
        self.outputs: List[int] = []
        self.vmax: List[int] = []   # largest value of each wire
        self.extra_luts: List[Tuple[int, ...]] = []   # circuit-local tables, LUT index NUM_FIXED_LUTS + i

    def _add(self, g, vmax: int = 1) -> int:
        self.gates.append(g)
        self.vmax.append(vmax)
        return len(self.gates) - 1

    def _bits(self, *ws: int):
        for w in ws:
            if self.vmax[w] != 1:
                raise ValueError(f"{self.name}: wire {w} holds values up to {self.vmax[w]}, not a bit; "
                                 "only a `lut` gate can read it")

    def input(self, shared: bool) -> int:
        if shared:
            self.num_shared_inputs += 1
            return self._add(("in", True, self.num_shared_inputs - 1))
        self.num_instance_inputs += 1
        return self._add(("in", False, self.num_instance_inputs - 1))

    def inputs(self, count: int, shared: bool) -> List[int]:
        return [self.input(shared) for _ in range(count)]

    def input_block(self, shared: bool) -> int:
        """A fresh client message block (values up to MAX_BLOCK_VALUE): only
        `lut` gates may read it, like a carry state."""
        w = self.input(shared)
        self.vmax[w] = MAX_BLOCK_VALUE
        return w

    def inputs_block(self, count: int, shared: bool) -> List[int]:
        return [self.input_block(shared) for _ in range(count)]

    def const(self, b: int) -> int:
        return self._add(("const", int(b) & 1))

    def iconst(self) -> int:
        self.num_iconsts += 1
        return self._add(("iconst", self.num_iconsts - 1))

    def xor(self, a: int, b: int) -> int:
        self._bits(a, b)
        return self._add(("xor", a, b))

    def xor_all(self, ws: Sequence[int]) -> int:
        acc = ws[0]
        for w in ws[1:]:
            acc = self.xor(acc, w)
        return acc

    def not_(self, a: int) -> int:
        self._bits(a)
        return self._add(("not", a))

    def xnor(self, a: int, b: int) -> int:
        return self.not_(self.xor(a, b))

    def and_(self, a: int, b: int) -> int:
        self._bits(a, b)
        return self._add(("and", a, b))

    def add_lut(self, table: Sequence[int]) -> int:
        """A LUT of this circuit: f over the 16 values of the padded message
        space, outputs in [0, MAX_VALUE]; returns its LUT index."""
        table = tuple(int(v) for v in table)
        if len(table) != TOTAL_MOD or min(table) < 0 or max(table) > MAX_VALUE:
            raise ValueError(f"{self.name}: a LUT maps the {TOTAL_MOD} values to [0, {MAX_VALUE}]")
        self.extra_luts.append(table)
        return NUM_FIXED_LUTS + len(self.extra_luts) - 1

    def lut_tables(self) -> List[List[int]]:
        """every table a `lut` gate of this circuit may name, by LUT index"""
        return lut_functions() + [list(t) for t in self.extra_luts]

    def lut_vmax(self, lut: int) -> int:
        return LUT_VMAX[lut] if lut < NUM_FIXED_LUTS else max(self.extra_luts[lut - NUM_FIXED_LUTS])

    def lut(self, terms: Sequence[Tuple[int, int]], c0: int, lut: int) -> int:
        if not 0 <= lut < NUM_FIXED_LUTS + len(self.extra_luts):
            raise ValueError(f"{self.name}: unknown LUT {lut}")
        return self._add(("lut", tuple((int(w), int(c)) for w, c in terms), int(c0), int(lut)), self.lut_vmax(lut))

    def mat(self, a: int) -> int:
        self._bits(a)
        return self._add(("mat", a))

    def output(self, ws: Sequence[int]):
        self._bits(*ws)
        self.outputs.extend(ws)

    def output_blocks(self, ws: Sequence[int]):
        """Outputs that are message blocks: wires holding values up to
        MAX_BLOCK_VALUE (a LUT wire packing two bits, or a bit).  A block
        input passed straight through is refreshed by a PBS on a circuit-local
        identity table (the parity refresh of bit inputs would keep x mod 2)."""
        for w in ws:
            if self.vmax[w] > MAX_BLOCK_VALUE:
                raise ValueError(f"{self.name}: wire {w} holds values up to {self.vmax[w]}, more than a "
                                 f"block's {MAX_BLOCK_VALUE}")
        ident = tuple(x if x <= MAX_BLOCK_VALUE else 0 for x in range(TOTAL_MOD))
        for w in ws:
            if self.gates[w][0] == "in" and self.vmax[w] > 1:
                lut = (NUM_FIXED_LUTS + self.extra_luts.index(ident) if ident in self.extra_luts
                       else self.add_lut(ident))
                w = self.lut([(w, 1)], 0, lut)
            self.outputs.append(w)

    def evaluate(self, shared_bits, instance_bits, iconst_bits) -> List[int]:
        """Direct evaluation of one instance (the reference semantics)."""
        luts = self.lut_tables()
        val: List[int] = []
        for g in self.gates:
            op = g[0]
            if op == "in":
                v = int(shared_bits[g[2]] if g[1] else instance_bits[g[2]])
            elif op == "const":
                v = g[1]
            elif op == "iconst":
                v = int(iconst_bits[g[1]])
            elif op == "xor":
                v = val[g[1]] ^ val[g[2]]
            elif op == "not":
                v = val[g[1]] ^ 1
            elif op == "and":
                v = val[g[1]] & val[g[2]]
            elif op == "lut":
                x = g[2] + sum(c * val[w] for w, c in g[1])
                assert 0 <= x <= MAX_VALUE, (g, x)
                v = luts[g[3]][x]
            else:  # mat
                v = val[g[1]]
            val.append(v)
        return [val[w] for w in self.outputs]


# ---------------------------------------------------------------------------
# compiled schedule
# ---------------------------------------------------------------------------
@dataclass
class Row:
    terms: List[Tuple[int, int]]          # (atom, coef)
    body: int                             # shared body constant (message units)
    iterms: List[Tuple[int, int]]         # (iconst index, coef): per-instance body part
    lut: int
    out: int                              # atom made by this row
    layer: int
    shared: bool


@dataclass
class Schedule:
    """Tables of a compiled circuit, laid out for `num_instances` instances.
    Only the addressing depends on the instance count: `for_instances` gives
    the same tables for another count without compiling again.

    Slots: shared slots [0, num_shared_slots) hold one LWE each; per-instance
    slot s >= num_shared_slots holds `num_instances` LWEs at pool rows
    num_shared_slots + (s - num_shared_slots) * num_instances + instance.
    Layer L has logical rows layer_rows[L] .. layer_rows[L+1], the first
    layer_shared_rows[L] of them shared (one output each), the others one
    output per instance.  Row r reads terms row_offsets[r] .. row_offsets[r+1]
    (term_slots, term_coefs) and adds the body constant
    body_base[r] + sum(coef * iconst[instance][idx]) over its iterms."""
    circuit_name: str
    num_instances: int
    num_shared_slots: int
    num_instance_slots: int
    layer_rows: np.ndarray        # u32 [L + 1]
    layer_shared_rows: np.ndarray  # u32 [L]
    row_offsets: np.ndarray       # u32 [R + 1]
    term_slots: np.ndarray        # u32 [T]
    term_coefs: np.ndarray        # i64 [T]
    body_base: np.ndarray         # i64 [R]
    iterm_rows: np.ndarray        # i64 [Ti]: row of each per-instance body term
    iterm_index: np.ndarray       # i64 [Ti]: iconst index
    iterm_coefs: np.ndarray       # i64 [Ti]
    row_lut: np.ndarray           # u32 [R]
    row_dest: np.ndarray          # u32 [R]: destination slot
    frees: List[np.ndarray]       # slots whose last reader is layer L (poisoned after it)
    shared_input_slots: np.ndarray
    instance_input_slots: np.ndarray
    output_slots: np.ndarray
    num_iconsts: int
    pbs_per_instance_rows: int = 0
    pbs_shared_rows: int = 0
    extra_luts: Tuple[Tuple[int, ...], ...] = ()   # the circuit's own tables, after lut_functions()

    def lut_tables(self) -> List[List[int]]:
        """the f tables of the LUT indexes in row_lut"""
        return lut_functions() + [list(t) for t in self.extra_luts]

    @property
    def num_layers(self) -> int:
        return len(self.layer_shared_rows)

    @property
    def peak_slots(self) -> int:
        return self.num_shared_slots + self.num_instance_slots

    @property
    def pool_rows(self) -> int:
        return self.num_shared_slots + self.num_instance_slots * self.num_instances

    def for_instances(self, num_instances: int) -> "Schedule":
        return dataclasses.replace(self, num_instances=num_instances)

    def pbs_count(self) -> int:
        """PBS of one call: shared rows once, the others once per instance."""
        return self.pbs_shared_rows + self.pbs_per_instance_rows * self.num_instances

    def layer_outputs(self, L: int) -> int:
        rows = int(self.layer_rows[L + 1] - self.layer_rows[L])
        sh = int(self.layer_shared_rows[L])
        return sh + (rows - sh) * self.num_instances

    def addr(self, slots: np.ndarray, inst) -> np.ndarray:
        """pool row of `slots` for instance(s) `inst` (broadcasting)"""
        slots = np.asarray(slots, dtype=np.int64)
        S, I = self.num_shared_slots, self.num_instances
        return np.where(slots < S, slots, S + (slots - S) * I + np.asarray(inst, dtype=np.int64))

    def body(self, iconst_bits: Optional[np.ndarray]) -> np.ndarray:
        """body constants [R, num_instances] in message units (int64)"""
        R = len(self.body_base)
        out = np.repeat(self.body_base[:, None], self.num_instances, axis=1)
        if len(self.iterm_rows):
            bits = np.asarray(iconst_bits, dtype=np.int64).reshape(self.num_instances, self.num_iconsts)
            np.add.at(out, self.iterm_rows, self.iterm_coefs[:, None] * bits[:, self.iterm_index].T)
        assert out.shape == (R, self.num_instances)
        return out

    def output_rows(self) -> np.ndarray:
        """pool rows of the outputs, instance-major: [num_instances * outputs]"""
        inst = np.arange(self.num_instances)[:, None]
        return self.addr(self.output_slots[None, :], inst).reshape(-1)

    def gpu_tables(self):
        """Per-output-row LUT and destination pool row of every layer, in the
        order the linear kernel writes its outputs (shared rows, then the
        per-instance rows instance-minor)."""
        luts, dests = [], []
        I = self.num_instances
        for L in range(self.num_layers):
            r0, r1 = int(self.layer_rows[L]), int(self.layer_rows[L + 1])
            sh = int(self.layer_shared_rows[L])
            luts.append(self.row_lut[r0:r0 + sh])
            dests.append(self.row_dest[r0:r0 + sh])
            luts.append(np.repeat(self.row_lut[r0 + sh:r1], I))
            dests.append(self.addr(np.repeat(self.row_dest[r0 + sh:r1], I), np.tile(np.arange(I), r1 - r0 - sh)))
        return (np.concatenate(luts).astype(np.uint64) if luts else np.zeros(0, np.uint64),
                np.concatenate(dests).astype(np.uint64) if dests else np.zeros(0, np.uint64))


@dataclass
class _Atom:
    ready: int
    vmax: int
    shared: bool


class _Form:
    """Parity of a set of atoms, a shared constant bit and per-instance bits."""
    __slots__ = ("atoms", "c", "k")

    def __init__(self, atoms=frozenset(), c=0, k=frozenset()):
        self.atoms, self.c, self.k = frozenset(atoms), c, frozenset(k)

    def __xor__(self, o):
        return _Form(self.atoms ^ o.atoms, self.c ^ o.c, self.k ^ o.k)


class _Compiler:
    def __init__(self, circuit: Circuit):
        self.circ = circuit
        self.atoms: List[_Atom] = []
        self.rows: List[Row] = []
        self.memo: Dict[tuple, int] = {}
        self.input_atoms: Dict[Tuple[bool, int], int] = {}

    def new_atom(self, ready, vmax, shared) -> int:
        self.atoms.append(_Atom(ready, vmax, shared))
        return len(self.atoms) - 1

    def emit(self, terms, body, iterms, lut) -> int:
        """one PBS row; returns its atom (memoized on the whole row)"""
        terms = sorted(terms)
        iterms = sorted(iterms)
        key = (tuple(terms), body, tuple(iterms), lut)
        if key in self.memo:
            return self.memo[key]
        noise = sum(abs(c) for _, c in terms)
        lo = body + sum(min(0, c) * self.atoms[a].vmax for a, c in terms) + sum(min(0, c) for _, c in iterms)
        hi = body + sum(max(0, c) * self.atoms[a].vmax for a, c in terms) + sum(max(0, c) for _, c in iterms)
        assert noise <= MAX_NOISE_LEVEL and 0 <= lo and hi <= MAX_VALUE, (terms, body, iterms, lut)
        layer = 1 + max([self.atoms[a].ready for a, _ in terms], default=0)
        shared = all(self.atoms[a].shared for a, _ in terms) and not iterms
        out = self.new_atom(layer, self.circ.lut_vmax(lut), shared)
        self.rows.append(Row(terms, body, iterms, lut, out, layer, shared))
        self.memo[key] = out
        return out

    # -- parity reductions -------------------------------------------------
    def _plan(self, atoms, t):
        """earliest-first merging of `atoms` down to <= t: (ready times, merges)"""
        ready = sorted(self.atoms[a].ready for a in atoms)
        merges = 0
        while len(ready) > t:
            k = min(MAX_TERMS, len(ready) - t + 1)
            grp, ready = ready[:k], ready[k:]
            ready.append(max(grp) + 1)
            ready.sort()
            merges += 1
        return (max(ready, default=0), merges)

    def reduce(self, atoms, t) -> frozenset:
        atoms = sorted(atoms, key=lambda a: (self.atoms[a].ready, a))
        while len(atoms) > t:
            k = min(MAX_TERMS, len(atoms) - t + 1)
            grp, atoms = atoms[:k], atoms[k:]
            atoms.append(self.emit([(a, 1) for a in grp], 0, [], LUT_PARITY))
            atoms.sort(key=lambda a: (self.atoms[a].ready, a))
        return frozenset(atoms)

    def materialize(self, f: _Form) -> int:
        """the form as one stored atom"""
        if len(f.atoms) == 1 and f.c == 0 and not f.k:
            return next(iter(f.atoms))
        atoms = self.reduce(f.atoms, MAX_TERMS)
        return self.emit([(a, 1) for a in atoms], f.c, [(k, 1) for k in f.k], LUT_PARITY)

    def and_gate(self, fa: _Form, fb: _Form) -> _Form:
        if fa.k:
            fa = _Form({self.materialize(fa)})
        if fb.k:
            fb = _Form({self.materialize(fb)})
        for x, y in ((fa, fb), (fb, fa)):
            if not y.atoms:  # constant operand
                return x if y.c else _Form()
        best = None
        # (high operand, low operand, atoms allowed in each): w = |low| + 1
        for hi, lo in ((fa, fb), (fb, fa)):
            for th, tl in ((1, 1), (2, 1), (1, 2)):
                rh, mh = self._plan(hi.atoms, th)
                rl, ml = self._plan(lo.atoms, tl)
                cost = (max(rh, rl), mh + ml, th + tl)
                if best is None or cost < best[0]:
                    best = (cost, hi, lo, th, tl)
        _, hi, lo, th, tl = best
        ah, al = self.reduce(hi.atoms, th), self.reduce(lo.atoms, tl)
        w = len(al) + 1
        terms = [(a, w) for a in ah] + [(a, 1) for a in al]
        return _Form({self.emit(terms, 0, [], lut_and(w, hi.c, lo.c))})

    def lut_gate(self, forms_terms, c0, lut) -> _Form:
        terms, iterms, body = [], [], c0
        for f, coef in forms_terms:
            if not f.atoms and not f.k:
                body += coef * f.c
            elif not f.atoms and len(f.k) == 1 and f.c == 0:
                iterms.append((next(iter(f.k)), coef))
            else:
                if len(f.atoms) != 1 or f.k:
                    f = _Form({self.materialize(f)})
                a = next(iter(f.atoms))
                if f.c:  # value of NOT a = 1 - a
                    terms.append((a, -coef))
                    body += coef
                else:
                    terms.append((a, coef))
        return _Form({self.emit(terms, body, iterms, lut)})

    def run(self):
        forms: List[_Form] = []
        for gi, g in enumerate(self.circ.gates):
            op = g[0]
            if op == "in":
                a = self.new_atom(0, self.circ.vmax[gi], g[1])   # 1, or MAX_BLOCK_VALUE for a block input
                self.input_atoms[(g[1], g[2])] = a
                f = _Form({a})
            elif op == "const":
                f = _Form(c=g[1])
            elif op == "iconst":
                f = _Form(k={g[1]})
            elif op == "xor":
                f = forms[g[1]] ^ forms[g[2]]
            elif op == "not":
                f = forms[g[1]] ^ _Form(c=1)
            elif op == "and":
                f = self.and_gate(forms[g[1]], forms[g[2]])
            elif op == "lut":
                f = self.lut_gate([(forms[w], c) for w, c in g[1]], g[2], g[3])
            else:  # mat
                f = _Form({self.materialize(forms[g[1]])})
            forms.append(f)
        # every output is a PBS output of its own
        outs = []
        inputs = set(self.input_atoms.values())
        for w in self.circ.outputs:
            f = forms[w]
            if len(f.atoms) == 1 and f.c == 0 and not f.k:
                a = next(iter(f.atoms))
                if a in inputs and self.atoms[a].vmax > 1:
                    # `output_blocks` refreshes block inputs itself; parity would keep x mod 2
                    raise ValueError(f"{self.circ.name}: a block input is output without a refresh")
                # a client bit passed through is refreshed by a PBS of its own
                outs.append(self.emit([(a, 1)], 0, [], LUT_PARITY) if a in inputs else a)
            else:
                outs.append(self.materialize(f))
        return outs


def compile_circuit(circuit: Circuit, num_instances: int = 1) -> Schedule:
    comp = _Compiler(circuit)
    outs = comp.run()
    rows = comp.rows
    atoms = comp.atoms
    num_layers = max([r.layer for r in rows], default=0)
    # last layer reading each atom; outputs live to the end
    last = {}
    for r in rows:
        for a, _ in r.terms:
            last[a] = max(last.get(a, 0), r.layer)
    for a in outs:
        last[a] = num_layers + 1
    by_layer: List[List[Row]] = [[] for _ in range(num_layers + 1)]
    for r in rows:
        by_layer[r.layer].append(r)
    # slot allocation: inputs first, then per layer, freeing after the last reader
    slot: Dict[int, int] = {}
    free = {True: [], False: []}
    count = {True: 0, False: 0}

    def alloc(shared):
        if free[shared]:
            return free[shared].pop()
        count[shared] += 1
        return count[shared] - 1

    for (shared, _), a in sorted(comp.input_atoms.items(), key=lambda kv: (not kv[0][0], kv[0][1])):
        slot[a] = alloc(shared)
    frees_by_layer: List[List[Tuple[bool, int]]] = [[] for _ in range(num_layers + 1)]
    for a in slot:
        if a not in last:  # an input no row reads
            frees_by_layer[0].append((atoms[a].shared, slot[a]))
    for L in range(1, num_layers + 1):
        dying = sorted({a for r in by_layer[L] for a, _ in r.terms if last[a] == L})
        for a in dying:
            frees_by_layer[L].append((atoms[a].shared, slot[a]))
            free[atoms[a].shared].append(slot[a])
        free[True].sort(reverse=True)
        free[False].sort(reverse=True)
        dead = []
        for r in sorted(by_layer[L], key=lambda r: (not r.shared, r.out)):
            slot[r.out] = alloc(r.shared)
            if r.out not in last:  # a gate nothing reads: its slot is free after the layer
                dead.append((r.shared, slot[r.out]))
        for sh, s in dead:  # not reused within the layer: no two rows write one slot
            free[sh].append(s)
    S = count[True]

    def gslot(a):  # global slot id: shared, then per-instance
        return slot[a] if atoms[a].shared else S + slot[a]

    ordered: List[Row] = []
    layer_rows, layer_shared = [0], []
    for L in range(1, num_layers + 1):
        rs = sorted(by_layer[L], key=lambda r: (not r.shared, r.out))
        ordered.extend(rs)
        layer_rows.append(len(ordered))
        layer_shared.append(sum(r.shared for r in rs))
    offs, tslots, tcoefs, ir, ii, ic = [0], [], [], [], [], []
    for i, r in enumerate(ordered):
        for a, c in r.terms:
            tslots.append(gslot(a))
            tcoefs.append(c)
        offs.append(len(tslots))
        for k, c in r.iterms:
            ir.append(i)
            ii.append(k)
            ic.append(c)
    frees = [np.array(sorted(s if sh else S + s for sh, s in frees_by_layer[L]), dtype=np.int64)
             for L in range(num_layers + 1)]
    return Schedule(
        circuit_name=circuit.name, num_instances=num_instances, num_shared_slots=S,
        num_instance_slots=count[False],
        layer_rows=np.array(layer_rows, dtype=np.uint32), layer_shared_rows=np.array(layer_shared, dtype=np.uint32),
        row_offsets=np.array(offs, dtype=np.uint32), term_slots=np.array(tslots, dtype=np.uint32),
        term_coefs=np.array(tcoefs, dtype=np.int64), body_base=np.array([r.body for r in ordered], dtype=np.int64),
        iterm_rows=np.array(ir, dtype=np.int64), iterm_index=np.array(ii, dtype=np.int64),
        iterm_coefs=np.array(ic, dtype=np.int64), row_lut=np.array([r.lut for r in ordered], dtype=np.uint32),
        row_dest=np.array([gslot(r.out) for r in ordered], dtype=np.uint32), frees=frees,
        shared_input_slots=np.array([gslot(comp.input_atoms[(True, i)]) for i in range(circuit.num_shared_inputs)],
                                    dtype=np.int64),
        instance_input_slots=np.array([gslot(comp.input_atoms[(False, i)])
                                       for i in range(circuit.num_instance_inputs)], dtype=np.int64),
        output_slots=np.array([gslot(a) for a in outs], dtype=np.int64), num_iconsts=circuit.num_iconsts,
        pbs_per_instance_rows=sum(not r.shared for r in ordered), pbs_shared_rows=sum(r.shared for r in ordered),
        extra_luts=tuple(circuit.extra_luts))


# one compiled schedule per live circuit object, whatever the instance counts
_CACHE: "weakref.WeakKeyDictionary[Circuit, Schedule]" = weakref.WeakKeyDictionary()


def schedule(circuit: Circuit, num_instances: int) -> Schedule:
    """The circuit's schedule for `num_instances` instances; the circuit is
    compiled once (the compile does not depend on the instance count)."""
    base = _CACHE.get(circuit)
    if base is None:
        base = _CACHE[circuit] = compile_circuit(circuit)
    return base.for_instances(num_instances)


# ---------------------------------------------------------------------------
# cleartext executor
# ---------------------------------------------------------------------------
POISON = -(1 << 20)


def run_cleartext(sched: Schedule, shared_bits, instance_bits=None, iconst_bits=None) -> np.ndarray:
    """Run the schedule on plaintext values, tracking each slot's noise level;
    asserts the budget rule on every row and poisons freed slots.  Returns the
    outputs [num_instances, outputs]."""
    I = sched.num_instances
    val = np.full(sched.pool_rows, POISON, dtype=np.int64)
    lvl = np.full(sched.pool_rows, 1 << 20, dtype=np.int64)
    val[sched.addr(sched.shared_input_slots, 0)] = np.asarray(shared_bits, dtype=np.int64).reshape(-1)
    if len(sched.instance_input_slots):
        inst = np.asarray(instance_bits, dtype=np.int64).reshape(I, -1)
        rows = sched.addr(sched.instance_input_slots[None, :], np.arange(I)[:, None])
        val[rows] = inst
    written = np.concatenate([sched.addr(sched.shared_input_slots, 0),
                              sched.addr(sched.instance_input_slots[None, :], np.arange(I)[:, None]).reshape(-1)])
    lvl[written] = 1
    body = sched.body(iconst_bits) if sched.num_iconsts else np.repeat(sched.body_base[:, None], I, axis=1)
    luts = np.array(sched.lut_tables(), dtype=np.int64)

    def poison(slots):
        if len(slots):
            rows = sched.addr(slots[None, :], np.arange(I)[:, None]).reshape(-1)
            val[rows] = POISON
            lvl[rows] = 1 << 20

    poison(sched.frees[0])
    for L in range(sched.num_layers):
        r0, r1 = int(sched.layer_rows[L]), int(sched.layer_rows[L + 1])
        results = []
        for r in range(r0, r1):
            t0, t1 = int(sched.row_offsets[r]), int(sched.row_offsets[r + 1])
            slots, coefs = sched.term_slots[t0:t1].astype(np.int64), sched.term_coefs[t0:t1]
            insts = np.arange(I) if r - r0 >= int(sched.layer_shared_rows[L]) else np.zeros(1, dtype=np.int64)
            addrs = sched.addr(slots[None, :], insts[:, None])           # [instances, terms]
            x = (val[addrs] * coefs[None, :]).sum(1) + body[r, insts]
            noise = (lvl[addrs] * np.abs(coefs)[None, :]).sum(1)
            assert np.all(noise <= MAX_NOISE_LEVEL), (sched.circuit_name, L, r, noise)
            assert np.all((x >= 0) & (x <= MAX_VALUE)), (sched.circuit_name, L, r, x)
            results.append((sched.addr(int(sched.row_dest[r]), insts), luts[sched.row_lut[r], x]))
        poison(sched.frees[L + 1])
        for rows, v in results:
            val[rows] = v
            lvl[rows] = 1
    out = val[sched.output_rows()].reshape(I, -1)
    assert np.all(out >= 0), "an output slot was freed before the end"
    return out
