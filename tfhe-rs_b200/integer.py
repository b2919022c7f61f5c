"""Radix-integer multiplication on top of the batched KS -> PBS entry points
(FheUint64 x FheUint64, 32 blocks of 2+2 bits).

Host-side orchestration only: every ciphertext operation that is not a plain
wrapping add is a keyswitch + programmable bootstrap issued through the C ABI
with per-sample LUT indexes, exactly what the reference's integer layer does
with `execute_keyswitch_async` + `execute_pbs_async`
(backends/tfhe-cuda-backend/cuda/src/integer/integer.cuh:869-1000).

The algorithm restates the reference's CPU `unchecked_mul_parallelized`:
  * terms: for every block i of rhs, lhs shifted by i blocks with the bivariate
    LUT (x*y) % 4, and shifted by i+1 blocks with (x*y) / 4
    (tfhe/src/integer/server_key/radix_parallel/mul.rs:333-398; bivariate
    packing lhs*4 + rhs, shortint/server_key/bivariate_pbs.rs);
  * column-wise partial sums in chunks of 5 blocks (15 / 3), message and carry
    extraction, until every column holds at most 5 blocks
    (radix_parallel/sum.rs:14-160);
  * full carry propagation (sequential variant of full_propagate_parallelized).

The arithmetic on encrypted blocks is engine-agnostic (`BlockEngine`): the GPU
engine keeps blocks in device memory (torch int64 tensors: wrapping adds are
plumbing) and sends every LUT evaluation to libtfhe_cuda_backend_b200.so; the
tests additionally run the same host logic over a CPU engine backed by the
oracle (tests/ only).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

MSG_MOD = 4      # message modulus of PARAM_MESSAGE_2_CARRY_2
TOTAL_MOD = 16   # message * carry modulus
CHUNK = (TOTAL_MOD - 1) // (MSG_MOD - 1)  # = 5, ServerKey::max_sum_size(Degree(3))

LUT_MUL_LSB, LUT_MUL_MSB, LUT_MSG, LUT_CARRY = 0, 1, 2, 3
LUT_STATE, LUT_COMBINE, LUT_CARRY_BIT = 4, 5, 6
ST_NONE, ST_PROPAGATE, ST_GENERATE = 0, 1, 2


def lut_functions() -> List[List[int]]:
    """f tables over the 4-bit padded message space, in LUT index order."""
    lsb = [((x // MSG_MOD) * (x % MSG_MOD)) % MSG_MOD for x in range(TOTAL_MOD)]
    msb = [((x // MSG_MOD) * (x % MSG_MOD)) // MSG_MOD for x in range(TOTAL_MOD)]
    msg = [x % MSG_MOD for x in range(TOTAL_MOD)]
    carry = [x // MSG_MOD for x in range(TOTAL_MOD)]
    # carry-propagation states of a block value (message + incoming carry <= 7)
    state = [ST_GENERATE if x >= MSG_MOD else (ST_PROPAGATE if x == MSG_MOD - 1 else ST_NONE)
             for x in range(TOTAL_MOD)]
    # prefix operator on packed (cur * 4 + prev): a propagating block inherits the previous state
    combine = [((x % MSG_MOD) if (x // MSG_MOD) == ST_PROPAGATE else min(x // MSG_MOD, ST_GENERATE))
               for x in range(TOTAL_MOD)]
    carry_bit = [1 if x == ST_GENERATE else 0 for x in range(TOTAL_MOD)]
    return [lsb, msb, msg, carry, state, combine, carry_bit]


class BlockEngine:
    """What the radix algorithms need from a backend.  Blocks are rows of an
    array-like `[count, big_lwe_dimension + 1]` with wrapping u64 arithmetic."""

    def zeros(self, count: int):
        raise NotImplementedError

    def stack(self, rows: Sequence):
        raise NotImplementedError

    def add(self, a, b):
        raise NotImplementedError

    def scalar_mul(self, a, s: int):
        raise NotImplementedError

    def apply_luts(self, blocks, lut_ids: Sequence[int]):
        """KS -> PBS of every row of `blocks` with LUT `lut_ids[row]`."""
        raise NotImplementedError

    # batched plumbing (defaults work for numpy arrays and torch tensors alike)
    def take(self, blocks, idx: Sequence[int]):
        """rows `idx` of `blocks` as a new array"""
        return blocks[list(idx)]

    def cat(self, parts: Sequence):
        return self.stack([row for part in parts for row in part])

    def sum_groups(self, blocks, group: int):
        """wrapping sum of every `group` consecutive rows"""
        return blocks.reshape(blocks.shape[0] // group, group, blocks.shape[1]).sum(1)


def _bivariate_pack(engine: BlockEngine, lhs_rows, rhs_rows):
    """lhs * 4 + rhs (unchecked_apply_lookup_table_bivariate's linear part)."""
    return engine.add(engine.scalar_mul(lhs_rows, MSG_MOD), rhs_rows)


def compute_terms_for_mul_low(engine: BlockEngine, lhs, rhs, num_blocks: int):
    """All partial-product blocks in ONE batched LUT evaluation.  Returns
    `columns`: list (per output block) of lists of row handles."""
    lhs_idx, rhs_idx, lut_ids, col = [], [], [], []
    for i in range(num_blocks):          # rhs block
        for j in range(num_blocks - i):  # lhs block, result column i + j
            lhs_idx.append(j)
            rhs_idx.append(i)
            lut_ids.append(LUT_MUL_LSB)
            col.append(i + j)
            if i + j + 1 < num_blocks:   # carry part lands one block higher
                lhs_idx.append(j)
                rhs_idx.append(i)
                lut_ids.append(LUT_MUL_MSB)
                col.append(i + j + 1)
    packed = _bivariate_pack(engine, lhs[lhs_idx], rhs[rhs_idx])
    out = engine.apply_luts(packed, lut_ids)
    columns = [[] for _ in range(num_blocks)]
    for r, c in enumerate(col):
        columns[c].append(out[r])
    return columns


def partial_sum_columns(engine: BlockEngine, columns):
    """radix_parallel/sum.rs:14-160 on column lists; every round is one batched
    LUT evaluation (message + carry extraction of every full chunk).  The chunk
    sums of a round are ONE stacked gather + grouped sum, not one add per row."""
    n = len(columns)
    while any(len(c) > CHUNK for c in columns):
        flat, meta = [], []
        new_cols = [[] for _ in range(n)]
        for ci, colm in enumerate(columns):
            if len(colm) < CHUNK:
                new_cols[ci].extend(colm)
                continue
            full = (len(colm) // CHUNK) * CHUNK
            flat.extend(colm[:full])
            meta.extend([ci] * (full // CHUNK))
            new_cols[ci].extend(colm[full:])
        sums = engine.sum_groups(engine.stack(flat), CHUNK)
        pick, ids, dest = [], [], []
        for r, ci in enumerate(meta):
            pick.append(r)
            ids.append(LUT_MSG)
            dest.append(ci)
            if ci + 1 < n:
                pick.append(r)
                ids.append(LUT_CARRY)
                dest.append(ci + 1)
        out = engine.apply_luts(engine.take(sums, pick), ids)
        for r, d in enumerate(dest):
            new_cols[d].append(out[r])
        columns = new_cols
    # final column sums: pad every column to the longest with zero blocks
    width = max(1, max(len(c) for c in columns))
    zero = engine.zeros(1)[0]
    flat = [row for colm in columns for row in (list(colm) + [zero] * (width - len(colm)))]
    return engine.sum_groups(engine.stack(flat), width)


def _split_and_shift_carries(engine: BlockEngine, blocks, n: int):
    """Blocks may hold any value <= 15: extract message and carry of every
    block in one batched round and add each carry one block up (value <= 6).
    Returns the stacked [n, L] result."""
    out = engine.apply_luts(engine.take(blocks, [i for i in range(n) for _ in (0, 1)]), [LUT_MSG, LUT_CARRY] * n)
    msgs = engine.take(out, list(range(0, 2 * n, 2)))
    if n == 1:
        return msgs
    carries = engine.take(out, list(range(1, 2 * (n - 1), 2)))
    return engine.add(msgs, engine.cat([engine.zeros(1), carries]))


def full_propagate(engine: BlockEngine, blocks, num_blocks: int):
    """Sequential carry ripple (one LUT round per block) after the parallel
    message/carry split; kept as the simple cross-check of the parallel scan."""
    vals = _split_and_shift_carries(engine, blocks, num_blocks)
    out = []
    cur = vals[0]
    for i in range(num_blocks):
        if i + 1 < num_blocks:
            res = engine.apply_luts(engine.stack([cur, cur]), [LUT_MSG, LUT_CARRY])
            out.append(res[0])
            cur = engine.add(vals[i + 1], res[1])
        else:
            res = engine.apply_luts(engine.stack([cur]), [LUT_MSG])
            out.append(res[0])
    return engine.stack(out)


def full_propagate_parallel(engine: BlockEngine, blocks, num_blocks: int):
    """Carry propagation in 4 + ceil(log2(blocks)) batched LUT rounds instead of
    `blocks` sequential ones (role of the reference's parallel
    `propagate_single_carry_parallelized`, integer/server_key/radix_parallel/
    add.rs): split every block into message and carry, add the carry one block
    up (value <= 6), classify blocks as generate / propagate / none, run a
    Hillis-Steele prefix scan with the bivariate operator, turn the incoming
    state into a carry bit, add it and extract the message."""
    n = num_blocks
    vals = _split_and_shift_carries(engine, blocks, n)
    states = engine.apply_luts(vals, [LUT_STATE] * n)
    d = 1
    while d < n:
        idx = list(range(d, n))
        packed = engine.add(engine.scalar_mul(engine.take(states, idx), MSG_MOD),
                            engine.take(states, [i - d for i in idx]))
        comb = engine.apply_luts(packed, [LUT_COMBINE] * len(idx))
        states = engine.cat([states[:d], comb])
        d *= 2
    if n == 1:
        return engine.apply_luts(vals, [LUT_MSG])
    # carry into block i = [inclusive prefix state of blocks 0..i-1 == generate]
    bits = engine.apply_luts(states[: n - 1], [LUT_CARRY_BIT] * (n - 1))
    finals = engine.add(vals, engine.cat([engine.zeros(1), bits]))
    return engine.apply_luts(finals, [LUT_MSG] * n)


def unchecked_mul(engine: BlockEngine, lhs, rhs, parallel_carry: bool = True):
    """radix_parallel/mul.rs:437-470 (clean inputs: carries empty)."""
    num_blocks = lhs.shape[0]
    assert rhs.shape[0] == num_blocks
    columns = compute_terms_for_mul_low(engine, lhs, rhs, num_blocks)
    summed = partial_sum_columns(engine, columns)
    if parallel_carry:
        return full_propagate_parallel(engine, summed, num_blocks)
    return full_propagate(engine, summed, num_blocks)


# ---------------------------------------------------------------------------
# GPU engine
# ---------------------------------------------------------------------------
class CudaBlockEngine(BlockEngine):
    """Blocks live on the GPU as an int64 tensor [count, kN + 1]; LUT
    evaluations go through CudaServerKey.apply_lookup_table (C ABI)."""

    def __init__(self, server_key, lut_glwe_list_np: np.ndarray, glwe_dimension: int, polynomial_size: int):
        import torch

        from . import gpu

        self.torch, self.gpu = torch, gpu
        self.skey = server_key
        self.streams = server_key.streams
        self.luts = gpu.CudaGlweCiphertextList.from_glwe_ciphertext_list(
            lut_glwe_list_np, glwe_dimension, polynomial_size, self.streams)
        self.big = server_key.big_dim
        self.pbs_count = 0

    def from_numpy(self, a: np.ndarray):
        t = self.torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64))
        with self.torch.cuda.stream(self.streams.streams[0]):
            return t.to(self.streams.device(0))

    def to_numpy(self, t) -> np.ndarray:
        self.streams.synchronize()
        return t.cpu().numpy().view(np.uint64)

    def zeros(self, count):
        with self.torch.cuda.stream(self.streams.streams[0]):
            return self.torch.zeros((count, self.big + 1), dtype=self.torch.int64, device=self.streams.device(0))

    def stack(self, rows):
        with self.torch.cuda.stream(self.streams.streams[0]):
            return self.torch.stack(list(rows))

    def add(self, a, b):
        with self.torch.cuda.stream(self.streams.streams[0]):
            return a + b  # int64 add wraps mod 2^64

    def scalar_mul(self, a, s):
        with self.torch.cuda.stream(self.streams.streams[0]):
            return a * int(s)

    def take(self, blocks, idx):
        with self.torch.cuda.stream(self.streams.streams[0]):
            index = self.torch.tensor(list(idx), dtype=self.torch.int64).to(self.streams.device(0), non_blocking=True)
            return blocks.index_select(0, index)

    def cat(self, parts):
        with self.torch.cuda.stream(self.streams.streams[0]):
            return self.torch.cat(list(parts), dim=0)

    def sum_groups(self, blocks, group):
        with self.torch.cuda.stream(self.streams.streams[0]):
            return blocks.view(blocks.shape[0] // group, group, blocks.shape[1]).sum(1)

    def apply_luts(self, blocks, lut_ids):
        gpu = self.gpu
        count = blocks.shape[0]
        with self.torch.cuda.stream(self.streams.streams[0]):
            flat = blocks.contiguous().view(-1)
            ids = self.torch.tensor(list(lut_ids), dtype=self.torch.int64).to(self.streams.device(0))
        cts = gpu.CudaLweCiphertextList(gpu.CudaVec(flat, np.uint64), self.big, count)
        out = self.skey.apply_lookup_table(cts, self.luts, gpu.CudaVec(ids, np.uint64))
        self.pbs_count += count
        return out.d_vec.t.view(count, self.big + 1)


class CudaUnsignedRadixCiphertext:
    """integer/gpu/ciphertext: a vector of shortint blocks on one GPU, least
    significant first.  It may hold `num_inputs` integers of `num_blocks`
    blocks each, instance-major: `blocks` is [num_inputs * num_blocks,
    big + 1]; the radix operations run them as instances of one schedule."""
    signed = False

    def __init__(self, blocks, num_inputs: int = 1):
        self.blocks = blocks
        self.num_inputs = num_inputs

    @property
    def num_blocks(self):
        return self.blocks.shape[0] // self.num_inputs


class CudaSignedRadixCiphertext(CudaUnsignedRadixCiphertext):
    """A two's-complement radix integer: the sign is bit 1 of the top block."""
    signed = True


class CudaBooleanBlock:
    """One block holding 0 or 1 per input: `blocks` is [num_inputs, big + 1]."""

    def __init__(self, blocks, num_inputs: int = 1):
        self.blocks = blocks
        self.num_inputs = num_inputs


class CudaRadixServerKey:
    """Mirror of integer::gpu::CudaServerKey: the multiplication path
    (integer/gpu/server_key/radix/mul.rs:167), and comparisons, selects,
    additions, subtractions, bitwise operations, their clear-operand forms,
    signed overflow flags, abs, erc7984's transfer (`radix`), products and
    sums (`radix_mul`), divisions (`radix_div`), shifts, rotations and bit counts (`radix_bits`), vector find
    and the key-value store's encrypted-key operations (`radix_find`), and the oblivious bitonic shuffle
    of a list of integers by OPRF sort keys (`radix_shuffle`), compiled to KS -> PBS
    layers and run by a bit-circuit runner of its own (created on first use) with `b200_bit_circuit_64_async`.

    Those operations take ciphertexts of one kind (unsigned or signed), one
    block count and one `num_inputs`, on 2_2 keys, and raise ValueError before
    any GPU work otherwise.  The work runs on the server key's first stream
    after the caller's current stream; inputs may be dropped as soon as a
    call returns, and the caller's stream waits for the result (see
    `bit_circuit_gpu`)."""

    _runner = None

    def __init__(self, server_key, lut_glwe_list_np=None, glwe_dimension=1, polynomial_size=2048):
        if lut_glwe_list_np is None:  # the 7 accumulators of lut_functions(), 2+2-bit blocks, one padding bit
            from . import algorithms

            delta = (1 << 63) // TOTAL_MOD
            lut_glwe_list_np = np.stack([
                algorithms.generate_programmable_bootstrap_glwe_lut(polynomial_size, glwe_dimension + 1, TOTAL_MOD,
                                                                    delta, f) for f in lut_functions()])
        self.engine = CudaBlockEngine(server_key, lut_glwe_list_np, glwe_dimension, polynomial_size)

    def unchecked_mul(self, lhs: CudaUnsignedRadixCiphertext, rhs: CudaUnsignedRadixCiphertext):
        return CudaUnsignedRadixCiphertext(unchecked_mul(self.engine, lhs.blocks, rhs.blocks))

    # -- compiled radix circuits ------------------------------------------------
    @property
    def runner(self):
        """The bit-circuit runner of the radix circuits, created on first use
        (its device tables are its own: AES or Trivium runners keep theirs)."""
        if self._runner is None:
            skey = self.engine.skey
            moduli = (getattr(skey, "message_modulus", None), getattr(skey, "carry_modulus", None))
            if moduli != (MSG_MOD, TOTAL_MOD // MSG_MOD):
                raise ValueError(f"radix circuits need a 2_2 server key, got message / carry moduli {moduli}")
            from . import bit_circuit_gpu

            self._runner = bit_circuit_gpu.CudaBitCircuitRunner(skey)
        return self._runner

    @staticmethod
    def _operands(*cts):
        """(ciphertext type, num_blocks, num_inputs) shared by all operands"""
        from . import radix

        first = cts[0]
        for ct in cts:
            if not isinstance(ct, CudaUnsignedRadixCiphertext):
                raise ValueError(f"expected a radix ciphertext, got {type(ct).__name__}")
            if type(ct) is not type(first):
                raise ValueError(f"operands differ in signedness: {type(first).__name__} and {type(ct).__name__}")
            I = ct.num_inputs
            if isinstance(I, bool) or not isinstance(I, (int, np.integer)) or I < 1 or ct.blocks.shape[0] % I:
                raise ValueError(f"{ct.blocks.shape[0]} blocks do not hold num_inputs = {I!r} integers")
            if I != first.num_inputs:
                raise ValueError(f"operands differ in num_inputs: {first.num_inputs} and {I}")
            if ct.num_blocks != first.num_blocks:
                raise ValueError(f"operands differ in block count: {first.num_blocks} and {ct.num_blocks}")
        return type(first), radix.check_num_blocks(first.num_blocks), int(first.num_inputs)

    def _run(self, op, signed, n, I, blocks, iconsts=None):
        """the circuit of (op, n, signed) on the operands' blocks, concatenated
        per instance; returns the outputs [I, outputs, big + 1]"""
        from . import radix

        return self._run_circuit(radix.circuit(op, n, signed), I, blocks, iconsts)

    def _run_circuit(self, circuit, I, blocks, iconsts=None):
        """`circuit` on the operands' blocks, concatenated per instance;
        returns the outputs [I, outputs, big + 1]"""
        import torch

        W = blocks[0].shape[1]
        parts = [b.reshape(I, -1, W) for b in blocks]
        inst = parts[0] if len(parts) == 1 else torch.cat(parts, 1)
        return self.runner.run(circuit, None, inst.reshape(-1, W), iconsts, I).view(I, -1, W)

    @staticmethod
    def _radix(kind, out, I):
        return kind(out.reshape(-1, out.shape[-1]), I)

    def _binary(self, op, lhs, rhs):
        kind, n, I = self._operands(lhs, rhs)
        return kind, I, self._run(op, kind.signed, n, I, [lhs.blocks, rhs.blocks])

    def _compare(self, op, lhs, rhs) -> CudaBooleanBlock:
        _, I, out = self._binary(op, lhs, rhs)
        return CudaBooleanBlock(out[:, 0], I)

    def _scalar_iconsts(self, ct, scalar):
        """(kind, n, I, iconsts) of a clear operand: `scalar` is one clear
        integer for every input, or one per input"""
        from . import radix

        kind, n, I = self._operands(ct)
        scalars = [scalar] * I if np.ndim(scalar) == 0 else list(scalar)
        if len(scalars) != I:
            raise ValueError(f"expected one scalar or {I}, got {len(scalars)}")
        return kind, n, I, radix.scalar_iconsts(scalars, n, kind.signed)

    def _scalar_compare(self, op, lhs, scalar) -> CudaBooleanBlock:
        """`scalar` is one clear integer for every input, or one per input"""
        kind, n, I, iconsts = self._scalar_iconsts(lhs, scalar)
        return CudaBooleanBlock(self._run(f"scalar_{op}", kind.signed, n, I, [lhs.blocks], iconsts)[:, 0], I)

    def _scalar_arith(self, op, ct, scalar):
        """the blocks of op with a clear rhs, then its flag if it has one"""
        kind, n, I, iconsts = self._scalar_iconsts(ct, scalar)
        out = self._run(f"scalar_{op}", kind.signed, n, I, [ct.blocks], iconsts)
        if out.shape[1] == n:
            return self._radix(kind, out, I)
        return self._radix(kind, out[:, :n], I), CudaBooleanBlock(out[:, n], I)

    def eq(self, lhs, rhs):
        return self._compare("eq", lhs, rhs)

    def ne(self, lhs, rhs):
        return self._compare("ne", lhs, rhs)

    def gt(self, lhs, rhs):
        return self._compare("gt", lhs, rhs)

    def ge(self, lhs, rhs):
        return self._compare("ge", lhs, rhs)

    def lt(self, lhs, rhs):
        return self._compare("lt", lhs, rhs)

    def le(self, lhs, rhs):
        return self._compare("le", lhs, rhs)

    def scalar_eq(self, lhs, scalar):
        return self._scalar_compare("eq", lhs, scalar)

    def scalar_ne(self, lhs, scalar):
        return self._scalar_compare("ne", lhs, scalar)

    def scalar_gt(self, lhs, scalar):
        return self._scalar_compare("gt", lhs, scalar)

    def scalar_ge(self, lhs, scalar):
        return self._scalar_compare("ge", lhs, scalar)

    def scalar_lt(self, lhs, scalar):
        return self._scalar_compare("lt", lhs, scalar)

    def scalar_le(self, lhs, scalar):
        return self._scalar_compare("le", lhs, scalar)

    def min(self, lhs, rhs):
        kind, I, out = self._binary("min", lhs, rhs)
        return self._radix(kind, out, I)

    def max(self, lhs, rhs):
        kind, I, out = self._binary("max", lhs, rhs)
        return self._radix(kind, out, I)

    def if_then_else(self, condition: CudaBooleanBlock, true_ct, false_ct):
        """true_ct where the condition holds, else false_ct, per input"""
        kind, n, I = self._operands(true_ct, false_ct)
        if not isinstance(condition, CudaBooleanBlock) or condition.num_inputs != I \
                or condition.blocks.shape[0] != I:
            raise ValueError(f"the condition must be a CudaBooleanBlock of {I} input(s)")
        out = self._run("if_then_else", False, n, I, [condition.blocks, true_ct.blocks, false_ct.blocks])
        return self._radix(kind, out, I)

    def add(self, lhs, rhs):
        """lhs + rhs, wrapping mod 4^num_blocks"""
        kind, I, out = self._binary("add", lhs, rhs)
        return self._radix(kind, out, I)

    def sub(self, lhs, rhs):
        """lhs - rhs, wrapping mod 4^num_blocks"""
        kind, I, out = self._binary("sub", lhs, rhs)
        return self._radix(kind, out, I)

    def neg(self, ct):
        """-ct, wrapping mod 4^num_blocks"""
        kind, n, I = self._operands(ct)
        return self._radix(kind, self._run("neg", False, n, I, [ct.blocks]), I)

    def _overflowing(self, op, lhs, rhs):
        kind, n, I = self._operands(lhs, rhs)
        if kind.signed:
            raise ValueError(f"unsigned_{op} takes unsigned integers")
        out = self._run(op, False, n, I, [lhs.blocks, rhs.blocks])
        return self._radix(kind, out[:, :n], I), CudaBooleanBlock(out[:, n], I)

    def unsigned_overflowing_add(self, lhs, rhs):
        """(lhs + rhs wrapping, [lhs + rhs >= 4^num_blocks])"""
        return self._overflowing("overflowing_add", lhs, rhs)

    def unsigned_overflowing_sub(self, lhs, rhs):
        """(lhs - rhs wrapping, [lhs < rhs])"""
        return self._overflowing("overflowing_sub", lhs, rhs)

    def _signed_overflowing(self, op, lhs, rhs):
        kind, n, I = self._operands(lhs, rhs)
        if not kind.signed:
            raise ValueError(f"signed_{op} takes signed integers")
        out = self._run(f"signed_{op}", True, n, I, [lhs.blocks, rhs.blocks])
        return self._radix(kind, out[:, :n], I), CudaBooleanBlock(out[:, n], I)

    def signed_overflowing_add(self, lhs, rhs):
        """(lhs + rhs wrapping, [the exact lhs + rhs is outside [MIN, MAX]])
        for signed integers"""
        return self._signed_overflowing("overflowing_add", lhs, rhs)

    def signed_overflowing_sub(self, lhs, rhs):
        """(lhs - rhs wrapping, [the exact lhs - rhs is outside [MIN, MAX]])
        for signed integers"""
        return self._signed_overflowing("overflowing_sub", lhs, rhs)

    def scalar_add(self, ct, scalar):
        """ct + scalar, wrapping mod 4^num_blocks; `scalar` is one clear
        integer for every input, or one per input, in the integer's range
        (else ValueError)"""
        return self._scalar_arith("add", ct, scalar)

    def scalar_sub(self, ct, scalar):
        """ct - scalar, wrapping mod 4^num_blocks, `scalar` as in `scalar_add`"""
        return self._scalar_arith("sub", ct, scalar)

    def unsigned_overflowing_scalar_add(self, ct, scalar):
        """(ct + scalar wrapping, [ct + scalar >= 4^num_blocks]) for an
        unsigned ct, `scalar` as in `scalar_add`"""
        if not isinstance(ct, CudaUnsignedRadixCiphertext) or ct.signed:
            raise ValueError("unsigned_overflowing_scalar_add takes an unsigned integer")
        return self._scalar_arith("overflowing_add", ct, scalar)

    def signed_overflowing_scalar_add(self, ct, scalar):
        """(ct + scalar wrapping, [the exact sum is outside [MIN, MAX]]) for a
        signed ct, `scalar` as in `scalar_add`"""
        if not isinstance(ct, CudaSignedRadixCiphertext):
            raise ValueError("signed_overflowing_scalar_add takes a signed integer")
        return self._scalar_arith("signed_overflowing_add", ct, scalar)

    def signed_overflowing_scalar_sub(self, ct, scalar):
        """(ct - scalar wrapping, [the exact difference is outside [MIN,
        MAX]]) for a signed ct, `scalar` as in `scalar_add`"""
        if not isinstance(ct, CudaSignedRadixCiphertext):
            raise ValueError("signed_overflowing_scalar_sub takes a signed integer")
        return self._scalar_arith("signed_overflowing_sub", ct, scalar)

    def abs(self, ct):
        """|ct| wrapping (abs(MIN) is MIN) for a signed ct; an unsigned ct comes
        back as a copy (on the caller's current stream), with no bootstrap"""
        kind, n, I = self._operands(ct)
        if not kind.signed:
            return kind(ct.blocks.clone(), I)
        return self._radix(kind, self._run("abs", True, n, I, [ct.blocks]), I)

    def bitand(self, lhs, rhs):
        kind, I, out = self._binary("bitand", lhs, rhs)
        return self._radix(kind, out, I)

    def bitor(self, lhs, rhs):
        kind, I, out = self._binary("bitor", lhs, rhs)
        return self._radix(kind, out, I)

    def bitxor(self, lhs, rhs):
        kind, I, out = self._binary("bitxor", lhs, rhs)
        return self._radix(kind, out, I)

    def bitnot(self, ct):
        kind, n, I = self._operands(ct)
        return self._radix(kind, self._run("bitnot", False, n, I, [ct.blocks]), I)

    def scalar_bitand(self, ct, scalar):
        """ct & scalar on the two's-complement bits, `scalar` as in `scalar_add`"""
        return self._scalar_arith("bitand", ct, scalar)

    def scalar_bitor(self, ct, scalar):
        """ct | scalar on the two's-complement bits, `scalar` as in `scalar_add`"""
        return self._scalar_arith("bitor", ct, scalar)

    def scalar_bitxor(self, ct, scalar):
        """ct ^ scalar on the two's-complement bits, `scalar` as in `scalar_add`"""
        return self._scalar_arith("bitxor", ct, scalar)

    def transfer(self, from_amount, to_amount, amount):
        """erc7984's `transfer_whitepaper` on unsigned balances, in one
        circuit: sent = amount if from_amount >= amount else 0; returns
        (from_amount - sent, to_amount + sent)."""
        kind, n, I = self._operands(from_amount, to_amount, amount)
        if kind.signed:
            raise ValueError("transfer takes unsigned integers")
        out = self._run("transfer", False, n, I, [from_amount.blocks, to_amount.blocks, amount.blocks])
        return self._radix(kind, out[:, :n], I), self._radix(kind, out[:, n:], I)

    # -- products and sums (`radix_mul`) ---------------------------------------
    def mul(self, lhs, rhs):
        """lhs * rhs wrapping mod 4^num_blocks, per input (the low half of the
        product, the same bits for signed and unsigned integers)"""
        from . import radix_mul

        kind, n, I = self._operands(lhs, rhs)
        return self._radix(kind, self._run_circuit(radix_mul.circuit("mul", n), I, [lhs.blocks, rhs.blocks]), I)

    def scalar_mul(self, ct, scalar):
        """ct * scalar wrapping mod 4^num_blocks; `scalar` is one clear integer
        for every input, or one per input, in the integer's range (else
        ValueError)"""
        from . import radix_mul

        kind, n, I, iconsts = self._scalar_iconsts(ct, scalar)
        return self._radix(kind, self._run_circuit(radix_mul.circuit("scalar_mul", n), I, [ct.blocks], iconsts), I)

    def unsigned_overflowing_mul(self, lhs, rhs):
        """(lhs * rhs wrapping, [lhs * rhs >= 4^num_blocks]) for unsigned
        integers"""
        from . import radix_mul

        kind, n, I = self._operands(lhs, rhs)
        if kind.signed:
            raise ValueError("unsigned_overflowing_mul takes unsigned integers")
        out = self._run_circuit(radix_mul.circuit("unsigned_overflowing_mul", n), I, [lhs.blocks, rhs.blocks])
        return self._radix(kind, out[:, :n], I), CudaBooleanBlock(out[:, n], I)

    def signed_overflowing_mul(self, lhs, rhs):
        """(lhs * rhs wrapping, [the exact lhs * rhs is outside [MIN, MAX]])
        for signed integers"""
        from . import radix_mul

        kind, n, I = self._operands(lhs, rhs)
        if not kind.signed:
            raise ValueError("signed_overflowing_mul takes signed integers")
        out = self._run_circuit(radix_mul.circuit("signed_overflowing_mul", n), I, [lhs.blocks, rhs.blocks])
        return self._radix(kind, out[:, :n], I), CudaBooleanBlock(out[:, n], I)

    def sum_ciphertexts(self, cts):
        """the wrapping sum of a list of integers of one kind, block count and
        num_inputs, per input; None for an empty list (tfhe-rs' Option)"""
        from . import radix_mul

        cts = list(cts)
        if not cts:
            return None
        kind, n, I = self._operands(*cts)
        out = self._run_circuit(radix_mul.circuit("sum", n, len(cts)), I, [ct.blocks for ct in cts])
        return self._radix(kind, out, I)

    # -- division (`radix_div`) --------------------------------------------------
    def _div(self, op, lhs, rhs):
        from . import radix_div

        kind, n, I = self._operands(lhs, rhs)
        out = self._run_circuit(radix_div.circuit(op, n, kind.signed), I, [lhs.blocks, rhs.blocks])
        return self._div_results(op, kind, n, I, out)

    def _scalar_div(self, op, lhs, scalar):
        """`scalar` is one clear divisor for every input, or one per input"""
        from . import radix_div

        kind, n, I = self._operands(lhs)
        scalars = [scalar] * I if np.ndim(scalar) == 0 else list(scalar)
        if len(scalars) != I:
            raise ValueError(f"expected one scalar or {I}, got {len(scalars)}")
        iconsts = radix_div.scalar_iconsts(scalars, n, kind.signed)
        out = self._run_circuit(radix_div.circuit(f"scalar_{op}", n, kind.signed), I, [lhs.blocks], iconsts)
        return self._div_results(op, kind, n, I, out)

    def _div_results(self, op, kind, n, I, out):
        if op == "div_rem":
            return self._radix(kind, out[:, :n], I), self._radix(kind, out[:, n:], I)
        return self._radix(kind, out, I)

    def div_rem(self, numerator, divisor):
        """(quotient, remainder) of numerator / divisor, per input.  Unsigned:
        n // d and n % d.  Signed: the quotient truncated toward zero (MIN / -1
        wraps to MIN) and the remainder with the sign of the numerator.  By an
        encrypted zero: unsigned, (2^bits - 1, n); signed, (-1 if n >= 0 else
        1, n), as tfhe-rs computes."""
        return self._div("div_rem", numerator, divisor)

    def div(self, numerator, divisor):
        """the quotient of `div_rem`"""
        return self._div("div", numerator, divisor)

    def rem(self, numerator, divisor):
        """the remainder of `div_rem`"""
        return self._div("rem", numerator, divisor)

    def scalar_div_rem(self, numerator, divisor):
        """`div_rem` by a clear divisor (one for every input, or one per input);
        a zero divisor or one outside the integer's range raises ValueError"""
        return self._scalar_div("div_rem", numerator, divisor)

    def scalar_div(self, numerator, divisor):
        """the quotient of `scalar_div_rem`"""
        return self._scalar_div("div", numerator, divisor)

    def scalar_rem(self, numerator, divisor):
        """the remainder of `scalar_div_rem`"""
        return self._scalar_div("rem", numerator, divisor)

    # -- shifts, rotations and bit counts (`radix_bits`) ------------------------
    def _shift(self, op, ct, amount):
        from . import radix_bits

        kind, n, I = self._operands(ct)
        if not isinstance(amount, CudaUnsignedRadixCiphertext) or amount.signed:
            raise ValueError(f"the amount of {op} must be a CudaUnsignedRadixCiphertext, got {type(amount).__name__}")
        _, amount_blocks, amount_inputs = self._operands(amount)
        if amount_inputs != I:
            raise ValueError(f"the amount holds {amount_inputs} input(s), the integer {I}")
        out = self._run_circuit(radix_bits.circuit(op, n, kind.signed, amount_blocks), I, [ct.blocks, amount.blocks])
        return self._radix(kind, out, I)

    def _scalar_shift(self, op, ct, amount):
        from . import radix_bits

        kind, n, I = self._operands(ct)
        circuit = radix_bits.circuit(f"scalar_{op}", n, kind.signed, amount)
        return self._radix(kind, self._run_circuit(circuit, I, [ct.blocks]), I)

    def _count(self, op, ct):
        from . import radix_bits

        kind, n, I = self._operands(ct)
        out = self._run_circuit(radix_bits.circuit(op, n, kind.signed), I, [ct.blocks])
        w = radix_bits.result_blocks(op, n)
        count = self._radix(CudaUnsignedRadixCiphertext, out[:, :w], I)
        return (count, CudaBooleanBlock(out[:, w], I)) if op == "checked_ilog2" else count

    def left_shift(self, ct, amount):
        """ct << amount per input, `amount` an unsigned radix ciphertext of any
        block count in [1, 64]; 0 when amount >= 2 * num_blocks"""
        return self._shift("left_shift", ct, amount)

    def right_shift(self, ct, amount):
        """ct >> amount per input (arithmetic for a signed ct); when amount >=
        2 * num_blocks, 0, or -1 for a negative signed ct"""
        return self._shift("right_shift", ct, amount)

    def rotate_left(self, ct, amount):
        """ct rotated left by (amount mod 2^m) mod bits, bits = 2 * num_blocks
        and m = floor(log2 bits) + [bits is not a power of 2]: the amount bits
        tfhe-rs' barrel shifter reads"""
        return self._shift("rotate_left", ct, amount)

    def rotate_right(self, ct, amount):
        """ct rotated right, the amount read as in `rotate_left`"""
        return self._shift("rotate_right", ct, amount)

    def scalar_left_shift(self, ct, amount):
        """ct << amount, `amount` a clear non-negative int for every input"""
        return self._scalar_shift("left_shift", ct, amount)

    def scalar_right_shift(self, ct, amount):
        """ct >> amount (arithmetic for a signed ct), `amount` a clear
        non-negative int for every input"""
        return self._scalar_shift("right_shift", ct, amount)

    def scalar_rotate_left(self, ct, amount):
        """ct rotated left by amount mod 2 * num_blocks"""
        return self._scalar_shift("rotate_left", ct, amount)

    def scalar_rotate_right(self, ct, amount):
        """ct rotated right by amount mod 2 * num_blocks"""
        return self._scalar_shift("rotate_right", ct, amount)

    def leading_zeros(self, ct):
        """the leading zero bits of ct's bit pattern (signed integers too), an
        unsigned integer of ceil((floor(log2 bits) + 1) / 2) blocks"""
        return self._count("leading_zeros", ct)

    def leading_ones(self, ct):
        """the leading one bits of ct's bit pattern, as `leading_zeros`"""
        return self._count("leading_ones", ct)

    def trailing_zeros(self, ct):
        """the trailing zero bits of ct's bit pattern, as `leading_zeros`"""
        return self._count("trailing_zeros", ct)

    def trailing_ones(self, ct):
        """the trailing one bits of ct's bit pattern, as `leading_zeros`"""
        return self._count("trailing_ones", ct)

    def count_ones(self, ct):
        """the one bits of ct's bit pattern, an unsigned integer of 16 blocks"""
        return self._count("count_ones", ct)

    def count_zeros(self, ct):
        """the zero bits of ct's bit pattern, an unsigned integer of 16 blocks"""
        return self._count("count_zeros", ct)

    def ilog2(self, ct):
        """floor(log2) of ct's bit pattern (a signed integer is read as its bit
        pattern, as tfhe-rs does): (bits - 1) - leading_zeros, an unsigned
        integer of ceil((floor(log2(bits - 1)) + 2) / 2) blocks; all ones for 0"""
        return self._count("ilog2", ct)

    def checked_ilog2(self, ct):
        """(`ilog2`, ct > 0): the flag compares with ct's own signedness, as
        tfhe-rs does, so it is 0 for a negative signed ct"""
        return self._count("checked_ilog2", ct)

    # -- vector find and the key-value store (`radix_find`, `kv_store`) ---------
    # Lists are Python sequences of ciphertexts holding one integer each, of
    # one kind and block count; indexes are unsigned.  Empty lists and stores
    # give tfhe-rs' trivial results.
    def match_value(self, ct, matches):
        """(the output of the (input, output) pair of `matches` whose input
        equals the unsigned ct, else 0, on enough blocks for the largest
        output; [a match was found]).  Inputs must be unique and fit ct."""
        from . import radix_find

        return radix_find.match_value(self, ct, matches)

    def match_value_or(self, ct, matches, or_value):
        """the output of the matching pair, or the clear `or_value` when none
        matches, on enough blocks for both"""
        from . import radix_find

        return radix_find.match_value_or(self, ct, matches, or_value)

    def contains(self, cts, value):
        """[the encrypted value equals an entry of cts]"""
        from . import radix_find

        return radix_find.contains(self, cts, value)

    def contains_clear(self, cts, clear):
        """[the clear value equals an entry of cts]"""
        from . import radix_find

        return radix_find.contains_clear(self, cts, clear)

    def is_in_clears(self, ct, clears):
        """[ct equals one of the clears]"""
        from . import radix_find

        return radix_find.is_in_clears(self, ct, clears)

    def index_in_clears(self, ct, clears):
        """(index of ct in clears, found) on enough blocks for len - 1; 0 when
        not found"""
        from . import radix_find

        return radix_find.index_in_clears(self, ct, clears)

    def first_index_in_clears(self, ct, clears):
        """(index of the first occurrence of ct in clears, found)"""
        from . import radix_find

        return radix_find.index_in_clears(self, ct, clears, first=True)

    def index_of(self, cts, value):
        """(index of the encrypted value in cts, found)"""
        from . import radix_find

        return radix_find.index_of(self, cts, value=value)

    def index_of_clear(self, cts, clear):
        """(index of the clear value in cts, found)"""
        from . import radix_find

        return radix_find.index_of(self, cts, clear=clear)

    def first_index_of(self, cts, value):
        """(index of the first entry of cts equal to the encrypted value, found)"""
        from . import radix_find

        return radix_find.index_of(self, cts, value=value, first=True)

    def first_index_of_clear(self, cts, clear):
        """(index of the first entry of cts equal to the clear value, found)"""
        from . import radix_find

        return radix_find.index_of(self, cts, clear=clear, first=True)

    def all_eq_slices(self, lhs, rhs):
        """[lhs and rhs have one length and equal entries pairwise]"""
        from . import radix_find

        return radix_find.all_eq_slices(self, lhs, rhs)

    def contains_sub_slice(self, lhs, pattern):
        """[the non-empty pattern occurs in lhs as a contiguous run]"""
        from . import radix_find

        return radix_find.contains_sub_slice(self, lhs, pattern)

    def kv_store_get(self, store, key):
        """(the value of `store` (a kv_store.CudaKVStore) under the key equal
        to the encrypted `key`, else 0; found)"""
        from . import radix_find

        return radix_find.kv_store_get(self, store, key)

    def kv_store_update(self, store, key, new_value):
        """store[key] = new_value for the encrypted key, every entry rewritten
        as sel_i ? new_value : v_i in one call; returns found"""
        from . import radix_find

        return radix_find.kv_store_update(self, store, key, new_value)

    def kv_store_map(self, store, key, func):
        """(old, new, found): old = store[key], new = func(old) (any callable
        on a ciphertext, for example a method of this key), store[key] = new"""
        from . import radix_find

        return radix_find.kv_store_map(self, store, key, func)

    def kv_store_contains_key(self, store, key):
        from . import radix_find

        return radix_find.kv_store_contains_key(self, store, key)

    def kv_store_contains_value(self, store, value):
        from . import radix_find

        return radix_find.kv_store_contains_value(self, store, value)

    def kv_store_contains_clear_value(self, store, clear):
        from . import radix_find

        return radix_find.kv_store_contains_clear_value(self, store, clear)

    # -- oblivious shuffle (`radix_shuffle`) --------------------------------------
    def bitonic_shuffle(self, oprf_key, data, key_size, seed):
        """`data` (single-integer radix ciphertexts of one kind and block count)
        permuted uniformly at random: sorted by sort keys of `key_size` (a
        radix_shuffle.BitonicShuffleKeySize) drawn from `seed` by `oprf_key`
        (an oprf.CudaOprfServerKey) through a bitonic network.  Returns a new
        list; lists of length 0 or 1 come back as they are."""
        from . import radix_shuffle

        return radix_shuffle.bitonic_shuffle(self, oprf_key, data, key_size, seed)

    def bitonic_shuffle_and_re_randomize(self, oprf_key, data, key_size, seed, re_randomization_key, prf_context):
        """`bitonic_shuffle` with the sort keys re-randomized by one list of
        zeros whose seed derives from `prf_context` (a
        rerand.ReRandomizationContext, left as it was), the OPRF seed and the
        keys' bit layout; the same permutation as `bitonic_shuffle`."""
        from . import radix_shuffle

        return radix_shuffle.bitonic_shuffle_and_re_randomize(self, oprf_key, data, key_size, seed,
                                                              re_randomization_key, prf_context)

    def bitonic_shuffle_with_keys(self, data, keys):
        """`data` sorted by `keys` (unsigned radix ciphertexts of one block
        count, one per element) through the bitonic network; equal keys are
        ordered as tfhe-rs orders them."""
        from . import radix_shuffle

        return radix_shuffle.bitonic_shuffle_with_keys(self, data, keys)
