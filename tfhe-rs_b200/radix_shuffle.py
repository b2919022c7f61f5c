"""Oblivious shuffle of encrypted integers: `bitonic_shuffle`,
`bitonic_shuffle_and_re_randomize` and `bitonic_shuffle_with_keys` of
`integer.CudaRadixServerKey`.  A list is permuted uniformly at random, the
permutation a function of a public seed and the OPRF secret key only: one
OPRF sort key per element (optionally re-randomized), then a bitonic sorting
network of compare-and-swaps on the keys, each swap moving key and data
together.  Host code only: the sort keys come from `oprf.cuh` (and
`rerand.cuh`), and every compare-and-swap runs on the KS and PBS kernels
through `b200_bit_circuit_64_async`.

Semantics are tfhe-rs' (`radix_parallel/bitonic_shuffle.rs`);
`tests/shuffle_model.py` restates them on Python integers:

  * network: for n = next_power_of_two(len), phase in 0..log n, step in
    phase..0, the pairs (i, j = i ^ 2^step), j > i, ascending iff bit
    phase + 1 of i is 0 (`network`);
  * swap rule: an ascending pair swaps iff key_i > key_j, a descending pair
    iff key_i <= key_j; with equal keys this asymmetry decides the
    permutation;
  * padding: when len is not a power of two every key gets one zero block on
    top, and n - len elements are appended with keys of all digits 3 (above
    every real key) and data 0; the result is the first len elements;
  * key size (`BitonicShuffleKeySize`): ceil(bits / 2) blocks.

One compare-and-swap circuit per (key blocks K, data blocks D), compiled once
(`circuit`); a pair is one instance, its direction a per-instance constant
bit.  gt = `radix.compare` (2K - 1 PBS); every block x_i, x_j of the pair
then takes 4 PBS in two layers: A = keep_if(cond, x_j), B = keep_if(not cond,
x_i), with cond = gt XOR desc folded into their input as the body constant
8 desc, then x_i' = A + B and x_j' = x_i + x_j - A - B (noise 4), both
identity PBS.  Every output is a PBS output holding a value <= 3, so it feeds
the next stage's comparison of 4 k_i + k_j.

Each network stage is one `runner.run` over its n / 2 pairs, fed by one
index gather from the element store; the outputs, in pair order, are the next
stage's store, addressed through the element -> row map, so no scatter runs
between stages.  log n (log n + 1) / 2 calls per shuffle.
"""
from __future__ import annotations

import functools
import math
from typing import List, Tuple

import numpy as np

from . import bit_circuit as bc
from . import radix
from .radix import MSG_MOD, blocks_of

MSG_BITS = 2   # log2(MSG_MOD): random bits per OPRF block
U32_MAX = 2 ** 32 - 1


# ---------------------------------------------------------------------------
# the network and the key size
# ---------------------------------------------------------------------------
@functools.lru_cache(maxsize=16)
def network(n: int) -> Tuple[Tuple[Tuple[int, int, bool], ...], ...]:
    """tfhe-rs `bitonic_network(n)`, n a power of two >= 2: the stages, each
    the disjoint (i, j, ascending) compare-and-swaps of one layer"""
    if n < 2 or n & (n - 1):
        raise ValueError(f"a bitonic network needs a power of two >= 2, got {n}")
    log_n = n.bit_length() - 1
    stages = []
    for phase in range(log_n):
        for step in range(phase, -1, -1):
            stages.append(tuple((i, i ^ (1 << step), (i >> (phase + 1)) & 1 == 0)
                                for i in range(n) if i ^ (1 << step) > i))
    return tuple(stages)


def next_power_of_two(n: int) -> int:
    return 1 if n <= 1 else 1 << (n - 1).bit_length()


def _saturating_u32(x: float) -> int:
    """Rust's `f64 as u32`: NaN and values below 0 give 0, above u32::MAX
    give u32::MAX, others truncate"""
    if x != x or x <= 0:
        return 0
    return U32_MAX if x >= U32_MAX else int(x)


class BitonicShuffleKeySize:
    """Width of the random sort keys (tfhe-rs BitonicShuffleKeySize): by a
    target collision probability p, bits = ceil(log2(len^2 / (2 p))), or by a
    bit count; blocks = ceil(bits / 2).  Larger keys make ties rarer, and so
    the permutation closer to uniform, at the cost of wider comparisons."""

    def __init__(self, probability=None, bits=None):
        self.probability, self.bits = probability, bits

    @classmethod
    def collision_probability(cls, p) -> "BitonicShuffleKeySize":
        if isinstance(p, bool) or not isinstance(p, (int, float, np.floating, np.integer)) or not 0.0 < p < 1.0:
            raise ValueError(f"a collision probability must lie in (0, 1), got {p!r}")
        return cls(probability=float(p))

    @classmethod
    def num_bits(cls, b) -> "BitonicShuffleKeySize":
        if isinstance(b, bool) or not isinstance(b, (int, np.integer)) or not 0 <= b <= U32_MAX:
            raise ValueError(f"a key bit count is an integer in [0, 2^32), got {b!r}")
        return cls(bits=int(b))

    def num_blocks(self, num_elements: int) -> int:
        """key blocks for a list of `num_elements` (0 is a valid answer, which
        the shuffles reject)"""
        if self.bits is not None:
            bits = self.bits
        else:
            x = float(num_elements * num_elements) / (2.0 * self.probability)
            bits = _saturating_u32(math.ceil(math.log2(x))) if x > 0 else 0   # log2(0) = -inf -> 0
        return -(-bits // MSG_BITS)

    def __repr__(self):
        return (f"BitonicShuffleKeySize.collision_probability({self.probability!r})" if self.bits is None
                else f"BitonicShuffleKeySize.num_bits({self.bits})")


# ---------------------------------------------------------------------------
# the compare-and-swap circuit
# ---------------------------------------------------------------------------
def swap_blocks(c: bc.Circuit, cond: int, desc: int, xi: List[int], xj: List[int]) -> Tuple[List[int], List[int]]:
    """(cond XOR desc ? xj : xi, cond XOR desc ? xi : xj) of two block lists:
    4 PBS per block pair, two layers"""
    a = radix.keep_if(c, cond, blocks_of(xj), 1, flip=desc)
    b = radix.keep_if(c, cond, blocks_of(xi), 0, flip=desc)
    ident = lambda v: v % MSG_MOD  # noqa: E731
    new_i = [radix._pbs(c, [(p, 1), (q, 1)], 0, ident) for p, q in zip(a, b)]
    # x_i + x_j - A - B is the other operand; the body 6 keeps the input >= 0
    new_j = [radix._pbs(c, [(x, 1), (y, 1), (p, -1), (q, -1)], 2 * (MSG_MOD - 1),
                        lambda v: (v - 2 * (MSG_MOD - 1)) % MSG_MOD)
             for x, y, p, q in zip(xi, xj, a, b)]
    return new_i, new_j


def circuit(key_blocks: int, data_blocks: int) -> bc.Circuit:
    """The compare-and-swap of one pair, its instance.  Inputs k_i (key
    blocks), d_i (data blocks), k_j, d_j; one per-instance constant, desc
    (1 for a descending pair).  Outputs k_i', d_i', k_j', d_j', swapped iff
    (k_i > k_j) XOR desc.  The radix.CIRCUIT_CACHE_SIZE most recent circuits
    are kept."""
    return _circuit(radix.check_num_blocks(key_blocks), radix.check_num_blocks(data_blocks))


@functools.lru_cache(maxsize=radix.CIRCUIT_CACHE_SIZE)
def _circuit(nk: int, nd: int) -> bc.Circuit:
    c = bc.Circuit(f"shuffle_cas_{nk}_{nd}")
    ki, di = c.inputs_block(nk, False), c.inputs_block(nd, False)
    kj, dj = c.inputs_block(nk, False), c.inputs_block(nd, False)
    desc = c.iconst()
    gt = radix.compare(c, blocks_of(ki), blocks_of(kj), "gt")
    new_i, new_j = swap_blocks(c, gt, desc, ki + di, kj + dj)
    c.output_blocks(new_i + new_j)
    return c


def stage_inputs(stage) -> Tuple[np.ndarray, np.ndarray]:
    """(element indexes [pairs, 2] (i, j), desc bits [pairs, 1]) of a stage"""
    pairs = np.array([(i, j) for i, j, _ in stage], dtype=np.int64).reshape(-1, 2)
    desc = np.array([[0 if asc else 1] for _, _, asc in stage], dtype=np.int64)
    return pairs, desc


def cost(length: int, key_blocks: int, data_blocks: int) -> Tuple[int, int, int]:
    """(PBS per stage, PBS layers per stage, stages) of a shuffle of
    `length` elements whose keys have `key_blocks` blocks (before the
    padding block, added when length is not a power of two)"""
    if length <= 1:
        return 0, 0, 0
    n = next_power_of_two(length)
    nk = key_blocks + (n != length)
    s = bc.schedule(circuit(nk, data_blocks), n // 2)
    log_n = n.bit_length() - 1
    return s.pbs_count(), s.num_layers, log_n * (log_n + 1) // 2


# ---------------------------------------------------------------------------
# the operations on `integer.CudaRadixServerKey`
# ---------------------------------------------------------------------------
def _check_2_2(key):
    """a 2_2 server key, checked without creating the runner"""
    if key._runner is not None:
        return
    skey = key.engine.skey
    moduli = (getattr(skey, "message_modulus", None), getattr(skey, "carry_modulus", None))
    if moduli != (MSG_MOD, bc.TOTAL_MOD // MSG_MOD):
        raise ValueError(f"bitonic shuffles need a 2_2 server key, got message / carry moduli {moduli}")


def _check_data(key, data, what: str = "data"):
    """(kind, num_blocks) of a list of single-integer radix ciphertexts of one
    kind and block count; (None, None) for an empty list"""
    if not data:
        return None, None
    kind, n, I = key._operands(*data)
    if I != 1:
        raise ValueError(f"every entry of the {what} must hold one integer (num_inputs = 1), got {I}")
    return kind, n


def _key_blocks(key_size, length: int) -> int:
    if not isinstance(key_size, BitonicShuffleKeySize):
        raise ValueError(f"key_size must be a BitonicShuffleKeySize, got {key_size!r}")
    nk = key_size.num_blocks(length)
    if nk == 0:
        raise ValueError(f"{key_size!r} gives sort keys of 0 blocks for {length} elements: at least 1 is needed")
    return _check_key_width(nk, length)


def _check_key_width(nk: int, length: int) -> int:
    """nk, if the keys fit a radix circuit with the padding block"""
    if nk + (next_power_of_two(length) != length) > radix.MAX_BLOCKS:
        raise ValueError(f"sort keys of {nk} blocks for {length} elements do not fit {radix.MAX_BLOCKS} blocks "
                         "(one more is added when the length is not a power of two)")
    return nk


def _check_oprf(oprf_key):
    from . import oprf

    if not isinstance(oprf_key, oprf.CudaOprfServerKey):
        raise ValueError(f"oprf_key must be an oprf.CudaOprfServerKey, got {type(oprf_key).__name__}")
    if oprf_key.message_bits != MSG_BITS:
        raise ValueError(f"the OPRF key makes blocks of {oprf_key.message_bits} message bits, the shuffle "
                         f"needs {MSG_BITS}")


def _shuffle(key, data, key_blocks, nk: int):
    """Sort `data` (a non-empty list) by its keys, `key_blocks` [len, nk, W],
    through the network; returns the new list"""
    import torch

    length, nd = len(data), data[0].num_blocks
    kind = type(data[0])
    runner = key.runner
    W = data[0].blocks.shape[-1]
    keys = key_blocks.reshape(length, nk, W)
    values = torch.stack([d.blocks for d in data])
    n = next_power_of_two(length)
    if n != length:
        # a trivial zero block on top of every key, then n - len elements of
        # key 4^(nk + 1) - 1 (above every real key) and data 0
        keys = torch.cat([keys, runner.trivial([0]).view(1, 1, W).expand(length, 1, W)], 1)
        nk += 1
        keys = torch.cat([keys, runner.trivial([MSG_MOD - 1] * nk).view(1, nk, W).expand(n - length, nk, W)])
        values = torch.cat([values, runner.trivial([0] * nd).view(1, nd, W).expand(n - length, nd, W)])
    E = nk + nd
    circ = circuit(nk, nd)
    store = torch.cat([keys, values], 1).reshape(n * E, W)
    row = np.arange(n, dtype=np.int64)    # row of each element in `store` (units of E blocks)
    dev = store.device
    for stage in network(n):
        pairs, desc = stage_inputs(stage)
        src = torch.as_tensor((row[pairs.reshape(-1)][:, None] * E + np.arange(E)[None, :]).reshape(-1),
                              device=dev)
        store = runner.run(circ, None, store.index_select(0, src), desc, n // 2)
        row[pairs.reshape(-1)] = np.arange(n)
    out = store.view(n, E, W)
    keep = torch.as_tensor(row[:length], device=dev)
    picked = out.index_select(0, keep)[:, nk:].contiguous()
    return [kind(picked[e], 1) for e in range(length)]


def bitonic_shuffle_with_keys(key, data, keys):
    """`data` sorted by the unsigned radix `keys` (one per element, one block
    count) through the bitonic network, ties and padding as tfhe-rs has them"""
    import torch

    from . import integer

    data, keys = list(data), list(keys)
    _check_2_2(key)
    if len(data) != len(keys):
        raise ValueError(f"data and keys must have the same length, got {len(data)} and {len(keys)}")
    _check_data(key, data)
    kkind, nk = _check_data(key, keys, "keys")
    if keys and kkind is not integer.CudaUnsignedRadixCiphertext:
        raise ValueError(f"sort keys must be unsigned radix ciphertexts, got {kkind.__name__}")
    if keys:
        _check_key_width(nk, len(keys))
    if len(data) <= 1:
        return data
    return _shuffle(key, data, torch.cat([k.blocks for k in keys]), nk)


def _oprf_shuffle(key, oprf_key, data, key_size, draw):
    """the argument checks, then `draw(chunks)` the sort keys' block lists"""
    import torch

    data = list(data)
    _check_2_2(key)
    _check_oprf(oprf_key)
    _check_data(key, data)
    nk = _key_blocks(key_size, len(data))
    if len(data) <= 1:
        return data
    chunks = draw([MSG_BITS * nk] * len(data))
    # the sort keys were made, and their memory allocated, on the OPRF key's stream
    cur = torch.cuda.current_stream(data[0].blocks.device)
    cur.wait_stream(oprf_key.streams.streams[0])
    W = data[0].blocks.shape[-1]
    flat = torch.cat([c.d_vec.t.view(nk, W) for c in chunks])
    for c in chunks:
        c.d_vec.t.record_stream(cur)
    return _shuffle(key, data, flat, nk)


def bitonic_shuffle(key, oprf_key, data, key_size, seed):
    """tfhe-rs `bitonic_shuffle`: sort keys of `key_size` drawn by
    `oprf_key.generate_oblivious_pseudo_random_bits_chunks(seed, ...)`"""
    return _oprf_shuffle(key, oprf_key, data, key_size,
                         lambda chunks: oprf_key.generate_oblivious_pseudo_random_bits_chunks(seed, chunks))


def bitonic_shuffle_and_re_randomize(key, oprf_key, data, key_size, seed, re_randomization_key, prf_context):
    """tfhe-rs `re_randomized_keys_bitonic_shuffle`: the sort keys
    re-randomized by one list of zeros (`CudaOprfServerKey.
    generate_oblivious_pseudo_random_bits_chunks_and_re_randomize`)"""
    from . import rerand

    if not isinstance(re_randomization_key, rerand.CudaReRandomizationKey):
        raise ValueError(f"{re_randomization_key!r} is not a CudaReRandomizationKey")
    if not isinstance(prf_context, rerand.ReRandomizationContext):
        raise ValueError(f"{prf_context!r} is not a ReRandomizationContext")
    return _oprf_shuffle(key, oprf_key, data, key_size,
                         lambda chunks: oprf_key.generate_oblivious_pseudo_random_bits_chunks_and_re_randomize(
                             seed, chunks, re_randomization_key, prf_context))
