"""Ciphertext re-randomization on the GPU: a fresh compact-public-key
encryption of zero, drawn from a public seed, added to every block before the
server computes on it (tfhe-rs shortint/ciphertext/re_randomization.rs,
integer/gpu/ciphertext/re_randomization.rs).

tfhe-rs encrypts the zeros on the CPU (prepare_cpk_zero_for_rerand) and uploads
them.  Here only the 40-byte XofSeed of every ciphertext crosses to the device:
b200_cpk_encrypt_zeros_from_seeds_64_async runs the XOF initialisation, the
AES key schedule, the binary random vector, the TUniform noise and both
negacyclic products on the GPU, bit for bit what tfhe-rs computes from the same
seed, and b200_rerand_64_async expands the zeros, keyswitches them when the
key asks for it and adds them to the blocks.

Seeds come from a ReRandomizationContext: the data that identifies the
ciphertexts is hashed, then ReRandomizationSeedGen.next_seed gives one seed per
ciphertext.  The Shake256 hasher is supported; Blake3 (tfhe-rs' default) is
not, for lack of an implementation here.  Seeds derived elsewhere can be passed
as ReRandomizationSeed(seed_bytes, public_encryption_domain_separator).
"""
from __future__ import annotations

import hashlib
from typing import Optional, Sequence

import numpy as np

from .compact_list import MAX_LWE_DIMENSION, MIN_LWE_DIMENSION

DOMAIN_SEP_LEN = 8  # XofSeed::DOMAIN_SEP_LEN
RERAND_SEED_BYTES = 32  # RERAND_SEED_BITS / 8
XOF_SEED_BYTES = DOMAIN_SEP_LEN + RERAND_SEED_BYTES


def _check_separator(sep, what: str) -> bytes:
    if not isinstance(sep, (bytes, bytearray)) or len(sep) != DOMAIN_SEP_LEN:
        raise ValueError(f"the {what} must be {DOMAIN_SEP_LEN} bytes, got {sep!r}")
    return bytes(sep)


class ReRandomizationSeed:
    """XofSeed of one encryption of zeros: `data` = the 8-byte public
    encryption domain separator followed by the 32-byte seed
    (XofSeed::new(seed, sep), tfhe-csprng seeders/mod.rs)."""

    def __init__(self, seed: bytes, public_encryption_domain_separator: bytes):
        if not isinstance(seed, (bytes, bytearray)) or len(seed) != RERAND_SEED_BYTES:
            raise ValueError(f"a re-randomization seed is {RERAND_SEED_BYTES} bytes, got "
                             f"{len(seed) if isinstance(seed, (bytes, bytearray)) else seed!r}")
        sep = _check_separator(public_encryption_domain_separator, "public encryption domain separator")
        self.data = sep + bytes(seed)


class ReRandomizationSeedGen:
    """next_seed: the context's hash state, then the seed index as 8 LE bytes,
    32 bytes squeezed out (ReRandomizationSeedGen::next_seed)."""

    def __init__(self, hash_state, public_encryption_domain_separator: bytes):
        self._state = hash_state
        self._sep = public_encryption_domain_separator
        self.next_seed_index = 0

    def next_seed(self) -> ReRandomizationSeed:
        h = self._state.copy()
        h.update(self.next_seed_index.to_bytes(8, "little"))
        self.next_seed_index += 1
        return ReRandomizationSeed(h.digest(RERAND_SEED_BYTES), self._sep)


class ReRandomizationContext:
    """Hash state fed with the data that identifies the ciphertexts, in call
    order (ReRandomizationContext, re_randomization.rs:126-237).  The state
    starts with the seeder domain separator."""

    def __init__(self, rerand_seeder_domain_separator: bytes, public_encryption_domain_separator: bytes,
                 hash_algo: str = "shake256"):
        if hash_algo == "blake3":
            raise ValueError("the Blake3 seed hasher is not available: use hash_algo='shake256'")
        if hash_algo != "shake256":
            raise ValueError(f"unknown seed hasher {hash_algo!r}: 'shake256' is supported")
        seeder_sep = _check_separator(rerand_seeder_domain_separator, "seeder domain separator")
        self._sep = _check_separator(public_encryption_domain_separator, "public encryption domain separator")
        self._state = hashlib.shake_256(seeder_sep)

    def add_bytes(self, data: bytes):
        self._state.update(bytes(data))

    def add_ciphertext(self, ciphertext):
        """The ciphertext's u64 words, little endian (add_ciphertext_data_slice).
        Several ciphertexts added one after the other hash like
        add_ciphertext_iterator over them."""
        words = np.ascontiguousarray(ciphertext, dtype=np.uint64).reshape(-1)
        self._state.update(words.astype("<u8").tobytes())

    def finalize(self) -> ReRandomizationSeedGen:
        return ReRandomizationSeedGen(self._state.copy(), self._sep)

    def copy(self) -> "ReRandomizationContext":
        """An independent context with the same hash state (the Rust type's
        Clone): one context can serve several calls."""
        out = ReRandomizationContext.__new__(ReRandomizationContext)
        out._sep, out._state = self._sep, self._state.copy()
        return out


def new_prf_rerand_seed(context: ReRandomizationContext, prf_seed, random_bits_rle: bytes) -> ReRandomizationSeed:
    """The seed of the zeros that re-randomize one OPRF call's blocks
    (ReRandomizationSeed::new_prf_rerand_seed, re_randomization.rs): a copy of
    the context, then the OPRF seed's bytes, then the RLE of the call's random
    bits (`oprf.rle_bytes`), finalized; its first seed.  `context` is left as
    it was."""
    from . import oprf

    if not isinstance(context, ReRandomizationContext):
        raise ValueError(f"{context!r} is not a ReRandomizationContext")
    ctx = context.copy()
    ctx.add_bytes(oprf.seed_bytes(prf_seed))
    ctx.add_bytes(random_bits_rle)
    return ctx.finalize().next_seed()


def seeds_array(seeds: Sequence[ReRandomizationSeed]) -> np.ndarray:
    """[len(seeds)][40] u8, the layout b200_cpk_encrypt_zeros_from_seeds_64_async reads."""
    if len(seeds) == 0:
        raise ValueError("no seed")
    for s in seeds:
        if not isinstance(s, ReRandomizationSeed):
            raise ValueError(f"{s!r} is not a ReRandomizationSeed")
    return np.frombuffer(b"".join(s.data for s in seeds), dtype=np.uint8).reshape(len(seeds), XOF_SEED_BYTES)


def tuniform_bytes(noise_bound_log2: int) -> int:
    """Stream bytes of one TUniform(b) sample: ceil((b + 2) / 8)."""
    return (noise_bound_log2 + 2 + 7) // 8


def zero_list_stream_bytes(count: int, n: int, noise_bound_log2: int) -> int:
    """Stream bytes one list of `count` zeros consumes: the r bits of its bins,
    then the mask and the body noise."""
    bins = -(-count // n)
    return bins * n // 8 + (bins * n + count) * tuniform_bytes(noise_bound_log2)


def bin_counts(counts: Sequence[int], n: int) -> np.ndarray:
    """Bodies per bin of n of lists of `counts` zeros, list after list."""
    counts = np.asarray(counts, dtype=np.int64)
    bins = -(-counts // n)
    out = np.full(int(bins.sum()), n, dtype=np.uint32)
    out[np.cumsum(bins) - 1] = counts - (bins - 1) * n
    return out


class CudaCompactPublicKey:
    """Compact public key resident on one GPU (tfhe-rs CompactPublicKey): the
    mask then the body polynomial of n words, and the TUniform bound of its
    encryption noise."""

    def __init__(self, d_vec, lwe_dimension: int, noise_bound_log2: int):
        n = lwe_dimension
        if not (MIN_LWE_DIMENSION <= n <= MAX_LWE_DIMENSION and n & (n - 1) == 0):
            raise ValueError(f"the compact lwe_dimension must be a power of two in "
                             f"[{MIN_LWE_DIMENSION}, {MAX_LWE_DIMENSION}], got {n}")
        if not 0 <= noise_bound_log2 <= 62:
            raise ValueError(f"noise_bound_log2 must be in [0, 62], got {noise_bound_log2}")
        if len(d_vec) != 2 * n:
            raise ValueError(f"a compact public key of dimension {n} has {2 * n} words, got {len(d_vec)}")
        self.d_vec, self.lwe_dimension, self.noise_bound_log2 = d_vec, n, noise_bound_log2

    @classmethod
    def from_compact_public_key(cls, mask: np.ndarray, body: np.ndarray, noise_bound_log2: int, streams,
                                stream_index: int = 0) -> "CudaCompactPublicKey":
        from . import gpu

        mask = np.ascontiguousarray(mask, dtype=np.uint64).reshape(-1)
        body = np.ascontiguousarray(body, dtype=np.uint64).reshape(-1)
        if mask.size != body.size:
            raise ValueError(f"mask ({mask.size} words) and body ({body.size}) differ in size")
        return cls(gpu.CudaVec.from_cpu_async(np.concatenate([mask, body]), streams, stream_index), mask.size,
                   noise_bound_log2)


class CudaReRandomizationKey:
    """What re-randomizes blocks (CudaReRandomizationKey): `derived(cpk)`, a
    compact key derived from the blocks' own key, whose zeros are added as
    they are; or `legacy(cpk, ksk, ...)`, a dedicated compact key whose zeros
    are keyswitched to the blocks' key first."""

    def __init__(self, cpk: CudaCompactPublicKey, ksk=None):
        self.cpk, self.ksk = cpk, ksk

    @classmethod
    def derived(cls, cpk: CudaCompactPublicKey) -> "CudaReRandomizationKey":
        if not isinstance(cpk, CudaCompactPublicKey):
            raise ValueError(f"{cpk!r} is not a CudaCompactPublicKey")
        return cls(cpk)

    @classmethod
    def legacy(cls, cpk: CudaCompactPublicKey, ksk, base_log: Optional[int] = None,
               level: Optional[int] = None) -> "CudaReRandomizationKey":
        """ksk: a CudaLweKeyswitchKey from the compact key to the blocks' key;
        base_log / level, when given, must be its decomposition."""
        if not isinstance(cpk, CudaCompactPublicKey):
            raise ValueError(f"{cpk!r} is not a CudaCompactPublicKey")
        if ksk.input_key_lwe_dimension != cpk.lwe_dimension:
            raise ValueError(f"the keyswitching key takes dimension {ksk.input_key_lwe_dimension}, the compact "
                             f"public key has {cpk.lwe_dimension}")
        if (base_log is not None and base_log != ksk.decomp_base_log) or (
                level is not None and level != ksk.decomp_level_count):
            raise ValueError(f"the keyswitching key decomposes with base_log {ksk.decomp_base_log}, level "
                             f"{ksk.decomp_level_count}; got {base_log}, {level}")
        if not (1 <= ksk.decomp_level_count and ksk.decomp_base_log * ksk.decomp_level_count <= 63):
            raise ValueError("unsupported keyswitch decomposition")
        return cls(cpk, ksk)

    @property
    def output_lwe_dimension(self) -> int:
        return self.ksk.output_key_lwe_dimension if self.ksk is not None else self.cpk.lwe_dimension


def _check_entries_and_seeds(counts: Sequence[int], seeds: Sequence[ReRandomizationSeed]):
    if len(counts) == 0:
        raise ValueError("empty batch")
    if len(seeds) != len(counts):
        raise ValueError(f"{len(counts)} ciphertexts and {len(seeds)} seeds: one seed each")


def encrypt_zeros_from_seeds(cpk: CudaCompactPublicKey, seeds: Sequence[ReRandomizationSeed], entries: np.ndarray,
                             streams, out=None, accumulate: bool = False, stream_index: int = 0):
    """b200_cpk_encrypt_zeros_from_seeds_64_async: entries [k][3] u64 {seed
    index, first stream byte, count}; returns the CudaVec of the flattened
    zero lists (written into, or with accumulate added into, `out`)."""
    import ctypes as C

    from . import _lib, gpu

    seeds_u8 = seeds_array(seeds)
    entries = np.ascontiguousarray(entries, dtype=np.uint64).reshape(-1, 3)
    if entries.shape[0] == 0:
        raise ValueError("empty batch")
    if entries[:, 2].min() < 1 or entries[:, 2].max() >= 2 ** 32:
        raise ValueError("every entry must encrypt between 1 and 2^32 - 1 zeros")
    if entries[:, 0].max() >= len(seeds):
        raise ValueError(f"an entry uses seed {int(entries[:, 0].max())} of {len(seeds)}")
    n = cpk.lwe_dimension
    counts = entries[:, 2].astype(np.int64)
    words = int((-(-counts // n) * n + counts).sum())
    if out is None:
        if accumulate:
            raise ValueError("accumulate needs an output buffer")
        out = gpu.CudaVec.new(words, streams, stream_index)
    elif len(out) != words:
        raise ValueError(f"the zero lists take {words} words, the buffer holds {len(out)}")
    _lib.lib().b200_cpk_encrypt_zeros_from_seeds_64_async(
        streams.ptr(stream_index), streams.gpu_indexes[stream_index], out.as_c_ptr(), cpk.d_vec.as_c_ptr(),
        seeds_u8.ctypes.data_as(C.POINTER(C.c_uint8)), len(seeds), entries.ctypes.data_as(C.POINTER(C.c_uint64)),
        entries.shape[0], n, cpk.noise_bound_log2, accumulate)
    return out


def re_randomize(ciphertexts, seeds: Sequence[ReRandomizationSeed], key: CudaReRandomizationKey, streams,
                 stream_index: int = 0):
    """Re-randomizes every ciphertext in place (CudaRadixCiphertext::
    re_randomize): CudaUnsignedRadixCiphertext, CudaSignedRadixCiphertext or
    CudaBooleanBlock, one seed each.  Ciphertext i gets the zeros of one list
    of num_blocks_i encryptions drawn from seeds[i] (prepare_cpk_zero_for_rerand).
    One generation call and one b200_rerand_64_async cover the whole batch."""
    import ctypes as C

    import torch

    from . import _lib

    if not isinstance(key, CudaReRandomizationKey):
        raise ValueError(f"{key!r} is not a CudaReRandomizationKey")
    ciphertexts = list(ciphertexts)
    nb = [int(ct.blocks.shape[0]) for ct in ciphertexts]
    _check_entries_and_seeds(nb, seeds)
    d = key.output_lwe_dimension
    for i, ct in enumerate(ciphertexts):
        if ct.blocks.ndim != 2 or ct.blocks.shape[1] != d + 1:
            raise ValueError(f"ciphertext {i} has LWE size {ct.blocks.shape[-1]}, the key re-randomizes LWE "
                             f"size {d + 1}")
        if nb[i] < 1:
            raise ValueError(f"ciphertext {i} has no block")
    cpk = key.cpk
    n = cpk.lwe_dimension
    entries = np.zeros((len(nb), 3), dtype=np.uint64)
    entries[:, 0] = np.arange(len(nb))
    entries[:, 2] = nb
    zeros = encrypt_zeros_from_seeds(cpk, seeds, entries, streams, stream_index=stream_index)
    counts = bin_counts(nb, n)
    with torch.cuda.stream(streams.streams[stream_index]):
        single = len(ciphertexts) == 1 and ciphertexts[0].blocks.is_contiguous()
        blocks = ciphertexts[0].blocks if single else torch.cat([ct.blocks for ct in ciphertexts])
        ksk = key.ksk
        _lib.lib().b200_rerand_64_async(
            streams.ptr(stream_index), streams.gpu_indexes[stream_index], blocks.data_ptr(), zeros.as_c_ptr(),
            counts.ctypes.data_as(C.POINTER(C.c_uint32)), counts.size, n,
            ksk.d_vec.as_c_ptr() if ksk is not None else None, ksk.decomp_base_log if ksk is not None else 0,
            ksk.decomp_level_count if ksk is not None else 0, d)
        if not single:
            at = 0
            for ct, k in zip(ciphertexts, nb):
                ct.blocks.copy_(blocks[at:at + k])
                at += k
    return ciphertexts


def re_randomize_compact_lists(lists, cpk: CudaCompactPublicKey, seed: ReRandomizationSeed, streams,
                               stream_index: int = 0):
    """Adds zeros to a CudaFlattenedVecCompactCiphertextList in place
    (re_randomize_compact_ciphertext_lists, re_randomization.rs:466-490): one
    generator runs across the lists, list k starting where list k - 1 ended."""
    if not isinstance(cpk, CudaCompactPublicKey):
        raise ValueError(f"{cpk!r} is not a CudaCompactPublicKey")
    if not isinstance(seed, ReRandomizationSeed):
        raise ValueError(f"{seed!r} is not a ReRandomizationSeed")
    if lists.lwe_dimension != cpk.lwe_dimension:
        raise ValueError(f"the lists have dimension {lists.lwe_dimension}, the compact public key "
                         f"{cpk.lwe_dimension}")
    counts = lists.list_counts
    if counts is None:
        raise ValueError("the lists were flattened without their list boundaries (list_counts)")
    counts = np.asarray(counts, dtype=np.int64)
    if counts.size == 0:
        raise ValueError("empty batch")
    if not np.array_equal(bin_counts(counts, cpk.lwe_dimension), lists.num_lwe_per_compact_list):
        raise ValueError("list_counts do not match the bins of the flattened lists")
    consumed = np.array([zero_list_stream_bytes(int(c), cpk.lwe_dimension, cpk.noise_bound_log2) for c in counts],
                        dtype=np.uint64)
    entries = np.zeros((counts.size, 3), dtype=np.uint64)
    entries[1:, 1] = np.cumsum(consumed)[:-1]
    entries[:, 2] = counts
    encrypt_zeros_from_seeds(cpk, [seed], entries, streams, out=lists.d_flattened_vec, accumulate=True,
                             stream_index=stream_index)
    return lists
