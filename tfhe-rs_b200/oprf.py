"""Oblivious pseudo-random generation (OPRF): encrypted random integers drawn
from a public seed, with no client involved.

Restates tfhe-rs' `create_random_from_seed_modulus_switched`
(tfhe/src/shortint/oprf.rs) on the host side and hands the rest to
`b200_grouped_oprf_64_async`:

  1. block plan: a chunk of `bc` random bits is `bc // r` blocks of `r` bits
     plus one block of `bc % r` bits when that is not 0 (r = log2(message
     modulus));
  2. SHA3-256("TFHE_PRF" || seed bytes || RLE of the plan) -> 32-byte digest;
  3. XofSeed(digest, "PRF_INIT") -> `xof_init_128` (tfhe-csprng
     generators/aes_ctr/mod.rs): a CBC-MAC chain of AES-128 under the zero key
     gives the AES key and the first counter of the mask stream;
  4. on the GPU: the masks are expanded from (key, counter), every block is
     bootstrapped with the LUT of its bit count (`generate_oprf_lut`) and its
     correction (p - 1) * delta / 2 is added to the body.

Only (key, counter), the LUT indexes and the corrections cross to the device;
the switched LWEs never do.  The AES-128 here is used for the few blocks of the
XOF initialisation; the mask stream itself is generated on the GPU.
"""
from __future__ import annotations

import hashlib
from typing import List, Sequence, Tuple, Union

import numpy as np

PRF_DOMAIN_SEPARATOR = b"TFHE_PRF"
PRF_XOF_SEED_DOMAIN_SEPARATOR = b"PRF_INIT"
MASK_128 = (1 << 128) - 1
MASK_64 = (1 << 64) - 1


# ---------------------------------------------------------------------------
# AES-128 (FIPS-197), vectorised over blocks
# ---------------------------------------------------------------------------
def _xtime(a: int) -> int:
    return ((a << 1) ^ (0x1B if a & 0x80 else 0)) & 0xFF


def _gf_mul(a: int, b: int) -> int:
    p = 0
    while b:
        if b & 1:
            p ^= a
        a = _xtime(a)
        b >>= 1
    return p


def _make_sbox() -> np.ndarray:
    sbox = np.zeros(256, dtype=np.uint8)
    for x in range(256):
        inv = 0
        if x:
            inv, base, e = 1, x, 254
            while e:
                if e & 1:
                    inv = _gf_mul(inv, base)
                base = _gf_mul(base, base)
                e >>= 1
        rotl = lambda v, s: ((v << s) | (v >> (8 - s))) & 0xFF
        sbox[x] = inv ^ rotl(inv, 1) ^ rotl(inv, 2) ^ rotl(inv, 3) ^ rotl(inv, 4) ^ 0x63
    return sbox


_SBOX = _make_sbox()
_XTIME = np.array([_xtime(a) for a in range(256)], dtype=np.uint8)
# state byte i = row i % 4 of column i // 4; ShiftRows moves row r left by r
_SHIFT_ROWS = np.array([r + 4 * ((c + r) % 4) for c in range(4) for r in range(4)])


def aes128_round_keys(key: bytes) -> np.ndarray:
    """The 11 round keys of a 16-byte key, [11][16] u8."""
    assert len(key) == 16
    rk = [list(key)]
    rcon = 1
    for _ in range(10):
        prev = rk[-1]
        t = [_SBOX[prev[13]] ^ rcon, _SBOX[prev[14]], _SBOX[prev[15]], _SBOX[prev[12]]]
        rcon = _xtime(rcon)
        cur = []
        for c in range(4):
            word = t if c == 0 else cur[4 * (c - 1): 4 * c]
            cur.extend(int(prev[4 * c + b]) ^ int(word[b]) for b in range(4))
        rk.append(cur)
    return np.array(rk, dtype=np.uint8)


def aes128_encrypt(key: bytes, blocks: np.ndarray) -> np.ndarray:
    """AES-128 of every row of `blocks` ([m][16] u8) under `key`."""
    rk = aes128_round_keys(key)
    s = np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, 16) ^ rk[0]
    for r in range(1, 11):
        s = _SBOX[s][:, _SHIFT_ROWS]
        if r < 10:
            a = s.reshape(-1, 4, 4)
            a1 = np.roll(a, -1, axis=2)
            everything = a ^ a1 ^ np.roll(a, -2, axis=2) ^ np.roll(a, -3, axis=2)
            s = (a ^ everything ^ _XTIME[a ^ a1]).reshape(-1, 16)
        s = s ^ rk[r]
    return s


def aes_ctr_bytes(key: bytes, counter: int, first_byte: int, count: int) -> np.ndarray:
    """Bytes [first_byte, first_byte + count) of the counter-mode table
    byte p = AES_K(le128(counter + p // 16))[p % 16]."""
    b0 = first_byte // 16
    nblk = (first_byte + count + 15) // 16 - b0
    ctr = [((counter + b0 + i) & MASK_128).to_bytes(16, "little") for i in range(nblk)]
    table = aes128_encrypt(key, np.frombuffer(b"".join(ctr), dtype=np.uint8)).reshape(-1)
    off = first_byte - 16 * b0
    return table[off: off + count]


# ---------------------------------------------------------------------------
# seed -> (AES key, first counter)
# ---------------------------------------------------------------------------
def xof_seed_bytes(seed: bytes, domain_separator: bytes) -> bytes:
    """XofSeed::new(seed, sep).data = sep || seed (tfhe-csprng seeders/mod.rs)."""
    assert len(domain_separator) == 8
    return bytes(domain_separator) + bytes(seed)


def xof_init_128(xof_seed: bytes) -> Tuple[bytes, int]:
    """(AES key bytes, first AES index) of RandomGenerator::new(XofSeed): the
    seed's 16-byte little-endian blocks (last one zero-padded), then its bit
    length, chained as c_i = AES_0(c_{i-1} ^ m_i); key = last c, index = the
    one before it."""
    blocks = [int.from_bytes(xof_seed[i: i + 16].ljust(16, b"\0"), "little") for i in range(0, len(xof_seed), 16)]
    blocks.append(8 * len(xof_seed))
    zero = bytes(16)
    prev_c = c = 0
    for m in blocks:
        prev_c = c
        out = aes128_encrypt(zero, np.frombuffer((prev_c ^ m).to_bytes(16, "little"), dtype=np.uint8))
        c = int.from_bytes(out.tobytes(), "little")
    return c.to_bytes(16, "little"), prev_c


def seed_bytes(seed: Union[int, bytes, bytearray, Sequence[int]]) -> bytes:
    """OprfSeed::into_bytes: Seed(u128) -> 16 little-endian bytes, bytes as given."""
    if isinstance(seed, int):
        return (seed & MASK_128).to_bytes(16, "little")
    return bytes(seed)


def block_plan(bit_chunks: Sequence[int], random_bits_per_block: int) -> List[int]:
    """Random bits carried by every block, chunks laid out one after the other."""
    assert random_bits_per_block > 0, "random_bits_per_block must be > 0"
    bits = []
    for bc in bit_chunks:
        full, last = divmod(int(bc), random_bits_per_block)
        bits.extend([random_bits_per_block] * full)
        if last:
            bits.append(last)
    return bits


def rle_bytes(bit_chunks: Sequence[int], random_bits_per_block: int, bits_per_block: int) -> bytes:
    """u64 LE words: bits_per_block, r, then per chunk num_blocks,
    [num_full, r] if num_full, [1, last_bits] if last_bits."""
    words = [bits_per_block, random_bits_per_block]
    for bc in bit_chunks:
        full, last = divmod(int(bc), random_bits_per_block)
        words.append(full + (1 if last else 0))
        if full:
            words += [full, random_bits_per_block]
        if last:
            words += [1, last]
    return b"".join(int(w).to_bytes(8, "little") for w in words)


def derive_mask_stream(seed, bit_chunks: Sequence[int], random_bits_per_block: int,
                       bits_per_block: int) -> Tuple[bytes, int, List[int]]:
    """(AES key, first counter, bits per block) of the mask stream of one
    OPRF call; the stream starts at byte 0 of that counter."""
    assert bits_per_block >= random_bits_per_block
    h = hashlib.sha3_256()
    h.update(PRF_DOMAIN_SEPARATOR)
    h.update(seed_bytes(seed))
    h.update(rle_bytes(bit_chunks, random_bits_per_block, bits_per_block))
    key, counter = xof_init_128(xof_seed_bytes(h.digest(), PRF_XOF_SEED_DOMAIN_SEPARATOR))
    return key, counter, block_plan(bit_chunks, random_bits_per_block)


# ---------------------------------------------------------------------------
# LUTs and corrections (oprf.rs generate_oprf_lut; oprf.h int_grouped_oprf_memory)
# ---------------------------------------------------------------------------
def oprf_delta(message_bits: int, carry_bits: int) -> int:
    return 1 << (64 - (1 + message_bits + carry_bits))


def oprf_lut(random_bits: int, message_bits: int, carry_bits: int, glwe_dimension: int,
             polynomial_size: int) -> np.ndarray:
    """Accumulator of p = 2^random_bits: body[x] = (2 (x // (2N / p)) + 1) delta / 2, masks 0."""
    p = 1 << random_bits
    N = polynomial_size
    assert 2 * N >= p
    delta = oprf_delta(message_bits, carry_bits)
    poly_delta = 2 * N // p
    x = np.arange(N, dtype=np.uint64) // np.uint64(poly_delta)
    with np.errstate(over="ignore"):
        body = (np.uint64(2) * x + np.uint64(1)) * np.uint64(delta) // np.uint64(2)
    out = np.zeros((glwe_dimension + 1) * N, dtype=np.uint64)
    out[glwe_dimension * N:] = body
    return out


def oprf_correction(random_bits: int, message_bits: int, carry_bits: int) -> int:
    """Plaintext added after the sample extraction: (p - 1) * delta / 2."""
    return (((1 << random_bits) - 1) * oprf_delta(message_bits, carry_bits) // 2) & MASK_64


# ---------------------------------------------------------------------------
# device entry points
# ---------------------------------------------------------------------------
def cuda_oprf_expand_seeded_lwe(lwe_out, aes_key: bytes, counter: int, first_byte_index: int, lwe_dimension: int,
                                num_blocks: int, log_modulus: int, streams, stream_index: int = 0):
    """Expands num_blocks seeded OPRF masks into `lwe_out` (CudaVec of
    num_blocks * (lwe_dimension + 1) u64)."""
    from . import _lib

    assert len(lwe_out) >= num_blocks * (lwe_dimension + 1)
    _lib.lib().b200_oprf_expand_seeded_lwe_64_async(
        streams.ptr(stream_index), streams.gpu_indexes[stream_index], lwe_out.as_c_ptr(), bytes(aes_key),
        counter & MASK_64, (counter >> 64) & MASK_64, first_byte_index, lwe_dimension, num_blocks, log_modulus)


class CudaOprfServerKey:
    """OPRF bootstrapping key resident on one GPU (the role of tfhe-rs'
    `CudaOprfServerKey`): a classic (CudaLweBootstrapKey) or multi-bit
    (CudaLweMultiBitBootstrapKey) key from the OPRF LWE secret key to the
    target GLWE key, in the 64-bit Fourier format of every other key.
    Outputs are blocks of the target parameters (message_modulus,
    carry_modulus) under the GLWE key, fresh out of a PBS."""

    def __init__(self, bsk, streams, message_modulus: int = 4, carry_modulus: int = 4):
        from . import gpu

        assert message_modulus & (message_modulus - 1) == 0 and carry_modulus & (carry_modulus - 1) == 0
        self.bsk, self.streams = bsk, streams
        self.multi_bit = isinstance(bsk, gpu.CudaLweMultiBitBootstrapKey)
        self.message_bits = message_modulus.bit_length() - 1
        self.carry_bits = carry_modulus.bit_length() - 1
        self.bits_per_block = 1 + self.message_bits + self.carry_bits
        luts = np.stack([oprf_lut(b, self.message_bits, self.carry_bits, bsk.glwe_dimension, bsk.polynomial_size)
                         for b in range(1, self.message_bits + 1)])
        self.d_luts = gpu.CudaVec.from_cpu_async(luts, streams)

    @property
    def big_dim(self) -> int:
        return self.bsk.glwe_dimension * self.bsk.polynomial_size

    def _generate_flat(self, seed, bit_chunks: Sequence[int]):
        """All blocks of `bit_chunks`, chunk after chunk, as one
        CudaLweCiphertextList."""
        from . import _lib, gpu

        key, counter, bits = derive_mask_stream(seed, bit_chunks, self.message_bits, self.bits_per_block)
        count = len(bits)
        out = gpu.CudaLweCiphertextList.new(self.big_dim, count, self.streams)
        if count == 0:
            return out
        b = np.asarray(bits, dtype=np.uint64)
        corrections = np.array([oprf_correction(int(x), self.message_bits, self.carry_bits) for x in bits],
                               dtype=np.uint64)
        d_idx = gpu.CudaVec.from_cpu_async(b - np.uint64(1), self.streams)
        d_corr = gpu.CudaVec.from_cpu_async(corrections, self.streams)
        k = self.bsk
        scratch = gpu.PbsScratch(self.streams, k.input_lwe_dimension, k.glwe_dimension, k.polynomial_size,
                                 k.decomp_level_count, count,
                                 centered=getattr(k, "ms_noise_reduction_configuration", None) is not None,
                                 multi_bit=self.multi_bit)
        try:
            _lib.lib().b200_grouped_oprf_64_async(
                self.streams.ptr(0), self.streams.gpu_indexes[0], out.d_vec.as_c_ptr(), key, counter & MASK_64,
                counter >> 64, self.d_luts.as_c_ptr(), d_idx.as_c_ptr(), d_corr.as_c_ptr(), k.d_vec.as_c_ptr(),
                scratch.buf, k.input_lwe_dimension, k.glwe_dimension, k.polynomial_size, k.decomp_base_log,
                k.decomp_level_count, k.grouping_factor if self.multi_bit else 1, count)
        finally:
            scratch.close()  # synchronises the stream: d_idx / d_corr may go
        return out

    def generate_oblivious_pseudo_random_bits_chunks(self, seed, bit_chunks: Sequence[int]):
        """One CudaLweCiphertextList per chunk of `bit_chunks` random bits
        (shortint generate_oblivious_pseudo_random_bits_chunks): ceil(bc / r)
        blocks, each encrypting a uniform value of r bits, the last one of
        bc % r bits when that is not 0; r = log2(message_modulus)."""
        flat = self._generate_flat(seed, bit_chunks)
        return self._chunks(flat.d_vec.t.view(flat.lwe_ciphertext_count, self.big_dim + 1), bit_chunks)

    def generate_oblivious_pseudo_random_bits_chunks_and_re_randomize(self, seed, bit_chunks: Sequence[int],
                                                                      re_randomization_key, prf_context):
        """`generate_oblivious_pseudo_random_bits_chunks`, then every block of
        every chunk re-randomized with one list of zeros drawn from one seed,
        `rerand.new_prf_rerand_seed(prf_context, seed, RLE of the chunks)`
        (shortint generate_pseudo_random_bits_chunks_and_re_randomize), on
        `rerand.re_randomize`.  prf_context: a rerand.ReRandomizationContext,
        left as it was."""
        from . import rerand
        from .integer import CudaUnsignedRadixCiphertext

        if not isinstance(re_randomization_key, rerand.CudaReRandomizationKey):
            raise ValueError(f"{re_randomization_key!r} is not a CudaReRandomizationKey")
        rr_seed = rerand.new_prf_rerand_seed(prf_context, seed,
                                             rle_bytes(bit_chunks, self.message_bits, self.bits_per_block))
        flat = self._generate_flat(seed, bit_chunks)
        t = flat.d_vec.t.view(flat.lwe_ciphertext_count, self.big_dim + 1)
        if flat.lwe_ciphertext_count:
            rerand.re_randomize([CudaUnsignedRadixCiphertext(t)], [rr_seed], re_randomization_key, self.streams)
        return self._chunks(t, bit_chunks)

    def _chunks(self, t, bit_chunks: Sequence[int]):
        """CudaLweCiphertextList views of the flat blocks `t`, one per chunk"""
        from . import gpu

        chunks, at = [], 0
        for bc in bit_chunks:
            n = -(-int(bc) // self.message_bits)
            chunks.append(gpu.CudaLweCiphertextList(gpu.CudaVec(t[at: at + n].reshape(-1), np.uint64),
                                                    self.big_dim, n))
            at += n
        return chunks

    def generate_oblivious_pseudo_random_unsigned_integer(self, seed, num_blocks: int):
        """Uniform integer in [0, message_modulus^num_blocks)
        (par_generate_oblivious_pseudo_random_unsigned_integer)."""
        from .integer import CudaUnsignedRadixCiphertext

        flat = self._generate_flat(seed, [num_blocks * self.message_bits])
        return CudaUnsignedRadixCiphertext(flat.d_vec.t.view(num_blocks, self.big_dim + 1))

    def generate_oblivious_pseudo_random_unsigned_integer_bounded(self, seed, random_bits_count: int,
                                                                  num_blocks: int):
        """Uniform integer in [0, 2^random_bits_count) on num_blocks blocks; the
        blocks above the random ones are trivial zeros
        (par_generate_oblivious_pseudo_random_unsigned_integer_bounded)."""
        import torch

        from .integer import CudaUnsignedRadixCiphertext

        range_bits = self.message_bits * num_blocks
        assert 0 < range_bits and random_bits_count <= range_bits, (
            f"The range asked for a random value in [0, 2^{random_bits_count}[ does not fit in the available "
            f"range [0, 2^{range_bits}[")
        flat = self._generate_flat(seed, [random_bits_count])
        t = flat.d_vec.t.view(flat.lwe_ciphertext_count, self.big_dim + 1)
        pad = num_blocks - flat.lwe_ciphertext_count
        if pad:
            with torch.cuda.stream(self.streams.streams[0]):
                t = torch.cat([t, torch.zeros((pad, self.big_dim + 1), dtype=t.dtype, device=t.device)])
        return CudaUnsignedRadixCiphertext(t)
