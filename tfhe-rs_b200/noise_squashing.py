"""Noise squashing on the GPU (tfhe-rs `squash_noise`,
shortint/integer NoiseSquashingKey::squash_radix_ciphertext_noise): radix
blocks are packed two per LWE, keyswitched to the small key and bootstrapped
with a 128-bit key (cuda_programmable_bootstrap_128_async, or
cuda_multi_bit_programmable_bootstrap_128_async for the multi-bit squashing
keys of tfhe-rs' GPU parameters) into u128 LWEs whose noise is far below their
message step, ready for threshold decryption.

u128 words are stored as two u64, low then high (a (..., 2) numpy u64 array on
the host)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from . import gpu
from .compact_list import CudaBooleanBlock, CudaSignedRadixCiphertext
from .integer import CudaUnsignedRadixCiphertext


def identity_lut_128(glwe_dimension: int, polynomial_size: int, plaintext_modulus: int) -> np.ndarray:
    """The u128 GLWE LUT of the identity over `plaintext_modulus` values with
    delta = 2^127 / plaintext_modulus (one padding bit):
    generate_programmable_bootstrap_glwe_lut on the u128 torus, (k+1)*N x 2 u64."""
    N, p = polynomial_size, plaintext_modulus
    if p < 1 or N % p:
        raise ValueError(f"plaintext modulus {p} must divide the polynomial size {N}")
    delta = (1 << 127) // p
    box, half = N // p, (N // p) // 2
    body = [(i // box) * delta for i in range(N)]
    for j in range(half):
        body[j] = -body[j]
    body = [body[(j + half) % N] & ((1 << 128) - 1) for j in range(N)]
    out = np.zeros(((glwe_dimension + 1) * N, 2), dtype=np.uint64)
    out[glwe_dimension * N:, 0] = [x & (2**64 - 1) for x in body]
    out[glwe_dimension * N:, 1] = [x >> 64 for x in body]
    return out


def _check_squash_shape(polynomial_size, decomp_base_log, decomp_level_count, message_modulus, carry_modulus):
    if message_modulus < 1 or carry_modulus < 1:
        raise ValueError("moduli must be positive")
    if message_modulus > carry_modulus:
        raise ValueError(f"message modulus {message_modulus} > carry modulus {carry_modulus}: "
                         "pairs of blocks cannot be packed")
    if not (256 <= polynomial_size <= 4096 and polynomial_size & (polynomial_size - 1) == 0):
        raise ValueError(f"polynomial size {polynomial_size} is not a power of two in [256, 4096]")
    if decomp_level_count < 1 or decomp_base_log < 1 or decomp_base_log * decomp_level_count > 128:
        raise ValueError("unsupported decomposition")


@dataclass
class CudaNoiseSquashingKey:
    """The 128-bit bootstrap key in the engine's double-double Fourier layout,
    the identity LUT (uploaded once) and the moduli it squashes for.
    grouping_factor is 1 for a classic key, g for a multi-bit one."""

    d_bsk: gpu.CudaVec  # n*(k+1)^2*l*N*2 f64 words (classic), (n/g)*2^g*(k+1)^2*l*N*2 (multi-bit)
    d_lut: gpu.CudaVec  # (k+1)*N u128 words
    input_lwe_dimension: int
    glwe_dimension: int
    polynomial_size: int
    decomp_base_log: int
    decomp_level_count: int
    message_modulus: int
    carry_modulus: int
    centered: bool
    streams: gpu.CudaStreams
    grouping_factor: int = 1

    @property
    def output_lwe_dimension(self) -> int:
        return self.glwe_dimension * self.polynomial_size

    @classmethod
    def from_bootstrap_key_128(cls, h_bsk: np.ndarray, input_lwe_dimension: int, glwe_dimension: int,
                               polynomial_size: int, decomp_base_log: int, decomp_level_count: int,
                               message_modulus: int, carry_modulus: int, centered: bool,
                               streams: gpu.CudaStreams) -> "CudaNoiseSquashingKey":
        """h_bsk: standard-domain u128 key [i][level][row][col][N], (..., 2) u64."""
        k1 = glwe_dimension + 1
        words = input_lwe_dimension * k1 * k1 * decomp_level_count * polynomial_size
        h_bsk = np.ascontiguousarray(h_bsk, dtype=np.uint64).reshape(-1)
        if h_bsk.size != 2 * words:
            raise ValueError(f"128-bit bootstrap key has {h_bsk.size // 2} words, its parameters need {words}")
        _check_squash_shape(polynomial_size, decomp_base_log, decomp_level_count, message_modulus, carry_modulus)
        d_bsk = gpu.CudaVec.new(2 * words, streams, np_dtype=np.float64)
        _lib.lib().cuda_convert_lwe_programmable_bootstrap_key_128_async(
            streams.ptr(0), streams.gpu_indexes[0], d_bsk.as_c_ptr(), h_bsk.ctypes.data, input_lwe_dimension,
            glwe_dimension, decomp_level_count, polynomial_size)
        lut = identity_lut_128(glwe_dimension, polynomial_size, message_modulus * carry_modulus)
        d_lut = gpu.CudaVec.from_cpu_async(lut.reshape(-1), streams)
        streams.synchronize_one(0)  # h_bsk may be freed by the caller
        return cls(d_bsk, d_lut, input_lwe_dimension, glwe_dimension, polynomial_size, decomp_base_log,
                   decomp_level_count, message_modulus, carry_modulus, centered, streams)

    @classmethod
    def from_multi_bit_bootstrap_key_128(cls, h_bsk: np.ndarray, input_lwe_dimension: int, glwe_dimension: int,
                                         polynomial_size: int, decomp_base_log: int, decomp_level_count: int,
                                         grouping_factor: int, message_modulus: int, carry_modulus: int,
                                         streams: gpu.CudaStreams) -> "CudaNoiseSquashingKey":
        """h_bsk: standard-domain u128 multi-bit key [group][2^g][level][row][col][N], (..., 2) u64
        (tfhe-rs' LweMultiBitBootstrapKey layout).  The body's modulus switch is the plain one."""
        g = grouping_factor
        if g not in (2, 3, 4):
            raise ValueError(f"grouping factor {g} is not 2, 3 or 4")
        if input_lwe_dimension < g or input_lwe_dimension % g:
            raise ValueError(f"input LWE dimension {input_lwe_dimension} is not a multiple of the grouping factor {g}")
        _check_squash_shape(polynomial_size, decomp_base_log, decomp_level_count, message_modulus, carry_modulus)
        k1 = glwe_dimension + 1
        words = (input_lwe_dimension // g << g) * k1 * k1 * decomp_level_count * polynomial_size
        h_bsk = np.ascontiguousarray(h_bsk, dtype=np.uint64).reshape(-1)
        if h_bsk.size != 2 * words:
            raise ValueError(f"multi-bit 128-bit bootstrap key has {h_bsk.size // 2} words, its parameters need "
                             f"{words}")
        d_bsk = gpu.CudaVec.new(2 * words, streams, np_dtype=np.float64)
        _lib.lib().cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async(
            streams.ptr(0), streams.gpu_indexes[0], d_bsk.as_c_ptr(), h_bsk.ctypes.data, input_lwe_dimension,
            glwe_dimension, decomp_level_count, polynomial_size, g)
        lut = identity_lut_128(glwe_dimension, polynomial_size, message_modulus * carry_modulus)
        d_lut = gpu.CudaVec.from_cpu_async(lut.reshape(-1), streams)
        streams.synchronize_one(0)  # h_bsk may be freed by the caller
        return cls(d_bsk, d_lut, input_lwe_dimension, glwe_dimension, polynomial_size, decomp_base_log,
                   decomp_level_count, message_modulus, carry_modulus, False, streams, g)

    def squash_radix_ciphertext_noise(self, server_key, ct) -> "CudaSquashedNoiseRadixCiphertext":
        return squash_radix_ciphertext_noise(self, server_key, ct)


@dataclass
class CudaSquashedNoiseRadixCiphertext:
    """ceil(original_block_count / 2) packed u128 LWEs on the device."""

    d_vec: gpu.CudaVec  # packed x (k*N + 1) u128 words
    original_block_count: int
    kind: str  # "unsigned", "signed" or "boolean"
    lwe_dimension: int
    message_modulus: int
    carry_modulus: int
    streams: gpu.CudaStreams

    @property
    def packed_block_count(self) -> int:
        return (self.original_block_count + 1) // 2

    def to_host(self) -> np.ndarray:
        """(packed, lwe_dimension + 1, 2) u64: the u128 LWEs, low word first."""
        return self.d_vec.to_cpu(self.streams).reshape(self.packed_block_count, self.lwe_dimension + 1, 2)


def squash_radix_ciphertext_noise(key: CudaNoiseSquashingKey, server_key,
                                  ct) -> CudaSquashedNoiseRadixCiphertext:
    """Squash the noise of an unsigned or signed radix ciphertext or a boolean
    block with one b200_apply_noise_squashing_64_async call
    (b200_apply_noise_squashing_multi_bit_64_async for a multi-bit key).  `server_key`
    (server_key.CudaServerKey) provides the keyswitch key to the small key."""
    kinds = {CudaUnsignedRadixCiphertext: "unsigned", CudaSignedRadixCiphertext: "signed",
             CudaBooleanBlock: "boolean"}
    kind = kinds.get(type(ct))
    if kind is None:
        raise ValueError(f"cannot squash a {type(ct).__name__}")
    ksk = server_key.ksk
    for name in ("message_modulus", "carry_modulus"):
        if getattr(server_key, name) != getattr(key, name):
            raise ValueError(f"{name} differs between the server key ({getattr(server_key, name)}) and the "
                             f"squashing key ({getattr(key, name)})")
    blocks = ct.blocks
    if blocks.dim() != 2 or blocks.shape[0] < 1:
        raise ValueError("a radix ciphertext needs at least one block")
    if blocks.shape[1] != ksk.input_key_lwe_dimension + 1:
        raise ValueError(f"blocks of dimension {blocks.shape[1] - 1} do not match the keyswitch key's input "
                         f"dimension {ksk.input_key_lwe_dimension}")
    if ksk.output_key_lwe_dimension != key.input_lwe_dimension:
        raise ValueError(f"keyswitch output dimension {ksk.output_key_lwe_dimension} does not match the squashing "
                         f"key's input dimension {key.input_lwe_dimension}")
    if blocks.device != key.streams.device(0):
        raise ValueError("the ciphertext is not on the squashing key's GPU")
    num_blocks = int(blocks.shape[0])
    packed = (num_blocks + 1) // 2
    width = key.output_lwe_dimension + 1
    st = key.streams
    blocks = blocks.contiguous()
    out = gpu.CudaVec.new(2 * packed * width, st)
    L = _lib.lib()
    gi, sp = st.gpu_indexes[0], st.ptr(0)
    buf = C.POINTER(C.c_int8)()
    if key.grouping_factor > 1:
        L.scratch_cuda_multi_bit_programmable_bootstrap_128_async(sp, gi, C.byref(buf), key.glwe_dimension,
                                                                  key.polynomial_size, key.decomp_level_count,
                                                                  packed, True)
        torch.cuda.current_stream(st.device(0)).synchronize()  # blocks written on other streams
        L.b200_apply_noise_squashing_multi_bit_64_async(
            sp, gi, out.as_c_ptr(), blocks.data_ptr(), num_blocks, ksk.input_key_lwe_dimension, key.message_modulus,
            ksk.d_vec.as_c_ptr(), ksk.decomp_base_log, ksk.decomp_level_count, key.d_lut.as_c_ptr(),
            key.d_bsk.as_c_ptr(), buf, key.input_lwe_dimension, key.glwe_dimension, key.polynomial_size,
            key.grouping_factor, key.decomp_base_log, key.decomp_level_count)
        L.cleanup_cuda_multi_bit_programmable_bootstrap_128(sp, gi, C.byref(buf))
    else:
        L.scratch_cuda_programmable_bootstrap_128_async(sp, gi, C.byref(buf), key.input_lwe_dimension,
                                                         key.glwe_dimension, key.polynomial_size,
                                                         key.decomp_level_count, packed, True,
                                                         1 if key.centered else 0)
        torch.cuda.current_stream(st.device(0)).synchronize()  # blocks written on other streams
        L.b200_apply_noise_squashing_64_async(
            sp, gi, out.as_c_ptr(), blocks.data_ptr(), num_blocks, ksk.input_key_lwe_dimension, key.message_modulus,
            ksk.d_vec.as_c_ptr(), ksk.decomp_base_log, ksk.decomp_level_count, key.d_lut.as_c_ptr(),
            key.d_bsk.as_c_ptr(), buf, key.input_lwe_dimension, key.glwe_dimension, key.polynomial_size,
            key.decomp_base_log, key.decomp_level_count)
        L.cleanup_cuda_programmable_bootstrap_128(sp, gi, C.byref(buf))
    return CudaSquashedNoiseRadixCiphertext(out, num_blocks, kind, key.output_lwe_dimension, key.message_modulus,
                                            key.carry_modulus, st)
