"""Homomorphic Trivium and Kreyvium on encrypted bits, and the keystream
applied to a clear stream ciphertext: the server side of transciphering, the
GPU twin of tfhe-rs' `CudaServerKey::{trivium_generate_keystream,
trivium_init, trivium_next, kreyvium_generate_keystream, kreyvium_init,
kreyvium_next}` and `transciphering::apply_keystream`.

Inputs are shortint blocks of a 2_2 parameter set holding one bit each.  A
key or IV is one block per bit in tfhe-rs' order: block i is bit i % 8 of byte
i // 8 (LSB first).  Registers are indexed by age, block 0 the newest bit:

  * Trivium (80-bit key and IV): a[i] = key[79 - i], b[i] = iv[79 - i],
    c[108..110] = 1 (`TriviumRef` of tfhe-rs' tests);
  * Kreyvium (128-bit key and IV): a[i] = key[127 - i], b[i] = iv[127 - i],
    c[i] = iv[43 - i] for i < 44, ones at c[44..109]; round t also reads
    K*[t] = key[127 - t % 128] into t3 and IV*[t] = iv[127 - t % 128] into the
    AND feeding b (tfhe-rs' `transciphering::ciphers::kreyvium`).

Both run 18 * 64 warm-up rounds; keystream bit j is the output of round j
after them.  A round is one bit-circuit step (`bit_circuit`): t1, t2, t3 and
the keystream bit are XOR forms, and each new state bit is a refresh point
(`mat`), one parity PBS over at most 5 level-1 atoms fed by one AND PBS.
K* and IV* are a renaming: the 128-bit rotating registers are the caller's
key and IV blocks read at a rotation offset, never bootstrapped.

`next` outputs only the keystream and the new state bits; the host shifts the
registers by tensor slicing.  A state bit passed through unchanged costs no
PBS (the compiler would refresh every input it outputs).

`num_inputs` independent (key, IV) pairs run bit-sliced, as instances of one
schedule, concatenated instance-major in every input, state and output.

`apply_keystream` XORs encrypted keystream bits with clear stream-ciphertext
bits and packs them two per block: block j = (k[2j] ^ i[2j]) + 2 (k[2j+1] ^
i[2j+1]), one PBS on k0 + 2 k1 + 4 i0 + 8 i1 (noise level 3, the clear bits
in the body), one instance per block."""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

from . import bit_circuit as bc

WARMUP = 18 * 64
A_BITS, B_BITS, C_BITS = 93, 84, 111
KEY_BITS = {"trivium": 80, "kreyvium": 128}
ROTATION = 128                    # length of Kreyvium's K* and IV* registers
MAX_COUNTER = (1 << 64) - 1       # keystream position, a u64 in tfhe-rs
CIRCUIT_CACHE_SIZE = 16           # compiled (kind, num_steps) circuits kept

# block = (k0 ^ i0) + 2 (k1 ^ i1) of the linear step k0 + 2 k1 + 4 i0 + 8 i1
XOR_PACK_LUT = [((x & 1) ^ ((x >> 2) & 1)) | ((((x >> 1) & 1) ^ ((x >> 3) & 1)) << 1)
                for x in range(bc.TOTAL_MOD)]


# ---------------------------------------------------------------------------
# circuits
# ---------------------------------------------------------------------------
def _load(c: bc.Circuit, cipher: str, key: Sequence[int], iv: Sequence[int]):
    """registers a, b, c (index 0 newest) loaded from the key and IV wires"""
    zero, one = c.const(0), c.const(1)
    if cipher == "trivium":
        a = [key[79 - i] for i in range(80)] + [zero] * (A_BITS - 80)
        b = [iv[79 - i] for i in range(80)] + [zero] * (B_BITS - 80)
        r = [zero] * (C_BITS - 3) + [one] * 3
    else:
        a = [key[127 - i] for i in range(A_BITS)]
        b = [iv[127 - i] for i in range(B_BITS)]
        r = [iv[43 - i] for i in range(44)] + [one] * 66 + [zero]
    return a, b, r


def rounds(c: bc.Circuit, a, b, r, steps: int, out_from: int = 0, key=None, iv=None):
    """`steps` rounds on registers a, b, r (lists of wires, index 0 newest).
    Kreyvium passes its key and IV wires at rotation 0: round t reads
    key[127 - t % 128] and iv[127 - t % 128].  Returns the keystream bits of
    the rounds >= out_from, and the registers after the last round."""
    z = []
    for t in range(steps):
        t1 = c.xor(a[65], a[92])
        t2 = c.xor(b[68], b[83])
        t3 = c.xor(r[65], r[110])
        a_and = c.and_(a[90], a[91])
        if key is not None:
            t3 = c.xor(t3, key[127 - t % ROTATION])
            a_and = c.xor(a_and, iv[127 - t % ROTATION])
        if t >= out_from:
            z.append(c.xor(c.xor(t1, t2), t3))
        na = c.mat(c.xor(c.xor(t3, a[68]), c.and_(r[108], r[109])))
        nb = c.mat(c.xor(c.xor(t1, b[77]), a_and))
        nc = c.mat(c.xor(c.xor(t2, r[86]), c.and_(b[81], b[82])))
        a, b, r = [na] + a[:-1], [nb] + b[:-1], [nc] + r[:-1]
    return z, a, b, r


def new_bits(num_steps: int) -> Tuple[int, int, int]:
    """state bits of a, b, c that `num_steps` rounds replace"""
    return min(num_steps, A_BITS), min(num_steps, B_BITS), min(num_steps, C_BITS)


@functools.lru_cache(maxsize=CIRCUIT_CACHE_SIZE)
def circuit(kind: str, num_steps: int = 0) -> bc.Circuit:
    """Per-instance inputs and outputs, cipher = 'trivium' or 'kreyvium':
      '<cipher>_keystream': key, iv -> num_steps keystream bits after the
          warm-up (warm-up and output compiled as one circuit);
      '<cipher>_init': key, iv -> a, b, c after the warm-up;
      '<cipher>_next': a, b, c (Kreyvium: then key and iv rotated to the
          state's offset) -> num_steps keystream bits, then the new bits of
          a, b and c (`new_bits`, newest first);
      'apply_keystream': k0, k1 and the clear bits i0, i1 (per-instance
          constants) -> one block (k0 ^ i0) + 2 (k1 ^ i1).
    The schedule of each circuit is compiled once (`bit_circuit.schedule`);
    the CIRCUIT_CACHE_SIZE most recent (kind, num_steps) are kept."""
    c = bc.Circuit(f"{kind}_{num_steps}" if num_steps else kind)
    if kind == "apply_keystream":
        k0, k1 = c.inputs(2, shared=False)
        i0, i1 = c.iconst(), c.iconst()
        c.output_blocks([c.lut([(k0, 1), (k1, 2), (i0, 4), (i1, 8)], 0, c.add_lut(XOR_PACK_LUT))])
        return c
    cipher, _, op = kind.partition("_")
    if cipher not in KEY_BITS or op not in ("keystream", "init", "next"):
        raise ValueError(f"unknown stream cipher circuit {kind!r}")
    if op != "init" and num_steps < 1:
        raise ValueError(f"{kind}: num_steps must be >= 1")
    kb = KEY_BITS[cipher]
    if op == "next":
        a, b, r = c.inputs(A_BITS, False), c.inputs(B_BITS, False), c.inputs(C_BITS, False)
        key = iv = None
        if cipher == "kreyvium":
            key, iv = c.inputs(kb, False), c.inputs(kb, False)
        z, a, b, r = rounds(c, a, b, r, num_steps, 0, key, iv)
        ma, mb, mc = new_bits(num_steps)
        c.output(z + a[:ma] + b[:mb] + r[:mc])
        return c
    key, iv = c.inputs(kb, False), c.inputs(kb, False)
    a, b, r = _load(c, cipher, key, iv)
    kiv = (key, iv) if cipher == "kreyvium" else (None, None)
    if op == "keystream":
        z, _, _, _ = rounds(c, a, b, r, WARMUP + num_steps, WARMUP, *kiv)
        c.output(z)
    else:
        _, a, b, r = rounds(c, a, b, r, WARMUP, WARMUP, *kiv)
        c.output(a + b + r)
    return c


def stream_bits(stream_bytes, n_bits: int) -> np.ndarray:
    """the first n_bits bits of `stream_bytes`, LSB first within each byte"""
    data = np.frombuffer(bytes(stream_bytes), dtype=np.uint8)
    return np.unpackbits(data, bitorder="little")[:n_bits].astype(np.int64)


def apply_keystream_iconsts(stream_bytes, n_bits: int) -> np.ndarray:
    """per-instance constants of the 'apply_keystream' circuit: [blocks, 2]
    clear bits (i0, i1), a missing odd last bit 0"""
    bits = stream_bits(stream_bytes, n_bits)
    if n_bits % 2:
        bits = np.append(bits, 0)
    return bits.reshape(-1, 2)


def _check_steps(num_steps) -> int:
    if isinstance(num_steps, bool) or not isinstance(num_steps, (int, np.integer)) or num_steps < 1:
        raise ValueError(f"num_steps must be an integer >= 1, got {num_steps!r}")
    return int(num_steps)


def _check_stream(stream_bytes, n_bits) -> bytes:
    if isinstance(n_bits, bool) or not isinstance(n_bits, (int, np.integer)) or n_bits < 1:
        raise ValueError(f"n_bits must be an integer >= 1, got {n_bits!r}")
    data = bytes(stream_bytes)
    if len(data) != (int(n_bits) + 7) // 8:
        raise ValueError(f"a stream of {n_bits} bits has {(int(n_bits) + 7) // 8} bytes, got {len(data)}")
    return data


# ---------------------------------------------------------------------------
# sessions
# ---------------------------------------------------------------------------
@dataclass(frozen=True)
class StreamCiphertext:
    """A clear stream-cipher ciphertext (tfhe-rs `StreamCiphertext`): `n_bits`
    message bits XORed with the keystream from bit `encryption_counter` on,
    packed LSB first into ceil(n_bits / 8) bytes."""
    kind: str
    encryption_counter: int
    n_bits: int
    bytes: bytes


class CudaTriviumState:
    """Trivium registers of `num_inputs` instances: a (93), b (84) and c (111)
    blocks per instance, index 0 the newest bit, instance-major.  `counter`
    is the keystream bits produced since the warm-up."""
    kind = "trivium"

    def __init__(self, a, b, c, num_inputs: int, counter: int = 0):
        self.a, self.b, self.c = a, b, c
        self.num_inputs = num_inputs
        self.counter = counter


class CudaKreyviumState(CudaTriviumState):
    """Kreyvium registers, plus the caller's key and IV blocks (copied at
    init) that K* and IV* read at rotation `offset`: the rounds run since the
    warm-up, mod 128 (the 1152 warm-up rounds are a multiple of 128)."""
    kind = "kreyvium"

    def __init__(self, a, b, c, key, iv, num_inputs: int, counter: int = 0, offset: int = 0):
        super().__init__(a, b, c, num_inputs, counter)
        self.key, self.iv = key, iv
        self.offset = offset


class CudaTriviumServerKey:
    """Trivium and Kreyvium on a `server_key.CudaServerKey` (classic or
    multi-bit, 2_2 blocks); ciphertexts are `integer.CudaUnsignedRadixCiphertext`
    of one bit per block (or tensors of blocks).  Streams, chunking and input
    lifetimes are those of `CudaAesServerKey`: the work runs on the server
    key's first stream after the caller's current stream, instances run in
    chunks that fit in free device memory, inputs may be dropped as soon as a
    call returns, and the caller's stream waits for the result."""

    def __init__(self, server_key):
        from . import bit_circuit_gpu

        self.skey = server_key
        self.runner = bit_circuit_gpu.CudaBitCircuitRunner(server_key)

    # -- helpers -------------------------------------------------------------
    @staticmethod
    def _blocks(ct, count: int, what: str):
        blocks = ct.blocks if hasattr(ct, "blocks") else ct
        if blocks.shape[0] != count:
            raise ValueError(f"{what}: expected {count} blocks, got {blocks.shape[0]}")
        return blocks

    @staticmethod
    def _num_inputs(num_inputs) -> int:
        if isinstance(num_inputs, bool) or not isinstance(num_inputs, (int, np.integer)) or num_inputs < 1:
            raise ValueError(f"num_inputs must be an integer >= 1, got {num_inputs!r}")
        return int(num_inputs)

    def _key_iv(self, cipher, key, iv, num_inputs):
        import torch

        I = self._num_inputs(num_inputs)
        kb = KEY_BITS[cipher]
        key = self._blocks(key, kb * I, f"{cipher} key")
        iv = self._blocks(iv, kb * I, f"{cipher} iv")
        W = key.shape[1]
        return I, W, torch.cat([key.reshape(I, kb, W), iv.reshape(I, kb, W)], 1).reshape(-1, W), key, iv

    def _run(self, kind, num_steps, instance, num_inputs):
        return self.runner.run(circuit(kind, num_steps), None, instance, None, num_inputs)

    @staticmethod
    def _radix(t):
        from .integer import CudaUnsignedRadixCiphertext

        return CudaUnsignedRadixCiphertext(t)

    # -- generic over the two ciphers ----------------------------------------
    def _generate_keystream(self, cipher, key, iv, num_steps, num_inputs):
        n = _check_steps(num_steps)
        I, _, inst, _, _ = self._key_iv(cipher, key, iv, num_inputs)
        return self._radix(self._run(f"{cipher}_keystream", n, inst, I))

    def _init(self, cipher, key, iv, num_inputs):
        I, W, inst, key, iv = self._key_iv(cipher, key, iv, num_inputs)
        out = self._run(f"{cipher}_init", 0, inst, I).view(I, A_BITS + B_BITS + C_BITS, W)
        a = self._radix(out[:, :A_BITS].reshape(-1, W))
        b = self._radix(out[:, A_BITS:A_BITS + B_BITS].reshape(-1, W))
        c = self._radix(out[:, A_BITS + B_BITS:].reshape(-1, W))
        if cipher == "trivium":
            return CudaTriviumState(a, b, c, I)
        # the state owns its copy: the caller may drop or reuse its key and IV
        return CudaKreyviumState(a, b, c, self._radix(key.clone()), self._radix(iv.clone()), I)

    def _next(self, cipher, state, num_steps):
        import torch

        expected = CudaKreyviumState if cipher == "kreyvium" else CudaTriviumState
        if type(state) is not expected:
            raise ValueError(f"{cipher}_next: expected a {expected.__name__}, got {type(state).__name__}")
        n = _check_steps(num_steps)
        if state.counter + n > MAX_COUNTER:
            raise ValueError(f"{cipher}: the keystream ends at bit 2^64 - 1; the state is at {state.counter}")
        I = state.num_inputs
        regs = [self._blocks(r, L * I, f"{cipher} state") for r, L in
                ((state.a, A_BITS), (state.b, B_BITS), (state.c, C_BITS))]
        W = regs[0].shape[1]
        regs = [r.reshape(I, -1, W) for r in regs]
        parts = list(regs)
        if cipher == "kreyvium":
            # K*/IV* at rotation `offset`: input m is key[(m - offset) % 128]
            for t in (state.key, state.iv):
                parts.append(torch.roll(self._blocks(t, ROTATION * I, "kreyvium state").reshape(I, ROTATION, W),
                                        state.offset, 1))
        out = self._run(f"{cipher}_next", n, torch.cat(parts, 1).reshape(-1, W), I).view(I, -1, W)
        o = n
        new = []
        for r, m in zip(regs, new_bits(n)):
            new.append(self._radix(torch.cat([out[:, o:o + m], r[:, :r.shape[1] - m]], 1).reshape(-1, W)))
            o += m
        state.a, state.b, state.c = new
        state.counter += n
        if cipher == "kreyvium":
            state.offset = (state.offset + n) % ROTATION
        return self._radix(out[:, :n].reshape(-1, W))

    # -- Trivium ---------------------------------------------------------------
    def trivium_generate_keystream(self, key, iv, num_steps: int, num_inputs: int = 1):
        """num_steps keystream bits per (key, IV) pair after the warm-up,
        warm-up and output in one schedule: num_inputs * num_steps blocks."""
        return self._generate_keystream("trivium", key, iv, num_steps, num_inputs)

    def trivium_init(self, key, iv, num_inputs: int = 1) -> CudaTriviumState:
        """The state after the warm-up: keys and IVs of 80 blocks per input."""
        return self._init("trivium", key, iv, num_inputs)

    def trivium_next(self, state: CudaTriviumState, num_steps: int):
        """The next num_steps keystream bits of every input (num_inputs *
        num_steps blocks); advances `state`."""
        return self._next("trivium", state, num_steps)

    # -- Kreyvium --------------------------------------------------------------
    def kreyvium_generate_keystream(self, key, iv, num_steps: int, num_inputs: int = 1):
        return self._generate_keystream("kreyvium", key, iv, num_steps, num_inputs)

    def kreyvium_init(self, key, iv, num_inputs: int = 1) -> CudaKreyviumState:
        """The state after the warm-up: keys and IVs of 128 blocks per input."""
        return self._init("kreyvium", key, iv, num_inputs)

    def kreyvium_next(self, state: CudaKreyviumState, num_steps: int):
        return self._next("kreyvium", state, num_steps)

    # -- transciphering ----------------------------------------------------------
    def transcipher(self, state, stream_ciphertext: StreamCiphertext):
        """The stream ciphertext as ceil(n_bits / 2) blocks of two message
        bits (`apply_keystream`), from the next n_bits keystream bits of a
        one-input state.  Like tfhe-rs' `check_transcipher_input`, the
        ciphertext's kind must be the state's and its encryption counter the
        state's counter; nothing runs otherwise."""
        sc = stream_ciphertext
        if not isinstance(state, CudaTriviumState):
            raise ValueError(f"transcipher: expected a Trivium or Kreyvium state, got {type(state).__name__}")
        if sc.kind != state.kind:
            raise ValueError(f"stream ciphertext kind mismatch: session {state.kind!r}, ciphertext {sc.kind!r}")
        if sc.encryption_counter != state.counter:
            raise ValueError(f"stream ciphertext counter mismatch: session at {state.counter}, ciphertext at "
                             f"{sc.encryption_counter}")
        if state.num_inputs != 1:
            raise ValueError(f"transcipher: the state holds {state.num_inputs} streams, not one")
        _check_stream(sc.bytes, sc.n_bits)
        keystream = self._next(state.kind, state, sc.n_bits)
        return apply_keystream(self, keystream, sc.bytes, sc.n_bits)


def apply_keystream(server_key, keystream_bits, stream_bytes, n_bits: int):
    """tfhe-rs `apply_keystream` for 2_2 blocks: n_bits encrypted keystream
    bits (one per block: Trivium, Kreyvium or `aes_ctr` output) XORed with the
    clear bits of `stream_bytes` (ceil(n_bits / 8) bytes, LSB first) and
    packed into ceil(n_bits / 2) blocks, block j = (k[2j] ^ i[2j]) +
    2 (k[2j+1] ^ i[2j+1]); an odd last block holds one bit.  One PBS per
    block.  `server_key` is a `CudaTriviumServerKey` or `CudaAesServerKey`
    (whose bit-circuit runner does the work)."""
    import torch

    data = _check_stream(stream_bytes, n_bits)
    n_bits = int(n_bits)
    blocks = CudaTriviumServerKey._blocks(keystream_bits, n_bits, "apply_keystream keystream")
    num_blocks = (n_bits + 1) // 2
    if n_bits % 2:  # k1 of the last block: a trivial encryption of 0
        blocks = torch.cat([blocks, torch.zeros((1, blocks.shape[1]), dtype=blocks.dtype, device=blocks.device)])
    out = server_key.runner.run(circuit("apply_keystream"), None, blocks, apply_keystream_iconsts(data, n_bits),
                                num_blocks)
    return CudaTriviumServerKey._radix(out)
