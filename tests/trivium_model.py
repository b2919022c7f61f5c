"""Plain Trivium and Kreyvium, and the client side of transciphering with them
(tests only: the package has no client key).

Conventions are tfhe-rs': a key or IV is a list of bits, bit i being bit i % 8
of byte i // 8 (LSB first), and it is encrypted one bit per 2_2 block in that
order.  Registers are indexed by age, index 0 the newest bit.  Trivium loads
a[i] = key[79 - i], b[i] = iv[79 - i], c[108..110] = 1; Kreyvium loads
a[i] = key[127 - i], b[i] = iv[127 - i], c[i] = iv[43 - i] for i < 44, ones at
c[44..109], and reads key[127 - t % 128] and iv[127 - t % 128] in round t.
Both run 18 * 64 warm-up rounds; keystream bit j is output round j after it."""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

WARMUP = 18 * 64


def bits_lsb_first(data: bytes, n_bits: int = None) -> List[int]:
    n_bits = 8 * len(data) if n_bits is None else n_bits
    return [(data[i // 8] >> (i % 8)) & 1 for i in range(n_bits)]


def pack_lsb_first(bits: Sequence[int]) -> bytes:
    out = bytearray((len(bits) + 7) // 8)
    for i, b in enumerate(bits):
        out[i // 8] |= (int(b) & 1) << (i % 8)
    return bytes(out)


class Trivium:
    def __init__(self, key: Sequence[int], iv: Sequence[int]):
        assert len(key) == len(iv) == 80
        self.a = [int(key[79 - i]) if i < 80 else 0 for i in range(93)]
        self.b = [int(iv[79 - i]) if i < 80 else 0 for i in range(84)]
        self.c = [1 if i >= 108 else 0 for i in range(111)]
        self.t = 0  # rounds run, warm-up included
        for _ in range(WARMUP):
            self.step()

    def taps(self):
        return 0, 0

    def step(self) -> int:
        a, b, c = self.a, self.b, self.c
        k, v = self.taps()
        t1 = a[65] ^ a[92]
        t2 = b[68] ^ b[83]
        t3 = c[65] ^ c[110] ^ k
        z = t1 ^ t2 ^ t3
        na = t3 ^ a[68] ^ (c[108] & c[109])
        nb = t1 ^ b[77] ^ (a[90] & a[91]) ^ v
        nc = t2 ^ c[86] ^ (b[81] & b[82])
        self.a, self.b, self.c = [na] + a[:-1], [nb] + b[:-1], [nc] + c[:-1]
        self.t += 1
        return z

    def keystream(self, n: int) -> List[int]:
        return [self.step() for _ in range(n)]

    @property
    def counter(self) -> int:
        return self.t - WARMUP


class Kreyvium(Trivium):
    def __init__(self, key: Sequence[int], iv: Sequence[int]):
        assert len(key) == len(iv) == 128
        self.key, self.iv = [int(x) for x in key], [int(x) for x in iv]
        self.a = [self.key[127 - i] for i in range(93)]
        self.b = [self.iv[127 - i] for i in range(84)]
        self.c = [self.iv[43 - i] if i < 44 else (1 if i < 110 else 0) for i in range(111)]
        self.t = 0
        for _ in range(WARMUP):
            self.step()

    def taps(self):
        return self.key[127 - self.t % 128], self.iv[127 - self.t % 128]


def encrypt_bits(oracle, keys, rng, bits) -> np.ndarray:
    """one shortint block per bit: message in {0, 1} at delta = 2^63 / 16"""
    P = keys.params
    return oracle.lwe_encrypt_batch(rng, keys.glwe_sk, np.asarray(bits, dtype=np.uint64) * np.uint64(P.delta),
                                    P.lwe_noise_log2)


def decrypt_messages(oracle, keys, blocks, vmax: int = 1) -> np.ndarray:
    """decrypt every block, checking that each holds a value up to `vmax`"""
    P = keys.params
    d = oracle.decode(oracle.lwe_decrypt_batch(keys.glwe_sk, np.asarray(blocks)), P.delta, 16)
    assert all(int(x) <= vmax for x in d), d
    return d.astype(np.int64)


def blocks_to_bits(values: Sequence[int], n_bits: int) -> List[int]:
    """2_2 blocks of apply_keystream (block j = bit 2j + 2 * bit 2j+1) -> bits"""
    out = []
    for v in values:
        out += [int(v) & 1, (int(v) >> 1) & 1]
    assert all(b == 0 for b in out[n_bits:])
    return out[:n_bits]
