"""Plain model of the bitonic shuffle on Python integers: the network, the
swap rule with its tie asymmetry, the padding and the key-size rule of
tfhe-rs (tfhe/src/integer/server_key/radix_parallel/bitonic_shuffle.rs),
written independently of `tfhe-rs_b200/radix_shuffle.py`."""
import math


def network(n):
    """bitonic_network(n): stages of (i, j, ascending)"""
    assert n >= 2 and n & (n - 1) == 0
    log_n = n.bit_length() - 1
    out = []
    for phase in range(log_n):
        for step in reversed(range(phase + 1)):
            out.append([(i, i ^ (1 << step), (i >> (phase + 1)) & 1 == 0)
                        for i in range(n) if (i ^ (1 << step)) > i])
    return out


# the reference's own unit test (bitonic_network_builds_expected_pairs_for_n8)
NETWORK_8 = [
    [(0, 1, True), (2, 3, False), (4, 5, True), (6, 7, False)],
    [(0, 2, True), (1, 3, True), (4, 6, False), (5, 7, False)],
    [(0, 1, True), (2, 3, True), (4, 5, False), (6, 7, False)],
    [(0, 4, True), (1, 5, True), (2, 6, True), (3, 7, True)],
    [(0, 2, True), (1, 3, True), (4, 6, True), (5, 7, True)],
    [(0, 1, True), (2, 3, True), (4, 5, True), (6, 7, True)],
]


def shuffle(data, keys, key_blocks):
    """unchecked_bitonic_shuffle_with_keys on integers: keys of `key_blocks`
    2-bit blocks; returns the shuffled data"""
    assert len(data) == len(keys)
    n = len(data)
    if n <= 1:
        return list(data)
    data, keys = list(data), list(keys)
    padded = 1 << (n - 1).bit_length()
    if padded > n:
        # an extra zero block on every key (values unchanged), padding keys of
        # all digits 3 over key_blocks + 1 blocks
        keys += [4 ** (key_blocks + 1) - 1] * (padded - n)
        data += [0] * (padded - n)
    for stage in network(padded):
        for i, j, asc in stage:
            swap = keys[i] > keys[j] if asc else keys[i] <= keys[j]
            if swap:
                keys[i], keys[j] = keys[j], keys[i]
                data[i], data[j] = data[j], data[i]
    return data[:n]


def key_blocks_for_probability(length, p):
    """num_blocks_of_keys(CollisionProbability(p)) at 2-bit blocks: Rust's
    `as u32` saturates -inf and negatives to 0"""
    assert 0 < p < 1
    x = (length * length) / (2.0 * p)
    bits = 0 if x == 0 else max(0, math.ceil(math.log2(x)))
    return (bits + 1) // 2


def key_blocks_for_bits(bits):
    return (bits + 1) // 2
