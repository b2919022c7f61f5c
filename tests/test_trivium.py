"""Homomorphic Trivium and Kreyvium, and the keystream applied into 2_2 blocks
(tfhe-rs_b200/trivium.py).

CPU: the plain models against tfhe-rs' known-answer vectors
(tests/golden/trivium_vectors_v1.json); `CudaTriviumServerKey`'s host code on
a cleartext runner (the compiled schedules on `bit_circuit.run_cleartext`,
which asserts the noise budget on every row, with blocks holding plain
messages): fused keystreams against init + next, several instances, Kreyvium's
rotation offset, apply_keystream and transcipher; the pinned schedule counts;
the argument checks; the compiler's circuit-local LUTs and block outputs; one
Trivium keystream and one apply_keystream through real LWE keyswitches and
PBS on the oracle.

GPU: `CudaTriviumServerKey` on classic P22 and multi-bit g = 4: every output
block decrypts to the plain model's."""
import json
import os
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import aes, bit_circuit as bc, trivium as T

from tests import aes_model as AM
from tests import trivium_model as M

VECTORS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "trivium_vectors_v1.json")))


def vector_bits(v, n):
    if "key_hex" in v:
        return M.bits_lsb_first(bytes.fromhex(v["key_hex"])), M.bits_lsb_first(bytes.fromhex(v["iv_hex"]))
    key, iv = [0] * n, [0] * n
    for i in v["key_bits"]:
        key[i] = 1
    for i in v["iv_bits"]:
        iv[i] = 1
    return key, iv


def model(cipher, key, iv):
    return (M.Trivium if cipher == "trivium" else M.Kreyvium)(key, iv)


def test_plain_models_match_tfhe_rs_vectors():
    for v in VECTORS["trivium"]:
        key, iv = vector_bits(v, 80)
        assert M.pack_lsb_first(M.Trivium(key, iv).keystream(512)).hex().upper() == v["keystream_hex"], v["name"]
    for v in VECTORS["kreyvium"]:
        key, iv = vector_bits(v, 128)
        assert M.pack_lsb_first(M.Kreyvium(key, iv).keystream(64)).hex().upper() == v["keystream_hex"], v["name"]


# ---------------------------------------------------------------------------
# the host code on a cleartext runner
# ---------------------------------------------------------------------------
class CleartextRunner:
    """`CudaBitCircuitRunner.run` on the cleartext executor: a block is an
    int64 row [message]; counts the calls."""

    def __init__(self):
        self.calls = 0

    def run(self, circuit, shared, instance, iconsts, num_instances):
        import torch

        self.calls += 1
        s = bc.schedule(circuit, num_instances)
        sh = [] if shared is None else shared[:, 0].numpy()
        ins = None if instance is None else instance[:, 0].numpy().reshape(num_instances, -1)
        return torch.from_numpy(bc.run_cleartext(s, sh, ins, iconsts).reshape(-1, 1).astype(np.int64))


def cleartext_key():
    k = T.CudaTriviumServerKey.__new__(T.CudaTriviumServerKey)
    k.runner = CleartextRunner()
    return k


def blocks(bits):
    import torch

    return torch.tensor(np.asarray(bits, dtype=np.int64).reshape(-1, 1))


def values(ct):
    return [int(x) for x in ct.blocks[:, 0]]


@pytest.mark.parametrize("cipher", ["trivium", "kreyvium"])
def test_vectors_on_the_cleartext_runner(cipher):
    """All vectors as instances of one call, fused and as init + 8 x next(64)."""
    tk = cleartext_key()
    vs = VECTORS[cipher]
    kb = T.KEY_BITS[cipher]
    n = 512 if cipher == "trivium" else 64
    keys, ivs = zip(*[vector_bits(v, kb) for v in vs])
    want = [v["keystream_hex"] for v in vs]
    gen = getattr(tk, f"{cipher}_generate_keystream")(blocks(keys), blocks(ivs), n, len(vs))
    got = np.array(values(gen)).reshape(len(vs), n)
    assert [M.pack_lsb_first(g).hex().upper() for g in got] == want
    st = getattr(tk, f"{cipher}_init")(blocks(keys), blocks(ivs), num_inputs=len(vs))
    parts = [np.array(values(getattr(tk, f"{cipher}_next")(st, 64))).reshape(len(vs), 64) for _ in range(n // 64)]
    assert [M.pack_lsb_first(g).hex().upper() for g in np.concatenate(parts, 1)] == want
    assert st.counter == n


@pytest.mark.parametrize("cipher", ["trivium", "kreyvium"])
def test_fused_equals_init_then_next_of_several_lengths(cipher):
    """num_inputs = 3 with distinct random keys; next lengths that cross the
    64-round batches, a register length and (Kreyvium) the 128-round
    rotation of K* and IV* several times."""
    rng = np.random.default_rng(zlib.crc32(cipher.encode()))
    kb = T.KEY_BITS[cipher]
    keys, ivs = rng.integers(0, 2, (3, kb)), rng.integers(0, 2, (3, kb))
    steps = [1, 63, 100, 130, 7, 129]
    total = sum(steps)
    want = np.array([model(cipher, k, i).keystream(total) for k, i in zip(keys, ivs)])
    tk = cleartext_key()
    fused = np.array(values(getattr(tk, f"{cipher}_generate_keystream")(blocks(keys), blocks(ivs), total, 3)))
    assert np.array_equal(fused.reshape(3, total), want)
    st = getattr(tk, f"{cipher}_init")(blocks(keys), blocks(ivs), 3)
    got, offsets = [], []
    for n in steps:
        got.append(np.array(values(getattr(tk, f"{cipher}_next")(st, n))).reshape(3, n))
        offsets.append(getattr(st, "offset", None))
    assert np.array_equal(np.concatenate(got, 1), want)
    assert st.counter == total
    if cipher == "kreyvium":
        assert offsets == [s % 128 for s in np.cumsum(steps)]
        # the state's registers are the model's
        m = M.Kreyvium(keys[1], ivs[1])
        m.keystream(total)
        assert values(st.a)[93:186] == m.a and values(st.b)[84:168] == m.b and values(st.c)[111:222] == m.c
        assert values(st.key)[128:256] == list(keys[1])


def test_apply_keystream_all_cases_and_odd_lengths():
    tk = cleartext_key()
    # all 16 (k0, k1, i0, i1): block j of the 32-bit stream is case j
    k = [(j >> s) & 1 for j in range(16) for s in (0, 1)]
    i = [(j >> s) & 1 for j in range(16) for s in (2, 3)]
    out = values(T.apply_keystream(tk, blocks(k), M.pack_lsb_first(i), 32))
    assert out == [((j & 1) ^ ((j >> 2) & 1)) + 2 * (((j >> 1) & 1) ^ ((j >> 3) & 1)) for j in range(16)]
    rng = np.random.default_rng(3)
    for n_bits in (1, 2, 3, 13, 64, 101):
        ks = rng.integers(0, 2, n_bits)
        stream = bytes(rng.integers(0, 256, (n_bits + 7) // 8, dtype=np.uint8))
        out = values(T.apply_keystream(tk, blocks(ks), stream, n_bits))
        assert len(out) == (n_bits + 1) // 2 and max(out) <= 3
        assert M.blocks_to_bits(out, n_bits) == [int(a) ^ b for a, b in zip(ks, M.bits_lsb_first(stream, n_bits))]
        if n_bits % 2:
            assert out[-1] <= 1  # the odd last block holds one bit


def test_apply_keystream_on_an_aes_ctr_keystream():
    """aes_ctr's bits (one per block) are a keystream like any other."""
    key, iv = bytes(range(16)), int("f0f1f2f3f4f5f6f7f8f9fafbfcfdfeff", 16)
    s = bc.schedule(aes.circuit("aes_ctr"), 2)
    ks = bc.run_cleartext(s, np.concatenate([AM.key_bits(key), AM.u128_bits(iv)]), None,
                          aes.counter_bits(0, 2)).reshape(-1)
    assert [AM.bits_u128(ks[128 * j:128 * j + 128]) for j in range(2)] == AM.aes_ctr(key, iv, 0, 2)
    msg = bytes(range(100, 132))
    out = values(T.apply_keystream(cleartext_key(), blocks(ks), msg, 256))
    assert M.pack_lsb_first(M.blocks_to_bits(out, 256)) == bytes(
        a ^ b for a, b in zip(msg, M.pack_lsb_first([int(x) for x in ks])))


def stream_ciphertext(cipher, plain, msg: bytes, n_bits=None):
    """client side: the model's next n_bits keystream bits XORed into msg"""
    n_bits = 8 * len(msg) if n_bits is None else n_bits
    counter = plain.counter
    ks = plain.keystream(n_bits)
    bits = [a ^ b for a, b in zip(M.bits_lsb_first(msg, n_bits), ks)]
    return T.StreamCiphertext(cipher, counter, n_bits, M.pack_lsb_first(bits))


@pytest.mark.parametrize("cipher", ["trivium", "kreyvium"])
def test_transcipher_sessions(cipher):
    rng = np.random.default_rng(zlib.crc32(b"transcipher" + cipher.encode()))
    kb = T.KEY_BITS[cipher]
    key, iv = rng.integers(0, 2, kb), rng.integers(0, 2, kb)
    plain = model(cipher, key, iv)
    tk = cleartext_key()
    st = getattr(tk, f"{cipher}_init")(blocks(key), blocks(iv))
    for msg, n_bits in ((int(rng.integers(0, 1 << 63)).to_bytes(8, "little"), None), (bytes(range(37)), 293)):
        sc = stream_ciphertext(cipher, plain, msg, n_bits)
        out = values(tk.transcipher(st, sc))
        assert M.blocks_to_bits(out, sc.n_bits) == M.bits_lsb_first(msg, sc.n_bits)
    assert st.counter == 64 + 293
    # tfhe-rs' check_transcipher_input: kind and counter; nothing runs, the state stays
    calls = tk.runner.calls
    other = "kreyvium" if cipher == "trivium" else "trivium"
    with pytest.raises(ValueError, match="kind"):
        tk.transcipher(st, T.StreamCiphertext(other, st.counter, 8, b"\0"))
    with pytest.raises(ValueError, match="counter"):
        tk.transcipher(st, T.StreamCiphertext(cipher, st.counter - 1, 8, b"\0"))
    with pytest.raises(ValueError):
        tk.transcipher(st, T.StreamCiphertext(cipher, st.counter, 9, b"\0"))
    assert tk.runner.calls == calls and st.counter == 64 + 293


def test_argument_checks_raise_before_any_call():
    tk = cleartext_key()
    k80, k128 = blocks(np.zeros(80)), blocks(np.zeros(128))
    bad = [
        lambda: tk.trivium_generate_keystream(k80, blocks(np.zeros(79)), 64),
        lambda: tk.trivium_generate_keystream(k80, k80, 0),
        lambda: tk.trivium_generate_keystream(k80, k80, 64, num_inputs=0),
        lambda: tk.trivium_generate_keystream(k80, k80, 64, num_inputs=2),
        lambda: tk.trivium_init(k128, k128),
        lambda: tk.kreyvium_init(k80, k80),
        lambda: tk.kreyvium_generate_keystream(k128, k128, -3),
        lambda: tk.kreyvium_init(k128, k128, num_inputs=0),
        lambda: T.apply_keystream(tk, blocks(np.zeros(15)), b"\0\0", 16),
        lambda: T.apply_keystream(tk, blocks(np.zeros(16)), b"\0", 16),
        lambda: T.apply_keystream(tk, blocks(np.zeros(0)), b"", 0),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert tk.runner.calls == 0
    st = tk.trivium_init(k80, k80)
    calls = tk.runner.calls
    for f in (lambda: tk.trivium_next(st, 0), lambda: tk.kreyvium_next(st, 64)):
        with pytest.raises(ValueError):
            f()
    st.counter = T.MAX_COUNTER - 3
    with pytest.raises(ValueError):
        tk.trivium_next(st, 4)
    assert tk.runner.calls == calls
    tk.trivium_next(st, 3)


# ---------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------
# PBS count, PBS layers and peak slots of one instance; recorded in DESIGN §8i
PINNED = {
    ("trivium_keystream", 64): (7168, 27, 488),
    ("trivium_keystream", 512): (10752, 37, 941),
    ("trivium_init", 0): (6656, 26, 469),
    ("trivium_next", 64): (512, 2, 544),
    ("trivium_next", 512): (4096, 12, 930),
    ("kreyvium_keystream", 64): (7357, 28, 712),
    ("kreyvium_keystream", 512): (10941, 37, 1106),
    ("kreyvium_init", 0): (6845, 26, 712),
    ("kreyvium_next", 64): (512, 2, 800),
    ("kreyvium_next", 512): (4096, 12, 1130),
    ("apply_keystream", 0): (1, 1, 2),
}


@pytest.mark.parametrize("kind,n", sorted(PINNED))
def test_pinned_schedule_counts(kind, n):
    s = bc.schedule(T.circuit(kind, n), 1)
    assert (s.pbs_count(), s.num_layers, s.peak_slots) == PINNED[(kind, n)]


def test_schedule_depth_and_pass_through():
    """Trivium init + 512 steps is at most 37 layers (the reference: about 79
    sequential KS -> PBS calls); a 64-round next is 2 layers, and its PBS are
    the rounds' own: 3 ANDs, 3 new state bits and 2 for the keystream bit's
    parity of 6 (Trivium) or 7 (Kreyvium) atoms, none for the 288 - 3 * 64
    state bits passed through.  Outputting the whole state instead costs one
    refresh PBS per passed-through bit."""
    assert bc.schedule(T.circuit("trivium_keystream", 512), 1).num_layers <= 37
    assert bc.schedule(T.circuit("kreyvium_keystream", 512), 1).num_layers <= 37
    for cipher in ("trivium", "kreyvium"):
        s = bc.schedule(T.circuit(f"{cipher}_next", 64), 1)
        assert s.num_layers == 2 and s.pbs_count() == 64 * (3 + 3 + 2)
    c = bc.Circuit("trivium_next_whole_state")
    a, b, r = c.inputs(93, False), c.inputs(84, False), c.inputs(111, False)
    z, a, b, r = T.rounds(c, a, b, r, 64)
    c.output(z + a + b + r)
    assert bc.schedule(c, 1).pbs_count() == 64 * 8 + (288 - 3 * 64)
    # schedules serve any instance count; circuits are cached per (kind, num_steps)
    assert T.circuit("trivium_next", 64) is T.circuit("trivium_next", 64)
    assert bc.schedule(T.circuit("trivium_next", 64), 16).pbs_count() == 16 * 512


def test_circuit_local_luts_and_block_outputs():
    assert len(bc.lut_functions()) == 11
    c = bc.Circuit("blocks")
    x = c.inputs(3, False)
    pack = c.add_lut(T.XOR_PACK_LUT)
    assert pack == bc.NUM_FIXED_LUTS
    wide = c.add_lut([v % 8 for v in range(16)])
    blk = c.lut([(x[0], 1), (x[1], 2)], 0, pack)
    seven = c.lut([(x[0], 1), (x[1], 2), (x[2], 2)], 0, wide)
    with pytest.raises(ValueError):
        c.output([blk])             # a block is not a bit
    with pytest.raises(ValueError):
        c.output_blocks([seven])    # values above 3 are not a block
    for table in ([0] * 15, [16] + [0] * 15, [-1] + [0] * 15):
        with pytest.raises(ValueError):
            c.add_lut(table)
    with pytest.raises(ValueError):
        c.lut([(x[0], 1)], 0, bc.NUM_FIXED_LUTS + 2)
    c.output_blocks([blk, x[2]])
    s = bc.compile_circuit(c, 8)
    assert s.extra_luts == (tuple(T.XOR_PACK_LUT), tuple(v % 8 for v in range(16)))
    ins = np.array([[a, b, d] for a in (0, 1) for b in (0, 1) for d in (0, 1)])
    got = bc.run_cleartext(s, [], ins)
    assert np.array_equal(got, np.array([c.evaluate([], i, []) for i in ins]))
    assert [int(v) for v in got[:, 0]] == [a + 2 * b for a, b, _ in ins]


# ---------------------------------------------------------------------------
# real ciphertexts on the oracle
# ---------------------------------------------------------------------------
def run_oracle(oracle, keys, sched, instance_blocks, iconst_bits=None):
    """The schedule's tables on the oracle with per-instance inputs and the
    circuit's own LUTs: numpy linear step, oracle keyswitch and PBS, scatter
    into the pool (tests only)."""
    P = keys.params
    luts = np.stack([oracle.make_lut(P, f) for f in sched.lut_tables()])
    pool = np.zeros((sched.pool_rows, P.big_n + 1), dtype=np.uint64)
    I = sched.num_instances
    rows = sched.addr(sched.instance_input_slots[None, :], np.arange(I)[:, None]).reshape(-1)
    pool[rows] = instance_blocks
    body = sched.body(iconst_bits)
    lut_rows, dests = sched.gpu_tables()
    o = 0
    for L in range(sched.num_layers):
        r0, r1 = int(sched.layer_rows[L]), int(sched.layer_rows[L + 1])
        sh = int(sched.layer_shared_rows[L])
        staged = []
        for r in range(r0, r1):
            t0, t1 = int(sched.row_offsets[r]), int(sched.row_offsets[r + 1])
            for i in ([0] if r - r0 < sh else range(I)):
                acc = np.zeros(P.big_n + 1, dtype=np.uint64)
                with np.errstate(over="ignore"):
                    acc[-1] = np.uint64(int(body[r, i]) * P.delta % 2 ** 64)
                    for t in range(t0, t1):
                        row = sched.addr(int(sched.term_slots[t]), i)
                        acc += np.uint64(int(sched.term_coefs[t]) % 2 ** 64) * pool[row]
                staged.append(acc)
        n = len(staged)
        small = oracle.keyswitch_batch(keys, np.stack(staged))
        pool[dests[o:o + n].astype(np.int64)] = oracle.pbs_batch(keys, luts, small, lut_idx=lut_rows[o:o + n])
        o += n
    return pool[sched.output_rows()]


def test_trivium_keystream_and_apply_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_aes: 64 Trivium keystream bits of vector 4, then
    those bits applied to a message."""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=41)
    rng = oracle.Rng(0x7217)
    v = VECTORS["trivium"][3]
    key, iv = vector_bits(v, 80)
    enc = M.encrypt_bits(oracle, keys, rng, np.concatenate([key, iv]))
    ks = run_oracle(oracle, keys, bc.schedule(T.circuit("trivium_keystream", 64), 1), enc)
    bits = M.decrypt_messages(oracle, keys, ks)
    assert M.pack_lsb_first(bits).hex().upper() == v["keystream_hex"][:16]
    msg = b"transcip"
    stream = M.pack_lsb_first([a ^ b for a, b in zip(M.bits_lsb_first(msg), bits)])
    s = bc.schedule(T.circuit("apply_keystream"), 32)
    out = run_oracle(oracle, keys, s, ks, T.apply_keystream_iconsts(stream, 64))
    assert M.pack_lsb_first(M.blocks_to_bits(M.decrypt_messages(oracle, keys, out, vmax=3), 64)) == msg


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["classic", "multi_bit_g4"])
def gpu_triv(request, oracle, keyset):
    import torch

    from oracle import csprng
    from tfhe_rs_b200 import gpu, server_key

    assert torch.cuda.is_available()
    if request.param == "classic":
        P = oracle.PARAM_MESSAGE_2_CARRY_2_KS_PBS
    else:
        P = csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS
    keys = keyset(P, seed=0x7210 + P.grouping_factor)
    streams = gpu.CudaStreams.new_single_gpu(0)
    skey = server_key.upload_server_key(keys.bsk, keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log,
                                        pbs_level=P.pbs_level, ks_base_log=P.ks_base_log, ks_level=P.ks_level,
                                        grouping_factor=P.grouping_factor, centered_ms=P.centered_ms,
                                        streams=streams)
    tk = T.CudaTriviumServerKey(skey)
    rng = oracle.Rng(0x7211)

    def enc(bits):
        return torch.from_numpy(M.encrypt_bits(oracle, keys, rng, np.asarray(bits).reshape(-1)).view(np.int64)).to(
            streams.device(0))

    def dec(ct, vmax=1):
        """copy on the caller's current stream, which waits for the work stream"""
        return M.decrypt_messages(oracle, keys, ct.blocks.cpu().numpy().view(np.uint64), vmax)

    yield tk, enc, dec, request.param
    tk.runner.close()


def hexes(bits, count):
    return [M.pack_lsb_first(b).hex().upper() for b in np.asarray(bits).reshape(count, -1)]


@pytest.mark.gpu
def test_gpu_trivium_vectors(gpu_triv):
    """Vectors 1-4 as four inputs of one call: fused 512 steps, and init
    plus 8 x next(64)."""
    tk, enc, dec, _ = gpu_triv
    vs = VECTORS["trivium"]
    keys, ivs = zip(*[vector_bits(v, 80) for v in vs])
    want = [v["keystream_hex"] for v in vs]
    assert hexes(dec(tk.trivium_generate_keystream(enc(keys), enc(ivs), 512, num_inputs=4)), 4) == want
    st = tk.trivium_init(enc(keys), enc(ivs), num_inputs=4)
    parts = [dec(tk.trivium_next(st, 64)).reshape(4, 64) for _ in range(8)]
    assert hexes(np.concatenate(parts, 1), 4) == want


@pytest.mark.gpu
def test_gpu_kreyvium_vectors(gpu_triv):
    tk, enc, dec, _ = gpu_triv
    vs = VECTORS["kreyvium"]
    keys, ivs = zip(*[vector_bits(v, 128) for v in vs])
    want = [v["keystream_hex"] for v in vs]
    assert hexes(dec(tk.kreyvium_generate_keystream(enc(keys), enc(ivs), 64, num_inputs=4)), 4) == want
    st = tk.kreyvium_init(enc(keys), enc(ivs), num_inputs=4)
    parts = [dec(tk.kreyvium_next(st, n)).reshape(4, n) for n in (40, 24)]
    assert hexes(np.concatenate(parts, 1), 4) == want


@pytest.mark.gpu
@pytest.mark.parametrize("cipher", ["trivium", "kreyvium"])
def test_gpu_random_keys_three_inputs(gpu_triv, cipher):
    tk, enc, dec, _ = gpu_triv
    rng = np.random.default_rng(zlib.crc32(b"gpu" + cipher.encode()))
    kb = T.KEY_BITS[cipher]
    keys, ivs = rng.integers(0, 2, (3, kb)), rng.integers(0, 2, (3, kb))
    want = np.array([model(cipher, k, i).keystream(200) for k, i in zip(keys, ivs)])
    got = dec(getattr(tk, f"{cipher}_generate_keystream")(enc(keys), enc(ivs), 72, 3)).reshape(3, 72)
    assert np.array_equal(got, want[:, :72])
    st = getattr(tk, f"{cipher}_init")(enc(keys), enc(ivs), 3)
    got = [dec(getattr(tk, f"{cipher}_next")(st, n)).reshape(3, n) for n in (130, 70)]
    assert np.array_equal(np.concatenate(got, 1), want)


@pytest.mark.gpu
def test_gpu_transcipher_u64_and_1000_bytes(gpu_triv):
    """A Kreyvium session transciphers a u64, a 1,000-byte stream and an odd
    13-bit one; a Trivium session a u64 and 29 bits.  The blocks decrypt to
    the plaintext bits, two per block."""
    tk, enc, dec, _ = gpu_triv
    rng = np.random.default_rng(1000)
    for cipher, msgs in (("kreyvium", [(8, None), (1000, None), (2, 13)]), ("trivium", [(8, None), (4, 29)])):
        kb = T.KEY_BITS[cipher]
        key, iv = rng.integers(0, 2, kb), rng.integers(0, 2, kb)
        plain = model(cipher, key, iv)
        st = getattr(tk, f"{cipher}_init")(enc(key), enc(iv))
        for nbytes, n_bits in msgs:
            msg = bytes(rng.integers(0, 256, nbytes, dtype=np.uint8))
            if n_bits is not None:
                msg = M.pack_lsb_first(M.bits_lsb_first(msg, n_bits))
            sc = stream_ciphertext(cipher, plain, msg, n_bits)
            out = tk.transcipher(st, sc)
            assert out.blocks.shape[0] == (sc.n_bits + 1) // 2
            assert M.blocks_to_bits(dec(out, vmax=3), sc.n_bits) == M.bits_lsb_first(msg, sc.n_bits)
        assert st.counter == plain.counter


@pytest.mark.gpu
def test_gpu_apply_keystream_on_aes_ctr(gpu_triv):
    """apply_keystream works on aes_ctr's keystream bits (same server key)."""
    tk, enc, dec, _ = gpu_triv
    key, iv = bytes(range(16)), int("f0f1f2f3f4f5f6f7f8f9fafbfcfdfeff", 16)
    ask = aes.CudaAesServerKey(tk.skey)
    ks = ask.aes_ctr(enc(AM.key_bits(key)), enc(AM.u128_bits(iv)), 0, 1)
    msg = bytes(range(16))
    kbits = [int(b) for b in AM.u128_bits(AM.aes_ctr(key, iv, 0, 1)[0])]
    stream = bytes(a ^ b for a, b in zip(msg, M.pack_lsb_first(kbits)))
    out = T.apply_keystream(ask, ks, stream, 128)
    assert M.pack_lsb_first(M.blocks_to_bits(dec(out, vmax=3), 128)) == msg
    ask.runner.close()


@pytest.mark.gpu
def test_gpu_dropped_inputs_and_state_after_key_drop(gpu_triv):
    """Calls enqueued back to back whose inputs the caller drops at once, the
    caller's stream then scribbling over fresh memory of their shapes; a
    Kreyvium state used after its key and IV were dropped and scribbled
    over.  Results are read on the caller's stream with no explicit
    synchronisation."""
    import torch

    tk, enc, dec, _ = gpu_triv
    rng = np.random.default_rng(77)
    big = tk.skey.big_dim
    dev = tk.runner.device
    scribbles, outs, cases = [], [], []
    for j in range(3):
        key, iv = rng.integers(0, 2, 80), rng.integers(0, 2, 80)
        cases.append((key, iv))
        outs.append(tk.trivium_generate_keystream(enc(key), enc(iv), 64))
        scribbles += [torch.full((rows, big + 1), -1, dtype=torch.int64, device=dev) for rows in (80, 80, 160)]
    kkey, kiv = rng.integers(0, 2, 128), rng.integers(0, 2, 128)
    k_ct, iv_ct = enc(kkey), enc(kiv)
    st = tk.kreyvium_init(k_ct, iv_ct)
    del k_ct, iv_ct
    scribbles += [torch.full((rows, big + 1), -1, dtype=torch.int64, device=dev) for rows in (128, 128, 256)]
    first = tk.kreyvium_next(st, 100)
    second = tk.kreyvium_next(st, 60)   # K* / IV* wrap past 128
    for (key, iv), out in zip(cases, outs):
        assert list(dec(out)) == M.Trivium(key, iv).keystream(64)
    plain = M.Kreyvium(kkey, kiv)
    assert list(dec(first)) + list(dec(second)) == plain.keystream(160)


@pytest.mark.gpu
def test_gpu_next_launch_count(gpu_triv):
    """One next(64) call is its schedule's 2 layers of 256 rows, each the
    linear kernel, the int8 keyswitch's 2 kernels and one PBS kernel (the
    N = 2048 register kernel on classic P22; on multi-bit g = 4 the fused
    kernel, which takes layers wider than the SM count): 2 * 4 launches."""
    from tfhe_rs_b200 import _lib

    tk, enc, dec, _ = gpu_triv
    L = _lib.lib()
    st = tk.trivium_init(enc(np.zeros(80)), enc(np.zeros(80)))
    tk.trivium_next(st, 64)               # warm-up: tables and scratch
    tk.runner.streams.synchronize()
    s = bc.schedule(T.circuit("trivium_next", 64), 1)
    assert s.num_layers == 2 and [s.layer_outputs(i) for i in range(2)] == [256, 256]
    before = L.b200_kernel_launch_count()
    out = tk.trivium_next(st, 64)
    tk.runner.streams.synchronize()
    assert L.b200_kernel_launch_count() - before == 2 * (1 + 2 + 1)
    assert list(dec(out)) == M.Trivium([0] * 80, [0] * 80).keystream(128)[64:]
