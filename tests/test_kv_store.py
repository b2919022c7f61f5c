"""The encrypted key-value store (tfhe-rs_b200/kv_store.py and the kv_store_*
methods of integer.CudaRadixServerKey).

CPU: insert / remove / get / update / map / contains sequences on the
cleartext runner of test_radix_find, checked against a Python dict, with
4-block keys and 1-, 2- and 8-block values, unsigned and signed; the empty
store's trivial results; argument checks; one `kv_store_get` of 2-block keys
and values over 5 entries through real LWE keyswitches and PBS on the oracle.

GPU: get, update and map (`scalar_add` through the server key) on a
64-entry FheUint64 -> FheUint64 store and one get on a 1024-entry store, on
classic P22 and multi-bit g = 4; every output block decrypts to the model's
value."""
import zlib

import numpy as np
import pytest

from tfhe_rs_b200 import bit_circuit as bc, kv_store as KV, radix as R, radix_find as F

from tests import find_model as FM
from tests import trivium_model as M
from tests.test_radix import wrap
from tests.test_radix_find import cleartext_key, flag, gpu_find, one, radix_of, run_oracle_shared  # noqa: F401
from tests.test_trivium import run_oracle


def store_of(d, nv, signed=False):
    s = KV.CudaKVStore()
    for k, v in d.items():
        assert s.insert(k, one(v, nv, signed)) is None
    return s


def contents(s, signed=False):
    return {k: radix_of(s.get(k), signed)[0] for k in s.keys()}


@pytest.mark.parametrize("nv", [1, 2, 8])
@pytest.mark.parametrize("signed", [False, True])
def test_store_sequences_against_a_dict(nv, signed):
    """4-block keys, nv-block values: a random sequence of clear inserts and
    removes and encrypted gets, updates, maps and contains"""
    key = cleartext_key()
    nk = 4
    rng = np.random.default_rng(zlib.crc32(f"kv{nv}{signed}".encode()))
    klo, khi = R.scalar_range(nk, signed)
    vlo, vhi = R.scalar_range(nv, signed)
    keys = [int(k) for k in rng.choice(np.arange(klo, khi), 10, replace=False)]
    s, d = KV.CudaKVStore(), {}
    for step in range(40):
        op = int(rng.integers(0, 7))
        k = keys[int(rng.integers(0, len(keys)))]
        v = int(rng.integers(vlo, vhi))
        q = one(k, nk, signed)
        if op == 0:
            old = s.insert(k, one(v, nv, signed))
            assert (None if old is None else radix_of(old, signed)[0]) == d.get(k)
            d[k] = v
        elif op == 1:
            old = s.remove(k)
            assert (None if old is None else radix_of(old, signed)[0]) == d.pop(k, None)
        elif op == 2:
            got, found = key.kv_store_get(s, q)
            want, wfound = FM.kv_store_get(d, k, nk)
            assert (radix_of(got, signed), flag(found)) == (want if not d else (want, nv), wfound)
        elif op == 3:
            found = key.kv_store_update(s, q, one(v, nv, signed))
            assert flag(found) == FM.kv_store_update(d, k, v)
        elif op == 4:
            def f(ct):
                return key.scalar_add(ct, 1)
            old, new, found = key.kv_store_map(s, q, f)
            o, nw, fd = FM.kv_store_map(d, k, lambda x: wrap(x + 1, nv if d else nk, signed), nk)
            assert (radix_of(old, signed)[0], radix_of(new, signed)[0], flag(found)) == (o, nw, fd)
        elif op == 5:
            assert flag(key.kv_store_contains_key(s, q)) == int(k in d)
            assert flag(key.kv_store_contains_clear_value(s, v)) == int(v in d.values())
        else:
            assert flag(key.kv_store_contains_value(s, one(v, nv, signed))) == int(v in d.values())
        assert len(s) == len(d) and contents(s, signed) == d, step


def test_empty_store_gives_trivial_results():
    key = cleartext_key()
    s = KV.CudaKVStore()
    q = one(7, 3)
    assert (radix_of(key.kv_store_get(s, q)[0]), flag(key.kv_store_get(s, q)[1])) == ((0, 3), 0)
    assert flag(key.kv_store_update(s, q, one(1, 3))) == 0
    old, new, found = key.kv_store_map(s, q, lambda ct: key.scalar_add(ct, 5))
    assert (radix_of(old), radix_of(new), flag(found)) == ((0, 3), (5, 3), 0)
    assert flag(key.kv_store_contains_key(s, q)) == 0 and flag(key.kv_store_contains_value(s, q)) == 0
    assert flag(key.kv_store_contains_clear_value(s, 1)) == 0
    assert key.runner.calls == 1 and len(s) == 0   # map's scalar_add


def test_store_argument_checks():
    key = cleartext_key()
    s = store_of({1: 2, 300: 3}, 2)
    bad = [
        lambda: key.kv_store_get(s, one(1, 4)),               # the clear key 300 does not fit 4 blocks
        lambda: key.kv_store_contains_key(s, one(1, 4, True)),
        lambda: key.kv_store_update(s, one(1, 5), one(1, 3)),  # value width
        lambda: key.kv_store_update(s, one(1, 5), one(1, 2, True)),
        lambda: key.kv_store_map(s, one(1, 5), lambda ct: one(1, 3)),
        lambda: s.insert(3, one(1, 3)),
        lambda: s.insert(3, one(1, 2, True)),
        lambda: s.insert(True, one(1, 2)),
        lambda: s.insert(1.5, one(1, 2)),
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    # only map's read (its two calls) ran, before the mapped value was refused
    assert key.runner.calls == 2 and len(s) == 2
    assert s.insert(4, integer_empty()) is None and len(s) == 2


def integer_empty():
    import torch

    from tfhe_rs_b200 import integer

    return integer.CudaUnsignedRadixCiphertext(torch.zeros((0, 1), dtype=torch.int64), 1)


def test_kv_store_get_on_the_oracle(oracle, keyset):
    """Real LWE encrypt -> (linear, KS, PBS) x layers -> decrypt at the toy
    2_2 parameters of test_radix: kv_store_get of a 2-block key over 5
    entries of 2-block values, present and absent"""
    P = oracle.Params("TOY_2_2_N512", n=32, k=1, N=512, pbs_base_log=23, pbs_level=1, ks_base_log=4, ks_level=4,
                      lwe_noise_log2=30, glwe_noise_log2=8)
    keys = keyset(P, seed=67)
    rng = oracle.Rng(0xC0DE)
    n, store = 2, {1: 9, 4: 15, 7: 0, 12: 3, 13: 6}
    ks = sorted(store)
    for x in (12, 5):
        s = bc.schedule(F.circuit("select", n, n), len(ks))
        query = M.encrypt_bits(oracle, keys, rng, R.to_digits(x, n))
        vals = M.encrypt_bits(oracle, keys, rng, [d for k in ks for d in R.to_digits(store[k], n)])
        per = run_oracle_shared(oracle, keys, s, query, vals, R.scalar_iconsts(ks, n, False))
        out = M.decrypt_messages(oracle, keys, run_oracle(oracle, keys, F.tree("select", len(ks), 1 + n), per),
                                 vmax=3)
        assert (R.from_digits(out[:n]), int(out[n])) == (store.get(x, 0), int(x in store))


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def gpu_store(enc_list, d, n):
    s = KV.CudaKVStore()
    for k, ct in zip(d, enc_list(list(d.values()), n)):
        s.insert(k, ct)
    return s


@pytest.mark.gpu
def test_gpu_store_of_64_fheuint64(gpu_find):
    rk, enc, enc_list, dec = gpu_find
    n = 32
    rng = np.random.default_rng(64)
    d = {int(k): int(v) for k, v in zip(rng.integers(0, 2 ** 64, 64, dtype=np.uint64),
                                         rng.integers(0, 2 ** 64, 64, dtype=np.uint64))}
    s = gpu_store(enc_list, d, n)
    present, absent = list(d)[41], next(k for k in range(10) if k not in d)
    for k in (present, absent):
        v, found = rk.kv_store_get(s, enc(k, n))
        assert (dec(v), dec(found)) == ((d.get(k, 0), n), int(k in d))
    assert dec(rk.kv_store_update(s, enc(present, n), enc(2 ** 64 - 3, n))) == 1
    d[present] = 2 ** 64 - 3
    old, new, found = rk.kv_store_map(s, enc(present, n), lambda ct: rk.scalar_add(ct, 5))
    assert (dec(old)[0], dec(new)[0], dec(found)) == (2 ** 64 - 3, 2, 1)
    d[present] = 2
    assert dec(rk.kv_store_update(s, enc(absent, n), enc(1, n))) == 0
    assert dec(rk.kv_store_contains_key(s, enc(present, n))) == 1
    assert dec(rk.kv_store_contains_clear_value(s, 2)) == 1
    assert dec(rk.kv_store_contains_value(s, enc(d[list(d)[3]], n))) == 1
    for k in (list(d)[0], present, list(d)[-1]):
        assert dec(s.get(k))[0] == d[k]


@pytest.mark.gpu
def test_gpu_store_of_1024_get(gpu_find):
    rk, enc, enc_list, dec = gpu_find
    n = 32
    rng = np.random.default_rng(1024)
    d = {int(k): int(v) for k, v in zip(rng.choice(2 ** 40, 1024, replace=False),
                                         rng.integers(0, 2 ** 64, 1024, dtype=np.uint64))}
    s = gpu_store(enc_list, d, n)
    k = list(d)[777]
    v, found = rk.kv_store_get(s, enc(k, n))
    assert (dec(v), dec(found)) == ((d[k], n), 1)
