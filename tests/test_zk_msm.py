"""BLS12-446 MSM (include/tfhe_b200_zk.h, csrc/bls12_446.cuh, csrc/msm.cuh)
against the plain-integer model of tests/bls12_446_model.py.

CPU: the header's constants, field and group law through its g++ build
(tests/emu/zk_host.cpp), the window digits, the ABI struct layout, the
exported symbols, the host-only C wrappers and argument checking.
GPU: G1 and G2 MSMs word for word against the model, edge batches, the managed
and unmanaged calls, and parity with the reference's zk library when built;
one MSM at and just below the smallest n of every window size, buckets at the
task and tree-pass edges, and the unmanaged call on a scratch of exactly the
reported size.  tests/test_zk_device_arith.py checks the device field and
curve code op by op."""
import ctypes as C
import os
import random
import re

import numpy as np
import pytest

from tests import bls12_446_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASK = (1 << 64) - 1


def limbs(v, n=7):
    return np.array([(v >> (64 * i)) & MASK for i in range(n)], dtype=np.uint64)


def val(a):
    return sum(int(w) << (64 * i) for i, w in enumerate(np.asarray(a, dtype=np.uint64).reshape(-1)))


def mont(v):
    return v * M.MONT_R % M.P


def unmont(v):
    return v * pow(M.MONT_R, -1, M.P) % M.P


@pytest.fixture(scope="module")
def host():
    from tests.emu.build_zk import build

    lib = C.CDLL(build())
    vp, i = C.c_void_p, C.c_int
    for name, args in {"zk_constants": [vp] * 5, "zk_fp_op": [i, vp, vp, vp], "zk_fp2_op": [i, vp, vp, vp],
                       "zk_g1_op": [i, vp, vp, vp, vp], "zk_g2_op": [i, vp, vp, vp, vp], "zk_num_windows": [i],
                       "zk_signed_digits": [vp, vp, i], "zk_struct_layout": [vp]}.items():
        getattr(lib, name).argtypes = args
    return lib


@pytest.fixture(scope="module")
def L():
    import tfhe_rs_b200

    return tfhe_rs_b200.lib()


# ---------------------------------------------------------------- CPU -----

def test_constants_derive_from_the_seed(host):
    p, r2, one, r = (np.zeros(n, np.uint64) for n in (7, 7, 7, 5))
    pinv = C.c_uint64()
    host.zk_constants(p.ctypes.data, r2.ctypes.data, one.ctypes.data, C.byref(pinv), r.ctypes.data)
    assert val(p) == M.P and M.P.bit_length() == 446 and M.P % 4 == 3 and 4 * M.P < M.MONT_R
    assert val(r) == M.R_ORDER and M.R_ORDER.bit_length() == 299
    assert val(r2) == M.R2 and val(one) == M.MONT_R % M.P
    assert pinv.value == M.PINV == 0xcd63fd900035fffd
    assert M.G1_ORDER == M.R_ORDER * (M.X - 1) ** 2 // 3


def test_generators_lie_on_their_curves_and_have_order_r():
    assert M.G1.on_curve(M.G1_GEN) and M.G2.on_curve(M.G2_GEN)
    assert M.G1.mul(M.R_ORDER, M.G1_GEN) is None and M.G2.mul(M.R_ORDER, M.G2_GEN) is None
    assert M.G1.mul(M.R_ORDER - 1, M.G1_GEN) == M.G1.neg(M.G1_GEN)


def _fp_values(rng, count):
    edge = [0, 1, 2, M.P - 1, M.P - 2, M.MONT_R % M.P, (M.MONT_R - 1) % M.P, M.P // 2, 1 << 445]
    return edge + [rng.randrange(M.P) for _ in range(count)]


def test_fp_matches_the_model(host):
    rng = random.Random(1)
    vals = _fp_values(rng, 40)
    pairs = [(a, b) for a in vals[:9] for b in vals[:9]] + [(rng.choice(vals), rng.choice(vals)) for _ in range(200)]
    out = np.zeros(7, np.uint64)

    def op(code, a, b=0):
        la, lb = limbs(a), limbs(b)
        host.zk_fp_op(code, out.ctypes.data, la.ctypes.data, lb.ctypes.data)
        return val(out)

    for a, b in pairs:
        am, bm = mont(a), mont(b)
        assert op(0, am, bm) == mont((a + b) % M.P)
        assert op(1, am, bm) == mont((a - b) % M.P)
        assert op(2, am, bm) == mont(a * b % M.P)
    for a in vals:
        am = mont(a)
        assert op(3, am) == mont(a * a % M.P)
        assert op(4, am) == mont(-a % M.P)
        assert op(5, am) == mont(pow(a, M.P - 2, M.P))
        assert op(6, a) == am and op(7, am) == a


def test_fp2_matches_the_model(host):
    rng = random.Random(2)
    vals = _fp_values(rng, 10)
    elems = [(a, b) for a in vals[:5] for b in vals[:5]] + [(rng.choice(vals), rng.choice(vals)) for _ in range(40)]
    out = np.zeros(14, np.uint64)

    def enc(x):
        return np.concatenate([limbs(mont(x[0])), limbs(mont(x[1]))])

    def op(code, a, b=(0, 0)):
        ea, eb = enc(a), enc(b)
        host.zk_fp2_op(code, out.ctypes.data, ea.ctypes.data, eb.ctypes.data)
        return unmont(val(out[:7])), unmont(val(out[7:]))

    for a in elems:
        b = rng.choice(elems)
        assert op(0, a, b) == M.f2_add(a, b)
        assert op(1, a, b) == M.f2_sub(a, b)
        assert op(2, a, b) == M.f2_mul(a, b)
        assert op(3, a) == M.f2_mul(a, a)
        assert op(4, a) == M.f2_neg(a)
        if a != (0, 0):
            assert op(5, a) == M.f2_inv(a)


def _mont_point(curve, p):
    from tfhe_rs_b200 import zk

    g = zk.G1 if curve is M.G1 else zk.G2
    if p is None:
        return zk.points(g, [None])
    if curve is M.G1:
        return zk.points(g, [(mont(p[0]), mont(p[1]))])
    return zk.points(g, [((mont(p[0][0]), mont(p[0][1])), (mont(p[1][0]), mont(p[1][1])))])


def _unmont_point(curve, a):
    if a["infinity"][0]:
        return None
    if curve is M.G1:
        return unmont(val(a["x"][0])), unmont(val(a["y"][0]))
    return ((unmont(val(a["x"][0][0])), unmont(val(a["x"][0][1]))),
            (unmont(val(a["y"][0][0])), unmont(val(a["y"][0][1]))))


def _proj_to_affine(curve, proj):
    w = proj.reshape(3, -1)
    X, Y, Z = (unmont(val(r)) if curve is M.G1 else (unmont(val(r[:7])), unmont(val(r[7:]))) for r in w)
    if Z in (0, (0, 0)):
        return None
    zi = curve.F.inv(Z)
    return curve.F.mul(X, zi), curve.F.mul(Y, zi)


@pytest.mark.parametrize("name", ["g1", "g2"])
def test_group_law_matches_the_model(host, name):
    curve = M.G1 if name == "g1" else M.G2
    fn = getattr(host, f"zk_{name}_op")
    rng = random.Random(3)
    P = curve.mul(rng.randrange(1, M.R_ORDER), curve.gen)
    Q = curve.mul(rng.randrange(1, M.R_ORDER), curve.gen)
    proj = np.zeros(3 * 7 * (1 if name == "g1" else 2), np.uint64)

    def run(mode, p, q):
        a, b = _mont_point(curve, p), _mont_point(curve, q)
        out = np.zeros(1, a.dtype)
        fn(mode, out.ctypes.data, proj.ctypes.data, a.ctypes.data, b.ctypes.data)
        return _unmont_point(curve, out)

    # generic, P + P, P + (-P), and the identity on either side
    for p, q in [(P, Q), (P, P), (P, curve.neg(P)), (None, P), (P, None), (None, None)]:
        for mode in (0, 1):  # mixed addition, XYZZ addition
            assert run(mode, p, q) == curve.add(p, q), (mode, p is None, q is None)
        assert run(2, p, p) == curve.add(p, p)
        # (X ZZZ, Y ZZ, ZZ ZZZ) is the same point; the identity is (0, 0, 0)
        proj[...] = 7
        assert run(3, p, q) == curve.add(p, q)
        assert _proj_to_affine(curve, proj) == curve.add(p, q)
        if curve.add(p, q) is None:
            assert not proj.any()


def _digit_scalars():
    r = M.R_ORDER
    top = (1 << 320) - 1
    return [0, 1, 2, r - 1, r, r + 1, top, top - 1, 1 << 319, (1 << 320) - (1 << 300), 0x80 << 312,
            0x7F << 312, sum(0x80 << (8 * i) for i in range(40))] + [random.Random(4).getrandbits(320)
                                                                     for _ in range(20)]


@pytest.mark.parametrize("c", range(4, 17))
def test_signed_digits_reconstruct_every_scalar(host, c):
    W = host.zk_num_windows(c)
    assert W == 320 // c + 1
    d = np.zeros(W, np.int32)
    half = 1 << (c - 1)
    for k in _digit_scalars():
        host.zk_signed_digits(d.ctypes.data, limbs(k, 5).ctypes.data, c)
        assert all(-half < int(x) <= half for x in d)
        assert sum(int(x) << (c * w) for w, x in enumerate(d)) == k
        assert d[-1] >= 0
    # a carry out of the top full window lands in the extra window
    host.zk_signed_digits(d.ctypes.data, limbs((1 << 320) - 1, 5).ctypes.data, c)
    assert d[-1] == (1 << (320 % c)) if 320 % c else d[-1] == 1


def test_struct_layout(host):
    from tfhe_rs_b200 import zk

    out = np.zeros(14, np.uint64)
    host.zk_struct_layout(out.ctypes.data)
    assert list(map(int, out)) == [56, 112, 40, 120, 56, 112, 232, 112, 224, 168, 112, 336, 224, 8]
    assert zk.G1_DTYPE.itemsize == 120 and zk.G1_DTYPE.fields["infinity"][1] == 112
    assert zk.G2_DTYPE.itemsize == 232 and zk.G2_DTYPE.fields["infinity"][1] == 224


def _zk_header_functions():
    text = open(os.path.join(ROOT, "include", "tfhe_b200_zk.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b([a-z_0-9]+)\s*\(", text)) - {"defined", "sizeof"})


def test_zk_header_equals_signatures_and_is_exported(L):
    from tfhe_rs_b200 import _lib

    declared = _zk_header_functions()
    assert set(declared) == set(_lib.ZK_SIGNATURES)
    assert len([n for n in declared if not n.startswith("b200_")]) == 25
    assert not set(_lib.ZK_SIGNATURES) & set(_lib.SIGNATURES)
    for name in declared:
        assert hasattr(L, name), name


def test_host_wrappers_match_the_model(L):
    from tfhe_rs_b200 import zk

    rng = random.Random(5)
    out = np.zeros(7, np.uint64)
    for v in _fp_values(rng, 10):
        L.fp_to_montgomery_wrapper(out.ctypes.data, limbs(v).ctypes.data)
        assert val(out) == mont(v)
        L.fp_from_montgomery_wrapper(out.ctypes.data, limbs(mont(v)).ctypes.data)
        assert val(out) == v
    r = np.zeros(5, np.uint64)
    L.scalar_modulus_limbs_wrapper(r.ctypes.data)
    assert val(r) == M.R_ORDER
    for name, curve in (("g1", M.G1), ("g2", M.G2)):
        g = zk.G1 if name == "g1" else zk.G2
        P = curve.mul(rng.randrange(1, M.R_ORDER), curve.gen)
        normal = zk.points(g, [P])
        assert getattr(L, f"is_on_curve_{name}_wrapper")(normal.ctypes.data)
        none = zk.points(g, [None])
        assert getattr(L, f"is_on_curve_{name}_wrapper")(none.ctypes.data)
        bad = normal.copy()
        bad["y"] = zk.points(g, [(P[0], curve.F.add(P[1], curve.F.one))])["y"]
        assert not getattr(L, f"is_on_curve_{name}_wrapper")(bad.ctypes.data)
        pm = _mont_point(curve, P)
        back = np.zeros(1, g.dtype)
        getattr(L, f"{name}_from_montgomery_wrapper")(back.ctypes.data, pm.ctypes.data)
        assert back.tobytes() == normal.tobytes()
        # affine -> projective (Z = 1) -> scaled by t -> affine and normalized
        proj = np.zeros(g.proj_shape, np.uint64)
        getattr(L, f"affine_to_projective_{name}_wrapper")(proj.ctypes.data, pm.ctypes.data)
        t = rng.randrange(2, M.P)
        if name == "g1":
            scaled = np.stack([limbs(mont(P[0] * t % M.P)), limbs(mont(P[1] * t % M.P)), limbs(mont(t))])
            assert val(proj[2]) == mont(1)
        else:
            tt = (t, rng.randrange(M.P))
            sc = [M.f2_mul(P[0], tt), M.f2_mul(P[1], tt), tt]
            scaled = np.stack([np.stack([limbs(mont(e[0])), limbs(mont(e[1]))]) for e in sc])
        aff = np.zeros(1, g.dtype)
        getattr(L, f"projective_to_affine_{name}_wrapper")(aff.ctypes.data, scaled.ctypes.data)
        assert aff.tobytes() == pm.tobytes()
        assert zk.normalized_to_affine(g, zk.normalize(g, scaled)) == P
        n1 = zk.normalize(g, scaled)
        assert val(n1[2]) == 1
        # the identity: Z = 0 stays 0, the infinity helpers
        zero = np.zeros(g.proj_shape, np.uint64)
        assert zk.normalized_to_affine(g, zk.normalize(g, zero)) is None
        getattr(L, f"projective_to_affine_{name}_wrapper")(aff.ctypes.data, zero.ctypes.data)
        assert aff["infinity"][0] and getattr(L, f"{name}_is_infinity_wrapper")(aff.ctypes.data)
        getattr(L, f"{name}_point_at_infinity_wrapper")(aff.ctypes.data)
        assert aff.tobytes() == zk.points(g, [None]).tobytes()
        proj[...] = 7
        getattr(L, f"{name}_projective_point_at_infinity_wrapper")(proj.ctypes.data)
        assert not proj.any()


def test_bad_arguments_raise_before_any_call(monkeypatch):
    from tfhe_rs_b200 import zk

    def no_gpu(*_):
        raise AssertionError("reached the library")

    monkeypatch.setattr(zk, "_check_gpu", no_gpu)
    pts = zk.points(zk.G1, [M.G1_GEN] * 3)
    ks = zk.scalars([1, 2, 3])
    with pytest.raises(ValueError):
        zk.g1_msm_gpu(pts, ks[:2])
    with pytest.raises(ValueError):
        zk.g1_msm_gpu(pts.view(np.uint8), ks)
    with pytest.raises(ValueError):
        zk.g2_msm_gpu(pts, ks)  # G1 points to a G2 MSM
    with pytest.raises(ValueError):
        zk.g1_msm_gpu(pts, ks.astype(np.int64))
    with pytest.raises(ValueError):
        zk.g1_msm_gpu(pts, ks[:, :4].copy())
    with pytest.raises(ValueError):
        zk.scalars([1 << 320])
    with pytest.raises(ValueError):
        zk.scalars([-1])
    with pytest.raises(ValueError):
        zk.scratch_size(zk.G1, 0)
    with pytest.raises(ValueError):
        zk.scratch_size(zk.G1, 1 << 32)
    # n = 0: the identity, no call
    assert zk.g1_msm_gpu(pts[:0], ks[:0]) is None and zk.g2_msm_gpu(zk.points(zk.G2, []), ks[:0]) is None
    assert not zk.msm_managed(zk.G2, zk.points(zk.G2, []), ks[:0]).any()


def test_n_of_2_pow_32_is_rejected(monkeypatch):
    from tfhe_rs_b200 import zk

    class Big(np.ndarray):
        def __len__(self):
            return 1 << 32

    pts = zk.points(zk.G1, [M.G1_GEN]).view(Big)
    ks = zk.scalars([1]).view(Big)
    monkeypatch.setattr(zk, "_check_gpu", lambda *_: (_ for _ in ()).throw(AssertionError("reached")))
    with pytest.raises(ValueError):
        zk.msm_managed(zk.G1, pts, ks)


# ---------------------------------------------------------------- GPU -----

_CACHE = {}


def _batch(name, n, seed=7):
    """(curve, zk group, logs, normal-form ABI points, Montgomery ABI points)"""
    from tfhe_rs_b200 import zk

    key = (name, n, seed)
    if key not in _CACHE:
        curve = M.G1 if name == "g1" else M.G2
        g = zk.G1 if name == "g1" else zk.G2
        logs, pts = M.known_multiples(curve, n, random.Random(seed))
        if name == "g1":
            mpts = [(mont(x), mont(y)) for x, y in pts]
        else:
            mpts = [((mont(x[0]), mont(x[1])), (mont(y[0]), mont(y[1]))) for x, y in pts]
        _CACHE[key] = (curve, g, logs, pts, zk.points(g, pts), zk.points(g, mpts))
    return _CACHE[key]


def _gpu_msm(name, normal, ks):
    from tfhe_rs_b200 import zk

    return (zk.g1_msm_gpu if name == "g1" else zk.g2_msm_gpu)(normal, ks)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
@pytest.mark.parametrize("n", [1, 2, 3, 31, 256, 1000, 4100, 65536])
def test_msm_random_scalars(name, n):
    from tfhe_rs_b200 import zk

    curve, g, logs, _, normal, _ = _batch(name, n)
    rng = random.Random(n)
    k = [rng.randrange(M.R_ORDER) for _ in range(n)]
    assert _gpu_msm(name, normal, zk.scalars(k)) == M.msm_by_logs(curve, k, logs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
def test_msm_edge_batches(name):
    from tfhe_rs_b200 import zk

    n = 300
    curve, g, logs, pts, normal, _ = _batch(name, n)
    r, top = M.R_ORDER, (1 << 320) - 1
    rng = random.Random(11)
    # all scalars 0
    assert _gpu_msm(name, normal, zk.scalars([0] * n)) is None
    # all scalars equal: every point of a window in one bucket
    for k in (5, r - 1, (1 << 299) + 12345):
        assert _gpu_msm(name, normal, zk.scalars([k] * n)) == M.msm_by_logs(curve, [k] * n, logs)
    # the same point n times
    same = zk.points(g, [pts[0]] * n)
    ks = [rng.randrange(r) for _ in range(n)]
    assert _gpu_msm(name, same, zk.scalars(ks)) == curve.mul(sum(ks) * logs[0] % r, curve.gen)
    assert _gpu_msm(name, same, zk.scalars([7] * n)) == curve.mul(7 * n * logs[0] % r, curve.gen)
    # pairs P, -P with equal scalars: the identity
    pairs = zk.points(g, [q for p in pts[:n // 2] for q in (p, curve.neg(p))])
    kk = [k for k in ks[:n // 2] for _ in (0, 1)]
    assert _gpu_msm(name, pairs, zk.scalars(kk)) is None
    # infinity-flagged points
    inf = normal.copy()
    holes = list(range(0, n, 3))
    inf["infinity"][holes] = True
    assert _gpu_msm(name, inf, zk.scalars(ks)) == M.msm_by_logs(curve, ks, logs, infinity=holes)
    # scalars r - 1, r, r + 1, 2^320 - 1 and other 320-bit values
    wide = [r - 1, r, r + 1, top, top - 1, 1 << 319] * (n // 6)
    wide += [rng.getrandbits(320) for _ in range(n - len(wide))]
    assert _gpu_msm(name, normal, zk.scalars(wide)) == M.msm_by_logs(curve, wide, logs)
    # one point, scalar 2^320 - 1
    assert _gpu_msm(name, normal[:1], zk.scalars([top])) == curve.mul(top * logs[0] % r, curve.gen)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
def test_managed_and_unmanaged_calls_agree(name):
    import torch

    from tfhe_rs_b200 import gpu, zk

    n = 1000
    curve, g, logs, _, normal, montp = _batch(name, n)
    rng = random.Random(13)
    ks = zk.scalars([rng.randrange(M.R_ORDER) for _ in range(n)])
    a = zk.msm_managed(g, normal, ks, points_in_montgomery=False)
    b = zk.msm_managed(g, montp, ks, points_in_montgomery=True)
    streams = gpu.CudaStreams.new_single_gpu(0)
    c = zk.msm_device(g, zk.to_device(montp, streams), zk.to_device(ks, streams), streams)
    side = torch.cuda.Stream(device=0)  # a non-default stream of another owner
    s2 = gpu.CudaStreams.new_single_gpu(0)
    s2.streams[0] = side
    d = zk.msm_device(g, zk.to_device(montp, s2), zk.to_device(ks, s2), s2)
    assert a.tobytes() == b.tobytes() == c.tobytes() == d.tobytes()
    expect = M.msm_by_logs(curve, [zk.limbs_to_int(k) for k in ks], logs)
    assert zk.normalized_to_affine(g, zk.normalize(g, a)) == expect
    cfg = zk._lib.lib().b200_last_msm_config().decode()
    assert "msm_accumulate_kernel" in cfg and cfg.startswith("c=")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
@pytest.mark.parametrize("n", [1, 31, 1000, 4100])
def test_parity_with_the_reference_library(name, n):
    from tfhe_rs_b200 import _lib, zk

    if not os.path.exists(_lib.REF_ZK_LIB_PATH):
        pytest.skip("oracle/_ref/libzk_cuda_backend_ref.so was not built")
    R = _lib.load_zk()
    L = _lib.lib()
    curve, g, logs, _, normal, _ = _batch(name, n)
    rng = random.Random(17 + n)
    ks = zk.scalars([rng.randrange(M.R_ORDER) for _ in range(n)])
    results = []
    for lib in (L, R):
        raw = np.zeros(g.proj_shape, np.uint64)
        stream = L.cuda_create_stream_ffi(0)
        tracker = C.c_uint64(0)
        getattr(lib, f"{name}_msm_managed_wrapper")(stream, 0, raw.ctypes.data, normal.ctypes.data, ks.ctypes.data,
                                                    n, False, C.byref(tracker))
        L.cuda_destroy_stream(stream, 0)
        out = np.zeros(g.proj_shape, np.uint64)
        getattr(lib, f"{name}_projective_from_montgomery_normalized_wrapper")(out.ctypes.data, raw.ctypes.data)
        results.append(out)
    assert results[0].tobytes() == results[1].tobytes()
    assert zk.normalized_to_affine(g, results[0]) == M.msm_by_logs(curve, [zk.limbs_to_int(k) for k in ks], logs)


# ---------------------------------------------------- every window plan ---
# msm_plan picks c in [4, 16] for G1 and [4, 14] for G2 minimising
# num_windows(c) (n + 3 2^(c-1)); the smallest n of each c:
PLAN_THRESHOLDS = {4: 1, 5: 74, 6: 188, 7: 457, 8: 1383, 9: 2381, 10: 7681, 11: 13825, 12: 24577, 13: 70657,
                   14: 129025, 15: 516097, 16: 983041}
C_MAX = {"g1": 16, "g2": 14}
POOL = 2048  # points are drawn cyclically from this many known multiples


def _plan_c(n, cmax):
    best = pc = None
    for c in range(4, cmax + 1):
        cost = (320 // c + 1) * (n + 3 * (1 << (c - 1)))
        if best is None or cost < best:
            best, pc = cost, c
    return pc


def test_plan_thresholds_follow_the_cost_formula():
    for name, cmax in C_MAX.items():
        for c in range(4, cmax + 1):
            n = PLAN_THRESHOLDS[c]
            assert _plan_c(n, cmax) == c and (n == 1 or _plan_c(n - 1, cmax) == c - 1), (name, c)
    assert _plan_c(1 << 31, 14) == 14 and _plan_c(1 << 31, 16) == 16


PLAN_ROWS = [(name, n) for name, cmax in C_MAX.items() for c in range(4, cmax + 1)
             for n in sorted({PLAN_THRESHOLDS[c], PLAN_THRESHOLDS[c] - 1} - {0})]
SEEN_C = {"g1": set(), "g2": set()}
COMPLETED_PLANS = set()


def _pool(name):
    """(curve, logs, normal-form ABI pool, Montgomery ABI pool) of POOL points"""
    _, g, logs, _, normal, montp = _batch(name, POOL, seed=23)
    return (M.G1 if name == "g1" else M.G2), g, logs, normal, montp


def _cyclic(name, n, seed):
    """n points P_i = pool[i mod POOL], n random 320-bit scalars, and the
    model's sum k_i log(i mod POOL) G"""
    curve, g, logs, normal, montp = _pool(name)
    idx = np.arange(n) % POOL
    ks = np.random.default_rng(seed).integers(0, 1 << 64, size=(n, 5), dtype=np.uint64)
    # per pool point, the sum of its scalars: 32-bit halves summed exactly in
    # float64 (at most 481 terms below 2^32 each)
    halves = ks.view(np.uint32).reshape(n, 10)
    sums = [np.bincount(idx, weights=halves[:, h], minlength=POOL) for h in range(10)]
    e = sum(logs[j] * sum(int(sums[h][j]) << (32 * h) for h in range(10)) for j in range(POOL)) % M.R_ORDER
    return normal[idx], montp[idx], ks, curve.mul(e, curve.gen)


def _last_config():
    from tfhe_rs_b200 import _lib

    cfg = _lib.lib().b200_last_msm_config().decode()
    return {k: int(v) for k, v in re.findall(r"\b(c|windows|task|segments)=(\d+)", cfg)}


@pytest.mark.gpu
@pytest.mark.parametrize("name,n", PLAN_ROWS)
def test_msm_at_every_window_plan(name, n):
    """One MSM at the smallest n of each window size c, and at one less; the
    plan that ran is read back from b200_last_msm_config()."""
    c = _plan_c(n, C_MAX[name])
    normal, _, ks, expect = _cyclic(name, n, seed=n)
    assert _gpu_msm(name, normal, ks) == expect
    cfg = _last_config()
    assert cfg["c"] == c and cfg["windows"] == 320 // c + 1, cfg
    assert cfg["segments"] == min(1 << (c - 1), 64) and cfg["task"] == 8, cfg
    SEEN_C[name].add(c)
    COMPLETED_PLANS.add((name, n))


@pytest.mark.gpu
def test_window_plans_cover_every_c():
    """Runs after the plan table (same module): every c of each group ran."""
    if len(COMPLETED_PLANS) < len(PLAN_ROWS):
        pytest.skip("the plan table did not run in this session")
    assert SEEN_C == {"g1": set(range(4, 17)), "g2": set(range(4, 15))}, SEEN_C


@pytest.mark.gpu
@pytest.mark.parametrize("name,c", [(name, c) for name, cmax in C_MAX.items() for c in range(4, cmax + 1)])
def test_unmanaged_scratch_of_exactly_the_reported_size(name, c):
    """A scratch of exactly pippenger_scratch_size bytes, filled with a
    sentinel and followed by a sentinel guard: the result matches the model
    and the guard is untouched."""
    import torch

    from tfhe_rs_b200 import gpu, zk

    n = PLAN_THRESHOLDS[c]
    _, montp, ks, expect = _cyclic(name, n, seed=1000 + n)
    g = zk.G1 if name == "g1" else zk.G2
    streams = gpu.CudaStreams.new_single_gpu(0)
    need = zk.scratch_size(g, n)
    guard = 1 << 16
    buf = torch.full((need + guard,), 0xA5, dtype=torch.uint8, device=streams.device(0))
    torch.cuda.synchronize()
    raw = zk.msm_device(g, zk.to_device(montp, streams), zk.to_device(ks, streams), streams, scratch=buf[:need])
    assert _last_config()["c"] == c
    assert zk.normalized_to_affine(g, zk.normalize(g, raw)) == expect
    torch.cuda.synchronize()
    assert bool((buf[need:] == 0xA5).all()), "the MSM wrote past pippenger_scratch_size"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
@pytest.mark.parametrize("n", [7, 8, 9, 15, 16, 17, 63, 64, 65, 129])
def test_equal_scalars_at_task_and_tree_edges(name, n):
    """Every scalar equal: each window's digit puts all n points in one bucket,
    ceil(n / 8) tasks and log2 of that many tree passes."""
    from tfhe_rs_b200 import zk

    curve, g, logs, _, normal, _ = _batch(name, n)
    for k in ((1 << 299) + 12345, M.R_ORDER - 1, (1 << 320) - 1):
        assert _gpu_msm(name, normal, zk.scalars([k] * n)) == M.msm_by_logs(curve, [k] * n, logs), k


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g1", "g2"])
@pytest.mark.parametrize("c,groups", [(4, 8), (6, 32)])
def test_every_bucket_holds_nine_points(name, c, groups):
    """n = 9 groups: group j's scalar has digit j + 1 in every full window, so
    every non-empty bucket holds 9 points, two tasks each (8 + 1).  The task
    count is then within 10% of the plan's max_tasks bound."""
    from tfhe_rs_b200 import zk

    n = 9 * groups
    assert _plan_c(n, C_MAX[name]) == c
    W, B = 320 // c + 1, 1 << (c - 1)
    tasks = 2 * groups * (W - 1)
    max_tasks = n * W // 8 + min(W * B, n * W) + 1
    assert 0.9 * max_tasks < tasks <= max_tasks
    curve, g, logs, _, normal, _ = _batch(name, n)
    digit = [sum((j + 1) << (c * w) for w in range(W - 1)) for j in range(groups)]
    ks = [digit[i // 9] for i in range(n)]
    assert _gpu_msm(name, normal, zk.scalars(ks)) == M.msm_by_logs(curve, ks, logs)
    assert _last_config()["c"] == c
