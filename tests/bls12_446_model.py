"""Plain-integer model of BLS12-446 (the curve of tfhe-zk-pok's PKE v2): the
field constants derived from the BLS12 seed, Fp and Fp2 = Fp[u]/(u^2 + 1), the
affine group law of G1 (y^2 = x^3 + 1) and of its M-type twist G2
(y^2 = x^3 + (1 + u)), and a naive MSM.  Points are (x, y) tuples, the
identity is None; an Fp2 element is a (c0, c1) tuple."""
import json
import os

X = -0x600_8204000000020001
R_ORDER = X**4 - X**2 + 1
P = (X - 1) ** 2 * R_ORDER // 3 + X
assert ((X - 1) ** 2 * R_ORDER) % 3 == 0
MONT_R = 1 << 448
R2 = MONT_R * MONT_R % P
PINV = (-pow(P, -1, 1 << 64)) % (1 << 64)
G1_ORDER = P + 1 - (X + 1)  # #E(Fp): trace x + 1


def fp_inv(a):
    return pow(a, P - 2, P)


# ---- Fp2 ----
def f2_add(a, b):
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def f2_sub(a, b):
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def f2_neg(a):
    return (-a[0] % P, -a[1] % P)


def f2_mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def f2_inv(a):
    t = fp_inv((a[0] * a[0] + a[1] * a[1]) % P)
    return (a[0] * t % P, -a[1] * t % P)


class _Fp:
    zero, one = 0, 1
    add = staticmethod(lambda a, b: (a + b) % P)
    sub = staticmethod(lambda a, b: (a - b) % P)
    mul = staticmethod(lambda a, b: a * b % P)
    neg = staticmethod(lambda a: -a % P)
    inv = staticmethod(fp_inv)


class _Fp2:
    zero, one = (0, 0), (1, 0)
    add, sub, mul, neg, inv = (staticmethod(f) for f in (f2_add, f2_sub, f2_mul, f2_neg, f2_inv))


class Curve:
    def __init__(self, F, b, gen):
        self.F, self.b, self.gen = F, b, gen

    def on_curve(self, p):
        if p is None:
            return True
        F = self.F
        x, y = p
        return F.mul(y, y) == F.add(F.mul(F.mul(x, x), x), self.b)

    def neg(self, p):
        return None if p is None else (p[0], self.F.neg(p[1]))

    def add(self, p, q):
        F = self.F
        if p is None:
            return q
        if q is None:
            return p
        if p[0] == q[0]:
            if p[1] != q[1] or p[1] == F.zero:
                return None
            lam = F.mul(F.mul(F.add(F.add(p[0], p[0]), p[0]), p[0]), F.inv(F.add(p[1], p[1])))
        else:
            lam = F.mul(F.sub(q[1], p[1]), F.inv(F.sub(q[0], p[0])))
        x3 = F.sub(F.sub(F.mul(lam, lam), p[0]), q[0])
        return (x3, F.sub(F.mul(lam, F.sub(p[0], x3)), p[1]))

    def mul(self, k, p):
        if k < 0:
            k, p = -k, self.neg(p)
        acc = None
        while k:
            if k & 1:
                acc = self.add(acc, p)
            p = self.add(p, p)
            k >>= 1
        return acc

    def msm(self, scalars, points):
        acc = None
        for k, p in zip(scalars, points):
            acc = self.add(acc, self.mul(k, p))
        return acc


def _load_generators():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bls12_446_v1.json")) as f:
        g = json.load(f)
    g1 = (int(g["g1"]["x"]), int(g["g1"]["y"]))
    g2 = (tuple(int(v) for v in g["g2"]["x"]), tuple(int(v) for v in g["g2"]["y"]))
    return g1, g2


G1_GEN, G2_GEN = _load_generators()
G1 = Curve(_Fp, 1, G1_GEN)
G2 = Curve(_Fp2, (1, 1), G2_GEN)


def known_multiples(curve, count, rng):
    """(a_i, a_i * G): points whose discrete logs are known, so an MSM over them
    is one scalar multiplication by sum k_i a_i mod r.  Successive points are
    built by one addition each."""
    step = rng.randrange(1, R_ORDER)
    a0 = rng.randrange(1, R_ORDER)
    logs, pts = [], []
    p, ps, a = curve.mul(a0, curve.gen), curve.mul(step, curve.gen), a0
    for _ in range(count):
        logs.append(a)
        pts.append(p)
        p, a = curve.add(p, ps), (a + step) % R_ORDER
    return logs, pts


def msm_by_logs(curve, scalars, logs, infinity=()):
    """sum k_i (a_i G) computed as (sum k_i a_i mod r) G; indexes in `infinity`
    hold the identity instead of a_i G."""
    skip = set(infinity)
    e = sum(k * a for i, (k, a) in enumerate(zip(scalars, logs)) if i not in skip) % R_ORDER
    return curve.mul(e, curve.gen)
