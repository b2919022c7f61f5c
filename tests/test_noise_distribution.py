"""Noise and failure probability of the GPU KS -> PBS and compression atomic
patterns, against the reference's noise model (tests/noise_model.py).

Every bit circuit, radix circuit and compressed list rests on one claim: a LUT
input sum c_i w_i + c_0 over PBS outputs with sum |c_i| <= 5, keyswitched and
then modulus-switched inside the PBS, decodes wrongly with the parameter set's
own p_fail.  Decryption cannot see a p_fail of 2^-129 become 2^-40, and a
variance bound cannot see a bias, which the x5 dot product turns straight into
lost margin.  So this file measures the chains the way tfhe-rs measures its own
GPU backend (integer/gpu/server_key/radix/tests_noise_distribution/
br_dp_ks_ms.rs and br_dp_packingks_ms.rs):

* CPU: the restated model lands on the published log2 p_fail of both parameter
  sets and on the reference's compression figure; broken models do not; the
  statistics agree with scipy; noiseless grid inputs switch exactly.
* GPU (classic P22 and multi-bit g = 4 keys): mean and variance after every
  stage (BR, DP, KS, MS; BR, DP, packing KS, storage MS) against the model,
  with tfhe-rs' acceptance rules; the p_fail at an inflated precision over
  10^6 runs, counted by decryption and by a second PBS; and controls with a
  wrong switch that must fail the same check.
"""
import math

import numpy as np
import pytest

from tests import compression_model as CM
from tests import noise_model as M

# log2_p_fail of the parameter files, written as literals:
# shortint/parameters/v1_4/classic/tuniform/p_fail_2_minus_128/ks_pbs.rs (P22) and
# shortint/parameters/v1_1/multi_bit/tuniform/p_fail_2_minus_128/ks_pbs_gpu.rs (g = 4)
PUBLISHED_LOG2_PFAIL = {"classic": -129.581, "mb4": -134.345}
# The parameter files print log2_p_fail to three decimals, so a faithful
# restatement lands within 0.0005 of them; 0.002 leaves room for the last-digit
# differences of f64 arithmetic and nothing more.  Every broken model below
# moves the result by at least 0.9 bit.
LOG2_PFAIL_TOL = 0.002
MAX_NOISE_LEVEL = 5  # MaxNoiseLevel of both 2_2 sets
# shortint/server_key/tests/noise_distribution/utils/mod.rs:1008-1018: the
# reference's own compression figure (P22 with its compression parameters)
REF_COMPRESSION_VARIANCE = 1.0216297411906617e-05
REF_COMPRESSION_LOG2_PFAIL = -280.4295428516361


def _params(kind):
    from oracle import csprng
    from oracle import oracle as O

    return {"classic": O.PARAM_MESSAGE_2_CARRY_2_KS_PBS,
            "mb4": csprng.PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS}[kind]


def _comp_params(kind):
    return {"classic": CM.COMP_PARAM_MESSAGE_2_CARRY_2_KS_PBS_TUNIFORM_2M128,
            "mb4": CM.COMP_PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2_KS_PBS_TUNIFORM_2M128}[kind]


# ---------------------------------------------------------------------------
# CPU: the model
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["classic", "mb4"])
def test_chain_reproduces_published_log2_pfail(kind):
    """BR -> DP(x5) -> KS -> MS at max noise level 5 gives the optimizer's
    log2_p_fail of the parameter file (see LOG2_PFAIL_TOL for the tolerance)."""
    got = M.chain_log2_pfail(_params(kind), MAX_NOISE_LEVEL)
    assert abs(got - PUBLISHED_LOG2_PFAIL[kind]) <= LOG2_PFAIL_TOL, got


@pytest.mark.parametrize("kind,control", [("classic", "scalar_4"), ("classic", "no_keyswitch"),
                                          ("classic", "standard_switch"), ("mb4", "scalar_4"),
                                          ("mb4", "no_keyswitch")])
def test_broken_chains_miss_published_log2_pfail(kind, control):
    """Negative controls: each broken chain leaves the tolerance."""
    P = _params(kind)
    got = {"scalar_4": lambda: M.chain_log2_pfail(P, 4),
           "no_keyswitch": lambda: M.chain_log2_pfail(P, MAX_NOISE_LEVEL, with_ks=False),
           "standard_switch": lambda: M.chain_log2_pfail(P, MAX_NOISE_LEVEL, ms=M.MS_STANDARD)}[control]()
    assert abs(got - PUBLISHED_LOG2_PFAIL[kind]) > 0.9, got


def test_packing_chain_reproduces_reference_compression_figure():
    """BR -> DP(x carry modulus) -> packing KS -> storage MS with P22 and its
    compression parameters gives the reference's variance and log2 p_fail at
    the compression precision (message 4, carry 1), and a broken chain does
    not."""
    P, cp = _params("classic"), _comp_params("classic")
    v = M.br_dp_packing_ks_ms(P, cp, 4)["ms"].variance
    assert v == pytest.approx(REF_COMPRESSION_VARIANCE, rel=1e-12)
    lp = math.log2(M.expected_pfail_for_precision(M.precision_with_padding(4, 1), v))
    assert lp == pytest.approx(REF_COMPRESSION_LOG2_PFAIL, abs=1e-6)
    assert M.br_dp_packing_ks_ms(P, cp, 4, lwe_to_pack=1)["ms"].variance < 0.8 * v
    assert M.br_dp_packing_ks_ms(P, cp, 8)["ms"].variance != pytest.approx(v, rel=1e-3)


def test_secure_minimum_is_the_parameter_sets_noise():
    """The secure-noise minimum at the small and big dimensions is the
    variance of the TUniform bounds the parameter sets encrypt with (45 at
    n = 918 and 920, 17 at k N = 2048), up to its 2^(4.44 - 128) term."""
    for kind in ("classic", "mb4"):
        P = _params(kind)
        assert M.minimal_lwe_variance_tuniform(P.n) == pytest.approx(M.tuniform_variance(P.lwe_noise_log2), rel=1e-9)
        assert M.minimal_lwe_variance_tuniform(P.big_n) == pytest.approx(M.tuniform_variance(P.glwe_noise_log2),
                                                                         rel=1e-9)


def test_pfail_arithmetic():
    """precision_with_padding and equivalent_pfail_gaussian_noise: tfhe-rs'
    inflation of the carry modulus to 2^5 takes P22 from 5 to 8 bits and its
    2^-129.58 to the chain's own p_fail at 8 bits, and back."""
    P = _params("classic")
    assert M.precision_with_padding(4, 4) == 5 and M.precision_with_padding(4, 32) == 8
    assert M.precision_with_padding(64, 1) == 7
    v = M.br_dp_ks_ms(P, 25)["ms"].variance
    orig = M.expected_pfail_for_precision(5, v)
    new = M.equivalent_pfail_gaussian_noise(5, orig, 8)
    assert new == pytest.approx(M.expected_pfail_for_precision(8, v), rel=1e-9)
    assert new == pytest.approx(0.0992, abs=1e-4)
    assert math.log2(M.equivalent_pfail_gaussian_noise(8, new, 5)) == pytest.approx(math.log2(orig), abs=1e-6)
    G = _params("mb4")
    assert M.expected_pfail_for_precision(8, M.br_dp_ks_ms(G, 25)["ms"].variance) == pytest.approx(0.0930, abs=1e-4)


def test_statistics_agree_with_scipy():
    """The 99 % intervals: Clopper-Pearson against binomtest's exact interval,
    the mean interval's z against norm, the variance interval against chi2
    quantiles, and both Gaussian intervals cover 99 % of repeated draws."""
    from scipy import stats

    for n, k in [(1000, 1), (1000, 37), (10 ** 6, 99160), (10 ** 6, 221102)]:
        ref = stats.binomtest(k, n).proportion_ci(confidence_level=0.99, method="exact")
        lo, hi = M.clopper_pearson_ci(n, k)
        assert lo == pytest.approx(ref.low, rel=1e-9) and hi == pytest.approx(ref.high, rel=1e-9)
    lo, hi = M.gaussian_mean_ci(10_000, 0.0, 1.0)
    assert hi == pytest.approx(stats.norm.ppf(0.995) / 100.0, rel=1e-12) and lo == -hi
    lo, hi = M.gaussian_variance_ci(65536, 2.0)
    assert lo == pytest.approx(65535 * 2.0 / stats.chi2.isf(0.005, 65535), rel=1e-12)
    assert hi == pytest.approx(65535 * 2.0 / stats.chi2.ppf(0.005, 65535), rel=1e-12)
    rng = np.random.default_rng(99)
    draws = rng.normal(0.5, 2.0, (4000, 300))
    m_in = v_in = 0
    for x in draws:
        a, b = M.gaussian_mean_ci(x.size, x.mean(), x.std(ddof=1))
        m_in += a <= 0.5 <= b
        a, b = M.gaussian_variance_ci(x.size, M.sample_variance(x))
        v_in += a <= 4.0 <= b
    # 4000 trials at 0.99: the binomial 99.9 % range is about [3946, 3985]
    assert 3940 <= m_in <= 3990 and 3940 <= v_in <= 3990, (m_in, v_in)


def test_normality_check_restatement():
    """Shapiro-Francia: W' is the squared correlation of the sorted sample with
    the Blom scores; Gaussian samples pass at alpha 0.01 and uniform, Laplace
    and bimodal ones fail, where scipy's Shapiro-Wilk decides the same."""
    from scipy import stats

    rng = np.random.default_rng(7)
    x = rng.normal(size=5000)
    w, p, ok = M.normality_test(x)
    blom = stats.norm.ppf((np.arange(1, 5001) - 0.375) / 5000.25)
    assert w == pytest.approx(np.corrcoef(np.sort(x), blom)[0, 1] ** 2, rel=1e-12)
    assert ok and stats.shapiro(x).pvalue > 0.01
    for bad in (rng.uniform(size=5000), rng.laplace(size=5000),
                np.concatenate([rng.normal(-2, 1, 2500), rng.normal(2, 1, 2500)])):
        assert not M.normality_test(bad)[2] and stats.shapiro(bad).pvalue < 0.01
    with pytest.raises(AssertionError):
        M.normality_test(rng.normal(size=5001))


def test_acceptance_rules():
    """mean_and_variance_check and pfail_check decide as tfhe-rs does."""
    rng = np.random.default_rng(3)
    x = rng.normal(0.0, 1.0, 65536)
    v = M.sample_variance(x)
    assert M.mean_and_variance_check(x, 0.0, 2.0 * v, 0.5)[0]  # smaller, secure
    assert not M.mean_and_variance_check(x, 0.0, 2.0 * v, 1.5)[0]  # smaller, not secure
    assert M.mean_and_variance_check(x, 0.0, 0.995 * v, 0.0)[0]  # larger, inside the interval
    assert not M.mean_and_variance_check(x, 0.0, 0.9 * v, 0.0)[0]  # larger, outside it
    assert not M.mean_and_variance_check(x + 0.05, 0.0, 2.0 * v, 0.0)[0]  # a bias of 0.05 sigma
    # eight keys, each with its own offset: the keys are the units of the mean
    keyed = x + np.repeat(rng.normal(0.0, 0.03, 8), x.size // 8)
    assert not M.mean_and_variance_check(keyed, 0.0, 2.0 * v, 0.5)[0]
    assert M.mean_and_variance_check(keyed, 0.0, 2.0 * v, 0.5, groups=8)[0]
    assert not M.mean_and_variance_check(keyed + 0.2, 0.0, 2.0 * v, 0.5, groups=8)[0]
    assert M.pfail_check(10 ** 6, 0, 0.1, 8, 5)[0]
    assert M.pfail_check(10 ** 6, 90_000, 0.1, 8, 5)[0]
    assert M.pfail_check(10 ** 6, 100_500, 0.1, 8, 5)[0]
    ok, rep = M.pfail_check(10 ** 6, 102_000, 0.1, 8, 5)
    assert not ok and rep["ci"][0] > 0.1
    ok, rep = M.pfail_check(10 ** 6, 99_160, 0.09916, 8, 5)
    assert ok and rep["equivalent_log2_pfail"] == pytest.approx(-129.58, abs=0.05)


@pytest.mark.parametrize("centered", [False, True])
def test_grid_inputs_switch_exactly(oracle, centered):
    """A noiseless PBS input -- mask on the 2N grid, body <a, s> + Delta m
    exactly -- switches to exactly Delta m with either switch.  The centered
    correction is then exactly minus half a step of 1/(2N), the -1/(4N) mean
    the model expects after that switch."""
    P = _params("classic")
    log_mod = P.log_2N
    shift = 64 - log_mod
    rng = np.random.default_rng(11)
    s = rng.integers(0, 2, P.n, dtype=np.uint64)
    for m in range(P.p):
        a = rng.integers(0, 1 << log_mod, P.n, dtype=np.uint64) << np.uint64(shift)
        with np.errstate(over="ignore"):
            body = (a * s).sum(dtype=np.uint64) + np.uint64(m * P.delta)
        ct = np.concatenate([a, [body]]).astype(np.uint64)
        sw = oracle.modulus_switch_lwe(ct, log_mod, centered).astype(np.int64)
        phase = (sw[-1] - int((sw[:-1] * s.astype(np.int64)).sum())) % (1 << log_mod)
        assert phase == (m * P.delta) >> shift
        corr = int(oracle.lib().orc_centered_ms_body_correction(oracle.u64p(ct), P.n, log_mod))
        assert corr == 2 ** 64 - 2 ** (shift - 1)
        assert -(2 ** (shift - 1)) / 2.0 ** 64 == M.expected_average_after_ms(M.MS_CENTERED, P.N)


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
SAMPLES = 1 << 16  # per stage and row, as tfhe-rs' 1000 x 16 messages, rounded up
PFAIL_RUNS = 10 ** 6
CHUNK = 1 << 16
# DP rows over the slots x0..x4 of one instance, each an independent PBS
# output: tfhe-rs' case, the compiler's heaviest row shapes, a 5-wire parity
DP_ROWS = {"5x": [(0, 5)], "3x+y+z": [(0, 3), (1, 1), (2, 1)], "3cur+prev": [(0, 3), (1, 1)],
           "parity5": [(s, 1) for s in range(5)]}
INFLATED_PRECISION = 8  # carry modulus 2^5: message 4 x carry 32, with padding
COMP_INFLATED_PRECISION = 7  # compression: message 64, carry 1


def _report(**kw):
    """One JSON line per measurement (shown with pytest -s)."""
    import json

    print(json.dumps(kw, default=float))


class _Rig:
    """Keys of one parameter set on the GPU, and the stages of the chain as
    raw C-ABI calls on torch buffers of int64 words."""

    def __init__(self, kind, oracle, seed):
        import torch

        from tfhe_rs_b200 import _lib, gpu, server_key

        self.kind, self.P = kind, _params(kind)
        P = self.P
        self.keys = oracle.keygen(P, seed)
        self.torch, self.L, self.gpu = torch, _lib.lib(), gpu
        self.streams = gpu.CudaStreams.new_single_gpu(0)
        self.skey = server_key.upload_server_key(
            self.keys.bsk, self.keys.ksk, n=P.n, k=P.k, N=P.N, pbs_base_log=P.pbs_base_log, pbs_level=P.pbs_level,
            ks_base_log=P.ks_base_log, ks_level=P.ks_level, grouping_factor=P.grouping_factor,
            centered_ms=P.centered_ms, streams=self.streams)
        self.dev = self.streams.device(0)
        self.s_small = torch.from_numpy(self.keys.lwe_sk.astype(np.int64)).to(self.dev)
        self.s_big = torch.from_numpy(self.keys.glwe_sk.astype(np.int64)).to(self.dev)
        self.gen = torch.Generator(device=self.dev)
        self.gen.manual_seed(seed)

    def sp(self):
        """The stream of the C calls.  torch work runs on its own stream, so
        the device is synchronised before every launch and after it."""
        self.torch.cuda.synchronize()
        return self.streams.ptr(0)

    def grid_inputs(self, count):
        """encrypt_noiseless_pbs_input_dyn_lwe of message 0: mask words uniform
        on the 2N grid, body <a, s> exactly (centered representatives, so
        every product fits an int64)."""
        torch, P = self.torch, self.P
        half = 1 << (P.log_2N - 1)
        r = torch.randint(-half, half, (count, P.n), generator=self.gen, device=self.dev, dtype=torch.int64)
        dot = (r * self.s_small).sum(1)
        body = torch.remainder(dot + half, 2 * half) - half
        step = 1 << (64 - P.log_2N)
        return torch.cat([r * step, (body * step)[:, None]], 1).contiguous()

    def lut(self, precision):
        from tfhe_rs_b200 import algorithms

        p = 1 << (precision - 1)
        lut = algorithms.generate_programmable_bootstrap_glwe_lut(self.P.N, self.P.k + 1, p, (1 << 63) // p,
                                                                  lambda x: x)
        return self.gpu.CudaGlweCiphertextList.from_glwe_ciphertext_list(lut, self.P.k, self.P.N, self.streams)

    def pbs(self, d_in, lut, centered=None):
        """One KS-less PBS of every row of d_in (count x (n + 1)); `centered`
        overrides the classic key's switch."""
        import dataclasses

        gpu, P = self.gpu, self.P
        count = d_in.shape[0]
        cts = gpu.CudaLweCiphertextList(gpu.CudaVec(d_in.reshape(-1), np.uint64), P.n, count)
        key = self.skey
        if centered is not None and not key.multi_bit:
            conf = gpu.CudaModulusSwitchNoiseReductionConfiguration.CENTERED if centered else None
            key = dataclasses.replace(key, bsk=dataclasses.replace(key.bsk, ms_noise_reduction_configuration=conf))
        self.torch.cuda.synchronize()
        out = key.bootstrap(cts, lut)
        self.streams.synchronize()
        self.pbs_kernel = self.L.b200_last_pbs_kernel().decode()
        return out.d_vec.t.reshape(count, P.big_n + 1)

    def linear(self, pool, inst, rows):
        """b200_lwe_linear_combination_64_async: row r of instance i is
        sum c * pool[slot * inst + i]; outputs row-major, instance-minor."""
        torch = self.torch
        offs, slots, coefs = [0], [], []
        for terms in rows:
            slots += [s for s, _ in terms]
            coefs += [c for _, c in terms]
            offs.append(len(slots))
        up = lambda a, dt: torch.tensor(a, dtype=dt, device=self.dev)  # noqa: E731
        d_offs, d_slots, d_coefs = up(offs, torch.int32), up(slots, torch.int32), up(coefs, torch.int64)
        d_body = torch.zeros(len(rows) * inst, dtype=torch.int64, device=self.dev)
        out = torch.empty((len(rows) * inst, self.P.big_n + 1), dtype=torch.int64, device=self.dev)
        self.L.b200_lwe_linear_combination_64_async(
            self.sp(), 0, out.data_ptr(), pool.data_ptr(), self.P.big_n, 0, inst, len(rows), 0, d_offs.data_ptr(),
            d_slots.data_ptr(), d_coefs.data_ptr(), d_body.data_ptr())
        self.streams.synchronize()
        return out

    def keyswitch(self, d_big):
        torch, P = self.torch, self.P
        count = d_big.shape[0]
        out = torch.empty((count, P.n + 1), dtype=torch.int64, device=self.dev)
        idx = torch.arange(count, dtype=torch.int64, device=self.dev)
        self.L.cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
            self.sp(), 0, out.data_ptr(), idx.data_ptr(), d_big.data_ptr(), idx.data_ptr(),
            self.skey.ksk.d_vec.as_c_ptr(), P.big_n, P.n, P.ks_base_log, P.ks_level, count)
        self.streams.synchronize()
        self.ks_kernel = self.L.b200_last_keyswitch_kernel().decode()
        return out

    def switch(self, d_small, centered):
        """cuda_centered_modulus_switch_64_async (one LWE per call) or
        cuda_modulus_switch_64_async (every word) to 2N."""
        torch, P = self.torch, self.P
        out = torch.empty_like(d_small)
        if centered:
            w = (P.n + 1) * 8
            src, dst = d_small.data_ptr(), out.data_ptr()
            f = self.L.cuda_centered_modulus_switch_64_async
            sp = self.sp()
            for i in range(d_small.shape[0]):
                f(sp, 0, dst + i * w, src + i * w, P.n, P.log_2N)
        else:
            self.L.cuda_modulus_switch_64_async(self.sp(), 0, out.data_ptr(), d_small.data_ptr(), d_small.numel(),
                                                P.log_2N)
        self.streams.synchronize()
        return out

    def phase(self, d, key, log_mod=64):
        """b - <a, s> of every row, wrapping, in int64 (mod 2^log_mod,
        centered, when the words are switched values)."""
        torch = self.torch
        parts = [c[:, -1] - (c[:, :-1] * key).sum(1) for c in d.split(8192)]
        ph = torch.cat(parts)
        if log_mod < 64:
            half = 1 << (log_mod - 1)
            ph = torch.remainder(ph + half, 2 * half) - half
        return ph

    def noise(self, d, key, log_mod=64):
        """Torus noise of message-0 ciphertexts, as float64 numpy."""
        return self.phase(d, key, log_mod).double().cpu().numpy() / 2.0 ** log_mod


KEYS = 8  # independent key sets per parameter set
_RIGS = {}


def _rigs(kind, oracle):
    """KEYS independent key sets of one parameter set, made once per module.
    tfhe-rs draws a fresh client key for every sample: a fixed key adds a
    fixed offset to the noise (its key errors times the non-zero mean of the
    decomposition digits of the LUT), so one key cannot speak for the mean."""
    if kind not in _RIGS:
        base = {"classic": 0x401E_C1A5, "mb4": 0x401E_4B04}[kind]
        _RIGS[kind] = [_Rig(kind, oracle, base + 0x1000 * j) for j in range(KEYS)]
    return _RIGS[kind]


# The PBS output's variance bound of the rest of the suite (DESIGN section 5):
# 1.0625 x the formula, plus 4 standard errors of a sample variance.
PBS_VARIANCE_BOUND = 1.0625


def _check(kind, stage, row, parts, expected, secure_dim, normality=False):
    """tfhe-rs' mean_and_variance_check on the samples of every key (equal
    blocks, key after key), and its normality check on 5000 samples drawn
    across the keys.  tfhe-rs checks the variance after the switch only.  The
    PBS output and its dot products (stages "br" and "dp") keep tfhe-rs' mean
    rule but take the suite's PBS variance bound: on classic P22 the formula
    is about 2 % below what both these kernels and the CPU oracle measure
    (DESIGN section 5), which the chi^2 interval of 2^16 samples resolves."""
    x = np.concatenate(parts)
    ok, rep = M.mean_and_variance_check(x, expected.mean, expected.variance, M.minimal_lwe_variance_tuniform(secure_dim),
                                        groups=len(parts))
    if stage in ("br", "dp"):
        bound = PBS_VARIANCE_BOUND * (1.0 + 4.0 * math.sqrt(2.0 / (x.size - 1)))
        rep["variance_ok"] = rep["variance_ratio"] <= bound
        ok = rep["mean_ok"] and rep["variance_ok"]
    rep["key_means"] = [float(p.mean()) for p in parts]
    if normality:
        w, p, n_ok = M.normality_test(x[::-(-x.size // 5000)][:5000])
        rep.update(normality_p=p, normality_ok=n_ok)
        ok = ok and n_ok
    _report(set=kind, stage=stage, row=row, ok=ok, **rep)
    return ok


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["classic", "mb4"])
def test_gpu_br_dp_ks_ms_noise(kind, oracle):
    """BR (identity PBS of noiseless grid inputs) -> DP (the bit circuits'
    linear-combination kernel, every row shape) -> KS -> MS: mean and variance
    of every stage against the model under tfhe-rs' acceptance rule, and the
    normality of the noise before the switch.  Classic: the centered switch of
    cuda_centered_modulus_switch_64_async and, as a second model, the plain
    cuda_modulus_switch_64_async.  Multi-bit: the switch happens inside the
    PBS and is covered by the p_fail test."""
    rigs = _rigs(kind, oracle)
    torch, P = rigs[0].torch, rigs[0].P
    S = SAMPLES // len(rigs)
    noise = {}

    def add(stage, row, x):
        noise.setdefault((stage, row), []).append(x)

    for rig in rigs:
        lut = rig.lut(5)
        pool = torch.cat([rig.pbs(rig.grid_inputs(S), lut) for _ in range(5)])  # slot s of instance i: row s S + i
        add("br", "-", rig.noise(pool, rig.s_big))
        dp_out = rig.linear(pool, S, list(DP_ROWS.values()))
        del pool
        ks_out = rig.keyswitch(dp_out)
        switched = {}
        if not rig.skey.multi_bit:
            switched = {M.MS_CENTERED: rig.switch(ks_out, True), M.MS_STANDARD: rig.switch(ks_out, False)}
        for r, name in enumerate(DP_ROWS):
            sl = slice(r * S, (r + 1) * S)
            add("dp", name, rig.noise(dp_out[sl], rig.s_big))
            add("ks", name, rig.noise(ks_out[sl], rig.s_small))
            for ms, d in switched.items():
                add("ms_" + ms, name, rig.noise(d[sl], rig.s_small, P.log_2N))
        del dp_out, ks_out, switched
    _report(set=kind, pbs_kernel=rigs[0].pbs_kernel, keyswitch_kernel=rigs[0].ks_kernel)
    # the standard switch's model for these keys' mean Hamming weight
    ms_dim = {M.MS_STANDARD: 2.0 * float(np.mean([r.keys.lwe_sk.sum() for r in rigs]))}
    failures = []
    for (stage, row), parts in noise.items():
        sum_c2 = 1.0 if stage == "br" else float(sum(c * c for _, c in DP_ROWS[row]))
        ms = stage[3:] if stage.startswith("ms_") else None
        model = M.br_dp_ks_ms(P, sum_c2, ms=ms, ms_dimension=ms_dim.get(ms))[stage[:2]]
        secure = P.big_n if stage in ("br", "dp") else P.n
        if not _check(kind, stage, row, parts, model, secure, normality=stage == "ks"):
            failures.append((stage, row))
    assert rigs[0].ks_kernel.startswith("ks_"), rigs[0].ks_kernel
    assert not failures, failures


def _pfail_runs(rigs, pbs_switches=(None,), switch_kinds=()):
    """PFAIL_RUNS chains of message 0 at the inflated precision, spread over
    the keys: BR -> 5x -> KS, then the failures counted by a second PBS (one
    bit-circuit layer) with each requested switch (None: the key's own) and by
    decrypting each requested stand-alone switch of the KS output."""
    P = rigs[0].P
    torch = rigs[0].torch
    half_box = 1 << (P.log_2N - INFLATED_PRECISION - 1)  # 2^-(precision + 1) of the torus, in switched units
    delta = 1 << (64 - INFLATED_PRECISION)
    fails = {**{("pbs", c): 0 for c in pbs_switches}, **{k: 0 for k in switch_kinds}}
    per_key = PFAIL_RUNS // len(rigs)
    assert per_key * len(rigs) == PFAIL_RUNS
    for rig in rigs:
        lut = rig.lut(INFLATED_PRECISION)
        done = 0
        while done < per_key:
            c = min(CHUNK, per_key - done)
            br = rig.pbs(rig.grid_inputs(c), lut)
            ks = rig.keyswitch(rig.linear(br, c, [DP_ROWS["5x"]]))
            del br
            for centered in pbs_switches:
                ph = rig.phase(rig.pbs(ks, lut, centered=centered), rig.s_big)
                # decode(pt, delta) mod p != 0 with p = 2^(precision - 1) values
                dec = torch.div(ph + delta // 2, delta, rounding_mode="floor")
                fails[("pbs", centered)] += int((torch.remainder(dec, 1 << (INFLATED_PRECISION - 1)) != 0).sum())
            for kind in switch_kinds:
                sw = rig.phase(rig.switch(ks, kind == M.MS_CENTERED), rig.s_small, P.log_2N)
                fails[kind] += int(((sw >= half_box) | (sw < -half_box)).sum())
            done += c
    return fails


def _pfail_verdict(kind, label, fails, ms):
    P = _params(kind)
    v = M.br_dp_ks_ms(P, float(MAX_NOISE_LEVEL ** 2), ms=ms)["ms"].variance
    expected_new = M.expected_pfail_for_precision(INFLATED_PRECISION, v)
    ok, rep = M.pfail_check(PFAIL_RUNS, fails, expected_new, INFLATED_PRECISION, 5)
    rep["original_expected_log2_pfail"] = math.log2(M.expected_pfail_for_precision(5, v))
    _report(set=kind, check="pfail", count=label, ok=ok, **rep)
    return ok


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["classic", "mb4"])
def test_gpu_br_dp_ks_ms_pfail(kind, oracle):
    """p_fail with tfhe-rs' inflated carry modulus (2^5: precision 5 -> 8), 10^6
    chains of message 0, failures counted by a second PBS (every key) and by
    decrypting the switched LWE (classic).  Each count passes pfail_check's
    rule against the model.  On the classic key the same KS outputs also run
    through the standard switch, in the second PBS and in the stand-alone
    entry point: the model puts that p_fail (0.221) far outside the 99 %
    interval of the centered one (0.099), and the check must fail it."""
    import time

    rigs = _rigs(kind, oracle)
    multi = rigs[0].skey.multi_bit
    t0 = time.perf_counter()
    if multi:
        fails = _pfail_runs(rigs)
    else:
        fails = _pfail_runs(rigs, (None, False), (M.MS_CENTERED, M.MS_STANDARD))
    _report(set=kind, check="pfail_wall_s", seconds=time.perf_counter() - t0)
    ok = [_pfail_verdict(kind, "second_pbs", fails[("pbs", None)], M.ms_kind(rigs[0].P))]
    if not multi:
        ok.append(_pfail_verdict(kind, "decrypt_centered", fails[M.MS_CENTERED], M.MS_CENTERED))
        # controls: the standard switch judged against the centered chain's model must fail
        ok.append(not _pfail_verdict(kind, "decrypt_standard_control", fails[M.MS_STANDARD], M.MS_CENTERED))
        ok.append(not _pfail_verdict(kind, "second_pbs_standard_control", fails[("pbs", False)], M.MS_CENTERED))
    assert all(ok), ok


@pytest.mark.gpu
def test_gpu_multibit_tie_rule_control(oracle):
    """The reference tie rule on g = 4 (b200_set_multibit_tie_rule(1)) as a
    sensitivity control.  It only changes the blind rotation, so the model
    of the p_fail it causes is the chain with the BR variance measured under
    that rule.  The control is run only where that model puts the p_fail
    beyond the 99 % interval of the shipped chain's expected value at 10^6
    runs, and then the check must fail it."""
    rigs = _rigs("mb4", oracle)
    P, L = rigs[0].P, rigs[0].L
    L.b200_set_multibit_tie_rule(1)
    try:
        S = SAMPLES // len(rigs)
        br = M.sample_variance(np.concatenate([r.noise(r.pbs(r.grid_inputs(S), r.lut(5)), r.s_big) for r in rigs]))
        model = M.br_dp_ks_ms(P, 25.0)
        v = model["ms"].variance + 25.0 * (br - model["br"].variance)
        predicted = M.expected_pfail_for_precision(INFLATED_PRECISION, v)
        expected = M.expected_pfail_for_precision(INFLATED_PRECISION, model["ms"].variance)
        lo, _ = M.clopper_pearson_ci(PFAIL_RUNS, round(predicted * PFAIL_RUNS))
        keep = lo > expected
        _report(set="mb4", check="tie_rule_control", br_variance_ratio=br / model["br"].variance,
                predicted_pfail=predicted, expected_pfail=expected, predicted_ci_low=lo, kept=keep)
        if keep:
            fails = _pfail_runs(rigs)
            assert not _pfail_verdict("mb4", "second_pbs_tie_rule_control", fails[("pbs", None)], M.MS_MULTI_BIT)
    finally:
        L.b200_set_multibit_tie_rule(0)


def _glwe_phase(words, sk, k, N, log_mod):
    """Body minus sum_j A_j * S_j in Z_{2^log_mod}[X]/(X^N + 1) of G GLWEs given
    as (G, (k + 1) N) integer words; returns (G, N) centered int64."""
    words = np.asarray(words, dtype=np.uint64)
    acc = words[:, k * N:].copy()
    idx = np.arange(N)
    diff = idx[:, None] - idx[None, :]
    with np.errstate(over="ignore"):
        for j in range(k):
            s = sk[j * N:(j + 1) * N].astype(np.uint64)
            # negacyclic matrix: out[t] = sum_i a[i] s[t - i], s[t - i + N] negated
            mat = np.where(diff >= 0, s[diff % N], np.uint64(0) - s[diff % N])
            acc -= words[:, j * N:(j + 1) * N] @ mat.T
    mod = 1 << log_mod
    ph = (acc & np.uint64(mod - 1)).astype(np.int64) if log_mod < 64 else acc.view(np.int64)
    if log_mod < 64:
        ph = np.where(ph >= mod // 2, ph - mod, ph)
    return ph


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["classic", "mb4"])
def test_gpu_br_dp_packing_ks_ms(kind, oracle):
    """BR -> DP(x message modulus, the engine's compression scaling) ->
    packing KS -> storage MS on real GPU PBS outputs: the GLWE of
    cuda_packing_keyswitch_lwe_list_to_glwe_64_async and the list of
    b200_compress_lwe_ciphertexts_64_async, every coefficient decrypted under
    the compression GLWE key, mean and variance against the model
    (br_dp_packingks_ms.rs), normality before the switch; then the p_fail at
    the inflated compression precision (message 64, carry 1) over 10^6 stored
    coefficients.  Each key set has its own compression key."""
    import ctypes as C

    rigs = _rigs(kind, oracle)
    torch, P, L = rigs[0].torch, rigs[0].P, rigs[0].L
    cp = _comp_params(kind)
    lpg, W = cp.lwe_per_glwe, cp.words_per_glwe
    model = M.br_dp_packing_ks_ms(P, cp, 4)
    S = SAMPLES // len(rigs)
    per_key = -(-PFAIL_RUNS // (lpg * len(rigs))) * lpg  # whole GLWEs: 10^6 rounded up
    half_box = 1 << (cp.storage_log_modulus - COMP_INFLATED_PRECISION - 1)
    noise = {"dp": [], "packing_ks": [], "storage_ms": []}
    fails = 0
    for j, rig in enumerate(rigs):
        comp_sk = np.random.default_rng(0xC0DE + j).integers(0, 2, cp.big_n, dtype=np.uint64)
        d_pksk = rig.gpu.CudaVec.from_cpu_async(CM.gen_packing_ksk(0x9AC7 + j, rig.keys.glwe_sk, comp_sk, cp),
                                                rig.streams)
        lut = rig.lut(5)

        def compress(br):
            g = br.shape[0] // lpg
            packed = torch.empty(g * W, dtype=torch.int64, device=rig.dev)
            L.b200_compress_lwe_ciphertexts_64_async(rig.sp(), 0, packed.data_ptr(), br.data_ptr(), br.shape[0],
                                                     P.big_n, 4, d_pksk.as_c_ptr(), cp.k, cp.N, cp.ks_base_log,
                                                     cp.ks_level, lpg, cp.storage_log_modulus)
            rig.streams.synchronize()
            words = packed.cpu().numpy().view(np.uint64)
            fields = CM.unpack_integers(words, cp.storage_log_modulus, g * (cp.big_n + cp.N))
            return _glwe_phase(fields.reshape(g, -1), comp_sk, cp.k, cp.N, cp.storage_log_modulus).reshape(-1)

        br = rig.pbs(rig.grid_inputs(S), lut)
        dp = rig.linear(br, S, [[(0, 4)]])
        buf = C.POINTER(C.c_int8)()
        L.scratch_cuda_packing_keyswitch_lwe_list_to_glwe_64_async(rig.sp(), 0, C.byref(buf), P.big_n, cp.k, cp.N,
                                                                   lpg, True)
        glwes = torch.empty((S // lpg, (cp.k + 1) * cp.N), dtype=torch.int64, device=rig.dev)
        try:
            for g in range(S // lpg):
                L.cuda_packing_keyswitch_lwe_list_to_glwe_64_async(
                    rig.sp(), 0, glwes[g].data_ptr(), dp[g * lpg].data_ptr(), d_pksk.as_c_ptr(), buf, P.big_n,
                    cp.k, cp.N, cp.ks_base_log, cp.ks_level, lpg)
            rig.streams.synchronize()
        finally:
            L.cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_64(rig.sp(), 0, C.byref(buf), True)
        ks_kernel = L.b200_last_keyswitch_kernel().decode()
        noise["dp"].append(rig.noise(dp, rig.s_big))
        noise["packing_ks"].append(
            _glwe_phase(glwes.cpu().numpy().view(np.uint64), comp_sk, cp.k, cp.N, 64).reshape(-1) / 2.0 ** 64)
        noise["storage_ms"].append(compress(br) / 2.0 ** cp.storage_log_modulus)
        del br, dp, glwes
        done = 0
        while done < per_key:
            c = min(CHUNK // lpg * lpg, per_key - done)
            ph = compress(rig.pbs(rig.grid_inputs(c), lut))
            fails += int(((ph >= half_box) | (ph < -half_box)).sum())
            done += c
    _report(set=kind, packing_keyswitch_kernel=ks_kernel)
    ok = [_check(kind, "dp", "4x", noise["dp"], model["dp"], P.big_n),
          _check(kind, "packing_ks", "4x", noise["packing_ks"], model["pks"], cp.big_n, normality=True),
          _check(kind, "storage_ms", "4x", noise["storage_ms"], model["ms"], cp.big_n)]
    runs = per_key * len(rigs)
    expected = M.expected_pfail_for_precision(COMP_INFLATED_PRECISION, model["ms"].variance)
    p_ok, rep = M.pfail_check(runs, fails, expected, COMP_INFLATED_PRECISION, M.precision_with_padding(4, 1))
    rep["original_expected_log2_pfail"] = math.log2(M.expected_pfail_for_precision(3, model["ms"].variance))
    _report(set=kind, check="compression_pfail", ok=p_ok, **rep)
    assert all(ok) and p_ok
