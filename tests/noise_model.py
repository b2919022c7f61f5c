"""Noise model of the KS -> PBS and compression atomic patterns: the reference's
additive-variance formulas, their composition along a chain, the p_fail
arithmetic and the acceptance statistics of its noise-distribution tests.

Each function restates the tfhe-rs function named in its docstring (paths
relative to tfhe/src/).  Variances are fractions of the torus squared, as in
the reference; moduli are passed as floats.  The PBS output formulas are the
ones of tests/noise_formula.py.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
from scipy import special, stats

from tests.noise_formula import multi_bit_pbs_variance_tuniform_fft, pbs_variance_tuniform_fft

Q64 = 2.0 ** 64
_LN2_SQ = 2.88539008177793  # 2 / ln 2, as the generated formulas write it
_L2E = math.log2(math.e)


# ---------------------------------------------------------------------------
# additive variances (core_crypto/commons/noise_formulas/)
# ---------------------------------------------------------------------------
def tuniform_variance(bound_log2: int, modulus: float = Q64) -> float:
    """TUniform::variance (commons/math/random/t_uniform.rs:75-81): values in
    [-2^b, 2^b], variance (2^(2b+1) + 1) / 6 integer units."""
    return (2.0 ** (2 * bound_log2 + 1) + 1.0) / 6.0 * modulus ** -2


def _tuniform_key_term(lwe_dimension: float, modulus: float) -> float:
    # the bracket shared by secure_noise.rs:59-68, lwe_keyswitch.rs:91-100 and
    # lwe_packing_keyswitch.rs:104-113
    bound = math.ceil(-0.025167785 * lwe_dimension + _L2E * math.log(modulus) + 4.10067100000001)
    return 2.0 ** (4.44 - _LN2_SQ * math.log(modulus)) + (1 / 3.0) * modulus ** -2 * (2.0 ** (2.0 * bound) + 0.5)


def minimal_lwe_variance_tuniform(lwe_dimension: int, modulus: float = Q64) -> float:
    """minimal_lwe_variance_for_132_bits_security_tuniform_impl
    (noise_formulas/secure_noise.rs:55-69)."""
    return _tuniform_key_term(lwe_dimension, modulus)


def keyswitch_variance_tuniform(n_in: int, n_out: int, base_log: int, level: int, q_in: float = Q64,
                                q_out: float = Q64) -> float:
    """keyswitch_additive_variance_132_bits_security_tuniform_impl
    (noise_formulas/lwe_keyswitch.rs:81-107)."""
    B = 2.0 ** base_log
    return (level * n_in * _tuniform_key_term(n_out, q_out) * (B ** 2 / 12.0 + 0.166666666666667)
            + n_in * (0.0208333333333333 * q_in ** -2 + 0.0416666666666667 * B ** (-2.0 * level))
            - q_in ** -2 / 12.0 + q_out ** -2 / 12.0)


def modulus_switch_variance(n: int, q: float, q_new: float) -> float:
    """modulus_switch_additive_variance_impl (noise_formulas/modulus_switch.rs:23-32)."""
    return n * (0.0208333333333333 * q ** -2 + 0.0416666666666667 * q_new ** -2) - q ** -2 / 12.0 + q_new ** -2 / 12.0


def centered_modulus_switch_variance(n: int, q: float, q_new: float) -> float:
    """centered_binary_shifted_modulus_switch_additive_variance_impl
    (noise_formulas/centered_mean_shifted_modulus_switch.rs:27-34)."""
    return n * (0.0416666666666667 * q ** -2 + 0.0208333333333333 * q_new ** -2)


def multi_bit_modulus_switch_variance(n: int, g: int, q: float, q_new: float) -> float:
    """multi_bit_modulus_switch_additive_variance_impl
    (noise_formulas/multi_bit_modulus_switch.rs:25-41)."""
    return ((1.0 / g) * n * q ** -2 * (1.0 - 2.0 ** -g) * (2.0 ** (-g - 2) + q_new ** -2 * (q ** 2 - q_new ** 2) / 12.0)
            - q ** -2 / 12.0 + q_new ** -2 / 12.0)


def packing_keyswitch_variance_tuniform(n_in: int, k_out: int, N_out: int, base_log: int, level: int,
                                        lwe_to_pack: int, q: float = Q64) -> float:
    """packing_keyswitch_additive_variance_132_bits_security_tuniform_impl
    (noise_formulas/lwe_packing_keyswitch.rs:92-119): per occupied slot."""
    B = 2.0 ** base_log
    return (level * n_in * lwe_to_pack * _tuniform_key_term(k_out * N_out, q) * (B ** 2 / 12.0 + 0.166666666666667)
            + 0.5 * n_in * (q ** -2 / 6.0 + B ** (-2.0 * level) / 12.0))


MS_STANDARD, MS_CENTERED, MS_MULTI_BIT = "standard", "centered", "multi_bit"


def expected_average_after_ms(kind: str, N: int) -> float:
    """NoiseSimulationModulusSwitchConfig::expected_average_after_ms
    (shortint/server_key/tests/noise_distribution/utils/noise_simulation.rs:963-974):
    the centered switch subtracts half a step of 1/(2N) before the blind
    rotation; the others are unbiased."""
    return -1.0 / (4.0 * N) if kind == MS_CENTERED else 0.0


def ms_additive_variance(kind: str, n: int, log_modulus: int, g: int = 1, q: float = Q64) -> float:
    """The switch of each NoiseSimulationModulusSwitchConfig
    (noise_formulas/noise_simulation/modulus_switch.rs:31-162)."""
    q_new = 2.0 ** log_modulus
    if kind == MS_CENTERED:
        return centered_modulus_switch_variance(n, q, q_new)
    if kind == MS_MULTI_BIT:
        return multi_bit_modulus_switch_variance(n, g, q, q_new)
    return modulus_switch_variance(n, q, q_new)


# ---------------------------------------------------------------------------
# composition (noise_formulas/noise_simulation/: every step adds its additive
# variance; a scalar c multiplies the variance by c^2, mod.rs:168-175; an
# uncorrelated sum adds the variances, mod.rs:177-195)
# ---------------------------------------------------------------------------
def br_variance(P) -> float:
    """Output variance of the blind rotation of a noiseless switched input
    (lwe_programmable_bootstrap.rs / lwe_multi_bit_programmable_bootstrap.rs
    through noise_formula.py)."""
    if P.grouping_factor > 1:
        return multi_bit_pbs_variance_tuniform_fft(P.n, P.k, P.N, P.pbs_base_log, P.pbs_level, P.grouping_factor)
    return pbs_variance_tuniform_fft(P.n, P.k, P.N, P.pbs_base_log, P.pbs_level)


def ms_kind(P) -> str:
    if P.grouping_factor > 1:
        return MS_MULTI_BIT
    return MS_CENTERED if P.centered_ms else MS_STANDARD


@dataclass(frozen=True)
class Stage:
    mean: float
    variance: float


def br_dp_ks_ms(P, sum_c2: float, ms: str | None = None, with_ks: bool = True, ms_dimension: float | None = None):
    """br_dp_ks_any_ms (shortint/server_key/tests/noise_distribution/br_dp_ks_ms.rs)
    on noise-simulation ciphertexts: the expected mean and variance after each
    stage, for a dot product with sum c_i^2 = sum_c2 over independent PBS
    outputs (the reference's `scalar` is the one-term case, sum_c2 = scalar^2).
    `ms` defaults to the parameter set's own switch; with_ks=False drops the
    keyswitch term (a negative control).  The means are those of noise that is
    unbiased until the switch.  `ms_dimension` replaces n in the switch's
    formula: the standard switch adds one rounding error per key bit set, so
    for given keys of mean Hamming weight w it is 2 w (the formula's n / 2 is
    the weight of a random key)."""
    ms = ms or ms_kind(P)
    br = br_variance(P)
    dp = sum_c2 * br
    ks = dp + (keyswitch_variance_tuniform(P.big_n, P.n, P.ks_base_log, P.ks_level) if with_ks else 0.0)
    after = ks + ms_additive_variance(ms, P.n if ms_dimension is None else ms_dimension, P.log_2N, P.grouping_factor)
    return {"br": Stage(0.0, br), "dp": Stage(0.0, dp), "ks": Stage(0.0, ks),
            "ms": Stage(expected_average_after_ms(ms, P.N), after)}


def br_dp_packing_ks_ms(P, cp, scalar: int, lwe_to_pack: int | None = None):
    """br_dp_packing_ks_ms (shortint/server_key/tests/noise_distribution/
    br_dp_packingks_ms.rs:33-110): PBS outputs times `scalar`, packed by the
    packing keyswitch into one GLWE of cp.lwe_per_glwe bodies, then the
    standard switch of the GLWE (k N mask words) to the storage modulus."""
    lwe_to_pack = cp.lwe_per_glwe if lwe_to_pack is None else lwe_to_pack
    br = br_variance(P)
    dp = scalar ** 2 * br
    pks = dp + packing_keyswitch_variance_tuniform(P.big_n, cp.k, cp.N, cp.ks_base_log, cp.ks_level, lwe_to_pack)
    after = pks + modulus_switch_variance(cp.big_n, Q64, 2.0 ** cp.storage_log_modulus)
    return {"br": Stage(0.0, br), "dp": Stage(0.0, dp), "pks": Stage(0.0, pks), "ms": Stage(0.0, after)}


# ---------------------------------------------------------------------------
# p_fail arithmetic (shortint/server_key/tests/noise_distribution/utils/mod.rs,
# core_crypto/commons/mod.rs)
# ---------------------------------------------------------------------------
def precision_with_padding(message_modulus: int, carry_modulus: int) -> int:
    """precision_with_padding (utils/mod.rs:929-938): log2(msg * carry) + 1."""
    c = message_modulus * carry_modulus
    assert c & (c - 1) == 0
    return c.bit_length() - 1 + 1


def expected_pfail_for_precision(precision: int, variance: float) -> float:
    """expected_pfail_for_precision (utils/mod.rs:940-954): a centred Gaussian
    of that variance leaves +-2^-(precision + 1)."""
    return float(special.erfc(2.0 ** -(precision + 1) / math.sqrt(variance) / math.sqrt(2.0)))


def equivalent_pfail_gaussian_noise(original_precision: int, original_pfail: float, new_precision: int) -> float:
    """equivalent_pfail_gaussian_noise (core_crypto/commons/mod.rs:300-321):
    each bit of precision halves the z-score's margin."""
    z = math.sqrt(2.0) * special.erfcinv(original_pfail)
    return float(special.erfc(z / 2.0 ** (new_precision - original_precision) / math.sqrt(2.0)))


def chain_log2_pfail(P, max_noise_level: int = 5, message_modulus: int = 4, carry_modulus: int = 4, **kw) -> float:
    """log2 p_fail of one bootstrap whose input is the chain at the
    parameter set's max noise level (the optimizer's figure)."""
    v = br_dp_ks_ms(P, float(max_noise_level) ** 2, **kw)["ms"].variance
    return math.log2(expected_pfail_for_precision(precision_with_padding(message_modulus, carry_modulus), v))


# ---------------------------------------------------------------------------
# acceptance statistics (core_crypto/commons/mod.rs, utils/mod.rs)
# ---------------------------------------------------------------------------
def sample_variance(x: np.ndarray) -> float:
    """test_tools::variance (commons/mod.rs:136-143): divides by n - 1."""
    return float(np.var(x, ddof=1))


def gaussian_mean_ci(count: int, mean: float, std: float, p: float = 0.99):
    """gaussian_mean_confidence_interval (commons/mod.rs:81-103)."""
    z = math.sqrt(2.0) * special.erfcinv(1.0 - p)
    d = z * std / math.sqrt(count)
    return mean - d, mean + d


def gaussian_variance_ci(count: int, variance: float, p: float = 0.99):
    """gaussian_variance_confidence_interval (commons/mod.rs:169-204): the chi^2
    interval with count - 1 degrees of freedom."""
    dof = count - 1.0
    a = 1.0 - p
    lo_q, hi_q = stats.chi2.ppf(a / 2.0, dof), stats.chi2.ppf(1.0 - a / 2.0, dof)
    return dof * variance / hi_q, dof * variance / lo_q


def clopper_pearson_ci(runs: int, fails: int, p: float = 0.99):
    """pfail_clopper_pearson_exact_confidence_interval (commons/mod.rs:111-133)."""
    a = 1.0 - p
    lo = stats.beta.ppf(a / 2.0, fails, runs - fails + 1.0)
    hi = stats.beta.ppf(1.0 - a / 2.0, fails + 1.0, runs - fails)
    return float(lo), float(hi)


def normality_test(samples: np.ndarray, alpha: float = 0.01):
    """normality_test_f64 (commons/mod.rs:334-391): the Shapiro-Francia W'
    against Blom scores, with Royston's log-normal approximation of its null
    distribution.  At most 5000 samples, as there.  Returns (W', p, passes)."""
    x = np.sort(np.asarray(samples, dtype=np.float64))
    n = x.size
    assert n <= 5000, "the approximation of the null distribution holds for n <= 5000"
    m = stats.norm.ppf((np.arange(1, n + 1) - 3.0 / 8.0) / (n + 0.25))
    c = m / np.sqrt(np.sum(m * m))
    w = float(np.sum(x * c) ** 2 / np.sum((x - x.mean()) ** 2))
    ln_n = math.log(n)
    u = math.log(ln_n) - ln_n
    mu = 1.0521 * u - 1.2725
    sigma = -0.26758 * (math.log(ln_n) + 2.0 / ln_n) + 1.0308
    p = float(1.0 - stats.norm.cdf((math.log(1.0 - w) - mu) / sigma))
    return w, p, p > alpha


def mean_and_variance_check(samples: np.ndarray, expected_mean: float, expected_variance: float,
                            secure_variance: float, groups: int = 1):
    """mean_and_variance_check (utils/mod.rs:75-213): the expected mean must
    lie in the 99 % interval of the measured mean; the measured variance must
    be <= expected and >= the secure minimum, or else the expected variance
    must lie in its 99 % interval.  Returns (ok, report).

    tfhe-rs draws a fresh key for every sample, so its samples are
    independent.  With `groups` > 1 the samples are that many equal blocks,
    one key each: a key fixes part of the noise's mean, the independent units
    of the mean are then the keys, and its 99 % interval is the Student t
    interval of the block means."""
    x = np.asarray(samples, dtype=np.float64)
    mean, var = float(x.mean()), sample_variance(x)
    if groups > 1:
        block_means = x.reshape(groups, -1).mean(axis=1)
        d = stats.t.ppf(0.995, groups - 1) * block_means.std(ddof=1) / math.sqrt(groups)
        m_lo, m_hi = mean - d, mean + d
    else:
        m_lo, m_hi = gaussian_mean_ci(x.size, mean, math.sqrt(var))
    v_lo, v_hi = gaussian_variance_ci(x.size, var)
    mean_ok = m_lo <= expected_mean <= m_hi
    if var <= expected_variance:
        var_ok = var >= secure_variance
    else:
        var_ok = v_lo <= expected_variance <= v_hi
    return mean_ok and var_ok, dict(samples=int(x.size), mean=mean, expected_mean=expected_mean, mean_ci=(m_lo, m_hi),
                                    variance=var, expected_variance=expected_variance, variance_ci=(v_lo, v_hi),
                                    variance_ratio=var / expected_variance, mean_ok=mean_ok, variance_ok=var_ok)


def pfail_check(runs: int, fails: int, expected_pfail: float, new_precision: int, original_precision: int):
    """pfail_check (utils/mod.rs:447-617): pass if the measured p_fail is <=
    the expected one, or if the expected one lies in the 99 % Clopper-Pearson
    interval.  Zero failures pass (the reference warns).  Also reports the
    measured p_fail brought back to the original precision."""
    measured = fails / runs
    rep = dict(runs=runs, fails=fails, measured_pfail=measured, expected_pfail=expected_pfail)
    if fails == 0:
        return True, rep
    lo, hi = clopper_pearson_ci(runs, fails)
    eq = equivalent_pfail_gaussian_noise(new_precision, measured, original_precision)
    rep.update(ci=(lo, hi), equivalent_log2_pfail=math.log2(eq) if eq > 0 else float("-inf"),
               equivalent_log2_ci=tuple(math.log2(equivalent_pfail_gaussian_noise(new_precision, b,
                                                                                   original_precision))
                                        for b in (lo, hi)))
    ok = measured <= expected_pfail or lo <= expected_pfail <= hi
    return ok, rep
