"""The ARIMA detector's numerical core (tad_arima.cu, compiled for the host) against plain high-precision restatements of the
same functions: the Kalman-filter likelihood and forecast and the Box-Cox likelihood against mpmath at 50 digits, the Box-Cox
MLE lambda and the start values against the SciPy/NumPy oracle, and tad_debug_arima_series -- the host reference of the
per-prefix GPU tests -- against the single-fit hook.  Runs without a GPU."""
import itertools

import numpy as np
import pytest

from oracle import arima_oracle as ao
from tests import arima_hooks as H

EPS = np.finfo(np.float64).eps


def _kalman_grid():
    rng = np.random.default_rng(1)
    pv = (0.0, 0.5, -0.5, 0.99, -0.99, 0.999999, -0.999999)
    for n in (3, 4, 33, 200):
        for scale in (1.0, 1e3, 1e9):
            y = (np.cumsum(rng.normal(size=n)) + 5.0) * scale
            # the longest series on a thinned parameter grid, to keep mpmath's share of the run short
            grid = itertools.product(pv, pv) if n < 200 else zip(pv, pv[::-1])
            for (phi, theta), s2 in itertools.product(grid, (1e-8, 1.0, 1e6)):
                yield y, (phi, theta, s2)


def test_kalman_filter_vs_mpmath():
    """arima_loglike and its one-step forecast against the recursion of oracle/arima_oracle.py:kalman_loglike at 50 digits.
    The filter starts the integrated state with the approximate-diffuse variance 1e6, and the first update subtracts it
    from itself (c00 = p00 - z0^2 / F): that costs about eps * 1e6 / s2 relative, so the bound scales with it.  Measured
    worst cases: 3.2e-10 (loglike) and 2.0e-10 (forecast) at s2 >= 1; 6.0e-3 and 9.9e-4 at s2 = 1e-8, where
    eps * 1e6 / s2 = 2.2e-2."""
    cases = list(_kalman_grid())
    out = H.core(H.OP_LOGLIKE, [y for y, _ in cases], [p for _, p in cases])
    worst = {}
    for (y, (phi, theta, s2)), (ll, fc) in zip(cases, out[:, :2]):
        ref = H.mp_kalman(y, phi, theta, s2)
        assert ref is not None and np.isfinite(ll), (len(y), phi, theta, s2)
        bound = 1e-9 + 0.5 * EPS * 1e6 / s2
        for what, got, want in (("loglike", ll, ref[0]), ("forecast", fc, ref[1])):
            err = float(abs((got - want) / want))
            assert err <= bound, (what, len(y), phi, theta, s2, err)
            key = (what, s2 >= 1.0)
            worst[key] = max(worst.get(key, 0.0), err)
    print("Kalman filter vs mpmath, worst relative error: " +
          ", ".join("%s s2%s %.2e" % (w, ">=1" if big else "=1e-8", e) for (w, big), e in sorted(worst.items())))


def _boxcox_sets():
    rng = np.random.default_rng(2)
    return {
        "noisy": np.maximum(np.rint(300 * (1 + 0.15 * rng.normal(size=50))), 1).astype(np.uint64),
        "wide": rng.integers(1, 2 ** 64 - 1, 40, dtype=np.uint64, endpoint=True),
        "top": np.array([2 ** 64 - 1, 2 ** 64 - 2, 2 ** 63, 2 ** 53 + 1, 2 ** 53, 10 ** 18, 5, 1], dtype=np.uint64),
    }


@pytest.mark.parametrize("lmb", [300.0, -300.0, 2.0, -2.0, 1e-10, -1e-10, 0.0])
def test_boxcox_llf_vs_mpmath(lmb):
    """boxcox_neg_llf against -scipy.stats.boxcox_llf at 50 digits, on values up to 2^64 - 1 and at lambdas of +-300, where
    x^lambda overflows a double (the likelihood is evaluated in log space so that Brent still finds the optimum there).
    1e-12 relative at every lambda but +-1e-10: there the log-space variance takes exp(z - max z) - mean of values that
    differ by about |lambda| * spread(log x), which leaves eps / (|lambda| * spread(log x)) of relative precision (8e-8
    measured on the noisy series).  Brent meets such lambdas only where the optimum is that close to zero, and there
    the lambda still agrees with SciPy's (test_lambda_vs_scipy_brent covers log-normal series)."""
    for name, v in _boxcox_sets().items():
        lx = np.log(v.astype(np.float64))
        got = H.core(H.OP_BOXCOX_LLF, [lx], [(lmb,)])[0, 0]
        want = H.mp_boxcox_neg_llf(lmb, lx)
        err = float(abs((got - want) / want))
        if lmb != 0.0 and abs(lmb) < 1e-6:
            bound = EPS / (abs(lmb) * np.ptp(lx))
        else:
            bound = 1e-12
        assert err <= bound, (name, lmb, err, bound)


def test_boxcox_transform_overflows_at_large_lambda():
    """The lambdas of +-300 above are ones where the transform itself is not finite: the likelihood is, the series is not."""
    v = _boxcox_sets()["wide"]
    calc, lam = H.series(v, lam=300.0)
    assert calc is None and lam == 300.0
    assert not np.isfinite(np.expm1(300.0 * np.log(v.astype(np.float64))) / 300.0).all()


def _lambda_series():
    rng = np.random.default_rng(3)
    for k in range(200):
        n = int(rng.integers(4, 120))
        kind = k % 5
        if kind == 0:
            v = 300 * (1 + 0.15 * rng.normal(size=n))
        elif kind == 1:
            v = np.exp(rng.normal(5.0, 1.0, n))                   # log-normal: the optimum is near lambda = 0
        elif kind == 2:
            v = rng.uniform(1, 1000, n)
        elif kind == 3:                                           # above 2^53: the u64 -> double rounding matters
            yield np.uint64(2 ** 60) + rng.integers(0, 2 ** 58, n, dtype=np.uint64)
            continue
        else:
            v = rng.gamma(2.0, 50.0, n) + 1
        yield np.maximum(np.rint(v), 1).astype(np.uint64)


def test_lambda_vs_scipy_brent():
    """The Box-Cox MLE lambda (boxcox_mle_lambda on log(x) as the kernel takes it) against ao.boxcox_mle, Brent as SciPy
    runs it, on 200 series.  Within 1e-7, or else an equally good optimum: the objective is flat to its last bit over an
    interval of about sqrt(eps / f'') around the optimum, and where the two Brent runs end at different points of it the
    exact (50-digit) objective at the engine's lambda is no worse than at SciPy's, to 1e-15 relative."""
    xs = list(_lambda_series())
    got = H.core(H.OP_LAMBDA, xs)[:, 0]
    off = 0
    for v, lam in zip(xs, got):
        x = v.astype(np.float64)
        want = ao.boxcox_mle(x)[1]
        if abs(lam - want) <= 1e-7:
            continue
        off += 1
        lx = np.log(x)
        fg, fw = H.mp_boxcox_neg_llf(lam, lx), H.mp_boxcox_neg_llf(want, lx)
        assert abs(lam - want) < 1e-4 and fg - fw <= 1e-15 * abs(fw), (len(v), lam, want)
    assert off <= len(xs) // 4, off


def _exact_start(y):
    """ao.start_params in exact rational arithmetic: the same regressions, solved by the minimum-norm (pseudo-inverse)
    solution of their normal equations with the rank taken exactly.  At an exact rank deficiency NumPy's SVD leaves
    rounding noise in residuals that are exactly zero (a linear series gives phi = 1 - 1e-16, kept as stationary, where
    the exact answer is phi = 1, which falls back to 0), so these cases are checked against this statement instead."""
    from fractions import Fraction as Fr
    d = [Fr(float(b)) - Fr(float(a)) for a, b in zip(y[:-1], y[1:])]
    m = len(d)

    def lstsq(rows):
        s11 = sum(a * a for a, _, _ in rows); s12 = sum(a * b for a, b, _ in rows); s22 = sum(b * b for _, b, _ in rows)
        r1 = sum(a * t for a, _, t in rows); r2 = sum(b * t for _, b, t in rows)
        det, tr = s11 * s22 - s12 * s12, s11 + s22
        if tr == 0:
            return Fr(0), Fr(0)
        if det != 0:
            return (r1 * s22 - r2 * s12) / det, (r2 * s11 - r1 * s12) / det
        return r1 / tr, r2 / tr                     # rank one: r lies in the range, pinv(A) r = r / trace(A)
    phi = theta = Fr(0)
    var = None
    if m >= 4:
        b1, b2 = lstsq([(d[t - 1], d[t - 2], d[t]) for t in range(2, m)])
        res = {t: d[t] - b1 * d[t - 1] - b2 * d[t - 2] for t in range(2, m)}
        phi, theta = lstsq([(d[t - 1], res[t - 1], d[t]) for t in range(3, m)])
        if m - 3 > 1:
            var = sum((d[t] - phi * d[t - 1] - theta * res[t - 1]) ** 2 for t in range(4, m)) / (m - 4)
    phi = phi if abs(phi) < 1 else Fr(0)
    theta = theta if abs(theta) < 1 else Fr(0)
    dmean = sum(d) / m
    dvar = sum((q - dmean) ** 2 for q in d) / m
    if var is None or var <= dvar / 10 ** 10 or var <= 0:
        var = dvar if dvar > 0 else Fr(1)
    return ao.untransform(float(phi), float(theta), float(var))


def _start_cases():
    rng = np.random.default_rng(4)
    degenerate, regular = [], []
    for n in range(4, 12):
        degenerate.append(np.arange(n) * 2.5 + 7.0)                             # linear: constant differences
        degenerate.append(np.cumsum(np.resize([1.0, 3.0], n)))                  # differences repeat with period 2
        degenerate.append(np.cumsum(np.resize([2.0, -2.0], n)) + 10.0)          # period 2, opposite regressors
        degenerate.append(np.resize([4.0, 4.0, 9.0], n))                        # repeated values
        regular.append(np.cumsum(rng.normal(size=n)) + 3.0)
    for n in (4, 5, 6, 7):                                                      # the variance falls back to var(diff)
        for _ in range(20):
            regular.append(rng.normal(size=n) * rng.choice([1e-3, 1.0, 1e4]))
    return degenerate, regular


def test_start_values_at_the_rank_deficient_edges():
    """arima_start at the rank-deficient edges of lstsq2 -- constant differences, period-2 differences, repeated values --
    against the exact statement of the algorithm, and on regular series and at n = 4..7 (too few points for a regression
    variance: the variance of the differences is taken) against ao.start_params (numpy.linalg.pinv).  At n = 5 the AR(2)
    regression fits its two points exactly, so the MA regressor is rounding noise of either implementation and theta a
    few 1e-9 from zero: the absolute tolerance of the regular cases covers that."""
    degenerate, regular = _start_cases()
    got = H.core(H.OP_START, degenerate + regular)[:, :3]
    for y, u in zip(degenerate, got):
        np.testing.assert_allclose(u, _exact_start(y), rtol=1e-12, atol=1e-15, err_msg=str(y))
    for y, u in zip(regular, got[len(degenerate):]):
        np.testing.assert_allclose(u, ao.untransform(*ao.start_params(y)), rtol=1e-9, atol=1e-8, err_msg=str(y))
        np.testing.assert_allclose(u, _exact_start(y), rtol=1e-9, atol=1e-8, err_msg=str(y))


def test_forward_difference_gradient_is_the_single_filter():
    """arima_fg runs the objective at u and at its three forward-difference neighbours as four filters in one loop; each
    must be the single filter's arithmetic exactly: f = arima_objective(u), g[c] = (objective(u + 1e-8 e_c) - f) / 1e-8."""
    rng = np.random.default_rng(5)
    ys, us = [], []
    for n in (3, 4, 7, 40, 150):
        for _ in range(6):
            ys.append(np.cumsum(rng.normal(size=n)) * rng.choice([1.0, 1e3]))
            us.append(rng.normal(size=3) * [1.0, 1.0, rng.choice([0.1, 1.0, 30.0])])
    out = H.core(H.OP_FG, ys, us)
    assert np.array_equal(out[:, 0], out[:, 4])
    assert np.array_equal(out[:, 1:4], (out[:, 5:8] - out[:, 4:5]) / 1e-8)


def test_series_hook_is_the_single_fit():
    """tad_debug_arima_series (the whole per-series path) on the golden series: its lambda is the single-fit hook's, its
    first three outputs the Box-Cox round trip, and its flags those of the reference's golden vector."""
    import json
    import os
    ref = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_test_vectors.json")))
    v = np.array(ref["throughput_list"], dtype=np.uint64)
    calc, lam = H.series(v)
    x = v.astype(np.float64)
    lam_h = H.core(H.OP_LAMBDA, [v])[0, 0]
    assert lam == lam_h and abs(lam - ao.boxcox_mle(x)[1]) < 1e-7
    np.testing.assert_allclose(calc[:3], x[:3], rtol=1e-14)
    # the flags of the reference golden vector
    assert list(np.abs(x - calc) > ref["stddev"]) == ref["expected_anomaly_list_arima"]


def test_series_hook_none_cases_and_nudges():
    """No rows for n <= 3, a zero value or constant values.  A one-ulp nudge of the transformed series leaves the first
    three points' round trip within 1e-14 and moves the prefix forecasts; each nudge mode is its own perturbation."""
    for vals in ([5, 6, 7], [5, 0, 7, 9, 11], [7, 7, 7, 7, 7]):
        assert H.series(np.array(vals, dtype=np.uint64))[0] is None
    rng = np.random.default_rng(6)
    v = np.maximum(np.rint(300 * (1 + 0.15 * rng.normal(size=40))), 1).astype(np.uint64)
    base, lam = H.series(v)
    assert np.array_equal(H.series(v, lam=lam)[0], base)
    runs = []
    for nudge in (1, -1, 7, 11):
        calc, lam2 = H.series(v, lam=lam, nudge=nudge)
        assert lam2 == lam and calc is not None
        assert (np.abs(calc - base) / base)[:3].max() <= 1e-14
        assert not np.array_equal(calc, base)
        runs.append(calc)
    assert len({c.tobytes() for c in runs}) == len(runs)
