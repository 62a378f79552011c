"""The GPU ARIMA detector prefix by prefix against its own core built for the host (tad_debug_arima_series: the kernels'
functions in the kernels' order), with optimiser path noise told apart from kernel error.

A prefix fit is path dependent: L-BFGS-B's stopping tests (pgtol 1e-8 on a forward-difference gradient of step 1e-8) sit at
the gradient's own noise level, so a one-ulp change of the series can end a fit elsewhere on a flat likelihood.  On the
GPU, FMA contraction and the device log/exp act as such a change.  So the host reference runs each series unnudged and
under one-ulp nudges -- up, down, and random directions per point; 4 runs for the longest series, up to 64 for short ones,
whose rare jumps to another optimum take many draws to show.  A prefix whose forecasts all agree within 1e-10 is stable.

Each job's rows are compared, prefix by prefix, with tad_debug_arima_series_device: the same functions on the device, one
thread per prefix fit, so any difference is the fit kernel's scheduling or its code generation.  The device reference's
transformed series is compared with the host's, and its fits with the host core's on that same series.  The same table then goes through the spill path
and through a fit that yields to queued jobs, and both must reproduce the first run's rows bit for bit."""
import os
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from theia_b200 import synth
from tests import arima_hooks as H
from tests.test_arima_core_precision import EPS, _boxcox_sets, _kalman_grid, _lambda_series
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

NUDGE_BUDGET = 40_000          # a series of n points gets about this / n^2 nudged runs (a fit's cost grows with its length)
STABLE = 1e-10                 # the host forecasts of a stable prefix all agree this closely (relative)
# FMA contraction.  nvcc contracts a * b + c into one rounding, and the same source contracts differently in the fit kernel,
# in the device reference's one-thread fit and on the host (which has none).  Built with --fmad=false (not the product
# build), an H100 gave: the kernel equal to the device reference bit for bit on every series, so the warp's hand-out, lane
# reuse and forecast slots add nothing; the device core within 6.7e-12 of the host core on every stable prefix; 63
# prefixes beyond 1e-3 against the host nudges' 1,933.  With contraction (the product build) the same table gives 1.06e-5
# on stable prefixes and 1,148 beyond 1e-3, and 85 of 147 series have some prefix not bit-equal to the device reference.
# The bounds below are those of the contracted build, about 10x the measured values.
STABLE_TOL = 1e-4              # device core vs host core on a stable prefix (measured 1.06e-5; 6.7e-12 uncontracted)
FAR_MAX = 0.21                 # share of prefixes the device core puts beyond 1e-3 of the host's (measured 18.5 %)
KERNEL_OFF_MAX = 0.07          # share of prefixes the kernel has not bit-equal to the device reference (measured 5.2 %)
TRANSFORM_ULPS = 4             # device vs host transformed series (log, expm1 and a divide per point)
MIN_STABLE_SHARE = 0.15        # measured: 18.7 % of this table's prefixes are stable
KEY0 = 0x0B000000


# ------------------------------------------------------------------------------------------------
# A. the device core against the host core and mpmath
# ------------------------------------------------------------------------------------------------
def test_device_lambda_is_the_host_lambda():
    """Within 1e-9, or else an equally good optimum: the device's log and exp move Brent's path as SciPy's arithmetic does
    (test_arima_core_precision.py::test_lambda_vs_scipy_brent), and the exact likelihood at the two lambdas agrees to the
    objective's double resolution."""
    xs = list(_lambda_series())
    host, dev = H.core(H.OP_LAMBDA, xs)[:, 0], H.core(H.OP_LAMBDA, xs, device=True)[:, 0]
    off = 0
    for v, h, d in zip(xs, host, dev):
        if abs(d - h) <= 1e-9:
            continue
        off += 1
        lx = np.log(v.astype(np.float64))
        fh, fd = H.mp_boxcox_neg_llf(h, lx), H.mp_boxcox_neg_llf(d, lx)
        assert abs(d - h) < 1e-4 and abs(fd - fh) <= 2e-15 * abs(fh), (len(v), h, d)
    print("device lambda vs host: %d of %d beyond 1e-9, worst %.2e" % (off, len(xs), np.abs(dev - host).max()))


def test_device_boxcox_llf_vs_mpmath():
    """Within four times the host's own error against mpmath, plus a few ulp."""
    xs, pars = [], []
    for v in _boxcox_sets().values():
        for lmb in (300.0, -300.0, 2.0, -2.0, 1e-10, -1e-10, 0.0):
            xs.append(np.log(v.astype(np.float64)))
            pars.append((lmb,))
    host, dev = H.core(H.OP_BOXCOX_LLF, xs, pars)[:, 0], H.core(H.OP_BOXCOX_LLF, xs, pars, device=True)[:, 0]
    for lx, (lmb,), h, d in zip(xs, pars, host, dev):
        want = H.mp_boxcox_neg_llf(lmb, lx)
        eh, ed = float(abs((h - want) / want)), float(abs((d - want) / want))
        assert ed <= 4 * eh + 8 * EPS, (lmb, eh, ed)


def test_device_kalman_filter_vs_mpmath():
    cases = [c for k, c in enumerate(_kalman_grid()) if k % 4 == 0]
    ys, ps = [y for y, _ in cases], [p for _, p in cases]
    host, dev = H.core(H.OP_LOGLIKE, ys, ps), H.core(H.OP_LOGLIKE, ys, ps, device=True)
    errs = []
    for y, p, h, d in zip(ys, ps, host, dev):
        ll, fc = H.mp_kalman(y, *p)
        errs.append([float(abs((a - want) / want)) for a, want in ((h[0], ll), (h[1], fc), (d[0], ll), (d[1], fc))])
    errs = np.array(errs)
    print("device Kalman filter vs mpmath: worst %.2e (host %.2e)" % (errs[:, 2:].max(), errs[:, :2].max()))
    # the error model of the host test (test_arima_core_precision.py::test_kalman_filter_vs_mpmath): the diffuse start
    # costs eps * 1e6 / s2.  FMA contraction rounds differently, not worse: at phi = +-0.999999 (1 / (1 - phi^2) = 5e5)
    # the device's error was measured at up to 6x the host's on the same series, both far inside this bound.
    for p, e in zip(ps, errs):
        assert e[2:].max() <= 1e-9 + 0.5 * EPS * 1e6 / p[2], (p, e)


def test_device_fused_gradient_is_the_single_filter():
    """arima_fg's four filters in one loop against four separate arima_objective calls, on the device: bit for bit."""
    rng = np.random.default_rng(5)
    ys, us = [], []
    for n in (3, 4, 7, 40, 150):
        for _ in range(12):
            ys.append(np.cumsum(rng.normal(size=n)) * rng.choice([1.0, 1e3]))
            us.append(rng.normal(size=3) * [1.0, 1.0, rng.choice([0.1, 1.0, 30.0])])
    out = H.core(H.OP_FG, ys, us, device=True)
    assert np.array_equal(out[:, 0], out[:, 4])
    assert np.array_equal(out[:, 1:4], (out[:, 5:8] - out[:, 4:5]) / 1e-8)


# ------------------------------------------------------------------------------------------------
# B. every prefix of a whole job
# ------------------------------------------------------------------------------------------------
def _noisy(rng, n, base=None, cv=0.15):
    v = (base if base is not None else rng.uniform(50, 500)) * (1.0 + cv * rng.normal(size=n))
    spike = rng.random(n) < 0.04
    v = np.where(spike, v * rng.choice([0.5, 2.0, 3.0], n), v)
    return np.maximum(np.rint(v), 1)


def _series_list():
    """(values u64, extra duplicate rows at existing times) per series, at the lengths where the fit's scheduling has
    edges: one fit, the start-value fallbacks, 31-34 fits around a warp's 32 lanes, 63-65, 97, and a handful of long
    series for the longest-first job list; then the series that yield no rows, one whose lambda overflows, values
    above 2^53 and (key, time) duplicates."""
    rng = np.random.default_rng(2024)
    out = []
    lengths = [4] * 12 + [5, 6, 7] * 8 + list(range(34, 38)) * 14 + [66, 67, 68] * 10 + [100] * 10 + [300, 420, 600]
    for n in lengths:
        out.append((_noisy(rng, n).astype(np.uint64), 0))
    for vals in ([5, 6], [5, 6, 7], [9, 4, 0, 7, 8, 6, 5, 3], [7] * 12):
        out.append((np.array(vals, dtype=np.uint64), 0))
    out.append((np.rint(1e6 * (1 + 1e-3 * rng.normal(size=24))).astype(np.uint64), 0))       # lambda in the hundreds
    for n in (12, 40, 70):                                                                     # above 2^53
        out.append(((2 ** 60 * (1 + 0.15 * rng.normal(size=n))).astype(np.uint64), 0))
    for n in (8, 35, 60):
        out.append((_noisy(rng, n).astype(np.uint64), n // 3))                                 # duplicates
    out.append((np.uint64(2 ** 53) + _noisy(rng, 30).astype(np.uint64), 10))
    return out


def _table(series, rng):
    cols = {k: [] for k in synth.COLUMN_DTYPES}
    for i, (v, dups) in enumerate(series):
        n = len(v)
        t = synth.T0 + 60 * (1 + np.arange(n))
        at = rng.integers(0, n, dups) if n else np.zeros(0, np.int64)
        extra = (v[at] // np.uint64(2) + rng.integers(0, 400, dups).astype(np.uint64)) if dups else np.zeros(0, np.uint64)
        m = n + dups
        cols["src_ip"].append(np.full(m, KEY0 + i, np.uint32)); cols["dst_ip"].append(np.full(m, 0x0A000001, np.uint32))
        cols["src_port"].append(np.full(m, 4000, np.uint16)); cols["dst_port"].append(np.full(m, 443, np.uint16))
        cols["proto"].append(np.full(m, 6, np.uint8)); cols["flow_start"].append(np.full(m, synth.T0, np.uint32))
        cols["flow_end"].append(np.concatenate([t, t[at]]).astype(np.uint32))
        cols["value"].append(np.concatenate([v, extra]).astype(np.uint64))
    tab = {k: np.concatenate(c) for k, c in cols.items()}
    perm = rng.permutation(len(tab["value"]))
    return {k: c[perm] for k, c in tab.items()}


def _reduced(table, reducer):
    """Per series, the values the kernel sees: (key, time) duplicates reduced by max or (wrapping) sum, in time order."""
    out = {}
    order = np.lexsort([table["flow_end"], table["src_ip"]])
    ip, te, val = table["src_ip"][order], table["flow_end"][order], table["value"][order]
    for s in np.unique(ip):
        m = ip == s
        times, inv = np.unique(te[m], return_inverse=True)
        v = np.zeros(len(times), np.uint64)
        if reducer == 0:
            np.maximum.at(v, inv, val[m])
        else:
            np.add.at(v, inv, val[m])
        out[int(s)] = (times, v)
    return out


def nudges(n):
    """The nudge modes of tad_debug_arima_series a series of n points is run under: all up, all down, then random."""
    return (1, -1) + tuple(range(7, 7 + int(np.clip(NUDGE_BUDGET // max(n, 1) ** 2, 4, 64)) - 2))


def _reference(v, lam, y):
    """The host core's fits on the transformed series y (the device's): unnudged and under nudges()."""
    base, _ = H.series(v, lam=lam, y=y)
    return base, [H.series(v, lam=lam, nudge=k, y=y)[0] for k in nudges(len(v))]


def _ulps(a, b):
    ia, ib = (np.asarray(q, np.float64).view(np.int64) for q in (a, b))
    ia, ib = (np.where(q < 0, np.int64(-2 ** 63) - q, q) for q in (ia, ib))      # ordered like the doubles
    return np.abs(ia - ib)


@pytest.fixture(scope="module")
def prefix_table():
    return _table(_series_list(), np.random.default_rng(7))


@pytest.fixture(scope="module")
def prefix_rows(engine, prefix_table):
    got, st = engine.run(prefix_table, algo="ARIMA", tad_id="prefix", emit_all=True)
    assert st["state"] == "COMPLETED"
    return got


def _check_prefixes(got, table, reducer):
    """One job's rows, series by series and prefix by prefix: (1) against the device reference, bit for bit on the train
    points and on all but KERNEL_OFF_MAX of the fits (code generation, see FMA above); (2) the
    device's transformed series against the host's; (3) the device reference's fits against the host core's on the same
    transformed series, and the kernel's rows too: stable prefixes within STABLE_TOL, and no more than FAR_MAX of all
    prefixes beyond 1e-3."""
    red = _reduced(table, reducer)
    keys = sorted(red)
    dev = dict(zip(keys, H.series_device([red[k][1] for k in keys])))
    valid = [k for k in keys if len(red[k][1]) > 3 and red[k][1].min() > 0 and red[k][1].min() != red[k][1].max()]
    lam = dict(zip(valid, H.core(H.OP_LAMBDA, [red[k][1] for k in valid], device=True)[:, 0]))
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:           # the hooks run without the GIL
        refs = dict(zip(valid, ex.map(lambda k: _reference(red[k][1], lam[k], dev[k][1]), valid)))
    want = {c: np.asarray(a) for c, a in oracle_rows(table, "EWMA", emit_all=True, reducer=reducer)[0].items()}
    errs, spreads, stables, worst_ulps, worst_trip, n_off, worst_off = [], [], [], 0, 0.0, 0, 0.0
    for k in keys:
        times, v = red[k]
        dcalc, dy = dev[k]
        g = got["src_ip"] == k
        # (1) the fit kernel's scheduling against one thread per prefix fit: the same rows, bit for bit
        assert g.any() == (dcalc is not None), "series %#x: emitted by %s only" % (k, "the kernel" if g.any() else "the reference")
        if not g.any():
            continue
        o = np.argsort(got["flow_end"][g])
        row = {c: np.asarray(a)[g][o] for c, a in got.items()}
        w = want["src_ip"] == k
        wo = np.argsort(want["flow_end"][w])
        assert np.array_equal(row["flow_end"], times) and np.array_equal(row["flow_end"], want["flow_end"][w][wo])
        for c in ("dst_ip", "src_port", "dst_port", "proto", "flow_start", "throughput"):
            assert np.array_equal(row[c], want[c][w][wo]), (k, c)
        assert np.array_equal(row["stddev"], want["stddev"][w][wo], equal_nan=True), k
        assert np.array_equal(row["throughput"], v.astype(np.float64)), k
        off = row["algo_calc"] != dcalc
        n_off += int(off.sum())
        # the train points and the inverse transform are the same instructions in both: exact
        assert not off[:3].any(), k
        if off.any():
            worst_off = max(worst_off, float((np.abs(row["algo_calc"] - dcalc) / dcalc).max()))
        x, sd = v.astype(np.float64), row["stddev"][0]
        assert np.array_equal(row["anomaly"].astype(bool), np.abs(x - row["algo_calc"]) > sd), k
        # (2) the device's log, Box-Cox lambda and transform against the host's at the same lambda
        hy = H.transform(v, lam[k])
        assert hy is not None, k
        worst_ulps = max(worst_ulps, int(_ulps(dy, hy).max()))
        # (3) the fits: the device core against the host core on the device's transformed series
        base, runs = refs[k]
        assert base is not None or any(r is not None for r in runs), "series %#x: emitted by the GPU only" % k
        if base is None:
            continue                            # emitted where a nudged host run emits too: nothing to compare with
        err = np.abs(dcalc - base) / np.abs(base)
        worst_trip = max(worst_trip, float(err[:3].max()))
        spread = np.max([np.abs(r - base) / np.abs(base) if r is not None else np.full(len(base), np.inf) for r in runs],
                        axis=0)
        kerr = np.abs(row["algo_calc"] - base) / np.abs(base)
        errs.append(np.maximum(err, kerr)[3:]); spreads.append(spread[3:]); stables.append(spread[3:] <= STABLE)
    err, spread, stable = np.concatenate(errs), np.concatenate(spreads), np.concatenate(stables)
    n_all, n_stable = len(err), int(stable.sum())
    worst = float(err[stable].max()) if n_stable else 0.0
    n_far, n_far_host = int((err > 1e-3).sum()), int((spread > 1e-3).sum())
    print("ARIMA prefixes (reducer %d): %d fits; kernel vs device reference: %d prefixes not bit-equal (worst %.2e); "
          "transform within %d ulp of the host's; t < 3 within %.1e; stable %.1f %% (worst error %.2e), %d unstable "
          "(worst error %.2e); beyond 1e-3: device %d, host nudges %d"
          % (reducer, n_all, n_off, worst_off, worst_ulps, worst_trip, 100.0 * n_stable / n_all, worst, n_all - n_stable,
             err[~stable].max(), n_far, n_far_host))
    assert n_all >= 4000 and n_stable >= MIN_STABLE_SHARE * n_all
    assert n_off <= KERNEL_OFF_MAX * n_all, n_off
    assert worst_ulps <= TRANSFORM_ULPS and worst_trip <= 1e-14
    assert worst <= STABLE_TOL, worst
    assert n_far <= FAR_MAX * n_all, n_far


def test_every_prefix_against_the_host_core(prefix_rows, prefix_table):
    _check_prefixes(prefix_rows, prefix_table, 0)


def test_duplicates_under_the_sum_reducer(engine, prefix_table):
    """The table's duplicate-bearing series (and the rest) with (key, time) duplicates summed instead of maxed."""
    got, st = engine.run(prefix_table, algo="ARIMA", tad_id="prefix-sum", emit_all=True, reducer=1)
    assert st["state"] == "COMPLETED"
    _check_prefixes(got, prefix_table, 1)


# ------------------------------------------------------------------------------------------------
# C. the same table through the spill path and through a fit that yields
# ------------------------------------------------------------------------------------------------
def test_spill_path_rows_are_the_same(prefix_rows, prefix_table):
    """Two hash buckets, and 10,000 two-point connections (too short to fit, so they add no rows) beside the table, so that
    each bucket holds more rows than the group kernel's largest class and every series takes the spill path."""
    from theia_b200.engine import TadEngine
    m = 10_000
    filler = {"src_ip": np.arange(m, dtype=np.uint32).repeat(2) + np.uint32(0x0C000000),
              "dst_ip": np.full(2 * m, 0x0A000001, np.uint32), "src_port": np.full(2 * m, 4000, np.uint16),
              "dst_port": np.full(2 * m, 443, np.uint16), "proto": np.full(2 * m, 6, np.uint8),
              "flow_start": np.full(2 * m, synth.T0, np.uint32),
              "flow_end": np.tile([synth.T0 + 60, synth.T0 + 120], m).astype(np.uint32),
              "value": np.tile([300, 410], m).astype(np.uint64)}
    table = {k: np.concatenate([prefix_table[k], filler[k]]) for k in prefix_table}
    os.environ["TAD_DEBUG_LOGB"] = "1"
    try:
        eng = TadEngine(device=0)
    finally:
        del os.environ["TAD_DEBUG_LOGB"]
    try:
        got, st = eng.run(table, algo="ARIMA", tad_id="prefix-spill", emit_all=True)
    finally:
        eng.close()
    assert st["state"] == "COMPLETED" and st["spill_rows"] == st["rows_kept"]
    assert_same_rows(got, prefix_rows, what="ARIMA through the spill path")


def test_yielding_fit_rows_are_the_same(engine, prefix_rows, prefix_table):
    """The table as the running fit while short EWMA jobs queue behind it back to back: the fit yields to them, and its
    resume launch fits again the prefixes it dropped in flight."""
    ewma = engine.columns_from_numpy(synth.make_flows(500, 50, seed=13))
    cols = engine.columns_from_numpy(prefix_table)
    engine.set_fit_sharing(256 << 20)
    stop, errors = threading.Event(), []

    def stream():
        try:
            while not stop.is_set():
                q = engine.submit(ewma, algo="EWMA", tad_id="queued")
                q.wait()
                q.release()
        except Exception as e:          # reported below
            errors.append(e)
    job = engine.submit(cols, algo="ARIMA", tad_id="prefix-yield", emit_all=True)
    th = threading.Thread(target=stream)
    try:
        t0 = time.time()
        while job.progress()["fits_done"] == 0:
            assert job.poll()["state"] in ("SCHEDULED", "RUNNING") and time.time() - t0 < 60.0, job.poll()
            time.sleep(0.002)
        th.start()
        job.wait()
        stop.set()
        th.join()
        rows, y = job.result(), job.yields()
    finally:
        stop.set()
        engine.set_fit_sharing(0)
        job.release()
        cols.free()
        ewma.free()
    print("ARIMA prefix table under queued jobs: %d yields, parked %.1f ms" % (y["yields"], y["parked_ms"]))
    assert not errors, errors
    assert y["yields"] >= 1
    assert_same_rows(rows, prefix_rows, what="ARIMA fit that yields")
