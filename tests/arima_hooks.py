"""Bindings of the ARIMA core's test hooks (tad_arima.cu; not part of the C ABI in theia_tad.h) and plain high-precision
restatements of the functions they run, shared by the host and device precision tests."""
import ctypes as C

import mpmath
import numpy as np

from oracle import arima_oracle as ao

DPS = 50
OP_LAMBDA, OP_BOXCOX_LLF, OP_LOGLIKE, OP_FG, OP_START = range(5)


def lib():
    from theia_b200 import _lib
    L = _lib.load()
    for name in ("tad_debug_arima_host", "tad_debug_arima_device"):
        getattr(L, name).argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        getattr(L, name).restype = C.c_int
    L.tad_debug_arima_series.argtypes = [C.c_void_p, C.c_uint32, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int]
    L.tad_debug_arima_series.restype = C.c_int
    L.tad_debug_arima_series_device.argtypes = [C.c_void_p] * 5 + [C.c_uint32] + [C.c_void_p] * 3
    L.tad_debug_arima_series_device.restype = C.c_int
    return L


def core(op, xs, pars=None, device=False):
    """One op of tad::arima_debug_case on every case: xs = the cases' inputs (u64 arrays for OP_LAMBDA, float64
    otherwise), pars = their parameters (up to 4 each).  Returns an array of 8 results per case."""
    words = [np.ascontiguousarray(x).view(np.uint64) if len(x) else np.zeros(0, np.uint64) for x in xs]
    lens = np.array([len(w) for w in words], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    x = np.concatenate(words + [np.zeros(1, np.uint64)])
    par = np.zeros((len(xs), 4))
    for c, p in enumerate(pars if pars is not None else []):
        par[c, :len(p)] = p
    out = np.zeros((len(xs), 8))
    L = lib()
    fn = L.tad_debug_arima_device if device else L.tad_debug_arima_host
    rc = fn(op, x.ctypes.data, offs.ctypes.data, lens.ctypes.data, par.ctypes.data, len(xs), out.ctypes.data)
    assert rc == 0, "tad_debug_arima_%s: error %d" % ("device" if device else "host", rc)
    return out


def series(values, lam=float("nan"), nudge=0, y=None):
    """tad_debug_arima_series on the host: (calc or None, lambda used).  y: the transformed series to fit instead of the
    values' own (then lam is its lambda)."""
    v = np.ascontiguousarray(values, dtype=np.uint64)
    calc = np.zeros(max(len(v), 1))
    lam_out = C.c_double()
    yy = np.ascontiguousarray(y, dtype=np.float64) if y is not None else None
    ok = lib().tad_debug_arima_series(v.ctypes.data, len(v), lam, nudge, calc.ctypes.data, C.byref(lam_out),
                                      yy.ctypes.data if yy is not None else None, int(yy is not None))
    return (calc[:len(v)] if ok else None), lam_out.value


def transform(values, lam):
    """The host's transformed series of tad_debug_arima_series at lambda lam (None if the series yields no rows)."""
    v = np.ascontiguousarray(values, dtype=np.uint64)
    y, lam_out = np.zeros(max(len(v), 1)), C.c_double()
    ok = lib().tad_debug_arima_series(v.ctypes.data, len(v), lam, 0, None, C.byref(lam_out), y.ctypes.data, 0)
    return y[:len(v)] if ok else None


def series_device(values, lams=None, ys=None):
    """tad_debug_arima_series_device on a list of series: [(calc or None, transformed series)].  lams: each series' lambda
    (NaN or None: the device's Brent MLE); ys: the transformed series to fit instead (then lams are their lambdas)."""
    lens = np.array([len(v) for v in values], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    v = np.concatenate([np.asarray(x, dtype=np.uint64) for x in values] + [np.zeros(1, np.uint64)])
    lam = np.full(len(values), np.nan) if lams is None else np.ascontiguousarray(lams, dtype=np.float64)
    y_in = np.concatenate([np.asarray(y, dtype=np.float64) for y in ys] + [np.zeros(1)]) if ys is not None else None
    calc, y_out, ok = np.zeros(len(v)), np.zeros(len(v)), np.zeros(len(values), dtype=np.int32)
    rc = lib().tad_debug_arima_series_device(v.ctypes.data, offs.ctypes.data, lens.ctypes.data, lam.ctypes.data,
                                             y_in.ctypes.data if y_in is not None else None, len(values), calc.ctypes.data,
                                             y_out.ctypes.data, ok.ctypes.data)
    assert rc == 0, "tad_debug_arima_series_device: error %d" % rc
    return [(calc[o:o + n].copy() if k else None, y_out[o:o + n].copy()) for o, n, k in zip(offs, lens, ok)]


def mp_kalman(y, phi, theta, s2):
    """oracle/arima_oracle.py:kalman_loglike in mpmath at DPS digits: (loglike, forecast), or None where the double
    filter gives up (F <= 0)."""
    with mpmath.workdps(DPS):
        mpf = mpmath.mpf
        phi, theta, s2 = mpf(phi), mpf(theta), mpf(s2)
        a0 = a1 = a2 = mpf(0)
        p00, p01, p02 = mpf(ao.DIFFUSE_VARIANCE), mpf(0), mpf(0)
        p11 = s2 * (1 + 2 * phi * theta + theta * theta) / (1 - phi * phi)
        p12, p22 = s2 * theta, s2 * theta * theta
        q11, q12, q22 = s2, s2 * theta, s2 * theta * theta
        ll = mpf(0)
        log2pi = mpmath.log(2 * mpmath.pi)
        for t, yt in enumerate(y):
            v = mpf(float(yt)) - (a0 + a1)
            F = p00 + 2 * p01 + p11
            if not F > 0:
                return None
            if t >= 1:
                ll += -(log2pi + mpmath.log(F) + v * v / F) / 2
            z0, z1, z2 = p00 + p01, p01 + p11, p02 + p12
            g = v / F
            f0, f1, f2 = a0 + z0 * g, a1 + z1 * g, a2 + z2 * g
            c00, c01, c02 = p00 - z0 * z0 / F, p01 - z0 * z1 / F, p02 - z0 * z2 / F
            c11, c12, c22 = p11 - z1 * z1 / F, p12 - z1 * z2 / F, p22 - z2 * z2 / F
            a0, a1, a2 = f0 + f1, phi * f1 + f2, mpf(0)
            p00 = c00 + 2 * c01 + c11
            p01 = phi * (c01 + c11) + c02 + c12
            p02 = mpf(0)
            p11 = phi * phi * c11 + 2 * phi * c12 + c22 + q11
            p12, p22 = q12, q22
        return ll, a0 + a1


def mp_boxcox_neg_llf(lmb, logx):
    """-scipy.stats.boxcox_llf(lmb, x) at DPS digits, from the double log values: (lmb - 1) sum(log x) is the Jacobian
    term, the variance that of x^lmb / lmb (of log x at lmb = 0); exact however large x^lmb gets."""
    with mpmath.workdps(DPS):
        lx = [mpmath.mpf(float(q)) for q in logx]
        n = len(lx)
        z = lx if lmb == 0 else [mpmath.exp(lmb * q) / lmb for q in lx]
        mean = mpmath.fsum(z) / n
        var = mpmath.fsum((q - mean) ** 2 for q in z) / n
        return -((lmb - 1) * mpmath.fsum(lx) - mpmath.mpf(n) / 2 * mpmath.log(var))
