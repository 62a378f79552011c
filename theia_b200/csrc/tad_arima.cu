// ARIMA detector (anomaly_detection.py:215-309): Box-Cox (MLE lambda) -> for every prefix of the
// series an ARIMA(1,1,1) state-space MLE fit and one-step forecast -> inverse Box-Cox -> flag.
//
// The per-fit algorithm is the one statsmodels 0.14 runs (see oracle/arima_oracle.py for the
// statement of it and for the parity status -- unpinned below ~1e-3 relative on algoCalc):
//   * 3-state Kalman filter likelihood, approximate-diffuse + stationary initialisation, burn 1;
//   * optimisation over the unconstrained parameters by L-BFGS with a More'-Thuente line search
//     (the unconstrained path of L-BFGS-B: m = 12, pgtol 1e-8, factr 1e2, maxiter 50,
//     forward-difference gradient with step 1e-8) on -loglike / nobs;
//   * Hannan-Rissanen start values.
// Compute-bound FP64 (about n^2/2 Kalman steps x ~100 likelihood evaluations per series), so the
// mapping is one WARP per series with one lane per prefix fit; the series lives in L1.
#include <algorithm>
#include <cfloat>
#include <vector>

#include "tad_kernels.h"

namespace tad {

inline namespace arima_core {

constexpr double kDiffuse = 1e6;
constexpr double kLog2Pi = 1.8378770664093454835606594728112;
constexpr int kLbfgsM = 12;

__device__ __forceinline__ SeriesEntry load_entry(const SeriesEntry *entries, const uint32_t *offsets, const uint32_t *sbase,
                                                  uint32_t B, uint32_t i)
{
    const uint32_t b = find_bucket(sbase, B, i);
    const uint4 *p = reinterpret_cast<const uint4 *>(entries + offsets[b] + (i - sbase[b]));
    const uint4 k = p[0], w = p[1];
    SeriesEntry e;
    e.a = ((uint64_t)k.y << 32) | k.x; e.b = ((uint64_t)k.w << 32) | k.z;
    e.proto = w.x; e.n = w.y; e.off = w.z; e.pad = w.w;
    return e;
}

// ------------------------------------------------------------------------------------------
// Box-Cox: llf(lambda) = (lambda - 1) sum(log x) - N/2 log var(x^lambda / lambda)   (scipy.stats.boxcox_llf)
// ------------------------------------------------------------------------------------------
// The variance of x^lambda / lambda is evaluated in log space (var = e^{2m} var(e^{z - m}) / lambda^2 with
// z = lambda log x, m = max z), so the likelihood stays finite for any lambda and Brent converges to the
// true optimum even when the transform itself would overflow (the caller then drops the series).
__host__ __device__ double boxcox_neg_llf(double lmb, const double *__restrict__ logx, uint32_t n, double sumlog)
{
    double logvar;
    if (lmb == 0.0) {
        double mean = 0.0;
        for (uint32_t i = 0; i < n; i++) mean += logx[i];
        mean /= n;
        double var = 0.0;
        for (uint32_t i = 0; i < n; i++) { const double d = logx[i] - mean; var += d * d; }
        logvar = log(var / n);
    } else {
        double m = -DBL_MAX;
        for (uint32_t i = 0; i < n; i++) m = fmax(m, lmb * logx[i]);
        double mean = 0.0;
        for (uint32_t i = 0; i < n; i++) mean += exp(lmb * logx[i] - m);
        mean /= n;
        double var = 0.0;
        for (uint32_t i = 0; i < n; i++) { const double d = exp(lmb * logx[i] - m) - mean; var += d * d; }
        logvar = log(var / n) + 2.0 * m - 2.0 * log(fabs(lmb));
    }
    return -((lmb - 1.0) * sumlog - 0.5 * n * logvar);
}

// scipy.optimize.brent(f, brack=(-2, 2)): bracket() followed by Brent's parabolic/golden iteration, tol 1.48e-8
__host__ __device__ double boxcox_mle_lambda(const double *__restrict__ logx, uint32_t n, double sumlog)
{
    auto f = [&](double l) { return boxcox_neg_llf(l, logx, n, sumlog); };
    const double gold = 1.618034, verysmall = 1e-21, grow = 110.0;
    double xa = -2.0, xb = 2.0;
    double fa = f(xa), fb = f(xb);
    if (fa < fb) { double t = xa; xa = xb; xb = t; t = fa; fa = fb; fb = t; }
    double xc = xb + gold * (xb - xa), fc = f(xc);
    int iter = 0;
    while (fc < fb && iter < 1000) {
        const double tmp1 = (xb - xa) * (fb - fc), tmp2 = (xb - xc) * (fb - fa);
        const double val = tmp2 - tmp1;
        const double denom = fabs(val) < verysmall ? 2.0 * verysmall : 2.0 * val;
        double w = xb - ((xb - xc) * tmp2 - (xb - xa) * tmp1) / denom;
        const double wlim = xb + grow * (xc - xb);
        double fw;
        iter++;
        if ((w - xc) * (xb - w) > 0.0) {
            fw = f(w);
            if (fw < fc) { xa = xb; xb = w; fa = fb; fb = fw; break; }
            else if (fw > fb) { xc = w; fc = fw; break; }
            w = xc + gold * (xc - xb); fw = f(w);
        } else if ((w - wlim) * (wlim - xc) >= 0.0) {
            w = wlim; fw = f(w);
        } else if ((w - wlim) * (xc - w) > 0.0) {
            fw = f(w);
            if (fw < fc) { xb = xc; xc = w; w = xc + gold * (xc - xb); fb = fc; fc = fw; fw = f(w); }
        } else {
            w = xc + gold * (xc - xb); fw = f(w);
        }
        xa = xb; xb = xc; xc = w; fa = fb; fb = fc; fc = fw;
    }
    const double mintol = 1.0e-11, cg = 0.3819660, tol = 1.48e-8;
    double x = xb, w = xb, v = xb, fx = fb, fw = fb, fv = fb;
    double a = xa < xc ? xa : xc, b = xa < xc ? xc : xa;
    double deltax = 0.0, rat = 0.0;
    for (iter = 0; iter < 500; iter++) {
        const double tol1 = tol * fabs(x) + mintol, tol2 = 2.0 * tol1, xmid = 0.5 * (a + b);
        if (fabs(x - xmid) < (tol2 - 0.5 * (b - a))) break;
        if (fabs(deltax) <= tol1) {
            deltax = x >= xmid ? a - x : b - x;
            rat = cg * deltax;
        } else {
            double tmp1 = (x - w) * (fx - fv), tmp2 = (x - v) * (fx - fw);
            double p = (x - v) * tmp2 - (x - w) * tmp1;
            tmp2 = 2.0 * (tmp2 - tmp1);
            if (tmp2 > 0.0) p = -p;
            tmp2 = fabs(tmp2);
            const double dx_temp = deltax;
            deltax = rat;
            if (p > tmp2 * (a - x) && p < tmp2 * (b - x) && fabs(p) < fabs(0.5 * tmp2 * dx_temp)) {
                rat = p / tmp2;
                const double u = x + rat;
                if ((u - a) < tol2 || (b - u) < tol2) rat = (xmid - x >= 0) ? tol1 : -tol1;
            } else {
                deltax = x >= xmid ? a - x : b - x;
                rat = cg * deltax;
            }
        }
        const double u = fabs(rat) < tol1 ? (rat >= 0 ? x + tol1 : x - tol1) : x + rat;
        const double fu = f(u);
        if (fu > fx) {
            if (u < x) a = u; else b = u;
            if (fu <= fw || w == x) { v = w; w = u; fv = fw; fw = fu; }
            else if (fu <= fv || v == x || v == w) { v = u; fv = fu; }
        } else {
            if (u >= x) a = x; else b = x;
            v = w; w = x; x = u; fv = fw; fw = fx; fx = fu;
        }
    }
    return x;
}

// ------------------------------------------------------------------------------------------
// ARIMA(1,1,1) likelihood (3-state Kalman filter, symmetric P as six scalars)
// ------------------------------------------------------------------------------------------
struct ArimaObj {
    const double *y;
    uint32_t n;
};

__host__ __device__ __forceinline__ void arima_transform(const double u[3], double &phi, double &theta, double &s2)
{
    phi = u[0] / sqrt(1.0 + u[0] * u[0]);
    theta = u[1] / sqrt(1.0 + u[1] * u[1]);
    s2 = u[2] * u[2];
}

// One filter: the state the recursion carries (a2 = p02 = 0, p12 = q12, p22 = q22 after every prediction step, so they are
// constants of the parameters) and one time step.  arima_loglike runs one of these; arima_fg runs FOUR side by side in one
// loop -- the objective at u and at its three forward-difference neighbours -- so that a lane has four independent FP64
// dependency chains in flight instead of one (the arithmetic of every chain is exactly that of the single filter).
struct Kalman {
    double phi, q11, q12, q22;
    double a0, a1, a2, p00, p01, p02, p11, p12, p22, ll;
    bool dead;                       // F <= 0 or not finite at some step: the likelihood is -1e300 (statsmodels raises)
};

__host__ __device__ __forceinline__ void kalman_init(Kalman &k, double phi, double theta, double s2)
{
    k.phi = phi;
    k.a0 = 0.0; k.a1 = 0.0; k.a2 = 0.0;
    k.p00 = kDiffuse; k.p01 = 0.0; k.p02 = 0.0;
    k.p11 = s2 * (1.0 + 2.0 * phi * theta + theta * theta) / (1.0 - phi * phi);
    k.p12 = s2 * theta; k.p22 = s2 * theta * theta;
    k.q11 = s2; k.q12 = s2 * theta; k.q22 = s2 * theta * theta;
    k.ll = 0.0;
    k.dead = false;
}

__host__ __device__ __forceinline__ void kalman_step(Kalman &k, double yt, bool count)
{
    const double v = yt - (k.a0 + k.a1);
    const double F = k.p00 + 2.0 * k.p01 + k.p11;
    if (!(F > 0.0) || !isfinite(F)) { k.dead = true; return; }
    if (count) k.ll += -0.5 * (kLog2Pi + log(F) + v * v / F);
    const double z0 = k.p00 + k.p01, z1 = k.p01 + k.p11, z2 = k.p02 + k.p12;
    const double g = v / F;
    const double f0 = k.a0 + z0 * g, f1 = k.a1 + z1 * g, f2 = k.a2 + z2 * g;
    const double c00 = k.p00 - z0 * z0 / F, c01 = k.p01 - z0 * z1 / F, c02 = k.p02 - z0 * z2 / F;
    const double c11 = k.p11 - z1 * z1 / F, c12 = k.p12 - z1 * z2 / F, c22 = k.p22 - z2 * z2 / F;
    k.a0 = f0 + f1; k.a1 = k.phi * f1 + f2; k.a2 = 0.0;
    k.p00 = c00 + 2.0 * c01 + c11;
    k.p01 = k.phi * (c01 + c11) + c02 + c12;
    k.p02 = 0.0;
    k.p11 = k.phi * k.phi * c11 + 2.0 * k.phi * c12 + c22 + k.q11;
    k.p12 = k.q12;
    k.p22 = k.q22;
}

__host__ __device__ double arima_loglike(const ArimaObj &o, double phi, double theta, double s2, double *forecast)
{
    Kalman k;
    kalman_init(k, phi, theta, s2);
    for (uint32_t t = 0; t < o.n && !k.dead; t++) kalman_step(k, o.y[t], t >= 1);
    if (k.dead) {
        if (forecast) *forecast = 0.0;
        return -1e300;
    }
    if (forecast) *forecast = k.a0 + k.a1;
    return k.ll;
}

__host__ __device__ __forceinline__ double arima_objective(const ArimaObj &o, const double u[3])
{
    double phi, theta, s2;
    arima_transform(u, phi, theta, s2);
    return -arima_loglike(o, phi, theta, s2, nullptr) / (double)o.n;
}

// f and the forward-difference gradient (step 1e-8, as SciPy's approx_fprime drives L-BFGS-B): four filters in one loop
__host__ __device__ void arima_fg(const ArimaObj &o, double u[3], double &f, double g[3])
{
    Kalman k[4];
    for (int c = 0; c < 4; c++) {
        double uc[3] = {u[0], u[1], u[2]};
        if (c > 0) uc[c - 1] = u[c - 1] + 1e-8;
        double phi, theta, s2;
        arima_transform(uc, phi, theta, s2);
        kalman_init(k[c], phi, theta, s2);
    }
    for (uint32_t t = 0; t < o.n; t++) {
        const double yt = o.y[t];
        const bool count = t >= 1;
#pragma unroll
        for (int c = 0; c < 4; c++)
            if (!k[c].dead) kalman_step(k[c], yt, count);
    }
    double fv[4];
    for (int c = 0; c < 4; c++) fv[c] = -(k[c].dead ? -1e300 : k[c].ll) / (double)o.n;
    f = fv[0];
    for (int c = 0; c < 3; c++) g[c] = (fv[c + 1] - f) / 1e-8;
}

// Least-squares solution of a two-regressor problem from its normal equations, following numpy.linalg.pinv:
// full rank -> the unique solution; rank one (singular value ratio below 1e-15) -> the minimum-norm solution
// b / trace(A); rank zero -> 0.
__host__ __device__ __forceinline__ void lstsq2(double s11, double s12, double s22, double r1, double r2, double &b1, double &b2)
{
    const double tr = s11 + s22, det = s11 * s22 - s12 * s12;
    b1 = 0.0; b2 = 0.0;
    if (!(tr > 0.0) || !isfinite(tr)) return;
    if (det > 1e-30 * tr * tr) {
        b1 = (r1 * s22 - r2 * s12) / det;
        b2 = (r2 * s11 - r1 * s12) / det;
    } else {
        b1 = r1 / tr;
        b2 = r2 / tr;
    }
}

// Hannan-Rissanen / conditional-sum-of-squares start values on the differenced data (k_ar = k_ma = 1)
__host__ __device__ void arima_start(const ArimaObj &o, double u[3])
{
    const double *y = o.y;
    const int m = (int)o.n - 1;                      // d[i] = y[i+1] - y[i]
    auto d = [&](int i) { return y[i + 1] - y[i]; };
    double phi0 = 0.0, th0 = 0.0, var = NAN;
    double dmean = 0.0;
    for (int i = 0; i < m; i++) dmean += d(i);
    dmean = m > 0 ? dmean / m : 0.0;
    double dvar = 0.0;
    for (int i = 0; i < m; i++) { const double e = d(i) - dmean; dvar += e * e; }
    dvar = m > 0 ? dvar / m : 0.0;
    if (m >= 4) {
        // AR(2) by least squares: d[t] ~ b1 d[t-1] + b2 d[t-2], t = 2..m-1
        double s11 = 0, s12 = 0, s22 = 0, r1 = 0, r2 = 0;
        for (int t = 2; t < m; t++) {
            const double x1 = d(t - 1), x2 = d(t - 2), yy = d(t);
            s11 += x1 * x1; s12 += x1 * x2; s22 += x2 * x2; r1 += x1 * yy; r2 += x2 * yy;
        }
        double b1, b2;
        lstsq2(s11, s12, s22, r1, r2, b1, b2);
        auto res = [&](int t) { return d(t) - b1 * d(t - 1) - b2 * d(t - 2); };      // residual at t >= 2
        // ARMA(1,1): d[t] ~ phi d[t-1] + theta res[t-1], t = 3..m-1
        s11 = s12 = s22 = r1 = r2 = 0;
        for (int t = 3; t < m; t++) {
            const double x1 = d(t - 1), x2 = res(t - 1), yy = d(t);
            s11 += x1 * x1; s12 += x1 * x2; s22 += x2 * x2; r1 += x1 * yy; r2 += x2 * yy;
        }
        lstsq2(s11, s12, s22, r1, r2, phi0, th0);
        if (m - 3 > 1) {
            double acc = 0.0;
            for (int t = 4; t < m; t++) { const double e = d(t) - phi0 * d(t - 1) - th0 * res(t - 1); acc += e * e; }
            var = acc / (m - 4);
        }
    }
    if (!(fabs(phi0) < 1.0)) phi0 = 0.0;
    if (!(fabs(th0) < 1.0)) th0 = 0.0;
    if (!isfinite(var) || var <= 1e-10 * dvar || var <= 0.0) var = dvar > 0.0 ? dvar : 1.0;
    u[0] = phi0 / sqrt(1.0 - phi0 * phi0);
    u[1] = th0 / sqrt(1.0 - th0 * th0);
    u[2] = sqrt(var);
}

// ------------------------------------------------------------------------------------------
// More'-Thuente line search (MINPACK-2 dcsrch / dcstep), as driven by L-BFGS-B's lnsrlb
// ------------------------------------------------------------------------------------------
struct LineSearch {
    bool brackt;
    int stage;
    double ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1;
};
enum { LS_FG = 0, LS_CONV = 1, LS_WARN = 2 };

__host__ __device__ void dcstep(double &stx, double &fx, double &dx, double &sty, double &fy, double &dy, double &stp, double fp, double dp,
                       bool &brackt, double stpmin, double stpmax)
{
    const double sgnd = dp * (dx / fabs(dx));
    double stpf;
    if (fp > fx) {
        const double theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
        const double s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
        double gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
        if (stp < stx) gamma = -gamma;
        const double p = (gamma - dx) + theta, q = ((gamma - dx) + gamma) + dp, r = p / q;
        const double stpc = stx + r * (stp - stx);
        const double stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / 2.0) * (stp - stx);
        stpf = fabs(stpc - stx) < fabs(stpq - stx) ? stpc : stpc + (stpq - stpc) / 2.0;
        brackt = true;
    } else if (sgnd < 0.0) {
        const double theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
        const double s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
        double gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
        if (stp > stx) gamma = -gamma;
        const double p = (gamma - dp) + theta, q = ((gamma - dp) + gamma) + dx, r = p / q;
        const double stpc = stp + r * (stx - stp);
        const double stpq = stp + (dp / (dp - dx)) * (stx - stp);
        stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
        brackt = true;
    } else if (fabs(dp) < fabs(dx)) {
        const double theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
        const double s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
        double gamma = s * sqrt(fmax(0.0, (theta / s) * (theta / s) - (dx / s) * (dp / s)));
        if (stp > stx) gamma = -gamma;
        const double p = (gamma - dp) + theta, q = (gamma + (dx - dp)) + gamma, r = p / q;
        double stpc;
        if (r < 0.0 && gamma != 0.0) stpc = stp + r * (stx - stp);
        else if (stp > stx) stpc = stpmax;
        else stpc = stpmin;
        const double stpq = stp + (dp / (dp - dx)) * (stx - stp);
        if (brackt) {
            stpf = fabs(stpc - stp) < fabs(stpq - stp) ? stpc : stpq;
            if (stp > stx) stpf = fmin(stp + 0.66 * (sty - stp), stpf);
            else stpf = fmax(stp + 0.66 * (sty - stp), stpf);
        } else {
            stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
            stpf = fmin(stpmax, stpf);
            stpf = fmax(stpmin, stpf);
        }
    } else {
        if (brackt) {
            const double theta = 3.0 * (fp - fy) / (sty - stp) + dy + dp;
            const double s = fmax(fabs(theta), fmax(fabs(dy), fabs(dp)));
            double gamma = s * sqrt((theta / s) * (theta / s) - (dy / s) * (dp / s));
            if (stp > sty) gamma = -gamma;
            const double p = (gamma - dp) + theta, q = ((gamma - dp) + gamma) + dy, r = p / q;
            stpf = stp + r * (sty - stp);
        } else if (stp > stx) stpf = stpmax;
        else stpf = stpmin;
    }
    if (fp > fx) {
        sty = stp; fy = fp; dy = dp;
    } else {
        if (sgnd < 0.0) { sty = stx; fy = fx; dy = dx; }
        stx = stp; fx = fp; dx = dp;
    }
    stp = stpf;
}

__host__ __device__ void dcsrch_start(LineSearch &ls, double stp, double f, double g, double ftol, double stpmin, double stpmax)
{
    ls.brackt = false;
    ls.stage = 1;
    ls.finit = f; ls.ginit = g; ls.gtest = ftol * g;
    ls.width = stpmax - stpmin; ls.width1 = ls.width / 0.5;
    ls.stx = 0.0; ls.fx = f; ls.gx = g;
    ls.sty = 0.0; ls.fy = f; ls.gy = g;
    ls.stmin = 0.0; ls.stmax = stp + 4.0 * stp;
}

__host__ __device__ int dcsrch_step(LineSearch &ls, double &stp, double f, double g, double ftol, double gtol, double xtol, double stpmin,
                           double stpmax)
{
    const double ftest = ls.finit + stp * ls.gtest;
    if (ls.stage == 1 && f <= ftest && g >= 0.0) ls.stage = 2;
    int task = LS_FG;
    if (ls.brackt && (stp <= ls.stmin || stp >= ls.stmax)) task = LS_WARN;
    if (ls.brackt && ls.stmax - ls.stmin <= xtol * ls.stmax) task = LS_WARN;
    if (stp == stpmax && f <= ftest && g <= ls.gtest) task = LS_WARN;
    if (stp == stpmin && (f > ftest || g >= ls.gtest)) task = LS_WARN;
    if (f <= ftest && fabs(g) <= gtol * (-ls.ginit)) task = LS_CONV;
    if (task != LS_FG) return task;
    if (ls.stage == 1 && f <= ls.fx && f > ftest) {
        const double fm = f - stp * ls.gtest;
        double fxm = ls.fx - ls.stx * ls.gtest, fym = ls.fy - ls.sty * ls.gtest;
        const double gm = g - ls.gtest;
        double gxm = ls.gx - ls.gtest, gym = ls.gy - ls.gtest;
        dcstep(ls.stx, fxm, gxm, ls.sty, fym, gym, stp, fm, gm, ls.brackt, ls.stmin, ls.stmax);
        ls.fx = fxm + ls.stx * ls.gtest; ls.fy = fym + ls.sty * ls.gtest;
        ls.gx = gxm + ls.gtest; ls.gy = gym + ls.gtest;
    } else {
        dcstep(ls.stx, ls.fx, ls.gx, ls.sty, ls.fy, ls.gy, stp, f, g, ls.brackt, ls.stmin, ls.stmax);
    }
    if (ls.brackt) {
        if (fabs(ls.sty - ls.stx) >= 0.66 * ls.width1) stp = ls.stx + 0.5 * (ls.sty - ls.stx);
        ls.width1 = ls.width;
        ls.width = fabs(ls.sty - ls.stx);
    }
    if (ls.brackt) {
        ls.stmin = fmin(ls.stx, ls.sty);
        ls.stmax = fmax(ls.stx, ls.sty);
    } else {
        ls.stmin = stp + 1.1 * (stp - ls.stx);
        ls.stmax = stp + 4.0 * (stp - ls.stx);
    }
    stp = fmax(stp, stpmin);
    stp = fmin(stp, stpmax);
    if ((ls.brackt && (stp <= ls.stmin || stp >= ls.stmax)) || (ls.brackt && ls.stmax - ls.stmin <= xtol * ls.stmax)) stp = ls.stx;
    return LS_FG;
}

// ------------------------------------------------------------------------------------------
// L-BFGS (the unconstrained path of L-BFGS-B 3.0 as SciPy drives it), written as a resumable state machine:
// the caller evaluates (f, g) at x, lbfgs_advance() consumes them and either leaves the next trial point in x
// (returns false) or ends the fit (returns true, x = the solution).  The host driver below loops over it; the fit
// kernel lets all lanes of a warp evaluate TOGETHER (the Kalman-filter likelihood, >95 % of the work, then runs
// converged) and only the cheap bookkeeping between two evaluations diverges.
// ------------------------------------------------------------------------------------------
struct Lbfgs {
    double S[kLbfgsM][3], Y[kLbfgsM][3], rho[kLbfgsM];
    int col, head, iter, ifun, state;        // state 0: first evaluation pending, 1: line-search evaluation pending
    double theta, f, g[3], d[3], stp, fold, xold[3], gold[3], gdold, gd;
    LineSearch ls;
};

__host__ __device__ __forceinline__ void lbfgs_init(Lbfgs &s)
{
    s.col = 0; s.head = 0; s.iter = 0; s.ifun = 0; s.state = 0; s.theta = 1.0;
}

// start iterations from (s.f, s.g) at x until a line search has its first trial point in x (false) or the fit ends (true)
__host__ __device__ bool lbfgs_begin_iter(Lbfgs &s, double x[3])
{
    const double stpmx = 1e10, ftol = 1e-3;
    for (;;) {
        if (s.iter >= 50) return true;
        // ---- direction d = -H g (two-loop recursion, H0 = I / theta) ------------------------
        double d[3] = {s.g[0], s.g[1], s.g[2]}, alpha[kLbfgsM];
        for (int k = s.col - 1; k >= 0; k--) {
            const int i = (s.head + k) % kLbfgsM;
            alpha[k] = s.rho[i] * (s.S[i][0] * d[0] + s.S[i][1] * d[1] + s.S[i][2] * d[2]);
            for (int c = 0; c < 3; c++) d[c] -= alpha[k] * s.Y[i][c];
        }
        for (int c = 0; c < 3; c++) d[c] /= s.theta;
        for (int k = 0; k < s.col; k++) {
            const int i = (s.head + k) % kLbfgsM;
            const double beta = s.rho[i] * (s.Y[i][0] * d[0] + s.Y[i][1] * d[1] + s.Y[i][2] * d[2]);
            for (int c = 0; c < 3; c++) d[c] += s.S[i][c] * (alpha[k] - beta);
        }
        for (int c = 0; c < 3; c++) s.d[c] = -d[c];
        // ---- line search ----------------------------------------------------------------------
        const double dnorm = sqrt(s.d[0] * s.d[0] + s.d[1] * s.d[1] + s.d[2] * s.d[2]);
        s.stp = s.iter == 0 ? fmin(1.0 / dnorm, stpmx) : 1.0;
        s.fold = s.f;
        for (int c = 0; c < 3; c++) { s.xold[c] = x[c]; s.gold[c] = s.g[c]; }
        s.gdold = s.g[0] * s.d[0] + s.g[1] * s.d[1] + s.g[2] * s.d[2];
        s.gd = s.gdold;
        const bool ok = s.gdold < 0.0 && isfinite(s.gdold) && dnorm > 0.0;
        if (ok) {
            dcsrch_start(s.ls, s.stp, s.f, s.gdold, ftol, 0.0, stpmx);
            s.ifun = 0;
            for (int c = 0; c < 3; c++) x[c] = s.xold[c] + s.stp * s.d[c];
            s.state = 1;
            return false;
        }
        // no descent direction: with stored pairs restart from steepest descent, else stop (x, f, g are unchanged)
        if (s.col == 0) return true;
        s.col = 0; s.head = 0; s.theta = 1.0;
    }
}

__host__ __device__ bool lbfgs_advance(Lbfgs &s, double x[3], double f, const double g[3])
{
    const double pgtol = 1e-8, factr = 1e2, epsmch = DBL_EPSILON, stpmx = 1e10;
    const double ftol = 1e-3, gtol = 0.9, xtol = 0.1;
    s.f = f;
    for (int c = 0; c < 3; c++) s.g[c] = g[c];
    if (s.state == 0) {
        if (fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2]))) <= pgtol) return true;
        return lbfgs_begin_iter(s, x);
    }
    // ---- an evaluation of the running line search ---------------------------------------------
    s.ifun++;
    s.gd = g[0] * s.d[0] + g[1] * s.d[1] + g[2] * s.d[2];
    bool ok = isfinite(f) && isfinite(s.gd);
    if (ok) {
        const int task = dcsrch_step(s.ls, s.stp, f, s.gd, ftol, gtol, xtol, 0.0, stpmx);
        if (task == LS_FG) {
            if (s.ifun >= 20) ok = false;
            else {
                for (int c = 0; c < 3; c++) x[c] = s.xold[c] + s.stp * s.d[c];
                return false;
            }
        }
    }
    if (!ok) {
        // line search failed: restore; with stored pairs restart from steepest descent, else stop
        s.f = s.fold;
        for (int c = 0; c < 3; c++) { x[c] = s.xold[c]; s.g[c] = s.gold[c]; }
        if (s.col == 0) return true;
        s.col = 0; s.head = 0; s.theta = 1.0;
        return lbfgs_begin_iter(s, x);
    }
    s.iter++;
    if (fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2]))) <= pgtol) return true;
    const double ddum = fmax(fabs(s.fold), fmax(fabs(f), 1.0));
    if (s.fold - f <= epsmch * factr * ddum) return true;
    // ---- update the limited-memory matrices ---------------------------------------------------
    double r[3], sv[3], rr = 0.0;
    for (int c = 0; c < 3; c++) { r[c] = g[c] - s.gold[c]; sv[c] = x[c] - s.xold[c]; rr += r[c] * r[c]; }
    double dr, dd;
    if (s.stp == 1.0) { dr = s.gd - s.gdold; dd = -s.gdold; }
    else { dr = (s.gd - s.gdold) * s.stp; dd = -s.gdold * s.stp; }
    if (dr > epsmch * dd) {
        int slot;
        if (s.col < kLbfgsM) { slot = (s.head + s.col) % kLbfgsM; s.col++; }
        else { slot = s.head; s.head = (s.head + 1) % kLbfgsM; }
        for (int c = 0; c < 3; c++) { s.S[slot][c] = sv[c]; s.Y[slot][c] = r[c]; }
        s.rho[slot] = 1.0 / dr;
        s.theta = rr / dr;
    }
    return lbfgs_begin_iter(s, x);
}

// one fit, evaluated and advanced in place (host tests; the sequential device path)
__host__ __device__ void arima_fit(const ArimaObj &o, double x[3])
{
    Lbfgs s;
    lbfgs_init(s);
    for (;;) {
        double f, g[3];
        arima_fg(o, x, f, g);
        if (lbfgs_advance(s, x, f, g)) return;
    }
}

}  // namespace arima_core

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------
// pred[t] of a prefix fit not written yet (a fit that can yield): a quiet NaN whose payload no computation makes.  The fit
// reads finite data only, so every NaN it can produce descends from the device's canonical NaN (0x7fffffffffffffff) or
// from NAN (0x7ff8000000000000), never from this payload.  A sentinel rather than a bitmap of written prefixes: it needs
// no buffer beyond pred[] and no atomics, and the resume launch reads the word it would overwrite anyway.
constexpr unsigned long long kPredUnset = 0x7ff80000000a7f17ull;

// The per-series steps of the detector, shared by the kernels and the host reference (tad_debug_arima_series), so that the
// reference runs the kernels' own arithmetic.
__host__ __device__ __forceinline__ double u64_to_double(uint64_t v)
{
#ifdef __CUDA_ARCH__
    return __ull2double_rn(v);
#else
    return (double)v;                                      // round to nearest, as __ull2double_rn
#endif
}

// log of the values into y[] and their sum; false if the series yields no rows: n <= 3, a zero value or constant values
__host__ __device__ __forceinline__ bool arima_log_series(const uint64_t *__restrict__ v, uint32_t n, double *__restrict__ y,
                                                          double &sumlog)
{
    bool valid = n > 3;                                   // anomaly_detection.py:232-234
    bool constant = true;
    sumlog = 0.0;
    for (uint32_t q = 0; q < n && valid; q++) {
        if (v[q] == 0) valid = false;                     // Box-Cox needs positive data (:260-264 -> None)
        if (v[q] != v[0]) constant = false;
        const double lx = log(u64_to_double(v[q]));
        y[q] = lx;
        sumlog += lx;
    }
    return valid && !constant;
}

// y[] = log x -> the Box-Cox transform at lambda l, in place; false if it is not finite (the series yields no rows)
__host__ __device__ __forceinline__ bool arima_boxcox_transform(double *__restrict__ y, uint32_t n, double l)
{
    bool finite = isfinite(l);
    for (uint32_t q = 0; q < n && finite; q++) {
        y[q] = l == 0.0 ? y[q] : expm1(l * y[q]) / l;     // scipy.special.boxcox
        finite = isfinite(y[q]);
    }
    return finite;
}

__host__ __device__ __forceinline__ double inv_boxcox_d(double y, double l)
{
    return l == 0.0 ? exp(y) : exp(log1p(l * y) / l);     // scipy.special.inv_boxcox
}

// one series: validity, Box-Cox lambda, transformed series into yb[]; returns its prefix fits (n - 3 with a lambda, else 0).
// unset (a fit that can yield): pred[], whose prefix forecasts [3, n) are marked kPredUnset.
__device__ __forceinline__ uint32_t arima_boxcox_series(const SeriesEntry *__restrict__ entries, const uint32_t *__restrict__ offsets,
                                                        const uint32_t *__restrict__ sbase, uint32_t B, uint32_t i,
                                                        const uint64_t *__restrict__ csr_v, double *__restrict__ yb,
                                                        double *__restrict__ lam, double *__restrict__ unset)
{
    const SeriesEntry e = load_entry(entries, offsets, sbase, B, i);
    const uint64_t *v = csr_v + e.off;
    double *y = yb + e.off;
    const uint32_t n = e.n;
    double sumlog;
    if (!arima_log_series(v, n, y, sumlog)) { lam[i] = NAN; return 0; }
    const double l = boxcox_mle_lambda(y, n, sumlog);
    const bool finite = arima_boxcox_transform(y, n, l);
    lam[i] = finite ? l : NAN;                             // overflowing transform -> the series yields no rows
    if (finite && unset)
        for (uint32_t q = 3; q < n; q++) unset[e.off + q] = __longlong_as_double((long long)kPredUnset);
    return finite ? n - 3 : 0u;
}

// one thread per series; *fits_total gains the prefix fits of the series (one atomic per warp)
__global__ void __launch_bounds__(128) arima_boxcox_kernel(const SeriesEntry *__restrict__ entries, const uint32_t *__restrict__ offsets,
                                                           const uint32_t *__restrict__ sbase, uint32_t B, uint32_t S,
                                                           const uint64_t *__restrict__ csr_v, double *__restrict__ yb,
                                                           double *__restrict__ lam, uint32_t *__restrict__ fits_total,
                                                           double *__restrict__ unset)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fits = i < S ? arima_boxcox_series(entries, offsets, sbase, B, i, csr_v, yb, lam, unset) : 0u;
    fits = __reduce_add_sync(0xffffffffu, fits);          // the grid covers whole warps
    if ((threadIdx.x & 31) == 0 && fits) atomicAdd(fits_total, fits);
}

// Prefix fits (pred[] in Box-Cox space), evaluation-synchronous, one warp per series: the fits t = n-1 .. 3 form a job
// list that the lanes work through dynamically (longest first, so the fits in flight have similar lengths).  Every round, all lanes that
// hold a job evaluate the objective and its forward-difference gradient TOGETHER -- the same Kalman-filter loop, each lane
// on its own prefix and parameters -- then each lane advances its own optimiser state (lbfgs_advance) to the next trial
// point; a lane whose fit has ended writes its forecast and takes the next job.  Per fit the arithmetic is the same as
// in arima_fit: only the scheduling differs.
// Cancel: lane 0 reads *cancel in every round (a volatile load from L2, so every round reads it anew) and the next round
// starts with it; once it is nonzero the warp leaves at once, dropping the fits in flight unfinished -- a cancelled job
// fails without reading pred[].  So the wait is bounded by one round (one evaluation of the longest prefix in flight),
// not by one fit (tens of rounds) or one series.  *fits_done gains the fits finished, one atomic per warp and round.
// Yield (resume != null): a cancel word of 2 ends the launch the same way; each warp then writes its series' resume point
// resume[2i], the longest prefix it has not finished (0 once all are done): every prefix above it has its forecast, and
// below it only those fitted while longer ones were in flight; resume[2i + 1] = the fits it dropped in flight, also added
// to resume[2S].  The kResume launch starts each series at its resume point and hands out only the prefixes whose pred[t]
// still holds kPredUnset, so the fits dropped in flight are fitted again from their start values and each fit finishes,
// and is counted, once.  The dropped fits are the unset prefixes above the point where the hand-out had got to, so they
// are the warp's first resume[2i + 1] hand-outs; resume[2S + 1] counts those that have finished again, which lets the host
// hold the next yield until all have (so no fit is dropped twice).  kMode: 0 a fit that cannot yield (resume is null),
// 1 one that can, 2 its resume launch; mode 0 is the fit kernel as it is without fit sharing.
// Stop: what lane 0 reads every round and whether it says leave -- CancelWord (one GPU: the job's cancel word) or StopBoard
// (several GPUs: the ranks' stop board, mode 0 only).
// arima_fit_series is the work of the warp that fits series i (lane = its lane): the one body of the fit kernels.
struct CancelWord {
    const volatile uint32_t *word;
    typedef uint32_t Read;
    __device__ __forceinline__ Read read() const { return *word; }
    __device__ __forceinline__ uint32_t stops(Read r) const { return r; }
};

// The stop board of a multi-GPU job: 8 u32 (one per rank, at most 8 ranks) in this rank's memory, word r written only by rank r, through its
// mapping, with the ordinal of a job rank r cancelled (0: none yet).  The warp leaves once any word equals this job's
// ordinal.  Unused words stay 0 (ordinals start at 1), so lane 0 reads all of them, one 32-byte sector in two 16-byte
// volatile loads, whatever the world size; the comparison waits for the next round, so the loads' latency overlaps the
// evaluation as the cancel word's does.
struct StopBoard {
    const uint32_t *board;
    uint32_t ordinal;
    struct Read {
        uint4 lo, hi;
    };
    __device__ __forceinline__ Read read() const
    {
        Read r;
        asm volatile("ld.volatile.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.lo.x), "=r"(r.lo.y), "=r"(r.lo.z), "=r"(r.lo.w)
                     : "l"(board));
        asm volatile("ld.volatile.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.hi.x), "=r"(r.hi.y), "=r"(r.hi.z), "=r"(r.hi.w)
                     : "l"(board + 4));
        return r;
    }
    __device__ __forceinline__ uint32_t stops(const Read &r) const
    {
        const uint32_t k = ordinal;
        return (r.lo.x == k) | (r.lo.y == k) | (r.lo.z == k) | (r.lo.w == k) | (r.hi.x == k) | (r.hi.y == k) |
               (r.hi.z == k) | (r.hi.w == k);
    }
};

template <int kMode, class Stop = CancelWord>
__device__ __forceinline__ void arima_fit_series(const SeriesEntry *__restrict__ entries, const uint32_t *__restrict__ offsets,
                                                 const uint32_t *__restrict__ sbase, uint32_t B, uint32_t S,
                                                 const double *__restrict__ yb, const double *__restrict__ lam,
                                                 double *__restrict__ pred, const Stop cancel,
                                                 uint32_t *__restrict__ fits_done, uint32_t *__restrict__ resume,
                                                 const uint32_t i, const uint32_t lane)
{
    if (i >= S) return;                                    // warp-uniform
    if (isnan(lam[i])) return;
    constexpr bool kResume = kMode == 2;
    int next;                                              // next job to hand out (warp-uniform), down to 3
    uint32_t redo = 0;                                     // kResume: hand-outs left that redo a dropped fit (warp-uniform)
    if (kResume) {
        next = (int)resume[2 * i];
        redo = resume[2 * i + 1];
        if (next < 3) return;                              // every prefix of the series has its forecast
    }
    const SeriesEntry e = load_entry(entries, offsets, sbase, B, i);
    const double *y = yb + e.off;
    double *p = pred + e.off;
    if (!kResume) {
        for (uint32_t t = lane; t < min(e.n, 3u); t += 32) p[t] = y[t];      // train = first three points (:241,255)
        next = (int)e.n - 1;
    }
    bool busy = false, redoing = false;
    ArimaObj o{y, 0};
    double u[3] = {0.0, 0.0, 0.0};
    Lbfgs st;
    // lane 0: the cancel word as read in the previous round; the first read is here, so that a warp which starts after
    // the cancel fits nothing
    typename Stop::Read stop = lane == 0 ? cancel.read() : typename Stop::Read{};
    for (;;) {
        if (__shfl_sync(0xffffffffu, cancel.stops(stop), 0)) break;      // cancelled: the fits in flight are dropped
        // ---- hand the next jobs to the idle lanes --------------------------------------------
        uint32_t idle = __ballot_sync(0xffffffffu, !busy);
        if (kResume) {
            // a prefix whose forecast is written is passed over; its idle lane takes the next one
            while (idle && next >= 3) {
                const int t = next - __popc(idle & ((1u << lane) - 1u));
                const bool take = !busy && t >= 3 && __double_as_longlong(p[t]) == (long long)kPredUnset;
                const uint32_t took = __ballot_sync(0xffffffffu, take);
                if (take) {
                    o.n = (uint32_t)t;
                    arima_start(o, u);
                    lbfgs_init(st);
                    busy = true;
                    redoing = __popc(took & ((1u << lane) - 1u)) < redo;      // longest first: in lane order
                }
                redo -= min(redo, (uint32_t)__popc(took));
                next -= __popc(idle);
                idle = __ballot_sync(0xffffffffu, !busy);
            }
        } else if (idle && next >= 3) {
            const int rank = __popc(idle & ((1u << lane) - 1u));
            if (!busy && next - rank >= 3) {
                o.n = (uint32_t)(next - rank);
                arima_start(o, u);
                lbfgs_init(st);
                busy = true;
            }
            next -= __popc(idle);
        }
        if (!__any_sync(0xffffffffu, busy)) break;
        // the next round's cancel word, read here so that its latency overlaps the evaluation
        if (lane == 0) stop = cancel.read();
        // ---- all busy lanes evaluate together -------------------------------------------------
        double f = 0.0, g[3] = {0.0, 0.0, 0.0};
        if (busy) arima_fg(o, u, f, g);
        __syncwarp();
        // ---- every lane advances its own optimiser --------------------------------------------
        bool ended = false;
        if (busy && lbfgs_advance(st, u, f, g)) {
            double phi, theta, s2, fc = 0.0;
            arima_transform(u, phi, theta, s2);
            arima_loglike(o, phi, theta, s2, &fc);
            p[o.n] = fc;
            busy = false;
            ended = true;
        }
        const uint32_t fin = __ballot_sync(0xffffffffu, ended);
        if (lane == 0 && fin) atomicAdd(fits_done, (uint32_t)__popc(fin));
        if (kResume) {
            const uint32_t again = __ballot_sync(0xffffffffu, ended && redoing);
            if (lane == 0 && again) atomicAdd(resume + 2 * S + 1, (uint32_t)__popc(again));
            if (ended) redoing = false;
        }
    }
    if (kMode != 0) {
        const int held = (int)__reduce_max_sync(0xffffffffu, busy ? o.n : 0u);    // the longest fit dropped in flight
        const uint32_t dropped = (uint32_t)__popc(__ballot_sync(0xffffffffu, busy));
        if (lane == 0) {
            resume[2 * i] = (uint32_t)max(max(next, held), 0);
            resume[2 * i + 1] = dropped;
            if (dropped) atomicAdd(resume + 2 * S, dropped);
        }
    }
}

template <int kMode>
__global__ void __launch_bounds__(128) arima_fit_sync_kernel(const SeriesEntry *__restrict__ entries, const uint32_t *__restrict__ offsets,
                                                             const uint32_t *__restrict__ sbase, uint32_t B, uint32_t S,
                                                             const double *__restrict__ yb, const double *__restrict__ lam,
                                                             double *__restrict__ pred, const volatile uint32_t *cancel,
                                                             uint32_t *__restrict__ fits_done, uint32_t *__restrict__ resume)
{
    arima_fit_series<kMode>(entries, offsets, sbase, B, S, yb, lam, pred, CancelWord{cancel}, fits_done, resume,
                            (blockIdx.x * blockDim.x + threadIdx.x) >> 5, threadIdx.x & 31);
}

// The fit kernel of a multi-GPU job (mode 0): it stops on the ranks' stop board instead of a cancel word.
__global__ void __launch_bounds__(128) arima_fit_board_kernel(const SeriesEntry *__restrict__ entries, const uint32_t *__restrict__ offsets,
                                                              const uint32_t *__restrict__ sbase, uint32_t B, uint32_t S,
                                                              const double *__restrict__ yb, const double *__restrict__ lam,
                                                              double *__restrict__ pred, StopBoard board,
                                                              uint32_t *__restrict__ fits_done)
{
    arima_fit_series<0>(entries, offsets, sbase, B, S, yb, lam, pred, board, fits_done, nullptr,
                        (blockIdx.x * blockDim.x + threadIdx.x) >> 5, threadIdx.x & 31);
}

// The lowest series of `a` a resume launch still has fits for (resume point >= 3), into *from (set to ~0 by the caller).
__global__ void __launch_bounds__(128) arima_unfinished_from_kernel(FitPart a, uint32_t *__restrict__ from)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool left = i < a.S && !isnan(a.lam[i]) && a.resume[2 * i] >= 3;
    const uint32_t lo = __reduce_min_sync(0xffffffffu, left ? i : ~0u);    // the grid covers whole warps
    if ((threadIdx.x & 31) == 0 && lo != ~0u) atomicMin(from, lo);
}

// Joint fit (fit sharing, TAD_FLAG_FIT_BESIDE): the fits of part b and the unfinished ones of a yielded fit, part a, in one
// launch, so that both share the SMs (a second launch beside a resume would not: the earlier grid's blocks are dispatched
// first and a block of a long series lives for minutes).  Part a runs as its resume launch (mode 2) over its series
// a_from ..< a_from + n_a, the series from its lowest unfinished one on; part b runs mode kModeB (1 its first launch, 2 its
// resume after a yield of its own).  The split: warps alternate between the two parts, a on the even warps and b on the odd,
// until the smaller part has all its series; the warps after that take the rest of the larger part.  So each part holds
// about half the warps while both have series left, and a yielded fit's finished series take no warp.  Each part reads
// its own cancel word and writes its own counters and resume points, so each leaves as a launch of its own would; the
// per-series work is arima_fit_series, so every forecast is the one its job computes alone.
template <int kModeB>
__global__ void __launch_bounds__(128) arima_fit_pair_kernel(FitPart a, uint32_t a_from, uint32_t n_a, FitPart b)
{
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t m = min(n_a, b.S);
    const bool on_b = w < 2 * m ? (w & 1) != 0 : b.S > n_a;
    const uint32_t at = w < 2 * m ? w >> 1 : w - m;
    if (kModeB == 2) {              // both parts resume: one call site
        arima_fit_series<2>(on_b ? b.entries : a.entries, on_b ? b.offsets : a.offsets, on_b ? b.sbase : a.sbase,
                            on_b ? b.B : a.B, on_b ? b.S : a.S, on_b ? b.y : a.y, on_b ? b.lam : a.lam, on_b ? b.pred : a.pred,
                            CancelWord{on_b ? b.cancel : a.cancel}, on_b ? b.fits_done : a.fits_done,
                            on_b ? b.resume : a.resume, on_b ? at : a_from + at, lane);
    } else if (on_b) {
        arima_fit_series<kModeB>(b.entries, b.offsets, b.sbase, b.B, b.S, b.y, b.lam, b.pred, CancelWord{b.cancel}, b.fits_done,
                                 b.resume, at, lane);
    } else {
        arima_fit_series<2>(a.entries, a.offsets, a.sbase, a.B, a.S, a.y, a.lam, a.pred, CancelWord{a.cancel}, a.fits_done,
                            a.resume, a_from + at, lane);
    }
}

// stddev_samp as in the other detectors (Welford, sequential in time order)
__device__ __forceinline__ double arima_stddev(const uint64_t *__restrict__ v, uint32_t n, bool &has_sd)
{
    double cnt = 0.0, avg = 0.0, m2 = 0.0;
    for (uint32_t i = 0; i < n; i++) {
        const double x = __ull2double_rn(v[i]);
        cnt = __dadd_rn(cnt, 1.0);
        const double d = __dsub_rn(x, avg);
        const double dn = __ddiv_rn(d, cnt);
        avg = __dadd_rn(avg, dn);
        m2 = __dadd_rn(m2, __dmul_rn(d, __dsub_rn(d, dn)));
    }
    has_sd = n >= 2;
    return has_sd ? __dsqrt_rn(__ddiv_rn(m2, __dsub_rn(cnt, 1.0))) : __longlong_as_double(0x7ff8000000000000LL);
}

template <int NT>
__global__ void __launch_bounds__(NT) detect_arima_kernel(const SeriesEntry *__restrict__ entries, const uint32_t *__restrict__ offsets,
                                                          const uint32_t *__restrict__ sbase, uint32_t B, uint32_t S,
                                                          const uint64_t *__restrict__ csr_v, const uint32_t *__restrict__ csr_t,
                                                          const double *__restrict__ pred, const double *__restrict__ lam,
                                                          OutCols out, uint32_t out_cap, uint32_t *__restrict__ stats, int emit_all)
{
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t total_s, base_s;
    const uint32_t i = blockIdx.x * NT + threadIdx.x;
    SeriesEntry e;
    e.n = 0;
    const uint64_t *v = nullptr;
    const double *p = nullptr;
    bool has_sd = false;
    double sd = 0.0, l = 0.0;
    uint32_t count = 0;
    if (i < S && !isnan(lam[i])) {                         // calc None -> the series contributes no rows
        e = load_entry(entries, offsets, sbase, B, i);
        l = lam[i];
        v = csr_v + e.off;
        p = pred + e.off;
        bool finite = true;
        for (uint32_t q = 0; q < e.n; q++) finite = finite && isfinite(inv_boxcox_d(p[q], l));
        if (!finite) e.n = 0;
        sd = arima_stddev(v, e.n, has_sd);
        if (emit_all) count = e.n;
        else if (has_sd)
            for (uint32_t q = 0; q < e.n; q++)
                count += fabs(__ull2double_rn(v[q]) - inv_boxcox_d(p[q], l)) > sd ? 1u : 0u;
    }
    // block exclusive scan of the counts
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = count;
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = lane < NT / 32 ? warp_sums[lane] : 0u;
        uint32_t winc = w;
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, winc, d);
            if (lane >= d) winc += o;
        }
        if (lane < NT / 32) warp_sums[lane] = winc - w;
        if (lane == NT / 32 - 1) total_s = winc;
    }
    __syncthreads();
    const uint32_t pre = warp_sums[warp] + inc - count;
    if (threadIdx.x == 0) base_s = total_s ? atomicAdd(&stats[ST_OUTCOUNT], total_s) : 0u;
    __syncthreads();
    if (count == 0) return;
    uint32_t idx = base_s + pre;
    const uint32_t *t = csr_t + e.off;
    for (uint32_t q = 0; q < e.n; q++) {
        const double x = __ull2double_rn(v[q]);
        const double calc = inv_boxcox_d(p[q], l);
        const bool flag = has_sd && fabs(x - calc) > sd;
        if (flag || emit_all) {
            if (idx < out_cap) {
                out.src_ip[idx] = (uint32_t)(e.a >> 32); out.dst_ip[idx] = (uint32_t)e.a;
                out.flow_start[idx] = (uint32_t)(e.b >> 32);
                out.src_port[idx] = (uint16_t)(e.b >> 16); out.dst_port[idx] = (uint16_t)e.b;
                out.proto[idx] = (uint8_t)e.proto; out.flow_end[idx] = t[q];
                out.stddev[idx] = sd; out.algo_calc[idx] = calc; out.throughput[idx] = x;
                out.anomaly[idx] = flag ? 1 : 0;
            }
            idx++;
        }
    }
}

// blocks of 128 threads for one warp per series
static uint32_t warp_blocks(uint64_t series) { return (uint32_t)((series * 32 + 127) / 128); }

cudaError_t launch_arima_boxcox(cudaStream_t st, const FitPart &p, const uint64_t *csr_v)
{
    if (p.S == 0) return cudaSuccess;
    arima_boxcox_kernel<<<(p.S + 127) / 128, 128, 0, st>>>(p.entries, p.offsets, p.sbase, p.B, p.S, csr_v, p.y, p.lam,
                                                           p.fits_total, p.resume ? p.pred : nullptr);
    return cudaGetLastError();
}

cudaError_t launch_arima_fit(cudaStream_t st, const FitPart &p, const uint64_t *csr_v, const uint32_t *board, uint32_t ordinal)
{
    const cudaError_t e = launch_arima_boxcox(st, p, csr_v);
    if (e != cudaSuccess || p.S == 0) return e;
    const uint32_t grid = warp_blocks(p.S);
    if (board)
        arima_fit_board_kernel<<<grid, 128, 0, st>>>(p.entries, p.offsets, p.sbase, p.B, p.S, p.y, p.lam, p.pred,
                                                     StopBoard{board, ordinal}, p.fits_done);
    else if (p.resume)
        arima_fit_sync_kernel<1><<<grid, 128, 0, st>>>(p.entries, p.offsets, p.sbase, p.B, p.S, p.y, p.lam, p.pred, p.cancel,
                                                       p.fits_done, p.resume);
    else
        arima_fit_sync_kernel<0><<<grid, 128, 0, st>>>(p.entries, p.offsets, p.sbase, p.B, p.S, p.y, p.lam, p.pred, p.cancel,
                                                       p.fits_done, nullptr);
    return cudaGetLastError();
}

cudaError_t launch_arima_resume(cudaStream_t st, const FitPart &p)
{
    if (p.S == 0) return cudaSuccess;
    arima_fit_sync_kernel<2><<<warp_blocks(p.S), 128, 0, st>>>(p.entries, p.offsets, p.sbase, p.B, p.S, p.y, p.lam, p.pred,
                                                               p.cancel, p.fits_done, p.resume);
    return cudaGetLastError();
}

cudaError_t launch_arima_unfinished(cudaStream_t st, const FitPart &a, uint32_t *from)
{
    cudaError_t e = cudaMemsetAsync(from, 0xff, 4, st);
    if (e != cudaSuccess || a.S == 0) return e;
    arima_unfinished_from_kernel<<<(a.S + 127) / 128, 128, 0, st>>>(a, from);
    return cudaGetLastError();
}

cudaError_t launch_arima_pair(cudaStream_t st, const FitPart &a, uint32_t a_from, uint32_t n_a, const FitPart &b, bool b_first)
{
    const uint64_t series = (uint64_t)n_a + b.S;
    if (series == 0) return cudaSuccess;
    if (b_first) arima_fit_pair_kernel<1><<<warp_blocks(series), 128, 0, st>>>(a, a_from, n_a, b);
    else arima_fit_pair_kernel<2><<<warp_blocks(series), 128, 0, st>>>(a, a_from, n_a, b);
    return cudaGetLastError();
}

cudaError_t launch_detect_arima(cudaStream_t st, const SeriesEntry *entries, const uint32_t *offsets, const uint32_t *sbase,
                                uint32_t B, uint32_t S, const uint64_t *csr_v, const uint32_t *csr_t, const double *scratch_pred,
                                const double *scratch_lam, const OutCols &out, uint32_t out_cap, uint32_t *stats, int emit_all)
{
    if (S == 0) return cudaSuccess;
    constexpr int NT = 128;
    detect_arima_kernel<NT><<<(S + NT - 1) / NT, NT, 0, st>>>(entries, offsets, sbase, B, S, csr_v, csr_t, scratch_pred,
                                                             scratch_lam, out, out_cap, stats, emit_all);
    return cudaGetLastError();
}

}  // namespace tad

// Host-side hook for the CPU tests of the numerical core (not part of the C ABI in theia_tad.h): runs the
// same start-value / L-BFGS / Kalman code the kernels run, on the host, for one history.
extern "C" int tad_debug_arima_fit(const double *y, uint32_t n, double *u_out, double *forecast, double *lambda_of_logx)
{
    if (lambda_of_logx) {        // y holds log(x): return the Box-Cox MLE lambda instead
        double sumlog = 0.0;
        for (uint32_t i = 0; i < n; i++) sumlog += y[i];
        *lambda_of_logx = tad::boxcox_mle_lambda(y, n, sumlog);
        return 0;
    }
    tad::ArimaObj o{y, n};
    double u[3];
    tad::arima_start(o, u);
    if (u_out) { u_out[3] = u[0]; u_out[4] = u[1]; u_out[5] = u[2]; }
    tad::arima_fit(o, u);
    double phi, theta, s2, fc = 0.0;
    tad::arima_transform(u, phi, theta, s2);
    const double ll = tad::arima_loglike(o, phi, theta, s2, &fc);
    if (u_out) { u_out[0] = u[0]; u_out[1] = u[1]; u_out[2] = u[2]; u_out[6] = -ll / n; }
    if (forecast) *forecast = fc;
    return 0;
}

namespace tad {

// The steps of the per-series reference (tad_debug_arima_series and tad_debug_arima_series_device), the same on the host and
// the device: the kernels' functions in the kernels' order.
// Transform: arima_log_series, the Box-Cox MLE lambda (or lambda_in if it is not NaN) and arima_boxcox_transform into y[];
// returns the lambda, or NaN if the series yields no rows; *tried = the lambda tried (NaN if none).
__host__ __device__ double arima_ref_transform(const uint64_t *v, uint32_t n, double lambda_in, double *y, double *tried)
{
    double sumlog;
    *tried = NAN;
    if (!arima_log_series(v, n, y, sumlog)) return NAN;
    const double l = isnan(lambda_in) ? boxcox_mle_lambda(y, n, sumlog) : lambda_in;
    *tried = l;
    return arima_boxcox_transform(y, n, l) ? l : NAN;
}

// every point one ulp up (nudge 1), down (-1), or in a random direction seeded by any other nonzero nudge
__host__ __device__ void arima_ref_nudge(double *y, uint32_t n, int nudge)
{
    uint64_t state = 0x9e3779b97f4a7c15ull * (uint64_t)(int64_t)nudge;
    for (uint32_t q = 0; q < n && nudge != 0; q++) {
        bool up = nudge == 1;
        if (nudge != 1 && nudge != -1) {
            state = state * 6364136223846793005ull + 1442695040888963407ull;
            up = (state >> 63) != 0;
        }
        y[q] = nextafter(y[q], up ? (double)INFINITY : -(double)INFINITY);
    }
}

// pred[t]: the train point for t < 3, else the forecast of the prefix fit on y[0 .. t) (start values, L-BFGS, forecast)
__host__ __device__ double arima_ref_prefix(const double *y, uint32_t t)
{
    if (t < 3) return y[t];
    const ArimaObj o{y, t};
    double u[3], phi, theta, s2, fc = 0.0;
    arima_start(o, u);
    arima_fit(o, u);
    arima_transform(u, phi, theta, s2);
    arima_loglike(o, phi, theta, s2, &fc);
    return fc;
}

// calc[] = the inverse transform of pred[]; false if any is not finite (the series yields no rows)
__host__ __device__ bool arima_ref_inverse(const double *p, uint32_t n, double l, double *calc)
{
    bool finite = true;
    for (uint32_t q = 0; q < n; q++) {
        calc[q] = inv_boxcox_d(p[q], l);
        finite = finite && isfinite(calc[q]);
    }
    return finite;
}

__global__ void __launch_bounds__(64) arima_ref_transform_kernel(const uint64_t *v, const uint32_t *off, const uint32_t *len,
                                                                 const double *lam_in, bool y_given, double *y, double *lam,
                                                                 uint32_t cases)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cases) return;
    double tried;
    lam[c] = y_given ? lam_in[c] : arima_ref_transform(v + off[c], len[c], lam_in[c], y + off[c], &tried);
}

__global__ void __launch_bounds__(64) arima_ref_prefix_kernel(const uint32_t *job_case, const uint32_t *job_t, uint32_t jobs,
                                                              const uint32_t *off, const double *lam, const double *y, double *p)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= jobs) return;
    const uint32_t c = job_case[j], t = job_t[j];
    if (!isnan(lam[c])) p[off[c] + t] = arima_ref_prefix(y + off[c], t);
}

__global__ void __launch_bounds__(64) arima_ref_inverse_kernel(const uint32_t *off, const uint32_t *len, const double *lam,
                                                               const double *p, double *calc, int32_t *ok, uint32_t cases)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < cases) ok[c] = !isnan(lam[c]) && arima_ref_inverse(p + off[c], len[c], lam[c], calc + off[c]);
}

}  // namespace tad

// Hooks of the per-prefix tests (not part of the C ABI in theia_tad.h): a series through the detector's whole path with the
// kernels' functions in the kernels' order, one prefix fit at a time (arima_fit, as a lane of the fit kernel runs it but
// without the warp's scheduling).  lambda_in: the lambda to transform with, or NaN for the Brent MLE.
// Host: nudge perturbs every transformed point by one ulp before the fits (arima_ref_nudge; 0 none) -- a fit whose forecast
// moves under such a nudge is path dependent, and the spread of the nudged runs measures by how much.  y_io (may be null)
// receives the transformed series before the nudge, or with y_given holds it on entry (then lambda_in is the lambda).
// Returns 1 if the series yields rows (calc[n] = the forecasts after the inverse transform; a null calc stops after the
// transform), else 0; *lambda_out = the lambda tried (NaN if there is none).
extern "C" int tad_debug_arima_series(const uint64_t *v, uint32_t n, double lambda_in, int nudge, double *calc,
                                      double *lambda_out, double *y_io, int y_given)
{
    std::vector<double> y(n), p(n);
    double l;
    if (y_given) {
        std::copy(y_io, y_io + n, y.begin());
        l = *lambda_out = lambda_in;
    } else {
        l = tad::arima_ref_transform(v, n, lambda_in, y.data(), lambda_out);
        if (y_io) std::copy(y.begin(), y.end(), y_io);
    }
    if (isnan(l)) return 0;
    if (!calc) return 1;                                   // the transform only
    tad::arima_ref_nudge(y.data(), n, nudge);
    for (uint32_t t = 0; t < n; t++) p[t] = tad::arima_ref_prefix(y.data(), t);
    return tad::arima_ref_inverse(p.data(), n, l, calc) ? 1 : 0;
}

// Device: `cases` series, series c on v[off[c] .. off[c] + len[c]) with lambda lam[c]; one thread per series for the transform
// and the inverse and one per prefix fit (longest first).  y_in (may be null): the transformed series, in v's layout, to fit
// instead (then lam[c] is the lambda).  calc and y_out (may be null) in v's layout; ok[c] = 1 if series c yields rows.
// Allocates and frees its own memory on the current device; returns once the results are copied back (0, or the CUDA error).
extern "C" int tad_debug_arima_series_device(const uint64_t *v, const uint32_t *off, const uint32_t *len, const double *lam,
                                             const double *y_in, uint32_t cases, double *calc, double *y_out, int32_t *ok)
{
    if (cases == 0) return 0;
    size_t words = 1;
    std::vector<std::pair<uint32_t, uint32_t>> jobs;                     // (t, case)
    for (uint32_t c = 0; c < cases; c++) {
        words = std::max(words, (size_t)off[c] + len[c]);
        for (uint32_t t = 0; t < len[c]; t++) jobs.emplace_back(t, c);
    }
    std::sort(jobs.begin(), jobs.end(), [](const auto &a, const auto &b) { return a.first > b.first; });
    std::vector<uint32_t> jc(jobs.size() + 1), jt(jobs.size() + 1);
    for (size_t j = 0; j < jobs.size(); j++) { jt[j] = jobs[j].first; jc[j] = jobs[j].second; }
    const uint32_t njobs = (uint32_t)jobs.size();
    uint64_t *dv = nullptr;
    uint32_t *doff = nullptr, *dlen = nullptr, *djc = nullptr, *djt = nullptr;
    double *dlam_in = nullptr, *dlam = nullptr, *dy = nullptr, *dp = nullptr, *dcalc = nullptr;
    int32_t *dok = nullptr;
    cudaError_t e = cudaMalloc(&dv, words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dy, words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dp, words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dcalc, words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&doff, cases * 4ull);
    if (e == cudaSuccess) e = cudaMalloc(&dlen, cases * 4ull);
    if (e == cudaSuccess) e = cudaMalloc(&dok, cases * 4ull);
    if (e == cudaSuccess) e = cudaMalloc(&dlam_in, cases * 8ull);
    if (e == cudaSuccess) e = cudaMalloc(&dlam, cases * 8ull);
    if (e == cudaSuccess) e = cudaMalloc(&djc, jc.size() * 4);
    if (e == cudaSuccess) e = cudaMalloc(&djt, jt.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpy(dv, v, words * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && y_in) e = cudaMemcpy(dy, y_in, words * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(doff, off, cases * 4ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dlen, len, cases * 4ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dlam_in, lam, cases * 8ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(djc, jc.data(), jc.size() * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(djt, jt.data(), jt.size() * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        const uint32_t cb = (cases + 63) / 64, jb = (njobs + 63) / 64;
        tad::arima_ref_transform_kernel<<<cb, 64>>>(dv, doff, dlen, dlam_in, y_in != nullptr, dy, dlam, cases);
        if (jb) tad::arima_ref_prefix_kernel<<<jb, 64>>>(djc, djt, njobs, doff, dlam, dy, dp);
        tad::arima_ref_inverse_kernel<<<cb, 64>>>(doff, dlen, dlam, dp, dcalc, dok, cases);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(calc, dcalc, words * 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && y_out) e = cudaMemcpy(y_out, dy, words * 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(ok, dok, cases * 4ull, cudaMemcpyDeviceToHost);
    for (void *q : {(void *)dv, (void *)dy, (void *)dp, (void *)dcalc, (void *)doff, (void *)dlen, (void *)dok, (void *)dlam_in,
                    (void *)dlam, (void *)djc, (void *)djt})
        cudaFree(q);
    return (int)e;
}

namespace tad {

// One case of tad_debug_arima_host / tad_debug_arima_device: the same core function on either side.  x: the case's n
// inputs (u64 values for op 0, doubles otherwise), par: 4 parameters, out: 8 results, tmp: n doubles of scratch.
//   op 0  x = values: out = {Box-Cox MLE lambda of log(x) as the kernel takes it, sum of the logs}
//   op 1  x = log values, par[0] = lambda: out[0] = boxcox_neg_llf
//   op 2  x = series, par = {phi, theta, s2}: out = {arima_loglike, forecast}
//   op 3  x = series, par = u: out[0..3] = arima_fg's f and g, out[4..7] = arima_objective at u, u + 1e-8 e_0, e_1, e_2
//   op 4  x = series: out[0..2] = arima_start
__host__ __device__ void arima_debug_case(int op, const void *x, uint32_t n, const double *par, double *out, double *tmp)
{
    const double *y = static_cast<const double *>(x);
    const ArimaObj o{y, n};
    for (int c = 0; c < 8; c++) out[c] = 0.0;
    if (op == 0) {
        double sumlog = 0.0;
        const uint64_t *v = static_cast<const uint64_t *>(x);
        for (uint32_t q = 0; q < n; q++) { tmp[q] = log(u64_to_double(v[q])); sumlog += tmp[q]; }
        out[0] = boxcox_mle_lambda(tmp, n, sumlog);
        out[1] = sumlog;
    } else if (op == 1) {
        double sumlog = 0.0;
        for (uint32_t q = 0; q < n; q++) sumlog += y[q];
        out[0] = boxcox_neg_llf(par[0], y, n, sumlog);
    } else if (op == 2) {
        out[0] = arima_loglike(o, par[0], par[1], par[2], &out[1]);
    } else if (op == 3) {
        double u[3] = {par[0], par[1], par[2]};
        arima_fg(o, u, out[0], out + 1);
        out[4] = arima_objective(o, u);
        for (int c = 0; c < 3; c++) {
            double uc[3] = {u[0], u[1], u[2]};
            uc[c] = u[c] + 1e-8;
            out[5 + c] = arima_objective(o, uc);
        }
    } else if (op == 4) {
        arima_start(o, out);
    }
}

__global__ void __launch_bounds__(64) arima_debug_kernel(int op, const uint8_t *x, const uint32_t *off, const uint32_t *len,
                                                         const double *par, double *out, double *tmp, uint32_t cases)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < cases) arima_debug_case(op, x + 8ull * off[c], len[c], par + 4ull * c, out + 8ull * c, tmp + off[c]);
}

}  // namespace tad

// Hooks for the precision tests of the numerical core (not part of the C ABI in theia_tad.h): `cases` cases of one op of
// tad::arima_debug_case, case c on the 8-byte words x[off[c] .. off[c] + len[c]) with par[4c ..] into out[8c ..].  The
// host hook runs them in turn; the device hook runs one thread per case on the current device, allocating and freeing its
// own memory, and returns once the results are copied back (0, or the CUDA error).
extern "C" int tad_debug_arima_host(int op, const void *x, const uint32_t *off, const uint32_t *len, const double *par,
                                    uint32_t cases, double *out)
{
    for (uint32_t c = 0; c < cases; c++) {
        std::vector<double> tmp(len[c] ? len[c] : 1);
        tad::arima_debug_case(op, static_cast<const uint64_t *>(x) + off[c], len[c], par + 4ull * c, out + 8ull * c, tmp.data());
    }
    return 0;
}

extern "C" int tad_debug_arima_device(int op, const void *x, const uint32_t *off, const uint32_t *len, const double *par,
                                      uint32_t cases, double *out)
{
    if (cases == 0) return 0;
    size_t words = 1;
    for (uint32_t c = 0; c < cases; c++) words = std::max(words, (size_t)off[c] + len[c]);
    uint8_t *dx = nullptr;
    uint32_t *doff = nullptr, *dlen = nullptr;
    double *dpar = nullptr, *dout = nullptr, *dtmp = nullptr;
    cudaError_t e = cudaMalloc(&dx, words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dtmp, words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&doff, cases * 4ull);
    if (e == cudaSuccess) e = cudaMalloc(&dlen, cases * 4ull);
    if (e == cudaSuccess) e = cudaMalloc(&dpar, cases * 32ull);
    if (e == cudaSuccess) e = cudaMalloc(&dout, cases * 64ull);
    if (e == cudaSuccess) e = cudaMemcpy(dx, x, words * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(doff, off, cases * 4ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dlen, len, cases * 4ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dpar, par, cases * 32ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        tad::arima_debug_kernel<<<(cases + 63) / 64, 64>>>(op, dx, doff, dlen, dpar, dout, dtmp, cases);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, cases * 64ull, cudaMemcpyDeviceToHost);
    for (void *p : {(void *)dx, (void *)dtmp, (void *)doff, (void *)dlen, (void *)dpar, (void *)dout}) cudaFree(p);
    return (int)e;
}
