// Generic fused log-density + reverse-mode gradient for a model given as ModelSpec IR (include/b200nuts.h: b200_ir;
// pymc_b200/ir.py).  One device function evaluates ANY model of the closed factor set, so a new model needs no new CUDA;
// it plugs into the same persistent NUTS / leapfrog / logp kernels as the hand-specialised models (same `eval` contract).
//
// It replaces one call of the compiled PyTensor function  q -> (logp, dlogp)  (pymc/model/core.py:232-267) and composes
// the joint density exactly the way the reference does:
//   1. constrain: x = backward(q) per value variable, + log|Jacobian|   (logprob/transforms.py:880-891, :1026-1073)
//   2. logp(x) = sum of factors (model/core.py:688-690), gx = d logp / d x accumulated factor by factor
//   3. chain rule through the transforms: g_q = gx * dx/dq + d log|J| / dq
// Determinism: no atomics.  A likelihood's gradient is PULLED: scalar targets by a team reduction over observations,
// indexed targets (group effects) through a CSR transpose of the index built at model-create time, so every sum has a
// fixed order and results are bit-identical from run to run and independent of how chains are sharded.
//
// Team scratch in global memory (L1/L2 resident), one slice per resident team: x[n] and the per-observation
// d loglik / d eta of the likelihood being processed.
//
// A random dispersion alpha (NegativeBinomial, Gamma) reaches its slot through the same team reduction as a likelihood's
// sigma.  Its normalising terms are not per observation: Gamma's once per evaluation, NegativeBinomial's over a table of
// the distinct nonzero counts (csrc/b200nuts.cu: prepare_ir), with digamma() of common.cuh for the gradient.
#pragma once
#include "common.cuh"

namespace b200 {

enum { IRT_NONE = 0, IRT_LOG = 1, IRT_INTERVAL = 2 };
enum { IRP_FLAT = 0, IRP_NORMAL, IRP_HALFNORMAL, IRP_CAUCHY, IRP_HALFCAUCHY, IRP_EXPONENTIAL, IRP_STUDENTT, IRP_UNIFORM,
       IRP_GAMMA, IRP_BETA, IRP_LOGNORMAL };
enum { IRL_NORMAL = 0, IRL_BERNOULLI_LOGIT, IRL_POISSON_LOG, IRL_STUDENTT, IRL_NORMAL_LOGVAR, IRL_BINOMIAL_LOGIT,
       IRL_NEGBINOMIAL_LOG, IRL_GAMMA_LOG };
enum { IRS_NONE = 0, IRS_CONST, IRS_REF, IRS_OBS };
constexpr double kNegBinPoissonAlpha = 1e10;  // above: NegativeBinomial -> Poisson(mu) limit (discrete.py:727-735)

struct IrParamD { int kind, ref; double value; };                     // kind 0: constant; 1: x[ref] (a scalar variable)
struct IrVarD { int offset, size, transform, pad; double lo, hi; };
struct IrPriorD { int dist, offset, size, pad; IrParamD p[3]; double c0; };      // c0: per-element constant of the density
struct IrFactorD { int offset, size; const int* idx; const int* rowptr; const int* rowobs; };  // CSR: element -> observations
// n_cols > 0: a design term, eta_i += sum_k X[i][k] x[f[0].offset + k], with coef = X row-major [N][n_cols] (the gradient
// reads it) and xt = X column-major [n_cols][N] (the forward pass reads it: consecutive threads take consecutive rows).
struct IrTermD { const double* coef; int n_factors, n_cols; IrFactorD f[3]; const double* xt; };
constexpr int kIrPartDoubles = 256;  // per-team slice partials of a design term's gradient, at the end of the team scratch

// sum_k X[i][k] b[k], k ascending
__device__ __forceinline__ double ir_design_row(const IrTermD& Tm, const double* b, int i, int N) {
    const double* xt = Tm.xt + i;
    double s = 0.0;
    for (int k = 0; k < Tm.n_cols; ++k) s = fma(xt[(long long)k * N], b[k], s);
    return s;
}

// g[k] += sum_i X[i][k] r[i] with the whole team, no atomics.  Columns go TS at a time; a block of kc < TS columns (the last
// one) splits the rows into S = TS / kc interleaved slices, thread t taking column t % kc and rows i = t / kc (mod S), so a
// warp reads adjacent rows of row-major X.  The slice partials meet in `part` and are added in slice order.  Every sum
// has a fixed order, so the result does not depend on the run or on the other teams.
template <int W>
__device__ __forceinline__ void ir_design_grad(const IrTermD& Tm, const double* r, int N, double* g, double* part, int tid) {
    constexpr int TS = 32 * W;
    const int K = Tm.n_cols;
    const double* X = Tm.coef;
    for (int c0 = 0; c0 < K; c0 += TS) {
        const int kc = min(K - c0, TS), S = TS / kc, c = tid % kc, s = tid / kc;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;  // four independent chains, combined in a fixed order
        if (s < S) {
            const double* xc = X + c0 + c;
            int i = s;
            for (; i + 3 * S < N; i += 4 * S) {
                a0 = fma(xc[(long long)i * K], r[i], a0);
                a1 = fma(xc[(long long)(i + S) * K], r[i + S], a1);
                a2 = fma(xc[(long long)(i + 2 * S) * K], r[i + 2 * S], a2);
                a3 = fma(xc[(long long)(i + 3 * S) * K], r[i + 3 * S], a3);
            }
            for (; i < N; i += S) a0 = fma(xc[(long long)i * K], r[i], a0);
        }
        const double a = (a0 + a1) + (a2 + a3);
        if (S == 1) {
            if (s == 0) g[c0 + c] += a;
        } else {  // uniform branch; only the last block can take it
            if (s < S) part[tid] = a;
            team_sync<W>();
            if (tid < kc) {
                double tot = part[c];
                for (int j = 1; j < S; ++j) tot += part[j * kc + c];
                g[c0 + c] += tot;
            }
        }
    }
}
// c0: sum of the constant parts over i.  Random dispersion (sigma_kind REF): Gamma keeps sum_i log y_i in sum_log_y;
// NegativeBinomial keeps the distinct nonzero y values u[k] with their counts cnt[k] (n_tab of them), over which the
// alpha-dependent normalising terms sum_i lgamma(y_i + a) - lgamma(a) and their digamma gradient are evaluated.
// yoff >= 0: a latent factor (a Normal / StudentT prior whose location is a linear predictor): y_i = x[yoff + i], the
// constrained values of a variable of size N, which also receives d logp / d y_i = -r_i; y is null.  -1: y is data.
struct IrLikD { int dist, n_terms, term0, sigma_kind; long long N; const double* y; const double* sigma_obs; IrParamD sigma;
                double nu, c0, sum_log_y; const double* tab_u; const double* tab_cnt; int n_tab, yoff; };
struct IrAr1D { int offset, size; IrParamD phi, sigma; double init_sigma; };

struct IrModel {
    struct Params {
        const IrVarD* vars; const IrPriorD* priors; const IrLikD* liks; const IrTermD* terms; const IrAr1D* ar1;
        int n_vars, n_priors, n_liks, n_ar1, n;
        double* scratch;            // [slots][stride]
        long long stride;           // doubles per team: n_pad + max N (+ kIrPartDoubles with a design term)
        int n_pad;
    };
    __host__ __device__ static size_t shared_bytes(const Params&) { return 0; }
    __device__ static void stage(const Params&, char*, uint64_t*) {}

    __device__ static __forceinline__ double par(const IrParamD& p, const double* x) { return p.kind ? x[p.ref] : p.value; }

    template <int NPL, int W, bool SMALL = false>
    __device__ __noinline__ static double eval(const Params& P, const char*, const double* q_s, double* g_s, int tid, double* red) {
        constexpr int TS = 32 * W;
        const int slot = (W == 1) ? (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) : (int)blockIdx.x;
        double* x = P.scratch + (long long)slot * P.stride;
        double* r = x + P.n_pad;
        const int n = P.n;
        double lp = 0.0;  // per-thread partial; reduced once at the end

        // ---- 1. constrain (+ log-Jacobians); gx accumulates in g_s -----------------------------------------------------
        for (int v = 0; v < P.n_vars; ++v) {
            const IrVarD V = P.vars[v];
            for (int j = tid; j < V.size; j += TS) {
                const int i = V.offset + j;
                const double z = q_s[i];
                double xv = z;
                if (V.transform == IRT_LOG) {
                    xv = exp(z);
                    lp += z;
                } else if (V.transform == IRT_INTERVAL) {
                    const double sg = sigmoid(z);
                    xv = V.lo + (V.hi - V.lo) * sg;
                    lp += log(V.hi - V.lo) - softplus(-z) - softplus(z);
                }
                x[i] = xv;
                g_s[i] = 0.0;
            }
        }
        team_sync<W>();

        // ---- 2a. priors ---------------------------------------------------------------------------------------------
        for (int k = 0; k < P.n_priors; ++k) {
            const IrPriorD F = P.priors[k];
            if (F.dist == IRP_FLAT) continue;
            const double a0 = par(F.p[0], x), a1 = par(F.p[1], x), a2 = par(F.p[2], x);
            double s[3] = {0.0, 0.0, 0.0};  // sums for the parameter gradients
            for (int j = tid; j < F.size; j += TS) {
                const int i = F.offset + j;
                const double xv = x[i];
                double gxi = 0.0;
                switch (F.dist) {
                    case IRP_NORMAL: {  // continuous.py:526-527
                        const double z = (xv - a0) / a1;
                        lp += -0.5 * z * z + F.c0 - log(a1);
                        gxi = -z / a1; s[0] += z / a1; s[1] += (z * z - 1.0) / a1;
                    } break;
                    case IRP_HALFNORMAL: {  // continuous.py:909-911
                        const double z = xv / a0;
                        lp += -0.5 * z * z + F.c0 - log(a0);
                        gxi = -z / a0; s[0] += (z * z - 1.0) / a0;
                    } break;
                    case IRP_CAUCHY: {  // continuous.py:2287-2288
                        const double u = xv - a0, den = a1 * a1 + u * u, t = u / a1;
                        lp += F.c0 - log(a1) - log1p(t * t);
                        gxi = -2.0 * u / den; s[0] += 2.0 * u / den; s[1] += (u * u - a1 * a1) / (a1 * den);
                    } break;
                    case IRP_HALFCAUCHY: {  // continuous.py:2383-2385
                        const double den = a0 * a0 + xv * xv, t = xv / a0;
                        lp += F.c0 - log(a0) - log1p(t * t);
                        gxi = -2.0 * xv / den; s[0] += (xv * xv - a0 * a0) / (a0 * den);
                    } break;
                    case IRP_EXPONENTIAL:  // continuous.py:1478-1480 (mu = 1 / lam)
                        lp += log(a0) - a0 * xv;
                        gxi = -a0; s[0] += 1.0 / a0 - xv;
                        break;
                    case IRP_STUDENTT: {  // continuous.py:1936-1944; a0 = nu (constant), a1 = mu, a2 = sigma
                        const double z = (xv - a1) / a2;
                        lp += F.c0 - log(a2) - 0.5 * (a0 + 1.0) * log1p(z * z / a0);
                        const double w = (a0 + 1.0) * z / (a2 * (a0 + z * z));
                        gxi = -w; s[1] += w; s[2] += -1.0 / a2 + w * z;
                    } break;
                    case IRP_UNIFORM: lp += F.c0; break;  // continuous.py:309-314
                    case IRP_GAMMA:  // continuous.py:2512-2515
                        lp += F.c0 + (a0 - 1.0) * log(xv) - a1 * xv;
                        gxi = (a0 - 1.0) / xv - a1;
                        break;
                    case IRP_BETA:  // continuous.py:1250-1256
                        lp += F.c0 + (a0 - 1.0) * log(xv) + (a1 - 1.0) * log1p(-xv);
                        gxi = (a0 - 1.0) / xv - (a1 - 1.0) / (1.0 - xv);
                        break;
                    case IRP_LOGNORMAL: {  // continuous.py:1807-1814
                        const double lx = log(xv), z = (lx - a0) / a1;
                        lp += -0.5 * z * z - lx + F.c0 - log(a1);
                        gxi = (-z / a1 - 1.0) / xv; s[0] += z / a1; s[1] += (z * z - 1.0) / a1;
                    } break;
                    default: break;
                }
                g_s[i] += gxi;
            }
            const bool any_ref = F.p[0].kind | F.p[1].kind | F.p[2].kind;
            if (any_ref) {  // uniform branch: the descriptor is the same for every thread
                team_sync<W>();
                team_sum_n<W>(s, tid, red);
                if (tid == 0) {
#pragma unroll
                    for (int a = 0; a < 3; ++a)
                        if (F.p[a].kind) g_s[F.p[a].ref] += s[a];
                }
            }
            team_sync<W>();
        }

        // ---- 2b. likelihoods: eta_i = sum_t coef_t[i] prod_f x_f[idx_f[i]] ----------------------------------------------
        for (int l = 0; l < P.n_liks; ++l) {
            const IrLikD L = P.liks[l];
            const int N = (int)L.N;
            const double sg_s = (L.sigma_kind == IRS_REF) ? x[L.sigma.ref] : L.sigma.value;
            const bool disp = L.dist == IRL_NEGBINOMIAL_LOG || L.dist == IRL_GAMMA_LOG;  // sg_s is the dispersion alpha
            const double la = disp ? log(sg_s) : 0.0;
            double s_sig = 0.0;
            for (int i = tid; i < N; i += TS) {
                double eta = 0.0;
                for (int t = 0; t < L.n_terms; ++t) {
                    const IrTermD& Tm = P.terms[L.term0 + t];
                    if (Tm.n_cols) {
                        eta += ir_design_row(Tm, x + Tm.f[0].offset, i, N);
                        continue;
                    }
                    double pr = Tm.coef ? Tm.coef[i] : 1.0;
                    for (int f = 0; f < Tm.n_factors; ++f) {
                        const IrFactorD& Fc = Tm.f[f];
                        pr *= x[Fc.offset + (Fc.idx ? Fc.idx[i] : (Fc.size == 1 ? 0 : i))];
                    }
                    eta += pr;
                }
                const double yi = L.yoff >= 0 ? x[L.yoff + i] : L.y[i];
                double ri = 0.0;
                switch (L.dist) {
                    case IRL_NORMAL: {  // continuous.py:526-527
                        const double sg = (L.sigma_kind == IRS_OBS) ? L.sigma_obs[i] : sg_s;
                        const double z = (yi - eta) / sg;
                        lp += -0.5 * z * z - log(sg);
                        ri = z / sg; s_sig += (z * z - 1.0) / sg;
                    } break;
                    case IRL_BERNOULLI_LOGIT:  // discrete.py:362-367 in PyTensor's stabilised forms
                        lp += yi * eta - softplus(eta);
                        ri = yi - sigmoid(eta);
                        break;
                    case IRL_POISSON_LOG: {  // discrete.py:581-586
                        const double mu = exp(eta);
                        lp += yi * eta - mu;
                        ri = yi - mu;
                    } break;
                    case IRL_STUDENTT: {  // continuous.py:1936-1944
                        const double sg = (L.sigma_kind == IRS_OBS) ? L.sigma_obs[i] : sg_s;
                        const double z = (yi - eta) / sg;
                        lp += -log(sg) - 0.5 * (L.nu + 1.0) * log1p(z * z / L.nu);
                        ri = (L.nu + 1.0) * z / (sg * (L.nu + z * z)); s_sig += -1.0 / sg + ri * z;
                    } break;
                    case IRL_NORMAL_LOGVAR: {  // Normal(0, exp(eta / 2))
                        const double w = yi * yi * exp(-eta);
                        lp += -0.5 * w - 0.5 * eta;
                        ri = 0.5 * w - 0.5;
                    } break;
                    case IRL_BINOMIAL_LOGIT: {  // discrete.py:141-152 in PyTensor's stabilised forms; binomln(n, y) is in c0
                        const double nt = (L.sigma_kind == IRS_OBS) ? L.sigma_obs[i] : sg_s;
                        lp += yi * eta - nt * softplus(eta);
                        ri = yi - nt * sigmoid(eta);
                    } break;
                    case IRL_NEGBINOMIAL_LOG:  // discrete.py:700-745, n = a, p = a / (mu + a); the lgamma part is in c0 / below
                        if (sg_s > kNegBinPoissonAlpha) {  // uniform branch: the Poisson(mu) limit
                            const double mu = exp(eta);
                            lp += yi * eta - mu;
                            ri = yi - mu;
                        } else {
                            // d = eta - log a: lse = logaddexp(eta, log a) = log a + softplus(d) = eta + softplus(-d), with
                            // s = mu / (mu + a) and sc = a / (mu + a) from one exp, so nothing overflows for any finite eta
                            const double d = eta - la, e = exp(-fabs(d)), l1 = log1p(e), h = 1.0 / (1.0 + e);
                            const double s = d >= 0 ? h : e * h, sc = d >= 0 ? e * h : h;
                            const double sp = fmax(d, 0.0) + l1;  // lse - log a
                            lp -= yi * (fmax(-d, 0.0) + l1) + sg_s * sp;
                            ri = yi * sc - sg_s * s;                         // a (y - mu) / (mu + a)
                            s_sig += 1.0 - sp - sc * (1.0 + yi / sg_s);      // d/da except psi(y + a) - psi(a)
                        }
                        break;
                    case IRL_GAMMA_LOG: {  // continuous.py:2512-2521, beta = a exp(-eta); the eta-free part once below
                        const double w = yi * exp(-eta);
                        lp -= sg_s * (eta + w);
                        ri = sg_s * (w - 1.0);
                        s_sig -= eta + w;
                    } break;
                    default: break;
                }
                r[i] = ri;
                if (L.yoff >= 0) g_s[L.yoff + i] -= ri;  // this thread owns element i of the latent variable
            }
            if (disp && L.sigma_kind == IRS_REF) {  // uniform branch: the alpha-dependent normalising terms
                const double a = sg_s;
                const IrLikD& Lt = P.liks[l];  // read here, not kept live through the observation loop
                if (L.dist == IRL_GAMMA_LOG) {
                    if (tid == 0) {
                        const double sly = Lt.sum_log_y;
                        lp += (double)N * (a * la - lgamma(a)) + (a - 1.0) * sly;
                        s_sig += (double)N * (la + 1.0 - digamma(a)) + sly;
                    }
                } else if (a <= kNegBinPoissonAlpha) {
                    // sum_i lgamma(y_i + a) - lgamma(a) over the distinct values: team-strided, fixed order
                    const double lga = lgamma(a), pa = digamma(a);
                    const double* tu = Lt.tab_u;
                    const double* tc = Lt.tab_cnt;
                    const int n_tab = Lt.n_tab;
                    for (int k = tid; k < n_tab; k += TS) {
                        const double u = tu[k], c = tc[k];
                        lp = fma(c, lgamma(u + a) - lga, lp);
                        s_sig = fma(c, digamma(u + a) - pa, s_sig);
                    }
                }
            }
            if (tid == 0) lp += L.c0;
            team_sync<W>();
            if (L.sigma_kind == IRS_REF) {
                const double tot = team_sum<W>(s_sig, tid, red);
                if (tid == 0) g_s[L.sigma.ref] += tot;
                team_sync<W>();
            }
            // gradient of every (term, factor): d eta_i / d x_f = coef * (other factors)
            for (int t = 0; t < L.n_terms; ++t) {
                const IrTermD& Tm = P.terms[L.term0 + t];
                if (Tm.n_cols) {  // uniform branch: the residuals r are complete after the barrier above
                    ir_design_grad<W>(Tm, r, N, g_s + Tm.f[0].offset, x + P.stride - kIrPartDoubles, tid);
                    team_sync<W>();
                    continue;
                }
                for (int f = 0; f < Tm.n_factors; ++f) {
                    const IrFactorD& Fc = Tm.f[f];
                    auto others = [&](int i) -> double {
                        double pr = Tm.coef ? Tm.coef[i] : 1.0;
                        for (int f2 = 0; f2 < Tm.n_factors; ++f2) {
                            if (f2 == f) continue;
                            const IrFactorD& F2 = Tm.f[f2];
                            pr *= x[F2.offset + (F2.idx ? F2.idx[i] : (F2.size == 1 ? 0 : i))];
                        }
                        return pr;
                    };
                    if (!Fc.idx && Fc.size == 1) {  // scalar target: team reduction over the observations
                        double a = 0.0;
                        for (int i = tid; i < N; i += TS) a = fma(r[i], others(i), a);
                        a = team_sum<W>(a, tid, red);
                        if (tid == 0) g_s[Fc.offset] += a;
                    } else if (!Fc.idx) {  // elementwise target (vector variable of the likelihood's length)
                        for (int i = tid; i < N; i += TS) g_s[Fc.offset + i] += r[i] * others(i);
                    } else {  // indexed target: pull through the CSR transpose of idx (fixed order)
                        for (int j = tid; j < Fc.size; j += TS) {
                            double a = 0.0;
                            for (int e = Fc.rowptr[j]; e < Fc.rowptr[j + 1]; ++e) {
                                const int i = Fc.rowobs[e];
                                a = fma(r[i], others(i), a);
                            }
                            g_s[Fc.offset + j] += a;
                        }
                    }
                    team_sync<W>();
                }
            }
        }

        // ---- 2c. AR(1): h_0 ~ Normal(0, init_sigma), h_t - phi h_{t-1} ~ Normal(0, sigma)  (timeseries.py:646-676) ------
        for (int k = 0; k < P.n_ar1; ++k) {
            const IrAr1D A = P.ar1[k];
            const double phi = par(A.phi, x), sg = par(A.sigma, x);
            const double i2 = 1.0 / (sg * sg);
            const double* h = x + A.offset;
            double s[2] = {0.0, 0.0};  // sum e h_{t-1}, sum e^2
            for (int t = tid; t < A.size; t += TS) {
                const double ht = h[t];
                double g = 0.0;
                if (t >= 1) {
                    const double hm = h[t - 1], e = ht - phi * hm;
                    g -= e * i2;
                    s[0] = fma(e, hm, s[0]);
                    s[1] = fma(e, e, s[1]);
                } else {
                    const double zi = ht / A.init_sigma;
                    g -= zi / A.init_sigma;
                    lp += -0.5 * zi * zi - B200_HALF_LOG_2PI - log(A.init_sigma);
                }
                if (t + 1 < A.size) g = fma(phi * i2, h[t + 1] - phi * ht, g);
                g_s[A.offset + t] += g;
            }
            team_sync<W>();
            team_sum_n<W>(s, tid, red);
            if (tid == 0) {
                lp += -0.5 * s[1] * i2 - (A.size - 1) * (B200_HALF_LOG_2PI + log(sg));
                if (A.phi.kind) g_s[A.phi.ref] += s[0] * i2;
                if (A.sigma.kind) g_s[A.sigma.ref] += (s[1] * i2 - (double)(A.size - 1)) / sg;
            }
            team_sync<W>();
        }

        // ---- 3. chain rule through the transforms -------------------------------------------------------------------------
        for (int v = 0; v < P.n_vars; ++v) {
            const IrVarD V = P.vars[v];
            if (V.transform == IRT_NONE) continue;
            for (int j = tid; j < V.size; j += TS) {
                const int i = V.offset + j;
                const double xv = x[i];
                if (V.transform == IRT_LOG) {
                    g_s[i] = fma(g_s[i], xv, 1.0);
                } else {
                    // dx/dz = (hi - lo) s (1 - s), s = sigmoid(z), in the form e / (1 + e)^2 with e = exp(-|z|): s recovered
                    // from x, or 1 - s, cancels at large |z| (relative error 1e-3 at |z| = 30)
                    const double sg = (xv - V.lo) / (V.hi - V.lo);
                    const double e = exp(-fabs(q_s[i]));
                    g_s[i] = fma(g_s[i], (V.hi - V.lo) * (e / ((1.0 + e) * (1.0 + e))), 1.0 - 2.0 * sg);
                }
            }
        }
        for (int i = n + tid; i < TS * NPL; i += TS) g_s[i] = 0.0;  // padding of the state vectors
        team_sync<W>();
        return team_sum<W>(lp, tid, red);
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// Pointwise log-likelihood of one likelihood factor for a batch of (unconstrained) draws: out[d][i] = log p(y_i | draw d).
// What pm.compute_log_likelihood evaluates per draw through a compiled function (pymc/stats/log_density.py:31-77,
// :129-195) -- the `log_likelihood` group LOO / WAIC need.  One warp per draw; the constrained values go through the
// team scratch slice like in eval().  Elementwise constants (log 2pi, lgamma) are included, unlike in eval() where they are
// folded into one constant per factor.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ir_pointwise_kernel(const IrModel::Params P, int lik, long long D,
                                                           const double* __restrict__ draws /*[D][n]*/,
                                                           double* __restrict__ out /*[D][N]*/) {
    const int lane = threadIdx.x & 31;
    const int slot = (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5));
    double* x = P.scratch + (long long)slot * P.stride;
    const IrLikD L = P.liks[lik];
    const int N = (int)L.N, n = P.n;
    const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long d = slot; d < D; d += stride) {
        const double* q = draws + d * n;
        for (int v = 0; v < P.n_vars; ++v) {
            const IrVarD V = P.vars[v];
            for (int j = lane; j < V.size; j += 32) {
                const double z = q[V.offset + j];
                x[V.offset + j] = V.transform == IRT_LOG ? exp(z) : (V.transform == IRT_INTERVAL ? V.lo + (V.hi - V.lo) * sigmoid(z) : z);
            }
        }
        __syncwarp();
        const double sg_s = (L.sigma_kind == IRS_REF) ? x[L.sigma.ref] : L.sigma.value;
        const double la = (L.dist == IRL_NEGBINOMIAL_LOG || L.dist == IRL_GAMMA_LOG) ? log(sg_s) : 0.0;
        for (int i = lane; i < N; i += 32) {
            double eta = 0.0;
            for (int t = 0; t < L.n_terms; ++t) {
                const IrTermD& Tm = P.terms[L.term0 + t];
                if (Tm.n_cols) {
                    eta += ir_design_row(Tm, x + Tm.f[0].offset, i, N);
                    continue;
                }
                double pr = Tm.coef ? Tm.coef[i] : 1.0;
                for (int f = 0; f < Tm.n_factors; ++f) {
                    const IrFactorD& Fc = Tm.f[f];
                    pr *= x[Fc.offset + (Fc.idx ? Fc.idx[i] : (Fc.size == 1 ? 0 : i))];
                }
                eta += pr;
            }
            const double yi = L.y[i];
            double lp = 0.0;
            switch (L.dist) {
                case IRL_NORMAL: {
                    const double sg = (L.sigma_kind == IRS_OBS) ? L.sigma_obs[i] : sg_s, z = (yi - eta) / sg;
                    lp = -0.5 * z * z - log(sg) - B200_HALF_LOG_2PI;
                } break;
                case IRL_BERNOULLI_LOGIT: lp = yi * eta - softplus(eta); break;
                case IRL_POISSON_LOG: lp = yi * eta - exp(eta) - lgamma(yi + 1.0); break;
                case IRL_STUDENTT: {
                    const double sg = (L.sigma_kind == IRS_OBS) ? L.sigma_obs[i] : sg_s, z = (yi - eta) / sg;
                    lp = lgamma(0.5 * (L.nu + 1.0)) - lgamma(0.5 * L.nu) - 0.5 * log(L.nu * 3.14159265358979323846) - log(sg) -
                         0.5 * (L.nu + 1.0) * log1p(z * z / L.nu);
                } break;
                case IRL_NORMAL_LOGVAR: lp = -0.5 * yi * yi * exp(-eta) - 0.5 * eta - B200_HALF_LOG_2PI; break;
                case IRL_BINOMIAL_LOGIT: {
                    const double nt = (L.sigma_kind == IRS_OBS) ? L.sigma_obs[i] : sg_s;
                    lp = lgamma(nt + 1.0) - lgamma(yi + 1.0) - lgamma(nt - yi + 1.0) + yi * eta - nt * softplus(eta);
                } break;
                case IRL_NEGBINOMIAL_LOG:
                    if (sg_s > kNegBinPoissonAlpha) {
                        lp = yi * eta - exp(eta) - lgamma(yi + 1.0);
                    } else {
                        const double d = eta - la, l1 = log1p(exp(-fabs(d)));
                        lp = lgamma(yi + sg_s) - lgamma(sg_s) - lgamma(yi + 1.0) - yi * (fmax(-d, 0.0) + l1) - sg_s * (fmax(d, 0.0) + l1);
                    }
                    break;
                case IRL_GAMMA_LOG: lp = sg_s * (la - eta) - lgamma(sg_s) + (sg_s - 1.0) * log(yi) - sg_s * yi * exp(-eta); break;
                default: break;
            }
            out[d * N + i] = lp;
        }
        __syncwarp();
    }
}

}  // namespace b200
