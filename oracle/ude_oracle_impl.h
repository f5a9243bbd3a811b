/*
 * ude_oracle_impl.h -- precision-generic body of the oracle (included twice by
 * ude_oracle.c with REAL=double/SUF=_f64 and REAL=float/SUF=_f32).
 * TEST INFRASTRUCTURE ONLY -- see ude_oracle.h for scope and citations.
 */
#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)
#define FN(name) CAT(name, SUF)

/* ---------------------------------------------------------------- chain ---- */
/* Dense layer l: h <- act(W h + b), W is out x in stored column-major followed
 * by b -- the layout Lux ComponentVector (scenario_1.jl:113), DiffEqFlux
 * initial_params (seir_exposure.jl:115) and Flux.destructure
 * (Fisher-KPP-CNN.jl:106) produce. */
static inline REAL FN(act_fwd)(int act, REAL a)
{
    switch (act) {
    case UDE_ACT_TANH: return R_TANH(a);
    case UDE_ACT_RBF: return R_EXP(-(a * a));      /* rbf(x) = exp(-x^2), scenario_1.jl:59 */
    default: return a;
    }
}
/* derivative of the activation given pre-activation a and output h */
static inline REAL FN(act_der)(int act, REAL a, REAL h)
{
    switch (act) {
    case UDE_ACT_TANH: return (REAL)1 - h * h;
    case UDE_ACT_RBF: return (REAL)-2 * a * h;
    default: return (REAL)1;
    }
}

/* forward keeping every layer's pre-activation (pre) and output (hs); hs[0] = input */
static void FN(chain_forward_store)(const ude_model *m, const REAL *th, const REAL *x,
                                    REAL hs[][UDE_MAX_WIDTH], REAL pre[][UDE_MAX_WIDTH])
{
    for (int i = 0; i < m->widths[0]; ++i) hs[0][i] = x[i];
    const REAL *p = th;
    for (int l = 0; l < m->n_layers; ++l) {
        const int nin = m->widths[l], nout = m->widths[l + 1];
        const REAL *W = p, *b = p + (size_t)nin * nout;
        for (int j = 0; j < nout; ++j) {
            REAL a = b[j];
            for (int i = 0; i < nin; ++i) a += W[(size_t)i * nout + j] * hs[l][i];
            pre[l][j] = a;
            hs[l + 1][j] = FN(act_fwd)(m->acts[l], a);
        }
        p += (size_t)nin * nout + nout;
    }
}

void FN(ude_mlp_forward)(const ude_model *m, const REAL *th, const REAL *x, REAL *y)
{
    REAL hs[UDE_MAX_LAYERS + 1][UDE_MAX_WIDTH], pre[UDE_MAX_LAYERS][UDE_MAX_WIDTH];
    FN(chain_forward_store)(m, th, x, hs, pre);
    for (int j = 0; j < m->widths[m->n_layers]; ++j) y[j] = hs[m->n_layers][j];
}

/* reverse sweep: given dy (cotangent of the chain output) return dx and add w * dtheta */
static void FN(chain_vjp)(const ude_model *m, const REAL *th, REAL hs[][UDE_MAX_WIDTH],
                          REAL pre[][UDE_MAX_WIDTH], const REAL *dy, REAL *dx, REAL *gth, REAL w)
{
    size_t off[UDE_MAX_LAYERS];
    size_t o = 0;
    for (int l = 0; l < m->n_layers; ++l) {
        off[l] = o;
        o += (size_t)m->widths[l] * m->widths[l + 1] + m->widths[l + 1];
    }
    REAL g[UDE_MAX_WIDTH], gin[UDE_MAX_WIDTH];
    for (int j = 0; j < m->widths[m->n_layers]; ++j) g[j] = dy[j];
    for (int l = m->n_layers - 1; l >= 0; --l) {
        const int nin = m->widths[l], nout = m->widths[l + 1];
        const REAL *W = th + off[l];
        REAL *gW = gth ? gth + off[l] : NULL;
        REAL *gb = gth ? gW + (size_t)nin * nout : NULL;
        for (int j = 0; j < nout; ++j) g[j] *= FN(act_der)(m->acts[l], pre[l][j], hs[l + 1][j]);
        for (int i = 0; i < nin; ++i) {
            REAL s = 0;
            for (int j = 0; j < nout; ++j) {
                s += W[(size_t)i * nout + j] * g[j];
                if (gW) gW[(size_t)i * nout + j] += w * g[j] * hs[l][i];
            }
            gin[i] = s;
        }
        if (gb) for (int j = 0; j < nout; ++j) gb[j] += w * g[j];
        for (int i = 0; i < nin; ++i) g[i] = gin[i];
    }
    for (int i = 0; i < m->widths[0]; ++i) dx[i] = g[i];
}

static size_t FN(chain_len)(const ude_model *m)
{
    size_t o = 0;
    for (int l = 0; l < m->n_layers; ++l)
        o += (size_t)m->widths[l] * m->widths[l + 1] + m->widths[l + 1];
    return o;
}

/* ------------------------------------------------------------------ RHS ---- */
void FN(ude_rhs)(const ude_model *m, const REAL *th, const REAL *u, REAL *du)
{
    const REAL *thc = th + m->n_prefix;
    REAL hs[UDE_MAX_LAYERS + 1][UDE_MAX_WIDTH], pre[UDE_MAX_LAYERS][UDE_MAX_WIDTH];
    const int L = m->n_layers;
    switch (m->model) {
    case UDE_MODEL_LV: {
        /* du1 = a1*u1 + NN1(u); du2 = -a2*u2 + NN2(u)   (scenario_1.jl:69-73)
         * a1,a2 fixed (p_[1], p_[4]) | a2 = theta[0] (scenario_2.jl:90-95)
         * | a1,a2 = theta[0:2] (hudson_bay.jl:85-91) */
        REAL a1 = (REAL)m->consts[0], a2 = (REAL)m->consts[1];
        if (m->n_prefix == 1) a2 = th[0];
        if (m->n_prefix == 2) { a1 = th[0]; a2 = th[1]; }
        FN(chain_forward_store)(m, thc, u, hs, pre);
        du[0] = a1 * u[0] + hs[L][0];
        du[1] = -a2 * u[1] + hs[L][1];
        break;
    }
    case UDE_MODEL_SEIR: {
        /* seir_exposure.jl:117-130; consts = F, b0, alpha, kappa, mu, sigma, gamma, d, lambda (:33) */
        const REAL F = (REAL)m->consts[0], b0 = (REAL)m->consts[1], mu = (REAL)m->consts[4],
                   sg = (REAL)m->consts[5], gm = (REAL)m->consts[6], dd = (REAL)m->consts[7],
                   lm = (REAL)m->consts[8];
        const REAL S = u[0], E = u[1], I = u[2], R = u[3], N = u[4], D = u[5];
        REAL x[3] = { S / N, I, D / N };
        FN(chain_forward_store)(m, thc, x, hs, pre);
        const REAL z = hs[L][0];
        du[0] = -b0 * S * F / N - z - mu * S;
        du[1] = b0 * S * F / N + z - (sg + mu) * E;
        du[2] = sg * E - (gm + mu) * I;
        du[3] = gm * I - mu * R;
        du[4] = -mu * N;
        du[5] = dd * gm * I - lm * D;
        du[6] = sg * E;
        break;
    }
    case UDE_MODEL_FKPP: {
        /* Fisher-KPP-CNN.jl:111-126: pointwise reaction net + D0 * 3-tap periodic stencil;
         * theta suffix = [w1, w2, w3, conv bias (unused), D0] (:106-109) */
        const REAL *sx = thc + FN(chain_len)(m);
        const REAL w1 = sx[0], w2 = sx[1], w3 = sx[2], D0 = sx[4];
        const int n = m->d;
        for (int i = 0; i < n; ++i) {
            const REAL um = u[(i + n - 1) % n], up = u[(i + 1) % n];
            FN(chain_forward_store)(m, thc, &u[i], hs, pre);
            du[i] = hs[L][0] + D0 * (w1 * um + w2 * u[i] + w3 * up);
        }
        break;
    }
    case UDE_MODEL_SEIR_NODE: {
        /* seir_exposure.jl:55-64: dS,dE,dI,dR,dD = first five outputs of ann_node([S/N,E,I,R,N,D/N,C]); dN = -mu N; dC = sigma E */
        const REAL mu = (REAL)m->consts[4], sg = (REAL)m->consts[5];
        const REAL N = u[4];
        REAL x[7] = { u[0] / N, u[1], u[2], u[3], N, u[5] / N, u[6] };
        FN(chain_forward_store)(m, thc, x, hs, pre);
        du[0] = hs[L][0]; du[1] = hs[L][1]; du[2] = hs[L][2]; du[3] = hs[L][3];
        du[4] = -mu * N;
        du[5] = hs[L][4];
        du[6] = sg * u[1];
        break;
    }
    default: /* UDE_MODEL_NODE: du = NN(u) */
        FN(chain_forward_store)(m, thc, u, hs, pre);
        for (int k = 0; k < m->d; ++k) du[k] = hs[L][k];
    }
}

/* dlam = J_u^T lam; gth += w * J_theta^T lam  (what ReverseDiffVJP provides,
 * seir_exposure.jl:71) */
void FN(ude_rhs_vjp)(const ude_model *m, const REAL *th, const REAL *u, const REAL *lam,
                     REAL *dlam, REAL *gth, REAL w)
{
    const REAL *thc = th + m->n_prefix;
    REAL *gthc = gth ? gth + m->n_prefix : NULL;
    REAL hs[UDE_MAX_LAYERS + 1][UDE_MAX_WIDTH], pre[UDE_MAX_LAYERS][UDE_MAX_WIDTH];
    REAL dx[UDE_MAX_WIDTH];
    switch (m->model) {
    case UDE_MODEL_LV: {
        REAL a1 = (REAL)m->consts[0], a2 = (REAL)m->consts[1];
        if (m->n_prefix == 1) a2 = th[0];
        if (m->n_prefix == 2) { a1 = th[0]; a2 = th[1]; }
        FN(chain_forward_store)(m, thc, u, hs, pre);
        FN(chain_vjp)(m, thc, hs, pre, lam, dx, gthc, w);
        dlam[0] = a1 * lam[0] + dx[0];
        dlam[1] = -a2 * lam[1] + dx[1];
        if (gth && m->n_prefix == 1) gth[0] += w * (-u[1] * lam[1]);
        if (gth && m->n_prefix == 2) { gth[0] += w * (u[0] * lam[0]); gth[1] += w * (-u[1] * lam[1]); }
        break;
    }
    case UDE_MODEL_SEIR: {
        const REAL F = (REAL)m->consts[0], b0 = (REAL)m->consts[1], mu = (REAL)m->consts[4],
                   sg = (REAL)m->consts[5], gm = (REAL)m->consts[6], dd = (REAL)m->consts[7],
                   lm = (REAL)m->consts[8];
        const REAL S = u[0], I = u[2], N = u[4], D = u[5];
        (void)I;
        REAL x[3] = { S / N, u[2], D / N };
        FN(chain_forward_store)(m, thc, x, hs, pre);
        REAL dz = lam[1] - lam[0];               /* z enters dS with -, dE with + */
        FN(chain_vjp)(m, thc, hs, pre, &dz, dx, gthc, w);
        const REAL c = b0 * F / N;               /* d(b0*S*F/N)/dS */
        const REAL cN = -b0 * S * F / (N * N);   /* d(b0*S*F/N)/dN */
        /* columns of J: contributions to dlam[k] = sum_r lam[r] * d f_r / d u_k */
        dlam[0] = lam[0] * (-c - mu) + lam[1] * c + dx[0] / N;
        dlam[1] = lam[1] * (-(sg + mu)) + lam[2] * sg + lam[6] * sg;
        dlam[2] = lam[2] * (-(gm + mu)) + lam[3] * gm + lam[5] * dd * gm + dx[1];
        dlam[3] = lam[3] * (-mu);
        dlam[4] = lam[0] * (-cN) + lam[1] * cN + lam[4] * (-mu)
                  - dx[0] * S / (N * N) - dx[2] * D / (N * N);
        dlam[5] = lam[5] * (-lm) + dx[2] / N;
        dlam[6] = 0;
        break;
    }
    case UDE_MODEL_FKPP: {
        const size_t cl = FN(chain_len)(m);
        const REAL *sx = thc + cl;
        REAL *gsx = gthc ? gthc + cl : NULL;
        const REAL w1 = sx[0], w2 = sx[1], w3 = sx[2], D0 = sx[4];
        const int n = m->d;
        for (int i = 0; i < n; ++i) dlam[i] = 0;
        for (int i = 0; i < n; ++i) {
            const int im = (i + n - 1) % n, ip = (i + 1) % n;
            FN(chain_forward_store)(m, thc, &u[i], hs, pre);
            FN(chain_vjp)(m, thc, hs, pre, &lam[i], dx, gthc, w);
            dlam[i] += dx[0] + D0 * w2 * lam[i];
            dlam[im] += D0 * w1 * lam[i];
            dlam[ip] += D0 * w3 * lam[i];
            if (gsx) {
                gsx[0] += w * D0 * u[im] * lam[i];
                gsx[1] += w * D0 * u[i] * lam[i];
                gsx[2] += w * D0 * u[ip] * lam[i];
                gsx[4] += w * (w1 * u[im] + w2 * u[i] + w3 * u[ip]) * lam[i];
            }
        }
        break;
    }
    case UDE_MODEL_SEIR_NODE: {
        const REAL mu = (REAL)m->consts[4], sg = (REAL)m->consts[5];
        const REAL S = u[0], N = u[4], D = u[5];
        REAL x[7] = { S / N, u[1], u[2], u[3], N, D / N, u[6] };
        REAL dy[7] = { lam[0], lam[1], lam[2], lam[3], lam[5], 0, 0 };
        FN(chain_forward_store)(m, thc, x, hs, pre);
        FN(chain_vjp)(m, thc, hs, pre, dy, dx, gthc, w);
        dlam[0] = dx[0] / N;
        dlam[1] = dx[1] + sg * lam[6];
        dlam[2] = dx[2];
        dlam[3] = dx[3];
        dlam[4] = dx[4] - mu * lam[4] - dx[0] * S / (N * N) - dx[5] * D / (N * N);
        dlam[5] = dx[5] / N;
        dlam[6] = dx[6];
        break;
    }
    default:
        FN(chain_forward_store)(m, thc, u, hs, pre);
        FN(chain_vjp)(m, thc, hs, pre, lam, dx, gthc, w);
        for (int k = 0; k < m->d; ++k) dlam[k] = dx[k];
    }
}

/* ---------------------------------------------------------- RK stepping ---- */
/* one explicit RK step with the generic tableau; ks[s][d] receives the stage derivatives.
 * Tsit5: stage 7 argument IS u_new (row 7 = b, FSAL); Vern7: u_new from b. */
static void FN(rk_step)(const ude_model *m, const REAL *th, const ude_tableau *tb, const REAL *u,
                        REAL dt, const REAL *k1_in, REAL *ks, REAL *unew, REAL *err)
{
    const int d = m->d, s = tb->s;
    REAL g[UDE_MAX_STATE];
    if (k1_in) for (int k = 0; k < d; ++k) ks[k] = k1_in[k];
    else FN(ude_rhs)(m, th, u, ks);
    for (int i = 1; i < s; ++i) {
        for (int k = 0; k < d; ++k) {
            REAL acc = 0;
            for (int j = 0; j < i; ++j) {
                const REAL a = (REAL)tb->A[i][j];
                if (a != 0) acc += a * ks[(size_t)j * d + k];
            }
            g[k] = u[k] + dt * acc;
        }
        if (tb->fsal && i == s - 1) for (int k = 0; k < d; ++k) unew[k] = g[k];
        FN(ude_rhs)(m, th, g, ks + (size_t)i * d);
    }
    if (!tb->fsal) {
        for (int k = 0; k < d; ++k) {
            REAL acc = 0;
            for (int j = 0; j < s; ++j) {
                const REAL b = (REAL)tb->b[j];
                if (b != 0) acc += b * ks[(size_t)j * d + k];
            }
            unew[k] = u[k] + dt * acc;
        }
    }
    if (err) {
        for (int k = 0; k < d; ++k) {
            REAL acc = 0;
            for (int j = 0; j < s; ++j) {
                const REAL b = (REAL)tb->bt[j];
                if (b != 0) acc += b * ks[(size_t)j * d + k];
            }
            err[k] = dt * acc;
        }
    }
}

static int FN(all_finite)(const REAL *x, int n)
{
    for (int i = 0; i < n; ++i) if (!isfinite((double)x[i])) return 0;
    return 1;
}

int FN(ude_solve_fixed)(const ude_model *m, const REAL *th, const REAL *u0, REAL dt, int n_steps,
                        int solver, int save_every, REAL *out, REAL *dense)
{
    const ude_tableau *tb = ude_get_tableau(solver);
    const int d = m->d, s = tb->s;
    REAL u[UDE_MAX_STATE], un[UDE_MAX_STATE];
    REAL ks[UDE_MAX_STAGES * UDE_MAX_STATE], kf[UDE_MAX_STATE];
    int have_fsal = 0, isave = 0;
    for (int k = 0; k < d; ++k) u[k] = u0[k];
    for (int k = 0; k < d; ++k) out[(size_t)isave * d + k] = u[k];
    ++isave;
    for (int n = 0; n < n_steps; ++n) {
        FN(rk_step)(m, th, tb, u, dt, have_fsal ? kf : NULL, ks, un, NULL);
        if (dense) memcpy(dense + (size_t)n * s * d, ks, sizeof(REAL) * (size_t)s * d);
        if (tb->fsal) { memcpy(kf, ks + (size_t)(s - 1) * d, sizeof(REAL) * d); have_fsal = 1; }
        for (int k = 0; k < d; ++k) u[k] = un[k];
        if ((n + 1) % save_every == 0) {
            for (int k = 0; k < d; ++k) out[(size_t)isave * d + k] = u[k];
            ++isave;
        }
        if (!FN(all_finite)(u, d)) return -1;
    }
    return 0;
}

/* Tsit5 free 4th-order interpolant weights b_i(Theta), i = 1..7 (Tsitouras 2011;
 * the r_ij block of OrdinaryDiffEq's Tsit5ConstantCache) */
static void FN(tsit5_bTheta)(REAL Th, REAL *bw)
{
    const double *r = ude_tsit5_r;   /* r11 r12 r13 r14 | r22 r23 r24 | ... | r72 r73 r74 */
    const REAL T2 = Th * Th;
    bw[0] = Th * ((REAL)r[0] + Th * ((REAL)r[1] + Th * ((REAL)r[2] + Th * (REAL)r[3])));
    for (int i = 1; i < 7; ++i) {
        const double *ri = r + 4 + 3 * (i - 1);
        bw[i] = T2 * ((REAL)ri[0] + Th * ((REAL)ri[1] + Th * (REAL)ri[2]));
    }
}

/* RMS error norm of OrdinaryDiffEq (ODE_DEFAULT_NORM) on err/(abstol + reltol*max(|u|,|unew|)) */
static REAL FN(eest)(const REAL *err, const REAL *u, const REAL *un, int d, REAL abstol, REAL reltol)
{
    REAL acc = 0;
    for (int k = 0; k < d; ++k) {
        const REAL a = R_FABS(u[k]), b = R_FABS(un[k]);
        const REAL sc = abstol + reltol * (a > b ? a : b);
        const REAL e = err[k] / sc;
        acc += e * e;
    }
    return R_SQRT(acc / (REAL)d);
}

int FN(ude_solve_adaptive)(const ude_model *m, const REAL *th, const REAL *u0, const REAL *saveat,
                           int n_save, REAL abstol, REAL reltol, int solver, REAL *out,
                           int *n_rejected)
{
    const ude_tableau *tb = ude_get_tableau(solver);
    const int d = m->d, s = tb->s, order = tb->order;
    const REAL t0 = saveat[0], t1 = saveat[n_save - 1];
    /* OrdinaryDiffEq defaults: gamma=9/10, qmin=1/5, qmax=10, beta2=2/(5*order), beta1=7/(10*order),
     * qsteady_min = qsteady_max = 1 (explicit RK), qoldinit=1e-4 */
    const REAL gamma = (REAL)0.9, qmin = (REAL)0.2, qmax = (REAL)10;
    const REAL beta2 = (REAL)2 / ((REAL)5 * order), beta1 = (REAL)7 / ((REAL)10 * order);
    REAL qold = (REAL)1e-4;
    REAL u[UDE_MAX_STATE], un[UDE_MAX_STATE], err[UDE_MAX_STATE], f0[UDE_MAX_STATE], f1[UDE_MAX_STATE];
    REAL ks[UDE_MAX_STAGES * UDE_MAX_STATE], kf[UDE_MAX_STATE];
    for (int k = 0; k < d; ++k) u[k] = u0[k];
    for (int k = 0; k < d; ++k) out[k] = u[k];
    int isave = 1, nacc = 0, nrej = 0;
    /* initial dt: Hairer-Norsett-Wanner heuristic as in OrdinaryDiffEq's ode_determine_initdt */
    REAL dt;
    {
        FN(ude_rhs)(m, th, u, f0);
        REAL d0 = 0, d1 = 0, d2 = 0;
        for (int k = 0; k < d; ++k) {
            const REAL sk = abstol + reltol * R_FABS(u[k]);
            d0 += (u[k] / sk) * (u[k] / sk);
            d1 += (f0[k] / sk) * (f0[k] / sk);
        }
        d0 = R_SQRT(d0 / d); d1 = R_SQRT(d1 / d);
        REAL dt0 = (d0 < (REAL)1e-5 || d1 < (REAL)1e-5) ? (REAL)1e-6 : (REAL)0.01 * d0 / d1;
        if (dt0 > t1 - t0) dt0 = t1 - t0;
        for (int k = 0; k < d; ++k) un[k] = u[k] + dt0 * f0[k];
        FN(ude_rhs)(m, th, un, f1);
        for (int k = 0; k < d; ++k) {
            const REAL sk = abstol + reltol * R_FABS(u[k]);
            const REAL e = (f1[k] - f0[k]) / sk;
            d2 += e * e;
        }
        d2 = R_SQRT(d2 / d) / dt0;
        const REAL dm = d1 > d2 ? d1 : d2;
        REAL dt1 = dm <= (REAL)1e-15 ? (dt0 * (REAL)1e-3 > (REAL)1e-6 ? dt0 * (REAL)1e-3 : (REAL)1e-6)
                                     : R_POW((REAL)10, -((REAL)2 + R_LOG10(dm)) / (REAL)order);
        dt = (REAL)100 * dt0 < dt1 ? (REAL)100 * dt0 : dt1;
        if (dt > t1 - t0) dt = t1 - t0;
    }
    memcpy(kf, f0, sizeof(REAL) * d);
    int have_fsal = tb->fsal;
    REAL t = t0;
    const int use_interp = (solver == UDE_TSIT5);
    int guard = 0;
    while (isave < n_save && guard++ < 10000000) {
        REAL tend = use_interp ? t1 : saveat[isave];
        REAL h = dt;
        int clipped = 0;
        if (t + h >= tend - (REAL)1e-12 * R_FABS(tend)) { h = tend - t; clipped = 1; }
        FN(rk_step)(m, th, tb, u, h, have_fsal ? kf : NULL, ks, un, err);
        const REAL EEst = FN(eest)(err, u, un, d, abstol, reltol);
        if (!isfinite((double)EEst)) { if (n_rejected) *n_rejected = nrej; return -1; }
        const REAL q11 = R_POW(EEst, beta1);
        REAL q = q11 / R_POW(qold, beta2);
        q = q / gamma;
        if (q < (REAL)1 / qmax) q = (REAL)1 / qmax;
        if (q > (REAL)1 / qmin) q = (REAL)1 / qmin;
        if (EEst <= (REAL)1) {
            ++nacc;
            const REAL tn = t + h;
            if (use_interp) {
                while (isave < n_save && saveat[isave] <= tn + (REAL)1e-12 * R_FABS(tn)) {
                    REAL Th = (saveat[isave] - t) / h, bw[7];
                    if (Th > 1) Th = 1;
                    FN(tsit5_bTheta)(Th, bw);
                    for (int k = 0; k < d; ++k) {
                        REAL acc = 0;
                        for (int i = 0; i < 7; ++i) acc += bw[i] * ks[(size_t)i * d + k];
                        out[(size_t)isave * d + k] = u[k] + h * acc;
                    }
                    ++isave;
                }
            } else if (clipped) {
                for (int k = 0; k < d; ++k) out[(size_t)isave * d + k] = un[k];
                ++isave;
            }
            qold = EEst > (REAL)1e-4 ? EEst : (REAL)1e-4;
            /* qsteady_min = qsteady_max = 1 for explicit RK methods (OrdinaryDiffEq defaults; 6/5 is the implicit-solver band): no dead band */
            if (!clipped || h >= dt) dt = h / q; /* a clipped (shortened) step does not shrink the proposal */
            else { const REAL prop = h / q; if (prop > dt) dt = prop; }
            t = tn;
            for (int k = 0; k < d; ++k) u[k] = un[k];
            if (tb->fsal) { memcpy(kf, ks + (size_t)(s - 1) * d, sizeof(REAL) * d); have_fsal = 1; }
            else have_fsal = 0;   /* k1 kept from a rejected attempt is stale once u has moved */
        } else {
            ++nrej;
            REAL qr = q11 / gamma;
            if (qr > (REAL)1 / qmin) qr = (REAL)1 / qmin;
            dt = h / qr;
            /* k1 of the rejected step is still f(u): reuse it */
            memcpy(kf, ks, sizeof(REAL) * d);
            have_fsal = 1;
        }
    }
    if (n_rejected) *n_rejected = nrej;
    return isave == n_save ? nacc : -1;
}

/* ------------------------------------------------ RKC2 (stabilised explicit) -- */
/* Second-order Runge-Kutta-Chebyshev (Sommeijer, Shampine, Verwer 1998): the closed-form member of the family the
 * north star names as ROCK2 (Climate/NeuralPDE/npde.jl:61,82; ROCK2's own coefficient tables are not in the reference).
 * Per step with s stages:  Y0 = u, Y1 = Y0 + mt1 h F0,
 *   Yj = (1 - mu_j - nu_j) Y0 + mu_j Y_{j-1} + nu_j Y_{j-2} + mt_j h F_{j-1} + ga_j h F0,  u_next = Y_s.
 * Dense output = cubic Hermite on (u_n, f_n, u_{n+1}, f_{n+1}) (OrdinaryDiffEq's default interpolant for such methods).
 * The interpolating adjoint integrates lambda backwards with the SAME scheme; mu never feeds back, so its update is a fixed
 * linear combination h sum_k w_k G_k of the stage integrands, with w from running the recurrence on unit vectors. */
#ifndef UDE_RKC_TABLES_DEFINED
#define UDE_RKC_TABLES_DEFINED
#include <float.h>
#if LDBL_MANT_DIG <= DBL_MANT_DIG
#error "ude_rkc2_tables needs a long double wider than double (x86-64, aarch64 Linux) for fp64-accurate RKC2 tables"
#endif
#define UDE_RKC_MAX_STAGES 64
typedef struct {
    int s;
    double mt1;
    double mu[UDE_RKC_MAX_STAGES + 1], nu[UDE_RKC_MAX_STAGES + 1], mt[UDE_RKC_MAX_STAGES + 1], ga[UDE_RKC_MAX_STAGES + 1];
    double c[UDE_RKC_MAX_STAGES + 1];   /* stage abscissae, c[0] = 0, c[s] = 1 */
    double w[UDE_RKC_MAX_STAGES + 1];   /* quadrature weights of the stage integrands F_0..F_{s-1} */
    double beta;                        /* length of the real stability interval */
} ude_rkc_tables;

static void ude_rkc2_tables(int s, ude_rkc_tables *t)
{
    /* T_j, T_j', T_j'' and b_j in long double: in double the relative error of the three-term recurrences grows like
     * j^2 eps, which at s = 64 moves the tables' stability polynomial by ~1e-10 at the end of its interval */
    const long double eps = 2.0L / 13.0L;
    const long double w0 = 1.0L + eps / ((long double)s * s);
    long double T[UDE_RKC_MAX_STAGES + 1], dT[UDE_RKC_MAX_STAGES + 1], d2T[UDE_RKC_MAX_STAGES + 1], b[UDE_RKC_MAX_STAGES + 1] = {0};
    T[0] = 1; T[1] = w0; dT[0] = 0; dT[1] = 1; d2T[0] = 0; d2T[1] = 0;
    for (int j = 2; j <= s; ++j) {
        T[j] = 2 * w0 * T[j - 1] - T[j - 2];
        dT[j] = 2 * T[j - 1] + 2 * w0 * dT[j - 1] - dT[j - 2];
        d2T[j] = 4 * dT[j - 1] + 2 * w0 * d2T[j - 1] - d2T[j - 2];
    }
    const long double w1 = dT[s] / d2T[s];
    for (int j = 2; j <= s; ++j) b[j] = d2T[j] / (dT[j] * dT[j]);
    b[0] = b[1] = b[2];
    t->s = s;
    t->mt1 = (double)(b[1] * w1);
    t->beta = (double)((w0 + 1.0L) * d2T[s] / dT[s]);
    for (int j = 2; j <= s; ++j) {
        const long double mt = 2 * b[j] * w1 / b[j - 1];
        t->mu[j] = (double)(2 * b[j] * w0 / b[j - 1]);
        t->nu[j] = (double)(-b[j] / b[j - 2]);
        t->mt[j] = (double)mt;
        t->ga[j] = (double)(-(1.0L - b[j - 1] * T[j - 1]) * mt);
    }
    /* abscissae and quadrature weights from the recurrence itself (y' = 1, and unit impulses in F_k) */
    double W[UDE_RKC_MAX_STAGES + 1][UDE_RKC_MAX_STAGES + 1];
    memset(W, 0, sizeof W);
    t->c[0] = 0; t->c[1] = t->mt1;
    W[1][0] = t->mt1;
    for (int j = 2; j <= s; ++j) {
        t->c[j] = t->mu[j] * t->c[j - 1] + t->nu[j] * t->c[j - 2] + t->mt[j] + t->ga[j];
        for (int k = 0; k < j; ++k) W[j][k] = t->mu[j] * W[j - 1][k] + t->nu[j] * W[j - 2][k];
        W[j][j - 1] += t->mt[j];
        W[j][0] += t->ga[j];
    }
    for (int k = 0; k < s; ++k) t->w[k] = W[s][k];
}

int ude_rkc2_coefficients(int s, double *mt1, double *mu, double *nu, double *mt, double *ga, double *c, double *w, double *beta)
{
    if (s < 2 || s > UDE_RKC_MAX_STAGES) return -1;
    ude_rkc_tables t;
    ude_rkc2_tables(s, &t);
    *mt1 = t.mt1; *beta = t.beta;
    for (int j = 0; j <= s; ++j) { mu[j] = j >= 2 ? t.mu[j] : 0; nu[j] = j >= 2 ? t.nu[j] : 0; mt[j] = j >= 2 ? t.mt[j] : 0; ga[j] = j >= 2 ? t.ga[j] : 0; c[j] = t.c[j]; w[j] = j < s ? t.w[j] : 0; }
    return 0;
}
#endif

/* forward: out[n_save][d]; ustep[n_steps+1][d] and fstep[n_steps+1][d] (f(u_n)) are the record the adjoint reads */
int FN(ude_solve_rkc2_fixed)(const ude_model *m, const REAL *th, const REAL *u0, REAL dt, int n_steps, int stages,
                             int save_every, REAL *out, REAL *ustep, REAL *fstep)
{
    if (stages < 2 || stages > UDE_RKC_MAX_STAGES) return -2;
    ude_rkc_tables t;
    ude_rkc2_tables(stages, &t);
    const int d = m->d, s = stages;
    REAL u[UDE_MAX_STATE], F0[UDE_MAX_STATE], F[UDE_MAX_STATE], Y0[UDE_MAX_STATE], Y1[UDE_MAX_STATE], Y2[UDE_MAX_STATE];
    for (int k = 0; k < d; ++k) u[k] = u0[k];
    for (int k = 0; k < d; ++k) out[k] = u[k];
    int isave = 1;
    for (int n = 0; n < n_steps; ++n) {
        FN(ude_rhs)(m, th, u, F0);
        if (ustep) for (int k = 0; k < d; ++k) { ustep[(size_t)n * d + k] = u[k]; fstep[(size_t)n * d + k] = F0[k]; }
        for (int k = 0; k < d; ++k) { Y0[k] = u[k]; Y1[k] = u[k] + (REAL)t.mt1 * dt * F0[k]; }
        for (int j = 2; j <= s; ++j) {
            FN(ude_rhs)(m, th, Y1, F);
            const REAL mu = (REAL)t.mu[j], nu = (REAL)t.nu[j], mt = (REAL)t.mt[j], ga = (REAL)t.ga[j];
            for (int k = 0; k < d; ++k) Y2[k] = ((REAL)1 - mu - nu) * u[k] + mu * Y1[k] + nu * Y0[k] + mt * dt * F[k] + ga * dt * F0[k];
            for (int k = 0; k < d; ++k) { Y0[k] = Y1[k]; Y1[k] = Y2[k]; }
        }
        for (int k = 0; k < d; ++k) u[k] = Y1[k];
        if ((n + 1) % save_every == 0) {
            for (int k = 0; k < d; ++k) out[(size_t)isave * d + k] = u[k];
            ++isave;
        }
        if (!FN(all_finite)(u, d)) return -1;
    }
    if (ustep) {
        FN(ude_rhs)(m, th, u, F0);
        for (int k = 0; k < d; ++k) { ustep[(size_t)n_steps * d + k] = u[k]; fstep[(size_t)n_steps * d + k] = F0[k]; }
    }
    return 0;
}

/* interpolating adjoint of an RKC2 solve: lambda stepped backwards with RKC2 itself, u(t) by cubic Hermite */
void FN(ude_adjoint_rkc2_fixed)(const ude_model *m, const REAL *th, const REAL *ustep, const REAL *fstep, REAL dt, int n_steps,
                                int stages, int save_every, const REAL *dLdout, REAL *grad_theta, REAL *grad_u0)
{
    ude_rkc_tables t;
    ude_rkc2_tables(stages, &t);
    const int d = m->d, s = stages;
    REAL lam[UDE_MAX_STATE], x[UDE_MAX_STATE], F0[UDE_MAX_STATE], F[UDE_MAX_STATE], Y0[UDE_MAX_STATE], Y1[UDE_MAX_STATE], Y2[UDE_MAX_STATE];
    const int n_save = n_steps / save_every + 1;
    for (int k = 0; k < d; ++k) lam[k] = dLdout[(size_t)(n_save - 1) * d + k];
    for (int n = n_steps - 1; n >= 0; --n) {
        const REAL *y0 = ustep + (size_t)n * d, *y1 = ustep + (size_t)(n + 1) * d, *f0 = fstep + (size_t)n * d, *f1 = fstep + (size_t)(n + 1) * d;
        /* stage k of the backward step sits at t_{n+1} - c_k dt, i.e. Theta = 1 - c_k of the forward step */
        for (int j = 0; j < s; ++j) {
            const REAL Th = (REAL)1 - (REAL)t.c[j];
            for (int k = 0; k < d; ++k)
                x[k] = ((REAL)1 - Th) * y0[k] + Th * y1[k]
                     + Th * (Th - (REAL)1) * (((REAL)1 - (REAL)2 * Th) * (y1[k] - y0[k]) + (Th - (REAL)1) * dt * f0[k] + Th * dt * f1[k]);
            const REAL *Yj = j == 0 ? lam : Y1;
            REAL *Fj = j == 0 ? F0 : F;
            FN(ude_rhs_vjp)(m, th, x, Yj, Fj, grad_theta, dt * (REAL)t.w[j]);
            if (j == 0) {
                for (int k = 0; k < d; ++k) { Y0[k] = lam[k]; Y1[k] = lam[k] + (REAL)t.mt1 * dt * F0[k]; }
            } else {
                const int jj = j + 1;   /* F = G(Y_j) feeds Y_{j+1} */
                const REAL mu = (REAL)t.mu[jj], nu = (REAL)t.nu[jj], mt = (REAL)t.mt[jj], ga = (REAL)t.ga[jj];
                for (int k = 0; k < d; ++k) Y2[k] = ((REAL)1 - mu - nu) * lam[k] + mu * Y1[k] + nu * Y0[k] + mt * dt * F[k] + ga * dt * F0[k];
                for (int k = 0; k < d; ++k) { Y0[k] = Y1[k]; Y1[k] = Y2[k]; }
            }
        }
        for (int k = 0; k < d; ++k) lam[k] = Y1[k];
        if (n % save_every == 0)
            for (int k = 0; k < d; ++k) lam[k] += dLdout[(size_t)(n / save_every) * d + k];
    }
    for (int k = 0; k < d; ++k) grad_u0[k] = lam[k];
}

/* ------------------------------------------------ discrete adjoint ---------- */
/* Exact gradient of the DISCRETE fixed-step Tsit5 scheme (what ForwardDiffSensitivity, scenario_1.jl:86 /
 * scenario_2.jl:108 / hudson_bay.jl:102, computes in forward mode -- here by reverse accumulation through the
 * stages): with g_i = u_n + dt sum_{j<i} a_ij k_j, k_i = f(g_i), u_{n+1} = u_n + dt sum_{i<=6} b_i k_i,
 *   kbar_i = dt (b_i ubar_{n+1} + sum_{j>i} a_ji gbar_j),  gbar_i = J_u(g_i)^T kbar_i,
 *   ubar_n = ubar_{n+1} + sum_i gbar_i,  grad_theta += J_theta(g_i)^T kbar_i.
 * k_7 (FSAL) has weight 0 in the update and is the next step's k_1 = f(u_{n+1}), which that step accounts for. */
void FN(ude_adjoint_discrete_fixed)(const ude_model *m, const REAL *th, const REAL *out, const REAL *dense,
                                    REAL dt, int n_steps, int save_every, const REAL *dLdout,
                                    REAL *grad_theta, REAL *grad_u0)
{
    const ude_tableau *tb = ude_get_tableau(UDE_TSIT5);
    const int d = m->d, s = 7;
    REAL lam[UDE_MAX_STATE], kb[UDE_MAX_STATE], x[UDE_MAX_STATE];
    REAL gb[6 * UDE_MAX_STATE];
    const int n_save = n_steps / save_every + 1;
    for (int k = 0; k < d; ++k) lam[k] = dLdout[(size_t)(n_save - 1) * d + k];
    REAL *ustart = (REAL *)malloc(sizeof(REAL) * (size_t)(n_steps + 1) * d);
    for (int k = 0; k < d; ++k) ustart[k] = out[k];
    for (int n = 0; n < n_steps; ++n) {
        const REAL *ks = dense + (size_t)n * s * d;
        if ((n + 1) % save_every == 0) {
            for (int k = 0; k < d; ++k) ustart[(size_t)(n + 1) * d + k] = out[(size_t)((n + 1) / save_every) * d + k];
        } else {
            for (int k = 0; k < d; ++k) {
                REAL acc = 0;
                for (int j = 0; j < 6; ++j) acc += (REAL)tb->A[6][j] * ks[(size_t)j * d + k];
                ustart[(size_t)(n + 1) * d + k] = ustart[(size_t)n * d + k] + dt * acc;
            }
        }
    }
    for (int n = n_steps - 1; n >= 0; --n) {
        const REAL *ks = dense + (size_t)n * s * d;
        const REAL *u_n = ustart + (size_t)n * d;
        for (int i = 5; i >= 0; --i) {
            for (int k = 0; k < d; ++k) {
                REAL acc = 0;
                for (int j = 0; j < i; ++j) acc += (REAL)tb->A[i][j] * ks[(size_t)j * d + k];
                x[k] = u_n[k] + dt * acc;
                REAL c = (REAL)tb->A[6][i] * lam[k];
                for (int j = i + 1; j < 6; ++j) c += (REAL)tb->A[j][i] * gb[(size_t)j * d + k];
                kb[k] = dt * c;
            }
            FN(ude_rhs_vjp)(m, th, x, kb, gb + (size_t)i * d, grad_theta, (REAL)1);
        }
        for (int k = 0; k < d; ++k) {
            REAL acc = lam[k];
            for (int i = 0; i < 6; ++i) acc += gb[(size_t)i * d + k];
            lam[k] = acc;
        }
        if (n % save_every == 0)
            for (int k = 0; k < d; ++k) lam[k] += dLdout[(size_t)(n / save_every) * d + k];
    }
    for (int k = 0; k < d; ++k) grad_u0[k] = lam[k];
    free(ustart);
}

/* ------------------------------------------------ interpolating adjoint ---- */
/* InterpolatingAdjoint (seir_exposure.jl:71,140; Fisher-KPP-CNN.jl:136): the
 * augmented state [lambda; mu] is integrated from T back to t0 with the same
 * Runge-Kutta method and step; u(t) at the backward stage times comes from the
 * forward solution's dense output (Tsit5 4th-order interpolant over the stored
 * k_1..k_7 of the step containing t); at every save time the loss cotangent
 * dL/du(t_i) is added to lambda (discrete callback), which also invalidates
 * FSAL, so k_1 is re-evaluated after each jump.  mu' = -lambda^T df/dtheta never
 * feeds back, so its quadrature is accumulated straight into grad_theta. */
void FN(ude_adjoint_fixed)(const ude_model *m, const REAL *th, const REAL *out, const REAL *dense,
                           REAL dt, int n_steps, int save_every, const REAL *dLdout,
                           REAL *grad_theta, REAL *grad_u0)
{
    const ude_tableau *tb = ude_get_tableau(UDE_TSIT5);
    const int d = m->d, s = 7;
    REAL lam[UDE_MAX_STATE], g[UDE_MAX_STATE], uu[UDE_MAX_STATE], un[UDE_MAX_STATE];
    REAL kl[7 * UDE_MAX_STATE];
    const int n_save = n_steps / save_every + 1;
    for (int k = 0; k < d; ++k) lam[k] = dLdout[(size_t)(n_save - 1) * d + k];
    /* reconstruct u_n at every step start from the saved states + dense output */
    REAL *ustart = (REAL *)malloc(sizeof(REAL) * (size_t)(n_steps + 1) * d);
    for (int k = 0; k < d; ++k) ustart[k] = out[k];
    for (int n = 0; n < n_steps; ++n) {
        const REAL *ks = dense + (size_t)n * s * d;
        if ((n + 1) % save_every == 0) {
            for (int k = 0; k < d; ++k) ustart[(size_t)(n + 1) * d + k] = out[(size_t)((n + 1) / save_every) * d + k];
        } else {
            for (int k = 0; k < d; ++k) {
                REAL acc = 0;
                for (int j = 0; j < 6; ++j) acc += (REAL)tb->A[6][j] * ks[(size_t)j * d + k];
                ustart[(size_t)(n + 1) * d + k] = ustart[(size_t)n * d + k] + dt * acc;
            }
        }
    }
    for (int n = n_steps - 1; n >= 0; --n) {
        const REAL *ks = dense + (size_t)n * s * d;
        const REAL *u_n = ustart + (size_t)n * d;
        /* backward step from t_{n+1} to t_n; stage i at t_{n+1} - c_i dt, Theta_i = 1 - c_i */
        for (int i = 0; i < 6; ++i) {          /* k_7 only feeds FSAL/error: not needed */
            const REAL Th = (REAL)1 - (REAL)tb->c[i];
            REAL bw[7];
            FN(tsit5_bTheta)(Th, bw);
            for (int k = 0; k < d; ++k) {
                REAL acc = 0;
                for (int j = 0; j < 7; ++j) acc += bw[j] * ks[(size_t)j * d + k];
                uu[k] = u_n[k] + dt * acc;
            }
            for (int k = 0; k < d; ++k) {
                REAL acc = 0;
                for (int j = 0; j < i; ++j) {
                    const REAL a = (REAL)tb->A[i][j];
                    if (a != 0) acc += a * kl[(size_t)j * d + k];
                }
                g[k] = lam[k] + dt * acc;
            }
            /* kl_i = J_u^T g ; grad_theta += dt*b_i * J_theta^T g */
            FN(ude_rhs_vjp)(m, th, uu, g, kl + (size_t)i * d, grad_theta, dt * (REAL)tb->A[6][i]);
        }
        for (int k = 0; k < d; ++k) {
            REAL acc = 0;
            for (int j = 0; j < 6; ++j) acc += (REAL)tb->A[6][j] * kl[(size_t)j * d + k];
            un[k] = lam[k] + dt * acc;
        }
        for (int k = 0; k < d; ++k) lam[k] = un[k];
        if (n % save_every == 0)
            for (int k = 0; k < d; ++k) lam[k] += dLdout[(size_t)(n / save_every) * d + k];
    }
    for (int k = 0; k < d; ++k) grad_u0[k] = lam[k];
    free(ustart);
}

/* ---------------------------------------------- adaptive forward with dense output ---- */
/* Adaptive Tsit5 (same controller as ude_solve_adaptive) that also records every ACCEPTED step:
 * tgrid[0..nacc], ustep[(nacc+1) x d], dense[nacc x 7 x d] -- what InterpolatingAdjoint interpolates.
 * saveat values are produced by the interpolant.  Returns the number of accepted steps or -1
 * (non-finite state, or more than max_steps steps). */
int FN(ude_solve_adaptive_dense)(const ude_model *m, const REAL *th, const REAL *u0, const REAL *saveat,
                                 int n_save, REAL abstol, REAL reltol, int max_steps, REAL *out,
                                 REAL *tgrid, REAL *ustep, REAL *dense)
{
    const ude_tableau *tb = ude_get_tableau(UDE_TSIT5);
    const int d = m->d, s = 7, order = 5;
    const REAL t0 = saveat[0], t1 = saveat[n_save - 1];
    const REAL gamma = (REAL)0.9, qmin = (REAL)0.2, qmax = (REAL)10;
    const REAL beta2 = (REAL)2 / ((REAL)5 * order), beta1 = (REAL)7 / ((REAL)10 * order);
    REAL qold = (REAL)1e-4;
    REAL u[UDE_MAX_STATE], un[UDE_MAX_STATE], err[UDE_MAX_STATE], f0[UDE_MAX_STATE], f1[UDE_MAX_STATE];
    REAL ks[UDE_MAX_STAGES * UDE_MAX_STATE], kf[UDE_MAX_STATE];
    for (int k = 0; k < d; ++k) { u[k] = u0[k]; out[k] = u[k]; ustep[k] = u[k]; }
    tgrid[0] = t0;
    int isave = 1, nacc = 0;
    REAL dt;
    {
        FN(ude_rhs)(m, th, u, f0);
        REAL d0 = 0, d1 = 0, d2 = 0;
        for (int k = 0; k < d; ++k) {
            const REAL sk = abstol + reltol * R_FABS(u[k]);
            d0 += (u[k] / sk) * (u[k] / sk);
            d1 += (f0[k] / sk) * (f0[k] / sk);
        }
        d0 = R_SQRT(d0 / d); d1 = R_SQRT(d1 / d);
        REAL dt0 = (d0 < (REAL)1e-5 || d1 < (REAL)1e-5) ? (REAL)1e-6 : (REAL)0.01 * d0 / d1;
        if (dt0 > t1 - t0) dt0 = t1 - t0;
        for (int k = 0; k < d; ++k) un[k] = u[k] + dt0 * f0[k];
        FN(ude_rhs)(m, th, un, f1);
        for (int k = 0; k < d; ++k) {
            const REAL sk = abstol + reltol * R_FABS(u[k]);
            const REAL e = (f1[k] - f0[k]) / sk;
            d2 += e * e;
        }
        d2 = R_SQRT(d2 / d) / dt0;
        const REAL dm = d1 > d2 ? d1 : d2;
        REAL dt1 = dm <= (REAL)1e-15 ? (dt0 * (REAL)1e-3 > (REAL)1e-6 ? dt0 * (REAL)1e-3 : (REAL)1e-6)
                                     : R_POW((REAL)10, -((REAL)2 + R_LOG10(dm)) / (REAL)order);
        dt = (REAL)100 * dt0 < dt1 ? (REAL)100 * dt0 : dt1;
        if (dt > t1 - t0) dt = t1 - t0;
    }
    memcpy(kf, f0, sizeof(REAL) * d);
    REAL t = t0;
    int guard = 0;
    while (isave < n_save && guard++ < 100000000) {
        REAL h = dt;
        int clipped = 0;
        if (t + h >= t1 - (REAL)1e-7 * R_FABS(t1)) { h = t1 - t; clipped = 1; }
        FN(rk_step)(m, th, tb, u, h, kf, ks, un, err);
        const REAL EEst = FN(eest)(err, u, un, d, abstol, reltol);
        if (!isfinite((double)EEst)) return -1;
        const REAL q11 = R_POW(EEst, beta1);
        REAL q = q11 / R_POW(qold, beta2);
        q = q / gamma;
        if (q < (REAL)1 / qmax) q = (REAL)1 / qmax;
        if (q > (REAL)1 / qmin) q = (REAL)1 / qmin;
        if (EEst <= (REAL)1) {
            if (nacc >= max_steps) return -1;
            const REAL tn = clipped ? t1 : t + h;
            memcpy(dense + (size_t)nacc * s * d, ks, sizeof(REAL) * (size_t)s * d);
            while (isave < n_save && saveat[isave] <= tn + (REAL)1e-7 * R_FABS(tn)) {
                REAL Th = (saveat[isave] - t) / h, bw[7];
                if (Th > 1) Th = 1;
                FN(tsit5_bTheta)(Th, bw);
                for (int k = 0; k < d; ++k) {
                    REAL acc = 0;
                    for (int i = 0; i < 7; ++i) acc += bw[i] * ks[(size_t)i * d + k];
                    out[(size_t)isave * d + k] = u[k] + h * acc;
                }
                ++isave;
            }
            qold = EEst > (REAL)1e-4 ? EEst : (REAL)1e-4;
            /* qsteady_min = qsteady_max = 1 for explicit RK methods (OrdinaryDiffEq defaults; 6/5 is the implicit-solver band): no dead band */
            if (!clipped || h >= dt) dt = h / q;
            else { const REAL prop = h / q; if (prop > dt) dt = prop; }
            t = tn;
            ++nacc;
            tgrid[nacc] = t;
            for (int k = 0; k < d; ++k) { u[k] = un[k]; ustep[(size_t)nacc * d + k] = u[k]; }
            memcpy(kf, ks + (size_t)(s - 1) * d, sizeof(REAL) * d);
        } else {
            REAL qr = q11 / gamma;
            if (qr > (REAL)1 / qmin) qr = (REAL)1 / qmin;
            dt = h / qr;
            memcpy(kf, ks, sizeof(REAL) * d);
        }
    }
    return isave == n_save ? nacc : -1;
}

/* u(t) from the recorded dense output; *hint is the last step index used (monotone search) */
static void FN(dense_eval)(const REAL *tgrid, const REAL *ustep, const REAL *dense, int nacc, int d, REAL t,
                           int *hint, REAL *uu)
{
    int n = *hint;
    if (n < 0) n = 0;
    if (n >= nacc) n = nacc - 1;
    while (n > 0 && t < tgrid[n]) --n;
    while (n < nacc - 1 && t > tgrid[n + 1]) ++n;
    *hint = n;
    const REAL h = tgrid[n + 1] - tgrid[n];
    REAL Th = (t - tgrid[n]) / h, bw[7];
    if (Th < 0) Th = 0;
    if (Th > 1) Th = 1;
    FN(tsit5_bTheta)(Th, bw);
    const REAL *ks = dense + (size_t)n * 7 * d;
    for (int k = 0; k < d; ++k) {
        REAL acc = 0;
        for (int j = 0; j < 7; ++j) acc += bw[j] * ks[(size_t)j * d + k];
        uu[k] = ustep[(size_t)n * d + k] + h * acc;
    }
}

/* Interpolating adjoint that REPLAYS the accepted forward steps backwards: each forward step
 * [t_n, t_n+1] is one backward Tsit5 step, split at the save times that fall strictly inside it (the
 * loss jumps are tstops of the backward solve).  This is what the GPU kernels do for adaptive solves;
 * ude_adjoint_adaptive below is the reference-style error-controlled backward solve it is checked against. */
void FN(ude_adjoint_replay)(const ude_model *m, const REAL *th, const REAL *saveat, int n_save,
                            const REAL *tgrid, const REAL *ustep, const REAL *dense, int nacc,
                            const REAL *dLdout, REAL *grad_theta, REAL *grad_u0)
{
    const ude_tableau *tb = ude_get_tableau(UDE_TSIT5);
    const int d = m->d;
    REAL lam[UDE_MAX_STATE], g[UDE_MAX_STATE], uu[UDE_MAX_STATE], kl[7 * UDE_MAX_STATE];
    int isave = n_save - 1;
    for (int k = 0; k < d; ++k) lam[k] = dLdout[(size_t)isave * d + k];
    --isave;
    for (int n = nacc - 1; n >= 0; --n) {
        const REAL tn = tgrid[n], tn1 = tgrid[n + 1], hn = tn1 - tn;
        const REAL *ks = dense + (size_t)n * 7 * d;
        const REAL eps = (REAL)1e-6 * hn;
        REAL cur = tn1;
        while (cur > tn + eps) {
            REAL ta = tn;
            if (isave >= 0 && saveat[isave] > tn + eps) ta = saveat[isave];
            const REAL h = cur - ta;
            for (int i = 0; i < 6; ++i) {
                REAL Th = (cur - (REAL)tb->c[i] * h - tn) / hn, bw[7];
                if (Th < 0) Th = 0;
                if (Th > 1) Th = 1;
                FN(tsit5_bTheta)(Th, bw);
                for (int k = 0; k < d; ++k) {
                    REAL acc = 0;
                    for (int j = 0; j < 7; ++j) acc += bw[j] * ks[(size_t)j * d + k];
                    uu[k] = ustep[(size_t)n * d + k] + hn * acc;
                }
                for (int k = 0; k < d; ++k) {
                    REAL acc = 0;
                    for (int j = 0; j < i; ++j) {
                        const REAL a = (REAL)tb->A[i][j];
                        if (a != 0) acc += a * kl[(size_t)j * d + k];
                    }
                    g[k] = lam[k] + h * acc;
                }
                FN(ude_rhs_vjp)(m, th, uu, g, kl + (size_t)i * d, grad_theta, h * (REAL)tb->A[6][i]);
            }
            for (int k = 0; k < d; ++k) {
                REAL acc = 0;
                for (int j = 0; j < 6; ++j) acc += (REAL)tb->A[6][j] * kl[(size_t)j * d + k];
                lam[k] += h * acc;
            }
            cur = ta;
            if (isave >= 0 && R_FABS(saveat[isave] - ta) <= eps) {
                for (int k = 0; k < d; ++k) lam[k] += dLdout[(size_t)isave * d + k];
                --isave;
            }
        }
    }
    for (int k = 0; k < d; ++k) grad_u0[k] = lam[k];
}

/* Reference-style backward solve: the augmented state [lambda; mu] (d + P entries) is integrated from T to t0
 * with adaptive Tsit5 (same tolerances, PI controller, error norm over all d + P components), tstops at the
 * save times where dL/du(t_i) is added to lambda; u(t) from the forward dense output.  grad_theta is SET. */
int FN(ude_adjoint_adaptive)(const ude_model *m, const REAL *th, const REAL *saveat, int n_save,
                             const REAL *tgrid, const REAL *ustep, const REAL *dense, int nacc,
                             const REAL *dLdout, REAL abstol, REAL reltol, REAL *grad_theta, REAL *grad_u0)
{
    const ude_tableau *tb = ude_get_tableau(UDE_TSIT5);
    const int d = m->d, order = 5;
    const size_t P = ude_num_params(m), S = (size_t)d + P;
    const REAL gamma = (REAL)0.9, qmin = (REAL)0.2, qmax = (REAL)10;
    const REAL beta2 = (REAL)2 / ((REAL)5 * order), beta1 = (REAL)7 / ((REAL)10 * order);
    REAL qold = (REAL)1e-4;
    REAL *y = (REAL *)calloc(S, sizeof(REAL)), *yn = (REAL *)calloc(S, sizeof(REAL));
    REAL *K = (REAL *)calloc(7 * S, sizeof(REAL)), *gs = (REAL *)calloc(S, sizeof(REAL));
    REAL uu[UDE_MAX_STATE];
    int hint = nacc - 1, isave = n_save - 1, nsteps = 0;
    for (int k = 0; k < d; ++k) y[k] = dLdout[(size_t)isave * d + k];
    --isave;
    REAL t = saveat[n_save - 1];
    REAL dt = (saveat[n_save - 1] - saveat[0]) * (REAL)0.01;   /* backward step magnitude */
    int have_k1 = 0;
    while (isave >= 0) {
        const REAL tstop = saveat[isave];
        REAL h = dt;
        int clipped = 0;
        if (t - h <= tstop + (REAL)1e-7 * R_FABS(tstop)) { h = t - tstop; clipped = 1; }
        /* stages in reverse time: y' = +F(y, t - c h) with F = [J_u^T lam; J_theta^T lam] */
        for (int i = 0; i < 7; ++i) {
            if (i == 0 && have_k1) continue;
            for (size_t q = 0; q < S; ++q) {
                REAL acc = 0;
                for (int j = 0; j < i; ++j) {
                    const REAL a = (REAL)tb->A[i][j];
                    if (a != 0) acc += a * K[(size_t)j * S + q];
                }
                gs[q] = y[q] + h * acc;
            }
            FN(dense_eval)(tgrid, ustep, dense, nacc, d, t - (REAL)tb->c[i] * h, &hint, uu);
            REAL *Ki = K + (size_t)i * S;
            for (size_t q = d; q < S; ++q) Ki[q] = 0;
            FN(ude_rhs_vjp)(m, th, uu, gs, Ki, Ki + d, (REAL)1);
            if (i == 5) for (size_t q = 0; q < S; ++q) {   /* y_new = stage-7 argument (row 7 = b) */
                REAL acc = 0;
                for (int j = 0; j < 6; ++j) acc += (REAL)tb->A[6][j] * K[(size_t)j * S + q];
                yn[q] = y[q] + h * acc;
            }
        }
        REAL ee = 0;
        for (size_t q = 0; q < S; ++q) {
            REAL e = 0;
            for (int j = 0; j < 7; ++j) e += (REAL)tb->bt[j] * K[(size_t)j * S + q];
            e *= h;
            const REAL a = R_FABS(y[q]), b = R_FABS(yn[q]);
            const REAL sc = abstol + reltol * (a > b ? a : b);
            ee += (e / sc) * (e / sc);
        }
        const REAL EEst = R_SQRT(ee / (REAL)S);
        if (!isfinite((double)EEst) || ++nsteps > 10000000) { free(y); free(yn); free(K); free(gs); return -1; }
        const REAL q11 = R_POW(EEst, beta1);
        REAL q = q11 / R_POW(qold, beta2) / gamma;
        if (q < (REAL)1 / qmax) q = (REAL)1 / qmax;
        if (q > (REAL)1 / qmin) q = (REAL)1 / qmin;
        if (EEst <= (REAL)1) {
            qold = EEst > (REAL)1e-4 ? EEst : (REAL)1e-4;
            /* qsteady_min = qsteady_max = 1 for explicit RK methods (OrdinaryDiffEq defaults; 6/5 is the implicit-solver band): no dead band */
            if (!clipped || h >= dt) dt = h / q;
            else { const REAL prop = h / q; if (prop > dt) dt = prop; }
            t = clipped ? tstop : t - h;
            for (size_t qq = 0; qq < S; ++qq) y[qq] = yn[qq];
            memcpy(K, K + 6 * S, sizeof(REAL) * S);   /* FSAL */
            have_k1 = 1;
            if (clipped) {
                for (int k = 0; k < d; ++k) y[k] += dLdout[(size_t)isave * d + k];
                --isave;
                have_k1 = 0;                          /* the jump invalidates FSAL */
            }
        } else {
            REAL qr = q11 / gamma;
            if (qr > (REAL)1 / qmin) qr = (REAL)1 / qmin;
            dt = h / qr;
            have_k1 = 1;                              /* K[0] is still F(y, t) */
        }
    }
    for (int k = 0; k < d; ++k) grad_u0[k] = y[k];
    for (size_t q = 0; q < P; ++q) grad_theta[q] = y[d + q];
    free(y); free(yn); free(K); free(gs);
    return nsteps;
}

double FN(ude_ensemble_loss_grad)(const ude_model *m, const REAL *th, const REAL *u0, const REAL *y,
                                  const REAL *wmask, size_t N, REAL dt, int n_steps, int save_every,
                                  REAL *out, REAL *grad_theta, REAL *grad_u0, int n_threads)
{
    const int d = m->d;
    const int n_save = n_steps / save_every + 1;
    const size_t P = ude_num_params(m);
    double loss = 0;
    if (n_threads < 1) n_threads = 1;
    REAL *gpart = (REAL *)calloc((size_t)n_threads * P, sizeof(REAL));
#ifdef _OPENMP
#pragma omp parallel num_threads(n_threads) reduction(+ : loss)
#endif
    {
#ifdef _OPENMP
        const int tid = omp_get_thread_num();
#else
        const int tid = 0;
#endif
        REAL *gt = gpart + (size_t)tid * P;
        REAL *o = (REAL *)malloc(sizeof(REAL) * (size_t)n_save * d);
        REAL *dl = (REAL *)malloc(sizeof(REAL) * (size_t)n_save * d);
        REAL *dense = (REAL *)malloc(sizeof(REAL) * (size_t)n_steps * 7 * d);
        REAL u[UDE_MAX_STATE], gu[UDE_MAX_STATE];
#ifdef _OPENMP
#pragma omp for schedule(static)
#endif
        for (long long n = 0; n < (long long)N; ++n) {
            for (int k = 0; k < d; ++k) u[k] = u0[(size_t)k * N + n];
            FN(ude_solve_fixed)(m, th, u, dt, n_steps, UDE_TSIT5, save_every, o, dense);
            for (int i = 0; i < n_save; ++i)
                for (int k = 0; k < d; ++k) {
                    const size_t idx = ((size_t)i * d + k) * N + n;
                    const REAL r = o[(size_t)i * d + k] - y[idx];
                    loss += (double)(wmask[k] * r * r);
                    dl[(size_t)i * d + k] = (REAL)2 * wmask[k] * r;
                    if (out) out[idx] = o[(size_t)i * d + k];
                }
            FN(ude_adjoint_fixed)(m, th, o, dense, dt, n_steps, save_every, dl, gt, gu);
            if (grad_u0) for (int k = 0; k < d; ++k) grad_u0[(size_t)k * N + n] = gu[k];
        }
        free(o); free(dl); free(dense);
    }
    for (size_t p = 0; p < P; ++p) {
        double acc = 0;
        for (int t = 0; t < n_threads; ++t) acc += (double)gpart[(size_t)t * P + p];
        grad_theta[p] = (REAL)acc;
    }
    free(gpart);
    return loss;
}

#undef FN
#undef CAT
#undef CAT_
