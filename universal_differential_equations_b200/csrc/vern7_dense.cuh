// vern7_dense.cuh -- Vern7 with its lazy 7th-order dense output (B200UDE_FLAG_VERN7_DENSE): the adaptive forward that saves through
// the interpolant, and the interpolating adjoint over the Vern7 solve's own dense output, written once over the real type.
//
// The continuous extension is OrdinaryDiffEq's (Vern7ExtraStages / Vern7InterpolationCoefficients, serialized in the reference's
// Scenario_1_recovery_0.005.jld2 after the tableau; SURVEY.md App. A.3): six extra stages
//     k_i = f(u_n + h sum_j a_ij k_j),  i = 11..16  (k_11 = f(u_{n+1}) up to round-off),
// and u(t_n + theta h) = u_n + h sum_i b_i(theta) k_i over the 13 stages i in {1, 4..9, 11..16}; b_1 is a polynomial in theta of
// degree 7 without constant term, the others start at theta^2.  Stages 2, 3 and 10 carry no interpolation weight.
//
// Forward (adaptive): OrdinaryDiffEq's PI controller as in the tstops kernels, but the steps stop only at the end of tspan; a
// save time inside an accepted step is filled in from the interpolant (the extra stages are computed once for that step), a
// save time on the step end takes the step-end state.  The record is the discrete adjoint's: u_n of every accepted step,
// h_n, the step end times and the accepted count -- no stage store.  A fixed grid saves at step ends: its forward is the plain
// Vern7 kernel with the step record switched on.
//
// Adjoint (replay): the accepted steps backwards; per step the stages k_1..k_9 are recomputed from u_n and h_n with the forward's
// own expressions (bitwise the forward's) and the extra stages k_11..k_16 after them (stage 10 only feeds the error estimate).
// The step is split at the save times inside it, where the loss cotangent jumps into lambda; on each piece [t_a, t_b],
// h = t_b - t_a, lambda is stepped backwards with Vern7's 9 update stages,
//     g_i = lambda + h sum_{j<i} a_ij kl_j,   kl_i = J_u(x_i)^T g_i,   grad_theta += h b_i J_theta(x_i)^T g_i,
//     lambda += h sum_i b_i kl_i,
// with x_i = u(t_b - c_i h) from this step's interpolant.  One trajectory per thread; the gradient goes through the precision's
// warp_acc into a per-warp shared vector, one partial row per warp, fixed-order reduce: bitwise deterministic.  On an adaptive
// grid the warp loops over its longest record, shorter records shadow step 0 with zero weight, and every lane walks its own
// pieces with a warp-uniform trip count, so a trajectory's results do not depend on its neighbours.
//
// `Ops` is the precision of the runtime-shape model layer (ude_generic.cuh): k_generic.cu instantiates it in fp32 (Ops32),
// k_f64.cu in fp64 (Ops64).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ude_generic.cuh"
#include "vern7.cuh"

namespace b200ude {

// extra stages and interpolation polynomials of the lazy Vern7 dense output (OrdinaryDiffEq 6.19.2), bit-equal to the doubles
// the reference serialized (tests/test_vern7_dense_oracle.py parses this struct and compares)
struct Vern7Dense {
    // abscissae: the 9 update stages (0-based 0..8; stage 10, index 9, has c = 1 and is not used here) and the extra stages 10..15
    __host__ __device__ static constexpr double c(int i)
    {
        switch (i) {
        case 1: return 0.005;
        case 2: return 0.10888888888888888;
        case 3: return 0.16333333333333333;
        case 4: return 0.4555;
        case 5: return 0.6095094489978381;
        case 6: return 0.884;
        case 7: return 0.925;
        case 8: return 1.0;
        case 10: return 1.0;
        case 11: return 0.29;
        case 12: return 0.125;
        case 13: return 0.25;
        case 14: return 0.53;
        case 15: return 0.79;
        default: return 0.0;
        }
    }
    // a_ij of the extra stages (0-based rows 10..15); rows 0..9 are Vern7::a
    __host__ __device__ static constexpr double a(int i, int j)
    {
        switch (i * 16 + j) {
        case 10 * 16 + 0: return 0.04715561848627222;
        case 10 * 16 + 3: return 0.25750564298434153;
        case 10 * 16 + 4: return 0.2621665397741262;
        case 10 * 16 + 5: return 0.15216092656738558;
        case 10 * 16 + 6: return 0.49399691700324844;
        case 10 * 16 + 7: return -0.29430311714032503;
        case 10 * 16 + 8: return 0.0813174723249511;
        case 11 * 16 + 0: return 0.0523222769159969;
        case 11 * 16 + 3: return 0.22495861826705715;
        case 11 * 16 + 4: return 0.017443709248776376;
        case 11 * 16 + 5: return -0.007669379876829393;
        case 11 * 16 + 6: return 0.03435896044073285;
        case 11 * 16 + 7: return -0.0410209723009395;
        case 11 * 16 + 8: return 0.025651133005205617;
        case 11 * 16 + 10: return -0.0160443457;
        case 12 * 16 + 0: return 0.053053341257859085;
        case 12 * 16 + 3: return 0.12195301011401886;
        case 12 * 16 + 4: return 0.017746840737602496;
        case 12 * 16 + 5: return -0.0005928372667681495;
        case 12 * 16 + 6: return 0.008381833970853752;
        case 12 * 16 + 7: return -0.01293369259698612;
        case 12 * 16 + 8: return 0.009412056815253861;
        case 12 * 16 + 10: return -0.005353253107275676;
        case 12 * 16 + 11: return -0.06666729992455811;
        case 13 * 16 + 0: return 0.03887903257436304;
        case 13 * 16 + 3: return -0.0024403203308301317;
        case 13 * 16 + 4: return -0.0013928917214672623;
        case 13 * 16 + 5: return -0.00047446291558680135;
        case 13 * 16 + 6: return 0.00039207932413159514;
        case 13 * 16 + 7: return -0.00040554733285128004;
        case 13 * 16 + 8: return 0.00019897093147716726;
        case 13 * 16 + 10: return -0.00010278198793179169;
        case 13 * 16 + 11: return 0.03385661513870267;
        case 13 * 16 + 12: return 0.1814893063199928;
        case 14 * 16 + 0: return 0.05723681204690013;
        case 14 * 16 + 3: return 0.22265948066761182;
        case 14 * 16 + 4: return 0.12344864200186899;
        case 14 * 16 + 5: return 0.04006332526666491;
        case 14 * 16 + 6: return -0.05269894848581452;
        case 14 * 16 + 7: return 0.04765971214244523;
        case 14 * 16 + 8: return -0.02138895885042213;
        case 14 * 16 + 10: return 0.015193891064036402;
        case 14 * 16 + 11: return 0.12060546716289655;
        case 14 * 16 + 12: return -0.022779423016187374;
        case 15 * 16 + 0: return 0.051372038802756814;
        case 15 * 16 + 3: return 0.5414214473439406;
        case 15 * 16 + 4: return 0.350399806692184;
        case 15 * 16 + 5: return 0.14193112269692182;
        case 15 * 16 + 6: return 0.10527377478429423;
        case 15 * 16 + 7: return -0.031081847805874016;
        case 15 * 16 + 8: return -0.007401883149519145;
        case 15 * 16 + 10: return -0.006377932504865363;
        case 15 * 16 + 11: return -0.17325495908361865;
        case 15 * 16 + 12: return -0.18228156777622026;
        default: return 0.0;
        }
    }
    // b_i(theta) = sum_p r(i, p) theta^p: p = 1..7 for stage 0, p = 2..7 for stages 3..8 and 10..15
    __host__ __device__ static constexpr double r(int i, int p)
    {
        switch (i * 8 + p) {
        case 0 * 8 + 1: return 1.0;
        case 0 * 8 + 2: return -8.413387198332767;
        case 0 * 8 + 3: return 33.675508884490895;
        case 0 * 8 + 4: return -70.80159089484886;
        case 0 * 8 + 5: return 80.64695108301298;
        case 0 * 8 + 6: return -47.19413969837522;
        case 0 * 8 + 7: return 11.133813442539243;
        case 3 * 8 + 2: return 8.754921980674396;
        case 3 * 8 + 3: return -88.4596828699771;
        case 3 * 8 + 4: return 346.9017638429916;
        case 3 * 8 + 5: return -629.2580030059837;
        case 3 * 8 + 6: return 529.6773755604193;
        case 3 * 8 + 7: return -167.35886986514018;
        case 4 * 8 + 2: return 8.913387586637922;
        case 4 * 8 + 3: return -90.06081846893218;
        case 4 * 8 + 4: return 353.1807459217058;
        case 4 * 8 + 5: return -640.6476819744374;
        case 4 * 8 + 6: return 539.2646279047156;
        case 4 * 8 + 7: return -170.38809442991547;
        case 5 * 8 + 2: return 5.1733120298478;
        case 5 * 8 + 3: return -52.271115900055385;
        case 5 * 8 + 4: return 204.9853867374073;
        case 5 * 8 + 5: return -371.8306118563603;
        case 5 * 8 + 6: return 312.9880934374529;
        case 5 * 8 + 7: return -98.89290352172495;
        case 6 * 8 + 2: return 16.79537744079696;
        case 6 * 8 + 3: return -169.70040000059728;
        case 6 * 8 + 4: return 665.4937727009246;
        case 6 * 8 + 5: return -1207.1638892336007;
        case 6 * 8 + 6: return 1016.1291515818546;
        case 6 * 8 + 7: return -321.06001557237494;
        case 7 * 8 + 2: return -10.005997536098665;
        case 7 * 8 + 3: return 101.1005433052275;
        case 7 * 8 + 4: return -396.47391512378437;
        case 7 * 8 + 5: return 719.1787707014183;
        case 7 * 8 + 6: return -605.3681033918824;
        case 7 * 8 + 7: return 191.27439892797935;
        case 8 * 8 + 2: return 2.764708833638599;
        case 8 * 8 + 3: return -27.934602637390462;
        case 8 * 8 + 4: return 109.54779186137893;
        case 8 * 8 + 5: return -198.7128113064482;
        case 8 * 8 + 6: return 167.26633571640318;
        case 8 * 8 + 7: return -52.85010499525706;
        case 10 * 8 + 2: return -2.1696320280163506;
        case 10 * 8 + 3: return 22.016696037569876;
        case 10 * 8 + 4: return -86.90152427798948;
        case 10 * 8 + 5: return 159.22388973861476;
        case 10 * 8 + 6: return -135.9618306534588;
        case 10 * 8 + 7: return 43.792401183280006;
        case 11 * 8 + 2: return -4.890070188793804;
        case 11 * 8 + 3: return 22.75407737425176;
        case 11 * 8 + 4: return -30.78034218537731;
        case 11 * 8 + 5: return -2.797194317207249;
        case 11 * 8 + 6: return 31.369456637508403;
        case 11 * 8 + 7: return -15.655927320381801;
        case 12 * 8 + 2: return 10.862170929551967;
        case 12 * 8 + 3: return -50.542971417827104;
        case 12 * 8 + 4: return 68.37148040407511;
        case 12 * 8 + 5: return 6.213326521632409;
        case 12 * 8 + 6: return -69.68006323194157;
        case 12 * 8 + 7: return 34.776056794509195;
        case 13 * 8 + 2: return -11.37286691922923;
        case 13 * 8 + 3: return 130.79058078246717;
        case 13 * 8 + 4: return -488.65113677785604;
        case 13 * 8 + 5: return 832.2148793276441;
        case 13 * 8 + 6: return -664.7743368554426;
        case 13 * 8 + 7: return 201.79288044241662;
        case 14 * 8 + 2: return -5.919778732715007;
        case 14 * 8 + 3: return 63.27679965889219;
        case 14 * 8 + 4: return -265.432682088738;
        case 14 * 8 + 5: return 520.1009254140611;
        case 14 * 8 + 6: return -467.412109533902;
        case 14 * 8 + 7: return 155.3868452824017;
        case 15 * 8 + 2: return -10.492146197961823;
        case 15 * 8 + 3: return 105.35538525188011;
        case 15 * 8 + 4: return -409.43975011988937;
        case 15 * 8 + 5: return 732.831448907654;
        case 15 * 8 + 6: return -606.3044574733512;
        case 15 * 8 + 7: return 188.0495196316683;
        default: return 0.0;
        }
    }
    // stages with interpolation weight
    __host__ __device__ static constexpr bool weighted(int i) { return i == 0 || (i >= 3 && i <= 8) || i >= 10; }
};

namespace vern7_dense {

// the point stage i of a step from u with step h is evaluated at: g = u + h sum_j a_ij k_j (the expression of the Vern7 forward
// kernels)
template <class Ops, int I>
__device__ __forceinline__ void stage_point(const typename Ops::real *u, typename Ops::real h, const typename Ops::real (*k)[Ops::MAXD],
                                            typename Ops::real *g)
{
    using R = typename Ops::real;
    const int D = Ops::D();
    for (int c = 0; c < D; ++c) {
        R acc = (R)0;
#pragma unroll
        for (int j = 0; j < I; ++j) {
            constexpr bool ext = I >= 10;
            const double aij = ext ? Vern7Dense::a(I, j) : Vern7::a(I, j);
            if (aij != 0.0) acc = fma((R)aij, k[j][c], acc);
        }
        g[c] = fma(h, acc, u[c]);
    }
}

// stage i of a step from u with step h: k_i = f(g), g its stage point
template <class Ops, int I>
__device__ __forceinline__ void stage(const typename Ops::real *u, typename Ops::real h, typename Ops::real (*k)[Ops::MAXD],
                                      typename Ops::real *g)
{
    stage_point<Ops, I>(u, h, k, g);
    generic::model_rhs<Ops>(g, k[I]);
}

// the extra stages k_11..k_16 (indices 10..15) of a step whose k_1..k_9 are in k
template <class Ops>
__device__ __forceinline__ void extra_stages(const typename Ops::real *u, typename Ops::real h, typename Ops::real (*k)[Ops::MAXD],
                                             typename Ops::real *g)
{
    stage<Ops, 10>(u, h, k, g);
    stage<Ops, 11>(u, h, k, g);
    stage<Ops, 12>(u, h, k, g);
    stage<Ops, 13>(u, h, k, g);
    stage<Ops, 14>(u, h, k, g);
    stage<Ops, 15>(u, h, k, g);
}

// the interpolation weights b_i(th), i = 0..15, by Horner (zero for the stages without weight)
template <typename R>
__device__ __forceinline__ void interp_weights(R th, R *bw)
{
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (!Vern7Dense::weighted(i)) { bw[i] = (R)0; continue; }
        R acc = (R)Vern7Dense::r(i, 7);
#pragma unroll
        for (int q = 6; q >= 2; --q) acc = fma(acc, th, (R)Vern7Dense::r(i, q));
        bw[i] = i == 0 ? th * fma(acc, th, (R)Vern7Dense::r(0, 1)) : th * th * acc;
    }
}

// x = u(t_n + th h) = u + h sum_i b_i(th) k_i
template <class Ops>
__device__ __forceinline__ void interpolate(const typename Ops::real *u, typename Ops::real h, const typename Ops::real (*k)[Ops::MAXD],
                                            typename Ops::real th, typename Ops::real *x)
{
    using R = typename Ops::real;
    R bw[16];
    interp_weights<R>(th, bw);
    const int D = Ops::D();
    for (int c = 0; c < D; ++c) {
        R acc = (R)0;
#pragma unroll
        for (int i = 0; i < 16; ++i)
            if (Vern7Dense::weighted(i)) acc = fma(bw[i], k[i][c], acc);
        x[c] = fma(h, acc, u[c]);
    }
}

template <typename R>
struct Fwd {
    const R *u0;        // [D][N]
    R *out;             // [n_save][D][N]
    R *ustep;           // [max_steps+1][D][N]  u_n of every accepted step
    R *tgrid;           // [max_steps+1][N]     step end times (t0 first)
    R *hstep;           // [max_steps][N]       the step sizes the forward used
    int *nacc;          // [N]
    int32_t *status;    // [N] or nullptr
    int N, n_save, max_steps;
    R t0, save_dt, abstol, reltol;
};

// adaptive Vern7 with OrdinaryDiffEq's PI controller (PIControl<R, 7>), steps clipped at the end of tspan only,
// saveat by the interpolant
template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) forward_kernel(Fwd<typename Ops::real> p)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    constexpr int MAXD = Ops::MAXD;
    const int D = Ops::D();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const R t0 = p.t0, t1 = p.t0 + p.save_dt * (R)(p.n_save - 1);
    const R abstol = p.abstol, reltol = p.reltol;
    R u[MAXD], un[MAXD], g[MAXD], k[16][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    for (int c = 0; c < D; ++c) {
        p.out[(size_t)c * N + n] = u[c];
        p.ustep[(size_t)c * N + n] = u[c];
    }
    p.tgrid[n] = t0;
    generic::model_rhs<Ops>(u, k[0]);
    PIControl<R, 7> pi;
    {   // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
        R d0 = 0, d1 = 0, d2 = 0;
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = PR::sq(d0 / D); d1 = PR::sq(d1 / D);
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fma(dt0, k[0][c], u[c]);
        generic::model_rhs<Ops>(g, un);
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            const R e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = PR::sq(d2 / D) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    R t = t0;
    int nacc = 0, isave = 1, bad = 0;
    bool have_k1 = true;
    while (isave < p.n_save) {
        R h = pi.dt;
        bool clipped = false;
        if (t + h >= t1 - PR::clip * fabs(t1)) { h = t1 - t; clipped = true; }
        if (!have_k1) generic::model_rhs<Ops>(u, k[0]);
        stage<Ops, 1>(u, h, k, g);
        stage<Ops, 2>(u, h, k, g);
        stage<Ops, 3>(u, h, k, g);
        stage<Ops, 4>(u, h, k, g);
        stage<Ops, 5>(u, h, k, g);
        stage<Ops, 6>(u, h, k, g);
        stage<Ops, 7>(u, h, k, g);
        stage<Ops, 8>(u, h, k, g);
        stage<Ops, 9>(u, h, k, g);
        R ee = 0;
        for (int c = 0; c < D; ++c) {
            R acc = 0, e = 0;
#pragma unroll
            for (int j = 0; j < 10; ++j) {
                if (Vern7::b(j) != 0.0) acc = fma((R)Vern7::b(j), k[j][c], acc);
                if (Vern7::bt(j) != 0.0) e = fma((R)Vern7::bt(j), k[j][c], e);
            }
            un[c] = fma(h, acc, u[c]);
            e *= h;
            const R sc = abstol + reltol * fmax(fabs(u[c]), fabs(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const R EEst = PR::sq(ee / D);
        if (!(EEst <= PR::huge)) { bad = 1; break; }
        if (pi.judge(EEst)) {
            if (nacc >= p.max_steps) { bad = 2; break; }
            const R tn = clipped ? t1 : t + h;
            const R eps = PR::eta * (tn - t);
            bool ext = false;
            while (isave < p.n_save) {
                const R ts = t0 + p.save_dt * (R)isave;
                if (ts > tn + eps) break;
                R *dst = p.out + (size_t)isave * D * N + n;
                if (ts >= tn - eps) {   // on the step end
                    for (int c = 0; c < D; ++c) dst[(size_t)c * N] = un[c];
                } else {
                    if (!ext) { extra_stages<Ops>(u, h, k, g); ext = true; }
                    interpolate<Ops>(u, h, k, (ts - t) / h, g);
                    for (int c = 0; c < D; ++c) dst[(size_t)c * N] = g[c];
                }
                ++isave;
            }
            p.hstep[(size_t)nacc * N + n] = h;
            ++nacc;
            pi.accept(EEst, h, clipped);
            t = tn;
            p.tgrid[(size_t)nacc * N + n] = t;
            for (int c = 0; c < D; ++c) {
                u[c] = un[c];
                p.ustep[((size_t)nacc * D + c) * N + n] = un[c];
            }
            have_k1 = false;   // not FSAL
        } else {
            pi.reject(h);
            have_k1 = true;    // k_1 = f(u) is still valid after a rejection
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        for (int is = isave; is < p.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = PR::nan();
    }
    p.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

template <typename R>
struct Adj {
    const R *ustep;     // [steps+1][D][N]
    const R *tgrid;     // adaptive: [max_steps+1][N]; nullptr = fixed step
    const R *hstep;     // adaptive: [max_steps][N]
    const int *nacc;    // adaptive: [N]
    const R *cot;       // fused_l2 ? data : dL/dout, [n_save][D][N]
    const R *saved;     // adaptive fused_l2: the saved states the forward returned, [n_save][D][N]
    R *grad_u0;         // [D][N] or nullptr
    R *partial;         // [gridDim.x * BLOCK/32][P+1], last entry = partial loss
    int N, n_steps, save_every, n_save, fused_l2;
    R dt, t0, save_dt;
};

template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(Adj<typename Ops::real> p)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    constexpr int MAXD = Ops::MAXD;
    extern __shared__ __align__(16) unsigned char s_raw[];
    R *s_g = reinterpret_cast<R *>(s_raw);   // [BLOCK/32][P+1]
    const int D = Ops::D(), P = Ops::P();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    R *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = (R)0;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const bool adaptive = p.tgrid != nullptr;
    const int nst = adaptive ? p.nacc[n] : p.n_steps;   // this trajectory's steps
    int nmax = live ? nst : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    R lam[MAXD], u[MAXD], x[MAXD], g[MAXD], k[16][MAXD], kl[9][MAXD];
    R loss = (R)0;
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    // loss cotangent of save point `is` (fused L2: 2 w (u - data) of the state the forward saved there)
    auto jump = [&](int is) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)is * D + c) * N + n;
            if (p.fused_l2) {
                const R us = adaptive ? p.saved[idx] : p.ustep[((size_t)is * p.save_every * D + c) * N + n];
                const R r = us - p.cot[idx];
                const R wgt = Ops::lossw(c);
                loss = fma(wgt * r, r, loss);
                lam[c] = fma((R)2 * wgt, r, lam[c]);
            } else {
                lam[c] += p.cot[idx];
            }
        }
    };
    auto save_time = [&](int is) { return p.t0 + p.save_dt * (R)is; };
    int isave = p.n_save - 1;
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act = live && s < nst;
        const int sr = act ? s : 0;   // inactive lanes shadow step 0 (finite data) with zero weight
        const R h = adaptive ? p.hstep[(size_t)sr * N + n] : p.dt;
        const R tn = adaptive ? p.tgrid[(size_t)sr * N + n] : (R)0;
        const R tn1 = adaptive ? p.tgrid[(size_t)(sr + 1) * N + n] : p.dt;
        const R eps = PR::eta * (tn1 - tn);
        for (int c = 0; c < D; ++c) u[c] = p.ustep[((size_t)sr * D + c) * N + n];
        // k_1..k_9 as the forward evaluated them, then the extra stages
        generic::model_rhs<Ops>(u, k[0]);
        stage<Ops, 1>(u, h, k, g);
        stage<Ops, 2>(u, h, k, g);
        stage<Ops, 3>(u, h, k, g);
        stage<Ops, 4>(u, h, k, g);
        stage<Ops, 5>(u, h, k, g);
        stage<Ops, 6>(u, h, k, g);
        stage<Ops, 7>(u, h, k, g);
        stage<Ops, 8>(u, h, k, g);
        extra_stages<Ops>(u, h, k, g);
        R cur = tn1;
        bool top = true;
        while (true) {
            // the cotangents of the save points at cur (adaptive: also those the solve never reached, past its last step end)
            if (act) {
                if (adaptive) {
                    while (isave >= 0 && save_time(isave) >= cur - eps) { jump(isave); --isave; }
                } else if (top && (s + 1) % p.save_every == 0) {
                    jump(isave); --isave;
                }
            }
            top = false;
            const bool has = act && cur > tn + eps;
            if (!__any_sync(0xffffffffu, has)) break;
            R ta = tn;   // the piece [ta, cur]: down to the next save time inside the step, else to the step start
            if (adaptive && has && isave >= 0) {
                const R ts = save_time(isave);
                if (ts > tn + eps) ta = ts;
            }
            const R hs = has ? cur - ta : (R)0;
#pragma unroll
            for (int i = 0; i < 9; ++i) {
                const R th = fmin(fmax((cur - (R)Vern7Dense::c(i) * hs - tn) / h, (R)0), (R)1);
                interpolate<Ops>(u, h, k, th, x);
                for (int c = 0; c < D; ++c) {
                    R a2 = (R)0;
#pragma unroll
                    for (int j = 0; j < i; ++j)
                        if (Vern7::a(i, j) != 0.0) a2 = fma((R)Vern7::a(i, j), kl[j][c], a2);
                    g[c] = fma(hs, a2, lam[c]);
                }
                generic::model_vjp<Ops>(x, g, hs * (R)Vern7::b(i), has ? (R)1 : (R)0, kl[i], gw, lane);
            }
            if (has) {
                for (int c = 0; c < D; ++c) {
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 9; ++j)
                        if (Vern7::b(j) != 0.0) acc = fma((R)Vern7::b(j), kl[j][c], acc);
                    lam[c] = fma(hs, acc, lam[c]);
                }
                cur = ta;
            }
        }
    }
    if (live)
        while (isave >= 0) { jump(isave); --isave; }   // t0 (and, after a solve that failed at once, every save point)
    if (p.grad_u0 && live)
        for (int c = 0; c < D; ++c) p.grad_u0[(size_t)c * N + n] = lam[c];
    loss *= live ? (R)1 : (R)0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) gw[P] = loss;
    __syncwarp();
    R *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

}  // namespace vern7_dense
}  // namespace b200ude
