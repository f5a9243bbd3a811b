// b200ude.cu -- C-ABI entry points (include/b200ude.h) over the sm_90a kernels.
//
// No torch types, no exceptions across the boundary, no CPU fallback: if there is no usable
// CUDA device, or the requested configuration has no kernel, the call fails with a code and a
// message.  Nothing here includes or links the CPU oracle.
#include "../../include/b200ude.h"

#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <algorithm>
#include <atomic>
#include <string>
#include <type_traits>
#include <vector>

#include "params.h"

using namespace b200ude;

namespace {

thread_local std::string g_create_error;

// The route of a handle: the forward / adjoint kernel pair it runs, chosen once by resolve() at create.  The forward, the adjoint,
// the Tsit5 re-solve, num_params, partial_rows and the buffers of create read the route, not the descriptor's model, solver or
// flag bits; within a route the dtype, fixed or adaptive stepping and the ensemble size are data the launchers take.  Routes
// marked fp32 are fp32 only; the others take both dtypes.
//   R_LV32            LV 2 -> 32 -> 32 -> 2 tanh, fixed-step Tsit5, interpolating adjoint (fp32)             BASELINE config 2
//                     (k_lv32_*.cu): warp-collective or one trajectory per thread, chosen per call from the ensemble size
//   R_LV32_DISCRETE   the same forward, the discrete adjoint on one trajectory per thread (fp32)
//   R_LV32_ADAPTIVE   adaptive Tsit5: tensor-core kernels with CTA-uniform attempt loops (fp32)
//   R_LV5             LV 2 -> 5 -> 5 -> 5 -> 2, per-layer activations, n_prefix = 0, 1, 2 trainable linear rates (k_lv5.cu):
//                     scenario_1.jl:62-73, scenario_2.jl:79-98, hudson_bay.jl:77-91; fixed-step Tsit5, either adjoint (fp32)
//   R_SEIR64          SEIR exposure UDE 3 -> 64 -> 64 -> 1 tanh, tensor-core kernels (k_seir.cu), fixed-step Tsit5 (fp32)   BASELINE config 3
//   R_SEIR64_VERN7    its fixed-step Vern7; the interpolating adjoint runs over a Tsit5 re-solve, launched by the first adjoint (fp32)
//   R_SEIR64_ADAPTIVE its adaptive Tsit5, CTA-uniform attempt loops (fp32)
//   R_FKPP_FIXED      Fisher-KPP UPDE: pointwise chain 1 -> ... -> 1 + 3-tap periodic stencil (Fisher-KPP-CNN.jl:111-126), fixed-step
//                     Tsit5 (fp32)
//   R_FKPP16          Fisher-KPP with the 1 -> 16 -> 16 -> 1 tanh reaction chain (k_fkpp.cu), fixed-step Tsit5 (fp32)   BASELINE config 4
//   R_FKPP16_RKC2     the same chain on even grids, fixed-step RKC2 (fp32)
//   R_FKPP_ADAPTIVE   Fisher-KPP adaptive Tsit5, grid per CTA, any chain (fkpp_adaptive.cuh), full step record
//   R_FKPP_CHECKPOINT the same with B200UDE_FLAG_CHECKPOINT: u_n every `seg` accepted steps and the step sizes
//   R_FKPP_VERN7_DISCRETE  Fisher-KPP adaptive Vern7 with the discrete adjoint (fkpp_vern7_discrete.cuh)
//   runtime-shape kernels (RuntimeShape<R>: k_generic.cu fp32, k_f64.cu fp64): any LV / SEIR / SEIR_NODE / NODE form with chain
//   widths <= 64 and <= 5 layers, fixed step or adaptive -- functional coverage (seir_exposure.jl:52-64,114-130 shapes), not tuned
//   R_TSIT5           Tsit5, interpolating adjoint
//   R_VERN7           Vern7; the interpolating adjoint runs over a Tsit5 re-solve from the same u0, launched by the first adjoint
//   R_DISCRETE_TSIT5  fixed-step Tsit5, discrete adjoint (discrete_adjoint.cuh)
//   R_DISCRETE_VERN7  Vern7, discrete adjoint; saves at step ends (B200UDE_FLAG_DISCRETE_DENSE on a fixed grid lands here too)
//   R_VERN7_DENSE     Vern7 with its lazy dense output, interpolating adjoint over it (vern7_dense.cuh; B200UDE_FLAG_VERN7_DENSE)
//   R_VERN7_DENSE_DISCRETE  adaptive Vern7 saving through its interpolant, discrete adjoint through it (vern7_dense_discrete.cuh;
//                     B200UDE_FLAG_DISCRETE_DENSE)
//   R_FORCED          forced neural ODE with a readout network (FENEP.jl:41-62) (k_forced.cu), Tsit5
//   R_OPERATOR        wide-state operator UDE du = D1 NN(u) + D2 u (npde.jl:75-78), warp per trajectory (k_operator.cu), Tsit5 or RKC2
enum Route {
    R_LV32, R_LV32_DISCRETE, R_LV32_ADAPTIVE, R_LV5, R_SEIR64, R_SEIR64_VERN7, R_SEIR64_ADAPTIVE, R_FKPP_FIXED, R_FKPP16, R_FKPP16_RKC2,
    R_FKPP_ADAPTIVE, R_FKPP_CHECKPOINT, R_FKPP_VERN7_DISCRETE, R_TSIT5, R_VERN7, R_DISCRETE_TSIT5, R_DISCRETE_VERN7, R_VERN7_DENSE,
    R_VERN7_DENSE_DISCRETE, R_FORCED, R_OPERATOR
};

// parameters of a handle: the tuned chains' fixed counts, else n_prefix + the dense layers + n_suffix.  The forced model's f0 and f1
// lie back to back in `widths`: its layers l >= L0 read one entry further on
int num_params(const b200ude_desc *d, Route r)
{
    switch (r) {
    case R_LV32: case R_LV32_DISCRETE: case R_LV32_ADAPTIVE: return 2 * 32 + 32 + 32 * 32 + 32 + 32 * 2 + 2;
    case R_SEIR64: case R_SEIR64_VERN7: case R_SEIR64_ADAPTIVE: return 3 * 64 + 64 + 64 * 64 + 64 + 64 + 1;
    case R_FKPP16: case R_FKPP16_RKC2: return 16 + 16 + 256 + 16 + 16 + 1 + 5;
    case R_LV5: return 87 + d->n_prefix;
    default: break;
    }
    const int L0 = r == R_FORCED ? (int)d->consts[0] : d->n_layers;
    int P = d->n_prefix + d->n_suffix;
    for (int l = 0; l < d->n_layers; ++l) {
        const int a = l < L0 ? l : l + 1;
        P += d->widths[a] * d->widths[a + 1] + d->widths[a + 1];
    }
    return P;
}

std::atomic<uint64_t> g_serial{0};   // handles may be created from several host threads (one per GPU)

}  // namespace

struct b200ude_handle {
    b200ude_desc desc;
    Route route = R_TSIT5;
    bool f64 = false;   // dtype = B200UDE_F64: every real-valued device array of the handle and of the callers is double
    Variant var;
    ConstTables tab;    // fp32 runtime-shape and tuned kernels
    Tables64 tab64;     // fp64 runtime-shape kernels
    GenericShape gen;
    int P = 0, n_save = 0, D = 0;
    int DR = 0;      // rows per save of out / data / dL_dout: D, or D + r for the forced model
    size_t cap = 0;  // max trajectories
    size_t N = 0;    // trajectories of the last forward
    bool have_forward = false;
    bool have_theta = false;
    int sm_count = 0;
    size_t wm_fwd_max = 0, wm_adj_max = 0;   // largest ensembles the warp-collective LV kernels are chosen for (auto mode)
    // device buffers of the handle's real type (es() bytes per element)
    void *d_theta = nullptr;
    void *d_ustep = nullptr;
    void *d_dense = nullptr;
    void *d_partial = nullptr;
    size_t partial_blocks = 0;
    // adaptive stepping
    bool adaptive = false;
    void *d_tgrid = nullptr, *d_cot = nullptr;
    void *d_hstep = nullptr;   // discrete-adjoint Vern7, checkpointed Fisher-KPP: step sizes of the accepted steps
    int seg = 0;               // R_FKPP_CHECKPOINT: accepted steps per checkpoint (d_ustep: checkpoints, d_dense: scratch), else 0
    float *d_block_loss = nullptr;
    int *d_nacc = nullptr;
    const void *last_out = nullptr;
    // host-buffer path
    float *d_u0 = nullptr, *d_out = nullptr, *d_data = nullptr, *d_gu0 = nullptr, *d_grad = nullptr, *d_loss = nullptr;
    int32_t *d_status = nullptr;
    float *h_loss = nullptr;  // pinned
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;   // host-buffer path: the data upload overlaps the forward kernel
    cudaEvent_t data_ready = nullptr, data_ready2 = nullptr;
    RkcHost rkc;                    // R_FKPP16_RKC2: recurrence tables for desc.n_stages
    // fused reduce + all-reduce over NVLink peer memory (b200ude_peer_*)
    void *d_peer_buf = nullptr;     // this rank's exchange buffer (cudaMalloc, exported with CUDA IPC)
    PeerLinks peer;                 // every rank's buffer as mapped here
    bool peer_attached = false;
    // on-device optimiser (b200ude_adam_*, b200ude_train_adam)
    void *d_u0_keep = nullptr, *d_aux_out = nullptr;   // Vern7: u0 of the last forward, saved states of the Tsit5 re-solve
    bool vern7_pending = false;   // R_VERN7, R_SEIR64_VERN7: the Tsit5 re-solve the adjoint runs over is still to be launched
    float *d_adam_m = nullptr, *d_adam_v = nullptr, *d_train_out = nullptr;
    int *d_adam_t = nullptr;
    int adam_t = 0;   // host mirror of the step counter
    // forced neural ODE (R_FORCED): shape, the forcing coefficients [3J][cap], the last forward's out
    ForcedHost fh{};
    void *d_forcing = nullptr;
    size_t forcing_n = 0;   // trajectories of the last b200ude_set_forcing
    void *d_usave = nullptr;   // adaptive: the saved states of the last forward [n_save][D][cap], read by the replay adjoint
    // operator UDE (R_OPERATOR): shape, the padded operator block, the RKC2 tables (handle dtype); it shares d_usave (as
    // [n_save][cap][D]) and the record buffers with the forced model
    bool ops_set = false;
    OperatorHost oh{};
    void *d_ops = nullptr, *d_rkc = nullptr;
    int *d_sstep = nullptr;   // adaptive RKC2: the stage count of each accepted step [max_steps][cap]
    size_t dev_bytes = 0;
    std::string err;
    size_t es() const { return f64 ? sizeof(double) : sizeof(float); }
};

namespace {

int32_t fail(b200ude_handle *h, int32_t code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf;
    else g_create_error = buf;
    return code;
}

#define CUDA_TRY(h, expr)                                                                                \
    do {                                                                                                 \
        cudaError_t e_ = (expr);                                                                         \
        if (e_ != cudaSuccess) {                                                                         \
            return fail((h), (int32_t)e_, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
        }                                                                                                \
    } while (0)

cudaError_t dalloc_bytes(b200ude_handle *h, void **p, size_t bytes)
{
    cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) h->dev_bytes += bytes;
    return e;
}

template <class T>
cudaError_t dalloc(b200ude_handle *h, T **p, size_t count)
{
    return dalloc_bytes(h, (void **)p, count * sizeof(T));
}

// count elements of the handle's real type
cudaError_t dalloc_real(b200ude_handle *h, void **p, size_t count) { return dalloc_bytes(h, p, count * h->es()); }

// RKC2 (Sommeijer, Shampine, Verwer 1998) recurrence coefficients, stage abscissae and the quadrature weights of the stage
// integrands (from running the recurrence on unit impulses)
// in double: mt1, then mu, nu, mt, ga, c, w with 65 entries each
#if LDBL_MANT_DIG <= DBL_MANT_DIG
#error "rkc2_tables64 needs a long double wider than double (x86-64, aarch64 Linux) for fp64-accurate RKC2 tables"
#endif
void rkc2_tables64(int s, double &mt1, double *mu, double *nu, double *mt, double *ga, double *c, double *w)
{
    // T_j, T_j', T_j'' and b_j in long double (the oracle's ude_rkc2_tables): in double the relative error of the three-term
    // recurrences grows like j^2 eps, which at s = 64 moves the tables' stability polynomial by ~1e-10 at the end of its interval
    const long double eps = 2.0L / 13.0L, w0 = 1.0L + eps / ((long double)s * s);
    long double T[65], dT[65], d2T[65], b[65] = {0};
    for (int j = 0; j < 65; ++j) mu[j] = nu[j] = mt[j] = ga[j] = c[j] = w[j] = 0;
    double W[65][65];   // 33 KB of stack, host side only
    T[0] = 1; T[1] = w0; dT[0] = 0; dT[1] = 1; d2T[0] = 0; d2T[1] = 0;
    for (int j = 2; j <= s; ++j) {
        T[j] = 2 * w0 * T[j - 1] - T[j - 2];
        dT[j] = 2 * T[j - 1] + 2 * w0 * dT[j - 1] - dT[j - 2];
        d2T[j] = 4 * dT[j - 1] + 2 * w0 * d2T[j - 1] - d2T[j - 2];
    }
    const long double w1 = dT[s] / d2T[s];
    for (int j = 2; j <= s; ++j) b[j] = d2T[j] / (dT[j] * dT[j]);
    b[0] = b[1] = b[2];
    mt1 = (double)(b[1] * w1);
    for (int j = 2; j <= s; ++j) {
        const long double mtj = 2 * b[j] * w1 / b[j - 1];
        mu[j] = (double)(2 * b[j] * w0 / b[j - 1]);
        nu[j] = (double)(-b[j] / b[j - 2]);
        mt[j] = (double)mtj;
        ga[j] = (double)(-(1.0L - b[j - 1] * T[j - 1]) * mtj);
    }
    memset(W, 0, sizeof W);
    c[0] = 0; c[1] = mt1; W[1][0] = mt1;
    for (int j = 2; j <= s; ++j) {
        c[j] = mu[j] * c[j - 1] + nu[j] * c[j - 2] + mt[j] + ga[j];
        for (int k = 0; k < j; ++k) W[j][k] = mu[j] * W[j - 1][k] + nu[j] * W[j - 2][k];
        W[j][j - 1] += mt[j];
        W[j][0] += ga[j];
    }
    for (int j = 0; j < s; ++j) w[j] = W[s][j];
}

void rkc2_tables(int s, RkcHost *out)
{
    double mt1, mu[65], nu[65], mt[65], ga[65], c[65], w[65];
    rkc2_tables64(s, mt1, mu, nu, mt, ga, c, w);
    *out = RkcHost();
    out->s = s; out->mt1 = (float)mt1;
    for (int j = 0; j <= s; ++j) {
        out->mu[j] = (float)mu[j]; out->nu[j] = (float)nu[j]; out->mt[j] = (float)mt[j]; out->ga[j] = (float)ga[j]; out->c[j] = (float)c[j];
        out->w[j] = j < s ? (float)w[j] : 0.0f;
    }
}

// operator UDE RKC2 table layout (operator.cuh: mt1, then c, w, mu, nu, mt, ga with 65 entries each); k = 0..5 in that order
constexpr int op_rkc_len() { return 1 + 6 * 65; }
constexpr int op_rkc_off(int k) { return 1 + 65 * k; }

// length of the real stability interval of s-stage RKC2 (damping 2/13): (w0 + 1) T''_s(w0) / T'_s(w0) ~ 0.65 s^2
double rkc2_beta64(int s)
{
    const double w0 = 1.0 + (2.0 / 13.0) / ((double)s * s);
    double T0 = 1, T1 = w0, d0 = 0, d1 = 1, e0 = 0, e1 = 0;
    for (int j = 2; j <= s; ++j) {
        const double T2 = 2 * w0 * T1 - T0, d2 = 2 * T1 + 2 * w0 * d1 - d0, e2 = 4 * d1 + 2 * w0 * e1 - e0;
        T0 = T1; T1 = T2; d0 = d1; d1 = d2; e0 = e1; e1 = e2;
    }
    return (w0 + 1.0) * e1 / d1;
}

// n doubles -> dst (device) in the handle's dtype, synchronously
cudaError_t upload_as(void *dst, const double *src, size_t n, bool f64)
{
    if (f64) return cudaMemcpy(dst, src, n * sizeof(double), cudaMemcpyHostToDevice);
    std::vector<float> v(src, src + n);
    return cudaMemcpy(dst, v.data(), n * sizeof(float), cudaMemcpyHostToDevice);
}

int env_int(const char *name, int dflt)
{
    const char *s = getenv(name);
    return s && *s ? atoi(s) : dflt;
}

bool generic_ok(const b200ude_desc &d)
{
    if (d.n_layers < 1 || d.n_layers > 5) return false;
    for (int l = 0; l <= d.n_layers; ++l)
        if (d.widths[l] < 1 || d.widths[l] > 64) return false;
    for (int l = 0; l < d.n_layers; ++l)
        if (d.acts[l] < 0 || d.acts[l] > 2) return false;
    const int din = d.widths[0], dout = d.widths[d.n_layers];
    if (d.model == B200UDE_MODEL_LV) return d.state_dim == 2 && din == 2 && dout == 2 && d.n_prefix >= 0 && d.n_prefix <= 2 && d.n_consts >= 2;
    if (d.model == B200UDE_MODEL_SEIR) return d.state_dim == 7 && din == 3 && dout == 1 && d.n_prefix == 0 && d.n_consts >= 9;
    if (d.model == B200UDE_MODEL_FKPP) return d.state_dim >= 3 && d.state_dim <= 256 && din == 1 && dout == 1 && d.n_prefix == 0 && d.n_suffix == 5 && d.n_loss_weights == 0;
    if (d.model == B200UDE_MODEL_SEIR_NODE) return d.state_dim == 7 && din == 7 && dout == 7 && d.n_prefix == 0 && d.n_consts >= 9;
    if (d.model == B200UDE_MODEL_NODE) return d.state_dim >= 1 && d.state_dim <= 8 && din == d.state_dim && dout == d.state_dim && d.n_prefix == 0;
    return false;
}

// kernel family of the LV 2-32-32-2 chain for an ensemble of N: mode 1 = always warp-collective, 0 = never, -1 = by size
bool use_wm(int mode, size_t N, size_t n_max) { return mode > 0 || (mode < 0 && N <= n_max); }

template <typename R>
constexpr bool is_f32 = std::is_same<R, float>::value;

// the forced neural ODE's and the operator UDE's forward, and the launch of their adjoints (both dtypes; defined below)
int32_t do_forward_forced(b200ude_handle *h, const void *u0, size_t N, void *out, int32_t *status, cudaStream_t st);
int32_t do_adjoint_forced(b200ude_handle *h, bool l2, const void *cot, void *grad_u0, cudaStream_t st, int *rows);
int32_t do_forward_operator(b200ude_handle *h, const void *u0, size_t N, void *out, int32_t *status, cudaStream_t st);
int32_t do_adjoint_operator(b200ude_handle *h, bool l2, const void *cot, void *grad_u0, cudaStream_t st, int *rows);

// the kernels' parameter structs of each precision
FwdParams fwd_params(const b200ude_handle *h, const float *u0, float *out, void *ustep, void *dense, int32_t *status, size_t N)
{
    FwdParams p;
    p.u0 = u0; p.out = out; p.ustep = (float *)ustep; p.dense = (float *)dense; p.status = status; p.theta = (const float *)h->d_theta;
    p.N = (int)N; p.n_steps = h->desc.n_steps; p.save_every = h->desc.save_every; p.P = h->P; p.dt = (float)h->desc.dt;
    return p;
}
Fwd64Host fwd_params(const b200ude_handle *h, const double *u0, double *out, void *ustep, void *dense, int32_t *status, size_t N)
{
    return Fwd64Host{u0, out, (double *)ustep, (double *)dense, status, (int)N, h->desc.n_steps, h->desc.save_every, h->desc.dt};
}
AdjParams adj_params(const b200ude_handle *h, const float *cot, float *grad_u0, bool l2)
{
    AdjParams p;
    p.ustep = (const float *)h->d_ustep; p.dense = (const float *)h->d_dense; p.cot = cot; p.grad_u0 = grad_u0; p.partial = (float *)h->d_partial;
    p.theta = (const float *)h->d_theta; p.N = (int)h->N; p.n_steps = h->desc.n_steps; p.save_every = h->desc.save_every; p.P = h->P;
    p.fused_l2 = l2 ? 1 : 0;
    p.dt = (float)h->desc.dt;
    return p;
}
Adj64Host adj_params(const b200ude_handle *h, const double *cot, double *grad_u0, bool l2)
{
    return Adj64Host{(const double *)h->d_ustep, (const double *)h->d_dense, cot, grad_u0, (double *)h->d_partial, (int)h->N, h->desc.n_steps,
                     h->desc.save_every, l2 ? 1 : 0, h->desc.dt};
}
// Every kernel runs on the time axis s = t - t0, so the origin it is given is 0.  The autonomous models never see t, and this
// keeps the float spacing of their step and save times that of the span, not of |t0| (at t0 = 1900, ulp(t) = 1.2e-4 in fp32).
// The forced model, the one model that reads t, has W t0 folded into its phases instead (b200ude_set_forcing).
template <typename R>
typename RealParams<R>::Adapt adapt(const b200ude_handle *h)
{
    return {(R)0, (R)(h->desc.dt * h->desc.save_every), (R)h->desc.abstol, (R)h->desc.reltol, h->n_save, h->desc.max_steps,
            (R *)h->d_tgrid, h->d_nacc, (R *)h->d_hstep};
}
template <typename R>
const typename RealParams<R>::Tab &tables(const b200ude_handle *h)
{
    if constexpr (is_f32<R>) return h->tab;
    else return h->tab64;
}

// the forward kernel of the handle's route.  tsit5: the Tsit5 re-solve of a Vern7 route (R_VERN7, R_SEIR64_VERN7) that its
// interpolating adjoint runs over.  The fp32-only routes exist in the fp32 instantiation only.
template <typename R>
cudaError_t launch_forward(b200ude_handle *h, const typename RealParams<R>::Fwd &p, size_t N, bool tsit5, cudaStream_t st)
{
    using RS = RuntimeShape<R>;
    const auto &t = tables<R>(h);
    const auto ag = adapt<R>(h);
    const auto *agp = h->adaptive ? &ag : nullptr;
    switch (h->route) {
    case R_LV32:
    case R_LV32_DISCRETE:
        // small / medium ensembles: the warp-collective family (latency per stage ~4x lower); large ones: one trajectory per thread
        if constexpr (is_f32<R>)
            return use_wm(h->var.fwd_wm, N, h->wm_fwd_max) ? launch_fwd_lv32_wm(h->var, h->tab, p, st) : launch_fwd_lv32(h->var, h->tab, p, st);
        break;
    case R_LV32_ADAPTIVE: if constexpr (is_f32<R>) return launch_fwd_lv32_adaptive(h->var, h->tab, p, ag, st); break;
    case R_LV5: if constexpr (is_f32<R>) return launch_fwd_lv5(h->desc.n_prefix, h->var, h->tab, p, st); break;
    case R_SEIR64: if constexpr (is_f32<R>) return launch_fwd_seir(h->var, h->tab, p, st); break;
    case R_SEIR64_VERN7:
        if constexpr (is_f32<R>) return tsit5 ? launch_fwd_seir(h->var, h->tab, p, st) : launch_fwd_seir_vern7(h->var, h->tab, p, st);
        break;
    case R_SEIR64_ADAPTIVE: if constexpr (is_f32<R>) return launch_fwd_seir_adaptive(h->var, h->tab, p, ag, st); break;
    case R_FKPP_FIXED: if constexpr (is_f32<R>) return launch_fwd_fkpp(h->gen, h->tab, p, st); break;
    case R_FKPP16: if constexpr (is_f32<R>) return launch_fwd_fkpp16(h->var, h->tab, p, h->D, st); break;
    case R_FKPP16_RKC2: if constexpr (is_f32<R>) return launch_fwd_fkpp16_rkc(h->var, h->tab, h->rkc, p, h->D, st); break;
    case R_FKPP_ADAPTIVE:
    case R_FKPP_CHECKPOINT: return RS::fwd_fkpp_adaptive(h->gen, t, p, ag, h->seg, st);
    case R_FKPP_VERN7_DISCRETE: return RS::fwd_fkpp_vern7(h->gen, t, p, ag, st);
    case R_TSIT5:
    case R_DISCRETE_TSIT5: return RS::fwd(h->gen, t, p, 0, agp, st);
    case R_VERN7: return RS::fwd(h->gen, t, p, tsit5 ? 0 : 1, agp, st);
    case R_DISCRETE_VERN7: return RS::fwd(h->gen, t, p, 1, agp, st);
    // an adaptive solve saves through the interpolant; a fixed grid saves at step ends, as without the flag
    case R_VERN7_DENSE: return h->adaptive ? RS::fwd_vern7_dense(h->gen, t, p, ag, st) : RS::fwd(h->gen, t, p, 1, nullptr, st);
    case R_VERN7_DENSE_DISCRETE: return RS::fwd_vern7_dense(h->gen, t, p, ag, st);
    case R_FORCED:
    case R_OPERATOR: break;   // do_forward_forced, do_forward_operator
    }
    return cudaErrorNotSupported;
}

template <typename R>
int32_t do_forward(b200ude_handle *h, const R *u0, size_t N, R *out, int32_t *status, cudaStream_t st)
{
    CUDA_TRY(h, cudaSetDevice(h->desc.device));   // launches, symbol copies and function attributes go to the handle's device
    if (!h->have_theta) return fail(h, B200UDE_ESTATE, "forward: set_params has not been called");
    if (N == 0 || N > h->cap) return fail(h, B200UDE_EINVAL, "forward: N=%zu outside (0, max_trajectories=%zu]", N, h->cap);
    if (!u0 || !out) return fail(h, B200UDE_EINVAL, "forward: null pointer");
    switch (h->route) {
    case R_FORCED: return do_forward_forced(h, u0, N, out, status, st);
    case R_OPERATOR: return do_forward_operator(h, u0, N, out, status, st);
    case R_VERN7:
    case R_SEIR64_VERN7:
        // Vern7 writes the saved states only.  Its lazy dense output is not used here (R_VERN7_DENSE uses it), so the interpolating
        // adjoint runs over a Tsit5 re-solve from the same u0 with the same step / tolerances, launched by the first adjoint call
        // (do_adjoint); u0 is kept for that.
        CUDA_TRY(h, launch_forward<R>(h, fwd_params(h, u0, out, nullptr, nullptr, status, N), N, false, st));
        if (!h->d_u0_keep && dalloc_real(h, &h->d_u0_keep, (size_t)h->D * h->cap) != cudaSuccess)
            return fail(h, B200UDE_ENOMEM, "forward: device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
        CUDA_TRY(h, cudaMemcpyAsync(h->d_u0_keep, u0, sizeof(R) * (size_t)h->D * N, cudaMemcpyDeviceToDevice, st));
        h->N = N;
        h->have_forward = false;
        h->vern7_pending = true;
        return B200UDE_OK;
    default:
        // the Tsit5 and RKC2 solves write the dense record (stage derivatives) the interpolating adjoint reads; the routes that
        // recompute the stages from u_n (discrete adjoint of Vern7, Vern7's dense output) have none (d_dense = nullptr)
        CUDA_TRY(h, launch_forward<R>(h, fwd_params(h, u0, out, h->d_ustep, h->d_dense, status, N), N, false, st));
        h->last_out = out;
        h->N = N;
        h->have_forward = true;
        return B200UDE_OK;
    }
}

// partial rows -> grad_theta and the loss (nullptr: not written): fp64 reduce, fp32 reduce fused with the all-reduce over the
// attached peers, or fp32 reduce
int32_t reduce_partials(b200ude_handle *h, int rows, void *grad_theta, void *loss, bool peer, cudaStream_t st)
{
    if (h->f64) CUDA_TRY(h, launch_reduce_f64((const double *)h->d_partial, rows, h->P + 1, (double *)grad_theta, (double *)loss, st));
    else if (peer) CUDA_TRY(h, launch_reduce_exchange((const float *)h->d_partial, rows, h->P + 1, h->peer, (float *)grad_theta, (float *)loss, st));
    else CUDA_TRY(h, launch_reduce((const float *)h->d_partial, rows, h->P + 1, (float *)grad_theta, (float *)loss, st));
    return B200UDE_OK;
}

// split: two events (data of the first / second half of the trajectories resident) for the host-buffer path: the warp-collective LV
// adjoint then runs as two sub-range launches, the first one under the second half's upload
template <typename R>
int32_t do_adjoint(b200ude_handle *h, bool l2, const R *cot, R *loss, R *grad_theta, R *grad_u0, cudaStream_t st, bool peer = false,
                   const cudaEvent_t *split = nullptr, size_t split_at = 0)
{
    CUDA_TRY(h, cudaSetDevice(h->desc.device));
    if (peer && !h->peer_attached) return fail(h, B200UDE_ESTATE, "adjoint_l2_allreduce: b200ude_peer_attach has not been called");
    if (peer && h->adaptive) return fail(h, B200UDE_EUNSUPPORTED, "adjoint_l2_allreduce: not available with adaptive stepping (all-reduce the result of b200ude_adjoint_l2 instead)");
    // an fp64 operator handle names its missing operators before the missing forward solution
    if (h->f64 && h->route == R_OPERATOR && !h->ops_set)
        return fail(h, B200UDE_ESTATE, "adjoint: B200UDE_MODEL_OPERATOR needs its operators (call b200ude_set_operators first)");
    if (h->vern7_pending) {
        if (!h->d_aux_out && dalloc_real(h, &h->d_aux_out, (size_t)h->n_save * (size_t)h->D * h->cap) != cudaSuccess)
            return fail(h, B200UDE_ENOMEM, "adjoint: device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
        CUDA_TRY(h, launch_forward<R>(h, fwd_params(h, (const R *)h->d_u0_keep, (R *)h->d_aux_out, h->d_ustep, h->d_dense, nullptr, h->N),
                                      h->N, true, st));
        h->last_out = h->d_aux_out;
        h->vern7_pending = false;
        h->have_forward = true;
    }
    if (!h->have_forward) return fail(h, B200UDE_ESTATE, "adjoint: no stored forward solution (call b200ude_forward first)");
    if (!cot || !grad_theta) return fail(h, B200UDE_EINVAL, "adjoint: null pointer");
    const bool split_ok = split && h->route == R_LV32 && use_wm(h->var.adj_wm, h->N, h->wm_adj_max) && split_at > 0 && split_at < h->N;
    if (split && !split_ok) {   // every other kernel family reads the whole data array
        CUDA_TRY(h, cudaStreamWaitEvent(st, split[0], 0));
        CUDA_TRY(h, cudaStreamWaitEvent(st, split[1], 0));
    }
    using RS = RuntimeShape<R>;
    const auto &t = tables<R>(h);
    const auto ag = adapt<R>(h);
    const auto *agp = h->adaptive ? &ag : nullptr;
    auto p = adj_params(h, cot, grad_u0, l2);
    const R *saved = (const R *)h->last_out;   // the states the forward returned (after a Vern7 forward: the Tsit5 re-solve's)
    R *reduce_loss = loss;
    bool finish_l2 = false;   // fp32 two-stage L2 cotangent: its loss follows the reduce
    const Route r = h->route;
    if (h->adaptive && l2 && (r == R_LV32_ADAPTIVE || r == R_SEIR64_ADAPTIVE || r == R_FKPP_ADAPTIVE || r == R_FKPP_CHECKPOINT ||
                              r == R_TSIT5 || r == R_VERN7)) {
        // the replay of an adaptive Tsit5 solve: form the cotangent 2 w (out - data) from the interpolated saved states of the last
        // forward, in fp32 in two stages (the loss follows the reduce), in fp64 in one CTA that writes the loss itself
        if constexpr (is_f32<R>) {
            CUDA_TRY(h, launch_l2_cot(h->tab, saved, cot, (float *)h->d_cot, h->d_block_loss, h->D, h->N, h->n_save, st));
            finish_l2 = loss != nullptr;
        } else {
            CUDA_TRY(h, launch_l2_cot_f64(h->tab64, saved, cot, (double *)h->d_cot, loss, h->D, h->N, h->n_save, st));
            reduce_loss = nullptr;
        }
        p.cot = (const R *)h->d_cot;
        p.fused_l2 = 0;
    }
    int rows = 0;
    cudaError_t e = cudaErrorNotSupported;
    switch (r) {
    case R_LV32:
        if constexpr (is_f32<R>) {
            if (!split_ok) {
                e = use_wm(h->var.adj_wm, h->N, h->wm_adj_max) ? launch_adj_lv32_wm(h->var, h->tab, p, st, &rows)
                                                              : launch_adj_lv32(h->var, h->tab, p, st, &rows);
                break;
            }
            int g0 = 0, g1 = 0;
            AdjParams q = p;
            q.n0 = 0; q.n_cnt = (int)split_at; q.row0 = 0;
            e = cudaStreamWaitEvent(st, split[0], 0);
            if (e == cudaSuccess) e = launch_adj_lv32_wm(h->var, h->tab, q, st, &g0);
            if (e == cudaSuccess) {
                q.n0 = (int)split_at; q.n_cnt = (int)(h->N - split_at); q.row0 = g0;
                e = cudaStreamWaitEvent(st, split[1], 0);
                if (e == cudaSuccess) e = launch_adj_lv32_wm(h->var, h->tab, q, st, &g1);
            }
            rows = g0 + g1;
        }
        break;
    case R_LV32_DISCRETE: if constexpr (is_f32<R>) e = launch_adj_lv32(h->var, h->tab, p, st, &rows); break;
    case R_LV32_ADAPTIVE: if constexpr (is_f32<R>) e = launch_adj_lv32_adaptive(h->var, h->tab, p, ag, st, &rows); break;
    case R_LV5: if constexpr (is_f32<R>) e = launch_adj_lv5(h->desc.n_prefix, h->var, h->tab, p, st, &rows); break;
    case R_SEIR64:
    case R_SEIR64_VERN7: if constexpr (is_f32<R>) e = launch_adj_seir(h->var, h->tab, p, st, &rows); break;
    case R_SEIR64_ADAPTIVE: if constexpr (is_f32<R>) e = launch_adj_seir_adaptive(h->var, h->tab, p, ag, st, &rows); break;
    case R_FKPP_FIXED: if constexpr (is_f32<R>) e = launch_adj_fkpp(h->gen, h->tab, p, st, &rows); break;
    case R_FKPP16: if constexpr (is_f32<R>) e = launch_adj_fkpp16(h->var, h->tab, p, h->D, st, &rows); break;
    case R_FKPP16_RKC2: if constexpr (is_f32<R>) e = launch_adj_fkpp16_rkc(h->var, h->tab, h->rkc, p, h->D, st, &rows); break;
    case R_FKPP_ADAPTIVE:
    case R_FKPP_CHECKPOINT: e = RS::adj_fkpp_adaptive(h->gen, t, p, ag, h->seg, st, &rows); break;
    // grid-per-CTA kernels
    case R_FKPP_VERN7_DISCRETE: e = RS::adj_fkpp_vern7(h->gen, t, p, ag, st, &rows); break;
    case R_TSIT5:
    case R_VERN7: e = RS::adj(h->gen, t, p, agp, st, &rows); break;
    // over the recorded steps; the fused L2 reads the recorded step-end states
    case R_DISCRETE_TSIT5: e = RS::adj_discrete(h->gen, t, p, 0, agp, st, &rows); break;
    case R_DISCRETE_VERN7: e = RS::adj_discrete(h->gen, t, p, 1, agp, st, &rows); break;
    // over Vern7's own dense output / through its interpolated saves; the fused L2 reads the states the forward returned
    case R_VERN7_DENSE: e = RS::adj_vern7_dense(h->gen, t, p, agp, saved, st, &rows); break;
    case R_VERN7_DENSE_DISCRETE: e = RS::adj_vern7_dense_discrete(h->gen, t, p, ag, saved, st, &rows); break;
    case R_FORCED:
    case R_OPERATOR: {
        const int32_t rc = r == R_FORCED ? do_adjoint_forced(h, l2, cot, grad_u0, st, &rows) : do_adjoint_operator(h, l2, cot, grad_u0, st, &rows);
        if (rc) return rc;
        e = cudaSuccess;
        break;
    }
    }
    CUDA_TRY(h, e);
    const int32_t rc = reduce_partials(h, rows, grad_theta, reduce_loss, peer, st);
    if (rc) return rc;
    if constexpr (is_f32<R>) {
        if (finish_l2) CUDA_TRY(h, launch_l2_finish(h->d_block_loss, loss, st));
    }
    return B200UDE_OK;
}

// ---- ADAM on the device (Flux.ADAM(eta, (beta1, beta2)), eps = 1e-8: scenario_1.jl:114, seir_exposure.jl:160) ----
// One CTA: L = loss_scale * L_data + l2_reg * sum theta^2, g = loss_scale * grad + 2 l2_reg theta, then the
// bias-corrected update of theta in place.  The step counter lives in device memory so that the launch arguments
// do not change from iteration to iteration (the training loop is replayed as a CUDA graph).
struct AdamArgs {
    float *theta, *m, *v;
    const float *grad, *loss;   // loss may be null
    float *loss_history;        // [..] or null; slot (t - 1 - t_base) receives the pre-update loss
    int *t;
    int P, t_base, reg_from;   // the L2 term covers theta[reg_from:] (scenario_2.jl:113: sum(abs2, theta[2:end]) skips the trainable physics rate)
    float eta, beta1, beta2, eps, loss_scale, l2_reg;
};

__global__ void __launch_bounds__(1024, 1) adam_kernel(AdamArgs a)
{
    __shared__ float red[32];
    __shared__ int s_t;
    if (threadIdx.x == 0) s_t = *a.t + 1;
    float sq = 0.0f;
    if (a.l2_reg != 0.0f)
        for (int i = a.reg_from + threadIdx.x; i < a.P; i += blockDim.x) sq = fmaf(a.theta[i], a.theta[i], sq);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
    __syncthreads();
    const int t = s_t;
    if (threadIdx.x == 0) {
        float tot = 0.0f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];   // fixed order
        if (a.loss_history && a.loss) a.loss_history[t - 1 - a.t_base] = fmaf(a.loss_scale, *a.loss, a.l2_reg * tot);
        *a.t = t;
    }
    const float c1 = (float)(1.0 / (1.0 - pow((double)a.beta1, (double)t)));
    const float c2 = (float)(1.0 / (1.0 - pow((double)a.beta2, (double)t)));
    for (int i = threadIdx.x; i < a.P; i += blockDim.x) {
        const float th = a.theta[i];
        const float g = fmaf(a.loss_scale, a.grad[i], i >= a.reg_from ? 2.0f * a.l2_reg * th : 0.0f);
        const float m = fmaf(a.beta1, a.m[i], (1.0f - a.beta1) * g);
        const float v = fmaf(a.beta2, a.v[i], (1.0f - a.beta2) * g * g);
        a.m[i] = m;
        a.v[i] = v;
        a.theta[i] = th - a.eta * (m * c1) / (sqrtf(v * c2) + a.eps);
    }
}

int32_t ensure_adam(b200ude_handle *h)
{
    if (h->f64) return fail(h, B200UDE_EUNSUPPORTED, "adam: not available for B200UDE_F64 handles (update theta on the host side)");
    if (h->d_adam_m) return B200UDE_OK;
    bool ok = dalloc(h, &h->d_adam_m, (size_t)h->P) == cudaSuccess && dalloc(h, &h->d_adam_v, (size_t)h->P) == cudaSuccess &&
              dalloc(h, &h->d_adam_t, 1) == cudaSuccess;
    if (!ok) return fail(h, B200UDE_ENOMEM, "adam: device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    // synchronous with respect to the host and to every stream that is used afterwards
    cudaMemset(h->d_adam_m, 0, sizeof(float) * h->P);
    cudaMemset(h->d_adam_v, 0, sizeof(float) * h->P);
    cudaMemset(h->d_adam_t, 0, sizeof(int));
    cudaDeviceSynchronize();
    h->adam_t = 0;
    return B200UDE_OK;
}

int32_t check_adam(b200ude_handle *h, const b200ude_adam *o)
{
    if (!o || o->struct_size != sizeof(b200ude_adam)) return fail(h, B200UDE_EINVAL, "adam: bad options struct");
    if (!(o->eta > 0) || !(o->beta1 >= 0 && o->beta1 < 1) || !(o->beta2 >= 0 && o->beta2 < 1) || !(o->eps > 0))
        return fail(h, B200UDE_EINVAL, "adam: need eta > 0, 0 <= beta < 1, eps > 0");
    if (!h->have_theta) return fail(h, B200UDE_ESTATE, "adam: no parameters set (call b200ude_set_params first)");
    return ensure_adam(h);
}

cudaError_t launch_adam(b200ude_handle *h, const b200ude_adam *o, const float *grad, const float *loss, float *hist, int t_base, cudaStream_t st)
{
    AdamArgs a;
    a.theta = (float *)h->d_theta; a.m = h->d_adam_m; a.v = h->d_adam_v; a.grad = grad; a.loss = loss; a.loss_history = hist;
    a.t = h->d_adam_t; a.P = h->P; a.t_base = t_base; a.reg_from = h->desc.n_prefix > 0 ? h->desc.n_prefix : 0;
    a.eta = (float)o->eta; a.beta1 = (float)o->beta1; a.beta2 = (float)o->beta2; a.eps = (float)o->eps;
    a.loss_scale = (float)(o->loss_scale == 0.0 ? 1.0 : o->loss_scale); a.l2_reg = (float)o->l2_reg;
    adam_kernel<<<1, 1024, 0, st>>>(a);
    return cudaGetLastError();
}

// ---- forced neural ODE with a readout network (B200UDE_MODEL_FORCED; k_forced.cu), both dtypes ------------------------------
int32_t forced_check(const b200ude_desc *d)
{
    if (d->solver != B200UDE_TSIT5 || d->sensealg != B200UDE_INTERPOLATING_ADJOINT ||
        (d->flags & (B200UDE_FLAG_VERN7_DENSE | B200UDE_FLAG_DISCRETE_DENSE)))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: B200UDE_MODEL_FORCED (forced neural ODE with a readout) has kernels for Tsit5, fixed step or adaptive, with the "
                    "interpolating adjoint; not for Vern7, RKC2, the discrete adjoint, B200UDE_FLAG_VERN7_DENSE or B200UDE_FLAG_DISCRETE_DENSE");
    const char *why = nullptr;
    const int D = d->state_dim, NL = d->n_layers;
    const int L0 = (int)d->consts[0], J = (int)d->consts[1], L1 = NL - L0;
    if (d->n_consts != 2 || d->consts[0] != (double)L0 || d->consts[1] != (double)J) why = "n_consts must be 2 with consts[0] = L0 (layers of f0) and consts[1] = J (harmonics), both integers";
    else if (J < 1 || J > 4) why = "J = consts[1] must be 1..4";
    else if (L0 < 1 || L1 < 1) why = "consts[0] = L0 must leave at least one layer to each of f0 and f1 (n_layers = L0 + L1)";
    else if (NL > 5) why = "L0 + L1 <= 5 (the widths of both chains take n_layers + 2 <= 7 entries)";
    else if (D < 1 || D > 7) why = "state_dim must be 1..7 (the chains' input [u; gamma] has <= 8 entries)";
    else if (d->n_prefix != 0 || d->n_suffix != 0) why = "n_prefix and n_suffix must be 0";
    if (!why) {
        for (int l = 0; l <= NL + 1; ++l)
            if (d->widths[l] < 1 || d->widths[l] > 64) why = "every width must be 1..64";
        for (int l = 0; l < NL; ++l)
            if (d->acts[l] < 0 || d->acts[l] > 2) why = "unknown activation";
    }
    if (!why) {
        const int r = d->widths[L0];
        if (d->widths[0] != D + 1) why = "f0's input widths[0] must be state_dim + 1";
        else if (r > 8) why = "the readout width widths[L0] must be <= 8";
        else if (d->widths[L0 + 1] != D + 1) why = "f1's input widths[L0 + 1] must be state_dim + 1";
        else if (d->widths[NL + 1] != D) why = "f1's output widths[n_layers + 1] must be state_dim";
        else if (d->n_loss_weights != 0 && d->n_loss_weights != D + r) why = "n_loss_weights must be 0 or state_dim + r";
        else if (d->adaptive && (!(d->abstol > 0) || !(d->reltol > 0) || d->max_steps < 1)) why = "adaptive stepping needs abstol > 0, reltol > 0, max_steps >= 1";
    }
    if (why) return fail(nullptr, B200UDE_EINVAL, "create: B200UDE_MODEL_FORCED: %s", why);
    return B200UDE_OK;
}

ForcedRun forced_run(const b200ude_handle *h, size_t N)
{
    ForcedRun r{};
    r.forcing = h->d_forcing;
    r.ustep = h->d_ustep; r.dense = h->d_dense; r.partial = h->d_partial; r.tgrid = h->d_tgrid;
    r.nacc = h->d_nacc;
    r.usave = h->d_usave;
    r.N = (int)N; r.n_steps = h->desc.n_steps; r.save_every = h->desc.save_every; r.adaptive = h->adaptive ? 1 : 0;
    r.n_save = h->n_save; r.max_steps = h->desc.max_steps; r.fstride = (int)h->cap;
    r.t0 = 0; r.dt = h->desc.dt; r.save_dt = h->desc.dt * h->desc.save_every; r.abstol = h->desc.abstol; r.reltol = h->desc.reltol;   // s = t - t0 (adapt)
    return r;
}

int32_t do_forward_forced(b200ude_handle *h, const void *u0, size_t N, void *out, int32_t *status, cudaStream_t st)
{
    if (N > h->forcing_n)
        return fail(h, B200UDE_ESTATE, "forward: B200UDE_MODEL_FORCED needs the forcing of every trajectory (b200ude_set_forcing set %zu, N = %zu)",
                    h->forcing_n, N);
    ForcedRun r = forced_run(h, N);
    r.u0 = u0; r.out = out; r.status = status;
    CUDA_TRY(h, launch_fwd_forced(h->fh, r, st));
    h->N = N;
    h->have_forward = true;
    return B200UDE_OK;
}

// fused L2: the loss 2 w (out - data) over all d + r rows, the readout rows recomputed from the saved states
int32_t do_adjoint_forced(b200ude_handle *h, bool l2, const void *cot, void *grad_u0, cudaStream_t st, int *rows)
{
    if (h->N > h->forcing_n) return fail(h, B200UDE_ESTATE, "adjoint: the forcing was reset to fewer trajectories than the forward solved");
    ForcedRun r = forced_run(h, h->N);
    r.cot = cot; r.saved = h->d_usave; r.grad_u0 = grad_u0; r.fused_l2 = l2 ? 1 : 0;
    CUDA_TRY(h, launch_adj_forced(h->fh, r, st, rows));
    return B200UDE_OK;
}

// ---- wide-state operator UDE du = D1 NN(u) + D2 u (B200UDE_MODEL_OPERATOR; k_operator.cu), both dtypes ---------------------------
int32_t operator_check(const b200ude_desc *d)
{
    if (d->solver == B200UDE_VERN7 || d->sensealg != B200UDE_INTERPOLATING_ADJOINT ||
        (d->flags & (B200UDE_FLAG_VERN7_DENSE | B200UDE_FLAG_DISCRETE_DENSE)))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: B200UDE_MODEL_OPERATOR (operator UDE du = D1 NN(u) + D2 u) has kernels for Tsit5 and RKC2, fixed step or "
                    "adaptive, with the interpolating adjoint; not for Vern7, the discrete adjoint, B200UDE_FLAG_VERN7_DENSE or "
                    "B200UDE_FLAG_DISCRETE_DENSE");
    const char *why = nullptr;
    const int D = d->state_dim, NL = d->n_layers;
    // adaptive RKC2 picks each step's stage count from eigen_est, the one constant this model takes (consts[0])
    const bool ark = d->solver == B200UDE_RKC2 && d->adaptive;
    if (D < 1 || D > 64) why = "state_dim must be 1..64";
    else if (NL > 5) why = "n_layers must be 1..5";
    else if (d->n_prefix != 0 || d->n_suffix != 0 || (d->n_consts != 0 && !(ark && d->n_consts == 1)))
        why = "n_prefix, n_suffix and n_consts must be 0 (n_consts = 1 only for adaptive RKC2: eigen_est in consts[0])";
    if (!why) {
        for (int l = 0; l <= NL; ++l)
            if (d->widths[l] < 1 || d->widths[l] > 64) why = "every width must be 1..64";
        for (int l = 0; l < NL; ++l)
            if (d->acts[l] < 0 || d->acts[l] > 2) why = "unknown activation";
    }
    if (!why) {
        if (d->widths[0] != D) why = "the chain's input widths[0] must be state_dim";
        else if (d->n_loss_weights != 0 && (d->n_loss_weights != D || D > 16)) why = "n_loss_weights must be 0, or state_dim when state_dim <= 16";
        else if (d->solver == B200UDE_RKC2 && (d->n_stages < 2 || d->n_stages > 64)) why = "RKC2 needs 2 <= n_stages <= 64";
        else if (ark && d->n_consts != 1)
            why = "adaptive RKC2 needs eigen_est (a bound of the spectral radius of df/du) in consts[0] with n_consts = 1; without it "
                  "RKC2 runs with a fixed step (adaptive = 0)";
        else if (ark && !(std::isfinite(d->consts[0]) && d->consts[0] > 0)) why = "adaptive RKC2 needs a finite eigen_est > 0 in consts[0]";
        else if (d->adaptive && (!(d->abstol > 0) || !(d->reltol > 0) || d->max_steps < 1)) why = "adaptive stepping needs abstol > 0, reltol > 0, max_steps >= 1";
    }
    if (why) return fail(nullptr, B200UDE_EINVAL, "create: B200UDE_MODEL_OPERATOR: %s", why);
    return B200UDE_OK;
}

OperatorRun operator_run(const b200ude_handle *h, size_t N)
{
    OperatorRun r{};
    r.ustep = h->d_ustep; r.dense = h->d_dense; r.partial = h->d_partial; r.tgrid = h->d_tgrid;
    r.usave = h->d_usave;
    r.nacc = h->d_nacc;
    r.sstep = h->d_sstep;
    r.N = (int)N; r.n_steps = h->desc.n_steps; r.save_every = h->desc.save_every; r.n_save = h->n_save; r.max_steps = h->desc.max_steps;
    r.adaptive = h->adaptive ? 1 : 0;
    r.t0 = 0; r.dt = h->desc.dt; r.save_dt = h->desc.dt * h->desc.save_every; r.abstol = h->desc.abstol; r.reltol = h->desc.reltol;   // s = t - t0 (adapt)
    return r;
}

int32_t do_forward_operator(b200ude_handle *h, const void *u0, size_t N, void *out, int32_t *status, cudaStream_t st)
{
    if (!h->ops_set) return fail(h, B200UDE_ESTATE, "forward: B200UDE_MODEL_OPERATOR needs its operators (call b200ude_set_operators first)");
    OperatorRun r = operator_run(h, N);
    r.u0 = u0; r.out = out; r.status = status;
    CUDA_TRY(h, launch_fwd_operator(h->oh, r, st));
    h->N = N;
    h->have_forward = true;
    return B200UDE_OK;
}

// the operators are set: a forward solution exists (do_adjoint)
int32_t do_adjoint_operator(b200ude_handle *h, bool l2, const void *cot, void *grad_u0, cudaStream_t st, int *rows)
{
    OperatorRun r = operator_run(h, h->N);
    r.cot = cot; r.grad_u0 = grad_u0; r.fused_l2 = l2 ? 1 : 0;
    CUDA_TRY(h, launch_adj_operator(h->oh, r, st, rows));
    return B200UDE_OK;
}

// The descriptor checks and the route that runs the descriptor.  The refusals keep this order: the first check a descriptor fails
// names it.  The kernel-selection knobs (B200UDE_SEIR_TC, _FKPP_TUNED, _SEIR_VERN7_TC, _ADAPTIVE_TC, _FKPP_PACKED; default 1) are
// read here, so they take effect per handle at create.
int32_t resolve(const b200ude_desc &d, Route *route)
{
    const bool disc = d.sensealg == B200UDE_DISCRETE_ADJOINT, want64 = d.dtype == B200UDE_F64, adaptive = d.adaptive != 0;
    const bool fkpp = d.model == B200UDE_MODEL_FKPP;
    if ((d.flags & B200UDE_FLAG_CHECKPOINT) && !(fkpp && adaptive && d.solver == B200UDE_TSIT5 && d.sensealg == B200UDE_INTERPOLATING_ADJOINT))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: B200UDE_FLAG_CHECKPOINT applies to adaptive Tsit5 with the interpolating adjoint on the Fisher-KPP UPDE; not to "
                    "fixed step, Vern7, RKC2, the discrete adjoint or other models");
    if (d.model == B200UDE_MODEL_OPERATOR) {
        *route = R_OPERATOR;
        return operator_check(&d);
    }
    if (d.model == B200UDE_MODEL_FORCED) {
        *route = R_FORCED;
        return forced_check(&d);
    }
    if (d.n_loss_weights != 0 && d.n_loss_weights != d.state_dim) return fail(nullptr, B200UDE_EINVAL, "create: n_loss_weights must be 0 or state_dim");
    // the tuned chains
    const bool shape_ok = generic_ok(d);   // the runtime-shape envelope
    const bool lv_out = d.model == B200UDE_MODEL_LV && d.state_dim == 2 && d.acts[d.n_layers - 1] == B200UDE_ACT_IDENTITY;
    const bool lv32 = lv_out && d.n_layers == 3 && d.widths[0] == 2 && d.widths[1] == 32 && d.widths[2] == 32 && d.widths[3] == 2 &&
                      d.acts[0] == B200UDE_ACT_TANH && d.acts[1] == B200UDE_ACT_TANH && d.n_prefix == 0;
    const bool lv5 = lv_out && d.n_layers == 4 && d.widths[0] == 2 && d.widths[1] == 5 && d.widths[2] == 5 && d.widths[3] == 5 &&
                     d.widths[4] == 2 && d.n_prefix >= 0 && d.n_prefix <= 2;
    const bool tanh64 = d.n_layers == 3 && d.acts[0] == B200UDE_ACT_TANH && d.acts[1] == B200UDE_ACT_TANH && d.acts[2] == B200UDE_ACT_IDENTITY;
    const bool seir64 = shape_ok && tanh64 && d.model == B200UDE_MODEL_SEIR && d.widths[1] == 64 && d.widths[2] == 64 && d.n_suffix == 0 &&
                        env_int("B200UDE_SEIR_TC", 1);
    const bool fkpp16 = shape_ok && tanh64 && fkpp && d.widths[1] == 16 && d.widths[2] == 16 && env_int("B200UDE_FKPP_TUNED", 1);
    // discrete adjoint: the tuned LV kernels (fixed-step Tsit5 on 2-32-32-2 / 2-5-5-5-2, fp32), the runtime-shape kernels of
    // discrete_adjoint.cuh and, for the Fisher-KPP UPDE, the grid-per-CTA adaptive Vern7 kernels of fkpp_vern7_discrete.cuh.
    // Adaptive Tsit5 saves through its free interpolant, which an exact discrete adjoint would also have to differentiate;
    // fixed-step Fisher-KPP and RKC2 have no such kernels.
    // B200UDE_FLAG_DISCRETE_DENSE: the discrete adjoint of the Vern7 solve that saves through its lazy interpolant
    // (vern7_dense_discrete.cuh); on a fixed grid the saves are step ends and the flag selects nothing
    const bool disc_dense = (d.flags & B200UDE_FLAG_DISCRETE_DENSE) != 0;
    if (disc_dense && (d.solver != B200UDE_VERN7 || !disc || fkpp || (d.flags & B200UDE_FLAG_VERN7_DENSE)))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: B200UDE_FLAG_DISCRETE_DENSE applies to Vern7 with the discrete adjoint on the LV / SEIR / SEIR_NODE / NODE forms; "
                    "not to the interpolating adjoint (B200UDE_FLAG_VERN7_DENSE is its flag, and the two exclude each other), Tsit5, RKC2 or "
                    "the Fisher-KPP UPDE");
    const bool fkpp_v7 = fkpp && adaptive && d.solver == B200UDE_VERN7;
    if (disc && ((fkpp && !fkpp_v7) || d.solver == B200UDE_RKC2 || (adaptive && d.solver == B200UDE_TSIT5)))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: the discrete adjoint (ForwardDiffSensitivity) has kernels for fixed-step Tsit5 and for fixed-step or adaptive Vern7 on the "
                    "LV / SEIR / SEIR_NODE / NODE forms (chain widths <= 64), and for adaptive Vern7 on the Fisher-KPP UPDE, fp32 and fp64; "
                    "not for adaptive Tsit5, fixed-step Fisher-KPP or RKC2");
    // Vern7's lazy dense output (vern7_dense.cuh): saveat through the interpolant and the interpolating adjoint over it.  The
    // discrete adjoint through an interpolated save has its own flag (above)
    const bool v7dense = (d.flags & B200UDE_FLAG_VERN7_DENSE) != 0;
    if (v7dense && (d.solver != B200UDE_VERN7 || d.sensealg != B200UDE_INTERPOLATING_ADJOINT || fkpp))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: B200UDE_FLAG_VERN7_DENSE applies to Vern7 with the interpolating adjoint on the LV / SEIR / SEIR_NODE / NODE forms; "
                    "not to the discrete adjoint, Tsit5, RKC2 or the Fisher-KPP UPDE");
    const bool tol_ok = d.abstol > 0 && d.reltol > 0 && d.max_steps >= 1;
    if (want64) {
        // fp64: the runtime-shape one-trajectory-per-thread kernels (ude_generic.cuh in fp64, k_f64.cu): LV / SEIR / NODE forms, Tsit5 and Vern7,
        // fixed step and adaptive, interpolating or discrete adjoint; the Fisher-KPP UPDE with adaptive Tsit5 (fkpp_adaptive.cuh)
        if (!shape_ok || d.solver == B200UDE_RKC2)
            return fail(nullptr, B200UDE_EUNSUPPORTED,
                        "create: B200UDE_F64 kernels exist for the LV / SEIR / NODE forms (chain widths <= 64), Tsit5 / Vern7, and the Fisher-KPP UPDE "
                        "with adaptive Tsit5 and the interpolating adjoint");
        if (fkpp && (!adaptive || !(d.solver == B200UDE_TSIT5 || (fkpp_v7 && disc))))
            return fail(nullptr, B200UDE_EUNSUPPORTED,
                        "create: B200UDE_F64 Fisher-KPP runs adaptive Tsit5 (interpolating adjoint) and adaptive Vern7 with the discrete adjoint "
                        "only; fixed-step Fisher-KPP is fp32");
        if (adaptive && !tol_ok) return fail(nullptr, B200UDE_EINVAL, "create: adaptive stepping needs abstol > 0, reltol > 0, max_steps >= 1");
    }
    if (!want64 && d.solver == B200UDE_VERN7 && (!shape_ok || (fkpp && !(fkpp_v7 && disc))))
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: Vern7 kernels exist for the LV / SEIR / NODE forms, and for the Fisher-KPP UPDE adaptive with the discrete adjoint");
    if (!want64 && adaptive) {
        if (!tol_ok) return fail(nullptr, B200UDE_EINVAL, "create: adaptive stepping needs abstol > 0, reltol > 0, max_steps >= 1");
        if (!shape_ok)
            return fail(nullptr, B200UDE_EUNSUPPORTED, "create: adaptive stepping is implemented for the LV / SEIR / NODE forms and the Fisher-KPP UPDE (chain widths <= 64)");
        if (fkpp && d.solver != B200UDE_TSIT5 && !(fkpp_v7 && disc))
            return fail(nullptr, B200UDE_EUNSUPPORTED,
                        "create: adaptive stepping of the Fisher-KPP UPDE is implemented for Tsit5, and for Vern7 with the discrete adjoint");
    }
    if (d.solver == B200UDE_RKC2) {
        if (d.n_stages < 2 || d.n_stages > 64) return fail(nullptr, B200UDE_EINVAL, "create: RKC2 needs 2 <= n_stages <= 64 (stability interval ~ 0.65 n_stages^2 >= dt * spectral radius)");
        if (!fkpp16 || d.state_dim % 2 != 0 || adaptive || d.sensealg != B200UDE_INTERPOLATING_ADJOINT || !env_int("B200UDE_FKPP_PACKED", 1))
            return fail(nullptr, B200UDE_EUNSUPPORTED,
                        "create: RKC2 has kernels for the Fisher-KPP UPDE with the 1-16-16-1 chain on even grids (fixed step, interpolating adjoint)");
    }
    if (!shape_ok && !lv32 && !lv5)
        return fail(nullptr, B200UDE_EUNSUPPORTED,
                    "create: no sm_90a kernel for this model/chain (built: LV 2-32-32-2 tanh; LV 2-5-5-5-2; generic LV/SEIR/NODE chains with widths <= 64, <= 5 layers)");
    // every check passed: the tuned fp32 kernels where they exist, the runtime-shape kernels for the rest.  The Fisher-KPP UPDE runs
    // adaptive on grid-per-CTA kernels (fkpp_adaptive.cuh; fkpp_vern7_discrete.cuh for Vern7), the tuned 1-16-16-1 chain included
    const bool tsit5 = d.solver == B200UDE_TSIT5;
    if (fkpp && adaptive) *route = !tsit5 ? R_FKPP_VERN7_DISCRETE : (d.flags & B200UDE_FLAG_CHECKPOINT) ? R_FKPP_CHECKPOINT : R_FKPP_ADAPTIVE;
    else if (fkpp) *route = !fkpp16 ? R_FKPP_FIXED : tsit5 ? R_FKPP16 : R_FKPP16_RKC2;
    // fixed-step Tsit5 with the discrete adjoint: LV 2-32-32-2 / 2-5-5-5-2 keep their tuned kernels (the SEIR tensor-core kernels have none)
    else if (!want64 && tsit5 && !adaptive && (lv32 || lv5 || (seir64 && !disc))) *route = lv32 ? (disc ? R_LV32_DISCRETE : R_LV32) : lv5 ? R_LV5 : R_SEIR64;
    // adaptive: the headline chains on tensor-core kernels with CTA-uniform attempt loops
    else if (!want64 && tsit5 && adaptive && (lv32 || seir64) && env_int("B200UDE_ADAPTIVE_TC", 1)) *route = lv32 ? R_LV32_ADAPTIVE : R_SEIR64_ADAPTIVE;
    // fixed-step Vern7 of the SEIR 3-64-64-1 chain (and the Tsit5 re-solve its adjoint uses) on the tensor-core kernels
    else if (!want64 && d.solver == B200UDE_VERN7 && seir64 && !adaptive && !disc && !v7dense && env_int("B200UDE_SEIR_VERN7_TC", 1)) *route = R_SEIR64_VERN7;
    else if (tsit5) *route = disc ? R_DISCRETE_TSIT5 : R_TSIT5;
    else if (v7dense) *route = R_VERN7_DENSE;
    else *route = !disc ? R_VERN7 : adaptive && disc_dense ? R_VERN7_DENSE_DISCRETE : R_DISCRETE_VERN7;
    return B200UDE_OK;
}

int32_t probe_device(const b200ude_desc *d, cudaDeviceProp *prop)
{
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return fail(nullptr, B200UDE_ENODEVICE, "create: no CUDA device (%s)", cudaGetErrorString(e));
    if (d->device < 0 || d->device >= ndev) return fail(nullptr, B200UDE_EINVAL, "create: device %d of %d", d->device, ndev);
    e = cudaGetDeviceProperties(prop, d->device);
    if (e != cudaSuccess) return fail(nullptr, (int32_t)e, "create: cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop->major != 9 || prop->minor != 0)
        return fail(nullptr, B200UDE_ENODEVICE, "create: device %d is sm_%d%d; this library carries sm_90a code only", d->device, prop->major, prop->minor);
    return B200UDE_OK;
}

// partial gradient rows of the handle's adjoint kernels at max_trajectories
size_t partial_rows(const b200ude_handle *h)
{
    const int N = (int)h->cap;
    switch (h->route) {
    case R_OPERATOR: return (size_t)adj_rows_operator(N, h->oh.warps);
    case R_FORCED: return (size_t)adj_rows_forced(N, h->f64 ? 1 : 0);
    case R_LV32: case R_LV32_DISCRETE: case R_LV32_ADAPTIVE: return (size_t)std::max(adj_grid_lv32(N), adj_rows_lv32_wm(N));
    case R_LV5: return (size_t)adj_grid_lv5(N);
    case R_SEIR64: case R_SEIR64_VERN7: case R_SEIR64_ADAPTIVE: return (size_t)adj_rows_seir(N);
    case R_FKPP16: case R_FKPP16_RKC2: return (size_t)adj_rows_fkpp16(N, h->D);
    case R_FKPP_FIXED: case R_FKPP_ADAPTIVE: case R_FKPP_CHECKPOINT: case R_FKPP_VERN7_DISCRETE: return (size_t)adj_rows_fkpp(N, h->D);
    default: return (size_t)(h->f64 ? RuntimeShape<double>::adj_rows(N) : RuntimeShape<float>::adj_rows(N));
    }
}

int32_t f64_unsupported(b200ude_handle *h, const char *what)
{
    return fail(h, B200UDE_EUNSUPPORTED, "%s: not available for B200UDE_F64 handles (device-pointer forward / adjoint entry points only)", what);
}

}  // namespace

// ---- exported entry points ------------------------------------------------------------------------
extern "C" {

int32_t b200ude_version(void) { return B200UDE_ABI_VERSION; }

const char *b200ude_last_error(const b200ude_handle *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int32_t b200ude_create(const b200ude_desc *d, b200ude_handle **out)
{
    if (!d || !out) return fail(nullptr, B200UDE_EINVAL, "create: null argument");
    *out = nullptr;
    if (d->struct_size != sizeof(b200ude_desc))
        return fail(nullptr, B200UDE_EINVAL, "create: struct_size %u != %zu (ABI mismatch)", d->struct_size, sizeof(b200ude_desc));
    if (d->dtype != B200UDE_F32 && d->dtype != B200UDE_F64) return fail(nullptr, B200UDE_EINVAL, "create: unknown dtype %d", d->dtype);
    if (d->n_layers < 1 || d->n_layers > B200UDE_MAX_LAYERS) return fail(nullptr, B200UDE_EINVAL, "create: n_layers=%d out of range", d->n_layers);
    if (d->solver != B200UDE_TSIT5 && d->solver != B200UDE_VERN7 && d->solver != B200UDE_RKC2)
        return fail(nullptr, B200UDE_EINVAL, "create: unknown solver %d", d->solver);
    if (d->sensealg != B200UDE_INTERPOLATING_ADJOINT && d->sensealg != B200UDE_DISCRETE_ADJOINT)
        return fail(nullptr, B200UDE_EUNSUPPORTED, "create: unknown sensealg %d", d->sensealg);
    if (!(d->dt > 0) || d->n_steps < 1 || d->save_every < 1 || d->n_steps % d->save_every != 0)
        return fail(nullptr, B200UDE_EINVAL, "create: need dt>0, n_steps>=1, save_every>=1 dividing n_steps");
    if (d->max_trajectories == 0 || d->max_trajectories > (1ull << 26)) return fail(nullptr, B200UDE_EINVAL, "create: max_trajectories out of range");
    // the descriptor is validated before the device check, so that it is testable without a GPU
    Route route;
    int32_t rc = resolve(*d, &route);
    if (rc) return rc;
    const bool op = route == R_OPERATOR, forced = route == R_FORCED, want64 = d->dtype == B200UDE_F64;
    OperatorHost oh{};
    if (op) {
        oh.dtype = want64 ? 1 : 0; oh.D = d->state_dim; oh.M = d->widths[d->n_layers]; oh.L = d->n_layers;
        for (int l = 0; l < 6; ++l) oh.widths[l] = l <= d->n_layers ? d->widths[l] : 0;
        for (int l = 0; l < 5; ++l) oh.acts[l] = l < d->n_layers ? d->acts[l] : 0;
        oh.rkc2 = d->solver == B200UDE_RKC2 ? 1 : 0;
        oh.S = oh.rkc2 ? d->n_stages : 0;
        oh.rho = oh.rkc2 && d->adaptive ? d->consts[0] : 0.0;
        operator_layout(oh);
    }
    cudaDeviceProp prop;
    rc = probe_device(d, &prop);
    if (rc) return rc;
    const int P = op ? oh.P : num_params(d, route);
    if (route == R_FKPP_ADAPTIVE || route == R_FKPP_CHECKPOINT || route == R_FKPP_VERN7_DISCRETE) {
        // the adjoint keeps one gradient vector (P + 1 entries) per warp in shared memory: refuse here what could not launch
        const size_t smem = fkpp_adaptive_smem(d->state_dim, P, want64 ? (int)sizeof(double) : (int)sizeof(float)) + 16;   // + static
        if (smem > prop.sharedMemPerBlockOptin)
            return fail(nullptr, B200UDE_EUNSUPPORTED,
                        "create: adaptive Fisher-KPP with %d grid points and %d parameters needs %zu B of shared memory per CTA (device limit %zu B)",
                        d->state_dim, P, smem, (size_t)prop.sharedMemPerBlockOptin);
    }
    cudaError_t e = cudaSetDevice(d->device);
    if (e != cudaSuccess) return fail(nullptr, (int32_t)e, "create: cudaSetDevice: %s", cudaGetErrorString(e));
    if (op) {
        // four warps (trajectories) per CTA, fewer when their gradient vectors do not fit next to the kernels' static shared memory
        size_t stat = 0;
        e = operator_static_smem(oh.dtype, &stat);
        if (e != cudaSuccess) return fail(nullptr, (int32_t)e, "create: cudaFuncGetAttributes: %s", cudaGetErrorString(e));
        oh.dyn_cap = (int)(prop.sharedMemPerBlockOptin - stat);
        oh.warps = 4;
        while (oh.warps > 0 && operator_smem(oh, oh.warps) > (size_t)oh.dyn_cap) --oh.warps;
        if (oh.warps == 0)
            return fail(nullptr, B200UDE_EUNSUPPORTED,
                        "create: B200UDE_MODEL_OPERATOR with d = %d, m = %d and %d parameters needs %zu B of shared memory for one warp "
                        "(%zu B dynamic + %zu B static; device limit %zu B)",
                        oh.D, oh.M, oh.P, operator_smem(oh, 1) + stat, operator_smem(oh, 1), stat, (size_t)prop.sharedMemPerBlockOptin);
    }
    // the fp32 runtime-shape, Fisher-KPP and forced kernels read theta from the constant bank
    const bool tuned = route == R_LV32 || route == R_LV32_DISCRETE || route == R_LV32_ADAPTIVE || route == R_LV5 || route == R_SEIR64 ||
                       route == R_SEIR64_VERN7 || route == R_SEIR64_ADAPTIVE || route == R_FKPP16 || route == R_FKPP16_RKC2;
    if (!want64 && !tuned && !op && P > 12288)
        return fail(nullptr, B200UDE_EUNSUPPORTED, "create: %d parameters exceed the constant-bank budget", P);

    b200ude_handle *h = new (std::nothrow) b200ude_handle();
    if (!h) return fail(nullptr, B200UDE_ENOMEM, "create: out of host memory");
    const uint64_t serial = ++g_serial;   // taken once: the shape and the tables must agree
    h->desc = *d;
    h->route = route;
    h->f64 = want64;
    h->D = h->DR = d->state_dim;
    h->n_save = d->n_steps / d->save_every + 1;
    h->cap = (size_t)d->max_trajectories;
    h->sm_count = prop.multiProcessorCount;
    h->adaptive = d->adaptive != 0;
    h->P = P;
    h->oh = oh;
    h->var.approx_tanh = (d->flags & B200UDE_FLAG_APPROX_TANH) ? 1 : 0;
    h->var.discrete = d->sensealg == B200UDE_DISCRETE_ADJOINT ? 1 : 0;
    if (route == R_FKPP16_RKC2) rkc2_tables(d->n_stages, &h->rkc);
    // tuning knobs for experiments (defaults are the measured-best variant, see DESIGN.md)
    h->var.fwd_smem = env_int("B200UDE_FWD_SMEM", 0);
    // default: tensor-core (3xTF32 mma.sync) kernels; B200UDE_FWD_TC=0 / B200UDE_ADJ_TC=0 select the packed CUDA-core kernels
    h->var.fwd_tc = env_int("B200UDE_FWD_TC", 1);
    h->var.adj_tc = env_int("B200UDE_ADJ_TC", 2);   // 2: gradient GEMM on mma.sync (3xTF32), 1: on the FMA pipe
    // warp-collective mma.sync family (lv32_wm.cuh): -1 = chosen per call from the ensemble size, 0 = off, 1 = always
    h->var.fwd_wm = env_int("B200UDE_FWD_WM", -1);
    h->var.adj_wm = env_int("B200UDE_ADJ_WM", -1);
    h->var.wm_groups = env_int("B200UDE_WM_G", 0);
    h->var.wm_g2_min = h->sm_count * 4 * 2 * 32;   // 33 792 on 132 SMs
    h->var.wm_rows = env_int("B200UDE_WM_R", 0);
    h->var.wm_r1_max = env_int("B200UDE_WM_R1_MAX", h->sm_count * 4 * 8);   // one 8-trajectory warp per scheduler: 4224 on 132 SMs
    h->wm_fwd_max = (size_t)env_int("B200UDE_WM_FWD_MAX", 1 << 26);
    h->wm_adj_max = (size_t)env_int("B200UDE_WM_ADJ_MAX", 1 << 26);

    const size_t N = h->cap, D = (size_t)h->D, es = h->es();
    const size_t rec = h->adaptive ? (size_t)d->max_steps : (size_t)d->n_steps;   // capacity of the step record
    // the discrete adjoint of Vern7 and Vern7's dense output recompute the stages from u_n: no dense record, the step sizes instead
    // when adaptive
    const bool from_un = route == R_DISCRETE_VERN7 || route == R_VERN7_DENSE || route == R_VERN7_DENSE_DISCRETE || route == R_FKPP_VERN7_DISCRETE;
    const size_t dense_rows = oh.rkc2 ? rec + 1 : rec * 6 + 1;   // operator RKC2: f(u_n); Tsit5: the stages
    // R_FKPP_CHECKPOINT: u_n every K accepted steps in place of ustep, the adjoint's scratch area for one segment (6K + 1 stage
    // rows, K + 1 state rows) in place of dense, the step sizes.  K minimises max_steps / K + 7K, the rows of both
    if (route == R_FKPP_CHECKPOINT) h->seg = std::max(1, (int)std::lround(std::sqrt((double)d->max_steps / 7.0)));
    const size_t seg = (size_t)h->seg;
    const size_t ustep_rows = seg ? (rec + seg - 1) / seg + 1 : rec + 1, dense_alloc = seg ? 7 * seg + 2 : dense_rows;
    // theta: the fp32 runtime-shape and tuned kernels read it as float4
    const size_t theta_n = want64 || forced || op ? (size_t)P + 1 : (size_t)((P + 3) / 4) * 4;
    h->partial_blocks = partial_rows(h);
    bool ok = dalloc_real(h, &h->d_theta, theta_n) == cudaSuccess && dalloc_real(h, &h->d_ustep, ustep_rows * D * N) == cudaSuccess &&
              (from_un || dalloc_real(h, &h->d_dense, dense_alloc * D * N) == cudaSuccess) &&
              dalloc_real(h, &h->d_partial, h->partial_blocks * (size_t)(P + 1)) == cudaSuccess;
    if (!want64) ok = ok && dalloc(h, &h->d_grad, (size_t)P) == cudaSuccess && dalloc(h, &h->d_loss, 1) == cudaSuccess;
    if (h->adaptive) {
        ok = ok && dalloc_real(h, &h->d_tgrid, (rec + 1) * N) == cudaSuccess && dalloc(h, &h->d_nacc, N) == cudaSuccess;
        if (forced || op)   // the saved states of the last forward, read by the replay adjoint
            ok = ok && dalloc_real(h, &h->d_usave, (size_t)h->n_save * D * N) == cudaSuccess;
        else   // the cotangent of the fused L2 and, in fp32, its per-block losses
            ok = ok && dalloc_real(h, &h->d_cot, (size_t)h->n_save * D * N) == cudaSuccess &&
                 (!(from_un || seg) || dalloc_real(h, &h->d_hstep, rec * N) == cudaSuccess) &&
                 (want64 || dalloc(h, &h->d_block_loss, (size_t)L2_BLOCKS) == cudaSuccess);
    }
    if (forced) ok = ok && dalloc_real(h, &h->d_forcing, 3 * (size_t)d->consts[1] * N) == cudaSuccess;
    // operator RKC2 tables: one block for n_stages; adaptive, one block per stage count 2..n_stages and then beta[0..64]
    const bool op_ark = op && oh.rkc2 && h->adaptive;
    const size_t rkc_n = op_ark ? (size_t)(oh.S - 1) * op_rkc_len() + 65 : (size_t)op_rkc_len();
    if (op) ok = ok && dalloc_real(h, &h->d_ops, (size_t)oh.ops_elems) == cudaSuccess && (!oh.rkc2 || dalloc_real(h, &h->d_rkc, rkc_n) == cudaSuccess);
    if (op_ark) ok = ok && dalloc(h, &h->d_sstep, (size_t)d->max_steps * N) == cudaSuccess;
    if (ok) ok = cudaMemset(h->d_theta, 0, es * theta_n) == cudaSuccess;
    if (ok && op) {
        // the loss weights in front of the operator block; the operators follow in b200ude_set_operators
        std::vector<double> w64(oh.ops_elems, 0.0);
        for (int c = 0; c < 64; ++c) w64[c] = c < oh.D ? (d->n_loss_weights > 0 ? d->loss_weights[c] : 1.0) : 0.0;
        ok = upload_as(h->d_ops, w64.data(), w64.size(), want64) == cudaSuccess;
        if (ok && oh.rkc2) {
            std::vector<double> t(rkc_n, 0.0);
            for (int s = op_ark ? 2 : oh.S; s <= oh.S; ++s) {
                double *b = &t[op_ark ? (size_t)(s - 2) * op_rkc_len() : 0];
                rkc2_tables64(s, b[0], &b[op_rkc_off(2)], &b[op_rkc_off(3)], &b[op_rkc_off(4)], &b[op_rkc_off(5)], &b[op_rkc_off(0)], &b[op_rkc_off(1)]);
            }
            if (op_ark)
                for (int s = 2; s <= 64; ++s) t[(size_t)(oh.S - 1) * op_rkc_len() + s] = rkc2_beta64(s);
            ok = upload_as(h->d_rkc, t.data(), t.size(), want64) == cudaSuccess;
        }
    }
    if (!ok) {
        g_create_error = std::string("create: device allocation failed: ") + cudaGetErrorString(cudaGetLastError());
        b200ude_destroy(h);
        return B200UDE_ENOMEM;
    }
    if (cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->data_ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->data_ready2, cudaEventDisableTiming) != cudaSuccess ||
        (!want64 && cudaMallocHost((void **)&h->h_loss, sizeof(float)) != cudaSuccess)) {
        g_create_error = "create: stream / pinned allocation failed";
        b200ude_destroy(h);
        return B200UDE_ENOMEM;
    }

    // the shape and tables the kernels read
    GenericShape &g = h->gen;
    g.serial = serial;
    g.model = d->model; g.D = d->state_dim; g.din = d->widths[0]; g.dout = d->widths[d->n_layers];
    g.n_layers = d->n_layers; g.n_prefix = d->n_prefix; g.P = P;
    for (int l = 0; l < 8; ++l) { g.widths[l] = l <= d->n_layers ? d->widths[l] : 0; g.acts[l] = l < d->n_layers ? d->acts[l] : 0; }
    h->tab.serial = serial;
    h->tab.d_theta = (const float *)h->d_theta;
    h->tab.P = P;
    h->tab64.theta = (const double *)h->d_theta;
    for (int i = 0; i < 16; ++i) {
        h->tab64.consts[i] = i < d->n_consts ? d->consts[i] : 0.0;
        h->tab64.lossw[i] = d->n_loss_weights > 0 ? (i < d->n_loss_weights ? d->loss_weights[i] : 0.0) : 1.0;
        h->tab.consts[i] = (float)h->tab64.consts[i];
        h->tab.lossw[i] = (float)h->tab64.lossw[i];
    }
    for (int i = 0; i < 8; ++i) h->tab.acts[i] = i < d->n_layers ? d->acts[i] : 0;
    if (forced) {   // both chains back to back
        ForcedHost &f = h->fh;
        const int L0 = (int)d->consts[0];
        h->DR = d->state_dim + d->widths[L0];
        f.serial = serial; f.dtype = want64 ? 1 : 0; f.D = d->state_dim; f.R = d->widths[L0]; f.J = (int)d->consts[1]; f.L0 = L0;
        f.L1 = d->n_layers - L0; f.P = P;
        for (int l = 0; l < 8; ++l) {
            f.widths[l] = l <= d->n_layers + 1 ? d->widths[l] : 0;
            f.acts[l] = l < d->n_layers ? d->acts[l] : 0;
        }
        for (int i = 0; i < 16; ++i) f.lossw[i] = h->tab64.lossw[i];
        f.theta = h->d_theta;
    }
    h->oh.theta = h->d_theta;
    h->oh.ops = h->d_ops;
    h->oh.rkc = h->d_rkc;
    h->oh.beta = op_ark ? (const void *)((const unsigned char *)h->d_rkc + es * (size_t)(oh.S - 1) * op_rkc_len()) : nullptr;
    *out = h;
    return B200UDE_OK;
}

void b200ude_destroy(b200ude_handle *h)
{
    if (!h) return;
    cudaFree(h->d_theta); cudaFree(h->d_ustep); cudaFree(h->d_dense); cudaFree(h->d_partial);
    cudaFree(h->d_u0); cudaFree(h->d_out); cudaFree(h->d_data); cudaFree(h->d_gu0); cudaFree(h->d_grad);
    cudaFree(h->d_loss); cudaFree(h->d_status);
    b200ude_peer_detach(h);
    cudaFree(h->d_peer_buf);
    cudaFree(h->d_u0_keep); cudaFree(h->d_aux_out);
    cudaFree(h->d_adam_m); cudaFree(h->d_adam_v); cudaFree(h->d_adam_t); cudaFree(h->d_train_out);
    cudaFree(h->d_tgrid); cudaFree(h->d_nacc); cudaFree(h->d_cot); cudaFree(h->d_block_loss); cudaFree(h->d_hstep);
    cudaFree(h->d_forcing); cudaFree(h->d_usave);
    cudaFree(h->d_ops); cudaFree(h->d_rkc); cudaFree(h->d_sstep);
    if (h->h_loss) cudaFreeHost(h->h_loss);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->data_ready) cudaEventDestroy(h->data_ready);
    if (h->data_ready2) cudaEventDestroy(h->data_ready2);
    delete h;
}

size_t b200ude_num_params(const b200ude_handle *h) { return h ? (size_t)h->P : 0; }
size_t b200ude_num_save(const b200ude_handle *h) { return h ? (size_t)h->n_save : 0; }
size_t b200ude_device_bytes(const b200ude_handle *h) { return h ? h->dev_bytes : 0; }

int32_t b200ude_set_params(b200ude_handle *h, const void *theta, size_t P, int32_t mem, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (!theta || P != (size_t)h->P) return fail(h, B200UDE_EINVAL, "set_params: P=%zu, expected %d", P, h->P);
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(h, cudaMemcpyAsync(h->d_theta, theta, h->es() * P, mem == B200UDE_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    h->have_theta = true;
    return B200UDE_OK;
}

int32_t b200ude_set_forcing(b200ude_handle *h, const void *coef, size_t N, int32_t mem, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (h->route != R_FORCED) return fail(h, B200UDE_EUNSUPPORTED, "set_forcing: only B200UDE_MODEL_FORCED handles take a forcing (this handle: model %d)", h->desc.model);
    if (!coef || N == 0 || N > h->cap) return fail(h, B200UDE_EINVAL, "set_forcing: null pointer or N=%zu outside (0, max_trajectories=%zu]", N, h->cap);
    CUDA_TRY(h, cudaSetDevice(h->desc.device));
    const size_t es = h->es();
    CUDA_TRY(h, cudaMemcpy2DAsync(h->d_forcing, es * h->cap, coef, es * N, es * N, (size_t)3 * h->fh.J,
                                  mem == B200UDE_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, (cudaStream_t)stream));
    // the kernels run on s = t - t0: cos(W t + F) = cos(W s + (F + W t0)).  t0 = 0 leaves the coefficients as given.
    if (h->desc.t0 != 0) CUDA_TRY(h, launch_fold_forcing(h->fh.dtype, h->d_forcing, h->fh.J, (int)h->cap, (int)N, h->desc.t0, (cudaStream_t)stream));
    h->forcing_n = N;
    return B200UDE_OK;
}

int32_t b200ude_set_operators(b200ude_handle *h, const void *D1, const void *D2, int32_t mem, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (h->route != R_OPERATOR) return fail(h, B200UDE_EUNSUPPORTED, "set_operators: only B200UDE_MODEL_OPERATOR handles take operators (this handle: model %d)", h->desc.model);
    if (!D1) return fail(h, B200UDE_EINVAL, "set_operators: D1 is a null pointer");
    CUDA_TRY(h, cudaSetDevice(h->desc.device));
    const OperatorHost &o = h->oh;
    const size_t es = o.dtype == 1 ? sizeof(double) : sizeof(float);
    const cudaMemcpyKind kind = mem == B200UDE_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    // column-major d x m and d x d into the padded block: column k at (64 + k ld) elements
    unsigned char *base = (unsigned char *)h->d_ops + es * 64;
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(h, cudaMemcpy2DAsync(base, es * o.ld1, D1, es * o.D, es * o.D, (size_t)o.M, kind, st));
    if (D2) CUDA_TRY(h, cudaMemcpy2DAsync(base + es * o.ld1 * o.M, es * o.ld2, D2, es * o.D, es * o.D, (size_t)o.D, kind, st));
    h->oh.has_d2 = D2 ? 1 : 0;
    h->ops_set = true;
    return B200UDE_OK;
}

int32_t b200ude_forward(b200ude_handle *h, const void *u0, size_t N, void *out, int32_t *status, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (h->f64) return do_forward(h, (const double *)u0, N, (double *)out, status, (cudaStream_t)stream);
    return do_forward(h, (const float *)u0, N, (float *)out, status, (cudaStream_t)stream);
}

int32_t b200ude_adjoint(b200ude_handle *h, const void *dL_dout, void *grad_theta, void *grad_u0, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (h->f64) return do_adjoint<double>(h, false, (const double *)dL_dout, nullptr, (double *)grad_theta, (double *)grad_u0, (cudaStream_t)stream);
    return do_adjoint<float>(h, false, (const float *)dL_dout, nullptr, (float *)grad_theta, (float *)grad_u0,
                      (cudaStream_t)stream);
}

int32_t b200ude_adjoint_l2(b200ude_handle *h, const void *data, void *loss, void *grad_theta, void *grad_u0, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (h->f64) return do_adjoint(h, true, (const double *)data, (double *)loss, (double *)grad_theta, (double *)grad_u0, (cudaStream_t)stream);
    return do_adjoint(h, true, (const float *)data, (float *)loss, (float *)grad_theta, (float *)grad_u0,
                      (cudaStream_t)stream);
}

// ---- host-buffer entry points -------------------------------------------------------------------
static int32_t ensure_host_path(b200ude_handle *h)
{
    if (h->d_u0) return B200UDE_OK;
    const size_t N = h->cap, D = (size_t)h->D;
    bool ok = true;
    ok = ok && dalloc(h, &h->d_u0, D * N) == cudaSuccess;
    ok = ok && dalloc(h, &h->d_out, (size_t)h->n_save * h->DR * N) == cudaSuccess;
    ok = ok && dalloc(h, &h->d_data, (size_t)h->n_save * h->DR * N) == cudaSuccess;
    ok = ok && dalloc(h, &h->d_gu0, D * N) == cudaSuccess;
    ok = ok && dalloc(h, &h->d_status, N) == cudaSuccess;
    if (!ok) return fail(h, B200UDE_ENOMEM, "host path: device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    return B200UDE_OK;
}

int32_t b200ude_solve_host(b200ude_handle *h, const void *theta, const void *u0, size_t N, void *out, int32_t *status)
{
    if (!h) return B200UDE_EINVAL;
    if (h->f64) return f64_unsupported(h, "solve_host");
    if (!theta || !u0 || !out) return fail(h, B200UDE_EINVAL, "solve_host: null pointer");
    if (N == 0 || N > h->cap) return fail(h, B200UDE_EINVAL, "solve_host: N=%zu outside (0, %zu]", N, h->cap);
    int32_t rc = ensure_host_path(h);
    if (rc) return rc;
    cudaStream_t st = h->own_stream;
    const size_t D = (size_t)h->D;
    rc = b200ude_set_params(h, theta, (size_t)h->P, B200UDE_HOST, st);
    if (rc) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(h->d_u0, u0, sizeof(float) * D * N, cudaMemcpyHostToDevice, st));
    rc = do_forward(h, h->d_u0, N, h->d_out, status ? h->d_status : nullptr, st);
    if (rc) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(out, h->d_out, sizeof(float) * (size_t)h->n_save * h->DR * N, cudaMemcpyDeviceToHost, st));
    if (status) CUDA_TRY(h, cudaMemcpyAsync(status, h->d_status, sizeof(int32_t) * N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(h, cudaStreamSynchronize(st));
    return B200UDE_OK;
}

int32_t b200ude_loss_gradient_host(b200ude_handle *h, const void *theta, const void *u0, const void *data, size_t N,
                                   double *loss, void *grad_theta, void *grad_u0)
{
    if (!h) return B200UDE_EINVAL;
    if (h->f64) return f64_unsupported(h, "loss_gradient_host");
    if (!theta || !u0 || !data || !grad_theta) return fail(h, B200UDE_EINVAL, "loss_gradient_host: null pointer");
    if (N == 0 || N > h->cap) return fail(h, B200UDE_EINVAL, "loss_gradient_host: N=%zu outside (0, %zu]", N, h->cap);
    int32_t rc = ensure_host_path(h);
    if (rc) return rc;
    cudaStream_t st = h->own_stream;
    const size_t D = (size_t)h->D;
    rc = b200ude_set_params(h, theta, (size_t)h->P, B200UDE_HOST, st);
    if (rc) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(h->d_u0, u0, sizeof(float) * D * N, cudaMemcpyHostToDevice, st));
    // the data (n_save x larger than u0) is only needed by the adjoint: upload it on a second stream while
    // the forward kernel runs (pinned host memory makes the two overlap)
    // ... in two halves of the trajectories (strided copies: the layout is trajectory-fastest), so that the adjoint of the first half
    // can start under the second half's upload when the link is slower than the forward kernel
    const size_t half = N >= 8192 ? ((N / 2 + 15) / 16) * 16 : N;
    const size_t rows = (size_t)h->n_save * h->DR;
    CUDA_TRY(h, cudaMemcpy2DAsync(h->d_data, sizeof(float) * N, data, sizeof(float) * N, sizeof(float) * half, rows, cudaMemcpyHostToDevice, h->copy_stream));
    CUDA_TRY(h, cudaEventRecord(h->data_ready, h->copy_stream));
    if (half < N)
        CUDA_TRY(h, cudaMemcpy2DAsync(h->d_data + half, sizeof(float) * N, (const float *)data + half, sizeof(float) * N, sizeof(float) * (N - half), rows,
                                      cudaMemcpyHostToDevice, h->copy_stream));
    CUDA_TRY(h, cudaEventRecord(h->data_ready2, h->copy_stream));
    rc = do_forward(h, h->d_u0, N, h->d_out, nullptr, st);
    if (rc) return rc;
    const cudaEvent_t ev[2] = {h->data_ready, h->data_ready2};
    rc = do_adjoint(h, true, h->d_data, h->d_loss, h->d_grad, grad_u0 ? h->d_gu0 : nullptr, st, false, ev, half);
    if (rc) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(grad_theta, h->d_grad, sizeof(float) * (size_t)h->P, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(h, cudaMemcpyAsync(h->h_loss, h->d_loss, sizeof(float), cudaMemcpyDeviceToHost, st));
    if (grad_u0) CUDA_TRY(h, cudaMemcpyAsync(grad_u0, h->d_gu0, sizeof(float) * D * N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(h, cudaStreamSynchronize(st));
    if (loss) *loss = (double)*h->h_loss;
    return B200UDE_OK;
}

// ---- on-device optimiser ---------------------------------------------------------------------------
int32_t b200ude_get_params(b200ude_handle *h, void *theta, size_t P, int32_t mem, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (!theta || P != (size_t)h->P) return fail(h, B200UDE_EINVAL, "get_params: P=%zu, expected %d", P, h->P);
    CUDA_TRY(h, cudaMemcpyAsync(theta, h->d_theta, h->es() * P, mem == B200UDE_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                                (cudaStream_t)stream));
    if (mem != B200UDE_DEVICE) CUDA_TRY(h, cudaStreamSynchronize((cudaStream_t)stream));
    return B200UDE_OK;
}

int32_t b200ude_adam_reset(b200ude_handle *h, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    int32_t rc = ensure_adam(h);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(h, cudaMemsetAsync(h->d_adam_m, 0, sizeof(float) * h->P, st));
    CUDA_TRY(h, cudaMemsetAsync(h->d_adam_v, 0, sizeof(float) * h->P, st));
    CUDA_TRY(h, cudaMemsetAsync(h->d_adam_t, 0, sizeof(int), st));
    h->adam_t = 0;
    return B200UDE_OK;
}

int32_t b200ude_adam_step(b200ude_handle *h, const b200ude_adam *opt, const void *grad_theta, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (!grad_theta) return fail(h, B200UDE_EINVAL, "adam_step: null gradient");
    int32_t rc = check_adam(h, opt);
    if (rc) return rc;
    CUDA_TRY(h, launch_adam(h, opt, (const float *)grad_theta, nullptr, nullptr, h->adam_t, (cudaStream_t)stream));
    h->adam_t += 1;
    return B200UDE_OK;
}

int32_t b200ude_train_adam(b200ude_handle *h, const b200ude_adam *opt, const void *u0, const void *data, size_t N,
                           int32_t iters, void *loss_history, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    if (!u0 || !data || iters < 1) return fail(h, B200UDE_EINVAL, "train_adam: null pointer or iters < 1");
    if (N == 0 || N > h->cap) return fail(h, B200UDE_EINVAL, "train_adam: N=%zu outside (0, %zu]", N, h->cap);
    int32_t rc = check_adam(h, opt);
    if (rc) return rc;
    if (!h->d_train_out && dalloc(h, &h->d_train_out, (size_t)h->n_save * (size_t)h->DR * h->cap) != cudaSuccess)
        return fail(h, B200UDE_ENOMEM, "train_adam: device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    cudaStream_t st = stream ? (cudaStream_t)stream : h->own_stream;   // the legacy default stream cannot be captured
    if (!stream) {
        // own_stream is non-blocking: order it after everything the caller enqueued on the legacy default stream (set_params,
        // adam_reset, the producers of u0 / data); the call synchronises own_stream before it returns
        CUDA_TRY(h, cudaEventRecord(h->data_ready, (cudaStream_t)0));
        CUDA_TRY(h, cudaStreamWaitEvent(h->own_stream, h->data_ready, 0));
    }
    const int t_base = h->adam_t;
    auto one_iteration = [&]() -> int32_t {
        int32_t r = do_forward(h, (const float *)u0, N, h->d_train_out, nullptr, st);
        if (r) return r;
        // with peers attached (b200ude_peer_attach) the gradient and the loss are the sums over all ranks: every rank runs the
        // same iterations in lock step and applies the identical update to its replica of theta
        r = do_adjoint<float>(h, true, (const float *)data, h->d_loss, h->d_grad, nullptr, st, h->peer_attached);
        if (r) return r;
        CUDA_TRY(h, launch_adam(h, opt, h->d_grad, h->d_loss, (float *)loss_history, t_base, st));
        return B200UDE_OK;
    };
    // iteration 1 eagerly (one-time function attributes, constant tables), the rest as replays of one captured graph
    rc = one_iteration();
    if (rc) return rc;
    if (iters > 1) {
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        bool graphed = false;
        if (env_int("B200UDE_TRAIN_GRAPH", 1) && cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            const int32_t r = one_iteration();
            const cudaError_t ce = cudaStreamEndCapture(st, &graph);
            if (r == B200UDE_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) graphed = true;
            else cudaGetLastError();
        }
        for (int it = 1; it < iters; ++it) {
            if (graphed) CUDA_TRY(h, cudaGraphLaunch(exec, st));
            else if ((rc = one_iteration()) != 0) break;   // same kernels, launched one by one
        }
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        if (rc) return rc;
    }
    h->adam_t = t_base + iters;
    if (!stream) CUDA_TRY(h, cudaStreamSynchronize(st));
    return B200UDE_OK;
}

// ---- multi-GPU: fused final reduction + all-reduce over NVLink peer memory ------------------------------------
static size_t peer_buf_bytes(const b200ude_handle *h)
{
    const size_t P1pad = (size_t)((h->P + 1 + 31) / 32) * 32;
    return (size_t)PEER_HEADER_BYTES + sizeof(float) * 2 * 16 * P1pad;
}

int32_t b200ude_peer_export(b200ude_handle *h, void *handle_out)
{
    if (!h) return B200UDE_EINVAL;
    if (h->f64) return fail(h, B200UDE_EUNSUPPORTED, "peer_export: not available for B200UDE_F64 handles (all-reduce the result of b200ude_adjoint_l2)");
    if (!handle_out) return fail(h, B200UDE_EINVAL, "peer_export: null pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == B200UDE_PEER_HANDLE_BYTES, "CUDA IPC handle size");
    if (!h->d_peer_buf) {
        CUDA_TRY(h, cudaMalloc(&h->d_peer_buf, peer_buf_bytes(h)));
        h->dev_bytes += peer_buf_bytes(h);
        CUDA_TRY(h, cudaMemset(h->d_peer_buf, 0, peer_buf_bytes(h)));
        CUDA_TRY(h, cudaDeviceSynchronize());
    }
    cudaIpcMemHandle_t ipc;
    CUDA_TRY(h, cudaIpcGetMemHandle(&ipc, h->d_peer_buf));
    memcpy(handle_out, &ipc, sizeof(ipc));
    return B200UDE_OK;
}

int32_t b200ude_peer_attach(b200ude_handle *h, int32_t rank, int32_t world, const void *handles)
{
    if (!h) return B200UDE_EINVAL;
    if (!handles || world < 1 || world > 16 || rank < 0 || rank >= world) return fail(h, B200UDE_EINVAL, "peer_attach: need 1 <= world <= 16, 0 <= rank < world");
    if (!h->d_peer_buf) return fail(h, B200UDE_ESTATE, "peer_attach: call b200ude_peer_export first");
    if (h->peer_attached) return fail(h, B200UDE_ESTATE, "peer_attach: already attached");
    for (int r = 0; r < 16; ++r) h->peer.base[r] = nullptr;
    for (int r = 0; r < world; ++r) {
        if (r == rank) { h->peer.base[r] = h->d_peer_buf; continue; }
        cudaIpcMemHandle_t ipc;
        memcpy(&ipc, (const char *)handles + (size_t)r * sizeof(ipc), sizeof(ipc));
        cudaError_t e = cudaIpcOpenMemHandle(&h->peer.base[r], ipc, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            for (int q = 0; q < r; ++q) if (q != rank && h->peer.base[q]) cudaIpcCloseMemHandle(h->peer.base[q]);
            return fail(h, (int32_t)e, "peer_attach: cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
        }
    }
    h->peer.rank = rank; h->peer.world = world; h->peer.P1pad = ((h->P + 1 + 31) / 32) * 32;
    h->peer_attached = true;
    return B200UDE_OK;
}

int32_t b200ude_peer_detach(b200ude_handle *h)
{
    if (!h) return B200UDE_EINVAL;
    if (h->peer_attached)
        for (int r = 0; r < h->peer.world; ++r)
            if (r != h->peer.rank && h->peer.base[r]) cudaIpcCloseMemHandle(h->peer.base[r]);
    h->peer_attached = false;
    return B200UDE_OK;
}

int32_t b200ude_adjoint_l2_allreduce(b200ude_handle *h, const void *data, void *loss, void *grad_theta, void *grad_u0, void *stream)
{
    if (!h) return B200UDE_EINVAL;
    return do_adjoint(h, true, (const float *)data, (float *)loss, (float *)grad_theta, (float *)grad_u0, (cudaStream_t)stream, true);
}

int32_t b200ude_selftest_tanh(int32_t device, const void *x, void *y, size_t n, void *stream)
{
    if (!x || !y || n == 0) return fail(nullptr, B200UDE_EINVAL, "selftest_tanh: null pointer or n == 0");
    CUDA_TRY(nullptr, cudaSetDevice(device));
    CUDA_TRY(nullptr, launch_tanh_selftest((const float *)x, (float *)y, n, (cudaStream_t)stream));
    return B200UDE_OK;
}

}  // extern "C"
