// params.h -- plain structs shared by the C-ABI layer and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace b200ude {

// model and activation codes (B200UDE_MODEL_*, B200UDE_ACT_*)
constexpr int MODEL_LV = 0, MODEL_SEIR = 1, MODEL_FKPP = 2, MODEL_NODE = 3, MODEL_SEIR_NODE = 4, MODEL_FORCED = 5;
constexpr int ACT_IDENTITY = 0, ACT_TANH = 1, ACT_RBF = 2;

struct FwdParams {
    const float *u0;    // [D][N]
    float *out;         // [n_save][D][N]
    float *ustep;       // [n_steps+1][D][N]  state at every step start (adjoint's interpolation base)
    float *dense;       // [n_steps*6+1][D][N] stage derivatives: row n*6+i = k_{i+1} of step n; k_7(n) = k_1(n+1)
    int32_t *status;    // [N] or nullptr
    const float *theta; // device copy of theta (shared-memory weight variant only)
    int N, n_steps, save_every, P;
    float dt;
};

struct AdjParams {
    const float *ustep;   // [n_steps+1][D][N]
    const float *dense;   // [n_steps*6+1][D][N]
    const float *cot;     // fused_l2 ? data [n_save][D][N] : dL/dout [n_save][D][N]
    float *grad_u0;       // [D][N] or nullptr
    float *partial;       // [gridDim.x][P+1]  per-CTA partial gradient, last entry = partial loss
    const float *theta;   // device theta (shared-memory weight variant only)
    int N, n_steps, save_every, P;
    int fused_l2;         // 1: cot is the data, form 2 w (u - data) and the loss in-kernel
    float dt;
    // sub-range launches (warp-collective LV kernels only): trajectories [n0, n0 + n_cnt) of the N, partial rows from row0
    // (n_cnt = 0: all N).  Lets the host-buffer path start the adjoint of the first half while the second half's data still uploads.
    int n0 = 0, n_cnt = 0, row0 = 0;
};

// per-handle tables every launch pushes into the launching translation unit's constant bank
struct ConstTables {
    uint64_t serial;  // unique per handle: the small tables are re-sent only when it changes
    const float *d_theta;
    int P;
    float consts[16];
    float lossw[16];
    int acts[8];
};

struct Variant {
    int fwd_smem = 0;    // packed LV32 forward: 0 = constant-bank weights, 1 = shared-memory weights
    int approx_tanh = 0;
    int fwd_tc = 0;      // 1: tensor-core (3xTF32 mma.sync) forward kernel
    int adj_tc = 0;      // 1: tensor-core (3xTF32 mma.sync) adjoint kernel, FFMA gradient GEMM; 2: mma.sync gradient GEMM
    int discrete = 0;    // 1: discrete adjoint (exact gradient of the fixed-step scheme) instead of the interpolating adjoint
    int fwd_wm = 0;      // 1: warp-collective mma.sync forward kernel (lv32_wm.cuh)
    int adj_wm = 0;      // 1: warp-collective mma.sync adjoint kernel
    int wm_groups = 0;   // groups per warp in the warp-collective forward kernel: 1, 2, or 0 = by ensemble size (>= wm_g2_min -> 2)
    int wm_g2_min = 0;   // two groups per warp once that still leaves two warps per scheduler (SMs x 4 x 2 x 32; b200ude_create)
    int wm_rows = 0;     // trajectories per group / 8: 1, 2, or 0 = by ensemble size (<= wm_r1_max -> 1)
    int wm_r1_max = 0;      // 8 trajectories per warp while that still leaves one warp per scheduler (SMs x 4 x 8; b200ude_create)
};

// function attributes (dynamic shared-memory size) are per device: one-time flags are kept per device ordinal
struct PerDeviceOnce {
    bool done[64] = {};
    bool &flag()
    {
        int dev = 0;
        cudaGetDevice(&dev);
        return done[dev & 63];
    }
};

// "which handle's small tables are in this device's constant bank": the bank is per device, so the cache is too
// (one host thread per GPU may create and drive handles concurrently)
struct SerialCache {
    std::atomic<uint64_t> last[64] = {};
    static int dev()
    {
        int d = 0;
        cudaGetDevice(&d);
        return d & 63;
    }
    bool hit(uint64_t serial) const { return last[dev()].load(std::memory_order_acquire) == serial; }
    void set(uint64_t serial) { last[dev()].store(serial, std::memory_order_release); }
};

constexpr int FWD_BLOCK = 128;      // small-chain forward kernels
constexpr int FWD_BLOCK_LV32 = 32;  // packed LV32 forward: one warp (64 trajectories) per CTA -> even spread over the SMs
constexpr int ADJ_BLOCK_GEMM = 32;   // H=32 adjoint: one warp (64 trajectories) per CTA
constexpr int ADJ_BLOCK_LANE = 128;  // small-chain adjoint

// runtime shape of a UDE handled by the generic kernels (k_generic.cu)
struct GenericShape {
    uint64_t serial;
    int model, D, din, dout, n_layers, n_prefix, P;
    int widths[8];
    int acts[8];
};

// adaptive stepping: save grid + tolerances + the per-trajectory record of accepted steps
struct AdaptiveGrid {
    float t0, save_dt, abstol, reltol;
    int n_save, max_steps;
    float *tgrid;   // [max_steps+1][N]
    int *nacc;      // [N]
    float *hstep;   // [max_steps][N] step sizes (discrete-adjoint Vern7 and checkpointed Fisher-KPP handles only, else nullptr)
};
constexpr int L2_BLOCKS = 296;

// launchers (one translation unit per kernel family; each owns its constant-bank symbols)
cudaError_t launch_fwd_lv32(const Variant &, const ConstTables &, const FwdParams &, cudaStream_t);
cudaError_t launch_adj_lv32(const Variant &, const ConstTables &, const AdjParams &, cudaStream_t, int *grid_out);
cudaError_t launch_fwd_lv5(int n_prefix, const Variant &, const ConstTables &, const FwdParams &, cudaStream_t);
cudaError_t launch_adj_lv5(int n_prefix, const Variant &, const ConstTables &, const AdjParams &, cudaStream_t, int *grid_out);
int adj_grid_lv32(int N);
cudaError_t launch_fwd_lv32_wm(const Variant &, const ConstTables &, const FwdParams &, cudaStream_t);
cudaError_t launch_adj_lv32_wm(const Variant &, const ConstTables &, const AdjParams &, cudaStream_t, int *rows_out);
int adj_rows_lv32_wm(int N);
cudaError_t launch_tanh_selftest(const float *x, float *y, size_t n, cudaStream_t);
cudaError_t launch_fwd_lv32_adaptive(const Variant &, const ConstTables &, const FwdParams &, const AdaptiveGrid &, cudaStream_t);
cudaError_t launch_adj_lv32_adaptive(const Variant &, const ConstTables &, const AdjParams &, const AdaptiveGrid &, cudaStream_t, int *rows_out);
int adj_grid_lv5(int N);
cudaError_t launch_l2_cot(const ConstTables &, const float *out, const float *data, float *cot, float *block_loss, int D, size_t N, int n_save, cudaStream_t);
cudaError_t launch_l2_finish(const float *block_loss, float *loss, cudaStream_t);
cudaError_t launch_fwd_fkpp(const GenericShape &, const ConstTables &, const FwdParams &, cudaStream_t);
cudaError_t launch_adj_fkpp(const GenericShape &, const ConstTables &, const AdjParams &, cudaStream_t, int *rows_out);
int adj_rows_fkpp(int N, int Nx);
size_t fkpp_adaptive_smem(int Nx, int P, int real_bytes);   // per-CTA dynamic shared memory of the larger of the two adaptive kernels
cudaError_t launch_fwd_seir(const Variant &, const ConstTables &, const FwdParams &, cudaStream_t);
cudaError_t launch_adj_seir(const Variant &, const ConstTables &, const AdjParams &, cudaStream_t, int *rows_out);
cudaError_t launch_fwd_seir_vern7(const Variant &, const ConstTables &, const FwdParams &, cudaStream_t);
int adj_rows_seir(int N);
cudaError_t launch_fwd_seir_adaptive(const Variant &, const ConstTables &, const FwdParams &, const AdaptiveGrid &, cudaStream_t);
cudaError_t launch_adj_seir_adaptive(const Variant &, const ConstTables &, const AdjParams &, const AdaptiveGrid &, cudaStream_t, int *rows_out);
// RKC2 recurrence tables of a handle (computed on the host, b200ude.cu)
struct RkcHost {
    int s = 0;
    float mt1 = 0;
    float mu[65] = {}, nu[65] = {}, mt[65] = {}, ga[65] = {}, c[65] = {}, w[65] = {};
};
cudaError_t launch_fwd_fkpp16_rkc(const Variant &, const ConstTables &, const RkcHost &, const FwdParams &, int Nx, cudaStream_t);
cudaError_t launch_adj_fkpp16_rkc(const Variant &, const ConstTables &, const RkcHost &, const AdjParams &, int Nx, cudaStream_t, int *rows_out);
cudaError_t launch_fwd_fkpp16(const Variant &, const ConstTables &, const FwdParams &, int Nx, cudaStream_t);
cudaError_t launch_adj_fkpp16(const Variant &, const ConstTables &, const AdjParams &, int Nx, cudaStream_t, int *rows_out);
int adj_rows_fkpp16(int N, int Nx);
// exchange buffers of the fused reduce + all-reduce (ude_adjoint.cuh): every rank's buffer as mapped in this process
constexpr int PEER_HEADER_BYTES = 256;   // flags[16], ticket, padding
struct PeerLinks {
    void *base[16];
    int rank = 0, world = 0, P1pad = 0;
};
cudaError_t launch_reduce_exchange(const float *partial, int nblocks, int P1, const PeerLinks &, float *grad, float *loss, cudaStream_t);
cudaError_t launch_reduce(const float *partial, int nblocks, int P1, float *grad, float *loss, cudaStream_t);

// ---- the runtime-shape kernels (ude_generic.cuh and the headers written over its Ops) in both precisions: fp32 (k_generic.cu) and
// fp64 (dtype = B200UDE_F64, k_f64.cu).  Fwd64Host / Adj64Host / Adapt64Host are the parameters of the fp64 kernels, as FwdParams /
// AdjParams / AdaptiveGrid are of the fp32 ones ----
struct Tables64 {   // fp64 counterpart of ConstTables: theta, constants and loss weights of a handle
    const double *theta;
    double consts[16], lossw[16];
};
struct Fwd64Host {
    const double *u0;
    double *out, *ustep, *dense;
    int32_t *status;
    int N, n_steps, save_every;
    double dt;
};
struct Adj64Host {
    const double *ustep, *dense, *cot;
    double *grad_u0, *partial;
    int N, n_steps, save_every, fused_l2;
    double dt;
};
struct Adapt64Host {
    double t0, save_dt, abstol, reltol;
    int n_save, max_steps;
    double *tgrid;
    int *nacc;
    double *hstep;   // discrete-adjoint Vern7 and checkpointed Fisher-KPP handles only, else nullptr
};
template <typename R>
struct RealParams;
template <>
struct RealParams<float> {
    using Tab = ConstTables;
    using Fwd = FwdParams;
    using Adj = AdjParams;
    using Adapt = AdaptiveGrid;
};
template <>
struct RealParams<double> {
    using Tab = Tables64;
    using Fwd = Fwd64Host;
    using Adj = Adj64Host;
    using Adapt = Adapt64Host;
};
// launchers (ude_launch.cuh).  ag: the adaptive record, nullptr on a fixed grid.  The partial rows of every adjoint but the
// Fisher-KPP ones are adj_rows(N); the Fisher-KPP ones are adj_rows_fkpp(N, Nx)
template <typename R>
struct RuntimeShape {
    using Tab = typename RealParams<R>::Tab;
    using Fwd = typename RealParams<R>::Fwd;
    using Adj = typename RealParams<R>::Adj;
    using Adapt = typename RealParams<R>::Adapt;
    static int adj_rows(int N);
    // Tsit5 (solver 0) / Vern7 (solver 1) forward; Vern7 records u_n of every step when p.ustep is set (discrete adjoint)
    static cudaError_t fwd(const GenericShape &, const Tab &, const Fwd &, int solver, const Adapt *ag, cudaStream_t);
    // interpolating adjoint over the Tsit5 dense record, the replay of an adaptive solve when ag is set
    static cudaError_t adj(const GenericShape &, const Tab &, const Adj &, const Adapt *ag, cudaStream_t, int *rows_out);
    // discrete adjoint (discrete_adjoint.cuh) of a Tsit5 (solver 0) / Vern7 (solver 1) solve over its recorded steps
    static cudaError_t adj_discrete(const GenericShape &, const Tab &, const Adj &, int solver, const Adapt *ag, cudaStream_t, int *rows_out);
    // Vern7 with its lazy dense output (vern7_dense.cuh, B200UDE_FLAG_VERN7_DENSE): the adaptive forward saving through the interpolant
    // (record: p.ustep, ag.tgrid, ag.hstep, ag.nacc), and the interpolating adjoint over that dense output, ag = nullptr on a fixed grid
    // (record: p.ustep of fwd with solver 1).  saved: the forward's `out`, read by the fused L2 on an adaptive grid
    static cudaError_t fwd_vern7_dense(const GenericShape &, const Tab &, const Fwd &, const Adapt &, cudaStream_t);
    static cudaError_t adj_vern7_dense(const GenericShape &, const Tab &, const Adj &, const Adapt *ag, const R *saved, cudaStream_t, int *rows_out);
    // discrete adjoint of that adaptive forward through its interpolated saves (vern7_dense_discrete.cuh, B200UDE_FLAG_DISCRETE_DENSE)
    static cudaError_t adj_vern7_dense_discrete(const GenericShape &, const Tab &, const Adj &, const Adapt &, const R *saved, cudaStream_t,
                                                int *rows_out);
    // adaptive Tsit5 of the Fisher-KPP UPDE (fkpp_adaptive.cuh).  seg = 0: the full step record (p.ustep, p.dense); seg = K
    // (B200UDE_FLAG_CHECKPOINT): p.ustep holds u_n every K accepted steps, ag.hstep the step sizes, p.dense the adjoint's scratch area
    static cudaError_t fwd_fkpp_adaptive(const GenericShape &, const Tab &, const Fwd &, const Adapt &, int seg, cudaStream_t);
    static cudaError_t adj_fkpp_adaptive(const GenericShape &, const Tab &, const Adj &, const Adapt &, int seg, cudaStream_t, int *rows_out);
    // adaptive Vern7 of the Fisher-KPP UPDE with the discrete adjoint (fkpp_vern7_discrete.cuh): same geometry and shared memory as
    // adaptive Tsit5; the record is p.ustep / ag.tgrid / ag.hstep / ag.nacc; p.fused_l2 reads the recorded step-end states
    static cudaError_t fwd_fkpp_vern7(const GenericShape &, const Tab &, const Fwd &, const Adapt &, cudaStream_t);
    static cudaError_t adj_fkpp_vern7(const GenericShape &, const Tab &, const Adj &, const Adapt &, cudaStream_t, int *rows_out);
};
cudaError_t launch_reduce_f64(const double *partial, int nrows, int P1, double *grad, double *loss, cudaStream_t);
cudaError_t launch_l2_cot_f64(const Tables64 &, const double *out, const double *data, double *cot, double *loss, int D, size_t N, int n_save,
                              cudaStream_t);

// ---- forced neural ODE with a readout network (B200UDE_MODEL_FORCED; forced.cuh, k_forced.cu), fp32 and fp64 ----
struct ForcedHost {
    uint64_t serial;
    int dtype;               // 0 = float, 1 = double: every pointer below and in ForcedRun
    int D, R, J, L0, L1, P;  // states, readout outputs, harmonics, layers of f0 / f1, parameters
    int widths[8], acts[8];  // the descriptor's back-to-back lists
    double lossw[16];        // d + r weights
    const void *theta;       // the handle's device copy
};
struct ForcedRun {
    const void *u0, *forcing, *cot, *saved;   // saved: the recorded saved states of an adaptive forward (= usave)
    void *out, *ustep, *dense, *usave, *grad_u0, *partial, *tgrid;
    int32_t *status;
    int *nacc;
    int N, n_steps, save_every, fused_l2, adaptive, n_save, max_steps, fstride;
    double t0, dt, save_dt, abstol, reltol;   // t0: the origin of the kernels' time axis (0: they run on t - desc.t0)
};
int adj_rows_forced(int N, int dtype);
cudaError_t launch_fwd_forced(const ForcedHost &, const ForcedRun &, cudaStream_t);
cudaError_t launch_adj_forced(const ForcedHost &, const ForcedRun &, cudaStream_t, int *rows_out);
// phi_j -> remainder(phi_j + w_j t0, 2 pi), in double, for the first N trajectories of the forcing [3J][fstride] (in place)
cudaError_t launch_fold_forcing(int dtype, void *forcing, int J, int fstride, int N, double t0, cudaStream_t);

// ---- wide-state operator UDE du = D1 NN(u) + D2 u (B200UDE_MODEL_OPERATOR; operator.cuh, k_operator.cu), fp32 and fp64 ----
struct OperatorHost {
    int dtype;                // 0 = float, 1 = double: every pointer below and in OperatorRun
    int D, M, L, P, has_d2;   // states, chain outputs, layers, parameters, D2 given
    int widths[6], acts[5];
    int rkc2, S;              // RKC2 with S stages (else Tsit5)
    int warps;                // warps (trajectories) per CTA
    int dyn_cap;              // dynamic shared memory every launch is allowed: the device's opt-in limit less the kernels' static size
    // staged layout (operator_layout): odd leading dimensions, offsets, block sizes in elements
    int ld1, ld2, woff[5], soff[5], ldw[5], ops_elems, theta_elems, gstride;
    const void *ops;          // [64 loss weights | D1 (ld1 x M) | D2 (ld2 x D)], ops_elems elements
    const void *theta, *rkc;  // the handle's theta, RKC2 tables (adaptive RKC2: one block per stage count 2..S)
    const void *beta;         // adaptive RKC2: the real stability interval of s stages at index s (0..64)
    double rho;               // adaptive RKC2: eigen_est, the bound of the spectral radius of df/du (desc.consts[0])
};
struct OperatorRun {
    const void *u0, *cot;
    void *out, *ustep, *dense, *usave, *grad_u0, *partial, *tgrid;
    int32_t *status;
    int *nacc, *sstep;        // adaptive: accepted steps; adaptive RKC2: the stage count of each [max_steps][N]
    int N, n_steps, save_every, n_save, max_steps, fused_l2, adaptive;
    double t0, dt, save_dt, abstol, reltol;
};
void operator_layout(OperatorHost &);                      // fills P and the staged layout from D, M, L, widths
size_t operator_smem(const OperatorHost &, int warps);     // dynamic shared memory of a CTA (warps = 0: the forward kernels)
int adj_rows_operator(int N, int warps);
cudaError_t operator_static_smem(int dtype, size_t *bytes);   // the largest static shared memory of the dtype's eight kernels (current device)
cudaError_t launch_fwd_operator(const OperatorHost &, const OperatorRun &, cudaStream_t);
cudaError_t launch_adj_operator(const OperatorHost &, const OperatorRun &, cudaStream_t, int *rows_out);

}  // namespace b200ude
