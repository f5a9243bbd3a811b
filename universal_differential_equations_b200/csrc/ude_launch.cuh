// ude_launch.cuh -- host launchers of the runtime-shape kernels (ude_generic.cuh and the headers written over its Ops), written
// once over the real type.  The translation unit that owns precision R's __constant__ symbols specialises ShapeUnit<R> -- the
// model layer's Ops, the block size and the upload of those symbols -- and instantiates RuntimeShape<R> (params.h):
// k_generic.cu in fp32, k_f64.cu in fp64.
#pragma once
#include "ude_generic.cuh"
#include "fkpp_adaptive.cuh"
#include "discrete_adjoint.cuh"
#include "fkpp_vern7_discrete.cuh"
#include "vern7_dense.cuh"
#include "vern7_dense_discrete.cuh"

#include "params.h"

namespace b200ude {

template <typename R>
struct ShapeUnit;

namespace shape_launch {

// one trajectory per thread; the adjoints keep one gradient vector (P + 1 entries) per warp in shared memory
template <typename R, class Kern, class... Args>
cudaError_t adjoint(Kern kern, int N, int P, cudaStream_t st, int *rows_out, const Args &...args)
{
    constexpr int B = ShapeUnit<R>::BLOCK;
    const size_t smem = sizeof(R) * (size_t)(B / 32) * (P + 1);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (N + B - 1) / B;
    *rows_out = grid * (B / 32);
    kern<<<grid, B, smem, st>>>(args...);
    return cudaGetLastError();
}

// Fisher-KPP: `tpc` whole grids per CTA of `th` threads (fkpp_adapt::cta_geometry); rows_out = nullptr for a forward
template <class Kern, class Q>
cudaError_t fkpp(Kern kern, const Q &q, int th, size_t smem, cudaStream_t st, int *rows_out)
{
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (q.N + q.tpc - 1) / q.tpc;
    if (rows_out) *rows_out = grid * (th / 32);
    kern<<<grid, th, smem, st>>>(q);
    return cudaGetLastError();
}

}  // namespace shape_launch

template <typename R>
int RuntimeShape<R>::adj_rows(int N)
{
    constexpr int B = ShapeUnit<R>::BLOCK;
    return ((N + B - 1) / B) * (B / 32);
}

template <typename R>
cudaError_t RuntimeShape<R>::fwd(const GenericShape &g, const Tab &t, const Fwd &p, int solver, const Adapt *ag, cudaStream_t st)
{
    using U = ShapeUnit<R>;
    using Ops = typename U::Ops;
    constexpr int B = U::BLOCK;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + B - 1) / B;
    if (solver == 1) {   // Vern7: the step record only for the discrete adjoint (p.ustep set); the interpolating adjoint re-solves with Tsit5
        if (ag) generic::vern7_adaptive_forward_kernel<Ops, B><<<grid, B, 0, st>>>(p, *ag);
        else generic::vern7_forward_kernel<Ops, B><<<grid, B, 0, st>>>(p);
    } else {
        if (ag) generic::adaptive_forward_kernel<Ops, B><<<grid, B, 0, st>>>(p, *ag);
        else generic::forward_kernel<Ops, B><<<grid, B, 0, st>>>(p);
    }
    return cudaGetLastError();
}

template <typename R>
cudaError_t RuntimeShape<R>::adj(const GenericShape &g, const Tab &t, const Adj &p, const Adapt *ag, cudaStream_t st, int *rows_out)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    if (ag) return shape_launch::adjoint<R>(generic::adaptive_adjoint_kernel<typename U::Ops, U::BLOCK>, p.N, g.P, st, rows_out, p, *ag);
    return shape_launch::adjoint<R>(generic::adjoint_kernel<typename U::Ops, U::BLOCK>, p.N, g.P, st, rows_out, p);
}

template <typename R>
cudaError_t RuntimeShape<R>::adj_discrete(const GenericShape &g, const Tab &t, const Adj &p, int solver, const Adapt *ag, cudaStream_t st,
                                          int *rows_out)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    discrete::Params<R> q;
    q.ustep = p.ustep; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.tgrid = ag ? ag->tgrid : nullptr; q.hstep = ag ? ag->hstep : nullptr; q.nacc = ag ? ag->nacc : nullptr;
    q.N = p.N; q.n_steps = p.n_steps; q.save_every = p.save_every; q.n_save = p.n_steps / p.save_every + 1; q.fused_l2 = p.fused_l2;
    q.dt = p.dt; q.t0 = ag ? ag->t0 : R(0); q.save_dt = ag ? ag->save_dt : R(0);
    q.margin = Prec<R>::clip / 2;   // half the clipping margin of vern7_adaptive_forward_kernel
    auto kern = solver == 1 ? discrete::adjoint_kernel<typename U::Ops, discrete::Vern7Scheme, U::BLOCK>
                            : discrete::adjoint_kernel<typename U::Ops, discrete::Tsit5Scheme, U::BLOCK>;
    return shape_launch::adjoint<R>(kern, p.N, g.P, st, rows_out, q);
}

template <typename R>
cudaError_t RuntimeShape<R>::fwd_vern7_dense(const GenericShape &g, const Tab &t, const Fwd &p, const Adapt &ag, cudaStream_t st)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    vern7_dense::Fwd<R> q;
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.tgrid = ag.tgrid; q.hstep = ag.hstep; q.nacc = ag.nacc; q.status = p.status;
    q.N = p.N; q.n_save = ag.n_save; q.max_steps = ag.max_steps;
    q.t0 = ag.t0; q.save_dt = ag.save_dt; q.abstol = ag.abstol; q.reltol = ag.reltol;
    vern7_dense::forward_kernel<typename U::Ops, U::BLOCK><<<(p.N + U::BLOCK - 1) / U::BLOCK, U::BLOCK, 0, st>>>(q);
    return cudaGetLastError();
}

template <typename R>
cudaError_t RuntimeShape<R>::adj_vern7_dense(const GenericShape &g, const Tab &t, const Adj &p, const Adapt *ag, const R *saved,
                                             cudaStream_t st, int *rows_out)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    vern7_dense::Adj<R> q;
    q.ustep = p.ustep; q.tgrid = ag ? ag->tgrid : nullptr; q.hstep = ag ? ag->hstep : nullptr; q.nacc = ag ? ag->nacc : nullptr;
    q.cot = p.cot; q.saved = saved; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.n_steps = p.n_steps; q.save_every = p.save_every; q.n_save = p.n_steps / p.save_every + 1; q.fused_l2 = p.fused_l2;
    q.dt = p.dt; q.t0 = ag ? ag->t0 : R(0); q.save_dt = ag ? ag->save_dt : R(0);
    return shape_launch::adjoint<R>(vern7_dense::adjoint_kernel<typename U::Ops, U::BLOCK>, p.N, g.P, st, rows_out, q);
}

template <typename R>
cudaError_t RuntimeShape<R>::adj_vern7_dense_discrete(const GenericShape &g, const Tab &t, const Adj &p, const Adapt &ag, const R *saved,
                                                      cudaStream_t st, int *rows_out)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    vern7_dense_discrete::Params<R> q;
    q.ustep = p.ustep; q.tgrid = ag.tgrid; q.hstep = ag.hstep; q.nacc = ag.nacc; q.cot = p.cot; q.saved = saved;
    q.grad_u0 = p.grad_u0; q.partial = p.partial; q.N = p.N; q.n_save = ag.n_save; q.fused_l2 = p.fused_l2;
    q.t0 = ag.t0; q.save_dt = ag.save_dt;
    return shape_launch::adjoint<R>(vern7_dense_discrete::adjoint_kernel<typename U::Ops, U::BLOCK>, p.N, g.P, st, rows_out, q);
}

template <typename R>
cudaError_t RuntimeShape<R>::fwd_fkpp_adaptive(const GenericShape &g, const Tab &t, const Fwd &p, const Adapt &ag, int seg, cudaStream_t st)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    fkpp_adapt::Fwd<R> q;
    int th;
    fkpp_adapt::cta_geometry(g.D, &q.tpc, &th);
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.dense = p.dense; q.status = p.status; q.tgrid = ag.tgrid; q.nacc = ag.nacc;
    q.N = p.N; q.Nx = g.D; q.n_save = ag.n_save; q.max_steps = ag.max_steps;
    q.t0 = ag.t0; q.save_dt = ag.save_dt; q.abstol = ag.abstol; q.reltol = ag.reltol;
    q.hstep = ag.hstep; q.seg = seg;
    const size_t smem = fkpp_adapt::fwd_smem(g.D, sizeof(R));
    if (seg) return shape_launch::fkpp(fkpp_adapt::forward_kernel<typename U::Ops, true>, q, th, smem, st, nullptr);
    return shape_launch::fkpp(fkpp_adapt::forward_kernel<typename U::Ops, false>, q, th, smem, st, nullptr);
}

template <typename R>
cudaError_t RuntimeShape<R>::adj_fkpp_adaptive(const GenericShape &g, const Tab &t, const Adj &p, const Adapt &ag, int seg, cudaStream_t st,
                                               int *rows_out)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    fkpp_adapt::Adj<R> q;
    int th;
    fkpp_adapt::cta_geometry(g.D, &q.tpc, &th);
    q.ustep = p.ustep; q.dense = p.dense; q.tgrid = ag.tgrid; q.nacc = ag.nacc; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.Nx = g.D; q.n_save = ag.n_save; q.t0 = ag.t0; q.save_dt = ag.save_dt;
    // checkpointed: the handle's dense buffer is the adjoint's scratch area
    q.hstep = ag.hstep; q.scratch = seg ? const_cast<R *>(p.dense) : nullptr; q.seg = seg;
    const size_t smem = fkpp_adapt::adj_smem(g.D, g.P, sizeof(R));
    if (seg) return shape_launch::fkpp(fkpp_adapt::adjoint_kernel<typename U::Ops, true>, q, th, smem, st, rows_out);
    return shape_launch::fkpp(fkpp_adapt::adjoint_kernel<typename U::Ops, false>, q, th, smem, st, rows_out);
}

template <typename R>
cudaError_t RuntimeShape<R>::fwd_fkpp_vern7(const GenericShape &g, const Tab &t, const Fwd &p, const Adapt &ag, cudaStream_t st)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    fkpp_vern7::Fwd<R> q;
    int th;
    fkpp_adapt::cta_geometry(g.D, &q.tpc, &th);
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.hstep = ag.hstep; q.status = p.status; q.tgrid = ag.tgrid; q.nacc = ag.nacc;
    q.N = p.N; q.Nx = g.D; q.n_save = ag.n_save; q.max_steps = ag.max_steps;
    q.t0 = ag.t0; q.save_dt = ag.save_dt; q.abstol = ag.abstol; q.reltol = ag.reltol;
    return shape_launch::fkpp(fkpp_vern7::vern7_forward_kernel<typename U::Ops>, q, th, fkpp_adapt::fwd_smem(g.D, sizeof(R)), st, nullptr);
}

template <typename R>
cudaError_t RuntimeShape<R>::adj_fkpp_vern7(const GenericShape &g, const Tab &t, const Adj &p, const Adapt &ag, cudaStream_t st,
                                            int *rows_out)
{
    using U = ShapeUnit<R>;
    cudaError_t e = U::upload(g, t, st);
    if (e != cudaSuccess) return e;
    fkpp_vern7::Adj<R> q;
    int th;
    fkpp_adapt::cta_geometry(g.D, &q.tpc, &th);
    q.ustep = p.ustep; q.hstep = ag.hstep; q.tgrid = ag.tgrid; q.nacc = ag.nacc; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.Nx = g.D; q.n_save = ag.n_save; q.fused_l2 = p.fused_l2; q.t0 = ag.t0; q.save_dt = ag.save_dt;
    q.margin = Prec<R>::clip / 2;   // half the clipping margin of the forward
    return shape_launch::fkpp(fkpp_vern7::discrete_adjoint_kernel<typename U::Ops>, q, th, fkpp_adapt::adj_smem(g.D, g.P, sizeof(R)), st,
                              rows_out);
}

}  // namespace b200ude
