// step_control.cuh -- what every kernel written over the real type shares: the per-precision margins and math (Prec<R>), and
// OrdinaryDiffEq's step-size control of the adaptive solvers (PIControl).
//
// PIControl is the policy alone.  It takes norms that the kernel has already reduced -- per thread, by a warp butterfly or over
// a Fisher-KPP trajectory in a CTA -- and the kernel keeps its stage loop, its clip test, its saves and its step record.
#pragma once
#include <cuda_runtime.h>

namespace b200ude {

// per-precision margins and math of every kernel written over the real type
template <typename R>
struct Prec;
template <>
struct Prec<float> {
    static constexpr float clip = 1e-6f;   // a step within clip |t1| of the end of tspan (or a save time) is stretched to it
    static constexpr float eta = 1e-5f;    // a save time within eta h of a step end is that step end
    static constexpr float huge = 3.0e38f;
    static __device__ __forceinline__ float nan() { return __int_as_float(0x7fc00000); }
    static __device__ __forceinline__ float pw(float a, float b) { return powf(a, b); }
    static __device__ __forceinline__ float sq(float a) { return sqrtf(a); }
    static __device__ __forceinline__ float lg(float a) { return log10f(a); }
    static __device__ __forceinline__ float ex(float a) { return exp10f(a); }
};
template <>
struct Prec<double> {
    static constexpr double clip = 1e-12;
    static constexpr double eta = 1e-10;
    static constexpr double huge = 1.0e300;
    static __device__ __forceinline__ double nan() { return __longlong_as_double(0x7ff8000000000000LL); }
    static __device__ __forceinline__ double pw(double a, double b) { return pow(a, b); }
    static __device__ __forceinline__ double sq(double a) { return sqrt(a); }
    static __device__ __forceinline__ double lg(double a) { return log10(a); }
    static __device__ __forceinline__ double ex(double a) { return exp10(a); }
};

// OrdinaryDiffEq's default PI controller for a method of order ORDER (gamma 0.9, qmin 1/5, qmax 10, beta1 = 7 / (10 ORDER),
// beta2 = 2 / (5 ORDER)) and its Hairer-Norsett-Wanner initial step, whose exponent divides by HNW.  One attempt:
//   if (pi.judge(EEst)) { ...; pi.accept(EEst, h, clipped); } else pi.reject(h);
// where h is the step taken and `clipped` says it was shortened to a save time or to the end of tspan.
template <typename R, int ORDER, int HNW = ORDER>
struct PIControl {
    using PR = Prec<R>;
    static constexpr R gamma = (R)0.9, qmin = (R)0.2, qmax = (R)10;
    static constexpr R beta1 = (R)7 / (R)(10 * ORDER), beta2 = (R)2 / (R)(5 * ORDER);
    R dt;                 // the next step to try
    R qold = (R)1e-4;     // error estimate of the last accepted step, floored at 1e-4
    R q11, q;             // EEst^beta1 and the step ratio h / dt_next of the current attempt

    // first guess dt0 from d0 = ||u0|| and d1 = ||f(t0, u0)||
    static __device__ __forceinline__ R hnw_dt0(R d0, R d1, R span)
    {
        const R dt0 = (d0 < (R)1e-5 || d1 < (R)1e-5) ? (R)1e-6 : (R)0.01 * d0 / d1;
        return fmin(dt0, span);
    }
    // the initial step, from d2 = ||f(t0 + dt0, u0 + dt0 f(t0, u0)) - f(t0, u0)|| / dt0
    __device__ __forceinline__ void hnw(R dt0, R d1, R d2, R span)
    {
        const R dm = fmax(d1, d2);
        const R dt1 = dm <= (R)1e-15 ? fmax((R)1e-6, dt0 * (R)1e-3) : PR::ex(-((R)2 + PR::lg(dm)) / (R)HNW);
        dt = fmin(fmin((R)100 * dt0, dt1), span);
    }
    // true when a step with error estimate EEst (finite) is accepted
    __device__ __forceinline__ bool judge(R EEst)
    {
        q11 = PR::pw(EEst, beta1);
        q = fmin(fmax(q11 / PR::pw(qold, beta2) / gamma, (R)1 / qmax), (R)1 / qmin);
        return EEst <= (R)1;
    }
    // qsteady_min = qsteady_max = 1 for explicit RK methods in OrdinaryDiffEq (the 6/5 band is the implicit-solver default): no
    // dead band.  A clipped step does not shrink the step that follows it.
    __device__ __forceinline__ void accept(R EEst, R h, bool clipped)
    {
        qold = fmax(EEst, (R)1e-4);
        if (!clipped || h >= dt) dt = h / q;
        else dt = fmax(dt, h / q);
    }
    __device__ __forceinline__ void reject(R h) { dt = h / fmin((R)1 / qmin, q11 / gamma); }
};

}  // namespace b200ude
