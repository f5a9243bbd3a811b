// dmma.cu -- fp64 tensor-core (mma.sync.m8n8k4.f64, SASS DMMA.8x8x4) issue rate on H100 (sm_90a) as a function of warps per
// scheduler and independent accumulator chains per warp.  Sets the ceiling of the fused deep-BSDE sweeps (csrc/bsde.cu).
#include <cuda_runtime.h>
#include <cstdio>
#define ITER 2048
__device__ __forceinline__ void dmma(double (&c)[2], double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
template <int NACC>
__global__ void k_dmma(double *out)
{
    double d[NACC][2];
    double a = 1.0 + threadIdx.x * 1e-3, b = 0.5 + threadIdx.x * 1e-3;
#pragma unroll
    for (int i = 0; i < NACC; ++i) d[i][0] = d[i][1] = 0.0;
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) dmma(d[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; ++i) s += d[i][0] + d[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// the fused sweeps' inner loop: per k-step one A fragment and 14 B fragments from shared memory (8-byte loads, conflict-free
// layout of csrc/bsde.cu), 14 DMMAs; optionally a CTA barrier every 4 k-steps
template <int BARRIER>
__global__ void k_dmma_lds(double *out)
{
    __shared__ double slab[16 * 116], act[4 * 8 * 116];
    for (int i = threadIdx.x; i < 16 * 116; i += blockDim.x) slab[i] = 1.0 + i * 1e-6;
    for (int i = threadIdx.x; i < 4 * 8 * 116; i += blockDim.x) act[i] = 0.5 + i * 1e-6;
    __syncthreads();
    const int lane = threadIdx.x & 31, r = lane >> 2, c = lane & 3, warp = (threadIdx.x >> 5) & 3;
    double d[14][2];
#pragma unroll
    for (int i = 0; i < 14; ++i) d[i][0] = d[i][1] = 0.0;
    const double *wp = slab + c * 116 + r, *ap = act + warp * 8 * 116 + r * 116 + c;
    for (int it = 0; it < ITER / 4; ++it) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const double av = ap[4 * ks + 16 * (it & 3)];
            double bv[14];
#pragma unroll
            for (int i = 0; i < 14; ++i) bv[i] = wp[ks * 4 * 116 + 8 * i];
#pragma unroll
            for (int i = 0; i < 14; ++i) dmma(d[i], av, bv[i]);
        }
        if (BARRIER) __syncthreads();
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 14; ++i) s += d[i][0] + d[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int BARRIER>
static void run_lds(const char *name, int warps_per_smsp, int sms, double mhz)
{
    double *out;
    const int threads = 128 * warps_per_smsp;
    cudaMalloc(&out, sizeof(double) * sms * threads);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    k_dmma_lds<BARRIER><<<sms, threads>>>(out);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k_dmma_lds<BARRIER><<<sms, threads>>>(out);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    const double n = (double)sms * threads / 32 * ITER * 14;
    printf("%-28s %6d %10.4f %14.3f %12.2f\n", name, warps_per_smsp, ms, n / sms / (ms * 1e-3 * mhz * 1e6), n * 512 / (ms * 1e-3) / 1e12);
    cudaFree(out);
}
template <int NACC>
static void run(const char *name, int warps_per_smsp, int sms, double mhz)
{
    double *out;
    const int threads = 128 * warps_per_smsp;
    cudaMalloc(&out, sizeof(double) * sms * threads);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    k_dmma<NACC><<<sms, threads>>>(out);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k_dmma<NACC><<<sms, threads>>>(out);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    const double n = (double)sms * threads / 32 * ITER * NACC;
    const double per_clk_sm = n / sms / (ms * 1e-3 * mhz * 1e6);
    printf("%-28s %6d %10.4f %14.3f %12.2f\n", name, warps_per_smsp, ms, per_clk_sm, n * 512 / (ms * 1e-3) / 1e12);
    cudaFree(out);
}
int main()
{
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("# %s %d SMs %d MHz\n%-28s %6s %10s %14s %12s\n", p.name, p.multiProcessorCount, khz / 1000, "kernel", "w/SMSP", "ms", "dmma/clk/SM*", "TFLOP/s");
    const int sms = p.multiProcessorCount;
    const double mhz = khz / 1000.0;
    for (int w = 1; w <= 4; ++w) run<1>("f64 m8n8k4 1 chain", w, sms, mhz);
    for (int w = 1; w <= 4; ++w) run<4>("f64 m8n8k4 4 chains", w, sms, mhz);
    for (int w = 1; w <= 4; ++w) run<14>("f64 m8n8k4 14 chains", w, sms, mhz);
    for (int w = 1; w <= 3; ++w) run_lds<0>("14 chains, operands by LDS", w, sms, mhz);
    for (int w = 1; w <= 3; ++w) run_lds<1>("  + CTA barrier / 4 k-steps", w, sms, mhz);
    printf("# status: %s   (* per nominal clock)\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
