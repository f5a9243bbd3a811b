// mma.cu -- legacy warp-level tensor-core (mma.sync) throughput on H100 (sm_90a): TF32 m16n8k8,
// BF16 m16n8k16.  Decides whether the 32x32 layers of the UDE chain can be moved off the FP32 pipe
// with a 3xTF32 split.  Reports MMA instructions / clk / SM and dense TFLOP/s.
#include <cuda_runtime.h>
#include <cstdio>
#define ITER 4096
__device__ __forceinline__ void mma_tf32(float (&d)[4], const unsigned (&a)[4], const unsigned (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const unsigned (&a)[4], const unsigned (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
template <int KIND, int NACC>
__global__ void k_mma(float *out)
{
    float d[NACC][4];
    unsigned a[4] = {0x3f800000u + threadIdx.x, 0x3f800000u, 0x3f000000u, 0x3e800000u}, b[2] = {0x3f800000u, 0x3f000000u + threadIdx.x};
#pragma unroll
    for (int i = 0; i < NACC; ++i) { d[i][0] = d[i][1] = d[i][2] = d[i][3] = 0.f; }
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
            if (KIND == 0) mma_tf32(d[i], a, b);
            else mma_bf16(d[i], a, b);
        }
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < NACC; ++i) s += d[i][0] + d[i][1] + d[i][2] + d[i][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// mixed: FFMA stream (two per float2) and MMA stream interleaved in the same warp: do the pipes overlap?
__global__ void k_mix(float *out, float x)
{
    float d[8][4];
    unsigned a[4] = {0x3f800000u + threadIdx.x, 0x3f800000u, 0x3f000000u, 0x3e800000u}, b[2] = {0x3f800000u, 0x3f000000u + threadIdx.x};
    float2 f[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) { d[i][0] = d[i][1] = d[i][2] = d[i][3] = 0.f; }
#pragma unroll
    for (int i = 0; i < 16; ++i) f[i] = make_float2(threadIdx.x, i);
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            mma_tf32(d[i], a, b);
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                f[i * 2 + q] = make_float2(__fmaf_rn(f[i * 2 + q].x, x, f[i * 2 + q].x), __fmaf_rn(f[i * 2 + q].y, x, f[i * 2 + q].y));
            }
        }
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += d[i][0] + d[i][1] + d[i][2] + d[i][3];
#pragma unroll
    for (int i = 0; i < 16; ++i) s += f[i].x + f[i].y;
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main()
{
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    const int sms = prop.multiProcessorCount;
    int clk_khz = 0;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    float *out;
    cudaMalloc(&out, sizeof(float) * sms * 64 * 1024);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("# %s %d SMs %.0f MHz\n%-28s %6s %10s %14s %12s\n", prop.name, sms, clk_khz / 1000.0, "kernel", "w/SMSP", "ms", "mma/clk/SM*", "TFLOP/s");
    const int wl[] = {1, 2, 4, 8};
    for (int kid = 0; kid < 7; ++kid)
        for (int wi = 0; wi < 4; ++wi) {
            const int wps = wl[wi], threads = 128, blocks = sms * wps;
            float ms = 0;
            const char *name = "";
            double mmas = 0, flop_per_mma = 0, extra_flop = 0;
            for (int rep = 0; rep < 3; ++rep) {
                cudaEventRecord(e0);
                switch (kid) {
                case 0: k_mma<0, 1><<<blocks, threads>>>(out); name = "tf32 m16n8k8 1 chain"; mmas = ITER; flop_per_mma = 2.0 * 16 * 8 * 8; break;
                case 1: k_mma<0, 4><<<blocks, threads>>>(out); name = "tf32 m16n8k8 4 chains"; mmas = 4.0 * ITER; flop_per_mma = 2.0 * 16 * 8 * 8; break;
                case 2: k_mma<0, 16><<<blocks, threads>>>(out); name = "tf32 m16n8k8 16 chains"; mmas = 16.0 * ITER; flop_per_mma = 2.0 * 16 * 8 * 8; break;
                case 3: k_mma<1, 1><<<blocks, threads>>>(out); name = "bf16 m16n8k16 1 chain"; mmas = ITER; flop_per_mma = 2.0 * 16 * 8 * 16; break;
                case 4: k_mma<1, 4><<<blocks, threads>>>(out); name = "bf16 m16n8k16 4 chains"; mmas = 4.0 * ITER; flop_per_mma = 2.0 * 16 * 8 * 16; break;
                case 5: k_mma<1, 16><<<blocks, threads>>>(out); name = "bf16 m16n8k16 16 chains"; mmas = 16.0 * ITER; flop_per_mma = 2.0 * 16 * 8 * 16; break;
                case 6: k_mix<<<blocks, threads>>>(out, 1.0000001f); name = "mix 8 tf32 mma + 32 ffma"; mmas = 8.0 * ITER; flop_per_mma = 2.0 * 16 * 8 * 8; extra_flop = 16.0 * ITER * 2 * 2 * 32; break;
                }
                cudaEventRecord(e1);
                cudaEventSynchronize(e1);
                cudaEventElapsedTime(&ms, e0, e1);
            }
            const double warps = (double)blocks * threads / 32.0;
            const double per_clk_sm = mmas * warps / (ms * 1e-3 * clk_khz * 1e3) / sms;
            const double tflops = (mmas * flop_per_mma + extra_flop) * warps / (ms * 1e-3) / 1e12;
            printf("%-28s %6d %10.4f %14.3f %12.2f\n", name, wps, ms, per_clk_sm, tflops);
        }
    cudaError_t e = cudaDeviceSynchronize();
    printf("# status: %s\n", cudaGetErrorString(e));
    return e != cudaSuccess;
}
