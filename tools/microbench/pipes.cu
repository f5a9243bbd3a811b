// pipes.cu -- instruction-throughput microbenchmarks that set the FP32 roofline denominators for
// the UDE kernels on H100 (sm_90a): scalar FFMA vs float2 pairs (two FFMAs each), register vs uniform-register
// (constant-bank) operands, MUFU, LDC.128 / LDS.128 feeding rates.  Build: nvcc -gencode arch=compute_90a,code=sm_90a.
// Each kernel runs ITER iterations of an unrolled body on `warps` warps per SM sub-partition and
// reports instructions/clk/SM (from clock64) and the derived GFLOP/s at the measured wall time.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

__constant__ float cw[2048];

#define ITER 2048

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c)
{
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));   // sm_90 has no packed fp32 FMA
}
__device__ __forceinline__ float ffma_v(float a, float b, float c)
{
    float d;
    asm volatile("fma.rn.f32 %0, %1, %2, %3;" : "=f"(d) : "f"(a), "f"(b), "f"(c));
    return d;
}

// 0: scalar FFMA, 3 register operands, 16 independent chains
__global__ void k_ffma_reg(float *out, float x, float y)
{
    float a[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = threadIdx.x + i;
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < 16; ++i) a[i] = ffma_v(a[i], x, y);
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// 1: scalar FFMA, multiplier from the constant bank (uniform register operand)
__global__ void k_ffma_const(float *out, float y)
{
    float a[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = threadIdx.x + i;
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < 16; ++i) a[i] = fmaf(a[i], cw[r * 16 + i], y);
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// 2: float2 pairs (two FFMAs each), 3 register operands, 16 independent chains (32 FMA lanes-worth per thread)
__global__ void k_ffma2_reg(float *out, float x, float y)
{
    float2 a[16];
    const float2 xx = make_float2(x, x), yy = make_float2(y, y);
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = make_float2(threadIdx.x + i, i);
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < 16; ++i) a[i] = ffma2(a[i], xx, yy);
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += a[i].x + a[i].y;
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// 3: float2 pairs with a scalar (broadcast) multiplier from the constant bank
__global__ void k_ffma2_const(float *out, float y)
{
    float2 a[16];
    const float2 yy = make_float2(y, y);
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = make_float2(threadIdx.x + i, i);
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float w = cw[r * 16 + i];
                a[i] = ffma2(a[i], make_float2(w, w), yy);
            }
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += a[i].x + a[i].y;
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// 4: MUFU.EX2  5: MUFU.RCP  6: tanh.approx
template <int OP>
__global__ void k_mufu(float *out)
{
    float a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = 0.001f * (threadIdx.x + i);
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (OP == 0) asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
                if (OP == 1) asm volatile("rcp.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
                if (OP == 2) asm volatile("tanh.approx.f32 %0, %0;" : "+f"(a[i]));
            }
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// 7: the real inner loop shape, scalar: 32x32 layer, weights from the constant bank (LDC.128 : 4 FFMA)
__global__ void k_layer_const_t1(float *out)
{
    float h[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) h[i] = 0.01f * (threadIdx.x + i);
    float keep = 0.f;
    for (int it = 0; it < ITER / 16; ++it) {
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 32; ++i)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    float w;
                    asm volatile("ld.const.f32 %0, [%1];" : "=f"(w) : "l"(__cvta_generic_to_constant(cw + i * 32 + jb * 4 + jj)));
                    acc[jj] = fmaf(w, h[i], acc[jj]);
                }
            keep += acc[0] + acc[1] + acc[2] + acc[3];
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) h[i] += keep * 1e-30f;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = keep;
}
// 8: same with two trajectories per thread in float2 pairs (LDC.128 : 8 FFMA)
__global__ void k_layer_const_t2(float *out)
{
    float2 h[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) h[i] = make_float2(0.01f * (threadIdx.x + i), 0.02f * i);
    float2 keep = make_float2(0.f, 0.f);
    for (int it = 0; it < ITER / 16; ++it) {
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
            float2 acc[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) acc[jj] = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 32; ++i)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    float w;
                    asm volatile("ld.const.f32 %0, [%1];" : "=f"(w) : "l"(__cvta_generic_to_constant(cw + i * 32 + jb * 4 + jj)));
                    acc[jj] = ffma2(make_float2(w, w), h[i], acc[jj]);
                }
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) { keep.x += acc[jj].x; keep.y += acc[jj].y; }
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) { h[i].x += keep.x * 1e-30f; h[i].y += keep.y * 1e-30f; }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = keep.x + keep.y;
}
// 9/10: same two shapes with the weights in shared memory (broadcast LDS.128)
__global__ void k_layer_smem_t1(float *out)
{
    __shared__ __align__(16) float sw[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) sw[i] = cw[i];
    __syncthreads();
    float h[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) h[i] = 0.01f * (threadIdx.x + i);
    float keep = 0.f;
    for (int it = 0; it < ITER / 16; ++it) {
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                float4 w;
                asm volatile("ld.volatile.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(w.x), "=f"(w.y), "=f"(w.z), "=f"(w.w) : "r"((unsigned)__cvta_generic_to_shared(sw + i * 32 + jb * 4)));
                acc[0] = fmaf(w.x, h[i], acc[0]); acc[1] = fmaf(w.y, h[i], acc[1]);
                acc[2] = fmaf(w.z, h[i], acc[2]); acc[3] = fmaf(w.w, h[i], acc[3]);
            }
            keep += acc[0] + acc[1] + acc[2] + acc[3];
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) h[i] += keep * 1e-30f;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = keep;
}
__global__ void k_layer_smem_t2(float *out)
{
    __shared__ __align__(16) float sw[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) sw[i] = cw[i];
    __syncthreads();
    float2 h[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) h[i] = make_float2(0.01f * (threadIdx.x + i), 0.02f * i);
    float2 keep = make_float2(0.f, 0.f);
    for (int it = 0; it < ITER / 16; ++it) {
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
            float2 acc[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) acc[jj] = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                float4 w;
                asm volatile("ld.volatile.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(w.x), "=f"(w.y), "=f"(w.z), "=f"(w.w) : "r"((unsigned)__cvta_generic_to_shared(sw + i * 32 + jb * 4)));
                acc[0] = ffma2(make_float2(w.x, w.x), h[i], acc[0]); acc[1] = ffma2(make_float2(w.y, w.y), h[i], acc[1]);
                acc[2] = ffma2(make_float2(w.z, w.z), h[i], acc[2]); acc[3] = ffma2(make_float2(w.w, w.w), h[i], acc[3]);
            }
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) { keep.x += acc[jj].x; keep.y += acc[jj].y; }
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) { h[i].x += keep.x * 1e-30f; h[i].y += keep.y * 1e-30f; }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = keep.x + keep.y;
}

struct Case { const char *name; double fma_per_thread; double instr_per_thread; };

int main()
{
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    const int sms = prop.multiProcessorCount;
    int clk_khz = 0;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    printf("# device %s, %d SMs, max clock %.0f MHz\n", prop.name, sms, clk_khz / 1000.0);
    float *out;
    cudaMalloc(&out, sizeof(float) * sms * 64 * 1024);
    std::vector<float> hw(2048);
    for (int i = 0; i < 2048; ++i) hw[i] = 1.0f + 1e-6f * (i % 7);
    cudaMemcpyToSymbol(cw, hw.data(), sizeof(float) * 2048);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("%-22s %6s %12s %14s %14s\n", "kernel", "w/SMSP", "ms", "inst/clk/SM*", "TFLOP/s");
    const int wps_list[] = {1, 2, 4, 8};
    for (int kid = 0; kid < 11; ++kid) {
        for (int wi = 0; wi < 4; ++wi) {
            const int wps = wps_list[wi];
            const int threads = 128;             // 4 warps = one per SMSP
            const int blocks = sms * wps;        // wps warps per SMSP
            float ms = 0;
            const char *name = "";
            double fma = 0, inst = 0;
            for (int rep = 0; rep < 3; ++rep) {
                cudaEventRecord(e0);
                switch (kid) {
                case 0: k_ffma_reg<<<blocks, threads>>>(out, 1.0000001f, 1e-9f); name = "ffma_reg"; fma = 64.0 * ITER; inst = fma; break;
                case 1: k_ffma_const<<<blocks, threads>>>(out, 1e-9f); name = "ffma_const(UR)"; fma = 64.0 * ITER; inst = fma; break;
                case 2: k_ffma2_reg<<<blocks, threads>>>(out, 1.0000001f, 1e-9f); name = "ffma2_reg"; fma = 128.0 * ITER; inst = fma; break;
                case 3: k_ffma2_const<<<blocks, threads>>>(out, 1e-9f); name = "ffma2_const(UR)"; fma = 128.0 * ITER; inst = fma; break;
                case 4: k_mufu<0><<<blocks, threads>>>(out); name = "mufu_ex2"; fma = 0; inst = 64.0 * ITER; break;
                case 5: k_mufu<1><<<blocks, threads>>>(out); name = "mufu_rcp"; fma = 0; inst = 64.0 * ITER; break;
                case 6: k_mufu<2><<<blocks, threads>>>(out); name = "mufu_tanh"; fma = 0; inst = 64.0 * ITER; break;
                case 7: k_layer_const_t1<<<blocks, threads>>>(out); name = "layer32 const T1"; fma = 1024.0 * (ITER / 16); inst = fma * 1.25; break;
                case 8: k_layer_const_t2<<<blocks, threads>>>(out); name = "layer32 const T2"; fma = 2048.0 * (ITER / 16); inst = fma * 1.125; break;
                case 9: k_layer_smem_t1<<<blocks, threads>>>(out); name = "layer32 smem T1"; fma = 1024.0 * (ITER / 16); inst = fma * 1.25; break;
                case 10: k_layer_smem_t2<<<blocks, threads>>>(out); name = "layer32 smem T2"; fma = 2048.0 * (ITER / 16); inst = fma * 1.125; break;
                }
                cudaEventRecord(e1);
                cudaEventSynchronize(e1);
                cudaEventElapsedTime(&ms, e0, e1);
            }
            const double warps_total = (double)blocks * threads / 32.0;
            // instructions per clock per SM assuming the max clock (an under-estimate if clocks are lower)
            const double ipc = inst * warps_total / (ms * 1e-3 * clk_khz * 1e3) / sms;
            const double tflops = 2.0 * fma * blocks * threads / (ms * 1e-3) / 1e12;
            printf("%-22s %6d %12.4f %14.3f %14.2f\n", name, wps, ms, ipc, tflops);
        }
    }
    cudaError_t e = cudaDeviceSynchronize();
    printf("# status: %s\n", cudaGetErrorString(e));
    return e != cudaSuccess;
}
