// k_f64.cu -- double-precision kernels (dtype = B200UDE_F64): the runtime-shape kernels (ude_generic.cuh and the headers written
// over its Ops) in fp64 with their __constant__ symbol and launchers (ude_launch.cuh), + the fp64 reduction / L2 helpers.
#include "ude_launch.cuh"

namespace b200ude {

namespace f64 {
struct Shape64 {
    uint64_t serial;
    int model, D, din, dout, n_layers, n_prefix, P;
    int widths[6];
    int acts[5];
    int woff[5];          // offset of layer l's W in theta (column-major, out x in), its bias follows at woff + in*out
    const double *theta;  // the handle's device copy
    double consts[16], lossw[16];
};
static __constant__ Shape64 c_gen;
}  // namespace f64

// the fp64 precision of the runtime-shape model layer: shape, constants and loss weights from one small __constant__ struct,
// theta from the handle's device copy (global memory, L1-resident)
struct Ops64 {
    using real = double;
    using Fwd = Fwd64Host;
    using Adj = Adj64Host;
    using Adapt = Adapt64Host;
    static constexpr int MAXD = generic::MAXD;
    static __device__ __forceinline__ int model() { return f64::c_gen.model; }
    static __device__ __forceinline__ int D() { return f64::c_gen.D; }
    static __device__ __forceinline__ int din() { return f64::c_gen.din; }
    static __device__ __forceinline__ int dout() { return f64::c_gen.dout; }
    static __device__ __forceinline__ int n_layers() { return f64::c_gen.n_layers; }
    static __device__ __forceinline__ int n_prefix() { return f64::c_gen.n_prefix; }
    static __device__ __forceinline__ int P() { return f64::c_gen.P; }
    static __device__ __forceinline__ int width(int l) { return f64::c_gen.widths[l]; }
    static __device__ __forceinline__ int woff(int l) { return f64::c_gen.woff[l]; }
    static __device__ __forceinline__ int layer_act(int l) { return f64::c_gen.acts[l]; }
    static __device__ __forceinline__ const double &theta(int i) { return f64::c_gen.theta[i]; }
    static __device__ __forceinline__ const double &consts(int i) { return f64::c_gen.consts[i]; }
    static __device__ __forceinline__ const double &lossw(int c) { return f64::c_gen.lossw[c]; }
    static __device__ __forceinline__ double act(int k, double a) { return k == ACT_TANH ? tanh(a) : (k == ACT_RBF ? exp(-a * a) : a); }
};

static cudaError_t upload_shape(const GenericShape &g, const Tables64 &t, cudaStream_t st)
{
    // theta's address and the constants are per handle; the struct is small (0.4 KB): re-sent when the handle changes
    static SerialCache cache;
    if (cache.hit(g.serial)) return cudaSuccess;
    f64::Shape64 d;
    d.serial = g.serial; d.model = g.model; d.D = g.D; d.din = g.din; d.dout = g.dout; d.n_layers = g.n_layers; d.n_prefix = g.n_prefix; d.P = g.P;
    int off = g.n_prefix;
    for (int l = 0; l < 6; ++l) d.widths[l] = l <= g.n_layers ? g.widths[l] : 0;
    for (int l = 0; l < 5; ++l) {
        d.acts[l] = l < g.n_layers ? g.acts[l] : 0;
        d.woff[l] = off;
        if (l < g.n_layers) off += g.widths[l] * g.widths[l + 1] + g.widths[l + 1];
    }
    d.theta = t.theta;
    for (int i = 0; i < 16; ++i) { d.consts[i] = t.consts[i]; d.lossw[i] = t.lossw[i]; }
    cudaError_t e = cudaMemcpyToSymbolAsync(f64::c_gen, &d, sizeof(d), 0, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        e = cudaStreamSynchronize(st);   // `d` is a stack object
        cache.set(g.serial);
    }
    return e;
}

template <>
struct ShapeUnit<double> {
    using Ops = Ops64;
    static constexpr int BLOCK = 64;   // two warps per CTA: the per-warp gradient vector (P + 1 doubles) lives in shared memory
    static cudaError_t upload(const GenericShape &g, const Tables64 &t, cudaStream_t st) { return upload_shape(g, t, st); }
};
template struct RuntimeShape<double>;

// fixed-order sum of the per-warp partial rows (one warp per entry; lane l sums rows l, l + 32, ... then a fixed butterfly)
static __global__ void reduce64_kernel(const double *__restrict__ partial, int nrows, int P1, double *__restrict__ grad, double *__restrict__ loss)
{
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (q >= P1) return;
    double acc = 0.0;
    for (int b = lane; b < nrows; b += 32) acc += partial[(size_t)b * P1 + q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        if (q == P1 - 1) {
            if (loss) *loss = acc;
        } else {
            grad[q] = acc;
        }
    }
}
cudaError_t launch_reduce_f64(const double *partial, int nrows, int P1, double *grad, double *loss, cudaStream_t st)
{
    reduce64_kernel<<<(P1 + 7) / 8, 256, 0, st>>>(partial, nrows, P1, grad, loss);
    return cudaGetLastError();
}

// L2 cotangent 2 w (out - data) and loss for the adaptive path (generic cotangent); one CTA, fixed order
struct LossW64 { double w[16]; };
static __global__ void l2_cot64_kernel(const double *__restrict__ out, const double *__restrict__ data, double *__restrict__ cot,
                                       double *__restrict__ loss, LossW64 lw, int D, size_t N, size_t total)
{
    __shared__ double red[1024];
    double acc = 0.0;
    for (size_t e = threadIdx.x; e < total; e += blockDim.x) {
        const int c = (int)((e / N) % (size_t)D);
        const double wgt = D <= 16 ? lw.w[c] : 1.0;
        const double r = out[e] - data[e];
        cot[e] = 2.0 * wgt * r;
        acc = fma(wgt * r, r, acc);
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0 && loss) *loss = red[0];
}
cudaError_t launch_l2_cot_f64(const Tables64 &t, const double *out, const double *data, double *cot, double *loss, int D, size_t N, int n_save,
                              cudaStream_t st)
{
    LossW64 lw;
    for (int i = 0; i < 16; ++i) lw.w[i] = t.lossw[i];
    l2_cot64_kernel<<<1, 1024, 0, st>>>(out, data, cot, loss, lw, D, N, (size_t)n_save * D * N);
    return cudaGetLastError();
}

}  // namespace b200ude
