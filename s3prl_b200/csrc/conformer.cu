// Conformer convolution module between its two pointwise convs (wav2vec2_model.py:371-393):
//   GLU(pointwise_conv1 output) -> depthwise Conv1d(k, padding k/2, groups = D) -> BatchNorm1d (eval) -> SiLU
// with BatchNorm folded into the taps and a bias at finalize (w' = w * s, b' = beta - mean * s, s = gamma / sqrt(var +
// eps)). Memory-bound: every input element is read once from HBM (the halo rows come from L2), every output written once.
#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

static constexpr int kDwChannels = 64;  // channels per block
static constexpr int kDwFrames = 64;    // output frames per block
static constexpr int kDwThreads = 256;  // 32 channel pairs x 8 groups of 8 frames

static size_t depthwise_smem_bytes(int k) { return (size_t)(kDwFrames + k - 1 + k) * kDwChannels * sizeof(float); }

// x: [B][T][2D] fp32 (a = channels [0, D), gate = [D, 2D)), w: [D][k] folded taps, bias: [D]. Block (channel block,
// frame tile, utterance b): the GLU values of frames [t0 - k/2, t0 + 64 + k/2) are staged in shared memory, zero outside
// [0, T) of utterance b (the conv's zero padding) — no block reads another utterance's rows, so lanes and sharded
// batches see the same values. Padded frames inside [0, T) are used as they are, like the reference.
__global__ void __launch_bounds__(kDwThreads) depthwise_glu_kernel(const float* __restrict__ x,
                                                                   const float* __restrict__ w,
                                                                   const float* __restrict__ bias, int T, int D, int k,
                                                                   const OutPlanes op) {
    extern __shared__ float4 dw_smem4[];
    float* g = reinterpret_cast<float*>(dw_smem4);  // [kDwFrames + k - 1][64] GLU values
    const int rows = kDwFrames + k - 1;
    float* taps = g + (size_t)rows * kDwChannels;  // [k][64]
    const int c0 = blockIdx.x * kDwChannels, t0 = blockIdx.y * kDwFrames, b = blockIdx.z, half = k / 2;
    const int tid = threadIdx.x;
    for (int i = tid; i < k * kDwChannels; i += kDwThreads) {
        const int j = i / kDwChannels, c = i - j * kDwChannels;
        taps[i] = __ldg(w + (size_t)(c0 + c) * k + j);
    }
    pdl_wait();
    pdl_launch_dependents();
    const float* xb = x + (size_t)b * T * (2 * D);
    for (int i = tid; i < rows * (kDwChannels / 4); i += kDwThreads) {
        const int r = i / (kDwChannels / 4), c4 = i - r * (kDwChannels / 4);
        const int t = t0 - half + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t >= 0 && t < T) {
            const float* xr = xb + (size_t)t * (2 * D) + c0 + 4 * c4;
            const float4 a = __ldg(reinterpret_cast<const float4*>(xr));
            const float4 gt = __ldg(reinterpret_cast<const float4*>(xr + D));
            v = make_float4(a.x * sigmoid_fast(gt.x), a.y * sigmoid_fast(gt.y), a.z * sigmoid_fast(gt.z),
                            a.w * sigmoid_fast(gt.w));
        }
        dw_smem4[i] = v;
    }
    __syncthreads();
    const int cp = tid & 31, f0 = (tid >> 5) * 8;  // channel pair, first of this thread's 8 frames
    float2 acc[8];
#pragma unroll
    for (int f = 0; f < 8; ++f) acc[f] = make_float2(0.f, 0.f);
    const float2* g2 = reinterpret_cast<const float2*>(g);
    const float2* t2 = reinterpret_cast<const float2*>(taps);
    for (int j = 0; j < k; ++j) {
        const float2 wj = t2[j * (kDwChannels / 2) + cp];
#pragma unroll
        for (int f = 0; f < 8; ++f) {
            const float2 v = g2[(f0 + f + j) * (kDwChannels / 2) + cp];
            acc[f].x = fmaf(wj.x, v.x, acc[f].x);
            acc[f].y = fmaf(wj.y, v.y, acc[f].y);
        }
    }
    const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + c0) + cp);
#pragma unroll
    for (int f = 0; f < 8; ++f) {
        const int t = t0 + f0 + f;
        if (t >= T) break;
        store_planes2(op, silu(acc[f].x + bb.x), silu(acc[f].y + bb.y), ((size_t)b * T + t) * D + c0 + 2 * cp);
    }
}

cudaError_t launch_depthwise_glu(const float* x, int B, int T, int D, int k, const float* w, const float* bias,
                                 const OutPlanes& op, cudaStream_t s) {
    if (B < 1 || T < 1) return cudaSuccess;
    if (D % kDwChannels != 0 || k < 1 || k > kDwMaxKernel || k % 2 == 0 || op.hi == nullptr)
        return cudaErrorInvalidValue;
    const dim3 grid(D / kDwChannels, (T + kDwFrames - 1) / kDwFrames, B);
    return launch_pdl(depthwise_glu_kernel, grid, dim3(kDwThreads), depthwise_smem_bytes(k), s, x, w, bias, T, D, k, op);
}

}  // namespace s3b
