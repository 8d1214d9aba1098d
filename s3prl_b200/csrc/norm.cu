// Row-wise HBM-bound kernels: LayerNorm (+GELU) with fp32 and bf16 hi/lo outputs, Featurizer weighted sum.
//   LayerNorm(512) before post_extract_proj       hubert_model.py:338,483
//   encoder / per-layer LayerNorms (D=384..1920)   wav2vec2_model.py:3069-3070,3260-3322,3049-3050
//   per-frame LayerNorm+GELU of "layer_norm" conv blocks  wav2vec2_model.py:2887-2897
//   Featurizer._weighted_sum                      s3prl/upstream/interfaces.py:217-248
#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

// one warp per row; V4 = D / 128 float4 per lane; two-pass statistics held in registers
template <int V4>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, size_t M,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, int gelu, float eps,
                                                        float* out_f32, const OutPlanes op) {
    constexpr int D = V4 * 128;
    const int lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    pdl_wait();
    pdl_launch_dependents();
    if (row >= M) return;
    const float4* xr = reinterpret_cast<const float4*>(x + row * D);
    float4 v[V4];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        v[i] = xr[lane + 32 * i];
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const int c4 = lane + 32 * i;
        const float4 g = __ldg(g4 + c4), b = __ldg(b4 + c4);
        float4 y;
        y.x = (v[i].x - mean) * rstd * g.x + b.x;
        y.y = (v[i].y - mean) * rstd * g.y + b.y;
        y.z = (v[i].z - mean) * rstd * g.z + b.z;
        y.w = (v[i].w - mean) * rstd * g.w + b.w;
        if (gelu) y.x = gelu_erf(y.x), y.y = gelu_erf(y.y), y.z = gelu_erf(y.z), y.w = gelu_erf(y.w);
        if (out_f32 != nullptr) reinterpret_cast<float4*>(out_f32 + row * D)[c4] = y;
        if (op.hi != nullptr) store_planes4(op, y, row * D + 4 * (size_t)c4);
    }
}

cudaError_t launch_layernorm(const float* x, size_t M, int D, const float* gamma, const float* beta, int gelu,
                             float* out_f32, const OutPlanes& op, cudaStream_t s, float eps) {
    if (M == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((M + 7) / 8);
    cudaError_t e = cudaSuccess;
    switch (D) {
        case 384: e = launch_pdl(layernorm_kernel<3>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        case 512: e = launch_pdl(layernorm_kernel<4>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        case 640: e = launch_pdl(layernorm_kernel<5>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        case 768: e = launch_pdl(layernorm_kernel<6>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        case 1024: e = launch_pdl(layernorm_kernel<8>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        case 1280: e = launch_pdl(layernorm_kernel<10>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        case 1920: e = launch_pdl(layernorm_kernel<15>, dim3(blocks), dim3(256), 0, s, x, M, gamma, beta, gelu, eps, out_f32, op); break;
        default: return cudaErrorInvalidValue;
    }
    return e;
}

// ------------------------------------------------------------------------------------------------
// modified CPC's ChannelNorm + ReLU after conv 1..4 (s3prl/upstream/cpc/model.py): per frame over the 256 channels,
//   y = relu((x - mean) * rsqrt(var + 1e-5) * gamma + beta),  var unbiased (divided by 255)
// x: [B][T][256] fp32 (the conv GEMM's output). Output rows follow the next conv's padded operand layout: utterance b
// owns rows [b R, b R + R), and row r holds frame r - pad when that is in [0, T), zeros otherwise; every row is
// written. R = T, pad = 0 is the dense layout, the only one with an fp32 copy (out_f32 [B][T][256], may be null).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) channelnorm_relu_kernel(const float* __restrict__ x, int B, int T, int R,
                                                               int pad, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float* out_f32,
                                                               const OutPlanes op) {
    constexpr int D = 256, V4 = D / 128;
    const int lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= (size_t)B * R) return;
    const int b = (int)(row / R), t = (int)(row - (size_t)b * R) - pad;
    float4 y[V4];
    if (t < 0 || t >= T) {
#pragma unroll
        for (int i = 0; i < V4; ++i) y[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
        const size_t src = (size_t)b * T + t;
        const float4* xr = reinterpret_cast<const float4*>(x + src * D);
        float4 v[V4];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            v[i] = xr[lane + 32 * i];
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
        const float mean = warp_sum(s) * (1.0f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + bb * bb) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(q) * (1.0f / (D - 1)) + 1e-5f);
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            const int c4 = lane + 32 * i;
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
            const float4 be = __ldg(reinterpret_cast<const float4*>(beta) + c4);
            y[i].x = relu_nan((v[i].x - mean) * rstd * g.x + be.x);
            y[i].y = relu_nan((v[i].y - mean) * rstd * g.y + be.y);
            y[i].z = relu_nan((v[i].z - mean) * rstd * g.z + be.z);
            y[i].w = relu_nan((v[i].w - mean) * rstd * g.w + be.w);
            if (out_f32 != nullptr) reinterpret_cast<float4*>(out_f32 + src * D)[c4] = y[i];
        }
    }
#pragma unroll
    for (int i = 0; i < V4; ++i) store_planes4(op, y[i], row * D + 4 * (size_t)(lane + 32 * i));
}

cudaError_t launch_channelnorm_relu(const float* x, int B, int T, int R, int pad, const float* gamma,
                                    const float* beta, float* out_f32, const OutPlanes& op, cudaStream_t s) {
    const size_t rows = (size_t)B * R;
    if (rows == 0) return cudaSuccess;
    if (op.hi == nullptr || (out_f32 != nullptr && (R != T || pad != 0))) return cudaErrorInvalidValue;
    channelnorm_relu_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(x, B, T, R, pad, gamma, beta, out_f32, op);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Conformer attention input (wav2vec2_model.py:255-310, 541): y = self_attn_layer_norm(x) and its rotary embedding
//   rope(y)_t = y_t * cos_t + rotate_half(y_t) * sin_t,  rotate_half(u) = cat(-u[32:], u[:32]) per 64-wide head,
// t = frame index in the padded batch (row % T). y feeds linear_v, rope(y) linear_q / linear_k; both are written as
// operand planes. cs: [>= T][64] fp32, cos of the 32 angles then their sin. Lane l holds channels 4 (l + 32 i) + 0..3,
// i.e. head offset 4 (l & 15): its rotate_half partner (offset +- 32) is lane l ^ 8 with the same i.
// ------------------------------------------------------------------------------------------------
template <int V4>
__global__ void __launch_bounds__(256) layernorm_rope_kernel(const float* __restrict__ x, size_t M, int T,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta,
                                                             const float* __restrict__ cs, const OutPlanes op,
                                                             const OutPlanes op_rope) {
    constexpr int D = V4 * 128;
    const int lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    pdl_wait();
    pdl_launch_dependents();
    if (row >= M) return;  // warp-uniform: the shuffles below see full warps
    const float4* xr = reinterpret_cast<const float4*>(x + row * D);
    float4 v[V4];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        v[i] = xr[lane + 32 * i];
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + 1e-5f);
    const int t = (int)(row % (size_t)T);
    const float4 co = __ldg(reinterpret_cast<const float4*>(cs + (size_t)t * 64) + (lane & 7));
    const float4 si = __ldg(reinterpret_cast<const float4*>(cs + (size_t)t * 64 + 32) + (lane & 7));
    const float sgn = (lane & 8) ? 1.0f : -1.0f;  // first half of a head takes -u[d + 32], second half +u[d - 32]
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const int c4 = lane + 32 * i;
        const float4 g = __ldg(g4 + c4), b = __ldg(b4 + c4);
        float4 y;
        y.x = (v[i].x - mean) * rstd * g.x + b.x;
        y.y = (v[i].y - mean) * rstd * g.y + b.y;
        y.z = (v[i].z - mean) * rstd * g.z + b.z;
        y.w = (v[i].w - mean) * rstd * g.w + b.w;
        float4 u;
        u.x = sgn * __shfl_xor_sync(0xffffffffu, y.x, 8);
        u.y = sgn * __shfl_xor_sync(0xffffffffu, y.y, 8);
        u.z = sgn * __shfl_xor_sync(0xffffffffu, y.z, 8);
        u.w = sgn * __shfl_xor_sync(0xffffffffu, y.w, 8);
        float4 r;
        r.x = y.x * co.x + u.x * si.x;
        r.y = y.y * co.y + u.y * si.y;
        r.z = y.z * co.z + u.z * si.z;
        r.w = y.w * co.w + u.w * si.w;
        store_planes4(op, y, row * D + 4 * (size_t)c4);
        store_planes4(op_rope, r, row * D + 4 * (size_t)c4);
    }
}

cudaError_t launch_layernorm_rope(const float* x, size_t M, int T, int D, const float* gamma, const float* beta,
                                  const float* cs, const OutPlanes& op, const OutPlanes& op_rope, cudaStream_t s) {
    if (M == 0) return cudaSuccess;
    if (T < 1 || op.hi == nullptr || op_rope.hi == nullptr) return cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((M + 7) / 8);
#define S3B_LR(V) \
    return launch_pdl(layernorm_rope_kernel<V>, dim3(blocks), dim3(256), 0, s, x, M, T, gamma, beta, cs, op, op_rope)
    switch (D) {
        case 512: S3B_LR(4);
        case 768: S3B_LR(6);
        case 1024: S3B_LR(8);
        case 1280: S3B_LR(10);
        default: return cudaErrorInvalidValue;
    }
#undef S3B_LR
}

// ------------------------------------------------------------------------------------------------
// pos_conv combine: the grouped k=128 convolution is computed as a GEMM over FOUR taps per k-block,
//   Z_j[u] = sum_q x[u + 4q - 64] . W[4q + j]   (j = 0..3, N = 4 * cpg columns per group; model.cu posconv4_params)
// and the four column blocks are re-aligned here:  conv[t] = sum_j Z_j[t + j]. One warp per frame:
//   y = x + GELU(conv + bias)                      (wav2vec2_model.py:3064-3067)
//   post-LN models: y -> LayerNorm -> hidden state 0 (fp32) + bf16 hi/lo   (wav2vec2_model.py:3069-3070)
// mode 0: the above. mode 1 / 2 (data2vec conv blocks, pos_conv_depth > 1; taps rounded up to a multiple of four):
//   y = GELU(LayerNorm_noaffine(conv + bias))      (wav2vec2_model.py:3000-3019); mode 2 (last block): y = x + y, then
//   the optional encoder LayerNorm as in mode 0.
// z: [B][T + 3][G][4][cpg] fp32
// ------------------------------------------------------------------------------------------------
template <int V4>
__global__ void __launch_bounds__(256) posconv_combine_kernel(const float* __restrict__ z, const float* __restrict__ x,
                                                              const float* __restrict__ bias, int B, int T, int cpg,
                                                              const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, int do_ln, int mode,
                                                              float* __restrict__ out_f32, const OutPlanes op) {
    constexpr int D = V4 * 128;
    const int lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    pdl_wait();
    pdl_launch_dependents();
    if (row >= (size_t)B * T) return;
    const int b = (int)(row / T), t = (int)(row - (size_t)b * T);
    const float4* xr = reinterpret_cast<const float4*>(x + (mode == 1 ? 0 : row * D));  // mode 1 has no residual
    const float4* b4 = reinterpret_cast<const float4*>(bias);
    float4 v[V4];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const int c = 4 * (lane + 32 * i);
        const int g = c / cpg, co = c - g * cpg;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 zz = __ldg(reinterpret_cast<const float4*>(
                z + ((size_t)b * (T + 3) + t + j) * (size_t)(4 * D) + (size_t)g * 4 * cpg + j * cpg + co));
            acc.x += zz.x, acc.y += zz.y, acc.z += zz.z, acc.w += zz.w;
        }
        const float4 bb = __ldg(b4 + lane + 32 * i);
        if (mode == 0) {
            const float4 xx = xr[lane + 32 * i];
            v[i].x = xx.x + gelu_erf(acc.x + bb.x);
            v[i].y = xx.y + gelu_erf(acc.y + bb.y);
            v[i].z = xx.z + gelu_erf(acc.z + bb.z);
            v[i].w = xx.w + gelu_erf(acc.w + bb.w);
        } else {
            v[i] = make_float4(acc.x + bb.x, acc.y + bb.y, acc.z + bb.z, acc.w + bb.w);
        }
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    float mean = 0.f, rstd = 1.f;
    if (mode != 0) {
        // data2vec block: LayerNorm over the channels without affine, then GELU (wav2vec2_model.py:3012-3015); the
        // last block (mode 2) adds the residual x afterwards (:3064-3067)
        mean = warp_sum(s) * (1.0f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + bq * bq) + (c * c + d * d);
        }
        rstd = rsqrtf(warp_sum(q) * (1.0f / D) + 1e-5f);
        s = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            float4 y;
            y.x = gelu_erf((v[i].x - mean) * rstd);
            y.y = gelu_erf((v[i].y - mean) * rstd);
            y.z = gelu_erf((v[i].z - mean) * rstd);
            y.w = gelu_erf((v[i].w - mean) * rstd);
            if (mode == 2) {
                const float4 xx = xr[lane + 32 * i];
                y.x += xx.x, y.y += xx.y, y.z += xx.z, y.w += xx.w;
            }
            v[i] = y;
            s += (y.x + y.y) + (y.z + y.w);
        }
        mean = 0.f, rstd = 1.f;
    }
    if (do_ln) {
        mean = warp_sum(s) * (1.0f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + bq * bq) + (c * c + d * d);
        }
        rstd = rsqrtf(warp_sum(q) * (1.0f / D) + 1e-5f);
    }
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const int c4 = lane + 32 * i;
        float4 y = v[i];
        if (do_ln) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
            const float4 be = __ldg(reinterpret_cast<const float4*>(beta) + c4);
            y.x = (y.x - mean) * rstd * g.x + be.x;
            y.y = (y.y - mean) * rstd * g.y + be.y;
            y.z = (y.z - mean) * rstd * g.z + be.z;
            y.w = (y.w - mean) * rstd * g.w + be.w;
        }
        if (out_f32 != nullptr) reinterpret_cast<float4*>(out_f32 + row * D)[c4] = y;
        if (op.hi != nullptr) store_planes4(op, y, row * D + 4 * (size_t)c4);
    }
}

cudaError_t launch_posconv_combine(const float* z, const float* x, const float* bias, int B, int T, int D, int cpg,
                                   const float* gamma, const float* beta, int do_ln, int mode, float* out_f32,
                                   const OutPlanes& op, cudaStream_t s) {
    const size_t M = (size_t)B * T;
    if (M == 0) return cudaSuccess;
    if (cpg % 4 != 0) return cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((M + 7) / 8);
#define S3B_PC(V)                                                                                                   \
    return launch_pdl(posconv_combine_kernel<V>, dim3(blocks), dim3(256), 0, s, z, x, bias, B, T, cpg, gamma, beta, \
                      do_ln, mode, out_f32, op)
    switch (D) {
        case 384: S3B_PC(3);
        case 512: S3B_PC(4);
        case 640: S3B_PC(5);
        case 768: S3B_PC(6);
        case 1024: S3B_PC(8);
        case 1280: S3B_PC(10);
        default: return cudaErrorInvalidValue;
    }
#undef S3B_PC
}

// ------------------------------------------------------------------------------------------------
// Featurizer weighted sum: streams NL layers once (vs. torch.stack + mul + sum = >= 3 passes)
// ------------------------------------------------------------------------------------------------
static constexpr int kMaxLayers = 64;

__global__ void __launch_bounds__(256) weighted_sum_kernel(const float4* __restrict__ hs, int NL, size_t n4,
                                                           const float* __restrict__ w_dev,
                                                           float4* __restrict__ out) {
    __shared__ float lw[kMaxLayers];
    if ((int)threadIdx.x < NL) lw[threadIdx.x] = w_dev[threadIdx.x];
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int l = 0; l < NL; ++l) {
            const float4 v = hs[(size_t)l * n4 + i];
            const float w = lw[l];
            acc.x = fmaf(w, v.x, acc.x), acc.y = fmaf(w, v.y, acc.y);
            acc.z = fmaf(w, v.z, acc.z), acc.w = fmaf(w, v.w, acc.w);
        }
        out[i] = acc;
    }
}

cudaError_t launch_weighted_sum(const float* hs, int NL, size_t n_per_layer, const float* w_dev, float* out,
                                cudaStream_t s) {
    if (NL > kMaxLayers || (n_per_layer & 3) != 0) return cudaErrorInvalidValue;
    const size_t n4 = n_per_layer / 4;
    size_t blocks = (n4 + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks == 0) return cudaSuccess;
    weighted_sum_kernel<<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(hs), NL, n4, w_dev,
                                                         reinterpret_cast<float4*>(out));
    return cudaGetLastError();
}

// grad_w[l] = <hs[l], gout>; grid (chunks, NL); deterministic two-stage reduction would need a workspace,
// the 13..25 scalars tolerate atomics (fp32 atomicAdd of per-block partials accumulated in fp32).
__global__ void __launch_bounds__(256) weighted_sum_bwd_kernel(const float4* __restrict__ hs, size_t n4,
                                                               const float4* __restrict__ gout,
                                                               float* __restrict__ grad_w) {
    const int l = blockIdx.y;
    float acc = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const float4 v = hs[(size_t)l * n4 + i];
        const float4 g = gout[i];
        acc += (v.x * g.x + v.y * g.y) + (v.z * g.z + v.w * g.w);
    }
    __shared__ float red[8];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        atomicAdd(grad_w + l, t);
    }
}

cudaError_t launch_weighted_sum_bwd(const float* hs, int NL, size_t n_per_layer, const float* gout, float* grad_w,
                                    cudaStream_t s) {
    if ((n_per_layer & 3) != 0) return cudaErrorInvalidValue;
    cudaError_t e = cudaMemsetAsync(grad_w, 0, sizeof(float) * NL, s);
    if (e != cudaSuccess) return e;
    const size_t n4 = n_per_layer / 4;
    size_t bx = (n4 + 256 * 8 - 1) / (256 * 8);
    if (bx > 132) bx = 132;
    if (bx == 0) return cudaSuccess;
    dim3 grid((unsigned)bx, NL);
    weighted_sum_bwd_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const float4*>(hs), n4,
                                                 reinterpret_cast<const float4*>(gout), grad_w);
    return cudaGetLastError();
}

}  // namespace s3b
