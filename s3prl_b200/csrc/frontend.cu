// HBM-bound front-end kernels of the conv feature extractor and the small glue ops:
//   * waveform packing (+ optional per-utterance normalisation)       hubert/expert.py:56-66
//   * conv-0 (Conv1d(1,512,10,5)) fused with GroupNorm(512,512) + GELU (extractor_mode "default")
//     or per-frame LayerNorm(512) + GELU (extractor_mode "layer_norm") wav2vec2_model.py:2869-2934
//   * fp32 -> bf16 hi/lo split (weights at load time)
// Outputs are channels-last [B][L0][512] bf16 hi/lo so that conv-1 is a plain K-major GEMM operand.
#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

// ------------------------------------------------------------------------------------------------
// fp32 -> (hi, lo) bf16 split
// ------------------------------------------------------------------------------------------------
__global__ void split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                             __nv_bfloat16* __restrict__ lo, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        __nv_bfloat16 h, l;
        split_bf16(x[i], h, l);
        hi[i] = h;
        lo[i] = l;
    }
}

cudaError_t launch_split(const float* x, __nv_bfloat16* hi, __nv_bfloat16* lo, size_t n, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const int threads = 256;
    size_t blocks = (n + threads - 1) / threads;
    if (blocks > 132 * 16) blocks = 132 * 16;
    split_kernel<<<(unsigned)blocks, threads, 0, s>>>(x, hi, lo, n);
    return cudaGetLastError();
}

// fp32 -> f16q8 planes (common.cuh): activations (weight == 0) or weights (weight != 0: wh8 = e4m3(w * 2^ShiftB),
// wl8 = e4m3((w - w16) * 2^ShiftD)), the e4m3 pairs into the interleaved q8 plane
__global__ void split_q8_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ p16,
                                uint8_t* __restrict__ q8, size_t n2, int weight) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n2; i += stride) {
        const float a = x[2 * i], b = x[2 * i + 1];
        uint32_t h;
        uint16_t q_h, q_l;
        if (weight == 0) {
            split_q8_pack2(a, b, h, q_h, q_l);
        } else {
            asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));
            float ha, hb;
            asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %2; cvt.f32.f16 %0, lo; cvt.f32.f16 %1, hi; }"
                : "=f"(ha), "=f"(hb)
                : "r"(h));
            const float sb = (float)(1 << kQ8ShiftB), sd = (float)(1 << kQ8ShiftD);
            asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(q_h) : "f"(b * sb), "f"(a * sb));
            asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(q_l) : "f"((b - hb) * sd), "f"((a - ha) * sd));
        }
        reinterpret_cast<uint32_t*>(p16)[i] = h;
        *reinterpret_cast<uint16_t*>(q8 + q8_off(2 * i, 1)) = q_h;
        *reinterpret_cast<uint16_t*>(q8 + q8_off(2 * i, 0)) = q_l;
    }
}

cudaError_t launch_split_q8(const float* x, __nv_bfloat16* p16, uint8_t* q8, size_t n, int weight,
                            cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    if (n & 1) return cudaErrorInvalidValue;
    const size_t n2 = n / 2;
    size_t blocks = (n2 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    split_q8_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, p16, q8, n2, weight);
    return cudaGetLastError();
}

// the interleaved q8 plane of n elements -> separate h8 and l8 planes (the C ABI's back-to-back plane layout)
__global__ void q8_deinterleave_kernel(const uint8_t* __restrict__ q8, size_t n, uint8_t* __restrict__ h8,
                                       uint8_t* __restrict__ l8) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        h8[i] = q8[q8_off(i, 1)];
        l8[i] = q8[q8_off(i, 0)];
    }
}

cudaError_t launch_q8_deinterleave(const uint8_t* q8, size_t n, uint8_t* h8, uint8_t* l8, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    size_t blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    q8_deinterleave_kernel<<<(unsigned)blocks, 256, 0, s>>>(q8, n, h8, l8);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// pack B ragged waveforms into a zero-padded [B][Lpad] buffer; optional F.layer_norm(wav, wav.shape)
// (eps 1e-5, biased variance) per utterance (task_cfg.normalize, hubert/expert.py:57-58)
// ------------------------------------------------------------------------------------------------
__global__ void wav_stats_kernel(const float* const* __restrict__ wavs, const long long* __restrict__ lens,
                                 float* __restrict__ mean_rstd) {
    // one block per utterance; two-pass (mean, then centred second moment), fp32 with double block combine
    const int b = blockIdx.x;
    const float* w = wavs[b];
    const long long n = lens[b];
    __shared__ double red[32];
    __shared__ float s_mean;
    double acc = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) acc += (double)w[i];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
        s_mean = (float)(t / (double)n);
    }
    __syncthreads();
    const float mean = s_mean;
    acc = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float d = w[i] - mean;
        acc += (double)(d * d);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
        mean_rstd[2 * b] = mean;
        mean_rstd[2 * b + 1] = rsqrtf((float)(t / (double)n) + 1e-5f);
    }
}

__global__ void wav_pack_kernel(const float* const* __restrict__ wavs, const long long* __restrict__ lens,
                                const float* __restrict__ mean_rstd, float* __restrict__ out, long long Lpad) {
    const int b = blockIdx.y;
    const float* w = wavs[b];
    const long long n = lens[b];
    float mean = 0.f, rstd = 1.f;
    if (mean_rstd != nullptr) mean = mean_rstd[2 * b], rstd = mean_rstd[2 * b + 1];
    float* o = out + (size_t)b * Lpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < Lpad;
         i += (long long)gridDim.x * blockDim.x)
        o[i] = (i < n) ? (w[i] - mean) * rstd : 0.0f;
}

cudaError_t launch_wav_pack(const float* const* wavs, const long long* lens, int B, long long Lpad, int normalize,
                            float* mean_rstd_ws, float* out, cudaStream_t s) {
    if (normalize) wav_stats_kernel<<<B, 1024, 0, s>>>(wavs, lens, mean_rstd_ws);
    dim3 grid((unsigned)((Lpad + 1023) / 1024 < 64 ? (Lpad + 1023) / 1024 : 64), B);
    wav_pack_kernel<<<grid, 256, 0, s>>>(wavs, lens, normalize ? mean_rstd_ws : nullptr, out, Lpad);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// conv-0: z[b][t][c] = sum_{j<10} w[c][j] * x[b][5t+j]      (no bias in "default" mode)
// 256 threads, thread = channel pair (2*tid, 2*tid+1), block = TCH consecutive frames of one utterance.
// ------------------------------------------------------------------------------------------------
static constexpr int kC0 = 512;
static constexpr int kC0K = 10;
static constexpr int kC0S = 5;
static constexpr int kTCH = 256;                        // frames per block
static constexpr int kXTile = kTCH * kC0S + 8;          // samples staged per block (+ halo, padded)

__device__ __forceinline__ void conv0_load_tile(const float* __restrict__ xb, long long L, long long s0, float* xs) {
    for (int i = threadIdx.x; i < kXTile; i += blockDim.x) {
        const long long g = s0 + i;
        xs[i] = (g < L) ? xb[g] : 0.0f;
    }
}

// 4 consecutive frames x 2 channels from 25 staged samples
__device__ __forceinline__ void conv0_quad(const float* xs, int tl, const float (&w0)[kC0K], const float (&w1)[kC0K],
                                           float (&z0)[4], float (&z1)[4]) {
    float xv[28];
    const float4* x4 = reinterpret_cast<const float4*>(xs + tl * kC0S);  // tl % 4 == 0 -> 16B aligned
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const float4 v = x4[i];
        xv[4 * i] = v.x, xv[4 * i + 1] = v.y, xv[4 * i + 2] = v.z, xv[4 * i + 3] = v.w;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int j = 0; j < kC0K; ++j) {
            a0 = fmaf(w0[j], xv[q * kC0S + j], a0);
            a1 = fmaf(w1[j], xv[q * kC0S + j], a1);
        }
        z0[q] = a0, z1[q] = a1;
    }
}

// pass 1: second-order moments of the 10-sample conv windows. With z_t[c] = sum_j w[c][j] x[5t+j],
//   sum_t z_t[c]   = sum_j w[c][j] m_j,            m_j  = sum_t x[5t+j]
//   sum_t z_t[c]^2 = sum_jk w[c][j] w[c][k] R_jk,  R_jk = sum_t x[5t+j] x[5t+k]
// so the GroupNorm statistics of all 512 channels follow from 10 + 55 numbers per utterance: one cheap pass over
// the waveform instead of a full conv pass (the previous conv0_stats_kernel took 0.29 ms at C2).
// The moments are summed in fp64 (a product of two fp32 samples is exact there): var = w^T R w / L0 - mean^2 cancels
// by the channel's conditioning (sum_j |w_j| |x|)^2 / var(z), large where a filter rejects most of the signal (a
// high-pass filter on band-limited or DC-offset audio), and fp32 sums lose conditioning^2 * 2^-24 of var there.
static constexpr int kNMom = kC0K + kC0K * (kC0K + 1) / 2;  // 65
static constexpr int kMomSplit = 3;                          // threads per moment, each summing every third frame
static_assert(kMomSplit * kNMom <= 256, "one thread per (moment, frame phase)");

__global__ void __launch_bounds__(256) conv0_moments_kernel(const float* __restrict__ x, long long L, int L0,
                                                            double* __restrict__ part /*[B][nchunk][65]*/,
                                                            int nchunk) {
    __shared__ __align__(16) float xs[kXTile];
    __shared__ double red[kMomSplit][kNMom];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int t0 = chunk * kTCH;
    conv0_load_tile(x + (size_t)b * L, L, (long long)t0 * kC0S, xs);
    __syncthreads();
    const int nt = min(kTCH, L0 - t0);  // frames of this chunk inside [0, L0)
    if (threadIdx.x < kMomSplit * kNMom) {
        const int i = threadIdx.x % kNMom, phase = threadIdx.x / kNMom;
        // moment i: m_j (i = j < 10), then R_jk for j <= k in row order (the order conv0_finalize_kernel reads)
        int j = i, k = -1;
        if (i >= kC0K) {
            int r = i - kC0K;
            for (j = 0; r >= kC0K - j; ++j) r -= kC0K - j;
            k = j + r;
        }
        const int kk = k < 0 ? j : k;
        double acc = 0.0;
        for (int t = phase; t < nt; t += kMomSplit) {
            const double a = (double)xs[t * kC0S + j];
            acc = fma(a, k < 0 ? 1.0 : (double)xs[t * kC0S + kk], acc);
        }
        red[phase][i] = acc;
    }
    __syncthreads();
    if (threadIdx.x < kNMom) {
        double v = 0.0;
#pragma unroll
        for (int p = 0; p < kMomSplit; ++p) v += red[p][threadIdx.x];
        part[((size_t)b * nchunk + chunk) * kNMom + threadIdx.x] = v;
    }
}

// finalize: GroupNorm(512 groups == per channel) statistics over ALL L0 frames of the padded batch
// (Fp32GroupNorm, eps 1e-5, biased variance; wav2vec2_model.py:1841-1853, 2898-2904), in double:
//   y = (z - mean) * rstd * gamma + beta  =  z * scale + shift
__global__ void __launch_bounds__(kC0) conv0_finalize_kernel(const double* __restrict__ part, int nchunk, int L0,
                                                             const float* __restrict__ w,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta,
                                                             float* __restrict__ scale, float* __restrict__ shift) {
    __shared__ double mom[kNMom];
    const int b = blockIdx.x, c = threadIdx.x;
    if (c < kNMom) {
        double acc = 0.0;
        for (int k = 0; k < nchunk; ++k) acc += part[((size_t)b * nchunk + k) * kNMom + c];
        mom[c] = acc;
    }
    __syncthreads();
    double wc[kC0K];
#pragma unroll
    for (int j = 0; j < kC0K; ++j) wc[j] = (double)w[c * kC0K + j];
    double s = 0.0, q = 0.0;
    int idx = kC0K;
#pragma unroll
    for (int j = 0; j < kC0K; ++j) {
        s += wc[j] * mom[j];
#pragma unroll
        for (int k = j; k < kC0K; ++k) q += (k == j ? 1.0 : 2.0) * wc[j] * wc[k] * mom[idx++];
    }
    const double mean = s / (double)L0;
    double var = q / (double)L0 - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + 1e-5));
    const float g = gamma[c] * rstd;
    scale[b * kC0 + c] = g;
    shift[b * kC0 + c] = beta[c] - (float)mean * g;
}

// pass 2 ("default" mode): recompute z, GroupNorm affine, GELU, split, channels-last store
__global__ void __launch_bounds__(256) conv0_apply_gn_kernel(const float* __restrict__ x, long long L, int L0,
                                                             const float* __restrict__ w,
                                                             const float* __restrict__ scale,
                                                             const float* __restrict__ shift, const OutPlanes op) {
    __shared__ __align__(16) float xs[kXTile];
    const int b = blockIdx.y;
    const int t0 = blockIdx.x * kTCH;
    conv0_load_tile(x + (size_t)b * L, L, (long long)t0 * kC0S, xs);
    float w0[kC0K], w1[kC0K];
    const int c0 = 2 * threadIdx.x;
#pragma unroll
    for (int j = 0; j < kC0K; ++j) w0[j] = w[c0 * kC0K + j], w1[j] = w[(c0 + 1) * kC0K + j];
    const float sc0 = scale[b * kC0 + c0], sc1 = scale[b * kC0 + c0 + 1];
    const float sh0 = shift[b * kC0 + c0], sh1 = shift[b * kC0 + c0 + 1];
    __syncthreads();
    const int nt = min(kTCH, L0 - t0);
    const size_t e0 = ((size_t)b * L0 + t0) * kC0 + c0;  // element index of (frame t0, channel c0)
    for (int tl = 0; tl < nt; tl += 4) {
        float z0[4], z1[4];
        conv0_quad(xs, tl, w0, w1, z0, z1);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (tl + q < nt) {
                const float y0 = gelu_erf(fmaf(z0[q], sc0, sh0));
                const float y1 = gelu_erf(fmaf(z1[q], sc1, sh1));
                store_planes2(op, y0, y1, e0 + (size_t)(tl + q) * kC0);
            }
        }
    }
}

// "layer_norm" mode: z (+bias) -> LayerNorm over the 512 channels of each frame -> GELU
// (wav2vec2_model.py:2887-2897; Fp32LayerNorm eps 1e-5). Block-wide two-pass reduction per frame quad.
__global__ void __launch_bounds__(256) conv0_apply_ln_kernel(const float* __restrict__ x, long long L, int L0,
                                                             const float* __restrict__ w,
                                                             const float* __restrict__ cbias,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, const OutPlanes op) {
    __shared__ __align__(16) float xs[kXTile];
    __shared__ float red[8][4];
    __shared__ float stat[4];
    const int b = blockIdx.y;
    const int t0 = blockIdx.x * kTCH;
    conv0_load_tile(x + (size_t)b * L, L, (long long)t0 * kC0S, xs);
    float w0[kC0K], w1[kC0K];
    const int c0 = 2 * threadIdx.x;
#pragma unroll
    for (int j = 0; j < kC0K; ++j) w0[j] = w[c0 * kC0K + j], w1[j] = w[(c0 + 1) * kC0K + j];
    const float cb0 = cbias ? cbias[c0] : 0.f, cb1 = cbias ? cbias[c0 + 1] : 0.f;
    const float g0 = gamma[c0], g1 = gamma[c0 + 1], be0 = beta[c0], be1 = beta[c0 + 1];
    __syncthreads();
    const int nt = min(kTCH, L0 - t0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t e0 = ((size_t)b * L0 + t0) * kC0 + c0;
    for (int tl = 0; tl < nt; tl += 4) {
        float z0[4], z1[4], mean[4], rstd[4];
        conv0_quad(xs, tl, w0, w1, z0, z1);
#pragma unroll
        for (int q = 0; q < 4; ++q) z0[q] += cb0, z1[q] += cb1;
        // mean over 512 channels
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float s = warp_sum(z0[q] + z1[q]);
            if (lane == 0) red[warp][q] = s;
        }
        __syncthreads();
        if (threadIdx.x < 4) {
            float s = 0.f;
            for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
            stat[threadIdx.x] = s * (1.0f / kC0);
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) mean[q] = stat[q];
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float d0 = z0[q] - mean[q], d1 = z1[q] - mean[q];
            const float s = warp_sum(d0 * d0 + d1 * d1);
            if (lane == 0) red[warp][q] = s;
        }
        __syncthreads();
        if (threadIdx.x < 4) {
            float s = 0.f;
            for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
            stat[threadIdx.x] = rsqrtf(s * (1.0f / kC0) + 1e-5f);
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) rstd[q] = stat[q];
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (tl + q < nt) {
                const float y0 = gelu_erf(fmaf((z0[q] - mean[q]) * rstd[q], g0, be0));
                const float y1 = gelu_erf(fmaf((z1[q] - mean[q]) * rstd[q], g1, be1));
                store_planes2(op, y0, y1, e0 + (size_t)(tl + q) * kC0);
            }
        }
    }
}

cudaError_t launch_conv0_groupnorm(const float* x, int B, long long L, int L0, const float* w, const float* gamma,
                                   const float* beta, double* ws_part /*[B][nchunk][65]*/,
                                   float* ws_scale_shift /*[2][B][512]*/, const OutPlanes& op, cudaStream_t s) {
    const int nchunk = (L0 + kTCH - 1) / kTCH;
    float* scale = ws_scale_shift;
    float* shift = ws_scale_shift + (size_t)B * kC0;
    dim3 grid(nchunk, B);
    conv0_moments_kernel<<<grid, 256, 0, s>>>(x, L, L0, ws_part, nchunk);
    conv0_finalize_kernel<<<B, kC0, 0, s>>>(ws_part, nchunk, L0, w, gamma, beta, scale, shift);
    conv0_apply_gn_kernel<<<grid, 256, 0, s>>>(x, L, L0, w, scale, shift, op);
    return cudaGetLastError();
}

cudaError_t launch_conv0_layernorm(const float* x, int B, long long L, int L0, const float* w, const float* cbias,
                                   const float* gamma, const float* beta, const OutPlanes& op, cudaStream_t s) {
    const int nchunk = (L0 + kTCH - 1) / kTCH;
    dim3 grid(nchunk, B);
    conv0_apply_ln_kernel<<<grid, 256, 0, s>>>(x, L, L0, w, cbias, gamma, beta, op);
    return cudaGetLastError();
}

size_t conv0_ws_part_bytes(int B, int L0) { return (size_t)B * ((L0 + kTCH - 1) / kTCH) * kNMom * sizeof(double); }

// ------------------------------------------------------------------------------------------------
// modified CPC's conv 0 (s3prl/upstream/cpc/model.py CPCEncoder): Conv1d(1, 256, 10, stride 5, padding 3) + bias,
// ChannelNorm over the 256 channels of each frame (unbiased variance, eps inside the rsqrt), ReLU. One warp per
// output row; lane l holds channels 4 l .. 4 l + 3 and 128 + 4 l .. + 3. The output is conv 1's padded operand
// layout: utterance b owns rows [b R, b R + R), and row r holds frame r - pad when that is in [0, T0), zeros
// otherwise (every row is written, so a reused workspace never leaks into the result).
// ------------------------------------------------------------------------------------------------
static constexpr int kCpcC = 256;
static constexpr int kCpcK0 = 10;
static constexpr int kCpcS0 = 5;
static constexpr int kCpcP0 = 3;

__global__ void __launch_bounds__(256) cpc_conv0_kernel(const float* __restrict__ x, int B, long long L, int T0,
                                                        const float* __restrict__ w, const float* __restrict__ cbias,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, int R, int pad,
                                                        const OutPlanes op) {
    const int lane = threadIdx.x & 31;
    const size_t rows = (size_t)B * R;
    const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
    float wr[2][4][kCpcK0], cb[2][4], g[2][4], be[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int c = 128 * i + 4 * lane + e;
#pragma unroll
            for (int j = 0; j < kCpcK0; ++j) wr[i][e][j] = w[c * kCpcK0 + j];
            cb[i][e] = cbias[c], g[i][e] = gamma[c], be[i][e] = beta[c];
        }
    for (size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps) {
        const int b = (int)(row / R), t = (int)(row - (size_t)b * R) - pad;
        float4 y[2];
        if (t < 0 || t >= T0) {
            y[0] = y[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            const float* xb = x + (size_t)b * L;
            const long long s0 = (long long)t * kCpcS0 - kCpcP0;
            float xv[kCpcK0];
#pragma unroll
            for (int j = 0; j < kCpcK0; ++j) xv[j] = (s0 + j >= 0 && s0 + j < L) ? __ldg(xb + s0 + j) : 0.f;
            float z[2][4], s = 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float a = 0.f;
#pragma unroll
                    for (int j = 0; j < kCpcK0; ++j) a = fmaf(wr[i][e][j], xv[j], a);
                    z[i][e] = a + cb[i][e];
                    s += z[i][e];
                }
            const float mean = warp_sum(s) * (1.0f / kCpcC);
            float q = 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) q += (z[i][e] - mean) * (z[i][e] - mean);
            const float rstd = rsqrtf(warp_sum(q) * (1.0f / (kCpcC - 1)) + 1e-5f);
            float o[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) o[i][e] = relu_nan((z[i][e] - mean) * rstd * g[i][e] + be[i][e]);
            y[0] = make_float4(o[0][0], o[0][1], o[0][2], o[0][3]);
            y[1] = make_float4(o[1][0], o[1][1], o[1][2], o[1][3]);
        }
        store_planes4(op, y[0], row * kCpcC + 4 * lane);
        store_planes4(op, y[1], row * kCpcC + 128 + 4 * lane);
    }
}

cudaError_t launch_cpc_conv0(const float* x, int B, long long L, int T0, const float* w, const float* cbias,
                             const float* gamma, const float* beta, int R, int pad, const OutPlanes& op,
                             cudaStream_t s) {
    const size_t rows = (size_t)B * R;
    if (rows == 0) return cudaSuccess;
    size_t blocks = (rows + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    cpc_conv0_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, B, L, T0, w, cbias, gamma, beta, R, pad, op);
    return cudaGetLastError();
}

}  // namespace s3b
