// WavLM gated relative-position bias helpers (s3prl/upstream/wavlm/modules.py:418-462,534-551) and
// layout helpers used by the parity-test entry points.
#include <math.h>

#include <vector>

#include "common.cuh"
#include "wavlm.cuh"

namespace s3b {

int wavlm_rel_bucket(int rel, int num_buckets, int max_distance) {
    // bidirectional: half of the buckets for each sign
    int nb = num_buckets / 2;
    int bucket = (rel > 0) ? nb : 0;
    const int a = rel < 0 ? -rel : rel;
    const int max_exact = nb / 2;
    if (a < max_exact) return bucket + a;
    // fp32 op sequence of the reference: log(float(a) / max_exact) / log(max_distance / max_exact) * (nb - max_exact)
    const float ratio = (float)a / (float)max_exact;
    const float denom = (float)log((double)max_distance / (double)max_exact);
    const float val = (logf(ratio) / denom) * (float)(nb - max_exact);
    long long large = (long long)max_exact + (long long)val;  // .to(torch.long) truncates toward zero
    if (large > nb - 1) large = nb - 1;
    return bucket + (int)large;
}

__global__ void rel_table_kernel(const float* __restrict__ emb, const int* __restrict__ buckets, int H, int R,
                                 float* __restrict__ table) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int h = blockIdx.y;
    // pre-multiplied by log2(e): the attention kernel adds it to scores that live in the exp2 domain
    if (r < R) table[(size_t)h * R + r] = emb[(size_t)buckets[r] * H + h] * 1.4426950408889634f;
}

cudaError_t launch_wavlm_rel_table(const float* emb, int num_buckets, int max_distance, int H, int T, float* table,
                                   cudaStream_t s) {
    const int R = 2 * T - 1;
    std::vector<int> b(R);
    for (int r = 0; r < R; ++r) b[r] = wavlm_rel_bucket(r - (T - 1), num_buckets, max_distance);
    int* dev = nullptr;
    cudaError_t e = cudaMalloc(&dev, R * sizeof(int));
    if (e != cudaSuccess) return e;
    e = cudaMemcpyAsync(dev, b.data(), R * sizeof(int), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        dim3 grid((R + 255) / 256, H);
        rel_table_kernel<<<grid, 256, 0, s>>>(emb, dev, H, R, table);
        e = cudaGetLastError();
    }
    cudaStreamSynchronize(s);  // pageable staging + free: table rebuilt only when T changes
    cudaFree(dev);
    return e;
}

// eight lanes per (token, head): 64 inputs -> 8 outputs -> 2 gates. The reference sums the 8 grep_linear outputs in two
// groups of four before the sigmoids (modules.py:541-546: view(..., 2, 4).sum(-1)), so only the two summed weight
// rows (and summed biases) are needed: 2 x 64 FMAs per thread instead of 8 x 64 (same value up to fp32 summation
// order). The two combined rows are built in shared memory by every block.
__global__ void __launch_bounds__(256) wavlm_gate_kernel(const OutPlanes xp, size_t M, int T,
                                                         int H, int D, const float* __restrict__ gw,
                                                         const float* __restrict__ gb, const float* __restrict__ ga,
                                                         float* __restrict__ gate) {
    __shared__ __align__(16) float sw[2 * 64 + 2];
    if (gw != nullptr && threadIdx.x < 130) {
        const int i = threadIdx.x;
        if (i < 128) {
            const int g = i >> 6, c = i & 63;
            sw[i] = (gw[(4 * g) * 64 + c] + gw[(4 * g + 1) * 64 + c]) + (gw[(4 * g + 2) * 64 + c] + gw[(4 * g + 3) * 64 + c]);
        } else {
            const int g = i - 128;
            sw[i] = (gb[4 * g] + gb[4 * g + 1]) + (gb[4 * g + 2] + gb[4 * g + 3]);
        }
    }
    __syncthreads();
    // eight lanes per (token, head): lane c loads the c-th 16-byte chunk of the hi and lo planes, so a warp load covers
    // four contiguous 128-byte head rows (one thread per head made every load touch 32 different lines)
    const size_t gidx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t idx = gidx >> 3;
    const int c = (int)(gidx & 7);
    const bool ok = idx < M * (size_t)H;
    const size_t m = ok ? idx / H : 0;
    const int h = ok ? (int)(idx - m * H) : 0;
    const int b = (int)(m / T), t = (int)(m - (size_t)b * T);
    float g1 = 1.0f;
    if (gw != nullptr) {  // kernel-uniform
        float sa = 0.f, sb = 0.f;
        if (ok) {
            const size_t off = m * (size_t)D + (size_t)h * 64 + 8 * (size_t)c;
            float xv[8];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 v2 = load_planes2(xp, off + 2 * e);
                xv[2 * e] = v2.x, xv[2 * e + 1] = v2.y;
            }
            const float4* w0 = reinterpret_cast<const float4*>(sw);
            const float4* w1 = reinterpret_cast<const float4*>(sw + 64);
            const float4 a0 = w0[2 * c], a1 = w0[2 * c + 1], b0 = w1[2 * c], b1 = w1[2 * c + 1];
            sa = fmaf(a0.x, xv[0], sa), sa = fmaf(a0.y, xv[1], sa), sa = fmaf(a0.z, xv[2], sa), sa = fmaf(a0.w, xv[3], sa);
            sa = fmaf(a1.x, xv[4], sa), sa = fmaf(a1.y, xv[5], sa), sa = fmaf(a1.z, xv[6], sa), sa = fmaf(a1.w, xv[7], sa);
            sb = fmaf(b0.x, xv[0], sb), sb = fmaf(b0.y, xv[1], sb), sb = fmaf(b0.z, xv[2], sb), sb = fmaf(b0.w, xv[3], sb);
            sb = fmaf(b1.x, xv[4], sb), sb = fmaf(b1.y, xv[5], sb), sb = fmaf(b1.z, xv[6], sb), sb = fmaf(b1.w, xv[7], sb);
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        sa += sw[128], sb += sw[129];
        const float a = 1.0f / (1.0f + expf(-sa));
        const float bb = 1.0f / (1.0f + expf(-sb));
        g1 = a * (bb * ga[h] - 1.0f) + 2.0f;
    }
    if (ok && c == 0) gate[((size_t)b * H + h) * T + t] = g1;
}

cudaError_t launch_wavlm_gate(const OutPlanes& xp, size_t M, int B, int T, int H, int D, const float* grep_w,
                              const float* grep_b, const float* grep_a, float* gate, cudaStream_t s) {
    (void)B;
    const size_t n = M * (size_t)H * 8;  // eight lanes per (token, head)
    const unsigned blocks = (unsigned)((n + 255) / 256);
    wavlm_gate_kernel<<<blocks, 256, 0, s>>>(xp, M, T, H, D, grep_w, grep_b, grep_a, gate);
    return cudaGetLastError();
}

__global__ void qkv_scatter_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                   const float* __restrict__ v, int B, int T, int Tp, int H, int hd, float q_scale,
                                   __nv_bfloat16* q_hi, __nv_bfloat16* q_lo, __nv_bfloat16* k_hi,
                                   __nv_bfloat16* k_lo, __nv_bfloat16* vt_hi, __nv_bfloat16* vt_lo) {
    const int D = H * hd;
    const size_t n = (size_t)B * T * D;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t m = i / D;
        const int col = (int)(i - m * D);
        const int b = (int)(m / T), t = (int)(m - (size_t)b * T);
        const int h = col / hd, d = col - h * hd;
        const size_t bh = (size_t)b * H + h;
        __nv_bfloat16 hi, lo;
        split_bf16(q[i] * q_scale, hi, lo);
        q_hi[(bh * T + t) * hd + d] = hi, q_lo[(bh * T + t) * hd + d] = lo;
        split_bf16(k[i], hi, lo);
        k_hi[(bh * T + t) * hd + d] = hi, k_lo[(bh * T + t) * hd + d] = lo;
        split_bf16(v[i], hi, lo);
        vt_hi[(bh * hd + d) * (size_t)Tp + t] = hi, vt_lo[(bh * hd + d) * (size_t)Tp + t] = lo;
    }
}

cudaError_t launch_qkv_scatter(const float* q, const float* k, const float* v, int B, int T, int Tp, int H, int hd,
                               float q_scale, __nv_bfloat16* q_hi, __nv_bfloat16* q_lo, __nv_bfloat16* k_hi,
                               __nv_bfloat16* k_lo, __nv_bfloat16* vt_hi, __nv_bfloat16* vt_lo, cudaStream_t s) {
    qkv_scatter_kernel<<<132 * 4, 256, 0, s>>>(q, k, v, B, T, Tp, H, hd, q_scale, q_hi, q_lo, k_hi, k_lo, vt_hi, vt_lo);
    return cudaGetLastError();
}

// the value a consumer of the operand sees: the same decode as load_planes2, element pairs
__global__ void planes_to_f32_kernel(const OutPlanes p, size_t n2, float* __restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (size_t)gridDim.x * blockDim.x) {
        const float2 v = load_planes2(p, 2 * i);
        out[2 * i] = v.x, out[2 * i + 1] = v.y;
    }
}

cudaError_t launch_planes_to_f32(const OutPlanes& p, size_t n, float* out, cudaStream_t s) {
    if (n & 1) return cudaErrorInvalidValue;
    planes_to_f32_kernel<<<132 * 4, 256, 0, s>>>(p, n / 2, out);
    return cudaGetLastError();
}

}  // namespace s3b
