// The per-row LayerNorm of norm.cu's layernorm_kernel, shared with kernels that form their row in registers first
// (mae_ast.cu's positions + LayerNorm).
#pragma once
#include "common.cuh"

namespace s3b {

// y = LayerNorm_D(v) * gamma + beta (biased var), optional GELU, of one row held by a warp: v[i] = columns
// 4 (lane + 32 i) .. + 3, D = 128 V4. Two-pass statistics in registers. y goes to out_row (fp32, may be null) and to
// op at element offset e0 of the row (op.hi may be null). out_row may alias the row's source.
template <int V4>
__device__ __forceinline__ void layernorm_row(const float4 (&v)[V4], int lane, const float* __restrict__ gamma,
                                              const float* __restrict__ beta, int gelu, float eps, float* out_row,
                                              const OutPlanes& op, size_t e0) {
    constexpr int D = V4 * 128;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
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
        if (out_row != nullptr) reinterpret_cast<float4*>(out_row)[c4] = y;
        if (op.hi != nullptr) store_planes4(op, y, e0 + 4 * (size_t)c4);
    }
}

}  // namespace s3b
