// MAE-AST (s3prl/upstream/mae_ast/mae_ast.py) between post_extract_proj and the wav2vec 2.0 encoder layers: the
// sinusoidal positions of the valid tokens and, for the post-LN encoder, encoder.layer_norm. The front end is
// fbank.cu's mae_ast_fbank_kernel; the projection, the layers' GEMMs, attention and LayerNorm are the library's own.
#include "common.cuh"
#include "kernels.cuh"
#include "norm.cuh"

namespace s3b {

// one warp per row of x [B][N][768] (row b * N + tok): v = x + pe[tok] where tok < valid[b] (pe null: nothing added);
// ln: LayerNorm(v) -> x and op; else v -> x
__global__ void __launch_bounds__(256) mae_ast_embed_kernel(float* __restrict__ x, size_t M, int N,
                                                            const int* __restrict__ valid,
                                                            const float* __restrict__ pe, int ln,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, const OutPlanes op) {
    constexpr int V4 = 6, D = V4 * 128;
    const int lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int b = (int)(row / N), tok = (int)(row - (size_t)b * N);
    float4* xr = reinterpret_cast<float4*>(x + row * D);
    const bool add = pe != nullptr && tok < valid[b];
    const float4* pr = reinterpret_cast<const float4*>(pe + (size_t)tok * D);
    float4 v[V4];
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        v[i] = xr[lane + 32 * i];
        if (add) {
            const float4 p = __ldg(pr + lane + 32 * i);
            v[i].x += p.x, v[i].y += p.y, v[i].z += p.z, v[i].w += p.w;
        }
    }
    if (ln) {
        layernorm_row<V4>(v, lane, gamma, beta, 0, 1e-5f, x + row * D, op, row * D);
    } else if (add) {
#pragma unroll
        for (int i = 0; i < V4; ++i) xr[lane + 32 * i] = v[i];
    }
}

cudaError_t launch_mae_ast_embed(float* x, int B, int N, int D, const int* valid, const float* pe, int ln,
                                 const float* gamma, const float* beta, const OutPlanes& op, cudaStream_t s) {
    if (D != 768 || (ln && (gamma == nullptr || beta == nullptr))) return cudaErrorInvalidValue;
    const size_t M = (size_t)B * N;
    if (M == 0) return cudaSuccess;
    mae_ast_embed_kernel<<<(unsigned)((M + 7) / 8), 256, 0, s>>>(x, M, N, valid, pe, ln, gamma, beta, op);
    return cudaGetLastError();
}

}  // namespace s3b
