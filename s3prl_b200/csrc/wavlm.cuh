// WavLM-specific pieces and small test helpers (wavlm.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace s3b {

// Host: bucket index of relative position `rel` = key - query (bit-exact restatement of
// MultiheadAttention._relative_positions_bucket, s3prl/upstream/wavlm/modules.py:418-448, bidirectional).
int wavlm_rel_bucket(int rel, int num_buckets, int max_distance);

// table[h][r] = emb[bucket(r - (T-1))][h] for r in [0, 2T-1)  (compute_bias, modules.py:450-462; Toeplitz)
cudaError_t launch_wavlm_rel_table(const float* emb /*[num_buckets][H] device*/, int num_buckets, int max_distance,
                                   int H, int T, float* table /*[H][2T-1] device*/, cudaStream_t s);

// gate[b][h][t] = ga*(gb*grep_a[h]-1)+2, (ga,gb) = sigmoid(sum4(grep_linear(x[b,t,h*64:(h+1)*64])))
// (modules.py:534-551). grep_w == nullptr (gru_rel_pos off) -> gate = 1.
cudaError_t launch_wavlm_gate(const OutPlanes& xp, size_t M, int B, int T, int H, int D, const float* grep_w,
                              const float* grep_b, const float* grep_a, float* gate, cudaStream_t s);

// test helpers: fp32 [B][T][H*hd] q/k/v -> the attention kernel's operand layout; n (even) elements of an operand in
// either format -> fp32
cudaError_t launch_qkv_scatter(const float* q, const float* k, const float* v, int B, int T, int Tp, int H, int hd,
                               float q_scale, __nv_bfloat16* q_hi, __nv_bfloat16* q_lo, __nv_bfloat16* k_hi,
                               __nv_bfloat16* k_lo, __nv_bfloat16* vt_hi, __nv_bfloat16* vt_lo, cudaStream_t s);
cudaError_t launch_planes_to_f32(const OutPlanes& p, size_t n, float* out, cudaStream_t s);

}  // namespace s3b
