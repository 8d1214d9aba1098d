// Host-visible description of one error-compensated GEMM launch (gemm_sm90.cu).
// One kernel serves every contraction on the hot path: the strided conv stack
// (conv 1..6 as implicit GEMM on channels-last activations), post_extract_proj, the grouped positional
// conv (one k-block per tap, time shift expressed in the TMA row coordinate), QKV, out_proj, fc1, fc2.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace s3b {

struct GemmParams {
    // A operand (activations): bf16 hi / lo, 3-D tensor maps (k, row, batch), box {64, 128 / cluster_n, 1}, SWIZZLE_128B
    CUtensorMap a_hi, a_lo;
    // B operand (weights, one [N][K] K-major matrix): bf16 hi / lo, tensor maps (k, n, 1), box {64, bn, 1}
    CUtensorMap b_hi, b_lo;

    // scheme 1 ("f16q8", bn 128 or 256 only): fp16 main product + two e4m3 correction products.
    //   a_hi / b_hi are the fp16 planes (box {64, rows}, SWIZZLE_128B), a_q8 / b_q8 the interleaved e4m3 planes
    //   (common.cuh: q8_off) as byte maps of 2 K bytes per row (box {128, rows}, SWIZZLE_128B: one 64-wide k-block);
    //   a_lo / b_lo are unused. K % 128 == 0, and the kernel walks the 64-wide k-blocks twice: num_k_blocks stages of
    //   e4m3 corrections, then num_k_blocks of fp16 products.
    int scheme;
    CUtensorMap a_q8, b_q8;

    // ---- tiling: every k-block is 64 elements of K wide --------------------------------------------------------
    int batches;            // extent of A's 3rd dim that is tiled over
    int rows_per_batch;     // valid output rows per batch
    int tiles_m_per_batch;  // ceil(rows_per_batch / 128)
    int n_tiles;            // output column tiles
    int bn;                 // columns per tile, the kernel's BN (multiple of 16 <= 256, or 80 / 120: pos_conv groups)
    int num_k_blocks;       // k-blocks per output tile
    // 128-wide tiles: CTAs per thread-block cluster along N (0 or 1: no cluster, 2, 4; divides n_tiles). The CTAs of
    // a cluster take adjacent column tiles of the same rows, and each loads 128 / cluster_n rows of every A box for
    // all of them (TMA multicast): the A tensor maps then have box height 128 / cluster_n.
    int cluster_n;
    // k-block kb reads   A box at (a_k_per_ntile*n_tile + (kb % kb_per_row)*64,
    //                              row0 + kq*a_row_step + a_row_off + (kq >= a_gap_at ? a_gap : 0), batch)
    //                    with kq = kb / kb_per_row
    //                    B box at (kb*64, n_tile*bn, 0)
    int kb_per_row;
    int a_row_step;
    int a_row_off;
    int a_k_per_ntile;
    // a tap convolution that skips a band of taps (the NPC masked conv): k-block rows kq >= a_gap_at read a_gap rows
    // further on. a_gap 0 is the plain walk.
    int a_gap_at;
    int a_gap;

    // ---- epilogue: v = acc (+bias[n]) ; act ; (+residual[m][n]) ; row_mask[m] ? 0 -----------------
    // gelu: the activation: 0 = none, 1 = GELU (exact erf), 2 = SiLU (x * sigmoid(x), the Conformer's Swish),
    //       3 = ReLU, 4 = tanh
    // res_first: v = acc (+bias) (+residual) ; act instead (the NPC ConvBlock's act(out + res)); out_pre is then unused
    // The launch picks one kernel instantiation per output kind: out_f32, operand planes (out_hi ...), both (widths
    // >= 128 only) or the QKV scatter (widths >= 128 only). A launch with none of them is an error.
    int out_rows_per_batch;  // flat output row m = batch*out_rows_per_batch + row
    int ldo;                 // leading dimension (elements) of out_f32/out_hi/out_lo/residual
    const float* bias;
    const float* residual;
    const uint8_t* row_mask;
    int gelu;
    int res_first;
    float* out_f32;
    __nv_bfloat16* out_hi;
    __nv_bfloat16* out_lo;
    // out_fmt 1: out_hi is an fp16 plane and out_q8 the interleaved e4m3 plane of the f16q8 operand format;
    // out_fmt 0: out_hi / out_lo are the bf16 hi / lo planes.
    int out_fmt;
    uint8_t* out_q8;
    float* out_pre;  // optional: v BEFORE the residual add (fc2 output, "fairseq_layers_before_residual"), same layout

    // ---- epilogue, QKV scatter mode (qkv_mode != 0): columns [0,D) -> q*scale, [D,2D) -> k, [2D,3D) -> v
    // q,k: [B][H][T][hd] split bf16 ; v transposed: [B][H][hd][Tp] split bf16. Flat row m = b*T + t. hd (below) is
    // the head width, 64, 80 or 120 (D = H * hd).
    // qkv_col0: the scatter column of GEMM column 0 (the Conformer runs [q | k] with 0 and v alone with 2D; `bias` then
    // points at the launch's own columns)
    int qkv_mode;
    int T, Tp, H, D;
    float q_scale;
    int qkv_col0;
    __nv_bfloat16 *q_hi, *q_lo, *k_hi, *k_lo, *vt_hi, *vt_lo;

    double alg_flops;  // host-side accounting only: 2*M*N*K with the un-padded K

    // bf16x3: 16-wide MMA k-steps issued per 64-wide k-block (0 = all 4). pos_conv with 48 channels per group
    // loads 64-wide boxes but only the first 3 k-steps carry non-zero weights.
    int k_steps;

    int hd;                 // QKV scatter: head width
    unsigned int hd_magic;  // 2^32 / hd rounded up: column / hd = __umulhi(column, hd_magic) for columns < 2^16
    int qk_head_step;       // (T - 1) * hd
};

// Launch on `stream`. Returns cudaGetLastError() of the launch.
cudaError_t launch_gemm(const GemmParams& p, int sm_count, cudaStream_t stream);

// Encode a 3-D bf16 tensor map with the 128B swizzle (box0 = 64 elements). strides in ELEMENTS for dims 1 and 2.
// Returns 0 on success, else a CUresult / -1 (driver entry point missing).
int encode_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                        uint64_t stride2, uint32_t box0, uint32_t box1);
// Same for a byte plane (the interleaved e4m3 plane): box0 is 128 bytes, one SWIZZLE_128B row. Strides in bytes.
int encode_tmap_u8_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                      uint64_t stride2, uint32_t box0, uint32_t box1);

}  // namespace s3b
