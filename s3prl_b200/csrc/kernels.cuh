// Launchers of the non-GEMM kernels (frontend.cu, norm.cu, attention.cu, fbank.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace s3b {

// ---- frontend.cu ---------------------------------------------------------------------------------
cudaError_t launch_split(const float* x, __nv_bfloat16* hi, __nv_bfloat16* lo, size_t n, cudaStream_t s);
cudaError_t launch_wav_pack(const float* const* wavs, const long long* lens, int B, long long Lpad, int normalize,
                            float* mean_rstd_ws, float* out, cudaStream_t s);
size_t conv0_ws_part_bytes(int B, int L0);
cudaError_t launch_split_q8(const float* x, __nv_bfloat16* p16, uint8_t* h8, uint8_t* l8, size_t n, int weight,
                            cudaStream_t s);
cudaError_t launch_conv0_groupnorm(const float* x, int B, long long L, int L0, const float* w, const float* gamma,
                                   const float* beta, double* ws_part, float* ws_scale_shift, const OutPlanes& op,
                                   cudaStream_t s);
cudaError_t launch_conv0_layernorm(const float* x, int B, long long L, int L0, const float* w, const float* cbias,
                                   const float* gamma, const float* beta, const OutPlanes& op, cudaStream_t s);
// modified CPC's conv 0 (w [256][10], stride 5, padding 3, + bias) + ChannelNorm + ReLU over x [B][L] into T0 frames
// of conv 1's padded operand layout: R rows per utterance, row r = frame r - pad (zeros outside [0, T0))
cudaError_t launch_cpc_conv0(const float* x, int B, long long L, int T0, const float* w, const float* cbias,
                             const float* gamma, const float* beta, int R, int pad, const OutPlanes& op,
                             cudaStream_t s);

// ---- norm.cu -------------------------------------------------------------------------------------
// y = LayerNorm_D(x) * gamma + beta (biased var; eps 1e-5, SSAST's DeiT blocks 1e-6), optional GELU; D in {384, 512,
// 640, 768, 1024, 1280, 1920}. Any of out_f32 / (out_hi,out_lo) may be null. x and out_f32 may alias.
cudaError_t launch_layernorm(const float* x, size_t M, int D, const float* gamma, const float* beta, int gelu,
                             float* out_f32, const OutPlanes& op, cudaStream_t s, float eps = 1e-5f);
// modified CPC: y = relu(ChannelNorm_256(x)) (unbiased var, eps 1e-5) of x [B][T][256] into op with R rows per
// utterance, row r = frame r - pad (zeros outside [0, T)); out_f32 [B][T][256] only with R == T and pad == 0
cudaError_t launch_channelnorm_relu(const float* x, int B, int T, int R, int pad, const float* gamma,
                                    const float* beta, float* out_f32, const OutPlanes& op, cudaStream_t s);
// Conformer: y = LayerNorm_D(x) -> op, rope(y) -> op_rope; frame t = row % T, cs [>= T][64] = cos | sin of the 32 angles
cudaError_t launch_layernorm_rope(const float* x, size_t M, int T, int D, const float* gamma, const float* beta,
                                  const float* cs, const OutPlanes& op, const OutPlanes& op_rope, cudaStream_t s);
// out[m] = sum_l w[l] * hs[l][m]   (Featurizer._weighted_sum, interfaces.py:217-248; w already softmaxed)
cudaError_t launch_posconv_combine(const float* z, const float* x, const float* bias, int B, int T, int D, int cpg,
                                   const float* gamma, const float* beta, int do_ln, int mode, float* out_f32,
                                   const OutPlanes& op, cudaStream_t s);
cudaError_t launch_weighted_sum(const float* hs, int NL, size_t n_per_layer, const float* w, float* out,
                                cudaStream_t s);
// grad_w[l] = sum_m hs[l][m] * gout[m]
cudaError_t launch_weighted_sum_bwd(const float* hs, int NL, size_t n_per_layer, const float* gout, float* grad_w,
                                    cudaStream_t s);

// ---- conformer.cu --------------------------------------------------------------------------------
// out = SiLU(depthwise_conv_k(GLU(x)) + bias) per utterance, zero padding outside [0, T); x [B][T][2D] fp32,
// w [D][k] (BatchNorm folded in), bias [D]; D % 64 == 0, k odd, k <= kDwMaxKernel. out: operand planes [B][T][D].
static constexpr int kDwMaxKernel = 63;
cudaError_t launch_depthwise_glu(const float* x, int B, int T, int D, int k, const float* w, const float* bias,
                                 const OutPlanes& op, cudaStream_t s);

// ---- fbank.cu: the DeCoAR 2.0 front end -------------------------------------------------------------------------
// K of DeCoAR 2.0's post_extract_proj GEMM: the 80 mel bins, zero-padded to the f16q8 GEMM's K % 128 rule
static constexpr int kDecoar2K = 128;
// builds the fbank tables and the hamming window on the current device (synchronous; once per device)
cudaError_t init_fbank_tables();
// kaldi fbank with the hamming window into fb [B][max_frames][80] (frames t < m_b of each utterance), then CMVN over
// each utterance's m_b frames and y[::frame_step] into operand planes op [B * T][kDecoar2K] (zero beyond 80 columns and
// T_b = ceil(m_b / frame_step) rows). frame_step: 2 for DeCoAR 2.0, 1 for APC. Needs init_fbank_tables() on this
// device first. m_b >= 2 (m_b == 1 gives NaN, as the reference's unbiased std).
cudaError_t launch_decoar2_features(const float* const* wavs_dev, const long long* lens_dev, int B, int max_frames,
                                    int T, int frame_step, float* fb, const OutPlanes& op, cudaStream_t s);

// ---- fbank.cu: SSAST's front end -------------------------------------------------------------------------------
// kaldi fbank (hanning window, 128 mel bins) of each S-sample window of each utterance (zero past lens[b]), normalised
// (y + 4.2677393) / 9.1379948, rows from 1 + (S - 400) / 160 up to TL zero: out [B * nseg][TL][128], row block
// b * nseg + s. Needs init_fbank_tables() on this device first.
cudaError_t launch_ssast_fbank(const float* const* wavs_dev, const long long* lens_dev, int B, int nseg, int S,
                               int TL, float* out, cudaStream_t s);

// ---- ssast.cu: SSAST's patch operand, tokens and output layout ----------------------------------------------------
// The patch-embedding GEMM's A operand from the features feat [SB][TL][128]: frame model (patch_f 1) the features
// themselves as operand planes [SB][TL][128] (the implicit GEMM reads rows t and t + 1 of a segment); patch model
// (patch_f 12) the 16 x 16 patches at stride 10 gathered into planes [SB][12 * tdim][256], row fi * tdim + ti, column
// kf * 16 + kt = feat[sb][10 ti + kt][10 fi + kf].
cudaError_t launch_ssast_patches(const float* feat, int SB, int TL, int patch_f, int tdim, const OutPlanes& op,
                                 cudaStream_t s);
// x [SB][2 + P][D] holds the patch GEMM's output (+ bias) in rows 2..: row 0 = cls + pos[0], row 1 = dist + pos[1],
// row 2 + p += pos[2 + p]
cudaError_t launch_ssast_tokens(float* x, const float* cls, const float* dist, const float* pos, int SB, int P, int D,
                                cudaStream_t s);
// One hidden state from the residual stream x [B * nseg][2 + P][D]: out [B][T][patch_f * D], out[b][t][fi * D + d] =
// x[b * nseg + t / tdim][2 + fi * tdim + t % tdim][d] (class tokens dropped, frequency patches folded into channels,
// time trimmed to T <= nseg * tdim). D % 4 == 0.
cudaError_t launch_ssast_fold(const float* x, int B, int nseg, int P, int tdim, int patch_f, int D, int T, float* out,
                              cudaStream_t s);

// ---- gru.cu: the GRU recurrence of APC / VQ-APC (cluster-resident W_hh) ------------------------------------------
static constexpr int kGruHidden = 512;  // hidden size the kernel is built for
static constexpr int kGruGroup = 4;     // utterances per cluster
static constexpr int kGruCtas = 16;     // CTAs per cluster (non-portable cluster size), 32 hidden units each
struct GruParams {
    const float* xg;   // [B][T][3H]: W_i x + b_i, with b_hr / b_hz added to the r / z columns (gate order r, z, n)
    const float* whh;  // [3H][H] weight_hh_l0
    const float* bhn;  // [H] the n third of bias_hh_l0
    const float* res;  // optional [B][T][H]: added to the layer output (the residual), not to the state
    const int* len;    // [B] valid frames; frames t >= len[b] are written as zero
    const int* order;  // [B] utterance indices, longest first: cluster g runs order[4g .. 4g + 3]
    int B, T;
    float* out;        // [B][T][H] layer output (fp32)
    OutPlanes op;      // optional [B * T][H] operand planes of the same values (op.hi null: none)
};
cudaError_t launch_gru(const GruParams& p, cudaStream_t s);
// clusters of the recurrence kernel that can be co-resident on the current device (0: the kernel cannot run)
cudaError_t gru_max_active_clusters(int* n);
size_t gru_smem_bytes();
// xg[r][q * H + u] += bhh[q * H + u] for q in {0, 1} (r, z) and rows r < rows: the bias folding the model does in its
// GEMM epilogue, for the building-block entry point
cudaError_t launch_gru_fold_bias(float* xg, const float* bhh, size_t rows, cudaStream_t s);

// ---- lstm.cu: the LSTM recurrence of DeCoAR (grid-resident W_hh) --------------------------------------------------
static constexpr int kLstmHidden = 1024;    // hidden size the kernel is built for
static constexpr int kLstmGroup = 16;       // utterances staged per group-step
static constexpr int kLstmCtas = 128;       // CTAs of the cooperative grid (one per SM), 8 hidden units each
static constexpr int kLstmMaxBatch = 512;   // utterances per launch; launch_lstm splits larger batches
struct LstmParams {
    const float* xg;    // [B][T][4H]: W_ih x + b_ih (+ b_hh), gate order i, f, g, o
    const float* whh;   // [4H][H] weight_hh_l{k}
    const float* bhh;   // optional [4H], added to xg (null when the GEMM bias already holds it)
    const int* len;     // [B] valid frames; frames t >= len[b] are written as zero
    const int* order;   // [B] utterance indices, longest first
    int B, T;
    int direction;      // 0: t = 0 .. len - 1; 1: t = len - 1 .. 0 (outputs stay in natural time)
    float* out;         // optional [B][T][ldo] fp32 layer output, columns col0 .. col0 + H - 1
    int ldo, col0;
    OutPlanes op;       // optional operand planes of the same values, same layout (op.hi null: none)
    float* hbuf;        // [2][min(B, kLstmMaxBatch)][H] state exchange buffer (lstm_hbuf_floats)
    unsigned int* counter;  // grid-barrier counter, zeroed on the stream before every launch
};
cudaError_t launch_lstm(const LstmParams& p, cudaStream_t s);
size_t lstm_hbuf_floats(int B);
size_t lstm_smem_bytes();
// ok = 1 when the device can host the grid: >= kLstmCtas SMs, enough opt-in shared memory, cooperative launch and one
// CTA per SM; sms / smem_optin report the device's values for messages
cudaError_t lstm_fits(int* ok, int* sms, int* smem_optin);

// ---- cpc_lstm.cu: the LSTM recurrence of modified CPC (cluster-resident W_hh) -------------------------------------
static constexpr int kCpcLstmHidden = 256;  // hidden size the kernel is built for
static constexpr int kCpcLstmGroup = 4;     // utterances per cluster
static constexpr int kCpcLstmCtas = 8;      // CTAs per cluster (portable cluster size), 32 hidden units each
struct CpcLstmParams {
    const float* xg;   // [B][T][4H]: W_ih x + b_ih + b_hh, gate order i, f, g, o
    const float* whh;  // [4H][H] weight_hh_l{k}
    int B, T;          // every utterance runs all T steps; cluster g runs utterances 4g .. 4g + 3
    float* out;        // optional [B][T][H] layer output (fp32)
    OutPlanes op;      // optional [B * T][H] operand planes of the same values (op.hi null: none)
};
cudaError_t launch_cpc_lstm(const CpcLstmParams& p, cudaStream_t s);
// clusters of the recurrence kernel that can be co-resident on the current device (0: the kernel cannot run)
cudaError_t cpc_lstm_max_active_clusters(int* n);

// ---- peer.cu: fused weighted sum + push all-gather over peer memory --------------------------------------------------
cudaError_t launch_weighted_sum_push(const float* hs, int NL, size_t n_per_layer, size_t layer_stride, const float* w,
                                     float* const* peer_dst, uint32_t* const* peer_flag, int n_peers, uint32_t seq,
                                     unsigned int* counter, cudaStream_t s);
cudaError_t launch_wait_flags(const uint32_t* flags, int n, uint32_t seq, cudaStream_t s);

// ---- attention.cu --------------------------------------------------------------------------------
struct AttnParams {
    CUtensorMap q_hi, q_lo;    // [B*H][T][hd]  box {64, 128, 1}
    CUtensorMap k_hi, k_lo;    // [B*H][T][hd]  box {64,  64, 1}
    CUtensorMap vt_hi, vt_lo;  // [B*H][hd][Tp] (dim0 = T valid keys) box {64, hd, 1}
    int B, H, T, D;
    const int* kv_len;          // [B] valid (un-padded) key count, >= 1
    // optional WavLM gated relative position bias: S[q][k] += gate[b][h][q] * table[h][k - q + bias_center]
    const float* bias_table;    // [H][bias_stride], entry (h, k - q + bias_center); or null
    int bias_stride, bias_center;
    const float* gate;          // [B][H][T] or null
    OutPlanes ctx;  // [B*T][D] A operand of out_proj, in either operand format
    // optional timeline (debug): clock64 stamps of CTA `trace_block`, [2 roles][16 blocks][8 slots]
    long long* trace;
    int trace_block;
    int hd;  // head width: 64, 80 or 120 (D = H * hd); the bias above needs 64
};
cudaError_t launch_attention(const AttnParams& p, cudaStream_t s);

}  // namespace s3b
