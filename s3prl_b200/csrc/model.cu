// Host-side orchestration of the upstream forward + the C ABI (include/s3prl_b200.h).
//
// Reference call stack being replaced:
//   UpstreamExpert.forward                      s3prl/upstream/hubert/expert.py:56-72
//   HubertModel.forward / extract_features      s3prl/upstream/hubert/hubert_model.py:466-513,566-582
//   ConvFeatureExtractionModel.forward          s3prl/upstream/wav2vec2/wav2vec2_model.py:2927-2934
//   TransformerEncoder.extract_features         s3prl/upstream/wav2vec2/wav2vec2_model.py:3054-3121
//   TransformerSentenceEncoderLayer.forward     s3prl/upstream/wav2vec2/wav2vec2_model.py:3260-3322
//   WavLM TransformerEncoder / layer            s3prl/upstream/wavlm/WavLM.py:599-645,709-774
//   ConformerEncoder / ConformerEncoderLayer    s3prl/upstream/wav2vec2/wav2vec2_model.py:3132-3211,441-578 (rope)
// Data layout in HBM: every activation is token-major / channels-last ([B][L][C]); GEMM operands are kept as
// two bf16 planes (hi, lo); hidden states are written once, in fp32, straight into the caller's
// [NL+1][B][T][D] buffer (the reference's forward hooks become plain views of that buffer).
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/s3prl_b200.h"
#include "gemm.cuh"
#include "kernels.cuh"
#include "wavlm.cuh"

using namespace s3b;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;

static int fail(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return 1;
}
#define CUDA_OK(expr)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                           __FILE__, __LINE__);                                    \
    } while (0)
#define S3B_OK(expr)            \
    do {                        \
        int _r = (expr);        \
        if (_r != 0) return _r; \
    } while (0)

// ------------------------------------------------------------------------------------------------
// containers
// ------------------------------------------------------------------------------------------------
struct HostTensor {
    std::vector<int64_t> shape;
    std::vector<float> data;
    size_t numel() const { return data.size(); }
};

// bumped on every (re)allocation: cached launch plans hold raw device pointers and are rebuilt when it moves
static uint64_t g_alloc_generation = 1;

// Owns one device allocation: freed on destruction, moved but never copied (a copy would free it twice)
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr, o.bytes = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            if (p) cudaFree(p);
            p = o.p, bytes = o.bytes;
            o.p = nullptr, o.bytes = 0;
        }
        return *this;
    }
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    int ensure(size_t n) {
        n += 1 << 16;  // slack: TMA boxes may over-read the last rows of a view (never consumed)
        if (n <= bytes) return 0;
        if (p) cudaFree(p);
        p = nullptr, bytes = 0;
        ++g_alloc_generation;
        cudaError_t e = cudaMalloc(&p, n);
        if (e != cudaSuccess) return fail("cudaMalloc(%zu) failed: %s", n, cudaGetErrorString(e));
        // zero once so that never-written padding is finite (0 * garbage must not be NaN)
        e = cudaMemset(p, 0, n);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();  // callers may use non-blocking streams
        if (e != cudaSuccess) return fail("cudaMemset failed: %s", cudaGetErrorString(e));
        bytes = n;
        return 0;
    }
    template <class T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};
static_assert(!std::is_copy_constructible<DevBuf>::value, "DevBuf owns its allocation: a copy would free it twice");

// One GEMM operand in HBM, 4 bytes per element in either format:
//   fmt 0 (bf16x3 scheme): `hi` = bf16 hi plane, `lo` = bf16 lo plane
//   fmt 1 (f16q8 scheme) : `hi` = fp16 plane, `lo` holds the two e4m3 planes back to back (h8 at 0, l8 at l8_off)
struct SplitBuf {
    DevBuf hi, lo;
    size_t l8_off = 0;
    int ensure(size_t elems) {
        S3B_OK(hi.ensure(elems * 2));
        const size_t before = lo.bytes;
        S3B_OK(lo.ensure(elems * 2));
        if (lo.bytes != before) l8_off = (elems + 255) & ~(size_t)255;
        return 0;
    }
    __nv_bfloat16* h() const { return hi.as<__nv_bfloat16>(); }
    __nv_bfloat16* l() const { return lo.as<__nv_bfloat16>(); }
    uint8_t* h8() const { return lo.as<uint8_t>(); }
    uint8_t* l8() const { return lo.as<uint8_t>() + l8_off; }
    OutPlanes planes(int fmt) const { return OutPlanes{h(), fmt ? nullptr : l(), fmt ? h8() : nullptr, fmt ? l8() : nullptr, fmt}; }
};

// Streams, events and pinned host memory, released on destruction
struct StreamDestroy {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
struct EventDestroy {
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct PinnedFree {
    void operator()(char* p) const { cudaFreeHost(p); }
};
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;
using Event = std::unique_ptr<CUevent_st, EventDestroy>;
using PinnedBuf = std::unique_ptr<char, PinnedFree>;

// the stream / event on first use: a non-blocking stream, an event without timing
static int ensure_stream(Stream& s) {
    if (s) return 0;
    cudaStream_t h = nullptr;
    CUDA_OK(cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking));
    s.reset(h);
    return 0;
}
static int ensure_event(Event& e) {
    if (e) return 0;
    cudaEvent_t h = nullptr;
    CUDA_OK(cudaEventCreateWithFlags(&h, cudaEventDisableTiming));
    e.reset(h);
    return 0;
}

// Default operand scheme: 1 = f16q8 (fp16 product + two e4m3 corrections): parity class of bf16x3 on every golden, and
// 2 MMA slots per 16 of K instead of 3 (e4m3 wgmma runs at twice the fp16 rate); bf16x3 (0) stays available through
// S3B_GEMM_SCHEME=bf16x3 for activations beyond fp16's range (|x| > 65504 would turn into inf / NaN hidden states,
// loudly, under f16q8).
#ifndef S3B_DEFAULT_SCHEME
#define S3B_DEFAULT_SCHEME 1
#endif
// Frames (batch x T) from which a forward call is split into two utterance lanes (default_lanes below)
#ifndef S3B_LANE_MIN_FRAMES_DEFAULT
#define S3B_LANE_MIN_FRAMES_DEFAULT 12000
#endif

static const int kNumConv = 7;
static const int kConvK[kNumConv] = {10, 3, 3, 3, 3, 2, 2};
static const int kConvS[kNumConv] = {5, 2, 2, 2, 2, 2, 2};
static const int kConvDim = 512;

struct LayerW {
    SplitBuf qkv, out, fc1, fc2;
    DevBuf qkv_b, out_b, fc1_b, fc2_b, ln1_g, ln1_b, ln2_g, ln2_b;
    DevBuf grep_w, grep_b, grep_a;  // WavLM gate
    // Conformer (finalize_conformer_layer): qkv holds [linear_q; linear_k] ([2D][D]), v linear_v, qkv_b the three
    // biases; fc1 / fc2 are ffn2.w_1 / w_2 and ffn1_* the first half-step FFN (w_2 and its bias pre-scaled by 0.5);
    // ln1 = self_attn_layer_norm, ln2 = final_layer_norm; dw_w / dw_b the depthwise taps with BatchNorm folded in
    SplitBuf v, ffn1_w1, ffn1_w2, pw1, pw2;
    DevBuf ffn1_b1, ffn1_b2, ffn1_ln_g, ffn1_ln_b, ffn2_ln_g, ffn2_ln_b, conv_ln_g, conv_ln_b, dw_w, dw_b;
    // APC GRU layer: wih = weight_ih_l0 [3H][K] (tap_weight_layout, k = 1; layer 0: K = 80 zero-padded to kDecoar2K),
    // gru_b = bias_ih_l0 with bias_hh_l0's r and z thirds added (the input GEMM's bias), whh = weight_hh_l0 [3H][H]
    // fp32, bhn = bias_hh_l0[2H:]
    // DeCoAR LSTM layer k, direction d (layers[2k + d]): wih = weight_ih_lk [4H][H], gru_b = bias_ih_lk + bias_hh_lk,
    // whh = weight_hh_lk [4H][H] fp32
    SplitBuf wih;
    DevBuf gru_b, whh, bhn;
    // NPC block i (finalize_npc), each weight in tap_weight_layout: fc1 = blocks.i.conv with bn1 folded in
    // ([512][3 * Cp], Cp = 128 for block 0's 80 channels, 512 after), fc2 = blocks.i.linear with bn2 folded in
    // ([512][512]), out = masked_convs.i's unmasked taps ([512][u * 512]); fc1_b, fc2_b, out_b their biases
};

// per-category device-time profile (CUDA events around each launch on the launching stream)
// CAT_GRU (the GRU / LSTM recurrences) is read through s3b_profile_read_ex only: s3b_profile_read fills five entries
enum { CAT_GEMM = 0, CAT_ATTN = 1, CAT_CONV0 = 2, CAT_NORM = 3, CAT_MISC = 4, CAT_GRU = 5, CAT_COUNT = 6 };
struct ProfRec {
    int cat;
    Event a, b;
};
struct Profiler {
    bool on = false;
    std::vector<Event> pool;
    std::vector<ProfRec> recs;
    Event pending;
    double ms[CAT_COUNT] = {};
    double flops[CAT_COUNT] = {};
    long long launches[CAT_COUNT] = {};
    Event get() {
        if (!pool.empty()) {
            Event e = std::move(pool.back());
            pool.pop_back();
            return e;
        }
        cudaEvent_t e = nullptr;
        cudaEventCreate(&e);
        return Event(e);
    }
};

// Cached launch plan: the forward of one lane at a given (B, Lmax) as an ordered list of steps (build_steps).
// Encoding the ~22 CUtensorMaps of a layer costs ~300 driver calls per forward; they only depend on the workspace
// addresses, the weights and (B, T), so they are built once per shape and reused (ragged training batches change
// Lmax every step and rebuild; fixed-shape serving never does).
struct Fwd;
using Step = std::function<int(Fwd&)>;
struct Plan {
    int B = 0;
    int64_t Lmax = 0;
    uint64_t gen = 0;
    // A step enqueues its kernels on the stream of the Fwd it is handed. It may capture only what the plan key fixes:
    // weights, workspace and bookkeeping-block addresses, B, T, M, L[] and the tensor maps built from them. Everything
    // else it reads per call from that Fwd: the stream, the output slots (slot(), hs(), proj_out()), ffn_out /
    // ffn_stride, last_res and layer_done / user.
    std::vector<Step> steps;
};

// Per-lane working set. A forward call runs the batch as one or two utterance micro-batches ("lanes"): lane 0 on
// the caller's stream, lane 1 on an internal stream, every kernel enqueue alternating between the two so that one
// lane's tails / small kernels fill the SMs the other leaves idle. Utterances are independent given the shared
// max_len, so the result is bit-identical to the single-lane run (tests/test_properties_gpu.py).
struct Workspace {
    // bookkeeping block (one pinned host mirror, one async H2D copy per call): wav ptrs | lens | kv_len | row mask
    DevBuf book;
    PinnedBuf book_host;
    size_t book_host_bytes = 0;
    size_t book_valid = 0;  // bytes of the mirror that hold the last call's block
    Event book_copied;      // the previous call's H2D copy has been consumed: the mirror may be rewritten
    DevBuf wav_stats, wav_pad, c0_part, c0_ss, conv_f32, tmp_f32, x_f32, x1_f32, gate, pos_z, hs0;
    DevBuf glu_f32;  // Conformer: pointwise_conv1 output [M][2D]
    DevBuf fb_f32;   // DeCoAR 2.0 / APC: log-mel frames [B][m(Lmax)][80]
    DevBuf xg_f32;   // APC / DeCoAR: the input GEMM's output [M][3H] / [M][4H]
    DevBuf lstm_h, lstm_sync;  // DeCoAR: the recurrence's state exchange buffer and grid-barrier counter
    SplitBuf act[kNumConv], ln512_s, x_s, xs_s, q_s, k_s, vt_s, ctx_s, x1_s, h_s;
    Stream stream;  // lane stream (lane 1; lane 0 runs on the caller's stream)
    Event done;
    std::vector<std::unique_ptr<Plan>> plans;  // small LRU of cached tensor maps / launch descriptors keyed by (B, Lmax)
};

// What a model runs, fixed by the create function that made it
enum ModelKind {
    kConvEncoder,   // s3b_model_create, frontend 0: conv stack into the transformer / Conformer encoder
    kFbankEncoder,  // s3b_model_create, frontend 1 (DeCoAR 2.0): fbank + CMVN, every second frame, into the encoder
    kGruStack,      // s3b_apc_model_create (APC / VQ-APC): fbank + CMVN into a GRU stack
    kLstmStack,     // s3b_decoar_model_create (DeCoAR): fbank + CMVN, post_extract_proj, bidirectional LSTM stack
    kNpcStack,      // s3b_npc_model_create (NPC): fbank + CMVN into ConvBlocks and masked convs
    kCpcStack,      // s3b_cpc_model_create (modified CPC): padded strided conv stack with ChannelNorm into an LSTM stack
    kSsastEncoder,  // s3b_ssast_model_create (SSAST): windowed 128-bin fbank, patch embedding, pre-LN DeiT encoder
};

struct s3b_model {
    s3b_config cfg;
    ModelKind kind = kConvEncoder;
    // kGruStack: cfg holds num_layers and embed_dim = hidden, everything else zero
    int apc_residual = 0;
    // kLstmStack: cfg holds num_layers and embed_dim = 2 H (the forward | backward concat)
    int decoar_all_layers = 0;  // 1: decoar_layers (every layer's output), 0: decoar (the last one)
    // kNpcStack: cfg holds num_layers = n_blocks and embed_dim = hidden
    s3b_npc_config npc = {};
    // kCpcStack: cfg holds num_layers = the LSTM levels and embed_dim = 256. Weights: conv0_w [256][10], conv0_b and
    // norm0_g / norm0_b (conv 0's ChannelNorm), conv_w[1..4] [256][2 s * 256] (tap_weight_layout), conv_b[1..4] and
    // conv_ln_g / conv_ln_b[1..4]; per LSTM layer wih [1024][256], gru_b = bias_ih + bias_hh, whh [1024][256] fp32
    // kSsastEncoder: cfg holds the pre-LN encoder (num_layers, embed_dim, ffn_dim, num_heads, layer_norm_first = 1).
    // Weights: proj_w / proj_b the patch embedding ([768][256], tap_weight_layout for the frame model), cls_tok,
    // dist_tok [768], pos_tab [2 + P][768]; the blocks in layers (ln1 = norm1, ln2 = norm2, out = attn.proj)
    s3b_ssast_config ssast = {};
    DevBuf cls_tok, dist_tok, pos_tab;
    float ln_eps = 1e-5f;  // eps of the encoder layers' LayerNorms
    std::map<std::string, HostTensor> host;
    bool finalized = false;
    int sm_count = 132;
    int scheme = 0;  // tensor-core operand scheme of the conv / linear GEMMs: 0 = bf16x3, 1 = f16q8 (gemm.cuh)
    Profiler prof;
    long long launches_total = 0;  // kernels launched by this model since creation
    Stream copy_stream, compute_stream;
    Event fork_event;
    std::vector<Event> layer_events;

    // weights
    DevBuf conv0_w, conv0_b, norm0_g, norm0_b;           // conv 0 (+ GroupNorm or LN affine)
    SplitBuf conv_w[kNumConv];                             // 1..6, [512][kw*512] (tap-major K)
    DevBuf conv_b[kNumConv], conv_ln_g[kNumConv], conv_ln_b[kNumConv];
    DevBuf ln512_g, ln512_b, proj_b, pos_b, enc_ln_g, enc_ln_b;
    SplitBuf proj_w, pos_w, pos_w4;  // pos_w4: four-taps-per-k-block layout (posconv4_params)
    std::vector<SplitBuf> posd_w4;      // data2vec (pos_conv_depth > 1): one four-taps layout per conv block
    std::vector<DevBuf> posd_b;         //                                 and its bias
    SplitBuf pred1_w;                   // Distiller output_layer.0.weight [N*D][D]
    std::vector<SplitBuf> pred2_w;      // Distiller output_layer.2.weight, per task, transposed to [D out][D in]
    DevBuf pred1_b, pred2_b;            // biases [N*D]
    DevBuf rel_table_src;  // WavLM relative_attention_bias.weight [num_buckets][H]
    DevBuf rel_table;      // [H][2*rel_table_T - 1] gathered table (x log2 e), built at finalize for rel_table_T frames
    int rel_table_T = 0;
    // Conformer rotary embedding: rope_cs [rope_T][64] = cos | sin of fp32(t) * inv_freq[j], j < 32 (build_rope_table)
    DevBuf rope_cs;
    int rope_T = 0;
    std::vector<float> rope_inv_freq;
    std::vector<LayerW> layers;

    Workspace ws[2];
    DevBuf stage_wav, stage_out;  // s3b_forward_host staging
};

// ------------------------------------------------------------------------------------------------
// host helpers
// ------------------------------------------------------------------------------------------------
static int upload_f32(DevBuf& dst, const float* src, size_t n) {
    S3B_OK(dst.ensure(n * 4));
    CUDA_OK(cudaMemcpy(dst.p, src, n * 4, cudaMemcpyHostToDevice));
    return 0;
}
static int upload_split(SplitBuf& dst, const float* src, size_t n, int fmt = 0) {
    DevBuf tmp;
    S3B_OK(upload_f32(tmp, src, n));
    S3B_OK(dst.ensure(n));
    if (fmt != 0) CUDA_OK(launch_split_q8(tmp.as<float>(), dst.h(), dst.h8(), dst.l8(), n, 1, 0));
    else CUDA_OK(launch_split(tmp.as<float>(), dst.h(), dst.l(), n, 0));
    CUDA_OK(cudaDeviceSynchronize());
    return 0;
}
static const HostTensor* find(const s3b_model* m, const std::string& k) {
    auto it = m->host.find(k);
    return it == m->host.end() ? nullptr : &it->second;
}
static int need(const s3b_model* m, const std::string& k, std::initializer_list<int64_t> shape, const HostTensor** out) {
    const HostTensor* t = find(m, k);
    if (!t) return fail("missing tensor '%s'", k.c_str());
    std::vector<int64_t> want(shape);
    if (t->shape != want) {
        std::string got, exp;
        for (auto d : t->shape) got += std::to_string(d) + ",";
        for (auto d : want) exp += std::to_string(d) + ",";
        return fail("tensor '%s' has shape [%s], expected [%s]", k.c_str(), got.c_str(), exp.c_str());
    }
    *out = t;
    return 0;
}
static int upload_vec(s3b_model* m, const std::string& k, int64_t n, DevBuf& dst) {
    const HostTensor* t;
    S3B_OK(need(m, k, {n}, &t));
    return upload_f32(dst, t->data.data(), (size_t)n);
}

static bool posconv4_ok(const s3b_config& c);
static int pos_taps(const s3b_config& c);
static int pos_taps4(const s3b_config& c);

static int64_t conv_out_len(int64_t L, int i) { return L < kConvK[i] ? 0 : (L - kConvK[i]) / kConvS[i] + 1; }

static int64_t num_frames(int64_t L) {
    for (int i = 0; i < kNumConv; ++i) L = conv_out_len(L, i);
    return L;
}

// DeCoAR 2.0 (frontend 1): kaldi fbank frames m = 1 + (L - 400) / 160 (snip_edges), y[::2] keeps (m + 1) / 2 of them
static const int64_t kDecoar2MinLen = 560;  // two fbank frames: the unbiased std of one frame is NaN
static int64_t decoar2_frames(int64_t L) { return L < 400 ? 0 : (1 + (L - 400) / 160 + 1) / 2; }
static int64_t fbank_frames(int64_t L) { return L < 400 ? 0 : 1 + (L - 400) / 160; }
// modified CPC's encoder (cpc/model.py CPCEncoder): five Conv1d with k = 2 s, strides 5, 4, 2, 2, 2 and paddings
// 3, 2, 1, 1, 1, 256 channels each
static const int kCpcConvs = 5;
static const int kCpcStride[kCpcConvs] = {5, 4, 2, 2, 2};
static const int kCpcPad[kCpcConvs] = {3, 2, 1, 1, 1};
static const int kCpcDim = 256;
static int64_t cpc_conv_len(int64_t L, int i) {
    const int s = kCpcStride[i], k = 2 * s;
    return L + 2 * kCpcPad[i] < k ? 0 : (L + 2 * kCpcPad[i] - k) / s + 1;
}
static int64_t cpc_frames(int64_t L) {
    for (int i = 0; i < kCpcConvs; ++i) L = cpc_conv_len(L, i);
    return L;
}
// rows per utterance of conv i's (i >= 1) padded operand, whose view rows t, t + 1 feed output frame t (conv_params):
// pad zero rows, the Lout(i - 1) input frames (those that fit), zero rows up to s (Lout + 1)
static int64_t cpc_rows(int64_t Lout, int i) { return kCpcStride[i] * (Lout + 1); }

// SSAST (ssast/expert.py, ast_models.py): S samples per window, TL = S / 160 feature rows, P = patch_f * tdim patches
// per window (frame model: patch_f 1, tdim TL - 1; patch model: patch_f 12 frequency patches, tdim time patches) and
// `rate` samples per output frame
struct SsastGeom {
    int S, TL, patch_f, tdim, P, rate;
};
static SsastGeom ssast_geom(const s3b_ssast_config& c) {
    SsastGeom g;
    g.S = c.window_samples, g.TL = g.S / 160;
    g.patch_f = c.patch ? 12 : 1;
    g.tdim = c.patch ? (g.TL - 16) / 10 + 1 : g.TL - 1;
    g.P = g.patch_f * g.tdim;
    g.rate = c.patch ? 1600 : 160;
    return g;
}
static int64_t ssast_segments(const SsastGeom& g, int64_t L) { return (L + g.S - 1) / g.S; }
// len(range(0, L, rate)) frames, at most the nseg * tdim the windows make
static int64_t ssast_frames(const SsastGeom& g, int64_t L) {
    return L < 1 ? 0 : std::min(ssast_segments(g, L) * g.tdim, (L + g.rate - 1) / g.rate);
}

// frames of a batch padded to L for this model's front end (m NULL: the conv stack); on the fbank kinds and modified
// CPC also the valid frames of one utterance of L samples
static int64_t model_frames(const s3b_model* m, int64_t L) {
    if (m != nullptr && m->kind == kCpcStack) return cpc_frames(L);
    if (m != nullptr && m->kind == kSsastEncoder) return ssast_frames(ssast_geom(m->ssast), L);
    if (m == nullptr || m->kind == kConvEncoder) return num_frames(L);
    return m->kind == kFbankEncoder ? decoar2_frames(L) : fbank_frames(L);  // the recurrent stacks keep every frame
}
static int fail_too_short(const s3b_model* m, int64_t max_len) {
    return fail("max_len %lld too short: the %s yields no frame", (long long)max_len,
                m->kind == kConvEncoder || m->kind == kCpcStack ? "conv stack" : "fbank");
}

// ------------------------------------------------------------------------------------------------
// C ABI: library
// ------------------------------------------------------------------------------------------------
extern "C" int s3b_version(void) { return 200; }
extern "C" const char* s3b_last_error(void) { return g_last_error.c_str(); }
extern "C" int s3b_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

// Operand scheme of the GEMMs: "f16q8" = fp16 product + two e4m3 correction products (2 MMA slots
// per 16 of K), "bf16x3" = bf16 hi/lo, 3 MMAs. S3B_GEMM_SCHEME overrides the default.
static int default_scheme() {
    const char* e = getenv("S3B_GEMM_SCHEME");
    if (e != nullptr) return (strcmp(e, "f16q8") == 0 || strcmp(e, "1") == 0) ? 1 : 0;
    return S3B_DEFAULT_SCHEME;
}

// attention head widths the kernel is built for (attention.cu), and pos_conv group widths: multiples of 16 up to 64
// (one 64-wide k-block per tap, or four taps per k-block), 80 and 120 (two k-blocks per tap, one tap per k-block),
// 24 and 40 (four taps per k-block only: posconv4_only)
static bool head_dim_ok(int hd) { return hd == 64 || hd == 80 || hd == 120; }
static bool posconv4_only(int cpg) { return cpg == 24 || cpg == 40; }
static bool posconv_cpg_ok(int cpg) {
    return (cpg % 16 == 0 && cpg >= 16 && cpg <= 64) || cpg == 80 || cpg == 120 || posconv4_only(cpg);
}
static int head_dim(const s3b_config& c) { return c.embed_dim / c.num_heads; }

// ------------------------------------------------------------------------------------------------
// C ABI: model lifetime
// ------------------------------------------------------------------------------------------------
extern "C" int s3b_model_create(const s3b_config* cfg, s3b_model** out) {
    if (!cfg || !out) return fail("null argument");
    if (cfg->embed_dim % 128 != 0 || cfg->embed_dim > 1920) return fail("embed_dim must be a multiple of 128, <= 1920");
    if (cfg->num_heads < 1 || cfg->embed_dim % cfg->num_heads != 0 || !head_dim_ok(cfg->embed_dim / cfg->num_heads))
        return fail("head dim (embed_dim / num_heads = %d / %d) must be 64, 80 or 120", cfg->embed_dim, cfg->num_heads);
    const int hd = cfg->embed_dim / cfg->num_heads;
    if (cfg->ffn_dim % 256 != 0) return fail("ffn_dim must be a multiple of 256");
    if (cfg->pos_conv_groups < 1 || cfg->embed_dim % cfg->pos_conv_groups != 0)
        return fail("embed_dim %% pos_conv_groups != 0");
    const int cpg = cfg->embed_dim / cfg->pos_conv_groups;
    if (!posconv_cpg_ok(cpg))
        return fail("channels per pos_conv group (embed_dim / pos_conv_groups = %d) must be 16, 32, 48, 64, 80 or 120 "
                    "(or 24 or 40 with four taps per k-block)", cpg);
    if (cfg->pos_conv_depth < 0 || cfg->pos_conv_depth > 8) return fail("pos_conv_depth out of range (0..8)");
    if (posconv4_only(cpg) && (cfg->pos_conv_depth > 1 || cfg->pos_conv_kernel % 4 != 0))
        return fail("%d channels per pos_conv group need pos_conv_depth <= 1 and a pos_conv_kernel that is a multiple of 4 "
                    "(four taps per k-block), not depth %d, kernel %d", cpg, cfg->pos_conv_depth, cfg->pos_conv_kernel);
    if (cfg->pos_conv_depth <= 1 && cfg->pos_conv_kernel % 2 != 0) return fail("pos_conv_kernel must be even");
    if (cfg->pos_conv_depth > 1 && (cfg->pos_conv_kernel < 3 || (4 * cpg != 192 && 4 * cpg != 256)))
        return fail("pos_conv_depth > 1 needs 48 or 64 channels per group");
    if (cfg->pos_conv_depth > 1 && cfg->family != 1)
        return fail("pos_conv_depth > 1 (data2vec) goes with the wav2vec2 family (1)");
    if (cfg->num_layers < 1 || cfg->num_layers > 63) return fail("num_layers out of range");
    if (cfg->family < 0 || cfg->family > 3) return fail("family must be 0 (hubert), 1 (wav2vec2), 2 (wavlm) or 3 (distiller)");
    if (cfg->pred_heads < 0 || cfg->pred_heads > 12 || cfg->pred_heads * cfg->embed_dim > cfg->ffn_dim)
        return fail("pred_heads out of range (needs pred_heads * embed_dim <= ffn_dim)");
    if (cfg->no_feature_layer_norm && cfg->extractor_layer_norm)
        return fail("no_feature_layer_norm with extractor_mode layer_norm is not supported");
    if ((cfg->family == 3) != (cfg->no_feature_layer_norm != 0))
        return fail("the distiller family (3) and no_feature_layer_norm go together");
    if (cfg->conformer != 0 && cfg->conformer != 1) return fail("conformer must be 0 or 1");
    // the rotary table, the WavLM gate (grep_linear [8][64]) and the relative bias are 64-wide per head
    if (cfg->conformer && hd != 64)
        return fail("conformer = 1 needs 64-wide heads: head dim (embed_dim / num_heads) is %d", hd);
    if (cfg->family == 2 && hd != 64)
        return fail("family 2 (wavlm) needs 64-wide heads: head dim (embed_dim / num_heads) is %d", hd);
    if (cfg->conformer) {
        if (cfg->family != 1) return fail("the Conformer encoder goes with the wav2vec2 family (1)");
        if (cfg->relative_position || cfg->pred_heads) return fail("the Conformer encoder has no WavLM bias or prediction heads");
        if (cfg->depthwise_kernel < 1 || cfg->depthwise_kernel > kDwMaxKernel || cfg->depthwise_kernel % 2 == 0)
            return fail("depthwise_kernel %d: must be odd, 1..%d", cfg->depthwise_kernel, kDwMaxKernel);
    } else if (cfg->depthwise_kernel != 0) {
        return fail("depthwise_kernel is a Conformer field (conformer = 0)");
    }
    if (cfg->proj_hidden0 != 0 && cfg->proj_hidden0 != 1) return fail("proj_hidden0 must be 0 or 1");
    if (cfg->proj_hidden0 && (cfg->family != 0 || cfg->conformer || cfg->layer_norm_first || cfg->frontend != 0))
        return fail("proj_hidden0 = 1 (LightHuBERT) goes with the hubert family (0), a post-LN transformer encoder and the "
                    "conv stack");
    if (cfg->frontend != 0 && cfg->frontend != 1) return fail("frontend must be 0 (conv stack) or 1 (DeCoAR 2.0 fbank)");
    if (cfg->frontend == 1) {
        // DeCoAR 2.0 = fbank features into the wav2vec 2.0 TransformerEncoder (decoar2/decoar2.py:27-59)
        if (cfg->family != 1) return fail("frontend 1 (DeCoAR 2.0) goes with the wav2vec2 family (1), not %d", cfg->family);
        if (cfg->conformer) return fail("frontend 1 (DeCoAR 2.0) runs a transformer encoder, not a Conformer");
        if (cfg->pos_conv_depth > 1) return fail("frontend 1 (DeCoAR 2.0) needs pos_conv_depth <= 1");
        if (cfg->extractor_layer_norm || cfg->conv_bias || cfg->normalize_wav || cfg->no_feature_layer_norm)
            return fail("frontend 1 (DeCoAR 2.0) has no conv stack: extractor_layer_norm, conv_bias, normalize_wav and "
                        "no_feature_layer_norm must be 0");
    }
    s3b_model* m = new s3b_model();
    m->cfg = *cfg;
    m->kind = cfg->frontend == 1 ? kFbankEncoder : kConvEncoder;
    m->scheme = default_scheme();
    *out = m;
    return 0;
}

extern "C" int s3b_apc_model_create(const s3b_apc_config* cfg, s3b_model** out) {
    if (!cfg || !out) return fail("null argument");
    if (cfg->struct_size != (int32_t)sizeof(s3b_apc_config))
        return fail("s3b_apc_config.struct_size %d != %d (header / library mismatch)", cfg->struct_size,
                    (int)sizeof(s3b_apc_config));
    if (cfg->num_layers != 3) return fail("num_layers %d: the APC model is served with 3 GRU layers", cfg->num_layers);
    if (cfg->hidden != kGruHidden) return fail("hidden %d: the APC model is served with hidden size %d", cfg->hidden, kGruHidden);
    if (cfg->residual != 0 && cfg->residual != 1) return fail("residual must be 0 or 1, not %d", cfg->residual);
    for (int i = 0; i < 4; ++i)
        if (cfg->reserved[i] != 0) return fail("s3b_apc_config.reserved[%d] must be 0", i);
    s3b_model* m = new s3b_model();
    memset(&m->cfg, 0, sizeof(m->cfg));
    m->cfg.num_layers = cfg->num_layers, m->cfg.embed_dim = cfg->hidden;
    m->kind = kGruStack, m->apc_residual = cfg->residual;
    m->scheme = default_scheme();
    *out = m;
    return 0;
}

extern "C" int s3b_decoar_model_create(const s3b_decoar_config* cfg, s3b_model** out) {
    if (!cfg || !out) return fail("null argument");
    if (cfg->struct_size != (int32_t)sizeof(s3b_decoar_config))
        return fail("s3b_decoar_config.struct_size %d != %d (header / library mismatch)", cfg->struct_size,
                    (int)sizeof(s3b_decoar_config));
    if (cfg->num_layers != 4) return fail("num_layers %d: DeCoAR is served with 4 LSTM layers", cfg->num_layers);
    if (cfg->hidden != kLstmHidden)
        return fail("hidden %d: DeCoAR is served with hidden size %d", cfg->hidden, kLstmHidden);
    if (cfg->all_layers != 0 && cfg->all_layers != 1) return fail("all_layers must be 0 or 1, not %d", cfg->all_layers);
    for (int i = 0; i < 4; ++i)
        if (cfg->reserved[i] != 0) return fail("s3b_decoar_config.reserved[%d] must be 0", i);
    s3b_model* m = new s3b_model();
    memset(&m->cfg, 0, sizeof(m->cfg));
    m->cfg.num_layers = cfg->num_layers, m->cfg.embed_dim = 2 * cfg->hidden;
    m->kind = kLstmStack, m->decoar_all_layers = cfg->all_layers;
    m->scheme = default_scheme();
    *out = m;
    return 0;
}

// NPC's masked conv i zeroes a centred band of mask_size + 2 (i + 1) of its kernel_size taps (npc.py MaskConvBlock)
static int npc_mask_width(const s3b_npc_config& c, int i) { return c.mask_size + 2 * (i + 1); }

extern "C" int s3b_npc_model_create(const s3b_npc_config* cfg, s3b_model** out) {
    if (!cfg || !out) return fail("null argument");
    if (cfg->struct_size != (int32_t)sizeof(s3b_npc_config))
        return fail("s3b_npc_config.struct_size %d != %d (header / library mismatch)", cfg->struct_size,
                    (int)sizeof(s3b_npc_config));
    if (cfg->n_blocks < 1 || cfg->n_blocks > 32) return fail("n_blocks %d: must be 1..32", cfg->n_blocks);
    if (cfg->hidden != 512) return fail("hidden %d: NPC is served with hidden size 512", cfg->hidden);
    if (cfg->kernel_size < 1 || cfg->kernel_size > 127 || cfg->kernel_size % 2 == 0)
        return fail("kernel_size %d: must be odd, 1..127", cfg->kernel_size);
    if (cfg->mask_size < 1 || cfg->mask_size % 2 == 0) return fail("mask_size %d: must be odd and >= 1", cfg->mask_size);
    if (cfg->kernel_size <= cfg->mask_size + 2 * cfg->n_blocks)
        return fail("kernel_size %d must exceed mask_size + 2 n_blocks = %d (the widest mask leaves no tap)",
                    cfg->kernel_size, cfg->mask_size + 2 * cfg->n_blocks);
    if (cfg->residual != 0 && cfg->residual != 1) return fail("residual must be 0 or 1, not %d", cfg->residual);
    if (cfg->batch_norm != 0 && cfg->batch_norm != 1) return fail("batch_norm must be 0 or 1, not %d", cfg->batch_norm);
    if (cfg->act != 0 && cfg->act != 1) return fail("act must be 0 (relu) or 1 (tanh), not %d", cfg->act);
    for (int i = 0; i < 4; ++i)
        if (cfg->reserved[i] != 0) return fail("s3b_npc_config.reserved[%d] must be 0", i);
    s3b_model* m = new s3b_model();
    memset(&m->cfg, 0, sizeof(m->cfg));
    m->cfg.num_layers = cfg->n_blocks, m->cfg.embed_dim = cfg->hidden;
    m->kind = kNpcStack, m->npc = *cfg;
    m->scheme = default_scheme();
    *out = m;
    return 0;
}

extern "C" int s3b_cpc_model_create(const s3b_cpc_config* cfg, s3b_model** out) {
    if (!cfg || !out) return fail("null argument");
    if (cfg->struct_size != (int32_t)sizeof(s3b_cpc_config))
        return fail("s3b_cpc_config.struct_size %d != %d (header / library mismatch)", cfg->struct_size,
                    (int)sizeof(s3b_cpc_config));
    if (cfg->hidden != kCpcDim) return fail("hidden %d: modified CPC is served with hidden size %d", cfg->hidden, kCpcDim);
    if (cfg->num_layers < 1 || cfg->num_layers > 8) return fail("num_layers %d: must be 1..8", cfg->num_layers);
    for (int i = 0; i < 4; ++i)
        if (cfg->reserved[i] != 0) return fail("s3b_cpc_config.reserved[%d] must be 0", i);
    s3b_model* m = new s3b_model();
    memset(&m->cfg, 0, sizeof(m->cfg));
    m->cfg.num_layers = cfg->num_layers, m->cfg.embed_dim = cfg->hidden;
    m->kind = kCpcStack;
    m->scheme = default_scheme();
    *out = m;
    return 0;
}

extern "C" int s3b_ssast_model_create(const s3b_ssast_config* cfg, s3b_model** out) {
    if (!cfg || !out) return fail("null argument");
    if (cfg->struct_size != (int32_t)sizeof(s3b_ssast_config))
        return fail("s3b_ssast_config.struct_size %d != %d (header / library mismatch)", cfg->struct_size,
                    (int)sizeof(s3b_ssast_config));
    if (cfg->patch != 0 && cfg->patch != 1) return fail("patch must be 0 (frame model) or 1 (patch model), not %d", cfg->patch);
    if (cfg->embed_dim != 768 || cfg->num_heads != 12 || cfg->num_layers != 12)
        return fail("only SSAST base is served: embed_dim 768, num_heads 12, num_layers 12 (got %d, %d, %d)",
                    cfg->embed_dim, cfg->num_heads, cfg->num_layers);
    const int min_s = cfg->patch ? 2560 : 400;
    if (cfg->window_samples < min_s || cfg->window_samples > 160000)
        return fail("window_samples %d out of range: the %s model needs %d..160000 (one patch of %d frames .. 10 s)",
                    cfg->window_samples, cfg->patch ? "patch" : "frame", min_s, cfg->patch ? 16 : 2);
    for (int i = 0; i < 4; ++i)
        if (cfg->reserved[i] != 0) return fail("s3b_ssast_config.reserved[%d] must be 0", i);
    s3b_model* m = new s3b_model();
    m->kind = kSsastEncoder, m->ssast = *cfg;
    m->cfg.num_layers = cfg->num_layers, m->cfg.embed_dim = cfg->embed_dim, m->cfg.num_heads = cfg->num_heads;
    m->cfg.ffn_dim = 4 * cfg->embed_dim, m->cfg.layer_norm_first = 1;
    m->ln_eps = 1e-6f;
    m->scheme = default_scheme();
    *out = m;
    return 0;
}

extern "C" int s3b_model_set_tensor(s3b_model* m, const char* name, const float* data, const int64_t* shape,
                                    int32_t ndim) {
    if (!m || !name || !data || (!shape && ndim > 0)) return fail("null argument");
    if (m->finalized) return fail("model already finalized");
    HostTensor t;
    size_t n = 1;
    for (int i = 0; i < ndim; ++i) t.shape.push_back(shape[i]), n *= (size_t)shape[i];
    t.data.assign(data, data + n);
    m->host[name] = std::move(t);
    return 0;
}

extern "C" void s3b_model_destroy(s3b_model* m) { delete m; }

// WavLM: table[h][r] = log2(e) * emb[bucket(r - (Tmax - 1))][h], r in [0, 2 Tmax - 1). Built once for Tmax frames
// (the ungated bias is shared by all layers and all calls, WavLM.py:622-632); the attention kernel indexes it with
// the centre Tmax - 1, so a forward never allocates or synchronises for it (it used to rebuild per distinct T).
static int build_rel_table(s3b_model* m, int Tmax) {
    const s3b_config& c = m->cfg;
    S3B_OK(m->rel_table.ensure((size_t)c.num_heads * (2 * (size_t)Tmax - 1) * 4));
    CUDA_OK(launch_wavlm_rel_table(m->rel_table_src.as<float>(), c.num_buckets, c.max_distance, c.num_heads, Tmax,
                                   m->rel_table.as<float>(), 0));
    CUDA_OK(cudaDeviceSynchronize());
    m->rel_table_T = Tmax;
    return 0;
}

// The attention kernel's view of a table built for Tmax frames: row h starts at h * (2 Tmax - 1), and k - q = 0 sits
// at column Tmax - 1. The model's plans and s3b_attention_ex both go through here.
static void set_rel_bias(AttnParams& ap, const float* table, int Tmax, const float* gate) {
    ap.bias_table = table;
    ap.bias_stride = 2 * Tmax - 1, ap.bias_center = Tmax - 1;
    ap.gate = gate;
}

// Conformer rotary table for frames [0, Tmax): the reference's angle fp32(t) * inv_freq[j] is an fp32 product
// (RotaryPositionalEmbedding.forward, wav2vec2_model.py:66-70); its cos / sin are taken in double and rounded to fp32.
// inv_freq: the checkpoint's buffer, else 1 / 10000^(2j / 64) rounded to fp32.
static std::vector<float> rope_table(const std::vector<float>& inv_freq, int Tmax) {
    std::vector<float> cs((size_t)Tmax * 64);
    for (int t = 0; t < Tmax; ++t)
        for (int j = 0; j < 32; ++j) {
            const float a = (float)t * inv_freq[j];
            cs[(size_t)t * 64 + j] = (float)cos((double)a);
            cs[(size_t)t * 64 + 32 + j] = (float)sin((double)a);
        }
    return cs;
}
static std::vector<float> default_inv_freq() {
    std::vector<float> f(32);
    for (int j = 0; j < 32; ++j) f[j] = (float)(1.0 / pow(10000.0, (2.0 * j) / 64.0));
    return f;
}
// grown (synchronously) like rel_table when a batch has more frames; a forward reads m->rope_cs at launch time
static int build_rope_table(s3b_model* m, int Tmax) {
    const std::vector<float> cs = rope_table(m->rope_inv_freq, Tmax);
    CUDA_OK(cudaDeviceSynchronize());  // the previous table may still be read by enqueued work
    S3B_OK(upload_f32(m->rope_cs, cs.data(), cs.size()));
    m->rope_T = Tmax;
    return 0;
}

// BatchNorm1d (eval, eps 1e-5) folded into the depthwise conv (wav2vec2_model.py:387-388), in double:
// w' = w * s, b' = beta - mean * s, s = gamma / sqrt(var + eps). w: [D][k].
static void fold_depthwise_bn(const float* w, const float* gamma, const float* beta, const float* mean,
                              const float* var, int D, int k, std::vector<float>& wf, std::vector<float>& bf) {
    wf.resize((size_t)D * k), bf.resize(D);
    for (int c = 0; c < D; ++c) {
        const double s = (double)gamma[c] / sqrt((double)var[c] + 1e-5);
        for (int j = 0; j < k; ++j) wf[(size_t)c * k + j] = (float)((double)w[(size_t)c * k + j] * s);
        bf[c] = (float)((double)beta[c] - (double)mean[c] * s);
    }
}

// One ConformerEncoderLayer (wav2vec2_model.py:441-578) of a layer_type "conformer", pos_enc_type "rope" checkpoint.
static int finalize_conformer_layer(s3b_model* m, int l) {
    const s3b_config& c = m->cfg;
    const int D = c.embed_dim, F = c.ffn_dim, k = c.depthwise_kernel;
    LayerW& L = m->layers[l];
    const std::string p = "encoder.layers." + std::to_string(l) + ".";
    const HostTensor* t;
    // x = x + 0.5 * ffn(x): the 0.5 goes into w_2 and its bias (a power of two: exact in fp32 and in both operand
    // schemes), so that w_2 runs the plain bias + residual epilogue
    auto ffn = [&](const std::string& f, SplitBuf& w1, DevBuf& b1, SplitBuf& w2, DevBuf& b2, DevBuf& lg, DevBuf& lb) {
        S3B_OK(upload_vec(m, f + "layer_norm.weight", D, lg));
        S3B_OK(upload_vec(m, f + "layer_norm.bias", D, lb));
        S3B_OK(need(m, f + "w_1.weight", {F, D}, &t));
        S3B_OK(upload_split(w1, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, f + "w_1.bias", F, b1));
        S3B_OK(need(m, f + "w_2.weight", {D, F}, &t));
        std::vector<float> h(t->data);
        for (float& v : h) v *= 0.5f;
        S3B_OK(upload_split(w2, h.data(), h.size(), m->scheme));
        S3B_OK(need(m, f + "w_2.bias", {D}, &t));
        h = t->data;
        for (float& v : h) v *= 0.5f;
        return upload_f32(b2, h.data(), h.size());
    };
    S3B_OK(ffn(p + "ffn1.", L.ffn1_w1, L.ffn1_b1, L.ffn1_w2, L.ffn1_b2, L.ffn1_ln_g, L.ffn1_ln_b));
    S3B_OK(ffn(p + "ffn2.", L.fc1, L.fc1_b, L.fc2, L.fc2_b, L.ffn2_ln_g, L.ffn2_ln_b));
    // attention: [q | k] from rope(LN(x)) in one GEMM, v from LN(x) in another; biases [bq | bk | bv]
    const std::string a = p + "self_attn.";
    const HostTensor *wq, *wk, *wv, *bq, *bk, *bv;
    S3B_OK(need(m, a + "linear_q.weight", {D, D}, &wq));
    S3B_OK(need(m, a + "linear_k.weight", {D, D}, &wk));
    S3B_OK(need(m, a + "linear_v.weight", {D, D}, &wv));
    S3B_OK(need(m, a + "linear_q.bias", {D}, &bq));
    S3B_OK(need(m, a + "linear_k.bias", {D}, &bk));
    S3B_OK(need(m, a + "linear_v.bias", {D}, &bv));
    std::vector<float> w((size_t)2 * D * D), b((size_t)3 * D);
    memcpy(w.data(), wq->data.data(), (size_t)D * D * 4);
    memcpy(w.data() + (size_t)D * D, wk->data.data(), (size_t)D * D * 4);
    memcpy(b.data(), bq->data.data(), D * 4), memcpy(b.data() + D, bk->data.data(), D * 4);
    memcpy(b.data() + 2 * D, bv->data.data(), D * 4);
    S3B_OK(upload_split(L.qkv, w.data(), w.size(), m->scheme));
    S3B_OK(upload_split(L.v, wv->data.data(), wv->numel(), m->scheme));
    S3B_OK(upload_f32(L.qkv_b, b.data(), b.size()));
    S3B_OK(need(m, a + "linear_out.weight", {D, D}, &t));
    S3B_OK(upload_split(L.out, t->data.data(), t->numel(), m->scheme));
    S3B_OK(upload_vec(m, a + "linear_out.bias", D, L.out_b));
    if ((t = find(m, a + "rotary_emb.inv_freq")) != nullptr) {
        if (t->numel() != 32) return fail("'%srotary_emb.inv_freq' has %zu entries, expected 32", a.c_str(), t->numel());
        if (l == 0) m->rope_inv_freq = t->data;
        else if (t->data != m->rope_inv_freq) return fail("layer %d's rotary inv_freq differs from layer 0's", l);
    }
    S3B_OK(upload_vec(m, p + "self_attn_layer_norm.weight", D, L.ln1_g));
    S3B_OK(upload_vec(m, p + "self_attn_layer_norm.bias", D, L.ln1_b));
    S3B_OK(upload_vec(m, p + "final_layer_norm.weight", D, L.ln2_g));
    S3B_OK(upload_vec(m, p + "final_layer_norm.bias", D, L.ln2_b));
    // convolution module
    const std::string cm = p + "conv_module.";
    S3B_OK(upload_vec(m, cm + "layer_norm.weight", D, L.conv_ln_g));
    S3B_OK(upload_vec(m, cm + "layer_norm.bias", D, L.conv_ln_b));
    S3B_OK(need(m, cm + "pointwise_conv1.weight", {2 * D, D, 1}, &t));
    S3B_OK(upload_split(L.pw1, t->data.data(), t->numel(), m->scheme));
    S3B_OK(need(m, cm + "pointwise_conv2.weight", {D, D, 1}, &t));
    S3B_OK(upload_split(L.pw2, t->data.data(), t->numel(), m->scheme));
    const HostTensor *dw, *g, *be, *mu, *var;
    S3B_OK(need(m, cm + "depthwise_conv.weight", {D, 1, k}, &dw));
    S3B_OK(need(m, cm + "batch_norm.weight", {D}, &g));
    S3B_OK(need(m, cm + "batch_norm.bias", {D}, &be));
    S3B_OK(need(m, cm + "batch_norm.running_mean", {D}, &mu));
    S3B_OK(need(m, cm + "batch_norm.running_var", {D}, &var));
    std::vector<float> wf, bf;
    fold_depthwise_bn(dw->data.data(), g->data.data(), be->data.data(), mu->data.data(), var->data.data(), D, k, wf, bf);
    S3B_OK(upload_f32(L.dw_w, wf.data(), wf.size()));
    return upload_f32(L.dw_b, bf.data(), bf.size());
}

// ---- weight relayouts shared by s3b_model_finalize and the building-block entry points ----------------------------
// Every GEMM reads its weight as one [N][K] K-major matrix. A convolution weight w [N][cin][k] becomes
// [N][(k - mask) * Cp]: the taps outside the centred band of `mask` taps, in tap order, each zero-padded from cin to
// Cp channels, so that the K index tap * Cp + channel is the channels-last im2col row the convolution builders walk.
// k = 1 pads a linear's [N][cin] to [N][Cp]. T = double (NPC's BatchNorm folding) rounds each element to fp32 once.
template <class T>
static std::vector<float> tap_weight_layout(const T* w, int N, int cin, int k, int mask, int Cp) {
    const int u = k - mask, head = u / 2;
    std::vector<float> r((size_t)N * u * Cp, 0.f);
    for (int o = 0; o < N; ++o)
        for (int q = 0; q < u; ++q) {
            const int tap = q < head ? q : q + mask;
            for (int c = 0; c < cin; ++c) r[((size_t)o * u + q) * Cp + c] = (float)w[((size_t)o * cin + c) * k + tap];
        }
    return r;
}
// grouped positional conv, one tap per k-block (posconv_params): tap_weight_layout with each group's cpg channels
// zero-padded to Cp = posconv_kc(cpg), whole 64-wide k-blocks
static int posconv_kc(int cpg) { return (cpg + 63) / 64 * 64; }
// grouped positional conv, four taps per k-block (tap = 4q + j, posconv4_params), folded weight w [D][cpg][Kp], the
// tap count rounded up to K4 = a multiple of four with zero taps: [G * 4cpg][K4 / 4 * 64], row g * 4cpg + j * cpg + n,
// column q * 64 + channel (zero padded to 64); cpg <= 64 (24, 40, 48 or 64 where it runs)
static std::vector<float> posconv4_weight_layout(const float* w, int D, int G, int Kp) {
    const int cpg = D / G, Kq = (Kp + 3) / 4;
    std::vector<float> w4((size_t)D * 4 * Kq * 64, 0.0f);
    for (int g = 0; g < G; ++g)
        for (int k = 0; k < Kp; ++k)
            for (int n = 0; n < cpg; ++n)
                for (int ci = 0; ci < cpg; ++ci)
                    w4[((size_t)(g * 4 + k % 4) * cpg + n) * Kq * 64 + (k / 4) * 64 + ci] =
                        w[((size_t)(g * cpg + n) * cpg + ci) * Kp + k];
    return w4;
}

// APC (apc.py:36-48): rnn_layers.{l} = nn.GRU(in, H) with in = 80 for layer 0 and H after it. The recurrence kernel
// must be able to run at all: clusters of 16 CTAs with 209 KB of shared memory each.
static int finalize_apc(s3b_model* m) {
    const int NL = m->cfg.num_layers, H = m->cfg.embed_dim;
    m->layers.resize(NL);
    for (int l = 0; l < NL; ++l) {
        LayerW& L = m->layers[l];
        const std::string p = "rnn_layers." + std::to_string(l) + ".";
        const int in = l == 0 ? 80 : H, K = l == 0 ? kDecoar2K : H;
        const HostTensor *wih, *whh, *bih, *bhh;
        S3B_OK(need(m, p + "weight_ih_l0", {3 * H, in}, &wih));
        S3B_OK(need(m, p + "weight_hh_l0", {3 * H, H}, &whh));
        S3B_OK(need(m, p + "bias_ih_l0", {3 * H}, &bih));
        S3B_OK(need(m, p + "bias_hh_l0", {3 * H}, &bhh));
        const std::vector<float> w = tap_weight_layout(wih->data.data(), 3 * H, in, 1, 0, K);
        S3B_OK(upload_split(L.wih, w.data(), w.size(), m->scheme));
        // b_hr, b_hz sit outside r * (.) and fold into the GEMM's bias; b_hn does not
        std::vector<float> b(bih->data);
        for (int i = 0; i < 2 * H; ++i) b[i] += bhh->data[i];
        S3B_OK(upload_f32(L.gru_b, b.data(), b.size()));
        S3B_OK(upload_f32(L.whh, whh->data.data(), whh->numel()));
        S3B_OK(upload_f32(L.bhn, bhh->data.data() + 2 * H, H));
    }
    int clusters = 0;
    CUDA_OK(gru_max_active_clusters(&clusters));
    if (clusters < 1)
        return fail("the GRU recurrence kernel cannot run on this device: cudaOccupancyMaxActiveClusters reports 0 "
                    "clusters of %d CTAs with %zu bytes of shared memory each", kGruCtas, gru_smem_bytes());
    return 0;
}

// NPC (npc.py): per block i, ConvBlock conv [512][cin][3] -> bn1 -> act -> linear [512][512][1] -> bn2 (+ input) -> act,
// then MaskConvBlock tanh(conv1d(x, W * conv_mask)). BatchNorm (eval, eps 1e-5) folds into the conv in front of it in
// fp64: W' = W g / sqrt(v + eps), b' = (b - mu) g / sqrt(v + eps) + beta. The masked weight is multiplied by the file's
// conv_mask; weight left on a tap the config masks means the file's mask is not the config's, and the model is refused.
static int finalize_npc(s3b_model* m) {
    const s3b_npc_config& c = m->npc;
    const int NB = c.n_blocks, H = 512, k = c.kernel_size;
    m->layers.resize(NB);
    for (int i = 0; i < NB; ++i) {
        LayerW& L = m->layers[i];
        const std::string b = "blocks." + std::to_string(i) + ".";
        const int cin = i == 0 ? 80 : H, Cp = i == 0 ? kDecoar2K : H;
        for (int j = 0; j < 2; ++j) {
            const std::string conv = b + (j == 0 ? "conv." : "linear."), bn = b + (j == 0 ? "bn1." : "bn2.");
            const int kin = j == 0 ? cin : H, kw = j == 0 ? 3 : 1;
            const HostTensor *w, *bias;
            S3B_OK(need(m, conv + "weight", {H, kin, kw}, &w));
            S3B_OK(need(m, conv + "bias", {H}, &bias));
            std::vector<double> wd(w->data.begin(), w->data.end()), bd(bias->data.begin(), bias->data.end());
            if (c.batch_norm) {
                const HostTensor *g, *be, *mu, *var;
                S3B_OK(need(m, bn + "weight", {H}, &g));
                S3B_OK(need(m, bn + "bias", {H}, &be));
                S3B_OK(need(m, bn + "running_mean", {H}, &mu));
                S3B_OK(need(m, bn + "running_var", {H}, &var));
                for (int o = 0; o < H; ++o) {
                    const double sc = (double)g->data[o] / sqrt((double)var->data[o] + 1e-5);
                    for (size_t e = 0; e < (size_t)kin * kw; ++e) wd[(size_t)o * kin * kw + e] *= sc;
                    bd[o] = (bd[o] - (double)mu->data[o]) * sc + (double)be->data[o];
                }
            }
            const std::vector<float> wl = tap_weight_layout(wd.data(), H, kin, kw, 0, j == 0 ? Cp : H);
            const std::vector<float> bl(bd.begin(), bd.end());
            S3B_OK(upload_split(j == 0 ? L.fc1 : L.fc2, wl.data(), wl.size(), m->scheme));
            S3B_OK(upload_f32(j == 0 ? L.fc1_b : L.fc2_b, bl.data(), bl.size()));
        }
        const std::string mc = "masked_convs." + std::to_string(i) + ".";
        const HostTensor *w, *mask;
        S3B_OK(need(m, mc + "conv.weight", {H, H, k}, &w));
        S3B_OK(need(m, mc + "conv_mask", {H, H, k}, &mask));
        const int mw = npc_mask_width(c, i), head = (k - mw) / 2;
        std::vector<double> wd(w->numel());
        for (size_t e = 0; e < wd.size(); ++e) {
            wd[e] = (double)(w->data[e] * mask->data[e]);  // fp32, like the reference's conv_mask * weight
            const int tap = (int)(e % k);
            if (tap >= head && tap < head + mw && wd[e] != 0.0)
                return fail("%sconv_mask leaves weight on tap %d, which kernel_size %d and mask_size %d mask in block "
                            "%d (taps %d..%d): the checkpoint's mask is not the config's", mc.c_str(), tap, k,
                            c.mask_size, i, head, head + mw - 1);
        }
        const std::vector<float> wl = tap_weight_layout(wd.data(), H, H, k, mw, H);
        S3B_OK(upload_split(L.out, wl.data(), wl.size(), m->scheme));
        S3B_OK(upload_vec(m, mc + "conv.bias", H, L.out_b));
    }
    return 0;
}

// modified CPC (cpc/model.py CPCModel): gEncoder.conv{i} [256][cin][2 s] + bias, gEncoder.batchNorm{i} (ChannelNorm,
// affine [1][256][1]), then gAR.baseNet = nn.LSTM(256, 256, num_layers). Conv 1..4 become [256][2 s * 256] tap-major
// GEMM weights; the LSTM's two biases are summed into the input GEMM's bias.
static int finalize_cpc(s3b_model* m) {
    const int C = kCpcDim, H = kCpcDim, NL = m->cfg.num_layers;
    for (int i = 0; i < kCpcConvs; ++i) {
        const std::string conv = "gEncoder.conv" + std::to_string(i) + ".";
        const std::string bn = "gEncoder.batchNorm" + std::to_string(i) + ".";
        const int k = 2 * kCpcStride[i], cin = i == 0 ? 1 : C;
        const HostTensor *w, *g, *b;
        S3B_OK(need(m, conv + "weight", {C, cin, k}, &w));
        S3B_OK(need(m, bn + "weight", {1, C, 1}, &g));
        S3B_OK(need(m, bn + "bias", {1, C, 1}, &b));
        if (i == 0) {
            S3B_OK(upload_f32(m->conv0_w, w->data.data(), (size_t)C * k));
        } else {
            const std::vector<float> wl = tap_weight_layout(w->data.data(), C, C, k, 0, C);
            S3B_OK(upload_split(m->conv_w[i], wl.data(), wl.size(), m->scheme));
        }
        S3B_OK(upload_vec(m, conv + "bias", C, i == 0 ? m->conv0_b : m->conv_b[i]));
        S3B_OK(upload_f32(i == 0 ? m->norm0_g : m->conv_ln_g[i], g->data.data(), C));
        S3B_OK(upload_f32(i == 0 ? m->norm0_b : m->conv_ln_b[i], b->data.data(), C));
    }
    m->layers.resize(NL);
    for (int l = 0; l < NL; ++l) {
        LayerW& L = m->layers[l];
        const std::string s = "gAR.baseNet.", sl = "_l" + std::to_string(l);
        const HostTensor *wih, *whh, *bih, *bhh;
        S3B_OK(need(m, s + "weight_ih" + sl, {4 * H, C}, &wih));
        S3B_OK(need(m, s + "weight_hh" + sl, {4 * H, H}, &whh));
        S3B_OK(need(m, s + "bias_ih" + sl, {4 * H}, &bih));
        S3B_OK(need(m, s + "bias_hh" + sl, {4 * H}, &bhh));
        S3B_OK(upload_split(L.wih, wih->data.data(), wih->numel(), m->scheme));
        S3B_OK(upload_f32(L.whh, whh->data.data(), whh->numel()));
        std::vector<float> bsum(4 * H);
        for (int j = 0; j < 4 * H; ++j) bsum[j] = bih->data[j] + bhh->data[j];
        S3B_OK(upload_f32(L.gru_b, bsum.data(), bsum.size()));
    }
    int clusters = 0;
    CUDA_OK(cpc_lstm_max_active_clusters(&clusters));
    if (clusters < 1)
        return fail("the CPC LSTM recurrence kernel cannot run on this device (no cluster of %d CTAs fits)", kCpcLstmCtas);
    return 0;
}

// post_extract_proj of DeCoAR and DeCoAR 2.0: [N][80] zero-padded to K = kDecoar2K, the width of the CMVN kernel's
// operand planes
static int upload_fbank_proj(s3b_model* m, int N) {
    const HostTensor* t;
    S3B_OK(need(m, "post_extract_proj.weight", {N, 80}, &t));
    const std::vector<float> wp = tap_weight_layout(t->data.data(), N, 80, 1, 0, kDecoar2K);
    S3B_OK(upload_split(m->proj_w, wp.data(), wp.size(), m->scheme));
    return upload_vec(m, "post_extract_proj.bias", N, m->proj_b);
}

// DeCoAR (decoar.py): post_extract_proj = Linear(80, 1024), then {forward,backward}_lstm = nn.LSTM(1024, 1024,
// num_layers=4). The recurrence kernel needs the whole device: kLstmCtas co-resident CTAs, one per SM.
static int finalize_decoar(s3b_model* m) {
    const int NL = m->cfg.num_layers, H = kLstmHidden;
    S3B_OK(upload_fbank_proj(m, H));
    m->layers.resize(2 * NL);
    for (int l = 0; l < NL; ++l)
        for (int d = 0; d < 2; ++d) {
            LayerW& L = m->layers[2 * l + d];
            const std::string p = std::string(d == 0 ? "forward_lstm." : "backward_lstm."), k = std::to_string(l);
            const HostTensor *wih, *whh, *bih, *bhh;
            S3B_OK(need(m, p + "weight_ih_l" + k, {4 * H, H}, &wih));
            S3B_OK(need(m, p + "weight_hh_l" + k, {4 * H, H}, &whh));
            S3B_OK(need(m, p + "bias_ih_l" + k, {4 * H}, &bih));
            S3B_OK(need(m, p + "bias_hh_l" + k, {4 * H}, &bhh));
            S3B_OK(upload_split(L.wih, wih->data.data(), wih->numel(), m->scheme));
            std::vector<float> b(bih->data);
            for (int i = 0; i < 4 * H; ++i) b[i] += bhh->data[i];
            S3B_OK(upload_f32(L.gru_b, b.data(), b.size()));
            S3B_OK(upload_f32(L.whh, whh->data.data(), whh->numel()));
        }
    int ok = 0, sms = 0, smem = 0;
    CUDA_OK(lstm_fits(&ok, &sms, &smem));
    if (sms < kLstmCtas)
        return fail("the LSTM recurrence kernel needs %d SMs (one CTA each, all co-resident); this device has %d",
                    kLstmCtas, sms);
    if ((size_t)smem < lstm_smem_bytes())
        return fail("the LSTM recurrence kernel needs %zu bytes of shared memory per CTA; this device allows %d",
                    lstm_smem_bytes(), smem);
    if (!ok)
        return fail("the LSTM recurrence kernel cannot run on this device: %d co-resident CTAs with %zu bytes of "
                    "shared memory each (cooperative launch) do not fit", kLstmCtas, lstm_smem_bytes());
    return 0;
}

// SSAST (ast_models.py): the patch embedding, class tokens and positional table, then timm's DeiT blocks (norm1 ->
// attn.qkv [3D][D] with q | k | v rows, 64 per head -> attn.proj; norm2 -> mlp.fc1 -> GELU -> mlp.fc2)
static int finalize_ssast(s3b_model* m) {
    const SsastGeom g = ssast_geom(m->ssast);
    const int D = m->cfg.embed_dim, F = m->cfg.ffn_dim;
    const HostTensor* t;
    if (m->ssast.patch) {
        S3B_OK(need(m, "patch_embed.proj.weight", {D, 1, 16, 16}, &t));
        S3B_OK(upload_split(m->proj_w, t->data.data(), t->numel(), m->scheme));  // column kf * 16 + kt
    } else {
        // [D][1][128 f][2 dt] read as a conv of 2 taps over 128 channels: column dt * 128 + f
        S3B_OK(need(m, "patch_embed.proj.weight", {D, 1, 128, 2}, &t));
        const std::vector<float> w = tap_weight_layout(t->data.data(), D, 128, 2, 0, 128);
        S3B_OK(upload_split(m->proj_w, w.data(), w.size(), m->scheme));
    }
    S3B_OK(upload_vec(m, "patch_embed.proj.bias", D, m->proj_b));
    S3B_OK(need(m, "cls_token", {1, 1, D}, &t));
    S3B_OK(upload_f32(m->cls_tok, t->data.data(), t->numel()));
    S3B_OK(need(m, "dist_token", {1, 1, D}, &t));
    S3B_OK(upload_f32(m->dist_tok, t->data.data(), t->numel()));
    S3B_OK(need(m, "pos_embed", {1, 2 + g.P, D}, &t));
    S3B_OK(upload_f32(m->pos_tab, t->data.data(), t->numel()));
    m->layers.resize(m->cfg.num_layers);
    for (int l = 0; l < m->cfg.num_layers; ++l) {
        LayerW& L = m->layers[l];
        const std::string p = "blocks." + std::to_string(l) + ".";
        S3B_OK(need(m, p + "attn.qkv.weight", {3 * D, D}, &t));
        S3B_OK(upload_split(L.qkv, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "attn.qkv.bias", 3 * D, L.qkv_b));
        S3B_OK(need(m, p + "attn.proj.weight", {D, D}, &t));
        S3B_OK(upload_split(L.out, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "attn.proj.bias", D, L.out_b));
        S3B_OK(upload_vec(m, p + "norm1.weight", D, L.ln1_g));
        S3B_OK(upload_vec(m, p + "norm1.bias", D, L.ln1_b));
        S3B_OK(upload_vec(m, p + "norm2.weight", D, L.ln2_g));
        S3B_OK(upload_vec(m, p + "norm2.bias", D, L.ln2_b));
        S3B_OK(need(m, p + "mlp.fc1.weight", {F, D}, &t));
        S3B_OK(upload_split(L.fc1, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "mlp.fc1.bias", F, L.fc1_b));
        S3B_OK(need(m, p + "mlp.fc2.weight", {D, F}, &t));
        S3B_OK(upload_split(L.fc2, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "mlp.fc2.bias", D, L.fc2_b));
    }
    return 0;
}

// The conv-stack and fbank encoders: front end, pos_conv, transformer or Conformer layers, prediction heads
static int finalize_encoder(s3b_model* m) {
    const s3b_config& c = m->cfg;
    const int D = c.embed_dim, F = c.ffn_dim, C = kConvDim;
    const HostTensor* t;
    const std::string fe = "feature_extractor.conv_layers.";

    if (m->kind == kFbankEncoder) {
        S3B_OK(upload_fbank_proj(m, D));
    } else {
        // ---- conv 0 ------------------------------------------------------------------------------
        S3B_OK(need(m, fe + "0.0.weight", {C, 1, kConvK[0]}, &t));
        S3B_OK(upload_f32(m->conv0_w, t->data.data(), t->numel()));
        if (c.conv_bias) S3B_OK(upload_vec(m, fe + "0.0.bias", C, m->conv0_b));
        if (c.extractor_layer_norm) {
            S3B_OK(upload_vec(m, fe + "0.2.1.weight", C, m->norm0_g));
            S3B_OK(upload_vec(m, fe + "0.2.1.bias", C, m->norm0_b));
        } else {
            S3B_OK(upload_vec(m, fe + "0.2.weight", C, m->norm0_g));
            S3B_OK(upload_vec(m, fe + "0.2.bias", C, m->norm0_b));
        }
        // ---- conv 1..6 ---------------------------------------------------------------------------------------
        for (int i = 1; i < kNumConv; ++i) {
            const std::string p = fe + std::to_string(i);
            const int kw = kConvK[i];
            S3B_OK(need(m, p + ".0.weight", {C, C, kw}, &t));
            const std::vector<float> r = tap_weight_layout(t->data.data(), C, C, kw, 0, C);
            S3B_OK(upload_split(m->conv_w[i], r.data(), r.size(), m->scheme));
            if (c.conv_bias) S3B_OK(upload_vec(m, p + ".0.bias", C, m->conv_b[i]));
            if (c.extractor_layer_norm) {
                S3B_OK(upload_vec(m, p + ".2.1.weight", C, m->conv_ln_g[i]));
                S3B_OK(upload_vec(m, p + ".2.1.bias", C, m->conv_ln_b[i]));
            }
        }
        // ---- LayerNorm(512) + post_extract_proj ----------------------------------------------------------
        if (!c.no_feature_layer_norm) {
            S3B_OK(upload_vec(m, "layer_norm.weight", C, m->ln512_g));
            S3B_OK(upload_vec(m, "layer_norm.bias", C, m->ln512_b));
        }
        S3B_OK(need(m, "post_extract_proj.weight", {D, C}, &t));
        S3B_OK(upload_split(m->proj_w, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, "post_extract_proj.bias", D, m->proj_b));
    }
    // ---- data2vec pos_conv: pos_conv_depth plain Conv1d(k, padding k/2, groups) blocks (make_conv_block,
    //      wav2vec2_model.py:2995-3026). Four taps per k-block like pos_w4 below (posconv4_weight_layout)
    if (c.conformer) {
        // ConformerEncoder.extract_features never calls pos_conv (wav2vec2_model.py:3171-3211): its weights are unused
    } else if (c.pos_conv_depth > 1) {
        const int G = c.pos_conv_groups, cpg = D / G, Kp = pos_taps(c);
        m->posd_w4.resize(c.pos_conv_depth);
        m->posd_b.resize(c.pos_conv_depth);
        for (int i = 0; i < c.pos_conv_depth; ++i) {
            const std::string pre = "encoder.pos_conv." + std::to_string(i) + ".0.";
            const HostTensor* tw;
            S3B_OK(need(m, pre + "weight", {D, cpg, Kp}, &tw));
            const std::vector<float> w4 = posconv4_weight_layout(tw->data.data(), D, G, Kp);
            S3B_OK(upload_split(m->posd_w4[i], w4.data(), w4.size()));
            S3B_OK(upload_vec(m, pre + "bias", D, m->posd_b[i]));
        }
    } else {
    // ---- pos_conv: fold weight_norm(dim=2): W[o][c][k] = g[k] * v[o][c][k] / ||v[:,:,k]||  ---------------
    //      (make_conv_pos, wav2vec2_model.py:2937-2953), in the four-tap layout where posconv4_ok, else the one-tap one
        const int G = c.pos_conv_groups, cpg = D / G, Kp = c.pos_conv_kernel;
        const HostTensor *tg, *tv;
        S3B_OK(need(m, "encoder.pos_conv.0.weight_g", {1, 1, Kp}, &tg));
        S3B_OK(need(m, "encoder.pos_conv.0.weight_v", {D, cpg, Kp}, &tv));
        std::vector<double> nrm(Kp, 0.0);
        for (size_t oc = 0; oc < (size_t)D * cpg; ++oc)
            for (int k = 0; k < Kp; ++k) {
                const double v = tv->data[oc * Kp + k];
                nrm[k] += v * v;
            }
        std::vector<float> scale(Kp);
        for (int k = 0; k < Kp; ++k) scale[k] = (float)((double)tg->data[k] / sqrt(nrm[k]));
        std::vector<float> wf((size_t)D * cpg * Kp);
        for (size_t oc = 0; oc < (size_t)D * cpg; ++oc)
            for (int k = 0; k < Kp; ++k) wf[oc * Kp + k] = tv->data[oc * Kp + k] * scale[k];  // fp32, like torch's _weight_norm
        if (posconv4_ok(c)) {
            const std::vector<float> w4 = posconv4_weight_layout(wf.data(), D, G, Kp);
            S3B_OK(upload_split(m->pos_w4, w4.data(), w4.size()));
        } else {
            const std::vector<float> wb = tap_weight_layout(wf.data(), D, cpg, Kp, 0, posconv_kc(cpg));
            S3B_OK(upload_split(m->pos_w, wb.data(), wb.size()));
        }
        S3B_OK(upload_vec(m, "encoder.pos_conv.0.bias", D, m->pos_b));
    }
    S3B_OK(upload_vec(m, "encoder.layer_norm.weight", D, m->enc_ln_g));
    S3B_OK(upload_vec(m, "encoder.layer_norm.bias", D, m->enc_ln_b));
    // ---- transformer layers ------------------------------------------------------------------------
    m->layers.resize(c.num_layers);
    if (c.conformer) {
        m->rope_inv_freq = default_inv_freq();
        for (int l = 0; l < c.num_layers; ++l) S3B_OK(finalize_conformer_layer(m, l));
        S3B_OK(build_rope_table(m, 4096));  // utterances up to 82 s; rebuilt (synchronously) for longer batches
    }
    for (int l = 0; l < c.num_layers && !c.conformer; ++l) {
        LayerW& L = m->layers[l];
        const std::string p = "encoder.layers." + std::to_string(l) + ".";
        const HostTensor *wq, *wk, *wv, *bq, *bk, *bv;
        S3B_OK(need(m, p + "self_attn.q_proj.weight", {D, D}, &wq));
        S3B_OK(need(m, p + "self_attn.k_proj.weight", {D, D}, &wk));
        S3B_OK(need(m, p + "self_attn.v_proj.weight", {D, D}, &wv));
        S3B_OK(need(m, p + "self_attn.q_proj.bias", {D}, &bq));
        S3B_OK(need(m, p + "self_attn.k_proj.bias", {D}, &bk));
        S3B_OK(need(m, p + "self_attn.v_proj.bias", {D}, &bv));
        std::vector<float> w((size_t)3 * D * D), b((size_t)3 * D);
        memcpy(w.data(), wq->data.data(), (size_t)D * D * 4);
        memcpy(w.data() + (size_t)D * D, wk->data.data(), (size_t)D * D * 4);
        memcpy(w.data() + (size_t)2 * D * D, wv->data.data(), (size_t)D * D * 4);
        memcpy(b.data(), bq->data.data(), D * 4), memcpy(b.data() + D, bk->data.data(), D * 4);
        memcpy(b.data() + 2 * D, bv->data.data(), D * 4);
        S3B_OK(upload_split(L.qkv, w.data(), w.size(), m->scheme));
        S3B_OK(upload_f32(L.qkv_b, b.data(), b.size()));
        S3B_OK(need(m, p + "self_attn.out_proj.weight", {D, D}, &t));
        S3B_OK(upload_split(L.out, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "self_attn.out_proj.bias", D, L.out_b));
        S3B_OK(upload_vec(m, p + "self_attn_layer_norm.weight", D, L.ln1_g));
        S3B_OK(upload_vec(m, p + "self_attn_layer_norm.bias", D, L.ln1_b));
        S3B_OK(need(m, p + "fc1.weight", {F, D}, &t));
        S3B_OK(upload_split(L.fc1, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "fc1.bias", F, L.fc1_b));
        S3B_OK(need(m, p + "fc2.weight", {D, F}, &t));
        S3B_OK(upload_split(L.fc2, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, p + "fc2.bias", D, L.fc2_b));
        S3B_OK(upload_vec(m, p + "final_layer_norm.weight", D, L.ln2_g));
        S3B_OK(upload_vec(m, p + "final_layer_norm.bias", D, L.ln2_b));
        if (c.relative_position && c.gru_rel_pos) {
            S3B_OK(need(m, p + "self_attn.grep_linear.weight", {8, 64}, &t));
            S3B_OK(upload_f32(L.grep_w, t->data.data(), t->numel()));
            S3B_OK(upload_vec(m, p + "self_attn.grep_linear.bias", 8, L.grep_b));
            S3B_OK(need(m, p + "self_attn.grep_a", {1, c.num_heads, 1, 1}, &t));
            S3B_OK(upload_f32(L.grep_a, t->data.data(), t->numel()));
        }
    }
    if (c.pred_heads > 0) {
        // output_layer = Linear(D, N*D) -> GELU -> SplitLinear(D, N, D) (distiller/model.py:150-160); SplitLinear keeps
        // its weight as [task][in][out] (module.py:66-73): transposed per task to the [out][in] layout of the GEMM
        const int N = c.pred_heads;
        S3B_OK(need(m, "output_layer.0.weight", {(int64_t)N * D, D}, &t));
        S3B_OK(upload_split(m->pred1_w, t->data.data(), t->numel(), m->scheme));
        S3B_OK(upload_vec(m, "output_layer.0.bias", (int64_t)N * D, m->pred1_b));
        S3B_OK(need(m, "output_layer.2.weight", {N, D, D}, &t));
        m->pred2_w.resize(N);
        std::vector<float> wt((size_t)D * D);
        for (int k = 0; k < N; ++k) {
            for (int i = 0; i < D; ++i)
                for (int o = 0; o < D; ++o) wt[(size_t)o * D + i] = t->data[((size_t)k * D + i) * D + o];
            S3B_OK(upload_split(m->pred2_w[k], wt.data(), wt.size(), m->scheme));
        }
        const HostTensor* tb;
        S3B_OK(need(m, "output_layer.2.bias", {1, 1, N, D}, &tb));
        S3B_OK(upload_f32(m->pred2_b, tb->data.data(), tb->numel()));
    }
    if (c.relative_position) {
        S3B_OK(need(m, "encoder.layers.0.self_attn.relative_attention_bias.weight", {c.num_buckets, c.num_heads}, &t));
        S3B_OK(upload_f32(m->rel_table_src, t->data.data(), t->numel()));
        S3B_OK(build_rel_table(m, 4096));  // utterances up to 82 s; rebuilt (synchronously) for longer batches
    }
    return 0;
}

extern "C" int s3b_model_finalize(s3b_model* m) {
    if (!m) return fail("null model");
    if (m->finalized) return 0;
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    int dev = 0;
    CUDA_OK(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    CUDA_OK(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
        return fail("device is sm_%d%d; this library contains sm_90a code only", prop.major, prop.minor);
    m->sm_count = prop.multiProcessorCount;
    switch (m->kind) {
    case kGruStack: S3B_OK(finalize_apc(m)); break;
    case kLstmStack: S3B_OK(finalize_decoar(m)); break;
    case kNpcStack: S3B_OK(finalize_npc(m)); break;
    case kCpcStack: S3B_OK(finalize_cpc(m)); break;
    case kSsastEncoder: S3B_OK(finalize_ssast(m)); break;
    case kConvEncoder:
    case kFbankEncoder: S3B_OK(finalize_encoder(m)); break;
    }
    if (m->kind != kConvEncoder && m->kind != kCpcStack) CUDA_OK(init_fbank_tables());  // built here, not in a forward
    m->host.clear();
    m->finalized = true;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// frame bookkeeping
// ------------------------------------------------------------------------------------------------
extern "C" int64_t s3b_num_frames(const s3b_model* m, int64_t max_len) {
    const int64_t T = model_frames(m, max_len);
    return T > 0 ? T : -1;
}

extern "C" int32_t s3b_num_outputs(const s3b_model* m) {
    if (!m) return -1;
    switch (m->kind) {
    case kGruStack: return m->cfg.num_layers;  // the output of every GRU layer (+ residual)
    case kLstmStack: return m->decoar_all_layers ? m->cfg.num_layers : 1;  // decoar_layers: every layer; decoar: the last
    case kNpcStack: return 2 * m->cfg.num_layers + 1;  // every block, every masked conv, then feat
    case kCpcStack: return 2;                          // the encoder's output, then the last LSTM layer's
    case kSsastEncoder: return m->cfg.num_layers;      // every block's output
    default: return m->cfg.num_layers + 1 + m->cfg.pred_heads;
    }
}

extern "C" int s3b_valid_frames(const s3b_model* m, const int64_t* lens, int32_t batch, int64_t max_len,
                                int32_t* valid) {
    if (!m || !lens || !valid) return fail("null argument");
    const int64_t T = model_frames(m, max_len);
    if (T <= 0) return fail_too_short(m, max_len);
    const char* fbank_model = m->kind == kFbankEncoder ? "DeCoAR 2.0"
                              : m->kind == kGruStack   ? "APC"
                              : m->kind == kLstmStack  ? "DeCoAR"
                              : m->kind == kNpcStack   ? "NPC"
                                                       : nullptr;
    bool any_pad = false;
    for (int b = 0; b < batch; ++b) {
        if (lens[b] < 1 || lens[b] > max_len) return fail("lens[%d]=%lld out of range", b, (long long)lens[b]);
        if (fbank_model != nullptr && lens[b] < kDecoar2MinLen)
            return fail("lens[%d]=%lld: %s needs >= %lld samples (2 fbank frames; the CMVN std of one frame is NaN)", b,
                        (long long)lens[b], fbank_model, (long long)kDecoar2MinLen);
        any_pad |= lens[b] < max_len;
    }
    for (int b = 0; b < batch; ++b) {
        int64_t v;
        if (m->kind == kSsastEncoder) {
            // the frames of the utterance's own samples at the downsample rate; every frame is computed
            const int rate = ssast_geom(m->ssast).rate;
            v = (lens[b] + rate - 1) / rate;
        } else if (m->kind != kConvEncoder) {
            // pad_sequence of the per-utterance features (apc/expert.py:47-51, decoar2/expert.py:81-92); modified CPC:
            // the frames of the utterance's own conv chain (0 below 159 samples), though every frame is computed
            v = model_frames(m, lens[b]);
        } else if (m->cfg.family == 1) {
            // wav2vec2: conv-length rule, only when the batch has any padding (wav2vec2_model.py:2652-2671). The
            // reference evaluates floor((n - k) / s + 1) in fp32 WITHOUT clamping, so an utterance shorter than the
            // receptive field yields 0 or a negative length and `mask[b, length - 1] = 1` wraps around like any
            // negative Python index: valid = ((length - 1) mod T) + 1.
            if (!any_pad) {
                v = T;
            } else {
                float n = (float)lens[b];
                for (int i = 0; i < kNumConv; ++i) n = floorf((n - (float)kConvK[i]) / (float)kConvS[i] + 1.0f);
                int64_t idx = (int64_t)n - 1;
                if (idx < -T) return fail("lens[%d]=%lld: the reference's mask index %lld is out of range for T=%lld",
                                          b, (long long)lens[b], (long long)idx, (long long)T);
                if (idx < 0) idx += T;
                v = idx + 1;
            }
        } else if (m->cfg.family == 3) {
            // Distiller: conv length formula with truncating division, always applied (distiller/model.py:272-286)
            int64_t n = lens[b];
            for (int i = 0; i < kNumConv; ++i) n = (n - kConvK[i]) / kConvS[i] + 1;  // C++ division truncates
            if (n < 1) return fail("lens[%d]=%lld yields no valid frame: the reference's attention would see only padding",
                                   b, (long long)lens[b]);
            v = n;
        } else {
            // HuBERT / WavLM: frame t is padding iff all samples of chunk t are padding, chunk = Lmax // T
            const int64_t chunk = max_len / T;
            v = (lens[b] + chunk - 1) / chunk;
        }
        valid[b] = (int32_t)(v > T ? T : v);
    }
    return 0;
}

// WavLM relative-position buckets (modules.py:418-448), exported so that the product's integer rule can be pinned
// against the reference-generated table (tests/test_oracle_cpu.py); pure host arithmetic, no GPU needed.
extern "C" int s3b_wavlm_buckets(int32_t num_buckets, int32_t max_distance, const int32_t* rel, int32_t n,
                                 int32_t* out) {
    if (!rel || !out || n < 0) return fail("null argument");
    if (num_buckets < 4 || num_buckets % 4 != 0 || max_distance <= num_buckets / 4)
        return fail("num_buckets must be a positive multiple of 4 and max_distance > num_buckets / 4");
    for (int i = 0; i < n; ++i) out[i] = wavlm_rel_bucket(rel[i], num_buckets, max_distance);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// GEMM descriptors
// ------------------------------------------------------------------------------------------------
struct Epi {
    const float* bias = nullptr;
    const float* residual = nullptr;
    const uint8_t* row_mask = nullptr;
    int gelu = 0;
    int res_first = 0;  // the activation after the residual add (gemm.cuh)
    float* out_f32 = nullptr;
    OutPlanes op = no_planes();  // GEMM-operand output (either format)
};

// the two common epilogues: an fp32 output (+ bias, + residual), or operand planes (+ bias, + activation)
static Epi epi_f32(float* out, const float* bias = nullptr, const float* residual = nullptr) {
    Epi e;
    e.out_f32 = out, e.bias = bias, e.residual = residual;
    return e;
}
static Epi epi_planes(const OutPlanes& op, const float* bias = nullptr, int gelu = 0) {
    Epi e;
    e.op = op, e.bias = bias, e.gelu = gelu;
    return e;
}

static void set_epi(GemmParams& p, const Epi& e, int ldo) {
    p.bias = e.bias, p.residual = e.residual, p.row_mask = e.row_mask, p.gelu = e.gelu, p.res_first = e.res_first;
    p.out_f32 = e.out_f32, p.out_hi = e.op.hi, p.out_lo = e.op.lo, p.out_h8 = e.op.h8, p.out_l8 = e.op.l8;
    p.out_fmt = e.op.fmt, p.ldo = ldo;
    p.qkv_mode = 0;
}

// q pre-scaled by head_dim^-0.5 and log2(e): the attention kernel's softmax runs on exp2. For 64-wide heads that is
// log2(e) / 8, exact but for the rounding of log2(e); for 80 and 120 the product is rounded to one fp32 constant.
static const float kQScale = 0.125f * 1.4426950408889634f;
static float q_scale(int hd) { return hd == 64 ? kQScale : (float)(1.4426950408889634 / sqrt((double)hd)); }

// QKV epilogue of a [B*T][3D] linear: bias, then q (scaled), k as [B][H][T][hd] and v transposed as [B][H][hd][Tp]
// (Tp = T rounded up to 8), all as bf16 hi/lo planes. col0: the QKV column of the launch's first column (a launch
// covering only [k | v] or v), `bias` then starts at that column.
static void set_qkv_epi(GemmParams& p, const float* bias, int T, int H, int hd, const SplitBuf& q, const SplitBuf& k,
                        const SplitBuf& vt, int col0 = 0) {
    const int D = H * hd;
    set_epi(p, epi_f32(nullptr, bias), 3 * D);
    p.qkv_mode = 1, p.T = T, p.Tp = (T + 7) & ~7, p.H = H, p.D = D, p.q_scale = q_scale(hd), p.qkv_col0 = col0;
    p.hd = hd, p.hd_magic = 0xFFFFFFFFu / (unsigned)hd + 1u, p.qk_head_step = (T - 1) * hd;
    p.q_hi = q.h(), p.q_lo = q.l(), p.k_hi = k.h(), p.k_lo = k.l();
    p.vt_hi = vt.h(), p.vt_lo = vt.l();
}

// Tile width for a flat [M][N] linear layer. Both widths give bit-identical results. The rule comes from
// tools/gemm_shapes.py on an H100 80GB HBM3 at 400 W, at the encoder shapes of hubert_base (K = 768, 3072) and
// wav2vec2_large (K = 1024, 4096), M = 7984..15984, with the ping-pong kernel at 128 columns:
//  - bf16x3: 128 columns, 1.4x-2.2x faster than 256 at every measured shape.
//  - f16q8 with K <= 1024: 128 columns, 1.04x-1.5x faster than 256, except wav2vec2_large's fc1 (N = 4096), where
//    256 is 3-6% faster; hubert_base's fc1 (N = 3072) prefers 128 by 4%, so N does not make a clean cut.
//  - f16q8 with K >= 3072 (fc2): 256 columns are 21-28% faster when their last round of tiles fills at least half of
//    the SMs (or none is partial); otherwise that round runs half empty and 128 columns are 17% faster (hubert_base
//    fc2 at M = 7984: 189 tiles of 256 on 132 SMs). The K >= 2048 cut lies between measured Ks (1024 and 3072).
// The epilogue kind does not enter the rule: at K <= 1024 the GELU (fc1) and fp32 epilogues ranked the two widths the
// same way, but for the one shape above.
// Since f16q8's 128-wide tiles run in clusters of 2 (pick_cluster_n), hubert_base's shapes were re-measured (H100
// 80GB HBM3, 700 W) and the rule still holds there: at K = 768, 128 columns are 1.15x-1.65x faster than 256 (QKV,
// out_proj, fc1); fc2 at M = 7984 takes 128 columns, now 10% faster than 256 (0.146 against 0.161 ms), and at
// M = 15968 the two tie (256 columns 0.281 ms, 128 columns 0.282). wav2vec2_large's shapes were not re-measured.
// An N that is not a multiple of 128 takes the widest of 192, 64, 32 and 16 that divides it. forced != 0 (the tile
// width s3b_linear_ex or s3b_gemm_bench asks for) is taken wherever it divides N.
static int pick_bn(int64_t M, int N, int K, int scheme, int sm_count, int forced) {
    if (forced != 0 && N % forced == 0) return forced;
    if (N % 128 != 0) return N % 192 == 0 ? 192 : N % 64 == 0 ? 64 : N % 32 == 0 ? 32 : 16;
    if (N % 256 != 0 || scheme == 0 || K < 2048) return 128;
    const int sms = sm_count > 0 ? sm_count : 1;
    const int64_t tiles = (M + 127) / 128 * (N / 256);
    const int64_t last = tiles % sms;
    return (last == 0 || last >= sms / 2) ? 256 : 128;
}

// CTAs per cluster along N for a launch of n_tiles tiles of bn columns: 128-wide tiles take `preferred` (1, 2 or 4)
// where it divides n_tiles, every other width 1. The CTAs of a cluster load each A tile once between them (TMA
// multicast), which cuts the L2 -> SM operand traffic per tile. Results are bit-identical whatever the size.
// f16q8 linears prefer 2: tools/gemm_shapes.py --k-sweep (H100 80GB HBM3, 700 W; M = 7984, N = 2304) cuts the
// per-K cost of a round of 128-wide tiles from 18.2 to 14.5 ns and leaves the fixed cost at 2-3 us, and
// hubert_base's QKV, out_proj, fc1 and fc2 run 8-18% faster (4 helps fc1 by another 1%, the only one it divides).
// bf16x3 prefers 1: its per-K cost does not drop (15.8 ns, 16.3 in clusters of 2), and three of its four
// encoder linears run 2-3% slower in clusters of 2.
// S3B_GEMM_CLUSTER=1 / 2 / 4 replaces `preferred` at every call: 1 turns clusters off, for A/B runs of one build.
static int pick_cluster_n(int bn, int n_tiles, int preferred) {
    if (const char* e = getenv("S3B_GEMM_CLUSTER")) {
        const int v = atoi(e);
        if (v == 1 || v == 2 || v == 4) preferred = v;
    }
    return bn == 128 && n_tiles % preferred == 0 ? preferred : 1;
}

#define TMAP_OK(expr)                                                                     \
    do {                                                                                  \
        int _r = (expr);                                                                  \
        if (_r != 0) return fail("cuTensorMapEncodeTiled failed (%d) at %s:%d", _r, __FILE__, __LINE__); \
    } while (0)

// The A and B tensor maps of one launch in its operand scheme, the one place they are encoded. A: the (k, row, batch)
// view of [batches][rows][ka] from element a_off of A's planes, rows lda and batches bstride elements apart, boxes
// {64, a_box}. W: the [N][K] K-major weight, boxes {64, bn}.
static int gemm_tmaps(GemmParams& p, int scheme, const SplitBuf& A, size_t a_off, uint64_t ka, uint64_t rows,
                      uint64_t batches, uint64_t lda, uint64_t bstride, uint32_t a_box, const SplitBuf& W, int N, int K,
                      int bn) {
    const uint64_t wn = (uint64_t)N * K;
    TMAP_OK(encode_tmap_bf16_3d(&p.a_hi, A.h() + a_off, ka, rows, batches, lda, bstride, 64, a_box));
    TMAP_OK(encode_tmap_bf16_3d(&p.b_hi, W.h(), K, N, 1, K, wn, 64, bn));
    if (scheme != 0) {
        TMAP_OK(encode_tmap_u8_3d(&p.a_h8, A.h8() + a_off, ka, rows, batches, lda, bstride, 64, a_box));
        TMAP_OK(encode_tmap_u8_3d(&p.a_l8, A.l8() + a_off, ka, rows, batches, lda, bstride, 64, a_box));
        TMAP_OK(encode_tmap_u8_3d(&p.b_h8, W.h8(), K, N, 1, K, wn, 64, bn));
        TMAP_OK(encode_tmap_u8_3d(&p.b_l8, W.l8(), K, N, 1, K, wn, 64, bn));
    } else {
        TMAP_OK(encode_tmap_bf16_3d(&p.a_lo, A.l() + a_off, ka, rows, batches, lda, bstride, 64, a_box));
        TMAP_OK(encode_tmap_bf16_3d(&p.b_lo, W.l(), K, N, 1, K, wn, 64, bn));
    }
    p.scheme = scheme;
    return 0;
}

// out[M][N] = A[M][K] * W[N][K]^T with epilogue `e`, flat token-major A (hi/lo planes), K % 64 == 0
// scheme 1: A and W are f16q8 operands (SplitBuf fmt 1), K % 128 == 0, tile width 128 or 256.
// sm_count: SMs of the device the GEMM runs on (pick_bn's tile-width rule).
// lda / a_off: A is the [M][K] column slice starting at element a_off of rows that are lda elements apart (0 = dense).
// forced_bn: the tile width pick_bn takes wherever it divides N (0 = the rule's choice).
static int linear_params(GemmParams& p, const SplitBuf& A, const SplitBuf& W, int64_t M, int N, int K, int scheme,
                         int sm_count, const Epi& e, int64_t lda = 0, size_t a_off = 0, int forced_bn = 0) {
    memset(&p, 0, sizeof(p));
    if (lda == 0) lda = K;
    if (K % 64 != 0 || N % 16 != 0) return fail("linear: K %% 64 or N %% 16 violated (N=%d K=%d)", N, K);
    const int bn = pick_bn(M, N, K, scheme, sm_count, forced_bn);
    const int cn = pick_cluster_n(bn, N / bn, scheme != 0 ? 2 : 1);
    if (scheme != 0 && ((bn != 128 && bn != 256) || K % 128 != 0))
        return fail("f16q8 GEMM needs a tile width of 128 or 256 and K %% 128 == 0 (N=%d K=%d)", N, K);
    S3B_OK(gemm_tmaps(p, scheme, A, a_off, K, M, 1, lda, (uint64_t)M * lda, 128 / cn, W, N, K, bn));
    p.num_k_blocks = K / 64, p.kb_per_row = K / 64;
    p.batches = 1, p.rows_per_batch = (int)M, p.tiles_m_per_batch = (int)((M + 127) / 128);
    p.n_tiles = N / bn, p.bn = bn, p.cluster_n = cn;
    p.out_rows_per_batch = (int)M;
    p.alg_flops = 2.0 * (double)M * N * K;
    set_epi(p, e, N);
    return 0;
}

// Convolution of k taps into N channels (a multiple of 128) over channels-last operand planes A [B][Lin][Cp], with
// epilogue `e`, as one implicit GEMM over W [N][u * Cp] (tap_weight_layout; u = k - mask taps). Output row t of
// utterance b takes tap j from input row stride * t + j - pad of its own utterance, TMA zero-filling rows outside
// [0, Lin).
//  - stride 1 (NPC): same padding, pad = (k - 1) / 2 and Lout = Lin. Only the taps outside the centred band of `mask`
//    taps are contracted: one k-block row per tap (Cp / 64 k-blocks), and the rows after the left run of u / 2 taps
//    skip the band (a_gap).
//  - stride s >= 2, mask 0: no padding in the GEMM. Row t of the [ceil(Lin / s)][s Cp] view holds input rows
//    s t .. s t + s - 1, so taps 0 .. s - 1 come from view row t and taps s .. k - 1 from view row t + 1 (k <= 2 s).
//    conv 1..6 of the wav2vec 2.0 stack: s = 2, k in {2, 3}. Modified CPC's conv 1..4 (k = 2 s, padding p): A is the
//    producer's padded layout, Lin = s (Lout + 1) rows per utterance with p zero rows in front, so that the padding is
//    part of the operand and view rows t, t + 1 are exactly the output row's receptive field.
// alg_flops counts cin, the channels before padding.
static int conv_params(GemmParams& p, const SplitBuf& A, const SplitBuf& W, int B, int64_t Lin, int64_t Lout,
                       int stride, int N, int cin, int Cp, int k, int mask, int scheme, const Epi& e) {
    memset(&p, 0, sizeof(p));
    if (N % 128 != 0) return fail("conv: N %d must be a multiple of 128", N);
    const int u = k - mask, K = u * Cp, width = stride * Cp;
    // Tile: tools/gemm_shapes.py times the linear with conv i's M, N = 512 and K as a proxy (H100 80GB HBM3, 700 W,
    // hubert_base's conv stack at 32 x 10 s). f16q8 on 128-wide tiles in clusters of 4 (N = 512 is four tiles, which
    // then share each A tile) runs conv 1..6 in 6.96 ms, against 7.57 in clusters of 2, 7.97 on 256-wide tiles
    // (10-13% slower at every conv) and 9.49 on unclustered 128-wide tiles. bf16x3 stays on unclustered 128-wide
    // tiles: clusters of 2 and 4 are 2% and 10% slower there, and 256-wide tiles 70%.
    // N = 256 (modified CPC) has two tiles, which f16q8 clusters in twos.
    const int bn = 128;
    const int cn = pick_cluster_n(bn, N / bn, scheme != 0 ? std::min(4, N / bn) : 1);
    S3B_OK(gemm_tmaps(p, scheme, A, 0, width, (uint64_t)((Lin + stride - 1) / stride), B, width, (uint64_t)Lin * Cp,
                      128 / cn, W, N, K, bn));
    p.num_k_blocks = K / 64, p.kb_per_row = width / 64;
    p.batches = B, p.rows_per_batch = (int)Lout, p.tiles_m_per_batch = (int)((Lout + 127) / 128);
    p.n_tiles = N / bn, p.bn = bn, p.cluster_n = cn;
    p.a_row_step = 1, p.a_row_off = stride == 1 ? -((k - 1) / 2) : 0, p.a_gap_at = u / 2, p.a_gap = mask;
    p.out_rows_per_batch = (int)Lout;
    p.alg_flops = 2.0 * (double)B * Lout * N * cin * u;
    set_epi(p, e, N);
    return 0;
}

// taps of ONE positional conv: conv_pos, or max(3, conv_pos / depth) for the data2vec blocks
// (wav2vec2_model.py:2996-2998); pos_taps4 = rounded up to the four-taps-per-k-block layout (zero taps appended)
static int pos_taps(const s3b_config& c) {
    return c.pos_conv_depth > 1 ? std::max(3, c.pos_conv_kernel / c.pos_conv_depth) : c.pos_conv_kernel;
}
static int pos_taps4(const s3b_config& c) { return (pos_taps(c) + 3) / 4 * 4; }

// grouped positional conv over x [B][T][D]: one k-block per tap; A row coordinate = t + tap - K/2 (TMA zero-fills t<0,
// t>=T). Groups of 80 and 120 channels take two 64-wide k-blocks per tap: the A box of the second reads on into the
// next group's channels (or, for the last group, past D: TMA zero fill), which meet the zero-padded weights of
// posconv_kc. The tile is exactly the group's cpg columns wide, so no output column lands in a neighbouring group, and
// it reads its group's rows of W [D][Kp * Kc].
static int posconv_params(GemmParams& p, const s3b_config& c, const SplitBuf& x, const SplitBuf& W, int B, int T,
                          const Epi& e) {
    memset(&p, 0, sizeof(p));
    const int D = c.embed_dim, G = c.pos_conv_groups, cpg = D / G, Kp = c.pos_conv_kernel, Kc = posconv_kc(cpg);
    S3B_OK(gemm_tmaps(p, 0, x, 0, D, T, B, D, (uint64_t)T * D, 128, W, D, Kp * Kc, cpg));
    p.batches = B, p.rows_per_batch = T, p.tiles_m_per_batch = (T + 127) / 128;
    p.n_tiles = G, p.bn = cpg, p.num_k_blocks = Kp * (Kc / 64), p.kb_per_row = Kc / 64;
    p.a_row_step = 1, p.a_row_off = -(Kp / 2), p.a_k_per_ntile = cpg;
    p.out_rows_per_batch = T;
    p.alg_flops = 2.0 * (double)B * T * D * cpg * Kp;
    set_epi(p, e, D);
    return 0;
}

// pos_conv with FOUR taps per k-block: consecutive taps read the same activation rows shifted by one
// frame, so the one-tap formulation (N = cpg = 48 columns) is bound by the shared-memory reads of its A operand
// (4 KB per 24-cycle MMA). Writing tap = 4q + j,
//     Z_j[u] = sum_q x[u + 4q - Kp/2] . W[4q + j],      conv[t] = sum_j Z_j[t + j]
// gives one GEMM with N = 4*cpg (96, 160, 192 or 256) columns per group and Kp/4 k-blocks whose A rows advance by
// 4; the four column blocks are re-aligned by posconv_combine_kernel (norm.cu). Rows u in [0, T+3) per utterance.
// W: the [G * 4cpg][Kq * 64] matrix of posconv4_weight_layout, one group's rows per tile. At 24 and 40 channels per
// group the one-tap formulation would be bound by its A reads even more than at 48, so those widths run four taps only.
static bool posconv4_ok(const s3b_config& c) {
    const int cpg = c.embed_dim / c.pos_conv_groups;
    if (c.pos_conv_depth > 1) return true;  // the only formulation of the data2vec blocks (checked at create)
    return c.pos_conv_kernel % 4 == 0 && (posconv4_only(cpg) || cpg == 48 || cpg == 64);
}
static int posconv4_params(GemmParams& p, const s3b_config& c, const SplitBuf& x, const SplitBuf& W, int B, int T,
                           const Epi& e) {
    memset(&p, 0, sizeof(p));
    const int D = c.embed_dim, G = c.pos_conv_groups, cpg = D / G, Kq = pos_taps4(c) / 4, bn = 4 * cpg;
    S3B_OK(gemm_tmaps(p, 0, x, 0, D, T, B, D, (uint64_t)T * D, 128, W, 4 * D, Kq * 64, bn));
    p.batches = B, p.rows_per_batch = T + 3, p.tiles_m_per_batch = (T + 3 + 127) / 128;
    p.n_tiles = G, p.bn = bn, p.num_k_blocks = Kq, p.kb_per_row = 1;
    p.a_row_step = 4, p.a_row_off = -(pos_taps(c) / 2), p.a_k_per_ntile = cpg;
    p.out_rows_per_batch = T + 3;
    p.k_steps = (cpg + 15) / 16;  // 24, 40 or 48 channels per group: the box's last k-steps hold zero weights
    p.alg_flops = 2.0 * (double)B * T * D * cpg * pos_taps(c);
    set_epi(p, e, 4 * D);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// launch accounting / profiling
// ------------------------------------------------------------------------------------------------
// (m == nullptr: a building-block entry point, nothing to account)
static inline void prof_begin(s3b_model* m, cudaStream_t st) {
    if (m == nullptr || !m->prof.on) return;
    m->prof.pending = m->prof.get();
    cudaEventRecord(m->prof.pending.get(), st);
}
static inline void prof_end(s3b_model* m, cudaStream_t st, int cat, int nkernels, double flops) {
    if (m == nullptr) return;
    m->launches_total += nkernels;
    if (!m->prof.on) return;
    Event b = m->prof.get();
    cudaEventRecord(b.get(), st);
    m->prof.recs.push_back({cat, std::move(m->prof.pending), std::move(b)});
    m->prof.launches[cat] += nkernels;
    m->prof.flops[cat] += flops;
}
// One launch `expr` on stream st, accounted to model m as nk kernels of category cat and fl FLOPs
#define KLAUNCH(m, st, cat, nk, fl, expr) \
    do {                                  \
        prof_begin(m, st);                \
        CUDA_OK(expr);                    \
        prof_end(m, st, cat, nk, fl);     \
    } while (0)
#define KNORM(m, st, expr) KLAUNCH(m, st, CAT_NORM, 1, 0.0, expr)
#define KMISC(m, st, expr) KLAUNCH(m, st, CAT_MISC, 1, 0.0, expr)

// The feature extractor's front end (add_conv_frontend, s3b_frontend_f32): B ragged waveforms packed into
// wav_pad [B][Lmax] (+ per-utterance normalisation), then conv 0 (w [512][10]) with GroupNorm(512, 512) over all
// L0 frames (layer_norm 0) or per-frame LayerNorm(512) (layer_norm 1), GELU, written to operand planes `op`.
// Workspaces: wav_stats [B][2], c0_part conv0_ws_part_bytes(B, L0), c0_ss [2][B][512] (GroupNorm only).
static int launch_frontend(s3b_model* m, cudaStream_t st, const float* const* d_wavs, const long long* d_lens, int B,
                           long long Lmax, int L0, int normalize, const float* w, const float* bias, const float* gamma,
                           const float* beta, int layer_norm, float* wav_pad, float* wav_stats, double* c0_part,
                           float* c0_ss, const OutPlanes& op) {
    const double conv0_flops = 2.0 * kConvK[0] * kConvDim * (double)B * L0;
    KMISC(m, st, launch_wav_pack(d_wavs, d_lens, B, Lmax, normalize, wav_stats, wav_pad, st));
    if (layer_norm) {
        KLAUNCH(m, st, CAT_CONV0, 1, conv0_flops, launch_conv0_layernorm(wav_pad, B, Lmax, L0, w, bias, gamma, beta, op, st));
    } else {
        // a conv-0 bias (conv_bias with extractor_mode "default") is removed again by the per-channel GroupNorm
        // mean: it cancels exactly in (z + b) - mean(z + b), so the kernel never adds it
        KLAUNCH(m, st, CAT_CONV0, 3, conv0_flops,
                launch_conv0_groupnorm(wav_pad, B, Lmax, L0, w, gamma, beta, c0_part, c0_ss, op, st));
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// forward (one lane = one utterance micro-batch) as an ordered list of steps
// ------------------------------------------------------------------------------------------------
// layer_done: optional callback fired (host side) right after hidden state `l` has been enqueued completely
typedef int (*LayerDoneFn)(s3b_model*, int l, cudaStream_t st, void* user);

// What a lane's plan is built for: the model, the lane's workspace, the shape and what follows from it, and the
// device addresses of the bookkeeping block. Steps capture these by value.
struct Lane {
    s3b_model* m = nullptr;
    Workspace* w = nullptr;
    int B = 0;
    int64_t Lmax = 0;
    int64_t L[kNumConv];
    int T = 0;
    int64_t M = 0;
    // the encoder's attention batch: SB sequences of ST tokens, M = SB * ST rows. B and T for every model but SSAST,
    // whose sequences are the B * nseg windows of 2 + P tokens (T is then its output frames).
    int SB = 0, ST = 0;
    const float** d_wavs = nullptr;
    long long* d_lens = nullptr;
    int* d_kv = nullptr;
    int* d_ord = nullptr;  // APC / DeCoAR: utterances longest first (the recurrence kernels' grouping)
    uint8_t* d_mask = nullptr;
    // a [M][N] linear of the model's operand scheme, tiled for its device
    int linear(GemmParams& p, const SplitBuf& A, const SplitBuf& W, int N, int K, const Epi& e, int64_t lda = 0,
               size_t a_off = 0) const {
        return linear_params(p, A, W, M, N, K, m->scheme, m->sm_count, e, lda, a_off);
    }
};

// One forward call of one lane: the Lane, and what may change from call to call
struct Fwd : Lane {
    cudaStream_t st = nullptr;
    const float* const* wavs = nullptr;  // host array of device pointers (this lane's utterances)
    const int64_t* lens = nullptr;
    float* hidden = nullptr;   // this lane's first utterance inside hidden state 0
    size_t layer_stride = 0;   // elements between consecutive hidden states
    float* ffn_out = nullptr;  // optional: fc2 output (+bias) before the residual add, [NL][...] like hidden
    size_t ffn_stride = 0;
    float* last_res = nullptr;  // optional (pre-LN models): un-normalised output of the last layer
    LayerDoneFn layer_done = nullptr;
    void* user = nullptr;
    Plan* plan = nullptr;

    // slot 0 is the post_extract_proj output, padded frames zeroed: the distiller's feat_final, LightHuBERT's features
    bool proj_slot0() const { return m->cfg.family == 3 || m->cfg.proj_hidden0; }
    // Output slot i of the caller's buffer. Hidden state l (the input of layer l / the encoder output) lives in slot l —
    // except where proj_slot0(): the layer-0 input is then not exposed (internal scratch).
    float* slot(int i) const { return hidden + (size_t)i * layer_stride; }
    // post_extract_proj output; a pre-LN Conformer's hidden state 0 is that output itself (no pos_conv)
    float* proj_out() const {
        return (proj_slot0() || (m->cfg.conformer && m->cfg.layer_norm_first)) ? slot(0) : w->x_f32.as<float>();
    }
    // SSAST: the residual stream is internal (hidden states are a fold of it), one buffer that every layer updates
    float* hs(int l) const {
        if (m->kind == kSsastEncoder) return w->x_f32.as<float>();
        return (proj_slot0() && l == 0) ? w->hs0.as<float>() : slot(l);
    }
    // hidden state l has been enqueued completely
    int done(int l) const { return layer_done != nullptr ? layer_done(m, l, st, user) : 0; }
    int prepare();
};

static int build_steps(const Lane& lane, std::vector<Step>& steps);

int Fwd::prepare() {
    const s3b_config& c = m->cfg;
    const int D = c.embed_dim, F = c.ffn_dim, H = c.num_heads, C = kConvDim;
    if (B < 1) return fail("empty batch");
    const bool cpc = m->kind == kCpcStack, ssast = m->kind == kSsastEncoder;
    const bool fb = m->kind != kConvEncoder && !cpc;
    const bool recurrent = m->kind == kGruStack || m->kind == kLstmStack;
    {
        int64_t cur = Lmax;
        for (int i = 0; i < kNumConv; ++i)
            cur = L[i] = fb ? 0 : cpc ? (i < kCpcConvs ? cpc_conv_len(cur, i) : 0) : conv_out_len(cur, i);
    }
    const int64_t T64 = model_frames(m, Lmax);
    if (T64 < 1) return fail_too_short(m, Lmax);
    if ((int64_t)B * (fb ? fbank_frames(Lmax) : L[0]) > 2000000000LL) return fail("batch too large for 32-bit tile indexing");
    T = (int)T64;
    SB = B, ST = T;
    if (ssast) {
        const SsastGeom g = ssast_geom(m->ssast);
        SB = (int)(B * ssast_segments(g, Lmax)), ST = g.P + 2;
    }
    M = (int64_t)SB * ST;
    const int STp = (ST + 7) & ~7;
    if (layer_stride == 0) layer_stride = (size_t)B * T * D * (ssast ? ssast_geom(m->ssast).patch_f : 1);
    if (ffn_out != nullptr && ffn_stride == 0) ffn_stride = (size_t)M * D;
    if (c.relative_position && T > m->rel_table_T) S3B_OK(build_rel_table(m, 2 * T));
    if (c.conformer && T > m->rope_T) S3B_OK(build_rope_table(m, 2 * T));

    // ---- bookkeeping block: pinned host mirror -> one async copy ---------------------------------------------
    const size_t off_lens = (size_t)B * sizeof(void*);
    const size_t off_kv = off_lens + (size_t)B * sizeof(long long);
    const size_t off_ord = off_kv + (size_t)SB * sizeof(int);  // kv: the attention's valid keys per sequence
    const size_t off_mask = (off_ord + (recurrent ? (size_t)B * sizeof(int) : 0) + 15) & ~(size_t)15;
    const size_t book_bytes = off_mask + (size_t)M;
    S3B_OK(w->book.ensure(book_bytes));
    if (w->book_host_bytes < book_bytes) {
        if (w->book_copied) CUDA_OK(cudaEventSynchronize(w->book_copied.get()));
        w->book_host.reset(), w->book_host_bytes = 0;
        const size_t cap = book_bytes * 2 + 4096;
        void* hp = nullptr;
        CUDA_OK(cudaHostAlloc(&hp, cap, cudaHostAllocDefault));
        w->book_host.reset(static_cast<char*>(hp));
        w->book_host_bytes = cap, w->book_valid = 0;
    }
    S3B_OK(ensure_event(w->book_copied));
    {
        // build the block in a scratch vector first: when nothing changed since the last call (fixed-shape serving
        // loops, the bench) the mirror is left alone and the host never waits for the previous copy to be consumed
        static thread_local std::vector<char> scratch;
        scratch.assign(book_bytes, 0);
        char* hb = scratch.data();
        memcpy(hb, wavs, (size_t)B * sizeof(void*));
        long long* hl = reinterpret_cast<long long*>(hb + off_lens);
        int* hk = reinterpret_cast<int*>(hb + off_kv);
        uint8_t* hm = reinterpret_cast<uint8_t*>(hb + off_mask);
        S3B_OK(s3b_valid_frames(m, lens, B, Lmax, hk));
        for (int b = 0; b < B; ++b) hl[b] = (long long)lens[b];
        for (int b = 0; b < B; ++b)
            for (int t = hk[b]; t < T; ++t) hm[(size_t)b * T + t] = 1;
        if (ssast)  // no key mask: every token of a window attends to all 2 + P tokens of its window
            for (int i = 0; i < SB; ++i) hk[i] = ST;
        if (recurrent) {  // group utterances of similar length: a recurrence group stops at its own longest
            int* ho = reinterpret_cast<int*>(hb + off_ord);
            std::vector<int> ord(B);
            for (int b = 0; b < B; ++b) ord[b] = b;
            std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return hk[a] > hk[b]; });
            memcpy(ho, ord.data(), (size_t)B * sizeof(int));
        }
        if (w->book_valid != book_bytes || memcmp(w->book_host.get(), hb, book_bytes) != 0) {
            CUDA_OK(cudaEventSynchronize(w->book_copied.get()));  // normally long complete
            memcpy(w->book_host.get(), hb, book_bytes);
            w->book_valid = book_bytes;
        }
    }
    char* db = w->book.as<char>();
    d_wavs = reinterpret_cast<const float**>(db);
    d_lens = reinterpret_cast<long long*>(db + off_lens);
    d_kv = reinterpret_cast<int*>(db + off_kv);
    d_ord = reinterpret_cast<int*>(db + off_ord);
    d_mask = reinterpret_cast<uint8_t*>(db + off_mask);

    // ---- workspace ------------------------------------------------------------------------------------------
    if (ssast) {
        // the windows' features, then the patch GEMM's operand planes
        const SsastGeom g = ssast_geom(m->ssast);
        S3B_OK(w->fb_f32.ensure((size_t)SB * g.TL * 128 * 4));
        S3B_OK(w->ln512_s.ensure(m->ssast.patch ? (size_t)SB * g.P * 256 : (size_t)SB * g.TL * 128));
    } else if (cpc) {
        // conv i's input (i = 1..4) in its padded layout act[i - 1], conv i's fp32 output, the LSTM's operand planes
        // (encoder output, then each layer's), the input GEMM's output
        S3B_OK(w->wav_pad.ensure((size_t)B * Lmax * 4));
        for (int i = 1; i < kCpcConvs; ++i) S3B_OK(w->act[i - 1].ensure((size_t)B * cpc_rows(L[i], i) * kCpcDim));
        S3B_OK(w->conv_f32.ensure((size_t)B * L[1] * kCpcDim * 4));
        S3B_OK(w->x_s.ensure((size_t)M * kCpcDim));
        S3B_OK(w->xg_f32.ensure((size_t)M * 4 * kCpcDim * 4));
    } else if (fb) {
        S3B_OK(w->fb_f32.ensure((size_t)B * fbank_frames(Lmax) * 80 * 4));
        // the CMVN kernel's planes: the A operand of post_extract_proj (APC: of layer 0's input GEMM)
        S3B_OK(w->ln512_s.ensure((size_t)M * kDecoar2K));
    } else {
        S3B_OK(w->wav_pad.ensure((size_t)B * Lmax * 4));
        S3B_OK(w->wav_stats.ensure((size_t)B * 2 * 4));
        S3B_OK(w->c0_part.ensure(conv0_ws_part_bytes(B, (int)L[0])));
        S3B_OK(w->c0_ss.ensure((size_t)2 * B * C * 4));
        for (int i = 0; i < kNumConv - 1; ++i) S3B_OK(w->act[i].ensure((size_t)B * L[i] * C));
        S3B_OK(w->conv_f32.ensure((size_t)B * (c.extractor_layer_norm ? L[1] : L[6]) * C * 4));
        S3B_OK(w->ln512_s.ensure((size_t)M * C));
    }
    if (m->kind == kGruStack) {
        S3B_OK(w->x_s.ensure((size_t)M * D));  // layers 1..: the recurrence kernel's planes
        S3B_OK(w->xg_f32.ensure((size_t)M * 3 * D * 4));
    } else if (m->kind == kNpcStack) {
        S3B_OK(w->x_s.ensure((size_t)M * D));  // a block's output: the next block's and its masked conv's operand
        S3B_OK(w->h_s.ensure((size_t)M * D));  // a block's conv output: its linear's operand
    } else if (m->kind == kLstmStack) {
        const int H = kLstmHidden;
        S3B_OK(w->x_s.ensure((size_t)M * H));      // layer 0's operand: post_extract_proj's output
        S3B_OK(w->h_s.ensure((size_t)M * 2 * H));  // layers 1..: the previous layer's [M][2H] output
        S3B_OK(w->xg_f32.ensure((size_t)M * 4 * H * 4));
        S3B_OK(w->lstm_h.ensure(lstm_hbuf_floats(B) * 4));
        S3B_OK(w->lstm_sync.ensure(sizeof(unsigned int)));
    } else if (!cpc) {  // the encoder's buffers
        S3B_OK(w->tmp_f32.ensure((size_t)M * D * 4));
        S3B_OK(w->x_f32.ensure((size_t)M * D * 4));
        S3B_OK(w->x1_f32.ensure((size_t)M * D * 4));
        S3B_OK(w->x_s.ensure((size_t)M * D));
        S3B_OK(w->xs_s.ensure((size_t)M * D));
        S3B_OK(w->x1_s.ensure((size_t)M * D));
        S3B_OK(w->ctx_s.ensure((size_t)M * D));
        S3B_OK(w->q_s.ensure((size_t)M * D));
        S3B_OK(w->k_s.ensure((size_t)M * D));
        S3B_OK(w->vt_s.ensure((size_t)D * SB * STp));
        S3B_OK(w->h_s.ensure((size_t)M * F));
        if (c.conformer) S3B_OK(w->glu_f32.ensure((size_t)M * 2 * D * sizeof(float)));
        else if (!ssast && posconv4_ok(c)) S3B_OK(w->pos_z.ensure((size_t)B * (T + 3) * 4 * D * sizeof(float)));
        if (c.relative_position) S3B_OK(w->gate.ensure((size_t)B * H * T * 4));
        if (c.family == 3 || c.proj_hidden0) S3B_OK(w->hs0.ensure((size_t)M * D * 4));
    }

    // ---- launch plan (cached per (B, Lmax) while no buffer has been reallocated) --------------------------------
    plan = nullptr;
    for (size_t i = 0; i < w->plans.size(); ++i) {
        const Plan& pl = *w->plans[i];
        if (pl.B == B && pl.Lmax == Lmax && pl.gen == g_alloc_generation) {
            std::rotate(w->plans.begin(), w->plans.begin() + i, w->plans.begin() + i + 1);  // to the front
            plan = w->plans.front().get();
            break;
        }
    }
    if (plan == nullptr) {
        std::unique_ptr<Plan> pl(new Plan());
        S3B_OK(build_steps(*this, pl->steps));
        pl->B = B, pl->Lmax = Lmax, pl->gen = g_alloc_generation;
        w->plans.insert(w->plans.begin(), std::move(pl));
        if (w->plans.size() > 4) w->plans.pop_back();
        plan = w->plans.front().get();
    }
    return 0;
}

// The attention kernel's view of q / k / v^T planes as the QKV scatter writes them (q, k [B*H][T][hd], v^T
// [B*H][hd][Tp]): Q and K rows as 64-wide boxes, the last one reading past hd into TMA zero fill.
static int attn_tmaps(AttnParams& ap, const SplitBuf& q, const SplitBuf& k, const SplitBuf& vt, int B, int T, int H,
                      int hd) {
    const uint64_t BH = (uint64_t)B * H;
    const int Tp = (T + 7) & ~7;
    TMAP_OK(encode_tmap_bf16_3d(&ap.q_hi, q.h(), hd, T, BH, hd, (uint64_t)T * hd, 64, 128));
    TMAP_OK(encode_tmap_bf16_3d(&ap.q_lo, q.l(), hd, T, BH, hd, (uint64_t)T * hd, 64, 128));
    TMAP_OK(encode_tmap_bf16_3d(&ap.k_hi, k.h(), hd, T, BH, hd, (uint64_t)T * hd, 64, 64));
    TMAP_OK(encode_tmap_bf16_3d(&ap.k_lo, k.l(), hd, T, BH, hd, (uint64_t)T * hd, 64, 64));
    TMAP_OK(encode_tmap_bf16_3d(&ap.vt_hi, vt.h(), T, hd, BH, Tp, (uint64_t)hd * Tp, 64, hd));
    TMAP_OK(encode_tmap_bf16_3d(&ap.vt_lo, vt.l(), T, hd, BH, Tp, (uint64_t)hd * Tp, 64, hd));
    ap.B = B, ap.H = H, ap.T = T, ap.D = H * hd, ap.hd = hd;
    return 0;
}

// the attention kernel's view of a lane's q / k / v^T planes (QKV scatter epilogue) and its context output
static int attn_params(AttnParams& ap, const Workspace* w, int B, int T, int H, int hd, const int* d_kv, int scheme) {
    memset(&ap, 0, sizeof(ap));
    S3B_OK(attn_tmaps(ap, w->q_s, w->k_s, w->vt_s, B, T, H, hd));
    ap.kv_len = d_kv;
    ap.ctx = w->ctx_s.planes(scheme);
    return 0;
}

// one GEMM of a step on the call's stream
static int run_gemm(const Fwd& f, const GemmParams& p) {
    KLAUNCH(f.m, f.st, CAT_GEMM, 1, p.alg_flops, launch_gemm(p, f.m->sm_count, f.st));
    return 0;
}

// the bookkeeping block prepare() left in the pinned mirror, copied ahead of everything else on the lane's stream
static int copy_book(const Lane& lane, cudaStream_t st) {
    Workspace* w = lane.w;
    const size_t book_bytes = (size_t)(reinterpret_cast<char*>(lane.d_mask) - w->book.as<char>()) + (size_t)lane.M;
    CUDA_OK(cudaMemcpyAsync(w->book.p, w->book_host.get(), book_bytes, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaEventRecord(w->book_copied.get(), st));
    return 0;
}

// ConvFeatureExtractionModel.forward: waveform packing (+ normalisation) and conv 0 + norm + GELU -> act[0], then conv
// 1..6 as implicit GEMMs (+ per-frame LayerNorm + GELU in "layer_norm" mode), one step each
static int add_conv_frontend(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const s3b_config& c = m->cfg;
    const int B = lane.B, C = kConvDim, sch = m->scheme;
    steps.push_back([=](Fwd& f) {
        S3B_OK(copy_book(lane, f.st));
        return launch_frontend(m, f.st, lane.d_wavs, lane.d_lens, B, lane.Lmax, (int)lane.L[0], m->cfg.normalize_wav,
                               m->conv0_w.as<float>(), m->cfg.conv_bias ? m->conv0_b.as<float>() : nullptr,
                               m->norm0_g.as<float>(), m->norm0_b.as<float>(), m->cfg.extractor_layer_norm,
                               w->wav_pad.as<float>(), w->wav_stats.as<float>(), w->c0_part.as<double>(),
                               w->c0_ss.as<float>(), w->act[0].planes(sch));
    });
    const bool ln = c.extractor_layer_norm != 0;
    for (int i = 1; i < kNumConv; ++i) {
        const bool last = i == kNumConv - 1;
        const float* bias = c.conv_bias ? m->conv_b[i].as<float>() : nullptr;
        Epi e = epi_f32(w->conv_f32.as<float>(), bias);  // "layer_norm" mode: the LayerNorm kernel adds the GELU
        if (!ln) {
            if (!last) e = epi_planes(w->act[i].planes(sch), bias, 1);
            else if (c.no_feature_layer_norm) e = epi_planes(w->ln512_s.planes(sch), bias, 1);  // into post_extract_proj
            else e.gelu = 1;
        }
        GemmParams p;
        S3B_OK(conv_params(p, w->act[i - 1], m->conv_w[i], B, lane.L[i - 1], lane.L[i], 2, C, C, C, kConvK[i], 0, sch, e));
        const size_t rows = (size_t)B * lane.L[i];
        steps.push_back([=](Fwd& f) {
            S3B_OK(run_gemm(f, p));
            if (ln)
                KNORM(m, f.st, launch_layernorm(w->conv_f32.as<float>(), rows, C, m->conv_ln_g[i].as<float>(),
                                                m->conv_ln_b[i].as<float>(), 1, last ? w->conv_f32.as<float>() : nullptr,
                                                last ? no_planes() : w->act[i].planes(sch), f.st));
            return 0;
        });
    }
    return 0;
}

// kaldi fbank frames + CMVN (DeCoAR 2.0: every second frame) into the first GEMM's operand planes (profile category 2)
static int add_fbank_frontend(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const int frame_step = m->kind == kFbankEncoder ? 2 : 1;
    steps.push_back([=](Fwd& f) {
        S3B_OK(copy_book(lane, f.st));
        KLAUNCH(m, f.st, CAT_CONV0, 2, 0.0,
                launch_decoar2_features(lane.d_wavs, lane.d_lens, lane.B, (int)fbank_frames(lane.Lmax), lane.T,
                                        frame_step, w->fb_f32.as<float>(), w->ln512_s.planes(m->scheme), f.st));
        return 0;
    });
    return 0;
}

// LayerNorm(512) -> post_extract_proj, padded frames zeroed (x[padding_mask] = 0, wav2vec2_model.py:3061-3062). The
// distiller's output IS output slot 0, feat_final (zeroed like the reference's in-place x[padding_mask] = 0 on the
// same storage, distiller/module.py:303-304).
static int add_post_extract_proj(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const s3b_config& c = m->cfg;
    const int C = kConvDim, sch = m->scheme;
    const int64_t M = lane.M;
    const bool ln = !c.no_feature_layer_norm && m->kind == kConvEncoder;
    Epi e = epi_f32(nullptr, m->proj_b.as<float>());
    e.row_mask = lane.d_mask;
    if (!c.conformer) e.op = w->x_s.planes(0);  // operand of pos_conv, which stays on the bf16x3 kernel (48-channel groups)
    GemmParams p;
    S3B_OK(lane.linear(p, w->ln512_s, m->proj_w, c.embed_dim, m->kind == kFbankEncoder ? kDecoar2K : C, e));
    steps.push_back([=](Fwd& f) {
        if (ln)
            KNORM(m, f.st, launch_layernorm(w->conv_f32.as<float>(), (size_t)M, C, m->ln512_g.as<float>(),
                                            m->ln512_b.as<float>(), 0, nullptr, w->ln512_s.planes(sch), f.st));
        GemmParams q = p;
        q.out_f32 = f.proj_out();
        S3B_OK(run_gemm(f, q));
        return f.proj_slot0() ? f.done(0) : 0;
    });
    return 0;
}

// x = x + GELU(pos_conv(x)); post-LN models: encoder.layer_norm -> hidden state 0 and layer 0's operand planes
static int add_pos_conv(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const s3b_config& c = m->cfg;
    const int B = lane.B, T = lane.T, D = c.embed_dim, cpg = D / c.pos_conv_groups, sch = m->scheme;
    const int64_t M = lane.M;
    const bool ln = !c.layer_norm_first;
    float* z = w->pos_z.as<float>();
    if (c.pos_conv_depth > 1) {
        // data2vec: x_{i+1} = GELU(LayerNorm_noaffine(conv_i(x_i) + b_i)), x = x + x_depth (wav2vec2_model.py:3000-3019,
        // 3064-3067), every block a four-taps GEMM and the combine kernel, all in one step. Block i reads the operand
        // planes block i-1 wrote: x_s -> x1_s -> ctx_s -> x1_s ... (both are free here). Padded frames are NOT
        // re-zeroed between the blocks (the reference does not either).
        const int depth = c.pos_conv_depth;
        std::vector<const SplitBuf*> x(depth);
        std::vector<GemmParams> conv(depth);
        for (int i = 0; i < depth; ++i) {
            x[i] = i == 0 ? &w->x_s : (i & 1) ? &w->x1_s : &w->ctx_s;
            S3B_OK(posconv4_params(conv[i], c, *x[i], m->posd_w4[i], B, T, epi_f32(z)));
        }
        steps.push_back([=](Fwd& f) {
            for (int i = 0; i < depth; ++i) {
                const bool last = (i == depth - 1);
                S3B_OK(run_gemm(f, conv[i]));
                KNORM(m, f.st, launch_posconv_combine(z, last ? f.proj_out() : nullptr, m->posd_b[i].as<float>(), B, T,
                                                      D, cpg, m->enc_ln_g.as<float>(), m->enc_ln_b.as<float>(),
                                                      last && ln ? 1 : 0, last ? 2 : 1, last ? f.hs(0) : nullptr,
                                                      last ? (ln ? w->xs_s.planes(sch) : no_planes()) : x[i + 1]->planes(0),
                                                      f.st));
            }
            return f.proj_slot0() ? 0 : f.done(0);
        });
    } else if (posconv4_ok(c)) {
        // four taps per k-block into pos_z, then the combine kernel (+ LayerNorm)
        GemmParams p;
        S3B_OK(posconv4_params(p, c, w->x_s, m->pos_w4, B, T, epi_f32(z)));
        steps.push_back([=](Fwd& f) {
            S3B_OK(run_gemm(f, p));
            KNORM(m, f.st, launch_posconv_combine(z, f.proj_out(), m->pos_b.as<float>(), B, T, D, cpg,
                                                  m->enc_ln_g.as<float>(), m->enc_ln_b.as<float>(), ln ? 1 : 0, 0,
                                                  f.hs(0), ln ? w->xs_s.planes(sch) : no_planes(), f.st));
            return f.proj_slot0() ? 0 : f.done(0);
        });
    } else {
        // one tap per k-block: x + GELU(conv + bias) in the epilogue (pre-LN: straight into hidden state 0), then the
        // LayerNorm
        Epi e = epi_f32(w->tmp_f32.as<float>(), m->pos_b.as<float>());
        e.gelu = 1;
        GemmParams p;
        S3B_OK(posconv_params(p, c, w->x_s, m->pos_w, B, T, e));
        steps.push_back([=](Fwd& f) {
            GemmParams q = p;
            q.residual = f.proj_out();
            if (!ln) q.out_f32 = f.hs(0);
            S3B_OK(run_gemm(f, q));
            if (ln)
                KNORM(m, f.st, launch_layernorm(w->tmp_f32.as<float>(), (size_t)M, D, m->enc_ln_g.as<float>(),
                                                m->enc_ln_b.as<float>(), 0, f.hs(0), w->xs_s.planes(sch), f.st));
            return f.proj_slot0() ? 0 : f.done(0);
        });
    }
    return 0;
}

// TransformerSentenceEncoderLayer.forward (wav2vec2_model.py:3260-3322; WavLM.py:709-774) in five steps
static int add_transformer_layer(const Lane& lane, int l, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const s3b_config& c = m->cfg;
    const int B = lane.SB, T = lane.ST, D = c.embed_dim, F = c.ffn_dim, H = c.num_heads, hd = head_dim(c);
    const int sch = m->scheme;
    const size_t M = (size_t)lane.M;
    const LayerW* W = &m->layers[l];
    const bool pre = c.layer_norm_first != 0, rel = c.relative_position != 0, gru_rel = c.gru_rel_pos != 0;
    const bool last = l == c.num_layers - 1, heads = c.pred_heads > 0;
    // SSAST's encoder has no final norm on its outputs, and its hidden states are written by the fold step after the layer
    const bool ssast = m->kind == kSsastEncoder, enc_ln = pre && last && !ssast;
    const float eps = m->ln_eps;
    const double attn_flops = 4.0 * (double)T * T * D * B;
    float* x1 = w->x1_f32.as<float>();
    float* tmp = w->tmp_f32.as<float>();
    GemmParams qkv, out, fc1, fc2;
    AttnParams attn;
    S3B_OK(lane.linear(qkv, w->xs_s, W->qkv, 3 * D, D, Epi()));
    set_qkv_epi(qkv, W->qkv_b.as<float>(), T, H, hd, w->q_s, w->k_s, w->vt_s);
    S3B_OK(attn_params(attn, w, B, T, H, hd, lane.d_kv, sch));
    if (rel) set_rel_bias(attn, m->rel_table.as<float>(), m->rel_table_T, w->gate.as<float>());
    S3B_OK(lane.linear(out, w->ctx_s, W->out, D, D, epi_f32(pre ? x1 : tmp, W->out_b.as<float>())));
    S3B_OK(lane.linear(fc1, w->x1_s, W->fc1, F, D, epi_planes(w->h_s.planes(sch), W->fc1_b.as<float>(), 1)));
    S3B_OK(lane.linear(fc2, w->h_s, W->fc2, D, F, epi_f32(tmp, W->fc2_b.as<float>(), x1)));
    // pre-LN: xs = LN1(hidden state l); QKV projection, scattered per head; WavLM: the gate from the layer's attention
    // input (post-LN: hidden state l; pre-LN: the LN1 output), modules.py:534-551
    steps.push_back([=](Fwd& f) {
        if (pre)
            KNORM(m, f.st, launch_layernorm(f.hs(l), M, D, W->ln1_g.as<float>(), W->ln1_b.as<float>(), 0, nullptr,
                                            w->xs_s.planes(sch), f.st, eps));
        S3B_OK(run_gemm(f, qkv));
        if (rel)
            KMISC(m, f.st, launch_wavlm_gate(w->xs_s.planes(sch), M, B, T, H, D, gru_rel ? W->grep_w.as<float>() : nullptr,
                                             W->grep_b.as<float>(), W->grep_a.as<float>(), w->gate.as<float>(), f.st));
        return 0;
    });
    steps.push_back([=](Fwd& f) {
        KLAUNCH(m, f.st, CAT_ATTN, 1, attn_flops, launch_attention(attn, f.st));
        return 0;
    });
    // r1 = hidden state l + out_proj(ctx); pre-LN: x1_s = LN2(r1); post-LN: x1 = LN1(r1)
    steps.push_back([=](Fwd& f) {
        GemmParams p = out;
        p.residual = f.hs(l);
        S3B_OK(run_gemm(f, p));
        if (pre)
            KNORM(m, f.st, launch_layernorm(x1, M, D, W->ln2_g.as<float>(), W->ln2_b.as<float>(), 0, nullptr,
                                            w->x1_s.planes(sch), f.st, eps));
        else
            KNORM(m, f.st, launch_layernorm(tmp, M, D, W->ln1_g.as<float>(), W->ln1_b.as<float>(), 0, x1,
                                            w->x1_s.planes(sch), f.st));
        return 0;
    });
    steps.push_back([=](Fwd& f) { return run_gemm(f, fc1); });
    // fc2 + residual; the next layer's (or the prediction heads') operand planes
    steps.push_back([=](Fwd& f) {
        GemmParams p = fc2;
        // pre-LN: the sum IS hidden state l+1 (un-normalised residual stream), except after the last layer
        float* unnorm = (last && f.last_res != nullptr) ? f.last_res : tmp;
        if (pre) p.out_f32 = enc_ln ? unnorm : f.hs(l + 1);
        if (f.ffn_out != nullptr) p.out_pre = f.ffn_out + (size_t)l * f.ffn_stride;
        S3B_OK(run_gemm(f, p));
        if (pre) {
            if (enc_ln)  // encoder.layer_norm on the final output (wav2vec2_model.py:3049-3050)
                KNORM(m, f.st, launch_layernorm(unnorm, M, D, m->enc_ln_g.as<float>(), m->enc_ln_b.as<float>(), 0,
                                                f.hs(l + 1), heads ? w->xs_s.planes(sch) : no_planes(), f.st));
        } else {
            KNORM(m, f.st, launch_layernorm(tmp, M, D, W->ln2_g.as<float>(), W->ln2_b.as<float>(), 0, f.hs(l + 1),
                                            !last || heads ? w->xs_s.planes(sch) : no_planes(), f.st));
        }
        return ssast ? 0 : f.done(l + 1);
    });
    return 0;
}

// Distiller output layer on the encoder output (operand planes xs_s): Linear(D, N*D) + GELU -> h_s, then one [D][D]
// GEMM per task on its D-column slice of h_s into output slot NL + 1 + k (SplitLinear, distiller/module.py:77-90)
static int add_pred_heads(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const int D = m->cfg.embed_dim, N = m->cfg.pred_heads, NL = m->cfg.num_layers;
    GemmParams p1;
    S3B_OK(lane.linear(p1, w->xs_s, m->pred1_w, N * D, D, epi_planes(w->h_s.planes(m->scheme), m->pred1_b.as<float>(), 1)));
    steps.push_back([=](Fwd& f) { return run_gemm(f, p1); });
    for (int k = 0; k < N; ++k) {
        GemmParams p;
        S3B_OK(lane.linear(p, w->h_s, m->pred2_w[k], D, D, epi_f32(nullptr, m->pred2_b.as<float>() + (size_t)k * D),
                           (int64_t)N * D, (size_t)k * D));
        steps.push_back([=](Fwd& f) {
            GemmParams q = p;
            q.out_f32 = f.slot(NL + 1 + k);
            S3B_OK(run_gemm(f, q));
            return f.done(NL + 1 + k);
        });
    }
    return 0;
}

// ConformerEncoder before its layers: no pos_conv; post-LN models: encoder.layer_norm -> hidden state 0
// (wav2vec2_model.py:3183-3184)
static int add_conformer_input(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    float* x = lane.w->x_f32.as<float>();
    const bool ln = !m->cfg.layer_norm_first;
    const size_t M = (size_t)lane.M;
    const int D = m->cfg.embed_dim;
    steps.push_back([=](Fwd& f) {
        if (ln)
            KNORM(m, f.st, launch_layernorm(x, M, D, m->enc_ln_g.as<float>(), m->enc_ln_b.as<float>(), 0, f.hs(0),
                                            no_planes(), f.st));
        return f.done(0);
    });
    return 0;
}

// One Conformer layer (wav2vec2_model.py:537-578) in ten steps, nine GEMMs. Residual stream: hidden state l -> r1
// (x1_f32, after ffn1) -> r2 (x_f32, after attention) -> r3 (x1_f32, after the conv module) -> r4 (tmp_f32, after
// ffn2) -> final_layer_norm -> hidden state l+1. Operand planes: xs_s = LayerNorm outputs, x1_s = rope(LN) / depthwise
// output.
static int add_conformer_layer(const Lane& lane, int l, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const s3b_config& c = m->cfg;
    const int B = lane.B, T = lane.T, D = c.embed_dim, F = c.ffn_dim, H = c.num_heads, kw = c.depthwise_kernel;
    const int sch = m->scheme;
    const size_t M = (size_t)lane.M;
    const LayerW* W = &m->layers[l];
    const double attn_flops = 4.0 * (double)T * T * D * B;
    const OutPlanes xs = w->xs_s.planes(sch), x1s = w->x1_s.planes(sch), hs = w->h_s.planes(sch);
    float* r13 = w->x1_f32.as<float>();
    float* r2 = w->x_f32.as<float>();
    float* r4 = w->tmp_f32.as<float>();
    GemmParams ffn1_a, ffn1_b, qk, v, out, pw1, pw2, fc1, fc2;
    AttnParams attn;
    S3B_OK(lane.linear(ffn1_a, w->xs_s, W->ffn1_w1, F, D, epi_planes(hs, W->ffn1_b1.as<float>(), 2)));
    S3B_OK(lane.linear(ffn1_b, w->h_s, W->ffn1_w2, D, F, epi_f32(r13, W->ffn1_b2.as<float>())));
    S3B_OK(lane.linear(qk, w->x1_s, W->qkv, 2 * D, D, Epi()));
    set_qkv_epi(qk, W->qkv_b.as<float>(), T, H, 64, w->q_s, w->k_s, w->vt_s, 0);
    S3B_OK(lane.linear(v, w->xs_s, W->v, D, D, Epi()));
    set_qkv_epi(v, W->qkv_b.as<float>() + 2 * D, T, H, 64, w->q_s, w->k_s, w->vt_s, 2 * D);
    S3B_OK(attn_params(attn, w, B, T, H, 64, lane.d_kv, sch));
    S3B_OK(lane.linear(out, w->ctx_s, W->out, D, D, epi_f32(r2, W->out_b.as<float>(), r13)));
    S3B_OK(lane.linear(pw1, w->xs_s, W->pw1, 2 * D, D, epi_f32(w->glu_f32.as<float>())));
    S3B_OK(lane.linear(pw2, w->x1_s, W->pw2, D, D, epi_f32(r13, nullptr, r2)));
    S3B_OK(lane.linear(fc1, w->xs_s, W->fc1, F, D, epi_planes(hs, W->fc1_b.as<float>(), 2)));
    S3B_OK(lane.linear(fc2, w->h_s, W->fc2, D, F, epi_f32(r4, W->fc2_b.as<float>(), r13)));
    // ffn1: LayerNorm -> w_1 + SiLU
    steps.push_back([=](Fwd& f) {
        KNORM(m, f.st, launch_layernorm(f.hs(l), M, D, W->ffn1_ln_g.as<float>(), W->ffn1_ln_b.as<float>(), 0, nullptr,
                                        xs, f.st));
        return run_gemm(f, ffn1_a);
    });
    // r1 = x + 0.5 w_2(...) (0.5 folded into w_2)
    steps.push_back([=](Fwd& f) {
        GemmParams p = ffn1_b;
        p.residual = f.hs(l);
        return run_gemm(f, p);
    });
    // self_attn_layer_norm + RoPE -> [q | k] from rope(LN(r1)), v from LN(r1)
    steps.push_back([=](Fwd& f) {
        KNORM(m, f.st, launch_layernorm_rope(r13, M, T, D, W->ln1_g.as<float>(), W->ln1_b.as<float>(),
                                             m->rope_cs.as<float>(), xs, x1s, f.st));
        S3B_OK(run_gemm(f, qk));
        return run_gemm(f, v);
    });
    steps.push_back([=](Fwd& f) {
        KLAUNCH(m, f.st, CAT_ATTN, 1, attn_flops, launch_attention(attn, f.st));
        return 0;
    });
    // r2 = r1 + linear_out
    steps.push_back([=](Fwd& f) { return run_gemm(f, out); });
    // conv_module: LayerNorm -> pointwise_conv1 (no bias) -> fp32 [M][2D]
    steps.push_back([=](Fwd& f) {
        KNORM(m, f.st, launch_layernorm(r2, M, D, W->conv_ln_g.as<float>(), W->conv_ln_b.as<float>(), 0, nullptr, xs,
                                        f.st));
        return run_gemm(f, pw1);
    });
    // GLU -> depthwise conv -> BatchNorm -> SiLU
    steps.push_back([=](Fwd& f) {
        KMISC(m, f.st, launch_depthwise_glu(w->glu_f32.as<float>(), B, T, D, kw, W->dw_w.as<float>(),
                                            W->dw_b.as<float>(), x1s, f.st));
        return 0;
    });
    // r3 = r2 + pointwise_conv2 (no bias)
    steps.push_back([=](Fwd& f) { return run_gemm(f, pw2); });
    // ffn2: LayerNorm -> w_1 + SiLU
    steps.push_back([=](Fwd& f) {
        KNORM(m, f.st, launch_layernorm(r13, M, D, W->ffn2_ln_g.as<float>(), W->ffn2_ln_b.as<float>(), 0, nullptr, xs,
                                        f.st));
        return run_gemm(f, fc1);
    });
    // r4 = r3 + 0.5 w_2(...) -> final_layer_norm -> hidden state l+1 (pre-LN: encoder.layer_norm after the last layer,
    // wav2vec2_model.py:3049-3050)
    const bool enc_ln = c.layer_norm_first && l == c.num_layers - 1;
    steps.push_back([=](Fwd& f) {
        S3B_OK(run_gemm(f, fc2));
        KNORM(m, f.st, launch_layernorm(r4, M, D, W->ln2_g.as<float>(), W->ln2_b.as<float>(), 0,
                                        enc_ln ? r4 : f.hs(l + 1), no_planes(), f.st));
        if (enc_ln)
            KNORM(m, f.st, launch_layernorm(r4, M, D, m->enc_ln_g.as<float>(), m->enc_ln_b.as<float>(), 0, f.hs(l + 1),
                                            no_planes(), f.st));
        return f.done(l + 1);
    });
    return 0;
}

// APC: per GRU layer l, the input GEMM x_g = x W_ih^T + (b_ih + [b_hr, b_hz, 0]) over all B * T rows, fp32 [M][3D]
// (the recurrence ignores t >= m_b), then the recurrence, which writes hidden state l (+ layer l's input when
// residual, l > 0) and layer l + 1's operand planes
static int add_gru_stack(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const int D = m->cfg.embed_dim, NL = m->cfg.num_layers;
    const int64_t M = lane.M;
    for (int l = 0; l < NL; ++l) {
        const LayerW& W = m->layers[l];
        GemmParams in;
        S3B_OK(lane.linear(in, l == 0 ? w->ln512_s : w->x_s, W.wih, 3 * D, l == 0 ? kDecoar2K : D,
                           epi_f32(w->xg_f32.as<float>(), W.gru_b.as<float>())));
        steps.push_back([=](Fwd& f) { return run_gemm(f, in); });
        GruParams g;
        g.xg = w->xg_f32.as<float>(), g.whh = W.whh.as<float>(), g.bhn = W.bhn.as<float>();
        g.len = lane.d_kv, g.order = lane.d_ord, g.B = lane.B, g.T = lane.T;
        g.op = l + 1 < NL ? w->x_s.planes(m->scheme) : no_planes();
        const bool residual = m->apc_residual && l > 0;
        steps.push_back([=](Fwd& f) {
            GruParams q = g;
            q.res = residual ? f.slot(l - 1) : nullptr;
            q.out = f.slot(l);
            KLAUNCH(m, f.st, CAT_GRU, 1, 2.0 * 3 * D * D * (double)M, launch_gru(q, f.st));
            return f.done(l);
        });
    }
    return 0;
}

// DeCoAR: post_extract_proj [M][80 -> 128] x [1024][128]^T + b into layer 0's operand planes; then per layer l and
// direction d (0 forward, 1 backward) the input GEMM x_g = x W_ih^T + (b_ih + b_hh), fp32 [M][4H], and the recurrence,
// which writes columns [d H, d H + H) of layer l's [B][T][2H] output: an output slot (decoar_layers: every layer;
// decoar: the last) and, below the last layer, the operand planes of layer l + 1's GEMMs, which read their direction's
// half (row stride 2H). The two directions never run concurrently: each recurrence occupies the whole device.
static int add_lstm_stack(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const int NL = m->cfg.num_layers, H = kLstmHidden, B = lane.B, sch = m->scheme;
    const int64_t M = lane.M;
    const bool all_layers = m->decoar_all_layers != 0;
    GemmParams proj;
    S3B_OK(lane.linear(proj, w->ln512_s, m->proj_w, H, kDecoar2K, epi_planes(w->x_s.planes(sch), m->proj_b.as<float>())));
    steps.push_back([=](Fwd& f) { return run_gemm(f, proj); });
    for (int l = 0; l < NL; ++l) {
        const bool last = l == NL - 1;
        for (int d = 0; d < 2; ++d) {
            const LayerW& W = m->layers[2 * l + d];
            GemmParams in;
            S3B_OK(lane.linear(in, l == 0 ? w->x_s : w->h_s, W.wih, 4 * H, H,
                               epi_f32(w->xg_f32.as<float>(), W.gru_b.as<float>()), l == 0 ? 0 : 2 * H,
                               l == 0 ? 0 : (size_t)d * H));
            steps.push_back([=](Fwd& f) { return run_gemm(f, in); });
            LstmParams g;
            g.xg = w->xg_f32.as<float>(), g.whh = W.whh.as<float>(), g.bhh = nullptr;
            g.len = lane.d_kv, g.order = lane.d_ord, g.B = B, g.T = lane.T, g.direction = d;
            g.out = nullptr, g.ldo = 2 * H, g.col0 = d * H;
            g.op = last ? no_planes() : w->h_s.planes(sch);
            g.hbuf = w->lstm_h.as<float>(), g.counter = w->lstm_sync.as<unsigned int>();
            steps.push_back([=](Fwd& f) {
                LstmParams q = g;
                q.out = all_layers ? f.slot(l) : last ? f.slot(0) : nullptr;
                KLAUNCH(m, f.st, CAT_GRU, (B + kLstmMaxBatch - 1) / kLstmMaxBatch, 8.0 * H * H * (double)M,
                        launch_lstm(q, f.st));
                if (d == 0) return 0;
                return all_layers ? f.done(l) : last ? f.done(0) : 0;
            });
        }
    }
    return 0;
}

// NPC: per block i, the ConvBlock's conv (k = 3) into the linear's operand planes, the linear into hidden state 2i (fp32)
// and the operand planes that block i + 1 and masked conv i read, then masked conv i: tanh(conv + b) is hidden state
// 2i + 1 (out_pre), and that plus the running feat is feat, accumulated in place in the last output slot (the
// epilogue reads each residual element before it writes the same element). No row mask anywhere: frames t >= m_b hold
// the response to the zero features, as in the reference.
static int add_npc_stack(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const s3b_npc_config& c = m->npc;
    const int NB = c.n_blocks, B = lane.B, T = lane.T, sch = m->scheme, H = 512;
    const int act = c.act == 0 ? 3 : 4;  // ReLU or tanh (gemm.cuh)
    for (int i = 0; i < NB; ++i) {
        const LayerW& L = m->layers[i];
        const bool first = i == 0;
        GemmParams conv, lin, mc;
        S3B_OK(conv_params(conv, first ? w->ln512_s : w->x_s, L.fc1, B, T, T, 1, H, first ? 80 : H, first ? kDecoar2K : H,
                           3, 0, sch, epi_planes(w->h_s.planes(sch), L.fc1_b.as<float>(), act)));
        Epi el = epi_f32(nullptr, L.fc2_b.as<float>());
        el.op = w->x_s.planes(sch), el.gelu = act, el.res_first = 1;
        S3B_OK(conv_params(lin, w->h_s, L.fc2, B, T, T, 1, H, H, H, 1, 0, sch, el));
        Epi em = epi_f32(nullptr, L.out_b.as<float>());
        em.gelu = 4;
        S3B_OK(conv_params(mc, w->x_s, L.out, B, T, T, 1, H, H, H, c.kernel_size, npc_mask_width(c, i), sch, em));
        const bool residual = c.residual && !first;
        steps.push_back([=](Fwd& f) { return run_gemm(f, conv); });
        steps.push_back([=](Fwd& f) {
            GemmParams q = lin;
            q.out_f32 = f.slot(2 * i);
            q.residual = residual ? f.slot(2 * i - 2) : nullptr;
            S3B_OK(run_gemm(f, q));
            return f.done(2 * i);
        });
        steps.push_back([=](Fwd& f) {
            GemmParams q = mc;
            q.out_pre = f.slot(2 * i + 1);
            q.out_f32 = f.slot(2 * NB);
            q.residual = first ? nullptr : f.slot(2 * NB);
            S3B_OK(run_gemm(f, q));
            S3B_OK(f.done(2 * i + 1));
            return i == NB - 1 ? f.done(2 * NB) : 0;
        });
    }
    return 0;
}

// Modified CPC (cpc/expert.py, model.py): the padded waveforms into conv 0 + ChannelNorm + ReLU, written straight into
// conv 1's padded operand layout; conv 1..4 as implicit GEMMs (fp32 + bias) each followed by ChannelNorm + ReLU into
// the next conv's padded layout, conv 4's into hidden state 0 and the dense operand planes of the LSTM. Per LSTM layer
// the input GEMM x_g = x W_ih^T + (b_ih + b_hh), fp32 [M][1024], then the recurrence over all T frames of every
// utterance (the reference runs the padded batch unpacked): the last layer writes hidden state 1, the others the next
// layer's operand planes. Frames near and beyond an utterance's end hold the response to the zero samples, as in the
// reference.
static int add_cpc_stack(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const int B = lane.B, T = lane.T, C = kCpcDim, NL = m->cfg.num_layers, sch = m->scheme;
    const int64_t M = lane.M;
    steps.push_back([=](Fwd& f) {
        S3B_OK(copy_book(lane, f.st));
        KMISC(m, f.st, launch_wav_pack(lane.d_wavs, lane.d_lens, B, lane.Lmax, 0, nullptr, w->wav_pad.as<float>(), f.st));
        KLAUNCH(m, f.st, CAT_CONV0, 1, 2.0 * 10 * C * (double)B * lane.L[0],
                launch_cpc_conv0(w->wav_pad.as<float>(), B, lane.Lmax, (int)lane.L[0], m->conv0_w.as<float>(),
                                 m->conv0_b.as<float>(), m->norm0_g.as<float>(), m->norm0_b.as<float>(),
                                 (int)cpc_rows(lane.L[1], 1), kCpcPad[1], w->act[0].planes(sch), f.st));
        return 0;
    });
    for (int i = 1; i < kCpcConvs; ++i) {
        const bool last = i == kCpcConvs - 1;
        GemmParams p;
        S3B_OK(conv_params(p, w->act[i - 1], m->conv_w[i], B, cpc_rows(lane.L[i], i), lane.L[i], kCpcStride[i], C, C, C,
                           2 * kCpcStride[i], 0, sch, epi_f32(w->conv_f32.as<float>(), m->conv_b[i].as<float>())));
        const int Tout = (int)lane.L[i];
        const int R = last ? Tout : (int)cpc_rows(lane.L[i + 1], i + 1), pad = last ? 0 : kCpcPad[i + 1];
        const OutPlanes op = last ? w->x_s.planes(sch) : w->act[i].planes(sch);
        steps.push_back([=](Fwd& f) {
            S3B_OK(run_gemm(f, p));
            KNORM(m, f.st, launch_channelnorm_relu(w->conv_f32.as<float>(), B, Tout, R, pad, m->conv_ln_g[i].as<float>(),
                                                   m->conv_ln_b[i].as<float>(), last ? f.slot(0) : nullptr, op, f.st));
            return last ? f.done(0) : 0;
        });
    }
    for (int l = 0; l < NL; ++l) {
        const bool last = l == NL - 1;
        const LayerW& W = m->layers[l];
        GemmParams in;
        S3B_OK(lane.linear(in, w->x_s, W.wih, 4 * C, C, epi_f32(w->xg_f32.as<float>(), W.gru_b.as<float>())));
        steps.push_back([=](Fwd& f) { return run_gemm(f, in); });
        CpcLstmParams g;
        g.xg = w->xg_f32.as<float>(), g.whh = W.whh.as<float>(), g.B = B, g.T = T;
        g.out = nullptr, g.op = last ? no_planes() : w->x_s.planes(sch);
        steps.push_back([=](Fwd& f) {
            CpcLstmParams q = g;
            if (last) q.out = f.slot(1);
            KLAUNCH(m, f.st, CAT_GRU, 1, 8.0 * C * C * (double)M, launch_cpc_lstm(q, f.st));
            return last ? f.done(1) : 0;
        });
    }
    return 0;
}

// The patch GEMM of SSAST's embedding over the operand planes A (ssast_patches_kernel), its output (+ bias) written
// into rows 2.. of each window's 2 + P rows of x. Frame model: a convolution of 2 taps over the TL feature rows of a
// window (row t reads rows t and t + 1, K = 2 * 128); patch model: a [P][256] x [768][256]^T GEMM per window.
static int ssast_patch_params(GemmParams& p, const SsastGeom& g, const SplitBuf& A, const SplitBuf& W, int SB, int D,
                              int scheme, float* x, const float* bias) {
    const Epi e = epi_f32(x + 2 * (size_t)D, bias);
    if (g.patch_f == 1) S3B_OK(conv_params(p, A, W, SB, g.TL, g.tdim, 1, D, 128, 128, 2, 0, scheme, e));
    else S3B_OK(conv_params(p, A, W, SB, g.P, g.P, 1, D, 256, 256, 1, 0, scheme, e));
    p.out_rows_per_batch = g.P + 2;
    return 0;
}

// SSAST's front end (profile category 2): per window the normalised 128-bin fbank, the patch operand, the patch GEMM
// (category 0) and the token assembly, which leaves layer 0's input in x_f32
static int add_ssast_frontend(const Lane& lane, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const SsastGeom g = ssast_geom(m->ssast);
    const int D = m->cfg.embed_dim, SB = lane.SB, sch = m->scheme;
    const int nseg = SB / lane.B;
    GemmParams p;
    S3B_OK(ssast_patch_params(p, g, w->ln512_s, m->proj_w, SB, D, sch, w->x_f32.as<float>(), m->proj_b.as<float>()));
    steps.push_back([=](Fwd& f) {
        S3B_OK(copy_book(lane, f.st));
        KLAUNCH(m, f.st, CAT_CONV0, 1, 0.0,
                launch_ssast_fbank(lane.d_wavs, lane.d_lens, lane.B, nseg, g.S, g.TL, w->fb_f32.as<float>(), f.st));
        KLAUNCH(m, f.st, CAT_CONV0, 1, 0.0,
                launch_ssast_patches(w->fb_f32.as<float>(), SB, g.TL, g.patch_f, g.tdim, w->ln512_s.planes(sch), f.st));
        S3B_OK(run_gemm(f, p));
        KLAUNCH(m, f.st, CAT_CONV0, 1, 0.0,
                launch_ssast_tokens(w->x_f32.as<float>(), m->cls_tok.as<float>(), m->dist_tok.as<float>(),
                                    m->pos_tab.as<float>(), SB, g.P, D, f.st));
        return 0;
    });
    return 0;
}

// after SSAST layer l: its output, class tokens dropped and frequency patches folded into channels, into hidden state
// l (profile category 4: the only misc kernel of the model)
static int add_ssast_output(const Lane& lane, int l, std::vector<Step>& steps) {
    s3b_model* m = lane.m;
    Workspace* w = lane.w;
    const SsastGeom g = ssast_geom(m->ssast);
    const int B = lane.B, nseg = lane.SB / lane.B, T = lane.T, D = m->cfg.embed_dim;
    steps.push_back([=](Fwd& f) {
        KMISC(m, f.st, launch_ssast_fold(w->x_f32.as<float>(), B, nseg, g.P, g.tdim, g.patch_f, D, T, f.slot(l), f.st));
        return f.done(l);
    });
    return 0;
}

// One lane's forward at the lane's shape, in enqueue order
static int build_steps(const Lane& lane, std::vector<Step>& steps) {
    const s3b_model* m = lane.m;
    const s3b_config& c = m->cfg;
    switch (m->kind) {
    case kGruStack:
        S3B_OK(add_fbank_frontend(lane, steps));
        return add_gru_stack(lane, steps);
    case kLstmStack:
        S3B_OK(add_fbank_frontend(lane, steps));
        return add_lstm_stack(lane, steps);
    case kNpcStack:
        S3B_OK(add_fbank_frontend(lane, steps));
        return add_npc_stack(lane, steps);
    case kCpcStack: return add_cpc_stack(lane, steps);
    case kSsastEncoder:
        S3B_OK(add_ssast_frontend(lane, steps));
        for (int l = 0; l < c.num_layers; ++l) {
            S3B_OK(add_transformer_layer(lane, l, steps));
            S3B_OK(add_ssast_output(lane, l, steps));
        }
        return 0;
    case kFbankEncoder:
        S3B_OK(add_fbank_frontend(lane, steps));
        // six empty steps where the conv stack would be: with two lanes they keep lane 1's steps enqueued next to the
        // same lane-0 steps as in the conv encoder
        for (int i = 1; i < kNumConv; ++i) steps.push_back([](Fwd&) { return 0; });
        break;
    case kConvEncoder: S3B_OK(add_conv_frontend(lane, steps)); break;
    }
    S3B_OK(add_post_extract_proj(lane, steps));
    if (c.conformer) {
        S3B_OK(add_conformer_input(lane, steps));
        for (int l = 0; l < c.num_layers; ++l) S3B_OK(add_conformer_layer(lane, l, steps));
        return 0;
    }
    S3B_OK(add_pos_conv(lane, steps));
    for (int l = 0; l < c.num_layers; ++l) S3B_OK(add_transformer_layer(lane, l, steps));
    if (c.pred_heads > 0) S3B_OK(add_pred_heads(lane, steps));
    return 0;
}

// floats per frame of a hidden state: the encoder width, or SSAST's patch model's 12 frequency patches of it
static int out_width(const s3b_model* m) {
    return m->kind == kSsastEncoder ? ssast_geom(m->ssast).patch_f * m->cfg.embed_dim : m->cfg.embed_dim;
}

// Number of lanes for a batch: S3B_LANES overrides; otherwise two lanes when the batch can be split AND carries at
// least kLaneMinFrames frames (S3B_LANE_MIN_FRAMES overrides). Below that the halves no longer fill the SMs and the
// doubled launch count costs more than the overlap wins.
static constexpr int64_t kLaneMinFrames = S3B_LANE_MIN_FRAMES_DEFAULT;
static int default_lanes(int B, int64_t T) {
    static int env = -2;
    static long long min_frames = -1;
    if (env == -2) {
        const char* e = getenv("S3B_LANES");
        env = e ? atoi(e) : -1;
        const char* f = getenv("S3B_LANE_MIN_FRAMES");
        min_frames = f ? atoll(f) : (long long)kLaneMinFrames;
    }
    if (B < 2) return 1;
    if (env > 0) return env > 2 ? 2 : env;
    return (long long)B * T >= min_frames ? 2 : 1;
}

// Lanes a model can run: two grid-resident LSTM launches must never be in flight at once, so a DeCoAR model runs one
// (its recurrence occupies the whole device)
static int max_lanes(const s3b_model* m) { return m != nullptr && m->kind == kLstmStack ? 1 : 2; }

extern "C" int32_t s3b_default_lanes(const s3b_model* m, int32_t batch, int64_t max_len) {
    const int64_t T = model_frames(m, max_len);
    if (batch < 1 || T < 1) return -1;
    return std::min(default_lanes(batch, T), max_lanes(m));
}

static int forward_lanes(s3b_model* m, const float* const* wavs, const int64_t* lens, int B, int64_t Lmax,
                         float* hidden_out, cudaStream_t st, const s3b_forward_opts* o) {
    const s3b_config& c = m->cfg;
    if (B < 1) return fail("empty batch");
    const int64_t T = model_frames(m, Lmax);
    if (T < 1) return fail_too_short(m, Lmax);
    int lanes = std::min((o && o->lanes > 0) ? (int)o->lanes : default_lanes(B, T), max_lanes(m));
    if (lanes > B) lanes = B;
    const size_t frame = (size_t)T * out_width(m);
    const size_t layer_stride = (o && o->layer_stride > 0) ? (size_t)o->layer_stride : (size_t)B * frame;
    float* ffn_out = o ? o->ffn_out : nullptr;
    const size_t ffn_stride = (o && o->ffn_layer_stride > 0) ? (size_t)o->ffn_layer_stride : (size_t)B * frame;
    float* last_res = o ? o->last_residual : nullptr;

    Fwd f[2];
    int b0 = 0;
    for (int i = 0; i < lanes; ++i) {
        const int nb = (i == 0) ? (B + lanes - 1) / lanes : B - b0;
        f[i].m = m, f[i].w = &m->ws[i], f[i].wavs = wavs + b0, f[i].lens = lens + b0, f[i].B = nb, f[i].Lmax = Lmax;
        f[i].hidden = hidden_out + (size_t)b0 * frame, f[i].layer_stride = layer_stride;
        f[i].ffn_out = ffn_out ? ffn_out + (size_t)b0 * frame : nullptr, f[i].ffn_stride = ffn_stride;
        f[i].last_res = last_res ? last_res + (size_t)b0 * frame : nullptr;
        f[i].st = st;
        b0 += nb;
    }
    // profiling brackets every launch with events: lanes then run one after the other on the caller's stream so that
    // each kernel is timed alone, at its production shape
    const bool concurrent = lanes == 2 && !m->prof.on;
    if (concurrent) {
        Workspace& w1 = m->ws[1];
        S3B_OK(ensure_stream(w1.stream));
        S3B_OK(ensure_event(w1.done));
        S3B_OK(ensure_event(m->fork_event));
        f[1].st = w1.stream.get();
    }
    for (int i = 0; i < lanes; ++i) S3B_OK(f[i].prepare());
    if (concurrent) {
        const std::vector<Step>& s0 = f[0].plan->steps;
        const std::vector<Step>& s1 = f[1].plan->steps;
        if (s0.size() != s1.size()) return fail("internal: the lanes have %zu and %zu steps", s0.size(), s1.size());
        CUDA_OK(cudaEventRecord(m->fork_event.get(), st));
        CUDA_OK(cudaStreamWaitEvent(f[1].st, m->fork_event.get(), 0));
        // lane 1 trails lane 0 by two steps: while one lane runs a GEMM the other tends to be in a different kind
        // of kernel (attention, LayerNorm, another GEMM shape), which is what lets them share the SMs
        for (size_t s = 0; s < s0.size() + 2; ++s) {
            if (s < s0.size()) S3B_OK(s0[s](f[0]));
            if (s >= 2) S3B_OK(s1[s - 2](f[1]));
        }
        CUDA_OK(cudaEventRecord(m->ws[1].done.get(), f[1].st));
        CUDA_OK(cudaStreamWaitEvent(st, m->ws[1].done.get(), 0));
    } else {
        for (int i = 0; i < lanes; ++i)
            for (const Step& step : f[i].plan->steps) S3B_OK(step(f[i]));
    }
    return 0;
}

extern "C" int s3b_forward(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch,
                           int64_t max_len, float* hidden_out, void* stream) {
    if (!m || !wavs || !lens || !hidden_out) return fail("null argument");
    if (!m->finalized) return fail("model not finalized");
    return forward_lanes(m, wavs, lens, batch, max_len, hidden_out, (cudaStream_t)stream, nullptr);
}

extern "C" int s3b_forward_ex(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch,
                              int64_t max_len, float* hidden_out, void* stream, const s3b_forward_opts* opts) {
    if (!m || !wavs || !lens || !hidden_out) return fail("null argument");
    if (!m->finalized) return fail("model not finalized");
    if (opts != nullptr && opts->struct_size != (int32_t)sizeof(s3b_forward_opts))
        return fail("s3b_forward_opts.struct_size %d != %d (header / library mismatch)", opts->struct_size,
                    (int)sizeof(s3b_forward_opts));
    for (int b = 0; b < batch; ++b)
        if (lens[b] > max_len) return fail("lens[%d]=%lld exceeds max_len", b, (long long)lens[b]);
    if (opts != nullptr && (opts->ffn_out != nullptr || opts->last_residual != nullptr)) {
        const char* why =
            m->kind == kGruStack    ? "an APC model is a GRU stack, it has no feed-forward blocks or layer results"
            : m->kind == kLstmStack ? "a DeCoAR model is an LSTM stack, it has no feed-forward blocks or layer results"
            : m->kind == kNpcStack  ? "an NPC model is a conv stack, it has no feed-forward blocks or layer results"
            : m->kind == kCpcStack  ? "a modified CPC model is a conv stack and an LSTM, it has no feed-forward blocks or "
                                      "layer results"
            : m->kind == kSsastEncoder ? "the SSAST expert returns only its blocks' outputs (ssast/expert.py)"
            : m->cfg.conformer      ? "a Conformer encoder collects no layer results (wav2vec2_model.py:3199-3200)"
                                    : nullptr;
        if (why != nullptr) return fail("ffn_out / last_residual: %s", why);
    }
    return forward_lanes(m, wavs, lens, batch, max_len, hidden_out, (cudaStream_t)stream, opts);
}

static int forward_host_impl(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch,
                             int64_t max_len, float* hidden_out, float* hidden_dev) {
    const int64_t T = model_frames(m, max_len);
    if (T < 1) return fail_too_short(m, max_len);
    size_t total = 0;
    for (int b = 0; b < batch; ++b) total += (size_t)lens[b];
    S3B_OK(m->stage_wav.ensure(total * 4));
    const size_t frame_elems = (size_t)T * out_width(m);
    const size_t layer_elems = (size_t)batch * frame_elems;
    if (hidden_dev == nullptr) {
        S3B_OK(m->stage_out.ensure((size_t)s3b_num_outputs(m) * layer_elems * 4));
        hidden_dev = m->stage_out.as<float>();
    }
    S3B_OK(ensure_stream(m->copy_stream));
    S3B_OK(ensure_stream(m->compute_stream));
    while ((int)m->layer_events.size() < s3b_num_outputs(m)) {
        Event e;
        S3B_OK(ensure_event(e));
        m->layer_events.push_back(std::move(e));
    }
    cudaStream_t st = m->compute_stream.get();
    std::vector<const float*> ptrs(batch);
    size_t off = 0;
    for (int b = 0; b < batch; ++b) {
        float* d = m->stage_wav.as<float>() + off;
        CUDA_OK(cudaMemcpyAsync(d, wavs[b], (size_t)lens[b] * 4, cudaMemcpyHostToDevice, st));
        ptrs[b] = d;
        off += (size_t)lens[b];
    }
    // device->host copy of hidden state l overlaps the computation of layer l+1 (second stream).
    // The batch is processed as k utterance chunks (S3B_HOST_CHUNKS=k overrides the default below) so that chunk
    // c+1's conv stack overlaps chunk c's copies — nothing can leave the device before the first
    // hidden state exists (~5 ms at 32 x 10 s), which is what bounds the end-to-end time. Utterances
    // are independent given the shared max_len, so the result is bit-identical. Every chunk writes its utterances'
    // slice of the standard [NL+1][batch][T][D] device buffer (layer stride = the whole batch).
    struct Ctx {
        float* host;        // hidden_out + first utterance of the chunk
        const float* dev;   // same position in the device buffer
        size_t layer;       // elements between layers (batch * T * D), host and device alike
        size_t chunk;       // elements per layer of this chunk (Bc * T * D)
    };
    auto layer_done = [](s3b_model* mm, int l, cudaStream_t s, void* user) -> int {
        Ctx* c = static_cast<Ctx*>(user);
        CUDA_OK(cudaEventRecord(mm->layer_events[l].get(), s));
        CUDA_OK(cudaStreamWaitEvent(mm->copy_stream.get(), mm->layer_events[l].get(), 0));
        CUDA_OK(cudaMemcpyAsync(c->host + (size_t)l * c->layer, c->dev + (size_t)l * c->layer, c->chunk * 4,
                                cudaMemcpyDeviceToHost, mm->copy_stream.get()));
        return 0;
    };
    // default: two chunks from 16 utterances on (first-output latency ~ half, GEMMs at 16 utterances still run at
    // ~90 % of their 32-utterance rate); smaller batches are not copy-bound enough to pay for the smaller GEMMs
    int chunks = batch >= 16 ? 2 : 1;
    if (const char* e = getenv("S3B_HOST_CHUNKS")) chunks = atoi(e);
    if (chunks < 1) chunks = 1;
    if (chunks > batch) chunks = batch;
    std::vector<Ctx> ctxs(chunks);
    for (int c = 0; c < chunks; ++c) {
        const int b0 = (int)((int64_t)batch * c / chunks), b1 = (int)((int64_t)batch * (c + 1) / chunks);
        ctxs[c] = Ctx{hidden_out + (size_t)b0 * frame_elems, hidden_dev + (size_t)b0 * frame_elems, layer_elems,
                      (size_t)(b1 - b0) * frame_elems};
        Fwd f;
        f.m = m, f.w = &m->ws[0], f.st = st, f.wavs = ptrs.data() + b0, f.lens = lens + b0, f.B = b1 - b0;
        f.Lmax = max_len, f.hidden = hidden_dev + (size_t)b0 * frame_elems, f.layer_stride = layer_elems;
        f.layer_done = layer_done, f.user = &ctxs[c];
        S3B_OK(f.prepare());
        for (const Step& step : f.plan->steps) S3B_OK(step(f));
    }
    CUDA_OK(cudaStreamSynchronize(st));
    CUDA_OK(cudaStreamSynchronize(m->copy_stream.get()));
    return 0;
}

extern "C" int s3b_forward_host(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch,
                                int64_t max_len, float* hidden_out) {
    if (!m || !wavs || !lens || !hidden_out) return fail("null argument");
    if (!m->finalized) return fail("model not finalized");
    return forward_host_impl(m, wavs, lens, batch, max_len, hidden_out, nullptr);
}

extern "C" int s3b_forward_host_ex(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch,
                                   int64_t max_len, float* hidden_out, float* hidden_out_dev) {
    if (!m || !wavs || !lens || !hidden_out) return fail("null argument");
    if (!m->finalized) return fail("model not finalized");
    return forward_host_impl(m, wavs, lens, batch, max_len, hidden_out, hidden_out_dev);
}

// ------------------------------------------------------------------------------------------------
// profiling / accounting
// ------------------------------------------------------------------------------------------------
extern "C" int s3b_profile_enable(s3b_model* m, int32_t enable) {
    if (!m) return fail("null model");
    m->prof.on = enable != 0;
    return 0;
}

extern "C" int s3b_profile_read_ex(s3b_model* m, int32_t num_categories, double* ms, double* flops, int64_t* launches,
                                   int32_t reset) {
    if (!m || !ms || !flops || !launches) return fail("null argument");
    if (num_categories < 1 || num_categories > CAT_COUNT) return fail("num_categories must be 1..%d", (int)CAT_COUNT);
    CUDA_OK(cudaDeviceSynchronize());
    for (ProfRec& r : m->prof.recs) {
        float t = 0.f;
        CUDA_OK(cudaEventElapsedTime(&t, r.a.get(), r.b.get()));
        m->prof.ms[r.cat] += t;
        m->prof.pool.push_back(std::move(r.a));
        m->prof.pool.push_back(std::move(r.b));
    }
    m->prof.recs.clear();
    for (int c = 0; c < CAT_COUNT; ++c) {
        if (c < num_categories) ms[c] = m->prof.ms[c], flops[c] = m->prof.flops[c], launches[c] = m->prof.launches[c];
        if (reset) m->prof.ms[c] = 0, m->prof.flops[c] = 0, m->prof.launches[c] = 0;
    }
    return 0;
}

extern "C" int s3b_profile_read(s3b_model* m, double* ms, double* flops, int64_t* launches, int32_t reset) {
    return s3b_profile_read_ex(m, 5, ms, flops, launches, reset);
}

extern "C" int64_t s3b_launch_count(const s3b_model* m) { return m ? m->launches_total : -1; }

// ------------------------------------------------------------------------------------------------
// Featurizer
// ------------------------------------------------------------------------------------------------
// The weighted-sum kernels keep the layer weights in a 64-entry shared table and move hs / out / grad_out as float4.
// Checked before any CUDA call, so a bad argument is refused with its name even on a host without a device.
static int check_layers(int32_t num) {
    if (num < 1 || num > 64) return fail("num = %d: the weighted sum takes 1..64 layers", num);
    return 0;
}
static int check_float4(const void* ptr, const char* name) {
    if (reinterpret_cast<uintptr_t>(ptr) & 15) return fail("%s = %p is not 16-byte aligned (read as float4)", name, ptr);
    return 0;
}
static int check_ws_args(const float* hs, int32_t num, int64_t n_per_layer, const float* other, const char* other_name) {
    S3B_OK(check_layers(num));
    if (n_per_layer < 0 || (n_per_layer & 3) != 0)
        return fail("n_per_layer = %lld must be a non-negative multiple of 4", (long long)n_per_layer);
    S3B_OK(check_float4(hs, "hs"));
    return check_float4(other, other_name);
}

extern "C" int s3b_weighted_sum(const float* hs, int32_t num, int64_t n_per_layer, const float* w, float* out,
                                void* stream) {
    if (!hs || !w || !out) return fail("null argument");
    S3B_OK(check_ws_args(hs, num, n_per_layer, out, "out"));
    CUDA_OK(launch_weighted_sum(hs, num, (size_t)n_per_layer, w, out, (cudaStream_t)stream));
    return 0;
}
extern "C" int s3b_weighted_sum_backward(const float* hs, int32_t num, int64_t n_per_layer, const float* grad_out,
                                         float* grad_w, void* stream) {
    if (!hs || !grad_out || !grad_w) return fail("null argument");
    S3B_OK(check_ws_args(hs, num, n_per_layer, grad_out, "grad_out"));
    CUDA_OK(launch_weighted_sum_bwd(hs, num, (size_t)n_per_layer, grad_out, grad_w, (cudaStream_t)stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// peer-memory feature exchange (fused weighted sum + all-gather, csrc/peer.cu)
// ------------------------------------------------------------------------------------------------
struct s3b_peer {
    int rank = 0, world = 1, slots = 3;
    int64_t block = 0;       // floats per rank block
    void* base = nullptr;    // own allocation: [slots][world][block] floats | flags [slots][world] u32 | counter
    size_t bytes = 0, flags_off = 0, counter_off = 0;
    std::vector<void*> peer_base;  // every rank's allocation as mapped in THIS process (own: base)
    bool connected = false;
    s3b_peer() = default;
    s3b_peer(const s3b_peer&) = delete;
    s3b_peer& operator=(const s3b_peer&) = delete;
    ~s3b_peer() {
        for (int r = 0; r < (int)peer_base.size(); ++r)
            if (r != rank && peer_base[r]) cudaIpcCloseMemHandle(peer_base[r]);
        if (base) cudaFree(base);
    }
};

extern "C" int s3b_peer_create(int32_t rank, int32_t world, int64_t block_elems, int32_t slots, s3b_peer** out,
                               void* ipc_handle_out) {
    if (!out || !ipc_handle_out) return fail("null argument");
    if (world < 1 || world > 16 || rank < 0 || rank >= world) return fail("bad rank / world (max 16 ranks)");
    if (block_elems < 4 || (block_elems & 3) != 0) return fail("block_elems must be a positive multiple of 4");
    if (slots < 2 || slots > 8) return fail("slots must be in [2, 8]");
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    s3b_peer* p = new s3b_peer();
    p->rank = rank, p->world = world, p->slots = slots, p->block = block_elems;
    const size_t data = (size_t)slots * world * (size_t)block_elems * 4;
    p->flags_off = (data + 255) & ~(size_t)255;
    p->counter_off = p->flags_off + (((size_t)slots * world * 4 + 255) & ~(size_t)255);
    p->bytes = p->counter_off + 256;
    cudaError_t e = cudaMalloc(&p->base, p->bytes);
    if (e == cudaSuccess) e = cudaMemset(p->base, 0, p->bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p->base);
    if (e != cudaSuccess) {
        delete p;
        return fail("peer buffer allocation / IPC export failed: %s", cudaGetErrorString(e));
    }
    memcpy(ipc_handle_out, &h, sizeof(h));
    p->peer_base.assign(world, nullptr);
    p->peer_base[rank] = p->base;
    *out = p;
    return 0;
}

extern "C" int s3b_peer_connect(s3b_peer* p, const void* all_handles) {
    if (!p || !all_handles) return fail("null argument");
    if (p->connected) return 0;
    const cudaIpcMemHandle_t* hs = static_cast<const cudaIpcMemHandle_t*>(all_handles);
    for (int r = 0; r < p->world; ++r) {
        if (r == p->rank) continue;
        void* ptr = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&ptr, hs[r], cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail("cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
        }
        p->peer_base[r] = ptr;
    }
    p->connected = true;
    return 0;
}

extern "C" float* s3b_peer_slot(s3b_peer* p, uint32_t step) {
    if (!p) return nullptr;
    return static_cast<float*>(p->base) + (size_t)(step % p->slots) * p->world * (size_t)p->block;
}

extern "C" int s3b_peer_push(s3b_peer* p, const float* hs, int32_t num, int64_t layer_stride, const float* w,
                             uint32_t step, void* stream) {
    if (!p || !hs || !w) return fail("null argument");
    if (!p->connected && p->world > 1) return fail("s3b_peer_connect has not been called");
    S3B_OK(check_layers(num));
    if (layer_stride < p->block || (layer_stride & 3) != 0)
        return fail("layer_stride = %lld must be a multiple of 4 and >= block_elems = %lld", (long long)layer_stride,
                    (long long)p->block);
    S3B_OK(check_float4(hs, "hs"));
    const int slot = (int)(step % p->slots);
    float* dst[16];
    uint32_t* flag[16];
    for (int r = 0; r < p->world; ++r) {
        char* b = static_cast<char*>(p->peer_base[r]);
        dst[r] = reinterpret_cast<float*>(b) + ((size_t)slot * p->world + p->rank) * (size_t)p->block;
        flag[r] = reinterpret_cast<uint32_t*>(b + p->flags_off) + (size_t)slot * p->world + p->rank;
    }
    unsigned int* counter = reinterpret_cast<unsigned int*>(static_cast<char*>(p->base) + p->counter_off);
    CUDA_OK(launch_weighted_sum_push(hs, num, (size_t)p->block, (size_t)layer_stride, w, dst, flag, p->world, step + 1,
                                     counter, (cudaStream_t)stream));
    return 0;
}

extern "C" int s3b_peer_wait(s3b_peer* p, uint32_t step, void* stream) {
    if (!p) return fail("null argument");
    const uint32_t* flags = reinterpret_cast<const uint32_t*>(static_cast<char*>(p->base) + p->flags_off) +
                            (size_t)(step % p->slots) * p->world;
    CUDA_OK(launch_wait_flags(flags, p->world, step + 1, (cudaStream_t)stream));
    return 0;
}

extern "C" void s3b_peer_destroy(s3b_peer* p) { delete p; }

// ------------------------------------------------------------------------------------------------
// building blocks for parity tests
// ------------------------------------------------------------------------------------------------
static int device_sm_count(int* out) {
    int dev = 0;
    CUDA_OK(cudaGetDevice(&dev));
    CUDA_OK(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
    return 0;
}

// Operand scheme of a building-block call: -1 = the library default where the shape allows it (else bf16x3), 0 / 1 =
// exactly that scheme (linear_params / conv_params refuse an f16q8 request the shape cannot take)
static int resolve_scheme(int scheme, int K, int N, int* out) {
    if (scheme < -1 || scheme > 1) return fail("scheme must be -1 (default), 0 (bf16x3) or 1 (f16q8), not %d", scheme);
    if (scheme == -1) scheme = (K % 128 == 0 && N % 128 == 0) ? default_scheme() : 0;
    *out = scheme;
    return 0;
}

// fp32 -> operand planes of `scheme`, on the stream (weight != 0: the weight split of the f16q8 format)
static int split_operand(const float* x, SplitBuf& s, size_t n, int scheme, int weight, cudaStream_t st) {
    S3B_OK(s.ensure(n));
    if (scheme != 0) CUDA_OK(launch_split_q8(x, s.h(), s.h8(), s.l8(), n, weight, st));
    else CUDA_OK(launch_split(x, s.h(), s.l(), n, st));
    return 0;
}

// a device fp32 tensor of the caller (written on `st`) to the host, for the weight relayouts of s3b_model_finalize
static int download_f32(const float* src, size_t n, cudaStream_t st, std::vector<float>& dst) {
    dst.resize(n);
    CUDA_OK(cudaStreamSynchronize(st));
    CUDA_OK(cudaMemcpy(dst.data(), src, n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

static int check_out_fmt(int out_fmt) {
    if (out_fmt < -1 || out_fmt > 1) return fail("out_fmt must be -1 (fp32), 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    return 0;
}

extern "C" int s3b_linear_ex(const float* a, const float* w, const float* bias, const float* residual, int64_t M,
                             int32_t N, int32_t K, int32_t gelu, s3b_linear_opts* opts, float* out, void* stream) {
    if (!a || !w || !out) return fail("null argument");
    if (M < 1 || N < 1 || K < 1) return fail("bad sizes");
    s3b_linear_opts o;
    memset(&o, 0, sizeof(o));
    o.scheme = -1, o.out_fmt = -1;
    if (opts != nullptr) {
        if (opts->struct_size != (int32_t)sizeof(s3b_linear_opts))
            return fail("s3b_linear_opts.struct_size %d != %d (header / library mismatch)", opts->struct_size,
                        (int)sizeof(s3b_linear_opts));
        o = *opts;
    }
    int scheme = 0;
    S3B_OK(resolve_scheme(o.scheme, K, N, &scheme));
    S3B_OK(check_out_fmt(o.out_fmt));
    if (gelu < 0 || gelu > 2) return fail("gelu must be 0 (none), 1 (GELU) or 2 (SiLU), not %d", gelu);
    if (o.tile_n != 0 && o.tile_n != 128 && o.tile_n != 256) return fail("tile_n must be 0, 128 or 256, not %d", o.tile_n);
    if (o.tile_n != 0 && N % o.tile_n != 0) return fail("tile_n %d does not divide N = %d", o.tile_n, N);
    const int64_t lda = o.lda != 0 ? o.lda : K;
    if (o.a_off < 0 || o.a_off + K > lda || (o.lda != 0 && (lda % 16 != 0 || o.a_off % 16 != 0)))
        return fail("A slice [%lld, %lld) of rows of %lld elements: out of range or not a multiple of 16",
                    (long long)o.a_off, (long long)(o.a_off + K), (long long)lda);
    cudaStream_t st = (cudaStream_t)stream;
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    SplitBuf as, ws, os;
    S3B_OK(split_operand(a, as, (size_t)M * lda, scheme, 0, st));
    S3B_OK(split_operand(w, ws, (size_t)N * K, scheme, 1, st));
    Epi e;
    e.bias = bias, e.residual = residual, e.gelu = gelu, e.row_mask = o.row_mask;
    if (o.out_fmt < 0) {
        e.out_f32 = out;
    } else {
        S3B_OK(os.ensure((size_t)M * N));
        e.op = os.planes(o.out_fmt);
    }
    GemmParams p;
    S3B_OK(linear_params(p, as, ws, M, N, K, scheme, sms, e, lda, (size_t)o.a_off, o.tile_n));
    if (o.tile_n != 0 && p.bn != o.tile_n) return fail("tile_n %d requested, %d chosen", o.tile_n, p.bn);
    p.out_pre = o.out_pre;
    CUDA_OK(launch_gemm(p, sms, st));
    if (o.out_fmt >= 0) CUDA_OK(launch_planes_to_f32(os.planes(o.out_fmt), (size_t)M * N, out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (opts != nullptr) opts->scheme_used = scheme, opts->tile_n_used = p.bn;
    return 0;
}

extern "C" int s3b_linear_f32(const float* a, const float* w, const float* bias, const float* residual, int64_t M,
                              int32_t N, int32_t K, int32_t gelu, float* out, void* stream) {
    return s3b_linear_ex(a, w, bias, residual, M, N, K, gelu, nullptr, out, stream);
}

extern "C" int s3b_qkv_hd_f32(const float* x, const float* w, const float* b, int32_t B, int32_t T, int32_t H,
                              int32_t hd, int32_t scheme, float* q_out, float* k_out, float* vt_out, void* stream) {
    if (!x || !w || !b || !q_out || !k_out || !vt_out) return fail("null argument");
    if (B < 1 || T < 1 || H < 1) return fail("bad sizes");
    if (!head_dim_ok(hd)) return fail("head_dim must be 64, 80 or 120, not %d", hd);
    const int D = H * hd, Tp = (T + 7) & ~7;
    const int64_t M = (int64_t)B * T;
    int sch = 0;
    S3B_OK(resolve_scheme(scheme, D, 3 * D, &sch));
    cudaStream_t st = (cudaStream_t)stream;
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    SplitBuf xs, ws, qs, ks, vts;
    S3B_OK(split_operand(x, xs, (size_t)M * D, sch, 0, st));
    S3B_OK(split_operand(w, ws, (size_t)3 * D * D, sch, 1, st));
    S3B_OK(qs.ensure((size_t)M * D));
    S3B_OK(ks.ensure((size_t)M * D));
    S3B_OK(vts.ensure((size_t)B * D * Tp));
    GemmParams p;
    S3B_OK(linear_params(p, xs, ws, M, 3 * D, D, sch, sms, Epi()));
    set_qkv_epi(p, b, T, H, hd, qs, ks, vts);
    CUDA_OK(launch_gemm(p, sms, st));
    CUDA_OK(launch_planes_to_f32(qs.planes(0), (size_t)M * D, q_out, st));
    CUDA_OK(launch_planes_to_f32(ks.planes(0), (size_t)M * D, k_out, st));
    CUDA_OK(launch_planes_to_f32(vts.planes(0), (size_t)B * D * Tp, vt_out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_qkv_f32(const float* x, const float* w, const float* b, int32_t B, int32_t T, int32_t H,
                           int32_t scheme, float* q_out, float* k_out, float* vt_out, void* stream) {
    return s3b_qkv_hd_f32(x, w, b, B, T, H, 64, scheme, q_out, k_out, vt_out, stream);
}

extern "C" int s3b_conv_gemm_f32(const float* x, const float* w, const float* bias, int32_t B, int64_t Lin, int32_t kw,
                                 int32_t gelu, int32_t scheme, int32_t out_fmt, float* out, void* stream) {
    if (!x || !w || !out) return fail("null argument");
    if (kw != 2 && kw != 3) return fail("kw must be 2 or 3, not %d", kw);
    if (B < 1 || Lin < kw) return fail("bad sizes (batch %d, lin %lld, kw %d)", B, (long long)Lin, kw);
    S3B_OK(check_out_fmt(out_fmt));
    const int C = kConvDim;
    const int64_t Lout = (Lin - kw) / 2 + 1;
    int sch = 0;
    S3B_OK(resolve_scheme(scheme, kw * C, C, &sch));
    cudaStream_t st = (cudaStream_t)stream;
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    SplitBuf xs, ws, os;
    std::vector<float> wh;
    S3B_OK(download_f32(w, (size_t)C * C * kw, st, wh));
    const std::vector<float> wl = tap_weight_layout(wh.data(), C, C, kw, 0, C);
    S3B_OK(upload_split(ws, wl.data(), wl.size(), sch));
    S3B_OK(split_operand(x, xs, (size_t)B * Lin * C, sch, 0, st));
    Epi e;
    e.bias = bias, e.gelu = gelu;
    if (out_fmt < 0) {
        e.out_f32 = out;
    } else {
        S3B_OK(os.ensure((size_t)B * Lout * C));
        e.op = os.planes(out_fmt);
    }
    GemmParams p;
    S3B_OK(conv_params(p, xs, ws, B, Lin, Lout, 2, C, C, C, kw, 0, sch, e));
    CUDA_OK(launch_gemm(p, sms, st));
    if (out_fmt >= 0) CUDA_OK(launch_planes_to_f32(os.planes(out_fmt), (size_t)B * Lout * C, out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_posconv_f32(const float* x, const float* w, const float* bias, int32_t B, int32_t T, int32_t D,
                               int32_t G, int32_t k, int32_t taps, int32_t mode, const float* gamma, const float* beta,
                               int32_t out_fmt, float* out, void* stream) {
    if (!x || !w || !bias || !out || (gamma == nullptr) != (beta == nullptr)) return fail("null argument");
    if (B < 1 || T < 1) return fail("bad sizes");
    if (D != 384 && D != 512 && D != 640 && D != 768 && D != 1024 && D != 1280 && D != 1920)
        return fail("d must be 384, 512, 640, 768, 1024, 1280 or 1920, not %d", D);
    if (G < 1 || D % G != 0) return fail("d %d is not a multiple of groups %d", D, G);
    const int cpg = D / G;
    if (!posconv_cpg_ok(cpg))
        return fail("channels per group must be 16, 32, 48, 64, 80 or 120, or 24 or 40 with four taps per k-block (got %d)",
                    cpg);
    if (taps != 1 && taps != 4) return fail("taps_per_kblock must be 1 or 4, not %d", taps);
    if (mode < 0 || mode > 2) return fail("mode must be 0, 1 or 2, not %d", mode);
    if (k < 2) return fail("kernel size %d < 2", k);
    if (mode == 0 && k % (taps == 4 ? 4 : 2) != 0) return fail("conv_pos kernel %d: must be even (a multiple of 4 with "
                                                               "four taps per k-block)", k);
    if (taps == 4 && !posconv4_only(cpg) && cpg != 48 && cpg != 64)
        return fail("four taps per k-block need 24, 40, 48 or 64 channels per group");
    if (taps == 1 && posconv4_only(cpg)) return fail("%d channels per group run four taps per k-block only", cpg);
    if (taps == 1 && mode != 0) return fail("the data2vec blocks (mode 1, 2) run four taps per k-block only");
    if (taps == 1 && gamma == nullptr && out_fmt >= 0)  // add_pos_conv: the one-tap epilogue writes fp32 only
        return fail("one tap per k-block writes operand planes only through the LayerNorm (gamma)");
    S3B_OK(check_out_fmt(out_fmt));
    // one conv block of k taps: pos_taps(c) = k (the data2vec blocks' k = max(3, conv_pos / depth) is the caller's)
    s3b_config c;
    memset(&c, 0, sizeof(c));
    c.embed_dim = D, c.pos_conv_groups = G, c.pos_conv_kernel = k, c.pos_conv_depth = 1;
    const size_t M = (size_t)B * T;
    cudaStream_t st = (cudaStream_t)stream;
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    SplitBuf xs, ws, os;
    DevBuf z;
    std::vector<float> wh;
    S3B_OK(download_f32(w, (size_t)D * cpg * k, st, wh));
    const std::vector<float> wl = taps == 4 ? posconv4_weight_layout(wh.data(), D, G, k)
                                            : tap_weight_layout(wh.data(), D, cpg, k, 0, posconv_kc(cpg));
    S3B_OK(upload_split(ws, wl.data(), wl.size()));
    S3B_OK(split_operand(x, xs, M * D, 0, 0, st));
    OutPlanes op = no_planes();
    if (out_fmt >= 0) {
        S3B_OK(os.ensure(M * D));
        op = os.planes(out_fmt);
    }
    float* out_f32 = out_fmt < 0 ? out : nullptr;
    GemmParams p;
    if (taps == 4) {
        // add_pos_conv: Z = the four-tap GEMM, then the combine kernel (+ LayerNorm)
        S3B_OK(z.ensure((size_t)B * (T + 3) * 4 * D * sizeof(float)));
        S3B_OK(posconv4_params(p, c, xs, ws, B, T, epi_f32(z.as<float>())));
        CUDA_OK(launch_gemm(p, sms, st));
        CUDA_OK(launch_posconv_combine(z.as<float>(), x, bias, B, T, D, cpg, gamma, beta, gamma ? 1 : 0, mode,
                                       out_f32, op, st));
    } else {
        // add_pos_conv, one tap per k-block: x + GELU(conv + bias) in the epilogue, then the LayerNorm
        if (gamma != nullptr) S3B_OK(z.ensure(M * D * sizeof(float)));
        Epi e = epi_f32(gamma != nullptr ? z.as<float>() : out_f32, bias, x);
        e.gelu = 1;
        S3B_OK(posconv_params(p, c, xs, ws, B, T, e));
        CUDA_OK(launch_gemm(p, sms, st));
        if (gamma != nullptr) CUDA_OK(launch_layernorm(z.as<float>(), M, D, gamma, beta, 0, out_f32, op, st));
    }
    if (out_fmt >= 0) CUDA_OK(launch_planes_to_f32(op, M * D, out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_npc_conv_f32(const float* x, int32_t B, int32_t T, int32_t c_in, const float* w, int32_t k,
                                int32_t mask, const float* bias, const float* residual, int32_t act, int32_t res_first,
                                int32_t scheme, float* out, float* out_pre, void* stream) {
    if (!x || !w || !out) return fail("null argument");
    if (B < 1 || T < 1) return fail("bad sizes (batch %d, t %d)", B, T);
    if (c_in != 80 && c_in != 512) return fail("c_in must be 80 or 512, not %d", c_in);
    if (k < 1 || k > 127 || k % 2 == 0) return fail("k %d: must be odd, 1..127", k);
    if (mask < 0 || (mask > 0 && (mask % 2 == 0 || mask >= k))) return fail("mask %d: must be 0 or odd and < k %d", mask, k);
    if (act < 0 || act > 2) return fail("act must be 0 (none), 1 (ReLU) or 2 (tanh), not %d", act);
    if (res_first != 0 && res_first != 1) return fail("res_first must be 0 or 1, not %d", res_first);
    if (res_first && out_pre != nullptr) return fail("out_pre is the value before the residual add: not with res_first");
    const int N = 512, Cp = c_in == 80 ? kDecoar2K : 512, u = k - mask;
    const size_t M = (size_t)B * T;
    int sch = 0;
    S3B_OK(resolve_scheme(scheme, u * Cp, N, &sch));
    cudaStream_t st = (cudaStream_t)stream;
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    std::vector<float> wh;
    S3B_OK(download_f32(w, (size_t)N * c_in * k, st, wh));
    const std::vector<float> wl = tap_weight_layout(wh.data(), N, c_in, k, mask, Cp);
    SplitBuf xs, ws;
    S3B_OK(upload_split(ws, wl.data(), wl.size(), sch));
    DevBuf xpad;
    if (Cp != c_in) {  // 80 channels zero-padded to 128 per row, as the CMVN kernel writes them
        S3B_OK(xpad.ensure(M * Cp * 4));
        CUDA_OK(cudaMemcpy2DAsync(xpad.p, (size_t)Cp * 4, x, (size_t)c_in * 4, (size_t)c_in * 4, M,
                                  cudaMemcpyDeviceToDevice, st));
    }
    S3B_OK(split_operand(Cp != c_in ? xpad.as<float>() : x, xs, M * Cp, sch, 0, st));
    Epi e = epi_f32(out, bias, residual);
    e.gelu = act == 0 ? 0 : act == 1 ? 3 : 4, e.res_first = res_first;
    GemmParams p;
    S3B_OK(conv_params(p, xs, ws, B, T, T, 1, N, c_in, Cp, k, mask, sch, e));
    p.out_pre = out_pre;
    CUDA_OK(launch_gemm(p, sms, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_cpc_conv_f32(const float* x, int32_t B, int32_t L, int32_t layer, const float* w, const float* bias,
                                const float* gamma, const float* beta, int32_t scheme, float* out, void* stream) {
    if (!x || !w || !bias || !gamma || !beta || !out) return fail("null argument");
    if (layer < 0 || layer >= kCpcConvs) return fail("layer %d: must be 0..%d", layer, kCpcConvs - 1);
    if (B < 1 || L < 1) return fail("bad sizes (batch %d, length %d)", B, L);
    const int C = kCpcDim, s = kCpcStride[layer], k = 2 * s;
    const int64_t Tout = cpc_conv_len(L, layer);
    if (Tout < 1) return fail("length %d too short for conv %d (kernel %d, padding %d)", L, layer, k, kCpcPad[layer]);
    if ((int64_t)B * cpc_rows(Tout, layer) > 2000000000LL) return fail("batch too large for 32-bit indexing");
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    int sch = 0;
    S3B_OK(resolve_scheme(scheme, k * C, C, &sch));
    cudaStream_t st = (cudaStream_t)stream;
    const size_t M = (size_t)B * Tout;
    SplitBuf os;
    S3B_OK(os.ensure(M * C));
    if (layer == 0) {
        // conv 0 writes operand planes only (in the model: conv 1's); here the dense layout, decoded back to fp32
        CUDA_OK(launch_cpc_conv0(x, B, L, (int)Tout, w, bias, gamma, beta, (int)Tout, 0, os.planes(sch), st));
        CUDA_OK(launch_planes_to_f32(os.planes(sch), M * C, out, st));
        CUDA_OK(cudaStreamSynchronize(st));
        return 0;
    }
    // x [B][L][256] into the padded layout the model's producers write: pad zero rows, the frames that fit, zero rows
    const int64_t R = cpc_rows(Tout, layer), pad = kCpcPad[layer], n = std::min<int64_t>(L, R - pad);
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    std::vector<float> wh;
    S3B_OK(download_f32(w, (size_t)C * C * k, st, wh));
    const std::vector<float> wl = tap_weight_layout(wh.data(), C, C, k, 0, C);
    SplitBuf xs, ws;
    S3B_OK(upload_split(ws, wl.data(), wl.size(), sch));
    DevBuf xpad, z;
    S3B_OK(xpad.ensure((size_t)B * R * C * 4));
    CUDA_OK(cudaMemsetAsync(xpad.p, 0, (size_t)B * R * C * 4, st));
    CUDA_OK(cudaMemcpy2DAsync(xpad.as<float>() + pad * C, (size_t)R * C * 4, x, (size_t)L * C * 4, (size_t)n * C * 4, B,
                              cudaMemcpyDeviceToDevice, st));
    S3B_OK(split_operand(xpad.as<float>(), xs, (size_t)B * R * C, sch, 0, st));
    S3B_OK(z.ensure(M * C * 4));
    GemmParams p;
    S3B_OK(conv_params(p, xs, ws, B, R, Tout, s, C, C, C, k, 0, sch, epi_f32(z.as<float>(), bias)));
    CUDA_OK(launch_gemm(p, sms, st));
    CUDA_OK(launch_channelnorm_relu(z.as<float>(), B, (int)Tout, (int)Tout, 0, gamma, beta, out, os.planes(sch), st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_cpc_lstm_max_active_clusters(int32_t* out) {
    if (!out) return fail("null argument");
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    int n = 0;
    CUDA_OK(cpc_lstm_max_active_clusters(&n));
    *out = n;
    return 0;
}

extern "C" int s3b_cpc_lstm_f32(const float* xg, const float* whh, int32_t B, int32_t T, int32_t out_fmt, float* out,
                                float* planes_out, void* stream) {
    // add_cpc_stack's recurrence on this call's buffers
    if (!xg || !whh || !out) return fail("null argument");
    if (B < 1 || T < 1) return fail("bad sizes (batch %d, t %d)", B, T);
    if (out_fmt < -1 || out_fmt > 1) return fail("out_fmt must be -1 (none), 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    if (out_fmt >= 0 && planes_out == nullptr) return fail("out_fmt %d needs planes_out", out_fmt);
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t M = (size_t)B * T;
    SplitBuf os;
    CpcLstmParams g;
    g.xg = xg, g.whh = whh, g.B = B, g.T = T, g.out = out, g.op = no_planes();
    if (out_fmt >= 0) {
        S3B_OK(os.ensure(M * kCpcDim));
        g.op = os.planes(out_fmt);
    }
    CUDA_OK(launch_cpc_lstm(g, st));
    if (out_fmt >= 0) CUDA_OK(launch_planes_to_f32(g.op, M * kCpcDim, planes_out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

// Times `iters` back-to-back launches of the production GEMM (bias + GELU + split epilogue like fc1 when gelu != 0,
// bias + residual + fp32 output like out_proj / fc2 otherwise) on random operands; force_un in {0, 128, 256}.
extern "C" int s3b_gemm_bench(int64_t M, int32_t N, int32_t K, int32_t gelu, int32_t force_un, int32_t iters,
                              float* ms_per_launch) {
    if (!ms_per_launch || iters < 1) return fail("bad argument");
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    SplitBuf as, ws, os;
    DevBuf bias, res, out;
    S3B_OK(as.ensure((size_t)M * K));
    S3B_OK(ws.ensure((size_t)N * K));
    S3B_OK(bias.ensure((size_t)N * 4));
    S3B_OK(res.ensure((size_t)M * N * 4));
    S3B_OK(out.ensure((size_t)M * N * 4));
    S3B_OK(os.ensure((size_t)M * N));
    // finite, non-trivial operand bits: bf16 0x3c00..0x3cff ~ 0.0078..0.031
    CUDA_OK(cudaMemset(as.hi.p, 0x3c, (size_t)M * K * 2));
    CUDA_OK(cudaMemset(ws.hi.p, 0x3c, (size_t)N * K * 2));
    GemmParams p;
    int scheme = default_scheme();
    if (K % 128 != 0 || N % 128 != 0) scheme = 0;
    const Epi e = gelu ? epi_planes(os.planes(scheme), bias.as<float>(), 1)
                       : epi_f32(out.as<float>(), bias.as<float>(), res.as<float>());
    S3B_OK(linear_params(p, as, ws, M, N, K, scheme, sms, e, 0, 0, force_un));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaEventCreate(&e0), cudaEventCreate(&e1);
    const Event t0(e0), t1(e1);
    for (int i = 0; i < 3; ++i) launch_gemm(p, sms, 0);
    cudaEventRecord(e0, 0);
    for (int i = 0; i < iters; ++i) launch_gemm(p, sms, 0);
    cudaEventRecord(e1, 0);
    cudaError_t ce = cudaDeviceSynchronize();
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    *ms_per_launch = ms / iters;
    if (ce != cudaSuccess) return fail("gemm bench failed: %s", cudaGetErrorString(ce));
    if (ms_per_launch[0] >= 0) ms_per_launch[1] = (float)p.bn;
    return 0;
}

extern "C" int s3b_layernorm_eps_f32(const float* x, int64_t M, int32_t D, const float* gamma, const float* beta,
                                     int32_t gelu, float eps, float* out, void* stream) {
    if (!x || !gamma || !beta || !out) return fail("null argument");
    if (!(eps > 0.0f)) return fail("eps must be positive");
    CUDA_OK(launch_layernorm(x, (size_t)M, D, gamma, beta, gelu, out, no_planes(), (cudaStream_t)stream, eps));
    return 0;
}

extern "C" int s3b_layernorm_f32(const float* x, int64_t M, int32_t D, const float* gamma, const float* beta,
                                 int32_t gelu, float* out, void* stream) {
    if (!x || !gamma || !beta || !out) return fail("null argument");
    CUDA_OK(launch_layernorm(x, (size_t)M, D, gamma, beta, gelu, out, no_planes(), (cudaStream_t)stream));
    return 0;
}

extern "C" int s3b_attention_ex(const float* q, const float* k, const float* v, const int32_t* valid_frames,
                                int32_t B, int32_t T, int32_t H, const s3b_attention_opts* opts, float* out,
                                void* stream) {
    // Runs the production path: identity "QKV GEMM" is replaced by a scatter of the given q/k/v, then the
    // attention kernel (WavLM bias table built by the model's own launcher), then the context planes are decoded to fp32.
    if (!q || !k || !v || !valid_frames || !out) return fail("null argument");
    if (B < 1 || T < 1 || H < 1) return fail("bad sizes");
    s3b_attention_opts o;
    memset(&o, 0, sizeof(o));
    if (opts != nullptr) {
        if (opts->struct_size != (int32_t)sizeof(s3b_attention_opts))
            return fail("s3b_attention_opts.struct_size %d != %d (header / library mismatch)", opts->struct_size,
                        (int)sizeof(s3b_attention_opts));
        o = *opts;
    }
    if (o.ctx_format != 0 && o.ctx_format != 1) return fail("ctx_format must be 0 (bf16 hi/lo) or 1 (f16q8)");
    if (o.gate != nullptr && o.rel_emb == nullptr) return fail("a gate needs rel_emb");
    const int hd = o.head_dim != 0 ? o.head_dim : 64;
    if (!head_dim_ok(hd)) return fail("head_dim must be 64, 80 or 120 (0 = 64), not %d", o.head_dim);
    if (hd != 64 && o.rel_emb != nullptr) return fail("the relative position bias (rel_emb) needs head_dim 64");
    const int table_T = o.table_frames != 0 ? o.table_frames : 4096;  // s3b_model_finalize's table
    if (o.rel_emb != nullptr) {
        if (o.num_buckets < 4 || o.max_distance <= o.num_buckets / 4)
            return fail("num_buckets %d / max_distance %d out of range", o.num_buckets, o.max_distance);
        if (table_T < T) return fail("table_frames %d is below t = %d", table_T, T);
    }
    for (int b = 0; b < B; ++b)
        if (valid_frames[b] < 1 || valid_frames[b] > T) return fail("valid_frames[%d] = %d not in [1, %d]", b, valid_frames[b], T);
    cudaStream_t st = (cudaStream_t)stream;
    const int D = H * hd, Tp = (T + 7) & ~7;
    const size_t M = (size_t)B * T;
    SplitBuf qs, ks, vts, ctx;
    DevBuf kv, table;
    S3B_OK(qs.ensure(M * D));
    S3B_OK(ks.ensure(M * D));
    S3B_OK(vts.ensure((size_t)B * D * Tp));
    S3B_OK(ctx.ensure(M * D));
    S3B_OK(kv.ensure(B * sizeof(int)));
    CUDA_OK(cudaMemcpyAsync(kv.p, valid_frames, B * sizeof(int), cudaMemcpyHostToDevice, st));
    CUDA_OK(launch_qkv_scatter(q, k, v, B, T, Tp, H, hd, q_scale(hd), qs.h(), qs.l(), ks.h(), ks.l(), vts.h(), vts.l(),
                               st));
    AttnParams ap;
    memset(&ap, 0, sizeof(ap));
    S3B_OK(attn_tmaps(ap, qs, ks, vts, B, T, H, hd));
    ap.kv_len = kv.as<int>();
    if (o.rel_emb != nullptr) {
        S3B_OK(table.ensure((size_t)H * (2 * (size_t)table_T - 1) * 4));
        CUDA_OK(launch_wavlm_rel_table(o.rel_emb, o.num_buckets, o.max_distance, H, table_T, table.as<float>(), st));
        set_rel_bias(ap, table.as<float>(), table_T, o.gate);
    }
    ap.ctx = ctx.planes(o.ctx_format);
    DevBuf trace;
    const char* tb = getenv("S3B_ATTN_TRACE_BLOCK");  // debug: dump a clock64 timeline of one CTA to stderr
    if (tb != nullptr) {
        S3B_OK(trace.ensure(2 * 16 * 8 * sizeof(long long)));
        CUDA_OK(cudaMemsetAsync(trace.p, 0, 2 * 16 * 8 * sizeof(long long), st));
        ap.trace = trace.as<long long>(), ap.trace_block = atoi(tb);
    }
    CUDA_OK(launch_attention(ap, st));
    if (tb != nullptr) {
        std::vector<long long> h(2 * 16 * 8);
        CUDA_OK(cudaMemcpyAsync(h.data(), trace.p, h.size() * sizeof(long long), cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
        long long t0 = 0;
        for (long long v : h) if (v != 0 && (t0 == 0 || v < t0)) t0 = v;
        for (int role = 0; role < 2; ++role)
            for (int j = 0; j < 16; ++j) {
                if (h[(role * 16 + j) * 8] == 0) continue;
                fprintf(stderr, "attn-trace %s j=%2d:", role == 0 ? "ctrl" : "smax", j);
                for (int sl = 0; sl < 8; ++sl) fprintf(stderr, " %7lld", h[(role * 16 + j) * 8 + sl] ? h[(role * 16 + j) * 8 + sl] - t0 : -1);
                fprintf(stderr, "\n");
            }
    }
    CUDA_OK(launch_planes_to_f32(ctx.planes(o.ctx_format), M * D, out, st));
    const cudaError_t se = cudaStreamSynchronize(st);  // before the buffers are freed
    if (se != cudaSuccess) return fail("attention execution failed: %s", cudaGetErrorString(se));
    return 0;
}

extern "C" int s3b_attention_f32(const float* q, const float* k, const float* v, const int32_t* valid_frames,
                                 int32_t B, int32_t T, int32_t H, float* out, void* stream) {
    return s3b_attention_ex(q, k, v, valid_frames, B, T, H, nullptr, out, stream);
}

extern "C" int s3b_wavlm_gate_f32(const float* x, int32_t B, int32_t T, int32_t H, const float* grep_w,
                                  const float* grep_b, const float* grep_a, int32_t x_format, float* gate_out,
                                  void* stream) {
    // x goes into operand planes the way the model's producers write them (activation split, e4m3 residual scaled by
    // 2^11 in f16q8), then the production gate kernel reads it back from there
    if (!x || !gate_out || (grep_w && (!grep_b || !grep_a))) return fail("null argument");
    if (B < 1 || T < 1 || H < 1) return fail("bad sizes");
    if (x_format != 0 && x_format != 1) return fail("x_format must be 0 (bf16 hi/lo) or 1 (f16q8)");
    cudaStream_t st = (cudaStream_t)stream;
    const int D = H * 64;
    const size_t M = (size_t)B * T;
    SplitBuf xs;
    S3B_OK(xs.ensure(M * D));
    if (x_format != 0) CUDA_OK(launch_split_q8(x, xs.h(), xs.h8(), xs.l8(), M * D, 0, st));
    else CUDA_OK(launch_split(x, xs.h(), xs.l(), M * D, st));
    CUDA_OK(launch_wavlm_gate(xs.planes(x_format), M, B, T, H, D, grep_w, grep_b, grep_a, gate_out, st));
    const cudaError_t se = cudaStreamSynchronize(st);  // before xs is freed
    if (se != cudaSuccess) return fail("gate execution failed: %s", cudaGetErrorString(se));
    return 0;
}

extern "C" int s3b_frontend_f32(const float* const* wavs, const int64_t* lens, int32_t B, int64_t max_len,
                                int32_t normalize, const float* w, const float* bias, const float* gamma,
                                const float* beta, int32_t layer_norm, int32_t out_fmt, float* wav_out, float* out,
                                void* stream) {
    // the first step of add_conv_frontend (launch_frontend) on workspaces of this call; the conv-0 planes decoded to
    // fp32
    if (!wavs || !lens || !w || !gamma || !beta || !out) return fail("null argument");
    if (B < 1) return fail("bad batch %d", B);
    if (max_len < kConvK[0]) return fail("max_len %lld is below the conv-0 window of %d samples", (long long)max_len,
                                         kConvK[0]);
    for (int b = 0; b < B; ++b) {
        if (wavs[b] == nullptr) return fail("null argument: wavs[%d]", b);
        if (lens[b] < 1 || lens[b] > max_len)
            return fail("lens[%d] = %lld not in [1, %lld]", b, (long long)lens[b], (long long)max_len);
    }
    if (normalize != 0 && normalize != 1) return fail("normalize must be 0 or 1, not %d", normalize);
    if (layer_norm != 0 && layer_norm != 1) return fail("layer_norm must be 0 (GroupNorm) or 1 (LayerNorm), not %d", layer_norm);
    if (out_fmt != 0 && out_fmt != 1) return fail("out_fmt must be 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    const int64_t L0 = conv_out_len(max_len, 0);
    if ((int64_t)B * L0 > 2000000000LL) return fail("batch too large for 32-bit tile indexing");
    cudaStream_t st = (cudaStream_t)stream;
    DevBuf book, pad, stats, part, ss;
    SplitBuf os;
    S3B_OK(book.ensure((size_t)B * (sizeof(void*) + sizeof(long long))));
    std::vector<long long> hl(lens, lens + B);
    CUDA_OK(cudaMemcpyAsync(book.p, wavs, (size_t)B * sizeof(void*), cudaMemcpyHostToDevice, st));
    long long* d_lens = reinterpret_cast<long long*>(book.as<char>() + (size_t)B * sizeof(void*));
    CUDA_OK(cudaMemcpyAsync(d_lens, hl.data(), (size_t)B * sizeof(long long), cudaMemcpyHostToDevice, st));
    float* wav_pad = wav_out;
    if (wav_pad == nullptr) {
        S3B_OK(pad.ensure((size_t)B * max_len * 4));
        wav_pad = pad.as<float>();
    }
    S3B_OK(stats.ensure((size_t)B * 2 * 4));
    S3B_OK(part.ensure(conv0_ws_part_bytes(B, (int)L0)));
    S3B_OK(ss.ensure((size_t)2 * B * kConvDim * 4));
    S3B_OK(os.ensure((size_t)B * L0 * kConvDim));
    S3B_OK(launch_frontend(nullptr, st, book.as<const float*>(), d_lens, B, max_len, (int)L0, normalize, w, bias,
                           gamma, beta, layer_norm, wav_pad, stats.as<float>(), part.as<double>(), ss.as<float>(),
                           os.planes(out_fmt)));
    CUDA_OK(launch_planes_to_f32(os.planes(out_fmt), (size_t)B * L0 * kConvDim, out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

// add_fbank_frontend's step for a DeCoAR 2.0 (step 2) or APC (step 1) model on workspaces of this call; the operand
// planes decoded, columns 0..79 kept
static int fbank_cmvn_features(const float* const* wavs, const int64_t* lens, int32_t B, int step, int32_t out_fmt,
                               float* out, void* stream) {
    if (!wavs || !lens || !out) return fail("null argument");
    if (B < 1) return fail("bad batch %d", B);
    if (out_fmt != 0 && out_fmt != 1) return fail("out_fmt must be 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    int64_t max_len = 0;
    for (int b = 0; b < B; ++b) {
        if (wavs[b] == nullptr) return fail("null argument: wavs[%d]", b);
        if (lens[b] < kDecoar2MinLen)
            return fail("lens[%d] = %lld: %s needs >= %lld samples (2 fbank frames)", b, (long long)lens[b],
                        step == 1 ? "APC" : "DeCoAR 2.0",
                        (long long)kDecoar2MinLen);
        max_len = lens[b] > max_len ? lens[b] : max_len;
    }
    const int64_t mf = fbank_frames(max_len), T = step == 1 ? mf : decoar2_frames(max_len);
    if ((int64_t)B * mf > 2000000000LL) return fail("batch too large for 32-bit indexing");
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    CUDA_OK(init_fbank_tables());
    cudaStream_t st = (cudaStream_t)stream;
    const size_t rows = (size_t)B * T;
    DevBuf book, fbuf, dec;
    SplitBuf os;
    S3B_OK(book.ensure((size_t)B * (sizeof(void*) + sizeof(long long))));
    std::vector<long long> hl(lens, lens + B);
    CUDA_OK(cudaMemcpyAsync(book.p, wavs, (size_t)B * sizeof(void*), cudaMemcpyHostToDevice, st));
    long long* d_lens = reinterpret_cast<long long*>(book.as<char>() + (size_t)B * sizeof(void*));
    CUDA_OK(cudaMemcpyAsync(d_lens, hl.data(), (size_t)B * sizeof(long long), cudaMemcpyHostToDevice, st));
    S3B_OK(fbuf.ensure((size_t)B * mf * 80 * 4));
    S3B_OK(os.ensure(rows * kDecoar2K));
    S3B_OK(dec.ensure(rows * kDecoar2K * 4));
    CUDA_OK(launch_decoar2_features(book.as<const float*>(), d_lens, B, (int)mf, (int)T, step, fbuf.as<float>(),
                                    os.planes(out_fmt), st));
    CUDA_OK(launch_planes_to_f32(os.planes(out_fmt), rows * kDecoar2K, dec.as<float>(), st));
    CUDA_OK(cudaMemcpy2DAsync(out, 80 * sizeof(float), dec.p, kDecoar2K * sizeof(float), 80 * sizeof(float), rows,
                              cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

// SSAST's building blocks (add_ssast_frontend, add_ssast_output) on buffers of the call
extern "C" int s3b_ssast_fbank_f32(const float* const* wavs, const int64_t* lens, int32_t B, int64_t max_len,
                                   int32_t S, float* out, void* stream) {
    if (!wavs || !lens || !out) return fail("null argument");
    if (B < 1) return fail("bad batch %d", B);
    if (S < 400 || S > 160000) return fail("window_samples %d out of range (400..160000)", S);
    for (int b = 0; b < B; ++b) {
        if (wavs[b] == nullptr) return fail("null argument: wavs[%d]", b);
        if (lens[b] < 1 || lens[b] > max_len) return fail("lens[%d]=%lld out of range", b, (long long)lens[b]);
    }
    const int64_t nseg = (max_len + S - 1) / S;
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    CUDA_OK(init_fbank_tables());
    cudaStream_t st = (cudaStream_t)stream;
    DevBuf book;
    S3B_OK(book.ensure((size_t)B * (sizeof(void*) + sizeof(long long))));
    std::vector<long long> hl(lens, lens + B);
    CUDA_OK(cudaMemcpyAsync(book.p, wavs, (size_t)B * sizeof(void*), cudaMemcpyHostToDevice, st));
    long long* d_lens = reinterpret_cast<long long*>(book.as<char>() + (size_t)B * sizeof(void*));
    CUDA_OK(cudaMemcpyAsync(d_lens, hl.data(), (size_t)B * sizeof(long long), cudaMemcpyHostToDevice, st));
    CUDA_OK(launch_ssast_fbank(book.as<const float*>(), d_lens, B, (int)nseg, S, S / 160, out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_ssast_embed_f32(const float* feat, int32_t SB, int32_t TL, int32_t patch, const float* w,
                                   const float* bias, const float* cls, const float* dist, const float* pos,
                                   int32_t scheme, float* planes_out, float* out, void* stream) {
    if (!feat || !w || !bias || !cls || !dist || !pos || !out) return fail("null argument");
    if (patch != 0 && patch != 1) return fail("patch must be 0 or 1, not %d", patch);
    if (SB < 1 || TL < (patch ? 16 : 2)) return fail("bad sizes (segments %d, tl %d)", SB, TL);
    s3b_ssast_config c = {};
    c.patch = patch, c.window_samples = 160 * TL;
    const SsastGeom g = ssast_geom(c);
    const int D = 768, K = 256;
    int sch = 0;
    S3B_OK(resolve_scheme(scheme, K, D, &sch));
    cudaStream_t st = (cudaStream_t)stream;
    int sms = 0;
    S3B_OK(device_sm_count(&sms));
    std::vector<float> wh;
    S3B_OK(download_f32(w, (size_t)D * K, st, wh));
    const std::vector<float> wl = patch ? wh : tap_weight_layout(wh.data(), D, 128, 2, 0, 128);
    SplitBuf ws, as;
    S3B_OK(upload_split(ws, wl.data(), wl.size(), sch));
    const size_t an = patch ? (size_t)SB * g.P * K : (size_t)SB * TL * 128;
    S3B_OK(as.ensure(an));
    CUDA_OK(launch_ssast_patches(feat, SB, TL, g.patch_f, g.tdim, as.planes(sch), st));
    if (planes_out != nullptr) CUDA_OK(launch_planes_to_f32(as.planes(sch), an, planes_out, st));
    GemmParams p;
    S3B_OK(ssast_patch_params(p, g, as, ws, SB, D, sch, out, bias));
    CUDA_OK(launch_gemm(p, sms, st));
    CUDA_OK(launch_ssast_tokens(out, cls, dist, pos, SB, g.P, D, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_ssast_fold_f32(const float* x, int32_t B, int32_t nseg, int32_t TL, int32_t patch, int32_t T,
                                  float* out, void* stream) {
    if (!x || !out) return fail("null argument");
    if (patch != 0 && patch != 1) return fail("patch must be 0 or 1, not %d", patch);
    if (B < 1 || nseg < 1 || TL < (patch ? 16 : 2)) return fail("bad sizes (batch %d, nseg %d, tl %d)", B, nseg, TL);
    s3b_ssast_config c = {};
    c.patch = patch, c.window_samples = 160 * TL;
    const SsastGeom g = ssast_geom(c);
    if (T < 1 || T > nseg * g.tdim) return fail("t_out %d out of range (1..%d)", T, nseg * g.tdim);
    CUDA_OK(launch_ssast_fold(x, B, nseg, g.P, g.tdim, g.patch_f, 768, T, out, (cudaStream_t)stream));
    CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}

extern "C" int s3b_decoar2_features_f32(const float* const* wavs, const int64_t* lens, int32_t B, int32_t out_fmt,
                                        float* out, void* stream) {
    return fbank_cmvn_features(wavs, lens, B, 2, out_fmt, out, stream);
}

extern "C" int s3b_apc_features_f32(const float* const* wavs, const int64_t* lens, int32_t B, int32_t out_fmt,
                                    float* out, void* stream) {
    return fbank_cmvn_features(wavs, lens, B, 1, out_fmt, out, stream);
}

extern "C" int s3b_gru_max_active_clusters(int32_t* out) {
    if (!out) return fail("null argument");
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    int n = 0;
    CUDA_OK(gru_max_active_clusters(&n));
    *out = n;
    return 0;
}

extern "C" int s3b_gru_f32(const float* xg, const float* whh, const float* bhh, const float* residual,
                           const int32_t* lens, int32_t B, int32_t T, int32_t hidden, int32_t out_fmt, float* out,
                           float* planes_out, void* stream) {
    // add_gru_stack's recurrence on this call's buffers: b_hr / b_hz added to a copy of xg as the model's GEMM bias adds
    // them, utterances grouped longest first as the model groups them
    if (!xg || !whh || !bhh || !lens || !out) return fail("null argument");
    if (hidden != kGruHidden) return fail("hidden %d: the recurrence kernel is built for %d", hidden, kGruHidden);
    if (B < 1 || T < 1) return fail("bad sizes (batch %d, t %d)", B, T);
    if (out_fmt < -1 || out_fmt > 1) return fail("out_fmt must be -1 (none), 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    if (out_fmt >= 0 && planes_out == nullptr) return fail("out_fmt %d needs planes_out", out_fmt);
    for (int b = 0; b < B; ++b)
        if (lens[b] < 0 || lens[b] > T) return fail("lens[%d] = %d outside [0, %d]", b, lens[b], T);
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    cudaStream_t st = (cudaStream_t)stream;
    const int H = hidden;
    const size_t M = (size_t)B * T;
    DevBuf xgc, bk;
    SplitBuf os;
    std::vector<int> host(2 * (size_t)B);
    memcpy(host.data(), lens, (size_t)B * sizeof(int));
    std::vector<int> ord(B);
    for (int b = 0; b < B; ++b) ord[b] = b;
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return lens[a] > lens[b]; });
    memcpy(host.data() + B, ord.data(), (size_t)B * sizeof(int));
    S3B_OK(bk.ensure(host.size() * sizeof(int)));
    CUDA_OK(cudaMemcpyAsync(bk.p, host.data(), host.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    S3B_OK(xgc.ensure(M * 3 * H * 4));
    CUDA_OK(cudaMemcpyAsync(xgc.p, xg, M * 3 * H * 4, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(launch_gru_fold_bias(xgc.as<float>(), bhh, M, st));
    GruParams g;
    g.xg = xgc.as<float>(), g.whh = whh, g.bhn = bhh + 2 * H, g.res = residual;
    g.len = bk.as<int>(), g.order = bk.as<int>() + B, g.B = B, g.T = T;
    g.out = out;
    g.op = no_planes();
    if (out_fmt >= 0) {
        S3B_OK(os.ensure(M * H));
        g.op = os.planes(out_fmt);
    }
    CUDA_OK(launch_gru(g, st));
    if (out_fmt >= 0) CUDA_OK(launch_planes_to_f32(g.op, M * H, planes_out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_lstm_fits(int32_t* out) {
    if (!out) return fail("null argument");
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    int ok = 0, sms = 0, smem = 0;
    CUDA_OK(lstm_fits(&ok, &sms, &smem));
    *out = ok;
    return 0;
}

extern "C" int s3b_lstm_f32(const float* xg, const float* whh, const float* bhh, const int32_t* lens, int32_t B,
                            int32_t T, int32_t direction, int32_t out_fmt, float* out, float* planes_out,
                            void* stream) {
    // add_lstm_stack's recurrence on this call's buffers, utterances ordered longest first as the model orders them
    if (!xg || !whh || !lens || !out) return fail("null argument");
    if (B < 1 || T < 1) return fail("bad sizes (batch %d, t %d)", B, T);
    if (direction != 0 && direction != 1) return fail("direction must be 0 (forward) or 1 (backward), not %d", direction);
    if (out_fmt < -1 || out_fmt > 1) return fail("out_fmt must be -1 (none), 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    if (out_fmt >= 0 && planes_out == nullptr) return fail("out_fmt %d needs planes_out", out_fmt);
    for (int b = 0; b < B; ++b)
        if (lens[b] < 0 || lens[b] > T) return fail("lens[%d] = %d outside [0, %d]", b, lens[b], T);
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    int ok = 0, sms = 0, smem = 0;
    CUDA_OK(lstm_fits(&ok, &sms, &smem));
    if (!ok) return fail("the LSTM recurrence kernel cannot run on this device (%d SMs, %d bytes of shared memory)", sms, smem);
    cudaStream_t st = (cudaStream_t)stream;
    const int H = kLstmHidden;
    const size_t M = (size_t)B * T;
    DevBuf bk, hb, sync;
    SplitBuf os;
    std::vector<int> host(2 * (size_t)B);
    memcpy(host.data(), lens, (size_t)B * sizeof(int));
    std::vector<int> ord(B);
    for (int b = 0; b < B; ++b) ord[b] = b;
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return lens[a] > lens[b]; });
    memcpy(host.data() + B, ord.data(), (size_t)B * sizeof(int));
    S3B_OK(bk.ensure(host.size() * sizeof(int)));
    CUDA_OK(cudaMemcpyAsync(bk.p, host.data(), host.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    S3B_OK(hb.ensure(lstm_hbuf_floats(B) * 4));
    S3B_OK(sync.ensure(sizeof(unsigned int)));
    LstmParams g;
    g.xg = xg, g.whh = whh, g.bhh = bhh;
    g.len = bk.as<int>(), g.order = bk.as<int>() + B, g.B = B, g.T = T, g.direction = direction;
    g.out = out, g.ldo = 2 * H, g.col0 = direction * H;
    g.op = no_planes();
    if (out_fmt >= 0) {
        S3B_OK(os.ensure(M * 2 * H));
        g.op = os.planes(out_fmt);
    }
    g.hbuf = hb.as<float>(), g.counter = sync.as<unsigned int>();
    CUDA_OK(launch_lstm(g, st));
    if (out_fmt >= 0) CUDA_OK(launch_planes_to_f32(g.op, M * 2 * H, planes_out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_conformer_conv_f32(const float* x, int32_t B, int32_t T, int32_t D, int32_t k, const float* dw_w,
                                      const float* bn_gamma, const float* bn_beta, const float* bn_mean,
                                      const float* bn_var, int32_t out_fmt, float* out, void* stream) {
    // add_conformer_layer's depthwise step on this call's buffers: BatchNorm folded on the host like s3b_model_finalize does it
    if (!x || !dw_w || !bn_gamma || !bn_beta || !bn_mean || !bn_var || !out) return fail("null argument");
    if (B < 1 || T < 1) return fail("bad sizes (batch %d, t %d)", B, T);
    if (D < 64 || D % 64 != 0) return fail("d must be a positive multiple of 64, not %d", D);
    if (k < 1 || k > kDwMaxKernel || k % 2 == 0) return fail("kernel size %d: must be odd, 1..%d", k, kDwMaxKernel);
    if (out_fmt != 0 && out_fmt != 1) return fail("out_fmt must be 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t M = (size_t)B * T;
    DevBuf wb, bb;
    SplitBuf os;
    std::vector<float> w, g, be, mu, var, wf, bf;
    S3B_OK(download_f32(dw_w, (size_t)D * k, st, w));
    S3B_OK(download_f32(bn_gamma, D, st, g));
    S3B_OK(download_f32(bn_beta, D, st, be));
    S3B_OK(download_f32(bn_mean, D, st, mu));
    S3B_OK(download_f32(bn_var, D, st, var));
    fold_depthwise_bn(w.data(), g.data(), be.data(), mu.data(), var.data(), D, k, wf, bf);
    S3B_OK(upload_f32(wb, wf.data(), wf.size()));
    S3B_OK(upload_f32(bb, bf.data(), bf.size()));
    S3B_OK(os.ensure(M * D));
    CUDA_OK(launch_depthwise_glu(x, B, T, D, k, wb.as<float>(), bb.as<float>(), os.planes(out_fmt), st));
    CUDA_OK(launch_planes_to_f32(os.planes(out_fmt), M * D, out, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int s3b_layernorm_rope_f32(const float* x, int64_t M, int32_t T, int32_t D, const float* gamma,
                                      const float* beta, const float* inv_freq, int32_t out_fmt, float* out,
                                      float* out_rope, void* stream) {
    // add_conformer_layer's LayerNorm + RoPE kernel, with a table built for the t frames like build_rope_table
    if (!x || !gamma || !beta || !out || !out_rope) return fail("null argument");
    if (M < 1 || T < 1 || M % T != 0) return fail("m = %lld must be a positive multiple of t = %d", (long long)M, T);
    if (D != 512 && D != 768 && D != 1024 && D != 1280) return fail("d must be 512, 768, 1024 or 1280, not %d", D);
    if (out_fmt != 0 && out_fmt != 1) return fail("out_fmt must be 0 (bf16 hi/lo) or 1 (f16q8), not %d", out_fmt);
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<float> f = inv_freq ? std::vector<float>(inv_freq, inv_freq + 32) : default_inv_freq();
    const std::vector<float> cs = rope_table(f, T);
    DevBuf table;
    SplitBuf y, yr;
    S3B_OK(table.ensure(cs.size() * 4));
    CUDA_OK(cudaMemcpyAsync(table.p, cs.data(), cs.size() * 4, cudaMemcpyHostToDevice, st));
    S3B_OK(y.ensure((size_t)M * D));
    S3B_OK(yr.ensure((size_t)M * D));
    CUDA_OK(launch_layernorm_rope(x, (size_t)M, T, D, gamma, beta, table.as<float>(), y.planes(out_fmt),
                                  yr.planes(out_fmt), st));
    CUDA_OK(launch_planes_to_f32(y.planes(out_fmt), (size_t)M * D, out, st));
    CUDA_OK(launch_planes_to_f32(yr.planes(out_fmt), (size_t)M * D, out_rope, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// fbank baseline (s3prl/upstream/baseline/expert.py:69-79)
// ------------------------------------------------------------------------------------------------
#include "fbank.cuh"

extern "C" int64_t s3b_fbank_num_frames(int64_t len) { return len < 400 ? 0 : 1 + (len - 400) / 160; }

// Device memory owned by one call and released in the order of that call's stream (stream-ordered allocator). Every
// call stages its pointers and lengths, and keeps its intermediates, in blocks of its own, so a later call on another
// stream cannot overwrite what a call still queued will read.
struct StreamBuf {
    void* p = nullptr;
    cudaStream_t s;
    explicit StreamBuf(cudaStream_t st) : s(st) {}
    StreamBuf(const StreamBuf&) = delete;
    StreamBuf& operator=(const StreamBuf&) = delete;
    ~StreamBuf() {
        if (p) cudaFreeAsync(p, s);
    }
    int alloc(size_t n) {
        cudaError_t e = cudaMallocAsync(&p, n, s);
        if (e != cudaSuccess) {
            p = nullptr;
            return fail("cudaMallocAsync(%zu) failed: %s", n, cudaGetErrorString(e));
        }
        return 0;
    }
    template <class T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};

static int check_spectral_opts(const s3b_spectral_opts* opts) {
    if (opts != nullptr && opts->struct_size != (int32_t)sizeof(s3b_spectral_opts))
        return fail("s3b_spectral_opts.struct_size %d != %d (header / library mismatch)", opts->struct_size,
                    (int)sizeof(s3b_spectral_opts));
    if (opts != nullptr && opts->cmvn != 0 && opts->cmvn != 1) return fail("cmvn must be 0 or 1, not %d", opts->cmvn);
    return 0;
}

static int check_lengths(const int64_t* lens, int32_t batch) {
    for (int b = 0; b < batch; ++b)
        if (lens[b] < 0) return fail("lens[%d] = %lld is negative", b, (long long)lens[b]);
    return 0;
}

extern "C" int s3b_fbank_ex(const float* const* wavs, const int64_t* lens, int32_t batch,
                            const s3b_spectral_opts* opts, float* out, void* stream) {
    if (!wavs || !lens || !out) return fail("null argument");
    if (batch < 1) return fail("empty batch");
    S3B_OK(check_spectral_opts(opts));
    S3B_OK(check_lengths(lens, batch));
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    const int cmvn = opts ? opts->cmvn : 1;
    cudaStream_t st = (cudaStream_t)stream;
    int64_t max_len = 0;
    for (int b = 0; b < batch; ++b) max_len = lens[b] > max_len ? lens[b] : max_len;
    const int64_t max_frames = s3b_fbank_num_frames(max_len);
    if (max_frames < 1) return fail("waveforms shorter than one 25 ms frame");
    StreamBuf scratch(st);
    S3B_OK(scratch.alloc((size_t)batch * (sizeof(void*) + sizeof(long long))));
    std::vector<long long> l64(lens, lens + batch);
    const float** d_ptrs = scratch.as<const float*>();
    long long* d_lens = reinterpret_cast<long long*>(scratch.as<char>() + (size_t)batch * sizeof(void*));
    CUDA_OK(cudaMemcpyAsync(d_ptrs, wavs, batch * sizeof(void*), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(d_lens, l64.data(), batch * sizeof(long long), cudaMemcpyHostToDevice, st));
    CUDA_OK(launch_fbank(d_ptrs, d_lens, batch, (int)max_frames, cmvn, out, st));
    return 0;
}

extern "C" int s3b_fbank(const float* const* wavs, const int64_t* lens, int32_t batch, float* out, void* stream) {
    return s3b_fbank_ex(wavs, lens, batch, nullptr, out, stream);
}

// ------------------------------------------------------------------------------------------------
// mel / linear baselines (s3prl/upstream/baseline/expert.py:52-79 over preprocessor.py:150-223)
// ------------------------------------------------------------------------------------------------
extern "C" int s3b_trimmed_lengths(const float* const* wavs, const int64_t* lens, int32_t batch, int64_t* out) {
    if (!wavs || !lens || !out) return fail("null argument");
    S3B_OK(check_lengths(lens, batch));
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    DevBuf scratch;
    S3B_OK(scratch.ensure((size_t)batch * (sizeof(void*) + 2 * sizeof(long long))));
    const float** d_ptrs = scratch.as<const float*>();
    long long* d_lens = reinterpret_cast<long long*>(scratch.as<char>() + (size_t)batch * sizeof(void*));
    long long* d_out = d_lens + batch;
    std::vector<long long> l64(lens, lens + batch), res(batch);
    CUDA_OK(cudaMemcpy(d_ptrs, wavs, batch * sizeof(void*), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_lens, l64.data(), batch * sizeof(long long), cudaMemcpyHostToDevice));
    CUDA_OK(launch_trimmed_lengths(d_ptrs, d_lens, batch, d_out, 0));
    CUDA_OK(cudaMemcpy(res.data(), d_out, batch * sizeof(long long), cudaMemcpyDeviceToHost));
    for (int b = 0; b < batch; ++b) out[b] = res[b];
    return 0;
}

extern "C" int s3b_melspec_ex(const float* const* wavs, const int64_t* trimmed_lens, int32_t batch,
                              int64_t padded_len, int32_t mel, const int32_t* feats_len, const int32_t* final_len,
                              int32_t t_out, const s3b_spectral_opts* opts, float* out, void* stream) {
    S3B_OK(check_spectral_opts(opts));
    const int cmvn = opts ? opts->cmvn : 1;
    if (!wavs || !trimmed_lens || !out || (cmvn && (!feats_len || !final_len))) return fail("null argument");
    if (batch < 1 || padded_len < 1 || (cmvn && t_out < 1)) return fail("bad sizes");
    const int64_t n_frames = 1 + padded_len / 160;
    for (int b = 0; b < batch; ++b) {
        if (trimmed_lens[b] < 0 || trimmed_lens[b] > padded_len)
            return fail("trimmed_lens[%d] = %lld outside [0, padded_len = %lld]", b, (long long)trimmed_lens[b],
                        (long long)padded_len);
        if (!cmvn) continue;
        // mel_cmvn_kernel reads feats_len[b] rows of utterance b's n_frames-row block of tmp
        if (feats_len[b] < 0 || feats_len[b] > n_frames)
            return fail("feats_len[%d] = %d outside [0, 1 + padded_len / 160 = %lld]", b, feats_len[b],
                        (long long)n_frames);
        if (final_len[b] < 0 || final_len[b] > t_out)
            return fail("final_len[%d] = %d outside [0, t_out = %d]", b, final_len[b], t_out);
    }
    if (s3b_device_count() == 0) return fail("no CUDA device: s3prl_b200 has no CPU fallback");
    cudaStream_t st = (cudaStream_t)stream;
    const int dim = mel ? 80 : 201;
    StreamBuf scratch(st), tmp(st);
    S3B_OK(scratch.alloc((size_t)batch * (sizeof(void*) + sizeof(long long) + 2 * sizeof(int))));
    if (cmvn) S3B_OK(tmp.alloc((size_t)batch * n_frames * dim * 4));
    const float** d_ptrs = scratch.as<const float*>();
    long long* d_lens = reinterpret_cast<long long*>(scratch.as<char>() + (size_t)batch * sizeof(void*));
    int* d_fl = reinterpret_cast<int*>(d_lens + batch);
    int* d_kl = d_fl + batch;
    std::vector<long long> l64(trimmed_lens, trimmed_lens + batch);
    CUDA_OK(cudaMemcpyAsync(d_ptrs, wavs, batch * sizeof(void*), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(d_lens, l64.data(), batch * sizeof(long long), cudaMemcpyHostToDevice, st));
    if (cmvn) {
        CUDA_OK(cudaMemcpyAsync(d_fl, feats_len, batch * sizeof(int), cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaMemcpyAsync(d_kl, final_len, batch * sizeof(int), cudaMemcpyHostToDevice, st));
    }
    CUDA_OK(launch_melspec(d_ptrs, d_lens, batch, padded_len, mel, cmvn, d_fl, d_kl, t_out, tmp.as<float>(), out, st));
    return 0;
}

extern "C" int s3b_melspec(const float* const* wavs, const int64_t* trimmed_lens, int32_t batch, int64_t padded_len,
                           int32_t mel, const int32_t* feats_len, const int32_t* final_len, int32_t t_out, float* out,
                           void* stream) {
    return s3b_melspec_ex(wavs, trimmed_lens, batch, padded_len, mel, feats_len, final_len, t_out, nullptr, out,
                          stream);
}
