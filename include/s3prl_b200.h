/*
 * s3prl_b200 — C ABI of the Hopper (sm_90a, H100) upstream feature-extraction hot path.
 *
 * Plain pointers and sizes only (no torch types). Every entry point returns 0 on success and a
 * non-zero status otherwise; s3b_last_error() returns a thread-local message for the last failure.
 * The Python binding a reference maintainer would add is the ctypes stub in INTEGRATION.md
 * (ours: s3prl_b200/lib.py). Citations are to the reference tree s3prl/s3prl @ 0.4.18.
 */
#ifndef S3PRL_B200_H_
#define S3PRL_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct s3b_model s3b_model;

/* Architecture of one wav2vec2 / HuBERT / WavLM upstream.
 * Mirrors the fields of HubertConfig (s3prl/upstream/hubert/hubert_model.py:76-278),
 * Wav2Vec2Config (s3prl/upstream/wav2vec2/wav2vec2_model.py:2103-2350) and
 * WavLMConfig (s3prl/upstream/wavlm/WavLM.py:162-245) that the extraction forward reads. */
typedef struct s3b_config {
    int32_t family;               /* 0 = hubert, 1 = wav2vec2 and data2vec, 2 = wavlm, 3 = distiller (selects the frame-mask rule) */
    int32_t extractor_layer_norm; /* 0: extractor_mode "default" (GroupNorm after conv 0); 1: "layer_norm" */
    int32_t conv_bias;            /* conv_bias */
    int32_t layer_norm_first;     /* pre-LN transformer (large_ll60k, wavlm_large) */
    int32_t normalize_wav;        /* task_cfg.normalize: per-utterance F.layer_norm of the waveform */
    int32_t num_layers;           /* encoder_layers */
    int32_t embed_dim;            /* encoder_embed_dim (multiple of 128) */
    int32_t ffn_dim;              /* encoder_ffn_embed_dim */
    int32_t num_heads;            /* encoder_attention_heads; head dim embed_dim / num_heads: 64, 80 or 120 (64 for a
                                   * Conformer or the wavlm family) */
    int32_t pos_conv_kernel;      /* conv_pos (128; data2vec 95) */
    int32_t pos_conv_groups;      /* conv_pos_groups (16) */
    int32_t relative_position;    /* WavLM relative_position_embedding */
    int32_t num_buckets;          /* WavLM num_buckets (320) */
    int32_t max_distance;         /* WavLM max_distance (800) */
    int32_t gru_rel_pos;          /* WavLM gru_rel_pos */
    /* Distiller / DistilHuBERT (s3prl/upstream/distiller/model.py:81-269): */
    int32_t no_feature_layer_norm; /* 1: post_extract_proj takes the conv features directly (no LayerNorm(512)) */
    int32_t pred_heads;            /* n_tasks prediction heads Linear -> GELU -> SplitLinear on the encoder output (0: none) */
    int32_t pos_conv_depth;        /* 0 / 1: one weight-normed conv of pos_conv_kernel taps (make_conv_pos); > 1 (data2vec):
                                      that many blocks Conv1d(k) -> LayerNorm(no affine) -> GELU with
                                      k = max(3, pos_conv_kernel / pos_conv_depth) (wav2vec2_model.py:2995-3026) */
    /* wav2vec 2.0 Conformer (layer_type "conformer", attn_type "espnet", pos_enc_type "rope";
     * ConformerEncoder wav2vec2_model.py:3132-3211, ConformerEncoderLayer :441-578). 1 needs family 1; the positional
     * conv fields are then unused (the encoder has no pos_conv) and rotary attention is implied. */
    int32_t conformer;            /* 0: transformer layers; 1: Conformer layers */
    int32_t depthwise_kernel;     /* depthwise_conv_kernel_size of the convolution module: odd, 1..63 (conformer only) */
    /* 0: the waveform conv stack (feature_extractor.*, layer_norm.*) in front of post_extract_proj [D][512].
     * 1: DeCoAR 2.0 (s3prl/upstream/decoar2/{audio,decoar2,expert}.py): per utterance kaldi fbank (80 mel bins, 25 ms /
     *    10 ms, hamming window, snip_edges) -> CMVN over all m frames (unbiased std) -> every second frame, T_b =
     *    (m_b + 1) / 2, into post_extract_proj [D][80]; frame t of utterance b is padding iff t >= T_b. Needs family 1 and
     *    a transformer encoder with pos_conv_depth <= 1; the conv-stack fields (extractor_layer_norm, conv_bias,
     *    normalize_wav, no_feature_layer_norm) must be 0. Utterances need >= 560 samples (2 fbank frames). */
    int32_t frontend;
    /* 1: output slot 0 is the post_extract_proj output with its padded frames zeroed (LightHuBERT,
     * s3prl/upstream/lighthubert/lighthubert.py:687-783: hidden_states[0] is `features`, which the encoder's in-place
     * index_put zeroes), instead of the encoder's layer-0 input. Needs family 0, a post-LN transformer encoder and
     * frontend 0. 0: the encoder's layer-0 input, as for every other model of the family. */
    int32_t proj_hidden0;
    int32_t reserved[1];
} s3b_config;

/* Library / error ------------------------------------------------------------------------------ */
int s3b_version(void);
const char* s3b_last_error(void);
/* number of CUDA devices visible (0 on a GPU-less host; never fails) */
int s3b_device_count(void);

/* Model lifetime --------------------------------------------------------------------------------
 * Replaces load_converted_model + HubertModel(...).load_state_dict
 * (s3prl/upstream/hubert/convert.py:37-56, wav2vec2/convert.py:26-39, wavlm/expert.py:37-44).
 * Tensors are passed by their reference state-dict key, fp32, host memory, C-contiguous.
 * Unknown keys (pre-training heads: mask_emb, final_proj, quantizer.*, ...) are ignored.
 * s3b_model_finalize folds weight_norm of pos_conv, re-lays conv weights for channels-last implicit GEMM,
 * splits every GEMM weight into bf16 hi/lo, uploads to the current CUDA device. */
int s3b_model_create(const s3b_config* cfg, s3b_model** out);
int s3b_model_set_tensor(s3b_model* m, const char* name, const float* data, const int64_t* shape, int32_t ndim);

/* APC / VQ-APC (s3prl/upstream/apc/{expert,apc,audio}.py, vq_apc/expert.py). Per utterance kaldi fbank (80 mel bins,
 * 25 ms / 10 ms, hamming window, snip_edges), CMVN over all m frames (unbiased std), pad_sequence to T = max m, then
 * num_layers single-layer GRUs (gate order r, z, n; h_0 = 0) over the packed sequences; layer l > 0 adds its input when
 * residual is set. Frame t of utterance b is padding iff t >= m_b, and every output there is exactly 0.
 * Tensors (s3b_model_set_tensor, reference key names): rnn_layers.{l}.weight_ih_l0 [3H][80 or H], .weight_hh_l0
 * [3H][H], .bias_ih_l0 [3H], .bias_hh_l0 [3H]; other keys (postnet.*, vq_layers.*) are ignored.
 * The model then works with s3b_model_finalize, s3b_forward / _ex / _host / _host_ex, s3b_num_frames (m of max_len),
 * s3b_valid_frames (m_b; lens[b] >= 560 samples, since the std of one frame is NaN), s3b_default_lanes and the
 * profile calls. s3b_num_outputs = num_layers: hidden_out holds the output of every layer ([num_layers][batch][T][H]).
 * s3b_forward_ex refuses ffn_out and last_residual. Served: num_layers 3, hidden 512; finalize fails when the device
 * cannot hold one cluster of the recurrence kernel (16 CTAs, 209 KB of shared memory each). */
typedef struct s3b_apc_config {
    int32_t struct_size; /* sizeof(s3b_apc_config) */
    int32_t num_layers;  /* config["model"]["paras"]["num_layers"] */
    int32_t hidden;      /* hidden_size */
    int32_t residual;    /* residual: 0 or 1 */
    int32_t reserved[4]; /* 0 */
} s3b_apc_config;
int s3b_apc_model_create(const s3b_apc_config* cfg, s3b_model** out);

/* DeCoAR (s3prl/upstream/decoar/{expert,decoar,audio}.py, decoar_layers/{expert,decoar}.py). The APC front end
 * (kaldi fbank, 80 bins, hamming window, CMVN over all m frames with the unbiased std, pad_sequence to T = max m),
 * post_extract_proj = Linear(80, 1024), then two 4-layer nn.LSTM(1024, 1024) stacks (gate order i, f, g, o; h_0 =
 * c_0 = 0) over the packed sequences: forward_lstm in time order, backward_lstm over each utterance reversed within
 * its own length. Layer k's output is cat(forward, backward) [batch][T][2048]; frames t >= m_b are exactly 0.
 * Tensors (s3b_model_set_tensor, reference key names): post_extract_proj.{weight [1024][80], bias},
 * {forward,backward}_lstm.{weight_ih_l{k} [4096][1024], weight_hh_l{k} [4096][1024], bias_ih_l{k}, bias_hh_l{k}},
 * k = 0..3; other keys are ignored. s3b_num_outputs = 1 (all_layers 0, `decoar`: the last layer) or 4 (all_layers 1,
 * `decoar_layers`: every layer); hidden_out is [num_outputs][batch][T][2048]. The model works with the calls listed
 * for APC; s3b_forward_ex refuses ffn_out and last_residual. The recurrence is grid-resident: one cooperative launch
 * of 128 CTAs, one per SM, with 212.5 KiB of shared memory each (s3b_lstm_fits). So finalize fails on a device with
 * fewer than 128 SMs or less opt-in shared memory, and a forward always runs as one lane (s3b_default_lanes is 1 and
 * lanes = 2 runs as one): two such launches must never be in flight at once, so do not run two DeCoAR forwards
 * concurrently on one device. */
typedef struct s3b_decoar_config {
    int32_t struct_size; /* sizeof(s3b_decoar_config) */
    int32_t num_layers;  /* 4 */
    int32_t hidden;      /* 1024 */
    int32_t all_layers;  /* 0 = decoar, 1 = decoar_layers */
    int32_t reserved[4]; /* 0 */
} s3b_decoar_config;
int s3b_decoar_model_create(const s3b_decoar_config* cfg, s3b_model** out);
/* NPC (s3prl/upstream/npc/{expert,npc,audio}.py). The APC front end (kaldi fbank, 80 bins, hamming window, CMVN over
 * all m frames with the unbiased std, pad_sequence to T = max m), then n_blocks blocks: ConvBlock i is
 * act(bn2(linear(act(bn1(conv(x))))) (+ x when residual and i > 0)), with conv = Conv1d(k 3, padding 1) (80 input
 * channels in block 0, 512 after) and linear = Conv1d(512, 512, 1); masked conv i is tanh(Conv1d(512, 512,
 * kernel_size, padding (kernel_size - 1) / 2)) with a centred band of mask_size + 2 (i + 1) taps masked out; feat =
 * the sum of the masked convs. Frames t >= m_b are NOT zero: they hold the response to the zero padding features, and
 * valid frames near m_b read them, so an utterance's result depends on T (as in the reference).
 * Tensors (reference key names): blocks.{i}.conv.{weight [512][80 or 512][3], bias}, blocks.{i}.linear.{weight
 * [512][512][1], bias}, with batch_norm blocks.{i}.bn{1,2}.{weight, bias, running_mean, running_var};
 * masked_convs.{i}.conv.{weight [512][512][kernel_size], bias} and masked_convs.{i}.conv_mask (same shape). Other
 * keys (vq_layers.*, postnet.*, num_batches_tracked) are ignored. Finalize folds each BatchNorm (eps 1e-5) into the
 * conv before it, multiplies each masked weight by its conv_mask and fails, naming the block, if weight is left on
 * a tap the config masks; only the unmasked taps are computed.
 * s3b_num_outputs = 2 n_blocks + 1: hidden_out is [block 0, masked conv 0, block 1, ..., masked conv n-1, feat]
 * [batch][T][512]. The model works with the calls listed for APC; lens[b] >= 560 samples; s3b_forward_ex refuses
 * ffn_out and last_residual. Served: hidden 512, odd kernel_size > mask_size + 2 n_blocks, odd mask_size. */
typedef struct s3b_npc_config {
    int32_t struct_size; /* sizeof(s3b_npc_config) */
    int32_t n_blocks;    /* config["model"]["paras"]["n_blocks"], 1..32 */
    int32_t hidden;      /* hidden_size: 512 */
    int32_t kernel_size; /* masked conv kernel (odd) */
    int32_t mask_size;   /* odd; masked conv i masks mask_size + 2 (i + 1) centred taps */
    int32_t residual;    /* 0 or 1 */
    int32_t batch_norm;  /* 0 or 1 */
    int32_t act;         /* activate: 0 = relu, 1 = tanh */
    int32_t reserved[4]; /* 0 */
} s3b_npc_config;
int s3b_npc_model_create(const s3b_npc_config* cfg, s3b_model** out);
/* Modified CPC (s3prl/upstream/cpc/{expert,model}.py): pad_sequence of the waveforms (no normalisation), then the
 * encoder: five Conv1d(k = 2 s) with strides 5, 4, 2, 2, 2 and paddings 3, 2, 1, 1, 1 (1 -> 256 channels, then 256 ->
 * 256), each followed by ChannelNorm (per frame over the 256 channels, unbiased variance, rsqrt(var + 1e-5)) and ReLU;
 * then nn.LSTM(256, 256, num_layers) over the whole padded batch (no packing, h0 = c0 = 0, gate order i, f, g, o).
 * T = the conv chain over max_len (159 samples -> 1 frame, 16000 -> 100); max_len < 159 yields no frame. Individual
 * utterances may be shorter. Frames are not masked: the frames near and after an utterance's end hold the model's
 * response to the zero samples, so the last frame of an utterance (and those after it) depend on max_len.
 * Tensors (reference key names, CPCModel.state_dict()): gEncoder.conv{i}.{weight [256][1 or 256][2 s], bias [256]},
 * gEncoder.batchNorm{i}.{weight, bias} [1][256][1] for i = 0..4; gAR.baseNet.{weight_ih_l{k} [1024][256],
 * weight_hh_l{k} [1024][256], bias_ih_l{k}, bias_hh_l{k} [1024]} for k < num_layers.
 * s3b_num_outputs = 2: hidden_out is [encoder output, last LSTM layer's output] [batch][T][256]. s3b_forward_ex refuses
 * ffn_out and last_residual. Served: hidden 256, num_layers 1..8. */
typedef struct s3b_cpc_config {
    int32_t struct_size; /* sizeof(s3b_cpc_config) */
    int32_t hidden;      /* hiddenEncoder = hiddenGar: 256 */
    int32_t num_layers;  /* nLevelsGRU: LSTM layers, 1..8 */
    int32_t reserved[4]; /* 0 */
} s3b_cpc_config;
int s3b_cpc_model_create(const s3b_cpc_config* cfg, s3b_model** out);
/* SSAST (s3prl/upstream/ssast/{expert,audio,ast_models}.py): every utterance zero-padded to nseg = ceil(max_len / S)
 * windows of S = window_samples samples; per window kaldi fbank (128 mel bins, 25 ms / 10 ms, hanning window,
 * snip_edges), y = (y + 4.2677393) / 9.1379948, zero rows appended up to TL = S / 160 frames; the patch embedding
 * Conv2d over x[f][t] (frame model: kernel (128, 2), stride (128, 1), P = TL - 1 patches; patch model: kernel (16, 16),
 * stride (10, 10), P = 12 t_dim patches, t_dim = (TL - 16) / 10 + 1, in (f, t) row-major order); the sequence
 * [cls_token, dist_token, patches] + pos_embed; 12 pre-LN DeiT blocks (LayerNorm eps 1e-6, 12 heads of 64, FFN 3072,
 * exact GELU), every token of a window attending to the 2 + P tokens of its window. No final norm.
 * Hidden state l is block l's output without the class tokens: frame model [batch][T][768], patch model
 * [batch][T][12 * 768] with column block fi = frequency patch fi; T = min(nseg t_dim, ceil(max_len / rate)), rate 160
 * (frame) or 1600 (patch), t_dim = P for the frame model. Frames are not masked: windows past an utterance's end hold
 * the model's response to silence, as in the reference.
 * Tensors (timm names of ASTModel.v): patch_embed.proj.weight [768][1][128][2] or [768][1][16][16], patch_embed.proj.bias,
 * cls_token and dist_token [1][1][768], pos_embed [1][2 + P][768] (already re-gridded to the window, as the reference's
 * fine-tuning constructor does), blocks.{l}.{norm1, norm2}.{weight, bias}, blocks.{l}.attn.qkv.{weight [2304][768],
 * bias}, blocks.{l}.attn.proj.*, blocks.{l}.mlp.{fc1, fc2}.*; other keys are ignored.
 * s3b_num_outputs = num_layers (12); s3b_valid_frames gives min(T, ceil(lens[b] / rate)); s3b_forward_ex refuses ffn_out
 * and last_residual. Served: the base model only (embed_dim 768, num_heads 12, num_layers 12); window_samples from 400
 * (frame) or 2560 (patch) to 160000 (10 s). */
typedef struct s3b_ssast_config {
    int32_t struct_size;    /* sizeof(s3b_ssast_config) */
    int32_t patch;          /* 0 = frame model (base_f), 1 = patch model (base_p) */
    int32_t window_samples; /* int(window_secs * 16000) */
    int32_t embed_dim;      /* 768 */
    int32_t num_heads;      /* 12 */
    int32_t num_layers;     /* 12 */
    int32_t reserved[4];    /* 0 */
} s3b_ssast_config;
int s3b_ssast_model_create(const s3b_ssast_config* cfg, s3b_model** out);
/* MAE-AST (s3prl/upstream/mae_ast/{expert,mae_ast}.py): per utterance kaldi fbank (128 mel bins, povey window,
 * 25 ms / 10 ms, snip_edges), zero-padded to the batch's F = 1 + (max_len - 400) / 160 frames; y = (x - running_mean)
 * * rsqrt(running_var + 1e-5) * 0.5 on every element (padded frames too); unfold into (kt, kc) patches, (2, 128) for
 * the frame model and (16, 16) for the patch model: T' = F / kt time patches of nv = 128 / kc frequency patches, token
 * t * nv + fi, column i * kc + j; post_extract_proj Linear(256, 768); with sine_pos, rows 0 .. T' nv - 1 of the
 * checkpoint's sinusoid table added to the valid tokens; then num_layers wav2vec 2.0 encoder layers (12 heads of 64,
 * FFN 3072, exact GELU), post-LN with encoder.layer_norm on their input, or pre-LN without any encoder norm. Keys of
 * utterance b are valid for its first valid_b = min(ceil(n_b / kt), T') nv tokens, n_b its own fbank frames.
 * Hidden state l is layer l's output, [batch][T'][nv * 768]. s3b_num_outputs = num_layers; s3b_valid_frames gives
 * min(ceil(n_b / kt), T'), and refuses lens[b] < 400; s3b_forward_ex refuses ffn_out and last_residual, and a batch of
 * more than max_tokens tokens when sine_pos is set.
 * Tensors: post_extract_proj.{weight [768][256], bias}, batch_norm.running_mean [1], batch_norm.running_var [1],
 * enc_sine_pos_embed.pe [1][max_tokens][768] (sine_pos), encoder.layer_norm.* (post-LN), and per layer
 * encoder.layers.{l}.self_attn.{q,k,v,out}_proj.*, self_attn_layer_norm.*, fc1.*, fc2.*, final_layer_norm.*; other
 * keys are ignored. */
typedef struct s3b_mae_ast_config {
    int32_t struct_size;      /* sizeof(s3b_mae_ast_config) */
    int32_t patch;            /* 0 = frame model (2 x 128 patches), 1 = patch model (16 x 16) */
    int32_t embed_dim;        /* 768 */
    int32_t num_heads;        /* 12 */
    int32_t ffn_dim;          /* 3072 */
    int32_t num_layers;       /* encoder_layers, 1..63 */
    int32_t layer_norm_first; /* 0 = post-LN, 1 = pre-LN */
    int32_t sine_pos;         /* enc_sine_pos: 0 or 1 */
    int32_t max_tokens;       /* rows of enc_sine_pos_embed.pe (sine_pos 1), else 0 */
    int32_t reserved[4];      /* 0 */
} s3b_mae_ast_config;
int s3b_mae_ast_model_create(const s3b_mae_ast_config* cfg, s3b_model** out);
int s3b_model_finalize(s3b_model* m);
void s3b_model_destroy(s3b_model* m);

/* Frame bookkeeping (bit-exact integer rules) ------------------------------------
 * T = conv-stack output length for a padded batch of max length max_len
 * (ConvFeatureExtractionModel, wav2vec2_model.py:2857-2934); m may be NULL. For a DeCoAR 2.0 model (frontend 1)
 * T = (1 + (max_len - 400) / 160 + 1) / 2. Returns -1 if max_len is too short (below 400 samples for DeCoAR 2.0). */
int64_t s3b_num_frames(const s3b_model* m, int64_t max_len);
/* valid_frames[b] = number of un-padded frames of utterance b inside a batch padded to max_len:
 * HuBERT/WavLM chunk-all rule (hubert_model.py:454-464, WavLM.py:339-349) or the wav2vec2 conv-length
 * rule (wav2vec2_model.py:2610-2625,2652-2671); DeCoAR 2.0: (1 + (lens[b] - 400) / 160 + 1) / 2, lens[b] >= 560.
 * frame t of utterance b is padding iff t >= valid_frames[b]. */
int s3b_valid_frames(const s3b_model* m, const int64_t* lens, int32_t batch, int64_t max_len, int32_t* valid_frames);

/* The hot path ------------------------------------------------------------------------------------
 * Replaces UpstreamExpert.forward + hooks (hubert/expert.py:36-72, wav2vec2/expert.py:61-97,
 * wavlm/expert.py:45-87, interfaces.py:100-131).
 *  wavs        : host array of `batch` DEVICE pointers to fp32 waveforms (un-padded, any order)
 *  lens        : host array of `batch` lengths (samples)
 *  max_len     : padded batch length Lmax (>= max(lens); equal to it for single-GPU use; the global max of
 *                the un-sharded batch when the batch is sharded across ranks)
 *  hidden_out  : DEVICE buffer [s3b_num_outputs(m)][batch][T][embed_dim] fp32, T = s3b_num_frames(max_len):
 *                num_layers+1 hidden states (input of every layer + encoder output); for a distiller model
 *                (distiller/expert.py:44-63) feat_final, the num_layers layer outputs, then the pred_heads predictions
 *  stream      : cudaStream_t the work is enqueued on (asynchronous with respect to the host) */
int32_t s3b_num_outputs(const s3b_model* m);
int s3b_forward(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len,
                float* hidden_out, void* stream);
/* Same, end-to-end from HOST buffers: waveforms are host pointers, hidden_out is a host buffer; the
 * host<->device copies are part of the call, which returns after the result has landed. */
int s3b_forward_host(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len,
                     float* hidden_out);

/* Options of s3b_forward_ex (zero-initialise, set struct_size = sizeof(s3b_forward_opts)).
 *  lanes            : 0 = default (two utterance micro-batches enqueued alternately on two streams so that one
 *                     micro-batch's small kernels and tails fill the SMs the other leaves idle; bit-identical to
 *                     lanes = 1 because utterances are independent given max_len), 1 or 2
 *  layer_stride     : elements between consecutive hidden states in hidden_out; 0 = batch * T * embed_dim. A caller
 *                     that runs a sub-batch into its slice of a larger [NL+1][Btotal][T][D] buffer passes Btotal*T*D.
 *  ffn_out          : optional DEVICE [num_layers][batch][T][embed_dim]: fc2 output (+bias) of every layer BEFORE
 *                     the residual add = layer_results[i][2] of the reference (wav2vec2/expert.py:87-93,
 *                     feature_selection "fairseq_layers_before_residual"); ffn_layer_stride like layer_stride
 *  last_residual    : optional DEVICE [batch][T][embed_dim], layer_norm_first models only: output of the last layer
 *                     before encoder.layer_norm = layer_results[-1][0] ("fairseq_layers", wav2vec2/expert.py:81-86)
 *  A Conformer model refuses ffn_out and last_residual: its encoder collects no layer_results
 *  (wav2vec2_model.py:3199-3200), so the reference has no such outputs. */
typedef struct s3b_forward_opts {
    int32_t struct_size;
    int32_t lanes;
    int64_t layer_stride;
    float* ffn_out;
    int64_t ffn_layer_stride;
    float* last_residual;
    int64_t reserved[4];
} s3b_forward_opts;
int s3b_forward_ex(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len,
                   float* hidden_out, void* stream, const s3b_forward_opts* opts);
/* Lanes the library picks for a batch when opts->lanes == 0 (two from a measured frame count on, else one;
 * S3B_LANES / S3B_LANE_MIN_FRAMES override). No reference counterpart: scheduling only, results are bit-identical. */
int32_t s3b_default_lanes(const s3b_model* m, int32_t batch, int64_t max_len);
/* s3b_forward_host that also leaves the hidden states in a caller-owned DEVICE buffer [NL+1][batch][T][D]
 * (hidden_out_dev may be NULL = internal staging), so that a device-side consumer (Featurizer, all-gather) can run
 * without re-uploading them. */
int s3b_forward_host_ex(s3b_model* m, const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len,
                        float* hidden_out, float* hidden_out_dev);

/* WavLM relative-position bucket of rel[i] = key - query, bidirectional (integer rule, bit-exact with
 * MultiheadAttention._relative_positions_bucket, s3prl/upstream/wavlm/modules.py:418-448). Host arithmetic. */
int s3b_wavlm_buckets(int32_t num_buckets, int32_t max_distance, const int32_t* rel, int32_t n, int32_t* out);

/* Accounting --------------------------------------------------------------------------------------
 * Kernel categories: 0 = GEMM, 1 = attention, 2 = the front end before the GEMMs: conv-0 (+GroupNorm/LayerNorm+GELU), or
 * for a DeCoAR 2.0 model the fbank frame kernel and the CMVN / decimation kernel,
 * 3 = LayerNorm kernels (Conformer: LayerNorm + RoPE included), 4 = misc (waveform packing, WavLM gate, the
 * Conformer's GLU + depthwise conv). With profiling enabled every launch of
 * s3b_forward is bracketed by CUDA events on the launching stream; s3b_profile_read synchronises the device and
 * returns, per category, accumulated device milliseconds, ALGORITHMIC flops (2*M*N*K of the un-padded
 * contraction; 4*T^2*D per utterance and layer for attention) and kernel launches. Arrays have 5 entries.
 * s3b_profile_read_ex reads the first num_categories (1..6) categories; category 5 is the recurrence kernels: APC's GRU
 * (flops: 6*H*H per frame of the padded batch) and DeCoAR's LSTM (8*H*H per frame of the padded batch and direction).
 * reset clears all six. */
int s3b_profile_enable(s3b_model* m, int32_t enable);
int s3b_profile_read(s3b_model* m, double* ms, double* flops, int64_t* launches, int32_t reset);
int s3b_profile_read_ex(s3b_model* m, int32_t num_categories, double* ms, double* flops, int64_t* launches,
                        int32_t reset);
/* kernels launched by s3b_forward / s3b_forward_host on this model since creation */
int64_t s3b_launch_count(const s3b_model* m);

/* Featurizer (s3prl/upstream/interfaces.py:217-248) --------------------------------------------------
 * out[i] = sum_l w[l] * hs[l][i], hs = [num][n_per_layer] fp32 device, w = device (already softmaxed).
 * num in [1, 64]; n_per_layer a non-negative multiple of 4; hs, out and grad_out 16-byte aligned. */
int s3b_weighted_sum(const float* hs, int32_t num, int64_t n_per_layer, const float* w, float* out, void* stream);
/* grad_w[l] = sum_i hs[l][i] * grad_out[i] */
int s3b_weighted_sum_backward(const float* hs, int32_t num, int64_t n_per_layer, const float* grad_out,
                              float* grad_w, void* stream);

/* Fused Featurizer + all-gather over NVLink peer memory (multi-GPU step ---------------------------
 * One process per GPU on one NVSwitch node. Every rank creates an exchange object (the library cudaMalloc's
 * [slots][world][block_elems] floats + flags and exports them as a 64-byte CUDA IPC handle), the host side exchanges
 * the handles (torch.distributed.all_gather_object in s3prl_b200/parallel.py) and calls s3b_peer_connect with all of them.
 *  s3b_peer_push(step): ONE kernel computes sum_l w[l] * hs[l][i] over this rank's block (hs layers layer_stride
 *    elements apart) and stores it into slot step % slots of EVERY rank's buffer at this rank's position, then
 *    releases a per-(slot, rank) flag = step + 1 at system scope. num in [1, 64], layer_stride a multiple of 4 and
 *    >= block_elems, hs 16-byte aligned. Steps count from 0 and stay below 2^32 - 1: the flags are uint32 step + 1.
 *  s3b_peer_wait(step): stream-ordered wait until every rank's flag of that slot has reached step + 1: the local
 *    gathered buffer s3b_peer_slot(step) = [world][block_elems] is then complete.
 * Contract: a slot is rewritten `slots` steps later; the host protocol (parallel.FeatureGatherer) waits for step s-1
 * before pushing step s, so a writer never overtakes a reader by more than slots - 2 steps. */
typedef struct s3b_peer s3b_peer;
int s3b_peer_create(int32_t rank, int32_t world, int64_t block_elems, int32_t slots, s3b_peer** out,
                    void* ipc_handle_out /* 64 bytes */);
int s3b_peer_connect(s3b_peer* p, const void* all_handles /* world x 64 bytes, rank-major */);
float* s3b_peer_slot(s3b_peer* p, uint32_t step);
int s3b_peer_push(s3b_peer* p, const float* hs, int32_t num, int64_t layer_stride, const float* w, uint32_t step,
                  void* stream);
int s3b_peer_wait(s3b_peer* p, uint32_t step, void* stream);
void s3b_peer_destroy(s3b_peer* p);

/* fbank baseline upstream (s3prl/upstream/baseline/expert.py:69-79 over torchaudio.compliance.kaldi.fbank,
 * fbank.yaml: 80 mel bins, 25 ms / 10 ms, log; + 2 x ComputeDeltas(5) + per-utterance CMVN).
 *  wavs : host array of `batch` DEVICE pointers (fp32, un-padded), lens : host array of lengths
 *  out  : DEVICE buffer [batch][s3b_fbank_num_frames(max(lens))][240] fp32, zero beyond each utterance's frames
 *  Every lens[b] must be >= 0. */
int64_t s3b_fbank_num_frames(int64_t len);
int s3b_fbank(const float* const* wavs, const int64_t* lens, int32_t batch, float* out, void* stream);

/* Options of s3b_fbank_ex / s3b_melspec_ex (zero-initialise, set struct_size = sizeof(s3b_spectral_opts)).
 *  cmvn : 1 = per-utterance CMVN, as s3b_fbank / s3b_melspec (the fbank, mel and linear entries);
 *         0 = the features before CMVN (fbank: the fbank_no_cmvn entry, s3prl/upstream/baseline/fbank_no_cmvn.yaml)
 *  opts NULL is cmvn = 1. */
typedef struct s3b_spectral_opts {
    int32_t struct_size;
    int32_t cmvn;
    int64_t reserved[3];
} s3b_spectral_opts;
/* s3b_fbank with options. cmvn = 0: out holds [log-mel | delta | delta-delta] before CMVN, zero beyond each
 * utterance's frames. */
int s3b_fbank_ex(const float* const* wavs, const int64_t* lens, int32_t batch, const s3b_spectral_opts* opts,
                 float* out, void* stream);

/* mel / linear baseline upstreams (s3prl/upstream/baseline/expert.py:52-79 over OnlinePreprocessor.forward,
 * s3prl/upstream/baseline/preprocessor.py:150-223; mel.yaml / linear.yaml). The host side (Python, like the
 * reference) derives the data-dependent lengths; these entry points do the arithmetic.
 *  s3b_trimmed_lengths: out[b] = (index of the last non-zero sample) + 1, or lens[b] if all zero (synchronous).
 *  s3b_melspec: STFT power (n_fft 400, hop 160, hann, center/reflect over the row padded to `padded_len`) ->
 *    mel != 0: 80-bin HTK mel, else 201 linear bins -> log(x + 1e-10) -> CMVN over the first feats_len[b] frames
 *    -> first final_len[b] frames kept, zero up to t_out. out: DEVICE [batch][t_out][80 | 201] fp32.
 *    Refused: lens[b] < 0 (s3b_trimmed_lengths); trimmed_lens[b] outside [0, padded_len], feats_len[b] outside
 *    [0, 1 + padded_len / 160], final_len[b] outside [0, t_out] (s3b_melspec). */
int s3b_trimmed_lengths(const float* const* wavs, const int64_t* lens, int32_t batch, int64_t* out);
int s3b_melspec(const float* const* wavs, const int64_t* trimmed_lens, int32_t batch, int64_t padded_len, int32_t mel,
                const int32_t* feats_len, const int32_t* final_len, int32_t t_out, float* out, void* stream);
/* s3b_melspec with options. cmvn = 0: out is DEVICE [batch][1 + padded_len / 160][80 | 201], the log features of
 * every frame of the padded batch (the reference's feat before the per-utterance cut); feats_len, final_len and t_out
 * are then unused and may be NULL / 0. */
int s3b_melspec_ex(const float* const* wavs, const int64_t* trimmed_lens, int32_t batch, int64_t padded_len,
                   int32_t mel, const int32_t* feats_len, const int32_t* final_len, int32_t t_out,
                   const s3b_spectral_opts* opts, float* out, void* stream);

/* Building blocks exposed for parity tests (device pointers, fp32) -------------------------------------- */
/* out[M][N] = act(A[M][K] * W[N][K]^T + bias[N]) (+ residual[M][N]); K % 64 == 0, N % 16 == 0.
 * gelu selects act: 0 = none, 1 = GELU (exact erf), 2 = SiLU (x * sigmoid(x), the Conformer's Swish).
 * = s3b_linear_ex with opts NULL: the default operand scheme (S3B_GEMM_SCHEME) where it applies, else bf16x3. */
int s3b_linear_f32(const float* a, const float* w, const float* bias, const float* residual, int64_t m, int32_t n,
                   int32_t k, int32_t gelu, float* out, void* stream);
/* Options of s3b_linear_ex (zero-initialise, set struct_size = sizeof(s3b_linear_opts), scheme = out_fmt = -1).
 *  scheme      : -1 = the library default where it applies (else bf16x3), 0 = bf16x3, 1 = f16q8 (needs K % 128 == 0
 *                and N % 128 == 0; an impossible request is an error)
 *  tile_n      : 0 = the library's choice, 128 or 256 = that tile width (must divide N)
 *  out_fmt     : -1 = fp32 output; 0 / 1 = the output is written as operand planes (0 = bf16 hi/lo, 1 = f16q8) like
 *                fc1's, and out is decoded from them
 *  row_mask    : optional DEVICE uint8 [M]: rows != 0 are written as zero (post_extract_proj's padding mask)
 *  out_pre     : optional DEVICE fp32 [M][N]: the value before the residual add (fc2's ffn output)
 *  lda, a_off  : A is the [M][K] column slice starting at column a_off of a [M][lda] matrix (0, 0 = dense [M][K]);
 *                lda and a_off multiples of 16 (the distiller's SplitLinear)
 *  scheme_used, tile_n_used : filled in with the operand scheme and the tile width that ran */
typedef struct s3b_linear_opts {
    int32_t struct_size;
    int32_t scheme;
    int32_t tile_n;
    int32_t out_fmt;
    const uint8_t* row_mask;
    float* out_pre;
    int64_t lda;
    int64_t a_off;
    int32_t scheme_used;
    int32_t tile_n_used;
    int64_t reserved[2];
} s3b_linear_opts;
int s3b_linear_ex(const float* a, const float* w, const float* bias, const float* residual, int64_t m, int32_t n,
                  int32_t k, int32_t gelu, s3b_linear_opts* opts, float* out, void* stream);
/* The QKV projection as a layer runs it: x [batch][t][heads*64] times w [3D][D]^T + b [3D] through the GEMM's QKV
 * epilogue (q scaled by 1/8 * log2(e), per-head layout, v transposed), in operand scheme `scheme` (-1 / 0 / 1 as in
 * s3b_linear_opts). The bf16 hi/lo planes it writes are decoded to q_out, k_out [batch][heads][t][64] and
 * vt_out [batch][heads][64][(t + 7) & ~7]. The epilogue writes columns [0, t) of each vt_out row; the padding columns
 * t.. are never written by it and come back as the zero of a freshly allocated plane: this entry point allocates its
 * planes per call. A model's planes live as long as the model and are zeroed only when they are (re)allocated, so
 * there the padding columns hold whatever an earlier, differently shaped forward left, NaN included. The model path
 * does not rely on them: the attention kernel's tensor map of v^T has extent t, not (t + 7) & ~7, so the columns past
 * t are filled with zeros by the TMA load and the stored ones are never read. The same holds for q / k rows past t
 * and, for 80- and 120-wide heads, the box columns past head_dim. What the model path does rely on is written on every
 * call by the kernel that owns it: the CMVN kernel zero-fills columns 80..127 and rows past each utterance's frames of
 * the fbank models' [M][128] operand, and post_extract_proj's row mask zeroes padded frames.
 * tests/test_history_gpu.py holds a long-lived model to the result of a fresh one after calls of other shapes and
 * after a forward on non-finite waveforms. */
int s3b_qkv_f32(const float* x, const float* w, const float* b, int32_t batch, int32_t t, int32_t heads, int32_t scheme,
                float* q_out, float* k_out, float* vt_out, void* stream);
/* s3b_qkv_f32 for heads of head_dim (64, 80 or 120) channels: x [batch][t][heads*head_dim]; q scaled by
 * head_dim^-0.5 * log2(e) (one fp32 constant); q_out, k_out [batch][heads][t][head_dim],
 * vt_out [batch][heads][head_dim][(t + 7) & ~7]. */
int s3b_qkv_hd_f32(const float* x, const float* w, const float* b, int32_t batch, int32_t t, int32_t heads,
                   int32_t head_dim, int32_t scheme, float* q_out, float* k_out, float* vt_out, void* stream);
/* One conv of the feature extractor (Conv1d(512, 512, kw, stride 2), kw in {2, 3}) as the model runs it: implicit GEMM on
 * channels-last x [batch][lin][512], weight w [512][512][kw] (torch layout), optional bias [512], optional GELU, in
 * operand scheme `scheme`; out_fmt -1 = fp32 output, 0 / 1 = operand planes decoded to fp32.
 * out: [batch][(lin - kw) / 2 + 1][512]. */
int s3b_conv_gemm_f32(const float* x, const float* w, const float* bias, int32_t batch, int64_t lin, int32_t kw,
                      int32_t gelu, int32_t scheme, int32_t out_fmt, float* out, void* stream);
/* The positional conv as the model runs it (bf16x3): x [batch][t][d], folded weight w [d][d / groups][k], bias [d].
 * d in {384, 512, 640, 768, 1024, 1280, 1920}; d / groups in {16, 24, 32, 40, 48, 64, 80, 120} (80 and 120:
 * taps_per_kblock 1 only; 24 and 40: taps_per_kblock 4 only).
 *  taps_per_kblock 1: one k-block per tap (two above 64 channels per group), bias + GELU + residual in the GEMM epilogue, fp32 (then LayerNorm if gamma:
 *    as in the model, operand planes come only from that LayerNorm, so out_fmt >= 0 needs gamma);
 *  taps_per_kblock 4: four taps per k-block (zero taps appended up to a multiple of 4) + the combine kernel, mode
 *    0 = x + GELU(conv + bias); 1 = data2vec block GELU(LayerNorm_noaffine(conv + bias)); 2 = x + the mode-1 value.
 *  gamma, beta: optional LayerNorm(d) of the result (post-LN models' encoder LayerNorm); NULL = none.
 *  out_fmt -1 = fp32 output, 0 / 1 = operand planes decoded to fp32. out: [batch][t][d]. */
int s3b_posconv_f32(const float* x, const float* w, const float* bias, int32_t batch, int32_t t, int32_t d,
                    int32_t groups, int32_t k, int32_t taps_per_kblock, int32_t mode, const float* gamma,
                    const float* beta, int32_t out_fmt, float* out, void* stream);
/* One NPC convolution as the model runs it: same padding ((k - 1) / 2), implicit GEMM over channels-last
 * x [batch][t][c_in] (c_in 80, zero-padded to 128 per tap, or 512), weight w [512][c_in][k] (torch layout, device),
 * mask: 0 = every tap, else the odd width of a centred band of taps left out (the MaskConvBlock's conv_mask);
 * out = act(conv + bias) + residual, or act(conv + bias + residual) with res_first (the ConvBlock); act 0 = none,
 * 1 = ReLU, 2 = tanh; bias, residual ([batch][t][512]) optional; out_pre: optional act(conv + bias) before the
 * residual (not with res_first). scheme -1 / 0 / 1 as s3b_linear_ex. out: [batch][t][512] fp32. */
int s3b_npc_conv_f32(const float* x, int32_t batch, int32_t t, int32_t c_in, const float* w, int32_t k, int32_t mask,
                     const float* bias, const float* residual, int32_t act, int32_t res_first, int32_t scheme,
                     float* out, float* out_pre, void* stream);
/* One modified CPC conv + ChannelNorm + ReLU as the model runs it. layer 0: x is the padded waveform batch
 * [batch][len], w [256][1][10] (stride 5, padding 3); the model writes conv 0's output as operand planes only, so out
 * holds those planes (format of `scheme`) decoded to fp32. layer 1..4: x is channels-last [batch][len][256], w
 * [256][256][2 s] (torch layout; s = 4, 2, 2, 2, padding s / 2), computed as the model computes it: x split into operand
 * planes of `scheme` in the padded layout, one implicit GEMM (+ bias) in fp32, then the norm. bias, gamma, beta: [256];
 * all pointers device. scheme -1 / 0 / 1 as s3b_linear_ex. out: [batch][T][256] fp32, T = the conv's output length. */
int s3b_cpc_conv_f32(const float* x, int32_t batch, int32_t len, int32_t layer, const float* w, const float* bias,
                     const float* gamma, const float* beta, int32_t scheme, float* out, void* stream);
/* One modified CPC LSTM layer's recurrence as the model runs it: xg [batch][t][1024] = W_ih x + b_ih + b_hh (gate order
 * i, f, g, o), whh [1024][256]; every utterance runs all t steps from h0 = c0 = 0. out [batch][t][256] fp32; out_fmt 0 /
 * 1 also writes the same values as operand planes of that format, decoded into planes_out (-1: none). */
int s3b_cpc_lstm_f32(const float* xg, const float* whh, int32_t batch, int32_t t, int32_t out_fmt, float* out,
                     float* planes_out, void* stream);
/* clusters of the CPC recurrence kernel (8 CTAs, 4 utterances each) that can be co-resident on the current device */
int s3b_cpc_lstm_max_active_clusters(int32_t* out);
/* micro-benchmark of the production GEMM kernel: `iters` back-to-back launches of [M][K] x [N][K]^T with the fc1-style
 * epilogue (gelu != 0: bias + GELU + bf16 hi/lo output) or the out_proj-style one (bias + residual + fp32 output).
 * force_un in {0 = the library's choice, 128, 256} forces the tile width (columns per output tile) wherever it divides
 * n. out[0] = ms per launch, out[1] = tile width used. (tools/gemm_shapes.py) */
int s3b_gemm_bench(int64_t m, int32_t n, int32_t k, int32_t gelu, int32_t force_un, int32_t iters, float* out);
/* y = LayerNorm_D(x) (eps 1e-5), optional GELU; D in {384,512,640,768,1024,1280,1920} */
int s3b_layernorm_f32(const float* x, int64_t m, int32_t d, const float* gamma, const float* beta, int32_t gelu,
                      float* out, void* stream);
/* softmax(q k^T / 8 + key padding mask) v per (batch, head); q,k,v: [batch][T][heads*64] fp32; valid_frames: host,
 * [batch], each in [1, t]. The context comes back from bf16 hi/lo planes. = s3b_attention_ex with opts NULL. */
int s3b_attention_f32(const float* q, const float* k, const float* v, const int32_t* valid_frames, int32_t batch,
                      int32_t t, int32_t heads, float* out, void* stream);
/* Options of s3b_attention_ex (zero-initialise, set struct_size = sizeof(s3b_attention_opts)).
 *  rel_emb      : optional DEVICE fp32 [num_buckets][heads] (relative_attention_bias.weight, wavlm/modules.py:450-462):
 *                 scores get gate[b][h][q] * rel_emb[bucket(k - q)][h] before the key mask, through the table the
 *                 model builds (Toeplitz table for table_frames frames)
 *  table_frames : frames the table is built for (0 = 4096, as s3b_model_finalize); must be >= t
 *  gate         : optional DEVICE fp32 [batch][heads][t] (needs rel_emb); NULL = 1
 *  ctx_format   : operand format the kernel writes the context in: 0 = bf16 hi/lo, 1 = f16q8 (fp16 + e4m3 residual);
 *                 out is decoded from those planes with the arithmetic the library's kernels read an operand back with
 *  head_dim     : channels per head, 64, 80 or 120 (0 = 64): q, k, v are [batch][t][heads*head_dim] and the scores are
 *                 scaled by head_dim^-0.5; rel_emb needs 64 */
typedef struct s3b_attention_opts {
    int32_t struct_size;
    int32_t ctx_format;
    const float* rel_emb;
    int32_t num_buckets;
    int32_t max_distance;
    const float* gate;
    int32_t table_frames;
    int32_t head_dim;
    int64_t reserved[2];
} s3b_attention_opts;
int s3b_attention_ex(const float* q, const float* k, const float* v, const int32_t* valid_frames, int32_t batch,
                     int32_t t, int32_t heads, const s3b_attention_opts* opts, float* out, void* stream);
/* WavLM gate (wavlm/modules.py:534-551) through the model's kernel: x [batch][t][heads*64] fp32 is first written into
 * operand planes of x_format (0 = bf16 hi/lo, 1 = f16q8) like a LayerNorm output; grep_w [8][64], grep_b [8],
 * grep_a [heads] (grep_w NULL = gru_rel_pos off: gate 1). gate_out: DEVICE [batch][heads][t] fp32. */
int s3b_wavlm_gate_f32(const float* x, int32_t batch, int32_t t, int32_t heads, const float* grep_w,
                       const float* grep_b, const float* grep_a, int32_t x_format, float* gate_out, void* stream);
/* The feature extractor's front end as a forward runs it: ragged DEVICE waveforms (host array of pointers, lengths
 * lens[b] in [1, max_len]) packed into [batch][max_len] (normalize: per-utterance F.layer_norm over lens[b] samples),
 * then conv 0 (w [512][1][10], optional bias [512]) with GroupNorm(512, 512) over all L0 = (max_len - 10) / 5 + 1
 * frames (layer_norm 0; a bias is dropped as the model drops it) or per-frame LayerNorm(512) (layer_norm 1),
 * gamma / beta [512], GELU, written as operand planes of out_fmt (0 = bf16 hi/lo, 1 = f16q8) and decoded to
 * out [batch][L0][512]. max_len >= 10. wav_out (optional DEVICE [batch][max_len]): the packed waveform. */
int s3b_frontend_f32(const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len, int32_t normalize,
                     const float* w, const float* bias, const float* gamma, const float* beta, int32_t layer_norm,
                     int32_t out_fmt, float* wav_out, float* out, void* stream);
/* The DeCoAR 2.0 front end as a forward runs it (frontend = 1 of s3b_config): ragged DEVICE waveforms (host array of
 * pointers, host lengths lens[b] >= 560) -> kaldi fbank with the hamming window -> CMVN over each utterance's frames ->
 * every second frame, written as operand planes of out_fmt (0 = bf16 hi/lo, 1 = f16q8) and decoded to
 * out [batch][T][80], T = (1 + (max(lens) - 400) / 160 + 1) / 2, rows t >= T_b zero. */
int s3b_decoar2_features_f32(const float* const* wavs, const int64_t* lens, int32_t batch, int32_t out_fmt, float* out,
                             void* stream);
/* The APC front end as a forward runs it: s3b_decoar2_features_f32 without the decimation, every frame kept:
 * out [batch][T][80], T = 1 + (max(lens) - 400) / 160, rows t >= m_b zero; lens[b] >= 560. */
int s3b_apc_features_f32(const float* const* wavs, const int64_t* lens, int32_t batch, int32_t out_fmt, float* out,
                         void* stream);
/* The same front end (step 1: APC, DeCoAR, NPC; step 2: DeCoAR 2.0) written into the caller's DEVICE buffers instead of
 * workspaces of the call, undecoded: logmel [batch][m][80] fp32, the frame kernel's log-mel, m = 1 + (max(lens) - 400)
 * / 160 (rows past an utterance's frames are not written); planes: the operand planes of out_fmt as the first GEMM reads
 * them, each [batch][T][128] with T as above, back to back (4 * batch * T * 128 bytes, 4-byte aligned): out_fmt 0 the
 * bf16 hi plane then the bf16 lo plane, out_fmt 1 the fp16 plane, then the e4m3 plane of the fp16 values, then the
 * e4m3 plane of the residuals scaled by 2^11. */
int s3b_fbank_cmvn_planes(const float* const* wavs, const int64_t* lens, int32_t batch, int32_t step, int32_t out_fmt,
                          float* logmel, void* planes, void* stream);
/* One APC GRU layer's recurrence as a forward runs it (the model's kernel): xg [batch][t][3H] DEVICE = W_ih x + b_ih
 * (gate order r, z, n), whh [3H][H] and bhh [3H] DEVICE (weight_hh_l0, bias_hh_l0), optional residual [batch][t][H]
 * DEVICE added to the output, lens HOST [batch] valid frames in [0, t]. out [batch][t][H] DEVICE: h_t + residual for
 * t < lens[b], 0 beyond. out_fmt -1 = no operand planes; 0 / 1 = the planes the model feeds the next layer's GEMM
 * (bf16 hi/lo or f16q8), decoded to planes_out [batch][t][H]. hidden must be 512. */
/* cudaOccupancyMaxActiveClusters of the recurrence kernel on the current device: clusters of 16 CTAs (32 hidden units
 * and 209 KB of shared memory each) that can run at once; each runs 4 utterances. */
int s3b_gru_max_active_clusters(int32_t* out);
int s3b_gru_f32(const float* xg, const float* whh, const float* bhh, const float* residual, const int32_t* lens,
                int32_t batch, int32_t t, int32_t hidden, int32_t out_fmt, float* out, float* planes_out, void* stream);
/* 1 in *out when the current device can host DeCoAR's LSTM recurrence grid (128 co-resident CTAs, one per SM, with
 * their shared memory; cooperative launch), else 0. */
int s3b_lstm_fits(int32_t* out);
/* One DeCoAR LSTM layer and direction as a forward runs it (the model's kernel, H = 1024): xg [batch][t][4H] DEVICE =
 * W_ih x + b_ih (gate order i, f, g, o), whh [4H][H] DEVICE (weight_hh_l{k}), optional bhh [4H] DEVICE added to xg
 * (the model folds it into its GEMM bias), lens HOST [batch] valid frames in [0, t]. direction 0 runs frames 0 ..
 * lens[b] - 1, direction 1 runs them backwards. out [batch][t][2H] DEVICE: the kernel writes columns [direction * H,
 * direction * H + H) only: h of frame t for t < lens[b], 0 beyond. out_fmt -1 = no operand planes; 0 / 1 = the planes
 * the model feeds the next layer's GEMM (bf16 hi/lo or f16q8), decoded to planes_out [batch][t][2H] (same columns). */
int s3b_lstm_f32(const float* xg, const float* whh, const float* bhh, const int32_t* lens, int32_t batch, int32_t t,
                 int32_t direction, int32_t out_fmt, float* out, float* planes_out, void* stream);
/* The Conformer convolution module between its pointwise convs, as a forward runs it (wav2vec2_model.py:383-389):
 * x [batch][t][2d] (pointwise_conv1 output, channels-last) -> GLU (x[..., :d] * sigmoid(x[..., d:])) -> depthwise
 * Conv1d(k, padding k / 2, groups d, no bias; dw_w [d][1][k]) over each utterance's t frames -> BatchNorm1d (eval, eps
 * 1e-5; bn_gamma, bn_beta, bn_mean, bn_var [d], folded into the taps as the model folds them) -> SiLU, written as
 * operand planes of out_fmt (0 = bf16 hi/lo, 1 = f16q8) and decoded to out [batch][t][d]. d % 64 == 0, k odd <= 63. */
int s3b_conformer_conv_f32(const float* x, int32_t batch, int32_t t, int32_t d, int32_t k, const float* dw_w,
                           const float* bn_gamma, const float* bn_beta, const float* bn_mean, const float* bn_var,
                           int32_t out_fmt, float* out, void* stream);
/* The Conformer's attention input (wav2vec2_model.py:541, 255-310): y = LayerNorm_d(x) * gamma + beta (eps 1e-5) and
 * rope(y) per 64-wide head at frame index row % t, angles fp32(frame) * inv_freq[j] (inv_freq: host [32], NULL =
 * 1 / 10000^(2j / 64)), both written as operand planes of out_fmt and decoded to out [m][d] and out_rope [m][d].
 * x: [m][d] (m a multiple of t: rows of utterances of t frames); d in {512, 768, 1024, 1280}. */
int s3b_layernorm_rope_f32(const float* x, int64_t m, int32_t t, int32_t d, const float* gamma, const float* beta,
                           const float* inv_freq, int32_t out_fmt, float* out, float* out_rope, void* stream);

/* y = LayerNorm_D(x) with epsilon eps, otherwise s3b_layernorm_f32 (SSAST's blocks use 1e-6) */
int s3b_layernorm_eps_f32(const float* x, int64_t m, int32_t d, const float* gamma, const float* beta, int32_t gelu,
                          float eps, float* out, void* stream);
/* The same LayerNorm as a pre-LN layer's LN1 / LN2 runs it (SSAST: eps 1e-6): written only as operand planes of fmt
 * (0 bf16 hi/lo, 1 f16q8), decoded to out [m][d]. */
int s3b_layernorm_eps_planes_f32(const float* x, int64_t m, int32_t d, const float* gamma, const float* beta, float eps,
                                 int32_t fmt, float* out, void* stream);
/* SSAST's front end as a forward runs it: ragged DEVICE waveforms (host array of pointers, host lengths lens[b] in
 * [1, max_len]), nseg = ceil(max_len / window_samples) windows each -> out DEVICE [batch * nseg][TL][128], row block
 * b * nseg + s, TL = window_samples / 160 (the normalised fbank, zero rows appended). */
int s3b_ssast_fbank_f32(const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len,
                        int32_t window_samples, float* out, void* stream);
/* SSAST's patch embedding and token assembly as a forward runs them, on the features feat [segments][TL][128] (DEVICE):
 * the patch operand (patch 0: the features, patch 1: the 16 x 16 / stride-10 gather) written as operand planes of
 * `scheme` (-1 / 0 / 1 as s3b_linear_ex) and decoded into planes_out (optional; [segments][TL][128] or
 * [segments][P][256]), the (768, 256) patch GEMM + bias, then [cls + pos[0], dist + pos[1], patch p + pos[2 + p]] into
 * out [segments][2 + P][768]. w [768][1][128][2] or [768][1][16][16] (torch layout), bias, cls, dist [768],
 * pos [2 + P][768]; all DEVICE. */
int s3b_ssast_embed_f32(const float* feat, int32_t segments, int32_t tl, int32_t patch, const float* w,
                        const float* bias, const float* cls, const float* dist, const float* pos, int32_t scheme,
                        float* planes_out, float* out, void* stream);
/* The patch operand of s3b_ssast_embed_f32 (the features, or the 16 x 16 / stride-10 gather) as a forward writes it
 * from feat [segments][TL][128] (DEVICE), undecoded, into the caller's DEVICE buffer `planes`: the operand planes of
 * fmt (0 bf16 hi/lo, 1 f16q8), each [segments][TL][128] (patch 0) or [segments][P][256] (patch 1), back to back in
 * the layout of s3b_fbank_cmvn_planes (4 bytes per element, 4-byte aligned). */
int s3b_ssast_patch_planes(const float* feat, int32_t segments, int32_t tl, int32_t patch, int32_t fmt, void* planes,
                           void* stream);
/* One SSAST hidden state from the residual stream x [batch * nseg][2 + P][768] (DEVICE) as a forward writes it:
 * out [batch][t_out][768 or 12 * 768], class tokens dropped, frequency patches folded into channels; t_out <= nseg t_dim. */
int s3b_ssast_fold_f32(const float* x, int32_t batch, int32_t nseg, int32_t tl, int32_t patch, int32_t t_out,
                       float* out, void* stream);
/* MAE-AST's front end as a forward runs it: ragged DEVICE waveforms (host array of pointers, host lengths lens[b] in
 * [400, max_len]), the batch-normalised 128-bin fbank unfolded into the patch operand [batch * T' nv][256] (T' =
 * (1 + (max_len - 400) / 160) / kt), with y = log-mel * (0.5 / sqrt(running_var + 1e-5)) - running_mean * that.
 * out (optional): fp32, as the kernel computes it; planes_out (optional): the operand planes of `fmt` (0 bf16 hi/lo,
 * 1 f16q8) decoded. Both DEVICE. */
int s3b_mae_ast_fbank_f32(const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len, int32_t patch,
                          float running_mean, float running_var, int32_t fmt, float* out, float* planes_out,
                          void* stream);
/* The same front end with the forward's batch-norm constants, undecoded, into the caller's DEVICE buffer `planes`:
 * the operand planes of fmt, each [batch * T' nv][256], back to back in the layout of s3b_fbank_cmvn_planes (4 bytes
 * per element, 4-byte aligned). */
int s3b_mae_ast_fbank_planes(const float* const* wavs, const int64_t* lens, int32_t batch, int64_t max_len,
                             int32_t patch, float running_mean, float running_var, int32_t fmt, void* planes,
                             void* stream);
/* MAE-AST's positions and input norm as a forward runs them, in place on x [batch][n_tok][768] (DEVICE, the
 * projection's output): x[b][t] += pe[t] for t < valid[b] (host array; pe [>= n_tok][768] DEVICE, or NULL); with
 * gamma / beta (DEVICE, post-LN) then LayerNorm(eps 1e-5) into x and, when planes_out is given, its operand planes of
 * `fmt` decoded into planes_out [batch][n_tok][768] (DEVICE). */
int s3b_mae_ast_embed_f32(float* x, int32_t batch, int32_t n_tok, const int32_t* valid, const float* pe,
                          const float* gamma, const float* beta, int32_t fmt, float* planes_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* S3PRL_B200_H_ */
