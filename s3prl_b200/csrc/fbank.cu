// Kaldi-compatible log-mel filterbank + deltas + CMVN (the `fbank` baseline upstream).
// Replaces the per-utterance Python loop of s3prl/upstream/baseline/expert.py:46-50,69-79 over
//   torchaudio.compliance.kaldi.fbank(num_mel_bins=80, frame_length=25, frame_shift=10, use_log_fbank=True)
//     (torchaudio/compliance/kaldi.py: _get_window :154-218, get_mel_banks :436-512, fbank :514-646)
//   2 x ComputeDeltas(win_length=5), concatenated           s3prl/upstream/baseline/extracter.py:58-76
//   per-utterance CMVN with unbiased std                    s3prl/upstream/baseline/extracter.py:78-90
// One warp computes one 25 ms frame: DC removal, pre-emphasis, povey window, 512-point radix-2 FFT in shared
// memory, power spectrum, sparse triangular mel projection (the "matmul"), log. All fp32.
// The same frame kernel with a hamming window is the front end of DeCoAR 2.0 (s3prl/upstream/decoar2/audio.py:41-86),
// followed by decoar2_cmvn_kernel: per-utterance CMVN over all frames, every second frame kept, written as the
// operand planes of post_extract_proj. With a hanning window and 128 bins, per fixed-length window of the waveform, it
// is SSAST's front end (ssast_fbank_kernel).
#include <math.h>

#include <vector>

#include "common.cuh"
#include "fbank.cuh"
#include "kernels.cuh"

namespace s3b {

static constexpr int kWin = 400, kShift = 160, kFft = 512, kBins = 257, kMel = 80, kFeat = 240;
static constexpr int kMaxMelNnz = 1024;

struct FbankTables {
    float window[kWin];
    float tw_re[kFft / 2], tw_im[kFft / 2];  // exp(-2 pi i k / 512)
    int mel_start[kMel], mel_count[kMel], mel_off[kMel];
    float mel_w[kMaxMelNnz];
};
__device__ FbankTables g_tab;
static bool g_tab_ready[64] = {false};
// DeCoAR 2.0's window, torch.hamming_window(400, periodic=False, alpha=0.54, beta=0.46) (kaldi.py _get_window). A table
// of its own: g_tab.window stays the povey window of the fbank baseline, and both models can live in one process.
__device__ float g_hamming[kWin];
static bool g_hamming_ready[64] = {false};
// SSAST's front end: 128 mel bins and the hanning window, torch.hann_window(400, periodic=False) (kaldi.py _get_window),
// in tables of their own next to the 80-bin ones, so that every fbank model can live in one process
static constexpr int kSsastMel = 128;
struct MelTable {
    int start[kSsastMel], count[kSsastMel], off[kSsastMel];
    float w[kMaxMelNnz];
};
__device__ MelTable g_mel128;
__device__ float g_hann[kWin];
static bool g_ssast_ready[64] = {false};

// mel banks (kaldi.py:436-512): low 20 Hz, high = nyquist 8000 Hz, nbins bins over 256 fft bins, fp32 like torch
static void build_mel(int nbins, int* mel_start, int* mel_count, int* mel_off, float* mel_w) {
    const float low = 20.0f, high = 8000.0f, fft_bin_width = 16000.0f / kFft;
    auto mel = [](float f) { return 1127.0f * logf(1.0f + f / 700.0f); };
    const double mel_low = 1127.0 * log(1.0 + (double)low / 700.0), mel_high = 1127.0 * log(1.0 + (double)high / 700.0);
    const double delta = (mel_high - mel_low) / (nbins + 1);
    int off = 0;
    for (int j = 0; j < nbins; ++j) {
        const float left = (float)(mel_low + j * delta), center = (float)(mel_low + (j + 1.0) * delta),
                    right = (float)(mel_low + (j + 2.0) * delta);
        int start = -1, count = 0;
        for (int i = 0; i < kFft / 2; ++i) {
            const float m = mel(fft_bin_width * (float)i);
            const float up = (m - left) / (center - left), down = (right - m) / (right - center);
            const float w = fmaxf(0.0f, fminf(up, down));
            if (w > 0.0f) {
                if (start < 0) start = i;
                // weights of one triangle are contiguous in i
                if (off + count < kMaxMelNnz) mel_w[off + count] = w;
                ++count;
            }
        }
        mel_start[j] = start < 0 ? 0 : start, mel_count[j] = count, mel_off[j] = off;
        off += count;
    }
}

static void build_tables(FbankTables& t) {
    // povey window: hann(400, periodic=False) ** 0.85   (kaldi.py:98-100)
    for (int n = 0; n < kWin; ++n) {
        const double h = 0.5 - 0.5 * cos(2.0 * M_PI * n / (kWin - 1));
        t.window[n] = (float)pow(h, 0.85);
    }
    for (int k = 0; k < kFft / 2; ++k) {
        t.tw_re[k] = (float)cos(-2.0 * M_PI * k / kFft);
        t.tw_im[k] = (float)sin(-2.0 * M_PI * k / kFft);
    }
    build_mel(kMel, t.mel_start, t.mel_count, t.mel_off, t.mel_w);
}

static cudaError_t ensure_tables(cudaStream_t s) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 64 && g_tab_ready[dev]) return cudaSuccess;
    static FbankTables host;
    build_tables(host);
    e = cudaMemcpyToSymbolAsync(g_tab, &host, sizeof(host), 0, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(s);
    if (e == cudaSuccess && dev < 64) g_tab_ready[dev] = true;
    return e;
}

// Synchronous: the shared tables, the hamming window and SSAST's tables of the current device, built once. The fbank
// models call it at finalize, so that their forwards (asynchronous, graph-capturable) never build tables.
cudaError_t init_fbank_tables() {
    cudaError_t e = ensure_tables(0);
    if (e != cudaSuccess) return e;
    int dev = 0;
    e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (!(dev < 64 && g_hamming_ready[dev])) {
        float h[kWin];
        for (int n = 0; n < kWin; ++n) h[n] = (float)(0.54 - 0.46 * cos(2.0 * M_PI * n / (kWin - 1)));
        e = cudaMemcpyToSymbol(g_hamming, h, sizeof(h));
        if (e != cudaSuccess) return e;
        if (dev < 64) g_hamming_ready[dev] = true;
    }
    if (dev < 64 && g_ssast_ready[dev]) return cudaSuccess;
    float h[kWin];
    for (int n = 0; n < kWin; ++n) h[n] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * n / (kWin - 1)));
    e = cudaMemcpyToSymbol(g_hann, h, sizeof(h));
    if (e != cudaSuccess) return e;
    static MelTable mt;
    build_mel(kSsastMel, mt.start, mt.count, mt.off, mt.w);
    e = cudaMemcpyToSymbol(g_mel128, &mt, sizeof(mt));
    if (e == cudaSuccess && dev < 64) g_ssast_ready[dev] = true;
    return e;
}

__device__ __forceinline__ int bitrev9(int x) { return (int)(__brev((unsigned)x) >> 23); }

// One 25 ms frame per warp, 13 samples per lane in x (lane + 32 i, zero past 400): DC removal, pre-emphasis (replicate
// first sample), `window`, zero pad, 512-point radix-2 DIT FFT in re / im, power spectrum |X|^2 into pw[0, 257)
// (use_power=True; kaldi.py computes abs() then pow(2)). re, im, pw: this warp's shared rows.
__device__ __forceinline__ void frame_power(float (&x)[13], const float* __restrict__ window, float* re, float* im,
                                            float* pw, int lane) {
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 13; ++i) sum += x[i];
    const float mean = warp_sum(sum) / (float)kWin;
#pragma unroll
    for (int i = 0; i < 13; ++i) {
        const int n = lane + 32 * i;
        if (n < kWin) re[n] = x[i] - mean;
    }
    __syncwarp();
    float y[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int n = lane + 32 * i;
        float v = 0.f;
        if (n < kWin) v = (re[n] - 0.97f * re[n > 0 ? n - 1 : 0]) * window[n];
        y[i] = v;
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int n = lane + 32 * i;
        const int r = bitrev9(n);
        re[r] = y[i];
        im[r] = 0.f;
    }
    __syncwarp();
    // 9 radix-2 stages, 256 butterflies each (8 per lane)
    for (int s = 1; s <= 9; ++s) {
        const int half = 1 << (s - 1);
        const int tw_stride = kFft >> s;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int bf = lane + 32 * i;            // butterfly index 0..255
            const int j = bf & (half - 1);
            const int base = ((bf >> (s - 1)) << s) + j;
            const float wr = g_tab.tw_re[j * tw_stride], wi = g_tab.tw_im[j * tw_stride];
            const float ar = re[base], ai = im[base];
            const float br = re[base + half], bi = im[base + half];
            const float tr = br * wr - bi * wi, ti = br * wi + bi * wr;
            re[base] = ar + tr, im[base] = ai + ti;
            re[base + half] = ar - tr, im[base + half] = ai - ti;
        }
        __syncwarp();
    }
    for (int k = lane; k < kBins; k += 32) {
        const float a = sqrtf(re[k] * re[k] + im[k] * im[k]);
        pw[k] = a * a;
    }
    __syncwarp();
}

// grid: (ceil(max_frames / 4), B); block: 128 threads = 4 warps = 4 frames. kHamming: hamming instead of povey window;
// kLd: floats between consecutive frames of `out` (the log-mel goes to columns [0, 80))
template <bool kHamming, int kLd>
__global__ void __launch_bounds__(128) fbank_frames_kernel(const float* const* __restrict__ wavs,
                                                           const long long* __restrict__ lens, int max_frames,
                                                           float* __restrict__ out) {
    __shared__ float s_re[4][kFft], s_im[4][kFft], s_pw[4][kBins + 3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y;
    const int t = blockIdx.x * 4 + warp;
    const long long L = lens[b];
    const int m = L < kWin ? 0 : (int)(1 + (L - kWin) / kShift);  // snip_edges=True (kaldi.py:_get_strided)
    if (t >= m) return;  // warp-uniform
    const float* w = wavs[b] + (size_t)t * kShift;
    float x[13];
#pragma unroll
    for (int i = 0; i < 13; ++i) {
        const int n = lane + 32 * i;
        x[i] = n < kWin ? w[n] : 0.f;
    }
    float* pw = s_pw[warp];
    frame_power(x, kHamming ? g_hamming : g_tab.window, s_re[warp], s_im[warp], pw, lane);
    // mel projection + log(max(e, eps))
    float* o = out + ((size_t)b * max_frames + t) * kLd;
    for (int j = lane; j < kMel; j += 32) {
        const int st = g_tab.mel_start[j], cnt = g_tab.mel_count[j];
        const float* mw = g_tab.mel_w + g_tab.mel_off[j];
        float acc = 0.f;
        for (int i = 0; i < cnt; ++i) acc = fmaf(pw[st + i], mw[i], acc);
        o[j] = logf(fmaxf(acc, 1.1920928955078125e-07f));
    }
}

// SSAST's FeatureExtractor (s3prl/upstream/ssast/audio.py, expert.py) per window: kaldi.fbank of window s of
// utterance b, samples [s S, s S + S) of the waveform zero-padded past lens[b], with the hanning window and 128 mel
// bins, then y = (y + 4.2677393) / (4.5689974 * 2) and zero rows appended up to TL = target_length.
// out: [B * nseg][TL][128] fp32, row block b * nseg + s. grid (ceil(TL / 4), nseg, B); block 128 threads = 4 frames.
__global__ void __launch_bounds__(128) ssast_fbank_kernel(const float* const* __restrict__ wavs,
                                                          const long long* __restrict__ lens, int S, int TL,
                                                          float* __restrict__ out) {
    __shared__ float s_re[4][kFft], s_im[4][kFft], s_pw[4][kBins + 3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = blockIdx.y, b = blockIdx.z;
    const int t = blockIdx.x * 4 + warp;
    if (t >= TL) return;  // warp-uniform
    float* o = out + (((size_t)b * gridDim.y + s) * TL + t) * kSsastMel;
    if (t >= 1 + (S - kWin) / kShift) {  // the appended rows (snip_edges: frames of the window that fit)
        for (int j = lane; j < kSsastMel; j += 32) o[j] = 0.f;
        return;
    }
    const long long L = lens[b], start = (long long)s * S + (long long)t * kShift;
    const float* w = wavs[b];
    float x[13];
#pragma unroll
    for (int i = 0; i < 13; ++i) {
        const int n = lane + 32 * i;
        x[i] = (n < kWin && start + n < L) ? w[start + n] : 0.f;
    }
    float* pw = s_pw[warp];
    frame_power(x, g_hann, s_re[warp], s_im[warp], pw, lane);
    const float shift = (float)4.2677393, scale = (float)(4.5689974 * 2);
    for (int j = lane; j < kSsastMel; j += 32) {
        const int st = g_mel128.start[j], cnt = g_mel128.count[j];
        const float* mw = g_mel128.w + g_mel128.off[j];
        float acc = 0.f;
        for (int i = 0; i < cnt; ++i) acc = fmaf(pw[st + i], mw[i], acc);
        o[j] = (logf(fmaxf(acc, 1.1920928955078125e-07f)) + shift) / scale;
    }
}

cudaError_t launch_ssast_fbank(const float* const* wavs_dev, const long long* lens_dev, int B, int nseg, int S,
                               int TL, float* out, cudaStream_t s) {
    if (S < kWin || TL < 1 + (S - kWin) / kShift) return cudaErrorInvalidValue;
    if (B <= 0 || nseg <= 0) return cudaSuccess;
    ssast_fbank_kernel<<<dim3((TL + 3) / 4, nseg, B), 128, 0, s>>>(wavs_dev, lens_dev, S, TL, out);
    return cudaGetLastError();
}

// ComputeDeltas(win_length=5, mode="replicate") applied to columns [src, src+80) -> [src+80, src+160)
__global__ void delta_kernel(float* __restrict__ feat, const long long* __restrict__ lens, int max_frames, int src) {
    const int b = blockIdx.y;
    const long long L = lens[b];
    const int m = L < kWin ? 0 : (int)(1 + (L - kWin) / kShift);
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int t = idx / kMel, j = idx - t * kMel;
    if (t >= m) return;
    const float* c = feat + (size_t)b * max_frames * kFeat + src + j;
    auto at = [&](int tt) { return c[(size_t)min(max(tt, 0), m - 1) * kFeat]; };
    // F.conv1d with kernel [-2,-1,0,1,2] then / 10  (torchaudio functional.compute_deltas)
    const float v = (-2.f * at(t - 2) - at(t - 1) + 0.f * at(t) + at(t + 1) + 2.f * at(t + 2)) / 10.0f;
    feat[((size_t)b * max_frames + t) * kFeat + src + kMel + j] = v;
}

// CMVN per utterance and feature: (x - mean) / (1e-10 + std_unbiased); frames >= m are zero (pad_sequence)
__global__ void __launch_bounds__(256) cmvn_kernel(float* __restrict__ feat, const long long* __restrict__ lens,
                                                   int max_frames) {
    const int b = blockIdx.x;
    const int j = threadIdx.x;
    const long long L = lens[b];
    const int m = L < kWin ? 0 : (int)(1 + (L - kWin) / kShift);
    if (j >= kFeat) return;
    float* c = feat + (size_t)b * max_frames * kFeat + j;
    double s = 0.0;
    for (int t = 0; t < m; ++t) s += (double)c[(size_t)t * kFeat];
    const float mean = m > 0 ? (float)(s / m) : 0.f;
    double q = 0.0;
    for (int t = 0; t < m; ++t) {
        const float d = c[(size_t)t * kFeat] - mean;
        q += (double)(d * d);
    }
    const float sd = (float)sqrt(q / (double)(m - 1));  // m == 1 -> NaN, as torch.std does
    const float inv = 1.0f / (1e-10f + sd);
    for (int t = 0; t < m; ++t) c[(size_t)t * kFeat] = (c[(size_t)t * kFeat] - mean) * inv;
    for (int t = m; t < max_frames; ++t) c[(size_t)t * kFeat] = 0.f;
}

cudaError_t launch_fbank(const float* const* wavs_dev, const long long* lens_dev, int B, int max_frames, int cmvn,
                         float* out, cudaStream_t s) {
    cudaError_t e = ensure_tables(s);
    if (e != cudaSuccess) return e;
    if (max_frames <= 0 || B <= 0) return cudaSuccess;
    // without CMVN nothing else writes the rows past each utterance's frames
    if (!cmvn) {
        e = cudaMemsetAsync(out, 0, (size_t)B * max_frames * kFeat * sizeof(float), s);
        if (e != cudaSuccess) return e;
    }
    dim3 g1((max_frames + 3) / 4, B);
    fbank_frames_kernel<false, kFeat><<<g1, 128, 0, s>>>(wavs_dev, lens_dev, max_frames, out);
    dim3 g2((max_frames * kMel + 255) / 256, B);
    delta_kernel<<<g2, 256, 0, s>>>(out, lens_dev, max_frames, 0);
    delta_kernel<<<g2, 256, 0, s>>>(out, lens_dev, max_frames, kMel);
    if (cmvn) cmvn_kernel<<<B, 256, 0, s>>>(out, lens_dev, max_frames);
    return cudaGetLastError();
}

// DeCoAR 2.0 / APC CMVN (+ decimation) (decoar2/audio.py:13-38, 77-84; apc/audio.py:25-96): y = (x - mean_t) /
// (1e-10 + std_t) per utterance and mel bin over all m_b frames (unbiased std; the frames that y[::2] drops count too),
// then rows t < T_b = ceil(m_b / step) take frame step * t (step 2: DeCoAR 2.0's y[::2]; step 1: APC keeps every
// frame). Written as operand planes [B * T][128] of the first GEMM: columns 80..127 and rows t >= T_b zero.
// grid (B, 8): blockIdx.y is a 16-column slice of the operand rows (slices 5..7 only write zeros); block 256 threads.
// The statistics are a two-pass fp64 reduction over 16 frame lanes x 16 bins.
__global__ void __launch_bounds__(256) decoar2_cmvn_kernel(const float* __restrict__ feat,
                                                           const long long* __restrict__ lens, int max_frames, int T,
                                                           int step, OutPlanes op) {
    __shared__ double s_part[16][17];
    __shared__ float s_mean[16], s_sd[16];
    const int b = blockIdx.x, col0 = blockIdx.y * 16;
    const long long L = lens[b];
    const int m = L < kWin ? 0 : (int)(1 + (L - kWin) / kShift);
    const int tb = (m + step - 1) / step;
    const bool mel = col0 < kMel;  // block-uniform
    const float* base = feat + (size_t)b * max_frames * kMel + col0;
    if (mel) {
        const int j = threadIdx.x & 15, r = threadIdx.x >> 4;
        double s = 0.0;
        for (int t = r; t < m; t += 16) s += (double)base[(size_t)t * kMel + j];
        s_part[r][j] = s;
        __syncthreads();
        if (threadIdx.x < 16) {
            double a = 0.0;
#pragma unroll
            for (int i = 0; i < 16; ++i) a += s_part[i][threadIdx.x];
            s_mean[threadIdx.x] = (float)(a / m);
        }
        __syncthreads();
        const float mean = s_mean[j];
        double q = 0.0;
        for (int t = r; t < m; t += 16) {
            const float d = base[(size_t)t * kMel + j] - mean;
            q += (double)d * (double)d;
        }
        s_part[r][j] = q;
        __syncthreads();
        if (threadIdx.x < 16) {
            double a = 0.0;
#pragma unroll
            for (int i = 0; i < 16; ++i) a += s_part[i][threadIdx.x];
            s_sd[threadIdx.x] = (float)sqrt(a / (double)(m - 1));  // m == 1 -> NaN, as torch.std does
        }
        __syncthreads();
    }
    // 8 column pairs x 32 row lanes
    const int p = threadIdx.x & 7, r = threadIdx.x >> 3;
    float mean0 = 0.f, mean1 = 0.f, den0 = 1.f, den1 = 1.f;
    if (mel) {
        mean0 = s_mean[2 * p], mean1 = s_mean[2 * p + 1];
        den0 = 1e-10f + s_sd[2 * p], den1 = 1e-10f + s_sd[2 * p + 1];
    }
    for (int t = r; t < T; t += 32) {
        float y0 = 0.f, y1 = 0.f;
        if (mel && t < tb) {
            const float2 x = *reinterpret_cast<const float2*>(base + (size_t)(step * t) * kMel + 2 * p);
            y0 = (x.x - mean0) / den0;
            y1 = (x.y - mean1) / den1;
        }
        store_planes2(op, y0, y1, ((size_t)b * T + t) * kDecoar2K + col0 + 2 * p);
    }
}

cudaError_t launch_decoar2_features(const float* const* wavs_dev, const long long* lens_dev, int B, int max_frames,
                                    int T, int frame_step, float* fb, const OutPlanes& op, cudaStream_t s) {
    if (frame_step != 1 && frame_step != 2) return cudaErrorInvalidValue;
    if (max_frames <= 0 || B <= 0 || T <= 0) return cudaSuccess;
    dim3 g1((max_frames + 3) / 4, B);
    fbank_frames_kernel<true, kMel><<<g1, 128, 0, s>>>(wavs_dev, lens_dev, max_frames, fb);
    decoar2_cmvn_kernel<<<dim3(B, kDecoar2K / 16), 256, 0, s>>>(fb, lens_dev, max_frames, T, frame_step, op);
    return cudaGetLastError();
}

}  // namespace s3b
