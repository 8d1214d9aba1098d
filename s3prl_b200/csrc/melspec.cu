// `mel` / `linear` baseline upstreams: torch.stft power spectrogram (+ HTK mel filterbank), log, per-utterance CMVN.
// Replaces OnlinePreprocessor.forward (s3prl/upstream/baseline/preprocessor.py:150-223, mel.yaml / linear.yaml:
// win 25 ms, hop 10 ms, n_fft 400 -> 201 bins, hann window (periodic), center=True with reflect padding, power 2,
// torchaudio MelScale(n_mels=80, htk, f_min 0, f_max 8000), log(x + 1e-10), CMVN with unbiased std + 1e-10).
// One warp per frame: the 400-point DFT is evaluated directly from cos/sin tables (400 is not a power of two;
// 201 x 400 complex MACs per frame), then the dense 201 x 80 mel projection. All fp32.
#include <math.h>

#include <vector>

#include "common.cuh"
#include "fbank.cuh"

namespace s3b {

static constexpr int kNfft = 400, kHop = 160, kNbin = 201, kNmel = 80;

struct MelTables {
    float window[kNfft];  // hann(400), periodic
    float cs[kNfft], sn[kNfft];
    float fb[kNbin * kNmel];  // torchaudio.functional.melscale_fbanks(201, 0, 8000, 80, 16000, None, "htk")
};
__device__ MelTables g_mel;
static bool g_mel_ready[64] = {false};

static void build_mel_tables(MelTables& t) {
    for (int n = 0; n < kNfft; ++n) {
        t.window[n] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * n / kNfft));
        t.cs[n] = (float)cos(2.0 * M_PI * n / kNfft);
        t.sn[n] = (float)sin(2.0 * M_PI * n / kNfft);
    }
    auto hz2mel = [](double f) { return 2595.0 * log10(1.0 + f / 700.0); };
    auto mel2hz = [](double m) { return 700.0 * (pow(10.0, m / 2595.0) - 1.0); };
    const double m_min = hz2mel(0.0), m_max = hz2mel(8000.0);
    std::vector<double> f_pts(kNmel + 2);
    for (int i = 0; i < kNmel + 2; ++i) f_pts[i] = mel2hz(m_min + (m_max - m_min) * i / (kNmel + 1));
    for (int k = 0; k < kNbin; ++k) {
        const double f = 8000.0 * k / (kNbin - 1);
        for (int j = 0; j < kNmel; ++j) {
            const double down = (f - f_pts[j]) / (f_pts[j + 1] - f_pts[j]);
            const double up = (f_pts[j + 2] - f) / (f_pts[j + 2] - f_pts[j + 1]);
            const double w = fmax(0.0, fmin(down, up));
            t.fb[k * kNmel + j] = (float)w;
        }
    }
}

static cudaError_t ensure_mel_tables(cudaStream_t s) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 64 && g_mel_ready[dev]) return cudaSuccess;
    static MelTables host;
    build_mel_tables(host);
    e = cudaMemcpyToSymbolAsync(g_mel, &host, sizeof(host), 0, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(s);
    if (e == cudaSuccess && dev < 64) g_mel_ready[dev] = true;
    return e;
}

// length of each utterance after dropping trailing exact zeros (preprocessor.py:166-175: last non-zero index + 1,
// the full length if every sample is zero)
__global__ void trimmed_len_kernel(const float* const* __restrict__ wavs, const long long* __restrict__ lens,
                                   long long* __restrict__ out) {
    const int b = blockIdx.x;
    const float* w = wavs[b];
    const long long n = lens[b];
    long long last = -1;
    for (long long i = threadIdx.x; i < n; i += blockDim.x)
        if (w[i] != 0.0f) last = i;
    __shared__ long long red[32];
    for (int o = 16; o > 0; o >>= 1) {
        const long long other = __shfl_xor_sync(0xffffffffu, last, o);
        last = other > last ? other : last;
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = last;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) last = red[i] > last ? red[i] : last;
        out[b] = last < 0 ? n : last + 1;
    }
}

cudaError_t launch_trimmed_lengths(const float* const* wavs_dev, const long long* lens_dev, int B, long long* out_dev,
                                   cudaStream_t s) {
    trimmed_len_kernel<<<B, 1024, 0, s>>>(wavs_dev, lens_dev, out_dev);
    return cudaGetLastError();
}

// grid (ceil(n_frames / 4), B); block 128 = 4 warps = 4 frames. tmp: [B][n_frames][dim], dim = 80 (mel) or 201
__global__ void __launch_bounds__(128) stft_mel_kernel(const float* const* __restrict__ wavs,
                                                       const long long* __restrict__ lens, long long Lp, int n_frames,
                                                       int mel, float* __restrict__ tmp) {
    __shared__ float s_x[4][kNfft];
    __shared__ float s_cs[kNfft], s_sn[kNfft];
    __shared__ float s_pw[4][kNbin + 3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < kNfft; i += blockDim.x) s_cs[i] = g_mel.cs[i], s_sn[i] = g_mel.sn[i];
    const int b = blockIdx.y;
    const int t = blockIdx.x * 4 + warp;
    const long long len = lens[b];
    const float* w = wavs[b];
    if (t < n_frames) {
        for (int n = lane; n < kNfft; n += 32) {
            long long i = (long long)t * kHop - kNfft / 2 + n;  // center=True
            if (i < 0) i = -i;                                   // reflect padding of the padded row [0, Lp)
            if (i >= Lp) i = 2 * (Lp - 1) - i;
            const float v = (i >= 0 && i < len) ? w[i] : 0.0f;   // zero padding beyond this utterance
            s_x[warp][n] = v * g_mel.window[n];
        }
    }
    __syncthreads();
    if (t >= n_frames) return;
    float re[7], im[7];
    int idx[7], kk[7];
#pragma unroll
    for (int q = 0; q < 7; ++q) re[q] = 0.f, im[q] = 0.f, idx[q] = 0, kk[q] = lane + 32 * q;
    for (int n = 0; n < kNfft; ++n) {
        const float x = s_x[warp][n];
#pragma unroll
        for (int q = 0; q < 7; ++q) {
            re[q] = fmaf(x, s_cs[idx[q]], re[q]);
            im[q] = fmaf(-x, s_sn[idx[q]], im[q]);
            idx[q] += kk[q];
            if (idx[q] >= kNfft) idx[q] -= kNfft;
        }
    }
    float* pw = s_pw[warp];
#pragma unroll
    for (int q = 0; q < 7; ++q)
        if (kk[q] < kNbin) {
            const float a = sqrtf(re[q] * re[q] + im[q] * im[q]);  // abs().pow(2)
            pw[kk[q]] = a * a;
        }
    __syncwarp();
    if (mel) {
        float* o = tmp + ((size_t)b * n_frames + t) * kNmel;
        for (int j = lane; j < kNmel; j += 32) {
            float acc = 0.f;
            for (int k = 0; k < kNbin; ++k) acc = fmaf(pw[k], g_mel.fb[k * kNmel + j], acc);
            o[j] = logf(acc + 1e-10f);
        }
    } else {
        float* o = tmp + ((size_t)b * n_frames + t) * kNbin;
        for (int k = lane; k < kNbin; k += 32) o[k] = logf(pw[k] + 1e-10f);
    }
}

// CMVN over the first feats_len[b] frames, then keep final_len[b] frames, zero up to t_out (pad_sequence)
__global__ void __launch_bounds__(256) mel_cmvn_kernel(const float* __restrict__ tmp, int n_frames, int dim,
                                                       const int* __restrict__ feats_len,
                                                       const int* __restrict__ final_len, int t_out,
                                                       float* __restrict__ out) {
    const int b = blockIdx.x;
    const int m = feats_len[b];
    const int keep = min(final_len[b], m);
    for (int j = threadIdx.x; j < dim; j += blockDim.x) {
        const float* c = tmp + (size_t)b * n_frames * dim + j;
        double s = 0.0;
        for (int t = 0; t < m; ++t) s += (double)c[(size_t)t * dim];
        const float mean = m > 0 ? (float)(s / m) : 0.f;
        double q = 0.0;
        for (int t = 0; t < m; ++t) {
            const float d = c[(size_t)t * dim] - mean;
            q += (double)(d * d);
        }
        const float inv = 1.0f / ((float)sqrt(q / (double)(m - 1)) + 1e-10f);
        float* o = out + (size_t)b * t_out * dim + j;
        for (int t = 0; t < t_out; ++t) o[(size_t)t * dim] = t < keep ? (c[(size_t)t * dim] - mean) * inv : 0.f;
    }
}

cudaError_t launch_melspec(const float* const* wavs_dev, const long long* trim_lens_dev, int B, long long Lp,
                           int mel, int cmvn, const int* feats_len_dev, const int* final_len_dev, int t_out, float* tmp,
                           float* out, cudaStream_t s) {
    cudaError_t e = ensure_mel_tables(s);
    if (e != cudaSuccess) return e;
    const int n_frames = (int)(1 + Lp / kHop);
    dim3 g1((n_frames + 3) / 4, B);
    // without CMVN the log features of every frame of the padded batch are the output
    stft_mel_kernel<<<g1, 128, 0, s>>>(wavs_dev, trim_lens_dev, Lp, n_frames, mel, cmvn ? tmp : out);
    if (cmvn)
        mel_cmvn_kernel<<<B, 256, 0, s>>>(tmp, n_frames, mel ? kNmel : kNbin, feats_len_dev, final_len_dev, t_out,
                                          out);
    return cudaGetLastError();
}

}  // namespace s3b
