// fbank.cu launcher
#pragma once
#include <cuda_runtime.h>

namespace s3b {
// out: [B][max_frames][240] fp32 (80 log-mel | 80 delta | 80 delta-delta, CMVN applied when cmvn != 0, zero
// beyond each length)
cudaError_t launch_fbank(const float* const* wavs_dev, const long long* lens_dev, int B, int max_frames, int cmvn,
                         float* out, cudaStream_t s);
}  // namespace s3b

namespace s3b {
// melspec.cu
cudaError_t launch_trimmed_lengths(const float* const* wavs_dev, const long long* lens_dev, int B, long long* out_dev,
                                   cudaStream_t s);
// dim = 80 (mel != 0) or 201. cmvn != 0: tmp [B][1 + Lp/160][dim] scratch, out [B][t_out][dim];
// cmvn == 0: out [B][1 + Lp/160][dim] log features of every frame (tmp, feats_len, final_len and t_out unused)
cudaError_t launch_melspec(const float* const* wavs_dev, const long long* trim_lens_dev, int B, long long Lp, int mel,
                           int cmvn, const int* feats_len_dev, const int* final_len_dev, int t_out, float* tmp,
                           float* out, cudaStream_t s);
}  // namespace s3b
