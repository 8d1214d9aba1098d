// SSAST (s3prl/upstream/ssast/{expert,ast_models}.py) around the shared pre-LN encoder: the patch-embedding GEMM's
// operand, the class tokens and positional table, and the per-layer output layout. The fbank front end is fbank.cu's
// ssast_fbank_kernel; the patch GEMM, the layers' GEMMs, attention and LayerNorm are the library's own kernels.
#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

static constexpr int kSsastBins = 128, kPatch = 16, kPatchStride = 10;

// one thread per element pair; the frame model copies [SB][TL][128] into planes, the patch model gathers each pair
// (kt, kt + 1) of patch row (sb, fi, ti) from two consecutive frames of column 10 fi + kf
__global__ void __launch_bounds__(256) ssast_patches_kernel(const float* __restrict__ feat, size_t pairs, int TL,
                                                            int patch_f, int tdim, OutPlanes op) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pairs) return;
    const size_t e = 2 * i;
    if (patch_f == 1) {
        const float2 v = *reinterpret_cast<const float2*>(feat + e);
        store_planes2(op, v.x, v.y, e);
        return;
    }
    const int K = kPatch * kPatch, P = patch_f * tdim;
    const size_t row = e / K;
    const int col = (int)(e - row * K);
    const size_t sb = row / P;
    const int p = (int)(row - sb * P);
    const int fi = p / tdim, ti = p - fi * tdim, kf = col / kPatch, kt = col - kf * kPatch;
    const float* src = feat + ((sb * TL + (size_t)(ti * kPatchStride + kt)) * kSsastBins + fi * kPatchStride + kf);
    store_planes2(op, src[0], src[kSsastBins], e);
}

cudaError_t launch_ssast_patches(const float* feat, int SB, int TL, int patch_f, int tdim, const OutPlanes& op,
                                 cudaStream_t s) {
    if (patch_f != 1 && patch_f != 12) return cudaErrorInvalidValue;
    const size_t n = patch_f == 1 ? (size_t)SB * TL * kSsastBins : (size_t)SB * patch_f * tdim * kPatch * kPatch;
    if (n == 0) return cudaSuccess;
    const size_t pairs = n / 2;
    ssast_patches_kernel<<<(unsigned)((pairs + 255) / 256), 256, 0, s>>>(feat, pairs, TL, patch_f, tdim, op);
    return cudaGetLastError();
}

// one thread per float4 of x; pos [2 + P][D]
__global__ void __launch_bounds__(256) ssast_tokens_kernel(float4* __restrict__ x, const float4* __restrict__ cls,
                                                           const float4* __restrict__ dist,
                                                           const float4* __restrict__ pos, size_t n4, int rows,
                                                           int d4) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const size_t r = i / d4;
    const int c = (int)(i - r * d4);
    const int tok = (int)(r % rows);
    const float4 pe = pos[(size_t)tok * d4 + c];
    const float4 v = tok == 0 ? cls[c] : tok == 1 ? dist[c] : x[i];
    x[i] = make_float4(v.x + pe.x, v.y + pe.y, v.z + pe.z, v.w + pe.w);
}

cudaError_t launch_ssast_tokens(float* x, const float* cls, const float* dist, const float* pos, int SB, int P, int D,
                                cudaStream_t s) {
    if (D % 4 != 0) return cudaErrorInvalidValue;
    const size_t n4 = (size_t)SB * (P + 2) * (D / 4);
    if (n4 == 0) return cudaSuccess;
    ssast_tokens_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(cls), reinterpret_cast<const float4*>(dist),
        reinterpret_cast<const float4*>(pos), n4, P + 2, D / 4);
    return cudaGetLastError();
}

// one thread per float4 of out
__global__ void __launch_bounds__(256) ssast_fold_kernel(const float4* __restrict__ x, size_t n4, int nseg, int P,
                                                         int tdim, int patch_f, int d4, int T,
                                                         float4* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const int w4 = patch_f * d4;
    const size_t bt = i / w4;
    const int c = (int)(i - bt * w4);
    const size_t b = bt / T;
    const int t = (int)(bt - b * T);
    const int fi = c / d4, d = c - fi * d4;
    const int s = t / tdim, ti = t - s * tdim;
    const size_t row = (b * nseg + s) * (size_t)(P + 2) + 2 + fi * tdim + ti;
    out[i] = x[row * d4 + d];
}

cudaError_t launch_ssast_fold(const float* x, int B, int nseg, int P, int tdim, int patch_f, int D, int T, float* out,
                              cudaStream_t s) {
    if (D % 4 != 0 || T > nseg * tdim || P != patch_f * tdim) return cudaErrorInvalidValue;
    const size_t n4 = (size_t)B * T * patch_f * (D / 4);
    if (n4 == 0) return cudaSuccess;
    ssast_fold_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, s>>>(reinterpret_cast<const float4*>(x), n4, nseg, P,
                                                                     tdim, patch_f, D / 4, T,
                                                                     reinterpret_cast<float4*>(out));
    return cudaGetLastError();
}

}  // namespace s3b
