// Fused Featurizer weighted sum + all-gather over NVLink peer memory (one process per GPU on one NVSwitch node).
//
// The multi-GPU step of the path ends with the softmax-weighted layer sum of every rank's
// utterances being gathered on all ranks. Instead of "weighted_sum kernel -> NCCL all-gather" (two kernels, a 49 MB
// round trip through local HBM and a lock-step collective), ONE kernel streams the NL+1 local hidden states once and
// stores each result vector straight into every rank's gathered buffer (its own and the 7 peers', mapped through
// CUDA IPC), then publishes a per-(slot, rank) sequence flag with release semantics at system scope. A rank's
// stream waits for the flags of step s-1 at the start of step s (wait_flags_kernel), so ranks are coupled with one
// step of slack instead of per collective. Replaces Featurizer._weighted_sum + the gather of
// s3prl/upstream/interfaces.py:217-248 for the sharded run.
#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

static constexpr int kMaxPeers = 16;
static constexpr int kMaxLayersP = 64;

struct PushParams {
    const float4* hs;       // local hidden states, layer l at hs + l * layer_stride4
    size_t layer_stride4;
    size_t n4;              // float4 per layer (local block)
    int NL;
    const float* w;         // [NL] device
    float4* dst[kMaxPeers];     // every rank's gathered slot, already offset to THIS rank's block
    uint32_t* flag[kMaxPeers];  // every rank's flag word for (slot, this rank)
    int n_peers;
    uint32_t seq;
    unsigned int* counter;  // local: blocks done (reset by the last block)
};

__global__ void __launch_bounds__(256) weighted_sum_push_kernel(const __grid_constant__ PushParams p) {
    __shared__ float lw[kMaxLayersP];
    __shared__ bool is_last;
    if ((int)threadIdx.x < p.NL) lw[threadIdx.x] = p.w[threadIdx.x];
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int l = 0; l < p.NL; ++l) {  // same operation order as weighted_sum_kernel: bit-identical values
            const float4 v = p.hs[(size_t)l * p.layer_stride4 + i];
            const float wl = lw[l];
            acc.x = fmaf(wl, v.x, acc.x), acc.y = fmaf(wl, v.y, acc.y);
            acc.z = fmaf(wl, v.z, acc.z), acc.w = fmaf(wl, v.w, acc.w);
        }
#pragma unroll 4
        for (int r = 0; r < p.n_peers; ++r) p.dst[r][i] = acc;
    }
    // all stores of this block are performed system-wide before the block is counted
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(p.counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (is_last) {
        __threadfence_system();
        if (threadIdx.x < p.n_peers)
            asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p.flag[threadIdx.x]), "r"(p.seq) : "memory");
        if (threadIdx.x == 0) *p.counter = 0;
    }
}

__global__ void wait_flags_kernel(const uint32_t* flags, int n, uint32_t seq) {
    if ((int)threadIdx.x >= n) return;
    const long long t0 = clock64();
    uint32_t v;
    do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
        if (v >= seq) break;
        if (clock64() - t0 > 20000000000LL) {  // ~10 s: a peer died; fail the launch instead of hanging the GPU
            printf("s3b: peer flag timeout (rank slot %d: have %u, want %u)\n", (int)threadIdx.x, v, seq);
            __trap();
        }
    } while (true);
}

cudaError_t launch_weighted_sum_push(const float* hs, int NL, size_t n_per_layer, size_t layer_stride, const float* w,
                                     float* const* peer_dst, uint32_t* const* peer_flag, int n_peers, uint32_t seq,
                                     unsigned int* counter, cudaStream_t s) {
    if (NL > kMaxLayersP || n_peers > kMaxPeers || n_peers < 1 || (n_per_layer & 3) != 0 || (layer_stride & 3) != 0)
        return cudaErrorInvalidValue;
    PushParams p;
    p.hs = reinterpret_cast<const float4*>(hs);
    p.layer_stride4 = layer_stride / 4, p.n4 = n_per_layer / 4, p.NL = NL, p.w = w;
    for (int r = 0; r < n_peers; ++r) p.dst[r] = reinterpret_cast<float4*>(peer_dst[r]), p.flag[r] = peer_flag[r];
    p.n_peers = n_peers, p.seq = seq, p.counter = counter;
    size_t blocks = (p.n4 + 255) / 256;
    if (blocks > 132 * 4) blocks = 132 * 4;
    if (blocks == 0) blocks = 1;
    weighted_sum_push_kernel<<<(unsigned)blocks, 256, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_wait_flags(const uint32_t* flags, int n, uint32_t seq, cudaStream_t s) {
    if (n < 1 || n > 32) return cudaErrorInvalidValue;
    wait_flags_kernel<<<1, 32, 0, s>>>(flags, n, seq);
    return cudaGetLastError();
}

}  // namespace s3b
