// LSTM recurrence of modified CPC (s3prl/upstream/cpc/model.py CPCAR with mode "LSTM"): one nn.LSTM(256, 256) layer
// per launch over the whole padded batch (no packing: every utterance runs all T steps), h_0 = c_0 = 0, PyTorch's
// gate order i, f, g, o:
//   i = sigmoid(xg_i + W_hi h),  f = sigmoid(xg_f + W_hf h),  g = tanh(xg_g + W_hg h),  o = sigmoid(xg_o + W_ho h),
//   c' = f * c + i * g,  h' = o * tanh(c')
// where xg = W_ih x + b_ih + b_hh comes from one GEMM over all frames.
//
// One thread-block cluster of kCpcLstmCtas = 8 CTAs (a portable cluster size) runs a group of kCpcLstmGroup
// utterances. CTA c owns hidden units [32c, 32c + 32) and keeps their 128 rows of W_hh (4 gates x 32 units) resident in
// shared memory as fp32 (128 KiB). Every step each CTA computes its units for the group from the full previous state h
// (in its own shared memory), then pushes the new 32 values per utterance into every peer's state buffer through
// distributed shared memory; one cluster barrier per step closes the step. The state is double-buffered so that a
// step's pushes never land in the buffer peers are still reading. The cell state of a (unit, utterance) pair lives in
// the registers of the lanes that compute it.
//
// Arithmetic: plain fp32 FMAs. Lane l of a warp accumulates k = 128 i + 4 l .. + 3 (i = 0, 1) in a fixed order, and a
// butterfly over the 32 lanes completes each dot product. The tree depends neither on the utterance's slot in its
// group nor on the group, so an utterance's outputs are bit-identical in any batch.
#include <math.h>

#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

namespace {

constexpr int kH = kCpcLstmHidden;   // 256
constexpr int kG = kCpcLstmGroup;    // utterances per cluster
constexpr int kCtas = kCpcLstmCtas;  // CTAs per cluster
constexpr int kUnits = kH / kCtas;   // 32 hidden units per CTA
constexpr int kThreads = 256;        // 8 warps x 4 units
constexpr int kRows = 4 * kUnits;    // 128 W_hh rows per CTA
constexpr int kPairs = 4 * kG;       // (unit, utterance) pairs per warp: 16
constexpr int kVals = 4 * kPairs;    // dot products per warp and step: 64
static_assert(kThreads / 32 * 4 == kUnits && kPairs == 16, "warp tiling: 4 units x kG utterances per warp");

struct CpcLstmSmem {
    float w[kRows][kH];     // row 4 j + q = W_hh[q * 256 + 32 c + j]
    float h[2][kG][kH];     // double-buffered state of the group
    float hnew[kG][kUnits];  // this CTA's new state (pushed to the peers and written out)
};
static_assert(sizeof(CpcLstmSmem) <= 227 * 1024, "the recurrence kernel's shared memory exceeds 227 KB");

// grid: kCtas x number of groups, cluster (kCtas, 1, 1); block kThreads; dynamic smem sizeof(CpcLstmSmem)
__global__ void __launch_bounds__(kThreads, 1) cpc_lstm_kernel(CpcLstmParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    CpcLstmSmem& s = *reinterpret_cast<CpcLstmSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c = (int)cluster_rank();
    const int grp = blockIdx.x / kCtas;
    const int u0 = c * kUnits;

    // resident W_hh slice, h_0 = 0
    for (int i = tid; i < kRows * (kH / 4); i += kThreads) {
        const int r = i / (kH / 4), k4 = i % (kH / 4);
        const int j = r / 4, q = r % 4;
        reinterpret_cast<float4*>(&s.w[r][0])[k4] =
            reinterpret_cast<const float4*>(p.whh + ((size_t)q * kH + u0 + j) * kH)[k4];
    }
    for (int i = tid; i < kG * kH; i += kThreads) (&s.h[0][0][0])[i] = 0.f;
    // every CTA of the cluster is running and initialised before any peer writes into its shared memory
    cluster_sync();

    // after the butterfly, lanes l and l ^ 1 both hold pair (unit jl, slot gl); the even one writes
    const int pair = lane >> 1, jl = pair / kG, gl = pair % kG;
    const int j = warp * 4 + jl, unit = u0 + j;
    const int bq = grp * kG + gl;  // the utterance of slot gl (>= B: an empty slot, computed and never written)
    const bool live = bq < p.B;
    const bool writer = (lane & 1) == 0;
    const float* xg_u = p.xg + (size_t)(live ? bq : 0) * p.T * 4 * kH + unit;
    auto xg_at = [=](int t, int q) -> float { return (live && t < p.T) ? xg_u[(size_t)t * 4 * kH + q * kH] : 0.f; };
    float x0 = xg_at(0, 0), x1 = xg_at(0, 1), x2 = xg_at(0, 2), x3 = xg_at(0, 3);
    float cell = 0.f;

    for (int t = 0; t < p.T; ++t) {
        const int cur = t & 1;
        // prefetch step t + 1's inputs; their latency hides behind this step's dot products
        const float n0 = xg_at(t + 1, 0), n1 = xg_at(t + 1, 1), n2 = xg_at(t + 1, 2), n3 = xg_at(t + 1, 3);

        float acc[kVals];
#pragma unroll
        for (int v = 0; v < kVals; ++v) acc[v] = 0.f;
#pragma unroll
        for (int i = 0; i < kH / 128; ++i) {
            const int k = 128 * i + 4 * lane;
            float4 hv[kG];
#pragma unroll
            for (int g = 0; g < kG; ++g) hv[g] = *reinterpret_cast<const float4*>(&s.h[cur][g][k]);
#pragma unroll
            for (int ju = 0; ju < 4; ++ju)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 wv = *reinterpret_cast<const float4*>(&s.w[4 * (warp * 4 + ju) + q][k]);
#pragma unroll
                    for (int g = 0; g < kG; ++g) {
                        float& a = acc[(ju * kG + g) * 4 + q];
                        a = fmaf(wv.x, hv[g].x, a);
                        a = fmaf(wv.y, hv[g].y, a);
                        a = fmaf(wv.z, hv[g].z, a);
                        a = fmaf(wv.w, hv[g].w, a);
                    }
                }
        }
        // butterfly reduce-scatter: offsets 16, 8, 4, 2 halve the kept values (64 -> 4), offset 1 completes them.
        // Value index v = pair * 4 + gate; after the four halvings lane l keeps pair l >> 1.
        halve<16, kVals / 2>(acc, lane);
        halve<8, kVals / 4>(acc, lane);
        halve<4, kVals / 8>(acc, lane);
        halve<2, kVals / 16>(acc, lane);
        const float hi = acc[0] + __shfl_xor_sync(0xffffffffu, acc[0], 1);
        const float hf = acc[1] + __shfl_xor_sync(0xffffffffu, acc[1], 1);
        const float hg = acc[2] + __shfl_xor_sync(0xffffffffu, acc[2], 1);
        const float ho = acc[3] + __shfl_xor_sync(0xffffffffu, acc[3], 1);

        const float gi = sigmoid_f(x0 + hi), gf = sigmoid_f(x1 + hf), gg = tanhf(x2 + hg), go = sigmoid_f(x3 + ho);
        cell = gf * cell + gi * gg;
        if (writer) s.hnew[gl][j] = go * tanhf(cell);
        __syncthreads();
        // push the new state to every CTA of the cluster (own included): 8 peers x kG x 8 float4, one per thread
        const int nxt = cur ^ 1;
        for (int i = tid; i < kCtas * kG * (kUnits / 4); i += kThreads) {
            const int peer = i / (kG * (kUnits / 4)), rem = i % (kG * (kUnits / 4));
            const int g = rem / (kUnits / 4), q4 = rem % (kUnits / 4);
            const float4 v = reinterpret_cast<const float4*>(&s.hnew[g][0])[q4];
            st_cluster_f4(peer_addr(&s.h[nxt][g][u0 + 4 * q4], (uint32_t)peer), v);
        }
        // layer output (fp32 hidden state and / or the next layer's operand planes), two columns per thread
        if (tid < kG * (kUnits / 2)) {
            const int g = tid / (kUnits / 2), cp = tid % (kUnits / 2);
            const int bo = grp * kG + g;
            if (bo < p.B) {
                const float o0 = s.hnew[g][2 * cp], o1 = s.hnew[g][2 * cp + 1];
                const size_t e = ((size_t)bo * p.T + t) * kH + u0 + 2 * cp;
                if (p.out != nullptr) *reinterpret_cast<float2*>(p.out + e) = make_float2(o0, o1);
                if (p.op.hi != nullptr) store_planes2(p.op, o0, o1, e);
            }
        }
        x0 = n0, x1 = n1, x2 = n2, x3 = n3;
        cluster_sync();
    }
}

cudaLaunchConfig_t cpc_lstm_config(int groups, cudaStream_t s, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kCtas * groups);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = sizeof(CpcLstmSmem);
    cfg.stream = s;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kCtas, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

PerDeviceOnce g_cpc_lstm_attr;

cudaError_t cpc_lstm_set_attributes() {
    bool& done = g_cpc_lstm_attr.current();
    if (done) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(cpc_lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(CpcLstmSmem));
    if (e == cudaSuccess) done = true;
    return e;
}

}  // namespace

cudaError_t cpc_lstm_max_active_clusters(int* n) {
    cudaError_t e = cpc_lstm_set_attributes();
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = cpc_lstm_config(1, 0, attr);
    return cudaOccupancyMaxActiveClusters(n, cpc_lstm_kernel, &cfg);
}

cudaError_t launch_cpc_lstm(const CpcLstmParams& p, cudaStream_t s) {
    if (p.B <= 0 || p.T <= 0) return cudaSuccess;
    cudaError_t e = cpc_lstm_set_attributes();
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = cpc_lstm_config((p.B + kG - 1) / kG, s, attr);
    return cudaLaunchKernelEx(&cfg, cpc_lstm_kernel, p);
}

}  // namespace s3b
