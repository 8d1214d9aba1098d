// GRU recurrence of APC / VQ-APC (s3prl/upstream/apc/apc.py:101-169): one nn.GRU(512, 512) layer per launch over
// packed (ragged) sequences, h_0 = 0, PyTorch's gate order r, z, n:
//   r = sigmoid(xg_r + W_hr h),  z = sigmoid(xg_z + W_hz h),  n = tanh(xg_n + r * (W_hn h + b_hn)),
//   h' = (1 - z) * n + z * h
// where xg = W_i x + b_i (+ b_hr, b_hz folded into the r and z columns) comes from one GEMM over all frames.
//
// One thread-block cluster of kGruCtas = 16 CTAs runs a group of kGruGroup utterances. CTA c of the cluster owns hidden
// units [32c, 32c + 32) and keeps their 96 rows of W_hh resident in shared memory as fp32 (192 KB). Every step, each
// CTA computes its units for the group from the full previous state h (in its own shared memory), then pushes the new
// 32 values per utterance into every peer's state buffer through distributed shared memory; one cluster barrier
// (arrive.release / wait.acquire) per step closes the step. The state is double-buffered so that a step's pushes never
// land in the buffer peers are still reading. No CTA ever waits on a CTA outside its cluster.
//
// Arithmetic: plain fp32 FMAs. Lane l of a warp accumulates k = 128 i + 4 l .. + 3 (i = 0..3) in a fixed order, and a
// butterfly over the 32 lanes completes each dot product. The tree depends neither on the utterance's slot in its
// group nor on the group, so an utterance's outputs are bit-identical in any batch.
#include <math.h>

#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

namespace {

constexpr int kH = kGruHidden;       // 512
constexpr int kG = kGruGroup;        // utterances per cluster
constexpr int kCtas = kGruCtas;      // CTAs per cluster
constexpr int kUnits = kH / kCtas;   // 32 hidden units per CTA
constexpr int kThreads = 256;        // 8 warps x 4 units
constexpr int kRows = 3 * kUnits;    // 96 W_hh rows per CTA
constexpr int kPairs = 4 * kG;       // (unit, utterance) pairs per warp: 16
constexpr int kVals = 3 * kPairs;    // dot products per warp and step: 48

struct GruSmem {
    float w[kRows][kH];         // row 3 j + q = W_hh[q * 512 + 32 c + j]
    float h[2][kG][kH];         // double-buffered state of the group
    float hnew[kG][kUnits];     // this CTA's new state (pushed to the peers)
    float out[kG][kUnits];      // this CTA's layer output (+ residual)
    float bhn[kUnits];
};
// one CTA per SM with the opt-in maximum of dynamic shared memory (227 KB on sm_90)
static_assert(sizeof(GruSmem) <= 227 * 1024, "the recurrence kernel's shared memory exceeds 227 KB");

// grid: kCtas x number of groups, cluster (kCtas, 1, 1); block kThreads; dynamic smem sizeof(GruSmem)
__global__ void __launch_bounds__(kThreads, 1) gru_cluster_kernel(GruParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GruSmem& s = *reinterpret_cast<GruSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c = (int)cluster_rank();
    const int grp = blockIdx.x / kCtas;
    const int u0 = c * kUnits;

    // the group: slots of the length-sorted order; a missing slot runs with length 0
    int b_of[kG], len_of[kG];
    int tg = 0;
#pragma unroll
    for (int g = 0; g < kG; ++g) {
        const int idx = grp * kG + g;
        b_of[g] = idx < p.B ? p.order[idx] : -1;
        len_of[g] = idx < p.B ? p.len[b_of[g]] : 0;
        tg = max(tg, len_of[g]);
    }

    // resident W_hh slice, b_hn, h_0 = 0
    for (int i = tid; i < kRows * (kH / 4); i += kThreads) {
        const int r = i / (kH / 4), k4 = i % (kH / 4);
        const int j = r / 3, q = r % 3;
        const float4 v = reinterpret_cast<const float4*>(p.whh + ((size_t)q * kH + u0 + j) * kH)[k4];
        reinterpret_cast<float4*>(&s.w[r][0])[k4] = v;
    }
    if (tid < kUnits) s.bhn[tid] = p.bhn[u0 + tid];
    for (int i = tid; i < kG * kH; i += kThreads) (&s.h[0][0][0])[i] = 0.f;
    // every CTA of the cluster is running and initialised before any peer writes into its shared memory
    cluster_sync();

    // this lane finalises pair (unit jl, slot gl) after the butterfly; lanes l and l ^ 1 both hold it, the even one
    // writes
    const int pair = lane >> 1, jl = pair / kG, gl = pair % kG;
    const int j = warp * 4 + jl, unit = u0 + j;
    int bq = 0, lq = 0;  // b_of[gl], len_of[gl] without a dynamically indexed (local-memory) array
#pragma unroll
    for (int g = 0; g < kG; ++g)
        if (g == gl) bq = b_of[g], lq = len_of[g];
    const bool writer = (lane & 1) == 0;
    const float* xg_u = p.xg + (size_t)bq * p.T * 3 * kH + unit;
    const float* res_u = p.res != nullptr ? p.res + (size_t)bq * p.T * kH + unit : nullptr;
    auto xg_at = [=](int t, int q) -> float { return (t < lq) ? xg_u[(size_t)t * 3 * kH + q * kH] : 0.f; };
    auto res_at = [=](int t) -> float { return (res_u != nullptr && t < lq) ? res_u[(size_t)t * kH] : 0.f; };
    float xr = xg_at(0, 0), xz = xg_at(0, 1), xn = xg_at(0, 2), xres = res_at(0);

    for (int t = 0; t < tg; ++t) {
        const int cur = t & 1;
        // prefetch step t + 1's inputs; their latency hides behind this step's dot products
        const float nxr = xg_at(t + 1, 0), nxz = xg_at(t + 1, 1), nxn = xg_at(t + 1, 2), nres = res_at(t + 1);

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
                for (int q = 0; q < 3; ++q) {
                    const float4 wv = *reinterpret_cast<const float4*>(&s.w[3 * (warp * 4 + ju) + q][k]);
#pragma unroll
                    for (int g = 0; g < kG; ++g) {
                        float& a = acc[(ju * kG + g) * 3 + q];
                        a = fmaf(wv.x, hv[g].x, a);
                        a = fmaf(wv.y, hv[g].y, a);
                        a = fmaf(wv.z, hv[g].z, a);
                        a = fmaf(wv.w, hv[g].w, a);
                    }
                }
        }
        // butterfly reduce-scatter: offsets 16, 8, 4, 2 halve the kept values (48 -> 3), offset 1 completes them.
        // Value index v = pair * 3 + gate; after the four halvings lane l keeps pair l >> 1.
        halve<16, kVals / 2>(acc, lane);
        halve<8, kVals / 4>(acc, lane);
        halve<4, kVals / 8>(acc, lane);
        halve<2, kVals / 16>(acc, lane);
        float hr = acc[0] + __shfl_xor_sync(0xffffffffu, acc[0], 1);
        float hz = acc[1] + __shfl_xor_sync(0xffffffffu, acc[1], 1);
        float hn = acc[2] + __shfl_xor_sync(0xffffffffu, acc[2], 1);

        if (writer) {
            const float hp = s.h[cur][gl][unit];
            const float r = sigmoid_f(xr + hr);
            const float z = sigmoid_f(xz + hz);
            const float n = tanhf(xn + r * (hn + s.bhn[j]));
            const float hq = (1.0f - z) * n + z * hp;
            s.hnew[gl][j] = hq;
            s.out[gl][j] = hq + xres;
        }
        __syncthreads();
        // push the new state to every CTA of the cluster (own included): 16 peers x kG x 8 float4
        const int nxt = cur ^ 1;
        for (int i = tid; i < kCtas * kG * (kUnits / 4); i += kThreads) {
            const int peer = i / (kG * (kUnits / 4)), rem = i % (kG * (kUnits / 4));
            const int g = rem / (kUnits / 4), q4 = rem % (kUnits / 4);
            const float4 v = reinterpret_cast<const float4*>(&s.hnew[g][0])[q4];
            st_cluster_f4(peer_addr(&s.h[nxt][g][u0 + 4 * q4], (uint32_t)peer), v);
        }
        // layer output (fp32 hidden state + the next layer's operand planes), two columns per thread
        if (tid < kG * (kUnits / 2)) {
            const int g = tid / (kUnits / 2), cp = tid % (kUnits / 2);
            int bo = 0, lo = 0;
#pragma unroll
            for (int gg = 0; gg < kG; ++gg)
                if (gg == g) bo = b_of[gg], lo = len_of[gg];
            if (t < lo) {
                const float o0 = s.out[g][2 * cp], o1 = s.out[g][2 * cp + 1];
                const size_t e = ((size_t)bo * p.T + t) * kH + u0 + 2 * cp;
                *reinterpret_cast<float2*>(p.out + e) = make_float2(o0, o1);
                if (p.op.hi != nullptr) store_planes2(p.op, o0, o1, e);
            }
        }
        xr = nxr, xz = nxz, xn = nxn, xres = nres;
        cluster_sync();
    }

    // frames t >= m_b are padding: exactly zero (pad_packed_sequence zero-fills; a residual of zero stays zero)
#pragma unroll
    for (int g = 0; g < kG; ++g) {
        if (b_of[g] < 0) continue;
        const int rows = p.T - len_of[g];
        for (int i = tid; i < rows * (kUnits / 2); i += kThreads) {
            const int t = len_of[g] + i / (kUnits / 2), cp = i % (kUnits / 2);
            const size_t e = ((size_t)b_of[g] * p.T + t) * kH + u0 + 2 * cp;
            *reinterpret_cast<float2*>(p.out + e) = make_float2(0.f, 0.f);
            if (p.op.hi != nullptr) store_planes2(p.op, 0.f, 0.f, e);
        }
    }
}

cudaLaunchConfig_t gru_config(int groups, cudaStream_t s, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kCtas * groups);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = sizeof(GruSmem);
    cfg.stream = s;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kCtas, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

PerDeviceOnce g_gru_attr;

cudaError_t gru_set_attributes() {
    bool& done = g_gru_attr.current();
    if (done) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(gru_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(GruSmem));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(gru_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e == cudaSuccess) done = true;
    return e;
}

// xg[(b, t)][q * 512 + u] += b_hh[q * 512 + u] for the r and z columns (q < 2)
__global__ void gru_fold_bias_kernel(float* xg, const float* bhh, size_t rows) {
    const size_t n = rows * 2 * kH;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / (2 * kH), col = i % (2 * kH);
        xg[r * 3 * kH + col] += bhh[col];
    }
}

}  // namespace

size_t gru_smem_bytes() { return sizeof(GruSmem); }

cudaError_t gru_max_active_clusters(int* n) {
    cudaError_t e = gru_set_attributes();
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = gru_config(1, 0, attr);
    return cudaOccupancyMaxActiveClusters(n, gru_cluster_kernel, &cfg);
}

cudaError_t launch_gru(const GruParams& p, cudaStream_t s) {
    if (p.B <= 0 || p.T <= 0) return cudaSuccess;
    cudaError_t e = gru_set_attributes();
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = gru_config((p.B + kG - 1) / kG, s, attr);
    return cudaLaunchKernelEx(&cfg, gru_cluster_kernel, p);
}

cudaError_t launch_gru_fold_bias(float* xg, const float* bhh, size_t rows, cudaStream_t s) {
    if (rows == 0) return cudaSuccess;
    gru_fold_bias_kernel<<<132 * 4, 256, 0, s>>>(xg, bhh, rows);
    return cudaGetLastError();
}

}  // namespace s3b
