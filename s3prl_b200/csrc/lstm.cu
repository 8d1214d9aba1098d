// LSTM recurrence of DeCoAR (s3prl/upstream/decoar/decoar.py, decoar_layers/decoar.py): one nn.LSTM(1024, 1024)
// layer and direction per launch over packed (ragged) sequences, h_0 = c_0 = 0, PyTorch's gate order i, f, g, o:
//   i = sigmoid(xg_i + W_hi h),  f = sigmoid(xg_f + W_hf h),  g = tanh(xg_g + W_hg h),  o = sigmoid(xg_o + W_ho h),
//   c' = f * c + i * g,  h' = o * tanh(c')
// where xg = W_ih x + b_ih + b_hh comes from one GEMM over all frames. The backward direction runs utterance b from
// frame m_b - 1 down to 0 in natural time (the reference's flipBatch before and after its LSTM).
//
// W_hh is 4096 x 1024 fp32 (16 MiB): too large for one thread-block cluster, so the recurrence is grid-resident.
// kLstmCtas = 128 CTAs, one per SM, are launched cooperatively (the driver makes all of them co-resident or refuses
// the launch). CTA c owns hidden units [8c, 8c + 8) and keeps their 32 rows of W_hh (4 gates x 8 units) in shared
// memory, 128 KiB; its cell states never leave shared memory. h_{t-1} of every utterance lives in a global double
// buffer [2][B][1024], indexed by the utterance's slot in the length order. Every step each CTA stages the state of
// a group of kLstmGroup utterances from L2 into shared memory, computes its 32 x 16 dot products, applies the cell
// and writes its 8 units of h_t. A grid barrier (one
// arrival counter per launch: release-add, acquire-spin) closes the step. Groups are length-sorted, longest first, so
// a step loops over the prefix of groups that still have a live utterance; one weight load serves the whole batch.
//
// Arithmetic: plain fp32 FMAs. Lane l of a warp accumulates k = 128 i + 4 l .. + 3 (i = 0..7) in a fixed order, and a
// butterfly over the 32 lanes completes each dot product. The tree depends neither on the utterance's slot in its
// group nor on the group, so an utterance's outputs are bit-identical in any batch.
#include <math.h>

#include "common.cuh"
#include "kernels.cuh"

namespace s3b {

namespace {

constexpr int kH = kLstmHidden;        // 1024
constexpr int kG = kLstmGroup;         // utterances per group
constexpr int kCtas = kLstmCtas;       // CTAs of the grid
constexpr int kUnits = kH / kCtas;     // 8 hidden units per CTA
constexpr int kRows = 4 * kUnits;      // 32 W_hh rows per CTA
constexpr int kThreads = 256;          // 8 warps: warp w runs units 2 (w & 3) .. + 1 for slots 8 (w >> 2) .. + 7
constexpr int kWarpUnits = 2;
constexpr int kWarpSlots = 8;
constexpr int kVals = 4 * kWarpUnits * kWarpSlots;  // dot products per warp and group-step: 64
constexpr int kMaxB = kLstmMaxBatch;   // utterances per launch (cell states resident in shared memory)
static_assert(kUnits == 8 && kThreads / 32 == (kUnits / kWarpUnits) * (kG / kWarpSlots), "warp tiling");

struct LstmSmem {
    float w[kRows][kH];          // row 4 j + q = W_hh[q * 1024 + 8 c + j]
    float h[kG][kH];             // h_{t-1} of the group being computed
    float hnew[kG][kUnits];      // this CTA's h_t of that group
    float cell[kMaxB][kUnits];   // cell states of this CTA's units, by slot of the length-sorted order
    int b_of[kMaxB], len_of[kMaxB];
};
// one CTA per SM with the opt-in maximum of dynamic shared memory (227 KB on sm_90)
static_assert(sizeof(LstmSmem) <= 227 * 1024, "the LSTM recurrence kernel's shared memory exceeds 227 KB");

__device__ __forceinline__ void grid_arrive(unsigned int* counter) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
}
__device__ __forceinline__ unsigned int grid_poll(const unsigned int* counter) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    return v;
}

// grid: kCtas (cooperative); block kThreads; dynamic smem sizeof(LstmSmem)
__global__ void __launch_bounds__(kThreads, 1) lstm_grid_kernel(LstmParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    LstmSmem& s = *reinterpret_cast<LstmSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c = blockIdx.x;
    const int u0 = c * kUnits;
    const int groups = (p.B + kG - 1) / kG;

    // resident W_hh slice, the batch in length order, c_0 = 0
    for (int i = tid; i < kRows * (kH / 4); i += kThreads) {
        const int r = i / (kH / 4), k4 = i % (kH / 4);
        const int j = r / 4, q = r % 4;
        reinterpret_cast<float4*>(&s.w[r][0])[k4] =
            reinterpret_cast<const float4*>(p.whh + ((size_t)q * kH + u0 + j) * kH)[k4];
    }
    int steps = 0;
    for (int i = tid; i < groups * kG; i += kThreads) {
        const int b = i < p.B ? p.order[i] : -1;
        s.b_of[i] = b;
        s.len_of[i] = b >= 0 ? p.len[b] : 0;
    }
    for (int i = tid; i < groups * kG * kUnits; i += kThreads) (&s.cell[0][0])[i] = 0.f;
    __syncthreads();
    if (p.B > 0) steps = s.len_of[0];

    // this lane's share after the butterfly: values 2 lane, 2 lane + 1 = gates (2 (lane & 1), + 1) of unit ju, slot
    // sl; the even lane of each pair gathers all four gates and runs the cell
    const int sl = lane >> 2, ju = (lane >> 1) & 1;
    const int j = kWarpUnits * (warp & 3) + ju;          // unit within the CTA
    const int slot = kWarpSlots * (warp >> 2) + sl;      // slot within the group
    const int unit = u0 + j;
    const bool cell_lane = (lane & 1) == 0;
    const int wrow = 4 * kWarpUnits * (warp & 3);        // first of the warp's 8 W_hh rows
    const int hslot = kWarpSlots * (warp >> 2);          // first of the warp's 8 slots

    for (int t = 0; t < steps; ++t) {
        const float* hprev = p.hbuf + (size_t)((t + 1) & 1) * p.B * kH;
        float* hnext = p.hbuf + (size_t)(t & 1) * p.B * kH;
        for (int gi = 0; gi < groups && s.len_of[gi * kG] > t; ++gi) {
            // this lane's gate inputs (issued before the dot products so that their latency hides behind them)
            const int bq = s.b_of[gi * kG + slot], lq = s.len_of[gi * kG + slot];
            const bool live = bq >= 0 && t < lq;
            const int tau = p.direction ? lq - 1 - t : t;
            float x4[4] = {0.f, 0.f, 0.f, 0.f};
            if (cell_lane && live) {
                const float* xr = p.xg + ((size_t)bq * p.T + tau) * 4 * kH + unit;
#pragma unroll
                for (int q = 0; q < 4; ++q) x4[q] = xr[q * kH];
                if (p.bhh != nullptr)
#pragma unroll
                    for (int q = 0; q < 4; ++q) x4[q] += p.bhh[q * kH + unit];
            }

            float acc[kVals];
#pragma unroll
            for (int v = 0; v < kVals; ++v) acc[v] = 0.f;
            __syncthreads();  // the previous group's readers of s.h and s.hnew are done
            if (t > 0) {  // h_0 = 0: the first step's products are exactly zero
                for (int i = tid; i < kG * (kH / 4); i += kThreads) {
                    const int g = i / (kH / 4), k4 = i % (kH / 4);
                    const int i_ = gi * kG + g;
                    const float4 v = s.b_of[i_] >= 0 ? __ldcg(reinterpret_cast<const float4*>(hprev + (size_t)i_ * kH) + k4)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
                    reinterpret_cast<float4*>(&s.h[g][0])[k4] = v;
                }
                __syncthreads();
#pragma unroll 2
                for (int i = 0; i < kH / 128; ++i) {
                    const int k = 128 * i + 4 * lane;
                    float4 hv[kWarpSlots];
#pragma unroll
                    for (int g = 0; g < kWarpSlots; ++g) hv[g] = *reinterpret_cast<const float4*>(&s.h[hslot + g][k]);
#pragma unroll
                    for (int r = 0; r < 4 * kWarpUnits; ++r) {
                        const float4 wv = *reinterpret_cast<const float4*>(&s.w[wrow + r][k]);
#pragma unroll
                        for (int g = 0; g < kWarpSlots; ++g) {
                            float& a = acc[g * 4 * kWarpUnits + r];  // value index: slot, unit, gate
                            a = fmaf(wv.x, hv[g].x, a);
                            a = fmaf(wv.y, hv[g].y, a);
                            a = fmaf(wv.z, hv[g].z, a);
                            a = fmaf(wv.w, hv[g].w, a);
                        }
                    }
                }
            }
            // butterfly reduce-scatter 64 -> 2: lane l keeps values 2 l and 2 l + 1
            halve<16, 32>(acc, lane);
            halve<8, 16>(acc, lane);
            halve<4, 8>(acc, lane);
            halve<2, 4>(acc, lane);
            halve<1, 2>(acc, lane);
            const float o0 = __shfl_xor_sync(0xffffffffu, acc[0], 1);
            const float o1 = __shfl_xor_sync(0xffffffffu, acc[1], 1);
            if (cell_lane) {
                // even lane: gates i, f in acc[0..1]; its odd partner held g, o
                const float gi_ = sigmoid_f(x4[0] + acc[0]);
                const float gf = sigmoid_f(x4[1] + acc[1]);
                const float gg = tanhf(x4[2] + o0);
                const float go = sigmoid_f(x4[3] + o1);
                float& cs = s.cell[gi * kG + slot][j];
                const float cn = gf * cs + gi_ * gg;
                const float hn = go * tanhf(cn);
                if (live) cs = cn;
                s.hnew[slot][j] = hn;
            }
            __syncthreads();
            // h_t into the exchange buffer (two float4 per utterance) and the layer output (two columns per thread)
            if (tid < kG * 2) {
                const int g = tid >> 1, half = tid & 1;
                const int i_ = gi * kG + g;
                if (s.b_of[i_] >= 0 && t < s.len_of[i_])
                    __stcg(reinterpret_cast<float4*>(hnext + (size_t)i_ * kH + u0) + half,
                           reinterpret_cast<const float4*>(&s.hnew[g][0])[half]);
            } else if (tid >= 64 && tid < 64 + kG * (kUnits / 2)) {
                const int g = (tid - 64) / (kUnits / 2), cp = (tid - 64) % (kUnits / 2);
                const int b = s.b_of[gi * kG + g], lo = s.len_of[gi * kG + g];
                if (b >= 0 && t < lo) {
                    const int tt = p.direction ? lo - 1 - t : t;
                    const float y0 = s.hnew[g][2 * cp], y1 = s.hnew[g][2 * cp + 1];
                    const size_t e = ((size_t)b * p.T + tt) * p.ldo + p.col0 + u0 + 2 * cp;
                    if (p.out != nullptr) *reinterpret_cast<float2*>(p.out + e) = make_float2(y0, y1);
                    if (p.op.hi != nullptr) store_planes2(p.op, y0, y1, e);
                }
            }
        }
        // grid barrier: every CTA's h_t is in L2 before any CTA stages it
        __syncthreads();
        if (tid == 0) {
            const unsigned int target = (unsigned int)(t + 1) * gridDim.x;
            __threadfence();
            grid_arrive(p.counter);
            while (grid_poll(p.counter) < target) {
            }
            __threadfence();
        }
        __syncthreads();
    }

    // frames t >= m_b are padding: exactly zero (pad_packed_sequence zero-fills)
    for (int i = 0; i < p.B; ++i) {
        const int b = s.b_of[i], lo = s.len_of[i];
        for (int r = tid; r < (p.T - lo) * (kUnits / 2); r += kThreads) {
            const int tt = lo + r / (kUnits / 2), cp = r % (kUnits / 2);
            const size_t e = ((size_t)b * p.T + tt) * p.ldo + p.col0 + u0 + 2 * cp;
            if (p.out != nullptr) *reinterpret_cast<float2*>(p.out + e) = make_float2(0.f, 0.f);
            if (p.op.hi != nullptr) store_planes2(p.op, 0.f, 0.f, e);
        }
    }
}

PerDeviceOnce g_lstm_attr;

cudaError_t lstm_set_attributes() {
    bool& done = g_lstm_attr.current();
    if (done) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(lstm_grid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(LstmSmem));
    if (e == cudaSuccess) done = true;
    return e;
}

}  // namespace

size_t lstm_smem_bytes() { return sizeof(LstmSmem); }

cudaError_t lstm_fits(int* ok, int* sms, int* smem_optin) {
    *ok = 0;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    int coop = 0;
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    if (e != cudaSuccess) return e;
    if (*sms < kCtas || (size_t)*smem_optin < sizeof(LstmSmem) || !coop) return cudaSuccess;
    e = lstm_set_attributes();
    if (e != cudaSuccess) return e;
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lstm_grid_kernel, kThreads, sizeof(LstmSmem));
    if (e != cudaSuccess) return e;
    *ok = per_sm * *sms >= kCtas ? 1 : 0;
    return cudaSuccess;
}

size_t lstm_hbuf_floats(int B) { return (size_t)2 * (B < kMaxB ? B : kMaxB) * kH; }

cudaError_t launch_lstm(const LstmParams& p, cudaStream_t s) {
    if (p.B <= 0 || p.T <= 0) return cudaSuccess;
    cudaError_t e = lstm_set_attributes();
    if (e != cudaSuccess) return e;
    // batches beyond kMaxB utterances run as consecutive launches of at most kMaxB (the longest first)
    for (int b0 = 0; b0 < p.B; b0 += kMaxB) {
        LstmParams q = p;
        q.order = p.order + b0;
        q.B = p.B - b0 < kMaxB ? p.B - b0 : kMaxB;
        e = cudaMemsetAsync(q.counter, 0, sizeof(unsigned int), s);
        if (e != cudaSuccess) return e;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(kCtas);
        cfg.blockDim = dim3(kThreads);
        cfg.dynamicSmemBytes = sizeof(LstmSmem);
        cfg.stream = s;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeCooperative;
        attr[0].val.cooperative = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        e = cudaLaunchKernelEx(&cfg, lstm_grid_kernel, q);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace s3b
