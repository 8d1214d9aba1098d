// Flash-style self-attention on Hopper warpgroup MMAs (wgmma) with error-compensated bf16 operands.
// Replaces F.multi_head_attention_forward -> SDPA with key_padding_mask
// (s3prl/upstream/wav2vec2/wav2vec2_model.py:1146-1168) and, when bias_table is given, WavLM's gated
// relative-position bias (s3prl/upstream/wavlm/modules.py:511-580).
//
// One CTA = one (batch, head, 128-query tile), 288 threads:
//   warps 0..3, 4..7 : two softmax / MMA warpgroups, 64 query rows each; S, P and O live in registers
//   warp 8           : TMA producer (Q once, then K / V^T blocks of 64 keys into a two-stage ring)
// Per 64-key block j and warpgroup:
//   S_j = Qhi*Khi^T + Qhi*Klo^T + Qlo*Khi^T     wgmma m64n64k16 from shared memory, 3 * ceil(HD / 16) instructions
//   scores (log2 domain: q was scaled by HD^-0.5 * log2(e)) -> running max m, p = 2^(s-m); O rescaled by alpha
//   O += Phi*Vhi + Phi*Vlo + Plo*Vhi            wgmma m64nHDk16 with A = P from registers (the S accumulator layout is
//                                               the A-fragment layout, so P never touches shared memory)
// Head width HD in {64, 80, 120}. Q and K rows are loaded as ceil(HD / 64) boxes of 64 elements (128-byte swizzle
// rows); the columns of the last box past HD are TMA out-of-bounds fill (zero), so the padded k-steps add nothing.
//   HD = 64      : two CTAs per SM (~97 KB shared memory each)
//   HD = 80, 120 : one CTA per SM (~169 / ~189 KB: the Q and K boxes double)
#include <math.h>

#include "common.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

namespace s3b {

static constexpr int kQTile = 128;
static constexpr int kKBlk = 64;
static constexpr int kQBytes = kQTile * 64 * 2;  // 16 KB per 64-wide box of a plane
static constexpr int kKBytes = kKBlk * 64 * 2;   // 8 KB per 64-wide box of a plane
static constexpr int kStages = 2;
static constexpr int kAttnThreads = 288;

// smem map (1024-aligned): Qhi[box] Qlo[box] | 2 x {Khi[box] Klo[box] Vhi Vlo} | barriers
template <int HD>
struct AttnCfg {
    static constexpr int kBoxes = (HD + 63) / 64;  // 64-wide boxes of a Q / K row
    static constexpr int kVBytes = HD * kKBlk * 2;  // V^T block: HD rows of 64 keys
    static constexpr int kOffQ = 0;
    static constexpr int kOffKV = 2 * kBoxes * kQBytes;
    static constexpr int kStage = 2 * kBoxes * kKBytes + 2 * kVBytes;
    static constexpr int kOffBar = kOffKV + kStages * kStage;
    static constexpr int kSmem = kOffBar + 128 + 1024;
    static constexpr int kMinBlocks = HD == 64 ? 2 : 1;
    static_assert(HD % 8 == 0 && HD <= 128 && kVBytes % 1024 == 0, "head width");
};

template <int HD, bool kBias>
__global__ void __launch_bounds__(kAttnThreads, AttnCfg<HD>::kMinBlocks)
    attention_kernel(const __grid_constant__ AttnParams p) {
    using Cfg = AttnCfg<HD>;
    constexpr int kBoxes = Cfg::kBoxes, kOffQ = Cfg::kOffQ, kOffKV = Cfg::kOffKV, kStage = Cfg::kStage;
    constexpr int kOffV = 2 * kBoxes * kKBytes;  // V^T planes within a stage
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bar_q = reinterpret_cast<uint64_t*>(smem + Cfg::kOffBar);
    uint64_t* full_bar = bar_q + 1;             // [kStages] K_j / V_j landed
    uint64_t* empty_bar = full_bar + kStages;   // [kStages] both warpgroups are done with the stage

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int q_tiles = (p.T + kQTile - 1) / kQTile;
    const int item = blockIdx.x;
    const int bh = item / q_tiles;
    const int q0 = (item - bh * q_tiles) * kQTile;
    const int b = bh / p.H;
    const int h = bh - b * p.H;

    if (warp == 8 && elect_one()) {
        tma_prefetch_desc(&p.q_hi);
        tma_prefetch_desc(&p.k_hi);
        tma_prefetch_desc(&p.vt_hi);
        mbar_init(bar_q, 1);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);  // one arrive per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();  // prologue overlapped the QKV GEMM's tail; global memory is touched only below
    pdl_launch_dependents();

    const int kv_len = p.kv_len[b];
    const int nblk = (kv_len + kKBlk - 1) / kKBlk;

    if (warp == 8) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            mbar_arrive_expect_tx(bar_q, 2 * kBoxes * kQBytes);
#pragma unroll
            for (int x = 0; x < kBoxes; ++x) {
                tma_load_3d(smem + kOffQ + x * kQBytes, &p.q_hi, bar_q, 64 * x, q0, bh);
                tma_load_3d(smem + kOffQ + (kBoxes + x) * kQBytes, &p.q_lo, bar_q, 64 * x, q0, bh);
            }
            for (int j = 0; j < nblk; ++j) {
                const int s = j % kStages;
                const int use = j / kStages;
                if (use > 0) mbar_wait(&empty_bar[s], (uint32_t)((use - 1) & 1));
                uint8_t* st = smem + kOffKV + s * kStage;
                mbar_arrive_expect_tx(&full_bar[s], kStage);
#pragma unroll
                for (int x = 0; x < kBoxes; ++x) {
                    tma_load_3d(st + x * kKBytes, &p.k_hi, &full_bar[s], 64 * x, j * kKBlk, bh);
                    tma_load_3d(st + (kBoxes + x) * kKBytes, &p.k_lo, &full_bar[s], 64 * x, j * kKBlk, bh);
                }
                tma_load_3d(st + kOffV, &p.vt_hi, &full_bar[s], j * kKBlk, 0, bh);
                tma_load_3d(st + kOffV + Cfg::kVBytes, &p.vt_lo, &full_bar[s], j * kKBlk, 0, bh);
            }
        }
        return;
    }

    // ===================== softmax / MMA warpgroups =====================
    // accumulator layout (m64nN): this thread holds rows r and r + 8, columns 8c + 2(lane%4) + {0,1}, c < N / 8,
    // in registers [4c + 2i + e] (i: row r / r + 8, e: column parity)
    const int wg = warp >> 2;
    const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cpair = 2 * (lane & 3);
    int q_row[2];
    bool row_ok[2];
    float gate[2] = {0.f, 0.f};
    const float* brow[2] = {nullptr, nullptr};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        q_row[i] = q0 + r_base + 8 * i;
        row_ok[i] = q_row[i] < p.T;
        if (kBias) {
            gate[i] = (p.gate == nullptr) ? 1.0f : (row_ok[i] ? p.gate[((size_t)b * p.H + h) * p.T + q_row[i]] : 0.f);
            brow[i] = p.bias_table + (size_t)h * p.bias_stride + (p.bias_center - (row_ok[i] ? q_row[i] : 0));  // by key
        }
    }
    const uint32_t qa = smem_u32(smem + kOffQ) + (uint32_t)(wg * 64 * 128);
    const uint64_t dq_hi = make_wgmma_desc<128>(qa), dq_lo = make_wgmma_desc<128>(qa + kBoxes * kQBytes);

    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};  // running row max (log2 domain)
    float l_run[2] = {0.f, 0.f};              // this thread's share of the row sum

    mbar_wait(bar_q, 0);
    for (int j = 0; j < nblk; ++j) {
        const int s = j % kStages;
        mbar_wait(&full_bar[s], (uint32_t)((j / kStages) & 1));
        const uint32_t st = smem_u32(smem + kOffKV + s * kStage);
        const uint64_t dk_hi = make_wgmma_desc<128>(st), dk_lo = make_wgmma_desc<128>(st + kBoxes * kKBytes);
        const uint64_t dv_hi = make_wgmma_desc<128>(st + kOffV), dv_lo = make_wgmma_desc<128>(st + kOffV + Cfg::kVBytes);

        float sc[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < (HD + 15) / 16; ++k) {
            // 16-wide k-step k: box k / 4 (descriptor address unit = 16 bytes), + 32 bytes per step inside the
            // 128-byte swizzle row
            const uint64_t ko = (uint64_t)(2 * (k % 4)), box = (uint64_t)(k / 4);
            const uint64_t dq_hi_k = dq_hi + box * (kQBytes >> 4), dq_lo_k = dq_lo + box * (kQBytes >> 4);
            const uint64_t dk_hi_k = dk_hi + box * (kKBytes >> 4), dk_lo_k = dk_lo + box * (kKBytes >> 4);
            Wgmma<64, 0>::ss(sc, dq_lo_k + ko, dk_hi_k + ko, k != 0 ? 1u : 0u);
            Wgmma<64, 0>::ss(sc, dq_hi_k + ko, dk_lo_k + ko, 1u);
            Wgmma<64, 0>::ss(sc, dq_hi_k + ko, dk_hi_k + ko, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();

        const int kbase = j * kKBlk + cpair;
        if (kBias) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int kk = kbase + 8 * c + e;
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        sc[4 * c + 2 * i + e] = fmaf(gate[i], (kk < p.T) ? __ldg(brow[i] + kk) : 0.f, sc[4 * c + 2 * i + e]);
                }
            }
        }
        if (j * kKBlk + kKBlk > kv_len) {  // block-uniform: only the last block is partially masked
#pragma unroll
            for (int c = 0; c < 8; ++c)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (kbase + 8 * c + e >= kv_len) sc[4 * c + e] = -INFINITY, sc[4 * c + 2 + e] = -INFINITY;
        }
        float alpha[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float mx = -INFINITY;
#pragma unroll
            for (int c = 0; c < 8; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * i], sc[4 * c + 2 * i + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[i], mx);  // finite: key j*64 is always valid
            alpha[i] = fast_exp2(m_run[i] - m_new);
            m_run[i] = m_new;
        }
        // P as the A fragments of the four 16-key k-steps: register q of step k = keys of column block 2k + q/2,
        // row r + 8 (q & 1)
        uint32_t phi[4][4], plo[4][4];
        float psum[2] = {0.f, 0.f};
#pragma unroll
        for (int c = 0; c < 8; ++c) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float p0 = fast_exp2(sc[4 * c + 2 * i] - m_run[i]);
                const float p1 = fast_exp2(sc[4 * c + 2 * i + 1] - m_run[i]);
                psum[i] += p0 + p1;
                split_pack2(p0, p1, phi[c >> 1][2 * (c & 1) + i], plo[c >> 1][2 * (c & 1) + i]);
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) l_run[i] = fmaf(l_run[i], alpha[i], psum[i]);
#pragma unroll
        for (int c = 0; c < HD / 8; ++c)
#pragma unroll
            for (int i = 0; i < 2; ++i) o[4 * c + 2 * i] *= alpha[i], o[4 * c + 2 * i + 1] *= alpha[i];

        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kKBlk / 16; ++k) {
            const uint64_t ko = (uint64_t)(2 * k);
            WgmmaRs<HD>::bf16(o, plo[k], dv_hi + ko, 1u);
            WgmmaRs<HD>::bf16(o, phi[k], dv_lo + ko, 1u);
            WgmmaRs<HD>::bf16(o, phi[k], dv_hi + ko, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);  // the producer may overwrite this K / V stage
    }

#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float l = l_run[i];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        if (!row_ok[i]) continue;
        const float inv = 1.0f / l;
        const size_t off = ((size_t)b * p.T + q_row[i]) * (size_t)p.D + (size_t)h * HD + cpair;
#pragma unroll
        for (int c = 0; c < HD / 8; ++c) store_planes2(p.ctx, o[4 * c + 2 * i] * inv, o[4 * c + 2 * i + 1] * inv, off + 8 * c);
    }
}

template <int HD, bool kBias>
static cudaError_t launch_width(const AttnParams& p, int n_items, cudaStream_t s) {
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.current();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(attention_kernel<HD, kBias>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             AttnCfg<HD>::kSmem);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    return launch_pdl(attention_kernel<HD, kBias>, dim3(n_items), dim3(kAttnThreads), AttnCfg<HD>::kSmem, s, p);
}

cudaError_t launch_attention(const AttnParams& p, cudaStream_t s) {
    const int q_tiles = (p.T + kQTile - 1) / kQTile;
    const int n_items = p.B * p.H * q_tiles;
    if (n_items <= 0) return cudaSuccess;
    switch (p.hd) {
        case 64:
            if (p.bias_table != nullptr) return launch_width<64, true>(p, n_items, s);
            return launch_width<64, false>(p, n_items, s);
        // the WavLM bias (relative table, gate) is 64-wide only
        case 80: return p.bias_table != nullptr ? cudaErrorInvalidValue : launch_width<80, false>(p, n_items, s);
        case 120: return p.bias_table != nullptr ? cudaErrorInvalidValue : launch_width<120, false>(p, n_items, s);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace s3b
