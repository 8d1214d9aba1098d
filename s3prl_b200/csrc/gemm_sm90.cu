// Persistent, warp-specialised Hopper (sm_90a) GEMM with error-compensated operands:
//   D[m][n] = sum_k A[m][k] * W[n][k],  fp32 accumulation in registers (wgmma)
//   scheme 0 (bf16x3): A = A_hi + A_lo, W = W_hi + W_lo (bf16),   D += A_hi*W_hi + A_hi*W_lo + A_lo*W_hi
//   scheme 1 (f16q8) : fp16 main product + two e4m3 correction products (common.cuh), the corrections first
//
// Replaces the reference's fp32 torch ops (cited per call site in model.cu):
//   nn.Conv1d(512,512,k,2) blocks      s3prl/upstream/wav2vec2/wav2vec2_model.py:2879,2927-2934
//   post_extract_proj                  s3prl/upstream/hubert/hubert_model.py:489-490
//   pos_conv (grouped Conv1d k=128)    s3prl/upstream/wav2vec2/wav2vec2_model.py:2937-2953,3064-3067
//   q/k/v/out projections, fc1, fc2    s3prl/upstream/wav2vec2/wav2vec2_model.py:1146-1168,3260-3322
//
// One CTA per SM, persistent over 128 x BN output tiles, one TMA producer warp filling a swizzled shared-memory ring of
// kStages stages in tile order. Two kernels consume it:
//   cooperative (every width but 128), 288 threads: warps 0..3 and 4..7 are two consumer warpgroups that share each
//     tile, 64 rows each (wgmma m64nBN); warp 8 is the producer. ptxas gives these kernels at most 168 registers a
//     thread, which holds the 128 accumulators of a 256-wide tile.
//   ping-pong (128-wide tiles), 384 threads: warpgroups 0 and 1 take alternate tiles, each a whole 128 x 128 tile
//     (two m64n128 wgmmas per k-step, 128 accumulators); warp 8 of warpgroup 2 is the producer. One warpgroup's
//     epilogue then overlaps the other's MMAs. setmaxnreg moves registers from the producer warpgroup to the consumers.
//     It may run in clusters of CN = 2 or 4 CTAs along N that load each A box once between them (TMA multicast).
// Both run the same k order and f16q8 pass order per output element, so the two widths agree bit for bit.
#include <stdio.h>

#include "common.cuh"
#include "gemm.cuh"
#include "wgmma.cuh"

namespace s3b {

static constexpr int kBlockM = 128;
static constexpr int kBlockK = 64;  // K elements per k-block, every scheme and width
static constexpr int kThreads = 288;
static constexpr int kPingPongThreads = 384;
static constexpr int kSmemBudget = 220 * 1024;

// A stage holds 64 elements of K of A (128 rows) and W (BN rows) in rows of 128 bytes with the 128-byte swizzle.
// bf16x3: four planes [A_hi A_lo W_hi W_lo] of 64 bf16 elements per row. f16q8: one A box and one W box per stage,
// pass 0 of interleaved e4m3 rows [l8 k0..31 | h8 k0..31 | l8 k32..63 | h8 k32..63] (common.cuh: q8_off), pass 1 of
// fp16 rows [A16 | W16]. f16q8 stages are 48 KB at BN = 256, which makes the ring four deep there (six at BN = 128).
template <int BN, int kScheme>
struct GemmCfg {
    static constexpr int RB = 128;                        // bytes of one box row = the swizzle span
    static constexpr int kAPlane = kBlockM * RB;          // one A box
    static constexpr int kBPlane = BN * RB;               // one W box
    static constexpr int kBoxes = kScheme == 0 ? 2 : 1;   // boxes of A and of W per stage
    static constexpr int kStageBytes = kBoxes * (kAPlane + kBPlane);
    static constexpr int kStages = (kSmemBudget - 2048) / kStageBytes > 6 ? 6 : (kSmemBudget - 2048) / kStageBytes;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(kStages >= 2, "tile too large for the shared-memory ring");
};

// Epilogue kinds, one kernel instantiation each (chosen per launch in launch_gemm). Every non-QKV kind computes
//   v = acc (+bias) ; GELU, SiLU, ReLU or tanh? ; out_pre = v? ; (+residual) ; row_mask ? 0
// or, with res_first, v = acc (+bias) (+residual) ; activation ; row_mask ? 0
// and stores v as fp32, as operand planes, or both.
enum EpiKind { kEpiF32 = 1, kEpiPlanes = 2, kEpiBoth = 3, kEpiQkv = 4 };

__device__ __forceinline__ void setmaxnreg_dec40() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void setmaxnreg_inc232() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

// ===================== the persistent tile walk ======================================================================
// CTAs walk cluster tiles: CN adjacent column tiles of one 128-row tile, one per CTA of a cluster of CN CTAs along x
// (cluster c = blockIdx.x / CN, rank = blockIdx.x % CN). Every CTA of a cluster therefore runs the same number of
// tiles with the same K, in lockstep. CN = 1 is the plain walk over tiles, CTA blockIdx.x taking tiles blockIdx.x,
// blockIdx.x + gridDim.x, ...
struct TileCoord {
    int n_tile, batch, row0;
};
template <int CN>
__device__ __forceinline__ TileCoord tile_coord(const GemmParams& p, int ctile, int rank) {
    const int groups = p.n_tiles / CN;
    const int mt = ctile / groups;
    TileCoord c;
    c.n_tile = (ctile - mt * groups) * CN + rank;
    c.batch = mt / p.tiles_m_per_batch;
    c.row0 = (mt - c.batch * p.tiles_m_per_batch) * kBlockM;
    return c;
}

// One A box of a stage. CN > 1: this CTA loads rows [rank * 128 / CN, (rank + 1) * 128 / CN) of the box (the tensor
// map's box height) into that slice of the plane, in every CTA of the cluster; its peers load the other slices.
template <int CN, int RB>
__device__ __forceinline__ void load_a(uint8_t* plane, const CUtensorMap* m, uint64_t* bar, int a_k, int a_row,
                                       int batch, int rank) {
    if constexpr (CN == 1) {
        tma_load_3d(plane, m, bar, a_k, a_row, batch);
    } else {
        constexpr int kRows = kBlockM / CN;
        tma_load_3d_multicast(plane + rank * kRows * RB, m, bar, a_k, a_row + rank * kRows, batch,
                              (uint16_t)((1u << CN) - 1u));
    }
}

// ===================== TMA producer: every tile of this CTA, kPasses * num_k_blocks stages each, in tile order ====
// With CN > 1 a stage is refilled only once every CTA of the cluster has released it (empty_bar counts the consumer
// warps of all of them): this CTA's A slice lands in the peers' stage too. Each full_bar still expects the whole stage,
// its own W box plus the CN A slices.
template <int BN, int kScheme, int CN>
__device__ __forceinline__ void produce(const GemmParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar) {
    using Cfg = GemmCfg<BN, kScheme>;
    constexpr int kPasses = kScheme == 0 ? 1 : 2;
    const int rank = CN == 1 ? 0 : (int)cluster_rank();
    const int num_ctiles = p.batches * p.tiles_m_per_batch * (p.n_tiles / CN);
    int stage = 0;
    uint32_t phase = 0;
    for (int ct = blockIdx.x / CN; ct < num_ctiles; ct += gridDim.x / CN) {
        const TileCoord tc = tile_coord<CN>(p, ct, rank);
        const int n_tile = tc.n_tile, batch = tc.batch, row0 = tc.row0;
        const int a_k0 = p.a_k_per_ntile * n_tile;
        const int b_n0 = n_tile * BN;
        for (int pass = 0; pass < kPasses; ++pass) {
            for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                const int kq = kb / p.kb_per_row;
                const int kr = kb - kq * p.kb_per_row;
                mbar_wait(&empty_bar[stage], phase ^ 1u);
                uint8_t* st = smem + stage * Cfg::kStageBytes;
                uint8_t* sb = st + Cfg::kBoxes * Cfg::kAPlane;
                mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)Cfg::kStageBytes);
                const int a_row = row0 + kq * p.a_row_step + p.a_row_off + (kq >= p.a_gap_at ? p.a_gap : 0);
                const int a_k = a_k0 + kr * kBlockK;
                const int b_k = kb * kBlockK;
                if constexpr (kScheme == 1) {
                    // one A box and one W box of 128-byte rows: pass 0 the q8 planes (2 bytes per element of K, so
                    // at twice the fp16 column), pass 1 the fp16 planes
                    const CUtensorMap* ma = pass == 0 ? &p.a_q8 : &p.a_hi;
                    const CUtensorMap* mb = pass == 0 ? &p.b_q8 : &p.b_hi;
                    const int q = pass == 0 ? 2 : 1;
                    load_a<CN, Cfg::RB>(st, ma, &full_bar[stage], q * a_k, a_row, batch, rank);
                    tma_load_3d(sb, mb, &full_bar[stage], q * b_k, b_n0, 0);
                } else {
                    load_a<CN, Cfg::RB>(st, &p.a_hi, &full_bar[stage], a_k, a_row, batch, rank);
                    load_a<CN, Cfg::RB>(st + Cfg::kAPlane, &p.a_lo, &full_bar[stage], a_k, a_row, batch, rank);
                    tma_load_3d(sb, &p.b_hi, &full_bar[stage], b_k, b_n0, 0);
                    tma_load_3d(sb + Cfg::kBPlane, &p.b_lo, &full_bar[stage], b_k, b_n0, 0);
                }
                if (++stage == Cfg::kStages) stage = 0, phase ^= 1u;
            }
        }
    }
    // CN > 1: the peers' consumers arrive on this CTA's empty barriers until they have consumed their last stage. The
    // producer waits for every stage's last release, so that this CTA outlives those remote arrives. (Every peer
    // multicast into this CTA has landed before its own consumers finish: they wait for whole stages.) A cluster
    // barrier before exit would do the same, but it makes ptxas spill the consumers' registers.
    if constexpr (CN > 1) {
        for (int i = 0; i < Cfg::kStages; ++i) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            if (++stage == Cfg::kStages) stage = 0, phase ^= 1u;
        }
    }
}

// Stage release by one consumer warp: CN > 1 arrives on the stage's empty barrier in every CTA of the cluster (lane r
// on CTA r's), as each of them multicasts into this CTA's copy of the stage.
template <int CN>
__device__ __forceinline__ void release_stage(uint64_t* empty_bar, int lane) {
    __syncwarp();
    if constexpr (CN == 1) {
        if (lane == 0) mbar_arrive(empty_bar);
    } else {
        if (lane < CN) mbar_arrive_cluster(peer_addr(empty_bar, (uint32_t)lane));
    }
}

// ===================== MMAs of one tile: kHalves 64-row halves of A starting at half `half0`, acc[h] per half ======
// Stage s is released (one arrive per warp of the warpgroup) once the wgmma group reading it has retired; one group
// stays in flight so that the tensor pipe is fed while this warpgroup waits for the next stage. Every output element
// sees the same wgmma sequence whichever kernel, warpgroup or half runs it.
template <int BN, int kScheme, int kHalves, int CN>
__device__ __forceinline__ void mma_tile(const GemmParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                         int half0, int lane, int& stage, uint32_t& phase,
                                         float (&acc)[kHalves][BN / 2]) {
    using Cfg = GemmCfg<BN, kScheme>;
    constexpr int RB = Cfg::RB;
    constexpr int kStages = Cfg::kStages;
    constexpr int kNR = BN / 2;
    constexpr int kPasses = kScheme == 0 ? 1 : 2;
    const int k_steps = p.k_steps > 0 ? p.k_steps : RB / 32;  // 16-wide k-steps per stage (scheme 0)
#pragma unroll
    for (int h = 0; h < kHalves; ++h)
#pragma unroll
        for (int i = 0; i < kNR; ++i) acc[h][i] = 0.f;

    int pending = -1;
    bool first = true;
    // The pass loop is unrolled so that every wgmma sits in straight-line code: with a runtime pass index the
    // rescale below is a branch ptxas treats as divergent, and it then serialises every wgmma of the kernel.
#pragma unroll
    for (int pass = 0; pass < kPasses; ++pass) {
        if (kScheme == 1 && pass == 1) {
            // the corrections carry 2^kQ8Scale: scale them back before the main product accumulates (exact)
            wgmma_wait<0>();
            if (pending >= 0) {
                release_stage<CN>(&empty_bar[pending], lane);
                pending = -1;
            }
            const float s = 1.0f / (float)(1 << kQ8Scale);
#pragma unroll
            for (int h = 0; h < kHalves; ++h)
#pragma unroll
                for (int i = 0; i < kNR; ++i) acc[h][i] *= s;
            wgmma_fence();
        }
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t st = smem_u32(smem + stage * Cfg::kStageBytes);
            const uint32_t b0 = st + Cfg::kBoxes * Cfg::kAPlane;
            wgmma_fence();
            if constexpr (kScheme == 0) {
                const uint64_t db0 = make_wgmma_desc<RB>(b0), db1 = make_wgmma_desc<RB>(b0 + Cfg::kBPlane);
#pragma unroll
                for (int k = 0; k < RB / 32; ++k) {
                    if (k < k_steps) {
                        // advance 16 bf16 (= 32 bytes) along K inside the swizzle atom: +2 in (addr >> 4) units
                        const uint64_t ko = (uint64_t)(k * 2);
#pragma unroll
                        for (int h = 0; h < kHalves; ++h) {
                            const uint32_t a0 = st + (half0 + h) * 64 * RB, a1 = a0 + Cfg::kAPlane;
                            const uint64_t da0 = make_wgmma_desc<RB>(a0), da1 = make_wgmma_desc<RB>(a1);
                            Wgmma<BN, 0>::ss(acc[h], da1 + ko, db0 + ko, first ? 0u : 1u);
                            Wgmma<BN, 0>::ss(acc[h], da0 + ko, db1 + ko, 1u);
                            Wgmma<BN, 0>::ss(acc[h], da0 + ko, db0 + ko, 1u);
                        }
                        first = false;
                    }
                }
            } else if (pass == 0) {  // (kScheme == 1 from here on: one A and one W box of 128-byte rows)
                // e4m3 MMAs of K = 32 (32 bytes) at byte 32 i of the rows: A chunk i x W chunk i ^ 1 gives
                // A_l8 x W_h8, A_h8 x W_l8 for k 0..31, then the same for k 32..63 (a half's 64 A rows start
                // 64 * 128 bytes apart)
                const uint64_t db = make_wgmma_desc<128>(b0);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
#pragma unroll
                    for (int h = 0; h < kHalves; ++h) {
                        const uint64_t da = make_wgmma_desc<128>(st + (half0 + h) * 64 * 128);
                        Wgmma<BN, 2>::ss(acc[h], da + (uint64_t)(2 * i), db + (uint64_t)(2 * (i ^ 1)),
                                         first ? 0u : 1u);
                    }
                    first = false;
                }
            } else {
                // A16[k..k+64) x W16[k..k+64), K = 16 per MMA
                const uint64_t db = make_wgmma_desc<128>(b0);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint64_t ko = (uint64_t)(k * 2);
#pragma unroll
                    for (int h = 0; h < kHalves; ++h) {
                        const uint64_t da = make_wgmma_desc<128>(st + (half0 + h) * 64 * 128);
                        Wgmma<BN, 1>::ss(acc[h], da + ko, db + ko, 1u);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (pending >= 0) release_stage<CN>(&empty_bar[pending], lane);
            pending = stage;
            if (++stage == kStages) stage = 0, phase ^= 1u;
        }
    }
    wgmma_wait<0>();
    if (pending >= 0) release_stage<CN>(&empty_bar[pending], lane);
}

// two consecutive columns of one operand-plane format (the arithmetic of store_planes2)
template <int kFmt>
__device__ __forceinline__ void store_plane_pair(const GemmParams& p, float x0, float x1, size_t off) {
    if constexpr (kFmt != 0) {
        uint32_t h;
        uint16_t a, b;
        split_q8_pack2(x0, x1, h, a, b);
        uint8_t* q = p.out_q8 + q8_off(off, 0);
        *reinterpret_cast<uint32_t*>(p.out_hi + off) = h;
        *reinterpret_cast<uint16_t*>(q + 32) = a;
        *reinterpret_cast<uint16_t*>(q) = b;
    } else {
        uint32_t h, l;
        split_pack2(x0, x1, h, l);
        *reinterpret_cast<uint32_t*>(p.out_hi + off) = h;
        *reinterpret_cast<uint32_t*>(p.out_lo + off) = l;
    }
}

// ===================== epilogue of one tile, straight from the accumulator registers ===============================
// acc[h] holds rows row_base + 64 h + {0, 8} (register 4j + 2i + {0,1}: row + 8i, columns col0 + 8j + {0,1}).
// Per-row work (flat row, mask, offsets, QKV's b and t) is done once per row, the bias once per chunk of kCh column
// pairs for all rows, and every load of a chunk is issued before any of its stores. Mode tests are uniform branches
// around whole chunks, never per pair.
// the largest divisor of kJ column pairs that is at most 8
constexpr int chunk_pairs(int kJ) {
    for (int c = 8; c > 1; --c)
        if (kJ % c == 0) return c;
    return 1;
}

template <int BN, int kEpi, int kHalves>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, float (&acc)[kHalves][BN / 2], int batch,
                                              int row_base, int col0) {
    constexpr int kJ = BN / 8;               // column pairs per row
    // pairs per chunk: the largest divisor of kJ up to 8 (5 at the pos_conv's 80-, 120- and 160-column tiles, 6 at
    // 96), but 2 next to the 128 accumulators of a 256-wide cooperative tile (168 registers at most)
    constexpr int kCh = BN * kHalves >= 256 && kHalves == 1 ? 2 : chunk_pairs(kJ);
    constexpr int kRows = 2 * kHalves;       // rows per thread
    static_assert(kJ % kCh == 0, "chunking");
    bool ok[kRows];
    size_t m[kRows];
#pragma unroll
    for (int s = 0; s < kRows; ++s) {
        const int row = row_base + 64 * (s >> 1) + 8 * (s & 1);
        ok[s] = row < p.rows_per_batch;
        m[s] = (size_t)batch * p.out_rows_per_batch + row;
    }
    const bool has_bias = p.bias != nullptr;

    if constexpr (kEpi == kEpiQkv) {
        // m = b*T + t ; col = which*D + h*hd + d (column pairs never straddle a head: hd is even)
        //   q, k: [B][H][T][hd] at (b*H*T + t)*hd + h*T*hd + d      v^T: [B][H][hd][Tp] at b*H*hd*Tp + t + (h*hd + d)*Tp
        // q / k column offset h*T*hd + d = within + h*(T-1)*hd, h = within / hd by a multiply-high with p.hd_magic
        // (exact for within < 2^16), once per column pair; (T-1)*hd is the host's p.qk_head_step
        const int T = p.T, D = p.D, hd = p.hd;
        size_t base_qk[kRows], base_v[kRows];
#pragma unroll
        for (int s = 0; s < kRows; ++s) {
            const int b = (int)m[s] / T;
            const int t = (int)m[s] - b * T;
            base_qk[s] = (size_t)(unsigned)(b * p.H * T + t) * (unsigned)hd;  // (b*H*T + t) <= B*T*H < 2^31
            base_v[s] = (size_t)(unsigned)(b * D) * (unsigned)p.Tp + t;
        }
        const int qcol = col0 + p.qkv_col0;
        int which = qcol / D;
        int within = qcol - which * D;
#pragma unroll
        for (int c = 0; c < kJ; c += kCh) {
            float2 bv[kCh];
            if (has_bias) {
#pragma unroll
                for (int jj = 0; jj < kCh; ++jj) bv[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * (c + jj)));
            }
#pragma unroll
            for (int jj = 0; jj < kCh; ++jj) {
                const int j = c + jj;
                const int h = (int)__umulhi((unsigned)within, p.hd_magic);
                if (which < 2) {
                    __nv_bfloat16* dst_hi = which == 0 ? p.q_hi : p.k_hi;
                    __nv_bfloat16* dst_lo = which == 0 ? p.q_lo : p.k_lo;
                    const int o_col = within + h * p.qk_head_step;
#pragma unroll
                    for (int s = 0; s < kRows; ++s) {
                        if (!ok[s]) continue;
                        float x0 = acc[s >> 1][4 * j + 2 * (s & 1)], x1 = acc[s >> 1][4 * j + 2 * (s & 1) + 1];
                        if (has_bias) x0 += bv[jj].x, x1 += bv[jj].y;
                        if (which == 0) x0 *= p.q_scale, x1 *= p.q_scale;
                        uint32_t hi, lo;
                        split_pack2(x0, x1, hi, lo);
                        *reinterpret_cast<uint32_t*>(dst_hi + base_qk[s] + o_col) = hi;
                        *reinterpret_cast<uint32_t*>(dst_lo + base_qk[s] + o_col) = lo;
                    }
                } else {
                    const int o_col = within * p.Tp;
#pragma unroll
                    for (int s = 0; s < kRows; ++s) {
                        if (!ok[s]) continue;
                        float x0 = acc[s >> 1][4 * j + 2 * (s & 1)], x1 = acc[s >> 1][4 * j + 2 * (s & 1) + 1];
                        if (has_bias) x0 += bv[jj].x, x1 += bv[jj].y;
                        __nv_bfloat16 h0, l0, h1, l1;
                        split_bf16(x0, h0, l0);
                        split_bf16(x1, h1, l1);
                        const size_t o = base_v[s] + o_col;
                        p.vt_hi[o] = h0, p.vt_lo[o] = l0;
                        p.vt_hi[o + p.Tp] = h1, p.vt_lo[o + p.Tp] = l1;
                    }
                }
                within += 8;
                if (within >= D) within -= D, ++which;
            }
        }
        return;
    } else {
        const int act = p.gelu;
        const bool has_res = p.residual != nullptr, has_pre = p.out_pre != nullptr;
        const bool res_first = has_res && p.res_first != 0, add_res_after = has_res && p.res_first == 0;
        const int fmt = p.out_fmt;
        size_t off[kRows];
        bool zero[kRows];
#pragma unroll
        for (int s = 0; s < kRows; ++s) {
            off[s] = m[s] * (size_t)p.ldo + col0;
            zero[s] = ok[s] && p.row_mask != nullptr && p.row_mask[m[s]] != 0;
        }
#pragma unroll
        for (int c = 0; c < kJ; c += kCh) {
            float2 bv[kCh];
            if (has_bias) {
#pragma unroll
                for (int jj = 0; jj < kCh; ++jj) bv[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * (c + jj)));
            }
#pragma unroll
            for (int s = 0; s < kRows; ++s) {
                if (!ok[s]) continue;
                float(&a)[BN / 2] = acc[s >> 1];
                const int r2 = 2 * (s & 1);
                float2 rv[kCh];
                if (has_res) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        rv[jj] = __ldg(reinterpret_cast<const float2*>(p.residual + off[s] + 8 * (c + jj)));
                }
                if (has_bias) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj) a[4 * (c + jj) + r2] += bv[jj].x, a[4 * (c + jj) + r2 + 1] += bv[jj].y;
                }
                if (res_first) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj) a[4 * (c + jj) + r2] += rv[jj].x, a[4 * (c + jj) + r2 + 1] += rv[jj].y;
                }
                if (act == 1) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        a[4 * (c + jj) + r2] = gelu_erf(a[4 * (c + jj) + r2]),
                        a[4 * (c + jj) + r2 + 1] = gelu_erf(a[4 * (c + jj) + r2 + 1]);
                } else if (act == 2) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        a[4 * (c + jj) + r2] = silu(a[4 * (c + jj) + r2]),
                        a[4 * (c + jj) + r2 + 1] = silu(a[4 * (c + jj) + r2 + 1]);
                } else if (act == 3) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        a[4 * (c + jj) + r2] = fmaxf(a[4 * (c + jj) + r2], 0.f),
                        a[4 * (c + jj) + r2 + 1] = fmaxf(a[4 * (c + jj) + r2 + 1], 0.f);
                } else if (act == 4) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        a[4 * (c + jj) + r2] = tanhf(a[4 * (c + jj) + r2]),
                        a[4 * (c + jj) + r2 + 1] = tanhf(a[4 * (c + jj) + r2 + 1]);
                }
                if (has_pre) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        *reinterpret_cast<float2*>(p.out_pre + off[s] + 8 * (c + jj)) =
                            make_float2(a[4 * (c + jj) + r2], a[4 * (c + jj) + r2 + 1]);
                }
                if (add_res_after) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj) a[4 * (c + jj) + r2] += rv[jj].x, a[4 * (c + jj) + r2 + 1] += rv[jj].y;
                }
                if (zero[s]) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj) a[4 * (c + jj) + r2] = 0.f, a[4 * (c + jj) + r2 + 1] = 0.f;
                }
                if constexpr ((kEpi & kEpiF32) != 0) {
#pragma unroll
                    for (int jj = 0; jj < kCh; ++jj)
                        *reinterpret_cast<float2*>(p.out_f32 + off[s] + 8 * (c + jj)) =
                            make_float2(a[4 * (c + jj) + r2], a[4 * (c + jj) + r2 + 1]);
                }
                if constexpr ((kEpi & kEpiPlanes) != 0) {
                    if (fmt != 0) {
#pragma unroll
                        for (int jj = 0; jj < kCh; ++jj)
                            store_plane_pair<1>(p, a[4 * (c + jj) + r2], a[4 * (c + jj) + r2 + 1], off[s] + 8 * (c + jj));
                    } else {
#pragma unroll
                        for (int jj = 0; jj < kCh; ++jj)
                            store_plane_pair<0>(p, a[4 * (c + jj) + r2], a[4 * (c + jj) + r2 + 1], off[s] + 8 * (c + jj));
                    }
                }
            }
        }
    }
}

template <int BN, int kScheme, int kEpi>
__global__ void __launch_bounds__(kThreads, 1) gemm_sm90_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = GemmCfg<BN, kScheme>;
    constexpr int kStages = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment is required by the 128B swizzle atoms (8 rows x 128 B)
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);  // [kStages]
    uint64_t* empty_bar = full_bar + kStages;                                              // [kStages]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 8 && elect_one()) {
        tma_prefetch_desc(&p.a_hi);
        tma_prefetch_desc(&p.b_hi);
        tma_prefetch_desc(kScheme == 0 ? &p.a_lo : &p.a_q8);
        tma_prefetch_desc(kScheme == 0 ? &p.b_lo : &p.b_q8);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);  // one arrive per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlapped the previous kernel's tail; global memory is touched only below
    pdl_launch_dependents();

    if (warp == 8) {
        if (elect_one()) produce<BN, kScheme, 1>(p, smem, full_bar, empty_bar);
        return;
    }

    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile =====================
    const int wg = warp >> 2;
    const int wq = warp & 3;
    const int num_tiles = p.batches * p.tiles_m_per_batch * p.n_tiles;
    int stage = 0;
    uint32_t phase = 0;
    float acc[1][BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_tile = tile % p.n_tiles;
        const int mt = tile / p.n_tiles;
        const int batch = mt / p.tiles_m_per_batch;
        const int row0 = (mt - batch * p.tiles_m_per_batch) * kBlockM;
        mma_tile<BN, kScheme, 1, 1>(p, smem, full_bar, empty_bar, wg, lane, stage, phase, acc);
        epilogue_tile<BN, kEpi, 1>(p, acc, batch, row0 + wg * 64 + wq * 16 + (lane >> 2), n_tile * BN + 2 * (lane & 3));
    }
}

// CN: CTAs per cluster along N, which share every A box (tile_coord, load_a, release_stage); 1 = no cluster
template <int kScheme, int kEpi, int CN>
__global__ void __launch_bounds__(kPingPongThreads, 1) gemm_sm90_pingpong_kernel(const __grid_constant__ GemmParams p) {
    constexpr int BN = 128;
    using Cfg = GemmCfg<BN, kScheme>;
    constexpr int kStages = Cfg::kStages;
    constexpr int kPasses = kScheme == 0 ? 1 : 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);  // [kStages]
    uint64_t* empty_bar = full_bar + kStages;                                              // [kStages]
    uint64_t* order_bar = empty_bar + kStages;  // [2]: order_bar[wg] = the other warpgroup finished its mainloop

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 8 && elect_one()) {
        tma_prefetch_desc(&p.a_hi);
        tma_prefetch_desc(&p.b_hi);
        tma_prefetch_desc(kScheme == 0 ? &p.a_lo : &p.a_q8);
        tma_prefetch_desc(kScheme == 0 ? &p.b_lo : &p.b_q8);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            // each stage is consumed by ONE warpgroup of each CTA of the cluster: one arrive per warp
            mbar_init(&empty_bar[s], 4 * CN);
        }
        mbar_init(&order_bar[0], 4);
        mbar_init(&order_bar[1], 4);
        fence_mbar_init();
    }
    // CN > 1: no peer multicasts into this CTA's ring or arrives on its barriers before they are initialised
    if constexpr (CN == 1) __syncthreads();
    else cluster_sync();
    pdl_wait();
    pdl_launch_dependents();

    if (warp >= 8) {
        setmaxnreg_dec40();
        if (warp == 8 && elect_one()) produce<BN, kScheme, CN>(p, smem, full_bar, empty_bar);
        return;
    }
    setmaxnreg_inc232();

    // ===================== consumers: warpgroup wg takes this CTA's tiles of ordinal wg, wg + 2, ... =============
    // The mainloops run in tile order, one warpgroup at a time: tile ordinal `ord` starts its MMAs once the other
    // warpgroup has finished those of ordinal ord - 1, and its epilogue then overlaps the other's MMAs of ord + 1.
    // The order also keeps every full-barrier wait at most one phase ahead of the producer: a warpgroup that waited
    // on a stage two ring laps ahead would see the parity of the earlier phase and read a stage not yet loaded.
    const int wg = warp >> 2;
    const int wq = warp & 3;
    const int num_ctiles = p.batches * p.tiles_m_per_batch * (p.n_tiles / CN);
    const int stages_per_tile = kPasses * p.num_k_blocks;
    float acc[2][BN / 2];
    int j = 0;  // tiles this warpgroup has done
    for (int ct = (int)(blockIdx.x + wg * gridDim.x) / CN, ord = wg; ct < num_ctiles;
         ct += 2 * (int)gridDim.x / CN, ord += 2, ++j) {
        // the producer fills the ring in tile order: tile ordinal `ord` starts at ring position ord * stages_per_tile
        const int g = ord * stages_per_tile;
        int stage = g % kStages;
        uint32_t phase = (uint32_t)(g / kStages) & 1u;
        if (ord > 0) mbar_wait(&order_bar[wg], (uint32_t)(j - (wg == 0 ? 1 : 0)) & 1u);
        mma_tile<BN, kScheme, 2, CN>(p, smem, full_bar, empty_bar, 0, lane, stage, phase, acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&order_bar[wg ^ 1]);
        const TileCoord tc = tile_coord<CN>(p, ct, CN == 1 ? 0 : (int)cluster_rank());
        epilogue_tile<BN, kEpi, 2>(p, acc, tc.batch, tc.row0 + wq * 16 + (lane >> 2), tc.n_tile * BN + 2 * (lane & 3));
    }
}

// Per device and kernel instantiation: the shared-memory attribute is set, and how many clusters of it can be resident
// at once (cudaOccupancyMaxActiveClusters; not every GPC holds a whole number of clusters of one-CTA-per-SM CTAs)
struct PersistentLaunch {
    bool attr_set[64] = {};
    int max_clusters[64] = {};
};

// One CTA per SM (cn = 1), or cn x as many clusters as fit at once, capped by the clusters of tiles there are
template <typename Kernel>
static cudaError_t launch_persistent(Kernel kernel, PersistentLaunch& state, int threads, int smem_bytes, int cn,
                                     const GemmParams& p, int sm_count, cudaStream_t stream) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    dev &= 63;
    if (!state.attr_set[dev]) {
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
        if (e != cudaSuccess) return e;
        state.attr_set[dev] = true;
    }
    const int num_ctiles = p.batches * p.tiles_m_per_batch * (p.n_tiles / cn);
    if (num_ctiles <= 0) return cudaSuccess;
    int clusters = sm_count;
    if (cn > 1) {
        if (state.max_clusters[dev] == 0) {
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3(cn * (sm_count / cn));
            cfg.blockDim = dim3(threads);
            cfg.dynamicSmemBytes = smem_bytes;
            cudaLaunchAttribute attr;
            attr.id = cudaLaunchAttributeClusterDimension;
            attr.val.clusterDim.x = (unsigned)cn, attr.val.clusterDim.y = 1, attr.val.clusterDim.z = 1;
            cfg.attrs = &attr;
            cfg.numAttrs = 1;
            e = cudaOccupancyMaxActiveClusters(&state.max_clusters[dev], kernel, &cfg);
            if (e != cudaSuccess) return e;
            if (state.max_clusters[dev] <= 0) return cudaErrorInvalidConfiguration;
        }
        clusters = state.max_clusters[dev];
    }
    const int grid = cn * (num_ctiles < clusters ? num_ctiles : clusters);
    return launch_pdl_cluster(kernel, dim3(grid), dim3(threads), smem_bytes, cn, stream, p);
}

template <int BN, int kScheme, int kEpi>
static cudaError_t launch_impl(const GemmParams& p, int sm_count, cudaStream_t stream) {
    constexpr int kSmem = GemmCfg<BN, kScheme>::kSmemBytes;
    if constexpr (BN == 128) {
        static PersistentLaunch state[3];
        switch (p.cluster_n) {
            case 0:
            case 1:
                return launch_persistent(gemm_sm90_pingpong_kernel<kScheme, kEpi, 1>, state[0], kPingPongThreads,
                                         kSmem, 1, p, sm_count, stream);
            case 2:
                if (p.n_tiles % 2 != 0) return cudaErrorInvalidValue;
                return launch_persistent(gemm_sm90_pingpong_kernel<kScheme, kEpi, 2>, state[1], kPingPongThreads,
                                         kSmem, 2, p, sm_count, stream);
            case 4:
                if (p.n_tiles % 4 != 0) return cudaErrorInvalidValue;
                return launch_persistent(gemm_sm90_pingpong_kernel<kScheme, kEpi, 4>, state[2], kPingPongThreads,
                                         kSmem, 4, p, sm_count, stream);
            default:
                return cudaErrorInvalidValue;
        }
    } else {
        static PersistentLaunch state;
        if (p.cluster_n > 1) return cudaErrorInvalidValue;
        return launch_persistent(gemm_sm90_kernel<BN, kScheme, kEpi>, state, kThreads, kSmem, 1, p, sm_count, stream);
    }
}

// QKV scatter and the fp32 + planes output run at the widths of the encoder's linears only (>= 128 columns)
template <int BN, int kScheme>
static cudaError_t launch_epi(const GemmParams& p, int sm_count, cudaStream_t stream) {
    const bool f32 = p.out_f32 != nullptr, planes = p.out_hi != nullptr;
    if constexpr (BN >= 128) {
        if (p.qkv_mode) return launch_impl<BN, kScheme, kEpiQkv>(p, sm_count, stream);
        if (f32 && planes) return launch_impl<BN, kScheme, kEpiBoth>(p, sm_count, stream);
    }
    if (p.qkv_mode || (f32 && planes)) return cudaErrorInvalidValue;
    if (planes) return launch_impl<BN, kScheme, kEpiPlanes>(p, sm_count, stream);
    if (f32) return launch_impl<BN, kScheme, kEpiF32>(p, sm_count, stream);
    return cudaErrorInvalidValue;  // no output
}

// f16q8 runs at the linears' and convs' widths only (128, 256)
template <int BN>
static cudaError_t launch_n(const GemmParams& p, int sm_count, cudaStream_t stream) {
    if (p.scheme == 0) return launch_epi<BN, 0>(p, sm_count, stream);
    if constexpr (BN == 256 || BN == 128) return launch_epi<BN, 1>(p, sm_count, stream);
    return cudaErrorInvalidValue;
}

cudaError_t launch_gemm(const GemmParams& p, int sm_count, cudaStream_t stream) {
    if (p.scheme != 0 && p.k_steps != 0) return cudaErrorInvalidValue;
    if (p.gelu < 0 || p.gelu > 4 || (p.res_first != 0 && p.out_pre != nullptr)) return cudaErrorInvalidValue;
    if (p.out_fmt != 0 && (p.qkv_mode || (p.out_hi != nullptr && p.out_q8 == nullptr)))
        return cudaErrorInvalidValue;
    switch (p.bn) {
        case 256: return launch_n<256>(p, sm_count, stream);
        case 192: return launch_n<192>(p, sm_count, stream);
        case 160: return launch_n<160>(p, sm_count, stream);
        case 128: return launch_n<128>(p, sm_count, stream);
        case 120: return launch_n<120>(p, sm_count, stream);
        case 96: return launch_n<96>(p, sm_count, stream);
        case 80: return launch_n<80>(p, sm_count, stream);
        case 64: return launch_n<64>(p, sm_count, stream);
        case 48: return launch_n<48>(p, sm_count, stream);
        case 32: return launch_n<32>(p, sm_count, stream);
        case 16: return launch_n<16>(p, sm_count, stream);
        default: return cudaErrorInvalidValue;
    }
}

// ------------------------------------------------------------------------------------------------
// tensor-map encoding through the driver entry point (no link-time libcuda dependency: the C-ABI
// library must load on a GPU-less host for the symbol-export test)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    return fn;
}

int encode_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                        uint64_t stride2, uint32_t box0, uint32_t box1) {
    PFN_encodeTiled fn = get_encode_fn();
    if (fn == nullptr) return -1;
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {stride1 * 2, stride2 * 2};  // bytes
    cuuint32_t box[3] = {box0, box1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    // the swizzle span equals the box row: 64 elements -> 128 B
    if (box0 != 64) return -2;
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return (int)r;
}


int encode_tmap_u8_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                      uint64_t stride2, uint32_t box0, uint32_t box1) {
    PFN_encodeTiled fn = get_encode_fn();
    if (fn == nullptr) return -1;
    // the swizzle span equals the box row: 128 bytes
    if (box0 != 128) return -2;
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {stride1, stride2};  // bytes
    cuuint32_t box[3] = {box0, box1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return (int)r;
}

}  // namespace s3b
