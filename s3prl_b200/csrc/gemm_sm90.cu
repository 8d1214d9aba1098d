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
// One CTA per SM, persistent over 128 x BN output tiles; 288 threads:
//   warps 0..3, 4..7 : two consumer warpgroups, 64 output rows each (wgmma m64nBN, accumulators in registers),
//                      then the epilogue straight from the accumulator registers
//   warp 8           : TMA producer (A and W boxes -> swizzled shared-memory ring of kStages stages)
// With 288 threads ptxas may give every thread up to 224 registers: the 128 accumulators of a 256-wide tile fit.
#include <stdio.h>

#include "common.cuh"
#include "gemm.cuh"
#include "wgmma.cuh"

namespace s3b {

static constexpr int kBlockM = 128;
static constexpr int kThreads = 288;
static constexpr int kSmemBudget = 220 * 1024;

// RB: bytes of one K row of a stage plane = the swizzle span (128: 64 bf16 elements, 64: 32 bf16 / 64 e4m3 elements).
// f16q8 uses RB = 64 with 64 elements of K per stage: pass 0 fills the four planes with 64-byte e4m3 rows
// [A_l8 A_h8 W_h8 W_l8], pass 1 fills [A16 | W16] with 128-byte fp16 rows (each spanning two planes). Both are
// 48 KB at BN = 256, which makes the ring four deep there (six at BN = 128).
template <int BN, int RB>
struct GemmCfg {
    static constexpr int kAPlane = kBlockM * RB;
    static constexpr int kBPlane = BN * RB;
    static constexpr int kStageBytes = 2 * kAPlane + 2 * kBPlane;
    static constexpr int kStages = (kSmemBudget - 2048) / kStageBytes > 6 ? 6 : (kSmemBudget - 2048) / kStageBytes;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(kStages >= 2, "tile too large for the shared-memory ring");
};

// Epilogue of one row pair (2 consecutive columns): v = acc (+bias) ; gelu? ; then the output modes of gemm.cuh
__device__ __forceinline__ void epilogue_pair(const GemmParams& p, size_t m, int col, bool masked, float x0, float x1) {
    if (p.bias != nullptr) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        x0 += b.x, x1 += b.y;
    }
    if (p.gelu) x0 = gelu_erf(x0), x1 = gelu_erf(x1);
    if (p.qkv_mode) {
        // m = b*T + t ; col = which*D + h*64 + d (column pairs never straddle a head)
        const int b = (int)(m / (size_t)p.T);
        const int t = (int)(m - (size_t)b * p.T);
        const int which = col / p.D;
        const int within = col - which * p.D;
        const int h = within >> 6;
        const int d = within & 63;
        const size_t bh = (size_t)b * p.H + h;
        if (which < 2) {
            if (which == 0) x0 *= p.q_scale, x1 *= p.q_scale;
            uint32_t hi, lo;
            split_pack2(x0, x1, hi, lo);
            const size_t o = (bh * p.T + t) * 64 + d;
            *reinterpret_cast<uint32_t*>((which == 0 ? p.q_hi : p.k_hi) + o) = hi;
            *reinterpret_cast<uint32_t*>((which == 0 ? p.q_lo : p.k_lo) + o) = lo;
        } else {
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(x0, h0, l0);
            split_bf16(x1, h1, l1);
            const size_t o = (bh * 64 + d) * (size_t)p.Tp + t;
            p.vt_hi[o] = h0, p.vt_lo[o] = l0;
            p.vt_hi[o + p.Tp] = h1, p.vt_lo[o + p.Tp] = l1;
        }
        return;
    }
    const size_t off = m * (size_t)p.ldo + col;
    if (p.out_pre != nullptr) *reinterpret_cast<float2*>(p.out_pre + off) = make_float2(x0, x1);
    if (p.residual != nullptr) {
        const float2 r = __ldg(reinterpret_cast<const float2*>(p.residual + off));
        x0 += r.x, x1 += r.y;
    }
    if (masked) x0 = 0.f, x1 = 0.f;
    if (p.out_f32 != nullptr) *reinterpret_cast<float2*>(p.out_f32 + off) = make_float2(x0, x1);
    if (p.out_hi != nullptr) {
        const OutPlanes o{p.out_hi, p.out_lo, p.out_h8, p.out_l8, p.out_fmt};
        store_planes2(o, x0, x1, off);
    }
}

template <int BN, int RB, int kScheme>
__global__ void __launch_bounds__(kThreads, 1) gemm_sm90_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = GemmCfg<BN, RB>;
    constexpr int kStages = Cfg::kStages;
    constexpr int kNR = BN / 2;  // accumulator registers per thread
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
        if (kScheme == 0) {
            tma_prefetch_desc(&p.a_lo);
            tma_prefetch_desc(&p.b_lo);
        }
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);  // one arrive per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlapped the previous kernel's tail; global memory is touched only below
    pdl_launch_dependents();

    const int tiles_m = p.batches * p.tiles_m_per_batch;
    const int num_tiles = tiles_m * p.n_tiles;
    // two_cta layout: the W boxes hold BN/2 rows and a stage takes two of them (gemm.cuh)
    const int b_boxes = p.two_cta ? 2 : 1;
    const int b_box_rows = BN / b_boxes;
    constexpr int kPasses = kScheme == 0 ? 1 : 2;

    if (warp == 8) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int n_tile = tile % p.n_tiles;
                const int mt = tile / p.n_tiles;
                const int batch = mt / p.tiles_m_per_batch;
                const int row0 = (mt - batch * p.tiles_m_per_batch) * kBlockM;
                const int a_k0 = p.a_k_per_ntile * n_tile;
                const int b_n0 = p.b_n_tiled ? n_tile * BN : 0;
                const int b_z0 = n_tile * p.b_z_per_ntile;
                for (int pass = 0; pass < kPasses; ++pass) {
                    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                        const int kq = kb / p.kb_per_row;
                        const int kr = kb - kq * p.kb_per_row;
                        mbar_wait(&empty_bar[stage], phase ^ 1u);
                        uint8_t* st = smem + stage * Cfg::kStageBytes;
                        uint8_t* sb = st + 2 * Cfg::kAPlane;
                        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)Cfg::kStageBytes);
                        const int a_row = row0 + kq * p.a_row_step + p.a_row_off;
                        const int a_k = a_k0 + kr * p.block_k;
                        const int b_k = (p.b_k_linear ? kb : kr) * p.block_k;
                        const int b_z = p.b_k_linear ? 0 : b_z0 + kq;
                        if (kScheme == 1 && pass == 1) {
                            // [A16 | W16]: one fp16 box of 128-byte rows each, spanning both planes of the stage
                            tma_load_3d(st, &p.a_hi, &full_bar[stage], a_k, a_row, batch);
                            for (int h = 0; h < b_boxes; ++h)
                                tma_load_3d(sb + h * b_box_rows * 128, &p.b_hi, &full_bar[stage], b_k, b_n0 + h * b_box_rows, b_z);
                        } else {
                            // planes: scheme 0 [A_hi A_lo W_hi W_lo]; scheme 1 pass 0 [A_l8 A_h8 W_h8 W_l8] (64-byte rows)
                            const CUtensorMap* ma0 = kScheme == 0 ? &p.a_hi : &p.a_l8;
                            const CUtensorMap* ma1 = kScheme == 0 ? &p.a_lo : &p.a_h8;
                            const CUtensorMap* mb0 = kScheme == 0 ? &p.b_hi : &p.b_h8;
                            const CUtensorMap* mb1 = kScheme == 0 ? &p.b_lo : &p.b_l8;
                            tma_load_3d(st, ma0, &full_bar[stage], a_k, a_row, batch);
                            tma_load_3d(st + Cfg::kAPlane, ma1, &full_bar[stage], a_k, a_row, batch);
                            for (int h = 0; h < b_boxes; ++h) {
                                const int rows = b_n0 + h * b_box_rows;
                                tma_load_3d(sb + h * b_box_rows * RB, mb0, &full_bar[stage], b_k, rows, b_z);
                                tma_load_3d(sb + Cfg::kBPlane + h * b_box_rows * RB, mb1, &full_bar[stage], b_k, rows, b_z);
                            }
                        }
                        if (++stage == kStages) stage = 0, phase ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====================
    const int wg = warp >> 2;
    const int wq = warp & 3;
    const int k_steps = p.k_steps > 0 ? p.k_steps : RB / 32;  // 16-wide k-steps per stage (scheme 0)
    int stage = 0;
    uint32_t phase = 0;
    float acc[kNR];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_tile = tile % p.n_tiles;
        const int mt = tile / p.n_tiles;
        const int batch = mt / p.tiles_m_per_batch;
        const int row0 = (mt - batch * p.tiles_m_per_batch) * kBlockM;
#pragma unroll
        for (int i = 0; i < kNR; ++i) acc[i] = 0.f;

        // Stage s is released once the wgmma group reading it has retired; one group stays in flight so that the
        // tensor pipe is fed while this warpgroup waits for the next stage.
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
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[pending]);
                    pending = -1;
                }
                const float s = 1.0f / (float)(1 << kQ8Scale);
#pragma unroll
                for (int i = 0; i < kNR; ++i) acc[i] *= s;
                wgmma_fence();
            }
            for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t st = smem_u32(smem + stage * Cfg::kStageBytes);
                const uint32_t a0 = st + wg * 64 * RB, a1 = a0 + Cfg::kAPlane;
                const uint32_t b0 = st + 2 * Cfg::kAPlane, b1 = b0 + Cfg::kBPlane;
                const uint64_t da0 = make_wgmma_desc<RB>(a0), da1 = make_wgmma_desc<RB>(a1);
                const uint64_t db0 = make_wgmma_desc<RB>(b0), db1 = make_wgmma_desc<RB>(b1);
                wgmma_fence();
                if constexpr (kScheme == 0) {
#pragma unroll
                    for (int k = 0; k < RB / 32; ++k) {
                        if (k < k_steps) {
                            // advance 16 bf16 (= 32 bytes) along K inside the swizzle atom: +2 in (addr >> 4) units
                            const uint64_t ko = (uint64_t)(k * 2);
                            Wgmma<BN, 0>::ss(acc, da1 + ko, db0 + ko, first ? 0u : 1u);
                            Wgmma<BN, 0>::ss(acc, da0 + ko, db1 + ko, 1u);
                            Wgmma<BN, 0>::ss(acc, da0 + ko, db0 + ko, 1u);
                            first = false;
                        }
                    }
                } else if (pass == 0) {  // (kScheme == 1 from here on, RB == 64)
                    // A_l8 x W_h8 and A_h8 x W_l8, K = 32 per MMA (32 bytes), two k-steps per 64-byte row
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        const uint64_t ko = (uint64_t)(k * 2);
                        Wgmma<BN, 2>::ss(acc, da0 + ko, db0 + ko, first ? 0u : 1u);
                        Wgmma<BN, 2>::ss(acc, da1 + ko, db1 + ko, 1u);
                        first = false;
                    }
                } else {
                    // A16[k..k+64) x W16[k..k+64), K = 16 per MMA: one box of 128-byte rows each, spanning both
                    // 64-byte planes of the stage (the warpgroup's 64 A rows start 64 * 128 bytes apart)
                    const uint64_t da = make_wgmma_desc<128>(st + wg * 64 * 128), db = make_wgmma_desc<128>(b0);
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint64_t ko = (uint64_t)(k * 2);
                        Wgmma<BN, 1>::ss(acc, da + ko, db + ko, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (pending >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[pending]);
                }
                pending = stage;
                if (++stage == kStages) stage = 0, phase ^= 1u;
            }
        }
        wgmma_wait<0>();
        if (pending >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[pending]);
        }

        // ===================== epilogue: thread holds rows r, r + 8 and columns 8j + 2(lane%4) + {0,1} ==========
        const int col0 = n_tile * BN + 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = row0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
            if (row >= p.rows_per_batch) continue;
            const size_t m = (size_t)batch * p.out_rows_per_batch + row;
            const bool masked = (p.row_mask != nullptr) && (p.row_mask[m] != 0);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) epilogue_pair(p, m, col0 + 8 * j, masked, acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
        }
    }
}

template <int BN, int RB, int kScheme>
static cudaError_t launch_impl(const GemmParams& p, int sm_count, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, RB>;
    auto kernel = gemm_sm90_kernel<BN, RB, kScheme>;
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.current();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    const int num_tiles = p.batches * p.tiles_m_per_batch * p.n_tiles;
    if (num_tiles <= 0) return cudaSuccess;
    const int grid = num_tiles < sm_count ? num_tiles : sm_count;
    return launch_pdl(kernel, dim3(grid), dim3(kThreads), Cfg::kSmemBytes, stream, p);
}

template <int BN>
static cudaError_t launch_n(const GemmParams& p, int sm_count, cudaStream_t stream) {
    if (p.scheme != 0) {
        if constexpr (BN == 256 || BN == 192 || BN == 128) return launch_impl<BN, 64, 1>(p, sm_count, stream);
        return cudaErrorInvalidValue;
    }
    if (p.block_k == 64) return launch_impl<BN, 128, 0>(p, sm_count, stream);
    return launch_impl<BN, 64, 0>(p, sm_count, stream);
}

cudaError_t launch_gemm_bf16x3(const GemmParams& p, int sm_count, cudaStream_t stream) {
    if (p.ln_gamma != nullptr) return cudaErrorNotSupported;  // LayerNorm is a separate launch (norm.cu)
    if (p.scheme != 0 ? (p.block_k != 64 || p.k_steps != 0) : (p.block_k != 64 && p.block_k != 32))
        return cudaErrorInvalidValue;
    if (p.scheme == 0 && p.block_k == 32 && (p.two_cta || p.k_steps != 0)) return cudaErrorInvalidValue;
    if (p.out_fmt != 0 && (p.qkv_mode || (p.out_hi != nullptr && (p.out_h8 == nullptr || p.out_l8 == nullptr))))
        return cudaErrorInvalidValue;
    switch (p.umma_n) {
        case 256: return launch_n<256>(p, sm_count, stream);
        case 192: return launch_n<192>(p, sm_count, stream);
        case 128: return launch_n<128>(p, sm_count, stream);
        case 64: return p.two_cta ? cudaErrorInvalidValue : launch_n<64>(p, sm_count, stream);
        case 48: return p.two_cta ? cudaErrorInvalidValue : launch_n<48>(p, sm_count, stream);
        case 32: return p.two_cta ? cudaErrorInvalidValue : launch_n<32>(p, sm_count, stream);
        case 16: return p.two_cta ? cudaErrorInvalidValue : launch_n<16>(p, sm_count, stream);
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
    // the swizzle span equals the box row: 64 elements -> 128 B, 32 elements -> 64 B
    if (box0 != 64 && box0 != 32) return -2;
    const CUtensorMapSwizzle sw = box0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return (int)r;
}


int encode_tmap_u8_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                      uint64_t stride2, uint32_t box0, uint32_t box1) {
    PFN_encodeTiled fn = get_encode_fn();
    if (fn == nullptr) return -1;
    // the swizzle span equals the box row: 128 e4m3 elements -> 128 B, 64 elements -> 64 B
    if (box0 != 128 && box0 != 64) return -2;
    const CUtensorMapSwizzle sw = box0 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {stride1, stride2};  // bytes == elements
    cuuint32_t box[3] = {box0, box1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return (int)r;
}

}  // namespace s3b
