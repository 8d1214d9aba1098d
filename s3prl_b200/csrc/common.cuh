// Shared device helpers for the sm_90a kernels: mbarrier / TMA / wgmma descriptor PTX wrappers,
// the bf16 hi+lo split used for error-compensated tensor-core products, exact-erf GELU.
//
// Numerics contract: every fp32 contraction on the hot path is computed as
//   x*w ~= hi(x)*hi(w) + hi(x)*lo(w) + lo(x)*hi(w)     (bf16 operands, fp32 accumulation)
// with hi(v) = bf16_rn(v), lo(v) = bf16_rn(v - hi(v)); relative error per product ~2^-16.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

namespace s3b {

// ----------------------------------------------------------------------------------------------
// small utilities
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float gelu_erf(float x) {
    // exact-erf GELU, nn.GELU() default (reference: wav2vec2_model.py:2893,2902,2904; 1899-1900):
    //   gelu(x) = 0.5 x (1 + erf(x/sqrt2)) = 0.5 x * (x >= 0 ? 2 - erfc(|x|/sqrt2) : erfc(|x|/sqrt2))
    // erfc(z) = t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-z^2), t = 1/(1 + p z)   (Abramowitz-Stegun 7.1.26,
    // |error| <= 1.5e-7). ~17 instructions with two MUFU ops instead of erff's ~27, and no cancellation for
    // x < 0: measured max |error| vs float64 4.2e-7 over [-12, 12] (torch's own fp32 GELU: 1.2e-6), see
    // tests/test_oracle_cpu.py::test_gelu_formula. conv0 and the fc1 epilogue are issue-bound on this function.
#ifdef S3B_GELU_LIBM
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
#else
    const float z = fabsf(x) * 0.70710678118654752440f;
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * (z * -1.4426950408889634f)));
    const float erfc_z = poly * t * e;
    return 0.5f * x * (x >= 0.0f ? 2.0f - erfc_z : erfc_z);
#endif
}

// sigmoid(x) = 1 / (1 + e^-x) and SiLU(x) = x * sigmoid(x) (the Conformer's Swish, torch.nn.SiLU); two MUFU ops,
// relative error a few ulp. x -> -inf: e^-x = inf, rcp = 0, so both go to 0 without a NaN.
__device__ __forceinline__ float sigmoid_fast(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return r;
}
__device__ __forceinline__ float silu(float x) { return x * sigmoid_fast(x); }
// ReLU that keeps a NaN, as torch.relu does (fmaxf(NaN, 0) would return 0 and hide it)
__device__ __forceinline__ float relu_nan(float x) { return x < 0.0f ? 0.0f : x; }

// hi/lo split of an fp32 value into two bf16 values (round-to-nearest-even both times)
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

__device__ __forceinline__ void fsub2(float& x, float& y, float a0, float a1, float b0, float b1) {
    x = __fsub_rn(a0, b0);
    y = __fsub_rn(a1, b1);
}

// pack two floats -> two bf16x2 words (hi word, lo word); element 0 in the low half.
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
    float ra, rb;
    fsub2(ra, rb, a, b, __uint_as_float(hi << 16), __uint_as_float(hi & 0xffff0000u));
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(rb), "f"(ra));
}

// ----------------------------------------------------------------------------------------------
// "f16q8" operand format: x ~= h16 + l8 * 2^-kQ8ShiftA with h16 = fp16_rn(x) and two e4m3 planes
//   h8 = e4m3(h16)                        (the operand of the  A_hi * W_lo  correction MMA)
//   l8 = e4m3((x - h16) * 2^kQ8ShiftA)    (the operand of the  A_lo * W_hi  correction MMA)
// Weights: w16 = fp16_rn(w), wh8 = e4m3(w * 2^kQ8ShiftB), wl8 = e4m3((w - w16) * 2^kQ8ShiftD). Both correction
// products therefore carry the factor 2^kQ8Scale (= ShiftA + ShiftB = ShiftD); they are accumulated FIRST and the first
// main fp16 MMA of a tile the accumulator registers are scaled back by 2^-15 (exact: a power of two).
// 4 bytes per activation element, like the bf16 hi/lo pair it replaces; 8 instructions per element pair.
// ----------------------------------------------------------------------------------------------
static constexpr int kQ8ShiftA = 11;  // activations: residual of an 11-bit significand, scaled into e4m3's range
static constexpr int kQ8ShiftB = 4;   // weights |w| <= 28 stay finite in e4m3 (satfinite clamps beyond)
static constexpr int kQ8ShiftD = 15;  // weight residuals (|w - w16| <= 2^-11 |w|)
static constexpr int kQ8Scale = 15;   // = kQ8ShiftA + kQ8ShiftB = kQ8ShiftD (activation h8 plane is unscaled)
static_assert(kQ8ShiftA + kQ8ShiftB == kQ8Scale && kQ8ShiftD == kQ8Scale, "correction products must share one scale");

// two floats -> fp16x2 word (element 0 in the low half), e4m3x2 of the fp16 values, e4m3x2 of the scaled residuals
__device__ __forceinline__ void split_q8_pack2(float a, float b, uint32_t& h16, uint16_t& h8, uint16_t& l8) {
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(h16) : "f"(b), "f"(a));
    asm("cvt.rn.satfinite.e4m3x2.f16x2 %0, %1;" : "=h"(h8) : "r"(h16));
    float ha, hb;
    asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %2; cvt.f32.f16 %0, lo; cvt.f32.f16 %1, hi; }"
        : "=f"(ha), "=f"(hb)
        : "r"(h16));
    float ra, rb;
    fsub2(ra, rb, a, b, ha, hb);
    const float sc = (float)(1 << kQ8ShiftA);
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(l8) : "f"(rb * sc), "f"(ra * sc));
}
// The two e4m3 planes of an operand are stored as ONE interleaved q8 plane of 2 bytes per element: every 32-element
// chunk of the flat element order is 64 bytes [l8 x 32 | h8 x 32]. A 64-element k-block of a row whose width is a
// multiple of 64 is then one 128-byte row [l8 k0..31 | h8 k0..31 | l8 k32..63 | h8 k32..63], which the GEMM loads as
// one box with the 128-byte swizzle. Byte offset of element `elem`, plane p (0 = l8, 1 = h8):
//   2 elem - (elem & 31) + 32 p  =  elem + (elem & ~31) + 32 p
__host__ __device__ __forceinline__ size_t q8_off(size_t elem, int p) { return elem + (elem & ~(size_t)31) + 32 * (size_t)p; }
// bytes of the q8 plane of n elements: the last chunk is whole
__host__ __device__ __forceinline__ size_t q8_bytes(size_t n) { return 2 * ((n + 31) & ~(size_t)31); }

// four consecutive elements (elem % 4 == 0, so inside one chunk) -> one 8-byte fp16 store + two 4-byte e4m3 stores
__device__ __forceinline__ void store_q8x4(const float4& y, __nv_bfloat16* p16, uint8_t* q8, size_t elem) {
    uint32_t h0, h1;
    uint16_t a0, a1, b0, b1;
    split_q8_pack2(y.x, y.y, h0, a0, b0);
    split_q8_pack2(y.z, y.w, h1, a1, b1);
    uint8_t* q = q8 + q8_off(elem, 0);
    *reinterpret_cast<uint2*>(p16 + elem) = make_uint2(h0, h1);
    *reinterpret_cast<uint32_t*>(q + 32) = (uint32_t)a0 | ((uint32_t)a1 << 16);
    *reinterpret_cast<uint32_t*>(q) = (uint32_t)b0 | ((uint32_t)b1 << 16);
}

// GEMM-operand output of a producer kernel (LayerNorm, conv-0, GEMM epilogues, attention, pos_conv combine):
// fmt 0 = bf16 hi / lo planes (bf16x3 scheme), fmt 1 = fp16 plane + the interleaved q8 plane (f16q8 scheme).
struct OutPlanes {
    __nv_bfloat16* hi;
    __nv_bfloat16* lo;
    uint8_t* q8;
    int fmt;
};
__host__ __device__ inline OutPlanes no_planes() { return OutPlanes{nullptr, nullptr, nullptr, 0}; }

// four consecutive elements starting at element index `elem` (elem % 4 == 0)
__device__ __forceinline__ void store_planes4(const OutPlanes& o, const float4& y, size_t elem) {
    if (o.fmt != 0) {
        store_q8x4(y, o.hi, o.q8, elem);
    } else {
        uint32_t h0, l0, h1, l1;
        split_pack2(y.x, y.y, h0, l0);
        split_pack2(y.z, y.w, h1, l1);
        *reinterpret_cast<uint2*>(o.hi + elem) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(o.lo + elem) = make_uint2(l0, l1);
    }
}
// eight consecutive elements (elem % 8 == 0): 16-byte stores on the 2-byte planes
__device__ __forceinline__ void store_planes8(const OutPlanes& o, const float (&y)[8], size_t elem) {
    if (o.fmt != 0) {
        uint32_t h[4];
        uint16_t a[4], b[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) split_q8_pack2(y[2 * e], y[2 * e + 1], h[e], a[e], b[e]);
        uint8_t* q = o.q8 + q8_off(elem, 0);
        *reinterpret_cast<uint4*>(o.hi + elem) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint2*>(q + 32) =
            make_uint2((uint32_t)a[0] | ((uint32_t)a[1] << 16), (uint32_t)a[2] | ((uint32_t)a[3] << 16));
        *reinterpret_cast<uint2*>(q) =
            make_uint2((uint32_t)b[0] | ((uint32_t)b[1] << 16), (uint32_t)b[2] | ((uint32_t)b[3] << 16));
    } else {
        uint32_t h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) split_pack2(y[2 * e], y[2 * e + 1], h[e], l[e]);
        *reinterpret_cast<uint4*>(o.hi + elem) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(o.lo + elem) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}
// two consecutive elements (elem % 2 == 0)
__device__ __forceinline__ void store_planes2(const OutPlanes& o, float y0, float y1, size_t elem) {
    if (o.fmt != 0) {
        uint32_t h;
        uint16_t a, b;
        split_q8_pack2(y0, y1, h, a, b);
        uint8_t* q = o.q8 + q8_off(elem, 0);
        *reinterpret_cast<uint32_t*>(o.hi + elem) = h;
        *reinterpret_cast<uint16_t*>(q + 32) = a;
        *reinterpret_cast<uint16_t*>(q) = b;
    } else {
        uint32_t h, l;
        split_pack2(y0, y1, h, l);
        *reinterpret_cast<uint32_t*>(o.hi + elem) = h;
        *reinterpret_cast<uint32_t*>(o.lo + elem) = l;
    }
}
// read back element pair `elem` (even) of an operand in either format
__device__ __forceinline__ float2 load_planes2(const OutPlanes& o, size_t elem) {
    const uint32_t h = *reinterpret_cast<const uint32_t*>(o.hi + elem);
    if (o.fmt != 0) {
        const uint16_t l = *reinterpret_cast<const uint16_t*>(o.q8 + q8_off(elem, 0));
        float h0, h1;
        asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %2; cvt.f32.f16 %0, lo; cvt.f32.f16 %1, hi; }"
            : "=f"(h0), "=f"(h1)
            : "r"(h));
        uint32_t lf;  // e4m3x2 -> f16x2
        asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(lf) : "h"(l));
        float l0, l1;
        asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %2; cvt.f32.f16 %0, lo; cvt.f32.f16 %1, hi; }"
            : "=f"(l0), "=f"(l1)
            : "r"(lf));
        const float inv = 1.0f / (float)(1 << kQ8ShiftA);
        return make_float2(fmaf(l0, inv, h0), fmaf(l1, inv, h1));
    }
    const uint32_t l = *reinterpret_cast<const uint32_t*>(o.lo + elem);
    return make_float2(__uint_as_float(h << 16) + __uint_as_float(l << 16),
                       __uint_as_float(h & 0xffff0000u) + __uint_as_float(l & 0xffff0000u));
}

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// One lane of a CONVERGED warp: ptxas knows that the region guarded by elect.sync is single-threaded and feeds
// TMA operands through uniform registers directly.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (launch error) instead of a hung GPU. No printf here: a function call
// anywhere in a kernel makes ptxas serialise all of its wgmma instructions.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 8000000000LL) __trap();  // ~4 s at 2 GHz
    }
}

// ----------------------------------------------------------------------------------------------
// thread-block clusters
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// address of the same shared-memory location in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t peer_addr(const void* p, uint32_t rank) {
    uint32_t out;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(out) : "r"(smem_u32(p)), "r"(rank));
    return out;
}
// store to a peer_addr address (distributed shared memory)
__device__ __forceinline__ void st_cluster_f4(uint32_t addr, float4 v) {
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}

// ----------------------------------------------------------------------------------------------
// the recurrences' dot products (gru.cu, lstm.cu, cpc_lstm.cu)
// ----------------------------------------------------------------------------------------------
// one butterfly level: lanes with bit kOff set keep values [kHalf, 2 kHalf), the others [0, kHalf); each adds its
// partner's copy of what it keeps. The kept values move to [0, kHalf).
template <int kOff, int kHalf, int kN>
__device__ __forceinline__ void halve(float (&acc)[kN], int lane) {
    static_assert(2 * kHalf <= kN, "halve: more values kept than held");
    const bool upper = (lane & kOff) != 0;
#pragma unroll
    for (int v = 0; v < kHalf; ++v) {
        const float send = upper ? acc[v] : acc[v + kHalf];
        const float keep = upper ? acc[v + kHalf] : acc[v];
        acc[v] = keep + __shfl_xor_sync(0xffffffffu, send, kOff);
    }
}

// the recurrences' sigmoid: IEEE division and expf, the accuracy of PyTorch's CPU and cuDNN cells
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// arrive on an mbarrier of any CTA of the cluster (a peer_addr address). The default .release.cta semantics: a
// .cluster-scoped release compiles to a MEMBAR.ALL.GPU that waits for every outstanding store of the thread (the GEMM
// epilogue's), and a consumer releasing a shared-memory stage that only wgmma read needs no such fence.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar_cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(bar_cluster_addr) : "memory");
}

// generic-proxy writes to smem -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), 128B-swizzled tiles
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// the same box into the same shared-memory offset of every CTA of the cluster in `cta_mask`, each completing the
// transaction bytes on its own mbarrier at `bar`'s offset
__device__ __forceinline__ void tma_load_3d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                                      int c1, int c2, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(cta_mask)
        : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (sm_90a) for a K-major tile stored as rows of ROW_BYTES bytes with the
// matching swizzle (the layout TMA produces for a {ROW_BYTES, rows} box): 8-row atoms are 8 * ROW_BYTES apart (SBO),
// LBO is unused for swizzled K-major tiles (set to 1). Layout type: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B.
// Advancing the start address by 32 bytes (+2) steps 16 bf16 / 32 e4m3 elements along K inside the swizzle row.
// ----------------------------------------------------------------------------------------------
template <int ROW_BYTES>
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t smem_addr) {
    static_assert(ROW_BYTES == 128 || ROW_BYTES == 64, "unsupported swizzle span");
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)((8 * ROW_BYTES) >> 4) << 32;
    d |= (uint64_t)(ROW_BYTES == 128 ? 1 : 2) << 62;
    return d;
}

}  // namespace s3b

// Programmatic dependent launch (PDL): a kernel launched with the stream-serialization attribute may start its
// prologue (barrier init, tensor-map prefetch) while the previous kernel of the stream drains;
// `pdl_wait()` blocks until that previous grid has completed and its writes are visible, so every global read or
// write of a kernel must come after it. `pdl_launch_dependents()` lets the next kernel's CTAs be scheduled as
// soon as every CTA of this grid has issued it. Both are no-ops for a normal launch. S3B_PDL=0 disables.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("S3B_PDL");
        v = (e != nullptr && e[0] == '0') ? 0 : 1;
    }
    return v != 0;
}

// cluster_x > 1: thread-block clusters of cluster_x CTAs along x (grid.x a multiple of it), in the same launch
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, int cluster_x,
                                      cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = (unsigned)cluster_x, attr[n].val.clusterDim.y = 1, attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
    return launch_pdl_cluster(kernel, grid, block, smem, 1, stream, args...);
}

// cudaFuncSetAttribute applies to the current device only: one "done" flag per device so that a process that
// drives several GPUs configures each of them.
struct PerDeviceOnce {
    bool done[64] = {};
    bool& current() {
        int d = 0;
        cudaGetDevice(&d);
        return done[d & 63];
    }
};
