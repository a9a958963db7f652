// reverb.cu — FIR convolutional reverb (SURVEY §8 a14) as a bf16 wgmma GEMM with register accumulators.
//
//   y[v][n] = sum_{k<L} bf16(h_c[k]) * bf16(x[v][n-k])          (per IR channel c; products exact, fp32 accumulate)
//
// For one IR channel all voices share h, so a tile of outputs is a plain GEMM with a long reduction:
//   D[128 voices][BN frames] = A[128][K] * Bt[BN][K]^T,   K = L + BN - 1 (padded to 64), BN in {256, 224, 192, 128}
//   A[v][j]  = xh[row v][H + n0 - Lr + j]         a TMA window of the bf16 sample history, K-major as stored;
//                                                 Lr = roundup(L-1, 8) keeps every box start 16-byte aligned (TMA rule)
//   Bt[i][j] = h[Lr - (j - i)]  (0 <= Lr-(j-i) < L)  Toeplitz expansion of the reversed IR, built ONCE per IR (12 MB per
//                                                 channel for L = 48000) and then L2-resident: it is the same for
//                                                 every time tile and every voice tile.
// The band is (L / K) = 99.5 % dense, so the GEMM does no meaningful wasted work.
//
// Kernel anatomy (persistent grid, one CTA per SM, tiles strided by the grid; 384 threads = 3 warpgroups):
//   warpgroup 0, warp 0   TMA producer   cp.async.bulk.tensor.2d -> 128B-swizzled smem stages, mbarrier expect_tx
//   warpgroups 1 and 2    consumers      each owns 64 of the tile's 128 voices: 4 x wgmma.mma_async m64nBNk16 per 64-wide
//                                        k-block, operands read from shared memory through descriptors, BN/2 accumulator
//                                        registers per thread; a stage is released once the k-block after it is in flight;
//                                        the epilogue stores the fragments straight to y
// 4 stages x (16 KB A + 32 KB B) = 192 KB of shared memory.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "device.cuh"
#include "kernels.cuh"
#include "plan.hpp"
#include "wgmma.cuh"

namespace fw {

constexpr uint32_t RV_BM = 128, RV_BN = 256, RV_BK = 64, RV_STAGES = 4, RV_THREADS = 384, RV_MIN_SLICE_KB = 16;
constexpr uint32_t RV_A_BYTES = RV_BM * RV_BK * 2, RV_B_BYTES = RV_BN * RV_BK * 2;
constexpr uint32_t RV_SMEM_BYTES = RV_STAGES * (RV_A_BYTES + RV_B_BYTES) + 1024 /*align*/ + 256 /*barriers*/;

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int32_t x, int32_t y) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}

// wgmma shared-memory descriptor, K-major operand, 128-byte swizzle: rows at 128 B pitch, 8-row groups at SBO = 1024 B,
// LBO = 1 (unused for swizzled K-major), layout type 1 (bits 62-63) = SWIZZLE_128B.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024u >> 4) << 32) | ((uint64_t)1 << 62);
}

// ---------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------
// Bt[c][i][j] = bf16(h_c[Lr-(j-i)]) where 0 <= Lr-(j-i) < L, else 0.    [ir_ch][256][Kpad]
__global__ void reverb_build_toeplitz(const float* __restrict__ ir, __nv_bfloat16* __restrict__ bt, uint32_t L, uint32_t Lr, uint32_t ir_ch, uint32_t kpad) {
    const size_t n = (size_t)ir_ch * RV_BN * kpad;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
        const uint32_t j = idx % kpad; const size_t ci = idx / kpad; const uint32_t i = ci % RV_BN, c = (uint32_t)(ci / RV_BN);
        float v = 0.0f;
        const int64_t k = (int64_t)Lr - ((int64_t)j - (int64_t)i);
        if (k >= 0 && k < (int64_t)L) v = ir[(size_t)c * L + (size_t)k];
        bt[idx] = __float2bfloat16_rn(v);
    }
}

// xh[c*V + v][cursor + t] = bf16(in[v][c][t]) for t < T: appends the call's block behind the history (8 samples per thread)
__global__ void reverb_prepare(const float* __restrict__ in, __nv_bfloat16* __restrict__ xh, uint32_t V, uint32_t C, uint32_t T, uint32_t in_pitch, uint32_t cursor,
                               uint32_t pitch, uint32_t zero_first, uint32_t chan_base) {
    pdl_launch_dependents();  // the GEMM's set-up (barriers, tensor maps) overlaps this kernel
    pdl_wait();
    const uint32_t row = blockIdx.x;  // c * V + v (rows on grid.x: no 65535 cap)
    const uint32_t c = row / V, v = row % V;
    __nv_bfloat16* dst = xh + ((size_t)chan_base * V + row) * pitch + cursor;
    const float* x = in + ((size_t)v * C + c) * in_pitch;
    const bool vec = (T % 8u) == 0 && (zero_first % 8u) == 0 && (in_pitch % 4u) == 0 && (cursor % 8u) == 0 && (pitch % 8u) == 0 &&
                     (reinterpret_cast<uintptr_t>(in) % 16u) == 0;
    if (vec) {
        for (uint32_t i = (blockIdx.y * blockDim.x + threadIdx.x) * 8u; i < T; i += gridDim.y * blockDim.x * 8u) {
            float4 a = __ldcs(reinterpret_cast<const float4*>(x + i)), b = __ldcs(reinterpret_cast<const float4*>(x + i + 4));
            if (i < zero_first) { a = make_float4(0.f, 0.f, 0.f, 0.f); b = a; }
            __nv_bfloat162 p0 = __floats2bfloat162_rn(a.x, a.y), p1 = __floats2bfloat162_rn(a.z, a.w), p2 = __floats2bfloat162_rn(b.x, b.y), p3 = __floats2bfloat162_rn(b.z, b.w);
            uint4 o;
            o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1); o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
            *reinterpret_cast<uint4*>(dst + i) = o;
        }
    } else {
        for (uint32_t i = blockIdx.y * blockDim.x + threadIdx.x; i < T; i += gridDim.y * blockDim.x) dst[i] = __float2bfloat16_rn(i < zero_first ? 0.0f : x[i]);
    }
}

struct ReverbGemmArgs {
    float* out;                   // row (v * C + c) at out + row * out_pitch
    uint32_t out_pitch, V, C, T, Lr, cursor, ir_ch, num_kb, chan_base;
    uint32_t tiles_n, tiles_m, total_tiles;  // output tiles along frames / voices (per channel); tiles_n * tiles_m * C
    // Tail wave: the last `tail_tiles` tiles (fewer than half a wave) are each split along K between `tail_split` CTAs; the
    // CTA with the first slice adds the others' partial sums (fix-up workspace, one flag per CTA).
    uint32_t full_tiles, tail_tiles, tail_split;
    float* ws; uint32_t* flags; uint32_t epoch;
};
struct RvSeg { uint32_t tile, k0, k1; };
// segment i of CTA P: whole tiles P, P + NP, ... of the full waves, then (at most) one slice of a tail tile
__device__ __forceinline__ uint32_t rv_seg_count(const ReverbGemmArgs& a, uint32_t P, uint32_t NP) {
    const uint32_t full = a.full_tiles > P ? (a.full_tiles - P + NP - 1) / NP : 0u;
    return full + (P < a.tail_tiles * a.tail_split ? 1u : 0u);
}
__device__ __forceinline__ RvSeg rv_seg(const ReverbGemmArgs& a, uint32_t P, uint32_t NP, uint32_t i) {
    const uint32_t t = P + i * NP;
    if (t < a.full_tiles) return RvSeg{t, 0u, a.num_kb};
    const uint32_t j = P / a.tail_split, sl = P % a.tail_split;
    return RvSeg{a.full_tiles + j, (uint32_t)((uint64_t)sl * a.num_kb / a.tail_split), (uint32_t)((uint64_t)(sl + 1) * a.num_kb / a.tail_split)};
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
// keeps the accumulators in their registers across the asynchronous MMAs (the compiler must not move or copy them)
template <uint32_t N> __device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
    for (uint32_t i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Persistent grid, one CTA per SM: CTA g computes tiles g, g + G, g + 2G, ... each over the whole reduction. All CTAs walk
// the k-blocks of their tiles IN STEP, and the Toeplitz operand B depends only on (channel, k-block): at any moment the whole
// chip reads the same few B blocks, so B streams through L2 once instead of living there; a split that hands every SM its own
// k-range would put the CTAs at as many different k-offsets. SM coverage comes from the tile width instead: BN is chosen per
// call among 256 / 224 / 192 / 128 frames so that the tile count fills whole waves of SMs, and a tail wave at most half full
// is split along K (see ReverbGemmArgs).
template <uint32_t BN>
__global__ void __launch_bounds__(RV_THREADS, 1) reverb_gemm_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const ReverbGemmArgs a) {
    constexpr uint32_t B_BYTES = BN * RV_BK * 2, NACC = BN / 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));  // SWIZZLE_128B wants 1024-byte tiles
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + RV_STAGES * RV_A_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + RV_STAGES * (RV_A_BYTES + RV_B_BYTES));
    uint64_t* empty_bar = full_bar + RV_STAGES;

    pdl_launch_dependents();  // the next kernel's launch latency hides behind this one; it waits for our results itself
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t P = blockIdx.x, NP = gridDim.x, num_kb = a.num_kb;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (uint32_t s = 0; s < RV_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }  // empty: one arrival per consumer warpgroup
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t tiles_per_ch = a.tiles_n * a.tiles_m;
    const uint32_t nseg = rv_seg_count(a, P, NP);

    if (warp == 0) {
        // ===== TMA producer =====
        pdl_wait();  // the history buffer is written by reverb_prepare just before us
        if (lane == 0) {
            uint32_t it = 0;
            for (uint32_t si = 0; si < nseg; ++si) {
                const RvSeg sg = rv_seg(a, P, NP, si);
                const uint32_t t = sg.tile;
                const uint32_t c = t / tiles_per_ch, rem = t % tiles_per_ch, mt = rem / a.tiles_n, nt = rem % a.tiles_n;
                const int32_t col_a0 = (int32_t)(a.cursor + nt * BN) - (int32_t)a.Lr;  // multiple of 8 elements = 16 bytes
                const int32_t row_a = (int32_t)((a.chan_base + c) * a.V + mt * RV_BM), row_b = (int32_t)(((a.chan_base + c) % a.ir_ch) * RV_BN);
                for (uint32_t kb = sg.k0; kb < sg.k1; ++kb, ++it) {
                    const uint32_t s = it % RV_STAGES, ph = (it / RV_STAGES) & 1u;
                    mbar_wait(&empty_bar[s], ph ^ 1u);
                    mbar_expect_tx(&full_bar[s], RV_A_BYTES + B_BYTES);
                    tma_load_2d(smem_a + s * RV_A_BYTES, &tm_a, &full_bar[s], col_a0 + (int32_t)(kb * RV_BK), row_a);
                    tma_load_2d(smem_b + s * RV_B_BYTES, &tm_b, &full_bar[s], (int32_t)(kb * RV_BK), row_b);
                }
            }
        }
    } else if (warp >= 4) {
        // ===== consumers: MMA + epilogue, 64 voices of the tile per warpgroup =====
        const uint32_t wg = (warp >> 2) - 1u, ctid = threadIdx.x - 128u, wtid = ctid & 127u;
        const uint32_t rrow = wg * 64u + (wtid >> 5) * 16u + (lane >> 2), ccol = (lane & 3u) * 2u;  // fragment origin: rows rrow, rrow + 8
        float acc[NACC];
        uint32_t it = 0;
        for (uint32_t seg = 0; seg < nseg; ++seg) {
            const RvSeg sg = rv_seg(a, P, NP, seg);
            uint32_t prev_s = 0;
            acc_fence(acc);
#pragma unroll 1
            for (uint32_t kb = sg.k0; kb < sg.k1; ++kb, ++it) {
                const uint32_t s = it % RV_STAGES, ph = (it / RV_STAGES) & 1u;
                mbar_wait(&full_bar[s], ph);
                const uint64_t adesc = wgmma_desc_sw128(smem_u32(smem_a + s * RV_A_BYTES + wg * (64u * RV_BK * 2u)));
                const uint64_t bdesc = wgmma_desc_sw128(smem_u32(smem_b + s * RV_B_BYTES));
                wgmma_fence();
#pragma unroll
                for (uint32_t k = 0; k < RV_BK / 16; ++k)  // +32 bytes per K=16 step inside the 128-byte swizzle atom
                    WgmmaBf16<BN>::mma(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb != sg.k0 || k != 0) ? 1u : 0u);
                wgmma_commit();
                if (kb != sg.k0) {  // the previous k-block's MMAs have retired: its stage goes back to the producer
                    wgmma_wait<1>();
                    if (wtid == 0) mbar_arrive(&empty_bar[prev_s]);
                }
                prev_s = s;
            }
            wgmma_wait<0>();
            acc_fence(acc);
            if (sg.k1 > sg.k0 && wtid == 0) mbar_arrive(&empty_bar[prev_s]);

            const uint32_t t = sg.tile;
            const uint32_t c = t / tiles_per_ch, rem = t % tiles_per_ch, mt = rem / a.tiles_n, nt = rem % a.tiles_n;
            const uint32_t n0 = nt * BN, v0 = mt * RV_BM + rrow;
            const bool partial = sg.k0 != 0;                                  // a later K-slice of a tail tile: park the partial sums
            const uint32_t n_follow = (sg.k0 == 0 && sg.k1 < num_kb) ? a.tail_split - 1u : 0u;  // first slice: add the others'
            float* ws_me = a.ws + (size_t)P * (RV_BM * RV_BN) + ctid;  // [register][consumer thread]
            if (partial) {
#pragma unroll
                for (uint32_t i = 0; i < NACC; ++i) __stcg(ws_me + (size_t)i * 256u, acc[i]);
                __threadfence();  // publish: all 256 consumer threads have stored, then one release store
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (ctid == 0) st_release_gpu(a.flags + P, a.epoch);
                continue;
            }
            if (n_follow) {  // the other slices run in this same wave on CTAs P + 1 ...: they finish when we do
                for (uint32_t f = lane; f < n_follow; f += 32u) while (ld_acquire_gpu(a.flags + P + 1u + f) != a.epoch) { }
                __syncwarp();
                for (uint32_t f = 0; f < n_follow; ++f) {  // ascending K: ((first + slice 1) + slice 2) ...
                    const float* wf = a.ws + (size_t)(P + 1u + f) * (RV_BM * RV_BN) + ctid;
#pragma unroll
                    for (uint32_t i = 0; i < NACC; ++i) acc[i] += __ldcg(wf + (size_t)i * 256u);
                }
            }
            float* dst0 = a.out + ((size_t)v0 * a.C + c) * a.out_pitch + n0 + ccol;
            float* dst1 = dst0 + (size_t)8u * a.C * a.out_pitch;
            const bool ok0 = v0 < a.V, ok1 = v0 + 8u < a.V;
            const bool vec = (a.out_pitch & 1u) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 7u) == 0;
#pragma unroll
            for (uint32_t j = 0; j < BN / 8; ++j) {
                const uint32_t col = n0 + ccol + j * 8u;
                if (vec && col + 2u <= a.T) {
                    if (ok0) __stcs(reinterpret_cast<float2*>(dst0 + j * 8u), make_float2(acc[4 * j], acc[4 * j + 1]));
                    if (ok1) __stcs(reinterpret_cast<float2*>(dst1 + j * 8u), make_float2(acc[4 * j + 2], acc[4 * j + 3]));
                } else {
#pragma unroll
                    for (uint32_t e = 0; e < 2; ++e) if (col + e < a.T) {
                        if (ok0) dst0[j * 8u + e] = acc[4 * j + e];
                        if (ok1) dst1[j * 8u + e] = acc[4 * j + 2 + e];
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr; cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
static bool make_map_bf16_2d(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t outer, uint64_t pitch_elems, uint32_t box_inner, uint32_t box_outer) {
    EncodeTiledFn fn = encode_tiled();
    if (!fn) return false;
    const cuuint64_t dims[2] = {inner, outer};
    const cuuint64_t strides[1] = {pitch_elems * 2};
    const cuuint32_t box[2] = {box_inner, box_outer};
    const cuuint32_t estr[2] = {1, 1};
    return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static uint32_t reverb_lr(uint32_t L) { return ((L - 1 + 7) / 8) * 8; }
uint32_t reverb_kpad(uint32_t L) { return ((reverb_lr(L) + RV_BN + RV_BK - 1) / RV_BK) * RV_BK; }
uint32_t reverb_hist(uint32_t L) { return ((L - 1 + 63) / 64) * 64; }  // history samples kept in front of each call's block

cudaError_t launch_reverb_build(const float* d_ir, void* d_bt, uint32_t L, uint32_t ir_ch, cudaStream_t st) {
    const size_t n = (size_t)ir_ch * RV_BN * reverb_kpad(L);
    reverb_build_toeplitz<<<(unsigned)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096), 256, 0, st>>>(d_ir, static_cast<__nv_bfloat16*>(d_bt), L, reverb_lr(L), ir_ch, reverb_kpad(L));
    return cudaGetLastError();
}

// One call: append the block (bf16) behind the history at `cursor`, run the GEMM over windows ending in it.
// The caller owns the cursor policy (compaction when the buffer is full); cursor is a multiple of 8 and >= Lr.
size_t reverb_ws_bytes() { return (size_t)reverb_grid_max() * RV_BM * RV_BN * sizeof(float); }  // one 128 x 256 f32 partial per CTA
uint32_t reverb_grid_max() {
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    return (uint32_t)sms;
}

template <uint32_t BN>
static cudaError_t launch_gemm(const CUtensorMap& tm_a, const CUtensorMap& tm_b, const ReverbGemmArgs& ga, uint32_t grid, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(reverb_gemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RV_SMEM_BYTES);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    return launch_ex(reverb_gemm_kernel<BN>, dim3(grid), dim3(RV_THREADS), RV_SMEM_BYTES, st, true, tm_a, tm_b, ga);
}

// Tile width for a call: least (waves) x (cycles per k-block) of a paper model (not fitted to per-width timings, and blind to
// the K-split of the tail). Cycles per k-block = max(MMA, shared-memory traffic at
// 128 B/clk): 128 x BN x 64 MACs at 2048 per clock = 4 x BN, against one TMA write of A and B plus each warpgroup's read of
// its half of A and all of B = (32 KB + 3 x BN x 128 B) / 128.
static uint32_t reverb_pick_bn(uint32_t T, uint32_t tiles_mc, uint32_t units) {
    static const uint32_t cand[4] = {256, 224, 192, 128};
    uint32_t best = 256; uint64_t best_cost = ~0ull;
    for (uint32_t bn : cand) {
        const uint64_t tiles = (uint64_t)((T + bn - 1) / bn) * tiles_mc, waves = (tiles + units - 1) / units;
        const uint64_t mma = 4ull * bn, smem = 256ull + 3ull * bn;
        const uint64_t cost = waves * ((mma > smem ? mma : smem) + 8u);
        if (cost < best_cost) { best_cost = cost; best = bn; }
    }
    return best;
}

cudaError_t launch_reverb(const ReverbCall& rc, cudaStream_t st, std::string* err) {
    const uint32_t in_pitch = rc.in_pitch ? rc.in_pitch : rc.T, out_pitch = rc.out_pitch ? rc.out_pitch : rc.T;
    {
        const uint32_t per_block = 256 * 8;
        dim3 grid(rc.C * rc.V, (rc.T + per_block - 1) / per_block < 32 ? (rc.T + per_block - 1) / per_block : 32);
        cudaError_t e = launch_ex(reverb_prepare, grid, dim3(256), 0, st, true, rc.in, static_cast<__nv_bfloat16*>(rc.xh), rc.V, rc.C, rc.T, in_pitch, rc.cursor, rc.pitch, rc.zero_first, rc.chan_base);
        if (e != cudaSuccess) return e;
    }
    const uint32_t sms = reverb_grid_max(), tiles_m = (rc.V + RV_BM - 1) / RV_BM;
    const uint32_t bn = reverb_pick_bn(rc.T, tiles_m * rc.C, sms);
    const uint32_t kpad = reverb_kpad(rc.L);  // pitch of the Toeplitz rows (built for the widest tile)
    CUtensorMap tm_a, tm_b;
    if (!make_map_bf16_2d(&tm_a, rc.xh, (uint64_t)rc.cursor + rc.T, (uint64_t)(rc.chan_base + rc.C) * rc.V, rc.pitch, RV_BK, RV_BM) ||
        !make_map_bf16_2d(&tm_b, rc.bt, kpad, (uint64_t)rc.ir_ch * RV_BN, kpad, RV_BK, bn)) {
        if (err) *err = "cuTensorMapEncodeTiled failed";
        return cudaErrorInvalidValue;
    }
    ReverbGemmArgs ga{};
    ga.out = rc.out; ga.out_pitch = out_pitch; ga.V = rc.V; ga.C = rc.C; ga.T = rc.T; ga.Lr = reverb_lr(rc.L); ga.cursor = rc.cursor; ga.ir_ch = rc.ir_ch;
    ga.num_kb = (reverb_lr(rc.L) + bn + RV_BK - 1) / RV_BK;  // Bt[i][j] is zero for j > Lr + i: a narrower tile has a shorter reduction
    ga.chan_base = rc.chan_base;
    ga.tiles_n = (rc.T + bn - 1) / bn; ga.tiles_m = tiles_m; ga.total_tiles = ga.tiles_n * ga.tiles_m * rc.C;
    if (ga.total_tiles == 0) return cudaSuccess;
    ga.full_tiles = ga.total_tiles; ga.tail_tiles = 0; ga.tail_split = 1; ga.ws = rc.ws; ga.flags = rc.flags; ga.epoch = rc.epoch;
    if (rc.ws && rc.flags && ga.total_tiles > sms) {  // a tail wave at most half full is split along K (see ReverbGemmArgs)
        const uint32_t rem = ga.total_tiles % sms;
        // as many slices as there are idle CTAs per tail tile, but never fewer than RV_MIN_SLICE_KB k-blocks in a slice: every slice
        // starts with a clearing MMA (an empty one would hand on stale accumulators), and a few k-blocks do not pay for the fix-up
        const uint32_t split = rem ? (sms / rem < ga.num_kb / RV_MIN_SLICE_KB ? sms / rem : ga.num_kb / RV_MIN_SLICE_KB) : 0u;
        if (split >= 2u) { ga.tail_tiles = rem; ga.tail_split = split; ga.full_tiles = ga.total_tiles - rem; }
    }
    const uint32_t G = ga.total_tiles < sms ? ga.total_tiles : sms;
    switch (bn) {
        case 224: return launch_gemm<224>(tm_a, tm_b, ga, G, st);
        case 192: return launch_gemm<192>(tm_a, tm_b, ga, G, st);
        case 128: return launch_gemm<128>(tm_a, tm_b, ga, G, st);
        default: return launch_gemm<256>(tm_a, tm_b, ga, G, st);
    }
}

}  // namespace fw
