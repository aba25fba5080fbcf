// coach_b200/csrc/nn_gemm_tc.cuh -- the gather-GEMM on the Hopper tensor cores (wgmma, fp32 register accumulators).
//
// Same contraction / tables / epilogue as nn_gemm_fast.cuh, computed as a 3-way BF16 operand split with fp32
// accumulation:
//     x = x1 + x2 + x3 (bf16 each, exact: truncation split);   A*B ~= a1 b1 + [a1 b2 + a2 b1 + a2 b2 + a1 b3 + a3 b1]
// Two accumulators per output tile: MAIN collects a1*b1, CORR collects the five correction products, so the
// truncation error of the small products stays relative to their 2^-8 smaller magnitude.  The host caps the reduction
// length per launch (split-R, summed afterwards in fp32 round-to-nearest by split_reduce_kernel), which bounds MAIN to
// <= 64 accumulating k16 steps.
//
// uint8 A operands (the Atari frames of conv1, forward and weight gradient) take the EXACT path when the caller
// declares a_u8_div (lut[v] == v / a_u8_div): the raw integers 0..255 are exact bf16 values, so A needs ONE plane and
// the product three MMAs (a b1 + [a b2 + a b3]); the 1 / a_u8_div scale is applied once to the accumulated sum.
//
// Operands are staged BY THE THREADS into the canonical no-swizzle wgmma shared-memory layouts (8 x 16-byte core
// matrices): the A operand needs table-driven gather addressing,
// uint8 conversion and the bf16 split, none of which TMA can do.  A is K-major when the reduction index is
// contiguous in memory (forward / data gradients) and MN-major for the weight gradients (A^T); B [R, N] row-major is
// always MN-major.  Within a warp the 8 lanes of a quarter-warp always write the 8 rows (16 B each) of ONE core
// matrix, i.e. 128 contiguous bytes: conflict-free 128-bit shared stores.
//
// The reduction-indexed gather tables of the CTA's slice (<= 1024 entries) are copied to shared memory once, so the
// per-chunk global loads have no dependent table load in front of them; the loads of chunk c+1 are issued into
// registers right after chunk c has been converted (their latency overlaps the barrier, the MMA issue and the wait
// for the stage).
//
// PLANES.  A producer that knows its output feeds another GEMM writes the bf16 hi / mid / lo planes next to the fp32
// result (EpiParams::c_planes, 8x8 core-tiled format of nn_gemm.cuh; weights are split once per step by
// cb200_split_planes).  GEMMs whose operands both have planes run in nn_gemm_tiled.cuh (bulk-copy fed, no conversion
// work).  The register-staged kernel below remains for uint8 sources (exact path), LUT sources and plane-less fp32
// operands; it accepts B planes too (conv1: weights / dY), which removes the B-side split.
//
// CTA = 128 threads = one warpgroup = one 128 x BN output tile (BN <= 64: the accumulators of both 64-row halves live
// in its registers).  Two shared-memory stages: while the tensor core works on chunk c (asynchronously, one wgmma
// commit group per chunk), all threads convert chunk c+1.  The accumulators are then staged through shared memory and
// thread t writes output row t in the epilogue: bias / activation / activation-derivative mask -> global.
#pragma once
#include <cuda_bf16.h>

#include "nn_gemm_fast.cuh"

namespace cb200 {
namespace gemm {

constexpr int kTcBM = 128;
constexpr int kTcBK = 32;
constexpr int kTcStages = 2;
constexpr int kTcMaxSlice = 1024;       // reduction indices per CTA (table entries held in shared memory)

__device__ __forceinline__ uint64_t gmma_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    // start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout_type = 0 (no swizzle) [62,64).  No swizzle: LBO is
    // the step between core matrices along K, SBO along M / N, for K-major and MN-major operands alike.
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    return d;
}
// D[64 x N] += A[64 x 16] * B[16 x N], bf16 operands from shared memory, fp32 accumulators in registers (the
// m64nNk16 fragment: thread (warp w, lane l) of the warpgroup holds rows 16 w + l / 4 and 16 w + l / 4 + 8, columns
// 8 j + 2 (l % 4) + {0, 1} in d[4 j .. 4 j + 3]).  kTA / kTB: the operand is MN-major (transposed), not K-major.
template <int kTA, int kTB>
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %20, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %18, %19;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "n"(kTA), "n"(kTB), "r"(1));
}
template <int kTA, int kTB>
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %36, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %34, %35;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "n"(kTA), "n"(kTB), "r"(1));
}
// one 64 x BN product: BN = 32 -> one n32 MMA, otherwise BN / 64 n64 MMAs on consecutive runs of eight column cores
// of B (SBO = 128 bytes between column cores: the next 64 columns start 1024 bytes further)
template <int BN, int kTA, int kTB>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db) {
    static_assert(BN == 32 || BN % 64 == 0, "BN");
    if constexpr (BN == 32) {
        wgmma_n32<kTA, kTB>(d, da, db);
    } else {
#pragma unroll
        for (int b = 0; b < BN / 64; ++b) wgmma_n64<kTA, kTB>(d + 32 * b, da, db + (uint64_t)(b * (1024 >> 4)));
    }
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// accumulator fragments (MAIN + CORR) of a 64-row slab -> fp32 tile in shared memory, row stride ld floats
template <int BN>
__device__ __forceinline__ void store_fragment(float* tile, int ld, int r0, const float* main, const float* corr) {
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    const int row = r0 + 16 * w + (l >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * (l & 3);
        *reinterpret_cast<float2*>(tile + (size_t)row * ld + col) =
            make_float2(main[4 * j] + corr[4 * j], main[4 * j + 1] + corr[4 * j + 1]);
        *reinterpret_cast<float2*>(tile + (size_t)(row + 8) * ld + col) =
            make_float2(main[4 * j + 2] + corr[4 * j + 2], main[4 * j + 3] + corr[4 * j + 3]);
    }
}

// 8 fp32 -> three 16-byte groups of bf16 (hi / mid / lo)
struct Split8 {
    uint4 h, m, l;
};
__device__ __forceinline__ Split8 split8(const float4& lo4, const float4& hi4) {
    // Truncation split: hi = top 8 significant bits of x, mid = top 8 of the (exact) remainder, lo = the rest (<= 8
    // bits, exact).  x == hi + mid + lo exactly for |x| >= 2^-110 (below that `lo` is an fp32 denormal whose low
    // half-word is cut: absolute error < 2^-133), and each piece is a bf16 (upper half-word).
    const float x[8] = {lo4.x, lo4.y, lo4.z, lo4.w, hi4.x, hi4.y, hi4.z, hi4.w};
    uint32_t hb[8], mb[8], lb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        hb[j] = __float_as_uint(x[j]) & 0xffff0000u;
        const float r1 = x[j] - __uint_as_float(hb[j]);
        mb[j] = __float_as_uint(r1) & 0xffff0000u;
        lb[j] = __float_as_uint(r1 - __uint_as_float(mb[j]));
    }
    Split8 s;
    // pack the upper half-words of consecutive elements: result = (b[2i+1] & 0xffff0000) | (b[2i] >> 16)
    s.h = make_uint4(__byte_perm(hb[0], hb[1], 0x7632), __byte_perm(hb[2], hb[3], 0x7632),
                     __byte_perm(hb[4], hb[5], 0x7632), __byte_perm(hb[6], hb[7], 0x7632));
    s.m = make_uint4(__byte_perm(mb[0], mb[1], 0x7632), __byte_perm(mb[2], mb[3], 0x7632),
                     __byte_perm(mb[4], mb[5], 0x7632), __byte_perm(mb[6], mb[7], 0x7632));
    s.l = make_uint4(__byte_perm(lb[0], lb[1], 0x7632), __byte_perm(lb[2], lb[3], 0x7632),
                     __byte_perm(lb[4], lb[5], 0x7632), __byte_perm(lb[6], lb[7], 0x7632));
    return s;
}
// 8 bytes -> 8 bf16 holding the integers exactly.  0x4B0000vv is the float 2^23 + v; subtracting 2^23 leaves float(v),
// whose upper half-word is its bf16 (v < 256 has at most 8 significant bits).
__device__ __forceinline__ uint4 u8x8_to_bf16(uint32_t w0, uint32_t w1) {
    uint32_t f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        f[j] = __float_as_uint(__uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7440 + j)) - 8388608.f);
        f[4 + j] = __float_as_uint(__uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7440 + j)) - 8388608.f);
    }
    return make_uint4(__byte_perm(f[0], f[1], 0x7632), __byte_perm(f[2], f[3], 0x7632), __byte_perm(f[4], f[5], 0x7632),
                      __byte_perm(f[6], f[7], 0x7632));
}

__device__ __forceinline__ float4 as_float4(const uint4& q) {
    return make_float4(__uint_as_float(q.x), __uint_as_float(q.y), __uint_as_float(q.z), __uint_as_float(q.w));
}
__device__ __forceinline__ bool tap_ok(int ri, int ci, int oh, int ow) {
    const int y = (ri >> 16) - (ci >> 16), x = (ri & 0xffff) - (ci & 0xffff);
    return y >= 0 && y < oh && x >= 0 && x < ow;
}

// thread = output row of the accumulated tile (fp32 in shared memory, row stride ld) -> (1 / a_u8_div) -> bias /
// activation / activation-derivative mask -> fp32 result (+ bf16 planes) or split-R partial
template <int BN>
__device__ __forceinline__ void tc_epilogue(const EpiParams& ep, const float* tile, int ld, bool have_acc,
                                            int m0, int n0, int M, int m_end, int N, int split, bool u8,
                                            float a_u8_div, int unscaled_row, int col_lo = 0, int col_hi = BN) {
    // row = thread index modulo 128; a second group of four warps may take the other half of the columns
    // [col_lo, col_hi)
    const int tid = threadIdx.x & 127;
    const int m = m0 + tid;
    const bool scale_row = u8 && m != unscaled_row;
    const bool live = m < m_end;
    // everything that depends only on the row (the asm memory clobbers below would otherwise force re-evaluation)
    const bool vec = !ep.accumulate && (N % 8 == 0);
    const size_t part_row = ((size_t)split * M + (live ? m : 0)) * N;
    size_t c_row = 0, p_row = 0;
    if (live && ep.splits <= 1) {
        c_row = (ep.c_rowmap ? (size_t)__ldg(ep.c_rowmap + m) : (size_t)m) * ep.ldc;
        if (ep.c_planes || ep.mask_planes) p_row = plane_row((size_t)m, ep.c_prow_npix, ep.c_prow_batch);
    }
    const size_t p_base =
        (ep.c_planes || ep.mask_planes) ? (p_row >> 3) * (size_t)(ep.c_plane_cols >> 3) * 64 + (p_row & 7) * 8 : 0;
#pragma unroll 1
    for (int col = col_lo; col < col_hi; col += 16) {
        if (!live) continue;
        float v[16];
        if (have_acc) {
            const float4* r = reinterpret_cast<const float4*>(tile + (size_t)tid * ld + col);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 q = r[j];
                v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            if (scale_row) v[j] = __fdiv_rn(v[j], a_u8_div);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int nb = n0 + col + 8 * h;
            float* w = v + 8 * h;
            if (nb >= N) continue;
            if (vec) {
                // 2 x 128-bit stores per 8 columns (rows of C / the partial buffer are 16-byte aligned)
                float* dst;
                if (ep.splits > 1) {
                    dst = ep.partial + part_row + nb;
                } else {
                    const size_t elem = c_row + nb;
                    dst = ep.c + elem;
                    if (ep.bias) {
                        const float4 b0 = __ldg(reinterpret_cast<const float4*>(ep.bias + nb));
                        const float4 b1 = __ldg(reinterpret_cast<const float4*>(ep.bias + nb + 4));
                        w[0] += b0.x; w[1] += b0.y; w[2] += b0.z; w[3] += b0.w;
                        w[4] += b1.x; w[5] += b1.y; w[6] += b1.z; w[7] += b1.w;
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) w[j] = apply_act(w[j], ep.act);
                    if (ep.mask_planes) {
                        // mask from the planes of the activation (same tiled geometry as the result)
                        const uint16_t* mp = ep.mask_planes + p_base + (size_t)(nb >> 3) * 64;
                        const uint4 h = *reinterpret_cast<const uint4*>(mp);
                        float yy[8] = {__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u),
                                       __uint_as_float(h.y << 16), __uint_as_float(h.y & 0xffff0000u),
                                       __uint_as_float(h.z << 16), __uint_as_float(h.z & 0xffff0000u),
                                       __uint_as_float(h.w << 16), __uint_as_float(h.w & 0xffff0000u)};
                        if (ep.mask_act != CB200_ACT_RELU) {
#pragma unroll
                            for (int j = 0; j < 8; ++j)
                                yy[j] = mask_from_planes(mp + j, ep.mask_plane_stride, ep.mask_act);
                        }
#pragma unroll
                        for (int j = 0; j < 8; ++j) w[j] *= act_grad_from_output(yy[j], ep.mask_act);
                    } else if (ep.mask_y) {
                        const float4 y0 = *reinterpret_cast<const float4*>(ep.mask_y + elem);
                        const float4 y1 = *reinterpret_cast<const float4*>(ep.mask_y + elem + 4);
                        const float yy[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
#pragma unroll
                        for (int j = 0; j < 8; ++j) w[j] *= act_grad_from_output(yy[j], ep.mask_act);
                    }
                }
                if (ep.splits <= 1 && ep.c == nullptr) {
                    // fp32 result not wanted (only the planes are consumed): skip 40 % of the epilogue's write traffic
                } else if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
                    *reinterpret_cast<float4*>(dst) = make_float4(w[0], w[1], w[2], w[3]);
                    *reinterpret_cast<float4*>(dst + 4) = make_float4(w[4], w[5], w[6], w[7]);
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) dst[j] = w[j];
                }
                if (ep.c_planes && ep.splits <= 1) {
                    // one core-matrix row (8 columns of one plane row) = 16 bytes per plane
                    uint16_t* p = ep.c_planes + p_base + (size_t)(nb >> 3) * 64;
                    const Split8 sp = split8(make_float4(w[0], w[1], w[2], w[3]), make_float4(w[4], w[5], w[6], w[7]));
                    *reinterpret_cast<uint4*>(p) = sp.h;
                    *reinterpret_cast<uint4*>(p + ep.c_plane_stride) = sp.m;
                    *reinterpret_cast<uint4*>(p + 2 * ep.c_plane_stride) = sp.l;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int n = nb + j;
                    if (n >= N) continue;
                    if (ep.splits > 1)
                        ep.partial[part_row + n] = w[j];
                    else
                        epilogue_store(ep, m, n, w[j]);
                }
            }
        }
    }
}

// the operand stages, reused for the fp32 accumulator tile [128][BN + 4] once the main loop is done
template <int BN, bool kU8>
__host__ __device__ constexpr size_t tc_region_bytes() {
    constexpr size_t st = (size_t)kTcStages * ((kU8 ? 1 : 3) * kTcBM * kTcBK * 2 + 3 * BN * kTcBK * 2);
    constexpr size_t tile = (size_t)kTcBM * (BN + 4) * sizeof(float);
    return st > tile ? st : tile;
}
template <int BN, bool kU8>
constexpr size_t tc_smem_bytes() {
    return tc_region_bytes<BN, kU8>() + 1024 + 2 * kTcMaxSlice * sizeof(int32_t);
}

// kU8: A is uint8 and contracted exactly (see the header); otherwise A is fp32, or uint8 through the LUT (general).
template <int BN, bool kTransA, bool kU8>
__global__ void __launch_bounds__(128) gemm_tc_kernel(FastA a, const float* __restrict__ b, int ldb, EpiParams ep,
                                                      int M, int N, int R, int r_per_split, float a_u8_div,
                                                      const uint16_t* __restrict__ b_planes, int64_t b_plane_stride,
                                                      int b_prow_npix, int b_prow_batch) {
    constexpr int NA = kU8 ? 1 : 3;                       // bf16 planes of the A operand
    constexpr int A_SPLIT = kTcBM * kTcBK * 2;            // bytes of one bf16 plane of the A chunk (8 KB)
    constexpr int B_SPLIT = BN * kTcBK * 2;
    constexpr int STAGE = NA * A_SPLIT + 3 * B_SPLIT;
    static_assert(BN <= 64, "one warpgroup holds the accumulators of both 64-row halves");
    constexpr size_t REGION = tc_region_bytes<BN, kU8>();
    extern __shared__ __align__(1024) uint8_t smem[];
    float* lut_s = reinterpret_cast<float*>(smem + REGION);                          // 256 floats (uint8 via LUT)
    int32_t* tab_off = reinterpret_cast<int32_t*>(smem + REGION + 1024);
    int32_t* tab_info = tab_off + kTcMaxSlice;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * kTcBM, n0 = blockIdx.y * BN;
    const int split = blockIdx.z;
    const int r_lo = split * r_per_split;
    const int r_hi = min(R, r_lo + r_per_split);
    const bool has_info = a.rowinfo != nullptr;

    if (!kU8 && a.lut) {
        for (int i = tid; i < 256; i += 128) lut_s[i] = a.lut[i];
    }
    // reduction-indexed tables of this CTA's slice: K-major -> coloff / colinfo of every 4th reduction index (the
    // gather groups); MN-major -> rowoff / rowinfo of every reduction row
    if (!kTransA) {
        for (int j = tid; 4 * j < r_hi - r_lo; j += 128) {
            tab_off[j] = __ldg(a.coloff + r_lo + 4 * j);
            if (has_info) tab_info[j] = __ldg(a.colinfo + r_lo + 4 * j);
        }
    } else {
        for (int j = tid; j < r_hi - r_lo; j += 128) {
            tab_off[j] = __ldg(a.rowoff + r_lo + j);
            if (has_info) tab_info[j] = __ldg(a.rowinfo + r_lo + j);
        }
    }
    __syncthreads();
    if (!kU8 && a.lut) a.lut = lut_s;

    // ---- per-thread constants of the A loader ---------------------------------------------------------------------
    // K-major item (row, k-group of 8 = two gather groups of 4): lane l of warp w handles k-group l >> 3 of rows
    // 8 w + (l & 7) + 32 i, i < 4.  A quarter-warp covers 8 rows of one k-group (one core matrix in shared memory);
    // the four quarter-warps cover the 128 contiguous bytes (fp32) of each of those rows in global memory.
    // MN-major item (reduction row kk, group g of 8 logical columns): thread t handles kk = 8 i + (t & 7), g = t >> 3.
    const int kgrp = lane >> 3;
    int fix_off[4] = {-1, -1, -1, -1};     // K-major: rowoff[m_i];  MN-major: [0],[1] = coloff[k], coloff[k + 4]
    int fix_info[4] = {0, 0, 0, 0};
    if (!kTransA) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + 8 * warp + (lane & 7) + 32 * i;
            if (m < a.rows) {
                fix_off[i] = __ldg(a.rowoff + m);
                if (has_info) fix_info[i] = __ldg(a.rowinfo + m);
            }
        }
    } else {
        const int k = m0 + 8 * (tid >> 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int kc = k + 4 * h;
            if (kc < a.cols) {
                fix_off[h] = __ldg(a.coloff + kc);
                if (has_info) fix_info[h] = __ldg(a.colinfo + kc);
            } else if (kc == a.ones_col) {
                fix_off[h] = -2;
            }
        }
    }

    const int nchunks = (r_hi - r_lo + kTcBK - 1) / kTcBK;
    constexpr int NG = BN / 8;                               // 8-column groups of the B tile
    constexpr int NB_IT = kTcBK * NG / 128;                  // B items per thread
    static_assert(kTcBK * NG % 128 == 0, "B loader shape");
    // B item (reduction row kk, column group g): it = tid + 128 i -> kk = (it & 7) + 8 (it / (8 NG)), g = (it >> 3) % NG

    float4 va[kU8 ? 1 : 4][2];
    uint2 wa[kU8 ? 4 : 1];
    uint4 vb[NB_IT][3];                                      // two float4 (fp32 B) or the three plane rows (B planes)
    const uint8_t* src8 = static_cast<const uint8_t*>(a.src);
    const float* src32 = static_cast<const float*>(a.src);
    auto load_group = [&](int off, float4& v, uint32_t& w) {       // one gather group of 4 elements
        if (kU8) {
            w = __ldg(reinterpret_cast<const uint32_t*>(src8 + off));
        } else if (a.lut) {
            const uint32_t x = __ldg(reinterpret_cast<const uint32_t*>(src8 + off));
            v = make_float4(a.lut[x & 255], a.lut[(x >> 8) & 255], a.lut[(x >> 16) & 255], a.lut[x >> 24]);
        } else {
            v = __ldg(reinterpret_cast<const float4*>(src32 + off));
        }
    };
    auto fetch = [&](int c) {
        const int r0 = r_lo + c * kTcBK;
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!kTransA) {
            const int ra = r0 + kgrp * 8, rb = ra + 4;
            const int ja = (ra - r_lo) >> 2;
            const bool ina = ra < r_hi, inb = rb < r_hi;
            const int ca = ina ? tab_off[ja] : 0, cb = inb ? tab_off[ja + 1] : 0;
            int ia = 0, ib = 0;
            if (has_info) {
                ia = ina ? tab_info[ja] : 0;
                ib = inb ? tab_info[ja + 1] : 0;
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float4 v0 = z4, v1 = z4;
                uint32_t w0 = 0u, w1 = 0u;
                if (fix_off[i] >= 0) {
                    if (ina && (!has_info || tap_ok(fix_info[i], ia, a.oh, a.ow))) load_group(fix_off[i] + ca, v0, w0);
                    if (inb && (!has_info || tap_ok(fix_info[i], ib, a.oh, a.ow))) load_group(fix_off[i] + cb, v1, w1);
                }
                if (kU8) {
                    wa[kU8 ? i : 0] = make_uint2(w0, w1);
                } else {
                    va[kU8 ? 0 : i][0] = v0;
                    va[kU8 ? 0 : i][1] = v1;
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int mrow = r0 + 8 * i + (tid & 7);          // logical A row (reduction index)
                float4 v0 = z4, v1 = z4;
                uint32_t w0 = 0u, w1 = 0u;
                if (mrow < r_hi) {
                    const int ro = tab_off[mrow - r_lo];
                    const int ri = has_info ? tab_info[mrow - r_lo] : 0;
                    if (fix_off[0] >= 0) {
                        if (!has_info || tap_ok(ri, fix_info[0], a.oh, a.ow)) load_group(ro + fix_off[0], v0, w0);
                    } else if (fix_off[0] == -2) {
                        v0.x = 1.f;                               // bias-gradient row: sum_m 1 * dY[m, n]
                        w0 = 1u;
                    }
                    if (fix_off[1] >= 0) {
                        if (!has_info || tap_ok(ri, fix_info[1], a.oh, a.ow)) load_group(ro + fix_off[1], v1, w1);
                    } else if (fix_off[1] == -2) {
                        v1.x = 1.f;
                        w1 = 1u;
                    }
                }
                if (kU8) {
                    wa[kU8 ? i : 0] = make_uint2(w0, w1);
                } else {
                    va[kU8 ? 0 : i][0] = v0;
                    va[kU8 ? 0 : i][1] = v1;
                }
            }
        }
#pragma unroll
        for (int i = 0; i < NB_IT; ++i) {
            const int it = tid + i * 128;
            const int kk = (it & 7) + 8 * (it / (8 * NG)), g = (it >> 3) % NG;
            const int r = r0 + kk, n = n0 + 8 * g;
            const uint4 zq = make_uint4(0u, 0u, 0u, 0u);
            uint4 q0 = zq, q1 = zq, q2 = zq;
            if (r < r_hi && n < N) {
                if (b_planes) {                                   // tiled planes of B [R, ldb]: one core-matrix row
                    const uint16_t* p = b_planes + tiled_elem(plane_row((size_t)r, b_prow_npix, b_prow_batch), n, ldb);
                    q0 = __ldg(reinterpret_cast<const uint4*>(p));
                    q1 = __ldg(reinterpret_cast<const uint4*>(p + b_plane_stride));
                    q2 = __ldg(reinterpret_cast<const uint4*>(p + 2 * b_plane_stride));
                } else {
                    const float* p = b + (size_t)r * ldb + n;
                    q0 = __ldg(reinterpret_cast<const uint4*>(p));
                    if (n + 4 < N) q1 = __ldg(reinterpret_cast<const uint4*>(p + 4));
                }
            }
            vb[i][0] = q0;
            vb[i][1] = q1;
            vb[i][2] = q2;
        }
    };
    auto convert_store = [&](uint8_t* sA, uint8_t* sB) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int off;
            if (!kTransA) {
                const int rr = 8 * warp + (lane & 7) + 32 * i;
                off = kgrp * (kTcBM / 8) * 128 + (rr >> 3) * 128 + (rr & 7) * 16;
            } else {
                off = i * (kTcBM / 8) * 128 + (tid >> 3) * 128 + (tid & 7) * 16;
            }
            if (kU8) {
                *reinterpret_cast<uint4*>(sA + off) = u8x8_to_bf16(wa[kU8 ? i : 0].x, wa[kU8 ? i : 0].y);
            } else {
                const Split8 sp = split8(va[kU8 ? 0 : i][0], va[kU8 ? 0 : i][1]);
                *reinterpret_cast<uint4*>(sA + 0 * A_SPLIT + off) = sp.h;
                *reinterpret_cast<uint4*>(sA + (NA > 1 ? 1 : 0) * A_SPLIT + off) = sp.m;
                *reinterpret_cast<uint4*>(sA + (NA > 1 ? 2 : 0) * A_SPLIT + off) = sp.l;
            }
        }
#pragma unroll
        for (int i = 0; i < NB_IT; ++i) {
            const int it = tid + i * 128;
            const int kk = (it & 7) + 8 * (it / (8 * NG)), g = (it >> 3) % NG;
            const int off = (kk >> 3) * NG * 128 + g * 128 + (kk & 7) * 16;
            Split8 sp;
            if (b_planes) {
                sp.h = vb[i][0];
                sp.m = vb[i][1];
                sp.l = vb[i][2];
            } else {
                sp = split8(as_float4(vb[i][0]), as_float4(vb[i][1]));
            }
            *reinterpret_cast<uint4*>(sB + 0 * B_SPLIT + off) = sp.h;
            *reinterpret_cast<uint4*>(sB + 1 * B_SPLIT + off) = sp.m;
            *reinterpret_cast<uint4*>(sB + 2 * B_SPLIT + off) = sp.l;
        }
    };

    // accumulators of the two 64-row halves of the tile: MAIN collects a1*b1, CORR the correction products
    float acc[2][2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[h][0][j] = acc[h][1][j] = 0.f;
    constexpr int kTA = kTransA ? 1 : 0;
    if (nchunks > 0) fetch(0);
    for (int c = 0; c < nchunks; ++c) {
        const int s = c % kTcStages;
        uint8_t* sA = smem + s * STAGE;
        uint8_t* sB = sA + NA * A_SPLIT;
        // the MMAs of chunk c - 2 read this stage: at most the group of chunk c - 1 may still be in flight
        wgmma_wait<kTcStages - 1>();
        convert_store(sA, sB);
        if (c + 1 < nchunks) fetch(c + 1);
        fence_proxy_async_smem();          // generic-proxy stores -> visible to the tensor core (async proxy)
        __syncthreads();
        wgmma_fence();
        constexpr uint32_t A_LBO = (kTcBM / 8) * 128, B_LBO = (BN / 8) * 128, SBO = 128;
        const uint32_t a_base = smem_u32(sA), b_base = smem_u32(sB);
#pragma unroll
        for (int ks = 0; ks < kTcBK / 16; ++ks) {
            const uint32_t ao = ks * 2 * A_LBO, bo = ks * 2 * B_LBO;
            auto desc_b = [&](int sp) { return gmma_smem_desc(b_base + sp * B_SPLIT + bo, B_LBO, SBO); };
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                // rows 64 h .. 64 h + 63: eight 8-row core groups further (SBO = 128 bytes apart)
                auto desc_a = [&](int sp) { return gmma_smem_desc(a_base + sp * A_SPLIT + ao + h * 1024, A_LBO, SBO); };
                float* mn = acc[h][0];
                float* cr = acc[h][1];
                wgmma_tile<BN, kTA, 1>(mn, desc_a(0), desc_b(0));             // a1 b1
                wgmma_tile<BN, kTA, 1>(cr, desc_a(0), desc_b(2));             // a1 b3
                if (!kU8) {
                    wgmma_tile<BN, kTA, 1>(cr, desc_a(2), desc_b(0));         // a3 b1
                    wgmma_tile<BN, kTA, 1>(cr, desc_a(1), desc_b(1));         // a2 b2
                }
                wgmma_tile<BN, kTA, 1>(cr, desc_a(0), desc_b(1));             // a1 b2
                if (!kU8) wgmma_tile<BN, kTA, 1>(cr, desc_a(1), desc_b(0));   // a2 b1
            }
        }
        wgmma_commit();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        acc_fence<BN / 2>(acc[h][0]);
        acc_fence<BN / 2>(acc[h][1]);
    }
    __syncthreads();                       // every MMA of the CTA is complete: the stages become the result tile
    float* tile = reinterpret_cast<float*>(smem);
    constexpr int LD = BN + 4;
    store_fragment<BN>(tile, LD, 0, acc[0][0], acc[0][1]);
    store_fragment<BN>(tile, LD, 64, acc[1][0], acc[1][1]);
    __syncthreads();
    tc_epilogue<BN>(ep, tile, LD, nchunks > 0, m0, n0, M, M, N, split, kU8, a_u8_div,
                    (kU8 && kTransA) ? a.ones_col : -1);
}

}  // namespace gemm
}  // namespace cb200
