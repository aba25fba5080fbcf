// coach_b200/csrc/nn_gemm_tiled.cuh -- tensor-core GEMMs whose operands are pre-split bf16 planes in the 8x8
// core-tiled format (nn_gemm.cuh: tiled_elem): convolutions and dense layers as "multi-tap" contractions.
//
// Activations / gradients are plane matrices with rows = pixel * batch + b (pixel-major, batch-inner) and cols =
// channels; weights are stacks of [rows, n] blocks.  Two contraction shapes cover the whole learn step:
//
//   mode 0 (forward / data gradient; A is K-major):
//       C[q * B + b, n] = sum over the tap list of output pixel q, entries (a_pix, w_blk):
//                            sum_c  A[a_pix * B + b, c] * W[w_blk][c, n]
//     conv forward   : q = output pixel, one entry per kernel tap (a_pix = the input pixel under the tap)
//     conv data grad : q = INPUT pixel, entries = the taps whose output pixel exists (gather form: no zero padding, no
//                      stride-class decomposition -- invalid taps are simply not in the list), W = per-tap W^T
//     dense          : one pixel, one entry; a dense layer on a flattened conv map = one entry per pixel
//   mode 1 (weight gradient; A^T is MN-major):
//       C[t * Ca + c, n] = sum_q sum_b  A[a_pix(t, q) * B + b, c] * G[q * B + b, n]
//
// A CTA owns one 128 x BN output tile: 128 consecutive batch rows of one pixel (mode 0) or 128 rows of the stacked
// per-tap weight matrix (mode 1).  Because of the plane format every operand chunk (32 reduction indices) is a few
// contiguous runs of 128-byte core matrices, so the PRODUCER warp moves it with TMA (tensor-map boxes or 1-D bulk
// copies, completion counted in bytes on an mbarrier -- no registers, no shared-memory stores by threads).  Two
// CONSUMER warpgroups (rows 0-63 and 64-127 of the tile) issue the 3xBF16 product set of nn_gemm_tc.cuh with wgmma as
// soon as the "full" barrier of a stage flips, keep the fp32 accumulators in registers and release a stage on its
// "empty" barrier once wgmma.wait_group reports its MMAs complete.  At the end they stage the accumulators through
// shared memory and run tc_epilogue (bias / activation / derivative mask, fp32 result + planes).
//
// Tensor maps.  A plane set is a 4-D bf16 tensor (64 elements of a core | cores per 8-row group | row groups | 3
// planes); one TMA tile operation with box (64, cores, row groups, 3) fetches the hi / mid / lo planes of a whole
// operand chunk and lands them densely -- exactly the layouts below.  Mode 0 needs TWO operations per chunk (A, B),
// mode 1 one for G plus 1-D bulk copies for the A^T runs (one per tap and 8-row group: taps sit at unrelated pixels
// and the M direction must stay uniformly strided in shared memory).  Few large TMA operations keep the single
// producer warp's issue cost low.
//
// Shared-memory operand layouts (no swizzle; LBO = step between core matrices along K, SBO = along M / N):
//   A  K-major  [128 rows, 32 k] : core (rg, kg) at rg * 512 + kg * 128          LBO = 128,  SBO = 512
//   A^T MN-major [128 m,   32 k] : core (kg, mg) at kg * 2048 + mg * 128         LBO = 2048, SBO = 128
//   B  MN-major [32 k, BN n]     : core (kg, ng) at kg * (BN/8) * 128 + ng * 128 LBO = BN * 16, SBO = 128
#pragma once
#include <cuda.h>      // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint in nn.cu)

#include "nn_gemm_tc.cuh"

namespace cb200 {
namespace gemm {

struct TiledParams {
    int mode;
    int batch;                 // B, multiple of 32
    const uint16_t* a;         // planes of the A matrix [a_pixels * B, a_cols]
    long long a_stride;
    int a_cols;                // Ca, multiple of 32
    const uint16_t* b;         // mode 0: weight blocks [blocks][Ca, n];  mode 1: G [q_pixels * B, n]
    long long b_stride;
    int n;
    const int32_t* list_ptr;   // mode 0: [num_q + 1]
    const int2* list;          // mode 0: (a_pix, w_blk)
    const int32_t* a_pix;      // mode 1: [taps * num_q]
    int num_q, taps;
    int chunks_per_split;
    float a_u8_div;            // NA == 1: A holds raw uint8 values (exact in bf16); every sum is divided by this
    int bias_row;              // mode 1: also produce row M = sum over all rows of G (the bias gradient)
    int a_tma;                 // mode 1: the A^T operand of a chunk is one 5-D TMA box (tensor map tile_class[tile])
    uint8_t tile_class[64];
};

// NA = planes of the A operand: 3 (fp32 split) or 1 (uint8 values, exact: 3 products instead of 6)
// warps 0-7: two consumer warpgroups (rows 0-63 and 64-127 of the tile: wgmma, then the epilogue with half of the
// tile's columns per group of four warps), warp 8: producer
constexpr int kTlThreads = 288;
constexpr int kTlProducerWarp = 8;
constexpr int kTlConsumers = 256;

template <int BN, int NA>
struct TiledCfg {
    static constexpr int kStages = BN == 128 ? 4 : 3;
    static constexpr size_t kStageRegion = (size_t)kStages * (NA * kTcBM * kTcBK * 2 + 3 * BN * kTcBK * 2);
    static_assert(kStageRegion >= (size_t)kTcBM * (BN + 4) * sizeof(float), "result tile overlays the stages");
    static constexpr size_t kSmemBytes = kStageRegion + 128 + 1024;
};

__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], "
        "[%7];" ::"r"(smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], "
        "[%6];" ::"r"(smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kTlConsumers) : "memory"); }

// tmA: planes of A with box (64, 4, 16, NA) (mode 0 only); tmB: planes of the B operand with box (64, BN / 8, 4, 3)
// kCat (mode 0, BN <= 64, row-group interleaved B planes): the B box lands as [k-group][plane][column core]; each
// plane is then an MN-major operand with k-group stride 3 * (BN / 8) * 128 bytes, and the six narrow products are
// issued on it as on separate planes.  The interleaved operand would also allow three wide MMAs on one MAIN | CA | CB
// fragment (a1 x [b1|b2|b3] at N = 3 BN, a2 x [b1|b2], a3 x b1), reading each A plane once per k-step; measured on an
// H100 SXM (700 W) in the DQN step that form took 760 us of tiled-GEMM time per step against 724-727 us for the six
// narrow wgmma, so it is not used.
template <int BN, bool kTransA, int NA, bool kCat = false>
__global__ void __launch_bounds__(kTlThreads) gemm_tc_tiled_kernel(const __grid_constant__ CUtensorMap tmA,
                                                            const __grid_constant__ CUtensorMap tmB,
                                                            const __grid_constant__ CUtensorMap tmA1,
                                                            const __grid_constant__ CUtensorMap tmA2, TiledParams tp,
                                                            EpiParams ep, int M) {
    constexpr int S = TiledCfg<BN, NA>::kStages;
    constexpr int A_SPLIT = kTcBM * kTcBK * 2;            // 8 KB per plane
    constexpr int B_SPLIT = BN * kTcBK * 2;
    constexpr int STAGE = NA * A_SPLIT + 3 * B_SPLIT;
    constexpr int B_KG = (BN / 8) * 128;                  // bytes of one k-group (8 reduction rows) of the B tile
    constexpr size_t REGION = TiledCfg<BN, NA>::kStageRegion;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + REGION);       // [S]
    uint64_t* empty_bar = full_bar + S;                                    // [S]
    float* bias_part = reinterpret_cast<float*>(smem + REGION + 128);      // [256] partial column sums (bias row)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // Bias gradient (mode 1): the CTAs of the first M tile also form sum_rows G[row, :] -- the consumer threads add
    // the three exact bf16 planes of every G chunk in fp32 while the tensor core works on it.  This replaces a
    // separate column-sum pass over dY.
    const bool bias_cta = kTransA && tp.bias_row != 0 && blockIdx.x == 0;
    static_assert(!kCat || (!kTransA && BN <= 64), "kCat: mode 0, BN <= 64");
    const int B = tp.batch, Ca = tp.a_cols, N = tp.n;
    const int n0 = blockIdx.y * BN;
    const int split = blockIdx.z;

    // ---- tile decode ----------------------------------------------------------------------------------------------
    int q = 0, b0 = 0, m0, m_end, total, list_lo = 0;
    const int kc_per = Ca / kTcBK;                        // mode 0: chunks per tap
    const int bc_per = B / kTcBK;                         // mode 1: chunks per pixel
    if (!kTransA) {
        const int tiles_per_q = (B + kTcBM - 1) / kTcBM;
        q = blockIdx.x / tiles_per_q;
        b0 = (blockIdx.x % tiles_per_q) * kTcBM;
        m0 = q * B + b0;
        m_end = q * B + B;
        list_lo = __ldg(tp.list_ptr + q);
        total = (__ldg(tp.list_ptr + q + 1) - list_lo) * kc_per;
    } else {
        m0 = blockIdx.x * kTcBM;
        m_end = M - (tp.bias_row ? 1 : 0);       // the bias row is not part of any tile
        total = tp.num_q * bc_per;
    }
    const int c_lo = split * tp.chunks_per_split;
    const int c_hi = min(total, c_lo + tp.chunks_per_split);
    const int nchunks = max(0, c_hi - c_lo);

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_bar + s, 1);
            mbar_init(empty_bar + s, kTlConsumers / 32);   // one elected lane of each consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == kTlProducerWarp) {
        // ================= producer: bulk copies of the operand cores into the stage ring =========================
        // mode 1: taps covered by this M tile, and the channel range inside a tap
        const int taps_in_tile = kTransA ? (Ca >= kTcBM ? 1 : min(kTcBM / Ca, tp.taps - m0 / Ca)) : 0;
        const int t0 = kTransA ? m0 / Ca : 0;
        const int cw = kTransA ? min(Ca, kTcBM) : 0;                           // channels per tap inside the tile
        const int c0 = kTransA ? m0 % Ca : 0;
        // a tensor-map box always delivers (and counts) its full size, rows past the batch included
        const bool a_tma = kTransA && tp.a_tma != 0;
        const int a_cls = a_tma ? tp.tile_class[blockIdx.x & 63] : 0;
        const CUtensorMap* a_map = a_cls == 0 ? &tmA : (a_cls == 1 ? &tmA1 : &tmA2);
        const uint32_t a_bytes = (kTransA && !a_tma) ? (uint32_t)(taps_in_tile * 4 * (cw / 8) * 128) : (uint32_t)A_SPLIT;
        const uint32_t tx_bytes = (uint32_t)NA * a_bytes + 3u * (uint32_t)B_SPLIT;
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
            if (!kTransA || a_tma) asm volatile("prefetch.tensormap [%0];" ::"l"(a_map) : "memory");
        }
        for (int j = 0; j < nchunks; ++j) {
            const int s = j % S, u = j / S;
            if (u > 0) mbar_wait(empty_bar + s, (uint32_t)((u - 1) & 1));      // MMAs that read this stage are done
            uint8_t* sA = smem + s * STAGE;
            uint8_t* sB = sA + NA * A_SPLIT;
            uint64_t* bar = full_bar + s;
            if (lane == 0) mbar_expect_tx(bar, tx_bytes);
            __syncwarp();
            const int cj = c_lo + j;
            if (!kTransA) {
                if (lane == 0) {
                    const int e = cj / kc_per, kc = cj % kc_per;
                    const int2 ent = __ldg(tp.list + list_lo + e);
                    tma_load_4d(sA, &tmA, 0, kc * 4, (int)(((size_t)ent.x * B + b0) >> 3), 0, bar);
                    if (kCat) tma_load_4d(sB, &tmB, 0, n0 >> 3, 0, (ent.y * Ca + kc * kTcBK) >> 3, bar);
                    else tma_load_4d(sB, &tmB, 0, n0 >> 3, (ent.y * Ca + kc * kTcBK) >> 3, 0, bar);
                }
            } else {
                const int qq = cj / bc_per, bc = cj % bc_per;
                if (lane == 0) tma_load_4d(sB, &tmB, 0, n0 >> 3, (int)(((size_t)qq * B + (size_t)bc * kTcBK) >> 3), 0, bar);
                if (a_tma) {
                    // A^T: the taps of the tile sit a constant number of pixels apart -- one 5-D box (64 | cores | taps
                    // | 4 row groups | planes) lands as [plane][k-group][tap][core], the layout of the bulk path below
                    if (lane == 0) {
                        const int apix = __ldg(tp.a_pix + (size_t)t0 * tp.num_q + qq);
                        tma_load_5d(sA, a_map, 0, c0 >> 3, 0, (int)(((size_t)apix * B + (size_t)bc * kTcBK) >> 3), 0, bar);
                    }
                    continue;
                }
                // A^T: per tap of the tile, 4 k-groups (8 batch rows each) x a run of cw / 8 cores
                for (int idx = lane; idx < NA * 4 * taps_in_tile; idx += 32) {
                    const int p = idx / (4 * taps_in_tile), r = idx % (4 * taps_in_tile);
                    const int tt = r >> 2, kg = r & 3;
                    const int apix = __ldg(tp.a_pix + (size_t)(t0 + tt) * tp.num_q + qq);
                    const size_t rg = (((size_t)apix * B + (size_t)bc * kTcBK) >> 3) + kg;
                    bulk_g2s(sA + p * A_SPLIT + kg * 2048 + tt * (Ca >> 3) * 128,
                             tp.a + p * tp.a_stride + (rg * (size_t)(Ca >> 3) + (size_t)(c0 >> 3)) * 64,
                             (uint32_t)((cw >> 3) * 128), bar);
                }
            }
        }
    } else {
        // ================= consumers: warpgroup g computes rows 64 g .. 64 g + 63 of the tile =====================
        const int g = warp >> 2;
        constexpr int kTA = kTransA ? 1 : 0;
        // A K-major  [128 rows, 32 k]: core (rg, kg) at rg * 512 + kg * 128   -> rows 64 g start 8 * 512 g further
        // A^T MN-major [128 m, 32 k]: core (kg, mg) at kg * 2048 + mg * 128   -> rows 64 g start 8 * 128 g further
        constexpr uint32_t A_LBO = kTransA ? 2048u : 128u, A_SBO = kTransA ? 128u : 512u;
        constexpr uint32_t A_KS = kTransA ? 2u * 2048u : 256u;                 // bytes per k16 step
        const uint32_t a_half = (uint32_t)g * 8u * A_SBO;
        // B MN-major: k-group stride B_KG (plane stride B_SPLIT), or 3 * B_KG (plane stride B_KG) when interleaved
        constexpr uint32_t B_LBO = kCat ? 3u * (uint32_t)B_KG : (uint32_t)B_KG;
        constexpr uint32_t B_PLANE = kCat ? (uint32_t)B_KG : (uint32_t)B_SPLIT;
        const uint32_t smem_base = smem_u32(smem);
        float mn[BN / 2], cr[BN / 2];
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) mn[j] = cr[j] = 0.f;
        // bias row: thread t sums column t % BN over the reduction rows kk = t / BN (mod 256 / BN)
        float bsum = 0.f;
        const int bcol = tid % BN, brow0 = tid / BN;
        for (int j = 0; j < nchunks; ++j) {
            const int s = j % S, u = j / S;
            mbar_wait(full_bar + s, (uint32_t)(u & 1));                        // the bulk copies of this stage landed
            const uint32_t a_base = smem_base + s * STAGE + a_half, b_base = smem_base + s * STAGE + NA * A_SPLIT;
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < kTcBK / 16; ++ks) {
                const uint64_t a0 = gmma_smem_desc(a_base + ks * A_KS, A_LBO, A_SBO);
                const uint64_t a1 = a0 + (A_SPLIT >> 4), a2 = a0 + 2 * (A_SPLIT >> 4);
                const uint64_t b0d = gmma_smem_desc(b_base + ks * 2u * B_LBO, B_LBO, 128u);
                const uint64_t b1 = b0d + (B_PLANE >> 4), b2 = b0d + 2 * (B_PLANE >> 4);
                wgmma_tile<BN, kTA, 1>(mn, a0, b0d);           // a1 b1
                wgmma_tile<BN, kTA, 1>(cr, a0, b2);            // a1 b3
                if (NA == 3) {
                    wgmma_tile<BN, kTA, 1>(cr, a2, b0d);       // a3 b1
                    wgmma_tile<BN, kTA, 1>(cr, a1, b1);        // a2 b2
                }
                wgmma_tile<BN, kTA, 1>(cr, a0, b1);            // a1 b2
                if (NA == 3) wgmma_tile<BN, kTA, 1>(cr, a1, b0d);   // a2 b1
            }
            wgmma_commit();
            if (bias_cta) {
                const uint16_t* sb = reinterpret_cast<const uint16_t*>(smem + s * STAGE + NA * A_SPLIT);
                for (int kk = brow0; kk < kTcBK; kk += kTlConsumers / BN) {
                    const int e = ((kk >> 3) * B_KG + (bcol >> 3) * 128 + (kk & 7) * 16) / 2 + (bcol & 7);
                    const float g1 = __uint_as_float((uint32_t)sb[e] << 16);
                    const float g2 = __uint_as_float((uint32_t)sb[e + B_SPLIT / 2] << 16);
                    const float g3 = __uint_as_float((uint32_t)sb[e + B_SPLIT] << 16);
                    bsum += g1 + g2 + g3;
                }
            }
            // the MMAs of chunk j - 1 are complete: release its stage
            wgmma_wait<1>();
            __syncwarp();
            if (j > 0 && lane == 0)
                asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(empty_bar + (j - 1) % S))
                             : "memory");
        }
        wgmma_wait<0>();
        acc_fence<BN / 2>(mn);
        acc_fence<BN / 2>(cr);
        consumer_sync();                   // every MMA of the tile is complete: the stages become the result tile
        float* tile = reinterpret_cast<float*>(smem);
        constexpr int LD = BN + 4;
        store_fragment<BN>(tile, LD, 64 * g, mn, cr);
        if (bias_cta) bias_part[tid] = bsum;
        consumer_sync();
        {
            const int half = warp >> 2;                        // warps 0-3: low half of the columns, 4-7: high half
            tc_epilogue<BN>(ep, tile, LD, nchunks > 0, m0, n0, M, m_end, N, split, NA == 1, tp.a_u8_div, -1,
                            half * (BN / 2), half * (BN / 2) + BN / 2);
        }
        if (bias_cta && tid < BN) {
            // row `m_end` (= taps * Ca) of the result
            const int n = n0 + tid;
            float v = 0.f;
            for (int r = 0; r < kTlConsumers / BN; ++r) v += bias_part[r * BN + tid];
            if (n < N) {
                if (ep.splits > 1)
                    ep.partial[((size_t)split * M + m_end) * N + n] = v;
                else
                    epilogue_store(ep, m_end, n, v);
            }
        }
    }
}

}  // namespace gemm
}  // namespace cb200
