// coach_b200/csrc/nn_gemm.cuh -- fp32 tiled "gather-GEMM" core.
//
// Every dense contraction of the learn step -- conv forward as implicit GEMM over NHWC, conv weight / data gradients,
// dense forward / backward -- is one primitive:
//
//        C[m, n] (+)= sum_r A(m, r) * B(r, n)          A(m, r) = a_src[ a_rowoff[m] + a_coloff[r] ]
//
// i.e. the A operand is addressed through two small index tables (one entry per logical row, one per reduction
// index), which expresses im2col-on-the-fly (row = output pixel, col = (ky,kx,c) tap), the transposed convolution in
// gather form (row = input pixel, col = (tap, n); out-of-map taps masked through a_rowinfo / a_colinfo), plain dense
// matrices (rowoff = m*lda, coloff = r) and, with `a_transposed`, A^T for the weight gradients.  The tables are
// built once per layer geometry by the host code (coach_b200/architectures/layers.py).  B is always row-major
// [R, N]; the epilogue adds bias, applies the activation or an activation-derivative mask, remaps output rows
// (c_rowmap) or writes split-R partial sums that a second deterministic kernel reduces in fixed order.
//
// This file: the fp32 FFMA (CUDA-core) kernels, the shared epilogue and the plane format.  The reference trains in
// fp32 and the parity bar is 1e-5 relative, which TF32 / BF16 tensor-core operands only meet with 3-way operand
// splitting: that path is nn_gemm_tc.cuh (operands staged by the threads) and nn_gemm_tiled*.cuh (pre-split planes
// fed by TMA); the kernels here serve the shapes without a tensor-core form and the small batches.
//
// Tile: BM x BN outputs per CTA, reduction chunk BK, TM x TN outputs per thread.  Shared tiles are reduction-major
// (As[BK][BM], Bs[BK][BN]) and double buffered: operands of chunk c+1 are fetched into registers before the FMAs of
// chunk c and committed to the other buffer afterwards (one __syncthreads per chunk).
#pragma once
#include "common.cuh"

namespace cb200 {
namespace gemm {

template <int BM_, int BN_, int BK_, int TM_, int TN_>
struct Cfg {
    static constexpr int BM = BM_, BN = BN_, BK = BK_, TM = TM_, TN = TN_;
    static constexpr int TX = BN / TN, TY = BM / TM, T = TX * TY;
    static_assert(TM == 4 || TM == 8, "TM must be 4 or 8");
    static_assert(TN == 4 || TN == 8, "TN must be 4 or 8");
    static_assert(BM % TM == 0 && BN % TN == 0, "tile shape");
    static_assert((BM * BK) % T == 0 && (BN * BK) % T == 0, "loader shape");
};

// row / column owned by a thread: an 8-wide fragment is split in two groups of 4, half a tile apart, so that a
// quarter-warp reads 8 consecutive float4 from shared memory (no bank conflicts).
template <int BX, int TXN>
__device__ __forceinline__ int frag_index(int t, int i) {
    if (TXN == 8) return (i < 4) ? (t * 4 + i) : (BX / 2 + t * 4 + (i - 4));
    return t * 4 + i;
}

template <class C>
__device__ __forceinline__ void mma_chunk(const float* __restrict__ As, const float* __restrict__ Bs,
                                          float (&acc)[C::TM][C::TN], int ty, int tx) {
#pragma unroll
    for (int k = 0; k < C::BK; ++k) {
        float a[C::TM], b[C::TN];
        const float4 a0 = *reinterpret_cast<const float4*>(As + k * C::BM + ty * 4);
        a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
        if (C::TM == 8) {
            const float4 a1 = *reinterpret_cast<const float4*>(As + k * C::BM + C::BM / 2 + ty * 4);
            a[C::TM - 4] = a1.x; a[C::TM - 3] = a1.y; a[C::TM - 2] = a1.z; a[C::TM - 1] = a1.w;
        }
        const float4 b0 = *reinterpret_cast<const float4*>(Bs + k * C::BN + tx * 4);
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
        if (C::TN == 8) {
            const float4 b1 = *reinterpret_cast<const float4*>(Bs + k * C::BN + C::BN / 2 + tx * 4);
            b[C::TN - 4] = b1.x; b[C::TN - 3] = b1.y; b[C::TN - 2] = b1.z; b[C::TN - 1] = b1.w;
        }
#pragma unroll
        for (int i = 0; i < C::TM; ++i)
#pragma unroll
            for (int j = 0; j < C::TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
}

// A operand description (device copy of the relevant cb200_gemm_desc fields)
struct ASrc {
    const void* src;
    const float* lut;            // non-null: src is uint8 and value = lut[byte]   (x / 255 table, embedder.py:103-104)
    const int32_t* rowoff;       // [rows]
    const int32_t* coloff;       // [cols]
    const int32_t* rowinfo;      // optional (i << 16 | j) per row      } transposed-conv tap validity:
    const int32_t* colinfo;      // optional (a << 16 | b) per col      } 0 <= i-a < oh  and  0 <= j-b < ow
    int oh, ow;
    int rows, cols;              // logical extent of A (rows = m index, cols = r index) BEFORE any transposition
    __device__ __forceinline__ float at(int m, int r) const {
        if (m >= rows || r >= cols) return 0.f;
        if (rowinfo) {
            const int ri = __ldg(rowinfo + m), ci = __ldg(colinfo + r);
            const int y = (ri >> 16) - (ci >> 16), x = (ri & 0xffff) - (ci & 0xffff);
            if (y < 0 || y >= oh || x < 0 || x >= ow) return 0.f;
        }
        const int off = __ldg(rowoff + m) + __ldg(coloff + r);
        if (lut) return __ldg(lut + static_cast<const uint8_t*>(src)[off]);
        return __ldg(static_cast<const float*>(src) + off);
    }
};

template <class C, bool kTransposedA>
struct ALoader {
    // kTransposedA == false: tile element (row mm, red kk) = A(m0 + mm, r0 + kk); lanes walk kk (contiguous in memory)
    // kTransposedA == true : tile element (row mm, red kk) = A(r0 + kk, m0 + mm); lanes walk mm (contiguous in memory)
    static constexpr int ELEMS = C::BM * C::BK / C::T;
    ASrc a;
    float regs[ELEMS];
    __device__ __forceinline__ void coords(int idx, int& mm, int& kk) const {
        if (!kTransposedA) {
            kk = idx % C::BK;
            mm = idx / C::BK;
        } else {
            mm = idx % C::BM;
            kk = idx / C::BM;
        }
    }
    __device__ __forceinline__ void fetch(int m0, int r0, int r_hi, int tid) {
#pragma unroll
        for (int e = 0; e < ELEMS; ++e) {
            int mm, kk;
            coords(tid + e * C::T, mm, kk);
            const int r = r0 + kk;
            float v = 0.f;
            if (r < r_hi) v = kTransposedA ? a.at(r, m0 + mm) : a.at(m0 + mm, r);
            regs[e] = v;
        }
    }
    __device__ __forceinline__ void commit(float* As, int tid) const {
#pragma unroll
        for (int e = 0; e < ELEMS; ++e) {
            int mm, kk;
            coords(tid + e * C::T, mm, kk);
            As[kk * C::BM + mm] = regs[e];
        }
    }
};

// B[R, N] row-major with leading dimension ldb
template <class C>
struct BLoader {
    static constexpr int ELEMS = C::BN * C::BK / C::T;
    const float* b;
    int N, ldb;
    float regs[ELEMS];
    __device__ __forceinline__ void fetch(int n0, int r0, int r_hi, int tid) {
#pragma unroll
        for (int e = 0; e < ELEMS; ++e) {
            const int idx = tid + e * C::T;
            const int nn = idx % C::BN, kk = idx / C::BN;
            const int r = r0 + kk, n = n0 + nn;
            regs[e] = (r < r_hi && n < N) ? __ldg(b + (size_t)r * ldb + n) : 0.f;
        }
    }
    __device__ __forceinline__ void commit(float* Bs, int tid) const {
#pragma unroll
        for (int e = 0; e < ELEMS; ++e) Bs[tid + e * C::T] = regs[e];   // idx = kk*BN + nn already
    }
};

// ---- epilogue -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == CB200_ACT_RELU) return v > 0.f ? v : 0.f;
    if (act == CB200_ACT_TANH) return tanhf(v);
    return v;
}
// derivative of the activation expressed through its OUTPUT y (relu: y > 0; tanh: 1 - y^2)
__device__ __forceinline__ float act_grad_from_output(float y, int act) {
    if (act == CB200_ACT_RELU) return y > 0.f ? 1.f : 0.f;
    if (act == CB200_ACT_TANH) return 1.f - y * y;
    return 1.f;
}

struct EpiParams {
    float* c;                  // [M(rowmapped), ldc]
    int ldc;
    const float* bias;         // [N] or nullptr
    int act;
    const float* mask_y;       // same indexing as c, or nullptr:  c = v * act'(mask_y)
    int mask_act;
    const int32_t* c_rowmap;   // optional output-row remap
    float* partial;            // splits > 1: raw partial sums [splits][M][N]
    int splits;
    int accumulate;            // c += v instead of c = v (after bias/act/mask); used by multi-class data gradients
    uint16_t* c_planes;        // optional bf16 hi / mid / lo planes of c in the 8x8 core-tiled format (tiled_elem)
    int64_t c_plane_stride;    // elements between planes
    int c_plane_cols;          // columns of the tiled plane matrix (= n of this GEMM)
    int c_prow_npix;           // > 0: output row m = b * npix + q  (NHWC order) lands in plane row q * batch + b
    int c_prow_batch;          //      (pixel-major, batch-inner order of the planes); 0: plane row = m
    const uint16_t* mask_planes;   // optional: the activation whose derivative masks the result, given as tiled planes of
    int64_t mask_plane_stride;     // the SAME geometry as the result (replaces mask_y: no fp32 copy of it is needed)
};

// activation output y rebuilt from its planes for the derivative mask: relu only asks y > 0, which the hi plane answers
// (hi == 0 with y > 0 would need y < 2^-133); tanh needs the value
__device__ __forceinline__ float mask_from_planes(const uint16_t* p, int64_t stride, int act) {
    const float hi = __uint_as_float((uint32_t)p[0] << 16);
    if (act == CB200_ACT_RELU) return hi;
    return (hi + __uint_as_float((uint32_t)p[stride] << 16)) + __uint_as_float((uint32_t)p[2 * stride] << 16);
}

// Plane format.  A logical [rows, cols] matrix (both multiples of 8) is stored as 8x8 "core matrices" of 128 contiguous
// bytes, core (r / 8, c / 8) at ((r / 8) * (cols / 8) + c / 8) * 64 elements, element (r % 8, c % 8) inside it
// row-major.  This is exactly the unit the wgmma shared-memory descriptors address without swizzling (K-major A with
// M = rows, K = cols; MN-major A^T / B with K = rows, MN = cols all read the same 128 bytes), so any operand tile is a
// handful of contiguous runs of cores that a 1-D bulk copy (TMA) moves without touching a register.
// Activations / gradients use rows = pixel * batch + b (pixel-major, batch-inner), cols = channels: the im2col tile of
// one tap is then 128 consecutive rows of the plane matrix.
__device__ __forceinline__ size_t tiled_elem(size_t prow, int col, int pcols) {
    return ((prow >> 3) * (size_t)(pcols >> 3) + (size_t)(col >> 3)) * 64 + (prow & 7) * 8 + (col & 7);
}
// "Row-group interleaved" planes (B operands of the N <= 64 forward / data-gradient GEMMs): the three planes of one
// 8-row group sit next to each other -- (row group | plane | column core | 64) -- so that ONE TMA box delivers a
// [k-group][plane][column core] tile, i.e. a single MN-major operand [32 k, 3 * n] = [b1 | b2 | b3] fetched with one
// box instead of three (nn_gemm_tiled.cuh, kCat).  Plane stride argument -1.
__device__ __forceinline__ size_t tiled_elem_il(size_t prow, int col, int pcols, int plane) {
    return (((prow >> 3) * 3 + (size_t)plane) * (size_t)(pcols >> 3) + (size_t)(col >> 3)) * 64 + (prow & 7) * 8 + (col & 7);
}
__device__ __forceinline__ size_t plane_row(size_t m, int npix, int batch) {
    return npix > 0 ? (m % (size_t)npix) * (size_t)batch + m / (size_t)npix : m;
}

// Exact 3-way bf16 split of an fp32 value (truncation): x == hi + mid + lo, each the upper half-word of an fp32
// (exact for |x| >= 2^-110 and for 0; tinier values lose less than 2^-133, tests/test_tiled_host.py).
// The tensor-core GEMM (nn_gemm_tc.cuh) consumes operands in this form; producers that know their output feeds another
// GEMM write the planes next to the fp32 result so that consumers need no conversion work.
__device__ __forceinline__ void split3(float x, uint16_t& h, uint16_t& m, uint16_t& l) {
    const uint32_t hb = __float_as_uint(x) & 0xffff0000u;
    const float r1 = x - __uint_as_float(hb);
    const uint32_t mb = __float_as_uint(r1) & 0xffff0000u;
    const uint32_t lb = __float_as_uint(r1 - __uint_as_float(mb));
    h = (uint16_t)(hb >> 16);
    m = (uint16_t)(mb >> 16);
    l = (uint16_t)(lb >> 16);
}

__device__ __forceinline__ void epilogue_store(const EpiParams& ep, int m, int n, float v) {
    const size_t row = ep.c_rowmap ? (size_t)__ldg(ep.c_rowmap + m) : (size_t)m;
    if (ep.bias) v += __ldg(ep.bias + n);
    v = apply_act(v, ep.act);
    if (ep.mask_planes)
        v *= act_grad_from_output(
            mask_from_planes(ep.mask_planes + tiled_elem(plane_row((size_t)m, ep.c_prow_npix, ep.c_prow_batch), n,
                                                         ep.c_plane_cols),
                             ep.mask_plane_stride, ep.mask_act),
            ep.mask_act);
    else if (ep.mask_y) v *= act_grad_from_output(ep.mask_y[row * ep.ldc + n], ep.mask_act);
    if (ep.c) {             // c may be omitted when only the planes of the result are consumed (forward-only networks)
        float* dst = ep.c + row * ep.ldc + n;
        if (ep.accumulate) v += *dst;
        *dst = v;
    }
    if (ep.c_planes) {
        uint16_t* p = ep.c_planes + tiled_elem(plane_row((size_t)m, ep.c_prow_npix, ep.c_prow_batch), n, ep.c_plane_cols);
        split3(v, p[0], p[ep.c_plane_stride], p[2 * ep.c_plane_stride]);
    }
}

template <class C, bool kTransposedA>
__global__ void __launch_bounds__(C::T) gemm_kernel(ALoader<C, kTransposedA> al, BLoader<C> bl, EpiParams ep, int M,
                                                    int N, int R, int r_per_split) {
    __shared__ __align__(16) float As[2][C::BK * C::BM];
    __shared__ __align__(16) float Bs[2][C::BK * C::BN];
    const int tid = threadIdx.x;
    const int tx = tid % C::TX, ty = tid / C::TX;
    const int m0 = blockIdx.x * C::BM, n0 = blockIdx.y * C::BN;
    const int split = blockIdx.z;
    const int r_lo = split * r_per_split;
    const int r_hi = min(R, r_lo + r_per_split);
    float acc[C::TM][C::TN];
#pragma unroll
    for (int i = 0; i < C::TM; ++i)
#pragma unroll
        for (int j = 0; j < C::TN; ++j) acc[i][j] = 0.f;

    const int nchunks = (r_hi - r_lo + C::BK - 1) / C::BK;
    if (nchunks > 0) {
        al.fetch(m0, r_lo, r_hi, tid);
        bl.fetch(n0, r_lo, r_hi, tid);
        al.commit(As[0], tid);
        bl.commit(Bs[0], tid);
    }
    __syncthreads();
    for (int c = 0; c < nchunks; ++c) {
        const int cur = c & 1;
        if (c + 1 < nchunks) {
            al.fetch(m0, r_lo + (c + 1) * C::BK, r_hi, tid);
            bl.fetch(n0, r_lo + (c + 1) * C::BK, r_hi, tid);
        }
        mma_chunk<C>(As[cur], Bs[cur], acc, ty, tx);
        if (c + 1 < nchunks) {
            al.commit(As[cur ^ 1], tid);
            bl.commit(Bs[cur ^ 1], tid);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < C::TM; ++i) {
        const int m = m0 + frag_index<C::BM, C::TM>(ty, i);
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < C::TN; ++j) {
            const int n = n0 + frag_index<C::BN, C::TN>(tx, j);
            if (n >= N) continue;
            if (ep.splits > 1)
                ep.partial[((size_t)split * M + m) * N + n] = acc[i][j];
            else
                epilogue_store(ep, m, n, acc[i][j]);
        }
    }
}

// deterministic split reduction: fixed order over the split index, then the normal epilogue.
// kVec (M * N % 4 == 0, N % 4 == 0): four consecutive outputs per thread through 128-bit loads of the partials.
template <bool kVec>
__global__ void __launch_bounds__(256) split_reduce_kernel(EpiParams ep, int M, int N) {
    const int64_t total = (int64_t)M * N;
    if (kVec) {
        const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (i >= total) return;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < ep.splits; ++s) {
            const float4 p = *reinterpret_cast<const float4*>(ep.partial + (size_t)s * total + i);
            v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
        }
        const int m = (int)(i / N), n = (int)(i % N);
        epilogue_store(ep, m, n, v.x);
        epilogue_store(ep, m, n + 1, v.y);
        epilogue_store(ep, m, n + 2, v.z);
        epilogue_store(ep, m, n + 3, v.w);
    } else {
        const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= total) return;
        float v = 0.f;
        for (int s = 0; s < ep.splits; ++s) v += ep.partial[(size_t)s * total + i];
        epilogue_store(ep, (int)(i / N), (int)(i % N), v);
    }
}
// many splits (weight gradients: 56 ... 291 partial tiles): a block owns 32 consecutive outputs; its 8 warps walk the
// splits 8 apart with fully coalesced 128-byte reads, and the 8 partial sums are folded in a fixed order --
// deterministic, but a different association than the serial kernels, selected only by the split count.
__global__ void __launch_bounds__(256) split_reduce_wide_kernel(EpiParams ep, int M, int N) {
    __shared__ float red[8][32];
    const int64_t total = (int64_t)M * N;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * 32 + lane;
    float v = 0.f;
    if (i < total)
        for (int s = w; s < ep.splits; s += 8) v += ep.partial[(size_t)s * total + i];
    red[w][lane] = v;
    __syncthreads();
    if (w == 0 && i < total) {
        for (int k = 1; k < 8; ++k) v += red[k][lane];
        epilogue_store(ep, (int)(i / N), (int)(i % N), v);
    }
}

inline void launch_split_reduce(const EpiParams& ep, int M, int N, cudaStream_t st) {
    const int64_t total = (int64_t)M * N;
    if (ep.splits >= 16 && total <= (1 << 16)) {
        set_dispatch_reduce("reduce_wide");
        split_reduce_wide_kernel<<<(unsigned)((total + 31) / 32), 256, 0, st>>>(ep, M, N);
    } else if (N % 4 == 0 && total % 4 == 0 && (reinterpret_cast<uintptr_t>(ep.partial) & 15) == 0) {
        set_dispatch_reduce("reduce_vec");
        split_reduce_kernel<true><<<(unsigned)((total / 4 + 255) / 256), 256, 0, st>>>(ep, M, N);
    } else {
        set_dispatch_reduce("reduce_scalar");
        split_reduce_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ep, M, N);
    }
}

}  // namespace gemm
}  // namespace cb200
