// coach_b200/csrc/nn.cu -- C-ABI entry points of the dense contractions of the learn step (see nn_gemm.cuh).
#include <string>

#include "nn_gemm_skinny.cuh"
#include "nn_gemm_tiled.cuh"

namespace cb200 {
namespace gemm {

// kernel names for cb200_last_dispatch, built once per template instantiation
static std::string kernel_name(const char* kind, int a, int b, const char* c, const char* d = nullptr) {
    char s[64];
    if (b > 0) snprintf(s, sizeof(s), "%s<%d,%d,%s%s%s>", kind, a, b, c, d ? "," : "", d ? d : "");
    else snprintf(s, sizeof(s), "%s<%d,%s%s%s>", kind, a, c, d ? "," : "", d ? d : "");
    return s;
}

using CfgN64 = Cfg<128, 64, 16, 8, 8>;   // 128 threads, 8x8 per thread
using CfgN32 = Cfg<128, 32, 16, 8, 4>;   // 128 threads, 8x4 per thread
using CfgSmall = Cfg<32, 32, 16, 4, 4>;  // 64 threads: small-batch MLPs

static EpiParams make_epi(const cb200_gemm_desc& d, int splits) {
    return EpiParams{d.c,        d.ldc,       d.bias, d.act,        d.mask_y,
                     d.mask_act, d.c_rowmap,  d.workspace, splits,  d.accumulate,
                     static_cast<uint16_t*>(d.c_planes), d.c_plane_stride, d.c_plane_cols, d.c_prow_npix,
                     d.c_prow_batch, nullptr, 0};
}

template <class C, bool kT>
static void launch(const cb200_gemm_desc& d, int M, int R, int splits, int r_per_split, cudaStream_t st) {
    ALoader<C, kT> al;
    al.a.src = d.a_src;
    al.a.lut = d.a_lut;
    al.a.rowoff = d.a_rowoff;
    al.a.coloff = d.a_coloff;
    al.a.rowinfo = d.a_rowinfo;
    al.a.colinfo = d.a_colinfo;
    al.a.oh = d.a_oh;
    al.a.ow = d.a_ow;
    al.a.rows = d.a_rows;
    al.a.cols = d.a_cols;
    BLoader<C> bl;
    bl.b = d.b;
    bl.N = d.n;
    bl.ldb = d.ldb;
    const EpiParams ep = make_epi(d, splits);
    static const std::string name = kernel_name("ffma", C::BM, C::BN, kT ? "T" : "N");
    set_dispatch(name.c_str());
    dim3 grid((M + C::BM - 1) / C::BM, (d.n + C::BN - 1) / C::BN, splits);
    gemm_kernel<C, kT><<<grid, C::T, 0, st>>>(al, bl, ep, M, d.n, R, r_per_split);
    count_launch();
    if (splits > 1) {
        launch_split_reduce(ep, M, d.n, st);
        count_launch();
    }
}

template <class C, bool kT>
static void launch_fast(const cb200_gemm_desc& d, int M, int R, int splits, int r_per_split, cudaStream_t st) {
    FastA a;
    a.src = d.a_src;
    a.lut = d.a_lut;
    a.rowoff = d.a_rowoff;
    a.coloff = d.a_coloff;
    a.rowinfo = d.a_rowinfo;
    a.colinfo = d.a_colinfo;
    a.oh = d.a_oh;
    a.ow = d.a_ow;
    a.rows = d.a_rows;
    a.cols = d.a_cols;
    a.ones_col = (kT && d.a_ones_col) ? d.a_cols : -1;
    const EpiParams ep = make_epi(d, splits);
    static const std::string name = kernel_name("fast", C::BM, C::BN, kT ? "T" : "N");
    set_dispatch(name.c_str());
    dim3 grid((M + C::BM - 1) / C::BM, (d.n + C::BN - 1) / C::BN, splits);
    gemm_fast_kernel<C, kT><<<grid, C::T, 0, st>>>(a, d.b, d.ldb, ep, M, d.n, R, r_per_split);
    count_launch();
    if (splits > 1) {
        launch_split_reduce(ep, M, d.n, st);
        count_launch();
    }
}

template <int BN, bool kT, bool kU8>
static int launch_tc(const cb200_gemm_desc& d, int M, int R, int splits, int r_per_split, cudaStream_t st) {
    FastA a;
    a.src = d.a_src;
    a.lut = d.a_lut;
    a.rowoff = d.a_rowoff;
    a.coloff = d.a_coloff;
    a.rowinfo = d.a_rowinfo;
    a.colinfo = d.a_colinfo;
    a.oh = d.a_oh;
    a.ow = d.a_ow;
    a.rows = d.a_rows;
    a.cols = d.a_cols;
    a.ones_col = (kT && d.a_ones_col) ? d.a_cols : -1;
    const EpiParams ep = make_epi(d, splits);
    constexpr size_t smem = tc_smem_bytes<BN, kU8>();
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(gemm_tc_kernel<BN, kT, kU8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
            cudaSuccess)
            return -1;
        configured = true;
    }
    static const std::string names[2] = {kernel_name("tc", BN, 0, kT ? "T" : "N", kU8 ? "u8" : "f32"),
                                         kernel_name("tc", BN, 0, kT ? "T" : "N", "lut")};
    set_dispatch(names[!kU8 && d.a_lut ? 1 : 0].c_str());
    dim3 grid((M + kTcBM - 1) / kTcBM, (d.n + BN - 1) / BN, splits);
    const bool bp = d.b_planes != nullptr && d.n % 8 == 0 && d.ldb == d.n && R % 8 == 0;
    gemm_tc_kernel<BN, kT, kU8><<<grid, 128, smem, st>>>(a, d.b, d.ldb, ep, M, d.n, R, r_per_split, d.a_u8_div,
                                                         bp ? static_cast<const uint16_t*>(d.b_planes) : nullptr,
                                                         d.b_plane_stride, d.b_prow_npix, d.b_prow_batch);
    count_launch();
    if (splits > 1) {
        launch_split_reduce(ep, M, d.n, st);
        count_launch();
    }
    return 0;
}

// ---- tensor maps of plane sets -------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
// planes of a [rows, cols] matrix in the core-tiled format as a 4-D tensor (64 | cols / 8 | rows / 8 | 3) with box
// (64, box_cores, box_groups, 3)
static bool make_plane_map(CUtensorMap* map, const void* planes, int64_t plane_stride, int64_t rows, int cols,
                           int box_cores, int box_groups, int nplanes = 3, bool interleaved = false) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn) return false;
    cuuint64_t dims[4] = {64, (cuuint64_t)(cols / 8), (cuuint64_t)(rows / 8), (cuuint64_t)nplanes};
    cuuint64_t strides[3] = {128, (cuuint64_t)(cols / 8) * 128, (cuuint64_t)plane_stride * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)box_cores, (cuuint32_t)box_groups, (cuuint32_t)nplanes};
    if (interleaved) {
        // (64 | column cores | 3 planes | row groups): the box lands as [k-group][plane][column core]
        dims[2] = 3;
        dims[3] = (cuuint64_t)(rows / 8);
        strides[1] = (cuuint64_t)(cols / 8) * 128;
        strides[2] = 3 * (cuuint64_t)(cols / 8) * 128;
        box[2] = 3;
        box[3] = (cuuint32_t)box_groups;
    }
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(planes), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// A^T operand of the weight-gradient GEMM (mode 1): planes of A [pixels * B, cols] as a 5-D tensor
//   (64 | column cores | taps | row groups | planes)
// whose "taps" dimension steps `tap_delta` PIXELS (tap_delta * B / 8 row groups) and has `tap_extent` valid entries; it
// aliases the row-group dimension on purpose.  The box (64, box_cores, box_taps, 4, nplanes) lands as
// [plane][k-group][tap][core] -- the MN-major A^T tile of nn_gemm_tiled.cuh; taps past tap_extent are zero-filled.
static bool make_wgrad_map(CUtensorMap* map, const void* planes, int64_t plane_stride, int64_t rows, int cols, int batch,
                           int64_t tap_delta, int tap_extent, int box_cores, int box_taps, int nplanes) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn || tap_delta < 1) return false;
    const cuuint64_t rg_stride = (cuuint64_t)(cols / 8) * 128;
    cuuint64_t dims[5] = {64, (cuuint64_t)(cols / 8), (cuuint64_t)tap_extent, (cuuint64_t)(rows / 8), (cuuint64_t)nplanes};
    cuuint64_t strides[4] = {128, (cuuint64_t)tap_delta * (cuuint64_t)(batch / 8) * rg_stride, rg_stride,
                             (cuuint64_t)plane_stride * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)box_cores, (cuuint32_t)box_taps, 4, (cuuint32_t)nplanes};
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (nplanes == 1) strides[3] = (cuuint64_t)(rows / 8) * rg_stride;      // any valid stride: the dimension has one entry
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(planes), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int BN, bool kT, int NA, bool kCat = false>
static int launch_tiled(const CUtensorMap* maps, const TiledParams& tp, const EpiParams& ep,
                        int M, int gx, int splits, cudaStream_t st) {
    constexpr size_t smem = TiledCfg<BN, NA>::kSmemBytes;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(gemm_tc_tiled_kernel<BN, kT, NA, kCat>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem) != cudaSuccess)
            return -1;
        configured = true;
    }
    static const std::string name = kernel_name("tiled", BN, 0, kT ? "T" : "N",
                                                NA == 1 ? (kCat ? "1,cat" : "1") : (kCat ? "3,cat" : "3"));
    static const char* const fetch[4] = {"bulk", "tma1", "tma2", "tma3"};
    set_dispatch(name.c_str(), kT ? fetch[tp.a_tma] : nullptr);
    dim3 grid(gx, (tp.n + BN - 1) / BN, splits);
    // maps: [0] A (mode 0) / A^T class 0 (mode 1), [1] B, [2], [3] A^T classes 1 and 2
    gemm_tc_tiled_kernel<BN, kT, NA, kCat><<<grid, kTlThreads, smem, st>>>(maps[0], maps[1], maps[2], maps[3], tp, ep, M);
    count_launch();
    if (splits > 1) {
        launch_split_reduce(ep, M, tp.n, st);
        count_launch();
    }
    return 0;
}

// fp32 row-major matrices [rows, cols] -> tiled planes.  One launch converts a list of matrices that live in one fp32
// buffer (the parameter buffer): segment k = (src offset, rows, cols, plane offset), all in elements.
__global__ void __launch_bounds__(256) split_planes_kernel(const float* __restrict__ src, uint16_t* __restrict__ planes,
                                                           int64_t stride, const int64_t* __restrict__ segs) {
    const int64_t* sg = segs + 5 * blockIdx.y;
    const int64_t soff = sg[0], rows = sg[1], cols = sg[2], poff = sg[3];
    const bool il = sg[4] != 0;                            // row-group interleaved planes (tiled_elem_il)
    const int64_t groups = rows * (cols >> 3);             // one thread per (row, 8 columns) = one core-matrix row
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = g / (cols >> 3), c8 = g % (cols >> 3);
        const float* p = src + soff + r * cols + c8 * 8;
        const float4 v0 = __ldg(reinterpret_cast<const float4*>(p));
        const float4 v1 = __ldg(reinterpret_cast<const float4*>(p + 4));
        const Split8 sp = split8(v0, v1);
        if (il) {
            uint16_t* d = planes + poff + tiled_elem_il((size_t)r, (int)(c8 * 8), (int)cols, 0);
            const size_t ps = (size_t)(cols >> 3) * 64;
            *reinterpret_cast<uint4*>(d) = sp.h;
            *reinterpret_cast<uint4*>(d + ps) = sp.m;
            *reinterpret_cast<uint4*>(d + 2 * ps) = sp.l;
            continue;
        }
        uint16_t* d = planes + poff + tiled_elem((size_t)r, (int)(c8 * 8), (int)cols);
        *reinterpret_cast<uint4*>(d) = sp.h;
        *reinterpret_cast<uint4*>(d + stride) = sp.m;
        *reinterpret_cast<uint4*>(d + 2 * stride) = sp.l;
    }
}

// uint8 NHWC frames -> ONE exact bf16 plane of the space-to-depth view: pixel (Y, X) = (y / S, x / S), channel
// ((y % S) * S + x % S) * C + c, plane row (Y * (W / S) + X) * B + b.  A K x K stride-S convolution (K % S == 0) is a
// (K / S) x (K / S) stride-1 convolution of that view, whose channel count S * S * C (64 for Atari) suits the tiled
// tensor-core kernel.  One thread per (b, Y, X, y % S): S * C consecutive bytes -> S * C bf16.
__global__ void __launch_bounds__(256) u8_s2d_planes_kernel(const uint8_t* __restrict__ x, int B, int H, int W, int C,
                                                            int S, uint16_t* __restrict__ plane) {
    // Thread = (8-batch block, Y, pair of X, y % S, b % 8) with b % 8 fastest: the 8 lanes of a quarter-warp write the
    // 8 rows of one core matrix (128 contiguous bytes), and every thread reads the S * C bytes of two neighbouring
    // pixels' rows (a full 32-byte sector for the Atari 4 x 4 x 4 block).
    const int Hs = H / S, Ws = W / S, Cs = S * S * C, run = S * C;       // run: bytes per (pixel, y % S), multiple of 8
    const int Wp = (Ws + 1) / 2;
    const int64_t total = (int64_t)(B / 8) * Hs * Wp * S * 8;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int b8 = (int)(t & 7);
        int64_t r = t >> 3;
        const int dy = (int)(r % S);
        r /= S;
        const int xp = (int)(r % Wp);
        r /= Wp;
        const int Y = (int)(r % Hs);
        const int b = (int)(r / Hs) * 8 + b8;
#pragma unroll
        for (int xi = 0; xi < 2; ++xi) {
            const int X = 2 * xp + xi;
            if (X >= Ws) break;
            const uint8_t* src = x + (((size_t)b * H + (size_t)Y * S + dy) * W + (size_t)X * S) * C;
            const size_t prow = ((size_t)Y * Ws + X) * B + b;
            for (int g = 0; g < run; g += 8) {
                const uint2 w = __ldg(reinterpret_cast<const uint2*>(src + g));
                *reinterpret_cast<uint4*>(plane + tiled_elem(prow, dy * run + g, Cs)) = u8x8_to_bf16(w.x, w.y);
            }
        }
    }
}

// ---- small helpers -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_stage1(const float* __restrict__ x, int64_t rows, int64_t cols,
                                                     float* __restrict__ part, int nslab) {
    // grid.x = column blocks of CW = min(cols, 256) columns, grid.y = row slabs.  The 256 threads of a block form
    // RL = 256 / CW row lanes x CW columns (narrow matrices keep every thread busy and every load coalesced); the row
    // lanes are folded in a fixed order through shared memory.
    __shared__ float red[256];
    const int cw = cols < 256 ? (int)cols : 256;
    const int rl = 256 / cw;
    const int c_local = threadIdx.x % cw, lane_r = threadIdx.x / cw;
    const int64_t col = (int64_t)blockIdx.x * cw + c_local;
    const int slab = blockIdx.y;
    const int64_t per = (rows + nslab - 1) / nslab;
    const int64_t lo = slab * per, hi = min(rows, lo + per);
    float s = 0.f;
    if (col < cols && lane_r < rl)
        for (int64_t r = lo + lane_r; r < hi; r += rl) s += x[r * cols + col];
    red[threadIdx.x] = s;
    __syncthreads();
    if (lane_r == 0 && col < cols) {
        for (int k = 1; k < rl; ++k) s += red[k * cw + c_local];
        part[(int64_t)slab * cols + col] = s;
    }
}
__global__ void __launch_bounds__(1024) colsum_stage2(const float* __restrict__ part, int64_t cols, int nslab,
                                                      float* __restrict__ out) {
    // 1024 threads = RL row lanes x CW columns (up to 1024 partial rows: 32 per lane for a 32-column matrix), lanes
    // folded in a fixed order
    __shared__ float red[1024];
    const int cw = cols < 256 ? (int)cols : 256;
    const int rl = 1024 / cw;
    const int c_local = threadIdx.x % cw, lane_r = threadIdx.x / cw;
    const int64_t col = (int64_t)blockIdx.x * cw + c_local;
    float s = 0.f;
    if (col < cols && lane_r < rl)
        for (int k = lane_r; k < nslab; k += rl) s += part[(int64_t)k * cols + col];
    red[threadIdx.x] = s;
    __syncthreads();
    if (lane_r == 0 && col < cols) {
        for (int k = 1; k < rl; ++k) s += red[k * cw + c_local];
        out[col] = s;
    }
}

__global__ void __launch_bounds__(256) permute_kernel(const float* __restrict__ src, const int32_t* __restrict__ table,
                                                      int64_t n, float* __restrict__ dst, uint16_t* __restrict__ planes,
                                                      int64_t stride, int plane_cols) {
    // planes: dst seen as a [n / plane_cols, plane_cols] matrix in the tiled format
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = __ldg(src + __ldg(table + i));
        dst[i] = v;
        if (planes && stride < 0) {          // row-group interleaved planes
            uint16_t* p = planes + tiled_elem_il((size_t)(i / plane_cols), (int)(i % plane_cols), plane_cols, 0);
            const size_t ps = (size_t)(plane_cols >> 3) * 64;
            split3(v, p[0], p[ps], p[2 * ps]);
        } else if (planes) {
            uint16_t* p = planes + tiled_elem((size_t)(i / plane_cols), (int)(i % plane_cols), plane_cols);
            split3(v, p[0], p[stride], p[2 * stride]);
        }
    }
}

__global__ void transpose_kernel(const float* __restrict__ src, int64_t rows, int64_t cols, float* __restrict__ dst,
                                 uint16_t* __restrict__ planes, int64_t stride) {
    __shared__ float tile[32][33];
    const int64_t c0 = (int64_t)blockIdx.x * 32, r0 = (int64_t)blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = src[r * cols + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) {
            const float v = tile[threadIdx.x][i];
            dst[c * rows + r] = v;
            if (planes) {       // dst [cols, rows] in the tiled format
                uint16_t* p = planes + tiled_elem((size_t)c, (int)r, (int)rows);
                split3(v, p[0], p[stride], p[2 * stride]);
            }
        }
    }
}

}  // namespace gemm
}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_gemm(const cb200_gemm_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->a_src && d->a_rowoff && d->a_coloff && d->b && d->c, "null operand pointer");
    CB200_CHECK_ARG(d->a_rows > 0 && d->a_cols > 0 && d->n > 0 && d->ldb >= d->n && d->ldc >= d->n, "bad extents");
    CB200_CHECK_ARG((d->a_rowinfo == nullptr) == (d->a_colinfo == nullptr), "rowinfo / colinfo must come together");
    const bool tr = d->a_transposed != 0;
    const bool ones = tr && d->a_ones_col != 0;
    const int M = (tr ? d->a_cols : d->a_rows) + (ones ? 1 : 0);
    const int R = tr ? d->a_rows : d->a_cols;
    int splits = d->splits > 1 ? d->splits : 1;
    CB200_CHECK_ARG(splits == 1 || d->workspace, "split reduction needs a workspace");
    int r_per_split = (R + splits - 1) / splits;
    r_per_split = (r_per_split + 15) / 16 * 16;
    splits = (R + r_per_split - 1) / r_per_split;
    cudaStream_t st = as_stream(stream);
    // skinny dense products (heads): dedicated kernels, no split reduction
    if (d->a_lda > 0 && !d->a_lut && !d->a_rowinfo && !d->c_rowmap && tune_get("gemm_skinny", 1, 0, 1) != 0) {
        const float* a = static_cast<const float*>(d->a_src);
        const bool al16 = (reinterpret_cast<uintptr_t>(a) & 15) == 0 && d->a_lda % 4 == 0;
        const gemm::EpiParams ep = gemm::make_epi(*d, 1);
        if (!tr && d->n <= 8 && R % 4 == 0 && al16) {
            set_dispatch("skinny_n");
            gemm::skinny_n_kernel<<<(unsigned)((M + 7) / 8), 256, 0, st>>>(a, d->a_lda, d->b, d->ldb, ep, M, d->n, R);
            count_launch();
            CB200_CHECK_LAUNCH();
            return CB200_OK;
        }
        if (!tr && R <= 8 && d->n % 4 == 0 && d->ldb % 4 == 0 && (reinterpret_cast<uintptr_t>(d->b) & 15) == 0) {
            const int64_t groups = (int64_t)M * (d->n / 4);
            set_dispatch("skinny_r");
            gemm::skinny_r_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, st>>>(a, d->a_lda, d->b, d->ldb, ep, M,
                                                                                     d->n, R);
            count_launch();
            CB200_CHECK_LAUNCH();
            return CB200_OK;
        }
        if (tr && d->n <= 8) {
            const int kblocks = (d->a_cols + 31) / 32;
            set_dispatch("skinny_tn");
            gemm::skinny_tn_kernel<<<(unsigned)(kblocks + (ones ? 1 : 0)), 1024, 0, st>>>(
                a, d->a_lda, d->b, d->ldb, ep, d->a_rows, d->a_cols, d->n, d->a_cols);
            count_launch();
            CB200_CHECK_LAUNCH();
            return CB200_OK;
        }
    }
    const bool fast = d->a_vec4 && d->n % 4 == 0 && d->ldb % 4 == 0 && d->a_cols % 4 == 0 &&
                      (reinterpret_cast<uintptr_t>(d->b) & 15) == 0 && M > 64;
    CB200_CHECK_ARG(!ones || fast, "a_ones_col needs the vectorised or the skinny path");
    // tensor-core path (wgmma): operands split into 3 x bf16, fp32 accumulation; the reduction length per launch is
    // capped (split-R) -- see nn_gemm_tc.cuh
    const bool tc = fast && d->n % 16 == 0 && d->n >= 16 && tune_get("gemm_tc", 1, 0, 1) != 0 && d->ldc % 4 == 0 &&
                    ((reinterpret_cast<uintptr_t>(d->c) | reinterpret_cast<uintptr_t>(d->mask_y) |
                      reinterpret_cast<uintptr_t>(d->bias)) & 15) == 0 &&
                    r_per_split <= gemm::kTcMaxSlice;
    if (tc) {
        // uint8 A with a declared divisor: the integers are contracted exactly from one bf16 plane
        const bool u8 = d->a_lut != nullptr && d->a_u8_div > 0.f;
        int rc;
#define CB200_TC(BN_)                                                                                          \
    (u8 ? (tr ? gemm::launch_tc<BN_, true, true>(*d, M, R, splits, r_per_split, st)                           \
              : gemm::launch_tc<BN_, false, true>(*d, M, R, splits, r_per_split, st))                         \
        : (tr ? gemm::launch_tc<BN_, true, false>(*d, M, R, splits, r_per_split, st)                          \
              : gemm::launch_tc<BN_, false, false>(*d, M, R, splits, r_per_split, st)))
        // one warpgroup holds the accumulators of a 128 x BN tile: BN <= 64
        if (d->n <= 32) rc = CB200_TC(32);
        else rc = CB200_TC(64);
#undef CB200_TC
        CB200_CHECK_ARG(rc == 0, "could not configure shared memory for the tensor-core kernel");
        CB200_CHECK_LAUNCH();
        return CB200_OK;
    }
    if (fast) {
        if (d->n <= 32) {
            if (tr) gemm::launch_fast<gemm::FastCfg<256, 32>, true>(*d, M, R, splits, r_per_split, st);
            else gemm::launch_fast<gemm::FastCfg<256, 32>, false>(*d, M, R, splits, r_per_split, st);
        } else if (d->n <= 64) {
            if (tr) gemm::launch_fast<gemm::FastCfg<128, 64>, true>(*d, M, R, splits, r_per_split, st);
            else gemm::launch_fast<gemm::FastCfg<128, 64>, false>(*d, M, R, splits, r_per_split, st);
        } else {
            if (tr) gemm::launch_fast<gemm::FastCfg<128, 128>, true>(*d, M, R, splits, r_per_split, st);
            else gemm::launch_fast<gemm::FastCfg<128, 128>, false>(*d, M, R, splits, r_per_split, st);
        }
        CB200_CHECK_LAUNCH();
        return CB200_OK;
    }
    const bool small = (M <= 64);
    if (small) {
        if (tr) gemm::launch<gemm::CfgSmall, true>(*d, M, R, splits, r_per_split, st);
        else gemm::launch<gemm::CfgSmall, false>(*d, M, R, splits, r_per_split, st);
    } else if (d->n <= 32) {
        if (tr) gemm::launch<gemm::CfgN32, true>(*d, M, R, splits, r_per_split, st);
        else gemm::launch<gemm::CfgN32, false>(*d, M, R, splits, r_per_split, st);
    } else {
        if (tr) gemm::launch<gemm::CfgN64, true>(*d, M, R, splits, r_per_split, st);
        else gemm::launch<gemm::CfgN64, false>(*d, M, R, splits, r_per_split, st);
    }
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_gemm_tiled(const cb200_tgemm_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->mode == 0 || d->mode == 1, "mode must be 0 or 1");
    CB200_CHECK_ARG(d->a_planes && d->b_planes && (d->c || (d->c_planes && !d->mask_y)), "null operand pointer");
    CB200_CHECK_ARG(!d->mask_planes || (d->c_plane_cols == d->n && d->mask_plane_stride % 8 == 0 &&
                                        (reinterpret_cast<uintptr_t>(d->mask_planes) & 15) == 0),
                    "mask_planes need c_plane_cols == n and 16-byte alignment");
    CB200_CHECK_ARG(d->batch > 0 && d->batch % 32 == 0, "batch must be a multiple of 32");
    CB200_CHECK_ARG(d->a_cols > 0 && d->a_cols % 32 == 0 && (d->a_cols <= 128 ? 128 % d->a_cols == 0 : d->a_cols % 128 == 0),
                    "a_cols must be 32, 64, 128 or a multiple of 128");
    CB200_CHECK_ARG(d->n == 32 || (d->n > 0 && d->n % 64 == 0), "n must be 32 or a multiple of 64");
    CB200_CHECK_ARG(d->ldc >= d->n && d->ldc % 4 == 0, "ldc");
    CB200_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->a_planes) | reinterpret_cast<uintptr_t>(d->b_planes) |
                      reinterpret_cast<uintptr_t>(d->c_planes) | reinterpret_cast<uintptr_t>(d->c) |
                      reinterpret_cast<uintptr_t>(d->bias) | reinterpret_cast<uintptr_t>(d->mask_y)) & 15) == 0,
                    "operands must be 16-byte aligned");
    CB200_CHECK_ARG(d->a_plane_stride % 8 == 0 && d->b_plane_stride % 8 == 0 && d->c_plane_stride % 8 == 0, "plane strides");
    CB200_CHECK_ARG(!d->c_planes || d->c_plane_cols == d->n, "c_plane_cols must equal n");
    gemm::TiledParams tp;
    tp.mode = d->mode;
    tp.batch = d->batch;
    tp.a = static_cast<const uint16_t*>(d->a_planes);
    tp.a_stride = d->a_plane_stride;
    tp.a_cols = d->a_cols;
    tp.b = static_cast<const uint16_t*>(d->b_planes);
    tp.b_stride = d->b_plane_stride;
    tp.n = d->n;
    tp.list_ptr = d->list_ptr;
    tp.list = reinterpret_cast<const int2*>(d->list);
    tp.a_pix = d->a_pix;
    tp.num_q = d->num_q;
    tp.taps = d->taps;
    int M, gx, total;
    CB200_CHECK_ARG(d->a_rows > 0 && d->a_rows % 8 == 0 && d->b_rows > 0 && d->b_rows % 8 == 0, "a_rows / b_rows");
    const int bn = d->n <= 32 ? 32 : ((d->n <= 64 || d->n % 128 != 0) ? 64 : 128);
    const int na = d->a_num_planes == 1 ? 1 : 3;
    CB200_CHECK_ARG(na == 3 || d->a_u8_div > 0.f, "a single A plane means raw uint8 values: a_u8_div must be set");
    // row-group interleaved B planes: the three B planes reach shared memory as one [32 k, 3 n] operand (one TMA box
    // instead of three); the 3xBF16 product set is still issued as six narrow MMAs, one per plane pair
    const bool cat = d->b_interleaved != 0;
    CB200_CHECK_ARG(!cat || (d->mode == 0 && bn <= 64), "b_interleaved needs mode 0 and n <= 64 (or n % 128 != 0)");
    // the tensor maps depend only on the descriptor: built on the first call, kept in the descriptor
    cb200_tgemm_desc* md = const_cast<cb200_tgemm_desc*>(d);
    CUtensorMap* maps =
        reinterpret_cast<CUtensorMap*>((reinterpret_cast<uintptr_t>(md->tmap_storage) + 63) & ~(uintptr_t)63);
    const uint64_t key = (uint64_t)(reinterpret_cast<uintptr_t>(d->a_planes) ^ (reinterpret_cast<uintptr_t>(d->b_planes) << 1) ^ 1);
    if (md->tmap_key != key) {
        bool ok = gemm::make_plane_map(maps + 1, d->b_planes, d->b_plane_stride, d->b_rows, d->n, bn / 8, 4, 3, cat);
        if (d->mode == 0)
            ok = ok && gemm::make_plane_map(maps + 0, d->a_planes, d->a_plane_stride, d->a_rows, d->a_cols, 4, 16, na);
        else
            maps[0] = maps[1];
        maps[2] = maps[3] = maps[0];
        md->a_tma = 0;
        if (ok && d->mode == 1 && d->a_pix_host && tune_get("wgrad_tma", 1, 0, 1) != 0) {
            // Tap-stride classes of the 128-row tiles: tile i covers taps t0 .. t0 + box_taps - 1 (a_cols < 128) or a
            // 128-channel slice of one tap.  Usable when, inside every tile, consecutive taps sit the same positive
            // number of pixels apart at every output pixel, with at most three distinct (stride, valid taps) pairs.
            const int Ca = d->a_cols, cw = Ca < 128 ? Ca : 128, box_taps = 128 / cw;
            const int tiles = (d->taps * Ca + 127) / 128;
            struct Cls { int64_t delta; int extent; } cls[3];
            int ncls = 0;
            bool usable = tiles <= 64;
            for (int i = 0; usable && i < tiles; ++i) {
                const int t0 = Ca < 128 ? i * box_taps : (i * 128) / Ca;
                const int valid = Ca < 128 ? (d->taps - t0 < box_taps ? d->taps - t0 : box_taps) : 1;
                int64_t delta = 1;
                if (valid > 1) {
                    delta = (int64_t)d->a_pix_host[(size_t)(t0 + 1) * d->num_q] - d->a_pix_host[(size_t)t0 * d->num_q];
                    for (int t = t0; usable && t + 1 < t0 + valid; ++t)
                        for (int q = 0; q < d->num_q; ++q)
                            if ((int64_t)d->a_pix_host[(size_t)(t + 1) * d->num_q + q] -
                                    d->a_pix_host[(size_t)t * d->num_q + q] != delta) {
                                usable = false;
                                break;
                            }
                    if (delta < 1) usable = false;
                }
                int k = 0;
                while (k < ncls && !(cls[k].delta == delta && cls[k].extent == valid)) ++k;
                if (k == ncls) {
                    if (ncls == 3) { usable = false; break; }
                    cls[ncls].delta = delta;
                    cls[ncls].extent = valid;
                    ++ncls;
                }
                if (usable) md->a_tile_class[i] = (uint8_t)k;
            }
            if (usable) {
                static const int slot[3] = {0, 2, 3};
                for (int k = 0; usable && k < ncls; ++k)
                    usable = gemm::make_wgrad_map(maps + slot[k], d->a_planes, d->a_plane_stride, d->a_rows, Ca, d->batch,
                                                  cls[k].delta, cls[k].extent, cw / 8, box_taps, na);
                for (int k = ncls; k < 3; ++k) maps[slot[k]] = maps[slot[0]];
                if (usable) md->a_tma = ncls;
                else maps[0] = maps[2] = maps[3] = maps[1];
            }
            if (getenv("CB200_DEBUG"))
                fprintf(stderr, "cb200_gemm_tiled mode 1: taps %d a_cols %d num_q %d tiles %d -> A^T tensor maps: %d\n",
                        d->taps, d->a_cols, d->num_q, tiles, md->a_tma);
        }
        CB200_CHECK_ARG(ok, "cuTensorMapEncodeTiled failed (driver too old or bad plane geometry)");
        md->tmap_key = key;
    }
    tp.a_tma = d->mode == 1 ? md->a_tma : 0;
    for (int i = 0; i < 64; ++i) tp.tile_class[i] = md->a_tile_class[i];
    if (d->mode == 0) {
        CB200_CHECK_ARG(d->list_ptr && d->list && d->num_q > 0 && d->max_list_len > 0, "mode 0 needs the tap lists");
        M = d->num_q * d->batch;
        gx = d->num_q * ((d->batch + 127) / 128);
        total = d->max_list_len * (d->a_cols / 32);
    } else {
        CB200_CHECK_ARG(d->a_pix && d->num_q > 0 && d->taps > 0, "mode 1 needs the tap / pixel table");
        M = d->taps * d->a_cols;
        gx = (M + 127) / 128;
        total = d->num_q * (d->batch / 32);
        if (d->bias_row) M += 1;          // rows of the result (and of the split partials); tiles still cover M - 1
    }
    int splits = d->splits > 1 ? d->splits : 1;
    int cps = (total + splits - 1) / splits;
    splits = (total + cps - 1) / cps;
    // at most 32 reduction chunks (64 accumulating k16 steps) per launch slice; slices are summed in fp32
    CB200_CHECK_ARG(cps <= 32, "too few splits: more than 32 reduction chunks (1024 terms) per slice");
    CB200_CHECK_ARG(splits == 1 || d->workspace, "split reduction needs a workspace");
    tp.chunks_per_split = cps;
    tp.a_u8_div = d->a_u8_div;
    tp.bias_row = d->mode == 1 ? d->bias_row : 0;
    const gemm::EpiParams ep{d->c,        d->ldc,      d->bias,      d->act,  d->mask_y,
                             d->mask_act, d->c_rowmap, d->workspace, splits,  0,
                             static_cast<uint16_t*>(d->c_planes), d->c_plane_stride, d->c_plane_cols, 0, 0,
                             static_cast<const uint16_t*>(d->mask_planes), d->mask_plane_stride};
    cudaStream_t st = as_stream(stream);
    int rc;
#define CB200_TL(BN_) \
    (na == 1 ? (d->mode ? gemm::launch_tiled<BN_, true, 1>(maps, tp, ep, M, gx, splits, st)   \
                        : gemm::launch_tiled<BN_, false, 1>(maps, tp, ep, M, gx, splits, st)) \
             : (d->mode ? gemm::launch_tiled<BN_, true, 3>(maps, tp, ep, M, gx, splits, st)   \
                        : gemm::launch_tiled<BN_, false, 3>(maps, tp, ep, M, gx, splits, st)))
#define CB200_TLC(BN_) \
    (na == 1 ? gemm::launch_tiled<BN_, false, 1, true>(maps, tp, ep, M, gx, splits, st) \
             : gemm::launch_tiled<BN_, false, 3, true>(maps, tp, ep, M, gx, splits, st))
    if (cat) rc = bn == 32 ? CB200_TLC(32) : CB200_TLC(64);
    else if (bn == 32) rc = CB200_TL(32);
    else if (bn == 64) rc = CB200_TL(64);
    else rc = CB200_TL(128);
#undef CB200_TL
#undef CB200_TLC
    CB200_CHECK_ARG(rc == 0, "could not configure shared memory for the tiled tensor-core kernel");
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_u8_s2d_planes(const void* x, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t s, void* plane,
                        void* stream) {
    CB200_CHECK_ARG(x && plane && batch > 0 && batch % 8 == 0 && s > 0 && h % s == 0 && w % s == 0, "bad geometry");
    CB200_CHECK_ARG((s * c) % 8 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(plane)) & 15) == 0,
                    "s * c must be a multiple of 8 and the buffers 16-byte aligned");
    const int64_t total = (int64_t)batch * (h / s) * ((w / s + 1) / 2) * s;
    int64_t grid = (total + 255) / 256;
    if (grid > (int64_t)sm_count() * 16) grid = (int64_t)sm_count() * 16;
    gemm::u8_s2d_planes_kernel<<<(unsigned)grid, 256, 0, as_stream(stream)>>>(static_cast<const uint8_t*>(x), batch, h, w,
                                                                               c, s, static_cast<uint16_t*>(plane));
    count_launch();
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_split_planes(const float* src, void* planes, int64_t plane_stride, const int64_t* d_segments, int num_segments,
                       int64_t max_segment_elems, void* stream) {
    CB200_CHECK_ARG(src && planes && d_segments && num_segments > 0 && max_segment_elems > 0 && plane_stride % 8 == 0,
                    "bad arguments");
    CB200_CHECK_ARG(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(planes)) & 15) == 0,
                    "src and planes must be 16-byte aligned");
    int64_t gx = (max_segment_elems / 8 + 255) / 256;
    if (gx > (int64_t)sm_count() * 4) gx = (int64_t)sm_count() * 4;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, (unsigned)num_segments);
    gemm::split_planes_kernel<<<grid, 256, 0, as_stream(stream)>>>(src, static_cast<uint16_t*>(planes), plane_stride,
                                                                   d_segments);
    count_launch();
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_colsum(const float* x, int64_t rows, int64_t cols, float* out, float* workspace, void* stream) {
    CB200_CHECK_ARG(x && out && workspace && rows > 0 && cols > 0, "bad arguments");
    // slabs of about 8 rows per row lane (256 / min(cols, 256) lanes): enough blocks to fill the machine even for the
    // short, wide matrices of the dense layers; workspace holds <= 1024 partial rows
    const int64_t cw = cols < 256 ? cols : 256;
    const int64_t rl = 256 / cw;
    int nslab = (int)((rows + rl * 8 - 1) / (rl * 8));
    if (nslab > 1024) nslab = 1024;
    if (nslab < 1) nslab = 1;
    cudaStream_t st = as_stream(stream);
    dim3 g1((unsigned)((cols + 255) / 256), nslab);
    gemm::colsum_stage1<<<g1, 256, 0, st>>>(x, rows, cols, workspace, nslab);
    gemm::colsum_stage2<<<(unsigned)((cols + 255) / 256), 1024, 0, st>>>(workspace, cols, nslab, out);
    count_launch(2);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_permute_f32(const float* src, const int32_t* table, int64_t n, float* dst, void* dst_planes,
                      int64_t plane_stride, int32_t plane_cols, void* stream) {
    CB200_CHECK_ARG(!dst_planes || (plane_cols > 0 && plane_cols % 8 == 0 && n % (8 * (int64_t)plane_cols) == 0),
                    "planes: dst must be a [multiple of 8, plane_cols] matrix");
    CB200_CHECK_ARG(src && table && dst && n > 0, "bad arguments");
    int64_t grid = (n + 255) / 256;
    if (grid > (int64_t)sm_count() * 8) grid = (int64_t)sm_count() * 8;
    gemm::permute_kernel<<<(unsigned)grid, 256, 0, as_stream(stream)>>>(
        src, table, n, dst, static_cast<uint16_t*>(dst_planes), plane_stride, plane_cols);
    count_launch();
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_transpose(const float* src, int64_t rows, int64_t cols, float* dst, void* dst_planes, int64_t plane_stride,
                    void* stream) {
    CB200_CHECK_ARG(src && dst && rows > 0 && cols > 0, "bad arguments");
    // the planes of dst [cols, rows] have rows plane columns: whole 8-column cores, planes on core boundaries
    CB200_CHECK_ARG(!dst_planes || (rows % 8 == 0 && plane_stride % 8 == 0 && plane_stride >= rows * ((cols + 7) / 8 * 8)),
                    "planes: rows % 8 == 0, plane_stride % 8 == 0 and >= rows * cols rounded up to 8 rows");
    dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
    gemm::transpose_kernel<<<grid, dim3(32, 8), 0, as_stream(stream)>>>(src, rows, cols, dst,
                                                                        static_cast<uint16_t*>(dst_planes), plane_stride);
    count_launch();
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

}  // extern "C"
