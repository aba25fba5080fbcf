// coach_b200/csrc/replay.cu -- HBM-resident prioritized / uniform replay: segment trees, sampling, column gather.
//
// Reference arithmetic being replaced (file:line under /root/reference/rl_coach/):
//   memories/non_episodic/prioritized_experience_replay.py:43-156  SegmentTree
//   memories/non_episodic/prioritized_experience_replay.py:188-283 PER._update_priority/update_priorities/sample/store
//   memories/non_episodic/experience_replay.py:71-93,131-150        ExperienceReplay.sample/store
//   core_types.py:488-623                                           Batch column extraction (AoS -> SoA)
//
// Exactness rules for everything that feeds an index: fp64, explicit round-to-nearest intrinsics (__dadd_rn ...)
// so that nvcc can never contract a*b+c into an FMA (Python evaluates each operation separately), comparisons
// written exactly as the reference writes them (`val <= tree[left]`).
#include <math.h>
#include <string.h>

#include <cuda.h>      // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)

#include "common.cuh"

namespace cb200 {

// =====================================================================================================================
// Segment-tree descent: one warp, all lanes carry the same `val`.
// SegmentTree._retrieve (:76-92) walks one level per step; here each round fetches the next R<=5 levels below the
// current node (2+4+...+2^R <= 62 nodes, contiguous per level in the heap array) with two loads per lane and
// then replays the reference's comparisons out of registers with shuffles.  Same comparisons, same subtractions,
// same order => same leaf, bit for bit.
// =====================================================================================================================
// 8 bytes -> 8 bf16 holding the integers exactly (0x4B0000vv is the float 2^23 + v; minus 2^23 leaves float(v), whose
// upper half-word is its bf16)
__device__ __forceinline__ uint4 u8x8_to_bf16_s2d(uint32_t w0, uint32_t w1) {
    uint32_t f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        f[j] = __float_as_uint(__uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7440 + j)) - 8388608.f);
        f[4 + j] = __float_as_uint(__uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7440 + j)) - 8388608.f);
    }
    return make_uint4(__byte_perm(f[0], f[1], 0x7632), __byte_perm(f[2], f[3], 0x7632), __byte_perm(f[4], f[5], 0x7632),
                      __byte_perm(f[6], f[7], 0x7632));
}

struct Descent {
    int64_t leaf;
    double priority;   // tree[leaf + size - 1]
};

// Levels fetched per memory round trip.  7 levels = 254 nodes = 8 independent loads per lane: a 2^20-leaf tree is
// walked in 3 dependent round trips (7 + 7 + 6) instead of 20.  The fetched sub-tree is parked in a per-warp shared
// memory scratch (256 doubles) and the reference's comparisons are replayed out of it (one 16-byte broadcast read per
// level: the two children are adjacent elements).
constexpr int kRoundLevels = 7;
constexpr int kRoundRegs = ((2 << kRoundLevels) - 2 + 31) / 32;   // 8 loads per lane
constexpr int kScratchDoubles = 32 * kRoundRegs;                  // 256 per warp

__device__ __forceinline__ Descent warp_descent(const double* __restrict__ tree, int64_t size, int levels,
                                                double val, double* __restrict__ scratch /* per-warp, 16B aligned */) {
    const int lane = threadIdx.x & 31;
    uint64_t j = 1;   // 1-based heap index of the current node
    double p = 0.0;
    if (levels == 0) p = __ldcg(tree);
    int remaining = levels;
    while (remaining > 0) {
        const int r = remaining < kRoundLevels ? remaining : kRoundLevels;
        // element e of the sub-tree below j, in level order without the root: e + 2 = 2^k + off (k = level below j)
        //   -> 1-based node (j << k) + off = ((j - 1) << k) + (e + 2)
        double v[kRoundRegs];
#pragma unroll
        for (int q = 0; q < kRoundRegs; ++q) {
            const int e2 = lane + 32 * q + 2;
            const int k = 31 - __clz(e2);
            v[q] = (k <= r) ? __ldcg(tree + (((j - 1) << k) + e2 - 1)) : 0.0;
        }
        __syncwarp();          // previous round's reads of the scratch are done
#pragma unroll
        for (int q = 0; q < kRoundRegs; ++q) scratch[lane + 32 * q] = v[q];
        __syncwarp();
        uint32_t rel = 1;
        for (int s = 0; s < r; ++s) {
            const int el = 2 * rel - 2;             // left child; the right child is element el + 1 (el is even)
            const double2 lr = *reinterpret_cast<const double2*>(scratch + el);
            if (val <= lr.x) {   // :89
                rel = 2 * rel;
                p = lr.x;
            } else {             // :92
                val = __dsub_rn(val, lr.x);
                rel = 2 * rel + 1;
                p = lr.y;
            }
        }
        j = (j << r) + (rel - (1u << r));
        remaining -= r;
    }
    Descent d;
    d.leaf = (int64_t)j - size;
    d.priority = p;
    return d;
}

struct SampleParams {
    const double* sum_tree;
    const double* min_tree;
    int64_t size;
    int levels;
    const double* u;
    int64_t n;
    double nt;     // (double) num_transitions
    double beta;
    int64_t* idx_out;
    double* w_out;
    float* w32_out;
};

// PER.sample :232-245 for sample i (whole warp): the stratified draw and the tree descent.
__device__ __forceinline__ Descent per_sample_descend(const SampleParams& sp, int64_t i, double* scratch) {
    const double total = __ldcg(sp.sum_tree);
    const double segment = __ddiv_rn(total, (double)sp.n);                        // :232
    const double a = __dmul_rn(segment, (double)i);                               // :240
    const double b = __dmul_rn(segment, (double)(i + 1));                         // :241
    const double val = __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), __ldg(sp.u + i)));  // random.uniform :244
    return warp_descent(sp.sum_tree, sp.size, sp.levels, val, scratch);
}

// PER.sample :235-251: importance weight of one drawn leaf (one thread); off the gather's critical path
__device__ __forceinline__ void per_sample_publish(const SampleParams& sp, int64_t i, int64_t leaf, double priority) {
    if (sp.idx_out) sp.idx_out[i] = leaf;
    if (sp.w_out || sp.w32_out) {
        const double total = __ldcg(sp.sum_tree);
        const double min_probability = __ddiv_rn(__ldcg(sp.min_tree), total);       // :235
        const double max_weight = pow(__dmul_rn(min_probability, sp.nt), -sp.beta);  // :236
        const double prob = __ddiv_rn(priority, total);                             // :246
        const double weight = pow(__dmul_rn(sp.nt, prob), -sp.beta);                // :247
        const double w = __ddiv_rn(weight, max_weight);                             // :248
        if (sp.w_out) sp.w_out[i] = w;
        if (sp.w32_out) sp.w32_out[i] = (float)w;
    }
}

__global__ void __launch_bounds__(128) per_sample_kernel(SampleParams sp) {
    __shared__ __align__(16) double scratch[4][kScratchDoubles];
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (warp >= sp.n) return;
    const Descent d = per_sample_descend(sp, warp, scratch[threadIdx.x >> 5]);
    if ((threadIdx.x & 31) == 0) per_sample_publish(sp, warp, d.leaf, d.priority);
}

// =====================================================================================================================
// Tree update: leaves (last writer wins) then ancestors level by level.
// =====================================================================================================================
struct UpdateParams {
    double* sum_tree;
    double* min_tree;
    double* max_tree;
    int32_t* winner;
    int64_t size;
    int levels;
    const int64_t* idx;      // nullptr => ring mode: leaf = (cursor + i) % size, constant values
    const double* p_alpha;
    const double* p_raw;
    int64_t cursor;
    double c_alpha, c_raw;
    int64_t n;
    double* max_priority_out;
    int32_t* error_flags;    // optional: bit 1 (value 2) is set when a leaf index is out of range
};

// leaf of batch entry i, or -1 when the entry must not be applied: out of range (flagged), or carrying the negative
// priority marker cb200_per_priorities_device leaves for an invalid (negative / NaN) error
__device__ __forceinline__ int64_t upd_leaf(const UpdateParams& up, int64_t i) {
    if (up.idx) {
        const int64_t leaf = up.idx[i];
        if (leaf < 0 || leaf >= up.size) {
            if (up.error_flags) atomicOr(up.error_flags, 2);
            return -1;
        }
        if (up.p_alpha[i] < 0.0) return -1;
        return leaf;
    }
    return (up.cursor + i) & (up.size - 1);
}
__device__ __forceinline__ double py_min(double a, double b) { return (b < a) ? b : a; }   // builtin min(a, b)
__device__ __forceinline__ double py_max(double a, double b) { return (b > a) ? b : a; }   // builtin max(a, b)

__device__ __forceinline__ void recompute_parent(const UpdateParams& up, int64_t parent) {
    const int64_t l = 2 * parent + 1;                                                          // :71
    // children sit at l (odd) and l+1: not 16-byte aligned as a pair, so two 8-byte loads per tree
    const double sl = __ldcg(up.sum_tree + l), sr = __ldcg(up.sum_tree + l + 1);
    const double ml = __ldcg(up.min_tree + l), mr = __ldcg(up.min_tree + l + 1);
    const double xl = __ldcg(up.max_tree + l), xr = __ldcg(up.max_tree + l + 1);
    __stcg(up.sum_tree + parent, __dadd_rn(sl, sr));
    __stcg(up.min_tree + parent, py_min(ml, mr));
    __stcg(up.max_tree + parent, py_max(xl, xr));
}

// n <= 1024: one CTA does everything, __syncthreads between levels.
__global__ void __launch_bounds__(1024) per_update_cta_kernel(UpdateParams up) {
    const int i = threadIdx.x;
    int64_t leaf = -1;
    bool active = false;
    if (i < up.n) {
        leaf = upd_leaf(up, i);
        active = leaf >= 0 && leaf < up.size;
    }
    if (active) atomicMax(up.winner + leaf, i);
    __syncthreads();
    const bool win = active && (__ldcg(up.winner + leaf) == i);
    __syncthreads();
    int64_t node = leaf + up.size - 1;
    if (win) {
        const double pa = up.idx ? up.p_alpha[i] : up.c_alpha;
        const double pr = up.idx ? up.p_raw[i] : up.c_raw;
        __stcg(up.sum_tree + node, pa);
        __stcg(up.min_tree + node, pa);
        __stcg(up.max_tree + node, pr);
        __stcg(up.winner + leaf, -1);
    }
    if (active) {
        // pull every sibling on the path into L2 up front: the level loop below then only sees L2 latency
        int64_t nd = node;
        for (int l = 0; l < up.levels; ++l) {
            const int64_t sib = ((nd - 1) ^ 1) + 1;
            asm volatile("prefetch.global.L2 [%0];" ::"l"(up.sum_tree + sib));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(up.min_tree + sib));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(up.max_tree + sib));
            nd = (nd - 1) >> 1;
        }
    }
    __syncthreads();
    for (int l = 0; l < up.levels; ++l) {
        const int64_t parent = (node - 1) >> 1;   // :69
        // threads sharing a parent all compute the same value; let the lowest-numbered writer per pair do it when
        // cheap to know (sibling leaf within the same thread is not knowable) -- identical values, benign.
        if (active) recompute_parent(up, parent);
        node = parent;
        __syncthreads();
    }
    if (i == 0 && up.max_priority_out) *up.max_priority_out = __ldcg(up.max_tree);   // :201
}

// n <= 512, one launch, no global round trip between levels.
// The batch's leaves are sorted in shared memory (bitonic, key = leaf * 2048 + position), which (i) resolves duplicates
// -- the last writer of a leaf is the last key of its run -- and (ii) makes paths that meet adjacent: the threads whose
// paths pass through one node form a contiguous run [lo, hi], and a touched sibling is the run right next to it.  Each
// thread then walks its path bottom-up holding its node's (sum, min, max) in registers: the sibling's values come from
// the neighbouring run through shared memory when that sibling is itself being updated, otherwise from global memory,
// where they cannot change during the kernel and are therefore fetched a few levels ahead.  One __syncthreads per
// level on double-buffered shared arrays; every parent is op(left, right) of the final children, exactly what the
// reference's sequential updates leave behind (SegmentTree.update :62-73 recomputes each ancestor from its children).
constexpr int kUpdSortThreads = 512;     // 128 registers per thread: the bottom-level sibling values stay in registers
constexpr int kUpdAhead = 11;       // bottom levels whose untouched-sibling values a thread fetches up front (registers)
constexpr int kUpdTopLevels = 10;   // top levels of the three trees staged in shared memory (nodes 1 .. 1023, 1-based):
                                    // a sibling is found there when the child being left has index < 2^kUpdTopLevels, i.e.
                                    // from walk level l >= levels - (kUpdTopLevels - 1) on
constexpr int kUpdSortSmem = 80 * kUpdSortThreads + 3 * 8 * (1 << kUpdTopLevels);

__global__ void __launch_bounds__(kUpdSortThreads) per_update_sorted_kernel(UpdateParams up) {
    extern __shared__ __align__(16) uint8_t upd_smem[];      // kUpdSortSmem bytes (dynamic: above the 48 KB static limit)
    constexpr int T = kUpdSortThreads;
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(upd_smem);
    long long(*s_node)[T] = reinterpret_cast<long long(*)[T]>(upd_smem + 8 * T);
    double(*s_sum)[T] = reinterpret_cast<double(*)[T]>(upd_smem + 24 * T);
    double(*s_min)[T] = reinterpret_cast<double(*)[T]>(upd_smem + 40 * T);
    double(*s_max)[T] = reinterpret_cast<double(*)[T]>(upd_smem + 56 * T);
    short(*s_lo)[T] = reinterpret_cast<short(*)[T]>(upd_smem + 72 * T);
    short(*s_hi)[T] = reinterpret_cast<short(*)[T]>(upd_smem + 76 * T);
    // untouched siblings in the top kUpdTopLevels levels come from a shared-memory copy of those levels (loaded once,
    // coalesced, while the sort runs); only the bottom levels need per-thread global loads -- issued all at once, so
    // the whole walk costs two dependent global round trips (indices -> leaves / siblings) instead of one per few levels
    double* s_top = reinterpret_cast<double*>(upd_smem + 80 * T);          // [3][1 << kUpdTopLevels], 1-based heap index
    __shared__ int s_scan[kUpdSortThreads / 32];
    __shared__ int s_m;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int P = blockDim.x;                               // sort width = launch width (power of two >= n, >= 32)
    {
        // nodes 1 .. top_nodes: the top kUpdTopLevels levels, or the whole (small) tree
        const long long all_nodes = 2 * up.size - 1;
        const int top_nodes = (int)(all_nodes < (1 << kUpdTopLevels) - 1 ? all_nodes : (1 << kUpdTopLevels) - 1);
        for (int j = t; j < top_nodes; j += P) {
            s_top[j + 1] = __ldcg(up.sum_tree + j);
            s_top[(1 << kUpdTopLevels) + j + 1] = __ldcg(up.min_tree + j);
            s_top[2 * (1 << kUpdTopLevels) + j + 1] = __ldcg(up.max_tree + j);
        }
    }
    // ---- keys ------------------------------------------------------------------------------------------------------
    unsigned long long key = ~0ull;                         // invalid / padding: sorts last
    if (t < up.n) {
        const int64_t leaf = upd_leaf(up, t);
        if (leaf >= 0 && leaf < up.size) key = ((unsigned long long)leaf << 11) | (unsigned long long)t;
    }
    // ---- bitonic sort of the P keys, one per thread: exchanges at distance < 32 are warp shuffles, larger ones go
    // through shared memory (10 block-wide steps instead of 45 for P = 512) -----------------------------------------
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            unsigned long long other;
            if (j >= 32) {
                __syncthreads();                            // the previous step's readers are done
                s_key[t] = key;
                __syncthreads();
                other = s_key[t ^ j];
            } else {
                other = __shfl_xor_sync(0xffffffffu, key, j);
            }
            const bool keep_min = ((t & j) == 0) == ((t & k) == 0);
            key = keep_min ? (other < key ? other : key) : (other > key ? other : key);
        }
    }
    __syncthreads();
    s_key[t] = key;
    __syncthreads();
    // ---- last writer of every distinct leaf, compacted in leaf order ----------------------------------------------
    const bool winner = key != ~0ull && (t == P - 1 || (s_key[t + 1] >> 11) != (key >> 11));
    const unsigned ballot = __ballot_sync(0xffffffffu, winner);
    if (lane == 0) s_scan[warp] = __popc(ballot);
    __syncthreads();
    if (warp == 0) {
        int v = lane < (P >> 5) ? s_scan[lane] : 0;         // warps of this launch only
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        s_scan[lane] = incl - v;                            // exclusive prefix per warp
        if (lane == 31) s_m = incl;
    }
    __syncthreads();
    const int m = s_m;                                      // distinct leaves
    if (winner) {
        const int pos = s_scan[warp] + __popc(ballot & ((1u << lane) - 1u));
        s_node[1][pos] = (long long)key;                    // parked in the second buffer until the loop starts
    }
    __syncthreads();
    // ---- leaves -------------------------------------------------------------------------------------------------------
    long long node = 0;                                     // 1-based heap index of this thread's current node
    double v_sum = 0.0, v_min = 0.0, v_max = 0.0;
    int lo = t, hi = t;
    const bool act = t < m;
    if (act) {
        const unsigned long long k0 = (unsigned long long)s_node[1][t];
        const int64_t leaf = (int64_t)(k0 >> 11);
        const int src = (int)(k0 & 2047);
        const double pa = up.idx ? up.p_alpha[src] : up.c_alpha;
        const double pr = up.idx ? up.p_raw[src] : up.c_raw;
        node = leaf + up.size;
        __stcg(up.sum_tree + node - 1, pa);
        __stcg(up.min_tree + node - 1, pa);
        __stcg(up.max_tree + node - 1, pr);
        v_sum = v_min = pa;
        v_max = pr;
    }
    __syncthreads();                                        // s_node[1] is free again
    // untouched-sibling values of the bottom levels (node index >= 2^kUpdTopLevels): all loads in flight at once
    const int n_bottom = up.levels > kUpdTopLevels - 1 ? up.levels - (kUpdTopLevels - 1) : 0;   // levels 0 .. n_bottom - 1
    double p_sum[kUpdAhead], p_min[kUpdAhead], p_max[kUpdAhead];
#pragma unroll
    for (int w = 0; w < kUpdAhead; ++w) {
        p_sum[w] = p_min[w] = p_max[w] = 0.0;
        if (act && w < n_bottom) {
            const long long sib = ((node >> w) ^ 1) - 1;
            p_sum[w] = __ldcg(up.sum_tree + sib);
            p_min[w] = __ldcg(up.min_tree + sib);
            p_max[w] = __ldcg(up.max_tree + sib);
        }
    }
    const long long leaf_node = node;
    for (int l0 = 0; l0 < up.levels; l0 += kUpdAhead) {
#pragma unroll
        for (int w = 0; w < kUpdAhead; ++w) {
            const int l = l0 + w;
            if (l >= up.levels) break;
            const int buf = l & 1;
            if (act) {
                s_node[buf][t] = node;
                s_sum[buf][t] = v_sum;
                s_min[buf][t] = v_min;
                s_max[buf][t] = v_max;
                s_lo[buf][t] = (short)lo;
                s_hi[buf][t] = (short)hi;
            }
            __syncthreads();
            if (act) {
                const bool is_left = (node & 1) == 0;       // children of p: 2p (left), 2p + 1 (right)
                const int nb = is_left ? hi + 1 : lo - 1;
                const bool touched = nb >= 0 && nb < m && s_node[buf][nb] == (is_left ? node + 1 : node - 1);
                double o_sum, o_min, o_max;
                if (touched) {
                    o_sum = s_sum[buf][nb];
                    o_min = s_min[buf][nb];
                    o_max = s_max[buf][nb];
                    if (is_left) hi = s_hi[buf][nb];
                    else lo = s_lo[buf][nb];
                } else if (l < n_bottom) {
                    o_sum = p_sum[w];                       // (n_bottom <= kUpdAhead is checked by the launcher: l0 == 0 here)
                    o_min = p_min[w];
                    o_max = p_max[w];
                } else {
                    const int sib = (int)(node ^ 1);        // < 2^kUpdTopLevels: the staged copy of the top levels
                    o_sum = s_top[sib];
                    o_min = s_top[(1 << kUpdTopLevels) + sib];
                    o_max = s_top[2 * (1 << kUpdTopLevels) + sib];
                }
                const double l_sum = is_left ? v_sum : o_sum, r_sum = is_left ? o_sum : v_sum;
                const double l_min = is_left ? v_min : o_min, r_min = is_left ? o_min : v_min;
                const double l_max = is_left ? v_max : o_max, r_max = is_left ? o_max : v_max;
                v_sum = __dadd_rn(l_sum, r_sum);            // :72  tree[left] + tree[right]
                v_min = py_min(l_min, r_min);
                v_max = py_max(l_max, r_max);
                node >>= 1;
                if (t == lo) {                              // one writer per node
                    __stcg(up.sum_tree + node - 1, v_sum);
                    __stcg(up.min_tree + node - 1, v_min);
                    __stcg(up.max_tree + node - 1, v_max);
                }
            }
        }
    }
    (void)leaf_node;
    if (t == 0 && up.max_priority_out) *up.max_priority_out = m > 0 ? v_max : __ldcg(up.max_tree);   // :201
}

// large n: separate launches
__global__ void per_update_claim_kernel(UpdateParams up) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= up.n) return;
    const int64_t leaf = upd_leaf(up, i);
    if (leaf < 0 || leaf >= up.size) return;
    atomicMax(up.winner + leaf, (int32_t)(i & 0x7fffffff));
}
__global__ void per_update_leaf_kernel(UpdateParams up) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= up.n) return;
    const int64_t leaf = upd_leaf(up, i);
    if (leaf < 0 || leaf >= up.size) return;
    if (__ldcg(up.winner + leaf) != (int32_t)(i & 0x7fffffff)) return;
    const int64_t node = leaf + up.size - 1;
    up.sum_tree[node] = up.idx ? up.p_alpha[i] : up.c_alpha;
    up.min_tree[node] = up.idx ? up.p_alpha[i] : up.c_alpha;
    up.max_tree[node] = up.idx ? up.p_raw[i] : up.c_raw;
}
__global__ void per_update_reset_kernel(UpdateParams up) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= up.n) return;
    const int64_t leaf = upd_leaf(up, i);
    if (leaf < 0 || leaf >= up.size) return;
    up.winner[leaf] = -1;
}
__global__ void per_update_level_kernel(UpdateParams up, int shift) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= up.n) return;
    const int64_t leaf = upd_leaf(up, i);
    if (leaf < 0 || leaf >= up.size) return;
    // 1-based ancestor `shift` levels above the leaf, then 0-based
    const int64_t parent = ((leaf + up.size) >> shift) - 1;
    recompute_parent(up, parent);
}
__global__ void per_write_max_kernel(const double* max_tree, double* out) { *out = max_tree[0]; }

__global__ void per_init_kernel(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = 2 * size - 1;
    if (i < n) {
        sum_tree[i] = 0.0;                       // Operation.SUM initial_value :52
        min_tree[i] = __longlong_as_double(0x7ff0000000000000LL);   // +inf :51
        max_tree[i] = __longlong_as_double(0xfff0000000000000LL);   // -inf :50
    }
    if (i < size) winner[i] = -1;
}

__global__ void per_priorities_kernel(const double* err, int64_t n, double epsilon, double alpha, double* p_alpha,
                                      double* p_raw, int32_t* neg_flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double e = err[i];
    if (!(e >= 0)) {                           // :195 (negative; NaN too): flag it and mark the entry as "do not apply"
        if (neg_flag) atomicOr(neg_flag, 1);
        p_raw[i] = -1.0;
        p_alpha[i] = -1.0;
        return;
    }
    const double p = __dadd_rn(e, epsilon);    // :197
    p_raw[i] = p;
    p_alpha[i] = pow(p, alpha);                // :198
}

// =====================================================================================================================
// Column gather.
// =====================================================================================================================
constexpr int kStageBytes = 8192;       // smem stage capacity (one chunk of one row)
constexpr int kMaxStages = 32;
constexpr int kBarBytes = kMaxStages * 8;   // mbarrier array at the start of dynamic smem
constexpr int kGatherThreads = 128;
constexpr int kMaxCtaSamples = 16;      // descents a CTA may need for its contiguous item range (fused kernel)

struct BigColumn {
    const uint8_t* src;
    uint8_t* dst;
    int64_t row_bytes;
    int32_t nchunk;
    int32_t chunk_bytes;     // all chunks but the last
    int32_t last_bytes;
    int32_t first_item;      // prefix of nchunk over the preceding big columns
};
struct SmallColumn {
    const uint8_t* src;
    uint8_t* dst;
    int64_t row_bytes;
};
struct GatherParams {
    BigColumn big[CB200_MAX_COLUMNS];
    SmallColumn small[CB200_MAX_COLUMNS];
    int n_big, n_small;
    int items_per_sample;
    int64_t n;               // samples
    int64_t total_items;
    const int64_t* idx;      // plain gather: indices come from memory
    int stages;
    int stage_bytes;         // smem slot size (largest chunk, rounded up to 128 B)
};

// copy `bytes` from src to dst with the widest access the three alignments allow; executed by one warp
__device__ __forceinline__ void warp_copy_row(uint8_t* dst, const uint8_t* src, int64_t bytes, int lane) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src) | (uintptr_t)bytes;
    if ((a & 15) == 0) {
        for (int64_t o = (int64_t)lane * 16; o < bytes; o += 32 * 16) st_stream16(dst + o, ld_stream16(src + o));
    } else if ((a & 3) == 0) {
        for (int64_t o = (int64_t)lane * 4; o < bytes; o += 32 * 4)
            *reinterpret_cast<uint32_t*>(dst + o) = *reinterpret_cast<const uint32_t*>(src + o);
    } else {
        for (int64_t o = lane; o < bytes; o += 32) dst[o] = src[o];
    }
}

// Bulk-copy pipeline executed by ONE thread of the CTA: items [lo, hi) of the flattened (sample, column, chunk) space
// flow global -> smem stage -> global.  `leaf_of(sample)` yields the source row.
template <typename LeafFn>
__device__ __forceinline__ void bulk_pipeline(const GatherParams& gp, int64_t lo, int64_t hi, uint8_t* stage_mem,
                                              uint64_t* full_bar, LeafFn leaf_of) {
    const int S = gp.stages;
    const int64_t cnt = hi - lo;
    auto item_addr = [&](int64_t item, const uint8_t*& src, uint8_t*& dst, uint32_t& bytes) {
        const int64_t sample = item / gp.items_per_sample;
        const int r = (int)(item - sample * gp.items_per_sample);
        int c = 0;
#pragma unroll
        for (int q = 1; q < CB200_MAX_COLUMNS; ++q)
            if (q < gp.n_big && r >= gp.big[q].first_item) c = q;
        const BigColumn& col = gp.big[c];
        const int chunk = r - col.first_item;
        const int64_t off = (int64_t)chunk * col.chunk_bytes;
        bytes = (chunk == col.nchunk - 1) ? (uint32_t)col.last_bytes : (uint32_t)col.chunk_bytes;
        src = col.src + leaf_of(sample) * col.row_bytes + off;
        dst = col.dst + sample * col.row_bytes + off;
    };
    auto issue_load = [&](int64_t k) {
        const int st = (int)(k % S);
        const uint8_t* src;
        uint8_t* dst;
        uint32_t bytes;
        item_addr(lo + k, src, dst, bytes);
        mbar_expect_tx(full_bar + st, bytes);
        bulk_g2s(stage_mem + (size_t)st * gp.stage_bytes, src, bytes, full_bar + st);
    };
    fence_proxy_async_smem();   // the stage memory may have been used through the generic proxy (descent scratch)
    const int64_t pre = cnt < S ? cnt : S;
    for (int64_t k = 0; k < pre; ++k) issue_load(k);
    for (int64_t k = 0; k < cnt; ++k) {
        const int st = (int)(k % S);
        mbar_wait(full_bar + st, (uint32_t)((k / S) & 1));
        const uint8_t* src;
        uint8_t* dst;
        uint32_t bytes;
        item_addr(lo + k, src, dst, bytes);
        fence_proxy_async_smem();
        bulk_s2g(dst, stage_mem + (size_t)st * gp.stage_bytes, bytes);
        bulk_commit();
        // refill the stage whose store was issued one iteration ago (its smem read has had time to drain).  With one
        // stage that stage is this iteration's: its store must finish reading now, and the load of item k + 1 must be
        // in flight before the next wait, or that wait never completes.
        if (S > 1) {
            if (k >= 1 && (k - 1 + S) < cnt) {
                bulk_wait_read<1>();
                issue_load(k - 1 + S);
            }
        } else if (k + 1 < cnt) {
            bulk_wait_read<0>();
            issue_load(k + 1);
        }
    }
    bulk_wait_all<0>();
}

__device__ __forceinline__ void cta_item_range(int64_t total, int64_t& lo, int64_t& hi) {
    lo = total * blockIdx.x / gridDim.x;
    hi = total * (blockIdx.x + 1) / gridDim.x;
}

__device__ __forceinline__ void init_barriers(uint64_t* full_bar, int stages) {
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) mbar_init(full_bar + s, 1);
        fence_mbar_init();
    }
}

// plain gather: indices in memory (uniform ExperienceReplay, or PER after cb200_per_sample)
__global__ void __launch_bounds__(kGatherThreads) gather_bulk_kernel(GatherParams gp) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
    uint8_t* stage_mem = smem + kBarBytes;
    init_barriers(full_bar, gp.stages);
    __syncthreads();
    int64_t lo, hi;
    cta_item_range(gp.total_items, lo, hi);
    if (threadIdx.x == 0 && hi > lo) {
        const int64_t* idx = gp.idx;
        bulk_pipeline(gp, lo, hi, stage_mem, full_bar, [idx](int64_t s) { return __ldg(idx + s); });
    }
}

// small / unaligned columns: one warp per (sample, column)
__global__ void __launch_bounds__(256) gather_small_kernel(GatherParams gp) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t w = warp; w < gp.n * gp.n_small; w += nwarps) {
        const int64_t sample = w / gp.n_small;
        const SmallColumn& col = gp.small[w - sample * gp.n_small];
        const int64_t leaf = __ldg(gp.idx + sample);
        warp_copy_row(col.dst + sample * col.row_bytes, col.src + leaf * col.row_bytes, col.row_bytes, lane);
    }
}

// fused PER sample + gather
__global__ void __launch_bounds__(kGatherThreads) per_sample_gather_kernel(SampleParams sp, GatherParams gp) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
    int64_t* leaf_smem = reinterpret_cast<int64_t*>(smem + kBarBytes);                       // kMaxCtaSamples entries
    double* prio_smem = reinterpret_cast<double*>(smem + kBarBytes + kMaxCtaSamples * 8);    // kMaxCtaSamples entries
    uint8_t* stage_mem = smem + kBarBytes + kMaxCtaSamples * 16;
    init_barriers(full_bar, gp.stages);
    int64_t lo, hi;
    cta_item_range(gp.total_items, lo, hi);
    if (hi <= lo) return;
    const int ips = gp.items_per_sample;
    const int64_t s_lo = lo / ips, s_hi = (hi - 1) / ips;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    // phase A: descents for the samples this CTA touches, one warp each, in parallel (3 memory round trips)
    for (int64_t s = s_lo + warp; s <= s_hi; s += nwarp) {
        const Descent d = per_sample_descend(sp, s, reinterpret_cast<double*>(stage_mem) + warp * kScratchDoubles);
        if (lane == 0) {
            leaf_smem[(s - s_lo) % kMaxCtaSamples] = d.leaf;
            prio_smem[(s - s_lo) % kMaxCtaSamples] = d.priority;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // phase B (one thread): every chunk of this CTA goes in flight at once when the stages allow it
        bulk_pipeline(gp, lo, hi, stage_mem, full_bar,
                      [leaf_smem, s_lo](int64_t s) { return leaf_smem[(s - s_lo) % kMaxCtaSamples]; });
    } else if (warp >= 1 || nwarp == 1) {
        // meanwhile the other warps publish indices / importance weights and move the small columns of the samples
        // whose FIRST item belongs to this CTA (exactly one CTA per sample)
        const int w0 = warp - 1, nw = nwarp - 1;
        for (int64_t s = s_lo + w0; s <= s_hi; s += nw) {
            if (s * ips < lo) continue;
            const int64_t leaf = leaf_smem[(s - s_lo) % kMaxCtaSamples];
            if (lane == 0) per_sample_publish(sp, s, leaf, prio_smem[(s - s_lo) % kMaxCtaSamples]);
            for (int c = 0; c < gp.n_small; ++c) {
                const SmallColumn& col = gp.small[c];
                warp_copy_row(col.dst + s * col.row_bytes, col.src + leaf * col.row_bytes, col.row_bytes, lane);
            }
        }
    }
}

// =====================================================================================================================
// Fused input path of the image agents: PER sample (or given indices) -> gather the uint8 frames of the drawn slots ->
// bf16 plane of their space-to-depth(S) view, the operand format of the first convolution (nn.cu: u8_s2d_planes_kernel
// documents the view: pixel (Y, X) = (y / S, x / S), channel ((y % S) * S + x % S) * C + c, plane row
// (Y * (W / S) + X) * B + b, 8x8 core-tiled).  Replaces: staged uint8 copy written by the gather + two conversion
// passes that re-read it.  HBM traffic: the frames are read once; the planes (2 bytes per pixel value) are written once.
//
// One CTA = 8 consecutive samples (one 8-row group of the plane matrix: every 128-byte core is written whole) x one
// image column x one band of s2d rows.  Phase A: the CTA's 8 warps walk the sum tree for the 8 samples (3 dependent
// round trips, warp_descent).  Phase B: lanes 0..7 of warp 0 stream the band in chunks of `rows_per_chunk` s2d rows --
// one 1-D TMA bulk copy per sample and chunk (rows are contiguous in the ring), three chunks in flight on mbarriers --
// while all 256 threads convert the chunk that has landed: thread = (pixel slot, y % S, b): `S * C` bytes from shared
// memory (conflict-free: the per-sample stride is an odd multiple of 16 bytes) -> bf16 -> two 16-byte stores; the 8 b
// lanes of a quarter-warp complete one 128-byte core.  The band's first CTA also publishes indices / importance
// weights and copies the small columns.
// =====================================================================================================================
constexpr int kS2dThreads = 256;
constexpr int kS2dStages = 2;

struct S2dGatherParams {
    const uint8_t* src[2];     // ring columns (uint8 [capacity, H * W * C])
    uint16_t* plane[2];        // s2d planes [Hs * Ws * B, S * S * C] bf16, core-tiled
    int n_img;
    int64_t row_bytes;         // H * W * C
    int H, W, C, S;
    int B;                     // samples, multiple of 8
    int parts;                 // bands of s2d rows per (group, column)
    int rows_per_chunk;
    int chunk_stride;          // bytes per sample inside a stage (chunk bytes + padding: odd multiple of 16)
    const int64_t* idx_in;     // non-null: indices are given (uniform replay); null: sample the sum tree
    SmallColumn small[CB200_MAX_COLUMNS];
    int n_small;
    // frame-deduplicated ring (non-null `frames`): every H x W frame is stored ONCE in `frames` [frame slots, H * W];
    // src[k] is then the int32 [capacity, C] table of the frame slots that make up the stack of column k
    const uint8_t* frames;
    int frame_sub;             // bytes between the frames of one sample inside a stage (rows_per_chunk * S * W)
    int frame_tma;             // a stack whose 4 frames sit in consecutive slots is fetched by ONE 2-D TMA box (tmF)
};

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::
            "r"(smem_u32(smem_dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}

// tmF (frame-deduplicated ring): the frame store as a 2-D uint32 tensor (H * W / 4 words | frame slots) with box
// (rows_per_chunk * S * W / 4, 4): the bands of four consecutive frames in one operation, landing as [frame][band]
__global__ void __launch_bounds__(kS2dThreads) sample_gather_s2d_kernel(SampleParams sp, S2dGatherParams gp,
                                                                        const __grid_constant__ CUtensorMap tmF) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);                      // [kS2dStages]
    int64_t* leaf_smem = reinterpret_cast<int64_t*>(smem + 64);                  // [8]
    double* prio_smem = reinterpret_cast<double*>(smem + 128);                   // [8]
    uint8_t* stage_mem = smem + 256;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int part = blockIdx.x % gp.parts;
    const int col = (blockIdx.x / gp.parts) % gp.n_img;
    const int group = blockIdx.x / (gp.parts * gp.n_img);
    const int b0 = group * 8;
    const int S = gp.S, C = gp.C, Hs = gp.H / S, Ws = gp.W / S, run = S * C, Cs = S * run;
    const int s2d_row_bytes = S * gp.W * C;                                      // bytes of one s2d row of one sample
    const int per = (Hs + gp.parts - 1) / gp.parts;
    const int y_lo = part * per, y_hi = min(Hs, y_lo + per);
    if (tid == 0) {
        for (int s = 0; s < kS2dStages; ++s) mbar_init(full_bar + s, 1);
        fence_mbar_init();
    }
    // ---- phase A: one warp per sample ----------------------------------------------------------------------------
    {
        const int64_t smp = b0 + warp;
        if (gp.idx_in) {
            if (lane == 0) leaf_smem[warp] = __ldg(gp.idx_in + smp);
        } else {
            const Descent d = per_sample_descend(sp, smp, reinterpret_cast<double*>(stage_mem) + warp * kScratchDoubles);
            if (lane == 0) {
                leaf_smem[warp] = d.leaf;
                prio_smem[warp] = d.priority;
            }
        }
    }
    __syncthreads();
    const int nchunks = y_hi > y_lo ? (y_hi - y_lo + gp.rows_per_chunk - 1) / gp.rows_per_chunk : 0;
    auto issue = [&](int k) {        // executed by warp 0
        const int st = k % kS2dStages;
        const int ya = y_lo + k * gp.rows_per_chunk;
        const int rc = min(gp.rows_per_chunk, y_hi - ya);
        const uint32_t bytes = (uint32_t)(rc * s2d_row_bytes);
        if (lane == 0) mbar_expect_tx(full_bar + st, 8u * bytes);
        __syncwarp();
        if (gp.frames) {
            // lane = (sample, frame of its stack).  The four frames of a stack normally sit in consecutive slots (one
            // new frame per transition): their bands -- rc * S image rows of W bytes each -- then come with ONE 2-D
            // TMA box issued by the sample's first lane; otherwise (episode start: replicated first frame, wrap of the
            // frame store, a partial last chunk) one 1-D bulk copy per frame.
            const int4* fidx = reinterpret_cast<const int4*>(gp.src[col]);
            const uint32_t fbytes = (uint32_t)(rc * S * gp.W);
            const int smp = lane >> 2, c = lane & 3;
            const int4 f = __ldg(fidx + leaf_smem[smp]);
            uint8_t* dst = stage_mem + (size_t)st * 8 * gp.chunk_stride + (size_t)smp * gp.chunk_stride;
            const bool one_box = gp.frame_tma && rc == gp.rows_per_chunk && f.y == f.x + 1 && f.z == f.x + 2 &&
                                 f.w == f.x + 3;
            if (one_box) {
                if (c == 0) tma_load_2d(dst, &tmF, (ya * S * gp.W) >> 2, f.x, full_bar + st);
            } else {
                const int64_t fslot = c == 0 ? f.x : (c == 1 ? f.y : (c == 2 ? f.z : f.w));
                bulk_g2s(dst + (size_t)c * gp.frame_sub,
                         gp.frames + fslot * ((int64_t)gp.H * gp.W) + (size_t)ya * S * gp.W, fbytes, full_bar + st);
            }
        } else if (lane < 8) {
            bulk_g2s(stage_mem + (size_t)st * 8 * gp.chunk_stride + (size_t)lane * gp.chunk_stride,
                     gp.src[col] + leaf_smem[lane] * gp.row_bytes + (size_t)ya * s2d_row_bytes, bytes, full_bar + st);
        }
    };
    if (warp == 0) {
        fence_proxy_async_smem();      // the stage memory served as descent scratch through the generic proxy
        for (int k = 0; k < nchunks && k < kS2dStages; ++k) issue(k);
    } else if (part == 0 && col == 0) {
        // this (group)'s publisher: indices, importance weights, small columns -- off the copy's critical path
        for (int w = warp - 1; w < 8; w += 7) {
            const int64_t smp = b0 + w;
            const int64_t leaf = leaf_smem[w];
            if (lane == 0) {
                if (gp.idx_in == nullptr) per_sample_publish(sp, smp, leaf, prio_smem[w]);
            }
            for (int c = 0; c < gp.n_small; ++c) {
                const SmallColumn& sc = gp.small[c];
                warp_copy_row(sc.dst + smp * sc.row_bytes, sc.src + leaf * sc.row_bytes, sc.row_bytes, lane);
            }
        }
    }
    // ---- phase B: convert the chunks as they land ----------------------------------------------------------------
    const int per_pixel = 8 * S;                             // threads per s2d pixel: (y % S, b)
    const int slots = kS2dThreads / per_pixel;               // pixels converted per pass
    const int within = tid % per_pixel, slot = tid / per_pixel;
    const int dy = within >> 3, b = within & 7;
    uint16_t* plane = gp.plane[col];
    for (int k = 0; k < nchunks; ++k) {
        const int st = k % kS2dStages;
        const int ya = y_lo + k * gp.rows_per_chunk;
        const int rc = min(gp.rows_per_chunk, y_hi - ya);
        if (lane == 0) mbar_wait(full_bar + st, (uint32_t)((k / kS2dStages) & 1));   // one poller per warp
        __syncwarp();
        const uint8_t* sbase = stage_mem + (size_t)st * 8 * gp.chunk_stride + (size_t)b * gp.chunk_stride;
        if (slot < slots) {
            // pixel pi of the chunk: source = row (yl * S + dy) of the sample's band, S * C bytes at X; destination =
            // row group (pix * B + b0) / 8 of the plane matrix, cores (dy * run) / 8 ..., row b of each core.  All
            // strides are loop constants: the pixel index advances by `slots`, the addresses by fixed increments.
            const int npx = rc * Ws;
            const size_t core_stride = (size_t)(gp.B >> 3) * (size_t)(Cs >> 3) * 64;        // plane elements per pixel
            uint16_t* out0 = plane + ((size_t)(b0 >> 3) * (size_t)(Cs >> 3) + (size_t)((dy * run) >> 3)) * 64 + b * 8 +
                             (size_t)ya * Ws * core_stride;
            const int src_row = gp.W * C;                                                  // bytes per image row
            const uint8_t* src0 = sbase + (size_t)dy * src_row;
            int yl = slot / Ws, X = slot - yl * Ws;
            const int dyl = slots / Ws, dX = slots - dyl * Ws;
            for (int pi = slot; pi < npx; pi += slots) {
                const uint8_t* sp8 = src0 + (size_t)yl * S * src_row + X * run;
                uint16_t* o = out0 + (size_t)(yl * Ws + X) * core_stride;
                if (gp.frames) {
                    // planar frames (S == C == 4): 4 pixels of image row yl * S + dy from each of the 4 frames, byte-
                    // transposed into the stack's channel-last order (dx, c)
                    // (the 8 b-lanes of a quarter-warp sit a multiple of 128 bytes apart -- the TMA box needs that
                    // alignment -- i.e. in the same bank: each lane starts with another frame, 2-way conflicts remain)
                    const uint8_t* f = sbase + (size_t)((yl * S + dy) * gp.W + X * S);
                    const int r0 = gp.frame_tma ? (b & 3) : 0;      // (bulk path: odd 16-byte stride, no conflicts)
                    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(f + r0 * gp.frame_sub);
                    const uint32_t a1 = *reinterpret_cast<const uint32_t*>(f + ((r0 + 1) & 3) * gp.frame_sub);
                    const uint32_t a2 = *reinterpret_cast<const uint32_t*>(f + ((r0 + 2) & 3) * gp.frame_sub);
                    const uint32_t a3 = *reinterpret_cast<const uint32_t*>(f + ((r0 + 3) & 3) * gp.frame_sub);
                    // a_k holds frame (r0 + k) & 3
                    const uint32_t w0 = r0 == 0 ? a0 : (r0 == 1 ? a3 : (r0 == 2 ? a2 : a1));
                    const uint32_t w1 = r0 == 0 ? a1 : (r0 == 1 ? a0 : (r0 == 2 ? a3 : a2));
                    const uint32_t w2 = r0 == 0 ? a2 : (r0 == 1 ? a1 : (r0 == 2 ? a0 : a3));
                    const uint32_t w3 = r0 == 0 ? a3 : (r0 == 1 ? a2 : (r0 == 2 ? a1 : a0));
                    const uint32_t t0 = __byte_perm(w0, w1, 0x5140), t1 = __byte_perm(w2, w3, 0x5140);
                    const uint32_t t2 = __byte_perm(w0, w1, 0x7362), t3 = __byte_perm(w2, w3, 0x7362);
                    *reinterpret_cast<uint4*>(o) =
                        u8x8_to_bf16_s2d(__byte_perm(t0, t1, 0x5410), __byte_perm(t0, t1, 0x7632));
                    *reinterpret_cast<uint4*>(o + 64) =
                        u8x8_to_bf16_s2d(__byte_perm(t2, t3, 0x5410), __byte_perm(t2, t3, 0x7632));
                } else if (run == 16) {
                    const uint4 w = *reinterpret_cast<const uint4*>(sp8);
                    *reinterpret_cast<uint4*>(o) = u8x8_to_bf16_s2d(w.x, w.y);
                    *reinterpret_cast<uint4*>(o + 64) = u8x8_to_bf16_s2d(w.z, w.w);
                } else {
                    for (int g = 0; g < run; g += 8) {
                        const uint2 w = *reinterpret_cast<const uint2*>(sp8 + g);
                        *reinterpret_cast<uint4*>(o + (g >> 3) * 64) = u8x8_to_bf16_s2d(w.x, w.y);
                    }
                }
                X += dX;
                yl += dyl;
                if (X >= Ws) {
                    X -= Ws;
                    ++yl;
                }
            }
        }
        __syncthreads();                                     // everyone is done reading this stage
        if (warp == 0 && k + kS2dStages < nchunks) {
            fence_proxy_async_smem();
            issue(k + kS2dStages);
        }
    }
}

// Frame-deduplicated ring, un-fused readers: out[i, pix, c] = frames[fidx[idx[i], c], pix] -- the stacked observation
// the reference materialises with np.stack(frames, axis=-1) (observation_stacking_filter.py:37-41).
__global__ void __launch_bounds__(256) gather_stack_kernel(const uint8_t* __restrict__ frames, int64_t frame_bytes,
                                                           const int32_t* __restrict__ fidx, int K,
                                                           const int64_t* __restrict__ idx, int64_t n,
                                                           uint8_t* __restrict__ out) {
    const int64_t total = n * frame_bytes;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = t / frame_bytes, pix = t - i * frame_bytes;
        const int32_t* fi = fidx + idx[i] * K;
        uint8_t* o = out + t * K;
        for (int c = 0; c < K; ++c) o[c] = frames[(int64_t)__ldg(fi + c) * frame_bytes + pix];
    }
}

// generic row copy used by the ring append: dst row (cursor+i)%capacity <- src row i
__global__ void __launch_bounds__(256) scatter_ring_kernel(uint8_t* ring, const uint8_t* staged, int64_t row_bytes,
                                                           int64_t cursor, int64_t capacity, int64_t n,
                                                           int64_t piece_bytes, int pieces) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t w = warp; w < n * pieces; w += nwarps) {
        const int64_t i = w / pieces;
        const int64_t off = (w - i * pieces) * piece_bytes;
        const int64_t bytes = (off + piece_bytes <= row_bytes) ? piece_bytes : (row_bytes - off);
        if (bytes <= 0) continue;
        const int64_t slot = (cursor + i) % capacity;
        warp_copy_row(ring + slot * row_bytes + off, staged + i * row_bytes + off, bytes, lane);
    }
}

// all columns of a packed staging area in ONE launch: staged record i holds column c at staged[c] + i * staged_stride
struct ScatterPacked {
    uint8_t* ring[CB200_MAX_COLUMNS];
    const uint8_t* staged[CB200_MAX_COLUMNS];
    int64_t row_bytes[CB200_MAX_COLUMNS];
    int piece_start[CB200_MAX_COLUMNS + 1];      // prefix sums of the 4 KB pieces per row
    int n_cols;
    int64_t staged_stride;
};
__global__ void __launch_bounds__(256) scatter_ring_packed_kernel(ScatterPacked sp, int64_t cursor, int64_t capacity,
                                                                  int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int total = sp.piece_start[sp.n_cols];
    for (int64_t w = warp; w < n * total; w += nwarps) {
        const int64_t i = w / total;
        const int pp = (int)(w - i * total);
        int c = 0;
#pragma unroll
        for (int q = 1; q < CB200_MAX_COLUMNS; ++q)
            if (q < sp.n_cols && pp >= sp.piece_start[q]) c = q;
        const int64_t off = (int64_t)(pp - sp.piece_start[c]) * 4096;
        const int64_t bytes = (off + 4096 <= sp.row_bytes[c]) ? 4096 : (sp.row_bytes[c] - off);
        const int64_t slot = (cursor + i) % capacity;
        warp_copy_row(sp.ring[c] + slot * sp.row_bytes[c] + off, sp.staged[c] + i * sp.staged_stride + off, bytes, lane);
    }
}

// ---- host side ------------------------------------------------------------------------------------------------------
#define g_tune_ctas_per_sm (cb200::tune_get("gather_ctas_per_sm", 4, 1, 16))

static int ilog2_exact(int64_t size) {
    int l = 0;
    while (((int64_t)1 << l) < size) ++l;
    return (((int64_t)1 << l) == size) ? l : -1;
}

static int build_gather_params(const cb200_column* cols, int n_columns, int64_t n, GatherParams& gp) {
    gp.n_big = gp.n_small = 0;
    gp.items_per_sample = 0;
    gp.n = n;
    gp.idx = nullptr;
    gp.stages = 1;
    for (int c = 0; c < n_columns; ++c) {
        const cb200_column& col = cols[c];
        if (col.row_bytes <= 0 || !col.src || !col.dst) return -1;
        const bool aligned = (col.row_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(col.src) & 15) == 0) &&
                             ((reinterpret_cast<uintptr_t>(col.dst) & 15) == 0);
        if (aligned && col.row_bytes >= 2048) {
            BigColumn& b = gp.big[gp.n_big++];
            b.src = static_cast<const uint8_t*>(col.src);
            b.dst = static_cast<uint8_t*>(col.dst);
            b.row_bytes = col.row_bytes;
            int64_t nchunk = (col.row_bytes + kStageBytes - 1) / kStageBytes;
            int64_t cb = (((col.row_bytes + nchunk - 1) / nchunk) + 15) / 16 * 16;
            while (cb > kStageBytes) {   // cannot happen, but keep the invariant explicit
                ++nchunk;
                cb = (((col.row_bytes + nchunk - 1) / nchunk) + 15) / 16 * 16;
            }
            nchunk = (col.row_bytes + cb - 1) / cb;
            b.nchunk = (int32_t)nchunk;
            b.chunk_bytes = (int32_t)cb;
            b.last_bytes = (int32_t)(col.row_bytes - cb * (nchunk - 1));
            b.first_item = gp.items_per_sample;
            gp.items_per_sample += (int)nchunk;
        } else {
            SmallColumn& s = gp.small[gp.n_small++];
            s.src = static_cast<const uint8_t*>(col.src);
            s.dst = static_cast<uint8_t*>(col.dst);
            s.row_bytes = col.row_bytes;
        }
    }
    gp.total_items = (int64_t)gp.items_per_sample * n;
    int max_chunk = 16;
    for (int c = 0; c < gp.n_big; ++c) max_chunk = gp.big[c].chunk_bytes > max_chunk ? gp.big[c].chunk_bytes : max_chunk;
    gp.stage_bytes = (max_chunk + 127) / 128 * 128;
    return 0;
}

// grid + stage count: `ctas_per_sm` persistent CTAs per SM share the ~200 KB of shared memory; when the slots suffice
// every chunk of a CTA is loaded at once (the copy then costs one DRAM latency plus the drain).
static unsigned plan_bulk(GatherParams& gp, bool fused) {
    int64_t g = (int64_t)sm_count() * g_tune_ctas_per_sm;
    if (g > gp.total_items) g = gp.total_items;
    if (g < 1) g = 1;
    const int64_t items_per_cta = (gp.total_items + g - 1) / g;
    const int64_t budget = (int64_t)200 * 1024 / g_tune_ctas_per_sm - kBarBytes - (fused ? kMaxCtaSamples * 16 : 0);
    int64_t st = budget / gp.stage_bytes;
    if (st > items_per_cta) st = items_per_cta;
    const int forced = cb200::tune_get("gather_stages", 0, 0, kMaxStages);
    if (forced > 0 && forced < st) st = forced;
    if (st > kMaxStages) st = kMaxStages;
    if (st < 1) st = 1;
    gp.stages = (int)st;
    return (unsigned)g;
}

static size_t gather_smem_bytes(const GatherParams& gp, bool fused) {
    size_t stage = (size_t)gp.stages * gp.stage_bytes;
    const size_t scratch = (size_t)(kGatherThreads / 32) * kScratchDoubles * sizeof(double);   // phase-A alias
    if (fused && stage < scratch) stage = scratch;
    return kBarBytes + (fused ? kMaxCtaSamples * 16 : 0) + stage;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_l2_persist(const void* ptr, int64_t bytes, void* stream) {
    int dev = 0, max_persist = 0, max_window = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    CB200_CUDA(cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev));
    CB200_CUDA(cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev));
    cudaStreamAttrValue attr;
    memset(&attr, 0, sizeof(attr));
    if (ptr == nullptr || bytes <= 0) {
        attr.accessPolicyWindow.num_bytes = 0;     // clear the window
        CB200_CUDA(cudaStreamSetAttribute(as_stream(stream), cudaStreamAttributeAccessPolicyWindow, &attr));
        return CB200_OK;
    }
    if (max_persist <= 0 || max_window <= 0) return CB200_ERR_UNSUPPORTED;
    size_t want = (size_t)bytes;
    if (want > (size_t)max_window) want = (size_t)max_window;
    size_t carve = want < (size_t)max_persist ? want : (size_t)max_persist;
    CB200_CUDA(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve));
    attr.accessPolicyWindow.base_ptr = const_cast<void*>(ptr);
    attr.accessPolicyWindow.num_bytes = want;
    attr.accessPolicyWindow.hitRatio = 1.0f;
    attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    CB200_CUDA(cudaStreamSetAttribute(as_stream(stream), cudaStreamAttributeAccessPolicyWindow, &attr));
    return CB200_OK;
}

int cb200_per_init(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size, void* stream) {
    CB200_CHECK_ARG(sum_tree && min_tree && max_tree && winner, "null pointer");
    CB200_CHECK_ARG(ilog2_exact(size) >= 0, "size must be a positive power of 2");
    const int64_t n = 2 * size - 1;
    CB200_LAUNCH(per_init_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), sum_tree, min_tree, max_tree,
                 winner, size);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

static int run_update(UpdateParams& up, void* stream) {
    cudaStream_t st = as_stream(stream);
    if (up.n <= 0) return CB200_OK;
    if (up.n <= kUpdSortThreads && up.levels <= kUpdTopLevels - 1 + kUpdAhead && tune_get("per_update_sorted", 1, 0, 1)) {
        static bool configured = false;
        if (!configured) {
            CB200_CUDA(cudaFuncSetAttribute(per_update_sorted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            kUpdSortSmem));
            configured = true;
        }
        int threads = 32;
        while (threads < up.n) threads <<= 1;
        CB200_LAUNCH(per_update_sorted_kernel, 1, threads, kUpdSortSmem, st, up);
    } else if (up.n <= 1024) {
        int threads = (int)((up.n + 31) / 32 * 32);
        CB200_LAUNCH(per_update_cta_kernel, 1, threads, 0, st, up);
    } else {
        CB200_CHECK_ARG(up.n < ((int64_t)1 << 31), "n too large");
        const unsigned grid = (unsigned)((up.n + 255) / 256);
        CB200_LAUNCH(per_update_claim_kernel, grid, 256, 0, st, up);
        CB200_LAUNCH(per_update_leaf_kernel, grid, 256, 0, st, up);
        CB200_LAUNCH(per_update_reset_kernel, grid, 256, 0, st, up);
        for (int s = 1; s <= up.levels; ++s) CB200_LAUNCH(per_update_level_kernel, grid, 256, 0, st, up, s);
        if (up.max_priority_out) CB200_LAUNCH(per_write_max_kernel, 1, 1, 0, st, up.max_tree, up.max_priority_out);
    }
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_per_update(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size,
                     const int64_t* idx, const double* p_alpha, const double* p_raw, int64_t n,
                     double* max_priority_out, int32_t* error_flags, void* stream) {
    CB200_CHECK_ARG(sum_tree && min_tree && max_tree && winner, "null tree pointer");
    CB200_CHECK_ARG(n >= 0, "negative n");
    CB200_CHECK_ARG(n == 0 || (idx && p_alpha && p_raw), "null batch pointer");
    const int levels = ilog2_exact(size);
    CB200_CHECK_ARG(levels >= 0, "size must be a positive power of 2");
    UpdateParams up{sum_tree, min_tree, max_tree, winner, size, levels, idx, p_alpha, p_raw, 0, 0.0, 0.0, n,
                    max_priority_out, error_flags};
    return run_update(up, stream);
}

int cb200_per_store(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size,
                    int64_t cursor, int64_t n, double p_alpha, double p_raw, void* stream) {
    CB200_CHECK_ARG(sum_tree && min_tree && max_tree && winner, "null tree pointer");
    const int levels = ilog2_exact(size);
    CB200_CHECK_ARG(levels >= 0, "size must be a positive power of 2");
    CB200_CHECK_ARG(cursor >= 0 && cursor < size && n >= 0, "bad cursor / n");
    CB200_CHECK_ARG(n <= size, "storing more than one full ring per call is not supported");
    UpdateParams up{sum_tree, min_tree, max_tree, winner, size, levels, nullptr, nullptr, nullptr, cursor, p_alpha,
                    p_raw, n, nullptr, nullptr};
    return run_update(up, stream);
}

int cb200_per_priorities_device(const double* err, int64_t n, double epsilon, double alpha, double* p_alpha,
                                double* p_raw, int32_t* neg_flag, void* stream) {
    CB200_CHECK_ARG(n >= 0 && (n == 0 || (err && p_alpha && p_raw)), "bad arguments");
    if (n == 0) return CB200_OK;
    CB200_LAUNCH(per_priorities_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), err, n, epsilon, alpha,
                 p_alpha, p_raw, neg_flag);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_host_priorities(const double* h_err, int64_t n, double epsilon, double alpha, double* h_p_alpha,
                          double* h_p_raw) {
    CB200_CHECK_ARG(n >= 0 && (n == 0 || (h_err && h_p_alpha && h_p_raw)), "bad arguments");
    for (int64_t i = 0; i < n; ++i)
        if (!(h_err[i] >= 0)) {   // negative or NaN, as cb200_per_priorities_device
            set_error("cb200_host_priorities: The priorities must be non-negative values");
            return CB200_ERR_INVALID_ARGUMENT;
        }
    for (int64_t i = 0; i < n; ++i) {
        const double p = h_err[i] + epsilon;
        h_p_raw[i] = p;
        h_p_alpha[i] = pow(p, alpha);   // host libm == what Python's float ** float calls
    }
    return CB200_OK;
}

static int fill_sample_params(SampleParams& sp, const double* sum_tree, const double* min_tree, int64_t size,
                              const double* u, int64_t n, int64_t nt, double beta, int64_t* idx_out, double* w_out,
                              float* w32_out) {
    const int levels = ilog2_exact(size);
    if (levels < 0 || !sum_tree || !min_tree || !u || n <= 0) return -1;
    sp = SampleParams{sum_tree, min_tree, size, levels, u, n, (double)nt, beta, idx_out, w_out, w32_out};
    return 0;
}

int cb200_per_sample(const double* sum_tree, const double* min_tree, int64_t size, const double* u, int64_t n,
                     int64_t nt, double beta, int64_t* idx_out, double* w_out, float* w32_out, void* stream) {
    SampleParams sp;
    CB200_CHECK_ARG(fill_sample_params(sp, sum_tree, min_tree, size, u, n, nt, beta, idx_out, w_out, w32_out) == 0,
                    "bad arguments (size must be a power of 2, n > 0, non-null trees / uniforms)");
    CB200_CHECK_ARG(idx_out != nullptr, "idx_out is required");
    CB200_LAUNCH(per_sample_kernel, (unsigned)((n + 3) / 4), 128, 0, as_stream(stream), sp);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

static int launch_small_gather(const GatherParams& gp, cudaStream_t st) {
    if (gp.n_small == 0) return CB200_OK;
    const int64_t warps = gp.n * gp.n_small;
    unsigned grid = (unsigned)((warps + 7) / 8);
    const unsigned cap = (unsigned)sm_count() * 8;
    if (grid > cap) grid = cap;
    CB200_LAUNCH(gather_small_kernel, grid, 256, 0, st, gp);
    return CB200_OK;
}


int cb200_gather(const cb200_column* h_columns, int n_columns, const int64_t* idx, int64_t n, void* stream) {
    CB200_CHECK_ARG(h_columns && n_columns > 0 && n_columns <= CB200_MAX_COLUMNS, "bad column table");
    CB200_CHECK_ARG(idx && n > 0, "bad idx / n");
    GatherParams gp;
    CB200_CHECK_ARG(build_gather_params(h_columns, n_columns, n, gp) == 0, "bad column entry");
    gp.idx = idx;
    cudaStream_t st = as_stream(stream);
    if (gp.n_big > 0) {
        const unsigned grid = plan_bulk(gp, false);
        const size_t smem = gather_smem_bytes(gp, false);
        static size_t configured = 0;
        if (smem > configured) {
            CB200_CUDA(cudaFuncSetAttribute(gather_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            configured = smem;
        }
        CB200_LAUNCH(gather_bulk_kernel, grid, kGatherThreads, smem, st, gp);
    }
    launch_small_gather(gp, st);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_per_sample_gather(const double* sum_tree, const double* min_tree, int64_t size, const double* u, int64_t n,
                            int64_t nt, double beta, int64_t* idx_out, double* w_out, float* w32_out,
                            const cb200_column* h_columns, int n_columns, void* stream) {
    SampleParams sp;
    CB200_CHECK_ARG(fill_sample_params(sp, sum_tree, min_tree, size, u, n, nt, beta, idx_out, w_out, w32_out) == 0,
                    "bad arguments (size must be a power of 2, n > 0, non-null trees / uniforms)");
    CB200_CHECK_ARG(idx_out != nullptr, "idx_out is required");
    CB200_CHECK_ARG(h_columns && n_columns > 0 && n_columns <= CB200_MAX_COLUMNS, "bad column table");
    GatherParams gp;
    CB200_CHECK_ARG(build_gather_params(h_columns, n_columns, n, gp) == 0, "bad column entry");
    cudaStream_t st = as_stream(stream);
    // a CTA's contiguous item range must not span more than kMaxCtaSamples samples
    const unsigned grid = gp.n_big > 0 ? plan_bulk(gp, true) : 0;
    const bool fusable = gp.n_big > 0 &&
                         ((gp.total_items + grid - 1) / grid + gp.items_per_sample - 1) / gp.items_per_sample + 1 <=
                             kMaxCtaSamples;
    if (!fusable) {
        CB200_LAUNCH(per_sample_kernel, (unsigned)((n + 3) / 4), 128, 0, st, sp);
        CB200_CHECK_LAUNCH();
        return cb200_gather(h_columns, n_columns, idx_out, n, stream);
    }
    const size_t smem = gather_smem_bytes(gp, true);
    static size_t configured = 0;
    if (smem > configured) {
        CB200_CUDA(cudaFuncSetAttribute(per_sample_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem));
        configured = smem;
    }
    CB200_LAUNCH(per_sample_gather_kernel, grid, kGatherThreads, smem, st, sp, gp);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// frame store [slots, frame_bytes] as a 2-D uint32 tensor with box (band_bytes / 4, 4 slots); cached per geometry
static bool frame_store_map(CUtensorMap* out, const void* frames, int64_t frame_bytes, int64_t slots, int band_bytes) {
    static CUtensorMap cached;
    static const void* c_frames = nullptr;
    static int64_t c_bytes = 0, c_slots = 0;
    static int c_band = 0;
    if (c_frames == frames && c_bytes == frame_bytes && c_slots == slots && c_band == band_bytes) {
        *out = cached;
        return true;
    }
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return false;
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    if (frame_bytes % 16 || band_bytes % 16 || band_bytes / 4 > 256 || slots < 4) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)(frame_bytes / 4), (cuuint64_t)slots};
    const cuuint64_t strides[1] = {(cuuint64_t)frame_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)(band_bytes / 4), 4};
    const cuuint32_t estr[2] = {1, 1};
    if (fn(&cached, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<void*>(frames), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return false;
    c_frames = frames; c_bytes = frame_bytes; c_slots = slots; c_band = band_bytes;
    *out = cached;
    return true;
}

static int launch_gather_s2d(const SampleParams& sp, const int64_t* idx_in, int64_t n, const cb200_column* img,
                             int n_img, int h, int w, int c, int s, const cb200_column* small_cols, int n_small,
                             const void* frames, int64_t frame_slots, cudaStream_t st) {
    S2dGatherParams gp;
    memset(&gp, 0, sizeof(gp));
    gp.n_img = n_img;
    gp.row_bytes = (int64_t)h * w * c;
    gp.H = h; gp.W = w; gp.C = c; gp.S = s;
    gp.B = (int)n;
    gp.idx_in = idx_in;
    for (int k = 0; k < n_img; ++k) {
        gp.src[k] = static_cast<const uint8_t*>(img[k].src);
        gp.plane[k] = static_cast<uint16_t*>(img[k].dst);
    }
    gp.n_small = n_small;
    for (int k = 0; k < n_small; ++k) {
        gp.small[k].src = static_cast<const uint8_t*>(small_cols[k].src);
        gp.small[k].dst = static_cast<uint8_t*>(small_cols[k].dst);
        gp.small[k].row_bytes = small_cols[k].row_bytes;
    }
    const int hs = h / s;
    const int s2d_row_bytes = s * w * c;
    // chunks of about 2.7 KB per sample (two stages of 8 samples = 43 KB of shared memory: four CTAs per SM, whose
    // descents / copies / conversions overlap each other); the padded per-sample stride is an odd multiple of 16 bytes
    // bands: as many CTAs as fit in ONE wave of four per SM (a CTA is a chain of dependent round trips -- tree descent,
    // first chunk, conversion -- so a second, partial wave would double the kernel's duration)
    const int groups = (int)(n / 8) * n_img;
    int parts = (4 * sm_count()) / groups;
    if (parts < 1) parts = 1;
    if (parts > hs) parts = hs;
    gp.parts = parts;
    const int per_band = (hs + parts - 1) / parts;
    int rc = 2816 / s2d_row_bytes;
    if (rc < 1) rc = 1;
    if (rc > per_band) rc = per_band;
    gp.rows_per_chunk = rc;
    gp.frames = static_cast<const uint8_t*>(frames);
    gp.frame_sub = rc * s * w;
    int stride = rc * s2d_row_bytes;
    CUtensorMap tmF;
    memset(&tmF, 0, sizeof(tmF));
    // frame store, opt-in (cb200_tune("frame_tma", 1)): per-sample stage regions 128 bytes apart in alignment (TMA box
    // destination) when the tensor map can be built; otherwise (and for the verbatim ring) the padded odd-multiple-of-
    // 16 stride of the bulk-copy path.  The kernel is not bound by the number of copy requests, so the simpler path is
    // the default.
    gp.frame_tma = frames && frame_slots >= 4 && stride % 128 == 0 && tune_get("frame_tma", 0, 0, 1) != 0 &&
                   frame_store_map(&tmF, frames, (int64_t)h * w, frame_slots, rc * s * w);
    if (!gp.frame_tma && (stride / 16) % 2 == 0) stride += 16;
    gp.chunk_stride = stride;
    size_t smem = 256 + (size_t)kS2dStages * 8 * stride;
    const size_t scratch = 256 + 8 * kScratchDoubles * sizeof(double);     // phase A: per-warp descent scratch
    if (smem < scratch) smem = scratch;
    static size_t configured = 0;
    if (smem > configured) {
        if (cudaFuncSetAttribute(sample_gather_s2d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
            cudaSuccess) {
            // more than a CTA can hold: the caller refuses the geometry; clear the error so that the next launch's
            // check does not report it
            cudaGetLastError();
            return -1;
        }
        configured = smem;
    }
    CB200_LAUNCH(sample_gather_s2d_kernel, (unsigned)(groups * parts), kS2dThreads, smem, st, sp, gp, tmF);
    return 0;
}

static int check_s2d_args(const cb200_column* img, int n_img, int64_t n, int h, int w, int c, int s,
                          const cb200_column* small_cols, int n_small, const void* frames) {
    if (!img || n_img < 1 || n_img > 2 || n <= 0 || n % 8 != 0) return -1;
    if (s <= 0 || h % s || w % s || (s * c) % 8 != 0 || ((int64_t)s * w * c) % 16 != 0 || ((int64_t)h * w * c) % 16 != 0)
        return -1;
    // the conversion gives each s2d pixel 8 * s threads: beyond s = 32 a CTA has no thread for a pixel
    if (8 * s > kS2dThreads) return -1;
    if (n_small < 0 || n_small > CB200_MAX_COLUMNS || (n_small > 0 && !small_cols)) return -1;
    // frame-deduplicated ring: 4 x 4 space-to-depth blocks of 4-frame stacks; frames and their row bands 16-byte aligned
    if (frames && (s != 4 || c != 4 || ((int64_t)h * w) % 16 != 0 || ((int64_t)s * w) % 16 != 0 ||
                   (reinterpret_cast<uintptr_t>(frames) & 15)))
        return -1;
    for (int k = 0; k < n_img; ++k)
        if (!img[k].src || !img[k].dst ||
            img[k].row_bytes != (frames ? (int64_t)c * (int64_t)sizeof(int32_t) : (int64_t)h * w * c) ||
            ((reinterpret_cast<uintptr_t>(img[k].src) | reinterpret_cast<uintptr_t>(img[k].dst)) & 15))
            return -1;
    for (int k = 0; k < n_small; ++k)
        if (!small_cols[k].src || !small_cols[k].dst || small_cols[k].row_bytes <= 0) return -1;
    return 0;
}

int cb200_per_sample_gather_s2d(const double* sum_tree, const double* min_tree, int64_t size, const double* u, int64_t n,
                                int64_t nt, double beta, int64_t* idx_out, double* w_out, float* w32_out,
                                const cb200_column* image_columns, int n_image, int32_t h, int32_t w, int32_t c,
                                int32_t s, const cb200_column* small_columns, int n_small, const void* frames,
                                int64_t frame_slots, void* stream) {
    SampleParams sp;
    CB200_CHECK_ARG(fill_sample_params(sp, sum_tree, min_tree, size, u, n, nt, beta, idx_out, w_out, w32_out) == 0,
                    "bad arguments (size must be a power of 2, n > 0, non-null trees / uniforms)");
    CB200_CHECK_ARG(idx_out != nullptr, "idx_out is required");
    CB200_CHECK_ARG(check_s2d_args(image_columns, n_image, n, h, w, c, s, small_columns, n_small, frames) == 0,
                    "bad image geometry / column table (n % 8 == 0, s <= 32, 1-2 uint8 image columns, 16-byte aligned rows)");
    const int rc = launch_gather_s2d(sp, nullptr, n, image_columns, n_image, h, w, c, s, small_columns, n_small,
                                     frames, frame_slots, as_stream(stream));
    CB200_CHECK_ARG(rc == 0, "could not configure the fused sample + gather + space-to-depth kernel");
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_gather_s2d(const int64_t* idx, int64_t n, const cb200_column* image_columns, int n_image, int32_t h, int32_t w,
                     int32_t c, int32_t s, const cb200_column* small_columns, int n_small, const void* frames,
                     int64_t frame_slots, void* stream) {
    CB200_CHECK_ARG(idx != nullptr, "idx is required");
    CB200_CHECK_ARG(check_s2d_args(image_columns, n_image, n, h, w, c, s, small_columns, n_small, frames) == 0,
                    "bad image geometry / column table (n % 8 == 0, s <= 32, 1-2 uint8 image columns, 16-byte aligned rows)");
    SampleParams sp;
    memset(&sp, 0, sizeof(sp));
    const int rc = launch_gather_s2d(sp, idx, n, image_columns, n_image, h, w, c, s, small_columns, n_small, frames,
                                     frame_slots, as_stream(stream));
    CB200_CHECK_ARG(rc == 0, "could not configure the fused gather + space-to-depth kernel");
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_gather_stack(const void* frames, int64_t frame_bytes, const int32_t* frame_index, int32_t stack, const int64_t* idx,
                       int64_t n, void* out, void* stream) {
    CB200_CHECK_ARG(frames && frame_index && idx && out && frame_bytes > 0 && stack > 0 && n > 0, "bad arguments");
    const int64_t total = n * frame_bytes;
    unsigned grid = (unsigned)((total + 255) / 256);
    const unsigned cap = (unsigned)sm_count() * 16;
    if (grid > cap) grid = cap;
    CB200_LAUNCH(gather_stack_kernel, grid, 256, 0, as_stream(stream), static_cast<const uint8_t*>(frames), frame_bytes,
                 frame_index, (int)stack, idx, n, static_cast<uint8_t*>(out));
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_scatter_ring(const cb200_column* h_columns, int n_columns, int64_t cursor, int64_t capacity, int64_t n,
                       void* stream) {
    CB200_CHECK_ARG(h_columns && n_columns > 0 && n_columns <= CB200_MAX_COLUMNS, "bad column table");
    CB200_CHECK_ARG(capacity > 0 && cursor >= 0 && cursor < capacity && n >= 0 && n <= capacity, "bad ring arguments");
    if (n == 0) return CB200_OK;
    cudaStream_t st = as_stream(stream);
    for (int c = 0; c < n_columns; ++c) {
        const cb200_column& col = h_columns[c];
        CB200_CHECK_ARG(col.src && col.dst && col.row_bytes > 0, "bad column entry");
        const int64_t piece = 4096;
        const int pieces = (int)((col.row_bytes + piece - 1) / piece);
        const int64_t warps = n * pieces;
        unsigned grid = (unsigned)((warps + 7) / 8);
        const unsigned cap = (unsigned)sm_count() * 16;
        if (grid > cap) grid = cap;
        CB200_LAUNCH(scatter_ring_kernel, grid, 256, 0, st, static_cast<uint8_t*>(const_cast<void*>(col.src)),
                     static_cast<const uint8_t*>(col.dst), col.row_bytes, cursor, capacity, n, piece, pieces);
    }
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_scatter_ring_packed(const cb200_column* h_columns, int n_columns, int64_t staged_stride, int64_t cursor,
                              int64_t capacity, int64_t n, void* stream) {
    CB200_CHECK_ARG(h_columns && n_columns > 0 && n_columns <= CB200_MAX_COLUMNS, "bad column table");
    CB200_CHECK_ARG(capacity > 0 && cursor >= 0 && cursor < capacity && n >= 0 && n <= capacity && staged_stride > 0,
                    "bad ring arguments");
    if (n == 0) return CB200_OK;
    ScatterPacked sp;
    sp.n_cols = n_columns;
    sp.staged_stride = staged_stride;
    sp.piece_start[0] = 0;
    for (int c = 0; c < n_columns; ++c) {
        const cb200_column& col = h_columns[c];
        CB200_CHECK_ARG(col.src && col.dst && col.row_bytes > 0 && col.row_bytes <= staged_stride, "bad column entry");
        sp.ring[c] = static_cast<uint8_t*>(const_cast<void*>(col.src));
        sp.staged[c] = static_cast<const uint8_t*>(col.dst);
        sp.row_bytes[c] = col.row_bytes;
        sp.piece_start[c + 1] = sp.piece_start[c] + (int)((col.row_bytes + 4095) / 4096);
    }
    for (int c = n_columns; c < CB200_MAX_COLUMNS; ++c) {
        sp.ring[c] = nullptr;
        sp.staged[c] = nullptr;
        sp.row_bytes[c] = 0;
        sp.piece_start[c + 1] = sp.piece_start[n_columns];
    }
    const int64_t warps = n * sp.piece_start[n_columns];
    unsigned grid = (unsigned)((warps + 7) / 8);
    const unsigned cap = (unsigned)sm_count() * 16;
    if (grid > cap) grid = cap;
    CB200_LAUNCH(scatter_ring_packed_kernel, grid, 256, 0, as_stream(stream), sp, cursor, capacity, n);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

}  // extern "C"
