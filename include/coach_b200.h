/*
 * include/coach_b200.h -- C ABI of libcoach_b200.so (hand-written sm_90a CUDA behind Coach's
 * replay-sample -> learn_from_batch hot path).
 *
 * The reference (IntelLabs/coach, rl-coach 1.0.1) is pure Python and has no FFI of its own; its plugin boundary is
 * class substitution through `Parameters.path` strings (rl_coach/memories/memory.py:36-38,
 * rl_coach/agents/dqn_agent.py:64-66).  The Python classes in `coach_b200/` mirror those reference classes and bind
 * to the entry points below with ctypes (see INTEGRATION.md).  Every entry point:
 *   - takes plain device/host pointers, sizes and a CUDA stream handle (`void* stream` = cudaStream_t; NULL = the
 *     legacy default stream); no torch types appear anywhere in this ABI;
 *   - is asynchronous on `stream` unless stated otherwise and never synchronises the device;
 *   - returns CB200_OK (0) or a negative CB200_ERR_* code; `cb200_last_error()` returns a thread-local message.
 * Each declaration cites the reference code (file:line under /root/reference/rl_coach/) whose arithmetic it replaces.
 *
 * Pointers are DEVICE pointers unless the parameter name starts with `h_`.
 */
#ifndef COACH_B200_H
#define COACH_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CB200_ABI_VERSION 1

#define CB200_OK 0
#define CB200_ERR_INVALID_ARGUMENT (-1)
#define CB200_ERR_CUDA (-2)
#define CB200_ERR_UNSUPPORTED (-3)

int cb200_abi_version(void);
const char* cb200_last_error(void);
/* Thread-local name of the kernel the calling thread's last cb200_gemm / cb200_gemm_tiled call launched, e.g.
 * "tc<64,T,u8>+reduce_wide", "tiled<64,N,3,cat>", "tiled<128,T,3>/tma2", "ffma<32,32,N>", "skinny_n": the kernel
 * (template width(s), N / T = plain / transposed A, operand kind or A planes), "/fetch" of a mode-1 tiled call (bulk,
 * tma1 .. tma3 = number of A^T tensor-map classes) and "+reduce_wide|vec|scalar" when a split reduction followed.
 * Lets tests prove which variants they ran; valid until the thread's next call of this function. */
const char* cb200_last_dispatch(void);
/* Number of kernels launched through this library by the calling process so far (bench.py's `gpu_launches`). */
int64_t cb200_launch_count(void);
/* Multiprocessor count and compute capability of the current device (any pointer may be NULL). */
int cb200_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* Runtime switches for benchmark A/B runs (unknown keys are stored and ignored; the removed key "gemm_persistent" --
 * the persistent schedule of cb200_gemm_tiled -- is rejected with CB200_ERR_INVALID_ARGUMENT):
 *   "gather_ctas_per_sm" (persistent gather grid = SMs x this, default 4), "gather_stages" (0 = automatic)
 *   "gemm_tc" (1)          tensor-core (wgmma) path of cb200_gemm; 0 = fp32 CUDA-core kernels only
 *   "gemm_skinny" (1)      dedicated kernels for products with n <= 8 or k <= 8 */
int cb200_tune(const char* key, int value);

/* =====================================================================================================================
 * Segment trees (prioritized replay).  Layout = the reference's: one implicit binary heap per tree, float64,
 * 2*size-1 entries, root at [0], children of p at 2p+1 / 2p+2, leaves at [size-1, 2*size-1); `size` a power of two.
 * memories/non_episodic/prioritized_experience_replay.py:43-156 (SegmentTree).
 * ===================================================================================================================*/

/* Marks [ptr, ptr+bytes) as L2-persisting for kernels subsequently launched on `stream` (stream access-policy window
 * + persisting-L2 carve-out).  Used for the top levels of the sum tree (the first 2^k entries of the heap array are
 * its top k levels), which every sample's descent re-reads while ~100 MB of minibatch traffic per step would
 * otherwise evict them from the 50 MB L2.  ptr == NULL clears the window.  CB200_ERR_UNSUPPORTED if the device has
 * no persisting-L2 support. */
int cb200_l2_persist(const void* ptr, int64_t bytes, void* stream);

/* SegmentTree.__init__ :54-61 -- sum tree <- 0, min tree <- +inf, max tree <- -inf. `winner` (int32[size]) is the
 * scratch array used by cb200_per_update for last-writer-wins duplicate resolution; it is set to -1. */
int cb200_per_init(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size, void* stream);

/* PrioritizedExperienceReplay.update_priorities :203-217 + _update_priority :188-201 + SegmentTree.update/_propagate
 * :116-129,:63-74, for a whole batch at once.  Leaf idx[i] of the sum and min trees receives p_alpha[i], of the max
 * tree p_raw[i]; duplicates resolve last-writer-wins in batch order (the reference applies them sequentially); every
 * ancestor is then recomputed as op(left, right) level by level, which is bit-identical to the sequential reference
 * because parents are recomputed, never incrementally adjusted.  `max_priority_out` (device double, may be NULL)
 * receives max_tree[0] (= self.maximal_priority, :201).  n <= 1024 runs as ONE launch of one CTA that sorts the batch's
 * leaves in shared memory and walks all paths bottom-up without global round trips between levels; larger n uses one
 * launch per tree level.  Entries that must not be applied are skipped: a leaf outside [0, size) (the reference raises
 * ValueError :124-126; here bit 1 of *error_flags, device int32, may be NULL, is set) and entries whose p_alpha is
 * negative (the marker cb200_per_priorities_device leaves for a negative / NaN error). */
int cb200_per_update(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size,
                     const int64_t* idx, const double* p_alpha, const double* p_raw, int64_t n,
                     double* max_priority_out, int32_t* error_flags, void* stream);

/* priority = error + epsilon; p_raw = priority; p_alpha = priority ** alpha  (:197-200) computed ON DEVICE with CUDA's
 * pow (<= 2 ulp; glibc's pow, which the reference uses, is not correctly rounded either, so device and reference
 * can differ in the last bit of ~0.1% of leaves -- see cb200_host_priorities for the libm-exact route).
 * Bit 0 of *neg_flag (device int32, may be NULL) is set if any err[i] is negative or NaN (the reference raises
 * ValueError :195); such entries get p_alpha = p_raw = -1, which cb200_per_update skips, so an invalid error can never
 * reach the trees. */
int cb200_per_priorities_device(const double* err, int64_t n, double epsilon, double alpha, double* p_alpha,
                                double* p_raw, int32_t* neg_flag, void* stream);

/* Same arithmetic with the host's libm `pow` -- bit-identical to the reference on the same machine.  Synchronous,
 * HOST pointers; the agent overlaps it with the network backward pass.  Returns CB200_ERR_INVALID_ARGUMENT (and
 * processes nothing) if an error value is negative or NaN. */
int cb200_host_priorities(const double* h_err, int64_t n, double epsilon, double alpha, double* h_p_alpha,
                          double* h_p_raw);

/* PrioritizedExperienceReplay.store :264-283 + SegmentTree.add :102-114 for n consecutive transitions starting at
 * ring cursor `cursor` (wraps at size): every new leaf gets p_alpha (sum, min) / p_raw (max) where the caller passes
 * p_raw = maximal_priority and p_alpha = maximal_priority ** alpha. */
int cb200_per_store(double* sum_tree, double* min_tree, double* max_tree, int32_t* winner, int64_t size,
                    int64_t cursor, int64_t n, double p_alpha, double p_raw, void* stream);

/* PrioritizedExperienceReplay.sample :229-253 + SegmentTree._retrieve :76-92 for `n` samples.
 *   u[i]        raw random.random() draws (the host keeps Python's MT19937 stream; random.uniform(a,b)=a+(b-a)*u)
 *   nt          num_transitions() -- the reference's doubled count (store appends twice, :271/:280)
 *   idx_out     int64[n]  leaf indices (bit-exact)
 *   w_out       double[n] normalised importance weights ((nt*P)^-beta / max_w); w32_out float[n] the same rounded
 *               once to fp32 (what the TF placeholder receives); either may be NULL
 * One warp per sample; each round fetches a 7-level sub-tree (254 nodes, 8 coalesced loads per lane) into a per-warp
 * shared-memory scratch and replays the reference's comparisons from it, so a 2^20-leaf descent costs 3 dependent
 * memory round trips instead of 20. */
int cb200_per_sample(const double* sum_tree, const double* min_tree, int64_t size, const double* u, int64_t n,
                     int64_t nt, double beta, int64_t* idx_out, double* w_out, float* w32_out, void* stream);

/* =====================================================================================================================
 * Transition columns.  The replay ring is struct-of-arrays in HBM: one row-major [capacity, row_bytes] byte matrix
 * per transition field (state, next_state, action, reward, game_over, ...).  Replaces the AoS->SoA gather of
 * core_types.py:488-623 (Batch.states/next_states/actions/rewards/game_overs) and the list indexing of
 * experience_replay.py:90.
 * ===================================================================================================================*/
#define CB200_MAX_COLUMNS 8

typedef struct cb200_column {
    const void* src;     /* [capacity, row_bytes] ring column                                         */
    void* dst;           /* [n, row_bytes] staged minibatch column                                    */
    int64_t row_bytes;   /* bytes per transition in this column                                       */
} cb200_column;

/* dst[c][i, :] = src[c][idx[i], :] for every column c.  Rows that are 16-byte multiples and >= 2 KiB move through
 * shared memory with 1-D bulk async copies (TMA: cp.async.bulk global->shared->global, mbarrier completion) from a
 * persistent grid; smaller / unaligned rows use vectorised LSU copies. */
int cb200_gather(const cb200_column* h_columns, int n_columns, const int64_t* idx, int64_t n, void* stream);

/* Fused PER sample + gather (one launch): cb200_per_sample followed by cb200_gather on the freshly drawn indices
 * without leaving the kernel. */
int cb200_per_sample_gather(const double* sum_tree, const double* min_tree, int64_t size, const double* u, int64_t n,
                            int64_t nt, double beta, int64_t* idx_out, double* w_out, float* w32_out,
                            const cb200_column* h_columns, int n_columns, void* stream);

/* Fused input path of the image agents (one launch): PER sample -> gather the uint8 frames of the drawn slots -> bf16
 * plane of their space-to-depth(s) view, i.e. the operand of the first convolution (cb200_u8_s2d_planes documents the
 * view and the plane format).  Replaces, for the image columns, the staged uint8 copy of cb200_per_sample_gather
 * (memories/non_episodic/prioritized_experience_replay.py:219-262 + core_types.py:488-511) AND the conversion passes
 * over it (embedders/embedder.py:103 input rescale is applied by the GEMM, see cb200_tgemm_desc.a_u8_div).
 *   image_columns[k]: src = ring column (uint8 [capacity, h*w*c]), dst = plane (bf16 [(h/s)*(w/s)*n, s*s*c],
 *                     core-tiled), row_bytes = h*w*c; 1 or 2 columns (state, next_state)
 *   small_columns   : the remaining columns, copied row by row into their staged [n, row_bytes] buffers
 * n must be a multiple of 8 (whole 8-row groups of the plane matrix).  s is at most 32 (8*s threads convert one s2d
 * pixel, 256 per CTA), and an s2d row of s*w*c bytes above about 14.5 KB needs more than the 227 KiB of shared memory
 * a CTA can hold: both are refused (CB200_ERR_INVALID_ARGUMENT).  idx_out / w_out / w32_out as cb200_per_sample.
 * Frame-deduplicated ring (`frames` != NULL, s == c == 4): the ring stores every h x w frame ONCE in `frames`
 * (uint8 [frame slots, h*w]) -- the reference shares them between s, s' and neighbouring transitions through LazyStack
 * (filters/observation/observation_stacking_filter.py:27-41, agents/agent.py:905-973); image_columns[k].src is then the
 * int32 [capacity, c] table of the frame slots of each transition's stack (row_bytes = 4*c) and the kernel assembles
 * the last-axis stack while converting; frame_slots = rows of `frames` (a stack in four consecutive slots is fetched
 * by one 2-D TMA box per chunk). */
int cb200_per_sample_gather_s2d(const double* sum_tree, const double* min_tree, int64_t size, const double* u, int64_t n,
                                int64_t num_transitions, double beta, int64_t* idx_out, double* w_out, float* w32_out,
                                const cb200_column* image_columns, int n_image, int32_t h, int32_t w, int32_t c,
                                int32_t s, const cb200_column* small_columns, int n_small, const void* frames,
                                int64_t frame_slots, void* stream);

/* The same for given slot indices (uniform ExperienceReplay.sample, experience_replay.py:71-93). */
int cb200_gather_s2d(const int64_t* idx, int64_t n, const cb200_column* image_columns, int n_image, int32_t h, int32_t w,
                     int32_t c, int32_t s, const cb200_column* small_columns, int n_small, const void* frames,
                     int64_t frame_slots, void* stream);

/* Frame-deduplicated ring, un-fused readers (Batch.states() of the slots idx, core_types.py:488-511):
 * out[i, pix, c] = frames[frame_index[idx[i], c], pix], i.e. np.stack(frames, axis=-1) of observation_stacking_filter.py:
 * 37-41 as a uint8 [n, frame_bytes, stack] array. */
int cb200_gather_stack(const void* frames, int64_t frame_bytes, const int32_t* frame_index, int32_t stack, const int64_t* idx,
                       int64_t n, void* out, void* stream);

/* Ring append: src[c][(cursor + i) % capacity, :] = staged[c][i, :] (experience_replay.py:131-150 store; the
 * `cb200_column.src` member is the ring (written), `.dst` the staged rows (read)). */
int cb200_scatter_ring(const cb200_column* h_columns, int n_columns, int64_t cursor, int64_t capacity, int64_t n,
                       void* stream);

/* Same append for a PACKED staging area, all columns in one launch: column c of staged record i is at
 * h_columns[c].dst + i * staged_stride (the host staging area of DeviceRing.store is one pinned record per transition,
 * so a flush is one H2D copy and one kernel). */
int cb200_scatter_ring_packed(const cb200_column* h_columns, int n_columns, int64_t staged_stride, int64_t cursor,
                              int64_t capacity, int64_t n, void* stream);


/* =====================================================================================================================
 * Learn step: dense contractions.  One primitive ("gather-GEMM") covers conv forward (implicit im2col over NHWC),
 * conv weight / data gradients and dense forward / backward:
 *
 *      C[m, n] = epilogue( sum_r A(m, r) * B(r, n) ),      A(m, r) = a_src[ a_rowoff[m] + a_coloff[r] ]   (elements)
 *
 * Replaces the TensorFlow ops behind architectures/tensorflow_components/layers.py:108-183 (Conv2d / Dense),
 * embedders/embedder.py:95-124 (x / 255 input rescale, via a_lut) and tf.gradients over them
 * (architectures/tensorflow_components/architecture.py:193).  fp32 FFMA, deterministic (fixed reduction order).
 * ===================================================================================================================*/
#define CB200_ACT_NONE 0
#define CB200_ACT_RELU 1
#define CB200_ACT_TANH 2

typedef struct cb200_gemm_desc {
    /* A operand */
    const void* a_src;          /* fp32 (a_lut == NULL) or uint8 (value = a_lut[byte]) element array                */
    const float* a_lut;         /* 256-entry table, e.g. lut[v] = (float)v / 255.0f                                  */
    const int32_t* a_rowoff;    /* [a_rows] element offset contributed by the row index                              */
    const int32_t* a_coloff;    /* [a_cols] element offset contributed by the column (reduction) index               */
    const int32_t* a_rowinfo;   /* optional (i << 16 | j) per row   } A(m, r) = 0 unless 0 <= i - a < a_oh and       */
    const int32_t* a_colinfo;   /* optional (a << 16 | b) per col   }                    0 <= j - b < a_ow           */
    int32_t a_oh, a_ow;
    int32_t a_rows, a_cols;     /* logical extent of A                                                              */
    int32_t a_transposed;       /* 0: C[a_rows, N] = A * B   (reduction over a_cols)                                */
                                /* 1: C[a_cols, N] = A^T * B (reduction over a_rows; weight gradients)              */
    /* B operand: row-major [R, N] */
    const float* b;
    int32_t ldb;
    int32_t n;
    /* output / epilogue */
    float* c;                   /* [rows, ldc]                                                                       */
    int32_t ldc;
    const float* bias;          /* [n] or NULL                                                                       */
    int32_t act;                /* CB200_ACT_* applied after the bias                                                */
    const float* mask_y;        /* optional, indexed like c: c = value * act'(mask_y) with act' from the activation  */
    int32_t mask_act;           /*   OUTPUT (relu: y > 0, tanh: 1 - y*y) -- fuses the activation backward            */
    const int32_t* c_rowmap;    /* optional output row remap (transposed-conv stride classes)                        */
    int32_t accumulate;         /* c += value instead of c = value                                                   */
    /* split reduction */
    float* workspace;           /* >= splits * rows * n floats when splits > 1                                       */
    int32_t splits;             /* 0 / 1 = no split; k > 1 = k partial sums reduced in fixed order                   */
    /* fast-path hints (the tables are built by the caller, who knows their structure) */
    int32_t a_vec4;             /* 1: every aligned group of 4 column indices is contiguous in memory, a_cols % 4 == 0 */
                                /*    and every a_rowoff % 4 == 0  => 128-bit (fp32) / 32-bit (uint8) operand loads;  */
                                /*    a_colinfo must then be equal within each such group (the mask is per group)     */
    int32_t a_ones_col;         /* a_transposed only: 1 = append an output row a_cols holding sum_m B[m, :] (the bias  */
                                /*    gradient lands in c[a_cols, :], i.e. right behind the kernel gradient)          */
    float a_u8_div;             /* uint8 A only, 0 = not declared: the caller states a_lut[v] == (float)v / a_u8_div.  */
                                /*    The tensor-core path then contracts the raw integers (exact in bf16) and divides */
                                /*    each accumulated sum by a_u8_div once; other paths read a_lut and ignore this.   */
    /* bf16 operand planes (hi, mid, lo; x == hi + mid + lo exactly) in the 8x8 core-tiled format: a [rows, cols]    */
    /* matrix stores element (r, c) of plane p at                                                                    */
    /*     planes + p * plane_stride + ((r / 8) * (cols / 8) + c / 8) * 64 + (r % 8) * 8 + c % 8                     */
    /* Activations / gradients use rows = pixel * batch + b.  Consumed natively by cb200_gemm_tiled; this entry point */
    /* can read B planes (conv1: weights, dY) and write the planes of its result.                                    */
    const void* b_planes;       /* planes of b [R, n] (ldb == n)                                                     */
    int64_t b_plane_stride;
    int32_t b_prow_npix;        /* > 0: reduction row r = b * npix + q (NHWC) is plane row q * b_prow_batch + b       */
    int32_t b_prow_batch;
    void* c_planes;             /* if set, the epilogue also writes the planes of the final c values                */
    int64_t c_plane_stride;
    int32_t c_plane_cols;       /* columns of the plane matrix (= n)                                                */
    int32_t c_prow_npix;        /* > 0: output row m = b * npix + q is plane row q * c_prow_batch + b; 0: row m       */
    int32_t c_prow_batch;
    int32_t a_lda;              /* > 0: A is a plain row-major fp32 matrix with this leading dimension (the tables   */
                                /*    say the same); lets products with n <= 8 or a_cols <= 8 take the skinny kernels */
} cb200_gemm_desc;

int cb200_gemm(const cb200_gemm_desc* h_desc, void* stream);

/* =====================================================================================================================
 * Tensor-core GEMMs on pre-split operands (csrc/nn_gemm_tiled.cuh).  Convolutions and dense layers as "multi-tap"
 * contractions over plane matrices (rows = pixel * batch + b, cols = channels; weights = stacks of [a_cols, n] blocks):
 *   mode 0: C[q * B + b, :] = sum over the tap list of output pixel q, entries (a_pix, w_blk):
 *                                A[a_pix * B + b, :] * W[w_blk]                (forward, data gradient)
 *   mode 1: C[t * a_cols + c, :] = sum_q sum_b A[a_pix[t * num_q + q] * B + b, c] * G[q * B + b, :]   (weight gradient)
 * Replaces, for layers whose input already lives on the device as planes, the same reference code as cb200_gemm
 * (layers.py:108-183 forward, tf.gradients backward).  Operands move by 1-D bulk copies (TMA); 3xBF16 products with
 * fp32 accumulation (wgmma), at most 32 reduction chunks of 32 per launch slice (use `splits`).
 * ===================================================================================================================*/
typedef struct cb200_tgemm_desc {
    int32_t mode;
    int32_t batch;              /* B, multiple of 32                                                                 */
    const void* a_planes;       /* planes of A [a_pixels * B, a_cols]                                                */
    int64_t a_plane_stride;
    int32_t a_cols;             /* 32, 64, 128 or a multiple of 128                                                  */
    const void* b_planes;       /* mode 0: weight blocks [blocks][a_cols, n];  mode 1: G [num_q * B, n]               */
    int64_t b_plane_stride;
    int32_t n;                  /* 32 or a multiple of 64                                                            */
    const int32_t* list_ptr;    /* mode 0: [num_q + 1] offsets into list                                             */
    const int32_t* list;        /* mode 0: pairs (a_pix, w_blk)                                                      */
    int32_t max_list_len;       /* mode 0: longest tap list                                                          */
    const int32_t* a_pix;       /* mode 1: [taps * num_q] input pixel under tap t at output pixel q                  */
    int32_t num_q;
    int32_t taps;
    /* output / epilogue: as in cb200_gemm_desc; rows of C are q * B + b (mode 0) or t * a_cols + c (mode 1)          */
    /* c may be NULL when c_planes is set: only the planes of the result are produced (forward-only networks)         */
    float* c;
    int32_t ldc;
    const float* bias;
    int32_t act;
    const float* mask_y;
    int32_t mask_act;
    const int32_t* c_rowmap;    /* e.g. q * B + b -> b * num_q + q to store NHWC                                      */
    float* workspace;
    int32_t splits;
    void* c_planes;             /* tiled planes of C with plane row = C row, c_plane_cols == n                       */
    int64_t c_plane_stride;
    int32_t c_plane_cols;
    const void* mask_planes;    /* optional, instead of mask_y: the masking activation as tiled planes with the geometry */
    int64_t mask_plane_stride;  /*    of the result (rows q * B + b, n columns); c_plane_cols must be set to n            */
    int32_t bias_row;           /* mode 1: 1 = also produce row taps * a_cols = sum over all rows of G (the bias gradient, */
                                /*    stored right behind the kernel gradient); c / workspace / c_rowmap have one more row  */
    int32_t a_num_planes;       /* 3 (0 = 3): fp32 split;  1: A holds raw uint8 values as ONE exact bf16 plane, every    */
    float a_u8_div;             /*    accumulated sum is divided by a_u8_div (x / 255 input rescale, embedder.py:103)  */
    int64_t a_rows;             /* rows of the A plane matrix (a_pixels * B) and of the B operand's plane matrix      */
    int64_t b_rows;             /*   (mode 0: blocks * a_cols, mode 1: num_q * B): bounds of the TMA tensor maps      */
    int32_t b_interleaved;      /* mode 0, n <= 64 (or n % 128 != 0): the B planes are "row-group interleaved" --        */
                                /*   (row group | plane | column core | 64), written with plane_stride -1 by              */
                                /*   cb200_split_planes (segment layout 1) / cb200_permute_f32 -- and the 3xBF16 product  */
                                /*   set reads its three B planes from that one [b1|b2|b3] operand                         */
    const int32_t* a_pix_host;  /* mode 1, optional: HOST copy of a_pix.  When the taps that share a 128-row tile of the   */
                                /*   result sit a constant number of pixels apart (at most three distinct strides over   */
                                /*   the tiles: every convolution of the path), the A^T operand of a reduction chunk is  */
                                /*   ONE 5-D TMA box (64 | cores | taps | row groups | planes) instead of one 1-D bulk   */
                                /*   copy per (plane, tap, row group); NULL: bulk copies                                 */
    /* private: TMA tensor maps of the operands, built by the first call with this descriptor (keep the descriptor    */
    /* alive and unchanged between calls; zero-initialise)                                                            */
    uint64_t tmap_key;
    int32_t a_tma;              /* private: number of A^T tensor maps in use (0: bulk copies)                           */
    uint8_t a_tile_class[64];   /* private: tensor map of each 128-row tile                                             */
    uint8_t tmap_storage[4 * 128 + 64];
} cb200_tgemm_desc;

int cb200_gemm_tiled(const cb200_tgemm_desc* h_desc, void* stream);

/* uint8 NHWC frames [batch, h, w, c] -> one exact bf16 plane of the space-to-depth(s) view: plane row
 * ((y / s) * (w / s) + x / s) * batch + b, column ((y % s) * s + x % s) * c + ch; [h/s * w/s * batch, s*s*c] tiled.
 * Turns the strided first convolution (Atari: 8x8 stride 4 on 84x84x4) into a 2x2 stride-1 one on 64 channels. */
int cb200_u8_s2d_planes(const void* x, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t s, void* plane,
                        void* stream);

/* fp32 row-major matrices -> tiled planes, one launch for a list of matrices inside one fp32 buffer (the parameter
 * buffer, once per step): d_segments[k] = {src offset, rows, cols, plane offset, layout} in elements (device memory);
 * layout 0: three planes `plane_stride` apart; layout 1: row-group interleaved planes (cb200_tgemm_desc.b_interleaved),
 * the segment occupies 3 * rows * cols elements from its plane offset. */
int cb200_split_planes(const float* src, void* planes, int64_t plane_stride, const int64_t* d_segments,
                       int32_t num_segments, int64_t max_segment_elems, void* stream);

/* out[j] = sum_i x[i, j] for x [rows, cols] (bias gradients: tf.gradients wrt the bias of Dense / Conv2d), reduced in a
 * fixed order (two deterministic stages; `workspace` >= 1024 * cols floats). */
int cb200_colsum(const float* x, int64_t rows, int64_t cols, float* out, float* workspace, void* stream);

/* dst[i] = src[table[i]], i < n  (fp32; static permutations of weight tensors for the data-gradient GEMMs, e.g. the
 * per-stride-class [taps*N, Cin] matrices of the transposed convolution) */
/* (plane_stride -1: row-group interleaved planes, see cb200_tgemm_desc.b_interleaved) */
int cb200_permute_f32(const float* src, const int32_t* table, int64_t n, float* dst, void* dst_planes,
                      int64_t plane_stride, int32_t plane_cols, void* stream);
                      /* dst_planes optional (NULL): also write dst, seen as [n / plane_cols, plane_cols], as planes */

/* dst[c, r] = src[r, c]  (fp32; pre-transposition of weight matrices for the data-gradient GEMMs).
 * dst_planes optional (NULL): also write dst [cols, rows] as core-tiled planes `plane_stride` apart; needs rows % 8 == 0
 * (whole column cores), plane_stride % 8 == 0 and plane_stride >= rows * cols rounded up to a multiple of 8 rows.  When
 * cols % 8 != 0 the rows of the last row group past cols are not written. */
int cb200_transpose(const float* src, int64_t rows, int64_t cols, float* dst, void* dst_planes, int64_t plane_stride,
                    void* stream);


/* =====================================================================================================================
 * Learn step: element-wise / reduction kernels.
 * ===================================================================================================================*/

/* DQNAgent.learn_from_batch, agents/dqn_agent.py:92-103 (+ ddqn_agent.py:42-43 action selection):
 *   a*_i   = argmax_a q_select[i, a]                     (first maximum, np.argmax)
 *   y_i    = r_i + (1.0 - done_i) * discount * q_next[i, a*_i]        evaluated in fp64 like the Python loop
 *   err_i  = |y_i - q_online[i, act_i]|  (fp64)          -> td_err_out (the new priorities' input)
 *   targets = copy of q_online with targets[i, act_i] = (float) y_i
 * q_select = q_next for DQN, Q_online(s') for DDQN. */
int cb200_dqn_td_targets(const float* q_next, const float* q_select, const float* q_online, const int64_t* actions,
                         const double* rewards, const uint8_t* game_overs, double discount, int64_t batch,
                         int64_t n_actions, float* targets_out, double* td_err_out, void* stream);

/* Generic head loss of heads/head.py:165-177 for a Q / V style regression head:
 *   loss = mean_b( loss_weight * w_b * sum_a l(target_ba, out_ba) ),  l = Huber(delta=1) (tf.losses.huber_loss,
 *   q_head.py:44-45) or squared error (tf.losses.mean_squared_error);  w = importance weights (NULL => ones).
 *   d_out[b, a] = loss_weight * w_b / batch * l'(out_ba - target_ba)
 * loss_out: device float (fixed-order reduction). */
int cb200_regression_head_loss_grad(const float* out, const float* target, const float* weights, int64_t batch,
                                    int64_t width, int huber, float loss_weight, float* d_out, float* loss_out,
                                    void* stream);

/* Fused DQN / DDQN Q-head step: Q(s') of the target head, Q(s) [and Q(s'), DDQN] of the online head (q_head.py:52-54),
 * TD targets / errors (agents/dqn_agent.py:92-103, ddqn_agent.py:42-43; fp64, bit-exact given the Q values), Huber / MSE
 * head loss and dL/dQ (heads/head.py:165-177), and the head's backward pass: dL/dW, dL/db and the gradient w.r.t. the
 * feature layer's pre-activation (dQ W^T masked with relu'(h)), as fp32 and / or as operand planes.  Two launches
 * instead of the eight or nine of cb200_gemm x 5 + cb200_dqn_td_targets + cb200_regression_head_loss_grad. */
typedef struct cb200_dqn_head_desc {
    const float* h_next;        /* [batch, features] post-ReLU features of s' from the TARGET network                      */
    const float* h_online;      /* [batch, features] features of s from the online network                                */
    const float* h_select;      /* DDQN: features of s' from the ONLINE network (action selection); NULL for DQN          */
    const float* w_target;      /* target head kernel [features, n_actions] and bias                                      */
    const float* b_target;
    const float* w_online;
    const float* b_online;
    const int64_t* actions;     /* [batch]                                                                                 */
    const double* rewards;
    const uint8_t* game_overs;
    const float* weights;       /* importance weights [batch] or NULL                                                     */
    double discount;
    int32_t huber;              /* 1: tf.losses.huber_loss(delta 1), 0: mean squared error                                */
    int64_t batch;
    int32_t features;           /* 256 or 512                                                                              */
    int32_t n_actions;          /* <= 8                                                                                    */
    float* q_online;            /* out [batch, n_actions]                                                                  */
    float* q_next;              /* out, optional                                                                           */
    float* targets;             /* out [batch, n_actions]: Q(s) with the taken action's entry replaced by the TD target    */
    double* td_err;             /* out [batch]: |target - Q(s, a)| (the PER priorities' errors)                           */
    float* dq;                  /* out [batch, n_actions]: dL/dQ                                                           */
    float* loss;                /* out scalar, optional                                                                    */
    float* dh;                  /* out, optional: [batch, features] dL/d(pre-activation of the feature layer)             */
    void* dh_planes;            /* out, optional: the same as tiled bf16 hi / mid / lo planes                              */
    int64_t dh_plane_stride;
    float* dw;                  /* out [features, n_actions]: gradient of the online head kernel                          */
    float* db;                  /* out [n_actions]                                                                         */
    float* workspace;           /* ceil(batch / 16) * 8 * (features * n_actions + n_actions + 1) floats                    */
    /* Target rule of the taken action (CB200_TARGET_*); a zero-initialised tail means DQN / DDQN.  Every rule selects
     * a* = argmax Q_online(s') (first maximum; h_select required) and starts from the fp64 double-DQN target
     * y = r + ((1 - done) discount) Q_target(s')[a*], bit-exact given the Q values:
     *   MMC (mmc_agent.py:63-78):  target = (float)((1 - rho) y + rho R), fp64, R = mc_returns[i]
     *   PAL (pal_agent.py:70-106): t0 = (float)y; adv = max Qt(s) - Qt(s)[a]; nadv = max Qt(s') - Qt(s')[a*];
     *     m = adv (PAL) or min(adv, nadv) (persistent: nadv only when strictly smaller); t1 = t0 - (float)alpha m;
     *     t2 = (float)(1 - rho) t1; target = (float)((double)t2 + rho R) -- fp32 steps, as numpy evaluates them.
     * td_err is |target - Q(s, a)| of the final target for these rules.  Under every rule, a row whose action is outside
     * [0, n_actions) keeps Q(s) as its targets (dL/dQ = 0) and gets td_err = 0. */
    int32_t target_rule;
    const float* h_target_s;    /* PAL: [batch, features] features of s from the TARGET network                            */
    const double* mc_returns;   /* MMC / PAL: [batch] Monte Carlo returns (the replay's n_step_discounted_rewards)         */
    double pal_alpha;
    double mc_mixing_rate;      /* rho                                                                                     */
    float* q_select;            /* out, optional (MMC / PAL): [batch, n_actions] Q_online(s')                              */
    float* q_target_s;          /* out, optional (PAL): [batch, n_actions] Q_target(s)                                     */
} cb200_dqn_head_desc;

#define CB200_TARGET_DQN 0
#define CB200_TARGET_MMC 1
#define CB200_TARGET_PAL 2
#define CB200_TARGET_PAL_PERSISTENT 3

int cb200_dqn_head_fused(const cb200_dqn_head_desc* h_desc, void* stream);

/* Fused Bootstrapped DQN ensemble head (agents/bootstrapped_dqn_agent.py:26-30,57-86): `heads` Q heads on one feature
 * layer, head h owning the columns [h n_actions, (h + 1) n_actions) of one kernel [features, heads * n_actions].  Per
 * head and sample where masks[i, h] != 0: a* = argmax of the online head on s', target = r + (1 - done) * discount *
 * Q_target_h(s', a*) (fp64, bit-exact given the Q values, as cb200_dqn_head_fused); elsewhere the target is the online
 * prediction, so dL/dQ is exactly 0.  Per-head Huber / MSE loss mean_b(sum_a l) (heads/head.py:170-181), their sum,
 * dL/dQ, the head kernel's gradients, and the gradient w.r.t. the feature layer's pre-activation
 * grad_rescale * sum_h dQ_h W_h^T masked with relu'(h) (general_network.py:304-325), rescaled in fp32 before it is split
 * into operand planes.  features 256 or 512, n_actions <= 8, heads <= 64.  Deterministic: no atomics. */
typedef struct cb200_ensemble_head_desc {
    const float* h_next;        /* [batch, features] post-ReLU features of s' from the TARGET network                      */
    const float* h_online;      /* [batch, features] features of s from the online network                                */
    const float* h_select;      /* [batch, features] features of s' from the online network (per-head action selection)   */
    const float* w_target;      /* target head kernel [features, heads * n_actions] and bias [heads * n_actions]           */
    const float* b_target;
    const float* w_online;
    const float* b_online;
    const int64_t* actions;     /* [batch]                                                                                 */
    const double* rewards;
    const uint8_t* game_overs;
    const uint8_t* masks;       /* [batch, heads] bootstrap masks                                                          */
    double discount;
    int32_t huber;              /* 1: tf.losses.huber_loss(delta 1), 0: mean squared error                                */
    int64_t batch;
    int32_t features;           /* 256 or 512                                                                              */
    int32_t heads;              /* 1 .. 64                                                                                 */
    int32_t n_actions;          /* per head, <= 8                                                                          */
    float grad_rescale;         /* r of general_network.py:304-325                                                        */
    float* q_online;            /* out [batch, heads * n_actions]                                                          */
    float* q_next;              /* out, optional                                                                           */
    float* q_select;            /* out, optional                                                                           */
    float* targets;             /* out [batch, heads * n_actions]                                                          */
    float* dq;                  /* out [batch, heads * n_actions]: dL/dQ                                                   */
    float* losses;              /* out [heads]: per-head loss                                                              */
    float* loss;                /* out scalar, optional: sum of the per-head losses                                        */
    float* dh;                  /* out, optional: [batch, features] dL/d(pre-activation of the feature layer)             */
    void* dh_planes;            /* out, optional: the same as tiled bf16 hi / mid / lo planes                              */
    int64_t dh_plane_stride;
    float* dw;                  /* out [features, heads * n_actions]                                                       */
    float* db;                  /* out [heads * n_actions]                                                                 */
    float* workspace;           /* ceil(batch / 16) * 8 * ((features + 1) * heads * n_actions + heads) floats             */
} cb200_ensemble_head_desc;

int cb200_ensemble_head_fused(const cb200_ensemble_head_desc* e_desc, void* stream);

/* Fused N-step Q head (agents/n_step_q_agent.py:99-140): a plain QHead Dense(n_actions) on one feature layer, trained
 * on on-policy segments.  Segment s covers the rows [seg_offsets[s], seg_offsets[s] + seg_lengths[s]); a slot with
 * length 0 is unused.  The non-empty segments must be disjoint and together cover rows [0, n), n = the sum of the
 * lengths <= rows; rows [n, rows) are padding and get zero dq, dh and targets.  With S non-empty segments, per row i of a
 * segment of length L:
 *   targets[i] = Q_online(s_i) with the taken action's entry replaced by
 *     NSTEP (N-Step): R_i, walking i = L-1 .. 0 with R = r_i + discount R, in fp64.  R starts at 0 when the segment's
 *       last game_over is set, else at B = max_a Q_target(h_boot[s]) (fp32).  The first step after a bootstrap is
 *       numpy's python float * np.float32: (float)discount * B is rounded in fp32, then added to r_i in fp64.
 *     ONESTEP (1-Step): r_i + ((1 - done_i) discount) max_a Q_target(h_boot[i]), fp64 (as cb200_dqn_head_fused).
 *     NONE: nothing is replaced (the reference's fall-through): the loss and every gradient are 0.
 *   Every operation is an explicit _rn intrinsic; a row whose action is outside [0, n_actions) keeps Q(s).
 *   loss = (1/S) sum_s (1/L_s) sum_{i in s} sum_a l(Q - target), l Huber (delta 1) or squared error;
 *   dq = (1/S) (1/L_s) l'(Q - target), then dW = h^T dq, db = sum_i dq_i and dh = (dq W^T) relu'(h), as
 *   cb200_dqn_head_fused produces them.  features 256 or 512, n_actions <= 18.  Deterministic: per-warp partials reduced
 *   in a fixed order by a second launch, no atomics; repeat calls and graph replays give the same bits. */
typedef struct cb200_nstep_q_head_desc {
    const float* h_online;      /* [rows, features] post-ReLU features of s from the online network                      */
    const float* h_boot;        /* TARGET-network features: NSTEP [segments, features] of each segment's last s';
                                   ONESTEP [rows, features] of every row's s'; unused for NONE                            */
    const float* w_target;      /* target head kernel [features, n_actions] and bias                                      */
    const float* b_target;
    const float* w_online;
    const float* b_online;
    const int64_t* actions;     /* [rows]                                                                                 */
    const double* rewards;      /* [rows]                                                                                 */
    const uint8_t* game_overs;  /* [rows]                                                                                 */
    const int32_t* seg_offsets; /* [segments]                                                                             */
    const int32_t* seg_lengths; /* [segments], 0 = unused slot                                                           */
    int32_t segments;           /* slots in the table, 1 .. 2^20                                                         */
    int64_t rows;               /* rows of the feature / output buffers, 1 .. 2^24                                       */
    double discount;
    int32_t horizon;            /* CB200_NSTEP_*                                                                         */
    int32_t huber;              /* 1: tf.losses.huber_loss(delta 1), 0: mean squared error                                */
    int32_t features;           /* 256 or 512                                                                             */
    int32_t n_actions;          /* 1 .. 18                                                                                */
    float* q_online;            /* out [rows, n_actions]                                                                  */
    float* dq;                  /* out [rows, n_actions]: dL/dQ                                                           */
    float* loss;                /* out scalar, optional                                                                   */
    float* targets;             /* out, optional [rows, n_actions]                                                        */
    float* bootstrap;           /* out, optional: NSTEP [segments] B (0 for a terminal or unused segment);
                                   ONESTEP [rows] max_a Q_target(s'_i) (0 for padding rows)                               */
    float* dh;                  /* out, optional: [rows, features] dL/d(pre-activation of the feature layer)             */
    void* dh_planes;            /* out, optional: the same as tiled bf16 hi / mid / lo planes                             */
    int64_t dh_plane_stride;
    float* dw;                  /* out [features, n_actions]                                                              */
    float* db;                  /* out [n_actions]                                                                        */
    float* workspace;           /* ceil(segments / 4) * 4 * (features * n_actions + n_actions + 1) floats                */
} cb200_nstep_q_head_desc;

#define CB200_NSTEP_NONE 0
#define CB200_NSTEP_NSTEP 1
#define CB200_NSTEP_ONESTEP 2

int cb200_nstep_q_head(const cb200_nstep_q_head_desc* n_desc, void* stream);

/* Fused actor-critic head (agents/actor_critic_agent.py:111-165, heads/v_head.py, heads/policy_head.py): ONE
 * Dense(1 + n_actions) on one feature layer, column 0 the VHead V, columns 1..n_actions the PolicyHead logits, trained
 * on the segment table of cb200_nstep_q_head (slot s covers rows [seg_offsets[s], + seg_lengths[s]), length 0 = unused;
 * rows [n, rows) are padding and get zero outputs and dh).  Per segment of length L, with B = V(h_boot[s]) (0 when the
 * segment's last game_over is set) and gl = discount * gae_lambda (fp64), walking i = L-1 .. 0, all in fp64 with _rn:
 *   A_VALUE     R = r_i + discount R from R = B; the first step after a bootstrap is numpy's python float *
 *               np.float32: (float)discount * B rounded in fp32, then added to r_i.  target R, advantage R - V_i.
 *   GAE         delta_i = (r_i + fp32((float)discount * V_{i+1})) - V_i with V_L = B; advantage = the
 *               scipy.signal.lfilter([1], [1, -gl]) recurrence A_i = delta_i + gl A_{i+1}; target = the lfilter
 *               discounted sum of [r_0 .. r_{L-1}, B] with discount (GAE), or A_i + V_i (GAE_VALUE:
 *               estimate_state_value_using_gae).
 *   target and advantage are rounded to fp32.  p = softmax(logits) (fp32); u = p + FLT_EPSILON; ls = log u - log sum u;
 *   H = -sum_k u_k ls_k (tf Categorical(probs = p + eps), probs not renormalised).
 *   loss = (1/S) sum_s (1/L) sum_i [v_weight l(V_i - target_i) - p_weight ls_{a_i} A_i - beta_entropy H_i],
 *   l = squared error or Huber (delta 1); a row whose action is outside [0, n_actions) has no policy term.
 *   dz = dL/dZ over all 1 + n_actions columns, dW = h^T dz, db = sum_i dz_i, dh = (dz W^T) relu'(h).
 * features 256 or 512, n_actions <= 18.  Deterministic: per-warp partials reduced in a fixed order by a second launch,
 * no atomics; repeat calls and graph replays give the same bits. */
typedef struct cb200_actor_critic_head_desc {
    const float* h;             /* [rows, features] post-ReLU features of s                                               */
    const float* h_boot;        /* [segments, features] features of each segment's last s' (online network)             */
    const float* w;             /* head kernel [features, 1 + n_actions] and bias [1 + n_actions]                        */
    const float* b;
    const int64_t* actions;     /* [rows]                                                                                 */
    const double* rewards;      /* [rows]                                                                                 */
    const uint8_t* game_overs;  /* [rows]                                                                                 */
    const int32_t* seg_offsets; /* [segments]                                                                             */
    const int32_t* seg_lengths; /* [segments], 0 = unused slot                                                           */
    int32_t segments;           /* slots in the table, 1 .. 2^20                                                         */
    int64_t rows;               /* rows of the feature / output buffers, 1 .. 2^24                                       */
    double discount;
    double gae_lambda;
    int32_t mode;               /* CB200_AC_*                                                                             */
    int32_t huber;              /* VHead loss: 1 tf.losses.huber_loss(delta 1), 0 squared error                           */
    float beta_entropy;
    float v_weight;             /* VHead loss weight (0.5)                                                                */
    float p_weight;             /* PolicyHead loss weight (1.0)                                                           */
    int32_t features;           /* 256 or 512                                                                             */
    int32_t n_actions;          /* 1 .. 18                                                                                */
    float* z;                   /* out [rows, 1 + n_actions]: V | logits                                                  */
    float* dz;                  /* out, optional [rows, 1 + n_actions]: dL/dZ                                             */
    float* loss;                /* out scalar, optional                                                                   */
    float* probs;               /* out, optional [rows, n_actions]                                                        */
    float* targets;             /* out, optional [rows]: V targets (fp32)                                                 */
    float* advantages;          /* out, optional [rows] (fp32)                                                            */
    float* bootstrap;           /* out, optional [segments]: B                                                            */
    float* dh;                  /* out, optional: [rows, features] dL/d(pre-activation of the feature layer)             */
    void* dh_planes;            /* out, optional: the same as tiled bf16 hi / mid / lo planes                             */
    int64_t dh_plane_stride;
    float* dw;                  /* out [features, 1 + n_actions]                                                          */
    float* db;                  /* out [1 + n_actions]                                                                    */
    float* workspace;           /* ceil(segments / 4) * 4 * (features * (1 + n_actions) + n_actions + 2) floats          */
} cb200_actor_critic_head_desc;

#define CB200_AC_A_VALUE 0
#define CB200_AC_GAE 1
#define CB200_AC_GAE_VALUE 2

int cb200_actor_critic_head(const cb200_actor_critic_head_desc* ac_desc, void* stream);

/* Actor-critic head for continuous actions (actor_critic_agent.py:111-186, heads/policy_head.py:102-152 with
 * ContinuousEntropy): ONE Dense(1 + 2 action_dim) on one feature layer, column 0 V, columns 1..D (D = action_dim) the
 * pre-activation means, D+1..2D the pre-activation stds, over the segment table of cb200_actor_critic_head (segments
 * must not overlap; rows covered by no segment get zero outputs and dh).
 *   targets and advantages: cb200_actor_critic_head's A_VALUE / GAE / GAE_VALUE recurrences, the same operations.
 *   mean = tanh(z) * max_abs_range; std = softplus(z) + FLT_EPSILON with TF 1.x's softplus (x above -t, exp(x) below
 *   t, log(exp(x) + 1) between, t = log(FLT_EPSILON) + 2); all fp32.
 *   MultivariateNormalDiag(mean, std) at x = actions[i]: log pi = sum_d [-((x - mean) / std)^2 / 2 - log std -
 *   log(2 pi) / 2], H = sum_d [(1 + log(2 pi)) / 2 + log std].
 *   loss = (1/S) sum_s (1/L) sum_i [v_weight l(V_i - target_i) - p_weight log pi_i A_i - beta_entropy H_i] (S the
 *   non-empty segments), l = squared error or Huber (delta 1); dz = dL/dZ over the 1 + 2D columns (the std columns'
 *   softplus derivative is sigmoid(z)), dW = h^T dz, db = sum_i dz_i, dh = (dz W^T) relu'(h).
 * Parallel over rows (a row pass, one thread per segment for the recurrence, a row pass for the loss and dL/dZ);
 * dW, db and the loss are summed per 64-row chunk, then over the chunks in a fixed order: no atomics on floats, repeat
 * calls and graph replays give the same bits.  features 256 or 512, action_dim <= 17. */
typedef struct cb200_actor_critic_gaussian_head_desc {
    const float* h;             /* [rows, features] post-ReLU features of s                                               */
    const float* h_boot;        /* [segments, features] features of each segment's last s' (online network)             */
    const float* w;             /* head kernel [features, 1 + 2 action_dim] and bias [1 + 2 action_dim]                  */
    const float* b;
    const float* actions;       /* [rows, action_dim] the actions taken, as fp32                                          */
    const float* max_abs_range; /* [action_dim]                                                                           */
    const double* rewards;      /* [rows]                                                                                 */
    const uint8_t* game_overs;  /* [rows]                                                                                 */
    const int32_t* seg_offsets; /* [segments]                                                                             */
    const int32_t* seg_lengths; /* [segments], 0 = unused slot                                                           */
    int32_t segments;           /* slots in the table, 1 .. 2^20                                                         */
    int64_t rows;               /* rows of the feature / output buffers, 1 .. 2^24                                       */
    double discount;
    double gae_lambda;
    int32_t mode;               /* CB200_AC_*                                                                             */
    int32_t huber;              /* VHead loss: 1 tf.losses.huber_loss(delta 1), 0 squared error                           */
    float beta_entropy;
    float v_weight;             /* VHead loss weight (0.5)                                                                */
    float p_weight;             /* PolicyHead loss weight (1.0)                                                           */
    int32_t features;           /* 256 or 512                                                                             */
    int32_t action_dim;         /* 1 .. 17                                                                                */
    float* z;                   /* out [rows, 1 + 2 action_dim]: V | pre-tanh means | pre-softplus stds                   */
    float* dz;                  /* out, optional [rows, 1 + 2 action_dim]: dL/dZ                                          */
    float* loss;                /* out scalar, optional                                                                   */
    float* means;               /* out, optional [rows, action_dim]                                                       */
    float* stds;                /* out, optional [rows, action_dim]                                                       */
    float* targets;             /* out, optional [rows]: V targets (fp32)                                                 */
    float* advantages;          /* out, optional [rows] (fp32)                                                            */
    float* bootstrap;           /* out, optional [segments]: V(s'_last), 0 after a terminal state                        */
    float* dh;                  /* out, optional: [rows, features] dL/d(pre-activation of the feature layer)             */
    void* dh_planes;            /* out, optional: the same as tiled bf16 hi / mid / lo planes                             */
    int64_t dh_plane_stride;
    float* dw;                  /* out [features, 1 + 2 action_dim]                                                       */
    float* db;                  /* out [1 + 2 action_dim]                                                                 */
    float* workspace;           /* rows * (2 action_dim + 5) + segments + ceil(rows / 64) * (features + 1) *
                                   (2 action_dim + 1) + ceil(rows / 64) floats                                            */
} cb200_actor_critic_gaussian_head_desc;

int cb200_actor_critic_gaussian_head(const cb200_actor_critic_gaussian_head_desc* acg_desc, void* stream);

/* Acting from the continuous actor-critic head's outputs z [envs, 1 + 2 action_dim] (ContinuousEntropy, i.e.
 * exploration_policies/additive_noise.py:74-103 with the network's std): mean and std with the head's code (fp32);
 * with normals [envs, action_dim] (np.random.standard_normal) the action is numpy's normal(mean, std) =
 * (double) mean + (double) std * normal in fp64; normals NULL (evaluation): the mean.  actions [envs, action_dim] fp64
 * out; means and stds [envs, action_dim] fp32 out, optional. */
int cb200_gaussian_policy_act(const float* z, int64_t envs, int32_t action_dim, const float* max_abs_range,
                              const double* normals, double* actions, float* means, float* stds, void* stream);

/* Categorical acting (exploration_policies/categorical.py:36-47): z [envs, 1 + n_actions] as the actor-critic head
 * lays it out (V | logits); p = softmax(logits) with the head's code.  uniforms [envs] (np.random.random_sample):
 * np.random.choice's draw, cdf = cumsum(double(p)) in index order, cdf /= cdf[-1], action = the number of entries
 * <= u; uniforms NULL: the first argmax (evaluation).  actions [envs] out, probs [envs, n_actions] out, optional. */
int cb200_categorical_act(const float* z, int64_t envs, int32_t n_actions, const double* uniforms, int64_t* actions,
                          float* probs, void* stream);

/* Policy gradient targets (agents/policy_gradients_agent.py:47-67, policy_optimization_agent.py:58-71) over a segment
 * table of whole episodes (the table of cb200_nstep_q_head: slot s covers rows [seg_offsets[s], + seg_lengths[s]),
 * length 0 = unused), given each row's fp64 return R (cb200_nstep_returns with n_step -1).  Per row, in fp64 with every
 * operation rounded on its own, then rounded to fp32 into targets:
 *   TOTAL_RETURN            R_0 of the row's episode
 *   FUTURE_RETURN           R_i
 *   NORMALIZED_BY_EPISODE   (R_i - mean) / std, mean and std = np.mean / np.std (population) of the episode's returns
 *                           with numpy's pairwise summation, bit-identical; 0 when std == 0.  episode_stats (optional,
 *                           [segments, 2]) receives (mean, std) per slot.
 *   NORMALIZED_BY_TIMESTEP  R_i - m_i: the episodes are folded in slot order into the running-mean table (table_mean,
 *                           table_count [table_len], fp64, updated in place): n_i += 1; m_i -= m_i / n_i;
 *                           m_i += R_i / n_i, and m_i is the table right after the row's own episode was folded.
 *                           baselines (optional, [rows]) receives that m_i.  A row at a timestep >= table_len gets NaN
 *                           and leaves the table alone.
 * Rows covered by no segment are not written. */
#define CB200_PG_TOTAL_RETURN 0
#define CB200_PG_FUTURE_RETURN 1
#define CB200_PG_NORMALIZED_BY_EPISODE 2
#define CB200_PG_NORMALIZED_BY_TIMESTEP 3
int cb200_pg_targets(const double* returns, const int32_t* seg_offsets, const int32_t* seg_lengths, int32_t segments,
                     int64_t rows, int32_t rescaler, double* table_mean, double* table_count, int32_t table_len,
                     float* targets, double* baselines, double* episode_stats, void* stream);

/* Fused policy gradient head (heads/policy_head.py:54-150, policy_gradients_agent.py:69-86): ONE Dense(n_outputs) on
 * one feature layer, over the segment table above (segments must not overlap; rows covered by no segment get zero
 * outputs and dh).  With t_i the row's target and c = 1 / L for an episode of L rows:
 *   discrete    p = softmax(z) with cb200_actor_critic_head's code, Categorical(probs = p + eps) semantics:
 *               l_i = c (-log pi(a_i) t_i - beta_entropy H_i); an action outside [0, n_outputs) has no policy term.
 *   continuous  mean = tanh(z) * max_abs_range (fp32), MultivariateNormalDiag(mean, 1) (the std is the all-ones
 *               policy_stdev variable): log pi(x) = -|x - mean|^2 / 2 - D log(2 pi) / 2, H = D (1 + log(2 pi)) / 2
 *               (no gradient); l_i = c (-log pi(x_i) t_i - beta_entropy H).
 *   loss = sum_i l_i: the sum over the table's episodes of each episode's mean loss, and dz = dL/dZ, so the gradient
 *   is the sum of the episodes' gradients (what accumulate_gradients adds up).  dW = h^T dz, db = sum_i dz_i,
 *   dh = (dz W^T) relu'(h).
 * Parallel over rows; dW, db and the loss are summed per 64-row chunk, then over the chunks in a fixed order: no
 * atomics, repeat calls and graph replays give the same bits.  features 256 or 512; n_outputs <= 18 (discrete) or
 * <= 32 (continuous). */
typedef struct cb200_policy_gradient_head_desc {
    const float* h;             /* [rows, features] post-ReLU features                                                   */
    const float* w;             /* head kernel [features, n_outputs] and bias [n_outputs]                                */
    const float* b;
    const float* targets;       /* [rows] (cb200_pg_targets)                                                             */
    const int64_t* actions;     /* [rows], discrete                                                                      */
    const float* cont_actions;  /* [rows, n_outputs], continuous                                                         */
    const float* max_abs_range; /* [n_outputs], continuous                                                               */
    const int32_t* seg_offsets; /* [segments]                                                                            */
    const int32_t* seg_lengths; /* [segments], 0 = unused slot                                                           */
    int32_t segments;           /* 1 .. 2^20                                                                              */
    int64_t rows;               /* rows of the feature / output buffers, 1 .. 2^24                                       */
    int32_t continuous;         /* 0 discrete (Categorical), 1 bounded Gaussian                                          */
    int32_t features;           /* 256 or 512                                                                             */
    int32_t n_outputs;          /* actions (discrete) or action dimensions (continuous)                                  */
    float beta_entropy;
    float* z;                   /* out [rows, n_outputs]: the Dense outputs (logits / pre-tanh means)                    */
    float* policy;              /* out, optional [rows, n_outputs]: p (discrete) or the mean (continuous)                */
    float* dz;                  /* out, optional [rows, n_outputs]: dL/dZ                                                */
    float* loss;                /* out scalar, optional                                                                   */
    float* dh;                  /* out, optional: [rows, features] dL/d(pre-activation of the feature layer)             */
    void* dh_planes;            /* out, optional: the same as tiled bf16 hi / mid / lo planes                             */
    int64_t dh_plane_stride;
    float* dw;                  /* out [features, n_outputs]                                                             */
    float* db;                  /* out [n_outputs]                                                                        */
    float* workspace;           /* rows * (n_outputs + 1) + ceil(rows / 64) * (features * n_outputs + n_outputs + 1)    */
} cb200_policy_gradient_head_desc;

int cb200_policy_gradient_head(const cb200_policy_gradient_head_desc* pg_desc, void* stream);

/* Acting from a policy gradient head's outputs z [envs, n_outputs]:
 *   discrete    cb200_categorical_act's softmax and draw (uniforms in `draws` [envs], NULL: the first argmax) into
 *               actions [envs], probs [envs, n_outputs] optional.
 *   continuous  AdditiveNoise (exploration_policies/additive_noise.py:74-103): mean = tanh(z) * max_abs_range (fp32, the
 *               head's code); with draws [envs, n_outputs] (np.random.standard_normal) the action is numpy's
 *               normal(mean, scale) = (double) mean + scale[e, d] * draw in fp64 (scale [envs, n_outputs] fp64: each
 *               environment's noise times high - low); draws NULL (evaluation): the mean.  cont_actions [envs, n_outputs] fp64 out, means
 *               [envs, n_outputs] fp32 optional. */
int cb200_policy_act(const float* z, int64_t envs, int32_t n_outputs, int32_t continuous, const float* max_abs_range,
                     const double* draws, const double* scale, int64_t* actions, float* probs, double* cont_actions,
                     float* means, void* stream);

/* Acting values of an ensemble, q [envs, heads * n_actions] -> out [envs, n_actions], in the exploration policies' fp32
 * numpy arithmetic (exploration_policies/bootstrapped.py:70-84, ucb.py:70-83):
 *   SELECT  the row of head[e] (Bootstrapped, training)
 *   UCB     mean + lamb * std over the heads, population std (UCB, training)
 *   MEAN    mean over the heads (UCB, evaluation)
 *   VOTE    one-hot of the majority vote of the heads' argmaxes, ties to the lowest action (Bootstrapped, evaluation) */
#define CB200_ENSEMBLE_SELECT 0
#define CB200_ENSEMBLE_UCB 1
#define CB200_ENSEMBLE_MEAN 2
#define CB200_ENSEMBLE_VOTE 3
int cb200_ensemble_action_values(const float* q, int64_t envs, int32_t heads, int32_t n_actions, int32_t mode,
                                 const int32_t* head, float lamb, float* out, void* stream);

/* DuelingQHead (heads/dueling_q_head.py:33-47): q = v + (adv - mean_a adv); backward: d_v = sum_a dq,
 * d_adv = dq - mean_a dq. */
int cb200_dueling_combine_fwd(const float* v, const float* adv, int64_t batch, int64_t n_actions, float* q,
                              void* stream);
int cb200_dueling_combine_bwd(const float* dq, int64_t batch, int64_t n_actions, float* d_v, float* d_adv,
                              void* stream);

/* sum of squares of a flat fp32 buffer in a fixed order -> *out (device float); tf.global_norm =
 * sqrt(sum_t sum(t^2)) (architecture.py:194).  workspace >= 1024 floats. */
int cb200_sumsq(const float* x, int64_t n, float* out, float* workspace, void* stream);

/* tf.clip_by_global_norm (architecture.py:239-240): g *= clip / max(sqrt(*sumsq), clip)  -- in place, fp32 (sqrtf and
 * the division correctly rounded; finite g is untouched bit for bit while sqrt(*sumsq) <= clip).  A non-finite norm: *sumsq =
 * +inf scales by 0 (finite gradients become +-0), *sumsq = NaN scales by 1 (fmaxf drops the NaN: g passes unclipped,
 * and the NaN that made the norm NaN is still in g). */
int cb200_clip_by_global_norm(float* g, int64_t n, const float* sumsq, float clip, void* stream);

/* g *= s (apply_gradients `scaler`, architecture.py:485-493: 1/num_workers for sync training) */
int cb200_scale(float* g, int64_t n, float s, void* stream);

/* tf.train.AdamOptimizer step with TF-1.x semantics (general_network.py:390-394; kernel form of
 * tensorflow/core/kernels/training_ops.cc ApplyAdam):
 *   alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power)       (fp32; the powers are the fp32 running products)
 *   m += (g - m) * (1 - beta1);  v += (g*g - v) * (1 - beta2);  theta -= (m * alpha) / (sqrt(v) + epsilon)
 * over the whole flat parameter buffer in one launch. */
int cb200_adam_tf(float* theta, float* m, float* v, const float* g, int64_t n, float lr, float beta1, float beta2,
                  float epsilon, float beta1_power, float beta2_power, void* stream);

/* Same optimizer step with the running powers kept in DEVICE memory (state = {beta1_power, beta2_power}, initialised
 * to {beta1, beta2}); the step multiplies them afterwards.  All launch parameters are constant from step to step, so
 * a complete training step can be captured in a CUDA graph and replayed. */
int cb200_adam_tf_dev(float* theta, float* m, float* v, const float* g, int64_t n, float lr, float beta1, float beta2,
                      float epsilon, float* state, void* stream);

/* *x += delta on the device (minibatch cursor of a captured epoch loop, see cb200_gather_at) */
int cb200_add_i64(int64_t* x, int64_t delta, void* stream);

/* NetworkWrapper.update_target_network -> set_weights (architecture.py:598-607):
 *   target = rate * online + (1 - rate) * target   in fp32, rate and (1 - rate) rounded to fp32 first (numpy). */
int cb200_polyak(float* target, const float* online, int64_t n, double rate, void* stream);

/* PPOHead for continuous actions (heads/ppo_head.py:52-98,118-144): diagonal Gaussian policy with a state-independent
 * log-std variable, sigma = exp(logstd) + 1e-15; likelihood ratio exp(logp - logp_old) (:78), clipped to
 * 1 +- clip_eps (clip_eps = clip_likelihood_ratio_using_epsilon * clipping_decay rescaler, :80-84), surrogate
 * L = -mean(min(ratio*A, clip(ratio)*A)) (:85-90), entropy regulariser -beta*H (:93-95).  The old policy is given by
 * its mean per sample and its log-std vector (the frozen target network, clipped_ppo_agent.py:240).
 * Outputs d(L)/d(mu) [batch, action_dim], d(L)/d(logstd) [action_dim] and scalars[5] = {loss, KL(old||new), entropy,
 * mean ratio, mean clipped ratio} (the signals clipped_ppo_agent.py:227-230 fetches).  action_dim <= 32. */
int cb200_ppo_continuous_head(const float* mu, const float* logstd, const float* actions, const float* old_mu,
                              const float* old_logstd, const float* advantages, int64_t batch, int32_t action_dim,
                              float clip_eps, float beta_entropy, float* d_mu, float* d_logstd, float* scalars,
                              void* stream);

/* PPOHead for continuous actions with the KL penalty and no clipping (heads/ppo_head.py:64-97 with
 * clip_likelihood_ratio_using_epsilon None; agents/ppo_agent.py): the Gaussian terms of cb200_ppo_continuous_head and
 *   KLbar = mean_i KL_i(old || new)
 *   L     = -mean_i(ratio_i * A_i) + use_kl * (k * KLbar + high_kl_penalty * max(0, KLbar - kl_cutoff)^2) - beta * H
 * (the two KL terms are the head's regularizations, :68-72; kl_cutoff = 2 * target_kl_divergence).  kl_coef is a
 * DEVICE fp32 scalar k, read at run time, so a captured CUDA graph follows coefficient updates; it may be NULL when
 * use_kl == 0.  Outputs d(L)/d(mu) [batch, action_dim], d(L)/d(logstd) [action_dim] and optional scalars[5] =
 * {loss, KLbar, entropy, mean ratio, surrogate -mean(ratio * A)}.  One CTA with fixed-order reductions: repeat calls
 * give identical bits.  1 <= action_dim <= 32, batch >= 1. */
int cb200_ppo_kl_head(const float* mu, const float* logstd, const float* actions, const float* old_mu,
                      const float* old_logstd, const float* advantages, int64_t batch, int32_t action_dim,
                      const float* kl_coef, float kl_cutoff, float high_kl_penalty, int32_t use_kl, float beta_entropy,
                      float* d_mu, float* d_logstd, float* scalars, void* stream);

/* PPOHead for discrete actions with the clipped surrogate (heads/ppo_head.py:52-116; agents/clipped_ppo_agent.py).
 * logits [batch, n_actions] are the policy's last Dense outputs, p = softmax(logits); old_probs [batch, n_actions] the
 * frozen target network's softmax.  TF 1.x's Categorical(probs = x) takes logits log x, so
 *   log pi = log_softmax(log p), log pi_old = log_softmax(log old_probs), ratio = exp(log pi(a) - log pi_old(a)),
 *   clipped to 1 -+ e with e = fl32(clip_eps * *clip_rescaler) (TF's fp32 product),
 *   L = -mean_i min(ratio_i A_i, clip(ratio_i) A_i) - beta_entropy * mean_i H_i,  H_i = -sum_j p_j log pi_j.
 * clip_rescaler is a DEVICE fp32 scalar read at run time, so one captured CUDA graph follows the clipping schedule.
 * An action outside [0, n_actions) contributes no surrogate term: its row adds nothing to the loss's surrogate part,
 * the ratio sums or the surrogate gradient (it still adds its entropy and KL terms, and every mean divides by batch).
 * Outputs d(L)/d(logits) [batch, n_actions] and optional scalars[5] = {loss, mean KL(old||new), mean entropy,
 * mean ratio, mean clipped ratio} (the signals of cb200_ppo_continuous_head, in its order); a KL term whose old
 * probability is 0 counts as 0.  One CTA with fixed-order reductions: repeat calls give identical bits.
 * 1 <= n_actions <= 32, batch >= 1; a bad argument returns an error and writes nothing. */
int cb200_ppo_categorical_head(const float* logits, const int64_t* actions, const float* old_probs,
                               const float* advantages, int64_t batch, int32_t n_actions, float clip_eps,
                               const float* clip_rescaler, float beta_entropy, float* d_logits, float* scalars,
                               void* stream);

/* AdditiveNoise.get_action([mean, std]) of the PPO actor (exploration_policies/additive_noise.py:84-103):
 * stds [envs, action_dim] = exp(logstd) in fp32 (optional); with normals [envs, action_dim] (np.random.standard_normal,
 * what successive np.random.normal calls draw): actions = (double) mean + (double) std * n, multiply and add each
 * rounded on its own (numpy's normal).  normals NULL: only stds are written (evaluation acts on the mean). */
int cb200_ppo_gaussian_act(const float* mean, const float* logstd, int64_t envs, int32_t action_dim,
                           const double* normals, double* actions, float* stds, void* stream);

/* dst[c][i, :] = src[c][idx[*offset + i], :] for i < n (idx == NULL: rows *offset + i).  `offset` is a DEVICE scalar
 * so that the launch is identical for every minibatch of an epoch (CUDA-graph replay; only *offset changes).
 * Minibatch slicing of clipped_ppo_agent.py:232-265 after batch.shuffle(). */
int cb200_gather_at(const cb200_column* h_columns, int n_columns, const int64_t* idx, const int64_t* offset,
                    int64_t n, void* stream);

/* dz[r, c] = dy[r, c] * act'(y[r, c]) with independent leading dimensions: activation backward on a column block of a
 * wider buffer (the embedder part of a critic's concatenated [action, embedding] input, general_network.py:272-277). */
int cb200_act_backward(const float* dy, int32_t ld_dy, const float* y, int32_t ld_y, int64_t rows, int32_t cols,
                       int32_t act, float* dz, int32_t ld_dz, void* stream);

/* dst[r, c] = alpha * src[r, c] + beta * dst[r, c] on strided 2-D fp32 blocks (beta == 0: dst is not read).  Used for
 * the embedding merger concat, the actor's output scale and the -(1/B) * dQ/da seed of the actor update
 * (ddpg_agent.py:171-186). */
int cb200_axpby_2d(const float* src, int32_t ld_src, int64_t rows, int32_t cols, float alpha, float beta, float* dst,
                   int32_t ld_dst, void* stream);

/* Bootstrapped critic targets of DDPG / TD3 / SAC (ddpg_agent.py:156-164, td3_agent.py:172-181,
 * soft_actor_critic_agent.py:265-266): y = r + (1 - done) * discount * q_next in fp64 (numpy), optional clip (np.clip:
 * a NaN passes through), stored as fp32; bit-exact with the numpy expression.  With
 * use_non_zero_discount_for_terminal_states the product discount * q_next is fp32 (a Python float times a float32
 * array).  q_next is read with stride ld_q. */
int cb200_ac_td_targets(const double* rewards, const uint8_t* game_overs, const float* q_next, int32_t ld_q,
                        int64_t batch, double discount, int32_t use_non_zero_discount_for_terminal_states,
                        int32_t use_clip, double clip_lo, double clip_hi, float* targets_out, void* stream);

/* NAFHead (heads/naf_head.py:45-86), the per-sample nonlinear part: the three head projections come from ordinary Dense
 * layers (V: 1 output, mu: n_actions pre-tanh outputs, l: n_actions (n_actions + 1) / 2 outputs).  Per sample b:
 *   mu = tanh(z_mu) * scale                                    (scale: max_abs_range rounded to fp32)
 *   L  = lower triangle of l packed column by column: column c holds rows c .. A-1, starting at
 *        i_c = c A - c (c - 1) / 2, with L[c, c] = exp(l[i_c])
 *   d  = u - mu,  w = L^T d,  adv = -0.5 * d^T L L^T d = -0.5 * |w|^2,  Q = V + adv
 *   loss = mean_b l(Q_b - y_b), l = squared error or Huber (delta 1) (head.py:165-177; no importance weights)
 * and the gradients of the loss straight into the three layers' output gradients:
 *   d_zv = dL/dQ,  d_zmu = dL/dQ * (L w) * scale * (1 - tanh^2),  d_l[L[r, c]] = dL/dQ * (-d_r w_c), times L[c, c] on
 *   the diagonal.
 * The kernel evaluates w first (not P = L L^T as the TensorFlow graph does); its accuracy is stated against fp64
 * (tests/test_naf_gpu.py).  One warp per sample, n_actions <= 32.  The loss is reduced in a fixed order by a second
 * launch: the same bits on every call.
 * Acting mode (actions == NULL and targets == NULL): only mu and -- when given -- q = V are written; l, ld_l and
 * ld_actions are not read, and z_v only when q is given.
 * mu / z_mu / d_zmu use the row stride ld_mu, l / d_l ld_l, actions ld_actions; z_v, q, targets, d_zv, adv are [batch]. */
typedef struct cb200_naf_head_desc {
    const float* z_v;           /* [batch] V projection (acting: only read when q is given)                          */
    const float* z_mu;          /* [batch, ld_mu] mu projection before the tanh                                      */
    const float* l;             /* [batch, ld_l] l_vector projection (training only)                                 */
    const float* scale;         /* [n_actions] output scale of mu                                                    */
    const float* actions;       /* [batch, ld_actions] the head input u (the batch actions); NULL: acting mode       */
    const float* targets;       /* [batch] TD targets; NULL: acting mode                                             */
    int32_t huber;              /* replace_mse_with_huber_loss                                                       */
    int64_t batch;
    int32_t n_actions;          /* 1 .. 32                                                                           */
    int32_t ld_mu, ld_l, ld_actions;
    float* mu;                  /* [batch, ld_mu] scaled mu (always written)                                         */
    float* q;                   /* [batch] Q (training: required; acting: optional, = V)                             */
    float* loss;                /* [1] training: required                                                            */
    float* d_zv;                /* [batch] training: required                                                        */
    float* d_zmu;               /* [batch, ld_mu] training: required                                                 */
    float* d_l;                 /* [batch, ld_l] training: required                                                  */
    float* adv;                 /* [batch] training: optional                                                        */
} cb200_naf_head_desc;
int cb200_naf_head(const cb200_naf_head_desc* desc, void* stream);

/* tf.clip_by_value(g, -clip, clip) in place (architecture.py:241-245, GradientClippingMethod.ClipByValue); NaN passes
 * through, +-inf clips.  clip > 0. */
int cb200_clip_by_value(float* g, int64_t n, float clip, void* stream);

/* out = min(a, b) element-wise (clipped double-Q: td3_v_head.py:61, sac_q_head.py:84-86), as tf.minimum evaluates it:
 * b where b < a, else a (a tie of +0 and -0 gives a; a NaN in a passes through, a NaN in b gives a) */
int cb200_min2(const float* a, const float* b, int64_t n, float* out, void* stream);

/* TD3 target policy smoothing (td3_agent.py:162-164): a = clip(a + clip(noise, -noise_clip, noise_clip), lo, hi);
 * noise is the fp64 np.random.normal draw, the sum and both clips are evaluated in fp64 like numpy does and rounded
 * to fp32 once (bit-exact with the reference, tests/golden/agent_prologues.npz).  Both clips are np.clip's: a NaN
 * passes through and a value equal to a bound is kept. */
int cb200_td3_smooth_actions(float* actions, const double* noise, int64_t n, double noise_clip, double lo, double hi,
                             void* stream);

/* CategoricalQHead + distributional TD targets (agents/categorical_dqn_agent.py:105-165, rainbow_dqn_agent.py:93-140,
 * architectures/tensorflow_components/heads/categorical_q_head.py:41-57).  Inputs are the [batch, n_actions, n_atoms]
 * head logits of target(s'), online(s) and -- for the double-Q rule of Rainbow, else NULL -- online(s').  z = the fp64
 * support (np.linspace); gamma_n = discount (** n_step); bootstrap (fp64 per sample, NULL -> 1 - game_over) is
 * info['should_bootstrap_next_state'].  Writes: labels = TD_targets fed to the train op (online softmax, projected
 * distribution m on the taken action's row; projection accumulated in fp64 in the reference's loop order, bit-exact
 * given equal probabilities), dlogits = d(total loss)/d(online logits) (softmax - labels on the taken row, 0 elsewhere),
 * loss_rows [batch, n_actions] = tf.nn.softmax_cross_entropy_with_logits, total_loss = their sum
 * (general_network.py:360), td_err = loss_rows[b, action[b]] (what update_priorities is handed, :160-163), optional
 * q_online [batch, n_actions] fp64 (distribution_prediction_to_q_values) and target_actions.  next_is_prob != 0: `next`
 * / `select` already hold probabilities (parity tests feed the fixture's network outputs).  n_atoms 2 .. 1024 (above
 * 768 the kernel opts into more than 48 KB of dynamic shared memory).  The projection never writes outside the sample's
 * row: when (z[N-1] - z[0]) / (z[1] - z[0]) rounds above N - 1 (np.linspace supports often do) and a target clamps to
 * z[N-1], the share that would land on bin N is dropped -- the reference raises IndexError on the same sample; every
 * in-row share is unchanged. */
int cb200_c51_head(const float* next, const float* online, const float* select, const int64_t* actions,
                   const double* rewards, const uint8_t* game_overs, const double* bootstrap, const double* z,
                   double gamma_n, int32_t batch, int32_t n_actions, int32_t n_atoms, int32_t next_is_prob,
                   float* labels, float* dlogits, float* loss_rows, float* total_loss, double* td_err,
                   double* q_online, int64_t* target_actions, void* stream);

/* q_values output of the CategoricalQHead (categorical_q_head.py:56): q[r] = sum_j (double)softmax(logits[r, :])_j * z[j]
 * for rows = batch * n_actions rows of n_atoms logits; z = the fp32-rounded support cast back to fp64 (:36-37) */
int cb200_c51_q_values(const float* logits, const double* z, int64_t rows, int32_t n_atoms, double* q_out, void* stream);

/* QuantileRegressionQHead + the TD targets of QuantileRegressionDQNAgent (agents/qr_dqn_agent.py:97-137,
 * heads/quantile_regression_q_head.py:33-71).  Inputs are the [batch, n_actions, n_atoms] quantiles of target(s') and
 * online(s) (action-major, atom-inner).  Per sample b, with N = n_atoms:
 *   Q'[a]    = sum_j (double)next[a, j] * (1.0 / N) in fp64 (the head's q_values, np.dot with ones(N) / N);
 *              a* = the first argmax of Q'.  numpy's summation order is unspecified: Q' equals the reference's up to
 *              fp64 rounding, so only a near tie of two actions can choose differently.
 *   T_j      = (float)(r + ((1.0 - game_over) * discount) * (double)next[a*, j]), each operation an fp64 _rn operation
 *              in numpy's order: bit-exact with the reference's TD_targets as fed.
 *   sigma    = argsort of the taken row online[action, :], ties broken by index (kind='stable'); the reference assigns
 *              tau_i = tau_hat[sigma(i)] (NOT the rank tau_hat[sigma^-1(i)]), tau_hat_k = 0.5 * ((k + 1) / N + k / N)
 *              in fp64, fed as fp32 -- kept.
 *   pair (i, j), fp32, no contraction: e = T_j - theta_i, a = |e|, q = min(a, kappa), h = kappa (a - q) + 0.5 q^2,
 *              l = |tau_i - [e < 0]| h
 *   loss     = (sum over b, i, j of l) / N: summed over the batch, no importance weights.
 *   dq       = d loss / d online: -(1/N) sum_j |tau_i - [e < 0]| clamp(e, -kappa, kappa) on the taken row
 *              (tf.minimum sends its gradient to the first argument on ties), exactly 0 on every other row.  The
 *              products are fp32; their j-sum, which cancels, is accumulated in fp64 and rounded once.
 * kappa = 0 (the reference's "strict quantile loss") makes h, the loss and dq identically 0: the reference's
 * arithmetic, kept.  Each theta_i's j-sum runs in one thread in j order; the per-sample sums go to workspace and a
 * second launch reduces them in a fixed order: the same bits on every call (eager or graph replay).  An action outside
 * [0, n_actions) contributes 0 to the loss and dq, and its taus row is not written.  NaN quantiles give an unspecified
 * (in-range) order.  Limits: 1 <= n_atoms <= 1024, 1 <= n_actions <= 256, batch >= 1, kappa >= 0. */
typedef struct cb200_qr_head_desc {
    const float* next;          /* [batch, n_actions * n_atoms] target network on s'                                 */
    const float* online;        /* [batch, n_actions * n_atoms] online (training) network on s                        */
    const int64_t* actions;     /* [batch] taken actions                                                              */
    const double* rewards;      /* [batch]                                                                            */
    const uint8_t* game_overs;  /* [batch]                                                                            */
    double discount;
    float kappa;                /* huber_loss_interval                                                                */
    int32_t batch, n_actions, n_atoms;
    float* dq;                  /* [batch, n_actions * n_atoms] d loss / d online (the trunk's output gradient)       */
    float* loss;                /* [1] total loss                                                                     */
    float* targets;             /* [batch, n_atoms] optional: T as fed to the train op                                */
    float* taus;                /* [batch, n_atoms] optional: the quantile midpoints as fed (output_0_1)              */
    int64_t* target_actions;    /* [batch] optional: a*                                                               */
    float* workspace;           /* [batch] per-sample loss sums                                                       */
} cb200_qr_head_desc;
int cb200_qr_head(const cb200_qr_head_desc* desc, void* stream);

/* q_values output of the QuantileRegressionQHead (quantile_regression_q_head.py:65, qr_dqn_agent.py:72-73):
 * q[r] = sum_j (double)quantiles[r, j] * (1.0 / n_atoms) for `rows` rows of n_atoms, the arithmetic of Q' in
 * cb200_qr_head.  1 <= n_atoms <= 1024. */
int cb200_qr_q_values(const float* quantiles, int64_t rows, int32_t n_atoms, double* q_out, void* stream);

/* SACPolicyHead (heads/sac_head.py:60-97).  head_out [batch, 2*action_dim] = [mu | raw log-sigma]; log-sigma is clipped
 * to [-20, 2]; u = mu + exp(log_sigma) * eps; a = tanh(u); logp = MVN-diag log-prob of u minus the tanh squash
 * correction sum_j log(1 - a_j^2 + 1e-6).  Any output may be NULL. */
int cb200_sac_policy_sample(const float* head_out, const float* eps, int64_t batch, int32_t action_dim, float* raw_out,
                            float* actions_out, float* logp_out, void* stream);

/* d/d(head_out) of  mean_b logp(eps_logp)  -  sum_b <dq_da_b, tanh(mu + sigma * eps_q)_b>  -- the combination
 * policy_grads = dlogp_dphi - dq_dphi of soft_actor_critic_agent.py:213-232, each term with its own noise sample
 * (the reference evaluates them in separate sess.run calls which re-sample, sac_head.py:80). */
int cb200_sac_policy_grad(const float* head_out, const float* eps_logp, const float* eps_q, const float* dq_da,
                          int64_t batch, int32_t action_dim, float* d_head_out, void* stream);

/* qmin = min(q1, q2) (the rule of cb200_min2) and the seeds d mean_b(qmin) / dq1, dq2 (sac_q_head.py:84-86): the
 * seed float32(1) / float32(batch) goes to q1 where q1 <= q2 (tf.minimum's gradient rule), else to q2, and the other
 * seed is 0.  Outputs may be NULL. */
int cb200_sac_min_seed(const float* q1, const float* q2, int64_t batch, float* d1, float* d2, float* qmin,
                       void* stream);

/* out = a - b  (fp32) */
int cb200_sub(const float* a, const float* b, int64_t n, float* out, void* stream);

/* out[i] = (float) in[i] */
int cb200_f64_to_f32(const double* in, int64_t n, float* out, void* stream);

/* =====================================================================================================================
 * Scalar RL recurrences (fp64, as the reference computes them).
 * ===================================================================================================================*/

/* Generalised advantage estimation over a whole rollout of n transitions laid out episode after episode:
 * ActorCriticAgent.get_general_advantage_estimation_values (agents/actor_critic_agent.py:111-125: deltas, then
 * scipy.signal.lfilter([1],[1,-gamma*lambda]) on the reversed deltas) applied per episode as ClippedPPOAgent.
 * fill_advantages does (agents/clipped_ppo_agent.py:170-207): episodes end at game_over flags, the bootstrap value
 * appended at an episode end is 0 (:188), the value target is advantage + V(s_t) (:121), transitions after the last
 * game_over receive nothing (*n_valid = index of the last game_over + 1; later entries are still written but must be
 * ignored, cf. zip() truncation :203).  values[t] = V(s_t) (fp32 network output).  One block-wide scan of affine maps
 * (thread chunks -> warp shuffles -> shared memory). */
int cb200_gae_scan(const double* rewards, const float* values, const uint8_t* game_overs, int64_t n, double discount,
                   double gae_lambda, double* advantages, double* value_targets, int64_t* n_valid, void* stream);

/* x[:n_valid] = (x - mean) / std with the population std (clipped_ppo_agent.py:201), in place; x[n_valid:] = NaN.
 * n_valid may be NULL (= n).  mean_std_out (device double[2], may be NULL) receives mean and std. */
int cb200_standardize(double* x, int64_t n, const int64_t* n_valid, double* mean_std_out, void* stream);

/* Episode.update_discounted_rewards (core_types.py:771-790): out[t] = sum_{k < n_step} discount^k * r[t+k] inside t's
 * episode [ep_start[t], ep_end[t]), n_step == -1 => to the end of the episode; accumulated in the reference's order
 * (k ascending, running power of the discount), bit-identical to the numpy loop. */
int cb200_nstep_returns(const double* rewards, const int64_t* ep_start, const int64_t* ep_end, int64_t n,
                        double discount, int64_t n_step, double* out, void* stream);

/* NumpySharedRunningStats (utilities/shared_running_stats.py:115-164), used by ObservationNormalizationFilter
 * (filters/observation/observation_normalization_filter.py:71-78):
 *   push      : sum += sum_rows x, sumsq += sum_rows x^2   (fp64; the host adds `rows` to its count)
 *   finalize  : mean = sum/count; std = sqrt(max((sumsq - count*mean^2) / max(count-1, 1), epsilon)), every
 *               operation rounded on its own as numpy does (no fused multiply-add): bit-identical to the reference
 *               given the same sum, sumsq and count.  count > 0.
 *   normalize : clip((x - mean) / (std + 1e-15), lo, hi) -> fp32 (network feed) and/or fp64; bit-identical to numpy,
 *               np.clip's rules (a NaN passes through).  At least one of out32 / out64 must be given. */
int cb200_running_stats_push(const float* x, int64_t rows, int64_t cols, double* sum, double* sumsq, void* stream);
int cb200_running_stats_finalize(const double* sum, const double* sumsq, double count, double epsilon, int64_t cols,
                                 double* mean, double* std_out, void* stream);
int cb200_running_stats_normalize(const float* x, int64_t rows, int64_t cols, const double* mean, const double* std_in,
                                  double clip_lo, double clip_hi, float* out32, double* out64, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COACH_B200_H */
