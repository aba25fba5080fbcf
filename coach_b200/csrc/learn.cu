// coach_b200/csrc/learn.cu -- element-wise and reduction kernels of learn_from_batch (TD targets, head losses,
// global-norm clipping, TF-semantics Adam, polyak target update).  Reference lines are cited in include/coach_b200.h.
#include <math.h>

#include "common.cuh"

namespace cb200 {

// ---- DQN / DDQN TD targets ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dqn_td_targets_kernel(const float* __restrict__ q_next,
                                                             const float* __restrict__ q_select,
                                                             const float* __restrict__ q_online,
                                                             const int64_t* __restrict__ actions,
                                                             const double* __restrict__ rewards,
                                                             const uint8_t* __restrict__ game_overs, double discount,
                                                             int64_t B, int64_t A, float* __restrict__ targets,
                                                             double* __restrict__ td_err) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    // np.argmax: first maximum
    int64_t best = 0;
    float bv = q_select[i * A];
    for (int64_t a = 1; a < A; ++a) {
        const float v = q_select[i * A + a];
        if (v > bv) {
            bv = v;
            best = a;
        }
    }
    const int64_t act = actions[i];
    for (int64_t a = 0; a < A; ++a) targets[i * A + a] = q_online[i * A + a];
    // new_target = r + (1.0 - done) * discount * q'[a*]     (dqn_agent.py:100-101; left-to-right, fp64)
    const double not_done = __dsub_rn(1.0, game_overs[i] ? 1.0 : 0.0);
    const double t1 = __dmul_rn(__dmul_rn(not_done, discount), (double)q_next[i * A + best]);
    const double y = __dadd_rn(rewards[i], t1);
    if (act >= 0 && act < A) {
        td_err[i] = fabs(__dsub_rn(y, (double)q_online[i * A + act]));   // :102
        targets[i * A + act] = (float)y;                                 // :103 (fp32 array element assignment)
    } else {
        td_err[i] = 0.0;
    }
}

// ---- regression head loss (Huber / MSE) -----------------------------------------------------------------------------
// one CTA; fixed-order reduction => run-to-run bit-stable loss
__global__ void __launch_bounds__(1024) regression_head_kernel(const float* __restrict__ out,
                                                               const float* __restrict__ target,
                                                               const float* __restrict__ weights, int64_t B, int64_t W,
                                                               int huber, float loss_weight, float* __restrict__ d_out,
                                                               float* __restrict__ loss_out) {
    __shared__ float red[1024];
    float local = 0.f;
    const float inv_b = 1.0f / (float)B;
    for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
        const float w = loss_weight * (weights ? weights[b] : 1.0f);
        float row = 0.f;
        for (int64_t a = 0; a < W; ++a) {
            const float e = out[b * W + a] - target[b * W + a];     // predictions - labels
            float l, g;
            if (huber) {
                const float ae = fabsf(e);
                const float q = fminf(ae, 1.0f);                    // delta = 1
                const float lin = ae - q;
                l = 0.5f * q * q + lin;
                g = (ae <= 1.0f) ? e : (e > 0.f ? 1.0f : -1.0f);
            } else {
                l = e * e;
                g = 2.0f * e;
            }
            row += l;
            d_out[b * W + a] = w * inv_b * g;
        }
        local += w * row;
    }
    red[threadIdx.x] = local;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0 && loss_out) *loss_out = red[0] * inv_b;
}

// ---- fused DQN / DDQN Q-head step -----------------------------------------------------------------------------------
// Everything between the feature layer and the loss in ONE launch (+ one small reduction launch):
//   Q(s') of the target head, Q(s) of the online head [, Q(s') of the online head: DDQN action selection]
//   (q_head.py:52-54: Dense(num_actions) on the middleware output)  ->  TD targets / errors (dqn_agent.py:92-103,
//   fp64, bit-exact given the Q values)  ->  Huber / MSE head loss and dL/dQ (head.py:165-177)  ->  the head's own
//   backward: dL/dW = h^T dQ, dL/db = sum_b dQ, and the gradient w.r.t. the feature layer's pre-activation
//   dL/dz = (dQ W^T) * relu'(h), written as fp32 and as operand planes for the feature layer's tensor-core GEMMs.
// Replaces 8-9 launches of latency-bound kernels (three 512x512x6 skinny GEMMs, TD targets, loss, two backward GEMMs, a
// transpose) whose arithmetic is 12 MFLOP in total.
// One warp = kHeadRows batch rows; lane l owns features [l K/32, (l+1) K/32): its slice of a row of h is contiguous, so
// is its slice of W [K, A] (row-major), and the dL/dz planes get whole 16-byte core rows.  Dot products are reduced with
// an xor butterfly (every lane ends with the same bits); batch-wise sums (dW, db, loss) go through per-warp partials in
// global memory and a fixed-order second pass: run-to-run identical bits.
// exact 3-way bf16 truncation split of 8 fp32 values into three 16-byte groups (same arithmetic as gemm::split8 of
// nn_gemm_tc.cuh, restated here because that header defines kernels) and the core-tiled element index of nn_gemm.cuh
struct HeadSplit8 {
    uint4 h, m, l;
};
__device__ __forceinline__ HeadSplit8 head_split8(const float (&x)[8]) {
    uint32_t hb[8], mb[8], lb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        hb[j] = __float_as_uint(x[j]) & 0xffff0000u;
        const float r1 = x[j] - __uint_as_float(hb[j]);
        mb[j] = __float_as_uint(r1) & 0xffff0000u;
        lb[j] = __float_as_uint(r1 - __uint_as_float(mb[j]));
    }
    HeadSplit8 s;
    s.h = make_uint4(__byte_perm(hb[0], hb[1], 0x7632), __byte_perm(hb[2], hb[3], 0x7632),
                     __byte_perm(hb[4], hb[5], 0x7632), __byte_perm(hb[6], hb[7], 0x7632));
    s.m = make_uint4(__byte_perm(mb[0], mb[1], 0x7632), __byte_perm(mb[2], mb[3], 0x7632),
                     __byte_perm(mb[4], mb[5], 0x7632), __byte_perm(mb[6], mb[7], 0x7632));
    s.l = make_uint4(__byte_perm(lb[0], lb[1], 0x7632), __byte_perm(lb[2], lb[3], 0x7632),
                     __byte_perm(lb[4], lb[5], 0x7632), __byte_perm(lb[6], lb[7], 0x7632));
    return s;
}
__device__ __forceinline__ size_t head_tiled_elem(size_t prow, int col, int pcols) {
    return ((prow >> 3) * (size_t)(pcols >> 3) + (size_t)(col >> 3)) * 64 + (prow & 7) * 8 + (col & 7);
}

constexpr int kHeadMaxA = 8;
constexpr int kHeadRows = 2;
constexpr int kHeadWarps = 8;

struct HeadParams {
    const float *h_next, *h_online, *h_select;
    const float *w_target, *b_target, *w_online, *b_online;
    const int64_t* actions;
    const double* rewards;
    const uint8_t* game_overs;
    const float* weights;
    double discount;
    int huber, B, K, A;
    float *q_online, *q_next, *targets;
    double* td_err;
    float *dq, *loss, *dh;
    uint16_t* dh_planes;
    int64_t dh_plane_stride;
    float *dw, *db, *workspace;
    // target rules beyond DQN / DDQN (appended: the DQN rule reads nothing below)
    const float* h_target_s;
    const double* mc_returns;
    double pal_alpha, mc_mixing_rate;
    float *q_select, *q_target_s;
};

// Lane l owns features k = l + 32 j (j < KPL): a row of h is read with coalesced 128-byte loads and the head kernels,
// staged TRANSPOSED in shared memory (Wt[a][k]), are read conflict-free.  The row's dL/dz goes through a per-warp
// shared-memory row so that it leaves as whole 16-byte core rows / float4s.
template <int KPL>
__device__ __forceinline__ void head_dot(const float* __restrict__ hrow, const float* __restrict__ wt /* smem [A][K] */,
                                         const float* __restrict__ bias, int A, int K, int lane, float (&hv)[KPL],
                                         float (&q)[kHeadMaxA]) {
#pragma unroll
    for (int j = 0; j < KPL; ++j) hv[j] = __ldg(hrow + lane + 32 * j);
#pragma unroll
    for (int a = 0; a < kHeadMaxA; ++a) {
        q[a] = 0.f;
        if (a < A) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < KPL; ++j) s = fmaf(hv[j], wt[a * K + lane + 32 * j], s);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            q[a] = s + __ldg(bias + a);
        }
    }
}

// Per-row arithmetic shared by the DQN head and the ensemble head: every lane of the warp evaluates it on identical
// values (head_dot leaves the same bits in every lane).
// DDQN / DQN target action (ddqn_agent.py:42-43 / dqn_agent.py:78-79; np.argmax: first maximum) -> target Q of it
__device__ __forceinline__ float head_q_best(const float (&qs)[kHeadMaxA], const float (&qn)[kHeadMaxA], bool use_sel,
                                             int A) {
    float bv = use_sel ? qs[0] : qn[0];
    float q_best = qn[0];
#pragma unroll
    for (int a = 1; a < kHeadMaxA; ++a) {
        const float sv = use_sel ? qs[a] : qn[a];
        if (a < A && sv > bv) {
            bv = sv;
            q_best = qn[a];
        }
    }
    return q_best;
}
// new_target = r + (1.0 - done) * discount * q'[a*]   (dqn_agent.py:100-101; left-to-right, fp64)
__device__ __forceinline__ double head_td_target(double reward, uint8_t game_over, double discount, float q_best) {
    const double not_done = __dsub_rn(1.0, game_over ? 1.0 : 0.0);
    return __dadd_rn(reward, __dmul_rn(__dmul_rn(not_done, discount), (double)q_best));
}
// the fp32 target of the taken action under a target rule, given the double-DQN target y (fp64, head_td_target), the
// target head's Q values on s' (qn) and on s (qt, PAL only), q_best = qn[a*], and the sample's Monte Carlo return R.
// Every operation is an explicit _rn intrinsic: the reference's numpy rounding order, nothing FMA-contracted.
template <int RULE>
__device__ __forceinline__ float head_rule_target(double y, float q_best, const float (&qn)[kHeadMaxA],
                                                  const float (&qt)[kHeadMaxA], int64_t act, int A, double R,
                                                  double alpha, double rho) {
    if constexpr (RULE == CB200_TARGET_DQN) {
        return (float)y;                                                  // dqn_agent.py:103 (fp32 element assignment)
    } else if constexpr (RULE == CB200_TARGET_MMC) {
        // mmc_agent.py:72-78: (1 - rho) * one_step_target + rho * monte_carlo_target, all fp64, then stored as fp32
        return (float)__dadd_rn(__dmul_rn(__dsub_rn(1.0, rho), y), __dmul_rn(rho, R));
    } else {
        // pal_agent.py:83-106: every statement writes into the float32 TD_targets array (numpy 2 scalar promotion)
        float vt = qt[0], vn = qn[0], qta = qt[0];
#pragma unroll
        for (int a = 1; a < kHeadMaxA; ++a) {
            if (a < A) {
                vt = qt[a] > vt ? qt[a] : vt;                             // np.max(q_st_target, 1)
                vn = qn[a] > vn ? qn[a] : vn;                             // np.max(q_st_plus_1_target, 1)
                if (a == act) qta = qt[a];
            }
        }
        const float t0 = (float)y;
        const float adv = __fsub_rn(vt, qta);                             // advantage_learning_update
        const float nadv = __fsub_rn(vn, q_best);                         // next_advantage_learning_update
        // Python's min(adv, nadv): the first argument unless the second is strictly smaller
        const float m = (RULE == CB200_TARGET_PAL_PERSISTENT && nadv < adv) ? nadv : adv;
        const float t1 = __fsub_rn(t0, __fmul_rn((float)alpha, m));       // -= alpha * m (alpha demoted to fp32)
        const float t2 = __fmul_rn((float)__dsub_rn(1.0, rho), t1);       // (1 - rho) * t, 1 - rho in fp64 then demoted
        return (float)__dadd_rn((double)t2, __dmul_rn(rho, R));           // + rho * R: fp32 + fp64 -> fp64
    }
}

// head loss of one row and dL/dQ (head.py:165-177; tf.losses.huber_loss delta = 1 / mean_squared_error)
__device__ __forceinline__ float head_loss_grad(const float (&qo)[kHeadMaxA], const float (&tgt)[kHeadMaxA], int A,
                                                int huber, float w, float inv_b, float (&dq)[kHeadMaxA]) {
    float row = 0.f;
#pragma unroll
    for (int a = 0; a < kHeadMaxA; ++a) {
        dq[a] = 0.f;
        if (a < A) {
            const float e = qo[a] - tgt[a];
            float l, g;
            if (huber) {
                const float ae = fabsf(e);
                const float qq = fminf(ae, 1.0f);
                l = 0.5f * qq * qq + (ae - qq);
                g = (ae <= 1.0f) ? e : (e > 0.f ? 1.0f : -1.0f);
            } else {
                l = e * e;
                g = 2.0f * e;
            }
            row += l;
            dq[a] = w * inv_b * g;
        }
    }
    return row;
}
// one row of dL/dz, staged lane-strided in the warp's row buffer: lane l takes the KPL consecutive features
// [l KPL, (l + 1) KPL) and writes them as float4s and / or as whole 16-byte core rows of the three operand planes
template <int KPL>
__device__ __forceinline__ void head_store_dz(const float* rowbuf, int lane, int r, int K, float* dh,
                                              uint16_t* dh_planes, int64_t dh_plane_stride) {
    float dz[KPL];
#pragma unroll
    for (int j = 0; j < KPL / 4; ++j) {
        const float4 v = *reinterpret_cast<const float4*>(rowbuf + lane * KPL + 4 * j);
        dz[4 * j] = v.x; dz[4 * j + 1] = v.y; dz[4 * j + 2] = v.z; dz[4 * j + 3] = v.w;
    }
    if (dh) {
        float4* o = reinterpret_cast<float4*>(dh + (size_t)r * K + lane * KPL);
#pragma unroll
        for (int j = 0; j < KPL / 4; ++j) o[j] = make_float4(dz[4 * j], dz[4 * j + 1], dz[4 * j + 2], dz[4 * j + 3]);
    }
    if (dh_planes) {
#pragma unroll
        for (int c8 = 0; c8 < KPL / 8; ++c8) {
            const float x8[8] = {dz[8 * c8], dz[8 * c8 + 1], dz[8 * c8 + 2], dz[8 * c8 + 3],
                                 dz[8 * c8 + 4], dz[8 * c8 + 5], dz[8 * c8 + 6], dz[8 * c8 + 7]};
            const HeadSplit8 sp = head_split8(x8);
            uint16_t* d = dh_planes + head_tiled_elem((size_t)r, lane * KPL + 8 * c8, K);
            *reinterpret_cast<uint4*>(d) = sp.h;
            *reinterpret_cast<uint4*>(d + dh_plane_stride) = sp.m;
            *reinterpret_cast<uint4*>(d + 2 * dh_plane_stride) = sp.l;
        }
    }
}

// RULE: CB200_TARGET_* (the target of the taken action; see head_rule_target).  PAL adds one head_dot, the target
// head on h_target_s; the loss, dL/dQ and the backward pass are the same for every rule.
template <int KPL, int RULE>
__global__ void __launch_bounds__(32 * kHeadWarps) dqn_head_fused_kernel(HeadParams p) {
    constexpr bool kPal = RULE == CB200_TARGET_PAL || RULE == CB200_TARGET_PAL_PERSISTENT;
    extern __shared__ __align__(16) float head_smem[];     // Wt_online [A][K] | Wt_target [A][K] | row buffers [warps][K]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = blockIdx.x * kHeadWarps + warp;                        // global warp
    const int A = p.A, K = p.K;
    float* wt_on = head_smem;
    float* wt_tg = head_smem + A * K;
    float* rowbuf = head_smem + 2 * A * K + warp * K;
    for (int i = threadIdx.x; i < A * K; i += blockDim.x) {               // W [K, A] row-major -> Wt [A][K]
        const int k = i / A, a = i - k * A;
        wt_on[a * K + k] = __ldg(p.w_online + i);
        wt_tg[a * K + k] = __ldg(p.w_target + i);
    }
    __syncthreads();
    float acc_w[KPL][kHeadMaxA];                                          // this lane's slice of dW, over the warp's rows
    float acc_b[kHeadMaxA], acc_loss = 0.f;
#pragma unroll
    for (int j = 0; j < KPL; ++j)
#pragma unroll
        for (int a = 0; a < kHeadMaxA; ++a) acc_w[j][a] = 0.f;
#pragma unroll
    for (int a = 0; a < kHeadMaxA; ++a) acc_b[a] = 0.f;
    const float inv_b = 1.0f / (float)p.B;
    const bool use_sel = p.h_select != nullptr;
    for (int rr = 0; rr < kHeadRows; ++rr) {
        const int r = gw * kHeadRows + rr;
        if (r >= p.B) break;
        float hv[KPL], qn[kHeadMaxA], qs[kHeadMaxA], qo[kHeadMaxA], qt[kHeadMaxA];
        head_dot<KPL>(p.h_next + (size_t)r * K, wt_tg, p.b_target, A, K, lane, hv, qn);
        if (use_sel) head_dot<KPL>(p.h_select + (size_t)r * K, wt_on, p.b_online, A, K, lane, hv, qs);
        if constexpr (kPal) head_dot<KPL>(p.h_target_s + (size_t)r * K, wt_tg, p.b_target, A, K, lane, hv, qt);
        head_dot<KPL>(p.h_online + (size_t)r * K, wt_on, p.b_online, A, K, lane, hv, qo);    // hv = h_online slice
        // ---- TD target (every lane, identical values) -- dqn_agent.py:92-103 ------------------------------------------
        const float q_best = head_q_best(qs, qn, use_sel, A);
        const int64_t act = p.actions[r];
        const double y = head_td_target(p.rewards[r], p.game_overs[r], p.discount, q_best);
        float tgt[kHeadMaxA], dq[kHeadMaxA];
        double td = 0.0;
        if constexpr (RULE == CB200_TARGET_DQN) {
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a) {
                tgt[a] = qo[a];
                if (a < A && a == act) {
                    td = fabs(__dsub_rn(y, (double)qo[a]));
                    tgt[a] = (float)y;
                }
            }
        } else {
            const bool in_range = act >= 0 && act < A;
            const float ty = in_range ? head_rule_target<RULE>(y, q_best, qn, qt, act, A, p.mc_returns[r], p.pal_alpha,
                                                               p.mc_mixing_rate)
                                      : 0.f;
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a) {
                tgt[a] = qo[a];
                if (a < A && a == act) {
                    td = fabs(__dsub_rn((double)ty, (double)qo[a]));
                    tgt[a] = ty;
                }
            }
        }
        // ---- head loss and dL/dQ -----------------------------------------------------------------------------------------
        const float w = p.weights ? p.weights[r] : 1.0f;
        const float row = head_loss_grad(qo, tgt, A, p.huber, w, inv_b, dq);
        acc_loss += w * row;
        if (lane == 0) {
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a) {
                if (a < A) {
                    p.q_online[(size_t)r * A + a] = qo[a];
                    if (p.q_next) p.q_next[(size_t)r * A + a] = qn[a];
                    p.targets[(size_t)r * A + a] = tgt[a];
                    p.dq[(size_t)r * A + a] = dq[a];
                    if constexpr (RULE != CB200_TARGET_DQN) {
                        if (p.q_select) p.q_select[(size_t)r * A + a] = qs[a];
                        if (kPal && p.q_target_s) p.q_target_s[(size_t)r * A + a] = qt[a];
                    }
                }
            }
            p.td_err[r] = td;
        }
        // ---- backward of the head for this row ---------------------------------------------------------------------------
        __syncwarp();                                                     // the previous row's readers are done
#pragma unroll
        for (int j = 0; j < KPL; ++j) {
            float s = 0.f;
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a)
                if (a < A) {
                    s = fmaf(dq[a], wt_on[a * K + lane + 32 * j], s);
                    acc_w[j][a] = fmaf(hv[j], dq[a], acc_w[j][a]);
                }
            rowbuf[lane + 32 * j] = hv[j] > 0.f ? s : 0.f;                // relu'(h) on the post-activation value
        }
#pragma unroll
        for (int a = 0; a < kHeadMaxA; ++a) acc_b[a] += dq[a];
        __syncwarp();
        head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
    }
    // ---- per-warp partials: [dW (K * A) | db (A) | loss (1)] --------------------------------------------------------------
    float* part = p.workspace + (size_t)gw * ((size_t)K * A + A + 1);
#pragma unroll
    for (int j = 0; j < KPL; ++j)
#pragma unroll
        for (int a = 0; a < kHeadMaxA; ++a)
            if (a < A) part[((size_t)lane + 32 * j) * A + a] = acc_w[j][a];
    if (lane == 0) {
#pragma unroll
        for (int a = 0; a < kHeadMaxA; ++a)
            if (a < A) part[(size_t)K * A + a] = acc_b[a];
        part[(size_t)K * A + A] = acc_loss;
    }
}

// [nparts][n_out] partials -> dW | db | loss: a block owns 32 consecutive outputs, its 8 warps walk the partials 8
// apart (coalesced 128-byte reads) and the 8 sums are folded in a fixed order
__global__ void __launch_bounds__(256) dqn_head_reduce_kernel(const float* __restrict__ ws, int nparts, int n_out,
                                                              int KA, int A, float inv_b, float* __restrict__ dw,
                                                              float* __restrict__ db, float* __restrict__ loss) {
    __shared__ float red[8][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + lane;
    float s = 0.f;
    if (i < n_out)
        for (int q = w; q < nparts; q += 8) s += ws[(size_t)q * n_out + i];
    red[w][lane] = s;
    __syncthreads();
    if (w == 0 && i < n_out) {
        for (int k = 1; k < 8; ++k) s += red[k][lane];
        if (i < KA) dw[i] = s;
        else if (i < KA + A) db[i - KA] = s;
        else if (loss) *loss = s * inv_b;
    }
}

// ---- fused Bootstrapped DQN ensemble head ---------------------------------------------------------------------------
// H Q heads on one feature layer: head h owns the columns [h A, (h + 1) A) of one Dense(H A) kernel [K, H A]
// (bootstrapped_dqn_agent.py:26-30).  Per head: Q of the three bindings, the double-DQN target of the head's own
// selection where the sample's bootstrap mask is set (bootstrapped_dqn_agent.py:57-86; masked-out rows keep the online
// prediction, so their dL/dQ is exactly 0), the head's loss (head.py:170-181) and its kernel / bias gradients.  The
// gradient into the feature layer is r * sum_h dQ_h W_h^T, masked with relu'(h) (general_network.py:304-325: every head
// copy reads (1 - r) stop_gradient(x) + r x).
// Both networks' kernels of all heads do not fit in shared memory at H = 10, K = 512: the block stages one head at a
// time and walks the heads in order; each warp accumulates its rows' sum over heads in its own shared-memory rows (lane
// l owns features l + 32 j, as in head_dot), so no cross-block accumulation is needed and the bits are run-to-run
// stable.  Per-head batch sums (dW, db, loss) leave through per-warp partials and a fixed-order second pass.
struct EnsembleParams {
    const float *h_next, *h_online, *h_select;
    const float *w_target, *b_target, *w_online, *b_online;
    const int64_t* actions;
    const double* rewards;
    const uint8_t* game_overs;
    const uint8_t* masks;
    double discount;
    int huber, B, K, H, A;
    float rescale;
    float *q_online, *q_next, *q_select, *targets, *dq;
    float* dh;
    uint16_t* dh_planes;
    int64_t dh_plane_stride;
    float* workspace;
};

template <int KPL>
__global__ void __launch_bounds__(32 * kHeadWarps) ensemble_head_fused_kernel(EnsembleParams p) {
    // Wt_online [A][K] | Wt_target [A][K] of the current head | dz rows [warps][kHeadRows][K]
    extern __shared__ __align__(16) float head_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = blockIdx.x * kHeadWarps + warp;
    const int A = p.A, K = p.K, HA = p.H * p.A;
    float* wt_on = head_smem;
    float* wt_tg = head_smem + A * K;
    float* dzrows = head_smem + 2 * A * K + warp * kHeadRows * K;
#pragma unroll
    for (int rr = 0; rr < kHeadRows; ++rr)
#pragma unroll
        for (int j = 0; j < KPL; ++j) dzrows[rr * K + lane + 32 * j] = 0.f;
    const float inv_b = 1.0f / (float)p.B;
    const size_t per_head = (size_t)K * A + A + 1;
    float* part = p.workspace + (size_t)gw * per_head * p.H;
    for (int h = 0; h < p.H; ++h) {
        __syncthreads();                                                  // the previous head's readers are done
        for (int i = threadIdx.x; i < A * K; i += blockDim.x) {           // W[:, hA:(h+1)A] -> Wt [A][K]
            const int k = i / A, a = i - k * A;
            wt_on[a * K + k] = __ldg(p.w_online + (size_t)k * HA + h * A + a);
            wt_tg[a * K + k] = __ldg(p.w_target + (size_t)k * HA + h * A + a);
        }
        __syncthreads();
        float acc_w[KPL][kHeadMaxA];
        float acc_b[kHeadMaxA], acc_loss = 0.f;
#pragma unroll
        for (int j = 0; j < KPL; ++j)
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a) acc_w[j][a] = 0.f;
#pragma unroll
        for (int a = 0; a < kHeadMaxA; ++a) acc_b[a] = 0.f;
#pragma unroll
        for (int rr = 0; rr < kHeadRows; ++rr) {
            const int r = gw * kHeadRows + rr;
            if (r >= p.B) continue;
            float hv[KPL], qn[kHeadMaxA], qs[kHeadMaxA], qo[kHeadMaxA];
            head_dot<KPL>(p.h_next + (size_t)r * K, wt_tg, p.b_target + h * A, A, K, lane, hv, qn);
            head_dot<KPL>(p.h_select + (size_t)r * K, wt_on, p.b_online + h * A, A, K, lane, hv, qs);
            head_dot<KPL>(p.h_online + (size_t)r * K, wt_on, p.b_online + h * A, A, K, lane, hv, qo);
            const bool use = p.masks[(size_t)r * p.H + h] != 0;
            const float q_best = head_q_best(qs, qn, true, A);
            const int64_t act = p.actions[r];
            const double y = head_td_target(p.rewards[r], p.game_overs[r], p.discount, q_best);
            float tgt[kHeadMaxA], dq[kHeadMaxA];
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a) tgt[a] = (use && a < A && a == act) ? (float)y : qo[a];
            acc_loss += head_loss_grad(qo, tgt, A, p.huber, 1.0f, inv_b, dq);
            if (lane == 0) {
                const size_t o = (size_t)r * HA + h * A;
#pragma unroll
                for (int a = 0; a < kHeadMaxA; ++a) {
                    if (a < A) {
                        p.q_online[o + a] = qo[a];
                        if (p.q_next) p.q_next[o + a] = qn[a];
                        if (p.q_select) p.q_select[o + a] = qs[a];
                        p.targets[o + a] = tgt[a];
                        p.dq[o + a] = dq[a];
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < KPL; ++j) {
                float s = 0.f;
#pragma unroll
                for (int a = 0; a < kHeadMaxA; ++a)
                    if (a < A) {
                        s = fmaf(dq[a], wt_on[a * K + lane + 32 * j], s);
                        acc_w[j][a] = fmaf(hv[j], dq[a], acc_w[j][a]);
                    }
                dzrows[rr * K + lane + 32 * j] += s;
            }
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a) acc_b[a] += dq[a];
        }
        // per-warp partials of head h, head-major: [dW_h (K * A) | db_h (A) | loss_h (1)] -- the lanes' stores are as
        // dense as dqn_head_fused_kernel's; the reduction scatters the sums into the [K, H A] kernel layout once
        float* ph = part + (size_t)h * per_head;
#pragma unroll
        for (int j = 0; j < KPL; ++j)
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a)
                if (a < A) ph[((size_t)lane + 32 * j) * A + a] = acc_w[j][a];
        if (lane == 0) {
#pragma unroll
            for (int a = 0; a < kHeadMaxA; ++a)
                if (a < A) ph[(size_t)K * A + a] = acc_b[a];
            ph[(size_t)K * A + A] = acc_loss;
        }
    }
    // dL/dz = r * (sum over heads) * relu'(h), rescaled once in fp32 before the plane split
#pragma unroll
    for (int rr = 0; rr < kHeadRows; ++rr) {
        const int r = gw * kHeadRows + rr;
        if (r >= p.B) continue;
        float* row = dzrows + rr * K;
#pragma unroll
        for (int j = 0; j < KPL; ++j) {
            const float hv = __ldg(p.h_online + (size_t)r * K + lane + 32 * j);
            row[lane + 32 * j] = hv > 0.f ? __fmul_rn(p.rescale, row[lane + 32 * j]) : 0.f;
        }
        __syncwarp();
        head_store_dz<KPL>(row, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
    }
}

// [nparts][H][K A + A + 1] partials -> dW [K, H A] | db [H A] | per-head losses, in the fixed order of
// dqn_head_reduce_kernel
__global__ void __launch_bounds__(256) ensemble_head_reduce_kernel(const float* __restrict__ ws, int nparts, int n_out,
                                                                   int KA, int A, int HA, float inv_b,
                                                                   float* __restrict__ dw, float* __restrict__ db,
                                                                   float* __restrict__ losses) {
    __shared__ float red[8][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + lane;
    float s = 0.f;
    if (i < n_out)
        for (int q = w; q < nparts; q += 8) s += ws[(size_t)q * n_out + i];
    red[w][lane] = s;
    __syncthreads();
    if (w == 0 && i < n_out) {
        for (int k = 1; k < 8; ++k) s += red[k][lane];
        const int h = i / (KA + A + 1), j = i - h * (KA + A + 1);
        if (j < KA) dw[(size_t)(j / A) * HA + h * A + j % A] = s;
        else if (j < KA + A) db[h * A + j - KA] = s;
        else losses[h] = s * inv_b;
    }
}
// total loss = sum over the heads (general_network.py:352-360), in head order
__global__ void ensemble_loss_total_kernel(const float* __restrict__ losses, int H, float* __restrict__ total) {
    float s = losses[0];
    for (int h = 1; h < H; ++h) s = __fadd_rn(s, losses[h]);
    *total = s;
}

// ---- ensemble acting values: [E, H A] -> [E, A] ---------------------------------------------------------------------
// the exploration policies' numpy arithmetic (exploration_policies/bootstrapped.py:70-84, ucb.py:70-83) in fp32 with
// explicit rounding: numpy reduces axis 0 of a [H, A] array row after row, true-divides by H, and np.std squares the
// deviations from that mean, sums them in the same order, divides by H and takes the square root
__global__ void ensemble_action_values_kernel(const float* __restrict__ q, int E, int H, int A, int mode,
                                              const int32_t* __restrict__ head, float lamb, float* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const float* qe = q + (size_t)e * H * A;
    float* o = out + (size_t)e * A;
    if (mode == CB200_ENSEMBLE_SELECT) {
        const int h = head[e];
        for (int a = 0; a < A; ++a) o[a] = qe[(size_t)h * A + a];
        return;
    }
    if (mode == CB200_ENSEMBLE_VOTE) {
        // np.argmax per head (first maximum), np.bincount, np.argmax of the counts (first maximum), one-hot
        int best_c = 0, best_n = -1;
        for (int c = 0; c < A; ++c) {
            int n = 0;
            for (int h = 0; h < H; ++h) {
                const float* qh = qe + (size_t)h * A;
                int am = 0;
                for (int a = 1; a < A; ++a)
                    if (qh[a] > qh[am]) am = a;
                n += am == c;
            }
            if (n > best_n) {
                best_n = n;
                best_c = c;
            }
        }
        for (int a = 0; a < A; ++a) o[a] = a == best_c ? 1.0f : 0.0f;
        return;
    }
    const float fh = (float)H;
    for (int a = 0; a < A; ++a) {
        float s = qe[a];
        for (int h = 1; h < H; ++h) s = __fadd_rn(s, qe[(size_t)h * A + a]);
        const float mean = __fdiv_rn(s, fh);
        if (mode == CB200_ENSEMBLE_MEAN) {
            o[a] = mean;
            continue;
        }
        const float d0 = __fsub_rn(qe[a], mean);
        float ss = __fmul_rn(d0, d0);
        for (int h = 1; h < H; ++h) {
            const float d = __fsub_rn(qe[(size_t)h * A + a], mean);
            ss = __fadd_rn(ss, __fmul_rn(d, d));
        }
        const float sd = __fsqrt_rn(__fdiv_rn(ss, fh));
        o[a] = __fadd_rn(mean, __fmul_rn(lamb, sd));
    }
}

__global__ void dueling_fwd_kernel(const float* __restrict__ v, const float* __restrict__ adv, int64_t B, int64_t A,
                                   float* __restrict__ q) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    float s = 0.f;
    for (int64_t a = 0; a < A; ++a) s += adv[i * A + a];
    const float mean = s / (float)A;
    for (int64_t a = 0; a < A; ++a) q[i * A + a] = v[i] + (adv[i * A + a] - mean);
}
__global__ void dueling_bwd_kernel(const float* __restrict__ dq, int64_t B, int64_t A, float* __restrict__ d_v,
                                   float* __restrict__ d_adv) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    float s = 0.f;
    for (int64_t a = 0; a < A; ++a) s += dq[i * A + a];
    d_v[i] = s;
    const float mean = s / (float)A;
    for (int64_t a = 0; a < A; ++a) d_adv[i * A + a] = dq[i * A + a] - mean;
}

// ---- flat-buffer reductions / updates -------------------------------------------------------------------------------
constexpr int kRedBlocks = 1024;
__global__ void __launch_bounds__(256) sumsq_stage1(const float* __restrict__ x, int64_t n, float* __restrict__ part) {
    __shared__ float red[256];
    // contiguous slab per block, strided inside the block: fixed association order for a given n
    const int64_t per = (n + gridDim.x - 1) / gridDim.x;
    const int64_t lo = (int64_t)blockIdx.x * per, hi = min(n, lo + per);
    float s = 0.f;
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) s = fmaf(x[i], x[i], s);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}
__global__ void __launch_bounds__(1024) sumsq_stage2(const float* __restrict__ part, int nparts,
                                                     float* __restrict__ out) {
    __shared__ float red[1024];
    red[threadIdx.x] = (threadIdx.x < nparts) ? part[threadIdx.x] : 0.f;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = red[0];
}

__global__ void __launch_bounds__(256) clip_kernel(float* __restrict__ g, int64_t n, const float* __restrict__ sumsq,
                                                   float clip) {
    const float norm = sqrtf(*sumsq);
    const float scale = clip / fmaxf(norm, clip);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        g[i] *= scale;
}
// tf.clip_by_value: the comparisons are false for NaN, which passes through unchanged
__global__ void __launch_bounds__(256) clip_by_value_kernel(float* __restrict__ g, int64_t n, float clip) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = g[i];
        g[i] = x < -clip ? -clip : (x > clip ? clip : x);
    }
}
__global__ void __launch_bounds__(256) scale_kernel(float* __restrict__ g, int64_t n, float s) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        g[i] *= s;
}

__global__ void __launch_bounds__(256) adam_tf_kernel(float* __restrict__ theta, float* __restrict__ m,
                                                      float* __restrict__ v, const float* __restrict__ g, int64_t n,
                                                      float alpha, float one_minus_b1, float one_minus_b2, float eps) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gi = g[i];
        const float mi = __fadd_rn(m[i], __fmul_rn(__fsub_rn(gi, m[i]), one_minus_b1));
        const float vi = __fadd_rn(v[i], __fmul_rn(__fsub_rn(__fmul_rn(gi, gi), v[i]), one_minus_b2));
        m[i] = mi;
        v[i] = vi;
        theta[i] = __fsub_rn(theta[i], __fdiv_rn(__fmul_rn(mi, alpha), __fadd_rn(__fsqrt_rn(vi), eps)));
    }
}

// Adam with its step state on the device: state = {beta1_power, beta2_power}.  Launch-parameter-constant, so a whole
// training step can be captured in a CUDA graph and replayed; adam_state_advance_kernel multiplies the powers.
__global__ void __launch_bounds__(256) adam_tf_dev_kernel(float* __restrict__ theta, float* __restrict__ m,
                                                          float* __restrict__ v, const float* __restrict__ g,
                                                          int64_t n, float lr, float one_minus_b1, float one_minus_b2,
                                                          float eps, const float* __restrict__ state) {
    const float alpha = __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.0f, state[1]))), __fsub_rn(1.0f, state[0]));
    // four parameters per thread through 128-bit accesses (the flat buffers are 32-byte aligned and padded to a multiple
    // of 8 elements: architectures/network.py ParamStore); same per-element operations, same bits
    const bool vec = (n % 4 == 0) && (((uintptr_t)theta | (uintptr_t)m | (uintptr_t)v | (uintptr_t)g) % 16 == 0);
    auto upd = [&](float& th, float& mm, float& vv, float gi) {
        mm = __fadd_rn(mm, __fmul_rn(__fsub_rn(gi, mm), one_minus_b1));
        vv = __fadd_rn(vv, __fmul_rn(__fsub_rn(__fmul_rn(gi, gi), vv), one_minus_b2));
        th = __fsub_rn(th, __fdiv_rn(__fmul_rn(mm, alpha), __fadd_rn(__fsqrt_rn(vv), eps)));
    };
    if (vec) {
        const int64_t n4 = n / 4;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            const float4 g4 = reinterpret_cast<const float4*>(g)[i];
            float4 t4 = reinterpret_cast<float4*>(theta)[i], m4 = reinterpret_cast<float4*>(m)[i],
                   v4 = reinterpret_cast<float4*>(v)[i];
            upd(t4.x, m4.x, v4.x, g4.x);
            upd(t4.y, m4.y, v4.y, g4.y);
            upd(t4.z, m4.z, v4.z, g4.z);
            upd(t4.w, m4.w, v4.w, g4.w);
            reinterpret_cast<float4*>(m)[i] = m4;
            reinterpret_cast<float4*>(v)[i] = v4;
            reinterpret_cast<float4*>(theta)[i] = t4;
        }
        return;
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float th = theta[i], mm = m[i], vv = v[i];
        upd(th, mm, vv, g[i]);
        m[i] = mm;
        v[i] = vv;
        theta[i] = th;
    }
}
__global__ void adam_state_advance_kernel(float* state, float beta1, float beta2) {
    state[0] = __fmul_rn(state[0], beta1);
    state[1] = __fmul_rn(state[1], beta2);
}
__global__ void add_i64_kernel(int64_t* x, int64_t delta) { *x += delta; }

__global__ void __launch_bounds__(256) polyak_kernel(float* __restrict__ target, const float* __restrict__ online,
                                                     int64_t n, float rate, float one_minus_rate) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        target[i] = __fadd_rn(__fmul_rn(rate, online[i]), __fmul_rn(one_minus_rate, target[i]));
}

static unsigned flat_grid(int64_t n) {
    int64_t g = (n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (unsigned)g;
}

// ---- fused N-step Q head --------------------------------------------------------------------------------------------
// One warp = one segment (n_step_q_agent.py:99-140): the bootstrap max of the target head, then the segment's rows
// walked backwards (i = L-1 .. 0) carrying the fp64 return R, and per row Q_online(s), the target, the loss, dL/dQ and
// the head's backward pass.  Only the taken action's target differs from Q, so dL/dQ is zero off that column: per row
// one column of dW / db and dh = dq_a W[:, a] relu'(h).  dW / db accumulate in the warp's shared-memory slice ([A][K],
// lane l owns k = l + 32 j: conflict-free) and leave as per-warp partials for dqn_head_reduce_kernel's fixed-order sum.
// Lanes hold identical copies of every per-row scalar (the dot products end in an xor butterfly).
constexpr int kNsMaxA = 18;
constexpr int kNsWarps = 4;

struct NstepParams {
    const float *h_online, *h_boot, *w_target, *b_target, *w_online, *b_online;
    const int64_t* actions;
    const double* rewards;
    const uint8_t* game_overs;
    const int32_t *seg_off, *seg_len;
    int S, rows, horizon, huber, K, A;
    double discount;
    float *q_online, *dq, *targets, *bootstrap, *dh;
    uint16_t* dh_planes;
    int64_t dh_plane_stride;
    float* workspace;
};

template <int KPL, int MAXA = kNsMaxA>
__device__ __forceinline__ void ns_dot(const float* __restrict__ hrow, const float* __restrict__ wt /* smem [A][K] */,
                                       const float* __restrict__ bias, int A, int K, int lane, float (&hv)[KPL],
                                       float (&q)[MAXA]) {
#pragma unroll
    for (int j = 0; j < KPL; ++j) hv[j] = __ldg(hrow + lane + 32 * j);
#pragma unroll
    for (int a = 0; a < MAXA; ++a) {
        q[a] = 0.f;
        if (a < A) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < KPL; ++j) s = fmaf(hv[j], wt[a * K + lane + 32 * j], s);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            q[a] = s + __ldg(bias + a);
        }
    }
}
// np.max over the actions (a NaN propagates)
__device__ __forceinline__ float ns_max(const float (&q)[kNsMaxA], int A) {
    float m = q[0];
#pragma unroll
    for (int a = 1; a < kNsMaxA; ++a)
        if (a < A && (q[a] > m || q[a] != q[a])) m = q[a];
    return m;
}
// W [K, N] row-major -> Wt [N][K] in shared memory, by the whole block
__device__ __forceinline__ void seg_head_wt(const float* __restrict__ w, int N, int K, float* wt) {
    for (int i = threadIdx.x; i < N * K; i += blockDim.x) {
        const int k = i / N, n = i - k * N;
        wt[n * K + k] = __ldg(w + i);
    }
}
// non-empty segments and the rows they cover (every warp counts them; integer sums are order-free)
__device__ __forceinline__ void seg_count(const int32_t* __restrict__ seg_len, int S, int lane, int& nseg, int& used) {
    nseg = 0;
    used = 0;
    for (int s = lane; s < S; s += 32) {
        const int L = seg_len[s];
        if (L > 0) {
            nseg += 1;
            used += L;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        nseg += __shfl_xor_sync(0xffffffffu, nseg, o);
        used += __shfl_xor_sync(0xffffffffu, used, o);
    }
}

template <int KPL>
__global__ void __launch_bounds__(32 * kNsWarps, 1) nstep_q_head_kernel(NstepParams p) {
    // Wt_online [A][K] | Wt_target [A][K] | per warp: row buffer [K] | dW [A][K] | db [32]
    extern __shared__ __align__(16) float ns_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = blockIdx.x * kNsWarps + warp, nwarps = gridDim.x * kNsWarps;
    const int A = p.A, K = p.K;
    float* wt_on = ns_smem;
    float* wt_tg = ns_smem + A * K;
    float* rowbuf = ns_smem + 2 * A * K + warp * (K + A * K + 32);
    float* dwacc = rowbuf + K;
    float* dbacc = dwacc + A * K;
    for (int i = threadIdx.x; i < A * K; i += blockDim.x) {               // W [K, A] row-major -> Wt [A][K]
        const int k = i / A, a = i - k * A;
        wt_on[a * K + k] = __ldg(p.w_online + i);
        wt_tg[a * K + k] = __ldg(p.w_target + i);
    }
    for (int i = lane; i < A * K + 32; i += 32) dwacc[i] = 0.f;
    int nseg, used;
    seg_count(p.seg_len, p.S, lane, nseg, used);
    __syncthreads();
    const float w = nseg > 0 ? 1.0f / (float)nseg : 0.f;                 // the mean over segments
    float acc_loss = 0.f;
    if (gw < p.S) {
        const int s = gw, L = p.seg_len[s], o = p.seg_off[s];
        const bool valid = L > 0 && o >= 0 && (int64_t)o + L <= p.rows;
        float hv[KPL], q[kNsMaxA];
        float boot = 0.f;
        bool boot_pending = false;
        if (p.horizon == CB200_NSTEP_NSTEP) {
            if (valid && !p.game_overs[o + L - 1]) {                       // else R = 0
                ns_dot<KPL>(p.h_boot + (size_t)s * K, wt_tg, p.b_target, A, K, lane, hv, q);
                boot = ns_max(q, A);
                boot_pending = true;
            }
            if (p.bootstrap && lane == 0) p.bootstrap[s] = boot;
        }
        const float inv_l = valid ? 1.0f / (float)L : 0.f;
        double R = 0.0;
        float seg_sum = 0.f;
        for (int i = (valid ? L : 0) - 1; i >= 0; --i) {
            const int r = o + i;
            const int64_t act = p.actions[r];
            const bool in_range = act >= 0 && act < A;
            double y = 0.0;
            bool replace = false;
            if (p.horizon == CB200_NSTEP_NSTEP) {
                // R = r_i + discount * R; right after a bootstrap, python float * np.float32 is an fp32 product
                const double rw = p.rewards[r];
                R = boot_pending ? __dadd_rn(rw, (double)__fmul_rn((float)p.discount, boot))
                                 : __dadd_rn(rw, __dmul_rn(p.discount, R));
                boot_pending = false;
                y = R;
                replace = true;
            } else if (p.horizon == CB200_NSTEP_ONESTEP) {
                ns_dot<KPL>(p.h_boot + (size_t)r * K, wt_tg, p.b_target, A, K, lane, hv, q);
                const float qb = ns_max(q, A);
                if (p.bootstrap && lane == 0) p.bootstrap[r] = qb;
                y = head_td_target(p.rewards[r], p.game_overs[r], p.discount, qb);
                replace = true;
            }
            ns_dot<KPL>(p.h_online + (size_t)r * K, wt_on, p.b_online, A, K, lane, hv, q);   // hv = h_online slice
            float qa = 0.f;
#pragma unroll
            for (int a = 0; a < kNsMaxA; ++a)
                if (a == act) qa = q[a];
            const bool live = replace && in_range;
            const float ta = (float)y;
            float dqa = 0.f;
            if (live) {                                                     // head.py:165-177 on the taken entry
                const float e = qa - ta;
                float l, g;
                if (p.huber) {
                    const float ae = fabsf(e);
                    const float qq = fminf(ae, 1.0f);
                    l = 0.5f * qq * qq + (ae - qq);
                    g = (ae <= 1.0f) ? e : (e > 0.f ? 1.0f : -1.0f);
                } else {
                    l = e * e;
                    g = 2.0f * e;
                }
                seg_sum += l;
                dqa = w * inv_l * g;
            }
            if (lane == 0) {
#pragma unroll
                for (int a = 0; a < kNsMaxA; ++a) {
                    if (a < A) {
                        const bool here = live && a == act;
                        p.q_online[(size_t)r * A + a] = q[a];
                        p.dq[(size_t)r * A + a] = here ? dqa : 0.f;
                        if (p.targets) p.targets[(size_t)r * A + a] = here ? ta : q[a];
                    }
                }
                if (live) dbacc[act] += dqa;
            }
            __syncwarp();                                                   // the previous row's readers are done
#pragma unroll
            for (int j = 0; j < KPL; ++j) {
                const int k = lane + 32 * j;
                const float wv = live ? wt_on[act * K + k] : 0.f;
                rowbuf[k] = hv[j] > 0.f ? fmaf(dqa, wv, 0.f) : 0.f;         // relu'(h) on the post-activation value
                if (live) dwacc[act * K + k] = fmaf(hv[j], dqa, dwacc[act * K + k]);
            }
            __syncwarp();
            head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
        }
        acc_loss = __fmul_rn(__fmul_rn(seg_sum, inv_l), w);
    }
    // padding rows [used, rows): zero Q, dq, targets, dh
    for (int r = used + gw; r < p.rows; r += nwarps) {
        __syncwarp();
#pragma unroll
        for (int j = 0; j < KPL; ++j) rowbuf[lane + 32 * j] = 0.f;
        for (int a = lane; a < A; a += 32) {
            p.q_online[(size_t)r * A + a] = 0.f;
            p.dq[(size_t)r * A + a] = 0.f;
            if (p.targets) p.targets[(size_t)r * A + a] = 0.f;
        }
        if (p.horizon == CB200_NSTEP_ONESTEP && p.bootstrap && lane == 0) p.bootstrap[r] = 0.f;
        __syncwarp();
        head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
    }
    __syncwarp();
    // per-warp partials in dqn_head_reduce_kernel's layout: [dW (K * A) | db (A) | loss (1)]
    float* part = p.workspace + (size_t)gw * ((size_t)K * A + A + 1);
#pragma unroll
    for (int j = 0; j < KPL; ++j)
        for (int a = 0; a < A; ++a) part[((size_t)lane + 32 * j) * A + a] = dwacc[a * K + lane + 32 * j];
    if (lane == 0) {
        for (int a = 0; a < A; ++a) part[(size_t)K * A + a] = dbacc[a];
        part[(size_t)K * A + A] = acc_loss;
    }
}

// ---- fused actor-critic (A3C) head ----------------------------------------------------------------------------------
// One Dense(1 + A) on the feature layer: column 0 is the VHead, columns 1..A the PolicyHead logits.  One warp = one
// segment (actor_critic_agent.py:111-165), the segment table and the conventions of nstep_q_head_kernel: V of each
// segment's last s' (the online network: the reference bootstraps with online_network.predict), the rows walked
// backwards carrying the A_VALUE return or the GAE recurrences in fp64 in numpy's / scipy.signal.lfilter's operation
// order, then per row the softmax, the three loss terms and a dense dL/dZ over all 1 + A columns.  dW / db accumulate in
// the warp's shared-memory slice and leave as per-warp partials for dqn_head_reduce_kernel's fixed-order sum.
constexpr int kAcMaxN = kNsMaxA + 1;

struct AcParams {
    const float *h, *h_boot, *w, *b;
    const int64_t* actions;
    const double* rewards;
    const uint8_t* game_overs;
    const int32_t *seg_off, *seg_len;
    int S, rows, mode, huber, K, A;
    double discount, gae_lambda;
    float beta_entropy, v_weight, p_weight;
    float *z, *dz, *probs, *targets, *advantages, *bootstrap, *dh;
    uint16_t* dh_planes;
    int64_t dh_plane_stride;
    float* workspace;
};

// p = softmax(z[1..A]) in fp32: exp(x - max) / sum, the sum in index order.  cb200_categorical_act uses the same code, so
// acting and learning see the same probabilities.
__device__ __forceinline__ void ac_softmax(const float (&z)[kAcMaxN], int A, float (&p)[kNsMaxA]) {
    float m = z[1];
#pragma unroll
    for (int a = 1; a < kNsMaxA; ++a)
        if (a < A) m = fmaxf(m, z[a + 1]);
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a) {
        p[a] = a < A ? expf(z[a + 1] - m) : 0.f;
        s += p[a];
    }
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a) p[a] = p[a] / s;
}

// first-order scipy.signal.lfilter([1], [1, -c]) step, as its C loop evaluates it: y = z + 1 * x, then the delay
// z' = x * 0 - y * (-c)
__device__ __forceinline__ double ac_lfilter(double x, double& z, double c) {
    const double y = __dadd_rn(z, x);
    z = __dsub_rn(__dmul_rn(x, 0.0), __dmul_rn(y, -c));
    return y;
}

// One row i (walking i = L-1 .. 0) of a segment's backward recurrence (actor_critic_agent.py:111-150), shared by the
// discrete and the Gaussian heads: given the row's reward rw and V, the fp64 target and advantage in numpy's /
// scipy.signal.lfilter's operation order.  The state: vnext (V of the next row; first the bootstrap value, 0 after a
// terminal state), A_VALUE's R and boot_pending (true until the first step of a bootstrapped segment), GAE's filter
// delays za / zr (zr started with ac_lfilter(vnext, zr, gamma)); gl = discount * gae_lambda, gamma32 = (float) discount.
__device__ __forceinline__ void ac_recurrence_step(int mode, double rw, float v, double gamma, float gamma32, double gl,
                                                   float& vnext, double& R, bool& boot_pending, double& za, double& zr,
                                                   double& target, double& adv) {
    if (mode == CB200_AC_A_VALUE) {
        // R = r_i + discount * R; right after a bootstrap, python float * np.float32 is an fp32 product
        R = boot_pending ? __dadd_rn(rw, (double)__fmul_rn(gamma32, vnext)) : __dadd_rn(rw, __dmul_rn(gamma, R));
        boot_pending = false;
        target = R;
        adv = __dsub_rn(R, (double)v);
    } else {
        // deltas = rewards + discount * values[1:] - values[:-1]: every discount * value is an fp32 product
        const double delta = __dsub_rn(__dadd_rn(rw, (double)__fmul_rn(gamma32, vnext)), (double)v);
        adv = ac_lfilter(delta, za, gl);
        const double ret = ac_lfilter(rw, zr, gamma);
        target = mode == CB200_AC_GAE_VALUE ? __dadd_rn(adv, (double)v) : ret;
    }
    vnext = v;
}

// PolicyHead's discrete terms of one row (heads/policy_head.py:91-100), shared by the actor-critic and the policy
// gradient heads: p = softmax(logits z[1..A]); Categorical(probs = p + eps): ls = log_softmax(log(p + eps)) (probs not
// renormalised), H = -sum u ls, logp = ls[act] (0 for an action outside [0, A)), u_act = p[act] + eps, su = sum u.
__device__ __forceinline__ void ac_policy_terms(const float (&z)[kAcMaxN], int A, int64_t act, float (&pr)[kNsMaxA],
                                                float (&ls)[kNsMaxA], float& ent, float& logp, float& u_act,
                                                float& su) {
    const float eps = 1.1920928955078125e-07f;                            // np.finfo(np.float32).eps
    ac_softmax(z, A, pr);
    su = 0.f;
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a)
        if (a < A) su += pr[a] + eps;
    const float lse = logf(su);
    ent = 0.f;
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a)
        if (a < A) {
            ls[a] = logf(pr[a] + eps) - lse;
            ent = fmaf(-(pr[a] + eps), ls[a], ent);
        }
    logp = 0.f;
    u_act = 1.f;
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a)
        if (a == act) {
            logp = ls[a];
            u_act = pr[a] + eps;
        }
}
// dL/d(logits) of -cp' logp(a) - cb' H per row, given cp = -(row weight) * (policy weight) * advantage (0 for an
// action out of range) and cb = (row weight) * beta: d/du_k = cp ([k = a] / u_a - 1 / su) + cb ls_k with u = p + eps,
// then the softmax Jacobian dz_k = p_k (g_k - sum_j p_j g_j); written to dz[off + k]
template <int NOUT>
__device__ __forceinline__ void ac_policy_dz(const float (&pr)[kNsMaxA], const float (&ls)[kNsMaxA], int A,
                                             int64_t act, float u_act, float su, float cp, float cb, int off,
                                             float (&dz)[NOUT]) {
    const float inv_su = 1.0f / su;
    float g[kNsMaxA], pg = 0.f;
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a)
        if (a < A) {
            g[a] = fmaf(cb, ls[a], cp * ((a == act ? 1.0f / u_act : 0.f) - inv_su));
            pg = fmaf(pr[a], g[a], pg);
        }
#pragma unroll
    for (int a = 0; a < kNsMaxA; ++a) dz[a + off] = a < A ? pr[a] * (g[a] - pg) : 0.f;
}

template <int KPL>
__global__ void __launch_bounds__(32 * kNsWarps, 1) actor_critic_head_kernel(AcParams p) {
    // Wt [N][K] | per warp: row buffer [K] | dW [N][K] | db [32]
    extern __shared__ __align__(16) float ac_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = blockIdx.x * kNsWarps + warp, nwarps = gridDim.x * kNsWarps;
    const int A = p.A, K = p.K, N = p.A + 1;
    float* wt = ac_smem;
    float* rowbuf = ac_smem + N * K + warp * (K + N * K + 32);
    float* dwacc = rowbuf + K;
    float* dbacc = dwacc + N * K;
    seg_head_wt(p.w, N, K, wt);
    for (int i = lane; i < N * K + 32; i += 32) dwacc[i] = 0.f;
    int nseg, used;
    seg_count(p.seg_len, p.S, lane, nseg, used);
    __syncthreads();
    const float w = nseg > 0 ? 1.0f / (float)nseg : 0.f;                 // the mean over segments
    float acc_loss = 0.f;
    if (gw < p.S) {
        const int s = gw, L = p.seg_len[s], o = p.seg_off[s];
        const bool valid = L > 0 && o >= 0 && (int64_t)o + L <= p.rows;
        const bool terminal = valid && p.game_overs[o + L - 1];
        float hv[KPL], z[kAcMaxN];
        float vnext = 0.f;                                                // V(s'_last), 0 after a terminal state
        if (valid && !terminal) {
            ns_dot<KPL, kAcMaxN>(p.h_boot + (size_t)s * K, wt, p.b, 1, K, lane, hv, z);
            vnext = z[0];
        }
        if (p.bootstrap && lane == 0) p.bootstrap[s] = vnext;
        const double gamma = p.discount, gl = __dmul_rn(p.discount, p.gae_lambda);
        const float gamma32 = (float)p.discount;
        // A_VALUE: R; GAE: the advantage filter's delay za and the discounted-return filter's delay zr, started on
        // values[-1] (= vnext)
        double R = 0.0, za = 0.0, zr = 0.0;
        bool boot_pending = !terminal;
        if (p.mode != CB200_AC_A_VALUE) ac_lfilter((double)vnext, zr, gamma);
        const float inv_l = valid ? 1.0f / (float)L : 0.f;
        const float c = w * inv_l;
        float seg_sum = 0.f;
        for (int i = (valid ? L : 0) - 1; i >= 0; --i) {
            const int r = o + i;
            const double rw = p.rewards[r];
            ns_dot<KPL, kAcMaxN>(p.h + (size_t)r * K, wt, p.b, N, K, lane, hv, z);     // hv = this row's features
            const float v = z[0];
            double target, adv;
            ac_recurrence_step(p.mode, rw, v, gamma, gamma32, gl, vnext, R, boot_pending, za, zr, target, adv);
            const float t32 = (float)target, a32 = (float)adv;
            // policy: p = softmax(logits); Categorical(probs = p + eps): log_softmax(log(p + eps)), probs not renormalised
            float pr[kNsMaxA], ls[kNsMaxA], ent, logp, u_act, su;
            const int64_t act = p.actions[r];
            const bool in_range = act >= 0 && act < A;
            ac_policy_terms(z, A, act, pr, ls, ent, logp, u_act, su);
            // loss terms of this row: VHead (weight v_weight), -log pi(a) A (weight p_weight), -beta H
            const float e = v - t32;
            float lv, gv;
            if (p.huber) {
                const float ae = fabsf(e);
                const float qq = fminf(ae, 1.0f);
                lv = 0.5f * qq * qq + (ae - qq);
                gv = fmaxf(-1.0f, fminf(e, 1.0f));
            } else {
                lv = e * e;
                gv = 2.0f * e;
            }
            const float lp = in_range ? -p.p_weight * logp * a32 : 0.f;
            seg_sum += p.v_weight * lv + lp - p.beta_entropy * ent;
            // dL/dZ: d/du_k = c (-p_weight A ([k = a] / u_a - 1 / su) + beta ls_k) with u = p + eps, then the softmax
            // Jacobian dz_k = p_k (g_k - sum_j p_j g_j)
            const float cp = in_range ? -c * p.p_weight * a32 : 0.f, cb = c * p.beta_entropy;
            float dz[kAcMaxN];
            dz[0] = c * p.v_weight * gv;
            ac_policy_dz(pr, ls, A, act, u_act, su, cp, cb, 1, dz);
            if (lane == 0) {
#pragma unroll
                for (int n = 0; n < kAcMaxN; ++n)
                    if (n < N) {
                        p.z[(size_t)r * N + n] = z[n];
                        if (p.dz) p.dz[(size_t)r * N + n] = dz[n];
                    }
                if (p.probs) {
#pragma unroll
                    for (int a = 0; a < kNsMaxA; ++a)
                        if (a < A) p.probs[(size_t)r * A + a] = pr[a];
                }
                if (p.targets) p.targets[r] = t32;
                if (p.advantages) p.advantages[r] = a32;
#pragma unroll
                for (int n = 0; n < kAcMaxN; ++n)
                    if (n < N) dbacc[n] += dz[n];
            }
            __syncwarp();                                                   // the previous row's readers are done
#pragma unroll
            for (int j = 0; j < KPL; ++j) {
                const int k = lane + 32 * j;
                float sdh = 0.f;
#pragma unroll
                for (int n = 0; n < kAcMaxN; ++n)
                    if (n < N) {
                        sdh = fmaf(dz[n], wt[n * K + k], sdh);
                        dwacc[n * K + k] = fmaf(hv[j], dz[n], dwacc[n * K + k]);
                    }
                rowbuf[k] = hv[j] > 0.f ? sdh : 0.f;                        // relu'(h) on the post-activation value
            }
            __syncwarp();
            head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
        }
        acc_loss = __fmul_rn(__fmul_rn(seg_sum, inv_l), w);
    }
    // padding rows [used, rows): zero outputs and dh
    for (int r = used + gw; r < p.rows; r += nwarps) {
        __syncwarp();
#pragma unroll
        for (int j = 0; j < KPL; ++j) rowbuf[lane + 32 * j] = 0.f;
        for (int n = lane; n < N; n += 32) {
            p.z[(size_t)r * N + n] = 0.f;
            if (p.dz) p.dz[(size_t)r * N + n] = 0.f;
            if (p.probs && n < A) p.probs[(size_t)r * A + n] = 0.f;
        }
        if (lane == 0) {
            if (p.targets) p.targets[r] = 0.f;
            if (p.advantages) p.advantages[r] = 0.f;
        }
        __syncwarp();
        head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
    }
    __syncwarp();
    // per-warp partials in dqn_head_reduce_kernel's layout: [dW (K * N) | db (N) | loss (1)]
    float* part = p.workspace + (size_t)gw * ((size_t)K * N + N + 1);
#pragma unroll
    for (int j = 0; j < KPL; ++j)
        for (int n = 0; n < N; ++n) part[((size_t)lane + 32 * j) * N + n] = dwacc[n * K + lane + 32 * j];
    if (lane == 0) {
        for (int n = 0; n < N; ++n) part[(size_t)K * N + n] = dbacc[n];
        part[(size_t)K * N + N] = acc_loss;
    }
}

// one thread per environment: p = softmax of the policy logits (row e of z: A columns from column `first`, row stride
// ld), then np.random.choice's inverse-cdf draw (cdf = cumsum(float64(p)), cdf /= cdf[-1], the number of entries <= u)
// or the first argmax.  The actor-critic layout is ld = 1 + A, first = 1; the policy gradient layout ld = A, first = 0.
__global__ void categorical_act_kernel(const float* __restrict__ z, int ld, int first, int64_t envs, int A,
                                       const double* __restrict__ u, int64_t* __restrict__ actions,
                                       float* __restrict__ probs) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= envs) return;
    float zz[kAcMaxN], pr[kNsMaxA];
#pragma unroll
    for (int n = 0; n < kAcMaxN; ++n) zz[n] = (n >= 1 && n <= A) ? z[e * ld + first + n - 1] : 0.f;   // zz[0] unread
    ac_softmax(zz, A, pr);
    int pick = 0;
    if (u) {
        double cdf[kNsMaxA], c = 0.0;
#pragma unroll
        for (int a = 0; a < kNsMaxA; ++a)
            if (a < A) {
                c = __dadd_rn(c, (double)pr[a]);
                cdf[a] = c;
            }
        const double x = u[e];
#pragma unroll
        for (int a = 0; a < kNsMaxA; ++a)
            if (a < A) pick += __ddiv_rn(cdf[a], c) <= x ? 1 : 0;
        pick = min(pick, A - 1);
    } else {
        float m = pr[0];
#pragma unroll
        for (int a = 1; a < kNsMaxA; ++a)
            if (a < A && (pr[a] > m || (pr[a] != pr[a] && m == m))) {     // np.argmax: the first maximum (or NaN)
                m = pr[a];
                pick = a;
            }
    }
    actions[e] = pick;
    if (probs) {
#pragma unroll
        for (int a = 0; a < kNsMaxA; ++a)
            if (a < A) probs[e * A + a] = pr[a];
    }
}

// ---- policy gradients (REINFORCE) ------------------------------------------------------------------------------------
// Targets: the return-based rescalers of policy_gradients_agent.py:47-67 over whole episodes (one segment = one
// episode), given the fp64 returns of cb200_nstep_returns; every fp64 operation is an explicit _rn intrinsic.

// numpy's pairwise summation (np.add.reduce on a contiguous float64 array, loops_utils.h pairwise_sum) of f(i) for
// i < n: below 8 terms a running sum; up to 128 terms eight accumulators over the blocks of 8, folded
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the tail; above, the halves split at n/2 rounded down to a
// multiple of 8.  The recursion runs on an explicit stack (at most 18 levels for n < 2^24).
template <class F>
__device__ double np_pairwise_sum(F f, int n) {
    constexpr int kDepth = 20;
    int lo[kDepth], len[kDepth], stage[kDepth];
    double left[kDepth];
    int sp = 0;
    lo[0] = 0;
    len[0] = n;
    stage[0] = 0;
    double r = 0.0;
    for (;;) {
        if (len[sp] > 128) {                                              // descend into the left half
            int n2 = len[sp] / 2;
            n2 -= n2 % 8;
            stage[sp] = 1;
            lo[sp + 1] = lo[sp];
            len[sp + 1] = n2;
            ++sp;
            continue;
        }
        const int b = lo[sp], m = len[sp];
        if (m < 8) {
            r = -0.0;
            for (int i = 0; i < m; ++i) r = __dadd_rn(r, f(b + i));
        } else {
            double acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = f(b + j);
            int i = 8;
            for (; i < m - (m % 8); i += 8)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = __dadd_rn(acc[j], f(b + i + j));
            r = __dadd_rn(__dadd_rn(__dadd_rn(acc[0], acc[1]), __dadd_rn(acc[2], acc[3])),
                          __dadd_rn(__dadd_rn(acc[4], acc[5]), __dadd_rn(acc[6], acc[7])));
            for (; i < m; ++i) r = __dadd_rn(r, f(b + i));
        }
        // return r to the parents: a left half starts the right half, a right half completes its parent
        for (;;) {
            if (sp == 0) return r;
            --sp;
            if (stage[sp] == 1) {
                int n2 = len[sp] / 2;
                n2 -= n2 % 8;
                left[sp] = r;
                stage[sp] = 2;
                lo[sp + 1] = lo[sp] + n2;
                len[sp + 1] = len[sp] - n2;
                ++sp;
                break;
            }
            r = __dadd_rn(left[sp], r);
        }
    }
}

// one block per segment slot: TOTAL_RETURN (R_0 on every row), FUTURE_RETURN (R) and NORMALIZED_BY_EPISODE
// ((R - mean) / std with np.mean / np.std of the episode's returns, 0 when std == 0; policy_optimization_agent.py:62-71)
__global__ void __launch_bounds__(256) pg_segment_targets_kernel(const double* __restrict__ ret,
                                                                 const int32_t* __restrict__ seg_off,
                                                                 const int32_t* __restrict__ seg_len, int64_t rows,
                                                                 int mode, float* __restrict__ targets,
                                                                 double* __restrict__ stats) {
    __shared__ double mean_std[2];
    const int s = blockIdx.x, L = seg_len[s], o = seg_off[s];
    if (!(L > 0 && o >= 0 && (int64_t)o + L <= rows)) return;
    const double* R = ret + o;
    if (mode == CB200_PG_NORMALIZED_BY_EPISODE && threadIdx.x == 0) {
        const double n = (double)L;
        const double mean = __ddiv_rn(np_pairwise_sum([&](int i) { return R[i]; }, L), n);
        const double var = __ddiv_rn(np_pairwise_sum([&](int i) {
            const double x = __dsub_rn(R[i], mean);
            return __dmul_rn(x, x);
        }, L), n);
        mean_std[0] = mean;
        mean_std[1] = __dsqrt_rn(var);
        if (stats) {
            stats[2 * s] = mean;
            stats[2 * s + 1] = mean_std[1];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        double t;
        if (mode == CB200_PG_TOTAL_RETURN) {
            t = R[0];
        } else if (mode == CB200_PG_FUTURE_RETURN) {
            t = R[i];
        } else {
            const double sd = mean_std[1];
            t = sd != 0.0 ? __ddiv_rn(__dsub_rn(R[i], mean_std[0]), sd) : 0.0;
        }
        targets[o + i] = (float)t;
    }
}

// NORMALIZED_BY_TIMESTEP: one thread per timestep i, the segments folded in slot order into the running mean table
// (update_episode_statistics, policy_optimization_agent.py:58-71: n_i += 1; m_i -= m_i / n_i; m_i += R_i / n_i), and
// each row's baseline is the table right after its own segment's fold (learn_from_batch: R_i - m_i)
__global__ void __launch_bounds__(256) pg_timestep_targets_kernel(const double* __restrict__ ret,
                                                                  const int32_t* __restrict__ seg_off,
                                                                  const int32_t* __restrict__ seg_len, int S,
                                                                  int64_t rows, double* __restrict__ mean,
                                                                  double* __restrict__ count, int table_len,
                                                                  float* __restrict__ targets,
                                                                  double* __restrict__ baselines) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const bool in_table = i < table_len;
    double m = in_table ? mean[i] : 0.0, c = in_table ? count[i] : 0.0;
    bool touched = false;
    for (int s = 0; s < S; ++s) {
        const int L = seg_len[s], o = seg_off[s];
        if (!(L > 0 && o >= 0 && (int64_t)o + L <= rows) || i >= L) continue;
        const int64_t r = o + i;
        if (!in_table) {                                                  // longer than the table: no baseline
            targets[r] = __int_as_float(0x7fc00000);
            if (baselines) baselines[r] = __longlong_as_double(0x7ff8000000000000ll);
            continue;
        }
        const double x = ret[r];
        c = __dadd_rn(c, 1.0);
        m = __dsub_rn(m, __ddiv_rn(m, c));
        m = __dadd_rn(m, __ddiv_rn(x, c));
        touched = true;
        targets[r] = (float)__dsub_rn(x, m);
        if (baselines) baselines[r] = m;
    }
    if (touched) {
        mean[i] = m;
        count[i] = c;
    }
}

// Head: heads/policy_head.py:54-150 with policy_gradients_agent.py's loss, one Dense(N) on a feature layer.
// Parallel over rows: a block owns kPgBlockRows consecutive rows, maps each to its segment slot in shared memory and
// gives each warp kPgWarpRows of them; per row the xor-butterfly dot products of nstep_q_head_kernel, the row's loss,
// dL/dZ (written out) and dL/dh.  pg_head_dw_kernel then forms dW = h^T dZ, db and the loss per 64-row chunk, and
// dqn_head_reduce_kernel sums the chunks in a fixed order.
constexpr int kPgWarps = 8;
constexpr int kPgWarpRows = 8;
constexpr int kPgBlockRows = kPgWarps * kPgWarpRows;
constexpr int kPgChunk = 64;
constexpr int kPgMaxD = 32;

struct PgParams {
    const float *h, *w, *b, *targets, *cont_actions, *range;
    const int64_t* actions;
    const int32_t *seg_off, *seg_len;
    int S, rows, K, N, continuous;
    float beta_entropy;
    float *z, *policy, *dz, *rowloss, *dh;
    uint16_t* dh_planes;
    int64_t dh_plane_stride;
};

// the bounded Gaussian mean of the continuous head: tanh(z) * max_abs_range (policy_head.py:118-126); th = tanh(z)
__device__ __forceinline__ float pg_mean(float z, float range, float& th) {
    th = tanhf(z);
    return th * range;
}

template <int KPL>
__global__ void __launch_bounds__(32 * kPgWarps) pg_head_rows_kernel(PgParams p) {
    // Wt [N][K] | row buffers [warps][K] | segment slot of each of the block's rows
    extern __shared__ __align__(16) float pg_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = p.N, K = p.K;
    float* wt = pg_smem;
    float* rowbuf = pg_smem + N * K + warp * K;
    int* slot = reinterpret_cast<int*>(pg_smem + N * K + kPgWarps * K);
    const int r0 = blockIdx.x * kPgBlockRows;
    seg_head_wt(p.w, N, K, wt);
    for (int j = threadIdx.x; j < kPgBlockRows; j += blockDim.x) slot[j] = -1;
    __syncthreads();
    for (int s = threadIdx.x; s < p.S; s += blockDim.x) {
        const int L = p.seg_len[s], o = p.seg_off[s];
        if (!(L > 0 && o >= 0 && (int64_t)o + L <= p.rows)) continue;
        const int lo = max(o, r0), hi = min(o + L, r0 + kPgBlockRows);
        for (int r = lo; r < hi; ++r) slot[r - r0] = s;
    }
    __syncthreads();
    const float log2pi = 1.8378770664093453f;
    for (int rr = 0; rr < kPgWarpRows; ++rr) {
        const int r = r0 + warp * kPgWarpRows + rr;
        if (r >= p.rows) break;
        const int s = slot[r - r0];
        float hv[KPL], z[kPgMaxD], dz[kPgMaxD], pol[kPgMaxD];
        float row_loss = 0.f;
#pragma unroll
        for (int n = 0; n < kPgMaxD; ++n) z[n] = dz[n] = pol[n] = 0.f;
#pragma unroll
        for (int j = 0; j < KPL; ++j) hv[j] = 0.f;
        if (s >= 0) {
            ns_dot<KPL, kPgMaxD>(p.h + (size_t)r * K, wt, p.b, N, K, lane, hv, z);
            const float c = 1.0f / (float)p.seg_len[s];                   // the episode's mean
            const float t = p.targets[r];
            if (!p.continuous) {
                // -mean(log pi(a) t) - beta mean(H) with Categorical(probs = softmax + eps)
                float zz[kAcMaxN], pr[kNsMaxA], ls[kNsMaxA], ent, logp, u_act, su;
                zz[0] = 0.f;
#pragma unroll
                for (int a = 0; a < kNsMaxA; ++a) zz[a + 1] = z[a];
                const int64_t act = p.actions[r];
                const bool in_range = act >= 0 && act < N;
                ac_policy_terms(zz, N, act, pr, ls, ent, logp, u_act, su);
                row_loss = c * ((in_range ? -logp * t : 0.f) - p.beta_entropy * ent);
                ac_policy_dz(pr, ls, N, act, u_act, su, in_range ? -c * t : 0.f, c * p.beta_entropy, 0, dz);
#pragma unroll
                for (int a = 0; a < kNsMaxA; ++a) pol[a] = pr[a];
            } else {
                // MultivariateNormalDiag(mean, 1): log pi(x) = -|x - mean|^2 / 2 - D log(2 pi) / 2; its entropy
                // D (1 + log(2 pi)) / 2 is a constant (the std is the all-ones policy_stdev variable)
                float sq = 0.f;
#pragma unroll
                for (int d = 0; d < kPgMaxD; ++d)
                    if (d < N) {
                        const float rg = __ldg(p.range + d);
                        float th;
                        const float mu = pg_mean(z[d], rg, th);
                        const float diff = p.cont_actions[(size_t)r * N + d] - mu;
                        sq = fmaf(diff, diff, sq);
                        pol[d] = mu;
                        dz[d] = ((-c * t) * diff) * rg * (1.0f - th * th);
                    }
                const float logp = -0.5f * sq - 0.5f * (float)N * log2pi;
                const float ent = 0.5f * (float)N * (1.0f + log2pi);
                row_loss = c * (-logp * t - p.beta_entropy * ent);
            }
        }
        if (lane == 0) {
#pragma unroll
            for (int n = 0; n < kPgMaxD; ++n)
                if (n < N) {
                    p.z[(size_t)r * N + n] = z[n];
                    p.dz[(size_t)r * N + n] = dz[n];
                    if (p.policy) p.policy[(size_t)r * N + n] = pol[n];
                }
            p.rowloss[r] = row_loss;
        }
        __syncwarp();                                                     // the previous row's readers are done
#pragma unroll
        for (int j = 0; j < KPL; ++j) {
            const int k = lane + 32 * j;
            float sdh = 0.f;
            if (s >= 0) {
#pragma unroll
                for (int n = 0; n < kPgMaxD; ++n)
                    if (n < N) sdh = fmaf(dz[n], wt[n * K + k], sdh);
            }
            rowbuf[k] = (s >= 0 && hv[j] > 0.f) ? sdh : 0.f;              // relu'(h) on the post-activation value
        }
        __syncwarp();
        head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
    }
}

// per 64-row chunk: dW[k, n] = sum_r h[r, k] dz[r, n], db[n] = sum_r dz[r, n] and the loss sum_r l_r, in row order,
// into the chunk's partials [dW (K * N) | db (N) | loss (1)] (dqn_head_reduce_kernel's layout).  blockIdx.y strides over
// the chunks (gridDim.y is at most 65535; 2^24 rows make 262144 chunks).
__global__ void __launch_bounds__(256) pg_head_dw_kernel(const float* __restrict__ h, const float* __restrict__ dz,
                                                         const float* __restrict__ rowloss, int rows, int K, int N,
                                                         float* __restrict__ part) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int KN = K * N, n_out = KN + N + 1;
    if (i >= n_out) return;
    const int chunks = (rows + kPgChunk - 1) / kPgChunk;
    for (int ch = blockIdx.y; ch < chunks; ch += gridDim.y) {
        const int r0 = ch * kPgChunk, r1 = min(rows, r0 + kPgChunk);
        float s = 0.f;
        if (i < KN) {
            const int n = i / K, k = i - n * K;                           // a warp reads 32 consecutive features
            for (int r = r0; r < r1; ++r) s = fmaf(__ldg(h + (size_t)r * K + k), __ldg(dz + (size_t)r * N + n), s);
            part[(size_t)ch * n_out + (size_t)k * N + n] = s;
            continue;
        }
        if (i < KN + N) {
            for (int r = r0; r < r1; ++r) s += __ldg(dz + (size_t)r * N + (i - KN));
        } else {
            for (int r = r0; r < r1; ++r) s += __ldg(rowloss + r);
        }
        part[(size_t)ch * n_out + i] = s;
    }
}

// acting of a continuous policy gradient head: thread per (environment, dimension); mean = tanh(z) * range (fp32),
// then numpy's normal(loc = mean, scale) = loc + scale * z in fp64 on host standard normals (scale [envs, D]: each
// environment's own noise), or the mean
__global__ void pg_gaussian_act_kernel(const float* __restrict__ z, int64_t envs, int D, const float* __restrict__ range,
                                       const double* __restrict__ normals, const double* __restrict__ scale,
                                       double* __restrict__ actions, float* __restrict__ means) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= envs * D) return;
    const int d = (int)(i % D);
    float th;
    const float mu = pg_mean(z[i], range[d], th);
    actions[i] = normals ? __dadd_rn((double)mu, __dmul_rn(scale[i], normals[i])) : (double)mu;
    if (means) means[i] = mu;
}

// ---- actor-critic (A3C) head, continuous actions ----------------------------------------------------------------------
// ONE Dense(1 + 2D) on the feature layer: column 0 V, columns 1..D the pre-tanh means, D+1..2D the pre-softplus stds
// (policy_head.py:102-152 with ContinuousEntropy).  Segments are whole episodes (up to 1000 rows and more), so the head
// is parallel over rows, not over segments:
//   ac_gauss_rows_kernel      Z = hW + b of every row and each segment's bootstrap V(s'_last); every row's slot = -1
//   ac_gauss_segments_kernel  one thread per segment: the fp64 recurrence of the discrete head (AcRecurrence) on Z[:, 0]
//                             -> targets, advantages and the rows' segment slot
//   ac_gauss_grad_kernel      per row the three loss terms, dL/dZ over the 1 + 2D columns and dL/dh; rows no segment
//                             covers get zero outputs
// then pg_head_dw_kernel and dqn_head_reduce_kernel sum dW, db and the loss per 64-row chunk and over the chunks in a
// fixed order.
constexpr int kAcgMaxD = 17;                                              // Humanoid: every mujoco_v2 level
constexpr int kAcgMaxN = 1 + 2 * kAcgMaxD;

struct AcGaussParams {
    const float *h, *h_boot, *w, *b, *actions, *range;
    const double* rewards;
    const uint8_t* game_overs;
    const int32_t *seg_off, *seg_len;
    int S, rows, mode, huber, K, D, N;
    double discount, gae_lambda;
    float beta_entropy, v_weight, p_weight;
    float *z, *dz, *targets, *advantages, *bootstrap, *means, *stds, *rowloss, *dh;
    int32_t* row_seg;
    uint16_t* dh_planes;
    int64_t dh_plane_stride;
};

// softplus(x) + eps with TF 1.x's softplus (the Eigen functor): x above -threshold, exp(x) below threshold,
// log(exp(x) + 1) between, threshold = log(FLT_EPSILON) + 2; eps = np.finfo(np.float32).eps
__device__ __forceinline__ float acg_std(float x) {
    const float eps = 1.1920928955078125e-07f;
    const float threshold = logf(eps) + 2.0f;
    const float e = expf(x);
    const float sp = x > -threshold ? x : (x < threshold ? e : logf(e + 1.0f));
    return sp + eps;
}

// rows [0, rows) and then the S bootstrap rows, kPgBlockRows per block, kPgWarpRows per warp
template <int KPL>
__global__ void __launch_bounds__(32 * kPgWarps) ac_gauss_rows_kernel(AcGaussParams p) {
    extern __shared__ __align__(16) float acg_smem[];                     // Wt [N][K]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = p.N, K = p.K;
    float* wt = acg_smem;
    seg_head_wt(p.w, N, K, wt);
    __syncthreads();
    for (int rr = 0; rr < kPgWarpRows; ++rr) {
        const int r = blockIdx.x * kPgBlockRows + warp * kPgWarpRows + rr;
        float hv[KPL], z[kAcgMaxN];
        if (r < p.rows) {
            ns_dot<KPL, kAcgMaxN>(p.h + (size_t)r * K, wt, p.b, N, K, lane, hv, z);
            if (lane == 0) {
#pragma unroll
                for (int n = 0; n < kAcgMaxN; ++n)
                    if (n < N) p.z[(size_t)r * N + n] = z[n];
                p.row_seg[r] = -1;
            }
        } else if (r < p.rows + p.S) {
            // V(s'_last) of the online network, 0 after a terminal state or for an unused slot
            const int s = r - p.rows, L = p.seg_len[s], o = p.seg_off[s];
            const bool valid = L > 0 && o >= 0 && (int64_t)o + L <= p.rows;
            float vnext = 0.f;
            if (valid && !p.game_overs[o + L - 1]) {
                ns_dot<KPL, kAcgMaxN>(p.h_boot + (size_t)s * K, wt, p.b, 1, K, lane, hv, z);
                vnext = z[0];
            }
            if (lane == 0) p.bootstrap[s] = vnext;
        }
    }
}

__global__ void __launch_bounds__(128) ac_gauss_segments_kernel(AcGaussParams p) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= p.S) return;
    const int L = p.seg_len[s], o = p.seg_off[s];
    if (!(L > 0 && o >= 0 && (int64_t)o + L <= p.rows)) return;
    // the discrete head's state and start (actor_critic_head_kernel)
    float vnext = p.bootstrap[s];
    const double gamma = p.discount, gl = __dmul_rn(p.discount, p.gae_lambda);
    const float gamma32 = (float)p.discount;
    double R = 0.0, za = 0.0, zr = 0.0;
    bool boot_pending = !p.game_overs[o + L - 1];
    if (p.mode != CB200_AC_A_VALUE) ac_lfilter((double)vnext, zr, gamma);
    for (int i = L - 1; i >= 0; --i) {
        const int r = o + i;
        double target, adv;
        ac_recurrence_step(p.mode, p.rewards[r], p.z[(size_t)r * p.N], gamma, gamma32, gl, vnext, R, boot_pending, za,
                           zr, target, adv);
        p.targets[r] = (float)target;
        p.advantages[r] = (float)adv;
        p.row_seg[r] = s;
    }
}

template <int KPL>
__global__ void __launch_bounds__(32 * kPgWarps) ac_gauss_grad_kernel(AcGaussParams p) {
    // Wt [N][K] | row buffers [warps][K]
    extern __shared__ __align__(16) float acg_smem[];
    __shared__ int nseg_shared;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = p.N, K = p.K, D = p.D;
    float* wt = acg_smem;
    float* rowbuf = acg_smem + N * K + warp * K;
    if (threadIdx.x == 0) nseg_shared = 0;
    seg_head_wt(p.w, N, K, wt);
    __syncthreads();
    int mine = 0;                                                         // non-empty segments (order-free integer sum)
    for (int s = threadIdx.x; s < p.S; s += blockDim.x) mine += p.seg_len[s] > 0 ? 1 : 0;
    if (mine) atomicAdd(&nseg_shared, mine);
    __syncthreads();
    const int nseg = nseg_shared;
    const float w = nseg > 0 ? 1.0f / (float)nseg : 0.f;                 // the mean over segments
    const float log2pi = 1.8378770664093453f;
    for (int rr = 0; rr < kPgWarpRows; ++rr) {
        const int r = blockIdx.x * kPgBlockRows + warp * kPgWarpRows + rr;
        if (r >= p.rows) break;
        const int s = p.row_seg[r];
        // dL/dZ of V, of the mean block and of the std block (indexed by d only, so they stay in registers)
        float hv[KPL], dz0 = 0.f, dzm[kAcgMaxD], dzs[kAcgMaxD];
        float row_loss = 0.f;
#pragma unroll
        for (int d = 0; d < kAcgMaxD; ++d) dzm[d] = dzs[d] = 0.f;
#pragma unroll
        for (int j = 0; j < KPL; ++j) hv[j] = s >= 0 ? __ldg(p.h + (size_t)r * K + lane + 32 * j) : 0.f;
        if (s >= 0) {
            const float c = w * (1.0f / (float)p.seg_len[s]);            // the row weight 1 / (segments L)
            const float* zr = p.z + (size_t)r * N;
            const float v = zr[0], t32 = p.targets[r], a32 = p.advantages[r];
            const float e = v - t32;
            float lv, gv;
            if (p.huber) {
                const float ae = fabsf(e);
                const float qq = fminf(ae, 1.0f);
                lv = 0.5f * qq * qq + (ae - qq);
                gv = fmaxf(-1.0f, fminf(e, 1.0f));
            } else {
                lv = e * e;
                gv = 2.0f * e;
            }
            dz0 = c * p.v_weight * gv;
            // MultivariateNormalDiag(mean, std): log pi = sum_d -((x - mean) / std)^2 / 2 - log std - log(2 pi) / 2,
            // H = sum_d (1 + log(2 pi)) / 2 + log std
            const float cp = -c * p.p_weight * a32, cb = c * p.beta_entropy;
            float logp = 0.f, ent = 0.f;
#pragma unroll
            for (int d = 0; d < kAcgMaxD; ++d)
                if (d < D) {
                    const float rg = __ldg(p.range + d);
                    float th;
                    const float mu = pg_mean(zr[1 + d], rg, th);
                    const float zs = zr[1 + D + d];
                    const float sd = acg_std(zs);
                    const float diff = p.actions[(size_t)r * D + d] - mu;
                    const float y = diff / sd, lsd = logf(sd);
                    logp += -0.5f * y * y - lsd - 0.5f * log2pi;
                    ent += 0.5f * (1.0f + log2pi) + lsd;
                    dzm[d] = cp * (diff / (sd * sd)) * rg * (1.0f - th * th);
                    const float sig = 1.0f / (expf(-zs) + 1.0f);          // TF's SoftplusGrad: dy / (exp(-x) + 1)
                    dzs[d] = (cp * (diff * diff / (sd * sd * sd) - 1.0f / sd) - cb / sd) * sig;
                    if (lane == 0) {
                        if (p.means) p.means[(size_t)r * D + d] = mu;
                        if (p.stds) p.stds[(size_t)r * D + d] = sd;
                    }
                }
            row_loss = c * (p.v_weight * lv - p.p_weight * logp * a32 - p.beta_entropy * ent);
        }
        if (lane == 0) {
            float* dzr = p.dz + (size_t)r * N;
            dzr[0] = dz0;
#pragma unroll
            for (int d = 0; d < kAcgMaxD; ++d)
                if (d < D) {
                    dzr[1 + d] = dzm[d];
                    dzr[1 + D + d] = dzs[d];
                }
            if (s < 0) {
                for (int n = 0; n < N; ++n) p.z[(size_t)r * N + n] = 0.f;
                p.targets[r] = 0.f;
                p.advantages[r] = 0.f;
                for (int d = 0; d < D; ++d) {
                    if (p.means) p.means[(size_t)r * D + d] = 0.f;
                    if (p.stds) p.stds[(size_t)r * D + d] = 0.f;
                }
            }
            p.rowloss[r] = row_loss;
        }
        __syncwarp();                                                     // the previous row's readers are done
#pragma unroll
        for (int j = 0; j < KPL; ++j) {
            const int k = lane + 32 * j;
            float sdh = dz0 * wt[k];                                      // the columns in order
#pragma unroll
            for (int d = 0; d < kAcgMaxD; ++d)
                if (d < D) sdh = fmaf(dzm[d], wt[(1 + d) * K + k], sdh);
#pragma unroll
            for (int d = 0; d < kAcgMaxD; ++d)
                if (d < D) sdh = fmaf(dzs[d], wt[(1 + D + d) * K + k], sdh);
            rowbuf[k] = hv[j] > 0.f ? sdh : 0.f;                          // relu'(h) on the post-activation value
        }
        __syncwarp();
        head_store_dz<KPL>(rowbuf, lane, r, K, p.dh, p.dh_planes, p.dh_plane_stride);
    }
}

// acting of the continuous actor-critic head: thread per (environment, dimension) on z [envs, 1 + 2D]: the head's
// mean tanh(z) * range and std softplus(z) + eps (fp32), then numpy's normal(mean, std) = mean + std * n in fp64 on
// host standard normals, or the mean
__global__ void ac_gauss_act_kernel(const float* __restrict__ z, int64_t envs, int D, const float* __restrict__ range,
                                    const double* __restrict__ normals, double* __restrict__ actions,
                                    float* __restrict__ means, float* __restrict__ stds) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= envs * D) return;
    const int64_t e = i / D;
    const int d = (int)(i - e * D);
    const float* ze = z + e * (1 + 2 * D);
    float th;
    const float mu = pg_mean(ze[1 + d], range[d], th);
    const float sd = acg_std(ze[1 + D + d]);
    actions[i] = normals ? __dadd_rn((double)mu, __dmul_rn((double)sd, normals[i])) : (double)mu;
    if (means) means[i] = mu;
    if (stds) stds[i] = sd;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_dqn_td_targets(const float* q_next, const float* q_select, const float* q_online, const int64_t* actions,
                         const double* rewards, const uint8_t* game_overs, double discount, int64_t batch,
                         int64_t n_actions, float* targets_out, double* td_err_out, void* stream) {
    CB200_CHECK_ARG(q_next && q_select && q_online && actions && rewards && game_overs && targets_out && td_err_out,
                    "null pointer");
    CB200_CHECK_ARG(batch > 0 && n_actions > 0, "bad shape");
    CB200_LAUNCH(dqn_td_targets_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), q_next, q_select,
                 q_online, actions, rewards, game_overs, discount, batch, n_actions, targets_out, td_err_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_regression_head_loss_grad(const float* out, const float* target, const float* weights, int64_t batch,
                                    int64_t width, int huber, float loss_weight, float* d_out, float* loss_out,
                                    void* stream) {
    CB200_CHECK_ARG(out && target && d_out && batch > 0 && width > 0, "bad arguments");
    int threads = 32;
    while (threads < batch && threads < 1024) threads *= 2;
    CB200_LAUNCH(regression_head_kernel, 1, threads, 0, as_stream(stream), out, target, weights, batch, width, huber,
                 loss_weight, d_out, loss_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_dqn_head_fused(const cb200_dqn_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->h_next && d->h_online && d->w_target && d->b_target && d->w_online && d->b_online && d->actions &&
                        d->rewards && d->game_overs && d->q_online && d->targets && d->td_err && d->dq && d->dw && d->db &&
                        d->workspace,
                    "null pointer");
    CB200_CHECK_ARG(d->batch > 0 && d->n_actions > 0 && d->n_actions <= kHeadMaxA, "1 <= n_actions <= 8");
    CB200_CHECK_ARG(d->features == 256 || d->features == 512, "features must be 256 or 512");
    CB200_CHECK_ARG(!d->dh_planes || (d->dh_plane_stride % 8 == 0 && d->batch % 8 == 0), "planes: batch % 8, stride % 8");
    const int rule = d->target_rule;
    CB200_CHECK_ARG(rule >= CB200_TARGET_DQN && rule <= CB200_TARGET_PAL_PERSISTENT, "unknown target rule");
    CB200_CHECK_ARG(rule == CB200_TARGET_DQN || (d->h_select && d->mc_returns),
                    "MMC / PAL targets need h_select and mc_returns");
    CB200_CHECK_ARG(rule < CB200_TARGET_PAL || d->h_target_s, "PAL targets need h_target_s");
    HeadParams p;
    p.h_next = d->h_next; p.h_online = d->h_online; p.h_select = d->h_select;
    p.w_target = d->w_target; p.b_target = d->b_target; p.w_online = d->w_online; p.b_online = d->b_online;
    p.actions = d->actions; p.rewards = d->rewards; p.game_overs = d->game_overs; p.weights = d->weights;
    p.discount = d->discount; p.huber = d->huber; p.B = (int)d->batch; p.K = d->features; p.A = d->n_actions;
    p.q_online = d->q_online; p.q_next = d->q_next; p.targets = d->targets; p.td_err = d->td_err;
    p.dq = d->dq; p.loss = d->loss; p.dh = d->dh;
    p.dh_planes = static_cast<uint16_t*>(d->dh_planes); p.dh_plane_stride = d->dh_plane_stride;
    p.dw = d->dw; p.db = d->db; p.workspace = d->workspace;
    p.h_target_s = d->h_target_s; p.mc_returns = d->mc_returns;
    p.pal_alpha = d->pal_alpha; p.mc_mixing_rate = d->mc_mixing_rate;
    p.q_select = d->q_select; p.q_target_s = d->q_target_s;
    const int warps = (p.B + kHeadRows - 1) / kHeadRows;
    const unsigned grid = (unsigned)((warps + kHeadWarps - 1) / kHeadWarps);
    const int nparts = (int)grid * kHeadWarps;                 // idle warps of the last block write zero partials
    cudaStream_t st = as_stream(stream);
    const size_t smem = (size_t)(2 * p.A * p.K + kHeadWarps * p.K) * sizeof(float);      // <= 48 KB (A <= 8, K <= 512)
#define CB200_HEAD_LAUNCH(R)                                                                \
    if (p.K == 512) {                                                                       \
        CB200_LAUNCH((dqn_head_fused_kernel<16, R>), grid, 32 * kHeadWarps, smem, st, p);   \
    } else {                                                                                \
        CB200_LAUNCH((dqn_head_fused_kernel<8, R>), grid, 32 * kHeadWarps, smem, st, p);    \
    }
    switch (rule) {
        case CB200_TARGET_MMC: CB200_HEAD_LAUNCH(CB200_TARGET_MMC); break;
        case CB200_TARGET_PAL: CB200_HEAD_LAUNCH(CB200_TARGET_PAL); break;
        case CB200_TARGET_PAL_PERSISTENT: CB200_HEAD_LAUNCH(CB200_TARGET_PAL_PERSISTENT); break;
        default: CB200_HEAD_LAUNCH(CB200_TARGET_DQN); break;
    }
#undef CB200_HEAD_LAUNCH
    const int n_out = p.K * p.A + p.A + 1;
    CB200_LAUNCH(dqn_head_reduce_kernel, (unsigned)((n_out + 31) / 32), 256, 0, st, p.workspace, nparts, n_out,
                 p.K * p.A, p.A, 1.0f / (float)p.B, p.dw, p.db, p.loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ensemble_head_fused(const cb200_ensemble_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->h_next && d->h_online && d->h_select && d->w_target && d->b_target && d->w_online &&
                        d->b_online && d->actions && d->rewards && d->game_overs && d->masks && d->q_online &&
                        d->targets && d->dq && d->losses && d->dw && d->db && d->workspace,
                    "null pointer");
    CB200_CHECK_ARG(d->batch > 0 && d->batch <= (1 << 30), "bad batch");
    CB200_CHECK_ARG(d->n_actions > 0 && d->n_actions <= kHeadMaxA, "1 <= n_actions <= 8");
    CB200_CHECK_ARG(d->heads >= 1 && d->heads <= 64, "1 <= heads <= 64");
    CB200_CHECK_ARG(d->features == 256 || d->features == 512, "features must be 256 or 512");
    CB200_CHECK_ARG(!d->dh_planes || (d->dh_plane_stride % 8 == 0 && d->batch % 8 == 0), "planes: batch % 8, stride % 8");
    EnsembleParams p;
    p.h_next = d->h_next; p.h_online = d->h_online; p.h_select = d->h_select;
    p.w_target = d->w_target; p.b_target = d->b_target; p.w_online = d->w_online; p.b_online = d->b_online;
    p.actions = d->actions; p.rewards = d->rewards; p.game_overs = d->game_overs; p.masks = d->masks;
    p.discount = d->discount; p.huber = d->huber; p.B = (int)d->batch; p.K = d->features; p.H = d->heads;
    p.A = d->n_actions; p.rescale = d->grad_rescale;
    p.q_online = d->q_online; p.q_next = d->q_next; p.q_select = d->q_select; p.targets = d->targets; p.dq = d->dq;
    p.dh = d->dh; p.dh_planes = static_cast<uint16_t*>(d->dh_planes); p.dh_plane_stride = d->dh_plane_stride;
    p.workspace = d->workspace;
    const int warps = (p.B + kHeadRows - 1) / kHeadRows;
    const unsigned grid = (unsigned)((warps + kHeadWarps - 1) / kHeadWarps);
    const int nparts = (int)grid * kHeadWarps;
    cudaStream_t st = as_stream(stream);
    // <= 32 KB of staged head kernels + 32 KB of dz rows: above the 48 KB default, opted into once per instantiation
    // and device (the attribute is per device: one replay shard per GPU launches it on each)
    const size_t smem = (size_t)(2 * p.A * p.K + kHeadWarps * kHeadRows * p.K) * sizeof(float);
    static bool attr_set[kMaxDevices][2] = {};
    int dev = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    CB200_CHECK_ARG(dev < kMaxDevices, "device ordinal out of range");
    const int ti = p.K == 512 ? 1 : 0;
    if (!attr_set[dev][ti]) {
        if (ti)
            CB200_CUDA(cudaFuncSetAttribute(ensemble_head_fused_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            64 * 1024));
        else
            CB200_CUDA(cudaFuncSetAttribute(ensemble_head_fused_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            64 * 1024));
        attr_set[dev][ti] = true;
    }
    if (p.K == 512) {
        CB200_LAUNCH(ensemble_head_fused_kernel<16>, grid, 32 * kHeadWarps, smem, st, p);
    } else {
        CB200_LAUNCH(ensemble_head_fused_kernel<8>, grid, 32 * kHeadWarps, smem, st, p);
    }
    const int n_out = p.H * (p.K * p.A + p.A + 1);
    CB200_LAUNCH(ensemble_head_reduce_kernel, (unsigned)((n_out + 31) / 32), 256, 0, st, p.workspace, nparts, n_out,
                 p.K * p.A, p.A, p.H * p.A, 1.0f / (float)p.B, d->dw, d->db, d->losses);
    if (d->loss) CB200_LAUNCH(ensemble_loss_total_kernel, 1, 1, 0, st, d->losses, p.H, d->loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_nstep_q_head(const cb200_nstep_q_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->horizon >= CB200_NSTEP_NONE && d->horizon <= CB200_NSTEP_ONESTEP, "unknown horizon");
    CB200_CHECK_ARG(d->h_online && (d->horizon == CB200_NSTEP_NONE || d->h_boot) && d->w_target && d->b_target &&
                        d->w_online && d->b_online && d->actions && d->rewards && d->game_overs && d->seg_offsets &&
                        d->seg_lengths && d->q_online && d->dq && d->dw && d->db && d->workspace,
                    "null pointer");
    CB200_CHECK_ARG(d->segments >= 1 && d->segments <= (1 << 20), "1 <= segments <= 2^20");
    CB200_CHECK_ARG(d->rows >= 1 && d->rows <= (1 << 24), "1 <= rows <= 2^24");
    CB200_CHECK_ARG(d->n_actions >= 1 && d->n_actions <= kNsMaxA, "1 <= n_actions <= 18");
    CB200_CHECK_ARG(d->features == 256 || d->features == 512, "features must be 256 or 512");
    CB200_CHECK_ARG(!d->dh_planes || (d->dh_plane_stride % 8 == 0 && d->rows % 8 == 0), "planes: rows % 8, stride % 8");
    NstepParams p;
    p.h_online = d->h_online; p.h_boot = d->h_boot;
    p.w_target = d->w_target; p.b_target = d->b_target; p.w_online = d->w_online; p.b_online = d->b_online;
    p.actions = d->actions; p.rewards = d->rewards; p.game_overs = d->game_overs;
    p.seg_off = d->seg_offsets; p.seg_len = d->seg_lengths;
    p.S = d->segments; p.rows = (int)d->rows; p.horizon = d->horizon; p.huber = d->huber;
    p.K = d->features; p.A = d->n_actions; p.discount = d->discount;
    p.q_online = d->q_online; p.dq = d->dq; p.targets = d->targets; p.bootstrap = d->bootstrap; p.dh = d->dh;
    p.dh_planes = static_cast<uint16_t*>(d->dh_planes); p.dh_plane_stride = d->dh_plane_stride;
    p.workspace = d->workspace;
    const unsigned grid = (unsigned)((p.S + kNsWarps - 1) / kNsWarps);
    const int nparts = (int)grid * kNsWarps;                   // idle warps write zero partials
    cudaStream_t st = as_stream(stream);
    // up to 225 KB at K = 512, A = 18 (two staged kernels and four warps' dW slices): opted into once per instantiation
    // and device, at the size of the largest shape
    auto smem_of = [](int A, int K) { return (size_t)(2 * A * K + kNsWarps * (K + A * K + 32)) * sizeof(float); };
    const size_t smem = smem_of(p.A, p.K);
    static bool attr_set[kMaxDevices][2] = {};
    int dev = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    CB200_CHECK_ARG(dev < kMaxDevices, "device ordinal out of range");
    const int ti = p.K == 512 ? 1 : 0;
    if (!attr_set[dev][ti]) {
        if (ti)
            CB200_CUDA(cudaFuncSetAttribute(nstep_q_head_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_of(kNsMaxA, 512)));
        else
            CB200_CUDA(cudaFuncSetAttribute(nstep_q_head_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_of(kNsMaxA, 256)));
        attr_set[dev][ti] = true;
    }
    if (p.K == 512) {
        CB200_LAUNCH(nstep_q_head_kernel<16>, grid, 32 * kNsWarps, smem, st, p);
    } else {
        CB200_LAUNCH(nstep_q_head_kernel<8>, grid, 32 * kNsWarps, smem, st, p);
    }
    const int n_out = p.K * p.A + p.A + 1;
    CB200_LAUNCH(dqn_head_reduce_kernel, (unsigned)((n_out + 31) / 32), 256, 0, st, p.workspace, nparts, n_out,
                 p.K * p.A, p.A, 1.0f, d->dw, d->db, d->loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ensemble_action_values(const float* q, int64_t envs, int32_t heads, int32_t n_actions, int32_t mode,
                                 const int32_t* head, float lamb, float* out, void* stream) {
    CB200_CHECK_ARG(q && out && envs > 0 && envs <= (1 << 24) && heads >= 1 && n_actions >= 1, "bad arguments");
    CB200_CHECK_ARG(mode >= CB200_ENSEMBLE_SELECT && mode <= CB200_ENSEMBLE_VOTE, "unknown mode");
    CB200_CHECK_ARG(mode != CB200_ENSEMBLE_SELECT || head, "select mode needs the per-environment head indices");
    CB200_LAUNCH(ensemble_action_values_kernel, (unsigned)((envs + 127) / 128), 128, 0, as_stream(stream), q, (int)envs,
                 heads, n_actions, mode, head, lamb, out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_dueling_combine_fwd(const float* v, const float* adv, int64_t batch, int64_t n_actions, float* q,
                              void* stream) {
    CB200_CHECK_ARG(v && adv && q && batch > 0 && n_actions > 0, "bad arguments");
    CB200_LAUNCH(dueling_fwd_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), v, adv, batch,
                 n_actions, q);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_dueling_combine_bwd(const float* dq, int64_t batch, int64_t n_actions, float* d_v, float* d_adv,
                              void* stream) {
    CB200_CHECK_ARG(dq && d_v && d_adv && batch > 0 && n_actions > 0, "bad arguments");
    CB200_LAUNCH(dueling_bwd_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), dq, batch, n_actions,
                 d_v, d_adv);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_sumsq(const float* x, int64_t n, float* out, float* workspace, void* stream) {
    CB200_CHECK_ARG(x && out && workspace && n > 0, "bad arguments");
    int blocks = (int)((n + 4095) / 4096);
    if (blocks > kRedBlocks) blocks = kRedBlocks;
    CB200_LAUNCH(sumsq_stage1, blocks, 256, 0, as_stream(stream), x, n, workspace);
    CB200_LAUNCH(sumsq_stage2, 1, 1024, 0, as_stream(stream), workspace, blocks, out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_clip_by_global_norm(float* g, int64_t n, const float* sumsq, float clip, void* stream) {
    CB200_CHECK_ARG(g && sumsq && n > 0 && clip > 0, "bad arguments");
    CB200_LAUNCH(clip_kernel, flat_grid(n), 256, 0, as_stream(stream), g, n, sumsq, clip);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_clip_by_value(float* g, int64_t n, float clip, void* stream) {
    CB200_CHECK_ARG(g && n > 0 && clip > 0, "bad arguments");
    CB200_LAUNCH(clip_by_value_kernel, flat_grid(n), 256, 0, as_stream(stream), g, n, clip);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_scale(float* g, int64_t n, float s, void* stream) {
    CB200_CHECK_ARG(g && n > 0, "bad arguments");
    CB200_LAUNCH(scale_kernel, flat_grid(n), 256, 0, as_stream(stream), g, n, s);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_adam_tf(float* theta, float* m, float* v, const float* g, int64_t n, float lr, float beta1, float beta2,
                  float epsilon, float beta1_power, float beta2_power, void* stream) {
    CB200_CHECK_ARG(theta && m && v && g && n > 0, "bad arguments");
    const float alpha = lr * sqrtf(1.0f - beta2_power) / (1.0f - beta1_power);
    CB200_LAUNCH(adam_tf_kernel, flat_grid(n), 256, 0, as_stream(stream), theta, m, v, g, n, alpha, 1.0f - beta1,
                 1.0f - beta2, epsilon);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_adam_tf_dev(float* theta, float* m, float* v, const float* g, int64_t n, float lr, float beta1, float beta2,
                      float epsilon, float* state, void* stream) {
    CB200_CHECK_ARG(theta && m && v && g && state && n > 0, "bad arguments");
    CB200_LAUNCH(adam_tf_dev_kernel, flat_grid(n), 256, 0, as_stream(stream), theta, m, v, g, n, lr, 1.0f - beta1,
                 1.0f - beta2, epsilon, state);
    CB200_LAUNCH(adam_state_advance_kernel, 1, 1, 0, as_stream(stream), state, beta1, beta2);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_add_i64(int64_t* x, int64_t delta, void* stream) {
    CB200_CHECK_ARG(x != nullptr, "null pointer");
    CB200_LAUNCH(add_i64_kernel, 1, 1, 0, as_stream(stream), x, delta);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_polyak(float* target, const float* online, int64_t n, double rate, void* stream) {
    CB200_CHECK_ARG(target && online && n > 0, "bad arguments");
    CB200_LAUNCH(polyak_kernel, flat_grid(n), 256, 0, as_stream(stream), target, online, n, (float)rate,
                 (float)(1.0 - rate));
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_actor_critic_head(const cb200_actor_critic_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->mode >= CB200_AC_A_VALUE && d->mode <= CB200_AC_GAE_VALUE, "unknown mode");
    CB200_CHECK_ARG(d->h && d->h_boot && d->w && d->b && d->actions && d->rewards && d->game_overs && d->seg_offsets &&
                        d->seg_lengths && d->z && d->dw && d->db && d->workspace,
                    "null pointer");
    CB200_CHECK_ARG(d->segments >= 1 && d->segments <= (1 << 20), "1 <= segments <= 2^20");
    CB200_CHECK_ARG(d->rows >= 1 && d->rows <= (1 << 24), "1 <= rows <= 2^24");
    CB200_CHECK_ARG(d->n_actions >= 1 && d->n_actions <= kNsMaxA, "1 <= n_actions <= 18");
    CB200_CHECK_ARG(d->features == 256 || d->features == 512, "features must be 256 or 512");
    CB200_CHECK_ARG(!d->dh_planes || (d->dh_plane_stride % 8 == 0 && d->rows % 8 == 0), "planes: rows % 8, stride % 8");
    AcParams p;
    p.h = d->h; p.h_boot = d->h_boot; p.w = d->w; p.b = d->b;
    p.actions = d->actions; p.rewards = d->rewards; p.game_overs = d->game_overs;
    p.seg_off = d->seg_offsets; p.seg_len = d->seg_lengths;
    p.S = d->segments; p.rows = (int)d->rows; p.mode = d->mode; p.huber = d->huber;
    p.K = d->features; p.A = d->n_actions; p.discount = d->discount; p.gae_lambda = d->gae_lambda;
    p.beta_entropy = d->beta_entropy; p.v_weight = d->v_weight; p.p_weight = d->p_weight;
    p.z = d->z; p.dz = d->dz; p.probs = d->probs; p.targets = d->targets; p.advantages = d->advantages;
    p.bootstrap = d->bootstrap; p.dh = d->dh;
    p.dh_planes = static_cast<uint16_t*>(d->dh_planes); p.dh_plane_stride = d->dh_plane_stride;
    p.workspace = d->workspace;
    const unsigned grid = (unsigned)((p.S + kNsWarps - 1) / kNsWarps);
    const int nparts = (int)grid * kNsWarps;                   // idle warps write zero partials
    const int N = p.A + 1;
    cudaStream_t st = as_stream(stream);
    // up to 203 KB at K = 512, 1 + A = 19 (the staged kernel and four warps' dW slices): opted into once per
    // instantiation and device, at the size of the largest shape
    auto smem_of = [](int N, int K) { return (size_t)(N * K + kNsWarps * (K + N * K + 32)) * sizeof(float); };
    const size_t smem = smem_of(N, p.K);
    static bool attr_set[kMaxDevices][2] = {};
    int dev = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    CB200_CHECK_ARG(dev < kMaxDevices, "device ordinal out of range");
    const int ti = p.K == 512 ? 1 : 0;
    if (!attr_set[dev][ti]) {
        if (ti)
            CB200_CUDA(cudaFuncSetAttribute(actor_critic_head_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_of(kAcMaxN, 512)));
        else
            CB200_CUDA(cudaFuncSetAttribute(actor_critic_head_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_of(kAcMaxN, 256)));
        attr_set[dev][ti] = true;
    }
    if (p.K == 512) {
        CB200_LAUNCH(actor_critic_head_kernel<16>, grid, 32 * kNsWarps, smem, st, p);
    } else {
        CB200_LAUNCH(actor_critic_head_kernel<8>, grid, 32 * kNsWarps, smem, st, p);
    }
    const int n_out = p.K * N + N + 1;
    CB200_LAUNCH(dqn_head_reduce_kernel, (unsigned)((n_out + 31) / 32), 256, 0, st, p.workspace, nparts, n_out,
                 p.K * N, N, 1.0f, d->dw, d->db, d->loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_categorical_act(const float* z, int64_t envs, int32_t n_actions, const double* uniforms, int64_t* actions,
                          float* probs, void* stream) {
    CB200_CHECK_ARG(z && actions, "null pointer");
    CB200_CHECK_ARG(envs >= 1 && envs <= (1 << 24), "1 <= envs <= 2^24");
    CB200_CHECK_ARG(n_actions >= 1 && n_actions <= kNsMaxA, "1 <= n_actions <= 18");
    CB200_LAUNCH(categorical_act_kernel, (unsigned)((envs + 127) / 128), 128, 0, as_stream(stream), z, n_actions + 1, 1,
                 envs, n_actions, uniforms, actions, probs);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_pg_targets(const double* returns, const int32_t* seg_offsets, const int32_t* seg_lengths, int32_t segments,
                     int64_t rows, int32_t rescaler, double* table_mean, double* table_count, int32_t table_len,
                     float* targets, double* baselines, double* episode_stats, void* stream) {
    CB200_CHECK_ARG(returns && seg_offsets && seg_lengths && targets, "null pointer");
    CB200_CHECK_ARG(segments >= 1 && segments <= (1 << 20), "1 <= segments <= 2^20");
    CB200_CHECK_ARG(rows >= 1 && rows <= (1 << 24), "1 <= rows <= 2^24");
    CB200_CHECK_ARG(rescaler >= CB200_PG_TOTAL_RETURN && rescaler <= CB200_PG_NORMALIZED_BY_TIMESTEP,
                    "unknown rescaler");
    cudaStream_t st = as_stream(stream);
    if (rescaler == CB200_PG_NORMALIZED_BY_TIMESTEP) {
        CB200_CHECK_ARG(table_mean && table_count && table_len >= 1, "the timestep rescaler needs its table");
        CB200_LAUNCH(pg_timestep_targets_kernel, (unsigned)((rows + 255) / 256), 256, 0, st, returns, seg_offsets,
                     seg_lengths, segments, rows, table_mean, table_count, table_len, targets, baselines);
    } else {
        CB200_LAUNCH(pg_segment_targets_kernel, (unsigned)segments, 256, 0, st, returns, seg_offsets, seg_lengths, rows,
                     rescaler, targets, episode_stats);
    }
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_policy_gradient_head(const cb200_policy_gradient_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->h && d->w && d->b && d->targets && d->seg_offsets && d->seg_lengths && d->z && d->dw && d->db &&
                        d->workspace && (d->continuous ? (d->cont_actions && d->max_abs_range) : d->actions != nullptr),
                    "null pointer");
    CB200_CHECK_ARG(d->segments >= 1 && d->segments <= (1 << 20), "1 <= segments <= 2^20");
    CB200_CHECK_ARG(d->rows >= 1 && d->rows <= (1 << 24), "1 <= rows <= 2^24");
    CB200_CHECK_ARG(d->continuous ? (d->n_outputs >= 1 && d->n_outputs <= kPgMaxD)
                                  : (d->n_outputs >= 1 && d->n_outputs <= kNsMaxA),
                    "1 <= n_outputs <= 18 (discrete) / 32 (continuous)");
    CB200_CHECK_ARG(d->features == 256 || d->features == 512, "features must be 256 or 512");
    CB200_CHECK_ARG(!d->dh_planes || (d->dh_plane_stride % 8 == 0 && d->rows % 8 == 0), "planes: rows % 8, stride % 8");
    const int rows = (int)d->rows, K = d->features, N = d->n_outputs;
    PgParams p;
    p.h = d->h; p.w = d->w; p.b = d->b; p.targets = d->targets; p.cont_actions = d->cont_actions;
    p.range = d->max_abs_range; p.actions = d->actions;
    p.seg_off = d->seg_offsets; p.seg_len = d->seg_lengths;
    p.S = d->segments; p.rows = rows; p.K = K; p.N = N; p.continuous = d->continuous ? 1 : 0;
    p.beta_entropy = d->beta_entropy;
    p.z = d->z; p.policy = d->policy; p.dh = d->dh;
    p.dh_planes = static_cast<uint16_t*>(d->dh_planes); p.dh_plane_stride = d->dh_plane_stride;
    // workspace: dL/dZ [rows, N] (unless given) | per-row losses [rows] | chunk partials
    float* ws = d->workspace;
    p.dz = d->dz ? d->dz : ws;
    p.rowloss = ws + (size_t)rows * N;
    float* part = p.rowloss + rows;
    cudaStream_t st = as_stream(stream);
    // up to 80 KB at K = 512, N = 32 (the staged kernel and eight row buffers): opted into once per instantiation and
    // device, at the size of the largest shape
    auto smem_of = [](int N, int K) {
        return (size_t)(N * K + kPgWarps * K) * sizeof(float) + kPgBlockRows * sizeof(int);
    };
    static bool attr_set[kMaxDevices][2] = {};
    int dev = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    CB200_CHECK_ARG(dev < kMaxDevices, "device ordinal out of range");
    const int ti = K == 512 ? 1 : 0;
    if (!attr_set[dev][ti]) {
        if (ti)
            CB200_CUDA(cudaFuncSetAttribute(pg_head_rows_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_of(kPgMaxD, 512)));
        else
            CB200_CUDA(cudaFuncSetAttribute(pg_head_rows_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_of(kPgMaxD, 256)));
        attr_set[dev][ti] = true;
    }
    const unsigned grid = (unsigned)((rows + kPgBlockRows - 1) / kPgBlockRows);
    if (K == 512) {
        CB200_LAUNCH(pg_head_rows_kernel<16>, grid, 32 * kPgWarps, smem_of(N, K), st, p);
    } else {
        CB200_LAUNCH(pg_head_rows_kernel<8>, grid, 32 * kPgWarps, smem_of(N, K), st, p);
    }
    const int n_out = K * N + N + 1, chunks = (rows + kPgChunk - 1) / kPgChunk;
    const dim3 dw_grid((unsigned)((n_out + 255) / 256), (unsigned)min(chunks, 65535));
    CB200_LAUNCH(pg_head_dw_kernel, dw_grid, 256, 0, st, d->h, p.dz, p.rowloss, rows, K, N, part);
    CB200_LAUNCH(dqn_head_reduce_kernel, (unsigned)((n_out + 31) / 32), 256, 0, st, part, chunks, n_out, K * N, N, 1.0f,
                 d->dw, d->db, d->loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_policy_act(const float* z, int64_t envs, int32_t n_outputs, int32_t continuous, const float* max_abs_range,
                     const double* draws, const double* scale, int64_t* actions, float* probs, double* cont_actions,
                     float* means, void* stream) {
    CB200_CHECK_ARG(z != nullptr, "null pointer");
    CB200_CHECK_ARG(envs >= 1 && envs <= (1 << 24), "1 <= envs <= 2^24");
    cudaStream_t st = as_stream(stream);
    if (!continuous) {
        CB200_CHECK_ARG(actions != nullptr, "null pointer");
        CB200_CHECK_ARG(n_outputs >= 1 && n_outputs <= kNsMaxA, "1 <= n_outputs <= 18");
        CB200_LAUNCH(categorical_act_kernel, (unsigned)((envs + 127) / 128), 128, 0, st, z, n_outputs, 0, envs,
                     n_outputs, draws, actions, probs);
    } else {
        CB200_CHECK_ARG(max_abs_range && cont_actions && (!draws || scale), "null pointer");
        CB200_CHECK_ARG(n_outputs >= 1 && n_outputs <= kPgMaxD, "1 <= n_outputs <= 32");
        const int64_t n = envs * n_outputs;
        CB200_LAUNCH(pg_gaussian_act_kernel, (unsigned)((n + 127) / 128), 128, 0, st, z, envs, n_outputs, max_abs_range,
                     draws, scale, cont_actions, means);
    }
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_actor_critic_gaussian_head(const cb200_actor_critic_gaussian_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->mode >= CB200_AC_A_VALUE && d->mode <= CB200_AC_GAE_VALUE, "unknown mode");
    CB200_CHECK_ARG(d->h && d->h_boot && d->w && d->b && d->actions && d->max_abs_range && d->rewards &&
                        d->game_overs && d->seg_offsets && d->seg_lengths && d->z && d->dw && d->db && d->workspace,
                    "null pointer");
    CB200_CHECK_ARG(d->segments >= 1 && d->segments <= (1 << 20), "1 <= segments <= 2^20");
    CB200_CHECK_ARG(d->rows >= 1 && d->rows <= (1 << 24), "1 <= rows <= 2^24");
    CB200_CHECK_ARG(d->action_dim >= 1 && d->action_dim <= kAcgMaxD, "1 <= action_dim <= 17");
    CB200_CHECK_ARG(d->features == 256 || d->features == 512, "features must be 256 or 512");
    CB200_CHECK_ARG(!d->dh_planes || (d->dh_plane_stride % 8 == 0 && d->rows % 8 == 0), "planes: rows % 8, stride % 8");
    const int rows = (int)d->rows, K = d->features, D = d->action_dim, N = 1 + 2 * D, S = d->segments;
    AcGaussParams p;
    p.h = d->h; p.h_boot = d->h_boot; p.w = d->w; p.b = d->b; p.actions = d->actions; p.range = d->max_abs_range;
    p.rewards = d->rewards; p.game_overs = d->game_overs; p.seg_off = d->seg_offsets; p.seg_len = d->seg_lengths;
    p.S = S; p.rows = rows; p.mode = d->mode; p.huber = d->huber; p.K = K; p.D = D; p.N = N;
    p.discount = d->discount; p.gae_lambda = d->gae_lambda;
    p.beta_entropy = d->beta_entropy; p.v_weight = d->v_weight; p.p_weight = d->p_weight;
    p.z = d->z; p.means = d->means; p.stds = d->stds; p.dh = d->dh;
    p.dh_planes = static_cast<uint16_t*>(d->dh_planes); p.dh_plane_stride = d->dh_plane_stride;
    // workspace: dL/dZ [rows, N] | per-row losses | targets | advantages | row slots [rows] | bootstrap [segments] |
    // chunk partials; the optional outputs replace their workspace slices
    float* ws = d->workspace;
    p.dz = d->dz ? d->dz : ws;
    p.rowloss = ws + (size_t)rows * N;
    p.targets = d->targets ? d->targets : p.rowloss + rows;
    p.advantages = d->advantages ? d->advantages : p.rowloss + 2 * (size_t)rows;
    p.row_seg = reinterpret_cast<int32_t*>(p.rowloss + 3 * (size_t)rows);
    p.bootstrap = d->bootstrap ? d->bootstrap : p.rowloss + 4 * (size_t)rows;
    float* part = p.rowloss + 4 * (size_t)rows + S;
    cudaStream_t st = as_stream(stream);
    // up to 78 KB at K = 512, N = 35 (the staged kernel and eight row buffers): opted into once per instantiation and
    // device, at the size of the largest shape
    auto smem_of = [](int N, int K) { return (size_t)(N * K + kPgWarps * K) * sizeof(float); };
    static bool attr_set[kMaxDevices][2] = {};
    int dev = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    CB200_CHECK_ARG(dev < kMaxDevices, "device ordinal out of range");
    const int ti = K == 512 ? 1 : 0;
    if (!attr_set[dev][ti]) {
        const int most = (int)smem_of(kAcgMaxN, K);
        if (ti) {
            CB200_CUDA(cudaFuncSetAttribute(ac_gauss_rows_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
            CB200_CUDA(cudaFuncSetAttribute(ac_gauss_grad_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
        } else {
            CB200_CUDA(cudaFuncSetAttribute(ac_gauss_rows_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
            CB200_CUDA(cudaFuncSetAttribute(ac_gauss_grad_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
        }
        attr_set[dev][ti] = true;
    }
    const unsigned row_grid = (unsigned)((rows + S + kPgBlockRows - 1) / kPgBlockRows);
    const unsigned grad_grid = (unsigned)((rows + kPgBlockRows - 1) / kPgBlockRows);
    const size_t smem_rows = (size_t)N * K * sizeof(float), smem_grad = smem_of(N, K);
    if (K == 512) {
        CB200_LAUNCH(ac_gauss_rows_kernel<16>, row_grid, 32 * kPgWarps, smem_rows, st, p);
        CB200_LAUNCH(ac_gauss_segments_kernel, (unsigned)((S + 127) / 128), 128, 0, st, p);
        CB200_LAUNCH(ac_gauss_grad_kernel<16>, grad_grid, 32 * kPgWarps, smem_grad, st, p);
    } else {
        CB200_LAUNCH(ac_gauss_rows_kernel<8>, row_grid, 32 * kPgWarps, smem_rows, st, p);
        CB200_LAUNCH(ac_gauss_segments_kernel, (unsigned)((S + 127) / 128), 128, 0, st, p);
        CB200_LAUNCH(ac_gauss_grad_kernel<8>, grad_grid, 32 * kPgWarps, smem_grad, st, p);
    }
    const int n_out = K * N + N + 1, chunks = (rows + kPgChunk - 1) / kPgChunk;
    const dim3 dw_grid((unsigned)((n_out + 255) / 256), (unsigned)min(chunks, 65535));
    CB200_LAUNCH(pg_head_dw_kernel, dw_grid, 256, 0, st, d->h, p.dz, p.rowloss, rows, K, N, part);
    CB200_LAUNCH(dqn_head_reduce_kernel, (unsigned)((n_out + 31) / 32), 256, 0, st, part, chunks, n_out, K * N, N, 1.0f,
                 d->dw, d->db, d->loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_gaussian_policy_act(const float* z, int64_t envs, int32_t action_dim, const float* max_abs_range,
                              const double* normals, double* actions, float* means, float* stds, void* stream) {
    CB200_CHECK_ARG(z && max_abs_range && actions, "null pointer");
    CB200_CHECK_ARG(envs >= 1 && envs <= (1 << 24), "1 <= envs <= 2^24");
    CB200_CHECK_ARG(action_dim >= 1 && action_dim <= kAcgMaxD, "1 <= action_dim <= 17");
    const int64_t n = envs * action_dim;
    CB200_LAUNCH(ac_gauss_act_kernel, (unsigned)((n + 127) / 128), 128, 0, as_stream(stream), z, envs, action_dim,
                 max_abs_range, normals, actions, means, stds);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

}  // extern "C"
