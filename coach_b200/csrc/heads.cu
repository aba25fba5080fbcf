// coach_b200/csrc/heads.cu -- policy / value head losses of the actor-critic agents (ClippedPPO, DDPG/TD3, SAC) and
// the minibatch row gather used by the epoch loops.  Reference lines are cited in include/coach_b200.h.
#include <math.h>

#include "common.cuh"

namespace cb200 {

constexpr int kMaxActionDim = 32;
constexpr float kLog2Pi = 1.8378770664093453f;
constexpr float kTfEps = 1e-15f;          // `eps` of heads/ppo_head.py (std + eps)

// fixed-order block reduction of one float per thread (blockDim.x a power of two <= 1024)
__device__ __forceinline__ float block_sum(float v, float* red) {
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const float out = red[0];
    __syncthreads();
    return out;
}

// Per-element Gaussian terms of the two PPO heads (clipped and KL-penalty): sigma = exp(logstd) + eps, one dimension's
// KL(old || new) of diagonal Gaussians, the log-likelihood from its squared-z sum, the entropy and d sigma / d logstd
// over sigma.
__device__ __forceinline__ float ppo_sigma(float logstd) { return expf(logstd) + kTfEps; }
__device__ __forceinline__ float ppo_kl_term(float m, float old_m, float sig, float old_sig) {
    const float dm = (m - old_m) / sig;
    const float rs = old_sig / sig;
    return 0.5f * (rs * rs + dm * dm - 1.0f) - logf(rs);
}
__device__ __forceinline__ float ppo_logp(float q, float sum_log_sig, int A) {
    return -0.5f * q - sum_log_sig - 0.5f * A * kLog2Pi;
}
__device__ __forceinline__ float ppo_entropy(int A, float sum_log_sig) {
    return 0.5f * A * (1.0f + kLog2Pi) + sum_log_sig;
}
__device__ __forceinline__ float ppo_dsig(float sig) { return (sig - kTfEps) / sig; }

// =====================================================================================================================
// PPOHead, continuous actions (heads/ppo_head.py:52-144): diagonal Gaussian with state-independent log-std.
//   sigma_j   = exp(logstd_j) + eps
//   logp_i    = -0.5 * sum_j ((a_ij - mu_ij)/sigma_j)^2 - sum_j log sigma_j - 0.5*k*log(2 pi)
//   ratio_i   = exp(logp_i - logp_old_i);  clipped_i = clip(ratio_i, 1 - e, 1 + e),  e = clip_eps * rescaler
//   L         = -mean_i min(ratio_i * A_i, clipped_i * A_i)  -  beta * mean entropy
// Outputs the gradients wrt mu and logstd and the scalars the reference logs (loss, KL(old||new), entropy, mean
// ratio, mean clipped ratio).  One block; fixed reduction order.
// =====================================================================================================================
__global__ void __launch_bounds__(256) ppo_continuous_head_kernel(
    const float* __restrict__ mu, const float* __restrict__ logstd, const float* __restrict__ actions,
    const float* __restrict__ old_mu, const float* __restrict__ old_logstd, const float* __restrict__ advantages,
    int64_t B, int A, float clip_eps, float beta_entropy, float* __restrict__ d_mu, float* __restrict__ d_logstd,
    float* __restrict__ scalars /* [loss, kl, entropy, mean ratio, mean clipped ratio] */) {
    __shared__ float red[256];
    __shared__ float sig[kMaxActionDim], osig[kMaxActionDim], dls_part[kMaxActionDim];
    if (threadIdx.x < A) {
        sig[threadIdx.x] = ppo_sigma(logstd[threadIdx.x]);
        osig[threadIdx.x] = ppo_sigma(old_logstd[threadIdx.x]);
        dls_part[threadIdx.x] = 0.f;
    }
    __syncthreads();
    float sum_log_sig = 0.f, sum_log_osig = 0.f;
    for (int j = 0; j < A; ++j) {
        sum_log_sig += logf(sig[j]);
        sum_log_osig += logf(osig[j]);
    }
    const float inv_b = 1.0f / (float)B;
    const float lo = 1.0f - clip_eps, hi = 1.0f + clip_eps;
    float loss_acc = 0.f, kl_acc = 0.f, ratio_acc = 0.f, cratio_acc = 0.f;
    float dls_local[kMaxActionDim];
#pragma unroll
    for (int j = 0; j < kMaxActionDim; ++j) dls_local[j] = 0.f;
    for (int64_t i = threadIdx.x; i < B; i += blockDim.x) {
        float q = 0.f, qo = 0.f, kl = 0.f;
        for (int j = 0; j < A; ++j) {
            const float a = actions[i * A + j];
            const float z = (a - mu[i * A + j]) / sig[j];
            const float zo = (a - old_mu[i * A + j]) / osig[j];
            q += z * z;
            qo += zo * zo;
            kl += ppo_kl_term(mu[i * A + j], old_mu[i * A + j], sig[j], osig[j]);
        }
        const float logp = ppo_logp(q, sum_log_sig, A);
        const float logp_old = ppo_logp(qo, sum_log_osig, A);
        const float ratio = expf(logp - logp_old);
        const float cl = fminf(fmaxf(ratio, lo), hi);
        const float adv = advantages[i];
        const float s1 = ratio * adv, s2 = cl * adv;
        // tf.minimum passes the gradient to its first argument when s1 <= s2; clip_by_value passes it inside [lo, hi]
        float ds_dratio;
        if (s1 <= s2) ds_dratio = adv;
        else ds_dratio = (ratio >= lo && ratio <= hi) ? adv : 0.f;
        loss_acc += fminf(s1, s2);
        kl_acc += kl;
        ratio_acc += ratio;
        cratio_acc += cl;
        const float dlogp = -inv_b * ds_dratio * ratio;       // dL/dlogp_i
        for (int j = 0; j < A; ++j) {
            const float z = (actions[i * A + j] - mu[i * A + j]) / sig[j];
            d_mu[i * A + j] = dlogp * z / sig[j];
            // d logp / d logstd_j = (z^2 - 1) * exp(logstd_j) / sigma_j
            dls_local[j] += dlogp * (z * z - 1.0f) * ppo_dsig(sig[j]);
        }
    }
    const float loss_sum = block_sum(loss_acc, red);
    const float kl_sum = block_sum(kl_acc, red);
    const float ratio_sum = block_sum(ratio_acc, red);
    const float cratio_sum = block_sum(cratio_acc, red);
    for (int j = 0; j < A; ++j) {
        const float s = block_sum(dls_local[j], red);
        if (threadIdx.x == 0) dls_part[j] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float entropy = ppo_entropy(A, sum_log_sig);     // state independent
        for (int j = 0; j < A; ++j) {
            // entropy regulariser -beta * H:  dH/dlogstd_j = exp(logstd_j) / sigma_j
            d_logstd[j] = dls_part[j] - beta_entropy * ppo_dsig(sig[j]);
        }
        if (scalars) {
            scalars[0] = -loss_sum * inv_b - beta_entropy * entropy;
            scalars[1] = kl_sum * inv_b;
            scalars[2] = entropy;
            scalars[3] = ratio_sum * inv_b;
            scalars[4] = cratio_sum * inv_b;
        }
    }
}

// =====================================================================================================================
// dst[c][i, :] = src[c][idx[*offset + i], :] -- minibatch extraction inside a (CUDA-graph captured) epoch loop: the
// launch parameters stay constant, only the device scalar *offset changes between replays.
// =====================================================================================================================
struct AtColumns {
    const uint8_t* src[CB200_MAX_COLUMNS];
    uint8_t* dst[CB200_MAX_COLUMNS];
    int64_t row_bytes[CB200_MAX_COLUMNS];
    int n;
};
__global__ void __launch_bounds__(256) gather_at_kernel(AtColumns cols, const int64_t* __restrict__ idx,
                                                        const int64_t* __restrict__ offset_ptr, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t off = offset_ptr ? *offset_ptr : 0;
    for (int64_t w = warp; w < n * cols.n; w += nwarps) {
        const int64_t i = w / cols.n;
        const int c = (int)(w - i * cols.n);
        const int64_t row = idx ? idx[off + i] : (off + i);
        const uint8_t* s = cols.src[c] + row * cols.row_bytes[c];
        uint8_t* d = cols.dst[c] + i * cols.row_bytes[c];
        const int64_t bytes = cols.row_bytes[c];
        const uintptr_t al = reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d) | (uintptr_t)bytes;
        if ((al & 3) == 0) {
            for (int64_t o = (int64_t)lane * 4; o < bytes; o += 128)
                *reinterpret_cast<uint32_t*>(d + o) = *reinterpret_cast<const uint32_t*>(s + o);
        } else {
            for (int64_t o = lane; o < bytes; o += 32) d[o] = s[o];
        }
    }
}


// dz[r, c] = dy[r, c] * act'(y[r, c])  with independent leading dimensions (activation backward on a column block of a
// wider buffer, e.g. the embedder part of a concatenated critic input)
__global__ void __launch_bounds__(256) act_backward_kernel(const float* __restrict__ dy, int ld_dy,
                                                           const float* __restrict__ y, int ld_y, int64_t rows,
                                                           int cols, int act, float* __restrict__ dz, int ld_dz) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int64_t r = i / cols;
    const int c = (int)(i - r * cols);
    const float yy = y[r * ld_y + c];
    float g = 1.f;
    if (act == CB200_ACT_RELU) g = yy > 0.f ? 1.f : 0.f;
    else if (act == CB200_ACT_TANH) g = 1.f - yy * yy;
    dz[r * ld_dz + c] = dy[r * ld_dy + c] * g;
}

// dst[r, c] = alpha * src[r, c] + beta * dst[r, c]   (strided 2-D; beta == 0 never reads dst)
__global__ void __launch_bounds__(256) axpby_2d_kernel(const float* __restrict__ src, int ld_src, int64_t rows, int cols,
                                                       float alpha, float beta, float* __restrict__ dst, int ld_dst) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int64_t r = i / cols;
    const int c = (int)(i - r * cols);
    const float v = alpha * src[r * ld_src + c];
    dst[r * ld_dst + c] = (beta == 0.f) ? v : (v + beta * dst[r * ld_dst + c]);
}

// DDPG / TD3 / SAC bootstrapped targets, evaluated like the numpy expression (fp64 rewards, fp32 network output):
//   y = r + (1 - done) * discount * q_next      [done ignored when use_non_zero_discount_for_terminal_states]
//   optional clip (ddpg_agent.py:163-164) with np.clip's rules (NaN passes through, a value equal to a bound is kept);
//   written as fp32 (the TF placeholder dtype)
__global__ void __launch_bounds__(256) ac_td_targets_kernel(const double* __restrict__ rewards,
                                                            const uint8_t* __restrict__ dones,
                                                            const float* __restrict__ q_next, int ld_q, int64_t B,
                                                            double discount, int ignore_done, int use_clip,
                                                            double clip_lo, double clip_hi, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    double y;
    if (ignore_done) {
        // ddpg_agent.py:155: rewards + discount * q -- a Python float times a float32 array stays float32 in numpy, so
        // this product is rounded to fp32 before the fp64 add (pinned by tests/golden/agent_prologues.npz, "ddpg2")
        y = __dadd_rn(rewards[i], (double)__fmul_rn((float)discount, q_next[i * ld_q]));
    } else {
        // :157-158: (1.0 - game_overs) is a float64 array, the whole product is fp64
        const double nd = __dsub_rn(1.0, dones[i] ? 1.0 : 0.0);
        y = __dadd_rn(rewards[i], __dmul_rn(__dmul_rn(nd, discount), (double)q_next[i * ld_q]));
    }
    if (use_clip) y = y < clip_lo ? clip_lo : (y > clip_hi ? clip_hi : y);
    out[i] = (float)y;
}

// out[i] = min(a[i], b[i])  (TD3 / SAC clipped double-Q) as tf.minimum evaluates it (std::min): `a` unless b < a, so
// a tie of +0 and -0 keeps a's sign and a NaN in `a` passes through
__global__ void __launch_bounds__(256) min2_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n,
                                                   float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = b[i] < a[i] ? b[i] : a[i];
}

// TD3 target policy smoothing (td3_agent.py:162-164): a = clip(a + clip(noise, -c, c), lo, hi), in place.  The
// reference adds the fp64 numpy draw to the fp32 network output in fp64, clips in fp64 and the result is rounded to
// fp32 once when it is fed to the critic: same operations here (pinned by tests/golden/agent_prologues.npz).
__global__ void __launch_bounds__(256) td3_smooth_kernel(float* __restrict__ actions, const double* __restrict__ noise,
                                                         int64_t n, double noise_clip, double lo, double hi) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // np.clip: NaN passes through, a value equal to a bound is kept
    const double x = noise[i];
    const double nz = x < -noise_clip ? -noise_clip : (x > noise_clip ? noise_clip : x);
    const double y = __dadd_rn((double)actions[i], nz);
    actions[i] = (float)(y < lo ? lo : (y > hi ? hi : y));
}

// =====================================================================================================================
// CategoricalQHead + the distributional TD target of CategoricalDQNAgent / RainbowDQNAgent
// (agents/categorical_dqn_agent.py:105-165, rainbow_dqn_agent.py:93-140, heads/categorical_q_head.py:41-57).
// One warp per sample:
//   p_next[a, :]  = softmax(next logits[a, :])  (fp32)      Q[a] = sum_j (double)p[a, j] * z[j]   (np.dot with fp64 z)
//   a*            = argmax_a Q[a] of the target prediction  (of the `select` prediction for Rainbow's double-Q rule)
//   m[:]          = the projection of  r + boot * gamma_n * z_j  onto the support, accumulated in fp64 in the
//                   reference's order (j ascending; first the floor bin, then the ceil bin; an integral b_j adds
//                   nothing to either bin -- the reference's arithmetic, kept)
//   labels[a, :]  = online softmax for a != action (TD_targets starts as the online prediction), (float)m for the action
//   loss[a]       = sum_j labels_j * (log sum_k exp(x_k - max) - (x_j - max))         (tf.nn.softmax_cross_entropy)
//   dlogits[a, :] = softmax - labels for the taken action, exactly 0 elsewhere (labels ARE the softmax there)
// next_is_prob: the "next" / "select" inputs already hold probabilities (parity tests pin the projection bit for bit).
// =====================================================================================================================
struct C51Params {
    const float* next; const float* online; const float* select;
    const int64_t* actions; const double* rewards; const uint8_t* game_overs; const double* bootstrap;
    const double* z;
    double gamma_n;
    int B, A, N, next_is_prob;
    float* labels; float* dlogits; float* loss_rows; double* td_err; double* q_online; int64_t* target_actions;
};

constexpr int kC51Warps = 4;

__device__ __forceinline__ float warp_max(float v) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// softmax of one row of N logits into dst (shared); returns (max, sum of exp) to every lane
__device__ __forceinline__ void warp_softmax(const float* __restrict__ x, int N, int lane, float* dst, float& mx,
                                             float& sum) {
    float m = -INFINITY;
    for (int j = lane; j < N; j += 32) m = fmaxf(m, x[j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < N; j += 32) {
        const float e = expf(x[j] - m);
        dst[j] = e;
        s += e;
    }
    s = warp_sum(s);
    for (int j = lane; j < N; j += 32) dst[j] = dst[j] / s;
    mx = m;
    sum = s;
    __syncwarp();
}

__global__ void __launch_bounds__(kC51Warps * 32) c51_head_kernel(C51Params p) {
    extern __shared__ double c51_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * kC51Warps + warp;
    if (b >= p.B) return;
    const int A = p.A, N = p.N;
    double* s_m = c51_smem + (size_t)warp * N;                                         // [N] fp64 projection
    float* s_p = reinterpret_cast<float*>(c51_smem + (size_t)kC51Warps * N) + (size_t)warp * 2 * N;   // [2][N]
    float* s_sel = s_p + N;
    const int64_t row = (int64_t)b * A * N;

    // ---- target action ------------------------------------------------------------------------------------------
    int best = 0;
    double best_q = 0.0;
    const float* sel_src = p.select ? p.select : p.next;
    for (int a = 0; a < A; ++a) {
        float mx, sum;
        if (p.next_is_prob) {
            for (int j = lane; j < N; j += 32) s_sel[j] = sel_src[row + (int64_t)a * N + j];
            __syncwarp();
        } else {
            warp_softmax(sel_src + row + (int64_t)a * N, N, lane, s_sel, mx, sum);
        }
        double q = 0.0;
        for (int j = lane; j < N; j += 32) q += (double)s_sel[j] * p.z[j];
        q = warp_sum(q);
        if (a == 0 || q > best_q) { best_q = q; best = a; }                            // np.argmax: first maximum
        __syncwarp();
    }
    if (p.target_actions && lane == 0) p.target_actions[b] = best;
    {   // distribution of the target network for the chosen action
        float mx, sum;
        if (p.next_is_prob) {
            for (int j = lane; j < N; j += 32) s_p[j] = p.next[row + (int64_t)best * N + j];
            __syncwarp();
        } else {
            warp_softmax(p.next + row + (int64_t)best * N, N, lane, s_p, mx, sum);
        }
    }
    // ---- projection, sequential in j like the reference loop ---------------------------------------------------------
    for (int j = lane; j < N; j += 32) s_m[j] = 0.0;
    __syncwarp();
    if (lane == 0) {
        const double boot = p.bootstrap ? p.bootstrap[b] : __dsub_rn(1.0, p.game_overs[b] ? 1.0 : 0.0);
        const double coef = __dmul_rn(boot, p.gamma_n);
        const double r = p.rewards[b], z0 = p.z[0], zl = p.z[N - 1];
        const double dz = __dsub_rn(p.z[1], z0);
        for (int j = 0; j < N; ++j) {
            const double tz = fmax(fmin(__dadd_rn(r, __dmul_rn(coef, p.z[j])), zl), z0);
            const double bj = __ddiv_rn(__dsub_rn(tz, z0), dz);
            const double u = ceil(bj), l = floor(bj);
            const double pj = (double)s_p[j];
            // (z[N-1] - z[0]) / (z[1] - z[0]) of a linspace support can round above N - 1: a share that lands on bin N
            // is dropped (s_m[N] is the next warp's row)
            if ((int)l < N) s_m[(int)l] = __dadd_rn(s_m[(int)l], __dmul_rn(pj, __dsub_rn(u, bj)));
            if ((int)u < N) s_m[(int)u] = __dadd_rn(s_m[(int)u], __dmul_rn(pj, __dsub_rn(bj, l)));
        }
    }
    __syncwarp();
    // ---- online head: labels, cross entropy, gradient ---------------------------------------------------------------
    const int act = (int)p.actions[b];
    for (int a = 0; a < A; ++a) {
        const float* x = p.online + row + (int64_t)a * N;
        float mx, sum;
        warp_softmax(x, N, lane, s_sel, mx, sum);
        const float lse = logf(sum);
        float loss = 0.f;
        double q = 0.0;
        for (int j = lane; j < N; j += 32) {
            const float sm = s_sel[j];
            const float lab = (a == act) ? (float)s_m[j] : sm;
            loss += lab * (lse - (x[j] - mx));
            p.labels[row + (int64_t)a * N + j] = lab;
            p.dlogits[row + (int64_t)a * N + j] = (a == act) ? (sm - lab) : 0.f;
            q += (double)sm * p.z[j];
        }
        loss = warp_sum(loss);
        q = warp_sum(q);
        if (lane == 0) {
            p.loss_rows[(int64_t)b * A + a] = loss;
            if (p.q_online) p.q_online[(int64_t)b * A + a] = q;
            if (a == act) p.td_err[b] = (double)loss;
        }
        __syncwarp();
    }
}

// q_values of the CategoricalQHead (categorical_q_head.py:56): tensordot(cast(softmax, fp64), z), one warp per (b, a) row
__global__ void __launch_bounds__(128) c51_q_values_kernel(const float* __restrict__ logits, const double* __restrict__ z,
                                                           int64_t rows, int N, double* __restrict__ q) {
    const int64_t r = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const float* x = logits + r * N;
    float m = -INFINITY;
    for (int j = lane; j < N; j += 32) m = fmaxf(m, x[j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < N; j += 32) s += expf(x[j] - m);
    s = warp_sum(s);
    double acc = 0.0;
    for (int j = lane; j < N; j += 32) acc += (double)(expf(x[j] - m) / s) * z[j];
    acc = warp_sum(acc);
    if (lane == 0) q[r] = acc;
}

// total loss = tf.reduce_sum over the [B, A] loss tensor (general_network.py:360), one block, fixed order
__global__ void __launch_bounds__(256) c51_loss_sum_kernel(const float* __restrict__ loss_rows, int64_t n,
                                                           float* __restrict__ total) {
    __shared__ float red[256];
    float v = 0.f;
    for (int64_t i = threadIdx.x; i < n; i += 256) v += loss_rows[i];
    const float t = block_sum(v, red);
    if (threadIdx.x == 0) *total = t;
}

// =====================================================================================================================
// SACPolicyHead (heads/sac_head.py:60-97): head output z = [mu | log_sigma_raw]  (2A columns),
//   log_sigma = clip(log_sigma_raw, -20, 2);  u = mu + exp(log_sigma) * eps;  a = tanh(u);
//   log pi(a|s) = sum_j [ -0.5 eps_j^2 - log_sigma_j - 0.5 log(2 pi) ] - sum_j log(1 - tanh(u_j)^2 + 1e-6)
// (MultivariateNormalDiag.log_prob of the reparameterised sample, minus the squash correction :49-58).
// =====================================================================================================================
constexpr float kSacLogSigMin = -20.f, kSacLogSigMax = 2.f, kSacEps = 1e-6f;

__global__ void __launch_bounds__(256) sac_policy_sample_kernel(const float* __restrict__ z, const float* __restrict__ eps,
                                                                int64_t B, int A, float* __restrict__ raw,
                                                                float* __restrict__ act, float* __restrict__ logp) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    float lp = 0.f;
    for (int j = 0; j < A; ++j) {
        const float mu = z[i * 2 * A + j];
        const float ls = fminf(fmaxf(z[i * 2 * A + A + j], kSacLogSigMin), kSacLogSigMax);
        const float e = eps[i * A + j];
        const float u = mu + expf(ls) * e;
        const float t = tanhf(u);
        if (raw) raw[i * A + j] = u;
        if (act) act[i * A + j] = t;
        lp += -0.5f * e * e - ls - 0.5f * kLog2Pi - logf(1.0f - t * t + kSacEps);
    }
    if (logp) logp[i] = lp;
}

// gradient of  mean_b log pi(a~|s)  (noise eps_lp)  minus  sum_b <dq_da_b, a~_b>  (noise eps_q)  wrt the head output z:
// the two terms of policy_grads = dlogp_dphi - dq_dphi (soft_actor_critic_agent.py:213-232); each term was evaluated
// by its own sess.run and therefore with its own noise sample (SURVEY.md Q9).
__global__ void __launch_bounds__(256) sac_policy_grad_kernel(const float* __restrict__ z, const float* __restrict__ eps_lp,
                                                              const float* __restrict__ eps_q,
                                                              const float* __restrict__ dq_da, int64_t B, int A,
                                                              float* __restrict__ dz) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const float inv_b = 1.0f / (float)B;
    for (int j = 0; j < A; ++j) {
        const float mu = z[i * 2 * A + j];
        const float lsr = z[i * 2 * A + A + j];
        const float ls = fminf(fmaxf(lsr, kSacLogSigMin), kSacLogSigMax);
        const float in_range = (lsr >= kSacLogSigMin && lsr <= kSacLogSigMax) ? 1.f : 0.f;   // clip_by_value gradient
        const float sig = expf(ls);
        // --- d mean(log pi) ---
        const float e2 = eps_lp[i * A + j];
        const float u2 = mu + sig * e2, t2 = tanhf(u2);
        const float gprime = (-2.0f * t2 * (1.0f - t2 * t2)) / (1.0f - t2 * t2 + kSacEps);   // d/du log(1 - t^2 + eps)
        float d_mu = inv_b * (-gprime);
        float d_ls = inv_b * (-1.0f - gprime * sig * e2) * in_range;
        // --- minus sum <dq_da, tanh(mu + sig * eps3)> ---
        const float e3 = eps_q[i * A + j];
        const float u3 = mu + sig * e3, t3 = tanhf(u3);
        const float w = dq_da[i * A + j] * (1.0f - t3 * t3);
        d_mu -= w;
        d_ls -= w * sig * e3 * in_range;
        dz[i * 2 * A + j] = d_mu;
        dz[i * 2 * A + A + j] = d_ls;
    }
}

// seeds of d mean_b(min(q1, q2)) / dq_k (sac_q_head.py:84-86; tf.minimum sends the gradient to its first argument on
// ties), optionally also out = min(q1, q2)
__global__ void __launch_bounds__(256) sac_min_seed_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                           int64_t B, float* __restrict__ d1, float* __restrict__ d2,
                                                           float* __restrict__ qmin) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const bool first = q1[i] <= q2[i];
    const float s = 1.0f / (float)B;
    if (d1) d1[i] = first ? s : 0.f;
    if (d2) d2[i] = first ? 0.f : s;
    if (qmin) qmin[i] = q2[i] < q1[i] ? q2[i] : q1[i];      // the value as tf.minimum (std::min): q1 unless q2 < q1
}

// out[i] = a[i] - b[i]   (value targets = min Q - log pi, soft_actor_critic_agent.py:244)
__global__ void __launch_bounds__(256) sub_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n,
                                                  float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] - b[i];
}

// out[i] = (float) in[i]   (fp64 advantages / value targets -> fp32 network feeds)
__global__ void __launch_bounds__(256) f64_to_f32_kernel(const double* __restrict__ in, int64_t n,
                                                         float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}

// =====================================================================================================================
// NAFHead (heads/naf_head.py:45-86), see cb200_naf_head in the header.  One warp per sample; lane c owns action c and
// column c of L.  The sample's packed l vector is staged in shared memory (coalesced), so that lane c reads its column
// for w_c = sum_{r >= c} L[r, c] d_r and lane r its row for (L w)_r = sum_{c <= r} L[r, c] w_c; d and w travel by
// shuffles.  |w|^2 is an xor butterfly, which leaves the same bits in every lane.  The d_l column of each lane is
// written back into the staging buffer and stored coalesced.
constexpr int kNafWarps = 8;
constexpr int kNafMaxL = kMaxActionDim * (kMaxActionDim + 1) / 2;

struct NafParams {
    const float *z_v, *z_mu, *l, *scale, *actions, *targets;
    int huber, A, ld_mu, ld_l, ld_u;
    int64_t B;
    float *mu, *q, *d_zv, *d_zmu, *d_l, *adv;
};

// Huber (delta 1) / squared error of e = Q - y and the derivative dl/dQ, as regression_head_kernel (learn.cu) has them
__device__ __forceinline__ void naf_loss_terms(float e, int huber, float& l, float& g) {
    if (huber) {
        const float ae = fabsf(e);
        const float q = fminf(ae, 1.0f);
        l = 0.5f * q * q + (ae - q);
        g = (ae <= 1.0f) ? e : (e > 0.f ? 1.0f : -1.0f);
    } else {
        l = e * e;
        g = 2.0f * e;
    }
}

template <bool kTrain>
__global__ void __launch_bounds__(kNafWarps * 32) naf_head_kernel(const NafParams p) {
    __shared__ float s_l[kNafWarps][kNafMaxL];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t b = (int64_t)blockIdx.x * kNafWarps + wib;
    if (b >= p.B) return;                                              // whole warps only
    const int A = p.A;
    const bool own = lane < A;
    float t = 0.f, mu = 0.f;
    if (own) {
        t = tanhf(p.z_mu[b * p.ld_mu + lane]);
        mu = t * p.scale[lane];
        p.mu[b * p.ld_mu + lane] = mu;
    }
    if (!kTrain) {
        if (lane == 0 && p.q) p.q[b] = p.z_v[b];                       // u = mu: the advantage is 0
        return;
    }
    const float v = p.z_v[b];
    float* ls = s_l[wib];
    const int nl = A * (A + 1) / 2;
    for (int k = lane; k < nl; k += 32) ls[k] = p.l[b * p.ld_l + k];
    __syncwarp();
    const float d = own ? p.actions[b * p.ld_u + lane] - mu : 0.f;
    const int ic = lane * A - lane * (lane - 1) / 2;                   // start of column `lane`
    const float diag = own ? expf(ls[ic]) : 0.f;
    // w_c = sum_{r >= c} L[r, c] d_r
    float w = 0.f;
    for (int r = 0; r < A; ++r) {
        const float dr = __shfl_sync(0xffffffffu, d, r);
        if (own && r >= lane) w = fmaf(r == lane ? diag : ls[ic + r - lane], dr, w);
    }
    float ww = w * w;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ww += __shfl_xor_sync(0xffffffffu, ww, o);
    const float adv = -0.5f * ww;
    const float qv = v + adv;
    float lterm, g;
    naf_loss_terms(qv - p.targets[b], p.huber, lterm, g);
    const float dq = (1.0f / (float)p.B) * g;
    // (L w)_r = sum_{c <= r} L[r, c] w_c = dA/dmu_r
    float lw = 0.f;
    for (int c = 0; c < A; ++c) {
        const float wc = __shfl_sync(0xffffffffu, w, c);
        const int icc = c * A - c * (c - 1) / 2;
        if (own && c <= lane) lw = fmaf(c == lane ? diag : ls[icc + lane - c], wc, lw);
    }
    if (own) p.d_zmu[b * p.ld_mu + lane] = dq * lw * p.scale[lane] * (1.0f - t * t);
    if (lane == 0) {
        p.q[b] = qv;
        p.d_zv[b] = dq;
        if (p.adv) p.adv[b] = adv;
    }
    __syncwarp();                                                      // every read of the staged l is done
    // dA/dL[r, c] = -d_r w_c; the diagonal entries are exp(l): times L[c, c]
    for (int r = 0; r < A; ++r) {
        const float dr = __shfl_sync(0xffffffffu, d, r);
        if (own && r >= lane) {
            const float gl = dq * (-dr * w);
            ls[ic + r - lane] = r == lane ? gl * diag : gl;
        }
    }
    __syncwarp();
    for (int k = lane; k < nl; k += 32) p.d_l[b * p.ld_l + k] = ls[k];
}

// loss = mean_b l(q_b - y_b) in a fixed order (the per-thread strided sums and the tree of regression_head_kernel)
__global__ void __launch_bounds__(256) naf_loss_kernel(const float* __restrict__ q, const float* __restrict__ targets,
                                                       int64_t B, int huber, float* __restrict__ loss) {
    __shared__ float red[256];
    float local = 0.f;
    for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
        float l, g;
        naf_loss_terms(q[b] - targets[b], huber, l, g);
        local += l;
    }
    const float s = block_sum(local, red);
    if (threadIdx.x == 0) *loss = s * (1.0f / (float)B);
}

// =====================================================================================================================
// QuantileRegressionQHead + the TD targets of QuantileRegressionDQNAgent (agents/qr_dqn_agent.py:97-137,
// heads/quantile_regression_q_head.py:33-71), see cb200_qr_head in the header.  One CTA per sample:
//   Q'[a]   = sum_j (double)next[a, j] * (1.0 / N)        (qr_row_q; one warp per action)
//   a*      = first argmax of Q'
//   T_j     = (float)(r + ((1.0 - done) * gamma) * (double)next[a*, j])              (fp64, _rn: the numpy expression)
//   sigma   = argsort of the taken row, ties by index;  tau_i = (float)tau_hat[sigma(i)]   (the reference's permutation)
//   thread i: the pair terms (i, j) for j = 0 .. N-1 in order, in fp32 without contraction; the loss sums in fp32, the
//             gradient's terms (of both signs) in fp64
// The per-sample loss goes to the workspace; qr_loss_kernel sums it in a fixed order: the same bits on every call.
// =====================================================================================================================
constexpr int kQrThreads = 256;
constexpr int kQrMaxAtoms = 1024;
constexpr int kQrMaxActions = 256;

// the head's q_values for one row of N quantiles (np.dot with ones(N) / N in fp64): lanes stride j, then an xor
// butterfly, which leaves the same bits in every lane
__device__ __forceinline__ double qr_row_q(const float* __restrict__ row, int N, int lane) {
    const double p = __ddiv_rn(1.0, (double)N);
    double acc = 0.0;
    for (int j = lane; j < N; j += 32) acc = __dadd_rn(acc, __dmul_rn((double)row[j], p));
    return warp_sum(acc);
}

struct QrParams {
    const float* next; const float* online; const int64_t* actions; const double* rewards; const uint8_t* game_overs;
    double discount;
    float kappa;
    int B, A, N;
    float* dq; float* targets; float* taus; int64_t* target_actions; float* partial;
};

__global__ void __launch_bounds__(kQrThreads) qr_head_kernel(const QrParams p) {
    __shared__ float s_theta[kQrMaxAtoms], s_t[kQrMaxAtoms], s_tau[kQrMaxAtoms], s_g[kQrMaxAtoms];
    __shared__ int s_sigma[kQrMaxAtoms];
    __shared__ double s_q[kQrMaxActions];
    __shared__ float red[kQrThreads];
    __shared__ int s_best;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int A = p.A, N = p.N;
    const int64_t row = (int64_t)b * A * N;
    // ---- Q' and the target action ------------------------------------------------------------------------------------
    for (int a = warp; a < A; a += kQrThreads / 32) {
        const double q = qr_row_q(p.next + row + (int64_t)a * N, N, lane);
        if (lane == 0) s_q[a] = q;
    }
    const int64_t act64 = p.actions[b];
    const bool valid = act64 >= 0 && act64 < A;
    const int act = valid ? (int)act64 : 0;
    for (int i = tid; i < N; i += kQrThreads) {
        s_theta[i] = p.online[row + (int64_t)act * N + i];
        s_sigma[i] = i;                      // every slot holds an index even if NaNs make the ranks collide
    }
    __syncthreads();
    if (tid == 0) {
        int best = 0;
        for (int a = 1; a < A; ++a)
            if (s_q[a] > s_q[best]) best = a;                                    // np.argmax: first maximum
        s_best = best;
        if (p.target_actions) p.target_actions[b] = best;
    }
    // ---- ranks of the taken row (index tie-break = argsort kind='stable') --------------------------------------------
    for (int i = tid; i < N; i += kQrThreads) {
        const float v = s_theta[i];
        int r = 0;
        for (int k = 0; k < N; ++k) {
            const float u = s_theta[k];
            r += (u < v || (u == v && k < i)) ? 1 : 0;
        }
        s_sigma[r] = i;                                                          // sigma = argsort: sigma(rank(i)) = i
    }
    __syncthreads();
    // ---- TD targets and the permuted midpoints -----------------------------------------------------------------------
    const int best = s_best;
    const double coef = __dmul_rn(__dsub_rn(1.0, p.game_overs[b] ? 1.0 : 0.0), p.discount);
    const double r = p.rewards[b];
    for (int j = tid; j < N; j += kQrThreads) {
        const float t = __double2float_rn(__dadd_rn(r, __dmul_rn(coef, (double)p.next[row + (int64_t)best * N + j])));
        s_t[j] = t;
        if (p.targets) p.targets[(int64_t)b * N + j] = t;
        // tau_hat_k = 0.5 * (c[k + 1] + c[k]), c = arange(N + 1) / N in fp64
        const int k = s_sigma[j];
        const double mid = __dmul_rn(0.5, __dadd_rn(__ddiv_rn((double)(k + 1), (double)N),
                                                    __ddiv_rn((double)k, (double)N)));
        s_tau[j] = __double2float_rn(mid);
        if (p.taus && valid) p.taus[(int64_t)b * N + j] = s_tau[j];
    }
    __syncthreads();
    // ---- pair terms: thread i owns theta_i and sums over j in order ---------------------------------------------------
    const float kappa = p.kappa;
    const double inv_n = __ddiv_rn(1.0, (double)N);
    float loss = 0.f;
    for (int i = tid; i < N; i += kQrThreads) {
        const float th = s_theta[i], tau = s_tau[i];
        float li = 0.f;
        double gi = 0.0;                       // the gradient's j-sum cancels: accumulated in fp64, rounded once
        for (int j = 0; j < N; ++j) {
            const float e = __fsub_rn(s_t[j], th);
            const float ae = fabsf(e);
            const float q = fminf(ae, kappa);
            const float h = __fadd_rn(__fmul_rn(kappa, __fsub_rn(ae, q)), __fmul_rn(0.5f, __fmul_rn(q, q)));
            const float w = fabsf(__fsub_rn(tau, e < 0.f ? 1.0f : 0.0f));
            li = __fadd_rn(li, __fmul_rn(w, h));
            gi = __dadd_rn(gi, (double)__fmul_rn(w, fminf(fmaxf(e, -kappa), kappa)));
        }
        loss = __fadd_rn(loss, li);
        s_g[i] = valid ? __double2float_rn(__dmul_rn(-gi, inv_n)) : 0.f;
    }
    const float total = block_sum(valid ? loss : 0.f, red);                     // (its barriers also publish s_g)
    if (tid == 0) p.partial[b] = total;
    // ---- d loss / d quantiles: the taken row, 0 on every other action --------------------------------------------------
    for (int k = tid; k < A * N; k += kQrThreads) {
        const int a = k / N;
        p.dq[row + k] = (valid && a == act) ? s_g[k - a * N] : 0.f;
    }
}

// loss = (sum_b partial[b]) / N: one block, the strided per-thread sums and the tree of block_sum
__global__ void __launch_bounds__(256) qr_loss_kernel(const float* __restrict__ partial, int B, int N,
                                                      float* __restrict__ loss) {
    __shared__ float red[256];
    float v = 0.f;
    for (int b = threadIdx.x; b < B; b += 256) v = __fadd_rn(v, partial[b]);
    const float s = block_sum(v, red);
    if (threadIdx.x == 0) *loss = __fdiv_rn(s, (float)N);
}

// q_values of the QuantileRegressionQHead for acting, one warp per (b, a) row
__global__ void __launch_bounds__(128) qr_q_values_kernel(const float* __restrict__ quantiles, int64_t rows, int N,
                                                          double* __restrict__ q) {
    const int64_t r = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const double v = qr_row_q(quantiles + r * N, N, lane);
    if (lane == 0) q[r] = v;
}

// =====================================================================================================================
// PPOHead with the KL penalty instead of clipping (heads/ppo_head.py:64-97 with clip_likelihood_ratio_using_epsilon
// None): per minibatch of B rows
//   KLbar = mean_i KL_i(old || new),   ratio_i = exp(logp_i - logp_old_i)
//   L     = -mean_i ratio_i * A_i  +  use_kl * (k * KLbar + c * max(0, KLbar - cutoff)^2)  -  beta * H
// so every row's gradient depends on KLbar through f = k + 2 c max(0, KLbar - cutoff):
//   dL/dmu_ij     = (-A_i ratio_i z_ij + f dm_ij) / (B sigma_j),              z = (a - mu) / sigma, dm = (mu - mu_old) / sigma
//   dL/dlogstd_j  = [sum_i (-A_i ratio_i (z_ij^2 - 1) + f (1 - rs_j^2 - dm_ij^2)) / B - beta] (sigma_j - eps) / sigma_j,
//                   rs = sigma_old / sigma
// One CTA.  A warp owns a row at a time, lane j its dimension j (A <= 32), so the per-row sums are xor-shuffle trees
// whose result every lane holds bit for bit.  Pass 1 forms KLbar, pass 2 the gradients and the logged scalars.  Each
// warp accumulates its rows in order and the warps' partials are summed in warp order: no atomics, so repeat calls and
// graph replays give identical bits.  k is read from device memory so a captured graph follows coefficient updates.
// =====================================================================================================================
constexpr int kPpoKlThreads = 1024;
constexpr int kPpoKlWarps = kPpoKlThreads / 32;

__global__ void __launch_bounds__(kPpoKlThreads) ppo_kl_head_kernel(
    const float* __restrict__ mu, const float* __restrict__ logstd, const float* __restrict__ actions,
    const float* __restrict__ old_mu, const float* __restrict__ old_logstd, const float* __restrict__ advantages,
    int64_t B, int A, const float* __restrict__ kl_coef, float kl_cutoff, float high_kl_penalty, int use_kl,
    float beta_entropy, float* __restrict__ d_mu, float* __restrict__ d_logstd,
    float* __restrict__ scalars /* [loss, KLbar, entropy, mean ratio, surrogate] */) {
    __shared__ float dls_part[kPpoKlWarps][kMaxActionDim];
    __shared__ float row_part[3][kPpoKlWarps];          // per warp: KL, ratio, ratio * advantage
    __shared__ float kl_mean_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool on = lane < A;
    const float sig = on ? ppo_sigma(logstd[lane]) : 1.f;
    const float osig = on ? ppo_sigma(old_logstd[lane]) : 1.f;
    const float sum_log_sig = warp_sum(on ? logf(sig) : 0.f);
    const float sum_log_osig = warp_sum(on ? logf(osig) : 0.f);
    const float inv_b = 1.0f / (float)B;

    float kl_acc = 0.f;
    for (int64_t i = warp; i < B; i += kPpoKlWarps) {
        const float t = on ? ppo_kl_term(mu[i * A + lane], old_mu[i * A + lane], sig, osig) : 0.f;
        kl_acc += warp_sum(t);
    }
    if (lane == 0) row_part[0][warp] = kl_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kPpoKlWarps; ++w) s += row_part[0][w];
        kl_mean_s = s * inv_b;
    }
    __syncthreads();
    const float kl_mean = kl_mean_s;
    const float excess = fmaxf(0.f, kl_mean - kl_cutoff);
    const float coef = use_kl ? *kl_coef : 0.f;
    const float f_over_b = use_kl ? (coef + 2.0f * high_kl_penalty * excess) * inv_b : 0.f;

    float dls = 0.f, ratio_acc = 0.f, surr_acc = 0.f;
    for (int64_t i = warp; i < B; i += kPpoKlWarps) {
        float z = 0.f, zo = 0.f, dm = 0.f;
        if (on) {
            const float a = actions[i * A + lane], m = mu[i * A + lane], om = old_mu[i * A + lane];
            z = (a - m) / sig;
            zo = (a - om) / osig;
            dm = (m - om) / sig;
        }
        const float q = warp_sum(z * z), qo = warp_sum(zo * zo);
        const float ratio = expf(ppo_logp(q, sum_log_sig, A) - ppo_logp(qo, sum_log_osig, A));
        const float adv = advantages[i];
        ratio_acc += ratio;
        surr_acc += ratio * adv;
        const float dlogp = -inv_b * adv * ratio;          // dL/dlogp_i
        if (on) {
            const float rs = osig / sig;
            d_mu[i * A + lane] = (dlogp * z + f_over_b * dm) / sig;
            dls += dlogp * (z * z - 1.0f) + f_over_b * (1.0f - rs * rs - dm * dm);
        }
    }
    if (on) dls_part[warp][lane] = dls;
    if (lane == 0) {
        row_part[1][warp] = ratio_acc;
        row_part[2][warp] = surr_acc;
    }
    __syncthreads();
    if (threadIdx.x < A) {
        float s = 0.f;
        for (int w = 0; w < kPpoKlWarps; ++w) s += dls_part[w][threadIdx.x];
        const float ds = ppo_dsig(sig);
        d_logstd[threadIdx.x] = s * ds - beta_entropy * ds;
    }
    if (threadIdx.x == 0 && scalars) {
        float r = 0.f, sa = 0.f;
        for (int w = 0; w < kPpoKlWarps; ++w) {
            r += row_part[1][w];
            sa += row_part[2][w];
        }
        const float entropy = ppo_entropy(A, sum_log_sig);
        const float surrogate = -sa * inv_b;
        const float penalty = use_kl ? coef * kl_mean + high_kl_penalty * excess * excess : 0.f;
        scalars[0] = surrogate + penalty - beta_entropy * entropy;
        scalars[1] = kl_mean;
        scalars[2] = entropy;
        scalars[3] = r * inv_b;
        scalars[4] = surrogate;
    }
}

// AdditiveNoise.get_action([mean, std]) (exploration_policies/additive_noise.py:84-103) for the PPO actor:
// std = exp(logstd) (the head's policy_std output, no eps); actions = (double) mean + (double) std * n, one multiply
// and one add each rounded on its own, which is numpy's normal(mean, std) on the draws n.
__global__ void __launch_bounds__(256) ppo_gaussian_act_kernel(const float* __restrict__ mean,
                                                               const float* __restrict__ logstd, int64_t n, int A,
                                                               const double* __restrict__ normals,
                                                               double* __restrict__ actions, float* __restrict__ stds) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const float std = expf(logstd[k % A]);
        if (stds) stds[k] = std;
        if (normals) actions[k] = __dadd_rn((double)mean[k], __dmul_rn((double)std, normals[k]));
    }
}

// =====================================================================================================================
// PPOHead, discrete actions, clipped surrogate (heads/ppo_head.py:52-116).  TF 1.x's Categorical(probs = p) takes
// logits = log p, so per row i, with p = softmax(z_i) and q_i the old policy's probabilities:
//   log pi_j   = log_softmax(log p)_j = z_j - max z - log sum exp(z - max z)
//   log pio_j  = log_softmax(log q)_j
//   H_i        = -sum_j p_j log pi_j,   KL_i = sum_j softmax(log q)_j (log pio_j - log pi_j)  (0 where that weight is 0)
//   ratio_i    = exp(log pi_a - log pio_a),  clipped to 1 -+ e,  e = fl32(clip_eps * rescaler)
//   L          = -mean_i min(ratio_i A_i, clip(ratio_i) A_i)  -  beta * mean_i H_i
//   dL/dz_ij   = -(1/B) dmin/dratio_i ratio_i (onehot(a_i)_j - p_j)  +  (beta/B) p_j (log pi_j + H_i)
// A row whose action lies outside [0, A) has no surrogate term (nothing in the loss, ratio sums or gradient from it).
// One CTA.  A warp owns a row at a time and lane j its action j (A <= 32); the per-row sums are xor-shuffle trees, so
// every lane holds them bit for bit.  Each warp accumulates its rows in order and the warps' partials are summed in
// warp order: no atomics, repeat calls and graph replays give identical bits.  The rescaler is read from device
// memory so a captured graph follows a clipping schedule.
// =====================================================================================================================
constexpr int kPpoCatThreads = 1024;
constexpr int kPpoCatWarps = kPpoCatThreads / 32;

__global__ void __launch_bounds__(kPpoCatThreads) ppo_categorical_head_kernel(
    const float* __restrict__ logits, const int64_t* __restrict__ actions, const float* __restrict__ old_probs,
    const float* __restrict__ advantages, int64_t B, int A, float clip_eps, const float* __restrict__ clip_rescaler,
    float beta_entropy, float* __restrict__ d_logits,
    float* __restrict__ scalars /* [loss, KL(old||new), entropy, mean ratio, mean clipped ratio] */) {
    __shared__ float part[5][kPpoCatWarps];              // per warp: surrogate min, KL, entropy, ratio, clipped ratio
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool on = lane < A;
    const float inv_b = 1.0f / (float)B;
    const float e = __fmul_rn(clip_eps, *clip_rescaler);      // TF: 1 +- eps * rescaler, the product in fp32
    const float lo = 1.0f - e, hi = 1.0f + e;
    const float ent_w = beta_entropy * inv_b;
    float surr_acc = 0.f, kl_acc = 0.f, ent_acc = 0.f, ratio_acc = 0.f, cratio_acc = 0.f;
    for (int64_t i = warp; i < B; i += kPpoCatWarps) {
        const float z = on ? logits[i * A + lane] : -INFINITY;
        const float m = warp_max(z);
        const float ez = on ? expf(z - m) : 0.f;
        const float s = warp_sum(ez);
        const float p = ez / s;
        const float lp = on ? (z - m) - logf(s) : 0.f;
        const float lq = on ? logf(old_probs[i * A + lane]) : -INFINITY;
        const float mq = warp_max(lq);
        const float eq = on ? expf(lq - mq) : 0.f;
        const float sq = warp_sum(eq);
        const float qn = eq / sq;
        const float lpo = on ? (lq - mq) - logf(sq) : 0.f;
        const float H = -warp_sum(on ? p * lp : 0.f);
        kl_acc += warp_sum(qn > 0.f ? qn * (lpo - lp) : 0.f);
        ent_acc += H;
        const int64_t a = actions[i];
        const bool valid = a >= 0 && a < A;
        const int ai = valid ? (int)a : 0;
        const float lp_a = __shfl_sync(0xffffffffu, lp, ai), lpo_a = __shfl_sync(0xffffffffu, lpo, ai);
        float dlogp = 0.f;                                    // dL/dlog pi_a
        if (valid) {
            const float ratio = expf(lp_a - lpo_a);
            const float cl = fminf(fmaxf(ratio, lo), hi);
            const float adv = advantages[i];
            const float s1 = ratio * adv, s2 = cl * adv;
            // tf.minimum passes the gradient to its first argument when s1 <= s2; clip_by_value passes it inside
            // [lo, hi]
            float ds_dratio;
            if (s1 <= s2) ds_dratio = adv;
            else ds_dratio = (ratio >= lo && ratio <= hi) ? adv : 0.f;
            surr_acc += fminf(s1, s2);
            ratio_acc += ratio;
            cratio_acc += cl;
            dlogp = -inv_b * ds_dratio * ratio;
        }
        if (on) {
            const float onehot = (valid && lane == ai) ? 1.f : 0.f;
            d_logits[i * A + lane] = dlogp * (onehot - p) + ent_w * p * (lp + H);
        }
    }
    if (lane == 0) {
        part[0][warp] = surr_acc;
        part[1][warp] = kl_acc;
        part[2][warp] = ent_acc;
        part[3][warp] = ratio_acc;
        part[4][warp] = cratio_acc;
    }
    __syncthreads();
    if (threadIdx.x == 0 && scalars) {
        float t[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        for (int w = 0; w < kPpoCatWarps; ++w)
            for (int k = 0; k < 5; ++k) t[k] += part[k][w];
        const float entropy = t[2] * inv_b;
        scalars[0] = -t[0] * inv_b - beta_entropy * entropy;
        scalars[1] = t[1] * inv_b;
        scalars[2] = entropy;
        scalars[3] = t[3] * inv_b;
        scalars[4] = t[4] * inv_b;
    }
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_naf_head(const cb200_naf_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->n_actions >= 1 && d->n_actions <= kMaxActionDim, "1 <= n_actions <= 32");
    CB200_CHECK_ARG(d->batch > 0 && d->batch <= (int64_t)0x7fffffff * kNafWarps, "bad batch");
    CB200_CHECK_ARG(d->z_mu && d->scale && d->mu, "null pointer (z_mu, scale, mu)");
    CB200_CHECK_ARG(!d->actions == !d->targets, "actions and targets are both given (training) or both NULL (acting)");
    const bool train = d->actions != nullptr;
    CB200_CHECK_ARG(!(train || d->q) || d->z_v, "q needs z_v");
    CB200_CHECK_ARG(!train || (d->l && d->q && d->loss && d->d_zv && d->d_zmu && d->d_l),
                    "training needs l, q, loss, d_zv, d_zmu and d_l");
    const int A = d->n_actions;
    CB200_CHECK_ARG(d->ld_mu >= A && (!train || (d->ld_l >= A * (A + 1) / 2 && d->ld_actions >= A)),
                    "leading dimensions below the row widths");
    NafParams p;
    p.z_v = d->z_v; p.z_mu = d->z_mu; p.l = d->l; p.scale = d->scale; p.actions = d->actions; p.targets = d->targets;
    p.huber = d->huber; p.A = A; p.ld_mu = d->ld_mu; p.ld_l = d->ld_l; p.ld_u = d->ld_actions; p.B = d->batch;
    p.mu = d->mu; p.q = d->q; p.d_zv = d->d_zv; p.d_zmu = d->d_zmu; p.d_l = d->d_l; p.adv = d->adv;
    const unsigned grid = (unsigned)((d->batch + kNafWarps - 1) / kNafWarps);
    cudaStream_t st = as_stream(stream);
    if (train) {
        CB200_LAUNCH(naf_head_kernel<true>, grid, kNafWarps * 32, 0, st, p);
        CB200_LAUNCH(naf_loss_kernel, 1, 256, 0, st, d->q, d->targets, d->batch, d->huber, d->loss);
    } else {
        CB200_LAUNCH(naf_head_kernel<false>, grid, kNafWarps * 32, 0, st, p);
    }
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_qr_head(const cb200_qr_head_desc* d, void* stream) {
    CB200_CHECK_ARG(d != nullptr, "null descriptor");
    CB200_CHECK_ARG(d->n_atoms >= 1 && d->n_atoms <= kQrMaxAtoms, "1 <= n_atoms <= 1024");
    CB200_CHECK_ARG(d->n_actions >= 1 && d->n_actions <= kQrMaxActions, "1 <= n_actions <= 256");
    CB200_CHECK_ARG(d->batch >= 1, "batch >= 1");
    CB200_CHECK_ARG(d->kappa >= 0.f && d->kappa <= INFINITY, "huber_loss_interval >= 0");
    CB200_CHECK_ARG(d->next && d->online && d->actions && d->rewards && d->game_overs,
                    "null input (next, online, actions, rewards, game_overs)");
    CB200_CHECK_ARG(d->dq && d->loss && d->workspace, "null output (dq, loss, workspace)");
    QrParams p;
    p.next = d->next; p.online = d->online; p.actions = d->actions; p.rewards = d->rewards;
    p.game_overs = d->game_overs; p.discount = d->discount; p.kappa = d->kappa;
    p.B = d->batch; p.A = d->n_actions; p.N = d->n_atoms;
    p.dq = d->dq; p.targets = d->targets; p.taus = d->taus; p.target_actions = d->target_actions;
    p.partial = d->workspace;
    cudaStream_t st = as_stream(stream);
    CB200_LAUNCH(qr_head_kernel, (unsigned)d->batch, kQrThreads, 0, st, p);
    CB200_CHECK_LAUNCH();
    CB200_LAUNCH(qr_loss_kernel, 1, 256, 0, st, d->workspace, d->batch, d->n_atoms, d->loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_qr_q_values(const float* quantiles, int64_t rows, int32_t n_atoms, double* q_out, void* stream) {
    CB200_CHECK_ARG(quantiles && q_out && rows > 0 && n_atoms >= 1 && n_atoms <= kQrMaxAtoms, "bad arguments");
    CB200_LAUNCH(qr_q_values_kernel, (unsigned)((rows + 3) / 4), 128, 0, as_stream(stream), quantiles, rows, n_atoms,
                 q_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ppo_continuous_head(const float* mu, const float* logstd, const float* actions, const float* old_mu,
                              const float* old_logstd, const float* advantages, int64_t batch, int32_t action_dim,
                              float clip_eps, float beta_entropy, float* d_mu, float* d_logstd, float* scalars,
                              void* stream) {
    CB200_CHECK_ARG(mu && logstd && actions && old_mu && old_logstd && advantages && d_mu && d_logstd, "null pointer");
    CB200_CHECK_ARG(batch > 0 && action_dim > 0 && action_dim <= kMaxActionDim, "bad shape (action_dim <= 32)");
    CB200_LAUNCH(ppo_continuous_head_kernel, 1, 256, 0, as_stream(stream), mu, logstd, actions, old_mu, old_logstd,
                 advantages, batch, action_dim, clip_eps, beta_entropy, d_mu, d_logstd, scalars);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ppo_kl_head(const float* mu, const float* logstd, const float* actions, const float* old_mu,
                      const float* old_logstd, const float* advantages, int64_t batch, int32_t action_dim,
                      const float* kl_coef, float kl_cutoff, float high_kl_penalty, int32_t use_kl, float beta_entropy,
                      float* d_mu, float* d_logstd, float* scalars, void* stream) {
    CB200_CHECK_ARG(mu && logstd && actions && old_mu && old_logstd && advantages && d_mu && d_logstd, "null pointer");
    CB200_CHECK_ARG(batch > 0 && action_dim > 0 && action_dim <= kMaxActionDim, "bad shape (action_dim <= 32)");
    CB200_CHECK_ARG(!use_kl || kl_coef, "use_kl needs the device KL coefficient");
    CB200_LAUNCH(ppo_kl_head_kernel, 1, kPpoKlThreads, 0, as_stream(stream), mu, logstd, actions, old_mu, old_logstd,
                 advantages, batch, action_dim, kl_coef, kl_cutoff, high_kl_penalty, use_kl ? 1 : 0, beta_entropy,
                 d_mu, d_logstd, scalars);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ppo_categorical_head(const float* logits, const int64_t* actions, const float* old_probs,
                               const float* advantages, int64_t batch, int32_t n_actions, float clip_eps,
                               const float* clip_rescaler, float beta_entropy, float* d_logits, float* scalars,
                               void* stream) {
    CB200_CHECK_ARG(logits && actions && old_probs && advantages && clip_rescaler && d_logits, "null pointer");
    CB200_CHECK_ARG(batch > 0 && n_actions > 0 && n_actions <= kMaxActionDim, "bad shape (1 <= n_actions <= 32)");
    CB200_LAUNCH(ppo_categorical_head_kernel, 1, kPpoCatThreads, 0, as_stream(stream), logits, actions, old_probs,
                 advantages, batch, n_actions, clip_eps, clip_rescaler, beta_entropy, d_logits, scalars);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ppo_gaussian_act(const float* mean, const float* logstd, int64_t envs, int32_t action_dim,
                           const double* normals, double* actions, float* stds, void* stream) {
    CB200_CHECK_ARG(mean && logstd && envs > 0 && action_dim > 0 && action_dim <= kMaxActionDim, "bad arguments");
    CB200_CHECK_ARG(!normals || actions, "normals need actions");
    const int64_t n = envs * action_dim;
    int64_t grid = (n + 255) / 256;
    if (grid > (int64_t)sm_count() * 8) grid = (int64_t)sm_count() * 8;
    CB200_LAUNCH(ppo_gaussian_act_kernel, (unsigned)grid, 256, 0, as_stream(stream), mean, logstd, n, action_dim,
                 normals, actions, stds);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_gather_at(const cb200_column* h_columns, int n_columns, const int64_t* idx, const int64_t* offset,
                    int64_t n, void* stream) {
    CB200_CHECK_ARG(h_columns && n_columns > 0 && n_columns <= CB200_MAX_COLUMNS && n > 0, "bad arguments");
    AtColumns cols;
    cols.n = n_columns;
    for (int c = 0; c < n_columns; ++c) {
        CB200_CHECK_ARG(h_columns[c].src && h_columns[c].dst && h_columns[c].row_bytes > 0, "bad column entry");
        cols.src[c] = static_cast<const uint8_t*>(h_columns[c].src);
        cols.dst[c] = static_cast<uint8_t*>(h_columns[c].dst);
        cols.row_bytes[c] = h_columns[c].row_bytes;
    }
    int64_t grid = (n * n_columns + 7) / 8;
    if (grid > (int64_t)sm_count() * 8) grid = (int64_t)sm_count() * 8;
    CB200_LAUNCH(gather_at_kernel, (unsigned)grid, 256, 0, as_stream(stream), cols, idx, offset, n);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}


int cb200_act_backward(const float* dy, int32_t ld_dy, const float* y, int32_t ld_y, int64_t rows, int32_t cols,
                       int32_t act, float* dz, int32_t ld_dz, void* stream) {
    CB200_CHECK_ARG(dy && y && dz && rows > 0 && cols > 0 && ld_dy >= cols && ld_y >= cols && ld_dz >= cols,
                    "bad arguments");
    const int64_t n = rows * cols;
    CB200_LAUNCH(act_backward_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), dy, ld_dy, y, ld_y, rows,
                 cols, act, dz, ld_dz);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_axpby_2d(const float* src, int32_t ld_src, int64_t rows, int32_t cols, float alpha, float beta, float* dst,
                   int32_t ld_dst, void* stream) {
    CB200_CHECK_ARG(src && dst && rows > 0 && cols > 0 && ld_src >= cols && ld_dst >= cols, "bad arguments");
    const int64_t n = rows * cols;
    CB200_LAUNCH(axpby_2d_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), src, ld_src, rows, cols,
                 alpha, beta, dst, ld_dst);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_ac_td_targets(const double* rewards, const uint8_t* game_overs, const float* q_next, int32_t ld_q,
                        int64_t batch, double discount, int32_t use_non_zero_discount_for_terminal_states,
                        int32_t use_clip, double clip_lo, double clip_hi, float* targets_out, void* stream) {
    CB200_CHECK_ARG(rewards && game_overs && q_next && targets_out && batch > 0 && ld_q >= 1, "bad arguments");
    CB200_LAUNCH(ac_td_targets_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), rewards, game_overs,
                 q_next, ld_q, batch, discount, use_non_zero_discount_for_terminal_states, use_clip, clip_lo, clip_hi,
                 targets_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_min2(const float* a, const float* b, int64_t n, float* out, void* stream) {
    CB200_CHECK_ARG(a && b && out && n > 0, "bad arguments");
    CB200_LAUNCH(min2_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), a, b, n, out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_td3_smooth_actions(float* actions, const double* noise, int64_t n, double noise_clip, double lo, double hi,
                             void* stream) {
    CB200_CHECK_ARG(actions && noise && n > 0, "bad arguments");
    CB200_LAUNCH(td3_smooth_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), actions, noise, n,
                 noise_clip, lo, hi);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}


int cb200_c51_head(const float* next, const float* online, const float* select, const int64_t* actions,
                   const double* rewards, const uint8_t* game_overs, const double* bootstrap, const double* z,
                   double gamma_n, int32_t batch, int32_t n_actions, int32_t n_atoms, int32_t next_is_prob,
                   float* labels, float* dlogits, float* loss_rows, float* total_loss, double* td_err,
                   double* q_online, int64_t* target_actions, void* stream) {
    CB200_CHECK_ARG(next && online && actions && rewards && (game_overs || bootstrap) && z, "bad arguments");
    CB200_CHECK_ARG(labels && dlogits && loss_rows && total_loss && td_err, "bad output arguments");
    CB200_CHECK_ARG(batch > 0 && n_actions > 0 && n_atoms >= 2 && n_atoms <= 1024, "bad shape");
    C51Params p;
    p.next = next; p.online = online; p.select = select; p.actions = actions; p.rewards = rewards;
    p.game_overs = game_overs; p.bootstrap = bootstrap; p.z = z; p.gamma_n = gamma_n;
    p.B = batch; p.A = n_actions; p.N = n_atoms; p.next_is_prob = next_is_prob;
    p.labels = labels; p.dlogits = dlogits; p.loss_rows = loss_rows; p.td_err = td_err; p.q_online = q_online;
    p.target_actions = target_actions;
    const size_t smem = (size_t)kC51Warps * n_atoms * (sizeof(double) + 2 * sizeof(float));
    // above 768 atoms the kernel needs more than the 48 KB default (64 KB at 1024): opted into once per device
    if (smem > 48 * 1024) {
        static bool attr_set[kMaxDevices] = {};
        int dev = 0;
        CB200_CUDA(cudaGetDevice(&dev));
        CB200_CHECK_ARG(dev < kMaxDevices, "device ordinal out of range");
        if (!attr_set[dev]) {
            CB200_CUDA(cudaFuncSetAttribute(c51_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            kC51Warps * 1024 * (int)(sizeof(double) + 2 * sizeof(float))));
            attr_set[dev] = true;
        }
    }
    CB200_LAUNCH(c51_head_kernel, (unsigned)((batch + kC51Warps - 1) / kC51Warps), kC51Warps * 32, smem,
                 as_stream(stream), p);
    CB200_CHECK_LAUNCH();
    CB200_LAUNCH(c51_loss_sum_kernel, 1, 256, 0, as_stream(stream), loss_rows, (int64_t)batch * n_actions, total_loss);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}


int cb200_c51_q_values(const float* logits, const double* z, int64_t rows, int32_t n_atoms, double* q_out, void* stream) {
    CB200_CHECK_ARG(logits && z && q_out && rows > 0 && n_atoms >= 2, "bad arguments");
    CB200_LAUNCH(c51_q_values_kernel, (unsigned)((rows + 3) / 4), 128, 0, as_stream(stream), logits, z, rows, n_atoms,
                 q_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_sac_policy_sample(const float* head_out, const float* eps, int64_t batch, int32_t action_dim, float* raw_out,
                            float* actions_out, float* logp_out, void* stream) {
    CB200_CHECK_ARG(head_out && eps && batch > 0 && action_dim > 0, "bad arguments");
    CB200_LAUNCH(sac_policy_sample_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), head_out, eps,
                 batch, action_dim, raw_out, actions_out, logp_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_sac_policy_grad(const float* head_out, const float* eps_logp, const float* eps_q, const float* dq_da,
                          int64_t batch, int32_t action_dim, float* d_head_out, void* stream) {
    CB200_CHECK_ARG(head_out && eps_logp && eps_q && dq_da && d_head_out && batch > 0 && action_dim > 0,
                    "bad arguments");
    CB200_LAUNCH(sac_policy_grad_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), head_out, eps_logp,
                 eps_q, dq_da, batch, action_dim, d_head_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_sac_min_seed(const float* q1, const float* q2, int64_t batch, float* d1, float* d2, float* qmin,
                       void* stream) {
    CB200_CHECK_ARG(q1 && q2 && batch > 0, "bad arguments");
    CB200_LAUNCH(sac_min_seed_kernel, (unsigned)((batch + 255) / 256), 256, 0, as_stream(stream), q1, q2, batch, d1, d2,
                 qmin);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_sub(const float* a, const float* b, int64_t n, float* out, void* stream) {
    CB200_CHECK_ARG(a && b && out && n > 0, "bad arguments");
    CB200_LAUNCH(sub_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), a, b, n, out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_f64_to_f32(const double* in, int64_t n, float* out, void* stream) {
    CB200_CHECK_ARG(in && out && n > 0, "bad arguments");
    CB200_LAUNCH(f64_to_f32_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), in, n, out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

}  // extern "C"
