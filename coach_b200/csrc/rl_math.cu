// coach_b200/csrc/rl_math.cu -- scalar RL recurrences of the path on the GPU: GAE scan, n-step returns, running
// observation statistics + normalisation.  Reference lines are cited in include/coach_b200.h.
#include <math.h>

#include "common.cuh"

namespace cb200 {

// =====================================================================================================================
// GAE: A_t = delta_t + c_t * A_{t+1} over the whole rollout, with
//   delta_t = r_t + gamma * (1 - done_t) * V_{t+1} - V_t      (bootstrap value 0 at every episode end,
//   c_t     = gamma * lambda * (1 - done_t)                     clipped_ppo_agent.py:188)
// i.e. one first-order linear recurrence with per-element coefficients.  An affine map y -> a*y + b composes
// associatively, so the reverse recurrence is a block-wide scan of (a, b) pairs: each thread folds its contiguous
// chunk, a warp-shuffle scan combines the 32 lanes, a shared-memory pass combines the warps, and each thread then
// replays its chunk with the proper carry-in.  fp64 throughout (the reference computes in fp64).
// =====================================================================================================================
struct Affine {
    double a, b;   // y_out = a * y_in + b     (y_in = value coming from the right / later time steps)
};
__device__ __forceinline__ Affine compose(const Affine& left, const Affine& right) {
    // apply `right` first (later in time), then `left`:  left(right(y)) = left.a*(right.a*y + right.b) + left.b
    Affine r;
    r.a = left.a * right.a;
    r.b = left.a * right.b + left.b;
    return r;
}

constexpr int kGaeThreads = 1024;

__global__ void __launch_bounds__(kGaeThreads) gae_scan_kernel(const double* __restrict__ rewards,
                                                                const float* __restrict__ values,
                                                                const uint8_t* __restrict__ dones, int64_t n,
                                                                double gamma, double lambda,
                                                                double* __restrict__ adv, double* __restrict__ tgt,
                                                                int64_t* __restrict__ n_valid_out) {
    __shared__ Affine warp_tot[32];
    __shared__ long long last_done_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t per = (n + kGaeThreads - 1) / kGaeThreads;
    const int64_t lo = (int64_t)tid * per, hi = min(n, lo + per);
    if (tid == 0) last_done_s = -1;
    __syncthreads();
    const double gl = gamma * lambda;
    // pass 1: fold the chunk (reverse order) into one affine map; remember the last done flag
    Affine f{1.0, 0.0};
    long long my_last = -1;
    for (int64_t t = hi - 1; t >= lo; --t) {
        const double nd = dones[t] ? 0.0 : 1.0;
        if (dones[t] && my_last < 0) my_last = t;
        const double vnext = (t + 1 < n) ? (double)values[t + 1] : 0.0;
        const double delta = rewards[t] + gamma * nd * vnext - (double)values[t];
        Affine e{gl * nd, delta};
        f = compose(e, f);            // e is earlier in time than everything folded so far
    }
    if (my_last >= 0) atomicMax(&last_done_s, my_last);
    // reverse exclusive scan across threads: carry-in of thread i = composition of threads i+1 .. T-1 applied to 0
    // warp level (inclusive, reverse): after the loop `s` = f_i o f_{i+1} o ... o f_{warp end}
    Affine s = f;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        Affine o;
        o.a = __shfl_down_sync(0xffffffffu, s.a, off);
        o.b = __shfl_down_sync(0xffffffffu, s.b, off);
        if (lane + off < 32) s = compose(s, o);
    }
    if (lane == 0) warp_tot[warp] = s;
    __syncthreads();
    // carry from later warps
    Affine later{1.0, 0.0};
    for (int w = 31; w > warp; --w) later = compose(warp_tot[w], later);
    // exclusive within the warp: what lanes > lane produced
    Affine ex;
    ex.a = __shfl_down_sync(0xffffffffu, s.a, 1);
    ex.b = __shfl_down_sync(0xffffffffu, s.b, 1);
    if (lane == 31) ex = Affine{1.0, 0.0};
    const Affine carry = compose(ex, later);
    double y = carry.b;               // value of A at index hi (input to this chunk); carry applied to 0
    // pass 2: replay the chunk
    for (int64_t t = hi - 1; t >= lo; --t) {
        const double nd = dones[t] ? 0.0 : 1.0;
        const double vnext = (t + 1 < n) ? (double)values[t + 1] : 0.0;
        const double delta = rewards[t] + gamma * nd * vnext - (double)values[t];
        y = delta + gl * nd * y;
        adv[t] = y;
        tgt[t] = y + (double)values[t];      // estimate_state_value_using_gae: A + V[:-1] (actor_critic_agent.py:121)
    }
    __syncthreads();
    if (tid == 0 && n_valid_out) *n_valid_out = last_done_s + 1;   // transitions after the last done get nothing
}

// (x - mean) / std with the POPULATION std over the first n_valid entries (clipped_ppo_agent.py:201), in place;
// entries >= n_valid are set to NaN (the reference leaves them unset).  One block, fixed-order reductions.
__global__ void __launch_bounds__(1024) standardize_kernel(double* __restrict__ x, int64_t n,
                                                           const int64_t* __restrict__ n_valid_ptr,
                                                           double* __restrict__ mean_std_out) {
    __shared__ double red[1024];
    const int tid = threadIdx.x;
    const int64_t nv = n_valid_ptr ? min(n, *n_valid_ptr) : n;
    double s = 0.0;
    for (int64_t i = tid; i < nv; i += blockDim.x) s += x[i];
    red[tid] = s;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (tid < k) red[tid] += red[tid + k];
        __syncthreads();
    }
    const double mean = nv > 0 ? red[0] / (double)nv : 0.0;
    __syncthreads();
    s = 0.0;
    for (int64_t i = tid; i < nv; i += blockDim.x) {
        const double d = x[i] - mean;
        s += d * d;
    }
    red[tid] = s;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (tid < k) red[tid] += red[tid + k];
        __syncthreads();
    }
    const double sd = nv > 0 ? sqrt(red[0] / (double)nv) : 1.0;
    for (int64_t i = tid; i < n; i += blockDim.x) x[i] = (i < nv) ? (x[i] - mean) / sd : nan("");
    if (tid == 0 && mean_std_out) {
        mean_std_out[0] = mean;
        mean_std_out[1] = sd;
    }
}

// =====================================================================================================================
// n-step discounted returns, Episode.update_discounted_rewards (core_types.py:771-790):
//   out = r;  cur = g;  for i in 1..n-1: out += cur * shift(r, i);  cur *= g
// evaluated per element with exactly that operation order (explicit round-to-nearest ops, no FMA) => bit-identical to
// the numpy loop.  `ep_end[t]` = index one past the last transition of t's episode.
// =====================================================================================================================
__global__ void __launch_bounds__(256) nstep_kernel(const double* __restrict__ rewards,
                                                    const int64_t* __restrict__ ep_start,
                                                    const int64_t* __restrict__ ep_end, int64_t n, double discount,
                                                    int64_t n_step, double* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int64_t end = ep_end[t], len = end - ep_start[t];
    const int64_t cur_n = (n_step == -1 || n_step > len) ? len : n_step;
    double acc = rewards[t];
    double cur = discount;
    for (int64_t i = 1; i < cur_n; ++i) {
        const double r = (t + i < end) ? rewards[t + i] : 0.0;          // np.pad(..., constant 0)
        acc = __dadd_rn(acc, __dmul_rn(cur, r));
        cur = __dmul_rn(cur, discount);
    }
    out[t] = acc;
}

// =====================================================================================================================
// Running observation statistics (NumpySharedRunningStats, utilities/shared_running_stats.py:115-164)
// =====================================================================================================================
// column sums of x and x^2 in fp64, one block per feature, fixed order; accumulates into sum / sumsq
__global__ void __launch_bounds__(256) stats_push_kernel(const float* __restrict__ x, int64_t rows, int64_t cols,
                                                         double* __restrict__ sum, double* __restrict__ sumsq) {
    __shared__ double r1[256], r2[256];
    const int64_t c = blockIdx.x;
    double s = 0.0, q = 0.0;
    for (int64_t r = threadIdx.x; r < rows; r += blockDim.x) {
        const double v = (double)x[r * cols + c];
        s += v;
        q += v * v;
    }
    r1[threadIdx.x] = s;
    r2[threadIdx.x] = q;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) {
            r1[threadIdx.x] += r1[threadIdx.x + k];
            r2[threadIdx.x] += r2[threadIdx.x + k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        sum[c] += r1[0];
        sumsq[c] += r2[0];
    }
}
// mean = sum / count; std = sqrt(max((sumsq - count*mean^2) / max(count-1, 1), eps))   (:136-140), each operation
// rounded on its own like numpy's (explicit _rn: nvcc would otherwise fuse count*mean^2 into the subtraction), so the
// result is bit-identical to the reference's given the same sum, sumsq and count
__global__ void stats_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, double count,
                                      double epsilon, int64_t cols, double* __restrict__ mean,
                                      double* __restrict__ std_) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    const double m = sum[c] / count;
    mean[c] = m;
    const double var = __dsub_rn(sumsq[c], __dmul_rn(count, __dmul_rn(m, m))) / fmax(count - 1.0, 1.0);
    std_[c] = sqrt(fmax(var, epsilon));
}
// clip((x - mean) / (std + 1e-15), lo, hi)  (:162-164), fp64 math, fp32 result (what the network is fed).  The clip is
// np.clip's: a NaN passes through (a NaN observation stays visible) and an operand equal to a bound is kept as is.
__global__ void __launch_bounds__(256) stats_normalize_kernel(const float* __restrict__ x, int64_t rows, int64_t cols,
                                                              const double* __restrict__ mean,
                                                              const double* __restrict__ std_, double lo, double hi,
                                                              float* __restrict__ out32, double* __restrict__ out64) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int64_t c = i % cols;
    double v = ((double)x[i] - mean[c]) / (std_[c] + 1e-15);
    v = v < lo ? lo : (v > hi ? hi : v);
    if (out32) out32[i] = (float)v;
    if (out64) out64[i] = v;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_gae_scan(const double* rewards, const float* values, const uint8_t* game_overs, int64_t n, double discount,
                   double gae_lambda, double* advantages, double* value_targets, int64_t* n_valid, void* stream) {
    CB200_CHECK_ARG(rewards && values && game_overs && advantages && value_targets && n > 0, "bad arguments");
    CB200_LAUNCH(gae_scan_kernel, 1, kGaeThreads, 0, as_stream(stream), rewards, values, game_overs, n, discount,
                 gae_lambda, advantages, value_targets, n_valid);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_standardize(double* x, int64_t n, const int64_t* n_valid, double* mean_std_out, void* stream) {
    CB200_CHECK_ARG(x && n > 0, "bad arguments");
    CB200_LAUNCH(standardize_kernel, 1, 1024, 0, as_stream(stream), x, n, n_valid, mean_std_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_nstep_returns(const double* rewards, const int64_t* ep_start, const int64_t* ep_end, int64_t n,
                        double discount, int64_t n_step, double* out, void* stream) {
    CB200_CHECK_ARG(rewards && ep_start && ep_end && out && n > 0, "bad arguments");
    CB200_CHECK_ARG(n_step == -1 || n_step >= 1, "n-step should be an integer with value >= 1, or set to -1");
    CB200_LAUNCH(nstep_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), rewards, ep_start, ep_end, n,
                 discount, n_step, out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_running_stats_push(const float* x, int64_t rows, int64_t cols, double* sum, double* sumsq, void* stream) {
    CB200_CHECK_ARG(x && sum && sumsq && rows > 0 && cols > 0, "bad arguments");
    CB200_LAUNCH(stats_push_kernel, (unsigned)cols, 256, 0, as_stream(stream), x, rows, cols, sum, sumsq);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_running_stats_finalize(const double* sum, const double* sumsq, double count, double epsilon, int64_t cols,
                                 double* mean, double* std_out, void* stream) {
    CB200_CHECK_ARG(sum && sumsq && mean && std_out && cols > 0 && count > 0, "bad arguments");
    CB200_LAUNCH(stats_finalize_kernel, (unsigned)((cols + 127) / 128), 128, 0, as_stream(stream), sum, sumsq, count,
                 epsilon, cols, mean, std_out);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

int cb200_running_stats_normalize(const float* x, int64_t rows, int64_t cols, const double* mean, const double* std_in,
                                  double clip_lo, double clip_hi, float* out32, double* out64, void* stream) {
    CB200_CHECK_ARG(x && mean && std_in && (out32 || out64) && rows > 0 && cols > 0, "bad arguments");
    const int64_t n = rows * cols;
    CB200_LAUNCH(stats_normalize_kernel, (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), x, rows, cols, mean,
                 std_in, clip_lo, clip_hi, out32, out64);
    CB200_CHECK_LAUNCH();
    return CB200_OK;
}

}  // extern "C"
