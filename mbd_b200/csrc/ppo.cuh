// ppo.cuh — the PPO acting step, the observation statistics and GAE (mbd_ppo_* in include/mbd_b200.h).
// k_ppo_act: one warp per env, lane o = hidden unit o; the flat policy is staged once per CTA into shared memory, and a warp's
// layer input lives in its own shared row, so every unit is mbd_ppo_dense of include/mbd_ppo.h, the function the host harness runs.
#pragma once
#include "mbd_ppo.h"

namespace mbd {

constexpr int kPpoWarps = 8;
constexpr int kPpoThreads = 32 * kPpoWarps;
constexpr int kPpoRow = MBD_PPO_MAX_OBS + 2 * MBD_PPO_MAX_NU;   // per-warp scratch: layer input [128] | outputs [64]

// the last CTA of a launch advances the control words (every CTA has read them by then)
__device__ __forceinline__ void ppo_advance(int32_t* ctl, int mode) {
  __syncthreads();
  if (threadIdx.x != 0) return;
  __threadfence();
  if (atomicAdd(&ctl[2], 1) != (int)gridDim.x - 1) return;
  ctl[2] = 0;
  if (mode == MBD_PPO_RECORD || mode == MBD_PPO_EVAL_RECORD) {
    ctl[0] = 0;
  } else {
    ctl[0] = ctl[0] + 1;
    ctl[1] = ctl[1] + 1;
  }
  __threadfence();
}

__global__ void __launch_bounds__(kPpoThreads) k_ppo_act(mbd_ppo_plan p, int mode, int part) {
  extern __shared__ float ppo_sm[];
  const int O = p.O, nu = p.nu, B = p.B, H = MBD_PPO_HIDDEN;
  const int np = mbd_ppo_policy_size(O, nu);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool acting = mode == MBD_PPO_ACT || mode == MBD_PPO_EVAL;
  if (acting)
    for (int i = threadIdx.x; i < np; i += blockDim.x) ppo_sm[i] = p.policy_dev[i];
  float* x = ppo_sm + np + warp * kPpoRow;
  float* out = x + MBD_PPO_MAX_OBS;
  __syncthreads();
  const int t = p.act_ctl_dev[0];
  const int krow = p.act_ctl_dev[1];
  uint32_t k0 = 0, k1 = 0;
  if (acting && krow < p.act_key_rows) { k0 = p.act_keys_dev[2 * krow]; k1 = p.act_keys_dev[2 * krow + 1]; }
  const bool training = mode == MBD_PPO_ACT || mode == MBD_PPO_RECORD;
  const bool inside = (!acting || krow < p.act_key_rows) && (!training || t <= p.slots - (mode == MBD_PPO_ACT ? 1 : 0));
  for (int b = blockIdx.x * kPpoWarps + warp; inside && b < B; b += gridDim.x * kPpoWarps) {
    const float* ob = p.env_obs_dev + (size_t)b * O;
    if (training) {
      float* rec = p.obs_dev + ((size_t)t * B + b) * O;
      for (int i = lane; i < O; i += 32) rec[i] = ob[i];
      if (t > 0 && lane == 0) {
        const size_t r = (size_t)(t - 1) * B + b;
        p.reward_dev[r] = p.env_reward_dev[b];
        p.disc_dev[r] = 1.0f - p.env_done_dev[b];
        p.trunc_dev[r] = p.env_trunc_dev[b];
      }
    } else if (t > 0 && lane == 0) {   // EvalWrapper: the return of the first episode of every env
      const float a = p.active_dev[b];
      p.ret_dev[b] = p.ret_dev[b] + a * p.env_reward_dev[b];
      p.active_dev[b] = a * (1.0f - p.env_done_dev[b]);
    }
    if (!acting) continue;
    for (int i = lane; i < O; i += 32) x[i] = mbd_ppo_norm(ob[i], p.mean_dev[i], p.std_dev[i]);
    __syncwarp();
    int nin = O;
    for (int l = 0; l < MBD_PPO_LAYERS - 1; ++l) {
      const float* W = ppo_sm + mbd_ppo_layer_offset(O, l);
      const float h = mbd_swishf(mbd_ppo_dense(x, W, W + nin * H, nin, H, lane));
      __syncwarp();
      x[lane] = h;
      __syncwarp();
      nin = H;
    }
    const float* W5 = ppo_sm + mbd_ppo_layer_offset(O, MBD_PPO_LAYERS - 1);
    for (int o = lane; o < 2 * nu; o += 32) out[o] = mbd_ppo_dense(x, W5, W5 + H * 2 * nu, H, 2 * nu, o);
    __syncwarp();
    if (lane < nu) {
      float raw, act, lp;
      mbd_ppo_head(out[lane], out[nu + lane], mbd_ppo_eps(k0, k1, b, lane, B, nu, part), &raw, &act, &lp);
      p.env_actions_dev[(size_t)b * nu + lane] = act;
      if (mode == MBD_PPO_ACT) p.raw_dev[((size_t)t * B + b) * nu + lane] = raw;
      x[lane] = lp;
    }
    __syncwarp();
    if (mode == MBD_PPO_ACT && lane == 0) {
      float s = 0.0f;
      for (int j = 0; j < nu; ++j) s = s + x[j];   // j ascending
      p.logp_dev[(size_t)t * B + b] = s;
    }
    __syncwarp();
  }
  ppo_advance(p.act_ctl_dev, mode);
}

// running_statistics.update, (1): per chunk of MBD_PPO_STAT_ROWS rows and per column, S1 = sum d and S2 = sum d^2 with d = x - c,
// in float64, rows ascending.  The shift c is the batch's first row: a value inside the column's spread, so S2 - S1^2 / n keeps the
// batch's variance where a shift by the old mean would cancel it away (a column 1e4 from a fresh mean of 0 with a 1e-3 spread).
// Thread = column.
__global__ void __launch_bounds__(MBD_PPO_MAX_OBS) k_ppo_stat_partial(mbd_ppo_plan p, int rows) {
  const int j = threadIdx.x, O = p.O;
  if (j >= O) return;
  const double m = (double)p.obs_dev[j];
  const int r0 = blockIdx.x * MBD_PPO_STAT_ROWS;
  const int r1 = min(rows, r0 + MBD_PPO_STAT_ROWS);
  double s1 = 0.0, s2 = 0.0;
  for (int r = r0; r < r1; ++r) {
    const double d = (double)p.obs_dev[(size_t)r * O + j] - m;
    s1 = s1 + d;
    s2 = s2 + d * d;
  }
  p.stat_scratch_dev[(size_t)blockIdx.x * 2 * O + j] = s1;
  p.stat_scratch_dev[((size_t)blockIdx.x * 2 + 1) * O + j] = s2;
}

// (2): the chunk sums in chunk order give the batch mean c + S1 / n and the batch's summed variance M2 = S2 - (S1 / n) S1; the batch
// joins the old state by the pairwise combination (Chan, Golub and LeVeque), with delta = batch mean - old mean:
//   mean += delta n / count;  summed_var += M2 + delta^2 n_old n / count.
// That equals running_statistics.update's mean + sum (x - mean) / count and summed_var + sum (x - old mean)(x - new mean), and every
// term of the variance is non-negative.
__global__ void __launch_bounds__(MBD_PPO_MAX_OBS) k_ppo_stat_final(mbd_ppo_plan p, int rows, int chunks) {
  const int j = threadIdx.x, O = p.O;
  const double n0 = p.stat_dev[0], n = (double)rows;
  const double count = n0 + n;
  __syncthreads();   // every thread has read the old count before thread 0 writes the new one
  if (j >= O) return;
  double s1 = 0.0, s2 = 0.0;
  for (int c = 0; c < chunks; ++c) {
    s1 = s1 + p.stat_scratch_dev[(size_t)c * 2 * O + j];
    s2 = s2 + p.stat_scratch_dev[((size_t)c * 2 + 1) * O + j];
  }
  const double mb = s1 / n;
  const double m2 = s2 - mb * s1;
  const double delta = ((double)p.obs_dev[j] + mb) - p.stat_dev[1 + j];
  const double mean = p.stat_dev[1 + j] + delta * (n / count);
  const double var = p.stat_dev[1 + O + j] + m2 + delta * delta * (n0 * (n / count));
  const double sd = fmin(fmax(sqrt(var / count), 1e-6), 1e6);
  p.stat_dev[1 + j] = mean;
  p.stat_dev[1 + O + j] = var;
  if (j == 0) p.stat_dev[0] = count;
  ((float*)p.mean_dev)[j] = (float)mean;
  ((float*)p.std_dev)[j] = (float)sd;
}

// fixed-order sum of v over the CTA (blockDim.x a power of two): adjacent halves, stride blockDim / 2 down to 1
__device__ __forceinline__ float ppo_block_sum(float v, float* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] = sh[threadIdx.x] + sh[threadIdx.x + s];
    __syncthreads();
  }
  const float r = sh[0];
  __syncthreads();
  return r;
}

// CTA 0: compute_gae for trajectories i = thread, thread + blockDim, ..., then the advantage normalisation over the T * mb
// advantages; every thread sums its trajectories in ascending order, tau ascending within each, and the CTA sum is ppo_block_sum.
// CTAs 1 ..: the entropy noise normal(loss key, (T, mb, Nu)).
__global__ void __launch_bounds__(1024) k_ppo_gae(mbd_ppo_plan p, int part) {
  const int T = p.unroll, mb = p.mb, B = p.B;
  const int krow = *p.loss_ctl_dev;
  if (blockIdx.x > 0) {
    if (krow < 0 || krow >= p.loss_key_rows) return;
    const uint32_t k0 = p.loss_keys_dev[2 * krow], k1 = p.loss_keys_dev[2 * krow + 1];
    const uint32_t total = (uint32_t)T * (uint32_t)mb * (uint32_t)p.nu;
    for (uint32_t e = (blockIdx.x - 1) * blockDim.x + threadIdx.x; e < total; e += (gridDim.x - 1) * blockDim.x)
      p.ent_eps_dev[e] = mbd_bits_to_normal(mbd_random_bits_at(k0, k1, e, part ? 0u : total));
    return;
  }
  __shared__ float sh[1024];
  const float g = p.discount, lam = p.gae_lambda;
  float sum = 0.0f;
  for (int i = threadIdx.x; i < mb; i += blockDim.x) {
    const int n = p.traj_dev[i];
    const int u = n / B, b = n - u * B;
    const size_t base = (size_t)u * T;
    const float boot = p.values_dev[(size_t)T * mb + i];
    float acc = 0.0f, vnext = boot;
    for (int tau = T - 1; tau >= 0; --tau) {   // vs - v, reverse scan
      const size_t r = (base + tau) * B + b;
      const float rew = p.reward_dev[r] * p.reward_scaling;
      const float tr = p.trunc_dev[r];
      const float term = (1.0f - p.disc_dev[r]) * (1.0f - tr);
      const float tm = 1.0f - tr;
      const float v = p.values_dev[(size_t)tau * mb + i];
      const float delta = (rew + g * (1.0f - term) * vnext - v) * tm;
      acc = delta + g * (1.0f - term) * tm * lam * acc;
      p.vs_dev[(size_t)tau * mb + i] = acc + v;
      vnext = v;
    }
    for (int tau = 0; tau < T; ++tau) {   // advantages with vs_{t+1} (row T: the bootstrap value)
      const size_t r = (base + tau) * B + b;
      const float rew = p.reward_dev[r] * p.reward_scaling;
      const float tr = p.trunc_dev[r];
      const float term = (1.0f - p.disc_dev[r]) * (1.0f - tr);
      const float tm = 1.0f - tr;
      const float v = p.values_dev[(size_t)tau * mb + i];
      const float vsn = tau + 1 < T ? p.vs_dev[(size_t)(tau + 1) * mb + i] : boot;
      const float a = (rew + g * (1.0f - term) * vsn - v) * tm;
      p.adv_dev[(size_t)tau * mb + i] = a;
      sum = sum + a;
    }
  }
  const float cnt = (float)(T * mb);
  const float mean = MBD_DIV(ppo_block_sum(sum, sh), cnt);
  float sq = 0.0f;
  for (int i = threadIdx.x; i < mb; i += blockDim.x)
    for (int tau = 0; tau < T; ++tau) {
      const float d = p.adv_dev[(size_t)tau * mb + i] - mean;
      sq = sq + d * d;
    }
  const float sd = MBD_SQRT(MBD_DIV(ppo_block_sum(sq, sh), cnt));
  for (int i = threadIdx.x; i < mb; i += blockDim.x)
    for (int tau = 0; tau < T; ++tau) {
      float* a = p.adv_dev + (size_t)tau * mb + i;
      *a = MBD_DIV(*a - mean, sd + 1e-8f);
    }
}

}  // namespace mbd
