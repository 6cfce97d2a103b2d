// mpc.cuh — the step between two control steps of the receding-horizon controller (mbd_mpc_advance and mbd_mpc_pi_advance in
// include/mbd_b200.h).
// k_mpc_advance: one CTA per problem, so every per-problem word has exactly one writer and no atomic is needed.  The control
// counter c = mpc_ctl[b] is read by every thread before thread 0 advances it.
// sigma_log == nullptr (model-based diffusion: the sigmas are the schedule's and stay): sigma_warm is not read.  Otherwise (the
// path-integral baselines, whose update may rewrite sigma) ACT also logs params[b][0].sigma and resets rows 0 .. Nwarm to sigma_warm.
#pragma once

namespace mbd {

constexpr int kMpcThreads = 256;

__global__ void __launch_bounds__(kMpcThreads) k_mpc_advance(mbd_mpc_plan p, int mode, float sigma_warm, float* sigma_log) {
  extern __shared__ float mpc_sm[];   // [H * nu]: the plan P_c (ACT)
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int nu = p.nu, HNu = p.H * p.nu, S = p.state_words, nd = p.Ndiffuse, nw = p.Nwarm;
  const int c = p.mpc_ctl_dev[b];
  const float* st = p.env_state_dev + (size_t)b * S;
  if (mode == MBD_MPC_RECORD) {
    // after mbd_vec_step of control step c - 1 (ACT has advanced the counter): r_{c-1} and s_c
    if (c < 1 || c > p.Nstep) return;
    if (tid == 0) p.rewards_dev[(size_t)b * p.Nstep + c - 1] = p.env_reward_dev[b];
    float* row = p.states_dev + ((size_t)b * (p.Nstep + 1) + c) * S;
    for (int k = tid; k < S; k += blockDim.x) row[k] = st[k];
    return;
  }
  if (c < 0 || c >= p.Nstep) return;   // past the last control step: nothing to execute
  float* Y = p.Ybars_dev + (size_t)b * nd * HNu;
  for (int k = tid; k < HNu; k += blockDim.x) mpc_sm[k] = Y[k];   // P_c = Ybars[b][0]
  __syncthreads();
  // a_c = P_c[0], unclipped
  for (int k = tid; k < nu; k += blockDim.x) {
    p.env_actions_dev[(size_t)b * nu + k] = mpc_sm[k];
    p.actions_dev[((size_t)b * p.Nstep + c) * nu + k] = mpc_sm[k];
  }
  if (c == 0) {   // s_0, the state the first plan was solved from
    float* row = p.states_dev + (size_t)b * (p.Nstep + 1) * S;
    for (int k = tid; k < S; k += blockDim.x) row[k] = st[k];
  }
  const bool more = c + 1 < p.Nstep;
  if (more) {
    // shift(P_c) -> Ybars[b][Nwarm]: row h takes row h + 1, the last row is 0 (the cold start's prior mean)
    float* W = Y + (size_t)nw * HNu;
    for (int k = tid; k < HNu; k += blockDim.x) W[k] = k + nu < HNu ? mpc_sm[k + nu] : 0.0f;
    // the keys of control step c + 1 -> params[b][1 .. Nwarm].key; the coefficients stay those of the one schedule, and so does
    // sigma unless there is a sigma log: then rows 1 .. Nwarm restart from sigma_warm
    const uint32_t* kr = p.keys_dev + ((size_t)b * p.Nstep + c + 1) * nw * 2;
    mbd_step_params* sp = p.params_dev + (size_t)b * nd;
    for (int j = tid; j < nw; j += blockDim.x) {
      sp[j + 1].key[0] = kr[2 * j];
      sp[j + 1].key[1] = kr[2 * j + 1];
      if (sigma_log) sp[j + 1].sigma = sigma_warm;
    }
  }
  __syncthreads();   // every thread has read c
  if (tid == 0) {
    p.rew_hist_log_dev[(size_t)b * p.Nstep + c] = p.rew_hist_dev[(size_t)b * nd + 1];   // rews.mean() of diffusion step 1
    if (sigma_log) {
      // the sigma control step c ended with: CMA-ES's last update wrote it to row 0.  MPPI and CEM never write sigma, so row 0
      // takes sigma_warm too and their log reads the sigma they sampled with (1 at c = 0, then sigma_warm)
      mbd_step_params* sp = p.params_dev + (size_t)b * nd;
      sigma_log[(size_t)b * p.Nstep + c] = sp[0].sigma;
      if (more) sp[0].sigma = sigma_warm;
    }
    if (more) p.ctl_dev[b].i = nw;   // after the last control step the counter stays at 0, where the solve left it
    p.mpc_ctl_dev[b] = c + 1;
  }
}

// k_ens_draw (mbd_ens_draw): the planner ensemble of control step c = mpc_ctl[b], one thread per (problem b, member k).  It runs
// before the control step's diffusion steps, so c is the step about to be planned; past the last control step it writes nothing.
constexpr int kEnsDrawThreads = 128;

__global__ void __launch_bounds__(kEnsDrawThreads) k_ens_draw(mbd_ens_draw_plan p, int part) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.B * p.K) return;
  const int b = t / p.K, k = t - b * p.K;
  const int c = p.mpc_ctl_dev[b];
  if (c < 0 || c >= p.Nstep) return;
  const uint32_t* key = p.keys_dev + ((size_t)b * p.Nstep + c) * 2;
  const float* R = p.ranges_dev + (size_t)b * 4;
  uint32_t kf[2], kg[2];
  vec_split(key[0], key[1], 2, 0, part, kf);
  vec_split(key[0], key[1], 2, 1, part, kg);
  p.ens_factors_dev[(size_t)t * 2] = vec_uniform(kf, k, p.K, part, R[0], R[1]);
  p.ens_factors_dev[(size_t)t * 2 + 1] = vec_uniform(kg, k, p.K, part, R[2], R[3]);
}

}  // namespace mbd
