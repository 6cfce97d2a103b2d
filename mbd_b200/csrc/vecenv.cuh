// vecenv.cuh — launch (2) of the vector env's step, its reset, set_state and world poses (mbd_vec_* in include/mbd_b200.h).
// One thread per env.  The xpbd envs' kinematics run in float64 (include/mbd_kin64.h): a few thousand flops per env against the
// 7-20 positional substeps of launch (1), on a part that runs fp64 at half its fp32 rate; in return the observations reproduce the
// host env's float64 kinematics up to the final float32 rounding.
#pragma once
#include "mbd_kin64.h"

namespace mbd {

enum { kVecStep = 0, kVecSetState = 1, kVecReset = 2, kVecWorld = 3 };
constexpr int kVecThreads = 128;
constexpr int kVecMaxObs = 2 * MBD_K64_MAXQ;

struct VecDims { int S, O; };   // state words and obs words per env

// observation of one xpbd env from its float32 state rows: PipelineEnv._make_pipeline_state + the env's _get_obs
__device__ __forceinline__ void vec_obs_xpbd(const mbd_vec_plan& p, const float* st, float* ob) {
  const double* T = p.kin_dev;
  mbd_k64_world X;
  mbd_k64_world_of(T, st, &X);
  float q[MBD_K64_MAXQ], qd[MBD_K64_MAXQ];
  mbd_k64_inverse(T, &X, q, qd);
  const int nq = p.nq, nqd = p.nqd;
  const int q0 = p.obs_layout == MBD_VEC_OBS_SKIP2 ? 2 : (p.obs_layout == MBD_VEC_OBS_SKIP1 ? 1 : 0);
  int o = 0;
  for (int j = q0; j < nq; ++j) ob[o++] = q[j];
  if (p.obs_layout == MBD_VEC_OBS_HOPPER) ob[1] = (float)X.pos[0][2];   // hopper.py:_get_obs: position[1] = x.pos[0, 2]
  for (int j = 0; j < nqd; ++j) {
    float v = qd[j];
    if (p.obs_layout == MBD_VEC_OBS_HOPPER) v = fminf(fmaxf(v, -10.0f), 10.0f);   // np.clip(qd, -10, 10)
    ob[o++] = v;
  }
}

__device__ __forceinline__ void vec_obs(const mbd_vec_plan& p, const VecDims& d, const float* st, float* ob) {
  if (p.kind == MBD_VEC_XPBD) vec_obs_xpbd(p, st, ob);
  else for (int k = 0; k < d.S; ++k) ob[k] = st[k];
}

// split(key, num)[i] in the threefry layout of the samplers (prng.split)
__device__ __forceinline__ void vec_split(uint32_t k0, uint32_t k1, int num, int i, int part, uint32_t* o) {
  if (part) { mbd_threefry2x32(k0, k1, 0u, (uint32_t)i, &o[0], &o[1]); return; }
  o[0] = mbd_random_bits_at(k0, k1, 2u * i, 2u * num);
  o[1] = mbd_random_bits_at(k0, k1, 2u * i + 1u, 2u * num);
}
// prng.uniform(key, (n,), lo, hi)[j]
__device__ __forceinline__ float vec_uniform(const uint32_t* k, int j, int n, int part, float lo, float hi) {
  const float u = mbd_bits_to_unit(mbd_random_bits_at(k[0], k[1], (uint32_t)j, part ? 0u : (uint32_t)n));
  return fmaxf(lo, u * (hi - lo) + lo);
}

// env.reset(key) of one env: the state rows into st, reward / done of the initial state
__device__ __forceinline__ void vec_reset_one(const mbd_vec_plan& p, const VecDims& d, uint32_t k0, uint32_t k1, int part, float* st,
                                              float* rew, float* done) {
  const float* RT = p.reset_dev;
  const int kind = (int)RT[MBD_VEC_RT_KIND];
  const float lo = RT[MBD_VEC_RT_LO], hi = RT[MBD_VEC_RT_HI];
  const int nq = p.nq;
  *rew = 0.0f;
  *done = 0.0f;
  if (p.kind == MBD_VEC_CAR2D) {   // car2d.py: the constant x0
    for (int k = 0; k < d.S; ++k) st[k] = RT[MBD_VEC_RT_Q + k];
    return;
  }
  if (p.kind == MBD_VEC_PUSHT) {   // pushT.py:22-38: rng, rng_goal_xy = split(rng); q[5:] = U(-1, 1) * scale + offset
    uint32_t kg[2];
    vec_split(k0, k1, 2, 1, part, kg);
    for (int k = 0; k < MBD_PT_NQ; ++k) { st[k] = RT[MBD_VEC_RT_Q + k]; st[MBD_PT_NQ + k] = 0.0f; }
    for (int j = 0; j < 3; ++j) st[5 + j] = vec_uniform(kg, j, 3, part, -1.0f, 1.0f) * RT[MBD_VEC_RT_Q + nq + 5 + j] + RT[MBD_VEC_RT_Q + 5 + j];
    *rew = pusht_reward(st);
    *done = *rew > 0.95f ? 1.0f : 0.0f;
    return;
  }
  // xpbd envs: rng, rng1, rng2 = split(rng, 3); q = init_q + U(lo, hi) [+ offset]; qd = U(lo, hi) or clip(sigma N(0, 1), -1, 1)
  float q[MBD_K64_MAXQ], qd[MBD_K64_MAXQ];
  const int nqd = p.nqd;
  for (int j = 0; j < nq; ++j) q[j] = RT[MBD_VEC_RT_Q + j];
  for (int j = 0; j < nqd; ++j) qd[j] = 0.0f;
  if (kind == MBD_VEC_RESET_UNIFORM || kind == MBD_VEC_RESET_NORMAL) {
    uint32_t r1[2], r2[2];
    vec_split(k0, k1, 3, 1, part, r1);
    vec_split(k0, k1, 3, 2, part, r2);
    for (int j = 0; j < nq; ++j) q[j] = q[j] + vec_uniform(r1, j, nq, part, lo, hi);
    if (kind == MBD_VEC_RESET_UNIFORM) {
      for (int j = 0; j < nqd; ++j) qd[j] = vec_uniform(r2, j, nqd, part, lo, hi);
    } else {   // ant.py: ops.sample(rng2, nv, 0, 1, nv, sigma, 0), the planner's sampler: element j of a legacy draw of nv * nv words
      const uint32_t total = part ? 0u : (uint32_t)nqd * (uint32_t)nqd;
      for (int j = 0; j < nqd; ++j) qd[j] = sample_elem(r2[0], r2[1], (uint32_t)j, total, RT[MBD_VEC_RT_SIGMA], 0.0f);
    }
    if (RT[MBD_VEC_RT_HAS_OFF] != 0.0f)
      for (int j = 0; j < nq; ++j) q[j] = q[j] + RT[MBD_VEC_RT_Q + nq + j];   // cartpole.py: + [0, pi]
  }
  mbd_k64_pipeline_init(p.kin_dev, q, qd, st);
}

// domain randomisation: the factors of episode e of env b into factors[b] (mbd_vec_dr; envs.vec.dr_factors):
// kf, kg = split(fold_in(dk_b, e)); f = uniform(kf, (1,), flo, fhi)[0], g = uniform(kg, (1,), glo, ghi)[0]
__device__ __forceinline__ void vec_dr_draw(const mbd_vec_plan& p, const mbd_vec_dr& dr, int b, int e, int part) {
  uint32_t k[2], kf[2], kg[2];
  mbd_threefry2x32(dr.keys_dev[2 * b], dr.keys_dev[2 * b + 1], 0u, (uint32_t)e, &k[0], &k[1]);   // fold_in(dk_b, e)
  vec_split(k[0], k[1], 2, 0, part, kf);
  vec_split(k[0], k[1], 2, 1, part, kg);
  p.factors_dev[2 * b] = vec_uniform(kf, 0, 1, part, dr.range[0], dr.range[1]);
  p.factors_dev[2 * b + 1] = vec_uniform(kg, 0, 1, part, dr.range[2], dr.range[3]);
}

template <int MODE>
__global__ void __launch_bounds__(kVecThreads) k_vec(mbd_vec_plan p, VecDims d, const uint32_t* __restrict__ keys, int part,
                                                     float* __restrict__ wpos, float* __restrict__ wrot, mbd_vec_dr dr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  float* st = p.state_dev + (size_t)b * d.S;
  float* ob = p.obs_dev + (size_t)b * d.O;
  if (MODE == kVecWorld) {   // x.pos / x.rot of every link (PipelineEnv._make_pipeline_state)
    const int L = (int)p.kin_dev[0];
    mbd_k64_world X;
    mbd_k64_world_of(p.kin_dev, st, &X);
    for (int l = 0; l < L; ++l) {
      for (int k = 0; k < 3; ++k) wpos[((size_t)b * L + l) * 3 + k] = (float)X.pos[l][k];
      for (int k = 0; k < 4; ++k) wrot[((size_t)b * L + l) * 4 + k] = (float)X.rot[l][k];
    }
    return;
  }
  float o[kVecMaxObs];
  if (MODE == kVecReset || MODE == kVecSetState) {
    float rew = 0.0f, done = 0.0f;
    if (MODE == kVecReset) vec_reset_one(p, d, keys[2 * b], keys[2 * b + 1], part, st, &rew, &done);
    vec_obs(p, d, st, o);
    float* fs = p.first_state_dev + (size_t)b * d.S;
    float* fo = p.first_obs_dev + (size_t)b * d.O;
    for (int k = 0; k < d.S; ++k) fs[k] = st[k];
    for (int k = 0; k < d.O; ++k) { ob[k] = o[k]; fo[k] = o[k]; }
    p.reward_dev[b] = rew;
    p.done_dev[b] = done;
    p.truncation_dev[b] = 0.0f;
    p.steps_dev[b] = 0.0f;
    if (MODE == kVecReset && dr.keys_dev) {   // episode 0
      dr.episodes_dev[b] = 0;
      vec_dr_draw(p, dr, b, 0, part);
    }
    return;
  }
  // MODE == kVecStep: launch (1) left the next state in next_state and the step's reward in reward
  const float* nx = p.next_state_dev + (size_t)b * d.S;
  vec_obs(p, d, nx, o);
  const float done_prev = p.done_dev[b];
  float env_done = 0.0f;
  if (p.done_rule == MBD_VEC_DONE_COUNTER) env_done = done_prev + 1.0f;                        // humanoidtrack.py: done + 1
  else if (p.done_rule == MBD_VEC_DONE_PUSHT) env_done = p.reward_dev[b] > 0.95f ? 1.0f : 0.0f;   // pushT.py:64-66
  // [brax-recalled] AutoResetWrapper(EpisodeWrapper(env)), action_repeat = 1 (brax/envs/wrappers/training.py)
  const int ep = p.episode_length;
  float steps = (ep > 0 && done_prev != 0.0f) ? 0.0f : p.steps_dev[b];
  steps = steps + 1.0f;
  float done = env_done, trunc = 0.0f;
  if (ep > 0 && steps >= (float)ep) { done = 1.0f; trunc = 1.0f - env_done; }
  p.done_dev[b] = done;
  p.truncation_dev[b] = trunc;
  p.steps_dev[b] = steps;
  const bool reset = ep > 0 && done != 0.0f;
  const float* src = reset ? p.first_state_dev + (size_t)b * d.S : nx;
  for (int k = 0; k < d.S; ++k) st[k] = src[k];
  const float* fo = p.first_obs_dev + (size_t)b * d.O;
  for (int k = 0; k < d.O; ++k) ob[k] = reset ? fo[k] : o[k];
  // the next episode's factors; launch (1) of this step has read the old ones, launch (1) of the next step reads these
  if (reset && dr.keys_dev) {
    const int e = dr.episodes_dev[b] + 1;
    dr.episodes_dev[b] = e;
    vec_dr_draw(p, dr, b, e, part);
  }
}

}  // namespace mbd
