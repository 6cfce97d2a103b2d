/* mbd_ppo.h — the arithmetic of the PPO acting step (csrc/ppo.cuh) for one env, compiled for the device and for the host harness
 * (tests/host_ppo/), so that both produce the same bits (nvcc -fmad=false / gcc -ffp-contract=off, include/mbd_fp32.h).
 *
 * [brax-recalled] brax.training.agents.ppo.networks / distribution.NormalTanhDistribution (v0.10.x):
 *   logits = MLP(normalize(obs)), hidden (32, 32, 32, 32), swish between layers, no final activation;
 *   loc, s = split(logits, 2);  scale = softplus(s) + 0.001;  raw = normal(key) * scale + loc;
 *   log_prob = sum_j [ -0.5 (raw/scale - loc/scale)^2 - (0.5 log(2 pi) + log scale) - 2 (log 2 - raw - softplus(-2 raw)) ];
 *   action = tanh(raw).
 * Flat policy layout (mbd_b200/rl/networks.py): W1 [O][32] (in, out), b1 [32], W2 [32][32], b2, W3, b3, W4, b4, W5 [32][2 Nu], b5 [2 Nu].
 * Every sum runs over its inputs in ascending order from 0.0f and adds the bias last (Flax Dense: dot, then + bias).  The
 * transcendentals are the project's fp32 functions, so they are not XLA's bits. */
#ifndef MBD_PPO_H_
#define MBD_PPO_H_

#include "mbd_fp32.h"

#define MBD_PPO_HIDDEN 32
#define MBD_PPO_LAYERS 5

/* number of floats of the flat policy parameters */
MBD_HD int mbd_ppo_policy_size(int O, int nu) {
  return O * MBD_PPO_HIDDEN + MBD_PPO_HIDDEN + 3 * (MBD_PPO_HIDDEN * MBD_PPO_HIDDEN + MBD_PPO_HIDDEN) + MBD_PPO_HIDDEN * 2 * nu + 2 * nu;
}
/* offset of W_l (l = 0 .. 4) in the flat policy buffer; its bias follows the weights */
MBD_HD int mbd_ppo_layer_offset(int O, int l) {
  const int h = MBD_PPO_HIDDEN;
  return l == 0 ? 0 : O * h + h + (l - 1) * (h * h + h);
}

/* running_statistics.normalize without clipping: (x - mean) / std */
MBD_HD float mbd_ppo_norm(float x, float mean, float std) { return MBD_DIV(x - mean, std); }

/* unit o of a dense layer: sum_i x[i] W[i][o] (i ascending), then + b[o] */
MBD_HD float mbd_ppo_dense(const float* x, const float* W, const float* b, int nin, int nout, int o) {
  float acc = 0.0f;
  for (int i = 0; i < nin; ++i) acc = acc + x[i] * W[i * nout + o];
  return acc + b[o];
}

/* swish(x) = x / (1 + exp(-x)).  The exponent is capped at 80 so that the divisor stays inside the range where the device's exact
 * division is correctly rounded (below 2^126); for x < -80 the result is below 2e-33 in magnitude either way. */
MBD_HD float mbd_swishf(float x) {
  const float e = mbd_expf(fminf(-x, 80.0f));
  return MBD_DIV(x, 1.0f + e);
}
/* softplus(x) = max(x, 0) + log(1 + exp(-|x|)) (jax.nn.softplus = logaddexp(x, 0)); absolute error below 2^-23 + |x| ulp */
MBD_HD float mbd_softplusf(float x) {
  const float e = mbd_expf(-fabsf(x));
  return fmaxf(x, 0.0f) + mbd_logf(1.0f + e);
}
/* tanh(x) = sign(x) (1 - 2 / (exp(2|x|) + 1)); 2|x| is capped at 40, where the result is 1.0f already (absolute error ~1e-7) */
MBD_HD float mbd_tanhf(float x) {
  const float e = mbd_expf(fminf(2.0f * fabsf(x), 40.0f));
  const float t = 1.0f - MBD_DIV(2.0f, e + 1.0f);
  return x < 0.0f ? -t : t;
}

#define MBD_PPO_HALF_LOG_2PI 0.9189385175704956f /* float32(0.5 log(2 pi)) */
#define MBD_PPO_LOG2 0.6931471824645996f         /* float32(log 2) */
#define MBD_PPO_MIN_STD 0.001f

/* one action component: from the policy outputs (loc, s) and the standard normal eps, the raw action, the action tanh(raw) and
 * the component's log-probability term (Normal logpdf minus the tanh log-det-Jacobian) */
MBD_HD void mbd_ppo_head(float loc, float s, float eps, float* raw, float* act, float* lp) {
  const float scale = mbd_softplusf(s) + MBD_PPO_MIN_STD;
  const float r = eps * scale + loc;
  const float z = MBD_DIV(r, scale) - MBD_DIV(loc, scale);
  const float logpdf = -0.5f * (z * z) - (MBD_PPO_HALF_LOG_2PI + mbd_logf(scale));
  const float jac = 2.0f * (MBD_PPO_LOG2 - r - mbd_softplusf(-2.0f * r));
  *raw = r;
  *act = mbd_tanhf(r);
  *lp = logpdf - jac;
}

/* eps of env b, component j: jax.random.normal(key, (B, Nu))[b, j] (part: the threefry layout of mbd_set_prng_layout) */
MBD_HD float mbd_ppo_eps(uint32_t k0, uint32_t k1, int b, int j, int B, int nu, int part) {
  const uint32_t idx = (uint32_t)b * (uint32_t)nu + (uint32_t)j;
  return mbd_bits_to_normal(mbd_random_bits_at(k0, k1, idx, part ? 0u : (uint32_t)B * (uint32_t)nu));
}

#endif /* MBD_PPO_H_ */
