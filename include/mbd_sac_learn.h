/* mbd_sac_learn.h — the arithmetic of the fused SAC gradient update (csrc/sac_learn.cuh), compiled for the device and for the host
 * harness (tests/host_sac_learn/), so that both produce the same bits (nvcc -fmad=false / gcc -ffp-contract=off, include/mbd_fp32.h).
 *
 * One update is Brax's sgd_step as restated in mbd_b200/rl/sac.py (`losses`, `Learner.update`): the alpha, critic and actor losses
 * with the parameters from before the update, three Adam steps (torch.optim.Adam's formula, beta = (0.9, 0.999), eps = 1e-8), then
 * target += tau (q_new - target).
 *
 * Row phase (per batch row b; every loss term is written unscaled, the 1/n and 1/(2n) of the means come in the weight phase):
 *   x = normalize(obs), xn = normalize(next_obs); logits = policy(x), logits_n = policy(xn) (mbd_sac.h's units)
 *   alpha = mbd_expf(old log alpha)
 *   target = reward * reward_scaling + (discount * discounting) * (min_c Qt_c(xn, tanh raw_c) - alpha * lp_c)   raw_c from eps[1]
 *   err_c = (Q_c(x, action) - target) * (1 - trunc);  critic seed d3_c = err_c * (1 - trunc);  critic term = err_0^2 + err_1^2
 *   alpha term = -lp_a - target_entropy (eps[0]);  actor term = alpha * lp_p - min_c Q_c(x, tanh raw_p) (eps[2])
 *   actor seed: -1 into the critic that gives the min (critic 0 on a tie, torch.min's first index), 0 into the other
 * Backward of a row: dst[o] = (sum_k W[o][k] src[k], k ascending from 0.0f) where the layer's output h[o] > 0, else 0 (ReLU's
 * derivative at 0 is 0).  The action gradient of the actor row is sum over the critics c ascending of (sum_k W1_c[O + j][k] d1_c[k]),
 * the non-chosen critic contributing an exact zero.  The head: with t = tanh(raw_p) (the fp32 word of the forward) and exact z = eps,
 * d lp / d loc = 2 t and d lp / d scale = 2 t eps - 1 / scale, so
 *   g = gA (1 - t t) + alpha (2 t);  d loc = g;  d s = (g eps - alpha / scale) * sigmoid(s)   (mbd_sac_learn_head_grad)
 * Weight phase: dW[i][o] = (sum_b In[b][i] D[b][o], b ascending from 0.0f) / N, with In's row nin = 1 for the bias and N = n
 * (policy) or 2 n (Q); the alpha gradient is mbd_expf(log alpha) * (sum_b term_b / n), b ascending.  The owner of a parameter then
 * applies mbd_sac_adam and, for Q, mbd_sac_polyak. */
#ifndef MBD_SAC_LEARN_H_
#define MBD_SAC_LEARN_H_

#include "mbd_sac.h"

#define MBD_SAC_LEARN_MAX_BATCH 4096
#define MBD_SAC_ADAM_B1 0.9
#define MBD_SAC_ADAM_B2 0.999
#define MBD_SAC_ADAM_EPS 1e-8f
#define MBD_SAC_ALPHA_LR 3e-4f
#define MBD_SAC_LEARN_JOBS 9      /* weight-phase matrices: policy layers 0..2, critic 0 layers 0..2, critic 1 layers 0..2 */

/* ---- the Q buffer (mbd_b200/rl/networks.py: layer-major, W_l [2][in][out] then b_l [2][out]) ---- */
MBD_HD int mbd_sac_q_in(int O, int nu, int l) { return l == 0 ? O + nu : MBD_SAC_HIDDEN; }
MBD_HD int mbd_sac_q_out(int l) { return l == 2 ? 1 : MBD_SAC_HIDDEN; }
MBD_HD int mbd_sac_q_layer_offset(int O, int nu, int l) {
  int off = 0;
  for (int k = 0; k < l; ++k) off += 2 * (mbd_sac_q_in(O, nu, k) * mbd_sac_q_out(k) + mbd_sac_q_out(k));
  return off;
}
MBD_HD int mbd_sac_q_size(int O, int nu) { return mbd_sac_q_layer_offset(O, nu, 3); }
/* weights of critic c in layer l: [in][out] at this offset; its bias [out] at mbd_sac_q_bias */
MBD_HD int mbd_sac_q_w(int O, int nu, int l, int c) { return mbd_sac_q_layer_offset(O, nu, l) + c * mbd_sac_q_in(O, nu, l) * mbd_sac_q_out(l); }
MBD_HD int mbd_sac_q_bias(int O, int nu, int l, int c) {
  return mbd_sac_q_layer_offset(O, nu, l) + 2 * mbd_sac_q_in(O, nu, l) * mbd_sac_q_out(l) + c * mbd_sac_q_out(l);
}

/* ---- the scratch buffer of one update (floats; rows of the batch, row-major) ---- */
typedef struct mbd_sac_learn_layout {
  long long x, p1, p2, dp1, dp2, dp3;         /* policy: input [n][O], h1, h2 [n][256], deltas [n][256], [n][256], [n][2 Nu] */
  long long qin;                              /* critic input [n][O + Nu] = (x, action) */
  long long c1[2], c2[2], dc1[2], dc2[2], dc3[2];   /* critic c: h1, h2 [n][256], deltas [n][256], [n][256], [n] */
  long long terms;                            /* [3][n]: alpha term, critic term, actor term */
  long long total;
} mbd_sac_learn_layout;

MBD_HD mbd_sac_learn_layout mbd_sac_learn_layout_of(int O, int nu, int n) {
  const long long H = MBD_SAC_HIDDEN, N = n;
  mbd_sac_learn_layout L;
  long long k = 0;
  L.x = k; k += N * O;
  L.p1 = k; k += N * H;
  L.p2 = k; k += N * H;
  L.dp1 = k; k += N * H;
  L.dp2 = k; k += N * H;
  L.dp3 = k; k += N * 2 * nu;
  L.qin = k; k += N * (O + nu);
  for (int c = 0; c < 2; ++c) {
    L.c1[c] = k; k += N * H;
    L.c2[c] = k; k += N * H;
    L.dc1[c] = k; k += N * H;
    L.dc2[c] = k; k += N * H;
    L.dc3[c] = k; k += N;
  }
  L.terms = k; k += 3 * N;
  L.total = k;
  return L;
}

/* one weight-phase matrix: dW [nin + 1][nout] (row nin: the bias) from In (scratch offset, row stride nin) and D (offset, stride
 * nout); parameter (i, o) lives at w + i * nout + o for i < nin and at bias + o for i = nin */
typedef struct mbd_sac_learn_job {
  int is_q, critic, nin, nout;
  long long in, d;
  int w, bias;
} mbd_sac_learn_job;

MBD_HD mbd_sac_learn_job mbd_sac_learn_job_of(int O, int nu, int n, int j) {
  const mbd_sac_learn_layout L = mbd_sac_learn_layout_of(O, nu, n);
  mbd_sac_learn_job J;
  const int l = j % 3;
  J.is_q = j >= 3;
  J.critic = j >= 6 ? 1 : 0;
  if (!J.is_q) {
    J.nin = l == 0 ? O : MBD_SAC_HIDDEN;
    J.nout = l == 2 ? 2 * nu : MBD_SAC_HIDDEN;
    J.in = l == 0 ? L.x : l == 1 ? L.p1 : L.p2;
    J.d = l == 0 ? L.dp1 : l == 1 ? L.dp2 : L.dp3;
    J.w = mbd_sac_layer_offset(O, l);
    J.bias = J.w + J.nin * J.nout;
  } else {
    const int c = J.critic;
    J.nin = mbd_sac_q_in(O, nu, l);
    J.nout = mbd_sac_q_out(l);
    /* selects rather than L.c1[c]: a runtime index into the struct would put it in local memory on the device */
    J.in = l == 0 ? L.qin : l == 1 ? (c ? L.c1[1] : L.c1[0]) : (c ? L.c2[1] : L.c2[0]);
    J.d = l == 0 ? (c ? L.dc1[1] : L.dc1[0]) : l == 1 ? (c ? L.dc2[1] : L.dc2[0]) : (c ? L.dc3[1] : L.dc3[0]);
    J.w = mbd_sac_q_w(O, nu, l, c);
    J.bias = mbd_sac_q_bias(O, nu, l, c);
  }
  return J;
}

/* ---- the per-row pieces ---- */
MBD_HD float mbd_sac_sigmoidf(float s) {
  if (s >= 0.0f) return MBD_DIV(1.0f, 1.0f + mbd_expf(-s));
  const float e = mbd_expf(s);
  return MBD_DIV(e, 1.0f + e);
}

/* the actor row's head backward of component j: gA = d(-min Q) / d action, t = tanh(raw_p), eps, s = the scale logit */
MBD_HD void mbd_sac_learn_head_grad(float gA, float t, float eps, float s, float alpha, float* dloc, float* ds) {
  const float scale = mbd_softplusf(s) + MBD_PPO_MIN_STD;
  const float g = gA * (1.0f - t * t) + alpha * (2.0f * t);
  *dloc = g;
  *ds = (g * eps - MBD_DIV(alpha, scale)) * mbd_sac_sigmoidf(s);
}

/* Brax's target of one row: reward * reward_scaling + (discount * discounting) * (min(qt0, qt1) - alpha * lp_c) */
MBD_HD float mbd_sac_learn_target(float reward, float discount, float qt0, float qt1, float alpha, float lp_c, float reward_scaling,
                                  float discounting) {
  const float next_v = fminf(qt0, qt1) - alpha * lp_c;
  return reward * reward_scaling + (discount * discounting) * next_v;
}

/* ---- Adam (torch.optim.Adam, capturable) and Polyak ---- */
/* bias corrections of step t >= 1: 1 - beta^t in float64 (beta^t by squaring: correctly rounded * and - only, so host and device
 * agree), rounded to fp32; then step = lr / bc1 and bc2s = sqrt(bc2) in fp32 (correctly rounded) */
MBD_HD double mbd_sac_powi(double b, long long t) {
  double r = 1.0, p = b;
  while (t > 0) {
    if (t & 1) r = r * p;
    p = p * p;
    t >>= 1;
  }
  return r;
}
MBD_HD void mbd_sac_adam_scalars(float lr, long long t, float* step, float* bc2s) {
  const float bc1 = (float)(1.0 - mbd_sac_powi(MBD_SAC_ADAM_B1, t)), bc2 = (float)(1.0 - mbd_sac_powi(MBD_SAC_ADAM_B2, t));
  *step = MBD_DIV(lr, bc1);
  *bc2s = MBD_SQRT(bc2);
}
/* m = m + (1 - b1) (g - m) (torch's lerp_); v = v b2 + (1 - b2) g^2; p = p - step * (m / (sqrt(v) / bc2s + eps)).  v reaches the
 * subnormal range when a parameter's gradient stays tiny or rarely non-zero (v decays by 0.999 each update); MBD_SQRT is
 * correctly rounded there too (include/mbd_fp32.h). */
MBD_HD void mbd_sac_adam(float* p, float* m, float* v, float g, float step, float bc2s) {
  const float mm = *m + 0.1f * (g - *m);
  const float vv = *v * 0.999f + 0.001f * (g * g);
  const float denom = MBD_DIV(MBD_SQRT(vv), bc2s) + MBD_SAC_ADAM_EPS;
  *m = mm;
  *v = vv;
  *p = *p - step * MBD_DIV(mm, denom);
}
MBD_HD float mbd_sac_polyak(float target, float q, float tau) { return target + tau * (q - target); }

#endif /* MBD_SAC_LEARN_H_ */
