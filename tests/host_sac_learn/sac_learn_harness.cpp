// include/mbd_sac_learn.h built for the host (tests/test_sac_learn_cpu.py, tests/test_sac_learn_gpu.py): one fused SAC update row by
// row, in the association orders of csrc/sac_learn.cuh, so that it gives the kernel's bits.
#include <vector>

#include "mbd_sac_learn.h"

namespace {
const int H = MBD_SAC_HIDDEN;

// out[o] = (relu of) sum_i x[i] W[i][o] (i ascending from 0) + b[o]
void dense(const float* x, const float* W, const float* b, int nin, int nout, bool relu, float* out) {
  for (int o = 0; o < nout; ++o) {
    float acc = 0.0f;
    for (int i = 0; i < nin; ++i) acc = acc + x[i] * W[i * nout + o];
    const float y = acc + b[o];
    out[o] = relu ? mbd_sac_relu(y) : y;
  }
}
// hd[o] = sum_k W[o][k] d[k] (k ascending from 0) where hd[o] > 0, else 0
void back(const float* W, int nout, const float* d, float* hd) {
  for (int o = 0; o < H; ++o) {
    float acc = 0.0f;
    for (int k = 0; k < nout; ++k) acc = acc + W[o * nout + k] * d[k];
    hd[o] = hd[o] > 0.0f ? acc : 0.0f;
  }
}
}  // namespace

extern "C" {
// One update.  rows [n][row], eps [3][n][nu]; the parameters, moments and log alpha are updated in place; step: updates done before.
// Outputs the fp32 gradients (policy [P], q [Q], log alpha [1]) and the losses [3].
int sac_learn_update_host(float* policy, float* q, float* target_q, float* log_alpha, float* pm, float* pv, float* qm, float* qv,
                          float* amv, long long step, const float* mean, const float* std, const float* rows, const float* eps,
                          int O, int nu, int n, float lr, float reward_scaling, float discounting, float tau, float* gpolicy,
                          float* gq, float* galpha, float* losses) {
  const int R = mbd_sac_row(O, nu), QI = O + nu;
  const mbd_sac_learn_layout L = mbd_sac_learn_layout_of(O, nu, n);
  std::vector<float> scr((size_t)L.total, 0.0f);
  const float alpha = mbd_expf(log_alpha[0]);
  const float* Pw[3];
  for (int l = 0; l < 3; ++l) Pw[l] = policy + mbd_sac_layer_offset(O, l);
  std::vector<float> x(O), xn(O), h1(H), h2(H), ln(2 * nu), lg(2 * nu), tin(QI), cin(QI), ain(QI), tp(nu);
  std::vector<float> c1[2], c2[2], a1[2], a2[2];
  for (int c = 0; c < 2; ++c) { c1[c].resize(H); c2[c].resize(H); a1[c].resize(H); a2[c].resize(H); }
  std::vector<float> p1(H), p2(H), dp3(2 * nu);
  for (int b = 0; b < n; ++b) {
    const float* r = rows + (size_t)b * R;
    const float* e0 = eps + (size_t)b * nu;
    const float* e1 = eps + ((size_t)n + b) * nu;
    const float* e2 = eps + ((size_t)2 * n + b) * nu;
    for (int i = 0; i < O; ++i) {
      x[i] = mbd_ppo_norm(r[i], mean[i], std[i]);
      xn[i] = mbd_ppo_norm(r[mbd_sac_off_next_obs(O, nu) + i], mean[i], std[i]);
      tin[i] = xn[i];
      cin[i] = ain[i] = x[i];
      scr[L.x + (size_t)b * O + i] = x[i];
    }
    for (int j = 0; j < nu; ++j) cin[O + j] = r[mbd_sac_off_action(O) + j];
    for (int i = 0; i < QI; ++i) scr[L.qin + (size_t)b * QI + i] = cin[i];
    // the target
    dense(xn.data(), Pw[0], Pw[0] + O * H, O, H, true, h1.data());
    dense(h1.data(), Pw[1], Pw[1] + H * H, H, H, true, h2.data());
    dense(h2.data(), Pw[2], Pw[2] + H * 2 * nu, H, 2 * nu, false, ln.data());
    float lpc = 0.0f;
    for (int j = 0; j < nu; ++j) {
      float raw, act, lp;
      mbd_ppo_head(ln[j], ln[nu + j], e1[j], &raw, &act, &lp);
      tin[O + j] = act;
      lpc = lpc + lp;
    }
    float qt[2], one[1];
    for (int c = 0; c < 2; ++c) {
      dense(tin.data(), target_q + mbd_sac_q_w(O, nu, 0, c), target_q + mbd_sac_q_bias(O, nu, 0, c), QI, H, true, h1.data());
      dense(h1.data(), target_q + mbd_sac_q_w(O, nu, 1, c), target_q + mbd_sac_q_bias(O, nu, 1, c), H, H, true, h2.data());
      dense(h2.data(), target_q + mbd_sac_q_w(O, nu, 2, c), target_q + mbd_sac_q_bias(O, nu, 2, c), H, 1, false, one);
      qt[c] = one[0];
    }
    const float tgt = mbd_sac_learn_target(r[mbd_sac_off_reward(O, nu)], r[mbd_sac_off_discount(O, nu)], qt[0], qt[1], alpha, lpc,
                                           reward_scaling, discounting);
    // the policy on x and its heads
    dense(x.data(), Pw[0], Pw[0] + O * H, O, H, true, p1.data());
    dense(p1.data(), Pw[1], Pw[1] + H * H, H, H, true, p2.data());
    dense(p2.data(), Pw[2], Pw[2] + H * 2 * nu, H, 2 * nu, false, lg.data());
    for (int o = 0; o < H; ++o) { scr[L.p1 + (size_t)b * H + o] = p1[o]; scr[L.p2 + (size_t)b * H + o] = p2[o]; }
    float lpa = 0.0f, lpp = 0.0f;
    for (int j = 0; j < nu; ++j) {
      float raw, act, lp;
      mbd_ppo_head(lg[j], lg[nu + j], e0[j], &raw, &act, &lp);
      lpa = lpa + lp;
    }
    for (int j = 0; j < nu; ++j) {
      float raw, act, lp;
      mbd_ppo_head(lg[j], lg[nu + j], e2[j], &raw, &act, &lp);
      tp[j] = act;
      ain[O + j] = act;
      lpp = lpp + lp;
    }
    // both critics on (x, action) and (x, tanh raw_p)
    float qv[2], qa[2];
    for (int c = 0; c < 2; ++c) {
      const float *W1 = q + mbd_sac_q_w(O, nu, 0, c), *B1 = q + mbd_sac_q_bias(O, nu, 0, c);
      const float *W2 = q + mbd_sac_q_w(O, nu, 1, c), *B2 = q + mbd_sac_q_bias(O, nu, 1, c);
      const float *W3 = q + mbd_sac_q_w(O, nu, 2, c), *B3 = q + mbd_sac_q_bias(O, nu, 2, c);
      dense(cin.data(), W1, B1, QI, H, true, c1[c].data());
      dense(c1[c].data(), W2, B2, H, H, true, c2[c].data());
      dense(c2[c].data(), W3, B3, H, 1, false, one);
      qv[c] = one[0];
      dense(ain.data(), W1, B1, QI, H, true, a1[c].data());
      dense(a1[c].data(), W2, B2, H, H, true, a2[c].data());
      dense(a2[c].data(), W3, B3, H, 1, false, one);
      qa[c] = one[0];
      for (int o = 0; o < H; ++o) { scr[L.c1[c] + (size_t)b * H + o] = c1[c][o]; scr[L.c2[c] + (size_t)b * H + o] = c2[c][o]; }
    }
    const float m = 1.0f - r[mbd_sac_off_truncation(O, nu)];
    const float err0 = (qv[0] - tgt) * m, err1 = (qv[1] - tgt) * m;
    const float d3c[2] = {err0 * m, err1 * m};
    const int pick = qa[0] <= qa[1] ? 0 : 1;
    const float d3a[2] = {pick == 0 ? -1.0f : 0.0f, pick == 1 ? -1.0f : 0.0f};
    scr[L.terms + b] = -lpa - (-0.5f * (float)nu);
    scr[L.terms + n + b] = err0 * err0 + err1 * err1;
    scr[L.terms + 2 * n + b] = alpha * lpp - fminf(qa[0], qa[1]);
    float gac[2][32];
    for (int c = 0; c < 2; ++c) {
      scr[L.dc3[c] + b] = d3c[c];
      back(q + mbd_sac_q_w(O, nu, 2, c), 1, &d3c[c], c2[c].data());
      back(q + mbd_sac_q_w(O, nu, 1, c), H, c2[c].data(), c1[c].data());
      for (int o = 0; o < H; ++o) { scr[L.dc2[c] + (size_t)b * H + o] = c2[c][o]; scr[L.dc1[c] + (size_t)b * H + o] = c1[c][o]; }
      back(q + mbd_sac_q_w(O, nu, 2, c), 1, &d3a[c], a2[c].data());
      back(q + mbd_sac_q_w(O, nu, 1, c), H, a2[c].data(), a1[c].data());
      const float* W1 = q + mbd_sac_q_w(O, nu, 0, c);
      for (int j = 0; j < nu; ++j) {
        float acc = 0.0f;
        for (int k = 0; k < H; ++k) acc = acc + W1[(O + j) * H + k] * a1[c][k];
        gac[c][j] = acc;
      }
    }
    for (int j = 0; j < nu; ++j) {
      float dloc, ds;
      mbd_sac_learn_head_grad(gac[0][j] + gac[1][j], tp[j], e2[j], lg[nu + j], alpha, &dloc, &ds);
      dp3[j] = dloc;
      dp3[nu + j] = ds;
    }
    for (int j = 0; j < 2 * nu; ++j) scr[L.dp3 + (size_t)b * 2 * nu + j] = dp3[j];
    back(Pw[2], 2 * nu, dp3.data(), p2.data());
    back(Pw[1], H, p2.data(), p1.data());
    for (int o = 0; o < H; ++o) { scr[L.dp2 + (size_t)b * H + o] = p2[o]; scr[L.dp1 + (size_t)b * H + o] = p1[o]; }
  }
  // the weight phase
  const long long t = step + 1;
  float st, bc2s;
  mbd_sac_adam_scalars(lr, t, &st, &bc2s);
  for (int jb = 0; jb < MBD_SAC_LEARN_JOBS; ++jb) {
    const mbd_sac_learn_job J = mbd_sac_learn_job_of(O, nu, n, jb);
    const float N = J.is_q ? 2.0f * (float)n : (float)n;
    float* P = J.is_q ? q : policy;
    float* M = J.is_q ? qm : pm;
    float* V = J.is_q ? qv : pv;
    float* G = J.is_q ? gq : gpolicy;
    for (int i = 0; i <= J.nin; ++i)
      for (int o = 0; o < J.nout; ++o) {
        float acc = 0.0f;
        for (int b = 0; b < n; ++b) {
          const float a = i < J.nin ? scr[J.in + (size_t)b * J.nin + i] : 1.0f;
          acc = acc + a * scr[J.d + (size_t)b * J.nout + o];
        }
        const int k = i < J.nin ? J.w + i * J.nout + o : J.bias + o;
        const float g = MBD_DIV(acc, N);
        G[k] = g;
        mbd_sac_adam(P + k, M + k, V + k, g, st, bc2s);
        if (J.is_q) target_q[k] = mbd_sac_polyak(target_q[k], P[k], tau);
      }
  }
  float s[3];
  for (int w = 0; w < 3; ++w) {
    s[w] = 0.0f;
    for (int b = 0; b < n; ++b) s[w] = s[w] + scr[L.terms + (size_t)w * n + b];
  }
  const float ga = mbd_expf(log_alpha[0]) * MBD_DIV(s[0], (float)n);
  galpha[0] = ga;
  losses[0] = ga;
  losses[1] = 0.5f * MBD_DIV(s[1], 2.0f * (float)n);
  losses[2] = MBD_DIV(s[2], (float)n);
  mbd_sac_adam_scalars(MBD_SAC_ALPHA_LR, t, &st, &bc2s);
  mbd_sac_adam(log_alpha, amv, amv + 1, ga, st, bc2s);
  return 0;
}

// Adam on an array (the per-element step of the weight phase), for the optimiser checks
int sac_adam_host(float* p, float* m, float* v, const float* g, int n, float lr, long long t) {
  float st, bc2s;
  mbd_sac_adam_scalars(lr, t, &st, &bc2s);
  for (int i = 0; i < n; ++i) mbd_sac_adam(p + i, m + i, v + i, g[i], st, bc2s);
  return 0;
}
int sac_polyak_host(float* target, const float* q, int n, float tau) {
  for (int i = 0; i < n; ++i) target[i] = mbd_sac_polyak(target[i], q[i], tau);
  return 0;
}
int sac_learn_scratch_host(int O, int nu, int n, long long* out) {
  *out = mbd_sac_learn_layout_of(O, nu, n).total;
  return 0;
}
}
