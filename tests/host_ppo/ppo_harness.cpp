// include/mbd_ppo.h built for the host (tests/test_ppo_cpu.py, tests/test_ppo_gpu.py): the acting step of k_ppo_act, env by env.
#include "mbd_ppo.h"

extern "C" {
// policy: flat parameters; obs [B][O]; eps [B][nu] -> act, raw [B][nu], logp [B]
int ppo_act_host(const float* policy, const float* mean, const float* std, const float* obs, const float* eps, int B, int O, int nu,
                 float* act, float* raw, float* logp) {
  const int H = MBD_PPO_HIDDEN;
  float x[128], h[64];
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < O; ++i) x[i] = mbd_ppo_norm(obs[b * O + i], mean[i], std[i]);
    int nin = O;
    for (int l = 0; l < MBD_PPO_LAYERS - 1; ++l) {
      const float* W = policy + mbd_ppo_layer_offset(O, l);
      for (int o = 0; o < H; ++o) h[o] = mbd_swishf(mbd_ppo_dense(x, W, W + nin * H, nin, H, o));
      for (int o = 0; o < H; ++o) x[o] = h[o];
      nin = H;
    }
    const float* W5 = policy + mbd_ppo_layer_offset(O, MBD_PPO_LAYERS - 1);
    for (int o = 0; o < 2 * nu; ++o) h[o] = mbd_ppo_dense(x, W5, W5 + H * 2 * nu, H, 2 * nu, o);
    float s = 0.0f;
    for (int j = 0; j < nu; ++j) {
      float lp;
      mbd_ppo_head(h[j], h[nu + j], eps[b * nu + j], &raw[b * nu + j], &act[b * nu + j], &lp);
      s = s + lp;
    }
    logp[b] = s;
  }
  return 0;
}
// the header's composite functions elementwise (tests/test_fp32_spec.py): fn 0 = mbd_tanhf, 1 = mbd_softplusf, 2 = mbd_swishf
int ppo_fmap_host(int fn, const float* x, int n, float* out) {
  for (int i = 0; i < n; ++i) out[i] = fn == 0 ? mbd_tanhf(x[i]) : fn == 1 ? mbd_softplusf(x[i]) : mbd_swishf(x[i]);
  return 0;
}
// eps of env b, component j from the key (the in-kernel sampler)
int ppo_eps_host(uint32_t k0, uint32_t k1, int B, int nu, int part, float* eps) {
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < nu; ++j) eps[b * nu + j] = mbd_ppo_eps(k0, k1, b, j, B, nu, part);
  return 0;
}
}
