// include/mbd_sac.h built for the host (tests/test_sac_cpu.py, tests/test_sac_gpu.py): the acting step of k_sac_act env by env, and
// the replay sampler's arithmetic.
#include "mbd_sac.h"

extern "C" {
// policy: flat parameters; obs [B][O]; eps [B][nu] -> act, raw [B][nu], logp [B]
int sac_act_host(const float* policy, const float* mean, const float* std, const float* obs, const float* eps, int B, int O, int nu,
                 float* act, float* raw, float* logp) {
  const int H = MBD_SAC_HIDDEN;
  static float x[MBD_SAC_HIDDEN], h[MBD_SAC_HIDDEN];
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < O; ++i) x[i] = mbd_ppo_norm(obs[b * O + i], mean[i], std[i]);
    int nin = O;
    for (int l = 0; l < MBD_SAC_LAYERS - 1; ++l) {
      const float* W = policy + mbd_sac_layer_offset(O, l);
      for (int o = 0; o < H; ++o) h[o] = mbd_sac_hidden(x, W, W + nin * H, nin, o);
      for (int o = 0; o < H; ++o) x[o] = h[o];
      nin = H;
    }
    const float* W3 = policy + mbd_sac_layer_offset(O, MBD_SAC_LAYERS - 1);
    for (int o = 0; o < 2 * nu; ++o) h[o] = mbd_ppo_dense(x, W3, W3 + H * 2 * nu, H, 2 * nu, o);
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
// split(key, 2) in layout `part`: out [4]
int sac_split2_host(uint32_t k0, uint32_t k1, int part, uint32_t* out) {
  mbd_sac_split2(k0, k1, part, out);
  return 0;
}
// randint offsets from bit words hi / lo [n]
int sac_randint_host(const uint32_t* hi, const uint32_t* lo, int n, uint32_t span, uint32_t* out) {
  const uint32_t mult = mbd_sac_randint_mult(span);
  for (int i = 0; i < n; ++i) out[i] = mbd_sac_randint(hi[i], lo[i], span, mult);
  return 0;
}
}
