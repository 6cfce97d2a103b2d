/* mbd_sac.h — the arithmetic of the SAC acting step and replay sampler (csrc/sac.cuh), compiled for the device and for the host
 * harness (tests/host_sac/), so that both produce the same bits (nvcc -fmad=false / gcc -ffp-contract=off, include/mbd_fp32.h).
 *
 * [brax-recalled] brax.training.agents.sac.networks (v0.10.x): policy = MLP(normalize(obs)), hidden (256, 256), ReLU between layers,
 * none after the last, 2 Nu outputs; the action distribution is PPO's NormalTanh (include/mbd_ppo.h: mbd_ppo_head, mbd_ppo_eps).
 * Flat policy layout (mbd_b200/rl/networks.py): W1 [O][256] (in, out), b1 [256], W2 [256][256], b2 [256], W3 [256][2 Nu], b3 [2 Nu].
 * Unit o of a layer is mbd_ppo_dense: inputs summed in ascending order from 0.0f, the bias added last; relu(x) = fmaxf(x, 0).
 *
 * Replay row (one transition, float32): obs [O] | action [Nu] (= tanh(raw)) | reward | discount (1 - done) | next_obs [O] | truncation.
 *
 * [jax-recalled] jax.random.randint(key, shape, 0, span) with 32-bit words: k1, k2 = split(key); hi = bits(k1), lo = bits(k2);
 * mult = ((2^16 % span)^2) % span; offset = ((hi % span) * mult + lo % span) % span; every operation uint32 with wrap-around, and
 * span = 1 when maxval <= minval.  Restated exactly, wrap included (at span = 2^20 mult is 0 and the offset is lo % span). */
#ifndef MBD_SAC_H_
#define MBD_SAC_H_

#include "mbd_ppo.h"

#define MBD_SAC_HIDDEN 256
#define MBD_SAC_LAYERS 3

/* number of floats of the flat policy parameters */
MBD_HD int mbd_sac_policy_size(int O, int nu) {
  const int h = MBD_SAC_HIDDEN;
  return O * h + h + h * h + h + h * 2 * nu + 2 * nu;
}
/* offset of W_l (l = 0 .. 2) in the flat policy buffer; its bias follows the weights */
MBD_HD int mbd_sac_layer_offset(int O, int l) {
  const int h = MBD_SAC_HIDDEN;
  return l == 0 ? 0 : l == 1 ? O * h + h : O * h + h + h * h + h;
}
/* floats of one replay row and the offsets of its fields */
MBD_HD int mbd_sac_row(int O, int nu) { return 2 * O + nu + 3; }
MBD_HD int mbd_sac_off_action(int O) { return O; }
MBD_HD int mbd_sac_off_reward(int O, int nu) { return O + nu; }
MBD_HD int mbd_sac_off_discount(int O, int nu) { return O + nu + 1; }
MBD_HD int mbd_sac_off_next_obs(int O, int nu) { return O + nu + 2; }
MBD_HD int mbd_sac_off_truncation(int O, int nu) { return 2 * O + nu + 2; }

MBD_HD float mbd_sac_relu(float x) { return fmaxf(x, 0.0f); }

/* hidden unit o of layer l < 2: relu(mbd_ppo_dense) */
MBD_HD float mbd_sac_hidden(const float* x, const float* W, const float* b, int nin, int o) {
  return mbd_sac_relu(mbd_ppo_dense(x, W, b, nin, MBD_SAC_HIDDEN, o));
}

/* split(key, 2) in the threefry layout `part` (mbd_set_prng_layout): out = {key 0 word 0, word 1, key 1 word 0, word 1} */
MBD_HD void mbd_sac_split2(uint32_t k0, uint32_t k1, int part, uint32_t* out) {
  uint32_t a0, a1, b0, b1;
  if (part) {   /* key i = both words of block (0, i) */
    mbd_threefry2x32(k0, k1, 0u, 0u, &a0, &a1);
    mbd_threefry2x32(k0, k1, 0u, 1u, &b0, &b1);
    out[0] = a0; out[1] = a1; out[2] = b0; out[3] = b1;
  } else {      /* bits(key, 4): blocks (0, 2) and (1, 3); keys = rows of [o0(0), o0(1), o1(0), o1(1)] */
    mbd_threefry2x32(k0, k1, 0u, 2u, &a0, &a1);
    mbd_threefry2x32(k0, k1, 1u, 3u, &b0, &b1);
    out[0] = a0; out[1] = b0; out[2] = a1; out[3] = b1;
  }
}

/* randint's multiplier for span (uint32, wrapping) */
MBD_HD uint32_t mbd_sac_randint_mult(uint32_t span) {
  const uint32_t m = 65536u % span;
  return (m * m) % span;
}
/* randint's offset from the two bit words of an element */
MBD_HD uint32_t mbd_sac_randint(uint32_t hi, uint32_t lo, uint32_t span, uint32_t mult) {
  return ((hi % span) * mult + lo % span) % span;
}
/* physical ring row of logical row i: the ring holds the last `size` inserted rows, oldest first, and `pos` is the next write row
 * (pos < cap, i < size <= cap <= 2^24, so the sum stays far below 2^32) */
MBD_HD uint32_t mbd_sac_ring_row(uint32_t pos, uint32_t size, uint32_t cap, uint32_t i) {
  return (pos + cap - size + i) % cap;
}

#endif /* MBD_SAC_H_ */
