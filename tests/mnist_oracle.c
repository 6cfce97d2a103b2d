/* mnist_oracle.c — CPU restatement of the SIMT remainder of k_mnist_fwd<false> (csrc/mnist.cuh) (TEST INFRASTRUCTURE).
 *
 * Given the layer-1 pre-activations Z1 the device returns, this repeats everything after layer 1 in the device's fp32 order:
 * h1 = fmaxf(z1 + b1, 0); layers 2 and 3 summed k = 0 .. 31 from 0, then + bias; ReLU; mx = max over the classes in order;
 * s = z - mx; lse = mbd_logf(sum of mbd_expf(s) in class order); the label's s - lse; thread tau's running sum over images
 * tau, tau + 256, ...; the 256 partials folded by the lane / warp xor butterflies (an adjacent-pairwise tree); J = sum / M.
 * Compile with contraction off (-ffp-contract=off): an FMA happens only where mbd_fp32.h writes fmaf().
 * tests/mnist_oracle.py builds and loads it.                                                                                 */
#include <stddef.h>
#include <stdint.h>

#include "mbd_fp32.h"

#define THREADS 256
#define IN 784
#define H 32
#define OUT 10
#define OFF_B1 (IN * H)
#define OFF_W2 (OFF_B1 + H)
#define OFF_B2 (OFF_W2 + H * H)
#define OFF_W3 (OFF_B2 + H)
#define OFF_B3 (OFF_W3 + H * OUT)
#define HNU (OFF_B3 + OUT)

/* lp[label] of one image from its layer-1 pre-activations */
static float image_term(const float* row, const float* z1, int label) {
  float h1[H], h2[H], z3[OUT];
  for (int o = 0; o < H; ++o) {
    const float a = z1[o] + row[OFF_B1 + o];
    h1[o] = a > 0.0f ? a : 0.0f;
  }
  for (int o = 0; o < H; ++o) {
    float s = 0.0f;
    for (int k = 0; k < H; ++k) s = s + h1[k] * row[OFF_W2 + k * H + o];
    const float z = s + row[OFF_B2 + o];
    h2[o] = z > 0.0f ? z : 0.0f;
  }
  for (int o = 0; o < OUT; ++o) {
    float s = 0.0f;
    for (int k = 0; k < H; ++k) s = s + h2[k] * row[OFF_W3 + k * OUT + o];
    z3[o] = s + row[OFF_B3 + o];
  }
  float mx = z3[0];
  for (int o = 1; o < OUT; ++o) mx = z3[o] > mx ? z3[o] : mx;
  float se = 0.0f;
  for (int o = 0; o < OUT; ++o) { z3[o] = z3[o] - mx; se = se + mbd_expf(z3[o]); }
  return z3[label] - mbd_logf(se);
}

/* Js[n] of rows [n_models][HNU] from z1 [n_models][M][32] and the labels of the M images */
__attribute__((visibility("default"))) void mnist_js(const float* rows, const float* z1, const uint8_t* labels, int n_models, int M,
                                                     float* Js) {
  for (int n = 0; n < n_models; ++n) {
    const float* row = rows + (size_t)n * HNU;
    float p[THREADS];
    for (int t = 0; t < THREADS; ++t) {
      float acc = 0.0f;
      for (int m = t; m < M; m += THREADS) acc = acc + image_term(row, z1 + ((size_t)n * M + m) * H, labels[m]);
      p[t] = acc;
    }
    for (int w = THREADS; w > 1; w >>= 1)
      for (int k = 0; k < w / 2; ++k) p[k] = p[2 * k] + p[2 * k + 1];
    Js[n] = p[0] / (float)M;
  }
}
