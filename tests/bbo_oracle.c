/* bbo_oracle.c — CPU oracle of the black-box objectives of csrc/blackbox.cuh (TEST INFRASTRUCTURE).
 *
 * The same fp32 arithmetic in the same order as k_bbo, written out sample by sample: the per-element terms with
 * include/mbd_fp32.h's sin / cos / exp / sqrt, one running sum per "thread" tau (elements tau, tau + 256, ...), the 256
 * partials folded by an adjacent-pairwise tree.  Compile with contraction off (-ffp-contract=off): an FMA happens only where
 * mbd_fp32.h writes fmaf().  tests/bbo_oracle.py builds and loads it.                                                       */
#include <stdint.h>
#include <string.h>

#include "mbd_fp32.h"

#define BBO_THREADS 256
#define BBO_ACKLEY 1
#define BBO_RASTRIGIN 2
#define BBO_LEVY 3

/* the xor butterfly of k_bbo over 256 lanes: level by level, element 2k becomes p[2k] + p[2k + 1] */
static float tree256(float* p) {
  for (int n = BBO_THREADS; n > 1; n >>= 1)
    for (int k = 0; k < n / 2; ++k) p[k] = p[2 * k] + p[2 * k + 1];
  return p[0];
}

static float eval_one(int fn, const float* y, int dim, float x_min, float x_max) {
  const float c2pi = 6.28318548202514648f;
  const float span = x_max - x_min;
  float s[BBO_THREADS], c[BBO_THREADS];
  memset(s, 0, sizeof(s));
  memset(c, 0, sizeof(c));
  float p1 = 0.0f, p3 = 0.0f;
  for (int j = 0; j < dim; ++j) {
    const int t = j % BBO_THREADS;
    const float x = x_min + (span * (y[j] + 1.0f)) * 0.5f;
    if (fn == BBO_RASTRIGIN) {
      s[t] += x * x - 10.0f * mbd_cosf(c2pi * x);
    } else if (fn == BBO_ACKLEY) {
      s[t] += x * x;
      c[t] += mbd_cosf(c2pi * x);
    } else {
      const float w = 1.0f + (x - 1.0f) * 0.25f;
      const float d = w - 1.0f;
      if (j == 0) { const float q = mbd_sinf(MBD_PI_F * w); p1 = q * q; }
      if (j < dim - 1) {
        const float q = mbd_sinf(MBD_PI_F * w + 1.0f);
        s[t] += (d * d) * (1.0f + 10.0f * (q * q));
      } else {
        const float q = mbd_sinf(c2pi * w);
        p3 = (d * d) * (1.0f + q * q);
      }
    }
  }
  const float S = tree256(s);
  float f;
  if (fn == BBO_RASTRIGIN) {
    f = (float)(10 * dim) + S;
  } else if (fn == BBO_ACKLEY) {
    const float C = tree256(c);
    const float kb = -0.2f / sqrtf((float)dim);
    const float part1 = -20.0f * mbd_expf(kb * sqrtf(S));
    const float part2 = -mbd_expf(C / (float)dim);
    f = ((part1 + part2) + 20.0f) + 2.71828174591064453f;
  } else {
    f = (p1 + S) + p3;
  }
  return -f;
}

/* J = -f(Y0s[n]) for n < N; Y0s [N][dim].  Returns -1 for an unknown fn. */
__attribute__((visibility("default"))) int bbo_eval(int fn, const float* Y0s, int N, int dim, float x_min, float x_max, float* J) {
  if (fn < BBO_ACKLEY || fn > BBO_LEVY || dim < 1) return -1;
  for (int n = 0; n < N; ++n) J[n] = eval_one(fn, Y0s + (size_t)n * dim, dim, x_min, x_max);
  return 0;
}
