// blackbox.cuh — launch (1) of a black-box optimisation step (upstream mbd/blackbox/mbd_opt.py:64-75): sampling, clip and one
// objective value per sample.  Launches (2) and (3) are the MPPI tail of step_tail.cuh unchanged (mu <- sum_n w_n Y_n,
// mbd_opt.py:76-78), so a step is the same three parameterless, graph-capturable launches as every other solve here.
//
// k_bbo<FN, BATCH>: one CTA of kBboThreads per (sample n, problem b), grid (N, B).  Per element j of sample n:
//   eps   = normal(key_i)[n, j]                        (mbd_random_bits_at(key, n * dim + j, N * dim): jax.random.normal(key, (N, dim)))
//   mean  = Ybars[b][i][j], or on the first step (i == Ndiffuse - 1) normal(init_key_b)[n, j]  (mbd_opt.py:84, mu_0t per sample)
//   Y     = clip(eps * sigma_i + mean, -1, 1)  -> Y0s[b][n][j]
//   X     = x_min + ((x_max - x_min) * (Y + 1)) * 0.5  (the domain map of mbd_opt.py:35; * 0.5 is / 2.0 exactly)
// and the objective's per-element terms (fp32, no contraction; c2pi = fp32(2 pi), cpi = fp32(pi)):
//   Rastrigin  t_j = X * X - 10 * cos(c2pi * X);                     f = fp32(10 dim) + S
//   Ackley     q_j = X * X, c_j = cos(c2pi * X);                      f = ((-20 exp(kb * sqrt(Q)) + -exp(C / dim)) + 20) + fp32(e),
//              kb = fp32(-0.2) / sqrt(dim)
//   Levy       w = 1 + (X - 1) * 0.25; for j < dim - 1: t_j = (w - 1)^2 * (1 + 10 sin(cpi * w + 1)^2);
//              p1 = sin(cpi * w_0)^2, p3 = (w_{dim-1} - 1)^2 * (1 + sin(c2pi * w_{dim-1})^2);  f = (p1 + S) + p3
// Sums (S, Q, C): thread tau adds the terms of elements tau, tau + 256, ... in that order onto 0; the 256 partials are folded
// by an xor butterfly over lanes (offsets 1, 2, 4, 8, 16) and then over the 8 warp sums (1, 2, 4) — an adjacent-pairwise tree
// over the partials in thread order.  J = -f goes to rews[b][n] and is folded into best_hist[b][i] with an order-independent
// float max (Js.max() of mbd_opt.py:80 without a host read).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "mbd_b200.h"
#include "mbd_fp32.h"

namespace mbd {

constexpr int kBboThreads = 256;

struct BboArgs {
  const mbd_step_params* sp;   // [B][nd]: key and sigma of every step
  const mbd_step_ctl* ctl;     // [B]: the step index i (decremented by launch (3))
  const float* Ybars;          // [B][nd][dim]: row i = the mean of step i
  float* Y0s;                  // [B][N][dim]
  float* rews;                 // [B][N]: J = -f
  const uint32_t* init_keys;   // [B][2]: the first step's per-sample mean is normal(init_keys[b], (N, dim))
  float* best_hist;            // [B][nd]: row i = max_n J_n of step i
  int N, dim, nd, prng_part;
  float x_min, x_max;
};

// max over floats by the sign of the stored word: non-negative floats order as signed ints, negative floats in reverse as
// unsigned ints; a negative value can never replace a non-negative one (its unsigned image is larger) and vice versa, so the
// result is the maximum in any arrival order.  best_hist starts at -inf.
__device__ __forceinline__ void bbo_atomic_max(float* p, float v) {
  const int bits = __float_as_int(v);
  if (bits >= 0) atomicMax(reinterpret_cast<int*>(p), bits);
  else atomicMin(reinterpret_cast<unsigned int*>(p), (unsigned int)bits);
}

template <int K>
__device__ __forceinline__ void bbo_block_sum(float (&v)[K], float (*sh)[kBboThreads / 32]) {
#pragma unroll
  for (int k = 0; k < K; ++k)
    for (int o = 1; o < 32; o <<= 1) v[k] = v[k] + __shfl_xor_sync(0xffffffffu, v[k], o);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) sh[k][threadIdx.x >> 5] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      float r = threadIdx.x < kBboThreads / 32 ? sh[k][threadIdx.x] : 0.0f;
      for (int o = 1; o < kBboThreads / 32; o <<= 1) r = r + __shfl_xor_sync(0xffffffffu, r, o);
      v[k] = r;
    }
  }
}

template <int FN, bool BATCH>
__global__ void __launch_bounds__(kBboThreads) k_bbo(const BboArgs a) {
  constexpr float kTwoPi = 6.28318548202514648f;   // fp32(2 pi), what 2.0 * jnp.pi * X rounds the constant to
  constexpr int K = FN == MBD_BBO_ACKLEY ? 2 : 1;
  __shared__ float sh[K][kBboThreads / 32];
  __shared__ float s_p3;
  const unsigned b = batch_y<BATCH>();
  const int n = blockIdx.x;
  const int i = a.ctl[b].i;
  if (i < 1) return;   // replayed past the last step: launches (2) and (3) write nothing either
  const int dim = a.dim, N = a.N;
  const mbd_step_params& p = a.sp[(size_t)b * a.nd + i];
  const uint32_t k0 = p.key[0], k1 = p.key[1];
  const float sigma = p.sigma;
  const bool first = i == a.nd - 1;
  const uint32_t ik0 = a.init_keys[2 * b], ik1 = a.init_keys[2 * b + 1];
  const float* mean_row = a.Ybars + ((size_t)b * a.nd + i) * dim;
  float* y_row = a.Y0s + ((size_t)b * N + n) * dim;
  const uint32_t total = a.prng_part ? 0u : (uint32_t)N * (uint32_t)dim;   // 0 selects the partitionable layout
  const float span = a.x_max - a.x_min;
  float acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0f;
  float p1 = 0.0f;
  for (int j = threadIdx.x; j < dim; j += kBboThreads) {
    const uint32_t idx = (uint32_t)n * (uint32_t)dim + (uint32_t)j;
    const float mean = first ? mbd_bits_to_normal(mbd_random_bits_at(ik0, ik1, idx, total)) : mean_row[j];
    const float y = sample_elem(k0, k1, idx, total, sigma, mean);
    y_row[j] = y;
    const float x = a.x_min + (span * (y + 1.0f)) * 0.5f;
    if constexpr (FN == MBD_BBO_RASTRIGIN) {
      acc[0] += x * x - 10.0f * mbd_cosf(kTwoPi * x);
    } else if constexpr (FN == MBD_BBO_ACKLEY) {
      acc[0] += x * x;
      acc[1] += mbd_cosf(kTwoPi * x);
    } else {
      const float w = 1.0f + (x - 1.0f) * 0.25f;
      const float d = w - 1.0f;
      if (j == 0) { const float s = mbd_sinf(MBD_PI_F * w); p1 = s * s; }
      if (j < dim - 1) {
        const float s = mbd_sinf(MBD_PI_F * w + 1.0f);
        acc[0] += (d * d) * (1.0f + 10.0f * (s * s));
      } else {
        const float s = mbd_sinf(kTwoPi * w);
        s_p3 = (d * d) * (1.0f + s * s);
      }
    }
  }
  bbo_block_sum<K>(acc, sh);   // its __syncthreads also publishes s_p3
  if (threadIdx.x != 0) return;
  float f;
  if constexpr (FN == MBD_BBO_RASTRIGIN) {
    f = (float)(10 * dim) + acc[0];
  } else if constexpr (FN == MBD_BBO_ACKLEY) {
    const float kb = MBD_DIV(-0.2f, MBD_SQRT((float)dim));
    const float part1 = -20.0f * mbd_expf(kb * MBD_SQRT(acc[0]));
    const float part2 = -mbd_expf(MBD_DIV(acc[1], (float)dim));
    f = ((part1 + part2) + 20.0f) + 2.71828174591064453f;   // fp32(e)
  } else {
    f = (p1 + acc[0]) + s_p3;
  }
  const float J = -f;
  a.rews[(size_t)b * N + n] = J;
  bbo_atomic_max(a.best_hist + (size_t)b * a.nd + i, J);
}

}  // namespace mbd
