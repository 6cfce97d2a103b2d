// sac.cuh — the SAC acting step, the replay record and the replay sampler (mbd_sac_* in include/mbd_b200.h).
// k_sac_act: a CTA of 256 threads takes a tile of kSacTile envs, thread o = hidden unit o.  The 276 KB policy of hopper does not fit
// in shared memory, so the tile's layer inputs sit in shared memory instead and every weight is read from L2 once per tile.  Each
// thread keeps one accumulator per env and runs the inputs in ascending order, which is mbd_ppo_dense's order (include/mbd_sac.h).
#pragma once
#include "mbd_sac.h"

namespace mbd {

constexpr int kSacThreads = MBD_SAC_HIDDEN;
constexpr int kSacTile = 8;            // envs per CTA
constexpr int kSacSampleThreads = 256;

// the last CTA of a launch advances the control words ctl[0..1] (every CTA has read them by then); ticket ctl[tk]
__device__ __forceinline__ bool sac_last_cta(int32_t* ticket) {
  __syncthreads();
  if (threadIdx.x != 0) return false;
  __threadfence();
  if (atomicAdd(ticket, 1) != (int)gridDim.x - 1) return false;
  *ticket = 0;
  return true;
}

__global__ void __launch_bounds__(kSacThreads) k_sac_act(mbd_sac_plan p, int mode, int part) {
  __shared__ float xs[kSacTile][MBD_SAC_HIDDEN];
  __shared__ float hs[kSacTile][MBD_SAC_HIDDEN];
  __shared__ float outs[kSacTile][2 * MBD_PPO_MAX_NU];
  const int O = p.O, nu = p.nu, B = p.B, H = MBD_SAC_HIDDEN, R = mbd_sac_row(O, nu);
  const int o = threadIdx.x;
  const int e0 = blockIdx.x * kSacTile;
  const int ne = min(kSacTile, B - e0);
  const bool acting = mode != MBD_SAC_EVAL_RECORD;
  const int t = p.act_ctl_dev[0];
  const int krow = p.act_ctl_dev[1];
  const uint32_t pos = mode == MBD_SAC_ACT ? (uint32_t)p.ring_ctl_dev[0] : 0u;
  const bool inside = !acting || krow < p.act_key_rows;
  uint32_t k0 = 0, k1 = 0;
  if (acting && inside) { k0 = p.act_keys_dev[2 * krow]; k1 = p.act_keys_dev[2 * krow + 1]; }
  if (mode != MBD_SAC_ACT && t > 0 && o < ne && inside) {   // EvalWrapper: the return of the first episode of every env
    const int b = e0 + o;
    const float a = p.active_dev[b];
    p.ret_dev[b] = p.ret_dev[b] + a * p.env_reward_dev[b];
    p.active_dev[b] = a * (1.0f - p.env_done_dev[b]);
  }
  if (acting && inside) {
    for (int q = o; q < ne * O; q += blockDim.x) {
      const int e = q / O, i = q - e * O, b = e0 + e;
      const float ob = p.env_obs_dev[(size_t)b * O + i];
      xs[e][i] = mbd_ppo_norm(ob, p.mean_dev[i], p.std_dev[i]);
      if (mode == MBD_SAC_ACT) {
        p.stage_obs_dev[(size_t)b * O + i] = ob;
        p.ring_dev[(size_t)((pos + (uint32_t)b) % (uint32_t)p.capacity) * R + i] = ob;
      }
    }
    __syncthreads();
    // two hidden layers: acc[e] = sum_i x[e][i] W[i][o], i ascending, then + b[o], relu
    int nin = O;
    float (*src)[MBD_SAC_HIDDEN] = xs;
    float (*dst)[MBD_SAC_HIDDEN] = hs;
    for (int l = 0; l < MBD_SAC_LAYERS - 1; ++l) {
      const float* W = p.policy_dev + mbd_sac_layer_offset(O, l);
      float acc[kSacTile];
#pragma unroll
      for (int e = 0; e < kSacTile; ++e) acc[e] = 0.0f;
      for (int i = 0; i < nin; ++i) {
        const float w = __ldg(W + (size_t)i * H + o);
#pragma unroll
        for (int e = 0; e < kSacTile; ++e) acc[e] = acc[e] + src[e][i] * w;
      }
      const float bo = __ldg(W + (size_t)nin * H + o);
#pragma unroll
      for (int e = 0; e < kSacTile; ++e) dst[e][o] = mbd_sac_relu(acc[e] + bo);
      __syncthreads();
      float (*tmp)[MBD_SAC_HIDDEN] = src;
      src = dst;
      dst = tmp;
      nin = H;
    }
    // output layer: pair (e, j) of the tile, j < 2 Nu
    const float* W3 = p.policy_dev + mbd_sac_layer_offset(O, MBD_SAC_LAYERS - 1);
    for (int q = o; q < ne * 2 * nu; q += blockDim.x) {
      const int e = q / (2 * nu), j = q - e * 2 * nu;
      outs[e][j] = mbd_ppo_dense(src[e], W3, W3 + H * 2 * nu, H, 2 * nu, j);
    }
    __syncthreads();
    for (int q = o; q < ne * nu; q += blockDim.x) {
      const int e = q / nu, j = q - e * nu, b = e0 + e;
      float raw, act, lp;
      mbd_ppo_head(outs[e][j], outs[e][nu + j], mbd_ppo_eps(k0, k1, b, j, B, nu, part), &raw, &act, &lp);
      p.env_actions_dev[(size_t)b * nu + j] = act;
      if (mode == MBD_SAC_ACT)
        p.ring_dev[(size_t)((pos + (uint32_t)b) % (uint32_t)p.capacity) * R + mbd_sac_off_action(O) + j] = act;
    }
  }
  if (sac_last_cta(&p.act_ctl_dev[2])) {
    if (mode == MBD_SAC_EVAL_RECORD) {
      p.act_ctl_dev[0] = 0;
    } else {
      p.act_ctl_dev[0] = t + 1;
      p.act_ctl_dev[1] = krow + 1;
    }
    __threadfence();
  }
}

// the second half of a transition: element q = b * (O + 3) + w of the B envs' reward, discount, truncation and next obs
__global__ void __launch_bounds__(256) k_sac_record(mbd_sac_plan p) {
  const int O = p.O, nu = p.nu, R = mbd_sac_row(O, nu), per = O + 3;
  const uint32_t pos = (uint32_t)p.ring_ctl_dev[0], size = (uint32_t)p.ring_ctl_dev[1], cap = (uint32_t)p.capacity;
  const int n = p.B * per;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
    const int b = q / per, w = q - b * per;
    float* row = p.ring_dev + (size_t)((pos + (uint32_t)b) % cap) * R;
    if (w < O) row[mbd_sac_off_next_obs(O, nu) + w] = p.env_obs_dev[(size_t)b * O + w];
    else if (w == O) row[mbd_sac_off_reward(O, nu)] = p.env_reward_dev[b];
    else if (w == O + 1) row[mbd_sac_off_discount(O, nu)] = 1.0f - p.env_done_dev[b];
    else row[mbd_sac_off_truncation(O, nu)] = p.env_trunc_dev[b];
  }
  if (sac_last_cta(&p.ring_ctl_dev[2])) {
    p.ring_ctl_dev[0] = (int32_t)((pos + (uint32_t)p.B) % cap);
    p.ring_ctl_dev[1] = (int32_t)min(size + (uint32_t)p.B, cap);
    __threadfence();
  }
}

// One launch per training step.  Every thread derives (new buffer key, sample key) = split(buffer key) and (k1, k2) =
// split(sample key) itself; warp w draws the indices of rows 32 w .. 32 w + 31 (lane = row) and copies those rows, lane = word;
// the grid-stride loop over the three noise tensors follows.  The last CTA stores the new buffer key and s + 1.
__global__ void __launch_bounds__(kSacSampleThreads, 4) k_sac_sample(mbd_sac_plan p, int part) {
  const int O = p.O, nu = p.nu, R = mbd_sac_row(O, nu);
  const int s = p.sample_ctl_dev[0];
  const bool inside = s < p.noise_key_rows;
  const uint32_t bk0 = (uint32_t)p.sample_ctl_dev[2], bk1 = (uint32_t)p.sample_ctl_dev[3];
  uint32_t kb[4], kh[4];
  mbd_sac_split2(bk0, bk1, part, kb);           // kb[0..1]: the next buffer key, kb[2..3]: the sample key
  mbd_sac_split2(kb[2], kb[3], part, kh);       // kh[0..1]: k1 (high words), kh[2..3]: k2 (low words)
  const uint32_t nb0 = kb[0], nb1 = kb[1], h0 = kh[0], h1 = kh[1], l0 = kh[2], l1 = kh[3];
  const uint32_t total = (uint32_t)p.updates * (uint32_t)p.batch;
  const uint32_t size = (uint32_t)p.ring_ctl_dev[1], pos = (uint32_t)p.ring_ctl_dev[0], cap = (uint32_t)p.capacity;
  const uint32_t span = size == 0u ? 1u : size;
  const uint32_t mult = mbd_sac_randint_mult(span);
  const uint32_t cnt = part ? 0u : total;
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t w0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; inside && w0 * 32u < total; w0 += warps) {
    const uint32_t e = w0 * 32u + lane;
    uint32_t phys = 0u;
    if (e < total) {
      const uint32_t off = mbd_sac_randint(mbd_random_bits_at(h0, h1, e, cnt), mbd_random_bits_at(l0, l1, e, cnt), span, mult);
      p.idx_dev[e] = (int32_t)off;
      phys = mbd_sac_ring_row(pos, size, cap, off);
    }
    const int rows = (int)min(32u, total - w0 * 32u);
    for (int r = 0; r < rows; ++r) {
      const uint32_t ph = __shfl_sync(0xffffffffu, phys, r);
      const float* src = p.ring_dev + (size_t)ph * R;
      float* dst = p.batch_dev + (size_t)(w0 * 32u + r) * R;
      for (int c = lane; c < R; c += 32) dst[c] = src[c];
    }
  }
  const uint32_t per = (uint32_t)p.batch * (uint32_t)nu;        // one normal tensor (batch, Nu)
  const uint32_t ntot = 3u * (uint32_t)p.updates * per;
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; inside && q < ntot; q += gridDim.x * blockDim.x) {
    const uint32_t which = q / ((uint32_t)p.updates * per);
    const uint32_t rem = q - which * (uint32_t)p.updates * per;
    const uint32_t g = rem / per, i = rem - g * per;
    const uint32_t* key = p.noise_keys_dev + (((size_t)s * p.updates + g) * 3 + which) * 2;
    p.eps_dev[q] = mbd_bits_to_normal(mbd_random_bits_at(key[0], key[1], i, part ? 0u : per));
  }
  if (sac_last_cta(&p.sample_ctl_dev[1])) {
    p.sample_ctl_dev[0] = s + 1;
    p.sample_ctl_dev[2] = (int32_t)nb0;
    p.sample_ctl_dev[3] = (int32_t)nb1;
    __threadfence();
  }
}

}  // namespace mbd
