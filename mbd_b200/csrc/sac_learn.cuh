// sac_learn.cuh — the fused SAC gradient update (mbd_sac_update in include/mbd_b200.h): two launches, no float atomics.
// k_sac_learn_rows: a CTA of 256 threads takes kSlTile batch rows, thread o = hidden unit o.  It runs the policy on xn and the target
// critics (the target), the policy on x (the three heads), both critics on the stack (x, action) | (x, tanh raw_p) (2 kSlTile rows,
// same weights), forms each row's loss terms and backpropagates the critic and actor seeds to every layer's pre-activation.  The
// activations and deltas the weight gradients need go to the scratch buffer (include/mbd_sac_learn.h's layout); every layer input
// sits in shared memory as [unit][row], so a weight is read once per tile and the rows of a unit are two 16-byte loads.
// k_sac_learn_weights: a CTA takes a 64 x 64 tile of one of the nine dW matrices (thread = 4 x 4 outputs, strided by 16), sums over
// the batch in ascending row order and applies Adam (and the Polyak step for Q) to the parameters it owns; the last CTA reduces the
// three loss terms and steps log alpha, then advances the Adam step count and upd_ctl.
#pragma once
#include "mbd_sac_learn.h"

namespace mbd {

constexpr int kSlThreads = MBD_SAC_HIDDEN;
constexpr int kSlTile = 4;                   // batch rows per CTA (batch 512: 128 CTAs)
constexpr int kSlStack = 2 * kSlTile;        // the critic stack: critic rows, then actor rows
constexpr int kSlMaxIn = MBD_PPO_MAX_OBS + MBD_PPO_MAX_NU;
constexpr int kSwTile = 64, kSwK = 32;       // weight phase: output tile, rows per shared-memory stage

// shared memory of k_sac_learn_rows (floats; T = kSlTile rows, S = kSlStack)
constexpr int kSlOffXs = 0;                                        // [O][T] x
constexpr int kSlOffXn = kSlOffXs + MBD_PPO_MAX_OBS * kSlTile;     // [O][T] xn
constexpr int kSlOffQi = kSlOffXn + MBD_PPO_MAX_OBS * kSlTile;     // [O + Nu][S] the critic stack's input
constexpr int kSlOffC1 = kSlOffQi + kSlMaxIn * kSlStack;           // [2][256][S] critic h1 (then d1)
constexpr int kSlOffC2 = kSlOffC1 + 2 * MBD_SAC_HIDDEN * kSlStack; // [2][256][S] critic h2 (then d2)
constexpr int kSlOffP1 = kSlOffC2 + 2 * MBD_SAC_HIDDEN * kSlStack; // [256][T] policy h1 on x (then d1)
constexpr int kSlOffP2 = kSlOffP1 + MBD_SAC_HIDDEN * kSlTile;      // [256][T] policy h2 on x (then d2)
constexpr int kSlOffLg = kSlOffP2 + MBD_SAC_HIDDEN * kSlTile;      // [2 Nu][T] logits on x (then the policy's d3)
constexpr int kSlOffLn = kSlOffLg + 2 * MBD_PPO_MAX_NU * kSlTile;  // [2 Nu][T] logits on xn
constexpr int kSlOffTp = kSlOffLn + 2 * MBD_PPO_MAX_NU * kSlTile;  // [Nu][T] tanh raw_p
constexpr int kSlOffL0 = kSlOffTp + MBD_PPO_MAX_NU * kSlTile;      // [Nu][T] log-prob terms (eps 0, then eps 1)
constexpr int kSlOffL2 = kSlOffL0 + MBD_PPO_MAX_NU * kSlTile;      // [Nu][T] log-prob terms (eps 2)
constexpr int kSlOffGa = kSlOffL2 + MBD_PPO_MAX_NU * kSlTile;      // [2][Nu][T] action gradient through critic c
constexpr int kSlOffQo = kSlOffGa + 2 * MBD_PPO_MAX_NU * kSlTile;  // [2][S] critic outputs; [2][T] target critic outputs follow
constexpr int kSlOffD3 = kSlOffQo + 2 * kSlStack + 2 * kSlTile;    // [2][S] critic seeds
constexpr int kSlOffRow = kSlOffD3 + 2 * kSlStack;                 // [T] per row: target, lp_c, lp_a, lp_p, alpha scalar at [4][0]
constexpr int kSlFloats = kSlOffRow + 5 * kSlTile;
constexpr size_t kSlSmem = (size_t)kSlFloats * sizeof(float);

// dst[o][e] = (relu of) sum_i src[i][e] W[i][o] (i ascending from 0.0f) + b[o]; thread o, NR rows
template <int NR, bool RELU>
__device__ __forceinline__ void sl_dense(const float* __restrict__ W, const float* __restrict__ b, int nin, const float* src,
                                         float* dst) {
  const int o = threadIdx.x;
  float acc[NR];
#pragma unroll
  for (int e = 0; e < NR; ++e) acc[e] = 0.0f;
  for (int i = 0; i < nin; ++i) {
    const float w = __ldg(W + (size_t)i * MBD_SAC_HIDDEN + o);
    const float4* s4 = reinterpret_cast<const float4*>(src + i * NR);
#pragma unroll
    for (int q = 0; q < NR / 4; ++q) {
      const float4 v = s4[q];
      acc[4 * q + 0] = acc[4 * q + 0] + v.x * w;
      acc[4 * q + 1] = acc[4 * q + 1] + v.y * w;
      acc[4 * q + 2] = acc[4 * q + 2] + v.z * w;
      acc[4 * q + 3] = acc[4 * q + 3] + v.w * w;
    }
  }
  const float bo = __ldg(b + o);
#pragma unroll
  for (int e = 0; e < NR; ++e) {
    const float y = acc[e] + bo;
    dst[o * NR + e] = RELU ? mbd_sac_relu(y) : y;
  }
}

// the small output layer (256 -> nout): dst[j][e] = sum_i src[i][e] W[i][j] + b[j], thread = (e, j)
template <int NR>
__device__ __forceinline__ void sl_out(const float* __restrict__ W, const float* __restrict__ b, int nout, const float* src,
                                       float* dst) {
  for (int q = threadIdx.x; q < NR * nout; q += blockDim.x) {
    const int e = q / nout, j = q - e * nout;
    float acc = 0.0f;
    for (int i = 0; i < MBD_SAC_HIDDEN; ++i) acc = acc + src[i * NR + e] * __ldg(W + i * nout + j);
    dst[j * NR + e] = acc + __ldg(b + j);
  }
}

// backward through W [256][nout]: hd[o][e] = sum_k W[o][k] src[k][e] (k ascending from 0.0f) where hd[o][e] (the layer input's
// activation, overwritten in place) is > 0, else 0; thread o
template <int NR>
__device__ __forceinline__ void sl_back(const float* __restrict__ W, int nout, const float* src, float* hd) {
  const int o = threadIdx.x;
  float acc[NR];
#pragma unroll
  for (int e = 0; e < NR; ++e) acc[e] = 0.0f;
  const float* Wr = W + (size_t)o * nout;
  for (int k = 0; k < nout; ++k) {
    const float w = __ldg(Wr + k);
    const float4* s4 = reinterpret_cast<const float4*>(src + k * NR);
#pragma unroll
    for (int q = 0; q < NR / 4; ++q) {
      const float4 v = s4[q];
      acc[4 * q + 0] = acc[4 * q + 0] + w * v.x;
      acc[4 * q + 1] = acc[4 * q + 1] + w * v.y;
      acc[4 * q + 2] = acc[4 * q + 2] + w * v.z;
      acc[4 * q + 3] = acc[4 * q + 3] + w * v.w;
    }
  }
#pragma unroll
  for (int e = 0; e < NR; ++e) hd[o * NR + e] = hd[o * NR + e] > 0.0f ? acc[e] : 0.0f;
}

// rows [e0, e0 + ne) of a shared [256][NR] buffer (row offset r0) to the scratch matrix [n][256]
template <int NR>
__device__ __forceinline__ void sl_store(const float* s, int r0, float* g, int b0, int ne) {
  for (int q = threadIdx.x; q < ne * MBD_SAC_HIDDEN; q += blockDim.x) {
    const int e = q / MBD_SAC_HIDDEN, o = q - e * MBD_SAC_HIDDEN;
    g[(size_t)(b0 + e) * MBD_SAC_HIDDEN + o] = s[o * NR + r0 + e];
  }
}

__global__ void __launch_bounds__(kSlThreads) k_sac_learn_rows(mbd_sac_learn_plan p) {
  extern __shared__ float4 sl_smem4[];
  float* sm = reinterpret_cast<float*>(sl_smem4);
  const int O = p.O, nu = p.nu, n = p.batch, R = mbd_sac_row(O, nu), QI = O + nu, T = kSlTile, S = kSlStack;
  const long long g = p.upd_ctl_dev[0];
  if (g < 0 || g >= p.updates) return;
  const int b0 = blockIdx.x * T, ne = min(T, n - b0), tid = threadIdx.x;
  const mbd_sac_learn_layout L = mbd_sac_learn_layout_of(O, nu, n);
  float* scr = p.scratch_dev;
  const float* rows = p.batch_dev + (size_t)g * n * R;
  const float* eps0 = p.eps_dev + ((size_t)(0 * p.updates) + g) * n * nu;
  const float* eps1 = p.eps_dev + ((size_t)(1 * p.updates) + g) * n * nu;
  const float* eps2 = p.eps_dev + ((size_t)(2 * p.updates) + g) * n * nu;
  float *xs = sm + kSlOffXs, *xn = sm + kSlOffXn, *qi = sm + kSlOffQi, *c1 = sm + kSlOffC1, *c2 = sm + kSlOffC2;
  float *p1 = sm + kSlOffP1, *p2 = sm + kSlOffP2, *lg = sm + kSlOffLg, *ln = sm + kSlOffLn, *tp = sm + kSlOffTp;
  float *l0 = sm + kSlOffL0, *l2 = sm + kSlOffL2, *ga = sm + kSlOffGa, *qo = sm + kSlOffQo, *d3 = sm + kSlOffD3;
  float* rw = sm + kSlOffRow;
  const float alpha = mbd_expf(p.log_alpha_dev[0]);
  const float* Pw[3];
#pragma unroll
  for (int l = 0; l < 3; ++l) Pw[l] = p.policy_dev + mbd_sac_layer_offset(O, l);

  // inputs: x, xn, the critic stack (x, action | x, .) and the critic input scratch
  for (int q = tid; q < T * QI; q += blockDim.x) {
    const int e = q / QI, i = q - e * QI, b = b0 + e;
    const float* r = rows + (size_t)b * R;
    if (i < O) {
      const float x = e < ne ? mbd_ppo_norm(r[i], p.mean_dev[i], p.std_dev[i]) : 0.0f;
      const float y = e < ne ? mbd_ppo_norm(r[mbd_sac_off_next_obs(O, nu) + i], p.mean_dev[i], p.std_dev[i]) : 0.0f;
      xs[i * T + e] = x;
      xn[i * T + e] = y;
      qi[i * S + e] = x;
      qi[i * S + T + e] = x;
      if (e < ne) { scr[L.x + (size_t)b * O + i] = x; scr[L.qin + (size_t)b * QI + i] = x; }
    } else {
      const float a = e < ne ? r[mbd_sac_off_action(O) + i - O] : 0.0f;
      qi[i * S + e] = a;
      if (e < ne) scr[L.qin + (size_t)b * QI + i] = a;
    }
  }
  __syncthreads();

  // the target: policy on xn, the head with eps 1, both target critics on (xn, tanh raw_c); c1[0] holds their input [O + Nu][8]
  float* ti = c1;
  float *h1 = c1 + MBD_SAC_HIDDEN * S, *h2 = c2 + MBD_SAC_HIDDEN * S;    // critic 1's buffers as work space
  sl_dense<kSlTile, true>(Pw[0], Pw[0] + O * MBD_SAC_HIDDEN, O, xn, h1);
  __syncthreads();
  sl_dense<kSlTile, true>(Pw[1], Pw[1] + MBD_SAC_HIDDEN * MBD_SAC_HIDDEN, MBD_SAC_HIDDEN, h1, h2);
  __syncthreads();
  sl_out<kSlTile>(Pw[2], Pw[2] + MBD_SAC_HIDDEN * 2 * nu, 2 * nu, h2, ln);
  for (int q = tid; q < T * O; q += blockDim.x) {
    const int e = q / O, i = q - e * O;
    ti[i * T + e] = xn[i * T + e];
  }
  __syncthreads();
  for (int q = tid; q < T * nu; q += blockDim.x) {
    const int e = q / nu, j = q - e * nu;
    float raw, act, lp;
    mbd_ppo_head(ln[j * T + e], ln[(nu + j) * T + e], e < ne ? eps1[(size_t)(b0 + e) * nu + j] : 0.0f, &raw, &act, &lp);
    ti[(O + j) * T + e] = act;
    l0[j * T + e] = lp;
  }
  __syncthreads();
  if (tid < T) {
    float s = 0.0f;
    for (int j = 0; j < nu; ++j) s = s + l0[j * T + tid];
    rw[1 * T + tid] = s;
  }
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    sl_dense<kSlTile, true>(p.target_q_dev + mbd_sac_q_w(O, nu, 0, c), p.target_q_dev + mbd_sac_q_bias(O, nu, 0, c), QI, ti, h1);
    __syncthreads();
    sl_dense<kSlTile, true>(p.target_q_dev + mbd_sac_q_w(O, nu, 1, c), p.target_q_dev + mbd_sac_q_bias(O, nu, 1, c),
                            MBD_SAC_HIDDEN, h1, h2);
    __syncthreads();
    sl_out<kSlTile>(p.target_q_dev + mbd_sac_q_w(O, nu, 2, c), p.target_q_dev + mbd_sac_q_bias(O, nu, 2, c), 1, h2,
                    qo + 2 * S + c * T);
    __syncthreads();
  }
  if (tid < T) {
    const int e = tid;
    const float* r = rows + (size_t)(b0 + min(e, ne - 1)) * R;
    rw[0 * T + e] = mbd_sac_learn_target(r[mbd_sac_off_reward(O, nu)], r[mbd_sac_off_discount(O, nu)], qo[2 * S + e],
                                         qo[2 * S + T + e], alpha, rw[1 * T + e], p.reward_scaling, p.discounting);
  }

  // the policy on x and its heads with eps 0 (alpha loss) and eps 2 (actor loss)
  sl_dense<kSlTile, true>(Pw[0], Pw[0] + O * MBD_SAC_HIDDEN, O, xs, p1);
  __syncthreads();
  sl_store<kSlTile>(p1, 0, scr + L.p1, b0, ne);
  sl_dense<kSlTile, true>(Pw[1], Pw[1] + MBD_SAC_HIDDEN * MBD_SAC_HIDDEN, MBD_SAC_HIDDEN, p1, p2);
  __syncthreads();
  sl_store<kSlTile>(p2, 0, scr + L.p2, b0, ne);
  sl_out<kSlTile>(Pw[2], Pw[2] + MBD_SAC_HIDDEN * 2 * nu, 2 * nu, p2, lg);
  __syncthreads();
  for (int q = tid; q < T * nu; q += blockDim.x) {
    const int e = q / nu, j = q - e * nu;
    const size_t k = (size_t)(b0 + e) * nu + j;
    float raw, act, lp;
    mbd_ppo_head(lg[j * T + e], lg[(nu + j) * T + e], e < ne ? eps0[k] : 0.0f, &raw, &act, &lp);
    l0[j * T + e] = lp;
    mbd_ppo_head(lg[j * T + e], lg[(nu + j) * T + e], e < ne ? eps2[k] : 0.0f, &raw, &act, &lp);
    l2[j * T + e] = lp;
    tp[j * T + e] = act;
    qi[(O + j) * S + T + e] = act;
  }
  __syncthreads();
  if (tid < T) {
    float sa = 0.0f, sp = 0.0f;
    for (int j = 0; j < nu; ++j) sa = sa + l0[j * T + tid];
    for (int j = 0; j < nu; ++j) sp = sp + l2[j * T + tid];
    rw[2 * T + tid] = sa;
    rw[3 * T + tid] = sp;
  }

  // both critics on the stack
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float *a1 = c1 + c * MBD_SAC_HIDDEN * S, *a2 = c2 + c * MBD_SAC_HIDDEN * S;
    sl_dense<kSlStack, true>(p.q_dev + mbd_sac_q_w(O, nu, 0, c), p.q_dev + mbd_sac_q_bias(O, nu, 0, c), QI, qi, a1);
    __syncthreads();
    sl_store<kSlStack>(a1, 0, scr + L.c1[c], b0, ne);
    sl_dense<kSlStack, true>(p.q_dev + mbd_sac_q_w(O, nu, 1, c), p.q_dev + mbd_sac_q_bias(O, nu, 1, c), MBD_SAC_HIDDEN, a1, a2);
    __syncthreads();
    sl_store<kSlStack>(a2, 0, scr + L.c2[c], b0, ne);
    sl_out<kSlStack>(p.q_dev + mbd_sac_q_w(O, nu, 2, c), p.q_dev + mbd_sac_q_bias(O, nu, 2, c), 1, a2, qo + c * S);
  }
  __syncthreads();

  // the loss terms and the seeds
  if (tid < T) {
    const int e = tid, b = b0 + e;
    const bool in = e < ne;
    const float m = in ? 1.0f - rows[(size_t)b * R + mbd_sac_off_truncation(O, nu)] : 0.0f;
    const float tgt = rw[e];
    const float err0 = (qo[e] - tgt) * m, err1 = (qo[S + e] - tgt) * m;
    d3[e] = err0 * m;
    d3[S + e] = err1 * m;
    const float qa0 = qo[T + e], qa1 = qo[S + T + e];
    const int pick = qa0 <= qa1 ? 0 : 1;
    d3[T + e] = in && pick == 0 ? -1.0f : 0.0f;
    d3[S + T + e] = in && pick == 1 ? -1.0f : 0.0f;
    if (in) {
      scr[L.terms + b] = -rw[2 * T + e] - (-0.5f * (float)nu);
      scr[L.terms + n + b] = err0 * err0 + err1 * err1;
      scr[L.terms + 2 * n + b] = alpha * rw[3 * T + e] - fminf(qa0, qa1);
      scr[L.dc3[0] + b] = d3[e];
      scr[L.dc3[1] + b] = d3[S + e];
    }
  }
  __syncthreads();

  // critic backward on the stack: d2 into c2[c], d1 into c1[c]; the actor rows' action gradient through critic c
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float *a1 = c1 + c * MBD_SAC_HIDDEN * S, *a2 = c2 + c * MBD_SAC_HIDDEN * S;
    sl_back<kSlStack>(p.q_dev + mbd_sac_q_w(O, nu, 2, c), 1, d3 + c * S, a2);
    __syncthreads();
    sl_store<kSlStack>(a2, 0, scr + L.dc2[c], b0, ne);
    sl_back<kSlStack>(p.q_dev + mbd_sac_q_w(O, nu, 1, c), MBD_SAC_HIDDEN, a2, a1);
    __syncthreads();
    sl_store<kSlStack>(a1, 0, scr + L.dc1[c], b0, ne);
    const float* W1 = p.q_dev + mbd_sac_q_w(O, nu, 0, c);
    for (int q = tid; q < T * nu; q += blockDim.x) {
      const int e = q / nu, j = q - e * nu;
      const float* w = W1 + (size_t)(O + j) * MBD_SAC_HIDDEN;
      float acc = 0.0f;
      for (int k = 0; k < MBD_SAC_HIDDEN; ++k) acc = acc + __ldg(w + k) * a1[k * S + T + e];
      ga[(c * nu + j) * T + e] = acc;
    }
  }
  __syncthreads();

  // the head's backward into lg (the policy's d3), then the policy's backward
  for (int q = tid; q < T * nu; q += blockDim.x) {
    const int e = q / nu, j = q - e * nu;
    float dloc = 0.0f, ds = 0.0f;
    if (e < ne)
      mbd_sac_learn_head_grad(ga[j * T + e] + ga[(nu + j) * T + e], tp[j * T + e], eps2[(size_t)(b0 + e) * nu + j],
                              lg[(nu + j) * T + e], alpha, &dloc, &ds);
    lg[j * T + e] = dloc;      // each thread reads and writes its own (e, j) words only
    lg[(nu + j) * T + e] = ds;
    if (e < ne) {
      scr[L.dp3 + (size_t)(b0 + e) * 2 * nu + j] = dloc;
      scr[L.dp3 + (size_t)(b0 + e) * 2 * nu + nu + j] = ds;
    }
  }
  __syncthreads();
  sl_back<kSlTile>(Pw[2], 2 * nu, lg, p2);
  __syncthreads();
  sl_store<kSlTile>(p2, 0, scr + L.dp2, b0, ne);
  sl_back<kSlTile>(Pw[1], MBD_SAC_HIDDEN, p2, p1);
  __syncthreads();
  sl_store<kSlTile>(p1, 0, scr + L.dp1, b0, ne);
}
// the weight phase: CTA = one 64 x 64 tile of one job (the last CTA: log alpha and the loss scalars)
__global__ void __launch_bounds__(256) k_sac_learn_weights(mbd_sac_learn_plan p) {
  __shared__ float As[kSwK][kSwTile];
  __shared__ float Bs[kSwK][kSwTile];
  __shared__ int s_last;
  const int O = p.O, nu = p.nu, n = p.batch, tid = threadIdx.x;
  const long long g = p.upd_ctl_dev[0];
  if (g < 0 || g >= p.updates) return;
  const long long t = p.ctl_dev[0] + 1;
  int tile = blockIdx.x, j = 0;
  mbd_sac_learn_job J = mbd_sac_learn_job_of(O, nu, n, 0);
  int tr = 0, tc = 0;
  bool alpha_cta = true;
  for (j = 0; j < MBD_SAC_LEARN_JOBS; ++j) {
    J = mbd_sac_learn_job_of(O, nu, n, j);
    tr = (J.nin + 1 + kSwTile - 1) / kSwTile;
    tc = (J.nout + kSwTile - 1) / kSwTile;
    if (tile < tr * tc) { alpha_cta = false; break; }
    tile -= tr * tc;
  }
  const float* scr = p.scratch_dev;
  if (!alpha_cta) {
    const int i0 = (tile / tc) * kSwTile, o0 = (tile % tc) * kSwTile;
    const int ty = tid / 16, tx = tid % 16;
    const float* In = scr + J.in;
    const float* D = scr + J.d;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.0f;
    for (int k0 = 0; k0 < n; k0 += kSwK) {
      for (int q = tid; q < kSwK * kSwTile; q += 256) {
        const int kk = q / kSwTile, c = q - kk * kSwTile, b = k0 + kk, i = i0 + c, o = o0 + c;
        As[kk][c] = b < n && i < J.nin ? In[(size_t)b * J.nin + i] : (b < n && i == J.nin ? 1.0f : 0.0f);
        Bs[kk][c] = b < n && o < J.nout ? D[(size_t)b * J.nout + o] : 0.0f;
      }
      __syncthreads();
      const int kn = min(kSwK, n - k0);
      for (int kk = 0; kk < kn; ++kk) {
        float a[4], bb[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) a[r] = As[kk][ty + 16 * r];
#pragma unroll
        for (int c = 0; c < 4; ++c) bb[c] = Bs[kk][tx + 16 * c];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[r][c] = acc[r][c] + a[r] * bb[c];
      }
      __syncthreads();
    }
    const float N = J.is_q ? 2.0f * (float)n : (float)n;
    float step, bc2s;
    mbd_sac_adam_scalars(p.learning_rate, t, &step, &bc2s);
    float* P = J.is_q ? p.q_dev : p.policy_dev;
    float* M = J.is_q ? p.q_m_dev : p.policy_m_dev;
    float* V = J.is_q ? p.q_v_dev : p.policy_v_dev;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = i0 + ty + 16 * r;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int o = o0 + tx + 16 * c;
        if (i > J.nin || o >= J.nout) continue;
        const int k = i < J.nin ? J.w + i * J.nout + o : J.bias + o;
        mbd_sac_adam(P + k, M + k, V + k, MBD_DIV(acc[r][c], N), step, bc2s);
        if (J.is_q) p.target_q_dev[k] = mbd_sac_polyak(p.target_q_dev[k], P[k], p.tau);
      }
    }
  } else if (tid < 96 && (tid & 31) == 0) {
    // log alpha (thread 0), the loss scalars (threads 0, 32, 64): fixed-order sums over the batch
    const int w = tid >> 5;
    const float* terms = scr + mbd_sac_learn_layout_of(O, nu, n).terms + (size_t)w * n;
    float s = 0.0f;
    for (int b = 0; b < n; ++b) s = s + terms[b];
    const float mean = MBD_DIV(s, (float)n);
    if (w == 0) {
      const float ga = mbd_expf(p.log_alpha_dev[0]) * mean;
      p.losses_dev[0] = ga;
      float step, bc2s;
      mbd_sac_adam_scalars(MBD_SAC_ALPHA_LR, t, &step, &bc2s);
      mbd_sac_adam(p.log_alpha_dev, p.alpha_mv_dev, p.alpha_mv_dev + 1, ga, step, bc2s);
    } else if (w == 1) {
      p.losses_dev[1] = 0.5f * MBD_DIV(s, 2.0f * (float)n);
    } else {
      p.losses_dev[2] = mean;
    }
  }
  // the last CTA advances the step count and the update counter (every CTA has read them by then)
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(reinterpret_cast<unsigned long long*>(&p.ctl_dev[1]), 1ull) == (unsigned long long)gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && tid == 0) {
    p.ctl_dev[1] = 0;
    p.ctl_dev[0] = t;
    p.upd_ctl_dev[0] = g + 1;
    __threadfence();
  }
}

// CTAs of the weight phase: the tiles of the nine jobs and the alpha CTA
inline int sac_learn_weight_ctas(int O, int nu, int n) {
  int total = 1;
  for (int j = 0; j < MBD_SAC_LEARN_JOBS; ++j) {
    const mbd_sac_learn_job J = mbd_sac_learn_job_of(O, nu, n, j);
    total += ((J.nin + 1 + kSwTile - 1) / kSwTile) * ((J.nout + kSwTile - 1) / kSwTile);
  }
  return total;
}

}  // namespace mbd
