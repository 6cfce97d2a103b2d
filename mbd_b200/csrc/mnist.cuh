// mnist.cuh — model-based diffusion over the weights of a 784-32-32-10 MLP (upstream mbd/blackbox/mbd_mnist.py).
//
// One step is five parameterless launches (graph-capturable; everything that changes per step is read from device tables
// indexed by ctl->i):
//   (1) k_mnist_sample  Y0s[n] = mean + normal(kn) * sigma (* 0.1 on W1) * (uniform(ku) < 0.2), per tensor of the reference's
//                       order W1, b1, W2, b2, W3, b3 (add_noise_batch_to_params).  The PRNG counter of an element is its flat
//                       index in JAX's shape (n, in, out), whatever the row layout (below).
//   (2) k_mnist_fwd<false>  Js[n] = mean over the step's N minibatch images of log_softmax(MLP_n(x))[label]: one CTA per
//                       model n.  Layer 1 is a tensor-core GEMM (wgmma m64n32k8 TF32, split: see below); the epilogue runs
//                       layers 2 and 3, log-softmax and the label pick in fp32 SIMT.
//   (3) k_step_weights<false, RULE_MPPI> of step_tail.cuh, unchanged: mean / population std (guard) / softmax weights,
//                       rew_hist[i] = Js.mean().
//   (4) k_mnist_runs, (5) k_mnist_commit: Ybars[i - 1] = sum_n w_n Y0s_n in the tail's order (64-sample runs of sequential
//                       fmaf, then the adjacent-pairwise tree over the runs).  k_step_update cannot take a 26 506-column row
//                       (its control block holds 27 column tickets), so the MNIST step uses these two; the last CTA of (5)
//                       moves the step counter.
//   (6) k_mnist_fwd<true>   train / test correct-counts of the new mean into acc_hist[i] (every eval_every steps).
//
// Row layout of a parameter set (MNIST_HNU = 26 506 floats): W1T [32][784] (W1 transposed: the GEMM's B operand is K-major),
// b1 [32], W2 [32][32] (in, out), b2 [32], W3 [32][10], b3 [10].
//
// Layer 1 on the tensor cores.  Each of the two warpgroups of a CTA owns 128 image rows (two m64 blocks); per K tile of 16 the
// threads stage the pixels (as integer floats, padded rows) and the W1T tile (split into TF32 hi and lo blocks in the
// unswizzled K-major core-matrix layout) into double-buffered shared memory, then every warpgroup issues 8 wgmma (2 K steps x
// 2 row blocks x hi / lo) with A from registers and B from shared memory, while the next tile's global loads are in flight.
// TMA does not fit either operand: the pixels are a gather of minibatch rows, and a sample's W1T starts 26506 floats after
// the previous one, a row stride that is not a multiple of 16 bytes, which a tensor map requires.
//
// Layer 1 precision.  Z1[m][o] = (sum_k p_mk * W1[k][o]) / 255 with p the uint8 pixel: the pixel is an integer <= 255, exact in
// TF32; the weight is split w = hi + lo, hi = tf32_rna(w), lo = tf32_rna(w - hi) (|w - hi - lo| <= 2^-22 |w|), and both
// products are accumulated by the tensor core in fp32.  Each K tile of 16 is accumulated from zero on the tensor core (32
// products) and then added to the fp32 register sum with one FADD, so no tensor-core accumulation chain is longer than one
// tile.  The division by 255 is the fp32 epilogue (IEEE division).
//
// Layers 2 and 3 per (image, model), fp32, no contraction: z = ((0 + h_0 W_0o) + h_1 W_1o) + ... + h_31 W_31o, then + b_o;
// ReLU = fmaxf(z, 0).  log_softmax: mx = max_c z_c (c ascending), s_c = z_c - mx, lse = mbd_logf(sum_c mbd_expf(s_c)) (c
// ascending from 0), lp_c = s_c - lse.
//
// Reduction over the N images (train): thread tau adds lp[label] of images tau, tau + 256, ... in that order onto 0; the 256
// partials are folded by an xor butterfly over lanes (offsets 1, 2, 4, 8, 16) and then over the 8 warp sums (1, 2, 4); J is
// that sum / N.  No atomics.  Accuracy (eval): argmax over lp_c, first index wins; the integer counts are added with atomics
// (exact, order-independent).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "mbd_b200.h"
#include "mbd_fp32.h"

namespace mbd {

constexpr int kMnistIn = 784, kMnistH = 32, kMnistOut = 10;
constexpr int kMnistOffB1 = kMnistIn * kMnistH;                 // 25088
constexpr int kMnistOffW2 = kMnistOffB1 + kMnistH;              // 25120
constexpr int kMnistOffB2 = kMnistOffW2 + kMnistH * kMnistH;    // 26144
constexpr int kMnistOffW3 = kMnistOffB2 + kMnistH;              // 26176
constexpr int kMnistOffB3 = kMnistOffW3 + kMnistH * kMnistOut;  // 26496
constexpr int kMnistHNu = kMnistOffB3 + kMnistOut;              // 26506
constexpr int kMnistTail = kMnistHNu - kMnistOffB1;             // 1418: b1 .. b3
constexpr int kMnistThreads = 256;                              // one image row per thread per chunk
constexpr int kMnistKT = 16;                                    // K tile (784 = 49 * 16)
constexpr int kMnistKTiles = kMnistIn / kMnistKT;
constexpr int kMnistAS = kMnistKT + 4;                          // smem row stride: conflict-free fragment reads
constexpr int kMnistBBlk = kMnistH * 8;                         // one 32 x 8 TF32 block of W1T (1 KB)
constexpr int kMnistBFloats = 2 * 2 * (kMnistKT / 8) * kMnistBBlk;  // [buffer][hi, lo][K block]
constexpr int kMnistSmemFloats = 2 * kMnistThreads * kMnistAS + kMnistBFloats + kMnistTail + 2;
static_assert(kMnistIn % kMnistKT == 0, "K tile must divide 784");
static_assert(kMnistThreads * (kMnistH + 1) <= 2 * kMnistThreads * kMnistAS, "h1 reuses the A buffers");

// per-tensor (offset in the row, size, JAX shape (in, out)); tensor 0 (W1) is stored transposed
__device__ __forceinline__ int mnist_tensor_of(int j) {
  return j < kMnistOffB1 ? 0 : j < kMnistOffW2 ? 1 : j < kMnistOffB2 ? 2 : j < kMnistOffW3 ? 3 : j < kMnistOffB3 ? 4 : 5;
}

struct MnistArgs {
  const mbd_step_params* sp;   // [nd]: sigma of every step
  mbd_step_ctl* ctl;           // step index i
  float* Ybars;                // [nd][HNu]
  float* Y0s;                  // [N][HNu]
  float* rews;                 // [N]: J
  const float* weights;        // [N]: softmax weights of launch (3)
  float* runs;                 // [ceil(N/64)][HNu]
  const uint32_t* keys;        // [nd][12][2]: (kn, ku) of the six tensors
  const int32_t* idx;          // [nd][N]: the minibatch of every step
  const uint8_t* train_x;      // [n_train][784]
  const uint8_t* train_y;      // [n_train]
  const uint8_t* test_x;       // [n_test][784]
  const uint8_t* test_y;       // [n_test]
  int32_t* acc_hist;           // [nd][2]: train / test correct-counts of the mean after step i (-1: not evaluated)
  float* z1;                   // test only: [N models][N images][32] layer-1 pre-activations (before b1), or null
  const int32_t* idx_direct;   // test only: the image rows of a forward call without a step counter, or null
  int N, n_img, nd, n_train, n_test, eval_every, prng_part;
};

// does the step that produced Ybars[t - 1] (step t) get an accuracy evaluation?
__device__ __forceinline__ bool mnist_eval_step(const MnistArgs& a, int t) {
  return t == 1 || (a.nd - 1 - t) % a.eval_every == a.eval_every - 1;
}

// ---- (1) sampling -----------------------------------------------------------------------------------------------------
// grid (ceil(HNu / 256), N)
__global__ void __launch_bounds__(256) k_mnist_sample(const MnistArgs a) {
  const int i = a.ctl->i;
  if (i < 1) return;
  const int n = blockIdx.y;
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (n == 0 && j < 2 && mnist_eval_step(a, i)) a.acc_hist[2 * i + j] = 0;   // launch (6) adds this step's counts
  if (j >= kMnistHNu) return;
  const int t = mnist_tensor_of(j);
  constexpr int off[6] = {0, kMnistOffB1, kMnistOffW2, kMnistOffB2, kMnistOffW3, kMnistOffB3};
  constexpr int size[6] = {kMnistOffB1, kMnistH, kMnistH * kMnistH, kMnistH, kMnistH * kMnistOut, kMnistOut};
  int local = j - off[t];
  if (t == 0) local = (local % kMnistIn) * kMnistH + local / kMnistIn;   // stored (o, k) -> JAX (k, o)
  const uint32_t idx = (uint32_t)n * (uint32_t)size[t] + (uint32_t)local;
  const uint32_t total = a.prng_part ? 0u : (uint32_t)a.N * (uint32_t)size[t];
  const uint32_t* k = a.keys + ((size_t)i * 12 + 2 * t) * 2;
  const float sigma = a.sp[i].sigma;
  float noise = mbd_bits_to_normal(mbd_random_bits_at(k[0], k[1], idx, total)) * sigma;
  if (t == 0) noise = noise * 0.1f;
  const float upd = mbd_bits_to_unit(mbd_random_bits_at(k[2], k[3], idx, total)) < 0.2f ? 1.0f : 0.0f;
  a.Y0s[(size_t)n * kMnistHNu + j] = a.Ybars[(size_t)i * kMnistHNu + j] + noise * upd;
}

// ---- (2) / (6) forward ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// wgmma m64n32k8 TF32: A (16 rows x 8 K per warp, the mma.m16n8k8 fragment layout) from registers, B from shared memory
// through a matrix descriptor; fp32 accumulators d[4 * nb + q] at row g + 8 (q >> 1), column 8 nb + 2 (lane & 3) + (q & 1)
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[16]) {
#pragma unroll
  for (int q = 0; q < 16; ++q) asm volatile("" : "+f"(d[q])::"memory");
}
// descriptor of one K-major, unswizzled 32 (N) x 8 (K) TF32 block: core matrices of 8 rows x 16 bytes, the two K-adjacent ones
// 512 bytes apart (leading byte offset), the four N-adjacent ones 128 bytes apart (stride byte offset)
__device__ __forceinline__ uint64_t mnist_bdesc(const float* blk) {
  const uint32_t addr = static_cast<uint32_t>(__cvta_generic_to_shared(blk));
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)(512 >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
}
// float offset of W1T element (n, k) (k < 8) inside such a block
__device__ __forceinline__ int mnist_bofs(int n, int k) { return (k >> 2) * 128 + (n >> 3) * 32 + (n & 7) * 4 + (k & 3); }

// EVAL == false: grid N (model n = blockIdx.x), the images are the step's minibatch rows of the training set.
// EVAL == true: grid ceil(n_train / 256) + ceil(n_test / 256) (one chunk of 256 images each), model = Ybars[ctl->i].
template <bool EVAL>
__global__ void __launch_bounds__(kMnistThreads) k_mnist_fwd(const MnistArgs a) {
  extern __shared__ __align__(16) float sm[];   // 16 B: what an unswizzled wgmma operand needs; a larger alignment would pad the static smem of every kernel in this file
  float* As = sm;                                          // [2][256][kMnistAS] pixels (integers as floats)
  float* Bs = sm + 2 * kMnistThreads * kMnistAS;           // [2][hi, lo][2 K blocks][kMnistBBlk] W1T tile, TF32-rounded
  float* Ps = Bs + kMnistBFloats;                          // b1 .. b3 of the model
  float* H1 = sm;                                          // [256][33] after the GEMM (reuses As)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tq = lane & 3;
  const int wg = warp >> 2, wl = warp & 3;                 // warpgroup (rows 128 wg ..) and warp within it

  const float* W;
  const uint8_t* X;
  const uint8_t* Y;
  const int32_t* rows = nullptr;
  int n_img, first = 0, set = 0, t_step = 0;
  if constexpr (EVAL) {
    if (a.ctl->err != 0) return;   // launch (3) of a step past the end sets err: this step wrote nothing, neither does (6)
    const int i = a.ctl->i;        // launch (5) has moved the counter: the new mean is row i, produced by step i + 1
    t_step = i + 1;
    if (i < 0 || t_step >= a.nd || !mnist_eval_step(a, t_step)) return;
    W = a.Ybars + (size_t)i * kMnistHNu;
    const int tr_chunks = (a.n_train + kMnistThreads - 1) / kMnistThreads;
    set = (int)blockIdx.x >= tr_chunks;
    first = (set ? (int)blockIdx.x - tr_chunks : (int)blockIdx.x) * kMnistThreads;
    X = set ? a.test_x : a.train_x;
    Y = set ? a.test_y : a.train_y;
    n_img = set ? a.n_test : a.n_train;
  } else {
    if (a.idx_direct) {
      rows = a.idx_direct;
    } else {
      const int i = a.ctl->i;
      if (i < 1) return;
      rows = a.idx + (size_t)i * a.N;
    }
    W = a.Y0s + (size_t)blockIdx.x * kMnistHNu;
    X = a.train_x;
    Y = a.train_y;
    n_img = a.n_img;
  }
  for (int c = tid; c < kMnistTail; c += kMnistThreads) Ps[c] = W[kMnistOffB1 + c];
  const float* b1 = Ps;
  const float* W2 = Ps + kMnistH;
  const float* b2 = W2 + kMnistH * kMnistH;
  const float* W3 = b2 + kMnistH;
  const float* b3 = W3 + kMnistH * kMnistOut;

  float part = 0.0f;   // train: sum of this thread's lp[label]
  int correct = 0;     // eval
  const int chunk_end = EVAL ? first + kMnistThreads : n_img;
  for (int c0 = first; c0 < chunk_end && c0 < n_img; c0 += kMnistThreads) {
    // this thread's A row (pixels of one image) and B pair (two weights of W1T)
    const int m = c0 + tid;
    const bool valid = m < n_img;
    const uint8_t* xrow = valid ? X + (size_t)(EVAL ? m : rows[m]) * kMnistIn : nullptr;
    const int bo = tid >> 3, bk = (tid & 7) * 2;
    const float* wrow = W + (size_t)bo * kMnistIn + bk;
    uint4 ra = make_uint4(0u, 0u, 0u, 0u);
    float2 rb;
    auto load = [&](int kt) {
      if (valid) ra = *reinterpret_cast<const uint4*>(xrow + kt * kMnistKT);
      rb = *reinterpret_cast<const float2*>(wrow + kt * kMnistKT);
    };
    auto store = [&](int buf) {
      float* dst = As + (buf * kMnistThreads + tid) * kMnistAS;
      const uint32_t w4[4] = {ra.x, ra.y, ra.z, ra.w};
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int b = 0; b < 4; ++b) dst[4 * q + b] = (float)((w4[q] >> (8 * b)) & 0xffu);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float w = e ? rb.y : rb.x;
        const uint32_t hi = tf32_rna(w);
        const uint32_t lo = tf32_rna(w - __uint_as_float(hi));
        const int k = bk + e;
        float* blk = Bs + (buf * 2 * 2 + (k >> 3)) * kMnistBBlk;   // hi part; lo is 2 blocks further
        blk[mnist_bofs(bo, k & 7)] = __uint_as_float(hi);
        blk[2 * kMnistBBlk + mnist_bofs(bo, k & 7)] = __uint_as_float(lo);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic stores -> wgmma operand reads
    };
    float acc[2][16];
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int q = 0; q < 16; ++q) acc[mb][q] = 0.0f;
    load(0);
    __syncthreads();   // the previous chunk's epilogue is done with H1 (= As)
    store(0);
    __syncthreads();
    for (int kt = 0; kt < kMnistKTiles; ++kt) {
      const int buf = kt & 1;
      if (kt + 1 < kMnistKTiles) load(kt + 1);
      float tile[2][16];
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
        for (int q = 0; q < 16; ++q) tile[mb][q] = 0.0f;
        wgmma_fence_regs(tile[mb]);
      }
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int ks = 0; ks < kMnistKT / 8; ++ks) {
        const float* bhi = Bs + (buf * 2 * 2 + ks) * kMnistBBlk;
        const uint64_t dhi = mnist_bdesc(bhi), dlo = mnist_bdesc(bhi + 2 * kMnistBBlk);
#pragma unroll
        for (int mb = 0; mb < 2; ++mb) {
          const float* ap = As + (buf * kMnistThreads + wg * 128 + mb * 64 + wl * 16 + g) * kMnistAS + ks * 8 + tq;
          const uint32_t fa[4] = {__float_as_uint(ap[0]), __float_as_uint(ap[8 * kMnistAS]), __float_as_uint(ap[4]),
                                  __float_as_uint(ap[8 * kMnistAS + 4])};
          wgmma_tf32(tile[mb], fa, dhi);
          wgmma_tf32(tile[mb], fa, dlo);
        }
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        wgmma_fence_regs(tile[mb]);
#pragma unroll
        for (int q = 0; q < 16; ++q) acc[mb][q] = acc[mb][q] + tile[mb][q];
      }
      if (kt + 1 < kMnistKTiles) store(buf ^ 1);
      __syncthreads();
    }
    // epilogue 1: Z1 = acc / 255, h1 = relu(Z1 + b1) -> H1[row][o]
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int j = 0; j < 16; ++j) {
          const int q = j & 3;
          const int r = wg * 128 + mb * 64 + wl * 16 + g + (q >> 1) * 8;
          const int o = (j >> 2) * 8 + 2 * tq + (q & 1);
          const float z = MBD_DIV(acc[mb][j], 255.0f);
          if (!EVAL && a.z1 && c0 + r < n_img) a.z1[((size_t)blockIdx.x * n_img + c0 + r) * kMnistH + o] = z;
          H1[r * (kMnistH + 1) + o] = fmaxf(z + b1[o], 0.0f);
        }
    __syncthreads();
    // epilogue 2: layers 2 and 3, log-softmax, per image (thread tid = row tid of the chunk)
    if (valid) {
      float h2[kMnistH];
#pragma unroll
      for (int o = 0; o < kMnistH; ++o) {
        float s = 0.0f;
#pragma unroll
        for (int k = 0; k < kMnistH; ++k) s = s + H1[tid * (kMnistH + 1) + k] * W2[k * kMnistH + o];
        h2[o] = fmaxf(s + b2[o], 0.0f);
      }
      float z3[kMnistOut];
#pragma unroll
      for (int o = 0; o < kMnistOut; ++o) {
        float s = 0.0f;
#pragma unroll
        for (int k = 0; k < kMnistH; ++k) s = s + h2[k] * W3[k * kMnistOut + o];
        z3[o] = s + b3[o];
      }
      float mx = z3[0];
#pragma unroll
      for (int o = 1; o < kMnistOut; ++o) mx = fmaxf(mx, z3[o]);
      float se = 0.0f;
#pragma unroll
      for (int o = 0; o < kMnistOut; ++o) { z3[o] = z3[o] - mx; se = se + mbd_expf(z3[o]); }
      const float lse = mbd_logf(se);
      const int lab = Y[EVAL ? m : rows[m]];
      if constexpr (EVAL) {
        int best = 0;
        float bv = z3[0] - lse;
#pragma unroll
        for (int o = 1; o < kMnistOut; ++o) {
          const float v = z3[o] - lse;
          if (v > bv) { bv = v; best = o; }
        }
        correct += best == lab;
      } else {
        float v = 0.0f;
#pragma unroll
        for (int o = 0; o < kMnistOut; ++o) v = o == lab ? z3[o] - lse : v;
        part = part + v;
      }
    }
  }
  // fold the 256 per-thread partials: xor butterfly over lanes, then over the 8 warp sums
  __shared__ float s_red[kMnistThreads / 32];
  __shared__ int s_cnt[kMnistThreads / 32];
  for (int o = 1; o < 32; o <<= 1) {
    part = part + __shfl_xor_sync(0xffffffffu, part, o);
    correct += __shfl_xor_sync(0xffffffffu, correct, o);
  }
  if (lane == 0) { s_red[warp] = part; s_cnt[warp] = correct; }
  __syncthreads();
  if (warp == 0) {
    float r = lane < kMnistThreads / 32 ? s_red[lane] : 0.0f;
    int cn = lane < kMnistThreads / 32 ? s_cnt[lane] : 0;
    for (int o = 1; o < kMnistThreads / 32; o <<= 1) {
      r = r + __shfl_xor_sync(0xffffffffu, r, o);
      cn += __shfl_xor_sync(0xffffffffu, cn, o);
    }
    if (lane == 0) {
      if constexpr (EVAL) atomicAdd(a.acc_hist + 2 * t_step + set, cn);
      else a.rews[blockIdx.x] = MBD_DIV(r, (float)n_img);
    }
  }
}

// ---- (4) weighted-mean runs, (5) tree + step counter --------------------------------------------------------------------
// grid (ceil(N / 64), ceil(HNu / 256)); the order of k_step_update's runs (sequential fmaf from w_n0 * Y_n0)
__global__ void __launch_bounds__(256) k_mnist_runs(const MnistArgs a) {
  if (a.ctl->i < 1) return;
  const int j = blockIdx.y * 256 + threadIdx.x;
  if (j >= kMnistHNu) return;
  const int n0 = blockIdx.x * kTailRun, n1 = min(n0 + kTailRun, a.N);
  float acc = a.weights[n0] * a.Y0s[(size_t)n0 * kMnistHNu + j];
  for (int n = n0 + 1; n < n1; ++n) acc = fmaf(a.weights[n], a.Y0s[(size_t)n * kMnistHNu + j], acc);
  a.runs[(size_t)blockIdx.x * kMnistHNu + j] = acc;
}

// grid ceil(HNu / 256): Ybars[i - 1][j] = adjacent-pairwise tree over the runs; the last CTA moves ctl->i to i - 1
__global__ void __launch_bounds__(256) k_mnist_commit(const MnistArgs a) {
  __shared__ int s_last;
  mbd_step_ctl* ctl = a.ctl;
  const int step = ctl->i;
  if (step < 1) return;
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int nruns = (a.N + kTailRun - 1) / kTailRun;
  if (j < kMnistHNu) a.Ybars[(size_t)(step - 1) * kMnistHNu + j] = tree_sum_rows(a.runs, nruns, kMnistHNu, j);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&ctl->ticket[MBD_STEP_MAX_COLBLOCKS], 1u) == gridDim.x - 1;
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    ctl->ticket[MBD_STEP_MAX_COLBLOCKS] = 0u;
    ctl->epoch = ctl->epoch + 1u;
    ctl->i = step - 1;
  }
}

// ---- minibatch index table: random bits of one permutation round -------------------------------------------------------
__global__ void k_mnist_perm_bits(uint32_t k0, uint32_t k1, int n, int prng_part, uint32_t* bits, int32_t* iota) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  bits[e] = mbd_random_bits_at(k0, k1, (uint32_t)e, prng_part ? 0u : (uint32_t)n);
  if (iota) iota[e] = e;
}

}  // namespace mbd
