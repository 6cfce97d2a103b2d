/* mbd_b200.h — C ABI of the H100-native MBD hot path (libmbd_b200.so).
 *
 * The reference has no FFI layer (it is pure Python/JAX); the seams this library replaces are
 * the Python call sites of the jitted hot path.  Each entry point cites the reference
 * interface it stands in for.  Conventions: one host thread; every pointer marked `_dev` is
 * device memory owned by the caller (torch tensors on the Python side); the stream is passed
 * explicitly; return 0 on success, a negative MBD_E* code otherwise (no exceptions cross the
 * ABI, nothing is allocated after *_create).  See INTEGRATION.md for the ctypes stub.
 *
 * The structs and constants Python uses from this header, mbd_model.h, mbd_kin64.h, mbd_sac.h and mbd_sac_learn.h are mirrored
 * in mbd_b200/_lib.py and mbd_b200/model/blob.py; tests/test_abi.py compiles every mirror against these headers (offset, size
 * and kind of every field, every constant), so a change here is made there too.
 */
#ifndef MBD_B200_H_
#define MBD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MBD_OK 0
#define MBD_EINVAL (-1)  /* bad argument / bad blob */
#define MBD_ECUDA (-2)   /* CUDA runtime error (see mbd_last_error) */
#define MBD_ENOGPU (-3)  /* no CUDA device: there is deliberately NO CPU fallback */

typedef struct mbd_model mbd_model;
typedef void* mbd_stream; /* cudaStream_t */

const char* mbd_last_error(void);
int mbd_device_count(void);
/* rollout kernel mapping: 0 = auto (by shard size), 1 = v1 (one link per lane), 2 / 3 = v2 (one link per warp, lane = sample)
 * with CTA-wide / named-barrier phase synchronisation, 8 = packed kernel: two samples per lane (two independent chains per
 * thread), 64 samples per CTA, group barriers with decoupled leaves.  Fallbacks: 3 runs 2 on a tree that needs more than 15
 * named barriers; 8 runs 2 on a model that is not 11 hinge-only links with at most 2 contacts per link.  Any other value is
 * MBD_EINVAL.  All variants produce bit-identical results; the switch exists for tests and profiling. */
int mbd_set_kernel_variant(int v);
/* threefry counter layout of every in-kernel sampler (process-wide): 0 = legacy (jax_threefry_partitionable=False, what the JAX
 * known-answer vectors in tests/test_prng.py pin), 1 = partitionable (the default of JAX >= 0.5; [jax-recalled], unpinned).
 * The host-side key chain must use the same layout (mbd_b200.prng.set_layout). */
int mbd_set_prng_layout(int partitionable);
/* tuning hook: slot -> link order of the one-link-per-warp mapping (slot L-1 gets the highest warp id) */
int mbd_model_set_warp_order(mbd_model* m, const int* order, int n);

/* brax.io.mjcf.load(...) result made device resident — replaces the `sys` captured by the
 * jitted env.step (upstream mbd/envs/humanoidrun.py:15-17).  blob: include/mbd_model.h */
mbd_model* mbd_model_create(const uint32_t* blob_host, size_t nwords);
void mbd_model_destroy(mbd_model*);

/* eps = jax.random.normal(key,(Nsample,H,Nu)); Y0s = clip(eps*sigma + Ybar_i, -1, 1)
 * (upstream mbd/planners/mbd_planner.py:103-106) for global samples
 * [n_begin, n_begin+n_local) of n_total.  Y0s_dev [n_local, HNu]. */
int mbd_sample(const uint32_t key[2], int n_total, int n_begin, int n_local, int HNu, float sigma,
               const float* Ybar_dev, float* Y0s_dev, mbd_stream s);

/* jax.vmap(rollout_us, in_axes=(None,0))(state_init, Y0s)  (mbd_planner.py:109, utils.py:14-20)
 * for a Brax-positional env (HumanoidRun.step humanoidrun.py:34-41, HumanoidTrack.step
 * humanoidtrack.py:63-82).  state_init_dev [L,13]; Y0s_dev [n,H,Nu].
 * Outputs (NULL = not wanted): rewss_dev [n,H]; rews_dev [n] = rewss.mean(-1) (required);
 * logpd_dev [n] = vmap(env.eval_xref_logpd)(qs) when xref_dev [ntrack,href,3] is given;
 * final_state_dev [n,L,13]; track_pos_dev [n,H,ntrack,3].  nsub_override>0 replaces n_frames. */
int mbd_rollout(const mbd_model* m, const float* state_init_dev, const float* Y0s_dev, int n, int H,
                float* rewss_dev, float* rews_dev, const float* xref_dev, int href, float* logpd_dev,
                float* final_state_dev, float* track_pos_dev, int nsub_override, mbd_stream s);

/* mbd_rollout that also records the rollout: traj_dev [n,H,L,13] receives every link's state after each of the H env steps
 * (the layout of final_state_dev, once per step; row H-1 equals final_state_dev).  It runs the warp-per-link kernel whatever n is;
 * every output is bit-identical to mbd_rollout's.  traj_dev == NULL is exactly mbd_rollout. */
int mbd_rollout_traj(const mbd_model* m, const float* state_init_dev, const float* Y0s_dev, int n, int H,
                     float* rewss_dev, float* rews_dev, const float* xref_dev, int href, float* logpd_dev,
                     float* final_state_dev, float* track_pos_dev, int nsub_override, float* traj_dev, mbd_stream s);

/* mbd_sample + mbd_rollout fused in ONE kernel (each CTA draws the noise of its own samples,
 * writes Y0s once, then rolls them out): the hot path of reverse_once, mbd_planner.py:103-110. */
int mbd_sample_rollout(const mbd_model* m, const float* state_init_dev, const uint32_t key[2], int n_total,
                       int n_begin, int n_local, int H, float sigma, const float* Ybar_dev, float* Y0s_dev,
                       float* rews_dev, const float* xref_dev, int href, float* logpd_dev, mbd_stream s);

/* Car2d (self-contained env, upstream mbd/envs/car2d.py:77-102).
 * params_dev: [obs_center(11x2), obs_radius, dt, dt/2, dt/6]; x0_dev [3]; xref_dev [href,2] or NULL.
 * key == NULL: Y0s_dev is an input; else it is sampled first (fused) as in mbd_sample. */
int mbd_car2d_rollout(const float* params_dev, const float* x0_dev, const uint32_t* key, int n_total, int n_begin,
                      int n_local, int H, float sigma, const float* Ybar_dev, float* Y0s_dev, float* rewss_dev,
                      float* rews_dev, const float* xref_dev, int href, float* logpd_dev, float* traj_dev,
                      mbd_stream s);

/* rews.mean(), rews.std() (guard <1e-4 -> 1), logp0, demo blend, softmax
 * (mbd_planner.py:110-127) over the GLOBAL reward vector rews_all_dev [n_total] (all ranks'
 * samples, all-gathered by the caller); writes the softmax weights of the local slice
 * weights_dev [n_local] and scalars_dev[4] = {rews.mean(), rew_std, max logit, sum exp}.
 * logpd_all_dev NULL = enable_demo False.  logp_scratch_dev: n_total floats (receives logp0). */
int mbd_softmax_weights(const float* rews_all_dev, const float* logpd_all_dev, int n_total, int n_begin,
                        int n_local, float temp, float rew_xref, float* weights_dev, float* scalars_dev,
                        float* logp_scratch_dev, mbd_stream s);

/* partial of Ybar = einsum("n,nij->ij", weights, Y0s) over the local samples
 * (mbd_planner.py:128), deterministic order (64-sample runs, then a pairwise tree) so that
 * sharded and unsharded runs agree bit for bit.  scratch_dev: ceil(n_local/64)*HNu floats. */
int mbd_weighted_sum(const float* weights_dev, const float* Y0s_dev, int n_local, int HNu, float* scratch_dev,
                     float* partial_dev, mbd_stream s);

/* First stage of mbd_weighted_sum only: runs_dev [ceil(n_local/64)][HNu].  Returns the number of runs (> 0) or a
 * negative error.  With one rank the pairwise tree over the runs is the same tree mbd_update applies to its
 * `partials`, so `mbd_update(runs, P = nruns, ...)` finishes the weighted mean and the update in one launch. */
int mbd_weighted_sum_runs(const float* weights_dev, const float* Y0s_dev, int n_local, int HNu, float* runs_dev, mbd_stream s);

/* einsum("n,nij->ij", weights, (Y0s - mu_0t)**2): the CMA-ES spread update of
 * upstream mbd/planners/path_integral.py:39-45, same deterministic order as mbd_weighted_sum. */
int mbd_weighted_sqerr_sum(const float* weights_dev, const float* Y0s_dev, const float* mu_dev, int n_local, int HNu,
                           float* scratch_dev, float* partial_dev, mbd_stream s);

/* Test hook: the device build of the fp32 math specification, element-wise, so tests can compare it with float64 and with
 * the host build.  Ops: MBD_DIV (0), MBD_RCP (1), MBD_SQRT (2), mbd_atan2f (3) — the branch-free exact device sequences of
 * include/mbd_fp32.h — and the packed rollout kernel's atan2_ (csrc/pk_scalar.cuh): its scalar instantiation (4) and its
 * two-lane f2 instantiation with element i in the low (5) or the high (6) half, element n-1-i in the other;
 * mbd_logf (7), mbd_expf (8), the sine (9) and the cosine (10) of mbd_sincosf, mbd_erfinvf (11), mbd_bits_to_normal of a's
 * bits (12), mbd_tanhf (13), mbd_softplusf (14), mbd_swishf (15);  the packed kernel's scalar rcp_ (16), div_ (17),
 * div_nn_ (18), sqrt_ (19) and the low / high halves of their two-lane forms, paired like ops 5 and 6: rcp_ (20 / 21),
 * div_ (22 / 23), div_nn_ (24 / 25), sqrt_ (26 / 27);  and planted mistakes that exist only here, each a spec function
 * with one step removed: the sine without its third Cody-Waite constant (28), mbd_expf without its second (29), rcp as the
 * bare rcp.approx seed (30), sqrt without its final FMA (31), a division returning a * r after one Newton step (32), sqrt
 * without the exact scaling of arguments below 2^-100 (33). */
int mbd_test_arith(int op, const float* a_dev, const float* b_dev, float* out_dev, int n, mbd_stream s);

/* Test hook: err_dev[i] (double) = the error of op (as mbd_test_arith) at (a[i], b[i]) against a float64 reference from
 * CUDA's double libm, in metric (u = 2^-24): ulps of fl(ref) (0), u |ref| (1), u (1 + |ref|) (2), u absolute (3), u |a| (4),
 * exact: 0 when the result has the bits of fl(ref), else its distance in ulps and at least 1 (5), atan2 composed with the
 * rounding of its quotient (6).  Metrics 1-4 forgive 2^-149 where |ref| < 2^-126.  The reference of a division, reciprocal
 * or square root is the double operation, so fl(ref) is the correctly rounded float result. */
int mbd_test_err(int op, int metric, const float* a_dev, const float* b_dev, double* err_dev, int n, mbd_stream s);

/* Test hook: op and metric as mbd_test_err over the floats with bits first_bits + k * stride, k < count (uint32
 * arithmetic), with `other` as the other operand (the first one when other_first).  Writes per block (nblocks of 256
 * threads) the largest error (-1 for a block without inputs), the bits of the first input reaching it and the number of
 * inputs with a nonzero error; the reduction order is fixed, so the result is deterministic. */
int mbd_test_sweep(int op, int metric, uint32_t first_bits, uint32_t count, uint32_t stride, float other, int other_first,
                   int nblocks, double* err_dev, uint32_t* bits_dev, uint32_t* cnt_dev, mbd_stream s);

/* Ybar = tree-sum of the P rank partials; then score / Yim1 / Ybar_im1 literally as
 * mbd_planner.py:100,130-133.  coef = {sqrt(ab_i), 1/(1-ab_i), 1-ab_i, 1/sqrt(alpha_i), sqrt(ab_{i-1})}. */
int mbd_update(const float* partials_dev, int P, int HNu, const float* Ybar_i_dev, const float coef[5],
               float* Ybar_im1_dev, mbd_stream s);

/* pushT (upstream mbd/envs/pushT.py:16-66, the reference's one env on Brax's `generalized` backend; planar
 * reduced-coordinate pipeline restated in include/mbd_pusht.h).  params_dev [MBD_PT_NPARAM], x0_dev [16] = q | qd.
 * key != NULL: fused sampling exactly as mbd_car2d_rollout.  final_state_dev [n,16], traj_dev [n,H,16] optional. */
int mbd_pusht_rollout(const float* params_dev, const float* x0_dev, const uint32_t* key, int n_total, int n_begin,
                      int n_local, int H, float sigma, const float* Ybar_dev, float* Y0s_dev, float* rewss_dev,
                      float* rews_dev, float* final_state_dev, float* traj_dev, mbd_stream s);
enum { MBD_ENV_CAR2D = 0, MBD_ENV_PUSHT = 1 };

/* ---- one diffusion step as THREE parameterless launches (CUDA-graph capturable) -------------------------------------
 * reverse_once (mbd_planner.py:97-135) for any rank count: (1) sampling + rollouts, (2) global reward statistics /
 * demo blend / softmax in one 8-CTA thread-block cluster that pulls the peers' per-sample returns over NVLink itself,
 * (3) weighted-mean runs whose last CTA folds the tree, exchanges the rank partials over NVLink and applies the update
 * lines 130-133.  Everything that changes from step to step lives in DEVICE memory: params_dev[i] = {Y0s_rng key
 * (mbd_planner.py:103), sigmas[i], the five schedule scalars of mbd_update}, ctl_dev->i = the step index (the host loop
 * variable of mbd_planner.py:141), decremented by the last thread of launch (3); the iterate Ybar_i is row i of Ybars_dev
 * and the result is written to row i - 1, rews.mean() to rew_hist_dev[i].  The host therefore launches the same three
 * kernels Ndiffuse-1 times (or replays one captured graph) without touching a parameter. */
typedef struct mbd_step_params { uint32_t key[2]; float sigma; float coef[5]; } mbd_step_params; /* 32 bytes */
#define MBD_STEP_MAX_COLBLOCKS 27 /* H*Nu <= 27*256 */
typedef struct mbd_step_ctl {      /* 128 bytes, zero-initialised by the caller except `i` */
  int32_t i;                       /* current step index (Ndiffuse-1 ... 1) */
  uint32_t epoch;                  /* cross-GPU rendezvous counter (advanced once per step) */
  uint32_t err;                    /* 1: a cross-GPU rendezvous timed out (outputs are NaN-poisoned); 2: a step was launched with
                                    * i < 1, past the end of the solve (launches 2 and 3 returned without writing anything) */
  uint32_t pad;
  uint32_t ticket[28];             /* "last CTA done" tickets: per column block, [27] over the column blocks... see step_tail.cuh */
} mbd_step_ctl;
typedef struct mbd_step_plan {
  const mbd_model* model;            /* Brax-positional env; NULL = a flat-state env selected by env_kind: car2d (car_params_dev,
                                      * state_init_dev = x0[3]) or pushT (car_params_dev = the MBD_PT_* table, state_init_dev = q|qd [16]) */
  const float* car_params_dev;
  const float* state_init_dev;       /* [L,13] */
  const mbd_step_params* params_dev; /* [Ndiffuse] */
  mbd_step_ctl* ctl_dev;
  float* Ybars_dev;                  /* [Ndiffuse, H*Nu] */
  float* rew_hist_dev;               /* [Ndiffuse] or NULL */
  int32_t n_total, n_begin, n_local, H, nu;
  float temp, rew_xref;
  const float* xref_dev;             /* demo reference (enable_demo) or NULL */
  int32_t href;
  int32_t env_kind;                  /* model == NULL: MBD_ENV_CAR2D (0, the default) or MBD_ENV_PUSHT; sits in what was padding */
  float* Y0s_dev;                    /* [n_local, H*Nu] */
  float* rews_dev;                   /* [n_local]; P > 1: inside this rank's symmetric buffer at off_rews_words */
  float* logpd_dev;                  /* [n_local] or NULL; P > 1: at off_logpd_words */
  float* rews_all_dev;               /* [n_total] (unused when P == 1) */
  float* logpd_all_dev;              /* [n_total] or NULL */
  float* logp_dev;                   /* [n_total] scratch */
  float* weights_dev;                /* [n_local] */
  float* runs_dev;                   /* [ceil(n_local/64), H*Nu] */
  float* partial_dev;                /* [H*Nu]; P > 1: inside the symmetric buffer at off_partial_words */
  float* scalars_dev;                /* [4] = {rews.mean(), rew_std, max logit, sum exp} of the last step */
  int32_t P, rank;
  const uint64_t* peer_base_ptrs;    /* host array [P]: base address of every rank's symmetric buffer (NULL when P == 1) */
  uint64_t off_rews_words, off_logpd_words, off_partial_words, off_flags_words;  /* flags: 2 rows of 8 words, zeroed */
  uint64_t timeout_cycles;           /* cross-GPU rendezvous timeout in SM cycles; 0 = default (~20 s) */
  /* planner ensemble (appended; mbd_batch_step_launch / mbd_pi_batch_step_launch only, xpbd envs, DESIGN.md §5l).  Problem b
   * rolls every sample Y_bn out under ens_k models (f_bk, g_bk): every contact friction fl(mu * f_bk), every actuator gear
   * fl(gear * g_bk).  ens_rews[b][n][k] receives each member return r_bnk; the sample return the tail reads is
   * rews[b][n] = fl(fl(fl(r_bn0 + r_bn1) + ...) / ens_k), summed in member order.  NULL / 0 = today's step.
   * ens_worst = m >= 1 scores a sample by its m worst members instead (DESIGN.md §5m): NaN (0x7fffffff) if any r_bnk is NaN,
   * otherwise the K returns sorted ascending, ties by member index, s = r_(0), s = fl(s + r_(j)) for j = 1 .. m - 1, and
   * rews[b][n] = fl(s / m).  m = 1 is the minimum, m = K / 2 a discrete CVaR at 50 %.  0 = the ordered mean above. */
  const float* ens_factors_dev;      /* [B][ens_k][2]: friction factor, gear factor of every member of every problem */
  float* ens_rews_dev;               /* [B][N][ens_k] */
  int32_t ens_k;                     /* members per problem, 1 .. MBD_ENS_MAXK with a table, 0 without */
  int32_t ens_worst;                 /* 0 .. ens_k with a table (0 = the mean), 0 without */
} mbd_step_plan;
#define MBD_ENS_MAXK 16
/* Test entry point: the score launch of an ensemble step alone, on whatever the caller put into ens_rews_dev [count][K]:
 * rews_dev [count] <- the ordered mean (worst == 0) or the worst-m score (m = worst) of each row.  MBD_EINVAL before any CUDA call for a
 * NULL buffer, count < 1, K outside 1 .. MBD_ENS_MAXK or worst outside 0 .. K. */
int mbd_ens_score(const float* ens_rews_dev, float* rews_dev, int count, int K, int worst, mbd_stream s);
/* Members drawn afresh at every control step of the receding-horizon controllers (DESIGN.md §5m).  One launch, one thread per
 * (problem b, member k), graph-capturable: with c = mpc_ctl[b] and c < Nstep, (kf, kg) = split(keys[b][c]) and
 * ens_factors[b][k] = (uniform(kf, (K,), flo_b, fhi_b)[k], uniform(kg, (K,), glo_b, ghi_b)[k]) in the threefry layout of the
 * samplers (prng.split / prng.uniform); a problem with c outside 0 .. Nstep - 1 is not written.  MBD_EINVAL before any CUDA call
 * for a NULL plan or buffer, B outside 1 .. MBD_VEC_MAX_B, K outside 1 .. MBD_ENS_MAXK or Nstep < 1.  The ranges are the caller's
 * to check (finite, 0 <= lo <= hi). */
typedef struct mbd_ens_draw_plan {
  int32_t B, K, Nstep, pad;
  const uint32_t* keys_dev;          /* [B][Nstep][2]: the member key of every control step of every problem */
  const float* ranges_dev;           /* [B][4]: friction lo, friction hi, gear lo, gear hi */
  const int32_t* mpc_ctl_dev;        /* [B]: the control step counter of mbd_mpc_advance */
  float* ens_factors_dev;            /* [B][K][2]: mbd_step_plan.ens_factors_dev */
} mbd_ens_draw_plan;
int mbd_ens_draw(const mbd_ens_draw_plan* plan, mbd_stream s);
/* mbd_step_launch, mbd_step_launch_ev and mbd_step_tail_launch refuse an ensemble (MBD_EINVAL): the single-solve, sharded and
 * benchmark step keep their three launches. */
int mbd_step_launch(const mbd_step_plan* plan, mbd_stream s);
/* B independent solves of one env and shape in lockstep: three launches, graph-capturable.  Every per-problem buffer of
 * `plan` holds B consecutive single-problem blocks (state_init [B][state], params [B][Ndiffuse], ctl [B],
 * Ybars [B][Ndiffuse][HNu], rew_hist [B][Ndiffuse], Y0s [B][N][HNu], rews / logpd / logp / weights [B][N],
 * runs [B][nruns][HNu], scalars [B][4]); plan->n_total = n_local = N, n_begin = 0, P = 1.
 * temps_dev [B] or NULL (= plan->temp for every problem).  car_params / xref are shared by all problems.  Problem b draws
 * the noise of a stand-alone solve with its own key and reduces in the same order, so it reproduces mbd_step_launch on
 * its own buffers bit for bit.  MBD_EINVAL (with mbd_last_error) before any CUDA call for B < 1, P != 1, Ndiffuse < 2 or
 * a plan mbd_step_launch would refuse.
 * With a planner ensemble (ens_factors_dev) launch (1) becomes three launches: the batched sampler (the fused kernels' Y0s bits),
 * the ensemble rollout (rollout slot s of problem b is sample s / ens_k under member s % ens_k) and the ordered member mean into
 * rews; launches (2) and (3) follow unchanged.  MBD_EINVAL before any CUDA call for a table without ens_rews or ens_rews without a
 * table, ens_k outside 1 .. MBD_ENS_MAXK with a table or not 0 without one, a flat-state env (model NULL), a demo (xref) or
 * B * N * ens_k >= 2^31. */
int mbd_batch_step_launch(const mbd_step_plan* plan, int B, int Ndiffuse, const float* temps_dev, mbd_stream s);
/* ---- the path-integral baselines (upstream mbd/planners/path_integral.py:33-52) as the same three launches ----------------
 * B independent refinements of one env and shape in lockstep, laid out exactly as mbd_batch_step_launch (Ndiffuse = Nrefine
 * rows: Ybars row i = mu_0t of step i, the result goes to row i - 1, rews.mean() to rew_hist[i]).  Launch (1) is unchanged and
 * reads sigma_t from params[i].sigma; launch (2) computes the softmax weights of path_integral.py:116-124 (and, for CEM, selects
 * the top 10); launch (3) applies the method's update:
 *   MBD_PI_MPPI   Ybars[i-1] = sum_n w_n Y_n
 *   MBD_PI_CMAES  Ybars[i-1] as MPPI; sigma' = max(mean_j sqrt(sum_n w_n (Y_nj - Ybars[i]_j)^2) * sigma_i, 1e-3) (fp32) is written
 *                 to params[i-1].sigma (read by the next step's launch (1)) and to sigma_hist[i-1]
 *   MBD_PI_CEM    idx = argsort(w)[::-1][:10] (stable, so equal weights come highest index first); Ybars[i-1] = mean of those rows
 * A batch of one runs the single-problem (non-batched) kernel instantiations. */
enum { MBD_PI_MPPI = 1, MBD_PI_CMAES = 2, MBD_PI_CEM = 3 };
#define MBD_PI_IDX_STRIDE 16 /* ints per problem in cem_idx_dev: slots 0..9 = picked rows in rank order (-1 past the count), 10 = count */
typedef struct mbd_pi_bufs {        /* 24 bytes */
  float* sigma_hist_dev;            /* [B][Nrefine]; CMA-ES writes row i - 1 of each step (may be NULL for MPPI / CEM) */
  float* cma_scratch_dev;           /* CMA-ES: [B][ceil(N/64) + 1][H*Nu] (NULL otherwise) */
  int32_t* cem_idx_dev;             /* CEM: [B][MBD_PI_IDX_STRIDE] (NULL otherwise) */
} mbd_pi_bufs;
/* tail_only != 0: launches (2) and (3) only, on whatever the caller put into Y0s / rews / Ybars[i] / params[i] (tests); it ignores
 * the ensemble fields.  Otherwise a planner ensemble runs launch (1) as mbd_batch_step_launch does.
 * MBD_EINVAL (with mbd_last_error) before any CUDA call for an unknown method, P != 1, Nrefine < 2, B outside 1..65535, a demo
 * (xref), a missing buffer of the method, or a plan mbd_batch_step_launch would refuse. */
int mbd_pi_batch_step_launch(const mbd_step_plan* plan, int B, int Nrefine, int method, const float* temps_dev,
                             const mbd_pi_bufs* bufs, int tail_only, mbd_stream s);
/* ---- model-based diffusion as a black-box optimiser (upstream mbd/blackbox/mbd_opt.py:64-80) as the same three launches -------
 * B independent solves of one objective and shape in lockstep, laid out as mbd_batch_step_launch with H = 1 and nu = dim
 * (model, car_params, state_init and xref are not read and model / xref must be NULL).  Launch (1) (csrc/blackbox.cuh) draws
 * Y0s = clip(normal(params[i].key, (N, dim)) * params[i].sigma + mu, -1, 1), where mu is Ybars row i or, on the first step
 * (i == Ndiffuse - 1), the per-sample normal(init_keys[b], (N, dim)) of mbd_opt.py:84; it writes rews = J = -f(Y0s) and folds
 * max_n J_n into best_hist[b][i].  Launches (2) and (3) are those of MBD_PI_MPPI: Ybars[i-1] = sum_n w_n Y_n.
 * MBD_EINVAL (with mbd_last_error) before any CUDA call for an unknown fn, P != 1, Ndiffuse < 2, B outside 1..65535, H != 1, a
 * model or xref in the plan, missing bufs, x_min >= x_max, or a plan mbd_batch_step_launch would refuse (dim > 27 * 256,
 * N * dim >= 2^32). */
enum { MBD_BBO_ACKLEY = 1, MBD_BBO_RASTRIGIN = 2, MBD_BBO_LEVY = 3 };
typedef struct mbd_bbo_bufs {        /* 24 bytes */
  const uint32_t* init_keys_dev;     /* [B][2]: PRNGKey(seed) of each problem (the first step's per-sample mean) */
  float* best_hist_dev;              /* [B][Ndiffuse]: row i = max_n J_n of step i; initialised by the caller (-inf) */
  float x_min, x_max;                /* domain map X = x_min + (x_max - x_min) * (Y + 1) / 2 */
} mbd_bbo_bufs;
int mbd_bbo_batch_step_launch(const mbd_step_plan* plan, int B, int Ndiffuse, int fn, const float* temps_dev,
                              const mbd_bbo_bufs* bufs, mbd_stream s);

/* ---- model-based diffusion over the weights of a 784-32-32-10 MLP (upstream mbd/blackbox/mbd_mnist.py) ---------------------
 * One solve (B = 1) laid out as mbd_batch_step_launch with H = 1 and nu = 26506 (the parameter row of csrc/mnist.cuh: W1
 * transposed, b1, W2, b2, W3, b3).  A step is six parameterless launches (graph-capturable): sampling of the six tensors with the
 * keys of keys_dev[i]; the forward pass of all N models on the minibatch batch_idx_dev[i] (layer 1 on the tensor cores, split
 * TF32) -> rews = Js; the MPPI weights (mbd_pi_batch_step_launch's launch (2)) -> rew_hist[i] = Js.mean(); the weighted mean in
 * two launches -> Ybars[i - 1]; the accuracy of the new mean on the training and test sets -> acc_hist[i] (every eval_every
 * steps, others keep what the caller put there).  MBD_EINVAL (with mbd_last_error) before any CUDA call for layer sizes other
 * than 784-32-32-10, N < 1 or N > n_train, Ndiffuse < 2, missing buffers, a plan with a model / demo / P != 1 / H != 1 /
 * nu != 26506, or the other plan errors of mbd_batch_step_launch. */
#define MBD_MNIST_HNU 26506
typedef struct mbd_mnist_bufs {
  const uint8_t* train_images_dev;   /* [n_train][784] */
  const uint8_t* train_labels_dev;   /* [n_train] */
  const uint8_t* test_images_dev;    /* [n_test][784] */
  const uint8_t* test_labels_dev;    /* [n_test] */
  const uint32_t* keys_dev;          /* [Ndiffuse][12][2]: (noise key, mask key) of W1, b1, W2, b2, W3, b3 for every step */
  const int32_t* batch_idx_dev;      /* [Ndiffuse][N]: the minibatch of every step (mbd_mnist_batch_indices) */
  int32_t* acc_hist_dev;             /* [Ndiffuse][2]: train / test correct-counts of the mean after step i */
  int32_t layers[4];                 /* must be {784, 32, 32, 10} */
  int32_t n_train, n_test, eval_every;
} mbd_mnist_bufs;
int mbd_mnist_step_launch(const mbd_step_plan* plan, int Ndiffuse, const mbd_mnist_bufs* bufs, mbd_stream s);
/* Test entry point: Js[n] of models Y0s_dev [n_models][26506] on the images rows_dev [n_img] of the training set of bufs (no step
 * counter); z1_dev [n_models][n_img][32] (or NULL) receives the layer-1 pre-activations sum_k x_k W1[k][o] / 255 (before b1). */
int mbd_mnist_forward(const float* Y0s_dev, int n_models, const mbd_mnist_bufs* bufs, const int32_t* rows_dev, int n_img,
                      float* Js_dev, float* z1_dev, mbd_stream s);
/* The minibatch table: row t (1 <= t < Ndiffuse) = permutation(batch_rng_t, n_data)[:N] with two rounds of a stable sort by
 * random_bits(sub_r, (n_data,)); sub_keys_host [Ndiffuse][2][2] = the two round keys of every step.  scratch_dev NULL: writes the
 * scratch size needed to *scratch_bytes and returns.  Synchronous on the stream's work only (no host synchronisation). */
int mbd_mnist_batch_indices(const uint32_t* sub_keys_host, int Ndiffuse, int n_data, int N, int32_t* idx_dev, void* scratch_dev,
                            size_t* scratch_bytes, mbd_stream s);

/* ---- a batch of environments stepped together on the device (vmap(env.reset) / vmap(env.step) with Brax's training wrappers) --
 * B environments of one kind, each with its own state, stepped by two launches: (1) the env's rollout kernel with H = 1 and a
 * per-sample start state (state -> next_state, reward), (2) one thread per env that computes the observation (xpbd envs: com.to_world
 * and kinematics.inverse in float64 from the float32 state, rounded once: include/mbd_kin64.h), the env's done, the episode counters
 * and the auto-reset, and writes the chosen state back into state.  Both launches read everything from the plan, allocate nothing
 * and do not synchronise: a step can be captured in a CUDA graph.  Buffers (device, caller-owned, fixed for the plan's lifetime):
 *   state / next_state / first_state [B][S] (S = Lsim * 13, pushT 16, car2d 3), actions [B][Nu], obs / first_obs [B][O],
 *   reward / done / truncation / steps [B] (float32, steps counts env steps since the last reset).
 * episode_length > 0 adds Brax's EpisodeWrapper + AutoResetWrapper (action_repeat 1): steps is zeroed where the previous done was set,
 * then steps += 1; done = steps >= episode_length ? 1 : env_done; truncation = steps >= episode_length ? 1 - env_done : 0; where done
 * is set, state and obs are replaced by first_state and first_obs (reward and done of the step are returned as computed). */
enum { MBD_VEC_XPBD = 0, MBD_VEC_CAR2D = 1, MBD_VEC_PUSHT = 2 };
enum { MBD_VEC_OBS_QQD = 0,     /* q | qd (humanoids, cartpole) */
       MBD_VEC_OBS_HOPPER = 1,  /* q with q[1] = x.pos[0, 2], clip(qd, -10, 10) (hopper, walker2d) */
       MBD_VEC_OBS_SKIP2 = 2,   /* q[2:] | qd (ant) */
       MBD_VEC_OBS_SKIP1 = 3,   /* q[1:] | qd (halfcheetah) */
       MBD_VEC_OBS_STATE = 4 }; /* the flat state itself (pushT q | qd, car2d x) */
enum { MBD_VEC_DONE_ZERO = 0, MBD_VEC_DONE_COUNTER = 1 /* humanoidtrack: done = previous done + 1 */, MBD_VEC_DONE_PUSHT = 2 /* reward > 0.95 */ };
enum { MBD_VEC_RESET_NONE = 0 /* init_q, qd = 0 */, MBD_VEC_RESET_UNIFORM = 1 /* q, qd + U(lo, hi) */,
       MBD_VEC_RESET_NORMAL = 2 /* q + U(lo, hi), qd = clip(sigma N(0, 1), -1, 1) */, MBD_VEC_RESET_PUSHT = 3, MBD_VEC_RESET_CONST = 4 };
#define MBD_VEC_MAX_B 65536
/* reset table (float32, MBD_VEC_RT_* words then init_q [nq] and the q offset [nq]) */
enum { MBD_VEC_RT_KIND = 0, MBD_VEC_RT_LO = 1, MBD_VEC_RT_HI = 2, MBD_VEC_RT_SIGMA = 3, MBD_VEC_RT_HAS_OFF = 4, MBD_VEC_RT_Q = 8 };
typedef struct mbd_vec_plan {
  int32_t kind;                 /* MBD_VEC_* */
  int32_t B;
  const mbd_model* model;       /* MBD_VEC_XPBD: the env's model; NULL otherwise */
  const float* params_dev;      /* car2d / pushT parameter table (as mbd_car2d_rollout / mbd_pusht_rollout); NULL for xpbd */
  const double* kin_dev;        /* xpbd: the float64 kinematics table of include/mbd_kin64.h */
  const float* reset_dev;       /* reset table (MBD_VEC_RT_*) */
  int32_t obs_layout;           /* MBD_VEC_OBS_* */
  int32_t done_rule;            /* MBD_VEC_DONE_* */
  int32_t episode_length;       /* 0 = no episode wrapper / auto-reset */
  int32_t nq, nqd, nu;          /* joint coordinate / velocity / action sizes (flat envs: state size, 0, nu) */
  float* state_dev;
  float* next_state_dev;
  float* first_state_dev;
  float* actions_dev;
  float* obs_dev;
  float* first_obs_dev;
  float* reward_dev;
  float* done_dev;
  float* truncation_dev;
  float* steps_dev;
  float* factors_dev;           /* xpbd envs: [B][2] model factors (friction, actuator gear) of every env: env b steps with every contact
                                 * friction fl(mu * F[b][0]) and every actuator gear fl(gear * F[b][1]); NULL = the nominal model.  A
                                 * non-NULL table for car2d / pushT is MBD_EINVAL.  mbd_vec_reset_dr / mbd_vec_step_dr write it. */
} mbd_vec_plan;
/* env.reset(keys[b]) for every env b (keys_dev [B][2] uint32), in the threefry layout of mbd_set_prng_layout: state, first_state, obs,
 * first_obs, reward (0, pushT its reward), done, truncation 0, steps 0. */
int mbd_vec_reset(const mbd_vec_plan* plan, const uint32_t* keys_dev, mbd_stream s);
/* one env step of every env with the actions in plan->actions_dev (launches (1) and (2) above); with factors_dev, launch (1) is the
 * per-env-model instantiation of the same kernel choice */
int mbd_vec_step(const mbd_vec_plan* plan, mbd_stream s);
/* obs of the states the caller wrote into state_dev; first_state = state, first_obs = obs; reward, done, truncation, steps 0 */
int mbd_vec_set_state(const mbd_vec_plan* plan, mbd_stream s);
/* xpbd envs: world link poses x.pos [B][L][3], x.rot [B][L][4] of the current states (PipelineEnv._make_pipeline_state) */
int mbd_vec_world_poses(const mbd_vec_plan* plan, float* pos_dev, float* rot_dev, mbd_stream s);
/* domain randomisation (xpbd envs; DESIGN.md §5n): a new draw of the plan's factor table at every episode of every env.
 * keys_dev [B][2] uint32 is env b's DR key dk_b; episodes_dev [B] counts env b's episodes.  Episode e of env b steps with
 * factors_dev[b] = (f, g): kf, kg = split(threefry2x32(dk_b, (0, e))), f = uniform(kf, (1,), flo, fhi)[0],
 * g = uniform(kg, (1,), glo, ghi)[0], in the threefry layout of mbd_set_prng_layout.  range = {flo, fhi, glo, ghi}, finite, >= 0,
 * lo <= hi. */
typedef struct mbd_vec_dr {
  const uint32_t* keys_dev;
  int32_t* episodes_dev;
  float range[4];
} mbd_vec_dr;
/* mbd_vec_reset that also zeroes episodes and writes episode 0's factors into plan->factors_dev */
int mbd_vec_reset_dr(const mbd_vec_plan* plan, const mbd_vec_dr* dr, const uint32_t* keys_dev, mbd_stream s);
/* mbd_vec_step that, where an env auto-resets, adds 1 to its episode count and writes that episode's factors (the step that ends an
 * episode is computed under the old ones; launch (1) of the next step reads the new ones).  Both refuse, with MBD_EINVAL before any
 * CUDA call, dr == NULL, car2d / pushT, a plan without factors_dev, NULL keys_dev / episodes_dev and a bad range. */
int mbd_vec_step_dr(const mbd_vec_plan* plan, const mbd_vec_dr* dr, mbd_stream s);

/* ---- PPO on the vector env (Brax's ppo.train, v0.10.x line [brax-recalled]; mbd_b200/rl) ---------------------------------------
 * The acting step, the observation statistics and GAE on the device; the nets, the loss and Adam stay in torch.  A training step's
 * rollout is one time series of `slots` = U * T acting slots of B envs: obs [slots + 1][B][O], raw [slots][B][Nu], logp / reward /
 * disc / trunc [slots][B]; trajectory n = u * B + b is slots u * T ... u * T + T - 1 of env b and its bootstrap observation is slot
 * u * T + T.  act_ctl_dev [4] = {slot t, key row k, ticket (0), 0}: every act launch reads them, and its last CTA advances them.
 * MBD_EINVAL (with mbd_last_error) before any CUDA call for O outside 1..128, Nu outside 1..32, B outside 1..MBD_VEC_MAX_B or a
 * missing buffer of the entry point. */
enum { MBD_PPO_ACT = 0,          /* obs[t] = env obs; reward / disc / trunc [t - 1] = the env's (t > 0); raw[t], logp[t]; actions = tanh(raw)
                                  * with eps = normal(act_keys[k], (B, Nu)); t += 1, k += 1 */
       MBD_PPO_RECORD = 1,       /* the records of MBD_PPO_ACT without acting (after an unroll's last step); t = 0 */
       MBD_PPO_EVAL = 2,         /* t > 0: ret += active * reward, active *= 1 - done; then act as MBD_PPO_ACT without records; t += 1, k += 1 */
       MBD_PPO_EVAL_RECORD = 3 };/* the accumulation of MBD_PPO_EVAL without acting; t = 0 */
#define MBD_PPO_MAX_OBS 128
#define MBD_PPO_MAX_NU 32
#define MBD_PPO_MAX_MB 4096     /* trajectories per minibatch; a GAE thread takes every 1024th */
#define MBD_PPO_STAT_ROWS 256    /* rows per partial sum of mbd_ppo_obs_stats */
typedef struct mbd_ppo_plan {
  int32_t B, O, nu;              /* envs, observation size, action size */
  int32_t slots;                 /* acting slots of one training step (U * T) */
  int32_t unroll;                /* T */
  int32_t mb;                    /* trajectories per minibatch (GAE) */
  float reward_scaling, discount, gae_lambda;
  int32_t act_key_rows;          /* rows of act_keys_dev: an act launch past the table writes nothing */
  int32_t loss_key_rows;         /* rows of loss_keys_dev: a GAE launch past the table draws no noise */
  const float* policy_dev;       /* flat policy parameters (include/mbd_ppo.h) */
  const float* mean_dev;         /* [O] running mean (float32) */
  const float* std_dev;          /* [O] running std (float32) */
  const uint32_t* act_keys_dev;  /* [n][2] act keys, row k */
  int32_t* act_ctl_dev;          /* [4] */
  const float* env_obs_dev;      /* the vector env's obs [B][O], reward, done, truncation [B] and actions [B][Nu] */
  const float* env_reward_dev;
  const float* env_done_dev;
  const float* env_trunc_dev;
  float* env_actions_dev;
  float* obs_dev;                /* the rollout (MBD_PPO_ACT / MBD_PPO_RECORD, and GAE) */
  float* raw_dev;
  float* logp_dev;
  float* reward_dev;
  float* disc_dev;
  float* trunc_dev;
  float* ret_dev;                /* evaluation: [B] episode return and active flag */
  float* active_dev;
  double* stat_dev;              /* [1 + 2 O]: count, mean, summed variance (float64) */
  double* stat_scratch_dev;      /* [ceil(slots * B / MBD_PPO_STAT_ROWS)][2][O] */
  const uint32_t* loss_keys_dev; /* [n][2] loss keys, row *loss_ctl_dev */
  const int32_t* loss_ctl_dev;
  const int32_t* traj_dev;       /* [mb] trajectory ids of the minibatch */
  const float* values_dev;       /* [T + 1][mb] values of the minibatch's observations (row T: the bootstrap values) */
  float* vs_dev;                 /* [T][mb] value targets */
  float* adv_dev;                /* [T][mb] normalised advantages */
  float* ent_eps_dev;            /* [T][mb][Nu] = normal(loss key, (T, mb, Nu)) */
} mbd_ppo_plan;
/* one launch: the policy of every env (warp per env, lane per hidden unit) in the given MBD_PPO_* mode */
int mbd_ppo_act(const mbd_ppo_plan* plan, int mode, mbd_stream s);
/* running_statistics.update with obs rows 0 .. slots * B - 1 (two launches, float64 sums in a fixed order); writes mean_dev / std_dev
 * (std = clip(sqrt(summed_var / count), 1e-6, 1e6)) */
int mbd_ppo_obs_stats(const mbd_ppo_plan* plan, mbd_stream s);
/* one launch per minibatch: compute_gae with the truncation mask on the trajectories traj_dev (rewards * reward_scaling), the
 * advantage normalisation (adv - mean) / (std + 1e-8) (population std) and the entropy noise */
int mbd_ppo_gae(const mbd_ppo_plan* plan, mbd_stream s);

/* ---- SAC on the vector env (Brax's sac.train, v0.10.x line [brax-recalled]; mbd_b200/rl/sac.py) ---------------------------------
 * The acting step, the replay ring and its uniform sampler on the device; the losses and the three Adam optimisers stay in torch.
 * The ring holds `capacity` rows of include/mbd_sac.h's layout; ring_ctl_dev [4] = {pos (next write row), size, ticket (0), 0} gives
 * Brax's queue: logical row i (oldest first) is physical row (pos - size + i) mod capacity.  act_ctl_dev [4] is PPO's {step t, key
 * row k, ticket (0), 0}; sample_ctl_dev [4] = {training step s, ticket (0), buffer key word 0, word 1}.  Each launch's last CTA
 * advances its control words, so a training step is graph-capturable.  MBD_EINVAL (with mbd_last_error) before any CUDA call for O
 * outside 1..128, Nu outside 1..32, B outside 1..MBD_VEC_MAX_B, capacity outside B..MBD_SAC_MAX_CAPACITY or a missing buffer. */
enum { MBD_SAC_ACT = 0,          /* actions = tanh(raw), eps = normal(act_keys[k], (B, Nu)); obs and action into ring rows pos + b, obs
                                  * into stage_obs; k += 1 */
       MBD_SAC_EVAL = 1,         /* PPO's MBD_PPO_EVAL: t > 0: ret += active * reward, active *= 1 - done; then act without records */
       MBD_SAC_EVAL_RECORD = 2 };/* the accumulation of MBD_SAC_EVAL without acting; t = 0 */
#define MBD_SAC_MAX_CAPACITY (1 << 24)
typedef struct mbd_sac_plan {
  int32_t B, O, nu;              /* envs, observation size, action size */
  int32_t capacity;              /* ring rows (max_replay_size) */
  int32_t batch;                 /* rows per gradient update (batch_size) */
  int32_t updates;               /* gradient updates per training step (grad_updates_per_step) */
  int32_t act_key_rows;          /* rows of act_keys_dev: an act launch past the table writes nothing */
  int32_t noise_key_rows;        /* training steps of noise_keys_dev: a sample launch past the table writes nothing */
  const float* policy_dev;       /* flat policy parameters (include/mbd_sac.h) */
  const float* mean_dev;         /* [O] running mean (float32) */
  const float* std_dev;          /* [O] running std (float32) */
  const uint32_t* act_keys_dev;  /* [n][2] act keys, row k */
  int32_t* act_ctl_dev;          /* [4] */
  const float* env_obs_dev;      /* the vector env's obs [B][O], reward, done, truncation [B] and actions [B][Nu] */
  const float* env_reward_dev;
  const float* env_done_dev;
  const float* env_trunc_dev;
  float* env_actions_dev;
  float* ret_dev;                /* evaluation: [B] episode return and active flag */
  float* active_dev;
  float* stage_obs_dev;          /* [B][O] the acting observations (the statistics' input) */
  float* ring_dev;               /* [capacity][mbd_sac_row(O, Nu)] */
  int32_t* ring_ctl_dev;         /* [4] */
  int32_t* sample_ctl_dev;       /* [4] */
  const uint32_t* noise_keys_dev;/* [noise_key_rows][updates][3][2]: key_alpha, key_critic, key_actor of every update */
  int32_t* idx_dev;              /* [updates * batch] logical indices of the sample */
  float* batch_dev;              /* [updates][batch][row] the gathered rows */
  float* eps_dev;                /* [3][updates][batch][Nu] = normal(key_{alpha, critic, actor}, (batch, Nu)) of every update */
} mbd_sac_plan;
/* one launch: the policy of every env (CTA = a tile of envs, thread = hidden unit) in the given MBD_SAC_* mode */
int mbd_sac_act(const mbd_sac_plan* plan, int mode, mbd_stream s);
/* one launch after mbd_vec_step: reward, 1 - done, next obs and truncation into ring rows pos + b; pos += B, size = min(size + B, cap) */
int mbd_sac_record(const mbd_sac_plan* plan, mbd_stream s);
/* one launch per training step: buffer key, sample key = split(buffer key); updates * batch randint indices in 0 .. size - 1 from
 * sample key, the gathered rows, and the three noise tensors of every update from noise_keys row s; s += 1 */
int mbd_sac_sample(const mbd_sac_plan* plan, mbd_stream s);

/* ---- the fused SAC gradient update (include/mbd_sac_learn.h, csrc/sac_learn.cuh) ---------------------------------------------
 * One Brax sgd_step on the batch and noise of update g = *upd_ctl_dev (the sampler's batch_dev / eps_dev of mbd_sac_plan): the three
 * losses with the old parameters, Adam on the policy, Q and log alpha (torch.optim.Adam's formula, the step count ctl_dev[0] + 1),
 * then target_q += tau (q - target_q).  Two launches, no float atomics, graph-capturable: the second launch's last CTA stores the
 * step count and g + 1.  A launch with g outside 0 .. updates - 1 changes nothing.  MBD_EINVAL (with mbd_last_error) before any
 * CUDA call for O outside 1..128, Nu outside 1..32, batch outside 1..MBD_SAC_LEARN_MAX_BATCH, updates < 1, scratch_floats below
 * mbd_sac_learn_scratch(O, Nu, batch) or a missing buffer. */
typedef struct mbd_sac_learn_plan {
  int32_t O, nu, batch, updates;
  float learning_rate;           /* the policy's and Q's Adam rate (log alpha: 3e-4) */
  float reward_scaling, discounting, tau;
  float* policy_dev;             /* flat policy (include/mbd_sac.h), updated in place */
  float* q_dev;                  /* layer-major two-critic Q (mbd_b200/rl/networks.py) */
  float* target_q_dev;
  float* log_alpha_dev;          /* [1] */
  float* policy_m_dev;           /* Adam moments, the layouts of their parameters */
  float* policy_v_dev;
  float* q_m_dev;
  float* q_v_dev;
  float* alpha_mv_dev;           /* [2]: log alpha's m, v */
  int64_t* ctl_dev;              /* [2]: the Adam step count (updates done), ticket (0) */
  const float* mean_dev;         /* [O] observation statistics */
  const float* std_dev;
  const float* batch_dev;        /* [updates][batch][mbd_sac_row(O, Nu)] */
  const float* eps_dev;          /* [3][updates][batch][Nu]: the noise of the alpha, critic and actor losses */
  int64_t* upd_ctl_dev;          /* [1] the update of the training step */
  float* scratch_dev;            /* mbd_sac_learn_scratch(O, Nu, batch) floats */
  int64_t scratch_floats;
  float* losses_dev;             /* [3]: alpha, critic and actor loss of the last update */
} mbd_sac_learn_plan;
/* floats of the scratch buffer of one update */
int64_t mbd_sac_learn_scratch(int O, int nu, int batch);
/* one sgd_step (two launches) */
int mbd_sac_update(const mbd_sac_learn_plan* plan, mbd_stream s);

/* ---- model-based diffusion as a receding-horizon controller (mbd_b200/planners/mbd_mpc.py, DESIGN.md §5i) ----------------------
 * B closed loops of one env and shape, each planning with the buffers of mbd_batch_step_launch (params [B][Ndiffuse], ctl [B],
 * Ybars [B][Ndiffuse][H*nu], rew_hist [B][Ndiffuse]) from the vector env's state (mbd_vec_plan.state_dev, passed as the step plan's
 * state_init).  mpc_ctl_dev [B] holds the control step c of every problem (zeroed by the caller).  One launch, one CTA per problem,
 * graph-capturable.  MBD_EINVAL (with mbd_last_error) before any CUDA call for an unknown mode, B outside 1..MBD_VEC_MAX_B, H or nu
 * below 1, H * nu above 27 * 256, Ndiffuse < 2, Nwarm outside 1..Ndiffuse - 1, Nstep < 1, state_words < 1 or a missing buffer. */
enum { MBD_MPC_ACT = 0,     /* after control step c's last diffusion step: a_c = Ybars[b][0] row 0 into env_actions and actions[c];
                             * s_c into states[0] when c = 0; rew_hist[b][1] into rew_hist_log[c]; when c + 1 < Nstep: shift(P_c) into
                             * Ybars[b][Nwarm], keys row c + 1 into params[b][1 .. Nwarm].key, ctl.i = Nwarm; then c += 1.
                             * Nothing when c >= Nstep. */
       MBD_MPC_RECORD = 1 };/* after mbd_vec_step: the env's reward into rewards[c - 1], its state into states[c] (1 <= c <= Nstep) */
typedef struct mbd_mpc_plan {
  int32_t B, H, nu;                /* problems, horizon, action size */
  int32_t Ndiffuse, Nwarm, Nstep;  /* schedule rows, diffusion steps per warm control step, control steps */
  int32_t state_words;             /* S: words of one env state (the vector env's layout) */
  int32_t pad;
  mbd_step_params* params_dev;     /* [B][Ndiffuse] */
  mbd_step_ctl* ctl_dev;           /* [B] */
  float* Ybars_dev;                /* [B][Ndiffuse][H*nu] */
  const float* rew_hist_dev;       /* [B][Ndiffuse] */
  const uint32_t* keys_dev;        /* [B][Nstep][Nwarm][2]: row c = the keys of diffusion steps 1 .. Nwarm of control step c */
  int32_t* mpc_ctl_dev;            /* [B] */
  float* env_actions_dev;          /* the vector env's actions [B][nu], state [B][S] and reward [B] */
  const float* env_state_dev;
  const float* env_reward_dev;
  float* actions_dev;              /* [B][Nstep][nu] executed actions */
  float* rewards_dev;              /* [B][Nstep] */
  float* states_dev;               /* [B][Nstep + 1][S] */
  float* rew_hist_log_dev;         /* [B][Nstep]: rews.mean() of every control step's last diffusion step */
} mbd_mpc_plan;
int mbd_mpc_advance(const mbd_mpc_plan* plan, int mode, mbd_stream s);

/* ---- the path-integral baselines as receding-horizon controllers (mbd_b200/planners/pi_mpc.py, DESIGN.md §5j) -------------------
 * The same launch for B closed loops that plan with mbd_pi_batch_step_launch: base is the plan above with the baseline engine's
 * buffers (Ndiffuse = Nrefine).  The baselines read their sampling sigma from params[b][t].sigma and CMA-ES rewrites it, so ACT
 * does two more things: it stores params[b][0].sigma, the sigma control step c ended with, into sigma_log[b][c], and when
 * c + 1 < Nstep it writes sigma_warm into params[b][0 .. Nwarm].sigma, so every warm control step restarts from sigma_warm (a
 * reset, not a carry; row 0 is never sampled from, it only feeds the log of the methods that leave sigma alone).  RECORD is
 * mbd_mpc_advance's.  Refuses with MBD_EINVAL (and mbd_last_error) before any CUDA call everything mbd_mpc_advance refuses, a
 * sigma_warm that is <= 0, NaN or infinite, and in ACT mode a missing sigma_log_dev. */
typedef struct mbd_mpc_pi_plan {
  mbd_mpc_plan base;
  float sigma_warm;                /* the sigma every control step c >= 1 starts from */
  int32_t pad;
  float* sigma_log_dev;            /* [B][Nstep] */
} mbd_mpc_pi_plan;
int mbd_mpc_pi_advance(const mbd_mpc_pi_plan* plan, int mode, mbd_stream s);

/* Test / instrumentation entry point: launches (2) and (3) of mbd_step_launch only, on whatever the caller put into Y0s_dev,
 * rews_dev / logpd_dev (the symmetric-buffer slices when P > 1), Ybars_dev[i] and params_dev[i].  Same plan checks as
 * mbd_step_launch (H*Nu above 27*256 is MBD_EINVAL), except that state_init_dev and the env fields are not read. */
int mbd_step_tail_launch(const mbd_step_plan* plan, mbd_stream s);
/* the same three launches with CUDA events (mbd_event_create; NULL = skip) recorded before (1), between (1) and (2), between
 * (2) and (3), after (3): lets a caller time each kernel inside the real step on the launching stream (bench.py's roofline
 * and its per-kernel breakdown at every rank count) */
int mbd_step_launch_ev(const mbd_step_plan* plan, void* ev_before, void* ev_mid, void* ev_mid2, void* ev_after, mbd_stream s);
void* mbd_event_create(void);
void mbd_event_destroy(void* ev);
int mbd_event_record(void* ev, mbd_stream s);
int mbd_event_sync(void* ev);
float mbd_event_elapsed_ms(void* ev_a, void* ev_b);

/* Measured fp32 FFMA throughput of the current device in TFLOP/s (16 independent chains per thread, 2048 threads per SM):
 * the denominator of bench.py's fp32 roofline (SURVEY 8d).  Synchronises the stream. */
int mbd_ffma_peak(float* scratch_dev, int iters, float* tflops_out, mbd_stream s);

#ifdef __cplusplus
}
#endif
#endif /* MBD_B200_H_ */
