// xpbd_wpl.cuh — "warp per link, lane per sample" rollout kernel (v2).
//
// v1 (xpbd_device.cuh) maps one LINK per LANE: ncu showed 16.9 of 32 lanes active on average and
// 31 % of all issue slots spent in the contact code with <= 4 active lanes.  v2 transposes the
// mapping: a CTA owns 32 samples, warp w owns link w of all 32, lane = sample.  Every branch on
// the link's properties (jointed? ndof? contacts?) is warp-uniform, so no lane is ever masked,
// and joint-type specialisation (1-dof links skip the two unused Euler angles) is free.
// The link state (x_i, xd_i, x_i_prev, xd_i_before) stays in registers for the whole rollout;
// what other links need (parent pose, child reaction terms) is exchanged through shared memory,
// [link][field][lane] (conflict-free), with four CTA barriers per physics step:
//     A  joint torques        -> E[l] = T_l            | bar
//     B  gather children T, integrate, publish p,q     | bar
//     C  XPBD joint deltas     -> E[l] = parent deltas  | bar
//     D  gather children deltas, apply, contacts, project_xd, contact velocities, publish q,w | bar
// The arithmetic (association order, fmaf placement, child gather order) is IDENTICAL to v1 and
// to oracle/mbd_oracle.c: results are bit-exact across all three.
#pragma once

#include "xpbd_device.cuh"

// Optional per-phase clock64 accounting (scripts/gpu_phase_prof.py builds with -DMBD_PROFILE_PHASES; the
// product build compiles these macros to nothing).  Slots per link: A, wait, B, wait, C, wait, D, wait.
#ifdef MBD_PROFILE_PHASES
__device__ unsigned long long g_phase_cycles[16][8];
#define MBD_PH_BEGIN unsigned long long tprev_ = clock64();
#define MBD_PH(i) { unsigned long long t_ = clock64(); if (S.lane == 0) atomicAdd(&g_phase_cycles[c.l][i], t_ - tprev_); tprev_ = t_; }
#else
#define MBD_PH_BEGIN
#define MBD_PH(i)
#endif

namespace mbd {

constexpr int kWplLanes = 32;
constexpr int kXF = 10;  // published pose fields per link: p(3) q(4) w(3)
constexpr int kEF = 7;   // exchange fields per link: T(3)  |  dpp(3) dqp(4)

struct WplSmem {
  float* X;  // [L][kXF][32]
  float* E;  // [L][kEF][32]
  int lane;  // sample slot inside a row
  __device__ __forceinline__ float& x(int link, int f) const { return X[(link * kXF + f) * kWplLanes + lane]; }
  __device__ __forceinline__ float& e(int link, int f) const { return E[(link * kEF + f) * kWplLanes + lane]; }
  __device__ __forceinline__ v3 xp(int link) const { return V3(x(link, 0), x(link, 1), x(link, 2)); }
  __device__ __forceinline__ q4 xq(int link) const { return Q4(x(link, 3), x(link, 4), x(link, 5), x(link, 6)); }
  __device__ __forceinline__ v3 xw(int link) const { return V3(x(link, 7), x(link, 8), x(link, 9)); }
  __device__ __forceinline__ void put_p(int link, v3 p) const { x(link, 0) = p.x; x(link, 1) = p.y; x(link, 2) = p.z; }
  __device__ __forceinline__ void put_q(int link, q4 q) const { x(link, 3) = q.w; x(link, 4) = q.x; x(link, 5) = q.y; x(link, 6) = q.z; }
  __device__ __forceinline__ void put_w(int link, v3 w) const { x(link, 7) = w.x; x(link, 8) = w.y; x(link, 9) = w.z; }
  __device__ __forceinline__ v3 e3(int link, int f) const { return V3(e(link, f), e(link, f + 1), e(link, f + 2)); }
  __device__ __forceinline__ q4 e4(int link, int f) const { return Q4(e(link, f), e(link, f + 1), e(link, f + 2), e(link, f + 3)); }
  __device__ __forceinline__ void put_e3(int link, int f, v3 a) const { e(link, f) = a.x; e(link, f + 1) = a.y; e(link, f + 2) = a.z; }
  __device__ __forceinline__ void put_e4(int link, int f, q4 a) const { e(link, f) = a.w; e(link, f + 1) = a.x; e(link, f + 2) = a.y; e(link, f + 3) = a.z; }
};

// warp-uniform link configuration
// Only the integer topology stays in registers; the float constants are warp-uniform and are read
// from the shared-memory model table where they are used (broadcast LDS) — caching them cost ~40
// registers per thread and forced spills under the 2-CTAs/SM register cap.
struct WarpCfg {
  int l, ndof, parent, ncon, smask;   // smask: bit k = dof k is a slide dof (world-parented links only)
  int child[MBD_MAXCHILD];
};

// axis_angle_ang specialised for 1-dof links: only psi and the extra matrix entries are used
// (oracle computes the rest and discards it — same bits for what is used).
__device__ __forceinline__ void axis_angle_1dof(q4 j, float& psi, float& r10, float& r20) {
  float w = j.w, x = j.x, y = j.y, z = j.z;
  float r12 = 2.0f * fmaf(y, z, -(w * x));
  float r22 = 1.0f - 2.0f * fmaf(y, y, x * x);
  r10 = 2.0f * fmaf(x, y, w * z);
  r20 = 2.0f * fmaf(x, z, -(w * y));
  psi = mbd_atan2f(-r12, r22);
}

// ---- synchronisation policies --------------------------------------------------------------------
// SyncCta: four CTA-wide barriers per physics step (simple, any tree).
// (Round 1 also carried an mbarrier-polling edge protocol, "SyncP2P" / kernel variant 4, kept for comparison only: it was
// slower than the named barriers and compute-sanitizer's synccheck flags its unwaited phases — leaf links arrive on pose
// barriers that no child ever waits on — so it was removed in round 2 rather than exempted.)
struct SyncCta {
  __device__ __forceinline__ void wait_pose(int) {}
  __device__ __forceinline__ void arrive_terms(int) {}
  __device__ __forceinline__ void wait_terms(const int*) {}
  __device__ __forceinline__ void arrive_pose(int) {}
  __device__ __forceinline__ void phase_end() { __syncthreads(); }
  template <class C> __device__ __forceinline__ void end_A(const C&) { phase_end(); }
  template <class C> __device__ __forceinline__ void end_B(const C&) { phase_end(); }
  template <class C> __device__ __forceinline__ void end_C(const C&) { phase_end(); }
  template <class C> __device__ __forceinline__ void end_D(const C&) { phase_end(); }
};

// SyncGroup: the packed kernel's sync.  The phases are separated by CTA-wide named barriers (ids base .. base+3),
// except that LEAF links never hold anybody up where nobody depends on them:
//   * after A and after C a leaf only bar.arrive's (the next phase, B or D, gathers from CHILDREN: a leaf has none,
//     so it runs straight on; its parent still sees the leaf's terms because the arrival publishes them);
//   * after D the leaves with contacts ("late" leaves: their D phase is several times longer than anybody else's)
//     are left out of the barrier: everybody else syncs on id_x and then bar.arrive's on id_y, the late
//     leaves bar.sync on id_y — they wait for their parent's pose, nobody waits for them until the end of the
//     next A phase, which therefore overlaps the contact solve.
// Hazards: a leaf's X row is read by nobody; its E row is read by the parent in B and D, and rewritten by the leaf
// only in C (after the CTA-wide B->C barrier) and in A (after id_y, i.e. after the parent finished D).
template <int NL>
struct SyncGroup {
  // ids base+0: after A and after C; base+1: after B; base+2 / base+3: after D.  A warp never touches the same id
  // twice without a blocking CTA-wide barrier on ANOTHER id in between (a hardware barrier has one arrival
  // counter: a second arrival of the same warp would be counted into the generation that is still open).
  // bar.arrive orders the warp's earlier shared-memory writes before the barrier completes (CUTLASS NamedBarrier idiom).
  int base, count_x;   // count_x = 32 * (links that are not late leaves)
  static constexpr int kCount = 32 * NL;
  static __device__ __forceinline__ void bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
  static __device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
  template <class C> static __device__ __forceinline__ bool leaf(const C& c) { return c.child[0] < 0; }   // children are packed from slot 0
  __device__ __forceinline__ void wait_pose(int) {}
  __device__ __forceinline__ void arrive_terms(int) {}
  __device__ __forceinline__ void wait_terms(const int*) {}
  __device__ __forceinline__ void arrive_pose(int) {}
  template <class C> __device__ __forceinline__ void end_A(const C& c) { if (leaf(c)) bar_arrive(base, kCount); else bar_sync(base, kCount); }
  template <class C> __device__ __forceinline__ void end_B(const C&) { bar_sync(base + 1, kCount); }
  template <class C> __device__ __forceinline__ void end_C(const C& c) { end_A(c); }
  template <class C> __device__ __forceinline__ void end_D(const C& c) {
    if (leaf(c) && c.ncon > 0) { bar_sync(base + 3, kCount); }
    else { bar_sync(base + 2, count_x); bar_arrive(base + 3, kCount); }
  }
};

// (Round-2 experiment "SyncHood" — one rendezvous barrier per parent node, kernel variants 10 / 11 — measured 1-10 % slower than
// SyncGroup and compute-sanitizer's synccheck flags its bar.sync pattern as divergent: removed rather than exempted.)
// SyncNamed: a point-to-point protocol along the tree edges on hardware named barriers (bar.arrive / bar.sync, ids 1..15):
// waiting warps sleep in the barrier unit instead of polling an mbarrier, so they do not steal
// issue slots from the working warps.  Each node WITH children owns two ids:
//   pose id : the node bar.arrive's, each child bar.sync's      (count = 32 * (1 + nchildren))
//   terms id: each child bar.arrive's, the node bar.sync's      (same count)
// Needs 2 * (#nodes with children) <= 15; otherwise the caller falls back to SyncCta.
struct SyncNamed {
  int my_pose_id, my_terms_id, my_count;       // valid when this link has children (else 0)
  int par_pose_id, par_terms_id, par_count;    // ids owned by the parent (0 when parent is the world / none)
  // No fence before the arrival: bar.arrive / bar.sync order the arriving thread's earlier shared-memory accesses before the
  // barrier completes for every participant (the PTX ISA's own producer / consumer example is st.shared; bar.arrive on one side,
  // bar.sync; ld.shared on the other).  Round 1 had a __threadfence_block() here = four MEMBAR.SC.CTA per warp and substep.
  static __device__ __forceinline__ void bar_arrive(int id, int count) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
  }
  static __device__ __forceinline__ void bar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
  }
  __device__ __forceinline__ void wait_pose(int parent) {
    if (parent >= 0) bar_sync(par_pose_id, par_count);
  }
  __device__ __forceinline__ void arrive_terms(int) {
    if (par_terms_id) bar_arrive(par_terms_id, par_count);
  }
  __device__ __forceinline__ void wait_terms(const int*) {
    if (my_terms_id) bar_sync(my_terms_id, my_count);
  }
  __device__ __forceinline__ void arrive_pose(int) {
    if (my_pose_id) bar_arrive(my_pose_id, my_count);
  }
  __device__ __forceinline__ void phase_end() {}
  template <class C> __device__ __forceinline__ void end_A(const C&) {}
  template <class C> __device__ __forceinline__ void end_B(const C&) {}
  template <class C> __device__ __forceinline__ void end_C(const C&) {}
  template <class C> __device__ __forceinline__ void end_D(const C&) {}
  // returns false when the tree needs more ids than the hardware has
  __device__ __forceinline__ bool setup(const ModelSmem& M, int l, int L) {
    int nparents = 0, my_idx = -1, par_idx = -1, my_nch = 0, par_nch = 0;
    const int parent = M.li(MBD_F_PARENT, l);
    const bool jointed = M.li(MBD_F_NDOF, l) > 0;
    for (int k = 0; k < L; ++k) {
      int nch = 0;
      for (int j = 0; j < MBD_MAXCHILD; ++j) nch += M.li(MBD_F_CHILD0 + j, k) >= 0;
      if (nch > 0) {
        if (k == l) { my_idx = nparents; my_nch = nch; }
        if (k == parent) { par_idx = nparents; par_nch = nch; }
        ++nparents;
      }
    }
    my_pose_id = my_idx >= 0 ? 1 + 2 * my_idx : 0;
    my_terms_id = my_idx >= 0 ? 2 + 2 * my_idx : 0;
    my_count = 32 * (1 + my_nch);
    const bool linked = jointed && par_idx >= 0;
    par_pose_id = linked ? 1 + 2 * par_idx : 0;
    par_terms_id = linked ? 2 + 2 * par_idx : 0;
    par_count = 32 * (1 + par_nch);
    return 2 * nparents <= 15;
  }
};

// One brax.positional.pipeline.step for (link = this warp, sample = this lane).
// All threads of the CTA must call.  DR: every contact's friction is fl(mu * f_mu) (the vector env's per-env model factor).
template <int CMAX, bool DR = false, class Sync>
__device__ __forceinline__ void positional_step_wpl(const ModelSmem& M, const WarpCfg& c, const WplSmem& S,
                                                    Sync& Y, LinkState& s, const float tau[MBD_MAXDOF], float f_mu = 1.0f) {
  const bool jointed = c.ndof > 0;
  const bool has_parent = c.parent >= 0;
  const v3 p_prev = s.p;
  const q4 q_prev = s.q;  // x_i_prev
  MBD_PH_BEGIN

  // ---- A: joints.acceleration_update ----------------------------------------------------------
  v3 T = V3(0.0f, 0.0f, 0.0f);
  v3 Fa = V3(0.0f, 0.0f, 0.0f);   // linear acceleration from slide-dof forces (links with slide dofs only)
  Y.wait_pose(jointed ? c.parent : -1);
  if (jointed && c.smask != 0) {
    // links with slide dofs (planar roots, the cartpole cart; parent = world): oracle/mbd_oracle.c, "slide dofs"
    q4 a_p = qmul(Q4(1.0f, 0.0f, 0.0f, 0.0f), M.l4(MBD_F_PQ, c.l));
    q4 a_c = qmul(s.q, M.l4(MBD_F_JQ, c.l));
    q4 j = qmul(qconj(a_p), a_c);
    v3 jd = vinv_rotate(vsub(s.w, V3(0.0f, 0.0f, 0.0f)), a_p);
    v3 tq = vscale(jd, -M.lf(MBD_F_ANG_DAMP, c.l));
    JointAngles ja;
    axis_angle_ang(j, M.lf(MBD_F_PARITY, c.l), ja);
    v3 rcw = vrotate(M.l3(MBD_F_RC, c.l), s.q);
    v3 d = vsub(vadd(s.p, rcw), M.l3(MBD_F_RP, c.l));
    v3 va = vadd(s.v, vcross(s.w, rcw));
    v3 Fw = V3(0.0f, 0.0f, 0.0f);
#pragma unroll
    for (int k = 0; k < MBD_MAXDOF; ++k) {
      if (k < c.ndof) {
        int base = MBD_F_DOF0 + k * MBD_DOF_STRIDE;
        if ((c.smask >> k) & 1) {
          v3 ak = slide_axis(k, M.lf(MBD_F_PARITY, c.l), a_p);
          float x = vdot(d, ak), xd = vdot(va, ak);
          float f = fmaf(-M.lf(base + MBD_D_DAMP, c.l), xd, fmaf(-M.lf(base + MBD_D_STIFF, c.l), x, tau[k]));
          Fw = vfma(ak, f, Fw);
        } else {
          float vel = vdot(ja.ax[k], jd);
          float t = fmaf(-M.lf(base + MBD_D_DAMP, c.l), vel, fmaf(-M.lf(base + MBD_D_STIFF, c.l), ja.ang[k], tau[k]));
          tq = vfma(ja.ax[k], t, tq);
        }
      }
    }
    T = vrotate(tq, a_p);
    Fa = vscale(Fw, M.lf(MBD_F_INV_MASS, c.l));
    T = vadd(T, vcross(rcw, Fw));
    S.put_e3(c.l, 0, T);
  } else if (jointed) {
    q4 qp = Q4(1.0f, 0.0f, 0.0f, 0.0f);
    v3 wp = V3(0.0f, 0.0f, 0.0f);
    if (has_parent) { qp = S.xq(c.parent); wp = S.xw(c.parent); }
    q4 a_p = qmul(qp, M.l4(MBD_F_PQ, c.l));
    q4 a_c = qmul(s.q, M.l4(MBD_F_JQ, c.l));
    q4 j = qmul(qconj(a_p), a_c);
    v3 jd = vinv_rotate(vsub(s.w, wp), a_p);
    v3 tq = vscale(jd, -M.lf(MBD_F_ANG_DAMP, c.l));
    if (c.ndof == 1) {
      float psi, r10, r20;
      axis_angle_1dof(j, psi, r10, r20);
      float vel = vdot(V3(1.0f, 0.0f, 0.0f), jd);
      float t = fmaf(-M.lf(MBD_F_DOF0 + MBD_D_DAMP, c.l), vel, fmaf(-M.lf(MBD_F_DOF0 + MBD_D_STIFF, c.l), psi, tau[0]));
      tq = vfma(V3(1.0f, 0.0f, 0.0f), t, tq);
    } else {
      JointAngles ja;
      axis_angle_ang(j, M.lf(MBD_F_PARITY, c.l), ja);
#pragma unroll
      for (int k = 0; k < MBD_MAXDOF; ++k) {
        if (k < c.ndof) {
          int base = MBD_F_DOF0 + k * MBD_DOF_STRIDE;
          float vel = vdot(ja.ax[k], jd);
          float t = fmaf(-M.lf(base + MBD_D_DAMP, c.l), vel, fmaf(-M.lf(base + MBD_D_STIFF, c.l), ja.ang[k], tau[k]));
          tq = vfma(ja.ax[k], t, tq);
        }
      }
    }
    T = vrotate(tq, a_p);
    S.put_e3(c.l, 0, T);
  }
  MBD_PH(0)
  Y.arrive_terms(c.l);
  Y.end_A(c);
  MBD_PH(1)
  // ---- B: gather reaction torques, integrator.integrate_xdd, publish pose ---------------------------
  Y.wait_terms(c.child);
  {
    v3 acc = T;
#pragma unroll
    for (int k = 0; k < MBD_MAXCHILD; ++k)
      if (c.child[k] >= 0) acc = vsub(acc, S.e3(c.child[k], 0));
    s.w = V3(fmaf(acc.x, M.hf(MBD_H_DT), s.w.x * M.hf(MBD_H_ANG_DAMP)), fmaf(acc.y, M.hf(MBD_H_DT), s.w.y * M.hf(MBD_H_ANG_DAMP)), fmaf(acc.z, M.hf(MBD_H_DT), s.w.z * M.hf(MBD_H_ANG_DAMP)));
    v3 al = V3(M.hf(MBD_H_GX), M.hf(MBD_H_GY), M.hf(MBD_H_GZ));
    if (c.smask != 0) al = vadd(al, Fa);   // warp-uniform; g + 0 == g bit for bit, so the oracle adds unconditionally
    s.v = V3(fmaf(al.x, M.hf(MBD_H_DT), s.v.x * M.hf(MBD_H_VEL_DAMP)), fmaf(al.y, M.hf(MBD_H_DT), s.v.y * M.hf(MBD_H_VEL_DAMP)), fmaf(al.z, M.hf(MBD_H_DT), s.v.z * M.hf(MBD_H_VEL_DAMP)));
    s.q = qnormalize(qadd(s.q, vqmul(vscale(s.w, M.hf(MBD_H_HALF_DT)), s.q)));
    s.p = vfma(s.v, M.hf(MBD_H_DT), s.p);
    S.put_p(c.l, s.p);
    S.put_q(c.l, s.q);
  }
  MBD_PH(2)
  Y.arrive_pose(c.l);
  const v3 w_before = s.w, v_before = s.v;
  Y.end_B(c);
  MBD_PH(3)
  // ---- C: joints.position_update ---------------------------------------------------------------------
  v3 dpc = V3(0.0f, 0.0f, 0.0f);
  q4 dqc = Q4(0.0f, 0.0f, 0.0f, 0.0f);
  Y.wait_pose(jointed ? c.parent : -1);
  if (jointed) {
    v3 pp = V3(0.0f, 0.0f, 0.0f);
    q4 qp = Q4(1.0f, 0.0f, 0.0f, 0.0f);
    if (has_parent) { pp = S.xp(c.parent); qp = S.xq(c.parent); }
    const float im_c = M.lf(MBD_F_INV_MASS, c.l), im_p = M.lf(MBD_F_PINV_MASS, c.l), ii_p = M.lf(MBD_F_PINV_INERTIA, c.l);
    v3 rpw = vrotate(M.l3(MBD_F_RP, c.l), qp);
    v3 rcw = vrotate(M.l3(MBD_F_RC, c.l), s.q);
    v3 e = vsub(vadd(s.p, rcw), vadd(pp, rpw));
    q4 a_p = qmul(qp, M.l4(MBD_F_PQ, c.l));
    if (c.smask != 0) {   // prismatic dofs: what the limits allow along each slide axis is not an error
#pragma unroll
      for (int k = 0; k < MBD_MAXDOF; ++k)
        if (k < c.ndof && ((c.smask >> k) & 1)) {
          int base = MBD_F_DOF0 + k * MBD_DOF_STRIDE;
          v3 ak = slide_axis(k, M.lf(MBD_F_PARITY, c.l), a_p);
          float x = vdot(e, ak);
          e = vfma(ak, -clampf(x, M.lf(base + MBD_D_LO, c.l), M.lf(base + MBD_D_HI, c.l)), e);
        }
    }
    float cn;
    v3 n = vnormalize(e, &cn);
    v3 crc = vcross(rcw, n), crp = vcross(rpw, n);
    float w_c = im_c + vdot(crc, crc);
    float w_p = fmaf(ii_p, vdot(crp, crp), im_p);
    float dl = MBD_DIV(-cn, w_p + w_c + 1e-6f);
    v3 P = vscale(n, dl);
    v3 dp_c = vscale(P, im_c);
    // the exact factors 0.5 (and ii_p in {0,1}) are folded into the scale constants below: (x*0.5)*s == x*(0.5*s) bit for bit
    q4 dq_c = vqmul(vcross(rcw, P), s.q);
    v3 dp_p = vscale(P, -im_p);
    q4 dq_p = vqmul(vcross(rpw, P), qp);
    q4 a_c = qmul(s.q, M.l4(MBD_F_JQ, c.l));
    q4 j = qmul(qconj(a_p), a_c);
    v3 dqj;
    const int b0 = MBD_F_DOF0, b1 = MBD_F_DOF0 + MBD_DOF_STRIDE, b2 = MBD_F_DOF0 + 2 * MBD_DOF_STRIDE;
    if (c.ndof == 1) {
      float psi, r10, r20;
      axis_angle_1dof(j, psi, r10, r20);
      float e0 = (c.smask & 1) ? psi : psi - clampf(psi, M.lf(b0 + MBD_D_LO, c.l), M.lf(b0 + MBD_D_HI, c.l));
      dqj = V3(e0, -r20, r10);
    } else {
      JointAngles ja;
      axis_angle_ang(j, M.lf(MBD_F_PARITY, c.l), ja);
      float e0 = (c.smask & 1) ? ja.ang[0] : ja.ang[0] - clampf(ja.ang[0], M.lf(b0 + MBD_D_LO, c.l), M.lf(b0 + MBD_D_HI, c.l));
      float e1 = (c.smask & 2) ? ja.ang[1] : ja.ang[1] - clampf(ja.ang[1], M.lf(b1 + MBD_D_LO, c.l), M.lf(b1 + MBD_D_HI, c.l));
      float e2 = (c.smask & 4) ? ja.ang[2] : ja.ang[2] - clampf(ja.ang[2], M.lf(b2 + MBD_D_LO, c.l), M.lf(b2 + MBD_D_HI, c.l));
      dqj = vscale(ja.ax[0], e0);
      dqj = vfma(ja.ax[1], e1, dqj);
      dqj = vfma(ja.ax[2], e2, dqj);
    }
    v3 dq = vrotate(dqj, a_p);
    float th;
    v3 na = vnormalize(dq, &th);
    float nn = vdot(na, na);
    float dla = MBD_DIV(-th, fmaf(ii_p, nn, nn) + 1e-6f);
    v3 Pa = vscale(na, dla);
    q4 dqa_c = vqmul(Pa, s.q);
    q4 dqa_p = vqmul(Pa, qp);
    const float hsp = 0.5f * M.hf(MBD_H_SCALE_POS), hsa = 0.5f * M.hf(MBD_H_SCALE_ANG);
    dpc = vscale(dp_c, M.hf(MBD_H_SCALE_POS));
    dqc = qadd(qscale(dq_c, hsp), qscale(dqa_c, hsa));
    S.put_e3(c.l, 0, vscale(dp_p, M.hf(MBD_H_SCALE_POS)));
    S.put_e4(c.l, 3, qadd(qscale(dq_p, -hsp * ii_p), qscale(dqa_p, -hsa * ii_p)));
  }
  MBD_PH(4)
  Y.arrive_terms(c.l);
  Y.end_C(c);
  MBD_PH(5)
  // ---- D: gather child deltas, apply; contacts; project_xd; contact velocities; publish q,w ----------
  Y.wait_terms(c.child);
  {
    v3 dp = dpc;
    q4 dq = dqc;
#pragma unroll
    for (int k = 0; k < MBD_MAXCHILD; ++k) {
      if (c.child[k] >= 0) { dp = vadd(dp, S.e3(c.child[k], 0)); dq = qadd(dq, S.e4(c.child[k], 3)); }
    }
    s.p = vadd(s.p, dp);
    s.q = qnormalize(qadd(s.q, dq));
  }
  float dlam[CMAX];
  v3 cpos[CMAX];
  if (c.ncon > 0) {
    v3 dp = V3(0.0f, 0.0f, 0.0f);
    q4 dq = Q4(0.0f, 0.0f, 0.0f, 0.0f);
    const v3 p0 = s.p;
    const q4 q0 = s.q;
#pragma unroll
    for (int ci = 0; ci < CMAX; ++ci) {
      dlam[ci] = 0.0f; cpos[ci] = V3(0.0f, 0.0f, 0.0f);
      if (ci < c.ncon) {
        const float mu = DR ? M.lf(MBD_F_CON0 + ci * MBD_CON_STRIDE + 4, c.l) * f_mu : 0.0f;
        contact_position_plane<DR>(M, c.l, ci, M.lf(MBD_F_INV_MASS, c.l), p0, q0, p_prev, q_prev, dp, dq, dlam[ci], cpos[ci], mu);
      }
    }
    s.p = vfma(dp, M.hf(MBD_H_COLLIDE_SCALE), s.p);
    s.q = qnormalize(qadd(s.q, qscale(dq, 0.5f * M.hf(MBD_H_COLLIDE_SCALE))));
  }
  {
    s.v = vscale(vsub(s.p, p_prev), M.hf(MBD_H_INV_DT));
    q4 dq = qmul(s.q, qconj(q_prev));
    float sc = dq.w >= 0.0f ? M.hf(MBD_H_TWO_INV_DT) : -M.hf(MBD_H_TWO_INV_DT);
    s.w = V3(dq.x * sc, dq.y * sc, dq.z * sc);
  }
  if (c.ncon > 0) {
    v3 dv = V3(0.0f, 0.0f, 0.0f), dw = V3(0.0f, 0.0f, 0.0f);
    const v3 v0 = s.v, w0 = s.w;
#pragma unroll
    for (int ci = 0; ci < CMAX; ++ci)
      if (ci < c.ncon) {
        const float mu = DR ? M.lf(MBD_F_CON0 + ci * MBD_CON_STRIDE + 4, c.l) * f_mu : 0.0f;
        contact_velocity_plane<DR>(M, c.l, ci, M.lf(MBD_F_INV_MASS, c.l), M.hf(MBD_H_INV_DT), M.hf(MBD_H_ELASTICITY), s.p, v0, w0,
                                   v_before, w_before, cpos[ci], dlam[ci], dv, dw, mu);
      }
    s.v = vadd(s.v, dv);
    s.w = vadd(s.w, dw);
  }
  S.put_q(c.l, s.q);
  S.put_w(c.l, s.w);
  MBD_PH(6)
  Y.arrive_pose(c.l);
  Y.end_D(c);
  MBD_PH(7)
}

__device__ __forceinline__ v3 link_origin_w(const ModelSmem& M, int l, const LinkState& s) {
  return vsub(s.p, vrotate(M.l3(MBD_F_COM, l), s.q));
}
__device__ __forceinline__ v3 link_origin_vel_w(const ModelSmem& M, int l, const LinkState& s) {
  v3 rc = vrotate(M.l3(MBD_F_COM, l), s.q);
  return vadd(s.v, vcross(rc, s.w));
}

}  // namespace mbd
