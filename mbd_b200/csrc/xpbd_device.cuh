// xpbd_device.cuh — the Brax-positional (XPBD) physics step on sm_90a, one LINK per LANE.
//
// Mapping: a sample group is LPS (=16) consecutive lanes of a warp; lane l of the group owns
// link l (its COM-frame state x_i, xd_i lives in registers) and the joint that ties link l to
// its parent.  XPBD is Jacobi-parallel over joints, so the only cross-lane traffic is
//   * a parent-state fetch   (__shfl_sync from the parent's lane), and
//   * a child->parent gather (each lane pulls the reaction terms of its <=4 children),
// both inside the warp.  Model constants sit in shared memory as a field-major table
// (include/mbd_model.h) staged by one TMA bulk copy per CTA.
//
// Arithmetic contract: every expression below mirrors oracle/mbd_oracle.c operation for
// operation (same association, fmaf exactly where the oracle has fmaf; the file is compiled
// with -fmad=false so nothing else contracts).  tests/test_rollout_gpu.py asserts BIT-EXACT
// agreement of per-sample returns and final states.
//
// Reference path restated: brax.positional.pipeline.step as called from
// upstream mbd/envs/humanoidrun.py:36 (Brax itself is un-vendored: see DESIGN.md).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "mbd_fp32.h"
#include "mbd_model.h"

namespace mbd {

struct v3 { float x, y, z; };
struct q4 { float w, x, y, z; };

__device__ __forceinline__ v3 V3(float x, float y, float z) { v3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ q4 Q4(float w, float x, float y, float z) { q4 r; r.w = w; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ v3 vadd(v3 a, v3 b) { return V3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ v3 vsub(v3 a, v3 b) { return V3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ v3 vscale(v3 a, float s) { return V3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ v3 vfma(v3 b, float s, v3 a) { return V3(fmaf(b.x, s, a.x), fmaf(b.y, s, a.y), fmaf(b.z, s, a.z)); }
__device__ __forceinline__ float vdot(v3 a, v3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
__device__ __forceinline__ v3 vcross(v3 a, v3 b) {
  return V3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x)));
}
__device__ __forceinline__ v3 vnormalize(v3 a, float* norm) {
  float n = MBD_SQRT(vdot(a, a));
  float inv = (n == 0.0f) ? 0.0f : MBD_RCP(n);
  *norm = n;
  return vscale(a, inv);
}
__device__ __forceinline__ q4 qconj(q4 q) { return Q4(q.w, -q.x, -q.y, -q.z); }
__device__ __forceinline__ q4 qmul(q4 u, q4 v) {
  return Q4(fmaf(-u.z, v.z, fmaf(-u.y, v.y, fmaf(-u.x, v.x, u.w * v.w))),
            fmaf(-u.z, v.y, fmaf(u.y, v.z, fmaf(u.x, v.w, u.w * v.x))),
            fmaf(u.z, v.x, fmaf(u.y, v.w, fmaf(-u.x, v.z, u.w * v.y))),
            fmaf(u.z, v.w, fmaf(-u.y, v.x, fmaf(u.x, v.y, u.w * v.z))));
}
__device__ __forceinline__ q4 vqmul(v3 a, q4 q) {
  return Q4(fmaf(-a.z, q.z, fmaf(-a.y, q.y, -(a.x * q.x))),
            fmaf(-a.z, q.y, fmaf(a.y, q.z, a.x * q.w)),
            fmaf(a.z, q.x, fmaf(a.y, q.w, -(a.x * q.z))),
            fmaf(a.z, q.w, fmaf(-a.y, q.x, a.x * q.y)));
}
// Oracle form: t = 2(u x v); c = u x t; r = fma(w, t, v) + c.  Scaling by 2 is exact, so with t' = u x v and
// c' = u x t' (both exactly half of t, c):  fma(w, t, v) = fma(2w, t', v)  and  (.) + c = fma(2, c', (.))  — the same
// two roundings on the same real values, two instructions fewer.  Bit-identical to oracle/mbd_oracle.c::vrotate.
__device__ __forceinline__ v3 vrotate(v3 v, q4 q) {
  v3 u = V3(q.x, q.y, q.z);
  v3 t = vcross(u, v);
  v3 c = vcross(u, t);
  float w2 = q.w + q.w;
  return V3(fmaf(2.0f, c.x, fmaf(w2, t.x, v.x)), fmaf(2.0f, c.y, fmaf(w2, t.y, v.y)), fmaf(2.0f, c.z, fmaf(w2, t.z, v.z)));
}
__device__ __forceinline__ v3 vinv_rotate(v3 v, q4 q) { return vrotate(v, qconj(q)); }
__device__ __forceinline__ q4 qnormalize(q4 q) {
  float n = MBD_SQRT(fmaf(q.z, q.z, fmaf(q.y, q.y, fmaf(q.x, q.x, q.w * q.w))));
  float inv = MBD_RCP(n);
  return Q4(q.w * inv, q.x * inv, q.y * inv, q.z * inv);
}
__device__ __forceinline__ q4 qadd(q4 a, q4 b) { return Q4(a.w + b.w, a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ q4 qscale(q4 a, float s) { return Q4(a.w * s, a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

__device__ __forceinline__ v3 shfl3(v3 a, int src) {
  return V3(__shfl_sync(0xffffffffu, a.x, src), __shfl_sync(0xffffffffu, a.y, src), __shfl_sync(0xffffffffu, a.z, src));
}
__device__ __forceinline__ q4 shfl4(q4 a, int src) {
  return Q4(__shfl_sync(0xffffffffu, a.w, src), __shfl_sync(0xffffffffu, a.x, src), __shfl_sync(0xffffffffu, a.y, src),
            __shfl_sync(0xffffffffu, a.z, src));
}

// ---- shared-memory model table access ------------------------------------------------------
struct ModelSmem {
  const float* f;  // the blob in shared memory
  __device__ __forceinline__ float hf(int w) const { return f[w]; }
  __device__ __forceinline__ int hi(int w) const { return __float_as_int(f[w]); }
  __device__ __forceinline__ float lf(int field, int l) const { return f[MBD_HDR_WORDS + field * MBD_MAXL + l]; }
  __device__ __forceinline__ int li(int field, int l) const { return __float_as_int(lf(field, l)); }
  __device__ __forceinline__ v3 l3(int field, int l) const { return V3(lf(field, l), lf(field + 1, l), lf(field + 2, l)); }
  __device__ __forceinline__ q4 l4(int field, int l) const { return Q4(lf(field, l), lf(field + 1, l), lf(field + 2, l), lf(field + 3, l)); }
};

struct LinkState { v3 p; q4 q; v3 w; v3 v; };  // x_i.pos, x_i.rot, xd_i.ang, xd_i.vel

// ---- contact.get (MJX plane_sphere) + collisions.resolve_position / resolve_velocity ----------------
// Specialised for the ground-plane normal n = +z (the only contact class of the positional envs in scope):
//   r x n = (r.y, -r.x, 0);   P = dl*n = (0,0,dl);   r x P = (r.y dl, -r.x dl, 0);
//   tangential vectors have z = 0.  Same formulas as the general XPBD contact with n substituted —
// the oracle (oracle/mbd_oracle.c::contact_position_plane / contact_velocity_plane) uses the identical
// expressions.  vqmul_xy is vqmul with a.z = 0.
__device__ __forceinline__ q4 vqmul_xy(float ax, float ay, q4 q) {
  return Q4(fmaf(-ay, q.y, -(ax * q.x)), fmaf(ay, q.z, ax * q.w), fmaf(ay, q.w, -(ax * q.z)), fmaf(-ay, q.x, ax * q.y));
}

// one sphere-plane contact of link l: accumulates the position-level correction (dp, dq); returns dlambda and
// the contact point for the velocity pass.  DR (the vector env's per-env model): the friction is mu_dr, the caller's product
// fl(mu * f_mu) of the blob word and the env's friction factor, in the place of the blob word.
template <bool DR = false>
__device__ __forceinline__ void contact_position_plane(const ModelSmem& M, int l, int ci, float im, v3 p, q4 q, v3 p_prev, q4 q_prev,
                                                       v3& dp, q4& dq, float& dl_out, v3& cp_out, float mu_dr = 0.0f) {
  const int base = MBD_F_CON0 + ci * MBD_CON_STRIDE;
  const float radius = M.lf(base + 3, l), mu = DR ? mu_dr : M.lf(base + 4, l);
  v3 centre = vadd(p, vrotate(M.l3(base, l), q));
  float dist = centre.z - radius;
  v3 cp = V3(centre.x, centre.y, centre.z - (radius + 0.5f * dist));  // pos = c - n (r + dist/2)
  bool coll = dist < 0.0f;
  v3 r = vsub(cp, p);
  float w = im + fmaf(r.x, r.x, r.y * r.y);
  float dl = coll ? MBD_DIV(-dist, w + 1e-6f) : 0.0f;
  dp.z = dp.z + dl * im;
  dq = qadd(dq, vqmul_xy(r.y * dl, -(r.x * dl), q));  // the factor 0.5 is applied once by the caller (exact scaling)
  // static friction: cancel the tangential travel of the contact point since x_i_prev
  v3 rl = vinv_rotate(r, q);
  v3 pbar = vadd(p_prev, vrotate(rl, q_prev));
  float dx = cp.x - pbar.x, dy = cp.y - pbar.y;
  float ct = MBD_SQRT(fmaf(dy, dy, dx * dx));
  float inv = (ct == 0.0f) ? 0.0f : MBD_RCP(ct);
  float ntx = dx * inv, nty = dy * inv;
  float c1 = -(r.z * nty), c2 = r.z * ntx, c3 = fmaf(r.x, nty, -(r.y * ntx));
  float wt = im + fmaf(c3, c3, fmaf(c2, c2, c1 * c1));
  float dlt = MBD_DIV(-ct, wt + 1e-6f);
  bool stat = coll && (fabsf(dlt) < mu * fabsf(dl));
  float m = stat ? dlt : 0.0f;
  float ptx = ntx * m, pty = nty * m;
  dp.x = dp.x + ptx * im;
  dp.y = dp.y + pty * im;
  dq = qadd(dq, vqmul(V3(-(r.z * pty), r.z * ptx, fmaf(r.x, pty, -(r.y * ptx))), q));
  dl_out = dl;
  cp_out = cp;
}

template <bool DR = false>
__device__ __forceinline__ void contact_velocity_plane(const ModelSmem& M, int l, int ci, float im, float inv_dt, float elasticity, v3 p,
                                                       v3 v, v3 w, v3 v_before, v3 w_before, v3 cp, float dl, v3& dv, v3& dw,
                                                       float mu_dr = 0.0f) {
  const float mu = DR ? mu_dr : M.lf(MBD_F_CON0 + ci * MBD_CON_STRIDE + 4, l);
  v3 r = vsub(cp, p);
  v3 rel = vadd(v, vcross(w, r));
  float vn = rel.z;
  float vtn = MBD_SQRT(fmaf(rel.y, rel.y, rel.x * rel.x));
  float inv = (vtn == 0.0f) ? 0.0f : MBD_RCP(vtn);
  float tdx = rel.x * inv, tdy = rel.y * inv;
  float fr = mu * fabsf(dl) * inv_dt;
  float mag = fr < vtn ? fr : vtn;
  float c1 = -(r.z * tdy), c2 = r.z * tdx, c3 = fmaf(r.x, tdy, -(r.y * tdx));
  float wd = im + fmaf(c3, c3, fmaf(c2, c2, c1 * c1));
  float kd = MBD_RCP(wd + 1e-6f);
  float pdx = (tdx * -mag) * kd, pdy = (tdy * -mag) * kd;
  v3 rel_old = vadd(v_before, vcross(w_before, r));
  float vn_old = rel_old.z;
  float rest = -elasticity * vn_old;
  rest = rest < 0.0f ? rest : 0.0f;
  float wn = im + fmaf(r.x, r.x, r.y * r.y);
  float prz = (-vn + rest) * (MBD_RCP(wn + 1e-6f));
  v3 P = V3(pdx, pdy, (vn_old <= 0.0f) ? prz : 0.0f);
  if (dl == 0.0f) P = V3(0.0f, 0.0f, 0.0f);
  dv = vadd(dv, vscale(P, im));
  dw = vadd(dw, vcross(r, P));
}


struct JointAngles { float ang[3]; v3 ax[3]; float r10, r20; };

// kinematics.axis_angle_ang restated — see oracle/mbd_oracle.c::axis_angle_ang
__device__ __forceinline__ void axis_angle_ang(q4 j, float parity, JointAngles& o) {
  float w = j.w, x = j.x, y = j.y, z = j.z;
  float r00 = 1.0f - 2.0f * fmaf(z, z, y * y);
  float r01 = 2.0f * fmaf(x, y, -(w * z));
  float r02 = 2.0f * fmaf(x, z, w * y);
  float r12 = 2.0f * fmaf(y, z, -(w * x));
  float r22 = 1.0f - 2.0f * fmaf(y, y, x * x);
  o.r10 = 2.0f * fmaf(x, y, w * z);
  o.r20 = 2.0f * fmaf(x, z, -(w * y));
  float psi = mbd_atan2f(-r12, r22);
  float cth = MBD_SQRT(fmaf(r01, r01, r00 * r00));
  float theta = mbd_atan2f(r02, cth);
  float phi = mbd_atan2f(-r01, r00);
  float ln;
  v3 lon = vnormalize(V3(0.0f, r22, -r12), &ln);
  o.ang[0] = psi; o.ang[1] = theta; o.ang[2] = parity * phi;
  o.ax[0] = V3(1.0f, 0.0f, 0.0f);
  o.ax[1] = lon;
  o.ax[2] = V3(parity * r02, parity * r12, parity * r22);
}

// slide (prismatic) dof axis k of a link in world coordinates — oracle/mbd_oracle.c::slide_axis
__device__ __forceinline__ v3 slide_axis(int k, float parity, q4 a_p) {
  v3 e = k == 0 ? V3(1.0f, 0.0f, 0.0f) : (k == 1 ? V3(0.0f, 1.0f, 0.0f) : V3(0.0f, 0.0f, parity));
  return vrotate(e, a_p);
}

// Per-lane constants that stay in registers for the whole rollout.
struct LaneCfg {
  int l;         // link id (lane within the group)
  int gbase;     // first lane of this sample group inside the warp
  int ndof;      // -1 unused lane, 0 free root, 1..3
  int psrc;      // warp lane of the parent (own lane when parent is the world)
  int has_parent;
  int csrc[MBD_MAXCHILD];  // warp lanes of the children, -1 = none
  int ncon, smask;
  float inv_mass, pinv_mass, pinv_inertia, parity, ang_damp;
  q4 pq, jq;
  v3 rp, rc;
};

__device__ __forceinline__ void load_lane_cfg(const ModelSmem& M, int lane_in_warp, int lps, LaneCfg& c) {
  c.l = lane_in_warp % lps;
  c.gbase = lane_in_warp - c.l;
  int L = M.hi(MBD_H_NLINK);
  bool live = c.l < L && c.l < MBD_MAXL;
  int l = live ? c.l : 0;
  c.ndof = live ? M.li(MBD_F_NDOF, l) : -1;
  int par = live ? M.li(MBD_F_PARENT, l) : -1;
  c.has_parent = par >= 0;
  c.psrc = c.gbase + (par >= 0 ? par : c.l);
#pragma unroll
  for (int k = 0; k < MBD_MAXCHILD; ++k) {
    int ch = live ? M.li(MBD_F_CHILD0 + k, l) : -1;
    c.csrc[k] = ch >= 0 ? c.gbase + ch : -1;
  }
  c.ncon = live ? M.li(MBD_F_NCON, l) : 0;
  c.smask = (live && c.ndof > 0) ? M.li(MBD_F_SLIDE, l) : 0;
  c.inv_mass = M.lf(MBD_F_INV_MASS, l);
  c.pinv_mass = M.lf(MBD_F_PINV_MASS, l);
  c.pinv_inertia = M.lf(MBD_F_PINV_INERTIA, l);
  c.parity = M.lf(MBD_F_PARITY, l);
  c.ang_damp = M.lf(MBD_F_ANG_DAMP, l);
  c.pq = M.l4(MBD_F_PQ, l);
  c.jq = M.l4(MBD_F_JQ, l);
  c.rp = M.l3(MBD_F_RP, l);
  c.rc = M.l3(MBD_F_RC, l);
}

struct StepConsts { float dt, inv_dt, half_dt, two_inv_dt, vel_damp, ang_damp, scale_pos, scale_ang, collide_scale, elasticity; v3 g; };

__device__ __forceinline__ void load_step_consts(const ModelSmem& M, StepConsts& k) {
  k.dt = M.hf(MBD_H_DT); k.inv_dt = M.hf(MBD_H_INV_DT); k.half_dt = M.hf(MBD_H_HALF_DT); k.two_inv_dt = M.hf(MBD_H_TWO_INV_DT);
  k.vel_damp = M.hf(MBD_H_VEL_DAMP); k.ang_damp = M.hf(MBD_H_ANG_DAMP);
  k.scale_pos = M.hf(MBD_H_SCALE_POS); k.scale_ang = M.hf(MBD_H_SCALE_ANG);
  k.collide_scale = M.hf(MBD_H_COLLIDE_SCALE); k.elasticity = M.hf(MBD_H_ELASTICITY);
  k.g = V3(M.hf(MBD_H_GX), M.hf(MBD_H_GY), M.hf(MBD_H_GZ));
}

// One brax.positional.pipeline.step for the link owned by this lane.  tau[k] = gear*clip(act) of
// the lane's dof k (actuator.to_tau), already resolved by the caller.  All 32 lanes must call.
// DR: every contact's friction is fl(mu * f_mu) (the vector env's per-env model factor).
template <int CMAX, bool DR = false>
__device__ __forceinline__ void positional_step(const ModelSmem& M, const LaneCfg& c, const StepConsts& K,
                                                LinkState& s, const float tau[MBD_MAXDOF], float f_mu = 1.0f) {
  const bool jointed = c.ndof > 0;
  const LinkState prev = s;  // x_i_prev

  // ---- parent state (world = identity / zero) ----------------------------------------------
  q4 qp = shfl4(s.q, c.psrc);
  v3 wp = shfl3(s.w, c.psrc);
  if (!c.has_parent) { qp = Q4(1.0f, 0.0f, 0.0f, 0.0f); wp = V3(0.0f, 0.0f, 0.0f); }

  // ---- joints.acceleration_update ----------------------------------------------------------
  v3 T = V3(0.0f, 0.0f, 0.0f);
  v3 Fa = V3(0.0f, 0.0f, 0.0f);   // linear acceleration from slide-dof forces
  if (jointed) {
    q4 a_p = qmul(qp, c.pq);
    q4 a_c = qmul(s.q, c.jq);
    q4 j = qmul(qconj(a_p), a_c);
    v3 jd = vinv_rotate(vsub(s.w, wp), a_p);
    JointAngles ja;
    axis_angle_ang(j, c.parity, ja);
    v3 tq = vscale(jd, -c.ang_damp);
    v3 rcw_s = V3(0.0f, 0.0f, 0.0f), d_s = rcw_s, va_s = rcw_s, Fw = rcw_s;
    if (c.smask != 0) {
      rcw_s = vrotate(c.rc, s.q);
      d_s = vsub(vadd(s.p, rcw_s), c.rp);
      va_s = vadd(s.v, vcross(s.w, rcw_s));
    }
#pragma unroll
    for (int k = 0; k < MBD_MAXDOF; ++k) {
      if (k < c.ndof) {
        int base = MBD_F_DOF0 + k * MBD_DOF_STRIDE;
        if ((c.smask >> k) & 1) {
          v3 ak = slide_axis(k, c.parity, a_p);
          float x = vdot(d_s, ak), xd = vdot(va_s, ak);
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
    if (c.smask != 0) {
      Fa = vscale(Fw, c.inv_mass);
      T = vadd(T, vcross(rcw_s, Fw));
    }
  }
  // gather: acc = T_own - sum_children T_child (ascending child order)
  v3 acc = T;
#pragma unroll
  for (int k = 0; k < MBD_MAXCHILD; ++k) {
    int src = c.csrc[k];
    v3 tc = shfl3(T, src >= 0 ? src : 0);
    if (src >= 0) acc = vsub(acc, tc);
  }
  // ---- integrator.integrate_xdd ---------------------------------------------------------------
  s.w = V3(fmaf(acc.x, K.dt, s.w.x * K.ang_damp), fmaf(acc.y, K.dt, s.w.y * K.ang_damp), fmaf(acc.z, K.dt, s.w.z * K.ang_damp));
  const v3 al = vadd(K.g, Fa);   // g + 0 == g bit for bit on links without slide dofs
  s.v = V3(fmaf(al.x, K.dt, s.v.x * K.vel_damp), fmaf(al.y, K.dt, s.v.y * K.vel_damp), fmaf(al.z, K.dt, s.v.z * K.vel_damp));
  s.q = qnormalize(qadd(s.q, vqmul(vscale(s.w, K.half_dt), s.q)));
  s.p = vfma(s.v, K.dt, s.p);
  const v3 w_before = s.w, v_before = s.v;  // xd_i right after integration

  // ---- joints.position_update -------------------------------------------------------------------
  v3 pp = shfl3(s.p, c.psrc);
  qp = shfl4(s.q, c.psrc);
  if (!c.has_parent) { pp = V3(0.0f, 0.0f, 0.0f); qp = Q4(1.0f, 0.0f, 0.0f, 0.0f); }
  v3 dpc = V3(0.0f, 0.0f, 0.0f), dpp = V3(0.0f, 0.0f, 0.0f);
  q4 dqc = Q4(0.0f, 0.0f, 0.0f, 0.0f), dqp = Q4(0.0f, 0.0f, 0.0f, 0.0f);
  if (jointed) {
    const float im_c = c.inv_mass, im_p = c.pinv_mass, ii_p = c.pinv_inertia;
    v3 rpw = vrotate(c.rp, qp);
    v3 rcw = vrotate(c.rc, s.q);
    v3 e = vsub(vadd(s.p, rcw), vadd(pp, rpw));
    q4 a_p = qmul(qp, c.pq);
    if (c.smask != 0) {
#pragma unroll
      for (int k = 0; k < MBD_MAXDOF; ++k)
        if (k < c.ndof && ((c.smask >> k) & 1)) {
          int base = MBD_F_DOF0 + k * MBD_DOF_STRIDE;
          v3 ak = slide_axis(k, c.parity, a_p);
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
    q4 a_c = qmul(s.q, c.jq);
    q4 j = qmul(qconj(a_p), a_c);
    JointAngles ja;
    axis_angle_ang(j, c.parity, ja);
    const int b0 = MBD_F_DOF0, b1 = MBD_F_DOF0 + MBD_DOF_STRIDE, b2 = MBD_F_DOF0 + 2 * MBD_DOF_STRIDE;
    float e0 = (c.smask & 1) ? ja.ang[0] : ja.ang[0] - clampf(ja.ang[0], M.lf(b0 + MBD_D_LO, c.l), M.lf(b0 + MBD_D_HI, c.l));
    float e1 = (c.smask & 2) ? ja.ang[1] : ja.ang[1] - clampf(ja.ang[1], M.lf(b1 + MBD_D_LO, c.l), M.lf(b1 + MBD_D_HI, c.l));
    float e2 = (c.smask & 4) ? ja.ang[2] : ja.ang[2] - clampf(ja.ang[2], M.lf(b2 + MBD_D_LO, c.l), M.lf(b2 + MBD_D_HI, c.l));
    v3 dqj_n = vscale(ja.ax[0], e0);
    dqj_n = vfma(ja.ax[1], e1, dqj_n);
    dqj_n = vfma(ja.ax[2], e2, dqj_n);
    v3 dqj_1 = V3(e0, -ja.r20, ja.r10);
    v3 dqj = (c.ndof == 1) ? dqj_1 : dqj_n;
    v3 dq = vrotate(dqj, a_p);
    float th;
    v3 na = vnormalize(dq, &th);
    float nn = vdot(na, na);
    float dla = MBD_DIV(-th, fmaf(ii_p, nn, nn) + 1e-6f);
    v3 Pa = vscale(na, dla);
    q4 dqa_c = vqmul(Pa, s.q);
    q4 dqa_p = vqmul(Pa, qp);
    const float hsp = 0.5f * K.scale_pos, hsa = 0.5f * K.scale_ang;
    dpc = vscale(dp_c, K.scale_pos);
    dpp = vscale(dp_p, K.scale_pos);
    dqc = qadd(qscale(dq_c, hsp), qscale(dqa_c, hsa));
    dqp = qadd(qscale(dq_p, -hsp * ii_p), qscale(dqa_p, -hsa * ii_p));
  }
  {
    v3 dp = dpc;
    q4 dq = dqc;
#pragma unroll
    for (int k = 0; k < MBD_MAXCHILD; ++k) {
      int src = c.csrc[k];
      v3 a = shfl3(dpp, src >= 0 ? src : 0);
      q4 b = shfl4(dqp, src >= 0 ? src : 0);
      if (src >= 0) { dp = vadd(dp, a); dq = qadd(dq, b); }
    }
    s.p = vadd(s.p, dp);
    s.q = qnormalize(qadd(s.q, dq));
  }
  // ---- contact.get + collisions.resolve_position ---------------------------------------------------
  float dlam[CMAX];
  v3 cpos[CMAX];
#pragma unroll
  for (int ci = 0; ci < CMAX; ++ci) { dlam[ci] = 0.0f; cpos[ci] = V3(0.0f, 0.0f, 0.0f); }
  if (c.ncon > 0) {
    v3 dp = V3(0.0f, 0.0f, 0.0f);
    q4 dq = Q4(0.0f, 0.0f, 0.0f, 0.0f);
    const v3 p0 = s.p;
    const q4 q0 = s.q;
#pragma unroll
    for (int ci = 0; ci < CMAX; ++ci)
      if (ci < c.ncon) {
        const float mu = DR ? M.lf(MBD_F_CON0 + ci * MBD_CON_STRIDE + 4, c.l) * f_mu : 0.0f;
        contact_position_plane<DR>(M, c.l, ci, c.inv_mass, p0, q0, prev.p, prev.q, dp, dq, dlam[ci], cpos[ci], mu);
      }
    s.p = vfma(dp, K.collide_scale, s.p);
    s.q = qnormalize(qadd(s.q, qscale(dq, 0.5f * K.collide_scale)));
  }
  // ---- integrator.project_xd -----------------------------------------------------------------------
  {
    s.v = vscale(vsub(s.p, prev.p), K.inv_dt);
    q4 dq = qmul(s.q, qconj(prev.q));
    float sc = dq.w >= 0.0f ? K.two_inv_dt : -K.two_inv_dt;
    s.w = V3(dq.x * sc, dq.y * sc, dq.z * sc);
  }
  // ---- collisions.resolve_velocity -------------------------------------------------------------------
  if (c.ncon > 0) {
    v3 dv = V3(0.0f, 0.0f, 0.0f), dw = V3(0.0f, 0.0f, 0.0f);
    const v3 v0 = s.v, w0 = s.w;
#pragma unroll
    for (int ci = 0; ci < CMAX; ++ci)
      if (ci < c.ncon) {
        const float mu = DR ? M.lf(MBD_F_CON0 + ci * MBD_CON_STRIDE + 4, c.l) * f_mu : 0.0f;
        contact_velocity_plane<DR>(M, c.l, ci, c.inv_mass, K.inv_dt, K.elasticity, s.p, v0, w0, v_before, w_before, cpos[ci], dlam[ci],
                                   dv, dw, mu);
      }
    s.v = vadd(s.v, dv);
    s.w = vadd(s.w, dw);
  }
}

// post-step rewards of the Brax-backed envs, from the root link's world position x.pos[0]
__device__ __forceinline__ float reward_post(int kind, v3 x0) {
  if (kind == MBD_REWARD_HUMANOIDRUN) {  // humanoidrun.py:46-51
    float dz = clampf(fabsf(x0.z - 1.3f), -1.0f, 1.0f);
    return (x0.x - dz) - fabsf(x0.y) * 0.1f;
  }
  if (kind == MBD_REWARD_HUMANOIDSTANDUP)  // humanoidstandup.py:50-56
    return ((1.5f - clampf(fabsf(x0.z - 1.3f), -2.0f, 1.0f)) - fabsf(x0.x) * 0.1f) - fabsf(x0.y) * 0.1f;
  return x0.x - clampf(fabsf(x0.z - 1.0f), -1.0f, 1.0f) * 0.5f;  // hopper.py:57-65 (callers pass kinds with parameters to the functions below)
}
// hopper.py:57-65 (z0 = 1.0) / walker2d.py:56-61 (z0 = 1.1)
__device__ __forceinline__ float reward_hopper(const ModelSmem& M, v3 x0) {
  return x0.x - clampf(fabsf(x0.z - M.hf(MBD_H_RW0)), -1.0f, 1.0f) * 0.5f;
}
// cartpole.py:44 — oracle/mbd_oracle.c::reward_post(MBD_REWARD_CARTPOLE): cart = link 0 (state of the caller), q1 = rotation of link 1
__device__ __forceinline__ float reward_cartpole(const ModelSmem& M, const LinkState& cart, q4 q1) {
  q4 a_p = qmul(cart.q, M.l4(MBD_F_PQ, 1));
  q4 a_c = qmul(q1, M.l4(MBD_F_JQ, 1));
  JointAngles ja;
  axis_angle_ang(qmul(qconj(a_p), a_c), M.lf(MBD_F_PARITY, 1), ja);
  v3 rcw = vrotate(M.l3(MBD_F_RC, 0), cart.q);
  v3 va = vadd(cart.v, vcross(cart.w, rcw));
  float xd = vdot(va, slide_axis(0, M.lf(MBD_F_PARITY, 0), M.l4(MBD_F_PQ, 0)));
  return mbd_cosf(ja.ang[0]) - fabsf(xd);
}

// brax/envs/ant.py reward (oracle/mbd_oracle.c::reward_ant): forward velocity of the root + healthy reward - control cost;
// u = this sample's action row of the env step
__device__ __forceinline__ float reward_ant(const ModelSmem& M, float x_before, float x_after, const float* u, int nu) {
  const float env_dt = M.hf(MBD_H_RW0), healthy = M.hf(MBD_H_RW0 + 1), wc = M.hf(MBD_H_RW0 + 2);
  float fwd = (x_after - x_before) / env_dt;
  float ss = 0.0f;
  for (int k = 0; k < nu; ++k) ss = ss + u[k] * u[k];
  return (fwd + healthy) - wc * ss;
}

// com.to_world pieces
__device__ __forceinline__ v3 link_origin(const ModelSmem& M, const LaneCfg& c, const LinkState& s) {
  return vsub(s.p, vrotate(M.l3(MBD_F_COM, c.l < MBD_MAXL ? c.l : 0), s.q));
}
__device__ __forceinline__ v3 link_origin_vel(const ModelSmem& M, const LaneCfg& c, const LinkState& s) {
  v3 rc = vrotate(M.l3(MBD_F_COM, c.l < MBD_MAXL ? c.l : 0), s.q);
  return vadd(s.v, vcross(rc, s.w));
}

}  // namespace mbd
