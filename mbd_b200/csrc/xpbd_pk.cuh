// xpbd_pk.cuh — the Brax-positional (XPBD) step, warp per link, written once against the scalar layer of
// pk_scalar.cuh (T = f2: two samples per thread, every operation issued on both).
//
// Same algorithm, same association order and the same FMA placement as xpbd_wpl.cuh::positional_step_wpl and
// oracle/mbd_oracle.c — every expression below is the scalar expression with a*b -> mul, a+b -> add, a-b -> sub,
// fmaf -> fma, -a -> neg, c ? x : y -> sel.  The four phases are separate functions so that the host check build
// (tests/host_pk) can run them link by link, phase by phase, against the CPU oracle:
//   A  joints.acceleration_update: joint-frame spring/damper/motor torque  -> E[l][0..2]
//   B  gather the children's reactions, integrator.integrate_xdd           -> X[l] p, q
//   C  joints.position_update (XPBD joint deltas, child side kept, parent side published) -> E[l][0..6]
//   D  gather the children's deltas; contacts; integrator.project_xd; contact velocities  -> X[l] q, w
// Reference path restated: brax.positional.pipeline.step as called from upstream mbd/envs/humanoidrun.py:36
// (Brax itself is un-vendored: see DESIGN.md).
#pragma once

#include "mbd_model.h"
#include "pk_scalar.cuh"

namespace mbd {
namespace pk {

constexpr int kLanes = 32;
constexpr int kXF = 10;  // published pose fields per link: p(3) q(4) w(3)
constexpr int kEF = 7;   // exchange fields per link: T(3)  |  dpp(3) dqp(4)

template <class T> struct V { T x, y, z; };
template <class T> struct Q { T w, x, y, z; };
template <class T> PK_FN V<T> mkV(T x, T y, T z) { V<T> r; r.x = x; r.y = y; r.z = z; return r; }
template <class T> PK_FN Q<T> mkQ(T w, T x, T y, T z) { Q<T> r; r.w = w; r.x = x; r.y = y; r.z = z; return r; }
template <class T> PK_FN V<T> bcV(float x, float y, float z) { return mkV(bc<T>(x), bc<T>(y), bc<T>(z)); }
template <class T> PK_FN Q<T> bcQ(float w, float x, float y, float z) { return mkQ(bc<T>(w), bc<T>(x), bc<T>(y), bc<T>(z)); }
template <class T> PK_FN V<T> vadd(V<T> a, V<T> b) { return mkV(add(a.x, b.x), add(a.y, b.y), add(a.z, b.z)); }
template <class T> PK_FN V<T> vsub(V<T> a, V<T> b) { return mkV(sub(a.x, b.x), sub(a.y, b.y), sub(a.z, b.z)); }
template <class T> PK_FN V<T> vscale(V<T> a, T s) { return mkV(mul(a.x, s), mul(a.y, s), mul(a.z, s)); }
template <class T> PK_FN V<T> vfma(V<T> b, T s, V<T> a) { return mkV(fma(b.x, s, a.x), fma(b.y, s, a.y), fma(b.z, s, a.z)); }
template <class T> PK_FN T vdot(V<T> a, V<T> b) { return fma(a.z, b.z, fma(a.y, b.y, mul(a.x, b.x))); }
template <class T> PK_FN V<T> vcross(V<T> a, V<T> b) {
  return mkV(fma(a.y, b.z, neg(mul(a.z, b.y))), fma(a.z, b.x, neg(mul(a.x, b.z))), fma(a.x, b.y, neg(mul(a.y, b.x))));
}
template <class T, bool kExact = false> PK_FN V<T> vnormalize(V<T> a, T* norm) {   // kExact: sqrt_x (pk_scalar.cuh)
  const T zero = bc<T>(0.0f);
  T n = kExact ? sqrt_x(vdot(a, a)) : sqrt_(vdot(a, a));
  T inv = sel(eq(n, zero), zero, rcp_(n));
  *norm = n;
  return vscale(a, inv);
}
template <class T> PK_FN Q<T> qconj(Q<T> q) { return mkQ(q.w, neg(q.x), neg(q.y), neg(q.z)); }
template <class T> PK_FN Q<T> qmul(Q<T> u, Q<T> v) {
  return mkQ(fma(neg(u.z), v.z, fma(neg(u.y), v.y, fma(neg(u.x), v.x, mul(u.w, v.w)))),
             fma(neg(u.z), v.y, fma(u.y, v.z, fma(u.x, v.w, mul(u.w, v.x)))),
             fma(u.z, v.x, fma(u.y, v.w, fma(neg(u.x), v.z, mul(u.w, v.y)))),
             fma(u.z, v.w, fma(neg(u.y), v.x, fma(u.x, v.y, mul(u.w, v.z)))));
}
template <class T> PK_FN Q<T> vqmul(V<T> a, Q<T> q) {
  return mkQ(fma(neg(a.z), q.z, fma(neg(a.y), q.y, neg(mul(a.x, q.x)))),
             fma(neg(a.z), q.y, fma(a.y, q.z, mul(a.x, q.w))),
             fma(a.z, q.x, fma(a.y, q.w, neg(mul(a.x, q.z)))),
             fma(a.z, q.w, fma(neg(a.y), q.x, mul(a.x, q.y))));
}
template <class T> PK_FN Q<T> vqmul_xy(T ax, T ay, Q<T> q) {
  return mkQ(fma(neg(ay), q.y, neg(mul(ax, q.x))), fma(ay, q.z, mul(ax, q.w)), fma(ay, q.w, neg(mul(ax, q.z))), fma(neg(ay), q.x, mul(ax, q.y)));
}
// oracle form t = 2(u x v); c = u x t; r = fma(w, t, v) + c, with the exact doublings folded (xpbd_device.cuh::vrotate)
template <class T> PK_FN V<T> vrotate(V<T> v, Q<T> q) {
  V<T> u = mkV(q.x, q.y, q.z);
  V<T> t = vcross(u, v);
  V<T> c = vcross(u, t);
  T w2 = add(q.w, q.w);
  const T two = bc<T>(2.0f);
  return mkV(fma(two, c.x, fma(w2, t.x, v.x)), fma(two, c.y, fma(w2, t.y, v.y)), fma(two, c.z, fma(w2, t.z, v.z)));
}
template <class T> PK_FN V<T> vinv_rotate(V<T> v, Q<T> q) { return vrotate(v, qconj(q)); }
template <class T> PK_FN Q<T> qnormalize(Q<T> q) {
  T n = sqrt_(fma(q.z, q.z, fma(q.y, q.y, fma(q.x, q.x, mul(q.w, q.w)))));
  T inv = rcp_(n);
  return mkQ(mul(q.w, inv), mul(q.x, inv), mul(q.y, inv), mul(q.z, inv));
}
template <class T> PK_FN Q<T> qadd(Q<T> a, Q<T> b) { return mkQ(add(a.w, b.w), add(a.x, b.x), add(a.y, b.y), add(a.z, b.z)); }
// the same sums for operands that are (or may be) packed products: see add_nf in pk_scalar.cuh
template <class T> PK_FN V<T> vadd_nf(V<T> a, V<T> b) { return mkV(add_nf(a.x, b.x), add_nf(a.y, b.y), add_nf(a.z, b.z)); }
template <class T> PK_FN V<T> vsub_nf(V<T> a, V<T> b) { return mkV(sub_nf(a.x, b.x), sub_nf(a.y, b.y), sub_nf(a.z, b.z)); }
template <class T> PK_FN Q<T> qadd_nf(Q<T> a, Q<T> b) { return mkQ(add_nf(a.w, b.w), add_nf(a.x, b.x), add_nf(a.y, b.y), add_nf(a.z, b.z)); }
template <class T> PK_FN Q<T> qscale(Q<T> a, T s) { return mkQ(mul(a.w, s), mul(a.x, s), mul(a.y, s), mul(a.z, s)); }

// ---- model table: T-typed copy of the blob's float fields (f2: every word duplicated), ints from the blob -------------
template <class T>
struct Model {
  const T* t;        // [MBD_BLOB_WORDS] broadcast copies of the float fields
  const float* f;    // the blob (integer fields are read from here)
  PK_MFN T h(int w) const { return t[w]; }
  PK_MFN int hi(int w) const { return (int)mbd_f2u(f[w]); }
  PK_MFN T l(int field, int l_) const { return t[MBD_HDR_WORDS + field * MBD_MAXL + l_]; }
  PK_MFN int li(int field, int l_) const { return (int)mbd_f2u(f[MBD_HDR_WORDS + field * MBD_MAXL + l_]); }
  PK_MFN V<T> l3(int field, int l_) const { return mkV(l(field, l_), l(field + 1, l_), l(field + 2, l_)); }
  PK_MFN Q<T> l4(int field, int l_) const { return mkQ(l(field, l_), l(field + 1, l_), l(field + 2, l_), l(field + 3, l_)); }
};

// ---- exchange rows [link][field][lane] of T ---------------------------------------------------------------------------
template <class T>
struct Smem {
  T* X;  // [L][kXF][32]
  T* E;  // [L][kEF][32]
  int lane;
  PK_MFN T& x(int link, int f) const { return X[(link * kXF + f) * kLanes + lane]; }
  PK_MFN T& e(int link, int f) const { return E[(link * kEF + f) * kLanes + lane]; }
  PK_MFN V<T> xp(int link) const { return mkV(x(link, 0), x(link, 1), x(link, 2)); }
  PK_MFN Q<T> xq(int link) const { return mkQ(x(link, 3), x(link, 4), x(link, 5), x(link, 6)); }
  PK_MFN V<T> xw(int link) const { return mkV(x(link, 7), x(link, 8), x(link, 9)); }
  PK_MFN void put_p(int link, V<T> p) const { x(link, 0) = p.x; x(link, 1) = p.y; x(link, 2) = p.z; }
  PK_MFN void put_q(int link, Q<T> q) const { x(link, 3) = q.w; x(link, 4) = q.x; x(link, 5) = q.y; x(link, 6) = q.z; }
  PK_MFN void put_w(int link, V<T> w) const { x(link, 7) = w.x; x(link, 8) = w.y; x(link, 9) = w.z; }
  PK_MFN V<T> e3(int link, int f) const { return mkV(e(link, f), e(link, f + 1), e(link, f + 2)); }
  PK_MFN Q<T> e4(int link, int f) const { return mkQ(e(link, f), e(link, f + 1), e(link, f + 2), e(link, f + 3)); }
  PK_MFN void put_e3(int link, int f, V<T> a) const { e(link, f) = a.x; e(link, f + 1) = a.y; e(link, f + 2) = a.z; }
  PK_MFN void put_e4(int link, int f, Q<T> a) const { e(link, f) = a.w; e(link, f + 1) = a.x; e(link, f + 2) = a.y; e(link, f + 3) = a.z; }
};

struct Cfg {  // warp-uniform link topology
  int l, ndof, parent, ncon;
  int child[MBD_MAXCHILD];
};
template <class T> PK_FN void load_cfg(const Model<T>& M, int l, Cfg& c) {
  c.l = l;
  c.ndof = M.li(MBD_F_NDOF, l);
  c.parent = M.li(MBD_F_PARENT, l);
  c.ncon = M.li(MBD_F_NCON, l);
  for (int k = 0; k < MBD_MAXCHILD; ++k) c.child[k] = M.li(MBD_F_CHILD0 + k, l);
}

template <class T> struct State { V<T> p; Q<T> q; V<T> w; V<T> v; };  // x_i.pos, x_i.rot, xd_i.ang, xd_i.vel
// values one link carries from phase to phase inside a substep
template <class T, int CMAX> struct Carry {
  V<T> p_prev; Q<T> q_prev;    // x_i_prev
  V<T> Tq;                     // this link's joint torque in the world frame
  V<T> w_before, v_before;     // xd_i right after integration
  V<T> dpc; Q<T> dqc;          // this link's own joint deltas
};

// ---- kinematics.axis_angle_ang (xpbd_device.cuh::axis_angle_ang / xpbd_wpl.cuh::axis_angle_1dof) -----------------------
template <class T> struct Angles { T ang[3]; V<T> ax[3]; T r10, r20; };
template <class T> PK_FN void axis_angle_1dof(Q<T> j, T& psi, T& r10, T& r20) {
  const T one = bc<T>(1.0f), two = bc<T>(2.0f);
  T w = j.w, x = j.x, y = j.y, z = j.z;
  T r12 = mul(two, fma(y, z, neg(mul(w, x))));
  T r22 = sub_nf(one, mul(two, fma(y, y, mul(x, x))));
  r10 = mul(two, fma(x, y, mul(w, z)));
  r20 = mul(two, fma(x, z, neg(mul(w, y))));
  psi = atan2_(neg(r12), r22);
}
// third = false leaves ang[2] / ax[2] unset: phase A of a 2-dof joint never reads them, and their atan2_ is ~10 % of
// that phase's issue (phase C needs all three: the locked third axis enters dqj).  Warp-uniform, so a uniform branch.
template <class T> PK_FN void axis_angle_ang(Q<T> j, T parity, Angles<T>& o, bool third = true) {
  const T zero = bc<T>(0.0f), one = bc<T>(1.0f), two = bc<T>(2.0f);
  T w = j.w, x = j.x, y = j.y, z = j.z;
  T r00 = sub_nf(one, mul(two, fma(z, z, mul(y, y))));
  T r01 = mul(two, fma(x, y, neg(mul(w, z))));
  T r02 = mul(two, fma(x, z, mul(w, y)));
  T r12 = mul(two, fma(y, z, neg(mul(w, x))));
  T r22 = sub_nf(one, mul(two, fma(y, y, mul(x, x))));
  o.r10 = mul(two, fma(x, y, mul(w, z)));
  o.r20 = mul(two, fma(x, z, neg(mul(w, y))));
  T psi = atan2_(neg(r12), r22);
  T cth = sqrt_(fma(r01, r01, mul(r00, r00)));
  T theta = atan2_(r02, cth);
  T ln;
  V<T> lon = vnormalize(mkV(zero, r22, neg(r12)), &ln);
  o.ang[0] = psi; o.ang[1] = theta;
  o.ax[0] = mkV(one, zero, zero);
  o.ax[1] = lon;
  if (third) {
    T phi = atan2_(neg(r01), r00);
    o.ang[2] = mul(parity, phi);
    o.ax[2] = mkV(mul(parity, r02), mul(parity, r12), mul(parity, r22));
  }
}

// ---- contacts against the z = 0 plane (xpbd_device.cuh::contact_position_plane / contact_velocity_plane) ----------------
template <class T>
PK_FN void contact_position_plane(const Model<T>& M, int l, int ci, T im, V<T> p, Q<T> q, V<T> p_prev, Q<T> q_prev, V<T>& dp, Q<T>& dq,
                                  T& dl_out, V<T>& cp_out) {
  const T zero = bc<T>(0.0f);
  const int base = MBD_F_CON0 + ci * MBD_CON_STRIDE;
  const T radius = M.l(base + 3, l), mu = M.l(base + 4, l);
  V<T> centre = vadd(p, vrotate(M.l3(base, l), q));
  T dist = sub(centre.z, radius);
  V<T> cp = mkV(centre.x, centre.y, sub(centre.z, add_nf(radius, mul(bc<T>(0.5f), dist))));
  auto coll = lt(dist, zero);
  V<T> r = vsub(cp, p);
  T w = add(im, fma(r.x, r.x, mul(r.y, r.y)));
  T dl = sel(coll, div_(neg(dist), add(w, bc<T>(1e-6f))), zero);
  dp.z = add_nf(dp.z, mul(dl, im));
  dq = qadd(dq, vqmul_xy(mul(r.y, dl), neg(mul(r.x, dl)), q));
  V<T> rl = vinv_rotate(r, q);
  V<T> pbar = vadd(p_prev, vrotate(rl, q_prev));
  T dx = sub(cp.x, pbar.x), dy = sub(cp.y, pbar.y);
  T ct = sqrt_x(fma(dy, dy, mul(dx, dx)));
  T inv = sel(eq(ct, zero), zero, rcp_(ct));
  T ntx = mul(dx, inv), nty = mul(dy, inv);
  T c1 = neg(mul(r.z, nty)), c2 = mul(r.z, ntx), c3 = fma(r.x, nty, neg(mul(r.y, ntx)));
  T wt = add(im, fma(c3, c3, fma(c2, c2, mul(c1, c1))));
  T dlt = div_(neg(ct), add(wt, bc<T>(1e-6f)));
  auto stat = mand(coll, lt(abs_(dlt), mul(mu, abs_(dl))));
  T m = sel(stat, dlt, zero);
  T ptx = mul(ntx, m), pty = mul(nty, m);
  dp.x = add_nf(dp.x, mul(ptx, im));
  dp.y = add_nf(dp.y, mul(pty, im));
  dq = qadd(dq, vqmul(mkV(neg(mul(r.z, pty)), mul(r.z, ptx), fma(r.x, pty, neg(mul(r.y, ptx)))), q));
  dl_out = dl;
  cp_out = cp;
}

template <class T>
PK_FN void contact_velocity_plane(const Model<T>& M, int l, int ci, T im, T inv_dt, T elasticity, V<T> p, V<T> v, V<T> w, V<T> v_before,
                                  V<T> w_before, V<T> cp, T dl, V<T>& dv, V<T>& dw) {
  const T zero = bc<T>(0.0f);
  const T mu = M.l(MBD_F_CON0 + ci * MBD_CON_STRIDE + 4, l);
  V<T> r = vsub(cp, p);
  V<T> rel = vadd(v, vcross(w, r));   // v is a product (project_xd)
  T vn = rel.z;
  T vtn = sqrt_x(fma(rel.y, rel.y, mul(rel.x, rel.x)));
  T inv = sel(eq(vtn, zero), zero, rcp_(vtn));
  T tdx = mul(rel.x, inv), tdy = mul(rel.y, inv);
  T fr = mul(mul(mu, abs_(dl)), inv_dt);
  T mag = sel(lt(fr, vtn), fr, vtn);
  T c1 = neg(mul(r.z, tdy)), c2 = mul(r.z, tdx), c3 = fma(r.x, tdy, neg(mul(r.y, tdx)));
  T wd = add(im, fma(c3, c3, fma(c2, c2, mul(c1, c1))));
  T kd = rcp_(add(wd, bc<T>(1e-6f)));
  T pdx = mul(mul(tdx, neg(mag)), kd), pdy = mul(mul(tdy, neg(mag)), kd);
  V<T> rel_old = vadd(v_before, vcross(w_before, r));
  T vn_old = rel_old.z;
  T rest = mul(neg(elasticity), vn_old);
  rest = sel(lt(rest, zero), rest, zero);
  T wn = add(im, fma(r.x, r.x, mul(r.y, r.y)));
  T prz = mul(add(neg(vn), rest), rcp_(add(wn, bc<T>(1e-6f))));   // rest may be a product
  auto live = eq(dl, zero);   // dl == 0: no impulse at all
  V<T> P = mkV(sel(live, zero, pdx), sel(live, zero, pdy), sel(live, zero, sel(le(vn_old, zero), prz, zero)));
  dv = vadd_nf(dv, vscale(P, im));
  dw = vadd(dw, vcross(r, P));
}

// ---- phase A ------------------------------------------------------------------------------------------------------
template <class T, int CMAX>
PK_FN void phase_A(const Model<T>& M, const Cfg& c, const Smem<T>& S, State<T>& s, const T tau[MBD_MAXDOF], Carry<T, CMAX>& k) {
  const T zero = bc<T>(0.0f), one = bc<T>(1.0f);
  k.p_prev = s.p;
  k.q_prev = s.q;
  k.Tq = mkV(zero, zero, zero);
  if (c.ndof > 0) {
    Q<T> qp = mkQ(one, zero, zero, zero);
    V<T> wp = mkV(zero, zero, zero);
    if (c.parent >= 0) { qp = S.xq(c.parent); wp = S.xw(c.parent); }
    Q<T> a_p = qmul(qp, M.l4(MBD_F_PQ, c.l));
    Q<T> a_c = qmul(s.q, M.l4(MBD_F_JQ, c.l));
    Q<T> j = qmul(qconj(a_p), a_c);
    V<T> jd = vinv_rotate(vsub(s.w, wp), a_p);   // s.w is a product after project_xd
    V<T> tq = vscale(jd, neg(M.l(MBD_F_ANG_DAMP, c.l)));
    if (c.ndof == 1) {
      T psi, r10, r20;
      axis_angle_1dof(j, psi, r10, r20);
      T vel = vdot(mkV(one, zero, zero), jd);
      T t = fma(neg(M.l(MBD_F_DOF0 + MBD_D_DAMP, c.l)), vel, fma(neg(M.l(MBD_F_DOF0 + MBD_D_STIFF, c.l)), psi, tau[0]));
      tq = vfma(mkV(one, zero, zero), t, tq);
    } else {
      Angles<T> ja;
      axis_angle_ang(j, M.l(MBD_F_PARITY, c.l), ja, c.ndof > 2);
#if PK_DEVICE
#pragma unroll
#endif
      for (int d = 0; d < MBD_MAXDOF; ++d) {
        if (d < c.ndof) {
          int base = MBD_F_DOF0 + d * MBD_DOF_STRIDE;
          T vel = vdot(ja.ax[d], jd);
          T t = fma(neg(M.l(base + MBD_D_DAMP, c.l)), vel, fma(neg(M.l(base + MBD_D_STIFF, c.l)), ja.ang[d], tau[d]));
          tq = vfma(ja.ax[d], t, tq);
        }
      }
    }
    k.Tq = vrotate(tq, a_p);
    S.put_e3(c.l, 0, k.Tq);
  }
}

// ---- phase B ------------------------------------------------------------------------------------------------------
template <class T, int CMAX>
PK_FN void phase_B(const Model<T>& M, const Cfg& c, const Smem<T>& S, State<T>& s, Carry<T, CMAX>& k) {
  V<T> acc = k.Tq;
#if PK_DEVICE
#pragma unroll
#endif
  for (int i = 0; i < MBD_MAXCHILD; ++i)
    if (c.child[i] >= 0) acc = vsub(acc, S.e3(c.child[i], 0));
  const T dt = M.h(MBD_H_DT), ad = M.h(MBD_H_ANG_DAMP), vd = M.h(MBD_H_VEL_DAMP);
  s.w = mkV(fma(acc.x, dt, mul(s.w.x, ad)), fma(acc.y, dt, mul(s.w.y, ad)), fma(acc.z, dt, mul(s.w.z, ad)));
  s.v = mkV(fma(M.h(MBD_H_GX), dt, mul(s.v.x, vd)), fma(M.h(MBD_H_GY), dt, mul(s.v.y, vd)), fma(M.h(MBD_H_GZ), dt, mul(s.v.z, vd)));
  s.q = qnormalize(qadd(s.q, vqmul(vscale(s.w, M.h(MBD_H_HALF_DT)), s.q)));   // s.q is a product (qnormalize)
  s.p = vfma(s.v, dt, s.p);
  S.put_p(c.l, s.p);
  S.put_q(c.l, s.q);
  k.w_before = s.w;
  k.v_before = s.v;
}

// ---- phase C ------------------------------------------------------------------------------------------------------
template <class T, int CMAX>
PK_FN void phase_C(const Model<T>& M, const Cfg& c, const Smem<T>& S, State<T>& s, Carry<T, CMAX>& k) {
  const T zero = bc<T>(0.0f), one = bc<T>(1.0f);
  k.dpc = mkV(zero, zero, zero);
  k.dqc = mkQ(zero, zero, zero, zero);
  if (c.ndof > 0) {
    V<T> pp = mkV(zero, zero, zero);
    Q<T> qp = mkQ(one, zero, zero, zero);
    if (c.parent >= 0) { pp = S.xp(c.parent); qp = S.xq(c.parent); }
    const T im_c = M.l(MBD_F_INV_MASS, c.l), im_p = M.l(MBD_F_PINV_MASS, c.l), ii_p = M.l(MBD_F_PINV_INERTIA, c.l);
    V<T> rpw = vrotate(M.l3(MBD_F_RP, c.l), qp);
    V<T> rcw = vrotate(M.l3(MBD_F_RC, c.l), s.q);
    V<T> e = vsub(vadd(s.p, rcw), vadd(pp, rpw));
    T cn;
    V<T> n = vnormalize<T, true>(e, &cn);
    V<T> crc = vcross(rcw, n), crp = vcross(rpw, n);
    T w_c = add(im_c, vdot(crc, crc));
    T w_p = fma(ii_p, vdot(crp, crp), im_p);
    T dl = div_(neg(cn), add(add(w_p, w_c), bc<T>(1e-6f)));
    V<T> P = vscale(n, dl);
    V<T> dp_c = vscale(P, im_c);
    Q<T> dq_c = vqmul(vcross(rcw, P), s.q);
    V<T> dp_p = vscale(P, neg(im_p));
    Q<T> dq_p = vqmul(vcross(rpw, P), qp);
    Q<T> a_p = qmul(qp, M.l4(MBD_F_PQ, c.l));
    Q<T> a_c = qmul(s.q, M.l4(MBD_F_JQ, c.l));
    Q<T> j = qmul(qconj(a_p), a_c);
    V<T> dqj;
    const int b0 = MBD_F_DOF0, b1 = MBD_F_DOF0 + MBD_DOF_STRIDE, b2 = MBD_F_DOF0 + 2 * MBD_DOF_STRIDE;
    if (c.ndof == 1) {
      T psi, r10, r20;
      axis_angle_1dof(j, psi, r10, r20);
      T e0 = sub(psi, clamp_(psi, M.l(b0 + MBD_D_LO, c.l), M.l(b0 + MBD_D_HI, c.l)));
      dqj = mkV(e0, neg(r20), r10);
    } else {
      Angles<T> ja;
      axis_angle_ang(j, M.l(MBD_F_PARITY, c.l), ja);
      T e0 = sub(ja.ang[0], clamp_(ja.ang[0], M.l(b0 + MBD_D_LO, c.l), M.l(b0 + MBD_D_HI, c.l)));
      T e1 = sub(ja.ang[1], clamp_(ja.ang[1], M.l(b1 + MBD_D_LO, c.l), M.l(b1 + MBD_D_HI, c.l)));
      T e2 = sub(ja.ang[2], clamp_(ja.ang[2], M.l(b2 + MBD_D_LO, c.l), M.l(b2 + MBD_D_HI, c.l)));
      dqj = vscale(ja.ax[0], e0);
      dqj = vfma(ja.ax[1], e1, dqj);
      dqj = vfma(ja.ax[2], e2, dqj);
    }
    V<T> dq = vrotate(dqj, a_p);
    T th;
    V<T> na = vnormalize(dq, &th);
    T nn = vdot(na, na);
    T dla = div_(neg(th), add(fma(ii_p, nn, nn), bc<T>(1e-6f)));
    V<T> Pa = vscale(na, dla);
    Q<T> dqa_c = vqmul(Pa, s.q);
    Q<T> dqa_p = vqmul(Pa, qp);
    // the exact factors 0.5 (and ii_p in {0,1}) are folded into the scale constants: (x*0.5)*s == x*(0.5*s) bit for bit
    const T sp = M.h(MBD_H_SCALE_POS);
    const T hsp = mul(bc<T>(0.5f), sp), hsa = mul(bc<T>(0.5f), M.h(MBD_H_SCALE_ANG));
    k.dpc = vscale(dp_c, sp);
    k.dqc = qadd_nf(qscale(dq_c, hsp), qscale(dqa_c, hsa));
    S.put_e3(c.l, 0, vscale(dp_p, sp));
    S.put_e4(c.l, 3, qadd_nf(qscale(dq_p, mul(neg(hsp), ii_p)), qscale(dqa_p, mul(neg(hsa), ii_p))));
  }
}

// ---- phase D ------------------------------------------------------------------------------------------------------
template <class T, int CMAX>
PK_FN void phase_D(const Model<T>& M, const Cfg& c, const Smem<T>& S, State<T>& s, Carry<T, CMAX>& k) {
  const T zero = bc<T>(0.0f);
  {
    V<T> dp = k.dpc;
    Q<T> dq = k.dqc;
#if PK_DEVICE
#pragma unroll
#endif
    for (int i = 0; i < MBD_MAXCHILD; ++i) {
      if (c.child[i] >= 0) { dp = vadd(dp, S.e3(c.child[i], 0)); dq = qadd(dq, S.e4(c.child[i], 3)); }   // dp starts as a product
    }
    s.p = vadd(s.p, dp);
    s.q = qnormalize(qadd(s.q, dq));
  }
  T dlam[CMAX];
  V<T> cpos[CMAX];
  if (c.ncon > 0) {
    V<T> dp = mkV(zero, zero, zero);
    Q<T> dq = mkQ(zero, zero, zero, zero);
    const V<T> p0 = s.p;
    const Q<T> q0 = s.q;
#if PK_DEVICE
#pragma unroll
#endif
    for (int ci = 0; ci < CMAX; ++ci) {
      dlam[ci] = zero; cpos[ci] = mkV(zero, zero, zero);
      if (ci < c.ncon) contact_position_plane(M, c.l, ci, M.l(MBD_F_INV_MASS, c.l), p0, q0, k.p_prev, k.q_prev, dp, dq, dlam[ci], cpos[ci]);
    }
    const T cs = M.h(MBD_H_COLLIDE_SCALE);
    s.p = vfma(dp, cs, s.p);
    s.q = qnormalize(qadd_nf(s.q, qscale(dq, mul(bc<T>(0.5f), cs))));
  }
  {
    s.v = vscale(vsub(s.p, k.p_prev), M.h(MBD_H_INV_DT));
    Q<T> dq = qmul(s.q, qconj(k.q_prev));
    const T tid = M.h(MBD_H_TWO_INV_DT);
    T sc = sel(ge(dq.w, zero), tid, neg(tid));
    s.w = mkV(mul(dq.x, sc), mul(dq.y, sc), mul(dq.z, sc));
  }
  if (c.ncon > 0) {
    V<T> dv = mkV(zero, zero, zero), dw = mkV(zero, zero, zero);
    const V<T> v0 = s.v, w0 = s.w;
#if PK_DEVICE
#pragma unroll
#endif
    for (int ci = 0; ci < CMAX; ++ci)
      if (ci < c.ncon)
        contact_velocity_plane(M, c.l, ci, M.l(MBD_F_INV_MASS, c.l), M.h(MBD_H_INV_DT), M.h(MBD_H_ELASTICITY), s.p, v0, w0, k.v_before,
                               k.w_before, cpos[ci], dlam[ci], dv, dw);
    s.v = vadd(s.v, dv);   // s.v, s.w are products (project_xd)
    s.w = vadd(s.w, dw);
  }
  S.put_q(c.l, s.q);
  S.put_w(c.l, s.w);
}

// com.to_world pieces
template <class T> PK_FN V<T> link_origin_w(const Model<T>& M, int l, const State<T>& s) { return vsub(s.p, vrotate(M.l3(MBD_F_COM, l), s.q)); }
template <class T> PK_FN V<T> link_origin_vel_w(const Model<T>& M, int l, const State<T>& s) {
  V<T> rc = vrotate(M.l3(MBD_F_COM, l), s.q);
  return vadd(s.v, vcross(rc, s.w));
}

}  // namespace pk
}  // namespace mbd
