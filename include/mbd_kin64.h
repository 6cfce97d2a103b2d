/* mbd_kin64.h — float64 kinematics of the vector env (csrc/vecenv.cuh), compiled for the device and for the host.
 *
 * Restates, in float64 and in the same operation order, what the host env surface computes around one physics step:
 *   mbd_k64_pipeline_init  kinematics.forward + com.from_world (mbd_b200/model/kinematics.py: forward, pipeline_init), rounded
 *                          once to the float32 [Lsim,13] state row the kernels consume;
 *   mbd_k64_world          com.to_world of the simulated links (kinematics.to_world) rounded to float32, the cosmetic links at
 *                          their float32 init pose (PipelineEnv._static_x), i.e. the x / xd of PipelineEnv._make_pipeline_state;
 *   mbd_k64_inverse        kinematics.inverse on those float32 world poses, rounded once to float32 (q, qd).
 * Every float64 intermediate is a sum / product / quotient / sqrt / sin / cos / atan2 / hypot of float64 values, so the device and
 * numpy agree up to the last float64 bits, and the results — rounded once to float32 — are equal or one float32 ulp apart
 * (tests/test_vecenv_cpu.py holds this header, built with g++, to that bound on every shipped model).
 *
 * Table layout (doubles, packed by mbd_b200/envs/vec.py:pack_kin64):
 *   [0] L  [1] nq  [2] nqd  [3] nsim  [4] normalise free-joint quaternions (MBD_FREE_QUAT_NORMALIZE)  [5..7] unused
 *   [MBD_K64_SIM + i]       link index of simulated link i (state row i)
 *   [MBD_K64_LINK + l * MBD_K64_LS + f]   per link, fields MBD_K64_L_*
 *   [MBD_K64_DOF + d * MBD_K64_DS + f]    per dof: axis (3), is_slide, ref
 *   [MBD_K64_INITQ + j]     init_q (float64)
 */
#ifndef MBD_KIN64_H_
#define MBD_KIN64_H_

#include <math.h>

#ifdef __CUDACC__
#define MBD_K64 __host__ __device__ __forceinline__
#else
#define MBD_K64 static inline
#endif

#define MBD_K64_MAXL 16
#define MBD_K64_MAXQ 64
#define MBD_K64_SIM 8
#define MBD_K64_LINK (MBD_K64_SIM + MBD_K64_MAXL)
#define MBD_K64_LS 32
#define MBD_K64_DOF (MBD_K64_LINK + MBD_K64_MAXL * MBD_K64_LS)
#define MBD_K64_DS 5
#define MBD_K64_INITQ (MBD_K64_DOF + MBD_K64_MAXQ * MBD_K64_DS)
#define MBD_K64_WORDS (MBD_K64_INITQ + MBD_K64_MAXQ)
/* per-link fields */
#define MBD_K64_L_TYPE 0     /* -1 = free joint, else the number of stacked 1-dof joints */
#define MBD_K64_L_QS 1
#define MBD_K64_L_DS 2
#define MBD_K64_L_PARENT 3
#define MBD_K64_L_SIMIDX 4   /* state row of the link, -1 = not simulated (cosmetic) */
#define MBD_K64_L_POS 5      /* link.transform pos (3), rot (4) */
#define MBD_K64_L_ROT 8
#define MBD_K64_L_JPOS 12    /* link.joint pos (3), rot (4) */
#define MBD_K64_L_JROT 15
#define MBD_K64_L_COM 19
#define MBD_K64_L_PARITY 22
#define MBD_K64_L_SPOS 23    /* float32 world pose at init_q (PipelineEnv._static_x rounded), pos (3), rot (4) */
#define MBD_K64_L_SROT 26

/* world link frames of all links (float64) */
struct mbd_k64_world {
  double pos[MBD_K64_MAXL][3], rot[MBD_K64_MAXL][4], ang[MBD_K64_MAXL][3], vel[MBD_K64_MAXL][3];
};

MBD_K64 void mbd_k64_qmul(const double* u, const double* v, double* o) {
  const double w = u[0] * v[0] - u[1] * v[1] - u[2] * v[2] - u[3] * v[3];
  const double x = u[0] * v[1] + u[1] * v[0] + u[2] * v[3] - u[3] * v[2];
  const double y = u[0] * v[2] - u[1] * v[3] + u[2] * v[0] + u[3] * v[1];
  const double z = u[0] * v[3] + u[1] * v[2] - u[2] * v[1] + u[3] * v[0];
  o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}
MBD_K64 double mbd_k64_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
MBD_K64 void mbd_k64_cross(const double* a, const double* b, double* o) {
  const double x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  o[0] = x; o[1] = y; o[2] = z;
}
/* mjcf.rotate: 2 (u.v) u + (s^2 - u.u) v + 2 s (u x v) */
MBD_K64 void mbd_k64_rotate(const double* v, const double* q, double* o) {
  const double s = q[0], u[3] = {q[1], q[2], q[3]};
  const double a = 2.0 * mbd_k64_dot(u, v), b = s * s - mbd_k64_dot(u, u), c = 2.0 * s;
  double cr[3];
  mbd_k64_cross(u, v, cr);
  for (int i = 0; i < 3; ++i) o[i] = a * u[i] + b * v[i] + c * cr[i];
}
MBD_K64 double mbd_k64_norm(const double* a, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += a[i] * a[i];
  return sqrt(s);
}
MBD_K64 int mbd_k64_i(const double* T, int off) { return (int)T[off]; }
MBD_K64 const double* mbd_k64_lf(const double* T, int l, int f) { return T + MBD_K64_LINK + l * MBD_K64_LS + f; }

/* kinematics.forward on q [nq], qd [nqd] (float64 views of float32 inputs) */
MBD_K64 void mbd_k64_forward(const double* T, const double* q, const double* qd, mbd_k64_world* X) {
  const int L = mbd_k64_i(T, 0);
  const bool normalize = T[4] != 0.0;
  for (int l = 0; l < L; ++l) {
    const int type = (int)*mbd_k64_lf(T, l, MBD_K64_L_TYPE);
    const int qs = (int)*mbd_k64_lf(T, l, MBD_K64_L_QS), ds = (int)*mbd_k64_lf(T, l, MBD_K64_L_DS);
    const int par = (int)*mbd_k64_lf(T, l, MBD_K64_L_PARENT);
    if (type < 0) {
      for (int i = 0; i < 3; ++i) X->pos[l][i] = q[qs + i];
      const double n = normalize ? mbd_k64_norm(q + qs + 3, 4) : 1.0;
      for (int i = 0; i < 4; ++i) X->rot[l][i] = normalize ? q[qs + 3 + i] / n : q[qs + 3 + i];
      for (int i = 0; i < 3; ++i) { X->vel[l][i] = qd[ds + i]; X->ang[l][i] = qd[ds + 3 + i]; }
      continue;
    }
    double jrot[4] = {1.0, 0.0, 0.0, 0.0}, jang[3] = {0.0, 0.0, 0.0};
    double spos[3] = {0.0, 0.0, 0.0}, svel[3] = {0.0, 0.0, 0.0}, t[3], t2[3];
    for (int k = 0; k < type; ++k) {
      const double* dof = T + MBD_K64_DOF + (ds + k) * MBD_K64_DS;
      const double ref = dof[4];
      if (dof[3] != 0.0) {   // slide dof: translation along the axis (link-transform frame)
        const double d = q[qs + k] - ref;
        for (int i = 0; i < 3; ++i) t[i] = dof[i] * d;
        mbd_k64_rotate(t, jrot, t2);
        for (int i = 0; i < 3; ++i) spos[i] = spos[i] + t2[i];
        for (int i = 0; i < 3; ++i) t[i] = dof[i] * qd[ds + k];
        mbd_k64_rotate(t, jrot, t2);
        for (int i = 0; i < 3; ++i) svel[i] = svel[i] + t2[i];
        continue;
      }
      for (int i = 0; i < 3; ++i) t[i] = dof[i] * qd[ds + k];
      mbd_k64_rotate(t, jrot, t2);
      for (int i = 0; i < 3; ++i) jang[i] = jang[i] + t2[i];
      const double ang = q[qs + k] - ref;
      const double s = sin(ang / 2.0);
      const double ra[4] = {cos(ang / 2.0), dof[0] * s, dof[1] * s, dof[2] * s};
      double nr[4];
      mbd_k64_qmul(jrot, ra, nr);
      for (int i = 0; i < 4; ++i) jrot[i] = nr[i];
    }
    const double* jp = mbd_k64_lf(T, l, MBD_K64_L_JPOS);
    double jpos[3];
    mbd_k64_rotate(jp, jrot, t);
    for (int i = 0; i < 3; ++i) jpos[i] = jp[i] - t[i] + spos[i];
    const double zero3[3] = {0.0, 0.0, 0.0}, one4[4] = {1.0, 0.0, 0.0, 0.0};
    const double* ppos = par >= 0 ? X->pos[par] : zero3;
    const double* prot = par >= 0 ? X->rot[par] : one4;
    const double* pang = par >= 0 ? X->ang[par] : zero3;
    const double* pvel = par >= 0 ? X->vel[par] : zero3;
    double tpos[3], trot[4];
    mbd_k64_rotate(mbd_k64_lf(T, l, MBD_K64_L_POS), prot, t);
    for (int i = 0; i < 3; ++i) tpos[i] = ppos[i] + t[i];
    mbd_k64_qmul(prot, mbd_k64_lf(T, l, MBD_K64_L_ROT), trot);
    mbd_k64_rotate(jpos, trot, t);
    for (int i = 0; i < 3; ++i) X->pos[l][i] = tpos[i] + t[i];
    double xr[4];
    mbd_k64_qmul(trot, jrot, xr);
    const double n = mbd_k64_norm(xr, 4);
    for (int i = 0; i < 4; ++i) X->rot[l][i] = xr[i] / n;
    double w_rel[3];
    mbd_k64_rotate(jang, trot, w_rel);
    for (int i = 0; i < 3; ++i) X->ang[l][i] = pang[i] + w_rel[i];
    double anchor[3], d1[3], d2[3], c1[3], c2[3], sv[3];
    mbd_k64_rotate(jp, X->rot[l], t);
    for (int i = 0; i < 3; ++i) anchor[i] = X->pos[l][i] + t[i];
    for (int i = 0; i < 3; ++i) { d1[i] = X->pos[l][i] - ppos[i]; d2[i] = X->pos[l][i] - anchor[i]; }
    mbd_k64_cross(pang, d1, c1);
    mbd_k64_cross(w_rel, d2, c2);
    mbd_k64_rotate(svel, trot, sv);
    for (int i = 0; i < 3; ++i) X->vel[l][i] = pvel[i] + c1[i] + c2[i] + sv[i];
  }
}

/* kinematics.pipeline_init: q, qd (float32) -> state rows [nsim][13] (float32, rounded once) */
MBD_K64 void mbd_k64_pipeline_init(const double* T, const float* qf, const float* qdf, float* state) {
  double q[MBD_K64_MAXQ], qd[MBD_K64_MAXQ];
  const int nq = mbd_k64_i(T, 1), nqd = mbd_k64_i(T, 2), nsim = mbd_k64_i(T, 3);
  for (int j = 0; j < nq; ++j) q[j] = (double)qf[j];
  for (int j = 0; j < nqd; ++j) qd[j] = (double)qdf[j];
  mbd_k64_world X;
  mbd_k64_forward(T, q, qd, &X);
  for (int i = 0; i < nsim; ++i) {
    const int l = mbd_k64_i(T, MBD_K64_SIM + i);
    double rc[3], c[3];
    mbd_k64_rotate(mbd_k64_lf(T, l, MBD_K64_L_COM), X.rot[l], rc);
    mbd_k64_cross(X.ang[l], rc, c);
    float* o = state + i * 13;
    for (int k = 0; k < 3; ++k) o[k] = (float)(X.pos[l][k] + rc[k]);
    for (int k = 0; k < 4; ++k) o[3 + k] = (float)X.rot[l][k];
    for (int k = 0; k < 3; ++k) o[7 + k] = (float)X.ang[l][k];
    for (int k = 0; k < 3; ++k) o[10 + k] = (float)(X.vel[l][k] + c[k]);
  }
}

/* float32 world frames of all links from the state rows (PipelineEnv._make_pipeline_state): to_world of the simulated links,
 * rounded to float32; cosmetic links at their float32 init pose with zero motion.  Stored widened to float64. */
MBD_K64 void mbd_k64_world_of(const double* T, const float* state, mbd_k64_world* X) {
  const int L = mbd_k64_i(T, 0);
  for (int l = 0; l < L; ++l) {
    const int si = (int)*mbd_k64_lf(T, l, MBD_K64_L_SIMIDX);
    if (si < 0) {
      for (int k = 0; k < 3; ++k) { X->pos[l][k] = mbd_k64_lf(T, l, MBD_K64_L_SPOS)[k]; X->ang[l][k] = 0.0; X->vel[l][k] = 0.0; }
      for (int k = 0; k < 4; ++k) X->rot[l][k] = mbd_k64_lf(T, l, MBD_K64_L_SROT)[k];
      continue;
    }
    const float* s = state + si * 13;
    double p[3], r[4], w[3], v[3], rc[3], c[3];
    for (int k = 0; k < 3; ++k) { p[k] = s[k]; w[k] = s[7 + k]; v[k] = s[10 + k]; }
    for (int k = 0; k < 4; ++k) r[k] = s[3 + k];
    mbd_k64_rotate(mbd_k64_lf(T, l, MBD_K64_L_COM), r, rc);
    mbd_k64_cross(rc, w, c);
    for (int k = 0; k < 3; ++k) {
      X->pos[l][k] = (double)(float)(p[k] - rc[k]);
      X->vel[l][k] = (double)(float)(v[k] + c[k]);
      X->ang[l][k] = w[k];
    }
    for (int k = 0; k < 4; ++k) X->rot[l][k] = r[k];
  }
}

/* kinematics.inverse on the float32 world frames X: q [nq], qd [nqd] (float32, rounded once) */
MBD_K64 void mbd_k64_inverse(const double* T, const mbd_k64_world* X, float* qo, float* qdo) {
  const int nq = mbd_k64_i(T, 1), nqd = mbd_k64_i(T, 2), nsim = mbd_k64_i(T, 3);
  for (int j = 0; j < nq; ++j) qo[j] = (float)T[MBD_K64_INITQ + j];
  for (int j = 0; j < nqd; ++j) qdo[j] = 0.0f;
  const double zero3[3] = {0.0, 0.0, 0.0}, one4[4] = {1.0, 0.0, 0.0, 0.0};
  for (int i = 0; i < nsim; ++i) {
    const int l = mbd_k64_i(T, MBD_K64_SIM + i);
    const int type = (int)*mbd_k64_lf(T, l, MBD_K64_L_TYPE);
    const int qs = (int)*mbd_k64_lf(T, l, MBD_K64_L_QS), ds = (int)*mbd_k64_lf(T, l, MBD_K64_L_DS);
    if (type < 0) {
      for (int k = 0; k < 3; ++k) { qo[qs + k] = (float)X->pos[l][k]; qdo[ds + k] = (float)X->vel[l][k]; qdo[ds + 3 + k] = (float)X->ang[l][k]; }
      for (int k = 0; k < 4; ++k) qo[qs + 3 + k] = (float)X->rot[l][k];
      continue;
    }
    const int par = (int)*mbd_k64_lf(T, l, MBD_K64_L_PARENT);
    const double* prot = par >= 0 ? X->rot[par] : one4;
    const double* pang = par >= 0 ? X->ang[par] : zero3;
    const double* ppos = par >= 0 ? X->pos[par] : zero3;
    const double* lrot = mbd_k64_lf(T, l, MBD_K64_L_ROT);
    const double* jrot = mbd_k64_lf(T, l, MBD_K64_L_JROT);
    double t4[4], a_p[4], a_c[4], j[4];
    mbd_k64_qmul(prot, lrot, t4);
    mbd_k64_qmul(t4, jrot, a_p);
    mbd_k64_qmul(X->rot[l], jrot, a_c);
    const double a_pc[4] = {a_p[0], -a_p[1], -a_p[2], -a_p[3]};
    mbd_k64_qmul(a_pc, a_c, j);
    const double w = j[0], x = j[1], y = j[2], z = j[3];
    const double r00 = 1.0 - 2.0 * (y * y + z * z), r01 = 2.0 * (x * y - w * z), r02 = 2.0 * (x * z + w * y);
    const double r12 = 2.0 * (y * z - w * x), r22 = 1.0 - 2.0 * (x * x + y * y);
    const double ps = *mbd_k64_lf(T, l, MBD_K64_L_PARITY);
    const double ang[3] = {atan2(-r12, r22), atan2(r02, hypot(r00, r01)), ps * atan2(-r01, r00)};
    double lon[3] = {0.0, r22, -r12};
    const double ln = mbd_k64_norm(lon, 3) + 1e-30;
    for (int k = 0; k < 3; ++k) lon[k] = lon[k] / ln;
    const double axes[3][3] = {{1.0, 0.0, 0.0}, {lon[0], lon[1], lon[2]}, {ps * r02, ps * r12, ps * r22}};
    double dw[3], jd[3];
    // the host subtracts two float32 arrays here (xang[l] - xang[par]): a float32 difference
    for (int k = 0; k < 3; ++k) dw[k] = par >= 0 ? (double)((float)X->ang[l][k] - (float)pang[k]) : X->ang[l][k];
    mbd_k64_rotate(dw, a_pc, jd);
    // slide dofs: coordinate along the fixed parent-side axis
    double trot[4], t3[3], t3b[3], anchor_p[3], rcw[3], d[3], va[3], c[3];
    mbd_k64_qmul(prot, lrot, trot);
    const double* jp = mbd_k64_lf(T, l, MBD_K64_L_JPOS);
    mbd_k64_rotate(jp, lrot, t3);
    for (int k = 0; k < 3; ++k) t3[k] = mbd_k64_lf(T, l, MBD_K64_L_POS)[k] + t3[k];
    mbd_k64_rotate(t3, prot, t3b);
    for (int k = 0; k < 3; ++k) anchor_p[k] = ppos[k] + t3b[k];
    mbd_k64_rotate(jp, X->rot[l], rcw);
    for (int k = 0; k < 3; ++k) d[k] = X->pos[l][k] + rcw[k] - anchor_p[k];
    mbd_k64_cross(X->ang[l], rcw, c);
    for (int k = 0; k < 3; ++k) va[k] = X->vel[l][k] + c[k];
    for (int k = 0; k < type; ++k) {
      const double* dof = T + MBD_K64_DOF + (ds + k) * MBD_K64_DS;
      if (dof[3] != 0.0) {
        double aw[3];
        mbd_k64_rotate(dof, trot, aw);
        qo[qs + k] = (float)(dof[4] + mbd_k64_dot(d, aw));
        qdo[ds + k] = (float)mbd_k64_dot(va, aw);
        continue;
      }
      qo[qs + k] = (float)(ang[k] + dof[4]);
      qdo[ds + k] = (float)mbd_k64_dot(axes[k], jd);
    }
  }
}

#endif /* MBD_KIN64_H_ */
