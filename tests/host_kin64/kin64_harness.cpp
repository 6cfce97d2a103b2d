// include/mbd_kin64.h built for the host (tests/test_vecenv_cpu.py): the float64 kinematics of the vector env's reset and epilogue.
#include "mbd_kin64.h"

extern "C" {
// kinematics.pipeline_init for n configurations: q [n][nq], qd [n][nqd] -> state [n][nsim][13]
int kin64_pipeline_init(const double* T, int n, const float* q, const float* qd, float* state) {
  const int nq = (int)T[1], nqd = (int)T[2], nsim = (int)T[3];
  for (int i = 0; i < n; ++i) mbd_k64_pipeline_init(T, q + i * nq, qd + i * nqd, state + i * nsim * 13);
  return 0;
}
// PipelineEnv._make_pipeline_state for n states: state [n][nsim][13] -> q [n][nq], qd [n][nqd], x.pos [n][L][3], x.rot [n][L][4]
int kin64_state(const double* T, int n, const float* state, float* q, float* qd, float* pos, float* rot) {
  const int L = (int)T[0], nq = (int)T[1], nqd = (int)T[2], nsim = (int)T[3];
  for (int i = 0; i < n; ++i) {
    mbd_k64_world X;
    mbd_k64_world_of(T, state + i * nsim * 13, &X);
    mbd_k64_inverse(T, &X, q + i * nq, qd + i * nqd);
    for (int l = 0; l < L; ++l) {
      for (int k = 0; k < 3; ++k) pos[(i * L + l) * 3 + k] = (float)X.pos[l][k];
      for (int k = 0; k < 4; ++k) rot[(i * L + l) * 4 + k] = (float)X.rot[l][k];
    }
  }
  return 0;
}
}
