// TEST INFRASTRUCTURE ONLY: the rigid-body side of the CPU twin of the payload estimator (qm_control_b200/csrc/kernels/payload_est_kernel.cu), on the
// oracle's own machinery (orc::compute_rbd: the composite-rigid-body mass matrix, the RNEA nonlinear effects and the end-effector frame Jacobian with its
// time derivative).  Everything else of the estimator (regressor, RLS, commit) is restated in numpy by tests/_payload_est_twin.py.
// Compiled by tests/_payload_est_twin.py together with oracle/src/model.cpp; the product never loads it.
#include <cstring>
#include <string>

#include "info.h"
#include "model.h"

using namespace orc;

namespace {
struct Twin { Model m; };
}  // namespace

extern "C" {

void* twin_est_create(const char* urdf, const char* task, const char* reference) {
  try {
    auto troot = info_parse_file(task); auto rroot = info_parse_file(reference);
    Mat djs = info_matrix(*rroot, "defaultJointState", NJ, 1); std::vector<double> dj(NJ); for (int i = 0; i < NJ; ++i) dj[i] = djs(i, 0);
    Twin* t = new Twin(); t->m = load_model(urdf, dj, troot->str("model_settings.eeFrame")); return t;
  } catch (...) { return nullptr; }
}
void twin_est_destroy(void* t) { delete static_cast<Twin*>(t); }

// the nominal model (no payload) at (q, v): M[24][24], nle[24], the end-effector frame Jacobian Jee[6][24] (rows: linear, angular; LOCAL_WORLD_ALIGNED) and its
// bias dJee v[6], the frame's origin, rotation (row-major), linear and angular velocity; effort[18] = the URDF effort limits
void twin_est_rbd(void* tp, const double* q, const double* v, double* M, double* nle, double* Jee, double* dJv, double* pos, double* rot, double* vel, double* angvel,
                  double* effort) {
  const Model& m = static_cast<Twin*>(tp)->m; RbdData d; compute_rbd(m, q, v, d, 1);
  for (int i = 0; i < NQ; ++i) { nle[i] = d.nle[i]; for (int j = 0; j < NQ; ++j) M[i * NQ + j] = d.M(i, j); }
  for (int i = 0; i < 6; ++i) { double s = 0.0; for (int j = 0; j < NQ; ++j) { Jee[i * NQ + j] = d.Jee(i, j); s += d.dJee(i, j) * v[j]; } dJv[i] = s; }
  for (int i = 0; i < 3; ++i) { pos[i] = d.ee_pos[i]; vel[i] = d.ee_vel[i]; angvel[i] = d.ee_angvel[i]; for (int j = 0; j < 3; ++j) rot[3 * i + j] = d.ee_rot(i, j); }
  for (int j = 0; j < NJ; ++j) effort[j] = m.joint[j].effort;
}

}  // extern "C"
