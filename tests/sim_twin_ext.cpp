// TEST INFRASTRUCTURE ONLY: the CPU twin of the plant step with per-robot variation (qm_control_b200/csrc/kernels/sim_kernel.cu: mu[B],
// payload[B][8], wrench[B][12]), beside the plain twin of tests/sim_twin.cpp.  Same contact law and semi-implicit Euler integrator, on the oracle's own
// machinery (orc::compute_rbd, linalg.h's dense Cholesky), but the variation is reached by other means than the kernel's:
//   payload   each point mass is merged into the BodyDef of its frame's body (mass, COM, parallel-axis inertia) in a copy of the Model, which
//             compute_rbd then sees as the robot;  payload = [m_ee, o_ee(3), m_base, o_base(3)], offsets in model_settings.eeFrame / "base"
//   wrench    Q += Jbase^T [f; n] + Jee^T [f; n] with the LOCAL_WORLD_ALIGNED frame Jacobians;  wrench = [f_base, n_base, f_ee, n_ee] (world)
//   mu        the friction_mu of the params row
// Compiled by tests/_sim_twin_ext.py together with oracle/src/model.cpp; the product never loads it.
#include <cmath>
#include <cstring>
#include <string>

#include "info.h"
#include "model.h"

using namespace orc;

namespace {
struct Twin { Model m; };
// params: ground, radius, k, d, gamma, mu, joint_damping[18] (tests/_sim_twin.py's row)
struct Prm { double ground, radius, k, d, gamma, mu, jd[NJ]; };
Prm unpack(const double* p) { Prm o; o.ground = p[0]; o.radius = p[1]; o.k = p[2]; o.d = p[3]; o.gamma = p[4]; o.mu = p[5]; for (int j = 0; j < NJ; ++j) o.jd[j] = p[6 + j]; return o; }

// Eigen::Quaterniond(const Matrix3d&), out = x, y, z, w
void quat_xyzw(const M3<double>& R, double* o) {
  auto m = [&](int i, int j) { return R(i, j); };
  const double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0.0) { double s = std::sqrt(t + 1.0); o[3] = 0.5 * s; s = 0.5 / s; o[0] = (m(2, 1) - m(1, 2)) * s; o[1] = (m(0, 2) - m(2, 0)) * s; o[2] = (m(1, 0) - m(0, 1)) * s; return; }
  int i = 0; if (m(1, 1) > m(0, 0)) i = 1; if (m(2, 2) > m(i, i)) i = 2;
  const int j = (i + 1) % 3, k = (j + 1) % 3;
  double s = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0); o[i] = 0.5 * s; s = 0.5 / s;
  o[3] = (m(k, j) - m(j, k)) * s; o[j] = (m(j, i) + m(i, j)) * s; o[k] = (m(k, i) + m(i, k)) * s;
}

Model with_payload(const Model& m, const double* payload) {
  Model o = m; if (!payload) return o;
  for (int k = 0; k < 2; ++k) {
    const double mp = payload[4 * k]; if (mp == 0.0) continue;
    const FrameDef& fd = m.frames[k == 0 ? m.ee_frame : m.base_frame];
    const V3<double> c = fd.p + fd.R * V3<double>(payload[4 * k + 1], payload[4 * k + 2], payload[4 * k + 3]);   // in the body's frame
    BodyDef& b = o.body[fd.body]; const double mt = b.mass + mp; const V3<double> com = (1.0 / mt) * (b.mass * b.com + mp * c);
    const M3<double> Sb = skew(b.com - com), Sp = skew(c - com), Pb = transpose(Sb) * Sb, Pp = transpose(Sp) * Sp;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) b.I(i, j) += b.mass * Pb(i, j) + mp * Pp(i, j);
    b.mass = mt; b.com = com;
  }
  o.mass = total_mass(o); return o;
}

void saturate(const Model& m, const double* effort, double* tau) { for (int j = 0; j < NJ; ++j) tau[j] = std::min(std::max(effort[j], -m.joint[j].effort), m.joint[j].effort); }

// generalised acceleration at (q, v): false when M is not positive definite.  F12 = contact forces (world), mask = feet with F_n > 0.
bool accel(const Model& mdl, const Prm& p, const double* tau_sat, const double* wrench, const double* q, const double* v, double* qdd, double* F12, int* mask) {
  RbdData d; compute_rbd(mdl, q, v, d, 1);
  Vec Q(NQ, 0.0); *mask = 0;
  for (int f = 0; f < 4; ++f) {
    const double pen = p.ground - (d.foot_pos[f][2] - p.radius);
    double fn = 0.0; if (pen > 0.0) fn = std::max(0.0, p.k * pen - p.d * d.foot_vel[f][2]);
    const double vx = d.foot_vel[f][0], vy = d.foot_vel[f][1], vt = std::sqrt(vx * vx + vy * vy);
    double fx = 0.0, fy = 0.0; if (fn > 0.0 && vt > 0.0) { const double c = std::min(p.gamma, p.mu * fn / vt); fx = -c * vx; fy = -c * vy; }
    const double F[3] = {fx, fy, fn}; for (int i = 0; i < 3; ++i) F12[3 * f + i] = F[i];
    if (fn > 0.0) *mask |= 8 >> f;
    for (int c = 0; c < NQ; ++c) for (int i = 0; i < 3; ++i) Q[c] += d.Jfoot(3 * f + i, c) * F[i];
  }
  for (int c = 0; c < NQ; ++c) Q[c] -= d.nle[c];
  for (int j = 0; j < NJ; ++j) Q[6 + j] += tau_sat[j] - p.jd[j] * v[6 + j];
  if (wrench)
    for (int c = 0; c < NQ; ++c) for (int i = 0; i < 6; ++i) Q[c] += d.Jbase(i, c) * wrench[i] + d.Jee(i, c) * wrench[6 + i];
  Mat L; if (!cholesky(d.M, L)) return false;
  Mat x = chol_solve(L, col(Q)); for (int c = 0; c < NQ; ++c) qdd[c] = x(c, 0);
  return true;
}
}  // namespace

extern "C" {

void* twin_ext_create(const char* urdf, const char* task, const char* reference) {
  try {
    auto troot = info_parse_file(task); auto rroot = info_parse_file(reference);
    Mat djs = info_matrix(*rroot, "defaultJointState", NJ, 1); std::vector<double> dj(NJ); for (int i = 0; i < NJ; ++i) dj[i] = djs(i, 0);
    Twin* t = new Twin(); t->m = load_model(urdf, dj, troot->str("model_settings.eeFrame")); return t;
  } catch (...) { return nullptr; }
}
void twin_ext_destroy(void* t) { delete static_cast<Twin*>(t); }

// qdd[24], F12[12] and the contact mask of one substep's right-hand side; payload[8] / wrench[12] may be NULL; returns 0 / -1 (not PD)
int twin_accel_ext(void* tp, const double* params, const double* payload, const double* wrench, const double* effort, const double* q, const double* v, double* qdd, double* F12,
                   int* mask) {
  const Model m = with_payload(static_cast<Twin*>(tp)->m, payload); double tau[NJ]; saturate(m, effort, tau);
  return accel(m, unpack(params), tau, wrench, q, v, qdd, F12, mask) ? 0 : -1;
}

// `substeps` semi-implicit Euler steps of length h; q, v in-out; rbd[55], contact mask, status (4 = non-finite state, 8 = M not PD) out
void twin_step_ext(void* tp, const double* params, const double* payload, const double* wrench, int substeps, double h, const double* effort, double* q, double* v, double* rbd,
                   int* contact, int* status) {
  const Model m = with_payload(static_cast<Twin*>(tp)->m, payload); const Prm p = unpack(params);
  double tau[NJ]; saturate(m, effort, tau);
  int st = 0, mask = 0; double qdd[NQ], F[12];
  for (int k = 0; k < substeps; ++k) {
    if (!accel(m, p, tau, wrench, q, v, qdd, F, &mask)) { st |= 8; break; }
    for (int c = 0; c < NQ; ++c) { v[c] += h * qdd[c]; q[c] += h * v[c]; }
  }
  for (int c = 0; c < NQ; ++c) if (!std::isfinite(q[c]) || !std::isfinite(v[c])) st |= 4;
  RbdData d; compute_rbd(m, q, v, d, 0);
  rbd[0] = q[3]; rbd[1] = q[4]; rbd[2] = q[5]; rbd[3] = q[0]; rbd[4] = q[1]; rbd[5] = q[2];
  for (int j = 0; j < NJ; ++j) { rbd[6 + j] = q[6 + j]; rbd[30 + j] = v[6 + j]; }
  const M3<double> T = euler_rate_map<double>(q[3], q[4]); const V3<double> w = T * V3<double>(v[3], v[4], v[5]);
  for (int i = 0; i < 3; ++i) { rbd[24 + i] = w[i]; rbd[27 + i] = v[i]; rbd[48 + i] = d.ee_pos[i]; }
  quat_xyzw(d.ee_rot, rbd + 51);
  *contact = mask; *status = st;
}

// rigid-body quantities of the robot with its payload at (q, v): M[24][24], nle[24], Ag[6][24] (about the COM), dAg*v[6], com[3], total mass
void twin_rbd_ext(void* tp, const double* payload, const double* q, const double* v, double* M, double* nle, double* Ag, double* dAg_v, double* com, double* mass) {
  const Model m = with_payload(static_cast<Twin*>(tp)->m, payload); RbdData d; compute_rbd(m, q, v, d, 3);
  for (int i = 0; i < NQ; ++i) { nle[i] = d.nle[i]; for (int j = 0; j < NQ; ++j) M[i * NQ + j] = d.M(i, j); }
  for (int i = 0; i < 6; ++i) { dAg_v[i] = d.dAg_v[i]; for (int j = 0; j < NQ; ++j) Ag[i * NQ + j] = d.Ag(i, j); }
  for (int i = 0; i < 3; ++i) com[i] = d.com[i];
  *mass = m.mass;
}

}  // extern "C"
