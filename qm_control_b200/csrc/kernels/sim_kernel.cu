// Batched plant step: the physics Gazebo runs behind QMHWSim (qm_gazebo/src/QMHWSim.cpp), restated as forward dynamics of the 24-DoF tree with
// compliant foot-ground contact, so that the controller's joint efforts (qmb200_hw_write) turn into the next measured state rbd[55] on the device.
//
// One warp owns one robot (lanes over bodies / generalised coordinates, as in rbd.cuh).  One launch advances every robot by `substeps`
// semi-implicit Euler steps of length h with the effort held; q, v stay in shared memory between substeps.  Per substep, at (q, v):
//   M, nle                 rbd_kinematics<true> → rbd_inertias(gravity) → rbd_accumulate → rbd_mass_matrix_nle
//   contact (lanes 0..3)   foot sphere of radius r centred on the *_FOOT frame against the local tangent plane of the ground under its centre:
//                          height H and gradient (gx, gy) there (sim_api.cuh: ground_at; the plane z = ground: H = ground, g = 0),
//                          s = sqrt(1 + gx^2 + gy^2), normal n = (-gx, -gy, 1) / s, penetration delta = (H - (p_z - r s)) / s;
//                          F_n = max(0, k delta - d pdot.n) for delta > 0, else 0; v_t = pdot - (pdot.n) n;
//                          F = F_n n - v_t min(gamma, mu F_n / |v_t|) (regularised Coulomb).  The force acts at the sphere centre, so the
//                          sphere's rolling is not modelled: the contact point is the foot frame's point, not the lowest point of the sphere.
//                          With g = 0 every operation of the law reduces exactly (s = 1, r 1, / 1, n.pdot = pdot_z, v_t = (pdot_x, pdot_y, 0)),
//                          so flat ground, and a constant tile at height ground, give the plane law bit for bit.
//   Q                      [0_6; sat(effort) - damping .* qdot_j] + sum_f J_f^T F_f - nle      (J_f: point_jacobian of the foot frame)
//   solve                  M qddot = Q by the warp Cholesky (wlinalg.cuh); v += h qddot; q += h v
// After the last substep one kinematics-only pass at the final q gives the measured state rbd[55] (include/qmb200.h layout) with the
// end-effector pose as qm_estimation fills it from ground truth.
//
// Per-robot plant variation (each input optional: a NULL pointer is the same for the whole grid, so there is one code path):
//   mu[B]            the feet's Coulomb coefficient in place of prm.friction_mu
//   payload[B][8]    [m_ee, o_ee(3), m_base, o_base(3)]: point masses rigidly attached at o_ee (end-effector frame) and o_base (base frame).
//                    After rbd_inertias, lanes 0 / 1 add each one's spatial inertia about the world origin [m, m c, m(|c|^2 1 - c c^T)] to Ic and its
//                    RNEA force I_p (A + g) + V x* I_p V to F of the body it is fixed to, so M and nle include it through the existing passes.
//   wrench[B][12]    [f_base, n_base, f_ee, n_ee], world frame, each moment about its own frame's origin, held over the step: W = [n + p x f; f]
//                    about the world origin, Q_c += S_c . W over the base columns (base wrench) and the base + arm chain columns (EE wrench).
//   terrain          heightfield tile and origin per robot (SimTerrain); terrain.robot == NULL or tile -1 is the plane z = prm.ground_height
// A zero payload or wrench adds exact zeros and mu[b] == prm.friction_mu is the shared law, so neutral variation is bit-identical.
#include "payload.cuh"
#include "sim_api.cuh"
#include "wlinalg.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

namespace {
constexpr int SIM_WARPS = 2;   // robots per CTA: 2 x 15.2 KB of static shared memory
constexpr int NTRI = NQ * (NQ + 1) / 2;

struct SimWs {
  RbdWs rb;
  double q[NQ], v[NQ], nle[NQ], Q[NQ];
  double M[NQ * NQ];   // dense mass matrix; once packed into L it holds the four foot Jacobians (12 x 24)
  double L[NTRI];      // packed lower triangle of M, then its Cholesky factor
  double fc[4][3];     // contact force of each foot (world)
  double pf[4][3];     // foot frame origin (world)
  double W[2][6];      // external wrench [nO; f] about the world origin: [0] end effector, [1] base
};

// Lane 0: the end-effector frame, lane 1: the base frame.  Adds the payload point mass to Ic / F of the frame's body (payload.cuh) and writes the wrench about
// the world origin to w->W[lane] (sim_step_kernel's header has the layouts).
__device__ __forceinline__ void frame_loads(const DevModel* __restrict__ mdl, SimWs* w, int lane, const double* __restrict__ payload, const double* __restrict__ wrench) {
  RbdWs* ws = &w->rb; double R[9], po[3]; const int body = payload_frame(mdl, ws, lane, R, po);   // po: frame origin (world)
  if (payload) payload_add(mdl, ws, lane, body, R, po, payload, true);
  if (wrench) {
    const double f[3] = {wrench[0], wrench[1], wrench[2]}; double* W = w->W[lane];
    cross3(po, f, W); W[0] += wrench[3]; W[1] += wrench[4]; W[2] += wrench[5]; W[3] = f[0]; W[4] = f[1]; W[5] = f[2];
  }
}
}  // namespace

// TERRAIN: compiled once with the ground lookup and once for the plane alone (terrain.robot == NULL), which keeps the plane's register budget and its
// seven CTAs per SM; both run the same contact law, and the law gives the plane bit for bit at zero gradient.
template <bool TERRAIN>
__global__ void __launch_bounds__(32 * SIM_WARPS) sim_step_kernel(const DevModel* __restrict__ mdl, SimParams prm, int B, int substeps, double h,
                                                                  const double* __restrict__ effort /*[B][18]*/, double* __restrict__ q_io /*[B][24]*/,
                                                                  double* __restrict__ v_io /*[B][24]*/, double* __restrict__ rbd /*[B][55]*/,
                                                                  int32_t* __restrict__ contact, int32_t* __restrict__ status, const double* __restrict__ mu_b /*[B] or NULL*/,
                                                                  const double* __restrict__ payload /*[B][8] or NULL*/, const double* __restrict__ wrench /*[B][12] or NULL*/,
                                                                  SimTerrain terrain) {
  __shared__ SimWs s_ws[SIM_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x * SIM_WARPS + warp;
  if (b >= B) return;   // the whole warp leaves together
  SimWs* w = &s_ws[warp]; RbdWs* ws = &w->rb;
  double tau = 0.0, jdamp = 0.0;   // lane c >= 6: saturated effort and viscous damping of joint c - 6
  if (lane < NQ) { w->q[lane] = q_io[(size_t)b * NQ + lane]; w->v[lane] = v_io[(size_t)b * NQ + lane]; }
  if (lane >= 6 && lane < NQ) {
    const int j = lane - 6; const double lim = mdl->effort[j];
    tau = fmin(fmax(effort[(size_t)b * NJ + j], -lim), lim); jdamp = prm.joint_damping[j];
  }
  const double mu = mu_b ? mu_b[b] : prm.friction_mu;
  const double* pl = payload && lane < 2 ? payload + (size_t)b * 8 + 4 * lane : nullptr;      // lane 0: [m_ee, o_ee], lane 1: [m_base, o_base]
  const double* wr = wrench && lane < 2 ? wrench + (size_t)b * 12 + 6 * (1 - lane) : nullptr;  // lane 0: [f_ee, n_ee], lane 1: [f_base, n_base]
  const double* ter = terrain.robot ? terrain.robot + (size_t)b * 3 : nullptr;                   // [tile, origin_x, origin_y]
  const int je = mdl->ee_body - 1;
  const bool ee_col = lane < 6 || (lane - 6 >= mdl->chain_start[je] && lane - 6 <= je);   // columns of the EE's point_jacobian
  __syncwarp();
  int st = 0; unsigned in_contact = 0;
  for (int k = 0; k < substeps; ++k) {
    rbd_kinematics<true>(mdl, w->q, w->v, ws, lane);
    rbd_inertias(mdl, ws, lane, 1);
    if (payload || wrench) {
      if (lane < 2) frame_loads(mdl, w, lane, pl, wr);
      __syncwarp();
    }
    rbd_accumulate(mdl, ws, lane, true);
    rbd_mass_matrix_nle(mdl, ws, w->M, NQ, w->nle, lane);
    if (lane < NQ) { const double* row = w->M + lane * NQ; double* out = w->L + tri(lane); for (int c = 0; c <= lane; ++c) out[c] = row[c]; }
    double fn = 0.0;
    if (lane < 4) {
      const int f = lane;
      double pw[3], vel[3]; foot_point(mdl, ws, f, pw); point_vel(ws->V[mdl->foot_body[f]], pw, vel);
      double H = prm.ground_height, gx = 0.0, gy = 0.0;
      if (TERRAIN) ground_at(terrain, ter, prm.ground_height, pw[0], pw[1], H, gx, gy);
      const double s = sqrt(1.0 + gx * gx + gy * gy), n[3] = {-gx / s, -gy / s, 1.0 / s};
      const double pen = (H - (pw[2] - prm.foot_radius * s)) / s, vn = vel[0] * n[0] + vel[1] * n[1] + vel[2] * n[2];
      if (pen > 0.0) fn = fmax(0.0, prm.stiffness * pen - prm.damping * vn);
      const double t[3] = {vel[0] - vn * n[0], vel[1] - vn * n[1], vel[2] - vn * n[2]}, vt = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
      double F[3] = {0.0, 0.0, 0.0};
      if (fn > 0.0) {
        F[0] = fn * n[0]; F[1] = fn * n[1]; F[2] = fn * n[2];
        if (vt > 0.0) { const double c = fmin(prm.tangential_damping, mu * fn / vt); F[0] -= c * t[0]; F[1] -= c * t[1]; F[2] -= c * t[2]; }
      }
      w->fc[f][0] = F[0]; w->fc[f][1] = F[1]; w->fc[f][2] = F[2];
      w->pf[f][0] = pw[0]; w->pf[f][1] = pw[1]; w->pf[f][2] = pw[2];
    }
    const unsigned bal = __ballot_sync(FULL, lane < 4 && fn > 0.0);
    in_contact = ((bal & 1u) << 3) | ((bal & 2u) << 1) | ((bal & 4u) >> 1) | ((bal & 8u) >> 3);   // foot f → bit 3 - f (LF=8 RF=4 LH=2 RH=1)
    __syncwarp();
    for (int f = 0; f < 4; ++f) { const int j = mdl->foot_body[f] - 1; point_jacobian(ws, w->pf[f], mdl->chain_start[j], j, w->M + 3 * f * NQ, NQ, lane); }
    __syncwarp();
    if (lane < NQ) {
      double g = tau - jdamp * w->v[lane] - w->nle[lane];
#pragma unroll
      for (int f = 0; f < 4; ++f) g += w->M[(3 * f) * NQ + lane] * w->fc[f][0] + w->M[(3 * f + 1) * NQ + lane] * w->fc[f][1] + w->M[(3 * f + 2) * NQ + lane] * w->fc[f][2];
      if (wrench) {
        if (lane < 6) g += dot6(ws->S[lane], w->W[1]);
        if (ee_col) g += dot6(ws->S[lane], w->W[0]);
      }
      w->Q[lane] = g;
    }
    __syncwarp();
    if (!w_cholesky(w->L, NQ, lane)) { st |= QMB200_ST_NOT_PD; break; }
    w_chol_solve(w->L, NQ, w->Q, lane);
    if (lane < NQ) { const double vn = w->v[lane] + h * w->Q[lane]; w->v[lane] = vn; w->q[lane] += h * vn; }
    __syncwarp();
  }
  const bool bad = lane < NQ && !(isfinite(w->q[lane]) && isfinite(w->v[lane]));
  if (__any_sync(FULL, bad)) st |= QMB200_ST_NAN;
  rbd_kinematics<false>(mdl, w->q, w->v, ws, lane);
  double* r = rbd + (size_t)b * QMB200_RBD;
  if (lane < NQ) {
    q_io[(size_t)b * NQ + lane] = w->q[lane]; v_io[(size_t)b * NQ + lane] = w->v[lane];
    r[lane < 3 ? RBD_POS + lane : (lane < 6 ? RBD_ZYX + lane - 3 : RBD_JPOS + lane - 6)] = w->q[lane];
    if (lane < 3) r[RBD_V + lane] = w->v[lane]; else if (lane >= 6) r[RBD_JVEL + lane - 6] = w->v[lane];
  }
  if (lane == 0) {
    double T[9]; euler_rate_map_sc(ws->trig, T); const double ed[3] = {w->v[3], w->v[4], w->v[5]}; double om[3]; matvec3(T, ed, om);
    r[RBD_W] = om[0]; r[RBD_W + 1] = om[1]; r[RBD_W + 2] = om[2];                        // w_world = T(zyx) zyx_rates
    double pe[3], Re[9]; ee_pose(mdl, ws, pe, Re);
    r[RBD_EE_POS] = pe[0]; r[RBD_EE_POS + 1] = pe[1]; r[RBD_EE_POS + 2] = pe[2];
    rot_to_quat_xyzw(Re, r + RBD_EE_QUAT);
    contact[b] = (int32_t)in_contact; status[b] = st;
  }
}

int launch_sim_step(const DevModel* mdl, const SimParams& prm, int B, int substeps, double h, const double* effort, double* q, double* v, double* rbd, int32_t* contact,
                    int32_t* status, const double* mu, const double* payload, const double* wrench, const SimTerrain& terrain, cudaStream_t s) {
  const dim3 grid((B + SIM_WARPS - 1) / SIM_WARPS), block(32 * SIM_WARPS);
  if (terrain.robot) sim_step_kernel<true><<<grid, block, 0, s>>>(mdl, prm, B, substeps, h, effort, q, v, rbd, contact, status, mu, payload, wrench, terrain);
  else sim_step_kernel<false><<<grid, block, 0, s>>>(mdl, prm, B, substeps, h, effort, q, v, rbd, contact, status, mu, payload, wrench, terrain);
  return 1;
}

}  // namespace qmb
