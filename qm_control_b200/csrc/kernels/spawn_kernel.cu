// Per-episode spawns (include/qmb200.h: qmb200_spawn_sample_dev; DESIGN.md §4.12).
//   spawn_sample_kernel   one thread per robot: a masked robot draws its episode's spawn row (spawn_row, the host's core), moves its tile under it
//                         (the plant's robot terrain row and, linked, the estimator's ground map), stands on that ground (standing_on_tile, or the plane
//                         pose), and writes the state every consumer starts from: q, v = 0, the measured state rbd with the end-effector pose, the
//                         contact flags, the controller's observation, its held end-effector target turned with the base, and the reset rows of the
//                         estimators that run.  Unmasked robots are not written.
#include "spawn_api.cuh"
#include "state_est_api.cuh"
#include "attitude_api.cuh"
#include "slip_api.cuh"

namespace qmb {

namespace {
constexpr int SP_THREADS = 128;

__global__ void __launch_bounds__(SP_THREADS) spawn_sample_kernel(const DevModel* __restrict__ mdl, int B, const SpawnArgs a, const int32_t* __restrict__ mask,
                                                                  const int32_t* __restrict__ episode, double* __restrict__ rows, double* __restrict__ q,
                                                                  double* __restrict__ v, double* __restrict__ rbd, int32_t* __restrict__ contact,
                                                                  double* __restrict__ x_obs, double* __restrict__ last_ee, double* __restrict__ rbd_est) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  const DevModel& d = *mdl;
  double r[SP_DBL];
  spawn_row(a.lo + (size_t)b * SP_DBL, a.hi + (size_t)b * SP_DBL, a.seed, (uint64_t)(a.robot0 + b), (uint64_t)(int64_t)episode[b], r);
#pragma unroll
  for (int c = 0; c < SP_DBL; ++c) rows[(size_t)b * SP_DBL + c] = r[c];
  // the ground moves under the robot: the tile's origin is the run's minus the offset
  const double ter[3] = {r[SP_TILE], a.origin[2 * b] - r[SP_DX], a.origin[2 * b + 1] - r[SP_DY]};
  double* tr = a.ter.robot ? const_cast<double*>(a.ter.robot) + (size_t)b * 3 : nullptr;
  if (tr) { tr[0] = ter[0]; tr[1] = ter[1]; tr[2] = ter[2]; }
  if (a.ground) { double* g = a.ground + (size_t)b * 3; g[0] = ter[0]; g[1] = ter[1]; g[2] = ter[2]; }

  double* qb = q + (size_t)b * NQ;
  const double x = qb[0], y = qb[1], yaw0 = qb[3], yaw = r[SP_YAW];
  double z = a.z_plane, pitch = 0.0, roll = 0.0;
  if (tr && ter[0] >= 0.0) standing_on_tile(d, a.ter, ter, a.radius, a.delta0, a.qj, x, y, yaw, z, pitch, roll);
  const double base[6] = {x, y, z, yaw, pitch, roll};
#pragma unroll
  for (int i = 0; i < 6; ++i) qb[i] = base[i];
  for (int j = 0; j < NJ; ++j) qb[6 + j] = a.qj[j];
  for (int i = 0; i < NQ; ++i) v[(size_t)b * NQ + i] = 0.0;

  // the measured state at (q, 0), and the feet the plant's contact law presses into the ground there
  double Rb[9]; spawn_rot_zyx(yaw, pitch, roll, Rb);
  const double pb[3] = {x, y, z};
  double* s = rbd + (size_t)b * QMB200_RBD;
#pragma unroll
  for (int i = 0; i < 3; ++i) { s[RBD_ZYX + i] = base[3 + i]; s[RBD_POS + i] = base[i]; s[RBD_W + i] = 0.0; s[RBD_V + i] = 0.0; }
  for (int j = 0; j < NJ; ++j) { s[RBD_JPOS + j] = a.qj[j]; s[RBD_JVEL + j] = 0.0; }
  double pe[3], Re[9]; spawn_ee(d, a.qj, Rb, pb, pe, Re);
  s[RBD_EE_POS] = pe[0]; s[RBD_EE_POS + 1] = pe[1]; s[RBD_EE_POS + 2] = pe[2];
  rot_to_quat_xyzw(Re, s + RBD_EE_QUAT);
  int32_t in_contact = 0;
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    double pf[3], H = a.ground_height, gx = 0.0, gy = 0.0; spawn_foot(d, a.qj, Rb, pb, f, pf);
    if (tr) ground_at(a.ter, ter, a.ground_height, pf[0], pf[1], H, gx, gy);   // the plane where the plant has no terrain rows
    const double sc = sqrt(1.0 + gx * gx + gy * gy);
    if ((H - (pf[2] - a.radius * sc)) / sc > 0.0) in_contact |= 1 << (3 - f);   // foot f → bit 3 - f (LF=8 RF=4 LH=2 RH=1)
  }
  contact[b] = in_contact;
  // the observation: centroidal_from_rbd at rest, where w = v = 0 make both momentum rows exact zeros whatever the robot's SRBD constants
  double* xo = x_obs + (size_t)b * NX;
#pragma unroll
  for (int i = 0; i < 3; ++i) { xo[i] = 0.0; xo[3 + i] = 0.0; xo[6 + i] = base[i]; xo[9 + i] = base[3 + i]; }
  for (int j = 0; j < NJ; ++j) xo[12 + j] = a.qj[j];
  if (rbd_est) for (int i = 0; i < QMB200_RBD; ++i) rbd_est[(size_t)b * QMB200_RBD + i] = s[i];

  // the held end-effector target turns with the base about the vertical through it
  if (yaw != yaw0) {
    double* e = last_ee + (size_t)b * 7; const double dyaw = yaw - yaw0; double sn, c, sh, ch; spawn_sincos(dyaw, sn, c); spawn_sincos(0.5 * dyaw, sh, ch);
    const double ex = e[0] - x, ey = e[1] - y, qx = e[3], qy = e[4], qz = e[5], qw = e[6];
    e[0] = x + (c * ex - sn * ey); e[1] = y + (sn * ex + c * ey);
    e[3] = ch * qx - sh * qy; e[4] = ch * qy + sh * qx; e[5] = ch * qz + sh * qw; e[6] = ch * qw - sh * qz;   // Rz(dyaw) quaternion times e's
  }

  // the reset rows: the state estimator at the new base position with no call yet (its next call places the feet), the attitude filter, the detector
  if (a.se) state_est_reset_row(a.se_prm, base, a.se + (size_t)b * SE_DBL);   // base[0..2]: the base position
  if (a.at) attitude_reset_row(a.at_prm, a.at + (size_t)b * AT_DBL);
  if (a.sl) for (int i = 0; i < SL_DBL; ++i) a.sl[(size_t)b * SL_DBL + i] = 0.0;
}
}  // namespace

int launch_spawn_sample(const DevModel* mdl, int B, const SpawnArgs& a, const int32_t* mask, const int32_t* episode, double* rows, double* q, double* v, double* rbd,
                        int32_t* contact, double* x_obs, double* last_ee, double* rbd_est, cudaStream_t s) {
  spawn_sample_kernel<<<(B + SP_THREADS - 1) / SP_THREADS, SP_THREADS, 0, s>>>(mdl, B, a, mask, episode, rows, q, v, rbd, contact, x_obs, last_ee, rbd_est);
  return 1;
}

}  // namespace qmb
