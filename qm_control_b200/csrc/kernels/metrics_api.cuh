// Host-visible interface of the per-episode metrics (metrics_kernel.cu): one accumulator row per robot that every plant step adds one sample to, and the
// close that turns it into the episode's row of QMB200_METRICS columns (include/qmb200.h: qmb200_metrics_*; DESIGN.md §4.13).
// The per-robot core is host + device: tests/metrics_host.cpp compiles it with g++ and checks it against a numpy statement of the column table.
#pragma once
#include <cuda_runtime.h>

#include "../../../include/qmb200.h"
#include "node_eval.cuh"
#include "sim_api.cuh"

namespace qmb {

constexpr int MT_DBL = 18;   // QMB200_METRICS: the columns of a closed episode's row (include/qmb200.h)
// The accumulator row [QMB200_METRICS_ACC] of one open episode; all zeros: open and empty.  The first sample fixes the start and the "previous" columns.
enum MetricsAcc : int {
  MA_N = 0,          // samples
  MA_DUR,            // sum of dt (s)
  MA_STATUS,         // OR of the status words, as a double
  MA_X0, MA_Y0,      // base xy of the first sample
  MA_X, MA_Y,        // base xy of the last sample
  MA_FEET,           // [4][2] foot frame xy of the last sample, contact order
  MA_CONTACT = MA_FEET + 8,   // contact mask of the last sample
  MA_PATH,           // sum of the planar base displacement between consecutive samples
  MA_MIN_H,          // min of p_z - H(p_x, p_y)
  MA_MAX_TILT,       // max of max(|pitch|, |roll|)
  MA_N_CMD,          // cmd_vel samples
  MA_VEL_SQ,         // sum over cmd_vel samples of the squared planar velocity error
  MA_YAW_SQ,         // ... of the squared yaw-rate error
  MA_EE_SQ,          // sum of |p_ee - p_ref|^2
  MA_EE_MAX,         // max of |p_ee - p_ref|
  MA_ORI_SQ,         // sum of the squared angle of q_ref^-1 q_ee
  MA_ENERGY,         // sum of |tau_j qd_j| dt
  MA_TAU_SQ,         // sum of sum_j tau_j^2 / 18
  MA_SLIP,           // sum of the planar displacement of feet in contact at both ends of a pair
  MA_TOUCHDOWNS,     // 0 -> 1 transitions of the four contact bits
  MA_N_EST,          // samples with an estimate
  MA_EST_POS_SQ,     // sum of |p_est - p|^2
  MA_EST_VEL_SQ,     // sum of |v_est - v|^2
  MA_DBL             // QMB200_METRICS_ACC
};
static_assert(MT_DBL == QMB200_METRICS && MA_DBL == QMB200_METRICS_ACC, "metrics layouts of include/qmb200.h");

// sin of an angle in [0, pi]: the slerp weights of target_pose through spawn_sincos, whose device path needs no stack
struct BoundedSin { QMB_HD double operator()(double x) const { double s, c; spawn_sincos(x, s, c); return s; } };

// One sample of robot b after a plant step into its accumulator row a: r its rbd [55], contact its mask, tau the effort held over the step [18], cmd its
// command [7] (cmd[3]: the yaw rate), cmd_vel whether its target is the cmd_vel stream, the target rows (nk knots of times tt and states ts [nk][37]),
// t the sample's time (the plant clock at the end of the step), status its word, est its estimate rbd_est [55] or NULL; trow its plant terrain row or NULL.
QMB_HD void metrics_sample(const DevModel& d, const SimTerrain& terrain, const double* trow, double ground_height, double dt, const double* r, int contact,
                           const double* tau, const double* cmd, bool cmd_vel, int nk, const double* tt, const double* ts, double t, uint32_t status,
                           const double* est, double* a) {
  const bool first = a[MA_N] == 0.0;
  a[MA_N] += 1.0; a[MA_DUR] += dt;
  a[MA_STATUS] = (double)((uint64_t)a[MA_STATUS] | (uint64_t)status);
  const double x = r[RBD_POS], y = r[RBD_POS + 1];
  double H, gx, gy; ground_at(terrain, trow, ground_height, x, y, H, gx, gy);
  const double h = r[RBD_POS + 2] - H, tilt = fmax(fabs(r[RBD_ZYX + 1]), fabs(r[RBD_ZYX + 2]));
  if (first) { a[MA_X0] = x; a[MA_Y0] = y; a[MA_MIN_H] = h; a[MA_MAX_TILT] = tilt; }
  else {
    const double dx = x - a[MA_X], dy = y - a[MA_Y]; a[MA_PATH] += sqrt(dx * dx + dy * dy);
    a[MA_MIN_H] = fmin(a[MA_MIN_H], h); a[MA_MAX_TILT] = fmax(a[MA_MAX_TILT], tilt);
  }
  a[MA_X] = x; a[MA_Y] = y;
  // the feet: planar slip of the feet in contact at both ends of the pair, then the new foot positions and mask
  const int prev = (int)a[MA_CONTACT], now = contact & 15;
  double Rb[9]; spawn_rot_zyx(r[RBD_ZYX], r[RBD_ZYX + 1], r[RBD_ZYX + 2], Rb);
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    double pf[3]; spawn_foot(d, r + RBD_JPOS, Rb, r + RBD_POS, f, pf);
    double* last = a + MA_FEET + 2 * f;
    if (!first && contact_flag(prev, f) && contact_flag(now, f)) { const double ux = pf[0] - last[0], uy = pf[1] - last[1]; a[MA_SLIP] += sqrt(ux * ux + uy * uy); }
    last[0] = pf[0]; last[1] = pf[1];
  }
  if (!first) { int on = now & ~prev; int c = 0; for (int f = 0; f < 4; ++f) c += (on >> f) & 1; a[MA_TOUCHDOWNS] += c; }
  a[MA_CONTACT] = now;
  // tracking: the planar velocity and the yaw rate against the cmd_vel target, the end-effector pose against the target trajectory at t
  if (cmd_vel) {
    const double ex = r[RBD_V] - ts[0], ey = r[RBD_V + 1] - ts[1], ew = r[RBD_W + 2] - cmd[3];
    a[MA_N_CMD] += 1.0; a[MA_VEL_SQ] += ex * ex + ey * ey; a[MA_YAW_SQ] += ew * ew;
  }
  {
    double pref[3], qref[4]; ne::target_pose(ne::target_segment(tt, ts, nk, t), nk, pref, qref, BoundedSin());
    const double* pe = r + RBD_EE_POS; const double* qe = r + RBD_EE_QUAT;   // xyzw
    const double e0 = pe[0] - pref[0], e1 = pe[1] - pref[1], e2 = pe[2] - pref[2], e2s = e0 * e0 + e1 * e1 + e2 * e2, en = sqrt(e2s);
    a[MA_EE_SQ] += e2s; a[MA_EE_MAX] = first ? en : fmax(a[MA_EE_MAX], en);
    // q_ref^-1 q_ee = (rw qw + rv.qv, rw qv - qw rv - rv x qv) with the conjugate as the inverse (atan2 takes the ratio, so the norm does not matter)
    const double* rv = qref; const double rw = qref[3]; double cr[3]; cross3(rv, qe, cr);
    const double w = rw * qe[3] + rv[0] * qe[0] + rv[1] * qe[1] + rv[2] * qe[2];
    const double v0 = rw * qe[0] - qe[3] * rv[0] - cr[0], v1 = rw * qe[1] - qe[3] * rv[1] - cr[1], v2 = rw * qe[2] - qe[3] * rv[2] - cr[2];
    const double ang = 2.0 * atan2(sqrt(v0 * v0 + v1 * v1 + v2 * v2), fabs(w));
    a[MA_ORI_SQ] += ang * ang;
  }
  // effort: joint power and torque
  double p = 0.0, s = 0.0;
  for (int j = 0; j < NJ; ++j) { const double tj = tau[j]; p += fabs(tj * r[RBD_JVEL + j]); s += tj * tj; }
  a[MA_ENERGY] += p * dt; a[MA_TAU_SQ] += s / NJ;
  if (est) {
    double ep = 0.0, ev = 0.0;
    for (int i = 0; i < 3; ++i) { const double u = est[RBD_POS + i] - r[RBD_POS + i], v = est[RBD_V + i] - r[RBD_V + i]; ep += u * u; ev += v * v; }
    a[MA_N_EST] += 1.0; a[MA_EST_POS_SQ] += ep; a[MA_EST_VEL_SQ] += ev;
  }
}

// The row [QMB200_METRICS] of the episode accumulated in a, closed for reason `end`.  A mean over no samples is NaN.
QMB_HD void metrics_finish(const double* a, int end, double* o) {
  const double n = a[MA_N], nc = a[MA_N_CMD], ne = a[MA_N_EST], nan = NAN;
  auto rms = [](double sum, double cnt) { return cnt > 0.0 ? sqrt(sum / cnt) : NAN; };
  const double dx = a[MA_X] - a[MA_X0], dy = a[MA_Y] - a[MA_Y0];
  o[0] = a[MA_DUR]; o[1] = end; o[2] = a[MA_STATUS];
  o[3] = n > 0.0 ? sqrt(dx * dx + dy * dy) : nan; o[4] = a[MA_PATH];
  o[5] = n > 0.0 ? a[MA_MIN_H] : nan; o[6] = n > 0.0 ? a[MA_MAX_TILT] : nan;
  o[7] = rms(a[MA_VEL_SQ], nc); o[8] = rms(a[MA_YAW_SQ], nc);
  o[9] = rms(a[MA_EE_SQ], n); o[10] = n > 0.0 ? a[MA_EE_MAX] : nan; o[11] = rms(a[MA_ORI_SQ], n);
  o[12] = a[MA_ENERGY]; o[13] = rms(a[MA_TAU_SQ], n); o[14] = a[MA_SLIP]; o[15] = a[MA_TOUCHDOWNS];
  o[16] = rms(a[MA_EST_POS_SQ], ne); o[17] = rms(a[MA_EST_VEL_SQ], ne);
}

// the inputs of one metrics_step launch (qmb200_metrics_step_dev); kind, rbd_est NULL as there
struct MetricsStep {
  double dt; const double *rbd, *effort, *cmd, *target_times, *target_states, *time, *rbd_est; const int32_t *contact, *kind, *n_target, *status; double* acc;
};
// robot b's sample of one launch: its rows of p, its plant terrain row, its knot count clamped to [1, QMB200_KMAX] as the MPC clamps it
QMB_HD void metrics_step_robot(const DevModel& d, const SimTerrain& terrain, double ground_height, const MetricsStep& p, int b) {
  const int n = p.n_target[b], nk = n < 1 ? 1 : (n > QMB200_KMAX ? QMB200_KMAX : n);
  metrics_sample(d, terrain, terrain.robot ? terrain.robot + (size_t)b * 3 : nullptr, ground_height, p.dt, p.rbd + (size_t)b * QMB200_RBD, p.contact[b],
                 p.effort + (size_t)b * NJ, p.cmd + (size_t)b * 7, !p.kind || p.kind[b] == QMB200_TARGET_CMD_VEL, nk, p.target_times + (size_t)b * QMB200_KMAX,
                 p.target_states + (size_t)b * QMB200_KMAX * QMB200_TARGET, p.time[b] + p.dt, (uint32_t)p.status[b],
                 p.rbd_est ? p.rbd_est + (size_t)b * QMB200_RBD : nullptr, p.acc + (size_t)b * MA_DBL);
}
// a masked robot's close: refused (nothing written) for an end outside {0, 1, 2}; else its row into out [n_episodes][QMB200_METRICS] at `episode`, or
// QMB200_ST_OVERFLOW in status when episode lies outside [0, n_episodes), and its accumulator row a zeroed
QMB_HD void metrics_close_robot(double* a, int end, int episode, int n_episodes, double* out, int32_t& status) {
  if (end < 0 || end > 2) return;
  if (episode >= 0 && episode < n_episodes) metrics_finish(a, end, out + (size_t)episode * MT_DBL);
  else status |= QMB200_ST_OVERFLOW;
#pragma unroll
  for (int i = 0; i < MA_DBL; ++i) a[i] = 0.0;
}

int launch_metrics_step(const DevModel* mdl, const SimTerrain& terrain, double ground_height, int B, const MetricsStep& p, cudaStream_t s);
// metrics_close_robot for every robot with mask[b] != 0 on out [B][n_episodes][QMB200_METRICS]
int launch_metrics_close(int B, const int32_t* mask, const int32_t* end, const int32_t* episode, int n_episodes, double* acc, double* out, int32_t* status,
                         cudaStream_t s);

}  // namespace qmb
