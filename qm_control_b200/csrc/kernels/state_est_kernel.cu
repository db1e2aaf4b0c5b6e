// Sensor readings of the plant and the base state estimator that turns them into the controller's measurement (DESIGN.md §4.6).
//
// read_sensors_kernel, one thread per robot: QMHWSim::readSim's IMU block and joint handles restated on the plant state.  The IMU link sits at the base
// origin with the base's axes (robot.urdf unitree_imu), so with R = R(zyx) and the world angular velocity w = T(zyx) zyx_rates
//   quat   R exp([n_o]x) as xyzw                    gyro   R^T w + n_g          accel  R^T ((v_lin - v_prev_lin) / dt - g) + n_a,  g = (0, 0, -9.81)
//   joint  q[6:24] + n_q, v[6:24] + n_v
// The accelerometer reads the mean acceleration over the step, which under the plant's semi-implicit Euler substeps is exactly the velocity change the
// filter's prediction integrates.  Every noise term is sigma * sensor_normal(seed, robot, sample, channel); a zero sigma adds nothing.
//
// state_est_step_kernel, one warp per robot: a linear Kalman filter on x = [p_base, v_base, p_foot(4)] (world frame).  Per call:
//   attitude     R and zyx (yaw in (-pi, pi]) from the quaternion, w = R gyro: taken as measured, not filtered
//   legs         rbd_kinematics<true> at q = [0, zyx, joints], v = [0, T^-1 w, joint rates]: each foot's offset r_i from the base and its velocity
//                rd_i in world axes with the base translation removed, and the end-effector pose relative to the base
//   predict      p += v dt + a dt^2 / 2, v += a dt with a = R accel + g, feet constant; P = A P A^T + dt diag(q), a swing foot's q scaled by swing_scale
//   update       28 rows y = C x + noise: p - p_foot_i = -r_i (3 per foot), v = -rd_i (3 per foot), p_foot_i,z = foot_height (1 per foot), a swing
//                foot's variances scaled by swing_scale.  Every row of C is +1 at column a_r and -1 at column b_r (or nothing), so P C^T and
//                S = C P C^T + R are gathered from P by index; S by the warp Cholesky, K = P C^T S^-1 (one lane per row of K), x += K (y - C x),
//                P -= K C P symmetrised
//   ground map   (optional, per robot a tile of the plant's library and its origin) foot f's height row becomes h_f(x) = p_f,z - H(p_f,x, p_f,y) =
//                s_f c with c = foot_height - ground_height and s_f = sqrt(1 + gx_f^2 + gy_f^2): the plant holds a stance sphere centre at r - delta
//                along the normal of the local tangent plane.  H, g = (gx, gy) and s come from ground_at (sim_api.cuh) at the predicted foot xy,
//                and the row of C gains -gx_f, -gy_f at p_f,x, p_f,y; G = P C^T and S pick up those two terms, K and the updates are unchanged.
//                A tile of -1 is the plane row.
// The first call after a reset only places the feet at p + r_i.  rbd_est[55] = [zyx, p, joints, w, v, joint rates, end-effector pose].
// status: QMB200_ST_NAN for a non-finite input (nothing is written) or update (x and P are kept); QMB200_ST_NOT_PD when S fails the Cholesky (x and P are
// kept).  rbd_est is written in both of the last two cases, from the kept state.
//
// slip_step_kernel, one warp per robot, between the sensor reading (and the attitude filter) and the estimator step: the legs as the estimator reads
// them (read_legs), then for each foot f in contact u_f = v- + rd_f, the world velocity of the foot point under the estimator's prior v- = v_hat + a dt,
// and d^2_f = u_f^T (P_vv + dt process_base_vel 1 + meas_slip 1)^-1 u_f.  A foot becomes slipping when d^2_f > gate and is trusted again after hold
// consecutive calls with d^2_f < release; a foot out of contact is cleared.  stance = contact & ~slip is the mask the estimator step reads in place of
// contact, so a slipping foot is handled as a swing foot.  Before the estimator's first call after its reset (SE_N = 0) and on a non-finite reading
// (QMB200_ST_NAN) the contact mask passes through and the detector's state is untouched.
#include "state_est_api.cuh"
#include <type_traits>

#include "slip_api.cuh"
#include "rbd.cuh"
#include "wlinalg.cuh"

namespace qmb {

namespace {
constexpr int SE_WARPS = 2;   // robots per CTA
constexpr int SE_STRI = SE_NY * (SE_NY + 1) / 2;

struct SeWs {
  RbdWs rb;
  double q[NQ], v[NQ];
  double x[SE_NX], P[SE_TRI];
  double r[4][3], rd[4][3];   // foot offsets from the base and their velocities (world axes)
  double ee[7];               // end-effector position relative to the base (world axes) and orientation quat xyzw
  double a[3];                // base acceleration a = R accel + g (world)
  double G[SE_NX][SE_NY + 1]; // P C^T; rows padded to an odd number of doubles, so lanes walking their own row hit different banks
  double K[SE_NX][SE_NY + 1];
  double S[SE_STRI];          // C P C^T + R, packed lower, then its Cholesky factor
  double e[SE_NY];            // innovation y - C x
};
// with a ground map: per foot f the ground under its predicted position, (H_f, gx_f, gy_f, s_f = sqrt(1 + gx_f^2 + gy_f^2))
struct SeWsMap : SeWs {
  double hg[4][4];
};

// columns of measurement row r: +1 at a_r, -1 at b_r (b_r < 0: none)
__device__ __forceinline__ int col_a(int r) { return r < 12 ? r % 3 : (r < 24 ? 3 + (r - 12) % 3 : 6 + 3 * (r - 24) + 2); }
__device__ __forceinline__ int col_b(int r) { return r < 12 ? 6 + r : -1; }
__device__ __forceinline__ int row_foot(int r) { return r < 12 ? r / 3 : (r < 24 ? (r - 12) / 3 : r - 24); }
__device__ __forceinline__ double pk(const double* P, int i, int j) { return i >= j ? P[tri(i) + j] : P[tri(j) + i]; }
__device__ __forceinline__ double gpk(const double* P, int i, int j) { return j < 0 ? 0.0 : pk(P, i, j); }
// the row i of packed entry t: tri(i) <= t < tri(i + 1), from the root of i^2 + i = 2t and one integer correction for its rounding
__device__ __forceinline__ int tri_row(int t) {
  int i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  if (tri(i) > t) --i; else if (tri(i + 1) <= t) ++i;
  return i;
}

// The reading of one sensor row sn, shared by the estimator and the slip detector.  Lane 0: R and zyx from the quaternion, w = R gyro, a = R accel + g;
// lanes < NJ: the encoders; then rbd_kinematics<true> at q = [0, zyx, joints], v = [0, T^-1 w, joint rates] and, per foot f (lane f < 4), its offset
// r_f from the base and its velocity rd_f in world axes; with EE also the end-effector pose relative to the base (lane 4).  W: a warp workspace with
// rb, q, v, a, r, rd, a scratch e[>= 6] and, with EE, ee.  zyx and om: lane i < 3's euler angle and world angular velocity component.  Lanes 0..4 leave
// without a final __syncwarp: the caller syncs before it reads r, rd or ee from another lane.
template <bool EE, class W>
__device__ __forceinline__ void read_legs(const DevModel* __restrict__ mdl, const double* sn, W* w, int lane, double& zyx, double& om) {
  RbdWs* ws = &w->rb;
  if (lane == 0) {
    double qt[4] = {sn[SEN_QUAT], sn[SEN_QUAT + 1], sn[SEN_QUAT + 2], sn[SEN_QUAT + 3]};
    const double nn = 1.0 / sqrt(qt[0] * qt[0] + qt[1] * qt[1] + qt[2] * qt[2] + qt[3] * qt[3]);
    const double x = qt[0] * nn, y = qt[1] * nn, z = qt[2] * nn, qw = qt[3] * nn;
    const double R[9] = {1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * qw), 2.0 * (x * z + y * qw),
                         2.0 * (x * y + z * qw), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * qw),
                         2.0 * (x * z - y * qw), 2.0 * (y * z + x * qw), 1.0 - 2.0 * (x * x + y * y)};
    const double e[3] = {atan2(R[3], R[0]), asin(fmin(fmax(-R[6], -1.0), 1.0)), atan2(R[7], R[8])};
    const double gy[3] = {sn[SEN_GYRO], sn[SEN_GYRO + 1], sn[SEN_GYRO + 2]}, ac[3] = {sn[SEN_ACCEL], sn[SEN_ACCEL + 1], sn[SEN_ACCEL + 2]};
    double wv[3], a[3], T[9], Ti[9], ed[3]; matvec3(R, gy, wv); matvec3(R, ac, a); a[2] -= 9.81;
    euler_rate_map(e[0], e[1], T); inv3(T, Ti); matvec3(Ti, wv, ed);
    for (int i = 0; i < 3; ++i) { w->q[i] = 0.0; w->v[i] = 0.0; w->q[3 + i] = e[i]; w->v[3 + i] = ed[i]; w->a[i] = a[i]; w->e[i] = e[i]; w->e[3 + i] = wv[i]; }
  }
  if (lane < NJ) { w->q[6 + lane] = sn[SEN_JPOS + lane]; w->v[6 + lane] = sn[SEN_JVEL + lane]; }
  __syncwarp();
  if (lane < 3) { zyx = w->e[lane]; om = w->e[3 + lane]; }
  rbd_kinematics<true>(mdl, w->q, w->v, ws, lane);
  if (lane < 4) {
    const int f = lane;
    double pw[3], vel[3]; foot_point(mdl, ws, f, pw); point_vel(ws->V[mdl->foot_body[f]], pw, vel);
    for (int k = 0; k < 3; ++k) { w->r[f][k] = pw[k]; w->rd[f][k] = vel[k]; }
  }
  if constexpr (EE) {
    if (lane == 4) {
      double pe[3], Re[9]; ee_pose(mdl, ws, pe, Re);
      for (int k = 0; k < 3; ++k) w->ee[k] = pe[k];
      rot_to_quat_xyzw(Re, w->ee + 3);
    }
  }
}

constexpr int SL_WARPS = 4;   // robots per CTA of the slip detector
struct SlWs {
  RbdWs rb;
  double q[NQ], v[NQ];
  double r[4][3], rd[4][3];   // foot offsets from the base and their velocities (world axes)
  double a[3];                // base acceleration a = R accel + g (world)
  double e[6];                // read_legs' scratch
};
}  // namespace

__global__ void read_sensors_kernel(qmb200_sensor_params prm, int B, int64_t robot0, double dt, int64_t sample, const double* __restrict__ q,
                                    const double* __restrict__ v, const double* __restrict__ v_prev, double* __restrict__ sensors) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* qb = q + (size_t)b * NQ; const double* vb = v + (size_t)b * NQ; const double* vp = v_prev + (size_t)b * NQ;
  double* out = sensors + (size_t)b * QMB200_SENSORS;
  const uint64_t seed = prm.seed, robot = (uint64_t)(robot0 + b), smp = (uint64_t)sample;
  double R[9], T[9]; rot_zyx(qb[3], qb[4], qb[5], R); euler_rate_map(qb[3], qb[4], T);
  const double ed[3] = {vb[3], vb[4], vb[5]}; double om[3], gyro[3]; matvec3(T, ed, om); matTvec3(R, om, gyro);
  const double aw[3] = {(vb[0] - vp[0]) / dt, (vb[1] - vp[1]) / dt, (vb[2] - vp[2]) / dt + 9.81}; double acc[3]; matTvec3(R, aw, acc);
  if (prm.sigma_orientation > 0.0) {   // R exp([n]x), Rodrigues
    double n[3]; for (int i = 0; i < 3; ++i) n[i] = prm.sigma_orientation * sensor_normal(seed, robot, smp, CH_ORI + i);
    const double th = sqrt(dot3(n, n));
    if (th > 0.0) {
      const double s = sin(th) / th, c = (1.0 - cos(th)) / (th * th);
      const double E[9] = {1.0 - c * (n[1] * n[1] + n[2] * n[2]), c * n[0] * n[1] - s * n[2], c * n[0] * n[2] + s * n[1],
                           c * n[0] * n[1] + s * n[2], 1.0 - c * (n[0] * n[0] + n[2] * n[2]), c * n[1] * n[2] - s * n[0],
                           c * n[0] * n[2] - s * n[1], c * n[1] * n[2] + s * n[0], 1.0 - c * (n[0] * n[0] + n[1] * n[1])};
      double Rn[9]; matmul3(R, E, Rn); for (int i = 0; i < 9; ++i) R[i] = Rn[i];
    }
  }
  rot_to_quat_xyzw(R, out + SEN_QUAT);
  for (int i = 0; i < 3; ++i) {
    out[SEN_GYRO + i] = prm.sigma_gyro > 0.0 ? gyro[i] + prm.sigma_gyro * sensor_normal(seed, robot, smp, CH_GYRO + i) : gyro[i];
    out[SEN_ACCEL + i] = prm.sigma_accel > 0.0 ? acc[i] + prm.sigma_accel * sensor_normal(seed, robot, smp, CH_ACCEL + i) : acc[i];
  }
  for (int j = 0; j < NJ; ++j) {
    out[SEN_JPOS + j] = prm.sigma_joint_pos > 0.0 ? qb[6 + j] + prm.sigma_joint_pos * sensor_normal(seed, robot, smp, CH_JPOS + j) : qb[6 + j];
    out[SEN_JVEL + j] = prm.sigma_joint_vel > 0.0 ? vb[6 + j] + prm.sigma_joint_vel * sensor_normal(seed, robot, smp, CH_JVEL + j) : vb[6 + j];
  }
}

// MAP: compiled once with the ground map's foot-height rows and once for the plane alone (map.robot == NULL), which keeps the plane's code as it was.
template <bool MAP>
__global__ void __launch_bounds__(32 * SE_WARPS) state_est_step_kernel(const DevModel* __restrict__ mdl, qmb200_state_est_params prm, int B, double dt,
                                                                       const double* __restrict__ sensors, const int32_t* __restrict__ contact,
                                                                       double* __restrict__ state, double* __restrict__ rbd_est, int32_t* __restrict__ status,
                                                                       SimTerrain map, double ground_height) {
  using Ws = typename std::conditional<MAP, SeWsMap, SeWs>::type;
  __shared__ Ws s_ws[SE_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x * SE_WARPS + warp;
  if (b >= B) return;   // the whole warp leaves together
  Ws* w = &s_ws[warp];
  const double* sn = sensors + (size_t)b * QMB200_SENSORS; double* st = state + (size_t)b * SE_DBL; double* out = rbd_est + (size_t)b * QMB200_RBD;
  const double s0 = sn[lane], s1 = lane + 32 < QMB200_SENSORS ? sn[lane + 32] : 0.0;
  if (__any_sync(FULL, !(isfinite(s0) && isfinite(s1)))) { if (lane == 0) status[b] = QMB200_ST_NAN; return; }   // dt: checked by the API
  const int mask = contact[b];

  double zyx = 0.0, om = 0.0;   // lanes 0..2: this lane's euler angle and world angular velocity component
  read_legs<true>(mdl, sn, w, lane, zyx, om);
  if (lane < SE_NX) w->x[lane] = st[SE_X + lane];
  for (int t = lane; t < SE_TRI; t += 32) w->P[t] = st[SE_P + t];
  const double n_prev = st[SE_N];
  __syncwarp();

  int code = 0; bool commit = false;   // commit: x and P of the shared workspace replace the stored ones
  if (n_prev == 0.0) {   // first call after a reset: the feet where the legs put them
    if (lane < 12) w->x[6 + lane] = w->x[lane % 3] + w->r[lane / 3][lane % 3];
    commit = true;
  } else {
    // ---- predict: P = A P A^T + Q, A = [I dt I 0; 0 I 0; 0 0 I] ----
    double pn[6];
#pragma unroll
    for (int h = 0; h < 6; ++h) {
      const int t = lane + 32 * h; pn[h] = 0.0; if (t >= SE_TRI) continue;
      const int i = tri_row(t), j = t - tri(i);
      double p = w->P[t];
      if (i < 3) p += dt * pk(w->P, i + 3, j);
      if (j < 3) p += dt * pk(w->P, i, j + 3);
      if (i < 3 && j < 3) p += dt * dt * pk(w->P, i + 3, j + 3);
      if (i == j) {
        const double qv = i < 3 ? prm.process_base_pos : (i < 6 ? prm.process_base_vel : prm.process_foot * (contact_flag(mask, (i - 6) / 3) ? 1.0 : prm.swing_scale));
        p += dt * qv;
      }
      pn[h] = p;
    }
    double xn = 0.0;
    if (lane < SE_NX) xn = lane < 3 ? w->x[lane] + dt * w->x[lane + 3] + 0.5 * dt * dt * w->a[lane] : (lane < 6 ? w->x[lane] + dt * w->a[lane - 3] : w->x[lane]);
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 6; ++h) { const int t = lane + 32 * h; if (t < SE_TRI) w->P[t] = pn[h]; }
    if (lane < SE_NX) w->x[lane] = xn;
    __syncwarp();
    if constexpr (MAP) {   // the ground under each foot's predicted (= stored) position, from the plant's lookup
      if (lane < 4) {
        const int f = lane; double H, gx, gy;
        ground_at(map, map.robot + (size_t)b * 3, ground_height, w->x[6 + 3 * f], w->x[7 + 3 * f], H, gx, gy);
        w->hg[f][0] = H; w->hg[f][1] = gx; w->hg[f][2] = gy; w->hg[f][3] = sqrt(1.0 + gx * gx + gy * gy);
      }
      __syncwarp();
    }

    // ---- update: G = P C^T, S = C G + R, e = y - C x ----
    // With a map, height row 24 + f is h_f(x) = p_f,z - H(p_f,x, p_f,y) = s_f c, c = foot_height - ground_height: its row of C adds -gx_f at p_f,x and
    // -gy_f at p_f,y to the +1 at p_f,z.  A zero gradient and H = ground_height give the plane's numbers bit for bit.
    for (int t = lane; t < SE_NX * SE_NY; t += 32) {
      const int j = t / SE_NY, r = t % SE_NY;
      double g = pk(w->P, j, col_a(r)) - gpk(w->P, j, col_b(r));
      if constexpr (MAP) {
        if (r >= 24) { const int f = r - 24; g -= w->hg[f][1] * pk(w->P, j, 6 + 3 * f) + w->hg[f][2] * pk(w->P, j, 7 + 3 * f); }
      }
      w->G[j][r] = g;
    }
    if (lane < SE_NY) {
      const int r = lane, f = row_foot(r), a = col_a(r), bb = col_b(r);
      double yr = r < 12 ? -w->r[f][r % 3] : (r < 24 ? -w->rd[f][(r - 12) % 3] : prm.foot_height);
      if constexpr (MAP) {   // y_f - H_f = s_f c - H_f written so that H_f = ground_height, s_f = 1 leaves foot_height
        if (r >= 24) yr = prm.foot_height + (w->hg[f][0] - ground_height) + (w->hg[f][3] - 1.0) * (prm.foot_height - ground_height);
      }
      w->e[r] = yr - (w->x[a] - (bb < 0 ? 0.0 : w->x[bb]));
    }
    __syncwarp();
    for (int t = lane; t < SE_STRI; t += 32) {
      const int r = tri_row(t), c = t - tri(r), bb = col_b(r);
      double s = w->G[col_a(r)][c] - (bb < 0 ? 0.0 : w->G[bb][c]);
      if constexpr (MAP) {
        if (r >= 24) { const int f = r - 24; s -= w->hg[f][1] * w->G[6 + 3 * f][c] + w->hg[f][2] * w->G[7 + 3 * f][c]; }
      }
      if (r == c) s += (r < 12 ? prm.meas_foot_pos : (r < 24 ? prm.meas_foot_vel : prm.meas_foot_height)) * (contact_flag(mask, row_foot(r)) ? 1.0 : prm.swing_scale);
      w->S[t] = s;
    }
    __syncwarp();
    if (!w_cholesky(w->S, SE_NY, lane)) code = QMB200_ST_NOT_PD;
    __syncwarp();
    if (!code) {
      if (lane < SE_NX) {   // row lane of K = G S^-1: L L^T k = g
        double* k = w->K[lane];
        for (int r = 0; r < SE_NY; ++r) { double x = w->G[lane][r]; for (int c = 0; c < r; ++c) x -= w->S[tri(r) + c] * k[c]; k[r] = x / w->S[tri(r) + r]; }
        for (int r = SE_NY - 1; r >= 0; --r) { double x = k[r]; for (int c = r + 1; c < SE_NY; ++c) x -= w->S[tri(c) + r] * k[c]; k[r] = x / w->S[tri(r) + r]; }
      }
      __syncwarp();
      double xu = 0.0; bool bad = false;
      if (lane < SE_NX) { xu = w->x[lane]; for (int r = 0; r < SE_NY; ++r) xu += w->K[lane][r] * w->e[r]; bad = !isfinite(xu); }
#pragma unroll
      for (int h = 0; h < 6; ++h) {
        const int t = lane + 32 * h; if (t >= SE_TRI) continue;
        const int i = tri_row(t), j = t - tri(i);
        double kg = 0.0; for (int r = 0; r < SE_NY; ++r) kg += w->K[i][r] * w->G[j][r] + w->K[j][r] * w->G[i][r];
        pn[h] = w->P[t] - 0.5 * kg; bad = bad || !isfinite(pn[h]);
      }
      if (__any_sync(FULL, bad)) code = QMB200_ST_NAN;
      else {
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 6; ++h) { const int t = lane + 32 * h; if (t < SE_TRI) w->P[t] = pn[h]; }
        if (lane < SE_NX) w->x[lane] = xu;
        commit = true;
      }
    }
  }
  __syncwarp();
  if (commit) {
    if (lane < SE_NX) st[SE_X + lane] = w->x[lane];
    for (int t = lane; t < SE_TRI; t += 32) st[SE_P + t] = w->P[t];
  }
  // ---- the measurement the controller reads, from the stored state (lane i < 18 wrote st[i] itself) ----
  if (lane < 6) out[lane < 3 ? RBD_POS + lane : RBD_V + lane - 3] = st[SE_X + lane];
  if (lane < 3) { out[RBD_ZYX + lane] = zyx; out[RBD_W + lane] = om; }
  if (lane < NJ) { out[RBD_JPOS + lane] = w->q[6 + lane]; out[RBD_JVEL + lane] = w->v[6 + lane]; }
  if (lane < 7) out[RBD_EE_POS + lane] = lane < 3 ? w->ee[lane] + st[SE_X + lane] : w->ee[lane];   // position, then the quaternion at RBD_EE_QUAT
  if (lane == 0) { st[SE_N] = n_prev + 1.0; status[b] = code; }
}

__global__ void __launch_bounds__(32 * SL_WARPS) slip_step_kernel(const DevModel* __restrict__ mdl, qmb200_slip_params prm, double process_base_vel, int B,
                                                                  double dt, const double* __restrict__ sensors, const int32_t* __restrict__ contact,
                                                                  const double* __restrict__ se, double* __restrict__ state, int32_t* __restrict__ stance,
                                                                  int32_t* __restrict__ slip, int32_t* __restrict__ status) {
  __shared__ SlWs s_ws[SL_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x * SL_WARPS + warp;
  if (b >= B) return;   // the whole warp leaves together
  SlWs* w = &s_ws[warp];
  const double* sn = sensors + (size_t)b * QMB200_SENSORS; const double* sx = se + (size_t)b * SE_DBL; double* st = state + (size_t)b * SL_DBL;
  const int mask = contact[b];
  const double s0 = sn[lane], s1 = lane + 32 < QMB200_SENSORS ? sn[lane + 32] : 0.0;
  int code = 0;
  if (__any_sync(FULL, !(isfinite(s0) && isfinite(s1)))) code = QMB200_ST_NAN;
  if (code || sx[SE_N] == 0.0) {   // a non-finite reading, or the estimator's next call only places the feet: the contact mask passes through
    if (lane == 0) { stance[b] = mask; slip[b] = 0; status[b] = code; }
    return;
  }
  double zyx, om; read_legs<false>(mdl, sn, w, lane, zyx, om);
  __syncwarp();

  // ---- lane f < 4: d^2 of foot f's world velocity u = v- + rd_f under the prior N(v-, Sigma-) of the estimator's next prediction ----
  double d2 = 0.0; bool bad = false;
  if (lane < 4) {
    const int f = lane;
    double S[9], Si[9], u[3];
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) S[3 * i + j] = sx[SE_P + (i >= j ? tri(3 + i) + 3 + j : tri(3 + j) + 3 + i)];
      S[4 * i] += dt * process_base_vel + prm.meas_slip;
      u[i] = sx[SE_X + 3 + i] + dt * w->a[i] + w->rd[f][i];
    }
    inv3(S, Si);
    for (int i = 0; i < 3; ++i) d2 += u[i] * (Si[3 * i] * u[0] + Si[3 * i + 1] * u[1] + Si[3 * i + 2] * u[2]);
    bad = contact_flag(mask, f) && !isfinite(d2);
  }
  if (__any_sync(FULL, bad)) {   // not reached on a finite estimator state (Sigma >= meas_slip 1 > 0); the state is kept
    if (lane == 0) { stance[b] = mask; slip[b] = 0; status[b] = QMB200_ST_NAN; }
    return;
  }
  // ---- hysteresis: slipping above gate, trusted again after hold consecutive calls below release; a foot out of contact is cleared ----
  unsigned bit = 0u;
  if (lane < 4) {
    const int f = lane;
    bool sl = ((int)st[SL_MASK] >> (3 - f)) & 1; double hold = st[SL_HOLD + f], onset = st[SL_ONSET + f];
    if (!contact_flag(mask, f)) { sl = false; hold = 0.0; }
    else if (sl) {
      if (d2 < prm.release) { hold += 1.0; if (hold >= (double)prm.hold) { sl = false; hold = 0.0; } }
      else hold = 0.0;
    } else if (d2 > prm.gate) { sl = true; hold = 0.0; onset += 1.0; }
    st[SL_HOLD + f] = hold; st[SL_ONSET + f] = onset;
    bit = sl ? 1u << (3 - f) : 0u;
  }
  const int sm = (int)__reduce_or_sync(FULL, bit);
  if (lane == 0) { st[SL_MASK] = (double)sm; stance[b] = mask & ~sm; slip[b] = sm; status[b] = 0; }
}

int launch_slip_step(const DevModel* mdl, const qmb200_slip_params& prm, const qmb200_state_est_params& se_prm, int B, double dt, const double* sensors,
                     const int32_t* contact, const double* se, double* state, int32_t* stance, int32_t* slip, int32_t* status, cudaStream_t s) {
  slip_step_kernel<<<(B + SL_WARPS - 1) / SL_WARPS, 32 * SL_WARPS, 0, s>>>(mdl, prm, se_prm.process_base_vel, B, dt, sensors, contact, se, state, stance, slip, status);
  return 1;
}

int launch_read_sensors(const qmb200_sensor_params& prm, int B, int64_t robot0, double dt, int64_t sample, const double* q, const double* v, const double* v_prev,
                        double* sensors, cudaStream_t s) {
  read_sensors_kernel<<<(B + 127) / 128, 128, 0, s>>>(prm, B, robot0, dt, sample, q, v, v_prev, sensors);
  return 1;
}
int launch_state_est_step(const DevModel* mdl, const qmb200_state_est_params& prm, int B, double dt, const double* sensors, const int32_t* contact, double* state,
                          double* rbd_est, int32_t* status, const SimTerrain& map, double ground_height, cudaStream_t s) {
  const int grid = (B + SE_WARPS - 1) / SE_WARPS;
  if (map.robot) state_est_step_kernel<true><<<grid, 32 * SE_WARPS, 0, s>>>(mdl, prm, B, dt, sensors, contact, state, rbd_est, status, map, ground_height);
  else state_est_step_kernel<false><<<grid, 32 * SE_WARPS, 0, s>>>(mdl, prm, B, dt, sensors, contact, state, rbd_est, status, map, ground_height);
  return 1;
}

}  // namespace qmb
