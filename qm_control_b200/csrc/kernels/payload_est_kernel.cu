// Online estimate of the end-effector payload: per-robot recursive least squares on the arm rows of the nominal model (DESIGN.md §4.6).
//
// The six arm rows a (generalised coordinates 18..23) of the nominal model (no payload) leave a residual
//     y_a = M_nom[a, :] qdd + nle_nom[a] - sat(tau)_a
// that no foot contact enters (the feet's point Jacobians have zero arm columns) and no base payload enters (M[a, :] and nle[a] use only the arm subtree's
// composite quantities).  A load fixed to the end-effector frame enters it linearly in its ten inertial parameters in that frame about its origin,
// theta = [m, m c(3), I(6)]: the load needs the wrench [f; n] = Y(w, dw, a - g) theta at the frame origin (Newton-Euler, all in the frame's axes)
//     f = m a + dw x h + w x (w x h),   n = I dw + w x (I w) + h x a,   h = m c
// and y_a = -J_e,a^T [R f; R n] with the end-effector Jacobian's arm columns, so y = Phi theta with Phi = -J_e,a^T R Y (6 x 10).
//
// One warp owns one robot (lanes over bodies / columns, as in rbd.cuh and sim_kernel.cu).  Per call, from the measurement rbd [55] and the effort held over the
// interval of length dt that ended at it:
//   (q, v)      rbd → q, and v with euler rates = T(zyx)^-1 w_world (rbd_read, as the WBC's measured pass)
//   qdd         (v - v_prev) / dt, with the previous sample from the estimator state; M, nle, the end-effector twist and acceleration at the midpoint
//               state ((q + q_prev) / 2 with the euler difference unwrapped, (v + v_prev) / 2): rbd_kinematics<true> → rbd_inertias → rbd_accumulate →
//               rbd_mass_matrix_nle, then the end-effector body's acceleration A + sum_c S_c qdd_c
//   RLS         S = lambda 1 + Phi P Phi^T (warp Cholesky), K = P Phi^T S^-1, theta += K (y - Phi theta), P = (P - K Phi P) / lambda symmetrised, and scaled
//               down to trace_max when its trace exceeds it
// The first call after a reset only stores its sample.  status: QMB200_ST_NAN for a non-finite input (nothing is stored) or a non-finite update (theta and P are
// kept, the sample is stored); QMB200_ST_NOT_PD when S fails the Cholesky (theta and P are kept, the sample is stored).
#include "payload_est_api.cuh"
#include "rbd.cuh"
#include "wlinalg.cuh"

namespace qmb {

namespace {
constexpr int EST_WARPS = 2;   // robots per CTA

struct EstWs {
  RbdWs rb;
  double q[NQ], v[NQ], qdd[NQ], nle[NQ];
  double M[NQ * NQ];
  double kin[9];            // end-effector frame: angular velocity, angular acceleration, linear acceleration of the origin minus gravity (frame axes)
  double Re[9], pe[3];      // end-effector frame rotation and origin (world)
  double Phi[6][EST_NP], y[6], e[6];
  double P[EST_TRI], th[EST_NP];
  double G[EST_NP][6];      // P Phi^T
  double K[EST_NP][6];
  double S[21];             // lambda 1 + Phi P Phi^T, packed, then its Cholesky factor
};

// u^T I v for the symmetric I = (xx, xy, xz, yy, yz, zz) as the six coefficients of those parameters
__device__ __forceinline__ void bilinear6(const double* u, const double* v, double* o) {
  o[0] = u[0] * v[0]; o[1] = u[0] * v[1] + u[1] * v[0]; o[2] = u[0] * v[2] + u[2] * v[0];
  o[3] = u[1] * v[1]; o[4] = u[1] * v[2] + u[2] * v[1]; o[5] = u[2] * v[2];
}
__device__ __forceinline__ double packed(const double* P, int i, int j) { return i >= j ? P[tri(i) + j] : P[tri(j) + i]; }
}  // namespace

__global__ void __launch_bounds__(32 * EST_WARPS) payload_est_step_kernel(const DevModel* __restrict__ mdl, qmb200_payload_est_params prm, int B, double dt,
                                                                          const double* __restrict__ effort /*[B][18]*/, const double* __restrict__ rbd /*[B][55]*/,
                                                                          double* __restrict__ state /*[B][EST_DBL]*/, int32_t* __restrict__ status) {
  __shared__ EstWs s_ws[EST_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x * EST_WARPS + warp;
  if (b >= B) return;   // the whole warp leaves together
  EstWs* w = &s_ws[warp]; RbdWs* ws = &w->rb;
  const double* rb = rbd + (size_t)b * QMB200_RBD; double* st = state + (size_t)b * EST_DBL;

  // ---- the sample: q, v (euler rates) as the WBC's measured pass reads them ----
  rbd_read(rb, w->q, w->v, nullptr, lane);
  __syncwarp();
  double qk = 0.0, vk = 0.0, tau = 0.0;
  if (lane < NQ) { qk = w->q[lane]; vk = w->v[lane]; }
  if (lane >= 6 && lane < NQ) { const double lim = mdl->effort[lane - 6]; tau = fmin(fmax(effort[(size_t)b * NJ + lane - 6], -lim), lim); }
  const bool bad_in = (lane < NQ && !(isfinite(qk) && isfinite(vk))) || (lane >= 6 && lane < NQ && !isfinite(effort[(size_t)b * NJ + lane - 6]));
  if (__any_sync(FULL, bad_in)) { if (lane == 0) status[b] = QMB200_ST_NAN; return; }   // dt: checked by the API
  const double n_prev = st[EST_N];
  if (n_prev == 0.0) {   // first sample after a reset: store it
    if (lane < NQ) { st[EST_Q + lane] = qk; st[EST_V + lane] = vk; }
    if (lane == 0) { st[EST_N] = 1.0; status[b] = 0; }
    return;
  }

  // ---- finite-difference acceleration and the midpoint state ----
  if (lane < NQ) {
    const double qp = st[EST_Q + lane], vp = st[EST_V + lane];
    double dq = qk - qp;
    if (lane >= 3 && lane < 6) dq -= 6.283185307179586 * rint(dq * 0.15915494309189535);   // euler angles: the short way round
    w->q[lane] = qp + 0.5 * dq; w->v[lane] = 0.5 * (vk + vp); w->qdd[lane] = (vk - vp) / dt;
  }
  __syncwarp();
  rbd_kinematics<true>(mdl, w->q, w->v, ws, lane);
  rbd_inertias(mdl, ws, lane, 1);
  rbd_accumulate(mdl, ws, lane, true);
  rbd_mass_matrix_nle(mdl, ws, w->M, NQ, w->nle, lane);
  const int je = mdl->ee_body - 1, a0 = 6 + mdl->chain_start[je];   // arm columns [a0, 6 + je], the six rows of y
  if (lane >= a0 && lane <= 6 + je) {
    const double* row = w->M + lane * NQ; double acc = w->nle[lane] - tau;
    for (int c = 0; c < NQ; ++c) acc += row[c] * w->qdd[c];
    w->y[lane - a0] = acc;
  }
  if (lane == 0) {   // end-effector frame kinematics at the midpoint: pose, twist, acceleration with qdd
    const int eb = mdl->ee_body;
    double pe[3], Re[9]; ee_pose(mdl, ws, pe, Re);
    double Af[6]; for (int i = 0; i < 6; ++i) Af[i] = ws->A[eb][i];
    for (int c = 0; c <= 6 + je; ++c) {
      if (c >= 6 && c < a0) continue;
      const double qd = w->qdd[c]; for (int i = 0; i < 6; ++i) Af[i] += ws->S[c][i] * qd;
    }
    const double* V = ws->V[eb]; double vel[3], acc[3]; point_vel_acc(V, Af, pe, vel, acc);
    acc[2] += 9.81;                                           // a - g with g = -9.81 z (rbd_inertias' gravity)
    matTvec3(Re, V, w->kin); matTvec3(Re, Af, w->kin + 3); matTvec3(Re, acc, w->kin + 6);
    for (int i = 0; i < 9; ++i) w->Re[i] = Re[i];
    w->pe[0] = pe[0]; w->pe[1] = pe[1]; w->pe[2] = pe[2];
  }
  if (lane < EST_TRI) w->P[lane] = st[EST_P + lane];
  if (lane + 32 < EST_TRI) w->P[lane + 32] = st[EST_P + lane + 32];
  if (lane < EST_NP) w->th[lane] = st[EST_THETA + lane];
  __syncwarp();

  // ---- regressor rows: Phi[r] = -(J_v^T f + J_w^T n) per unit parameter, with the column's end-effector Jacobian in the frame's axes ----
  if (lane >= a0 && lane <= 6 + je) {
    const double* S = ws->S[lane]; double jv[3]; point_vel(S, w->pe, jv);
    double wf[3], wn[3]; matTvec3(w->Re, jv, wf); matTvec3(w->Re, S, wn);
    const double* om = w->kin; const double* al = w->kin + 3; const double* a = w->kin + 6;
    double* phi = w->Phi[lane - a0];
    phi[0] = -dot3(wf, a);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double e[3] = {i == 0 ? 1.0 : 0.0, i == 1 ? 1.0 : 0.0, i == 2 ? 1.0 : 0.0};
      double t1[3], t2[3], f[3], n[3]; cross3(al, e, f); cross3(om, e, t1); cross3(om, t1, t2); f[0] += t2[0]; f[1] += t2[1]; f[2] += t2[2]; cross3(e, a, n);
      phi[1 + i] = -(dot3(wf, f) + dot3(wn, n));
    }
    double u[3], c1[6], c2[6]; cross3(wn, om, u); bilinear6(wn, al, c1); bilinear6(u, om, c2);   // wn.(I al) + wn.(om x I om) = wn^T I al + (wn x om)^T I om
#pragma unroll
    for (int i = 0; i < 6; ++i) phi[4 + i] = -(c1[i] + c2[i]);
  }
  __syncwarp();

  // ---- RLS ----
  const double lam = prm.forgetting;
  for (int t = lane; t < EST_NP * 6; t += 32) {   // G = P Phi^T
    const int i = t / 6, r = t % 6; double g = 0.0;
    for (int j = 0; j < EST_NP; ++j) g += packed(w->P, i, j) * w->Phi[r][j];
    w->G[i][r] = g;
  }
  __syncwarp();
  if (lane < 21) {   // S = lambda 1 + Phi G, packed lower
    int r = 0; while (tri(r + 1) <= lane) ++r; const int c = lane - tri(r);
    double s = r == c ? lam : 0.0; for (int j = 0; j < EST_NP; ++j) s += w->Phi[r][j] * w->G[j][c];
    w->S[lane] = s;
  }
  if (lane >= 24 && lane < 30) { const int r = lane - 24; double p = w->y[r]; for (int j = 0; j < EST_NP; ++j) p -= w->Phi[r][j] * w->th[j]; w->e[r] = p; }
  __syncwarp();
  int code = 0;
  if (!w_cholesky(w->S, 6, lane)) code = QMB200_ST_NOT_PD;
  __syncwarp();
  if (!code) {
    if (lane < EST_NP) {   // row i of K = G S^-1: L L^T k = g
      double k[6]; for (int r = 0; r < 6; ++r) k[r] = w->G[lane][r];
      for (int r = 0; r < 6; ++r) { double x = k[r]; for (int c = 0; c < r; ++c) x -= w->S[tri(r) + c] * k[c]; k[r] = x / w->S[tri(r) + r]; }
      for (int r = 5; r >= 0; --r) { double x = k[r]; for (int c = r + 1; c < 6; ++c) x -= w->S[tri(c) + r] * k[c]; k[r] = x / w->S[tri(r) + r]; }
      for (int r = 0; r < 6; ++r) w->K[lane][r] = k[r];
    }
    __syncwarp();
    double th_new = 0.0, pn[2] = {0.0, 0.0}, diag = 0.0;
    if (lane < EST_NP) { th_new = w->th[lane]; for (int r = 0; r < 6; ++r) th_new += w->K[lane][r] * w->e[r]; }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = lane + 32 * h; if (t >= EST_TRI) break;
      int i = 0; while (tri(i + 1) <= t) ++i; const int j = t - tri(i);
      double kg = 0.0; for (int r = 0; r < 6; ++r) kg += w->K[i][r] * w->G[j][r] + w->K[j][r] * w->G[i][r];
      pn[h] = (w->P[t] - 0.5 * kg) / lam;
      if (i == j) diag += pn[h];
    }
    const double tr = warp_sum(diag);
    if (tr > prm.trace_max) { const double sc = prm.trace_max / tr; pn[0] *= sc; pn[1] *= sc; }
    const bool bad = !isfinite(th_new) || !isfinite(pn[0]) || !isfinite(pn[1]) || !isfinite(tr);
    if (__any_sync(FULL, bad)) code = QMB200_ST_NAN;
    else {
      if (lane < EST_NP) st[EST_THETA + lane] = th_new;
      st[EST_P + lane] = pn[0];
      if (lane + 32 < EST_TRI) st[EST_P + lane + 32] = pn[1];
    }
  }
  if (lane < NQ) { st[EST_Q + lane] = qk; st[EST_V + lane] = vk; }
  if (lane == 0) { st[EST_N] = n_prev + 1.0; status[b] = code; }
}

// One thread per robot: theta → [m, o] of the end-effector half of the model payload row and the robot's SRBD constants (srbd_payload_fold, as the host).
__global__ void payload_est_commit_kernel(const DevModel* __restrict__ mdl, qmb200_payload_est_params prm, int B, const double* __restrict__ state,
                                          double* __restrict__ mpayload /*[B][8]*/, double* __restrict__ srbd /*[B][SRBD_DBL]*/) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* th = state + (size_t)b * EST_DBL + EST_THETA; double* pl = mpayload + (size_t)b * 8;
  const double m0 = th[0], m = fmin(fmax(m0, 0.0), prm.mass_max);
  double o[3] = {0.0, 0.0, 0.0};
  if (m0 >= prm.mass_min) {
    o[0] = th[1] / m0; o[1] = th[2] / m0; o[2] = th[3] / m0;
    const double n = sqrt(dot3(o, o));
    if (n > prm.offset_max) { const double s = prm.offset_max / n; o[0] *= s; o[1] *= s; o[2] *= s; }
  }
  double row[8] = {m, o[0], o[1], o[2], pl[4], pl[5], pl[6], pl[7]};
  pl[0] = m; pl[1] = o[0]; pl[2] = o[1]; pl[3] = o[2];
  srbd_payload_fold(*mdl, row, srbd + (size_t)b * SRBD_DBL);
}

int launch_payload_est_step(const DevModel* mdl, const qmb200_payload_est_params& prm, int B, double dt, const double* effort, const double* rbd, double* state,
                            int32_t* status, cudaStream_t s) {
  payload_est_step_kernel<<<(B + EST_WARPS - 1) / EST_WARPS, 32 * EST_WARPS, 0, s>>>(mdl, prm, B, dt, effort, rbd, state, status);
  return 1;
}
int launch_payload_est_commit(const DevModel* mdl, const qmb200_payload_est_params& prm, int B, const double* state, double* mpayload, double* srbd, cudaStream_t s) {
  payload_est_commit_kernel<<<(B + 127) / 128, 128, 0, s>>>(mdl, prm, B, state, mpayload, srbd);
  return 1;
}

}  // namespace qmb
