// Warp-cooperative rigid-body algorithms for the 24-DoF quadruped-manipulator (base + 5 serial chains).
// Replaces the Pinocchio calls of WbcBase::updateMeasured / updateDesired (qm_wbc/src/WbcBase.cpp:150-190,
// 202-225): forwardKinematics, computeJointJacobians(+TimeVariation), crba, nonLinearEffects, dccrba.
//
// Formulation (GPU-first, not Pinocchio's): everything is expressed in WORLD coordinates with Plücker
// vectors taken about the world origin, so composite inertias and forces add without frame transforms and
// each lane owns one body.  Generalised velocity v = qdot with q = [p_base, euler ZYX, joints]
// (composite Translation+SphericalZYX root joint [upstream FactoryFunctions.cpp]).
//   motion vector  [w; vO]   (vO = velocity of the body-fixed point passing through the world origin)
//   force  vector  [nO; f]   (nO = moment about the world origin)
#pragma once
#include "dev_common.cuh"

namespace qmb {

struct RbdWs {
  double R[NB][9];      // body (joint) frame orientation in world
  double p[NB][3];      // body (joint) frame origin in world
  double S[NQ][6];      // motion subspace columns [w; vO] of the 24 generalised velocities
  double V[NB][6];      // spatial velocity
  double A[NB][6];      // spatial bias acceleration (qddot = 0, gravity NOT included)
  double Ic[NB][10];    // (composite) inertia about world origin: m, h=m*c (3), IO (xx,xy,xz,yy,yz,zz)
  double F[NB][6];      // (composite) spatial force [nO; f]
  double trig[6];       // sin/cos of the base euler angles z, y, x (one sincos pass per kinematics call)
};

// y = I * [w; vO] → [nO; f]
__device__ __forceinline__ void inertia_apply(const double* I, const double* mv, double* out) {
  const double m = I[0]; const double* h = I + 1; const double* io = I + 4; const double* w = mv; const double* v = mv + 3;
  out[0] = io[0] * w[0] + io[1] * w[1] + io[2] * w[2] + (h[1] * v[2] - h[2] * v[1]);
  out[1] = io[1] * w[0] + io[3] * w[1] + io[4] * w[2] + (h[2] * v[0] - h[0] * v[2]);
  out[2] = io[2] * w[0] + io[4] * w[1] + io[5] * w[2] + (h[0] * v[1] - h[1] * v[0]);
  out[3] = m * v[0] + (w[1] * h[2] - w[2] * h[1]);
  out[4] = m * v[1] + (w[2] * h[0] - w[0] * h[2]);
  out[5] = m * v[2] + (w[0] * h[1] - w[1] * h[0]);
}
__device__ __forceinline__ double dot6(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5]; }
// RNEA force of the inertia I moving with V under the bias acceleration A: F = I (A + g) + V x* I V, with g = +9.81 z (the base acceleration trick) or 0
__device__ __forceinline__ void rnea_force(const double* I, const double* V, const double* A, bool gravity, double* F) {
  double acc[6]; for (int i = 0; i < 6; ++i) acc[i] = A[i]; if (gravity) acc[5] += 9.81;
  double f1[6], mom[6]; inertia_apply(I, acc, f1); inertia_apply(I, V, mom);
  const double* w = V; const double* vv = V + 3;
  // V x* [n; f] = [w x n + v x f; w x f]
  double t1[3], t2[3]; cross3(w, mom, t1); cross3_add(vv, mom + 3, t1); cross3(w, mom + 3, t2);
  F[0] = f1[0] + t1[0]; F[1] = f1[1] + t1[1]; F[2] = f1[2] + t1[2]; F[3] = f1[3] + t2[0]; F[4] = f1[4] + t2[1]; F[5] = f1[5] + t2[2];
}

// The measured state rbd[55] as the rigid-body passes take it: q = [p, zyx, joints], v = [v_lin, zyx rates = T^-1 w_world, joint rates], into shared memory.
// T (euler_rate_map at zyx) is also stored when the caller keeps it, else pass NULL.  Lane 0 writes v[3..5] last: the caller synchronises the warp after.
__device__ __forceinline__ void rbd_read(const double* __restrict__ rb, double* q, double* v, double* T, int lane) {
  if (lane < 3) { q[lane] = rb[RBD_POS + lane]; q[3 + lane] = rb[RBD_ZYX + lane]; v[lane] = rb[RBD_V + lane]; }
  if (lane < NJ) { q[6 + lane] = rb[RBD_JPOS + lane]; v[6 + lane] = rb[RBD_JVEL + lane]; }
  __syncwarp();
  if (lane == 0) {
    double Tl[9], Ti[9]; double* Tm = T ? T : Tl; euler_rate_map(q[3], q[4], Tm); inv3(Tm, Ti);
    const double w[3] = {rb[RBD_W], rb[RBD_W + 1], rb[RBD_W + 2]}; matvec3(Ti, w, v + 3);
  }
}

// Pass 1: kinematics (+ optional velocities / bias accelerations).  q,v are in shared memory (24 each).
// Lane L < 19 owns body L.  with_vel: 0 = positions only, 1 = V and A as well.  max_depth limits the tree levels that are updated
// (3 = base + legs, 6 = arm as well).
// All trigonometry happens in ONE warp-wide pass (lanes 1..18: joint angles, folded straight into the joint-local rotation
// Rj * Rq(q_j); lanes 19..21: base euler angles -> ws->trig), so the level loop below is one 3x3 product per body.
template <bool with_vel, class WS>
__device__ __forceinline__ void rbd_kinematics(const DevModel* __restrict__ mdl, const double* q, const double* v, WS* ws, int lane, int max_depth = 6) {
  const int body = lane; const int j = body - 1;
  const int my_depth = (body >= 1 && body < NB) ? mdl->depth[body] : -1;
  double Rlq[9]; int ax = 0;
  {
    const bool is_joint = body >= 1 && body < NB, is_euler = lane >= NB && lane < NB + 3;
    double s = 0.0, c = 1.0; if (is_joint || is_euler) sincos(is_joint ? q[6 + j] : q[3 + lane - NB], &s, &c);
    if (is_euler) { ws->trig[2 * (lane - NB)] = s; ws->trig[2 * (lane - NB) + 1] = c; }
    if (is_joint) {
      ax = mdl->axis[j]; const double* Rl = mdl->Rj[j];
#pragma unroll
      for (int i = 0; i < 3; ++i) { const double r0 = Rl[3 * i], r1 = Rl[3 * i + 1], r2 = Rl[3 * i + 2];   // Rl * Rq(axis, q_j): Rq mixes the two columns after the axis
        if (ax == 0) { Rlq[3 * i] = r0; Rlq[3 * i + 1] = c * r1 + s * r2; Rlq[3 * i + 2] = -s * r1 + c * r2; }
        else if (ax == 1) { Rlq[3 * i] = c * r0 - s * r2; Rlq[3 * i + 1] = r1; Rlq[3 * i + 2] = s * r0 + c * r2; }
        else { Rlq[3 * i] = c * r0 + s * r1; Rlq[3 * i + 1] = -s * r0 + c * r1; Rlq[3 * i + 2] = r2; } }
    }
  }
  __syncwarp();
  // base (lane 0) and the 6 base columns of S
  if (lane == 0) {
    double R[9]; rot_zyx_sc(ws->trig, R);
#pragma unroll
    for (int i = 0; i < 9; ++i) ws->R[0][i] = R[i];
    ws->p[0][0] = q[0]; ws->p[0][1] = q[1]; ws->p[0][2] = q[2];
    double T[9]; euler_rate_map_sc(ws->trig, T);
    const double pb[3] = {q[0], q[1], q[2]};
#pragma unroll
    for (int k = 0; k < 3; ++k) {   // translation columns: w = 0, vO = e_k
      ws->S[k][0] = 0; ws->S[k][1] = 0; ws->S[k][2] = 0; ws->S[k][3] = (k == 0); ws->S[k][4] = (k == 1); ws->S[k][5] = (k == 2);
      const double w[3] = {T[k], T[3 + k], T[6 + k]}; double vo[3]; cross3(pb, w, vo);   // euler-rate columns: w = T[:,k], vO = p x w
      ws->S[3 + k][0] = w[0]; ws->S[3 + k][1] = w[1]; ws->S[3 + k][2] = w[2]; ws->S[3 + k][3] = vo[0]; ws->S[3 + k][4] = vo[1]; ws->S[3 + k][5] = vo[2];
    }
    if constexpr (with_vel) {
      const double ed[3] = {v[3], v[4], v[5]}; double w[3]; matvec3(T, ed, w);
      double wd[3]; euler_rate_map_dot_times_sc(ws->trig, ed, wd);
      const double pd[3] = {v[0], v[1], v[2]};
      double vo[3]; cross3(pb, w, vo); vo[0] += pd[0]; vo[1] += pd[1]; vo[2] += pd[2];
      double ao[3]; cross3(pd, w, ao); cross3_add(pb, wd, ao);
      ws->V[0][0] = w[0]; ws->V[0][1] = w[1]; ws->V[0][2] = w[2]; ws->V[0][3] = vo[0]; ws->V[0][4] = vo[1]; ws->V[0][5] = vo[2];
      ws->A[0][0] = wd[0]; ws->A[0][1] = wd[1]; ws->A[0][2] = wd[2]; ws->A[0][3] = ao[0]; ws->A[0][4] = ao[1]; ws->A[0][5] = ao[2];
    }
  }
  __syncwarp();
  for (int d = 1; d <= max_depth; ++d) {
    if (my_depth == d) {
      const int pb = mdl->parent[j];
      double Rp[9], Rw[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) Rp[i] = ws->R[pb][i];
      matmul3(Rp, Rlq, Rw);
      double pl[3] = {mdl->pj[j][0], mdl->pj[j][1], mdl->pj[j][2]}, pw[3]; matvec3(Rp, pl, pw);
      pw[0] += ws->p[pb][0]; pw[1] += ws->p[pb][1]; pw[2] += ws->p[pb][2];
#pragma unroll
      for (int i = 0; i < 9; ++i) ws->R[body][i] = Rw[i];
      ws->p[body][0] = pw[0]; ws->p[body][1] = pw[1]; ws->p[body][2] = pw[2];
      const double a[3] = {Rw[ax], Rw[3 + ax], Rw[6 + ax]}; double vo[3]; cross3(pw, a, vo);
      double* Sc = ws->S[6 + j]; Sc[0] = a[0]; Sc[1] = a[1]; Sc[2] = a[2]; Sc[3] = vo[0]; Sc[4] = vo[1]; Sc[5] = vo[2];
      if constexpr (with_vel) {
        const double qd = v[6 + j]; const double* Vp = ws->V[pb]; const double* Ap = ws->A[pb];
        // V = Vp + S qd ;  A = Ap + (Vp x S) qd   with motion cross [w;v]x[a;b] = [w x a; w x b + v x a]
        double c1[3], c2[3]; cross3(Vp, a, c1); cross3(Vp, vo, c2); cross3_add(Vp + 3, a, c2);
        double* Vb = ws->V[body]; double* Ab = ws->A[body];
        Vb[0] = Vp[0] + a[0] * qd; Vb[1] = Vp[1] + a[1] * qd; Vb[2] = Vp[2] + a[2] * qd; Vb[3] = Vp[3] + vo[0] * qd; Vb[4] = Vp[4] + vo[1] * qd; Vb[5] = Vp[5] + vo[2] * qd;
        Ab[0] = Ap[0] + c1[0] * qd; Ab[1] = Ap[1] + c1[1] * qd; Ab[2] = Ap[2] + c1[2] * qd; Ab[3] = Ap[3] + c2[0] * qd; Ab[4] = Ap[4] + c2[1] * qd; Ab[5] = Ap[5] + c2[2] * qd;
      }
    }
    __syncwarp();
  }
}

// Pass 2: per-body world inertias; optionally RNEA body forces (gravity: +9.81 z base acceleration trick).
// with_force: 0 none, 1 = F = I (A + Ag) + V x* I V with gravity, 2 = same without gravity (centroidal momentum rate bias)
__device__ __forceinline__ void rbd_inertias(const DevModel* __restrict__ mdl, RbdWs* ws, int lane, int with_force) {
  if (lane < NB) {
    const int b = lane; const double m = mdl->mass[b];
    double R[9]; for (int i = 0; i < 9; ++i) R[i] = ws->R[b][i];
    double cl[3] = {mdl->com[b][0], mdl->com[b][1], mdl->com[b][2]}, c[3]; matvec3(R, cl, c); c[0] += ws->p[b][0]; c[1] += ws->p[b][1]; c[2] += ws->p[b][2];
    double Il[9]; for (int i = 0; i < 9; ++i) Il[i] = mdl->Ib[b][i];
    double RI[9], Iw[9]; matmul3(R, Il, RI); matmul3_nt(RI, R, Iw);
    const double cc = dot3(c, c);
    double* I = ws->Ic[b]; I[0] = m; I[1] = m * c[0]; I[2] = m * c[1]; I[3] = m * c[2];
    I[4] = Iw[0] + m * (cc - c[0] * c[0]); I[5] = Iw[1] - m * c[0] * c[1]; I[6] = Iw[2] - m * c[0] * c[2];
    I[7] = Iw[4] + m * (cc - c[1] * c[1]); I[8] = Iw[5] - m * c[1] * c[2]; I[9] = Iw[8] + m * (cc - c[2] * c[2]);
    if (with_force) rnea_force(I, ws->V[b], ws->A[b], with_force == 1, ws->F[b]);
  }
  __syncwarp();
}

// Pass 3: leaf-to-root accumulation of composite inertias (and forces if with_force).
__device__ __forceinline__ void rbd_accumulate(const DevModel* __restrict__ mdl, RbdWs* ws, int lane, bool with_force) {
  const int body = lane; const int my_depth = (body >= 1 && body < NB) ? mdl->depth[body] : -1;
  for (int d = 6; d >= 2; --d) {   // every body at depth >= 2 is the only child of its parent
    if (my_depth == d) {
      const int pb = mdl->parent[body - 1];
      for (int i = 0; i < 10; ++i) ws->Ic[pb][i] += ws->Ic[body][i];
      if (with_force) for (int i = 0; i < 6; ++i) ws->F[pb][i] += ws->F[body][i];
    }
    __syncwarp();
  }
  // depth-1 bodies (4 hips + arm link 1) all hang off the base: lanes 0..15 each sum one component
  if (lane < 16) {
    const int comp = lane;
    double acc = (comp < 10) ? ws->Ic[0][comp] : ((with_force) ? ws->F[0][comp - 10] : 0.0);
    for (int b = 1; b < NB; ++b) if (mdl->depth[b] == 1) acc += (comp < 10) ? ws->Ic[b][comp] : (with_force ? ws->F[b][comp - 10] : 0.0);
    if (comp < 10) ws->Ic[0][comp] = acc; else if (with_force) ws->F[0][comp - 10] = acc;
  }
  __syncwarp();
}

// body index that generalised velocity column c moves (0 for the 6 base columns)
__device__ __forceinline__ int col_body(int c) { return c < 6 ? 0 : c - 5; }

// Mass matrix (dense 24x24, leading dimension ldm) and nonlinear effects from composite quantities.
__device__ __forceinline__ void rbd_mass_matrix_nle(const DevModel* __restrict__ mdl, const RbdWs* ws, double* M, int ldm, double* nle, int lane) {
  for (int i = lane; i < NQ * NQ; i += 32) M[(i / NQ) * ldm + (i % NQ)] = 0.0;
  __syncwarp();
  if (lane < NQ) {
    const int c = lane; const int b = col_body(c);
    double Fc[6]; inertia_apply(ws->Ic[b], ws->S[c], Fc);
    nle[c] = dot6(ws->S[c], ws->F[b]);
    if (c < 6) {
      for (int k = 0; k < 6; ++k) M[c * ldm + k] = dot6(ws->S[k], Fc);
    } else {
      // own column, ancestors on the chain, and the 6 base columns
      M[c * ldm + c] = dot6(ws->S[c], Fc);
      for (int a = mdl->chain_start[c - 6] + 6; a < c; ++a) { const double mv = dot6(ws->S[a], Fc); M[c * ldm + a] = mv; M[a * ldm + c] = mv; }
      for (int k = 0; k < 6; ++k) { const double mv = dot6(ws->S[k], Fc); M[c * ldm + k] = mv; M[k * ldm + c] = mv; }
    }
  }
  __syncwarp();
}

// velocity of the point pw (world) fixed on a body moving with the spatial velocity V = [w; vO]: w x pw + vO
__device__ __forceinline__ void point_vel(const double* V, const double* pw, double* vel) { cross3(V, pw, vel); vel[0] += V[3]; vel[1] += V[4]; vel[2] += V[5]; }

// Linear velocity Jacobian row block (3 x 24, LOCAL_WORLD_ALIGNED) of a point pw fixed on `body` whose chain
// covers joints [chain_first, chain_last]; lanes over columns.
__device__ __forceinline__ void point_jacobian(const RbdWs* ws, const double* pw, int chain_first, int chain_last, double* J, int ldj, int lane) {
  if (lane < NQ) {
    const int c = lane; double col[3] = {0, 0, 0};
    if (c < 6 || (c - 6 >= chain_first && c - 6 <= chain_last)) point_vel(ws->S[c], pw, col);
    J[c] = col[0]; J[ldj + c] = col[1]; J[2 * ldj + c] = col[2];
  }
}
// classical velocity / bias acceleration (Jdot*v) of a point fixed on a body moving with V, A
__device__ __forceinline__ void point_vel_acc(const double* V, const double* A, const double* pw, double* vel, double* acc) {
  point_vel(V, pw, vel); point_vel(A, pw, acc); cross3_add(V, vel, acc);
}

// world position of the point pl (body axes) fixed on `body`
__device__ __forceinline__ void body_point(const RbdWs* ws, int body, const double* pl, double* pw) {
  matvec3(ws->R[body], pl, pw); pw[0] += ws->p[body][0]; pw[1] += ws->p[body][1]; pw[2] += ws->p[body][2];
}
// origin of foot frame f (world)
__device__ __forceinline__ void foot_point(const DevModel* __restrict__ mdl, const RbdWs* ws, int f, double* pw) { body_point(ws, mdl->foot_body[f], mdl->foot_p[f], pw); }
// end-effector frame: origin pe and, unless Re is NULL, rotation Re (world)
__device__ __forceinline__ void ee_pose(const DevModel* __restrict__ mdl, const RbdWs* ws, double* pe, double* Re) {
  const int eb = mdl->ee_body; body_point(ws, eb, mdl->ee_p, pe); if (Re) matmul3(ws->R[eb], mdl->ee_R, Re);
}

}  // namespace qmb
