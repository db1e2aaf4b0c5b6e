// Point-mass payloads rigidly attached to the end-effector frame or to the base, for the warp rigid-body passes (rbd.cuh): the plant's robot params
// (sim_kernel.cu) and the controller's model payload (wbc_kernel.cu) add them the same way, between rbd_inertias and rbd_accumulate, so that M, nle and the
// composite inertias include them through the existing passes.
#pragma once
#include "rbd.cuh"

namespace qmb {

// frame 0: the end-effector frame (on body ee_body), 1: the base frame (body 0).  R = the body's world rotation, po = the frame's origin (world); returns the body.
__device__ __forceinline__ int payload_frame(const DevModel* __restrict__ mdl, const RbdWs* ws, int frame, double* R, double* po) {
  const int body = frame == 0 ? mdl->ee_body : 0;
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = ws->R[body][i];
  po[0] = 0.0; po[1] = 0.0; po[2] = 0.0; if (frame == 0) matvec3(R, mdl->ee_p, po);
  po[0] += ws->p[body][0]; po[1] += ws->p[body][1]; po[2] += ws->p[body][2];
  return body;
}

// pl = [m, o(3)]: a point mass m at offset o in the frame's axes.  Adds its spatial inertia about the world origin [m, m c, m(|c|^2 1 - c c^T)] to Ic[body] and its
// RNEA force I_p (A + g) + V x* I_p V to F[body], with g = +9.81 z as rbd_inertias' mode 1 (gravity) or g = 0 as its mode 2.  A zero mass adds exact zeros.
__device__ __forceinline__ void payload_add(const DevModel* __restrict__ mdl, RbdWs* ws, int frame, int body, const double* R, const double* po, const double* __restrict__ pl, bool gravity) {
  const double m = pl[0]; const double ol[3] = {pl[1], pl[2], pl[3]}; double ob[3] = {ol[0], ol[1], ol[2]};
  if (frame == 0) matvec3(mdl->ee_R, ol, ob);                                   // offset in the body's axes
  double c[3]; matvec3(R, ob, c); c[0] += po[0]; c[1] += po[1]; c[2] += po[2];   // point mass position (world)
  const double cc = dot3(c, c);
  double I[10] = {m, m * c[0], m * c[1], m * c[2], m * (cc - c[0] * c[0]), -m * c[0] * c[1], -m * c[0] * c[2], m * (cc - c[1] * c[1]), -m * c[1] * c[2], m * (cc - c[2] * c[2])};
  double* Ic = ws->Ic[body]; double* F = ws->F[body];
#pragma unroll
  for (int i = 0; i < 10; ++i) Ic[i] += I[i];
  double f[6]; rnea_force(I, ws->V[body], ws->A[body], gravity, f);
#pragma unroll
  for (int i = 0; i < 6; ++i) F[i] += f[i];
}

// both steps for the frame's payload pl
__device__ __forceinline__ void payload_load(const DevModel* __restrict__ mdl, RbdWs* ws, int frame, const double* __restrict__ pl, bool gravity) {
  double R[9], po[3]; const int body = payload_frame(mdl, ws, frame, R, po); payload_add(mdl, ws, frame, body, R, po, pl, gravity);
}

}  // namespace qmb
