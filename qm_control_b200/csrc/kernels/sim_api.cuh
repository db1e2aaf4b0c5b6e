// Host-visible interface of the batched plant step (sim_kernel.cu): rigid-body forward dynamics of the 24-DoF tree with compliant
// foot-ground contact, the stand-in for Gazebo's physics step behind QMHWSim (qm_gazebo/src/QMHWSim.cpp).
#pragma once
#include <cuda_runtime.h>

#include "dev_common.cuh"

namespace qmb {

// Contact and joint constants of the plant (include/qmb200.h: qmb200_sim_params; DESIGN.md §4.6 explains the defaults).
struct SimParams {
  double ground_height;        // height of the flat ground plane (m)
  double foot_radius;          // collision sphere of the *_FOOT links, centred on the foot frame (m)
  double stiffness;            // normal penalty spring k (N/m)
  double damping;              // normal damper d (N s/m)
  double tangential_damping;   // regularised Coulomb friction: viscous slope gamma below the friction cone (N s/m)
  double friction_mu;          // Coulomb coefficient mu
  double joint_damping[NJ];    // viscous joint damping (N m s/rad)
  int substeps_per_ms;         // semi-implicit Euler steps per millisecond of simulated time
};

// mu [B], payload [B][8], wrench [B][12]: optional per-robot plant variation (NULL = not used; sim_kernel.cu has the layouts)
int launch_sim_step(const DevModel* mdl, const SimParams& prm, int B, int substeps, double h, const double* effort, double* q, double* v, double* rbd, int32_t* contact,
                    int32_t* status, const double* mu, const double* payload, const double* wrench, cudaStream_t s);

}  // namespace qmb
