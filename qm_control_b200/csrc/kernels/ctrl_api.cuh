// Host-visible interface of the controller-side kernels (observation, target front-end, control law, hybrid-joint plant law).
#pragma once
#include <cuda_runtime.h>

#include "dev_common.cuh"
#include "mpc_api.cuh"

namespace qmb {

constexpr int HW_DEPTH = 32;   // command-delay ring entries per robot (delay 0.009 s at a 1 kHz loop needs 10; gazebo/config/default.yaml:2)

// constants of the target publisher node (QmTargetTrajectoriesPublisher_node.cpp:225-229)
struct TargetParams {
  double com_height;                     // reference.info comHeight
  double target_displacement_velocity;   // reference.info targetDisplacementVelocity
  double target_rotation_velocity;       // reference.info targetRotationVelocity
  double time_to_target;                 // task.info mpc.timeHorizon
  double default_joint_state[NJ];        // reference.info defaultJointState
};

struct ControlLawParams {
  static constexpr int ROBOTS = 7, THREADS = 128;   // 7 robots x 18 joints = 126 threads of a 128-thread CTA
  int variant;                // 0 QMController, 1 QMMpcController
  double arm_kp, arm_kd;      // dynamic_reconfigure kp_arm_wbc / kd_arm_wbc (qm_controllers/cfg/weight.cfg:7-8: 0.0, 0.5)
};

int launch_observation(const DevModel* mdl, int B, const double* rbd, const double* period, double* t_obs, double* x_obs, cudaStream_t s, const double* srbd /*[B][SRBD_DBL] or NULL*/);
// kinds [B] (device, or NULL: every robot `kind`): per-robot kind; robots outside [0, 2] are left untouched
int launch_target(const TargetParams& prm, int kind, const int32_t* kinds, int B, const double* cmd, const double* t_obs, const double* x_obs, const double* ee_state,
                  double* last_ee_target, int32_t* n_target, double* target_times, double* target_states, cudaStream_t s);
int launch_control_law(const ControlLawParams& prm, int B, const double* x_des, const double* u_des, const double* wbc_cmd, const double* t_obs, const double* x_obs,
                       double* joint_cmd, double* arm_pos_cmd, double* last_time, int32_t* status, cudaStream_t s,
                       const double* tuning /*[B][TUNING_DBL] or NULL: the robots' arm gains in place of prm's*/);
int launch_hw_write(int B, double delay, const double* time, const double* period, const double* joint_cmd, const double* joint_pos, const double* joint_vel,
                    double* ring_cmd, double* ring_stamp, int32_t* ring_state, double* effort, int32_t* status, cudaStream_t s);

}  // namespace qmb
