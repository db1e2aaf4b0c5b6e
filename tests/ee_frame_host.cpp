// TEST INFRASTRUCTURE: host build (g++) of the target front-end's per-robot body (qm_control_b200/csrc/kernels/ctrl_api.cuh: target_robot, the
// function ctrl_target_kernel runs) with its world and heading frames, so that the CPU suite can check it against the oracle and against a numpy
// statement of the heading rule (tests/test_ee_frame_cpu.py); with it the spawn's hold rule (spawn_api.cuh: spawn_turn_hold) and the frame setter's
// check (ee_frame_error).
#include <cstdio>

#include "kernels/ctrl_api.cuh"
#include "kernels/spawn_api.cuh"

using namespace qmb;

extern "C" {

// The parameters the handle builds from reference.info / task.info: com_height, target_displacement_velocity, target_rotation_velocity,
// time_to_target, default_joint_state [NJ]
// n robots: kind [n] (outside [0, 2]: untouched), frame [n] (EE_FRAME_*), cmd [n][7], t_obs [n], x_obs [n][NX], ee [n][7], le [n][7] in-out,
// n_target [n], tt [n][KMAX], ts [n][KMAX][TARGET_DIM] in-out
void eef_target(int n, const double* prm4, const double* qj, const int32_t* kind, const int32_t* frame, const double* cmd, const double* t_obs,
                const double* x_obs, const double* ee, double* le, int32_t* n_target, double* tt, double* ts) {
  TargetParams p{};
  p.com_height = prm4[0]; p.target_displacement_velocity = prm4[1]; p.target_rotation_velocity = prm4[2]; p.time_to_target = prm4[3];
  for (int j = 0; j < NJ; ++j) p.default_joint_state[j] = qj[j];
  for (int i = 0; i < n; ++i) {
    if (kind[i] < 0 || kind[i] > 2) continue;
    target_robot(p, kind[i], frame[i] == EE_FRAME_HEADING, cmd + (size_t)i * 7, t_obs[i], x_obs + (size_t)i * NX, ee + (size_t)i * 7, le + (size_t)i * 7,
                 n_target + i, tt + (size_t)i * KMAX, ts + (size_t)i * KMAX * TARGET_DIM);
  }
}

// n holds e [n][7] in-out turned by spawns from yaw0 [n] to yaw [n] about bases at (x, y) [n][2]; heading [n] != 0: heading-frame robots
void eef_spawn_hold(int n, double* e, const double* xy, const double* yaw0, const double* yaw, const int32_t* heading) {
  for (int i = 0; i < n; ++i) spawn_turn_hold(e + (size_t)i * 7, xy[2 * i], xy[2 * i + 1], yaw0[i], yaw[i], heading[i] != 0);
}
// qmb200_set_ee_frame's check of frame [B] → the message's length (0: accepted), the message into msg [cap]
int eef_frame_error(const int32_t* frame, int B, char* msg, int cap) {
  const std::string e = ee_frame_error(frame, (size_t)B);
  std::snprintf(msg, (size_t)cap, "%s", e.c_str()); return (int)e.size();
}

int eef_kmax() { return KMAX; }
int eef_target_dim() { return TARGET_DIM; }

}  // extern "C"
