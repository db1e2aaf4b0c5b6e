// TEST INFRASTRUCTURE: host build (g++) of the end-effector path code (DESIGN.md §4.20), so that the CPU suite can check it without a GPU
// (tests/test_ee_path_cpu.py): the target front-end's per-robot bodies (qm_control_b200/csrc/kernels/ctrl_api.cuh: target_robot and target_path, the
// functions ctrl_target_kernel runs), the path table's check (ee_paths_error) and the gait core's command rules with path rows (gait_api.cuh:
// gs_command_check, gs_step, the functions gait_command_kernel and gait_step_kernel run).
#include <cstdio>
#include <cstring>
#include <vector>

#include "kernels/ctrl_api.cuh"
#include "kernels/gait_api.cuh"

using namespace qmb;

extern "C" {

// ctrl_target_kernel's per-robot dispatch on n robots: kind [n] in [0, 2] → target_robot, TARGET_EE_PATH / _FOLLOW → target_path on ps [n][EE_PATH_STATE]
// and the table (n_paths, n_way [n_paths], way [n_paths][EE_PATH_MAX][8]); other kinds untouched.  prm4: com_height, target_displacement_velocity,
// target_rotation_velocity, time_to_target; qj [NJ]: default_joint_state.  le, ps, n_target, tt, ts in-out.
void eep_target(int n, const double* prm4, const double* qj, const int32_t* kind, const int32_t* frame, const double* cmd, const double* t_obs,
                const double* x_obs, const double* ee, double* le, double* ps, int n_paths, const int32_t* n_way, const double* way, int32_t* n_target,
                double* tt, double* ts) {
  TargetParams p{};
  p.com_height = prm4[0]; p.target_displacement_velocity = prm4[1]; p.target_rotation_velocity = prm4[2]; p.time_to_target = prm4[3];
  for (int j = 0; j < NJ; ++j) p.default_joint_state[j] = qj[j];
  for (int i = 0; i < n; ++i) {
    const bool hd = frame[i] == EE_FRAME_HEADING;
    if (kind[i] >= 0 && kind[i] <= 2)
      target_robot(p, kind[i], hd, cmd + (size_t)i * 7, t_obs[i], x_obs + (size_t)i * NX, ee + (size_t)i * 7, le + (size_t)i * 7, n_target + i,
                   tt + (size_t)i * KMAX, ts + (size_t)i * KMAX * TARGET_DIM);
    else if (kind[i] == TARGET_EE_PATH || kind[i] == TARGET_EE_PATH_FOLLOW)
      target_path(p, kind[i] == TARGET_EE_PATH, hd, cmd + (size_t)i * 7, t_obs[i], x_obs + (size_t)i * NX, ee + (size_t)i * 7, le + (size_t)i * 7,
                  ps + (size_t)i * EE_PATH_STATE, n_paths, n_way, way, n_target + i, tt + (size_t)i * KMAX, ts + (size_t)i * KMAX * TARGET_DIM);
  }
}

// qmb200_set_ee_paths's check → the message's length (0: accepted), the message into msg [cap]
int eep_paths_error(int n_paths, const int32_t* n_way, const double* way, double T, char* msg, int cap) {
  const std::string e = ee_paths_error(n_paths, n_way, way, T);
  std::snprintf(msg, (size_t)cap, "%s", e.c_str()); return (int)e.size();
}

// gait_command_kernel's check of n rows: tmpl [n], vel [n][4], ee_kind [n], ee [n][7] → out [n]; n_paths < 0: the check's default (no table)
void eep_check(int n, const int32_t* tmpl, const double* vel, const int32_t* ee_kind, const double* ee, int n_templates, int n_paths, int32_t* out) {
  for (int i = 0; i < n; ++i)
    out[i] = n_paths < 0 ? gs_command_check(tmpl[i], vel + 4 * i, ee_kind[i], ee + 7 * i, n_templates)
                         : gs_command_check(tmpl[i], vel + 4 * i, ee_kind[i], ee + 7 * i, n_templates, n_paths);
}

// B robots on one stance template stepped at the times t [n_ticks] by gs_step with a timeline of n_cmd rows per robot (t_cmd [B][n_cmd], ee_kind
// [B][n_cmd], ee [B][n_cmd][7], cmd_vel [B][n_cmd][4]; no template rows) and, before tick k, the pending rows of pend_set [n_ticks][B] (pend_kind
// [n_ticks][B], pend_ee [n_ticks][B][7], pend_vel [n_ticks][B][4]).  Out per tick: cmd [n_ticks][B][7] (zeros at the start), target_kind
// [n_ticks][B], src [n_ticks][B], status [n_ticks][B].
void eep_steps(int B, int n_ticks, const double* t, int n_cmd, const double* t_cmd, const int32_t* ee_kind, const double* ee, const double* cmd_vel,
               const int32_t* pend_set, const int32_t* pend_kind, const double* pend_ee, const double* pend_vel, double* cmd, int32_t* target_kind,
               int32_t* src, int32_t* status) {
  GsTemplate stance; std::memset(&stance, 0, sizeof(stance)); stance.n = 1; stance.md[0] = GS_STANCE; stance.sw[0] = 0.0; stance.sw[1] = 0.5;
  std::vector<int32_t> tmpl((size_t)B * n_cmd, -1);
  const GsCommands c{n_cmd, t_cmd, tmpl.data(), cmd_vel, ee_kind, ee};
  std::vector<GsRobot> r(B); std::vector<int32_t> cursor(B, 0); std::vector<GsPending> pend(B); std::vector<double> row((size_t)B * 7, 0.0);
  for (int b = 0; b < B; ++b) {
    std::memset(&r[b], 0, sizeof(GsRobot)); r[b].s.n = 0; r[b].s.md[0] = GS_STANCE; gs_insert(r[b].s, stance, t[0], 1.0, 0.4);
    std::memset(&pend[b], 0, sizeof(GsPending));
  }
  for (int k = 0; k < n_ticks; ++k)
    for (int b = 0; b < B; ++b) {
      const size_t kb = (size_t)k * B + b;
      if (pend_set[kb]) {
        GsPending& p = pend[b]; p.set = 1; p.tmpl = -1; p.ee_kind = pend_kind[kb]; p.pad = 0;
        for (int i = 0; i < 4; ++i) p.vel[i] = pend_vel[kb * 4 + i];
        for (int i = 0; i < 7; ++i) p.ee[i] = pend_ee[kb * 7 + i];
      }
      int32_t ne; double ev[QMB200_EMAX]; int32_t md[QMB200_EMAX + 1];
      status[kb] = gs_step(r[b], &cursor[b], &stance, c, b, t[k], 1.0, 0.4, &ne, ev, md, row.data() + (size_t)b * 7, target_kind + kb, &pend[b]);
      for (int i = 0; i < 7; ++i) cmd[kb * 7 + i] = row[(size_t)b * 7 + i];
      src[kb] = r[b].src;
    }
}

int eep_kmax() { return KMAX; }
int eep_target_dim() { return TARGET_DIM; }
int eep_path_max() { return EE_PATH_MAX; }
int eep_path_state() { return EE_PATH_STATE; }

}  // extern "C"
