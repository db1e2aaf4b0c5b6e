// TEST INFRASTRUCTURE: host build (g++) of the per-robot curriculum core (qm_control_b200/csrc/kernels/curriculum_api.cuh), the same functions the
// update kernel, qmb200_curriculum_attach and qmb200_curriculum_draw compile, so that the CPU suite can check it against a numpy statement
// (tests/test_curriculum_cpu.py).
#include <cstring>

#include "kernels/curriculum_api.cuh"

using namespace qmb;

namespace {
int message(const std::string& e, char* msg, int cap) {
  std::strncpy(msg, e.c_str(), cap - 1); msg[cap - 1] = 0;
  return e.empty() ? 0 : 1;
}
qmb200_curriculum_rule rule_of(int n_levels, int n_cond, const int32_t* column, const int32_t* op, const int32_t* role) {
  qmb200_curriculum_rule r{}; r.n_levels = n_levels; r.n_cond = n_cond;
  for (int i = 0; i < n_cond && i < QMB200_CURRICULUM_MAX_COND; ++i) { r.column[i] = column[i]; r.op[i] = op[i]; r.role[i] = role[i]; }
  return r;
}
}  // namespace

extern "C" {

// the boxes [m][width] of m robots at levels level[m] between base and top [m][width]
void cu_box(int m, int width, int round_col, int n_levels, const int32_t* level, const double* base, const double* top, double* out) {
  for (int i = 0; i < m; ++i) curriculum_box(base + (size_t)i * width, top + (size_t)i * width, width, round_col, level[i], n_levels, out + (size_t)i * width);
}
// k updates of one robot's state [CUS_INT] under its row [CU_DBL]: end[k] and metrics rows [k][QMB200_METRICS]; the state after each into states [k][CUS_INT]
void cu_stream(int n_levels, int n_cond, const int32_t* column, const int32_t* op, const int32_t* role, const double* row, int k, const int32_t* end,
               const double* metrics, int32_t* state, int32_t* states) {
  const qmb200_curriculum_rule r = rule_of(n_levels, n_cond, column, op, role);
  for (int j = 0; j < k; ++j) {
    if (end[j] == 1 || end[j] == 2) curriculum_step(n_levels, row, curriculum_outcome(r, row, end[j], metrics + (size_t)j * QMB200_METRICS), state);
    std::memcpy(states + (size_t)j * CUS_INT, state, CUS_INT * 4);
  }
}
// qmb200_curriculum_set's check: 0 when valid, else 1 with the message in msg
int cu_error(int n_levels, int n_cond, const int32_t* column, const int32_t* op, const int32_t* role, int B, const double* rows, char* msg, int cap) {
  qmb200_curriculum_rule r = rule_of(n_levels, n_cond, column, op, role); r.n_cond = n_cond;
  return message(curriculum_error(r, rows, (size_t)B), msg, cap);
}
// qmb200_curriculum_attach's checks of kind (0 episode, 1 spawn on n_tiles tiles, 2 timeline) on B robots' base and top boxes
int cu_attach_error(int kind, int n_tiles, int n_levels, int B, const double* base_lo, const double* base_hi, const double* top_lo, const double* top_hi, char* msg,
                    int cap) {
  const size_t b = (size_t)B;
  if (kind == 2) { const std::string e = curriculum_timeline_ends_error(base_lo, base_hi, top_lo, top_hi, b); if (!e.empty()) return message(e, msg, cap); }
  const int width = kind == 0 ? EP_DBL : kind == 1 ? SP_DBL : TL_DBL;
  const char* name = kind == 0 ? "episode" : kind == 1 ? "spawn" : "timeline";
  return message(curriculum_levels_error(name, base_lo, base_hi, top_lo, top_hi, b, width, kind == 1 ? SP_TILE : -1, n_levels, [&](const double* lo, const double* hi) {
    const std::string e = kind == 0 ? episode_ranges_error(lo, hi, b) : kind == 1 ? spawn_ranges_error(lo, hi, b, n_tiles) : timeline_ranges_error(lo, hi, b);
    return e.empty() ? e : e.substr(e.find(": ") + 2);
  }), msg, cap);
}

}  // extern "C"
