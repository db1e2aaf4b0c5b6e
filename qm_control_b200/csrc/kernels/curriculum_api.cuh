// Per-robot curricula (curriculum_kernel.cu; include/qmb200.h: qmb200_curriculum_*; DESIGN.md §4.15): the box of an attached draw kind at a robot's
// level, and the update of a robot's level from a closed episode.  Host + device: the update kernel, qmb200_curriculum_attach / _draw and
// tests/curriculum_host.cpp compile the same core, so host and device agree bit for bit.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cmath>
#include <string>
#include <vector>

#include "dev_common.cuh"
#include "episode_api.cuh"
#include "spawn_api.cuh"
#include "timeline_api.cuh"
#include "ee_path_draw_api.cuh"
#include "../../../include/qmb200.h"

namespace qmb {

// a curriculum row [CU_DBL] (_lib.CURRICULUM_LAYOUT) and a state row [CUS_INT] (_lib.CURRICULUM_STATE_LAYOUT)
constexpr int CU_START = 0, CU_UP_AFTER = 1, CU_DOWN_AFTER = 2, CU_THRESHOLD = 3, CU_DBL = 7;
constexpr int CUS_LEVEL = 0, CUS_PASS_RUN = 1, CUS_FAIL_RUN = 2, CUS_UPDATES = 3, CUS_INT = 4;
constexpr int CU_KINDS = 4;

// One column at `level` of n_levels: base at level 0 and top at the last level, byte for byte; between them base where both ends are equal (-0.0
// included; fma would turn -0.0 into +0.0), else fma(f, top - base, base) with f = level / (n_levels - 1), rounded to the nearest integer
// (floor(x + 0.5)) for a column that holds one (the spawn's tile)
QMB_HD double curriculum_value(double base, double top, int level, int n_levels, bool integer) {
  if (level <= 0) return base;
  if (level >= n_levels - 1) return top;
  if (base == top) return base;
  const double x = fma((double)level / (double)(n_levels - 1), top - base, base);
  return integer ? floor(x + 0.5) : x;
}
// one robot's box row [width] at `level` from its base and top rows; round_col: the integer column (-1: none)
QMB_HD void curriculum_box(const double* base, const double* top, int width, int round_col, int level, int n_levels, double* out) {
  for (int c = 0; c < width; ++c) out[c] = curriculum_value(base[c], top[c], level, n_levels, c == round_col);
}

// A closed episode's outcome: -1 fail (end 1, or a fail condition holds), 1 pass (end 2 and every pass condition holds), 0 neutral.  m: the episode's
// metrics row [QMB200_METRICS], read only when the rule has conditions; row: the robot's curriculum row.  A comparison with NaN is false.
QMB_HD int curriculum_outcome(const qmb200_curriculum_rule& r, const double* row, int end, const double* m) {
  bool fail = end == 1, pass = end == 2;
#pragma unroll
  for (int i = 0; i < QMB200_CURRICULUM_MAX_COND; ++i) {
    if (i >= r.n_cond) break;
    const double v = m[r.column[i]], t = row[CU_THRESHOLD + i];
    const bool holds = r.op[i] == QMB200_CURRICULUM_LE ? v <= t : v >= t;
    if (r.role[i] == QMB200_CURRICULUM_FAIL) fail = fail || holds; else pass = pass && holds;
  }
  return fail ? -1 : pass ? 1 : 0;
}
// One update of a robot's state s [CUS_INT] with an episode of outcome `outcome` (curriculum_outcome) under its row: a pass or a fail extends its run
// and ends the other; a run of up_after passes (down_after fails) moves the level one up (down), clamped to [0, n_levels), and starts the run again
QMB_HD void curriculum_step(int n_levels, const double* row, int outcome, int32_t* s) {
  s[CUS_UPDATES] += 1;
  if (outcome > 0) {
    s[CUS_FAIL_RUN] = 0; s[CUS_PASS_RUN] += 1;
    if ((double)s[CUS_PASS_RUN] >= row[CU_UP_AFTER]) { s[CUS_LEVEL] = s[CUS_LEVEL] + 1 < n_levels ? s[CUS_LEVEL] + 1 : n_levels - 1; s[CUS_PASS_RUN] = 0; }
  } else if (outcome < 0) {
    s[CUS_PASS_RUN] = 0; s[CUS_FAIL_RUN] += 1;
    if ((double)s[CUS_FAIL_RUN] >= row[CU_DOWN_AFTER]) { s[CUS_LEVEL] = s[CUS_LEVEL] > 0 ? s[CUS_LEVEL] - 1 : 0; s[CUS_FAIL_RUN] = 0; }
  }
}

// The check of qmb200_curriculum_set on a rule and rows [B][CU_DBL] ("" when valid): n_levels >= 2, at most QMB200_CURRICULUM_MAX_COND conditions of
// known columns, ops and roles; per robot an integer start_level in [0, n_levels), integer up_after and down_after in [1, 2^31), finite thresholds
inline std::string curriculum_error(const qmb200_curriculum_rule& r, const double* rows, size_t B) {
  if (r.n_levels < 2) return "rule n_levels must be >= 2";
  if (r.n_cond < 0 || r.n_cond > QMB200_CURRICULUM_MAX_COND) return "rule n_cond must lie in [0, " + std::to_string(QMB200_CURRICULUM_MAX_COND) + "]";
  for (int i = 0; i < r.n_cond; ++i) {
    const std::string f = "[" + std::to_string(i) + "]";
    if (r.column[i] < 0 || r.column[i] >= QMB200_METRICS) return "rule column" + f + " must be a metrics column in [0, " + std::to_string(QMB200_METRICS) + ")";
    if (r.op[i] != QMB200_CURRICULUM_GE && r.op[i] != QMB200_CURRICULUM_LE) return "rule op" + f + " must be QMB200_CURRICULUM_GE or QMB200_CURRICULUM_LE";
    if (r.role[i] != QMB200_CURRICULUM_PASS && r.role[i] != QMB200_CURRICULUM_FAIL) return "rule role" + f + " must be QMB200_CURRICULUM_PASS or QMB200_CURRICULUM_FAIL";
  }
  static const char* const names[CU_DBL] = {"start_level", "up_after", "down_after", "threshold[0]", "threshold[1]", "threshold[2]", "threshold[3]"};
  for (size_t b = 0; b < B; ++b) for (int c = 0; c < CU_DBL; ++c) {
    const double v = rows[b * CU_DBL + c]; const bool integer = std::isfinite(v) && std::floor(v) == v;
    const std::string why = c == CU_START ? (integer && v >= 0.0 && v < r.n_levels ? "" : "must be an integer in [0, " + std::to_string(r.n_levels) + ")")
                          : c < CU_THRESHOLD ? (integer && v >= 1.0 && v < 2147483648.0 ? "" : "must be an integer in [1, 2^31)")
                          : std::isfinite(v) ? "" : "must be finite";
    if (!why.empty()) return std::string(names[c]) + " of robot " + std::to_string(b) + ": " + why;
  }
  return "";
}
// The timeline's columns that are not interpolated, gait_set and ee_q*, must be equal in the base and top boxes lo, hi [B][TL_DBL] ("" when they are)
inline std::string curriculum_timeline_ends_error(const double* base_lo, const double* base_hi, const double* top_lo, const double* top_hi, size_t B) {
  static const char* const names[5] = {"gait_set", "ee_qx", "ee_qy", "ee_qz", "ee_qw"};
  static const int cols[5] = {TL_GAIT_SET, TL_EE_QUAT, TL_EE_QUAT + 1, TL_EE_QUAT + 2, TL_EE_QUAT + 3};
  for (size_t b = 0; b < B; ++b) for (int j = 0; j < 5; ++j) {
    const size_t i = b * TL_DBL + cols[j];
    if (!(top_lo[i] == base_lo[i] && top_hi[i] == base_hi[i])) return std::string("timeline ") + names[j] + " of robot " + std::to_string(b) + ": must be equal in the base and top boxes";
  }
  return "";
}
// The ee path's columns that are not interpolated, n_way and q*, must be equal in the base and top boxes lo, hi [B][EPR_DBL] ("" when they are)
inline std::string curriculum_ee_path_ends_error(const double* base_lo, const double* base_hi, const double* top_lo, const double* top_hi, size_t B) {
  static const char* const names[5] = {"n_way", "qx", "qy", "qz", "qw"};
  static const int cols[5] = {EPR_N_WAY, EPR_QUAT, EPR_QUAT + 1, EPR_QUAT + 2, EPR_QUAT + 3};
  for (size_t b = 0; b < B; ++b) for (int j = 0; j < 5; ++j) {
    const size_t i = b * EPR_DBL + cols[j];
    if (!(top_lo[i] == base_lo[i] && top_hi[i] == base_hi[i])) return std::string("ee_path ") + names[j] + " of robot " + std::to_string(b) + ": must be equal in the base and top boxes";
  }
  return "";
}
// The first level of n_levels whose boxes lo, hi [B][width] between base and top fail check(lo, hi) (a message naming the field and the robot, "" when
// valid): "<kind> level <l>: <message>", "" when every level passes
template <class Check>
std::string curriculum_levels_error(const char* kind, const double* base_lo, const double* base_hi, const double* top_lo, const double* top_hi, size_t B, int width,
                                    int round_col, int n_levels, Check check) {
  std::vector<double> lo(B * width), hi(B * width);
  for (int l = 0; l < n_levels; ++l) {
    for (size_t o = 0; o < B * width; o += width) {
      curriculum_box(base_lo + o, top_lo + o, width, round_col, l, n_levels, lo.data() + o); curriculum_box(base_hi + o, top_hi + o, width, round_col, l, n_levels, hi.data() + o);
    }
    if (const std::string e = check(lo.data(), hi.data()); !e.empty()) return std::string(kind) + " level " + std::to_string(l) + ": " + e;
  }
  return "";
}

#ifdef __CUDACC__
// An attached kind's boxes as the update reads and writes them: base lo, hi and top lo, hi [B][width] (the kind's width, a compile-time constant of the
// kernel), and the kind's device ranges lo, hi [B][width].  lo NULL: not attached.
struct CurriculumKind { const double *base_lo, *base_hi, *top_lo, *top_hi; double *lo, *hi; };
struct CurriculumArgs {
  qmb200_curriculum_rule rule; const double* rows; int32_t* state;   // the rule, the curriculum rows [B][CU_DBL], the state [B][CUS_INT]
  CurriculumKind kind[CU_KINDS];                                     // QMB200_CURRICULUM_EPISODE, _SPAWN, _TIMELINE, _EE_PATH
};
// one thread per robot: the masked robots with end 1 or 2 update their state from end and (with conditions) metrics[b][episode[b]]
int launch_curriculum_update(int B, const CurriculumArgs& a, const int32_t* mask, const int32_t* end, const int32_t* episode, const double* metrics, int n_episodes,
                             int32_t* level, int32_t* status, cudaStream_t s);
#endif

}  // namespace qmb
