// TEST INFRASTRUCTURE: host build (g++) of the per-episode end-effector path draw core (qm_control_b200/csrc/kernels/ee_path_draw_api.cuh), the same
// functions the sampler kernel and qmb200_ee_path_draw compile, with the path table's check and the curriculum's level checks of the kind, so that the
// CPU suite can check them against a numpy statement (tests/test_ee_path_draw_cpu.py).
#include <cstring>

#include "kernels/curriculum_api.cuh"

using namespace qmb;

namespace {
int message(const std::string& e, char* msg, int cap) {
  std::strncpy(msg, e.c_str(), cap - 1); msg[cap - 1] = 0;
  return e.empty() ? 0 : 1;
}
}  // namespace

extern "C" {

// the paths of m (seed, robot, episode) triples on ranges lo, hi [m][EPR_DBL]: n_way [m] and way [m][EE_PATH_MAX][8]
void epd_rows(int m, const uint64_t* seed, const uint64_t* robot, const uint64_t* episode, const double* lo, const double* hi, int32_t* n_way, double* way) {
  for (int i = 0; i < m; ++i)
    n_way[i] = ee_path_rows(lo + (size_t)i * EPR_DBL, hi + (size_t)i * EPR_DBL, seed[i], robot[i], episode[i], way + (size_t)i * EE_PATH_MAX * EE_PATH_WAY);
}
// qmb200_ee_path_set_ranges' check on B robots' ranges at horizon T: 0 when valid, else 1 with the message in msg
int epd_ranges_error(int B, const double* lo, const double* hi, double T, char* msg, int cap) { return message(ee_path_ranges_error(lo, hi, (size_t)B, T), msg, cap); }
// qmb200_set_ee_paths' check on n paths at horizon T
int epd_paths_error(int n, const int32_t* n_way, const double* way, double T, char* msg, int cap) { return message(ee_paths_error(n, n_way, way, T), msg, cap); }
// qmb200_curriculum_attach's checks of the ee path kind on B robots' base and top boxes at n_levels levels and horizon T
int epd_attach_error(int n_levels, int B, double T, const double* base_lo, const double* base_hi, const double* top_lo, const double* top_hi, char* msg, int cap) {
  const size_t b = (size_t)B;
  if (const std::string e = curriculum_ee_path_ends_error(base_lo, base_hi, top_lo, top_hi, b); !e.empty()) return message(e, msg, cap);
  return message(curriculum_levels_error("ee_path", base_lo, base_hi, top_lo, top_hi, b, EPR_DBL, -1, n_levels, [&](const double* lo, const double* hi) {
    const std::string e = ee_path_ranges_error(lo, hi, b, T);
    return e.empty() ? e : e.substr(e.find(": ") + 2);
  }), msg, cap);
}

}  // extern "C"
