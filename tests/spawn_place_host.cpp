// TEST INFRASTRUCTURE: host build (g++) of the "here" row and the place check (qm_control_b200/csrc/kernels/spawn_api.cuh: spawn_here_row,
// spawn_place_ok, spawn_wrap_yaw), the same functions spawn_here_kernel and spawn_place_kernel compile, so that the CPU suite can check them against
// numpy statements (tests/test_spawn_place_cpu.py).
#include "kernels/spawn_api.cuh"

using namespace qmb;

extern "C" {

// n cases: rbd [n][QMB200_RBD], q_start [n][NQ], origin [n][2], ter [n][3] used where has_ter[i] != 0 → rows [n][SP_DBL]
void sph_here(int n, const double* rbd, const double* q_start, const double* origin, const double* ter, const int32_t* has_ter, double* rows) {
  for (int i = 0; i < n; ++i)
    spawn_here_row(rbd + (size_t)i * QMB200_RBD, q_start + (size_t)i * NQ, origin + 2 * (size_t)i, has_ter[i] ? ter + 3 * (size_t)i : nullptr, rows + (size_t)i * SP_DBL);
}
// n rows [n][SP_DBL] on a library of n_tiles tiles, with (rows_set[i] != 0) or without robot terrain rows → ok [n]
void sph_place_ok(int n, const double* rows, int n_tiles, const int32_t* rows_set, int32_t* ok) {
  for (int i = 0; i < n; ++i) ok[i] = spawn_place_ok(rows + (size_t)i * SP_DBL, n_tiles, rows_set[i] != 0);
}

}  // extern "C"
