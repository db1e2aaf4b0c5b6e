// Per-episode end-effector paths (include/qmb200.h: qmb200_ee_path_sample_dev; DESIGN.md §4.21).
//   ee_path_sample_kernel   one thread per robot: a masked robot draws its episode's path from its ranges (ee_path_waypoint, the host's core), writes
//                           each of its n_way waypoints as it is drawn to its record row and to its row p0 + b of the path table (the waypoints past
//                           n_way are not written: target_path reads none of them), that row's n_way, and a
//                           pending start of that row into its gait pending slot (the bytes qmb200_gait_dev_command writes for the row
//                           tmpl -1, cmd_vel NaN, ee_kind QMB200_TARGET_EE_PATH, ee[0] = p0 + b).  Unmasked robots are not written.
#include "ee_path_draw_api.cuh"

namespace qmb {

namespace {
constexpr int EPD_THREADS = 128;

__global__ void __launch_bounds__(EPD_THREADS) ee_path_sample_kernel(int B, int64_t robot0, const double* __restrict__ lo, const double* __restrict__ hi,
                                                                     uint64_t seed, const int32_t* __restrict__ mask, const int32_t* __restrict__ episode,
                                                                     double* __restrict__ rows, const EePathTargets t) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  const double* l = lo + (size_t)b * EPR_DBL; const double* h = hi + (size_t)b * EPR_DBL;
  const uint64_t robot = (uint64_t)(robot0 + b), ep = (uint64_t)(int64_t)episode[b];
  const int n = ee_path_n_way(l), p = t.p0 + b;
  double* rec = rows + (size_t)b * EE_PATH_MAX * EE_PATH_WAY; double* tab = t.way + (size_t)p * EE_PATH_MAX * EE_PATH_WAY;
  double tp = 0.0;
  for (int i = 0; i < n; ++i) {
    double w[EE_PATH_WAY];
    ee_path_waypoint(l, h, seed, robot, ep, i, tp, w); tp = w[0];
#pragma unroll
    for (int k = 0; k < EE_PATH_WAY; ++k) { rec[(size_t)i * EE_PATH_WAY + k] = w[k]; tab[(size_t)i * EE_PATH_WAY + k] = w[k]; }
  }
  t.n_way[p] = n;
  GsPending& g = t.pending[b];
  const double nan = timeline_nan();
  g.set = 1; g.tmpl = -1; g.ee_kind = GS_SRC_EE_PATH; g.pad = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) g.vel[i] = nan;
  g.ee[0] = (double)p;
#pragma unroll
  for (int i = 1; i < 7; ++i) g.ee[i] = 0.0;
}
}  // namespace

int launch_ee_path_sample(int B, int64_t robot0, const double* lo, const double* hi, uint64_t seed, const int32_t* mask, const int32_t* episode, double* rows,
                          const EePathTargets& t, cudaStream_t s) {
  ee_path_sample_kernel<<<(B + EPD_THREADS - 1) / EPD_THREADS, EPD_THREADS, 0, s>>>(B, robot0, lo, hi, seed, mask, episode, rows, t);
  return 1;
}

}  // namespace qmb
