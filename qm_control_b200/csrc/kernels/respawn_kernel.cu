// Per-robot restart and robot-state snapshots (include/qmb200.h: qmb200_robot_image_*, qmb200_robot_state_*, qmb200_fall_detect; DESIGN.md §4.10, §4.17).
//   image_restore_kernel   one launch over a table of per-robot row blocks (the start image of each running component with the zeroed warm starts, WBC
//                          input and command FIFO; or a snapshot's blocks): grid.y picks the block, a grid-stride loop over its B x words 4-byte words
//                          writes the masked robots' words from their source rows (respawn_api.cuh: restore_source / restore_word).  Copies are
//                          bit-exact, so a restored robot holds exactly what its source row holds.
//   fall_detect_kernel     one thread per robot on the plant's rbd.
#include <cstdint>

#include "../../../include/qmb200.h"
#include "respawn_api.cuh"

namespace qmb {

namespace {
constexpr int RESTORE_THREADS = 256, FALL_THREADS = 128;

__global__ void __launch_bounds__(RESTORE_THREADS) image_restore_kernel(const RestoreTable t, int B, const int32_t* __restrict__ mask, const int32_t* __restrict__ row,
                                                                        int32_t* __restrict__ status) {
  const RestoreSeg g = t.seg[blockIdx.y];
  const int64_t n = (int64_t)B * g.words;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / g.words); int r;
    if (restore_source(B, mask, row, b, r)) g.dst[i] = restore_word(g, r, i - (int64_t)b * g.words);
  }
  if (status && blockIdx.y == 0)
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) status[b] = restore_status(B, mask, row, b);
}

__global__ void __launch_bounds__(FALL_THREADS) fall_detect_kernel(int B, const double* __restrict__ rbd, double z_min, double tilt_max, const SimTerrain terrain,
                                                                   double ground_height, int32_t* __restrict__ count, int32_t* __restrict__ fallen) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* r = rbd + (size_t)b * QMB200_RBD;   // [0, 3) zyx = (yaw, pitch, roll), [3, 6) base position
  bool finite = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) finite = finite && isfinite(r[i]);
  bool down = !finite;
  if (finite) {
    double H, gx, gy;
    ground_at(terrain, terrain.robot ? terrain.robot + (size_t)b * 3 : nullptr, ground_height, r[3], r[4], H, gx, gy);
    down = r[5] - H <= z_min || fabs(r[1]) >= tilt_max || fabs(r[2]) >= tilt_max;
  }
  fallen[b] = down ? 1 : 0;
  count[b] = down ? count[b] + 1 : 0;
}
}  // namespace

int launch_image_restore(const RestoreTable& t, int B, const int32_t* mask, cudaStream_t s, const int32_t* row, int32_t* status) {
  if (t.n == 0) return 0;
  int64_t widest = 0;
  for (int i = 0; i < t.n; ++i) widest = widest > t.seg[i].words ? widest : t.seg[i].words;
  const int64_t blocks = ((int64_t)B * widest + RESTORE_THREADS - 1) / RESTORE_THREADS;
  image_restore_kernel<<<dim3((unsigned)(blocks < 1024 ? blocks : 1024), (unsigned)t.n), RESTORE_THREADS, 0, s>>>(t, B, mask, row, status);
  return 1;
}

int launch_fall_detect(int B, const double* rbd, double z_min, double tilt_max, const SimTerrain& terrain, double ground_height, int32_t* count, int32_t* fallen,
                       cudaStream_t s) {
  fall_detect_kernel<<<(B + FALL_THREADS - 1) / FALL_THREADS, FALL_THREADS, 0, s>>>(B, rbd, z_min, tilt_max, terrain, ground_height, count, fallen);
  return 1;
}

}  // namespace qmb
