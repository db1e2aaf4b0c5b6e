// Host-visible interface of the per-robot restart (respawn_kernel.cu): the masked restore of a start image of every component's per-robot rows and
// the fall detector on the plant's rbd (include/qmb200.h: qmb200_robot_image_*, qmb200_fall_detect; DESIGN.md §4.10).
#pragma once
#include <cuda_runtime.h>

#include "sim_api.cuh"

namespace qmb {

// One block of per-robot rows [B][words] of 4-byte words, written for every masked robot: from src [B][words] (the image), or zeros when src is NULL.
struct RestoreSeg { uint32_t* dst; const uint32_t* src; int32_t words; };
constexpr int RESTORE_MAX_SEGS = 16;   // 8 imaged blocks when every component runs, 5 cold-start blocks
struct RestoreTable { RestoreSeg seg[RESTORE_MAX_SEGS]; int n; };

// one launch over every segment of the table: robot b's rows are written when mask[b] != 0, and left alone otherwise
int launch_image_restore(const RestoreTable& t, int B, const int32_t* mask, cudaStream_t s);

// one thread per robot on the plant's rbd [B][55]: fallen[b] = 1 when its base rows (zyx, p) hold a non-finite value, p_z - H(p_x, p_y) <= z_min
// (H: the plant's ground under the base) or |pitch|, |roll| >= tilt_max, else 0; count[b] (in-out) grows by one on a fallen call and drops to 0 otherwise
int launch_fall_detect(int B, const double* rbd, double z_min, double tilt_max, const SimTerrain& terrain, double ground_height, int32_t* count, int32_t* fallen,
                       cudaStream_t s);

}  // namespace qmb
