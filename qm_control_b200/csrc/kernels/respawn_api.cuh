// Host-visible interface of the per-robot restart (respawn_kernel.cu): the masked row gather behind the start image's restore and the robot-state
// snapshots, and the fall detector on the plant's rbd (include/qmb200.h: qmb200_robot_image_*, qmb200_robot_state_*, qmb200_fall_detect; DESIGN.md §4.10,
// §4.17).
#pragma once
#include <cuda_runtime.h>

#include "../../../include/qmb200.h"
#include "sim_api.cuh"

namespace qmb {

// One block of per-robot rows [B][words] of 4-byte words, written for every masked robot: from src [B][words] (an image or a snapshot), or zeros when
// src is NULL.
struct RestoreSeg { uint32_t* dst; const uint32_t* src; int32_t words; };
constexpr int RESTORE_MAX_SEGS = 40;   // a snapshot with every component running holds 33 blocks; the start image 8 imaged and 5 cold-start blocks
struct RestoreTable { RestoreSeg seg[RESTORE_MAX_SEGS]; int n; };

// The gather rule, one word at a time (the kernel's body; tests/restore_host.cpp builds it with g++).  Robot b is written when mask[b] != 0 (NULL mask:
// every robot) and its source row r = row[b] (NULL row: r = b) lies in [0, B); its word w then becomes src[r][w], or 0 when src is NULL.
QMB_HD bool restore_source(int B, const int32_t* mask, const int32_t* row, int b, int& r) {
  if (mask && !mask[b]) return false;
  r = row ? row[b] : b;
  return r >= 0 && r < B;
}
QMB_HD uint32_t restore_word(const RestoreSeg& g, int r, int64_t w) { return g.src ? g.src[(int64_t)r * g.words + w] : 0u; }
// robot b's status word of a gather: QMB200_ST_RESTORE when it is masked and its source row lies outside [0, B), else 0 (written, not OR-ed)
QMB_HD int32_t restore_status(int B, const int32_t* mask, const int32_t* row, int b) {
  int r = 0;
  return (mask && !mask[b]) || restore_source(B, mask, row, b, r) ? 0 : QMB200_ST_RESTORE;
}

// one launch over every segment of the table: robot b's rows are gathered from source row row[b] (NULL: b) when mask[b] != 0 (NULL: every robot), and
// left alone otherwise or when row[b] lies outside [0, B).  status (NULL: none) [B] receives restore_status.
int launch_image_restore(const RestoreTable& t, int B, const int32_t* mask, cudaStream_t s, const int32_t* row = nullptr, int32_t* status = nullptr);

// one thread per robot on the plant's rbd [B][55]: fallen[b] = 1 when its base rows (zyx, p) hold a non-finite value, p_z - H(p_x, p_y) <= z_min
// (H: the plant's ground under the base) or |pitch|, |roll| >= tilt_max, else 0; count[b] (in-out) grows by one on a fallen call and drops to 0 otherwise
int launch_fall_detect(int B, const double* rbd, double z_min, double tilt_max, const SimTerrain& terrain, double ground_height, int32_t* count, int32_t* fallen,
                       cudaStream_t s);

}  // namespace qmb
