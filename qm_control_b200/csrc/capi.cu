// C-ABI of libqmb200 (include/qmb200.h).  Host logic only: argument checks, device buffers, stream ordering,
// kernel launches.  No CPU fallback: every compute entry point launches the sm_90a kernels or fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/qmb200.h"
#include "host/qm_config.h"
#include "kernels/mpc_api.cuh"
#include "kernels/ctrl_api.cuh"
#include "kernels/sim_api.cuh"
#include "kernels/payload_est_api.cuh"
#include "kernels/state_est_api.cuh"
#include "kernels/attitude_api.cuh"
#include "kernels/slip_api.cuh"
#include "kernels/gait_api.cuh"
#include "kernels/respawn_api.cuh"
#include "kernels/episode_api.cuh"
#include "kernels/spawn_api.cuh"

namespace qmb {
void launch_wbc_update(const DevModel* mdl, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const double* period, const double* time,
                       double* input_last, int variant, double* cmd, int32_t* status, cudaStream_t stream, int b0 = 0, int b1 = -1, int32_t* diag = nullptr,
                       const double* srbd = nullptr, const double* payload = nullptr,    // srbd [B][SRBD_DBL] / payload [B][8]: the model payload (NULL: none)
                       const double* tuning = nullptr);                                  // tuning [B][TUNING_DBL]: the robot tuning rows (NULL: none)
int wbc_configure_device();   // per-device kernel attributes (opt-in shared memory): wbc_kernel.cu / mpc_kernels.cu
int mpc_configure_device();
}

using namespace qmb;

static thread_local std::string g_create_error;

// A per-robot array the kernels read, `width` doubles per robot: the host copy (empty = not set) and its device copy, allocated on the first set.
struct RobotArray {
  int width; std::vector<double> host; double* d = nullptr;
  const double* dev() const { return host.empty() ? nullptr : d; }
};

// Per-robot ranges of a per-episode draw (capi_episode.inc, capi_spawn.inc): lo, hi [B][width] (empty: none set), their device copies (dalloc: freed
// with allocs) and the seed
struct DrawRanges {
  int width; std::vector<double> lo, hi; double *d_lo = nullptr, *d_hi = nullptr; uint64_t seed = 0;
};

// The components a start image covers (capi_respawn.inc).  Each has a generation that its reset, stop and re-allocation bump, so a restore can tell
// that the rows it would write no longer belong to the state it imaged.
enum ImageComponent { IMG_STATE_EST, IMG_ATTITUDE, IMG_SLIP, IMG_PAYLOAD_EST, IMG_MODEL_PAYLOAD, IMG_GAIT, IMG_N };

struct qmb200_handle {
  HostModel hm;
  DevModel* d_model = nullptr;
  int B = 0, nmax = 0, variant = 0, device = 0;
  cudaStream_t stream = nullptr;
  std::string err, task_file, reference_file;   // task_file: qmb200_mpc_set_solver re-reads the sqp{} / ipm{} / ddp{} block; both: qmb200_gait_dev_reset
  int64_t launches = 0;
  // intermediates of the tick and update chains (policy evaluation → WBC → control law), WBC state, and the update chain's safety word
  double *d_xdes = nullptr, *d_udes = nullptr, *d_input_last = nullptr;
  int32_t *d_mode = nullptr, *d_wbc_diag = nullptr, *d_safety = nullptr;   // d_wbc_diag: per-robot WBC iteration counts (qmb200_wbc_get_diagnostics), kept out of the status word
  char* stage = nullptr; size_t stage_bytes = 0;   // device arena of the host-pointer entry points (Staging)
  MpcBuffers mpc;   // device buffers of the MPC path (kernels/mpc_api.cuh)
  std::vector<void*> allocs;
  bool profiling = false; cudaEvent_t ev[8] = {nullptr};   // [0..4] MPC kernels, [5..6] policy / wbc brackets, [7] flow kernel | LQ kernel
  double kernel_ms[7] = {0, 0, 0, 0, 0, 0, 0}; int64_t kernel_calls = 0; bool ev_pending = false;   // kernel_ms[6]: the flow kernel's share of [1]
  // tick pipeline: the batch is cut into `chunks` robot ranges, each running its MPC → policy → WBC chain on its own stream, so that
  // kernels with different bottlenecks (LQ: instruction latency, Riccati: shared-memory bandwidth, WBC) share the SMs
  static constexpr int MAX_CHUNKS = 8;
  TargetParams target_prm{}; ControlLawParams law_prm{0, 0.0, 0.5};   // controller-side constants (capi_ctrl.inc)
  double hw_delay = 0.0; double *hw_ring_cmd = nullptr, *hw_ring_stamp = nullptr; int32_t* hw_ring_state = nullptr;   // QMHWSim command-delay FIFO
  void* comm = nullptr; int comm_ranks = 0, comm_rank = 0; double* d_send = nullptr;   // NCCL communicator of this handle (capi_comm.inc) and the packed torque rows
  SimParams sim_prm{};   // plant step (capi_sim.inc)
  RobotArray mu{1}, payload{8};   // per-robot plant variation (qmb200_sim_set_robot_params)
  RobotArray terrain{3};          // per-robot [tile, origin_x, origin_y] on the tile library (qmb200_sim_set_robot_terrain)
  struct { std::vector<double> host; double* d = nullptr; int n_tiles = 0, nx = 0, ny = 0; double cell = 0.0; } tiles;   // heightfield library (qmb200_sim_set_terrain)
  RobotArray mpayload{8}, srbd{SRBD_DBL};   // the controller's model payload (qmb200_set_model_payload) and the robots' SRBD constants it gives
  RobotArray tuning{TUNING_DBL};            // per-robot controller parameters (qmb200_set_robot_tuning): Tuning, then the control law's arm kp / kd
  qmb200_payload_est_params est_prm{}; double* d_est = nullptr;   // payload estimator (capi_est.inc): parameters and state [B][EST_DBL], NULL when not running
  qmb200_sensor_params sensor_prm{};                               // sensor noise of qmb200_sim_read_sensors (capi_state_est.inc)
  qmb200_state_est_params se_prm{}; double* d_se = nullptr;        // base state estimator: parameters and state [B][SE_DBL], NULL when not running
  RobotArray se_ground{3};        // the estimator's ground map: per-robot [tile, origin_x, origin_y] on the tile library (qmb200_state_est_set_ground)
  qmb200_attitude_params at_prm{}; double* d_at = nullptr;         // attitude filter (capi_attitude.inc): parameters and state [B][AT_DBL], NULL when not running
  qmb200_slip_params sl_prm{}; double* d_sl = nullptr;             // slip detector (capi_slip.inc): parameters and state [B][SL_DBL], NULL when not running
  struct {   // device gait schedule (capi_gait.inc): template table, per-robot state (NULL when not running) and command timeline [B][n_cmd]
    std::vector<GsTemplate> table; GsTemplate* d_table = nullptr; GsRobot* d_robots = nullptr; int32_t* d_cursor = nullptr;
    double* d_t = nullptr; int32_t* d_tmpl = nullptr; double* d_vel = nullptr; int n_cmd = 0; double stance_time = 0.0;
    int32_t* d_ee_kind = nullptr; double* d_ee = nullptr;   // the timeline's end-effector commands [B][n_cmd] and [B][n_cmd][7], NULL when it has none
  } gs;
  bool model_on_device = false;   // a commit wrote mpayload / srbd on the device: model_rows_sync refreshes the host copies before they are read
  bool plant_on_device = false, tuning_on_device = false;   // an episode draw wrote mu / payload or tuning on the device: plant_ / tuning_rows_sync refresh them
  DrawRanges episode{EP_DBL};       // per-episode plant draws (capi_episode.inc)
  bool terrain_on_device = false;   // a spawn wrote the plant's robot terrain / the ground map on the device: terrain_rows_sync refreshes them
  struct SpawnRanges : DrawRanges {   // per-episode spawns (capi_spawn.inc), and device copies of the robots' tile origins at the set [B][2] and the
                                      // standing pose's joints [NJ]; terrain: the plant had robot terrain rows at the set
    double *d_origin = nullptr, *d_qj = nullptr; bool terrain = false;
  } spawn{{SP_DBL}};
  uint64_t gen[IMG_N] = {};       // generation of each imaged component (ImageComponent)
  struct {                        // start image (qmb200_robot_image_save): the running components' rows, one block after the other in d
    bool saved = false; char* d = nullptr; bool on[IMG_N] = {}; uint64_t gen[IMG_N] = {};
  } image;
  int chunks = 1; cudaStream_t cs[MAX_CHUNKS] = {nullptr}; cudaEvent_t fork_ev = nullptr, join_ev[MAX_CHUNKS] = {nullptr};
};

namespace {
template <class T> bool dalloc(qmb200_handle* h, T** p, size_t count) {
  void* q = nullptr; cudaError_t e = cudaMalloc(&q, count * sizeof(T));
  if (e != cudaSuccess) { h->err = std::string("cudaMalloc failed: ") + cudaGetErrorString(e); return false; }
  cudaMemsetAsync(q, 0, count * sizeof(T), h->stream); h->allocs.push_back(q); *p = static_cast<T*>(q); return true;   // zeroed in stream order with the handle's work
}
SimParams default_sim_params();   // capi_sim.inc
qmb200_payload_est_params default_est_params();   // capi_est.inc
qmb200_state_est_params default_state_est_params(const DevModel& d);   // capi_state_est.inc
qmb200_attitude_params default_attitude_params();   // capi_attitude.inc
qmb200_slip_params default_slip_params();   // capi_slip.inc
int fail(qmb200_handle* h, const std::string& msg) { if (h) h->err = msg; else g_create_error = msg; return -1; }
#define QMB_CUDA(h, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(h, std::string(#call) + ": " + cudaGetErrorString(e_)); } while (0)

// The model a config describes: the default WBC gains unless a gains file is given, time_horizon / dt overridden when > 0.
HostModel config_model(const qmb200_config* cfg) {
  HostModel hm = build_host_model(cfg->task_file, cfg->urdf_file, cfg->reference_file, cfg->wbc_gains_file ? cfg->wbc_gains_file : "");
  if (cfg->time_horizon > 0) hm.dev.time_horizon = cfg->time_horizon;
  if (cfg->dt > 0) hm.dev.dt = cfg->dt;
  return hm;
}
// Stream-ordered update of the replicated constants from h->hm.dev: kernels already queued keep the old values, later ones see the new.
int push_model(qmb200_handle* h) {
  QMB_CUDA(h, cudaMemcpyAsync(h->d_model, &h->hm.dev, sizeof(DevModel), cudaMemcpyHostToDevice, h->stream)); QMB_CUDA(h, cudaStreamSynchronize(h->stream)); return 0;
}

// Sets each array to `rows` ([B][width]; NULL clears it).  Work still queued on any stream may read the current device copies, so the copy waits
// for the device.  On failure the host copies, which say what is set, stay unchanged.
struct RobotRows { RobotArray* a; const double* rows; };
int set_robot_arrays(qmb200_handle* h, std::initializer_list<RobotRows> sets) {
  const size_t B = (size_t)h->B;
  QMB_CUDA(h, cudaSetDevice(h->device));
  for (const RobotRows& s : sets) if (s.rows && !s.a->d && !dalloc(h, &s.a->d, B * s.a->width)) return -4;
  QMB_CUDA(h, cudaDeviceSynchronize());
  for (const RobotRows& s : sets) if (s.rows) QMB_CUDA(h, cudaMemcpy(s.a->d, s.rows, B * s.a->width * 8, cudaMemcpyHostToDevice));
  for (const RobotRows& s : sets) { if (s.rows) s.a->host.assign(s.rows, s.rows + B * s.a->width); else s.a->host.clear(); }
  return 0;
}

// A host-pointer entry point is its _dev twin on the handle's stream, with the caller's arrays staged through one device arena per handle:
// in() copies an array to the device, inout() also copies it back after the call, out() only copies it back.  done(rc) queues the copies back,
// waits for the stream and reports the first CUDA error; when the _dev call failed it returns that call's code and copies nothing back.
// Every array declared out must be written in full by the kernels, since the arena holds whatever the previous call left there.
class Staging {
 public:
  // The widest entry point, qmb200_control_law, stages 242 doubles and one int32 per robot (qmb200_update: 238 and one); each of its at most
  // STAGE_SLICES slices starts on a 256-byte boundary, the alignment cudaMalloc gives.
  static constexpr size_t ROBOT_BYTES = 243 * 8, ALIGN = 256, STAGE_SLICES = 10;
  explicit Staging(qmb200_handle* h) : h_(h) {}
  int open() {
    QMB_CUDA(h_, cudaSetDevice(h_->device));
    if (!h_->stage) {
      const size_t bytes = (size_t)h_->B * ROBOT_BYTES + STAGE_SLICES * ALIGN;
      if (!dalloc(h_, &h_->stage, bytes)) return -4;   // zeroed on h->stream, the only stream that uses the arena
      h_->stage_bytes = bytes;
    }
    return 0;
  }
  template <class T> const T* in(const T* src, size_t n) {
    if (!src) return nullptr;
    T* d = slice<T>(n); note(cudaMemcpyAsync(d, src, n * sizeof(T), cudaMemcpyHostToDevice, h_->stream)); return d;
  }
  template <class T> T* inout(T* p, size_t n) { T* d = const_cast<T*>(in<T>(p, n)); back_.push_back({p, d, n * sizeof(T)}); return d; }
  template <class T> T* out(T* p, size_t n) { T* d = slice<T>(n); back_.push_back({p, d, n * sizeof(T)}); return d; }
  int done(int rc) {
    if (rc) return rc;
    for (const Back& b : back_) note(cudaMemcpyAsync(b.host, b.dev, b.bytes, cudaMemcpyDeviceToHost, h_->stream));
    note(cudaStreamSynchronize(h_->stream));
    return err_.empty() ? 0 : fail(h_, err_);
  }

 private:
  struct Back { void* host; const void* dev; size_t bytes; };
  qmb200_handle* h_; size_t used_ = 0; std::vector<Back> back_; std::string err_;
  void note(cudaError_t e) { if (e != cudaSuccess && err_.empty()) err_ = std::string("staging copy: ") + cudaGetErrorString(e); }
  template <class T> T* slice(size_t n) {
    const size_t at = used_, bytes = n * sizeof(T);
    if (at + bytes > h_->stage_bytes) { if (err_.empty()) err_ = "staging arena too small"; return reinterpret_cast<T*>(h_->stage); }
    used_ = (at + bytes + ALIGN - 1) / ALIGN * ALIGN; return reinterpret_cast<T*>(h_->stage + at);
  }
};

// WbcBase::update of robots [b0, b1) with the handle's model, WBC state (input_last, diagnostics), model payload and robot tuning rows
void wbc_launch(qmb200_handle* h, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const double* period, const double* time, double* cmd,
                int32_t* status, cudaStream_t s, int b0 = 0, int b1 = -1) {
  launch_wbc_update(h->d_model, h->B, x_des, u_des, rbd, mode, period, time, h->d_input_last, h->variant, cmd, status, s, b0, b1, h->d_wbc_diag, h->srbd.dev(), h->mpayload.dev(), h->tuning.dev());
  h->launches += 1;
}
}  // namespace

extern "C" {

int qmb200_create(const qmb200_config* cfg, qmb200_handle** out) {
  if (!cfg || !out) return fail(nullptr, "qmb200_create: null argument");
  if (!cfg->task_file || !cfg->urdf_file || !cfg->reference_file) return fail(nullptr, "qmb200_create: task/urdf/reference file required");
  if (cfg->batch < 1) return fail(nullptr, "qmb200_create: batch must be >= 1");
  qmb200_handle* h = new qmb200_handle();
  try {
    h->hm = config_model(cfg);
    // constants of the target publisher node (QmTargetTrajectoriesPublisher_node.cpp:225-229)
    InfoFile ref(cfg->reference_file), task(cfg->task_file);
    h->target_prm.com_height = ref.number("comHeight"); h->target_prm.target_displacement_velocity = ref.number("targetDisplacementVelocity");
    h->target_prm.target_rotation_velocity = ref.number("targetRotationVelocity"); h->target_prm.time_to_target = task.number("mpc.timeHorizon");
    for (int j = 0; j < NJ; ++j) h->target_prm.default_joint_state[j] = h->hm.default_joint_state[j];
  } catch (const std::exception& e) { g_create_error = e.what(); delete h; return -2; }
  h->task_file = cfg->task_file; h->reference_file = cfg->reference_file;
  h->sim_prm = default_sim_params(); h->est_prm = default_est_params(); h->se_prm = default_state_est_params(h->hm.dev); h->at_prm = default_attitude_params();
  h->sl_prm = default_slip_params();
  h->B = cfg->batch; h->variant = cfg->wbc_variant; h->device = cfg->device; h->law_prm.variant = cfg->wbc_variant == QMB200_WBC_HIERARCHICAL_MPC ? 1 : 0;
  const int nint = (int)std::ceil(h->hm.dev.time_horizon / h->hm.dev.dt - 1e-9);
  h->nmax = cfg->max_nodes > 0 ? cfg->max_nodes : nint + 1 + 20;
  int ndev = 0; cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) { g_create_error = std::string("qmb200_create: no CUDA device (") + cudaGetErrorString(e) + ") — this library has no CPU fallback"; delete h; return -3; }
  if (cudaSetDevice(cfg->device) != cudaSuccess) { g_create_error = "qmb200_create: cudaSetDevice failed"; delete h; return -3; }
  cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  // kernel attributes are per device: set them for THIS handle's device (a process may hold handles on several GPUs)
  if (wbc_configure_device() != 0 || mpc_configure_device() != 0) { g_create_error = std::string("qmb200_create: cudaFuncSetAttribute failed: ") + cudaGetErrorString(cudaGetLastError()); qmb200_destroy(h); return -3; }
  const size_t B = (size_t)h->B;
  bool ok = dalloc(h, &h->d_model, 1) && dalloc(h, &h->d_xdes, B * NX) && dalloc(h, &h->d_udes, B * NU) && dalloc(h, &h->d_input_last, B * NU) && dalloc(h, &h->d_mode, B) &&
            dalloc(h, &h->d_wbc_diag, B) && dalloc(h, &h->d_safety, B) && dalloc(h, &h->d_send, B * NJ);
  if (ok) { std::string merr; ok = mpc_alloc(h->mpc, h->B, h->nmax, merr, h->allocs, h->stream); if (!ok) h->err = merr; }
  if (!ok) { g_create_error = h->err; qmb200_destroy(h); return -4; }
  if (push_model(h)) { g_create_error = "qmb200_create: " + h->err; qmb200_destroy(h); return -4; }   // buffers zeroed, constants resident before any (user-stream) launch
  *out = h; return 0;
}

void qmb200_destroy(qmb200_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  qmb200_comm_destroy(h);
  if (h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
  for (int c = 0; c < qmb200_handle::MAX_CHUNKS; ++c) { if (h->cs[c]) { cudaStreamSynchronize(h->cs[c]); cudaStreamDestroy(h->cs[c]); } if (h->join_ev[c]) cudaEventDestroy(h->join_ev[c]); }
  if (h->fork_ev) cudaEventDestroy(h->fork_ev);
  for (void* p : h->allocs) cudaFree(p);
  if (h->tiles.d) cudaFree(h->tiles.d);
  if (h->d_est) cudaFree(h->d_est);
  if (h->d_se) cudaFree(h->d_se);
  if (h->d_at) cudaFree(h->d_at);
  if (h->d_sl) cudaFree(h->d_sl);
  cudaFree(h->gs.d_table); cudaFree(h->gs.d_robots); cudaFree(h->gs.d_cursor); cudaFree(h->gs.d_t); cudaFree(h->gs.d_tmpl); cudaFree(h->gs.d_vel);
  cudaFree(h->gs.d_ee_kind); cudaFree(h->gs.d_ee);
  cudaFree(h->image.d);
  delete h;
}

const char* qmb200_last_error(const qmb200_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int64_t qmb200_debug_model_blob(const qmb200_config* cfg, void* out, int64_t capacity) {
  if (!cfg || !cfg->task_file || !cfg->urdf_file || !cfg->reference_file) { g_create_error = "qmb200_debug_model_blob: task/urdf/reference file required"; return -1; }
  try {
    const HostModel hm = config_model(cfg);
    if (out && capacity >= (int64_t)sizeof(DevModel)) std::memcpy(out, &hm.dev, sizeof(DevModel));
    return (int64_t)sizeof(DevModel);
  } catch (const std::exception& e) { g_create_error = e.what(); return -2; }
}

// ------------------------------------------------------------------ model payload
static_assert(SRBD_DBL == QMB200_SRBD, "per-robot SRBD block of include/qmb200.h");
static_assert(RBD_EE_QUAT + 4 == QMB200_RBD, "rbd layout of include/qmb200.h");
}  // extern "C"
namespace {
// payload rows [n][8] as qmb200_sim_set_robot_params and qmb200_set_model_payload accept them: finite, masses >= 0; "" when valid
std::string payload_error(const double* payload, size_t n, const char* who) {
  for (size_t b = 0; b < n; ++b) {
    const double* p = payload + 8 * b;
    for (int i = 0; i < 8; ++i) if (!std::isfinite(p[i])) return std::string(who) + ": payload must be finite";
    if (p[0] < 0.0 || p[4] < 0.0) return std::string(who) + ": payload masses must be >= 0";
  }
  return "";
}
// After a kernel wrote robot rows on the device (a payload estimator commit, a restore, an episode draw) the device holds them: when on_device says so,
// wait for it and copy them into the host copies, which say what is set and what the getters report
int rows_sync(qmb200_handle* h, bool& on_device, std::initializer_list<RobotArray*> arrays) {
  if (!on_device) return 0;
  QMB_CUDA(h, cudaSetDevice(h->device)); QMB_CUDA(h, cudaDeviceSynchronize());
  for (RobotArray* a : arrays) if (!a->host.empty()) QMB_CUDA(h, cudaMemcpy(a->host.data(), a->d, a->host.size() * 8, cudaMemcpyDeviceToHost));
  on_device = false; return 0;
}
int model_rows_sync(const qmb200_handle* hc) { qmb200_handle* h = const_cast<qmb200_handle*>(hc); return rows_sync(h, h->model_on_device, {&h->mpayload, &h->srbd}); }
int plant_rows_sync(const qmb200_handle* hc) { qmb200_handle* h = const_cast<qmb200_handle*>(hc); return rows_sync(h, h->plant_on_device, {&h->mu, &h->payload}); }
int tuning_rows_sync(const qmb200_handle* hc) { qmb200_handle* h = const_cast<qmb200_handle*>(hc); return rows_sync(h, h->tuning_on_device, {&h->tuning}); }
int terrain_rows_sync(const qmb200_handle* hc) { qmb200_handle* h = const_cast<qmb200_handle*>(hc); return rows_sync(h, h->terrain_on_device, {&h->terrain, &h->se_ground}); }
// The ranged draws' set / get / draw path (qmb200_<kind>_set_ranges, _get_ranges, _draw; kind: "episode" or "spawn").
// Set: NULL lo and hi clear the ranges once no queued draw reads them; else error() checks them ("" when valid), the device copies are allocated, then
// prepare() makes sure the rows the sampler writes exist (it may fail, leaving the ranges as they were), and the ranges are copied and stored.
template <class Error, class Prepare>
int ranges_set(qmb200_handle* h, DrawRanges& r, const char* kind, const double* lo, const double* hi, int64_t seed, Error error, Prepare prepare) {
  const std::string who = std::string("qmb200_") + kind + "_set_ranges"; const size_t n = (size_t)h->B * r.width;
  if (!lo != !hi) return fail(h, who + ": lo and hi must both be set or both be NULL");
  if (!lo) {
    QMB_CUDA(h, cudaSetDevice(h->device)); QMB_CUDA(h, cudaDeviceSynchronize());   // no queued draw still reads the ranges
    r.lo.clear(); r.hi.clear(); r.seed = 0; return 0;
  }
  if (const std::string e = error(); !e.empty()) return fail(h, e);
  QMB_CUDA(h, cudaSetDevice(h->device));
  if (!r.d_lo && !dalloc(h, &r.d_lo, n)) return -4;
  if (!r.d_hi && !dalloc(h, &r.d_hi, n)) return -4;
  if (int rc = prepare()) return rc;
  QMB_CUDA(h, cudaDeviceSynchronize());   // no queued draw still reads the ranges
  QMB_CUDA(h, cudaMemcpy(r.d_lo, lo, n * 8, cudaMemcpyHostToDevice)); QMB_CUDA(h, cudaMemcpy(r.d_hi, hi, n * 8, cudaMemcpyHostToDevice));
  r.lo.assign(lo, lo + n); r.hi.assign(hi, hi + n); r.seed = (uint64_t)seed;
  return 0;
}
int ranges_get(const qmb200_handle* h, const DrawRanges& r, double* lo, double* hi, int64_t* seed, int32_t* is_set) {
  const size_t n = (size_t)h->B * r.width; const bool set = !r.lo.empty();
  if (lo) { if (set) std::memcpy(lo, r.lo.data(), n * 8); else std::memset(lo, 0, n * 8); }
  if (hi) { if (set) std::memcpy(hi, r.hi.data(), n * 8); else std::memset(hi, 0, n * 8); }
  if (seed) *seed = (int64_t)r.seed;
  if (is_set) *is_set = set ? 1 : 0;
  return 0;
}
int no_ranges(qmb200_handle* h, const char* who, const char* kind) {
  return fail(h, std::string(who) + ": no ranges are set (qmb200_" + kind + "_set_ranges sets them)");
}
// The rows [n][width] robots robot [n] draw in episodes episode [n] on the stored ranges, each row(lo, hi, seed, global robot, episode, out) on the host
int ranges_draw(qmb200_handle* h, const DrawRanges& r, const char* kind, int32_t n, const int32_t* robot, const int32_t* episode, double* rows,
                void (*row)(const double*, const double*, uint64_t, uint64_t, uint64_t, double*)) {
  const std::string who = std::string("qmb200_") + kind + "_draw";
  if (n < 0 || (n > 0 && (!robot || !episode || !rows))) return fail(h, who + ": n must be >= 0 and the buffers non-null");
  if (r.lo.empty()) return no_ranges(h, who.c_str(), kind);
  for (int32_t i = 0; i < n; ++i) if (robot[i] < 0 || robot[i] >= h->B) return fail(h, who + ": robot must be in [0, B)");
  const int64_t robot0 = (int64_t)h->comm_rank * h->B;
  for (int32_t i = 0; i < n; ++i) {
    const size_t b = (size_t)robot[i];
    row(r.lo.data() + b * r.width, r.hi.data() + b * r.width, r.seed, (uint64_t)(robot0 + robot[i]), (uint64_t)(int64_t)episode[i], rows + (size_t)i * r.width);
  }
  return 0;
}
// SRBD constants of n robots with payload rows [n][8] (NULL: none)
void srbd_rows(const HostModel& hm, const double* payload, size_t n, double* out) {
  for (size_t b = 0; b < n; ++b) srbd_constants(hm.dev, payload ? payload + 8 * b : nullptr, out + SRBD_DBL * b);
}
}  // namespace
extern "C" {

int qmb200_set_model_payload(qmb200_handle* h, const double* payload) {
  if (!h) return -1; const size_t B = (size_t)h->B;
  if (payload) { const std::string e = payload_error(payload, B, "qmb200_set_model_payload"); if (!e.empty()) return fail(h, e); }
  std::vector<double> srbd; if (payload) { srbd.resize(B * SRBD_DBL); srbd_rows(h->hm, payload, B, srbd.data()); }
  const int rc = set_robot_arrays(h, {{&h->mpayload, payload}, {&h->srbd, payload ? srbd.data() : nullptr}});
  if (!rc) h->model_on_device = false;   // set_robot_arrays waited for the device: the rows just written replace any committed ones
  h->gen[IMG_MODEL_PAYLOAD] += 1;
  return rc;
}
int qmb200_get_model_payload(const qmb200_handle* h, double* payload, int32_t* is_set) {
  if (!h) return -1; const size_t B = (size_t)h->B;
  if (int rc = model_rows_sync(h)) return rc;
  const std::vector<double>& p = h->mpayload.host;
  if (payload) { if (p.empty()) std::memset(payload, 0, B * 64); else std::memcpy(payload, p.data(), B * 64); }
  if (is_set) *is_set = p.empty() ? 0 : 1;
  return 0;
}
int qmb200_debug_srbd_constants(const qmb200_config* cfg, int32_t n, const double* payload, double* out) {
  if (!cfg || !cfg->task_file || !cfg->urdf_file || !cfg->reference_file) { g_create_error = "qmb200_debug_srbd_constants: task/urdf/reference file required"; return -1; }
  if (n < 0 || (n > 0 && !out)) { g_create_error = "qmb200_debug_srbd_constants: n must be >= 0 and out non-null"; return -1; }
  if (payload) { const std::string e = payload_error(payload, (size_t)n, "qmb200_debug_srbd_constants"); if (!e.empty()) { g_create_error = e; return -1; } }
  try {
    srbd_rows(config_model(cfg), payload, (size_t)n, out);
    return 0;
  } catch (const std::exception& e) { g_create_error = e.what(); return -2; }
}

// ------------------------------------------------------------------ robot tuning
static_assert(TUNING_DBL == QMB200_TUNING && TUNING_MODEL == 6 + sizeof(qmb200_wbc_gains) / 8, "tuning row of include/qmb200.h: Tuning, then the two arm gains");
}  // extern "C"
namespace {
// Field names of a tuning row (include/qmb200.h), for the validation messages; the 32 WBC gains in qmb200_wbc_gains order
const char* tuning_field(int i) {
  static const char* const head[14] = {"friction_mu", "wbc_friction", "mu_ee_pos", "mu_ee_ori", "mu_final_ee_pos", "mu_final_ee_ori", "kp_swing", "kd_swing",
                                       "base_height_kp", "base_height_kd", "kp_base_linear", "kd_base_linear", "kp_base_angular", "kd_base_angular"};
  static const char* const vec[6] = {"kp_arm_joint", "kd_arm_joint", "kp_ee_linear", "kd_ee_linear", "kp_ee_angular", "kd_ee_angular"};
  static const int start[7] = {14, 20, 26, 29, 32, 35, 38};
  static thread_local std::string name;
  if (i < 14) return head[i];
  if (i == TUNING_ARM_KP) return "kp_arm_wbc";
  if (i == TUNING_ARM_KD) return "kd_arm_wbc";
  int v = 0; while (i >= start[v + 1]) ++v;
  name = std::string(vec[v]) + "[" + std::to_string(i - start[v]) + "]"; return name.c_str();
}
// the handle's values as one tuning row: DevModel's tuned block and the control law's arm gains
void handle_tuning(const qmb200_handle* h, double* row) {
  std::memcpy(row, tuning_of(&h->hm.dev, nullptr, 0), sizeof(Tuning)); row[TUNING_ARM_KP] = h->law_prm.arm_kp; row[TUNING_ARM_KD] = h->law_prm.arm_kd;
}
}  // namespace
extern "C" {

int qmb200_set_robot_tuning(qmb200_handle* h, const double* rows) {
  if (!h) return -1; const size_t B = (size_t)h->B;
  if (rows) for (size_t b = 0; b < B; ++b) for (int i = 0; i < TUNING_DBL; ++i) {
    const double v = rows[b * TUNING_DBL + i];
    const char* why = !std::isfinite(v) ? "must be finite" : (i < 2 && !(v > 0.0)) ? "must be > 0" : (v < 0.0) ? "must be >= 0" : nullptr;
    if (why) return fail(h, std::string("qmb200_set_robot_tuning: ") + tuning_field(i) + " of robot " + std::to_string(b) + " " + why);
  }
  const int rc = set_robot_arrays(h, {{&h->tuning, rows}});
  if (!rc) h->tuning_on_device = false;   // set_robot_arrays waited for the device: the rows just written replace any drawn ones
  return rc;
}
int qmb200_get_robot_tuning(const qmb200_handle* h, double* rows, int32_t* is_set) {
  if (!h) return -1; const size_t B = (size_t)h->B;
  if (int rc = tuning_rows_sync(h)) return rc;
  const std::vector<double>& t = h->tuning.host;
  if (rows) { if (t.empty()) for (size_t b = 0; b < B; ++b) handle_tuning(h, rows + b * TUNING_DBL); else std::memcpy(rows, t.data(), B * TUNING_DBL * 8); }
  if (is_set) *is_set = t.empty() ? 0 : 1;
  return 0;
}
int qmb200_get_handle_tuning(const qmb200_handle* h, double* row) {
  if (!h) return -1; if (!row) return fail(const_cast<qmb200_handle*>(h), "qmb200_get_handle_tuning: null row");
  handle_tuning(h, row); return 0;
}

int qmb200_get_dims(const qmb200_handle* h, int32_t* batch, int32_t* nmax, int32_t* emax, int32_t* kmax) {
  if (!h) return -1; if (batch) *batch = h->B; if (nmax) *nmax = h->nmax; if (emax) *emax = QMB200_EMAX; if (kmax) *kmax = QMB200_KMAX; return 0;
}
int qmb200_get_model_info(const qmb200_handle* h, double* robot_mass, double* initial_state30, double* default_joint_state18, double* time_horizon, double* dt) {
  if (!h) return -1;
  if (robot_mass) *robot_mass = h->hm.dev.total_mass;
  if (initial_state30) std::memcpy(initial_state30, h->hm.initial_state, sizeof(double) * NX);
  if (default_joint_state18) std::memcpy(default_joint_state18, h->hm.default_joint_state, sizeof(double) * NJ);
  if (time_horizon) *time_horizon = h->hm.dev.time_horizon; if (dt) *dt = h->hm.dev.dt; return 0;
}
int qmb200_get_joint_name(const qmb200_handle* h, int32_t joint, char* out, int32_t capacity) {
  if (!h || joint < 0 || joint >= NJ || !out || capacity < 1) return -1; std::snprintf(out, capacity, "%s", h->hm.joint_names[joint].c_str()); return 0;
}
int64_t qmb200_launch_count(const qmb200_handle* h) { return h ? h->launches : 0; }
void* qmb200_stream(const qmb200_handle* h) { return h ? (void*)h->stream : nullptr; }

// ------------------------------------------------------------------ WBC
int qmb200_wbc_update_dev(qmb200_handle* h, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const double* period, const double* time,
                          double* cmd, int32_t* status, void* cuda_stream) {
  if (!h) return -1; if (!x_des || !u_des || !rbd || !mode || !period || !time || !cmd || !status) return fail(h, "qmb200_wbc_update_dev: null buffer");
  QMB_CUDA(h, cudaSetDevice(h->device));
  wbc_launch(h, x_des, u_des, rbd, mode, period, time, cmd, status, cuda_stream ? (cudaStream_t)cuda_stream : h->stream);
  QMB_CUDA(h, cudaGetLastError());
  return 0;
}

int qmb200_wbc_update(qmb200_handle* h, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const double* period, const double* time, double* cmd, int32_t* status) {
  if (!h) return -1; if (!x_des || !u_des || !rbd || !mode || !period || !time || !cmd || !status) return fail(h, "qmb200_wbc_update: null buffer");
  Staging st(h); if (int rc = st.open()) return rc; const size_t B = (size_t)h->B;
  return st.done(qmb200_wbc_update_dev(h, st.in(x_des, B * NX), st.in(u_des, B * NU), st.in(rbd, B * QMB200_RBD), st.in(mode, B), st.in(period, B), st.in(time, B),
                                       st.out(cmd, B * QMB200_CMD), st.out(status, B), h->stream));
}
int qmb200_wbc_set_input_last(qmb200_handle* h, const double* input_last) {
  if (!h) return -1; QMB_CUDA(h, cudaSetDevice(h->device));
  if (input_last) QMB_CUDA(h, cudaMemcpyAsync(h->d_input_last, input_last, (size_t)h->B * NU * 8, cudaMemcpyHostToDevice, h->stream)); else QMB_CUDA(h, cudaMemsetAsync(h->d_input_last, 0, (size_t)h->B * NU * 8, h->stream));
  QMB_CUDA(h, cudaStreamSynchronize(h->stream)); return 0;
}
int qmb200_wbc_get_input_last(qmb200_handle* h, double* input_last) {
  if (!h || !input_last) return -1; QMB_CUDA(h, cudaSetDevice(h->device));
  QMB_CUDA(h, cudaMemcpyAsync(input_last, h->d_input_last, (size_t)h->B * NU * 8, cudaMemcpyDeviceToHost, h->stream)); QMB_CUDA(h, cudaStreamSynchronize(h->stream)); return 0;
}

int qmb200_wbc_get_gains(const qmb200_handle* h, qmb200_wbc_gains* g) {
  if (!h || !g) return -1; const DevModel& d = h->hm.dev;
  g->kp_swing = d.kp_swing; g->kd_swing = d.kd_swing; g->base_height_kp = d.base_height_kp; g->base_height_kd = d.base_height_kd; g->kp_base_linear = d.base_linear_kp; g->kd_base_linear = d.base_linear_kd;
  g->kp_base_angular = d.base_angular_kp; g->kd_base_angular = d.base_angular_kd;
  for (int i = 0; i < 6; ++i) { g->kp_arm_joint[i] = d.arm_joint_kp[i]; g->kd_arm_joint[i] = d.arm_joint_kd[i]; }
  for (int i = 0; i < 3; ++i) { g->kp_ee_linear[i] = d.ee_linear_kp[i]; g->kd_ee_linear[i] = d.ee_linear_kd[i]; g->kp_ee_angular[i] = d.ee_angular_kp[i]; g->kd_ee_angular[i] = d.ee_angular_kd[i]; }
  return 0;
}
// the handle's gains: robots with a tuning row (qmb200_set_robot_tuning) use the row's instead until the rows are cleared
int qmb200_wbc_set_gains(qmb200_handle* h, const qmb200_wbc_gains* g) {
  if (!h) return -1; if (!g) return fail(h, "qmb200_wbc_set_gains: null gains");
  QMB_CUDA(h, cudaSetDevice(h->device)); DevModel& d = h->hm.dev;
  d.kp_swing = g->kp_swing; d.kd_swing = g->kd_swing; d.base_height_kp = g->base_height_kp; d.base_height_kd = g->base_height_kd; d.base_linear_kp = g->kp_base_linear; d.base_linear_kd = g->kd_base_linear;
  d.base_angular_kp = g->kp_base_angular; d.base_angular_kd = g->kd_base_angular;
  for (int i = 0; i < 6; ++i) { d.arm_joint_kp[i] = g->kp_arm_joint[i]; d.arm_joint_kd[i] = g->kd_arm_joint[i]; }
  for (int i = 0; i < 3; ++i) { d.ee_linear_kp[i] = g->kp_ee_linear[i]; d.ee_linear_kd[i] = g->kd_ee_linear[i]; d.ee_angular_kp[i] = g->kp_ee_angular[i]; d.ee_angular_kd[i] = g->kd_ee_angular[i]; }
  return push_model(h);
}

// Per-robot WBC diagnostics of the last update on this handle: it0 | it1 << 8 | it2 << 16 | nw << 24 (level-0 semismooth passes, active-set iterations of
// levels 1 and 2, final working-set size).  They used to ride in the status word, where they collided with the MPC / safety bits.
int qmb200_wbc_get_diagnostics(qmb200_handle* h, int32_t* diag) {
  if (!h || !diag) return -1; QMB_CUDA(h, cudaSetDevice(h->device));
  QMB_CUDA(h, cudaMemcpyAsync(diag, h->d_wbc_diag, (size_t)h->B * 4, cudaMemcpyDeviceToHost, h->stream)); QMB_CUDA(h, cudaStreamSynchronize(h->stream)); return 0;
}
// Iteration caps of the WBC solver (defaults 30 / 80; robots that hit a cap carry QMB200_ST_ITER_CAP).  <= 0 keeps the current value.
int qmb200_wbc_set_iteration_caps(qmb200_handle* h, int32_t level0_passes, int32_t active_set_iterations) {
  if (!h) return -1; QMB_CUDA(h, cudaSetDevice(h->device));
  if (level0_passes > 0) h->hm.dev.wbc_iter_cap0 = level0_passes; if (active_set_iterations > 0) h->hm.dev.wbc_iter_cap = active_set_iterations;
  return push_model(h);
}

}  // extern "C"

#include "capi_mpc.inc"
#include "capi_ctrl.inc"
#include "capi_comm.inc"
#include "capi_sim.inc"
#include "capi_est.inc"
#include "capi_state_est.inc"
#include "capi_attitude.inc"
#include "capi_slip.inc"
#include "capi_gait.inc"
#include "capi_respawn.inc"
#include "capi_episode.inc"
#include "capi_spawn.inc"
