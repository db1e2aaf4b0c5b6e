/* qmb200 — C ABI of the H100-native batched MPC+WBC solver (drop-in for qm_control's per-tick numerical path).
 *
 * Every entry point replaces one reference interface; the thin C++ subclasses a maintainer adds on the
 * reference side (B200Wbc : qm::WbcBase, B200Mpc : ocs2::MPC_BASE) are shown in INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes only; return 0 on success, negative on error (never throws);
 * qmb200_last_error() describes the last failure; the caller owns every buffer it passes; `_dev` variants
 * take device pointers and a cudaStream_t (as void*) and do not synchronise; one handle per GPU, calls on
 * one handle are serialised on its stream; batch = 1 works (plugin use).  All arithmetic is fp64
 * (ocs2::scalar_t).  Layouts are robot-major, fixed stride:
 *   state x[30]  = [h_lin/m(3), h_ang/m(3), base pos(3), base euler ZYX(3), joints(18: LF,LH,RF,RH,arm)]   task.info:150-189
 *   input u[30]  = [contact forces(12: LF,RF,LH,RH), joint velocities(18)]                                  task.info:252-286
 *   rbd[55]      = [euler ZYX(3), pos(3), joints(18), w_world(3), v_lin(3), joint vel(18), ee pos(3), ee quat xyzw(4)]
 *                                                                                  qm_estimation/src/StateEstimateBase.cpp:41-103
 *   cmd[54]      = [vdot(24), F(12), tau(18)]                                      qm_wbc/src/WbcBase.cpp:548-563
 *   mode         = 4-bit stance code LF=8 RF=4 LH=2 RH=1 (ocs2_legged_robot MotionPhaseDefinition)
 */
#ifndef QMB200_H
#define QMB200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QMB200_NX 30
#define QMB200_NU 30
#define QMB200_RBD 55
#define QMB200_CMD 54
#define QMB200_TARGET 37   /* 30-dim state + end-effector pose [pos(3), quat xyzw(4)] (QMController.cpp:106-112) */
#define QMB200_EMAX 32     /* max events of one robot's mode schedule window */
#define QMB200_KMAX 4      /* max knots of one robot's target trajectory */

#define QMB200_WBC_HIERARCHICAL 0      /* qm::HierarchicalWbc      (qm_wbc/src/HierarchicalWbc.cpp:18-44)    */
#define QMB200_WBC_HIERARCHICAL_MPC 1  /* qm::HierarchicalMpcWbc   (qm_wbc/src/HierarchicalMpcWbc.cpp:18-34) */

/* per-robot status bits (the reference ignores solver status, HoQp.cpp:143; here it is reported).
 * Layout of a status word:  bits 0..7   WBC flags (QMB200_ST_ITER_CAP | _OVERFLOW | _NAN) — qmb200_wbc_update, qmb200_update, qmb200_tick
 *                           bits 8..15  MPC flags shifted left by 8 — only in the merged word qmb200_tick / qmb200_tick_dev return
 *                                       (qmb200_mpc_solve / qmb200_mpc_get_solution report the MPC flags unshifted in their own status array)
 *                           bit 16      QMB200_ST_SAFETY — qmb200_update / qmb200_control_law
 *                           bit 17      QMB200_ST_COMMAND — qmb200_gait_dev_command(_dev), a rejected command row
 *                           bit 18      QMB200_ST_RESTORE — qmb200_robot_state_load(_dev), a source robot outside [0, B)
 *                           bit 19      QMB200_ST_SPAWN — qmb200_spawn_place(_dev), a rejected spawn row
 * Nothing else is ever OR-ed into a status word: the WBC's iteration counts live in qmb200_wbc_get_diagnostics. */
#define QMB200_ST_ITER_CAP 1
#define QMB200_ST_OVERFLOW 2      /* WBC: more rows than the working-set / level-0 buffers hold; MPC: node count > NMAX, event / target count out of range, swing phase not enclosed */
#define QMB200_ST_NAN 4
#define QMB200_ST_NOT_PD 8
#define QMB200_ST_NO_STEP 16      /* line search rejected every step size (solution = initial guess, as in SqpSolver::takeStep) */
#define QMB200_ST_CONVERGED 32    /* informational: SqpSolver::checkConvergence ended the SQP loop before sqp.sqpIteration (only when sqpIteration > 1) */
#define QMB200_ST_NEG_DT 64       /* an interval of the time grid has a non-positive duration: a pre-/post-event node within weakEpsilon (1e-6 s) of its neighbour but
                                     further than dt_min (1e-8 s), so getIntervalEnd - getIntervalStart < 0 [upstream ocs2_oc TimeDiscretization]; the stage cost is then
                                     weighted by a negative dt and the QP is not convex (comes with QMB200_ST_NOT_PD) */
#define QMB200_MPC_STATUS_SHIFT 8

typedef struct qmb200_handle qmb200_handle;

/* Replaces the constructor chain QMController::setupInterface/setupMpc/setupWbc
 * (qm_controllers/src/QMController.cpp:272-306,336-340) → QMInterface(taskFile, urdfFile, referenceFile)
 * (qm_interface/include/qm_interface/QMInterface.h:31-35). */
typedef struct {
  const char* task_file;        /* task.info */
  const char* urdf_file;        /* robot.urdf */
  const char* reference_file;   /* reference.info */
  const char* wbc_gains_file;   /* optional INFO file with a wbcGains{} block; NULL → defaults of qm_wbc/cfg/wbcWigeht.cfg:7-47 */
  int32_t batch;                /* robots per call on this GPU */
  int32_t device;               /* CUDA device ordinal */
  double time_horizon;          /* <= 0 → mpc.timeHorizon (task.info:140) */
  double dt;                    /* <= 0 → sqp.dt (task.info:78) */
  int32_t max_nodes;            /* <= 0 → ceil(horizon/dt) + 1 + 2*10 (room for 10 events inside the horizon).  At most 1060, given or by default: the
                                   setup kernel stages 48 B per node + 320 B per warp, four warps per CTA, in at most 200 KB of shared memory; a larger value
                                   fails qmb200_create ("max_nodes too large") */
  int32_t wbc_variant;          /* QMB200_WBC_* */
} qmb200_config;

int qmb200_create(const qmb200_config* cfg, qmb200_handle** out);
void qmb200_destroy(qmb200_handle* h);
const char* qmb200_last_error(const qmb200_handle* h);   /* h may be NULL (error of a failed create) */

/* dimensions of this handle: batch, node capacity NMAX, event capacity, target-knot capacity */
int qmb200_get_dims(const qmb200_handle* h, int32_t* batch, int32_t* nmax, int32_t* emax, int32_t* kmax);
/* CentroidalModelInfo / settings as the reference exposes them (QMInterface.h:37-54): robotMass, initialState[30] (task.info:150-189),
 * defaultJointState[18] (reference.info:6-26), time horizon, dt */
int qmb200_get_model_info(const qmb200_handle* h, double* robot_mass, double* initial_state30, double* default_joint_state18, double* time_horizon, double* dt);
int qmb200_get_joint_name(const qmb200_handle* h, int32_t joint, char* out, int32_t capacity);

/* ---- WBC seam: qm::WbcBase::update(stateDesired, inputDesired, rbdStateMeasured, mode, period, time) → vector_t
 *      (qm_wbc/include/qm_wbc/WbcBase.h:31-32), batched.  Host-pointer version copies in/out on the handle's stream
 *      and returns after the result is in cmd/status. */
int qmb200_wbc_update(qmb200_handle* h, const double* x_des /*[B][30]*/, const double* u_des /*[B][30]*/, const double* rbd /*[B][55]*/,
                      const int32_t* mode /*[B]*/, const double* period /*[B]*/, const double* time /*[B]*/, double* cmd /*[B][54]*/, int32_t* status /*[B]*/);
int qmb200_wbc_update_dev(qmb200_handle* h, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const double* period,
                          const double* time, double* cmd, int32_t* status, void* cuda_stream);
/* WbcBase::inputLast_ (WbcBase.cpp:42,212-213): set for all robots (NULL → zeros, the constructor state) / read back */
int qmb200_wbc_set_input_last(qmb200_handle* h, const double* input_last /*[B][30] or NULL*/);
int qmb200_wbc_get_input_last(qmb200_handle* h, double* input_last /*[B][30]*/);

/* WbcBase::dynamicCallback (qm_wbc/src/WbcBase.cpp:69-117, qm_wbc/cfg/wbcWigeht.cfg:7-47): the PD gains of the task formulators, replaceable at run time.
 * Takes effect for the next wbc_update / tick / update call on the handle's stream.  These are the handle's gains: while per-robot tuning rows are set
 * (qmb200_set_robot_tuning) every robot uses its row's gains instead, and the handle's apply again after the rows are cleared. */
typedef struct {
  double kp_swing, kd_swing, base_height_kp, base_height_kd, kp_base_linear, kd_base_linear, kp_base_angular, kd_base_angular;
  double kp_arm_joint[6], kd_arm_joint[6], kp_ee_linear[3], kd_ee_linear[3], kp_ee_angular[3], kd_ee_angular[3];
} qmb200_wbc_gains;
int qmb200_wbc_get_gains(const qmb200_handle* h, qmb200_wbc_gains* out);
int qmb200_wbc_set_gains(qmb200_handle* h, const qmb200_wbc_gains* gains);
/* Per-robot diagnostics of the last WBC update on this handle (the reference prints nothing: HoQp.cpp:143 drops qpOASES' return value):
 * diag[b] = it0 | it1 << 8 | it2 << 16 | nw << 24 — level-0 semismooth passes, active-set iterations of levels 1 and 2, final working-set size. */
int qmb200_wbc_get_diagnostics(qmb200_handle* h, int32_t* diag /*[B]*/);
/* Iteration caps of the WBC solver (defaults 30 / 80 ≙ nWSR = 100 of HoQp.cpp:141); a robot that hits one carries QMB200_ST_ITER_CAP.  <= 0 keeps the value. */
int qmb200_wbc_set_iteration_caps(qmb200_handle* h, int32_t level0_passes, int32_t active_set_iterations);

/* ---- MPC seam: ocs2::MPC_BASE::run → SqpSolver::run(t0, x0, t0+T), one SQP iteration (QMController.cpp:287-288,315-332),
 *      with the inputs the reference manager holds: mode schedule (SwitchedModelReferenceManager) and TargetTrajectories.
 *      The previous PrimalSolution (warm start, mpc.coldStart=false) lives in the handle. */
int qmb200_mpc_solve(qmb200_handle* h, const double* t0 /*[B]*/, const double* x0 /*[B][30]*/,
                     const int32_t* n_events /*[B]*/, const double* event_times /*[B][EMAX]*/, const int32_t* mode_sequence /*[B][EMAX+1]*/,
                     const int32_t* n_target /*[B]*/, const double* target_times /*[B][KMAX]*/, const double* target_states /*[B][KMAX][37]*/,
                     int32_t* n_nodes /*[B]*/, double* node_times /*[B][NMAX]*/, int32_t* node_events /*[B][NMAX]*/,
                     double* x_traj /*[B][NMAX][30]*/, double* u_traj /*[B][NMAX][30]*/, int32_t* status /*[B]*/, double* step_info /*[B][4] or NULL: alpha, cost, dyn SSE, eq SSE after the step*/);
int qmb200_mpc_solve_dev(qmb200_handle* h, const double* t0, const double* x0, const int32_t* n_events, const double* event_times, const int32_t* mode_sequence,
                         const int32_t* n_target, const double* target_times, const double* target_states, void* cuda_stream);
/* sqp.sqpIteration / costTol of the handle (task.info:28; the create-time values come from task.info): SqpSolver::runImpl runs up to that many
 * LQ → QP → line-search iterations per solve and leaves the loop early per robot on checkConvergence (step size, metrics, primal step) [upstream ocs2_sqp].
 * sqp_iterations <= 0 / cost_tol <= 0 keep the current value. */
int qmb200_mpc_set_iterations(qmb200_handle* h, int32_t sqp_iterations, double cost_tol);
/* drop the stored PrimalSolution: next solve starts from QMInitializer (qm_interface/src/initialization/QMInitializer.cpp:33-41) */
int qmb200_mpc_reset(qmb200_handle* h);
/* load a PrimalSolution as warm start (n_nodes[b] < 2 → cold start for robot b) */
int qmb200_mpc_set_solution(qmb200_handle* h, const int32_t* n_nodes, const double* node_times, const int32_t* node_events, const double* x_traj, const double* u_traj);
/* read the stored solution (device → host) */
int qmb200_mpc_get_solution(qmb200_handle* h, int32_t* n_nodes, double* node_times, int32_t* node_events, double* x_traj, double* u_traj, int32_t* status, double* step_info);

/* ---- MPC→WBC hand-off: MPC_MRT_Interface::evaluatePolicy(t, x, → optimizedState, optimizedInput, plannedMode) (QMController.cpp:141)
 *      on the stored solution and the mode schedule of the last solve. */
int qmb200_policy_eval(qmb200_handle* h, const double* t /*[B]*/, double* x_des /*[B][30]*/, double* u_des /*[B][30]*/, int32_t* mode /*[B]*/);
int qmb200_policy_eval_dev(qmb200_handle* h, const double* t, double* x_des, double* u_des, int32_t* mode, void* cuda_stream);

/* ---- one controller tick on the device: mpc_solve → policy_eval(t_eval) → wbc_update, torque buffer out.
 *      Host-pointer version: observation in, cmd out (the e2e path bench.py times). */
int qmb200_tick(qmb200_handle* h, const double* t0, const double* x0, const int32_t* n_events, const double* event_times, const int32_t* mode_sequence,
                const int32_t* n_target, const double* target_times, const double* target_states, const double* t_eval, const double* rbd,
                const double* period, double* cmd /*[B][54]*/, int32_t* status /*[B]*/);
int qmb200_tick_dev(qmb200_handle* h, const double* t0, const double* x0, const int32_t* n_events, const double* event_times, const int32_t* mode_sequence,
                    const int32_t* n_target, const double* target_times, const double* target_states, const double* t_eval, const double* rbd,
                    const double* period, double* cmd, int32_t* status, void* cuda_stream);

/* ---- observation: CentroidalModelRbdConversions::computeCentroidalStateFromRbdModel (QMController.cpp:238-241), host utility.  With a model payload set
 *      (qmb200_set_model_payload) row r uses robot r's SRBD constants and n must equal the batch size. */
int qmb200_centroidal_state_from_rbd(const qmb200_handle* h, int32_t n, const double* rbd /*[n][55]*/, double* x /*[n][30]*/);

/* ---- the controller's model payload: what the MPC and the WBC believe each robot carries.
 *   payload[B][8]  layout as qmb200_sim_set_robot_params: [m_ee, o_ee_x, o_ee_y, o_ee_z, m_base, o_base_x, o_base_y, o_base_z], two point masses (kg) rigidly
 *                  attached at o_ee (m, end-effector frame) and o_base (m, base frame); no rotational inertia.
 * Robot b then computes what a handle built from an edited URDF computes for it: the URDF with an extra link fixed to the end-effector frame's link at o_ee
 * carrying m_ee, and one fixed to the base link at o_base carrying m_base.  That is:
 *   - the MPC's SRBD constants (robotMass, centroidalInertiaNominal, comToBasePositionNominal, folded at defaultJointState as createCentroidalModelInfo
 *     does), used by every MPC solver, the observation and qmb200_centroidal_state_from_rbd.  Like the reference's model, the SRBD places the payload at
 *     its position in the default joint state: it does not follow the arm;
 *   - the WBC's rigid-body model (mass matrix, nonlinear effects, centroidal momentum terms), where the point masses follow the arm.
 * This is the controller's model, independent of the plant's robot params (qmb200_sim_set_robot_params): an estimate may differ from the truth.
 * Host array, copied to the device; synchronous (waits for the device).  NULL clears it (every robot back to the nominal model).  Rejects a non-finite entry and a
 * negative mass; on rejection the stored payload stays unchanged. */
#define QMB200_SRBD 24   /* per-robot SRBD constants: [robotMass, centroidalInertiaNominal(9, row-major), its inverse(9), comToBasePositionNominal(3), 0, 0] */
int qmb200_set_model_payload(qmb200_handle* h, const double* payload /*[B][8] or NULL*/);
/* The stored payload (zeros where none is set); is_set = 1 when one is set.  Either output may be NULL.  After a qmb200_payload_est_commit_dev it waits
 * for the device and returns the rows the kernels read. */
int qmb200_get_model_payload(const qmb200_handle* h, double* payload /*[B][8]*/, int32_t* is_set);

/* ---- per-robot controller tuning: the parameters the reference changes at run time for the whole controller, one row per robot.
 *   rows[B][QMB200_TUNING]  offset  0       friction_mu      MPC friction-cone coefficient (frictionConeSoftConstraint.frictionCoefficient, task.info:290-292)
 *                                   1       wbc_friction     WBC friction pyramid (frictionConeTask.frictionCoefficient, task.info:346-348; WbcBase.cpp:419-431,585-590)
 *                                   2-5     mu_ee_pos, mu_ee_ori, mu_final_ee_pos, mu_final_ee_ori   end-effector soft-constraint weights (endEffector /
 *                                           finalEndEffector muPosition / muOrientation, task.info:235-246)
 *                                   6-37    the 32 fields of qmb200_wbc_gains in struct order (WbcBase::dynamicCallback, wbcWigeht.cfg)
 *                                   38-39   kp_arm_wbc, kd_arm_wbc   the control law's arm gains (QMController::dynamicCallback, weight.cfg)
 * Robot b then computes what a handle whose task.info, gains file and arm gains hold row b computes, in every MPC solver (SQP, IPM, DDP), both WBC variants
 * and the control law.  Rows are indexed by the global robot index, like the model payload, so chunked ticks and sharded or permuted batches keep each
 * robot on its own row.  Precedence: while rows are set they replace the handle's values (qmb200_wbc_set_gains, qmb200_set_arm_gains and the task file's)
 * for every robot; those calls still set the handle's values, which apply again after a clear.
 * Host array, copied to the device; synchronous (waits for the device).  NULL clears the rows.  Rejects a non-finite entry, a friction coefficient <= 0 and a
 * negative weight or gain, naming the field and the robot; on rejection the stored rows stay unchanged. */
#define QMB200_TUNING 40
int qmb200_set_robot_tuning(qmb200_handle* h, const double* rows /*[B][QMB200_TUNING] or NULL*/);
/* The stored rows, or the handle's current values on every row when none are set; is_set = 1 when rows are set.  Either output may be NULL. */
int qmb200_get_robot_tuning(const qmb200_handle* h, double* rows /*[B][QMB200_TUNING]*/, int32_t* is_set);
/* The handle's own values as one row: what every robot uses while no rows are set (the task file's, qmb200_wbc_set_gains' and qmb200_set_arm_gains'). */
int qmb200_get_handle_tuning(const qmb200_handle* h, double* row /*[QMB200_TUNING]*/);

/* ---- online estimate of the end-effector payload (DESIGN.md §4.6): per-robot recursive least squares on the six arm rows of the nominal model, which see
 *      an end-effector load through its ten inertial parameters theta = [m, m c_x, m c_y, m c_z, I_xx, I_xy, I_xz, I_yy, I_yz, I_zz] (end-effector frame,
 *      about its origin) and see neither the foot contacts nor a base payload.  It reads only what the controller reads (the measurement rbd and the effort
 *      sent) and commits its estimate to the model payload on the device, so it can run inside a loop without host synchronisation.
 *      An external wrench on the end effector is indistinguishable from a load and biases the estimate while it acts; a wrench on the base does not.
 *   forgetting       RLS forgetting factor lambda in (0, 1]
 *   p0_mass, p0_first_moment, p0_inertia   prior variances of m (kg^2), of m c (kg^2 m^2) and of I (kg^2 m^4): P = diag(p0) at the reset
 *   trace_max        P is scaled down to this trace whenever it exceeds it (directions the motion does not excite would otherwise grow as lambda^-k)
 *   mass_min         below this estimated mass the committed offset is 0 (m c / m is noise there)
 *   mass_max         committed mass = clamp(m, 0, mass_max)
 *   offset_max       committed offset = m c / m with its norm clipped to offset_max (m) */
typedef struct qmb200_payload_est_params {
  double forgetting, p0_mass, p0_first_moment, p0_inertia, trace_max, mass_min, mass_max, offset_max;
} qmb200_payload_est_params;
int qmb200_payload_est_get_params(const qmb200_handle* h, qmb200_payload_est_params* out);
/* rejects non-finite values, forgetting outside (0, 1], a variance, trace_max, mass_min, mass_max or offset_max <= 0 and mass_min > mass_max */
int qmb200_payload_est_set_params(qmb200_handle* h, const qmb200_payload_est_params* p);
/* (Re)starts the estimator of every robot: theta = the end-effector point mass of prior [B][8] (layout as qmb200_set_model_payload; NULL: the current model
 * payload, zeros when none is set), P = diag(p0), no stored sample.  Sets the model payload to prior through qmb200_set_model_payload, so the kernels read
 * per-robot rows from then on.  Synchronous. */
int qmb200_payload_est_reset(qmb200_handle* h, const double* prior /*[B][8] or NULL*/);
/* One RLS update per robot from the measurement rbd (the plant's output, include/qmb200.h layout) and the effort [B][18] held over the dt seconds that ended
 * at it (clipped to the URDF effort limits as the plant does).  The first call after a reset only stores its sample.  status [B] (written, not OR-ed):
 * QMB200_ST_NAN for a non-finite input (nothing is stored) or update, QMB200_ST_NOT_PD when the innovation covariance fails its Cholesky; the robot
 * then keeps its theta and P. */
int qmb200_payload_est_step(qmb200_handle* h, double dt, const double* effort /*[B][18]*/, const double* rbd /*[B][55]*/, int32_t* status /*[B]*/);
int qmb200_payload_est_step_dev(qmb200_handle* h, double dt, const double* effort, const double* rbd, int32_t* status, void* cuda_stream);
/* In stream order on cuda_stream (NULL: the handle's): m = clamp(theta_0, 0, mass_max) and o = theta_1:4 / theta_0 (0 when theta_0 < mass_min, norm clipped to
 * offset_max) into the end-effector half [m_ee, o_ee] of every robot's model payload row, and the robot's SRBD constants from the whole row, as
 * qmb200_set_model_payload computes them.  The base half is left as it was.  No host copy. */
int qmb200_payload_est_commit_dev(qmb200_handle* h, void* cuda_stream);
/* Synchronous: theta [B][10], the diagonal of P [B][10] and the samples stored since the reset [B].  Any output may be NULL. */
int qmb200_payload_est_get(qmb200_handle* h, double* theta /*[B][10]*/, double* p_diag /*[B][10]*/, int32_t* samples /*[B]*/);
/* Releases the estimator state; the model payload keeps its last committed rows.  Step, commit and get fail until the next reset. */
int qmb200_payload_est_stop(qmb200_handle* h);
/* The model payload rows the kernels read, copied in stream order into payload (device, [B][8]) on cuda_stream (NULL: the handle's): a record of the committed
 * estimate without host synchronisation.  Fails when no model payload is set. */
int qmb200_get_model_payload_dev(const qmb200_handle* h, double* payload /*[B][8] device*/, void* cuda_stream);

/* ---- gait front-end: GaitSchedule::getModeSchedule tiling of a ModeSequenceTemplate (QMInterface.cpp:455-480, gait.info) for one robot:
 *      STANCE until t_start, then the template repeated; window [lo, hi]; returns the number of events written (<= EMAX) or negative. */
int qmb200_gait_schedule(const char* gait_file, const char* gait_name, double t_start, double lo, double hi,
                         double* event_times /*[EMAX]*/, int32_t* mode_sequence /*[EMAX+1]*/);

/* ---- stateful gait front-end: ocs2::legged_robot::GaitSchedule as QMInterface::loadGaitSchedule builds it (QMInterface.cpp:455-480) and
 *      GaitReceiver / SwitchedModelReferenceManager drive it [upstream ocs2_legged_robot, recalled]: the schedule starts as
 *      reference.info:initialModeSchedule with defaultModeSequenceTemplate as the active template; a gait command
 *      (GaitJoyPublisher.cpp:35-60 → a gait.info template) is inserted at the end of the current horizon after phaseTransitionStanceTime
 *      of stance (task.info:9); every solve asks for the window [t0 - T, tf + T] (trim + tile).  Host object, one per robot. */
typedef struct qmb200_gait qmb200_gait;
int qmb200_gait_create(const char* task_file, const char* reference_file, qmb200_gait** out);
void qmb200_gait_destroy(qmb200_gait* g);
/* GaitSchedule::insertModeSequenceTemplate(template, startTime, finalTime); GaitReceiver passes (finalTime of the solve, timeHorizon) */
int qmb200_gait_insert_template(qmb200_gait* g, const char* gait_file, const char* gait_name, double start_time, double final_time);
/* GaitSchedule::getModeSchedule(lowerBoundTime, upperBoundTime): returns the number of events written (<= EMAX) or negative */
int qmb200_gait_get_mode_schedule(qmb200_gait* g, double lower_bound_time, double upper_bound_time, double* event_times /*[EMAX]*/, int32_t* mode_sequence /*[EMAX+1]*/);

/* ---- device gait front-end: the GaitSchedule protocol above for every robot of the handle, on the device, rolled once per MPC tick so that a
 *      closed loop can switch gaits per robot without a host synchronisation (DESIGN.md §4.7).  Each robot holds a schedule of at most
 *      QMB200_GAIT_CAP events, its active template and a cursor into its own command timeline.  The arithmetic is that of qmb200_gait_insert_template /
 *      qmb200_gait_get_mode_schedule: a robot's windows equal, bit for bit, those of a qmb200_gait object driven through the same protocol. */
#define QMB200_GAIT_CAP 64    /* events of one robot's schedule while a step works on it */
#define QMB200_GAIT_MAXM 16   /* modes of one template */
/* The template table: templates names[0..n) of gait_file, in that order (a template's id is its index).  Rejects a name the file lacks, more than
 * QMB200_GAIT_MAXM modes and switching times that are not finite and strictly increasing.  Fails while the schedule runs (qmb200_gait_dev_stop first). */
int qmb200_gait_dev_set_templates(qmb200_handle* h, const char* gait_file, const char* const* names, int32_t n);
/* (Re)starts every robot's schedule: what qmb200_gait_create builds (reference.info's initialModeSchedule, task.info's phaseTransitionStanceTime)
 * followed by qmb200_gait_insert_template(template[b], t_start[b], T) with T the handle's time horizon: stance until t_start, then the template.
 * Clears the command timeline.  Rejects a template outside the table and a non-finite t_start.  Synchronous. */
int qmb200_gait_dev_reset(qmb200_handle* h, const int32_t* tmpl /*[B]*/, const double* t_start /*[B]*/);
/* The command timeline, n_cmd commands per robot (host arrays, copied): robot b's command c is due at t[b][c] (same clock as t_obs; sorted per robot,
 * +inf pads), inserts template tmpl[b][c] (-1: none) and sets cmd_vel[b][c] (vx, vy, vz, yaw rate; a NaN row: none).  Every cursor goes back to 0;
 * n_cmd = 0 clears the timeline.  Rejects a NaN time, unsorted times, a template outside [-1, n_templates) and a cmd_vel row neither finite nor all
 * NaN.  Synchronous. */
int qmb200_gait_dev_set_commands(qmb200_handle* h, int32_t n_cmd, const double* t /*[B][n_cmd]*/, const int32_t* tmpl /*[B][n_cmd]*/, const double* cmd_vel /*[B][n_cmd][4]*/);
/* The same timeline with end-effector commands (DESIGN.md §4.8): command c of robot b may instead of a cmd_vel row carry ee_kind[b][c] =
 * QMB200_TARGET_EE_CMD_VEL (ee_cmd[b][c][0:3] = vx, vy, vz of the end effector, world frame; [3:7] ignored) or QMB200_TARGET_EE_GOAL (ee_cmd[b][c] = goal
 * position, quaternion xyzw, world frame); -1: none (the row is ignored).  Besides the checks above it rejects an ee_kind outside {-1, 1, 2}, a command
 * with both a cmd_vel row and an end-effector command, a non-finite ee_cmd_vel or goal and a goal quaternion whose norm differs from 1 by more than
 * 1e-9.  ee_kind and ee_cmd both NULL: qmb200_gait_dev_set_commands.  ee_kind QMB200_TARGET_EE_PATH starts the path ee_cmd[b][c][0] (an integer index
 * of the path table in force, qmb200_set_ee_paths; [1:7] ignored).  Synchronous. */
int qmb200_gait_dev_set_commands_ee(qmb200_handle* h, int32_t n_cmd, const double* t /*[B][n_cmd]*/, const int32_t* tmpl /*[B][n_cmd]*/, const double* cmd_vel /*[B][n_cmd][4]*/,
                                    const int32_t* ee_kind /*[B][n_cmd] or NULL*/, const double* ee_cmd /*[B][n_cmd][7] or NULL*/);
/* One step per robot at t = t_obs[b], right before the MPC tick's target_trajectories: (1) every command of the robot due at t (time <= t) and not yet
 * applied, in order: a template is inserted with qmb200_gait_insert_template's arithmetic at (t + T, T) (GaitReceiver::preSolverRun: start = the
 * solve's final time, final = the time horizon), a cmd_vel row is written to cmd[b][0:4] (the target front-end's cmd[B][7]); (2) the window
 * getModeSchedule(t - T, t + 2T) is written to the MPC problem rows n_events[b], event_times[b][EMAX] (0 past the count) and modes[b][EMAX+1] (stance
 * past the count).  All or nothing per robot: status QMB200_ST_NAN (non-finite t) or QMB200_ST_OVERFLOW (the window would hold more than QMB200_EMAX
 * events, where qmb200_gait_get_mode_schedule returns -2, or the schedule more than QMB200_GAIT_CAP) leaves the robot's schedule, cursor, MPC rows and
 * cmd row as they were, so its due commands are applied by a later step.  status [B] is written, not OR-ed; tmpl [B] (active template) and mode [B]
 * (the stored schedule's mode at t, as the MPC reads it) are written when non-NULL. */
int qmb200_gait_dev_step(qmb200_handle* h, const double* t_obs /*[B]*/, int32_t* n_events /*[B] in-out*/, double* event_times /*[B][EMAX] in-out*/,
                         int32_t* mode_sequence /*[B][EMAX+1] in-out*/, double* cmd /*[B][7] in-out*/, int32_t* tmpl /*[B] or NULL*/, int32_t* mode /*[B] or NULL*/,
                         int32_t* status /*[B]*/);
int qmb200_gait_dev_step_dev(qmb200_handle* h, const double* t_obs, int32_t* n_events, double* event_times, int32_t* mode_sequence, double* cmd, int32_t* tmpl,
                             int32_t* mode, int32_t* status, void* cuda_stream);
/* The step with the publisher's target source (DESIGN.md §4.8).  Each robot's source is the cmd_vel stream after qmb200_gait_dev_reset.  Among the
 * robot's commands applied by the step, the last target command (cmd_vel, ee_cmd_vel or goal) sets the source: a cmd_vel row writes cmd[b][0:4], an
 * ee_cmd_vel row cmd[b][0:3], a goal row cmd[b][0:7].  target_kind [B] (or NULL) is the kind this tick's target call takes
 * (qmb200_target_trajectories_per_robot): QMB200_TARGET_EE_GOAL when the step applied a goal as its last target command (the goal is published once),
 * -1 while a published goal is held (the target call then leaves the robot's target and last_ee_target as they are), otherwise the source's stream,
 * QMB200_TARGET_CMD_VEL or QMB200_TARGET_EE_CMD_VEL.  A failed step (QMB200_ST_NAN / QMB200_ST_OVERFLOW) leaves the source unchanged and reports that
 * source's kind (-1 for a held goal).  target_kind is written for every robot.  A path row (ee_kind QMB200_TARGET_EE_PATH, ee[0] the path index) writes
 * cmd[b][0] and makes the path the source: QMB200_TARGET_EE_PATH on the tick that applied it, QMB200_TARGET_EE_PATH_FOLLOW after it (and from a
 * failed step) while the source is the path (qmb200_target_trajectories_path). */
int qmb200_gait_dev_step_ee(qmb200_handle* h, const double* t_obs /*[B]*/, int32_t* n_events /*[B] in-out*/, double* event_times /*[B][EMAX] in-out*/,
                            int32_t* mode_sequence /*[B][EMAX+1] in-out*/, double* cmd /*[B][7] in-out*/, int32_t* tmpl /*[B] or NULL*/, int32_t* mode /*[B] or NULL*/,
                            int32_t* status /*[B]*/, int32_t* target_kind /*[B] or NULL*/);
int qmb200_gait_dev_step_ee_dev(qmb200_handle* h, const double* t_obs, int32_t* n_events, double* event_times, int32_t* mode_sequence, double* cmd, int32_t* tmpl,
                                int32_t* mode, int32_t* status, int32_t* target_kind, void* cuda_stream);
/* Synchronous: each robot's stored schedule (count, event times [B][GAIT_CAP] with 0 past the count, modes [B][GAIT_CAP+1] with stance past it), active
 * template and cursor.  Any output may be NULL. */
int qmb200_gait_dev_get(qmb200_handle* h, int32_t* n_events /*[B]*/, double* event_times /*[B][QMB200_GAIT_CAP]*/, int32_t* mode_sequence /*[B][QMB200_GAIT_CAP+1]*/,
                        int32_t* tmpl /*[B]*/, int32_t* cursor /*[B]*/);
/* Synchronous: the loaded command timeline (qmb200_gait_dev_set_commands(_ee), qmb200_timeline_sample_dev): n_cmd, and t [B][n_cmd], tmpl [B][n_cmd],
 * cmd_vel [B][n_cmd][4], ee_kind [B][n_cmd] and ee_cmd [B][n_cmd][7] in the layouts qmb200_gait_dev_set_commands_ee takes (ee_kind -1 and ee_cmd zeros
 * when the timeline has no end-effector rows).  Any output may be NULL: a call with n_cmd alone sizes the others.  Fails while the schedule is not running. */
int qmb200_gait_dev_get_commands(qmb200_handle* h, int32_t* n_cmd, double* t /*[B][n_cmd]*/, int32_t* tmpl /*[B][n_cmd]*/, double* cmd_vel /*[B][n_cmd][4]*/,
                                 int32_t* ee_kind /*[B][n_cmd]*/, double* ee_cmd /*[B][n_cmd][7]*/);
/* One command per robot from device buffers, applied by the robot's next step (DESIGN.md §4.16): each robot has one pending slot beside its schedule,
 * empty after qmb200_gait_dev_reset.  For every robot with mask[b] != 0 the row tmpl[b] (-1: none), cmd_vel[b][4] (a NaN row: none), ee_kind[b] (-1,
 * QMB200_TARGET_EE_CMD_VEL, QMB200_TARGET_EE_GOAL or QMB200_TARGET_EE_PATH, whose index is checked against the path table in force) and ee[b][7] (as
 * ee_cmd of qmb200_gait_dev_set_commands_ee) is checked on the device with the rules
 * of qmb200_gait_dev_set_commands_ee; an accepted row overwrites the slot (a later command before the step replaces an earlier one), a rejected row
 * leaves it and gets status[b] = QMB200_ST_COMMAND.  status [B] is written, not OR-ed: 0 for accepted rows and for robots with mask[b] == 0, whose
 * slots are not written.  The next step applies a set slot after the robot's timeline rows due at t, as one more row due at t, and clears it when it
 * succeeds; a failed step leaves it set.  A restore (qmb200_robot_image_restore) clears the restored robots' slots.  Fails, writing nothing, while the
 * schedule is not running or when a buffer is NULL.  One launch, no synchronisation. */
int qmb200_gait_dev_command(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* tmpl /*[B]*/, const double* cmd_vel /*[B][4]*/, const int32_t* ee_kind /*[B]*/,
                            const double* ee /*[B][7]*/, int32_t* status /*[B]*/);
int qmb200_gait_dev_command_dev(qmb200_handle* h, const int32_t* mask, const int32_t* tmpl, const double* cmd_vel, const int32_t* ee_kind, const double* ee,
                                int32_t* status, void* cuda_stream);
/* Synchronous: each robot's pending slot, set [B] (1: a command waits for the next step), and the row last written to it: tmpl [B], cmd_vel [B][4],
 * ee_kind [B], ee [B][7] (zeros after a reset or restore).  Any output may be NULL.  Fails while the schedule is not running. */
int qmb200_gait_dev_get_pending(qmb200_handle* h, int32_t* set /*[B]*/, int32_t* tmpl /*[B]*/, double* cmd_vel /*[B][4]*/, int32_t* ee_kind /*[B]*/, double* ee /*[B][7]*/);
/* Releases the schedules, the pending slots and the timeline; the template table stays.  Step and get fail until the next reset.  Stopping a schedule
 * that is not running does nothing and returns 0. */
int qmb200_gait_dev_stop(qmb200_handle* h);

/* ---- controller side of the path (SURVEY.md section 8f): the steps of QMController::update around evaluatePolicy / WbcBase::update and the
 *      publisher that feeds the solver, batched on the device.  The caller owns the per-robot controller state these functions read and
 *      write (the members of QMController / QmTargetTrajectoriesInteractiveMarker they mirror); `_dev` variants take device pointers. */
#define QMB200_TARGET_CMD_VEL 0      /* cmdVelToTargetTrajectories      (QmTargetTrajectoriesPublisher_node.cpp:73-113): cmd = vx, vy, vz, yaw rate */
#define QMB200_TARGET_EE_CMD_VEL 1   /* EeCmdVelToTargetTrajectories    (:118-165): cmd = vx, vy, vz of the end effector */
#define QMB200_TARGET_EE_GOAL 2      /* EEgoalPoseToTargetTrajectories  (:172-208) + processFeedback (QmTargetTrajectoriesPublisher.cpp:94-109): cmd = pos(3), quat xyzw(4) */
#define QMB200_TARGET_EE_PATH 3      /* start of an end-effector path (qmb200_target_trajectories_path; DESIGN.md §4.20): cmd[0] = path index of the table */
#define QMB200_TARGET_EE_PATH_FOLLOW 4   /* the path in force (path_state) at the call's time */
#define QMB200_JOINT_CMD 5           /* HybridJointHandle::setCommand(posDes, velDes, kp, kd, ff) (HybridJointInterface.h:55-61) */
#define QMB200_ST_SAFETY 0x10000     /* SafetyChecker::check failed (SafetyChecker.h:22-35): the reference stops the controller */
#define QMB200_ST_COMMAND 0x20000    /* qmb200_gait_dev_command(_dev): the robot's command row was rejected (no other status word uses this bit) */
#define QMB200_ST_RESTORE (QMB200_ST_COMMAND << 1)   /* qmb200_robot_state_load(_dev): the robot's source row lies outside [0, B), the robot was not written
                                                        (bit 18; no other status word uses it) */
#define QMB200_ST_SPAWN (QMB200_ST_RESTORE << 1)     /* qmb200_spawn_place(_dev): the robot's spawn row was rejected, the robot was not written (bit 19; no
                                                        other status word uses it) */
#define QMB200_ST_HW_RING_FULL 2     /* qmb200_hw_write: more than 32 commands inside the delay window (the oldest was dropped) */

/* QMController::updateStateEstimation tail (QMController.cpp:236-243): t_obs += period; x_obs = computeCentroidalStateFromRbdModel(rbd) with
 * the yaw unwrapped against the previous x_obs[9] (angles::shortest_angular_distance). */
int qmb200_observation_update(qmb200_handle* h, const double* rbd /*[B][55]*/, const double* period /*[B]*/, double* t_obs /*[B] in-out*/, double* x_obs /*[B][30] in-out*/);
int qmb200_observation_update_dev(qmb200_handle* h, const double* rbd, const double* period, double* t_obs, double* x_obs, void* cuda_stream);

/* TargetTrajectories from a command (QmTargetTrajectoriesPublisher_node.cpp:44-208) in the layout qmb200_mpc_solve takes; constants from
 * reference.info (comHeight, defaultJointState, target*Velocity) and task.info (mpc.timeHorizon).  last_ee_target mirrors lastEeTarget_
 * (initial value qmb200_initial_ee_target: QmTargetTrajectoriesPublisher.h:55-57). */
int qmb200_target_trajectories(qmb200_handle* h, int32_t kind, const double* cmd /*[B][7]*/, const double* t_obs /*[B]*/, const double* x_obs /*[B][30]*/, const double* ee_state /*[B][7] pos, quat xyzw*/,
                               double* last_ee_target /*[B][7] in-out*/, int32_t* n_target /*[B]*/, double* target_times /*[B][KMAX]*/, double* target_states /*[B][KMAX][37]*/);
int qmb200_target_trajectories_dev(qmb200_handle* h, int32_t kind, const double* cmd, const double* t_obs, const double* x_obs, const double* ee_state, double* last_ee_target,
                                   int32_t* n_target, double* target_times, double* target_states, void* cuda_stream);
/* The same with a kind per robot: kind[b] in {QMB200_TARGET_CMD_VEL, _EE_CMD_VEL, _EE_GOAL} as above, or -1: robot b is left untouched (a held goal: its
 * n_target, target_times, target_states and last_ee_target keep the published 2-knot trajectory, which the MPC keeps tracking; past its final time
 * the target holds the final knot).  The host variant rejects a kind outside [-1, 2] and stages the target rows in-out; the _dev variant leaves a
 * robot whose kind lies outside [0, 2] untouched.  For QMB200_TARGET_EE_CMD_VEL and _EE_GOAL the base target is the end-effector target minus
 * (0.52, 0.09) in the world frame, as QmTargetTrajectoriesPublisher_node.cpp:152-153, 184-185 compute it: right for a robot facing +x only (the base
 * of a robot turned by yaw is asked to stand 0.52 m world-x behind the hand, not 0.52 m behind it along its own heading).  A robot whose end-effector
 * frame is QMB200_EE_FRAME_HEADING (qmb200_set_ee_frame) takes its targets in its heading frame instead; every target call reads the rows. */
int qmb200_target_trajectories_per_robot(qmb200_handle* h, const int32_t* kind /*[B]*/, const double* cmd /*[B][7]*/, const double* t_obs /*[B]*/, const double* x_obs /*[B][30]*/,
                                         const double* ee_state /*[B][7]*/, double* last_ee_target /*[B][7] in-out*/, int32_t* n_target /*[B] in-out*/,
                                         double* target_times /*[B][KMAX] in-out*/, double* target_states /*[B][KMAX][37] in-out*/);
int qmb200_target_trajectories_per_robot_dev(qmb200_handle* h, const int32_t* kind, const double* cmd, const double* t_obs, const double* x_obs, const double* ee_state,
                                             double* last_ee_target, int32_t* n_target, double* target_times, double* target_states, void* cuda_stream);
void qmb200_initial_ee_target(double* last_ee_target7);
/* Per-robot end-effector frames (DESIGN.md §4.19), read by every target call and by qmb200_spawn_sample(_dev) / qmb200_spawn_place(_dev).
 * QMB200_EE_FRAME_WORLD: upstream's arithmetic, bit for bit.  QMB200_EE_FRAME_HEADING: the robot's heading frame H of its observed base (x_obs[6:8],
 * the unwrapped yaw x_obs[9]; origin (x, y, 0), rotation Rz(yaw), z the world's) states its end-effector targets: last_ee_target is the hold in H
 * (qmb200_initial_ee_target is then the nominal hold at any start pose), a goal (QMB200_TARGET_EE_GOAL) is a pose in H at the publishing call, the
 * base offset (0.52, 0.09) of the end-effector kinds turns with the yaw, and a spawn leaves the hold as it is.  frame [B] of 0 / 1, or NULL to clear
 * (every robot in the world frame).  The setter rejects any other value, naming the robot, and writes nothing; it waits for the device.  A per-robot
 * setting like the tuning rows: robot-state snapshots hold the rows while they are set (block 32). */
#define QMB200_EE_FRAME_WORLD 0
#define QMB200_EE_FRAME_HEADING 1
int qmb200_set_ee_frame(qmb200_handle* h, const int32_t* frame /*[B] or NULL to clear*/);
/* frame [B] (zeros when none are set, may be NULL), is_set (may be NULL): whether rows are set */
int qmb200_get_ee_frame(const qmb200_handle* h, int32_t* frame /*[B]*/, int32_t* is_set);

/* End-effector paths (DESIGN.md §4.20): a handle-wide table of timed hand paths, shared by every robot as the gait templates are.  Path p has
 * n_way[p] waypoints way[p][i] = (tau, position(3), quaternion xyzw(4)), tau in seconds after the path starts.  A robot that starts path p at time t0
 * from the measured hand pose S follows the piecewise pose p(t) through (t0, S), (t0 + tau_1, w_1), ..., each segment a position lerp and an
 * Eigen-semantics slerp (the MPC's own target interpolation); a heading-frame robot (qmb200_set_ee_frame) states the waypoints in its heading frame at
 * the start, fixed for the rest of the path.  The setter rejects, naming the path and the waypoint, and writes nothing for: a non-finite value,
 * n_way outside [1, QMB200_EE_PATH_MAX], tau_1 <= 0, times that are not strictly increasing, a gap between consecutive waypoints under T/2 (T the
 * handle's MPC time horizon, qmb200_get_model_info's time_horizon: task.info's mpc.timeHorizon unless qmb200_create overrides it; every target then
 * sees the path to t + T within QMB200_KMAX knots), a quaternion norm more than 1e-9 from 1.
 * n_paths 0 or way NULL clears the table.  It waits for the device. */
#define QMB200_EE_PATH_MAX 32
int qmb200_set_ee_paths(qmb200_handle* h, int32_t n_paths, const int32_t* n_way /*[n_paths]*/, const double* way /*[n_paths][QMB200_EE_PATH_MAX][8]*/);
/* n_paths (may be NULL): the table's size; n_way [n_paths] and way [n_paths][QMB200_EE_PATH_MAX][8] (zeros past n_way) may be NULL: a call with
 * n_paths alone sizes the others */
int qmb200_get_ee_paths(const qmb200_handle* h, int32_t* n_paths, int32_t* n_way, double* way);
/* The per-robot target call with paths: kind[b] as qmb200_target_trajectories_per_robot takes it, or QMB200_TARGET_EE_PATH (start path cmd[b][0] now)
 * or QMB200_TARGET_EE_PATH_FOLLOW (the path of path_state[b]).  path_state [B][QMB200_EE_PATH_STATE] is caller-owned and in-out: path index, start
 * time t0, start heading (x0, y0, yaw0 = x_obs[6], [7], [9] at the start) and the hand's start pose [7] (world).  A start writes the row and
 * last_ee_target (as a goal of the final waypoint published now leaves it), then follows.  Following at t writes the knot p(t) at t and the next
 * (up to three) waypoints after t at t0 + tau: n_target = 2..4.  The base of knot 0 is the observed base at comHeight, level; a waypoint knot's base
 * is the hand minus the (0.52, 0.09) offset (turned with the current yaw for a heading robot), at comHeight, level, at the current yaw.  With no
 * waypoint after t the call writes nothing: the robot holds the last waypoint as a held goal.  A path index outside the current table leaves the
 * robot untouched.  Robots of the other kinds get exactly what qmb200_target_trajectories_per_robot writes.  The host variant rejects kinds outside
 * [-1, 4] and stages the rows in-out. */
#define QMB200_EE_PATH_STATE 12
int qmb200_target_trajectories_path(qmb200_handle* h, const int32_t* kind /*[B]*/, const double* cmd /*[B][7]*/, const double* t_obs /*[B]*/, const double* x_obs /*[B][30]*/,
                                    const double* ee_state /*[B][7]*/, double* last_ee_target /*[B][7] in-out*/, double* path_state /*[B][EE_PATH_STATE] in-out*/,
                                    int32_t* n_target /*[B] in-out*/, double* target_times /*[B][KMAX] in-out*/, double* target_states /*[B][KMAX][37] in-out*/);
int qmb200_target_trajectories_path_dev(qmb200_handle* h, const int32_t* kind, const double* cmd, const double* t_obs, const double* x_obs, const double* ee_state,
                                        double* last_ee_target, double* path_state, int32_t* n_target, double* target_times, double* target_states, void* cuda_stream);

/* SafetyChecker::check + QMController::updateControlLaw (QMController.cpp:159-165,177-190) or, for a handle created with
 * QMB200_WBC_HIERARCHICAL_MPC, QMMpcController::updateControlLaw (:427-445).  joint_cmd entries the reference does not write in a given call
 * (legs before t = 10 s; the position-controlled arm of QMMpcController) keep their previous value, as the joint handles do. */
int qmb200_control_law(qmb200_handle* h, const double* x_des /*[B][30]*/, const double* u_des /*[B][30]*/, const double* wbc_cmd /*[B][54]*/, const double* t_obs /*[B]*/, const double* x_obs /*[B][30]*/,
                       double* joint_cmd /*[B][18][5] in-out*/, double* arm_pos_cmd /*[B][6] in-out*/, double* last_time /*[B] in-out*/, int32_t* status /*[B]*/);
int qmb200_control_law_dev(qmb200_handle* h, const double* x_des, const double* u_des, const double* wbc_cmd, const double* t_obs, const double* x_obs, double* joint_cmd, double* arm_pos_cmd,
                           double* last_time, int32_t* status, void* cuda_stream);
/* dynamic_reconfigure kp_arm_wbc / kd_arm_wbc (QMController.cpp:357-362; defaults 0.0 / 0.5, qm_controllers/cfg/weight.cfg:7-8).  The handle's gains: while
 * per-robot tuning rows are set (qmb200_set_robot_tuning) every robot uses its row's instead, and these apply again after the rows are cleared. */
int qmb200_set_arm_gains(qmb200_handle* h, double kp_arm_wbc, double kd_arm_wbc);

/* Plant stand-in, QMHWSim::writeSim (qm_gazebo/src/QMHWSim.cpp:98-116): the commands pass a per-robot delay FIFO (kept in the handle) and
 * the joint effort is kp (posDes - q) + kd (velDes - qd) + ff.  time == period clears the FIFO (simulation reset). */
int qmb200_hw_write(qmb200_handle* h, const double* time /*[B]*/, const double* period /*[B]*/, const double* joint_cmd /*[B][18][5]*/, const double* joint_pos /*[B][18]*/, const double* joint_vel /*[B][18]*/,
                    double* effort /*[B][18]*/, int32_t* status /*[B]*/);
int qmb200_hw_write_dev(qmb200_handle* h, const double* time, const double* period, const double* joint_cmd, const double* joint_pos, const double* joint_vel, double* effort, int32_t* status, void* cuda_stream);
/* gazebo/delay (qm_gazebo/config/default.yaml:2; QMHWSim.cpp:33-35 defaults to 0); clears the FIFO */
int qmb200_hw_set_delay(qmb200_handle* h, double delay);

/* ---- plant: Gazebo's physics step behind QMHWSim (one writeSim → physics step → readSim cycle) plus the contact flags QMHWSim::readSim reports to the
 *      ContactSensorInterface (qm_gazebo/src/QMHWSim.cpp:71-90), batched on the device.  Forward dynamics of the 24-DoF tree with a compliant contact
 *      between each foot's collision sphere and the ground: a flat plane, or per robot a heightfield tile (qmb200_sim_set_terrain) (this project's
 *      contact law, not Gazebo/ODE's: DESIGN.md §4.6).  The caller owns
 *      the plant state q[24] = [p_base, euler ZYX, joints], v[24] = dq/dt. */
typedef struct {
  double ground_height;        /* plane z = ground_height (m) under robots without a terrain tile; default 0 */
  double foot_radius;          /* foot collision sphere, centred on the *_FOOT frame (m); default 0.0265 (robot.urdf *_FOOT <collision>) */
  double stiffness;            /* normal force F_n = max(0, stiffness * delta - damping * dz/dt), delta = penetration (N/m); default 1e6 */
  double damping;              /* (N s/m); default 1e3 */
  double tangential_damping;   /* friction F_t = -v_t * min(tangential_damping, friction_mu * F_n / |v_t|) (N s/m); default 1e3 */
  double friction_mu;          /* default 0.6 (robot.urdf mu1 / mu2 of the feet) */
  double joint_damping[18];    /* viscous joint damping (N m s/rad); default robot.urdf <dynamics damping>: 0.05 legs, 0 arm */
  int32_t substeps_per_ms;     /* semi-implicit Euler substeps per simulated millisecond; default 4 */
} qmb200_sim_params;
int qmb200_sim_get_params(const qmb200_handle* h, qmb200_sim_params* out);
/* rejects non-finite values, foot_radius / stiffness / damping / tangential_damping / friction_mu <= 0, joint_damping < 0, substeps_per_ms < 1 */
int qmb200_sim_set_params(qmb200_handle* h, const qmb200_sim_params* p);
/* Advance every robot by `duration` s (0 < duration <= 1) with the effort held, as one writeSim → physics step: effort is clipped to the URDF effort
 * limits (gazebo_ros_control DefaultRobotHWSim), q and v are updated in place; rbd = the measured state at the end (qm_estimation's ground-truth
 * layout, EE pose included); contact = 4-bit mask of the feet with a positive normal force in the last substep (LF=8 RF=4 LH=2 RH=1);
 * status = QMB200_ST_NAN (non-finite state) | QMB200_ST_NOT_PD (mass matrix not positive definite: the robot stops at that substep).
 * status is this plant's own word: nothing is OR-ed into the controller's. */
int qmb200_sim_step(qmb200_handle* h, double duration, const double* effort /*[B][18]*/, double* q /*[B][24] in-out*/, double* v /*[B][24] in-out*/,
                    double* rbd /*[B][55]*/, int32_t* contact /*[B]*/, int32_t* status /*[B]*/);
int qmb200_sim_step_dev(qmb200_handle* h, double duration, const double* effort, double* q, double* v, double* rbd, int32_t* contact, int32_t* status, void* cuda_stream);
/* Per-robot plant variation, kept in the handle and applied by every qmb200_sim_step(_ext)(_dev) call (plant properties, like qmb200_sim_params):
 *   friction_mu[B]   the feet's Coulomb coefficient of robot b, in place of qmb200_sim_params.friction_mu
 *   payload[B][8]    layout: [m_ee, o_ee_x, o_ee_y, o_ee_z, m_base, o_base_x, o_base_y, o_base_z]
 *                    two point masses (kg) rigidly attached at o_ee (m, end-effector frame) and o_base (m, base frame); no rotational inertia.
 * These are plant properties only: the controller's model (MPC, WBC) is set apart with qmb200_set_model_payload, so a run can tell the controller the
 * truth, an estimate or nothing (the model mismatch is then the experiment).  qmb200_sim_standing_state ignores friction_mu and payload, so
 * a payload shifts the static pre-load of the standing state (by micrometres per kilogram at the default stiffness); it does follow the robot terrain.
 * Host arrays, copied to the device; synchronous (waits for the device).  NULL clears that override.  Rejects a non-finite or <= 0 friction_mu,
 * a non-finite payload entry and a negative mass; on rejection the stored values stay unchanged. */
int qmb200_sim_set_robot_params(qmb200_handle* h, const double* friction_mu /*[B] or NULL*/, const double* payload /*[B][8] or NULL*/);
/* The stored values; where an override is not set: friction_mu = qmb200_sim_params.friction_mu, payload = 0.  set_mask: 1 = friction_mu, 2 = payload.
 * Any output may be NULL. */
int qmb200_sim_get_robot_params(const qmb200_handle* h, double* friction_mu /*[B]*/, double* payload /*[B][8]*/, int32_t* set_mask);
/* qmb200_sim_step(_dev) plus external wrenches held over the whole step; wrench NULL = qmb200_sim_step(_dev).
 *   wrench[B][12]    layout: [f_base_x, f_base_y, f_base_z, n_base_x, n_base_y, n_base_z, f_ee_x, f_ee_y, f_ee_z, n_ee_x, n_ee_y, n_ee_z]
 *                    forces (N) and moments (N m) in the world frame; each moment is about its own frame's origin (the base origin q[0:3], the
 *                    end-effector frame origin).  Not validated: a non-finite wrench shows as QMB200_ST_NAN. */
int qmb200_sim_step_ext(qmb200_handle* h, double duration, const double* effort /*[B][18]*/, const double* wrench /*[B][12] or NULL*/, double* q /*[B][24] in-out*/,
                        double* v /*[B][24] in-out*/, double* rbd /*[B][55]*/, int32_t* contact /*[B]*/, int32_t* status /*[B]*/);
int qmb200_sim_step_ext_dev(qmb200_handle* h, double duration, const double* effort, const double* wrench, double* q, double* v, double* rbd, int32_t* contact,
                            int32_t* status, void* cuda_stream);
/* Per-robot terrain: heightfield tiles under the feet in place of the plane z = ground_height, applied by every qmb200_sim_step(_ext)(_dev) call.
 * The library holds n_tiles tiles on one grid of nx x ny nodes (both >= 2) with spacing cell (m); heights[n_tiles][ny][nx] are absolute world z (m).
 * Robot b stands on tile[b] (-1: the plane z = ground_height) whose node (0, 0) lies at world origin[b] = (x, y), so node (i, j) lies at
 * origin + (i cell, j cell).  At a foot centre (x, y, z) the ground is bilinear in the cell under (x, y), with height H and gradient (gx, gy); outside the
 * tile the border height continues with zero gradient across the clamped axis.  Contact is against the local tangent plane: s = sqrt(1 + gx^2 + gy^2),
 * n = (-gx, -gy, 1) / s, penetration delta = (H - (z - r s)) / s, F_n = max(0, stiffness delta - damping v.n) for delta > 0, v_t = v - (v.n) n, friction
 * as above on v_t; F = F_n n + F_t.  With zero gradient this is the plane law bit for bit, so tile -1 or a constant tile at ground_height changes nothing.
 * No link other than the feet collides; tiles are not rotated.
 * qmb200_sim_set_terrain: heights NULL clears the library and with it the robot terrain and the state estimator's ground map.  Rejects n_tiles < 1, nx
 * or ny < 2, a non-finite or non-positive cell, a non-finite height, a library whose byte count overflows, and a library with fewer tiles than a robot
 * or the estimator's ground map (qmb200_state_est_set_ground) references.
 * qmb200_sim_set_robot_terrain: tile NULL clears the robot terrain (every robot on the plane); rejects a tile outside [-1, n_tiles) and a non-finite origin.
 * Both are synchronous (they wait for the device); on rejection the stored values stay unchanged. */
int qmb200_sim_set_terrain(qmb200_handle* h, int32_t n_tiles, int32_t nx, int32_t ny, double cell, const double* heights /*[n_tiles][ny][nx] or NULL: clear*/);
/* The library: n_tiles = 0 (nx = ny = 0, cell = 0) when none is set; heights [n_tiles][ny][nx] is written when non-NULL.  Any output may be NULL. */
int qmb200_sim_get_terrain(const qmb200_handle* h, int32_t* n_tiles, int32_t* nx, int32_t* ny, double* cell, double* heights /*or NULL*/);
int qmb200_sim_set_robot_terrain(qmb200_handle* h, const int32_t* tile /*[B] or NULL: clear*/, const double* origin /*[B][2]*/);
/* The robot terrain; where none is set tile = -1, origin = 0 and is_set = 0.  Any output may be NULL. */
int qmb200_sim_get_robot_terrain(const qmb200_handle* h, int32_t* tile /*[B]*/, double* origin /*[B][2]*/, int32_t* is_set);
/* Host utility: the nominal standing configuration (defaultJointState, base at the given x, y, yaw, zero roll and pitch) with the base height at
 * which the four foot spheres carry m g / 4 each at the static penetration of the current params; v = 0.  With robot terrain set n must equal the
 * batch size and row r stands on robot r's ground: roll and pitch tilt the base onto the plane fitted through the ground heights under the four feet
 * (a few fixed-point iterations, since the feet move with the tilt), and the base height puts the deepest foot at the static penetration m g / (4 k). */
int qmb200_sim_standing_state(const qmb200_handle* h, int32_t n, const double* xy_yaw /*[n][3]*/, double* q /*[n][24]*/, double* v /*[n][24]*/);

/* ---- sensors of the plant: the IMU block of QMHWSim::readSim (qm_gazebo/src/QMHWSim.cpp:51-69) and the joint handles it fills, batched on the device.
 *      The IMU link unitree_imu sits at the base origin with the base's axes (robot.urdf), so with R = R(zyx) and w the world angular velocity:
 *        sensors[QMB200_SENSORS] = [quat xyzw(4) of R exp([n_o]x), gyro(3) = R^T w + n_g, accel(3) = R^T((v_lin - v_prev_lin) / dt - g) + n_a, joint pos(18)
 *                                   = q[6:24] + n_q, joint vel(18) = v[6:24] + n_v],  g = (0, 0, -9.81)
 *      The accelerometer reads the mean acceleration over the step that started at v_prev.  The contact flags are the mask qmb200_sim_step returns.
 *      Each noise term is sigma * N(0, 1), drawn as a pure function of (seed, robot, sample, channel): a counter-based integer hash and Box-Muller, so a
 *      draw depends neither on the batch nor on the launch; robot = the robot's index in the handle's batch plus rank * batch with a communicator
 *      (qmb200_comm_init).  The orientation noise n_o ~ N(0, sigma_orientation^2 1) is a rotation vector in the body frame.  All sigmas default to 0 (the
 *      reference's readSim, whose noise is a TODO); qm_gazebo/config/default.yaml:3-8 gives the covariances 0.0012 / 0.0004 / 0.01 of orientation,
 *      angular velocity and linear acceleration, i.e. sigma 0.0346 rad, 0.02 rad/s and 0.1 m/s^2. */
#define QMB200_SENSORS 46
typedef struct qmb200_sensor_params {
  uint64_t seed;
  double sigma_orientation, sigma_gyro, sigma_accel, sigma_joint_pos, sigma_joint_vel;   /* rad, rad/s, m/s^2, rad, rad/s */
} qmb200_sensor_params;
int qmb200_sim_get_sensor_params(const qmb200_handle* h, qmb200_sensor_params* out);
/* rejects a non-finite or negative sigma; on rejection the stored values stay unchanged */
int qmb200_sim_set_sensor_params(qmb200_handle* h, const qmb200_sensor_params* p);
/* sensors [B][46] of the plant state (q, v) [B][24] after a step of dt s (finite, > 0) that started at velocity v_prev [B][24] (owned by the caller);
 * sample numbers the reading for the noise. */
int qmb200_sim_read_sensors(qmb200_handle* h, double dt, int64_t sample, const double* q /*[B][24]*/, const double* v /*[B][24]*/, const double* v_prev /*[B][24]*/,
                            double* sensors /*[B][46]*/);
int qmb200_sim_read_sensors_dev(qmb200_handle* h, double dt, int64_t sample, const double* q, const double* v, const double* v_prev, double* sensors, void* cuda_stream);

/* ---- base state estimation, the seam of StateEstimateBase::update (qm_estimation/src/StateEstimateBase.cpp:41-78, fed by
 *      QMController::updateStateEstimation, qm_controllers/src/QMController.cpp:202-244): a linear Kalman filter per robot on
 *      x = [p_base(3), v_base(3), p_foot(4 x 3, contact order LF, RF, LH, RH)] in the world frame, from the sensors above and the contact mask.
 *      Orientation and angular velocity come from the IMU as read (zyx from the quaternion, yaw in (-pi, pi]; w = R gyro); the legs' kinematics at the
 *      encoder readings give each foot's offset r_i from the base and its velocity.  Predict: p += v dt + a dt^2 / 2, v += a dt with a = R accel + g,
 *      feet constant, P = A P A^T + dt diag(process).  Update with 28 rows: p_base - p_foot_i = -r_i, v_base = -dr_i/dt and p_foot_i,z = foot_height per
 *      foot.  A foot not in contact has its process and measurement variances scaled by swing_scale.  The foot-height rows assume the plane
 *      z = ground_height unless a ground map is set (qmb200_state_est_set_ground below).
 *   process_base_pos, process_base_vel, process_foot    process noise per second: m^2/s, (m/s)^2/s, m^2/s
 *   meas_foot_pos, meas_foot_vel, meas_foot_height      measurement variances: m^2, (m/s)^2, m^2
 *   swing_scale                                         factor on a swing foot's variances
 *   foot_height                                         world z of a stance foot frame: ground_height + foot_radius - m g / (4 stiffness); the default is that of
 *                                                       the default plant params and the model's mass
 *   p0_base_pos, p0_base_vel, p0_foot                   P = diag(p0) at the reset (m^2, (m/s)^2, m^2) */
typedef struct qmb200_state_est_params {
  double process_base_pos, process_base_vel, process_foot, meas_foot_pos, meas_foot_vel, meas_foot_height, swing_scale, foot_height, p0_base_pos, p0_base_vel, p0_foot;
} qmb200_state_est_params;
int qmb200_state_est_get_params(const qmb200_handle* h, qmb200_state_est_params* out);
/* rejects a non-finite value and a negative one (foot_height may take any finite value); on rejection the stored values stay unchanged */
int qmb200_state_est_set_params(qmb200_handle* h, const qmb200_state_est_params* p);
/* (Re)starts the filter of every robot: p_base = base_pos [B][3] (required), v_base = 0, P = diag(p0), no call yet.  Synchronous. */
int qmb200_state_est_reset(qmb200_handle* h, const double* base_pos /*[B][3]*/);
/* One filter call per robot from sensors [B][46] (qmb200_sim_read_sensors) and the contact mask [B] (qmb200_sim_step) of a step of dt s (finite, > 0):
 * writes rbd_est [B][55] (include/qmb200.h layout: zyx, p, joints, w, v, joint rates, end-effector pose) for the controller.  The first call after a reset
 * only places the feet at p_base + r_i.  status [B] (written, not OR-ed): QMB200_ST_NAN for a non-finite input (nothing is written) or update,
 * QMB200_ST_NOT_PD when the innovation covariance fails its Cholesky; the robot then keeps x and P, and rbd_est is written from them. */
int qmb200_state_est_step(qmb200_handle* h, double dt, const double* sensors /*[B][46]*/, const int32_t* contact /*[B]*/, double* rbd_est /*[B][55]*/, int32_t* status /*[B]*/);
int qmb200_state_est_step_dev(qmb200_handle* h, double dt, const double* sensors, const int32_t* contact, double* rbd_est, int32_t* status, void* cuda_stream);
/* Synchronous: x [B][18], the diagonal of P [B][18] and the calls since the reset [B].  Any output may be NULL. */
int qmb200_state_est_get(qmb200_handle* h, double* x /*[B][18]*/, double* p_diag /*[B][18]*/, int32_t* samples /*[B]*/);
/* Releases the filter state.  Step and get fail until the next reset.  Stopping a filter that is not running does nothing and returns 0, as
 * qmb200_payload_est_stop does, so a caller's clean-up may stop unconditionally. */
int qmb200_state_est_stop(qmb200_handle* h);
/* The estimator's ground map: per robot a tile of the plant's library (qmb200_sim_set_terrain; -1: the plane) with its node (0, 0) at world origin[b],
 * as qmb200_sim_set_robot_terrain takes them but held apart from the plant's own rows, so a run may give the estimator a map that differs from the
 * ground.  With a map, foot f's height row is h_f = p_f,z - H(p_f,x, p_f,y) = s_f (foot_height - ground_height), s_f = sqrt(1 + gx^2 + gy^2): the
 * plant's contact law holds a stance sphere centre at r - delta along the normal of the local tangent plane.  H and its gradient come from the plant's
 * lookup at the predicted foot position, ground_height is the plant's when the step is launched, and the row is linearised there (-gx, -gy at the
 * foot's x and y).  A tile of -1 or a constant tile at ground_height gives the plane's numbers bit for bit.  tile NULL clears the map; rejects a tile
 * outside [-1, n_tiles) and a non-finite origin.  Synchronous; on rejection the stored map stays unchanged.  The map survives qmb200_state_est_reset
 * and _stop; qmb200_sim_set_terrain refuses a library without a tile the map references, and clearing the library clears the map. */
int qmb200_state_est_set_ground(qmb200_handle* h, const int32_t* tile /*[B] or NULL: clear*/, const double* origin /*[B][2]*/);
/* The ground map; where none is set tile = -1, origin = 0 and is_set = 0.  Any output may be NULL. */
int qmb200_state_est_get_ground(const qmb200_handle* h, int32_t* tile /*[B]*/, double* origin /*[B][2]*/, int32_t* is_set);

/* ---- attitude filter, between the sensors and the state estimator: a multiplicative (error-state) Kalman filter per robot on SO(3) with gyro-bias
 *      states.  The reference has none (StateEstimateBase::updateImu passes the IMU quaternion through); a real robot's IMU filters on board.
 *      Nominal q_hat (world <- body) and b_hat, error [dtheta, db] with R = R_hat Exp(dtheta) (body frame), P 6x6.  Per call, on the row sensors[46]
 *      (qmb200_sim_read_sensors): predict q_hat <- q_hat (x) Exp((gyro - b_hat) dt), P <- F P F^T + dt diag(process), F = [[Exp(w dt)^T, -dt 1], [0, 1]];
 *      update with the row's quaternion q_m: r = Log(q_hat^-1 (x) q_m) (sign with w >= 0, so q_m and -q_m agree), S = P_tt + meas_orientation 1,
 *      K = P H^T S^-1, q_hat <- q_hat (x) Exp(K_t r), b_hat += K_b r, P <- P - K H P.  The accelerometer is not used.  The row is rewritten in place:
 *      quaternion = q_hat (w >= 0), gyro = gyro - b_hat; every other column is untouched, so qmb200_state_est_step reads the filtered row unchanged.
 *   process_attitude, process_gyro_bias    process noise per second: rad^2/s (gyro white noise as angle random walk), (rad/s)^2/s (bias random walk)
 *   meas_orientation                       variance of each axis of the orientation reading's error, rad^2 (> 0)
 *   p0_attitude, p0_gyro_bias              P = diag(p0) at the reset: rad^2, (rad/s)^2 */
typedef struct qmb200_attitude_params {
  double process_attitude, process_gyro_bias, meas_orientation, p0_attitude, p0_gyro_bias;   /* rad^2/s, (rad/s)^2/s, rad^2, rad^2, (rad/s)^2 */
} qmb200_attitude_params;
int qmb200_attitude_get_params(const qmb200_handle* h, qmb200_attitude_params* out);
/* rejects a non-finite or negative value and meas_orientation <= 0; on rejection the stored values stay unchanged */
int qmb200_attitude_set_params(qmb200_handle* h, const qmb200_attitude_params* p);
/* (Re)starts the filter of every robot: b_hat = 0, P = diag(p0), no call yet; the next call takes q_hat from its reading.  Synchronous. */
int qmb200_attitude_reset(qmb200_handle* h);
/* One filter call per robot on sensors [B][46] (in-out) of a step of dt s (finite, > 0).  The first call after a reset sets q_hat to the normalised
 * reading.  status [B] (written, not OR-ed): QMB200_ST_NAN for a non-finite quaternion or gyro input (neither the row nor the state is touched) or
 * update (the robot keeps its state and the row is written from it). */
int qmb200_attitude_step(qmb200_handle* h, double dt, double* sensors /*[B][46] in-out*/, int32_t* status /*[B]*/);
int qmb200_attitude_step_dev(qmb200_handle* h, double dt, double* sensors, int32_t* status, void* cuda_stream);
/* Synchronous: q_hat [B][4] (xyzw, as stored: its sign is continuous from call to call), b_hat [B][3], the diagonal of P [B][6] and the calls since the
 * reset [B].  Any output may be NULL. */
int qmb200_attitude_get(qmb200_handle* h, double* quat /*[B][4]*/, double* gyro_bias /*[B][3]*/, double* p_diag /*[B][6]*/, int32_t* samples /*[B]*/);
/* Releases the filter state.  Step and get fail until the next reset.  Stopping a filter that is not running does nothing and returns 0. */
int qmb200_attitude_stop(qmb200_handle* h);

/* ---- slip detector, between the sensors (and the attitude filter) and the state estimator: per robot and foot in contact, a test of the foot's
 *      velocity against the estimator's prior.  The estimator's leg-velocity rows (v_base = -dr_i/dt) assume a stance foot at rest; a foot that slides
 *      breaks them.  Per call, from the row sensors[46] (the legs as qmb200_state_est_step reads them) and the estimator's stored state (read only):
 *      v- = v_hat + a dt (a = R accel + g), Sigma- = P_vv + dt process_base_vel 1; per foot i in contact u_i = v- + dr_i/dt (the world velocity of the
 *      foot point) and d2_i = u_i^T (Sigma- + meas_slip 1)^-1 u_i.  A foot becomes slipping when d2_i > gate and is trusted again after hold consecutive
 *      calls with d2_i < release (hold 0 acts as 1); a foot out of contact is cleared.  stance = contact & ~slip is the mask to pass to
 *      qmb200_state_est_step in place of the plant's: a slipping foot is then handled as a swing foot.
 *   gate, release     thresholds on d2 (chi-square, 3 degrees of freedom), 0 < release <= gate
 *   meas_slip         variance added per axis for a stance foot's own velocity (its creep under the compliant contact), (m/s)^2, >= 0
 *   hold              calls below release before a slipping foot is trusted again, >= 0 */
typedef struct qmb200_slip_params {
  double gate, release, meas_slip;   /* -, -, (m/s)^2 */
  int32_t hold;                      /* calls */
} qmb200_slip_params;
int qmb200_slip_get_params(const qmb200_handle* h, qmb200_slip_params* out);
/* rejects non-finite values, gate <= 0, release outside (0, gate], meas_slip < 0 and hold < 0; on rejection the stored values stay unchanged */
int qmb200_slip_set_params(qmb200_handle* h, const qmb200_slip_params* p);
/* (Re)starts the detector of every robot: no foot slipping, counters zero.  Synchronous. */
int qmb200_slip_reset(qmb200_handle* h);
/* One detector call per robot of a step of dt s (finite, > 0), before the estimator's step on the same row: from sensors [B][46] and the contact mask
 * contact_in [B], writes stance_out [B] = contact_in & ~slip_out and slip_out [B] (the feet in contact flagged as slipping, contact bit order).  Needs
 * the detector and the state estimator running.  Before the estimator's first call after its reset, and for a robot with a non-finite reading
 * (status QMB200_ST_NAN), contact_in passes through and the robot's detector state is untouched.  status [B] is written, not OR-ed. */
int qmb200_slip_step(qmb200_handle* h, double dt, const double* sensors /*[B][46]*/, const int32_t* contact_in /*[B]*/, int32_t* stance_out /*[B]*/,
                     int32_t* slip_out /*[B]*/, int32_t* status /*[B]*/);
int qmb200_slip_step_dev(qmb200_handle* h, double dt, const double* sensors, const int32_t* contact_in, int32_t* stance_out, int32_t* slip_out, int32_t* status,
                         void* cuda_stream);
/* Synchronous: the slip mask [B], per foot the calls below release counted towards hold [B][4] and the onsets since the reset [B][4] (feet in contact
 * order LF, RF, LH, RH).  Any output may be NULL. */
int qmb200_slip_get(qmb200_handle* h, int32_t* mask /*[B]*/, int32_t* hold /*[B][4]*/, int32_t* onsets /*[B][4]*/);
/* Releases the detector state.  Step and get fail until the next reset.  Stopping a detector that is not running does nothing and returns 0. */
int qmb200_slip_stop(qmb200_handle* h);

/* ---- per-robot restart: QMController::starting (QMController.cpp:98-126) for single robots of a batch, inside a stream-ordered loop (DESIGN.md §4.10).
 *      The start image holds, per robot, the rows of every component running when it is saved: the state estimator, attitude filter, slip detector and
 *      payload estimator states, the model payload rows (qmb200_set_model_payload, as a commit may have left them) and the device gait schedule with
 *      its timeline cursor.  Handle settings (parameters, tuning rows, plant robot params, terrain, ground map, gait templates, command timeline) are not
 *      state and are never written.  The gait schedule's pending command slots (qmb200_gait_dev_command) are cleared, not imaged.  The image is the
 *      handle's own robot-state snapshot (below) of blocks 0-7, with their generations: each reset, stop or re-allocation of an imaged component (and
 *      qmb200_gait_dev_set_commands, which resets the cursors) makes the image stale for it. */
/* Saves the image of the components running now, replacing any previous one.  Synchronous. */
int qmb200_robot_image_save(qmb200_handle* h);
/* Frees the image (qmb200_destroy does too).  Clearing when none is saved does nothing and returns 0. */
int qmb200_robot_image_clear(qmb200_handle* h);
/* One launch, no host work: for every robot with mask[b] != 0 the imaged rows return to the image, both MPC warm-start sides forget the robot's
 * solution (n_nodes = 0, what qmb200_mpc_reset does for all), its WBC last input is zeroed, its hw_write FIFO emptied and, while the device gait
 * schedule runs, its pending command dropped (a command decided on the old episode's state never reaches the new one).  Robots with mask[b] == 0
 * are not written.  Fails, naming the block and writing nothing, when no image is saved or, as qmb200_robot_state_load_dev does for blocks 0-7, an
 * imaged block was reset, stopped or re-allocated since or no longer exists, or one of those blocks exists now that was not imaged. */
int qmb200_robot_image_restore(qmb200_handle* h, const int32_t* mask /*[B]*/);
int qmb200_robot_image_restore_dev(qmb200_handle* h, const int32_t* mask /*[B] device*/, void* cuda_stream);

/* ---- robot-state snapshots: the start image generalised to any window boundary, with the warm state, restored onto any robot (DESIGN.md §4.17).
 *      A snapshot holds, per robot, every [B][...] block of the handle that a later solve, update, plant step or estimator step reads before it writes,
 *      in this order (block i is bit i of qmb200_robot_state_desc.blocks; a block is held when it exists now):
 *        0 state estimator  1 attitude filter  2 slip detector  3 payload estimator  4 model payload rows  5 their SRBD constants
 *        6 device gait schedule  7 its timeline cursor  8-12 the current MPC solution side (n_nodes, node times, events, x, u: the warm start)
 *        13 the WBC's last input  14-16 the hw_write FIFO (commands, stamps, head / count)  17 the pending gait command
 *        18 plant friction  19 plant payload  20 plant robot terrain  21 state estimator ground map  22 tuning rows
 *        23-27 the gait schedule's command timeline (t, template, cmd_vel, end-effector kind, end-effector row)
 *        28-31 the MPC's copy of the last solve's mode schedule (event count, event times, modes), which every policy evaluation (qmb200_update,
 *              qmb200_policy_eval) reads until the next solve, and that solve's status
 *        32 end-effector frame rows (qmb200_set_ee_frame; held while they are set): a robot branched from another takes its frame with its hold
 *      A load may therefore sit anywhere in a loop: before a solve, or between a solve and the updates that evaluate its policy.
 *      It holds no shared settings (tiles, templates, parameters, gains), no draw ranges, curriculum or start image, and no per-call intermediates.  The
 *      buffer is caller-owned device memory of B * qmb200_robot_state_bytes bytes, one block [B][bytes] after the other.  Each block carries the
 *      generation of what owns it, bumped when that is reset, stopped, allocated, re-allocated or cleared: a load refuses a snapshot whose rows no
 *      longer belong to the handle's state. */
#define QMB200_STATE_BLOCKS 33
typedef struct qmb200_robot_state_desc {
  int32_t batch;                        /* B of the handle that saved it */
  int32_t n_blocks;                     /* blocks held (set bits of blocks) */
  int64_t bytes;                        /* bytes per robot: the sum of the held blocks' row widths */
  uint64_t blocks;                      /* bit i: block i is held */
  uint64_t gen[QMB200_STATE_BLOCKS];    /* generation of each held block's owner at the save (0 where not held) */
} qmb200_robot_state_desc;
/* Bytes per robot of a snapshot of the blocks that exist now (> 0: the MPC solution side and the WBC input always do); -1 for a NULL handle. */
int64_t qmb200_robot_state_bytes(const qmb200_handle* h);
/* One launch on the stream, no host synchronisation: copies every robot's held blocks into buf (device, at least bytes = B * qmb200_robot_state_bytes)
 * in the handle's current state in stream order, and fills desc.  Fails before any launch, writing nothing, on a NULL or short buffer. */
int qmb200_robot_state_save_dev(qmb200_handle* h, void* buf /*device*/, int64_t bytes, qmb200_robot_state_desc* desc, void* cuda_stream);
/* One launch, no host synchronisation: every robot b with mask[b] != 0 takes robot source[b]'s rows of the snapshot (NULL source: its own, b), the MPC
 * solution into the side current at this call.  A source outside [0, B) leaves the robot untouched and sets status[b] = QMB200_ST_RESTORE; status [B]
 * (NULL: none) is written, not OR-ed, 0 for restored and unmasked robots.  The getters of the plant, model payload, tuning and terrain rows report the
 * loaded rows.  Fails before any launch, writing nothing and naming the block, when buf is NULL, the snapshot is of another batch, its block set differs
 * from the blocks that exist now or a block's generation moved since the save. */
int qmb200_robot_state_load_dev(qmb200_handle* h, const void* buf /*device*/, const qmb200_robot_state_desc* desc, const int32_t* mask /*[B] device*/,
                                const int32_t* source /*[B] device, NULL: b*/, int32_t* status /*[B] device, NULL: none*/, void* cuda_stream);
/* Host mask, source and status (staged on the handle's stream, synchronous); buf is device memory as for qmb200_robot_state_load_dev. */
int qmb200_robot_state_load(qmb200_handle* h, const void* buf, const qmb200_robot_state_desc* desc, const int32_t* mask /*[B]*/, const int32_t* source /*[B] or NULL*/,
                            int32_t* status /*[B] or NULL*/);
/* The fall rule of the closed-loop sweeps, one thread per robot on the plant's rbd [B][55]: robot b is fallen when its base rows (zyx, p) hold a
 * non-finite value, p_z - H(p_x, p_y) <= z_min with H the plant's ground under the base (its terrain tile, the plane ground_height otherwise), or
 * |pitch| or |roll| >= tilt_max.  fallen [B] = 1 / 0; count [B] (in-out) grows by one on a fallen call and drops to 0 otherwise.  Rejects a non-finite
 * z_min and tilt_max that is non-finite or <= 0. */
int qmb200_fall_detect(qmb200_handle* h, const double* rbd /*[B][55]*/, double z_min, double tilt_max, int32_t* count /*[B] in-out*/, int32_t* fallen /*[B]*/);
int qmb200_fall_detect_dev(qmb200_handle* h, const double* rbd, double z_min, double tilt_max, int32_t* count, int32_t* fallen, void* cuda_stream);

/* ---- per-episode plant draws (DESIGN.md §4.11): each episode of each robot gets a new plant, drawn on the device right after its restart.
 *   row[QMB200_EPISODE]  offset  0       friction_mu      the plant's Coulomb coefficient (qmb200_sim_set_robot_params)
 *                                1-8     payload          the plant's payload row, qmb200_sim_set_robot_params' layout
 *                                9-10    push_t_on, push_duration   s from the episode's start
 *                                11-22   wrench           the push, qmb200_sim_step_ext's layout
 *                                23-26   cmd_vel_x, cmd_vel_y, cmd_vel_z, cmd_yaw_rate   the base-frame velocity command
 * Column c of robot b in episode e is fma(u, hi[b][c] - lo[b][c], lo[b][c]) with u = ((mix64(h) >> 11) + 0.5) 2^-53 in (0, 1), h the splitmix64 finaliser
 * over (seed ^ a domain constant, global robot rank * B + b, e, c) in turn, as the sensor noise hashes its words: a pure function of those words and the
 * ranges, identical on host and device; a column with lo == hi is lo itself, byte for byte. */
#define QMB200_EPISODE 27
#define QMB200_EPISODE_MODEL_PAYLOAD 1   /* link: the payload also goes to the controller's model payload and its SRBD rows (qmb200_set_model_payload) */
#define QMB200_EPISODE_MPC_FRICTION 2    /* link: friction_mu also goes to the tuning rows' MPC friction coefficient (qmb200_set_robot_tuning) */
#define QMB200_EPISODE_WBC_FRICTION 4    /* link: friction_mu also goes to the tuning rows' WBC friction coefficient */
/* Per-robot ranges lo, hi [B][QMB200_EPISODE] and the seed (its 64 bits; the draw reads it as unsigned).  NULL lo and hi clear them.  Rejects a non-finite
 * bound, lo > hi, a non-finite hi - lo, friction_mu lo <= 0 and a negative lo of a payload mass, push_t_on or push_duration, naming the field and the
 * robot; on rejection the stored ranges stay unchanged.  Setting ranges makes sure the plant's robot params (qmb200_sim_set_robot_params) are set, at
 * the values in force where they were not, so the sampler has rows to write.  Host arrays; synchronous. */
int qmb200_episode_set_ranges(qmb200_handle* h, const double* lo /*[B][QMB200_EPISODE] or NULL*/, const double* hi /*[B][QMB200_EPISODE] or NULL*/, int64_t seed);
/* The stored ranges and seed (zeros when none are set); is_set = 1 when ranges are set.  Any output may be NULL. */
int qmb200_episode_get_ranges(const qmb200_handle* h, double* lo /*[B][QMB200_EPISODE]*/, double* hi /*[B][QMB200_EPISODE]*/, int64_t* seed, int32_t* is_set);
/* One launch, no host work: every robot with mask[b] != 0 draws episode[b]'s row into rows[b] and the plant's robot params friction_mu[b] and payload[b];
 * link (QMB200_EPISODE_* bits) also writes the model payload row with its SRBD row (srbd_payload_fold, as a payload estimator commit does) and the tuning
 * rows' friction coefficients.  Robots with mask[b] == 0 are not written.  The getters (qmb200_sim_get_robot_params, qmb200_get_model_payload,
 * qmb200_get_robot_tuning) wait for the device and report the rows written.  Fails, writing nothing, when no ranges are set, the plant's robot params
 * were cleared since, a link's rows are not set, or the model payload link is asked while the payload estimator runs.  The start image
 * (qmb200_robot_image_save) holds no plant or tuning rows: restore first, then sample. */
int qmb200_episode_sample(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* episode /*[B]*/, int32_t link, double* rows /*[B][QMB200_EPISODE] in-out*/);
int qmb200_episode_sample_dev(qmb200_handle* h, const int32_t* mask, const int32_t* episode, int32_t link, double* rows, void* cuda_stream);
/* Host only: the rows [n][QMB200_EPISODE] of robots robot[n] (in [0, B)) in episodes episode[n] on the stored ranges and seed, what the sampler draws. */
int qmb200_episode_draw(const qmb200_handle* h, int32_t n, const int32_t* robot /*[n]*/, const int32_t* episode /*[n]*/, double* rows /*[n][QMB200_EPISODE]*/);

/* ---- per-episode spawns (DESIGN.md §4.12): each episode of each robot starts on new ground, drawn on the device right after its restart.
 *   row[QMB200_SPAWN]  0  tile    the plant's tile for the episode, an integer in [-1, n_tiles) (-1: the plane)
 *                      1  dx      the robot stands dx, dy m further along its tile, world axes: the tile's origin becomes the robot's origin at the set
 *                      2  dy      minus (dx, dy).  The base's world x, y do not move; the ground moves under it.  Tiles are not rotated.
 *                      3  yaw     the base yaw, in [-pi, pi]
 * Column c of robot b in episode e: a uniform u in (0, 1) of (seed ^ a domain constant of its own, global robot rank * B + b, e, c) as the episode draw
 * hashes them; dx, dy and yaw are fma(u, hi - lo, lo), the tile is lo + min(floor(u (hi - lo + 1)), hi - lo); a column with lo == hi is lo itself. */
#define QMB200_SPAWN 4
#define QMB200_SPAWN_GROUND_MAP 1   /* link: the drawn terrain row also goes to the state estimator's ground map (qmb200_state_est_set_ground) */
/* Per-robot ranges lo, hi [B][QMB200_SPAWN] and the seed.  NULL lo and hi clear them.  Rejects a non-finite bound, lo > hi, a non-finite hi - lo, tile
 * bounds that are not integers in [-1, n_tiles) of the library in force and yaw bounds outside [-pi, pi], naming the field and the robot; on rejection
 * the stored ranges stay unchanged.  The set takes the robots' tile origins from the plant's robot terrain rows in force (zeros where none are set),
 * and when any tile bound is >= 0 makes sure those rows exist (tile -1, origin 0 where they were not set).  Host arrays; synchronous. */
int qmb200_spawn_set_ranges(qmb200_handle* h, const double* lo /*[B][QMB200_SPAWN] or NULL*/, const double* hi /*[B][QMB200_SPAWN] or NULL*/, int64_t seed);
/* The stored ranges and seed (zeros when none are set); is_set = 1 when ranges are set.  Any output may be NULL. */
int qmb200_spawn_get_ranges(const qmb200_handle* h, double* lo /*[B][QMB200_SPAWN]*/, double* hi /*[B][QMB200_SPAWN]*/, int64_t* seed, int32_t* is_set);
/* One launch, no host work: every robot with mask[b] != 0 draws episode[b]'s spawn row into rows[b] and stands there.  It writes the plant's robot terrain
 * row [tile, origin - (dx, dy)] (when the plant has robot terrain rows) and, with link QMB200_SPAWN_GROUND_MAP, the estimator's ground-map row to the same
 * values; q[b]: x, y as given, the standing pose on that ground (qmb200_sim_standing_state's, on the plane bit for bit), the drawn yaw, defaultJointState;
 * v[b] = 0; rbd[b] the measured state at (q, 0) with the end-effector pose; contact[b] the feet the plant's contact law presses into the ground there;
 * x_obs[b] the observation of rbd[b] (qmb200_centroidal_state_from_rbd); last_ee[b] (the held end-effector target, position and quaternion xyzw) turned
 * about the vertical through the base by the drawn yaw minus the given q[b]'s yaw; rbd_est[b] = rbd[b] when rbd_est is given; and the rows the resets
 * write for every component that runs: the state estimator's as qmb200_state_est_reset at the new base position (its next call places the feet), the
 * attitude filter's as qmb200_attitude_reset, the slip detector's zeroed.  Robots with mask[b] == 0 are not written.  The getters
 * (qmb200_sim_get_robot_terrain, qmb200_state_est_get_ground, qmb200_sim_standing_state) wait for the device and report the rows written.  Fails,
 * writing nothing, when no ranges are set, the library has fewer tiles than a stored bound, the ground-map link has no map, or the plant's robot terrain
 * rows were cleared since the set. */
int qmb200_spawn_sample(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* episode /*[B]*/, int32_t link, double* rows /*[B][QMB200_SPAWN] in-out*/,
                        double* q /*[B][24] in-out*/, double* v /*[B][24] in-out*/, double* rbd /*[B][55] in-out*/, int32_t* contact /*[B] in-out*/,
                        double* x_obs /*[B][30] in-out*/, double* last_ee /*[B][7] in-out*/, double* rbd_est /*[B][55] in-out or NULL*/);
int qmb200_spawn_sample_dev(qmb200_handle* h, const int32_t* mask, const int32_t* episode, int32_t link, double* rows, double* q, double* v, double* rbd, int32_t* contact,
                            double* x_obs, double* last_ee, double* rbd_est, void* cuda_stream);
/* One launch, no host work (DESIGN.md §4.18): every robot with mask[b] != 0 stands on the given row rows[b] exactly as qmb200_spawn_sample_dev stands a
 * robot on a drawn row, writing the same buffers and rows; its offsets count from origin[b] (the tile's origin becomes origin[b] - (dx, dy)).  No ranges
 * are needed.  The row is checked on the device: the tile an integer in [-1, n_tiles) of the library in force, a tile >= 0 only where the plant has
 * robot terrain rows, dx and dy finite, the yaw in [-pi, pi].  A rejected robot is not written and gets status[b] = QMB200_ST_SPAWN; status [B] is
 * written, not OR-ed: 0 for accepted robots and for robots with mask[b] == 0, which are not written.  Fails, writing nothing, on a NULL buffer (rbd_est
 * may be NULL), unknown link bits, or the ground-map link without a map. */
int qmb200_spawn_place(qmb200_handle* h, const int32_t* mask /*[B]*/, const double* rows /*[B][QMB200_SPAWN]*/, const double* origin /*[B][2]*/, int32_t link,
                       double* q /*[B][24] in-out*/, double* v /*[B][24] in-out*/, double* rbd /*[B][55] in-out*/, int32_t* contact /*[B] in-out*/,
                       double* x_obs /*[B][30] in-out*/, double* last_ee /*[B][7] in-out*/, double* rbd_est /*[B][55] in-out or NULL*/, int32_t* status /*[B]*/);
int qmb200_spawn_place_dev(qmb200_handle* h, const int32_t* mask, const double* rows, const double* origin, int32_t link, double* q, double* v, double* rbd,
                           int32_t* contact, double* x_obs, double* last_ee, double* rbd_est, int32_t* status, void* cuda_stream);
/* One launch, no host work (DESIGN.md §4.18): every robot with mask[b] != 0 writes into rows[b] the spawn row that, once the robot is back at its start
 * pose q_start[b] and placed with qmb200_spawn_place(_dev) and the same origin, stands it on the ground point under its base now (rbd[b]) with its
 * heading now: tile = the plant's robot terrain tile (-1 without robot terrain rows), (dx, dy) = (x - x_start, y - y_start) + (origin - the robot
 * terrain origin now) (origin itself without rows), yaw = rbd[b]'s yaw wrapped into [-pi, pi].  On the plane only the heading carries over: a spawn
 * keeps the base's world x, y.  Rows of robots with mask[b] == 0 are not written.  Fails, writing nothing, on a NULL buffer. */
int qmb200_spawn_here(qmb200_handle* h, const int32_t* mask /*[B]*/, const double* rbd /*[B][55]*/, const double* q_start /*[B][24]*/, const double* origin /*[B][2]*/,
                      double* rows /*[B][QMB200_SPAWN] in-out*/);
int qmb200_spawn_here_dev(qmb200_handle* h, const int32_t* mask, const double* rbd, const double* q_start, const double* origin, double* rows, void* cuda_stream);
/* Host only: the rows [n][QMB200_SPAWN] of robots robot[n] (in [0, B)) in episodes episode[n] on the stored ranges and seed, what the sampler draws. */
int qmb200_spawn_draw(const qmb200_handle* h, int32_t n, const int32_t* robot /*[n]*/, const int32_t* episode /*[n]*/, double* rows /*[n][QMB200_SPAWN]*/);

/* ---- per-episode metrics (DESIGN.md §4.13): each robot's episode is scored on the device from the plant's truth, one sample per plant step.
 * A sample is the plant's state after one step: its rbd, its contact mask and the effort held over the step.  The first sample of an episode opens it
 * (the start xy, the foot positions, the contact mask); per-sample terms count from the first sample, displacement terms (path, slip, touchdowns)
 * between consecutive samples from the second on.  A closed episode is one row of QMB200_METRICS doubles:
 *   0  duration          sum of dt over the samples (samples x dt at a fixed step) (s)
 *   1  end               why it closed: 0 run end (truncated), 1 respawn on a fall, 2 respawn at the episode length limit
 *   2  status            bitwise OR of the status words passed with its samples, as a double
 *   3  distance          planar distance between the base xy of the first and of the last sample (m)
 *   4  path_length       sum of the planar base displacement between consecutive samples (m)
 *   5  min_height        min of p_z - H(p_x, p_y), H the plant's ground under the base (its terrain row in force at the sample, as qmb200_fall_detect) (m)
 *   6  max_tilt          max of max(|pitch|, |roll|) (rad)
 *   7  vel_err_rms       RMS over the cmd_vel samples of |v_xy - v_ref,xy|, v_ref = target_states[b][0][0:2] (the cmd_vel target's world velocity) (m/s)
 *   8  yaw_rate_err_rms  RMS over the same samples of omega_z - cmd[b][3] (rad/s)
 *   9  ee_pos_err_rms    RMS of |p_ee - p_ref(t)|, p_ref the target trajectory's end-effector position at the sample's time, as the MPC interpolates it (m)
 *  10  ee_pos_err_max    max of the same (m)
 *  11  ee_ori_err_rms    RMS of the angle of q_ref^-1 q_ee, 2 atan2(|vec|, |w|) (rad)
 *  12  energy            sum over the samples and the 18 joints of |tau_j qd_j| dt (J)
 *  13  torque_rms        sqrt(mean over the samples of sum_j tau_j^2 / 18) (N m)
 *  14  slip              sum over feet and consecutive sample pairs with the foot's contact bit set in both of its foot frame's planar displacement (m)
 *  15  touchdowns        count of 0 -> 1 transitions of the four contact bits
 *  16  est_pos_err_rms   RMS of |p_est - p| over the samples passed with an estimate rbd_est (m)
 *  17  est_vel_err_rms   RMS of |v_est - v| over the same samples (m/s)
 * A cmd_vel sample is one whose robot's target kind is QMB200_TARGET_CMD_VEL (kind [B], or every robot when kind is NULL).  An RMS, max, min or distance
 * over no samples is NaN.
 * The open episode of each robot is an accumulator row of QMB200_METRICS_ACC doubles, owned by the caller; all zeros is an open, empty episode:
 *   0 samples  1 sum of dt  2 status OR  3-4 first base xy  5-6 last base xy  7-14 last foot xy [4][2] (contact order)  15 last contact mask  16 path
 *   17 min height  18 max tilt  19 cmd_vel samples  20-21 their squared velocity and yaw-rate errors  22 squared EE position errors  23 max EE error
 *   24 squared EE angles  25 energy  26 sum of sum_j tau_j^2 / 18  27 slip  28 touchdowns  29 samples with an estimate  30-31 their squared errors */
#define QMB200_METRICS 18
#define QMB200_METRICS_ACC 32
/* One launch, no host work: one sample of every robot into acc [B][QMB200_METRICS_ACC] (in-out).  rbd [B][55], contact [B] and effort [B][18] are the
 * plant's state after the step and the effort held over it; cmd [B][7] the target commands (cmd[b][3]: the commanded yaw rate); kind [B] or NULL the
 * robots' target kinds; n_target [B] (clamped to [1, QMB200_KMAX] as the MPC does), target_times [B][QMB200_KMAX] and target_states
 * [B][QMB200_KMAX][QMB200_TARGET] the target trajectories in force; time [B] the plant clock at the start of the step, so the sample lies at time + dt;
 * status [B] the words to OR into the episode's; rbd_est [B][55] or NULL the estimate.  The foot frames come from the joints of rbd, the ground from the
 * plant's terrain (qmb200_sim_set_terrain, qmb200_sim_set_robot_terrain).  Fails, writing nothing, on a null required buffer and a dt that is not finite
 * and > 0. */
int qmb200_metrics_step(qmb200_handle* h, double dt, const double* rbd /*[B][55]*/, const int32_t* contact /*[B]*/, const double* effort /*[B][18]*/,
                        const double* cmd /*[B][7]*/, const int32_t* kind /*[B] or NULL*/, const int32_t* n_target /*[B]*/, const double* target_times,
                        const double* target_states, const double* time /*[B]*/, const int32_t* status /*[B]*/, const double* rbd_est /*[B][55] or NULL*/,
                        double* acc /*[B][QMB200_METRICS_ACC] in-out*/);
int qmb200_metrics_step_dev(qmb200_handle* h, double dt, const double* rbd, const int32_t* contact, const double* effort, const double* cmd, const int32_t* kind,
                            const int32_t* n_target, const double* target_times, const double* target_states, const double* time, const int32_t* status,
                            const double* rbd_est, double* acc, void* cuda_stream);
/* One launch, no host work: every robot with mask[b] != 0 closes its episode: its row, with end[b] as column 1, goes to out[b][episode[b]] (out
 * [B][n_episodes][QMB200_METRICS], in-out) and its accumulator row is zeroed, which opens the next episode.  When episode[b] lies outside [0, n_episodes)
 * no row is written, QMB200_ST_OVERFLOW is OR-ed into status[b] and the accumulator is still zeroed.  Robots with mask[b] == 0 are not written.  Fails,
 * writing nothing, on a null buffer and n_episodes < 1; the host variant also on a masked end outside {0, 1, 2}, which the device variant, unable to read
 * it on the host, refuses per robot by writing nothing of that robot. */
int qmb200_metrics_close(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* end /*[B]*/, const int32_t* episode /*[B]*/, int32_t n_episodes,
                         double* acc /*[B][QMB200_METRICS_ACC] in-out*/, double* out /*[B][n_episodes][QMB200_METRICS] in-out*/, int32_t* status /*[B] in-out*/);
int qmb200_metrics_close_dev(qmb200_handle* h, const int32_t* mask, const int32_t* end, const int32_t* episode, int32_t n_episodes, double* acc, double* out,
                             int32_t* status, void* cuda_stream);

/* ---- per-episode command timelines (DESIGN.md §4.14): each episode of each robot gets a new command timeline, drawn on the device right after its
 *      restart into the device gait schedule's timeline, which the gait step then consumes as it consumes a loaded one.
 *   ranges row[QMB200_TIMELINE]  0      t_first      slot 0's time on the robot's observation clock (s)
 *                                1      gap          time from slot j - 1 to slot j (s), lo >= 0
 *                                2      p_gait       probability that a slot inserts a gait; fixed (lo == hi), in [0, 1]
 *                                3      gait_set     bitmask of the templates a gait slot picks among; fixed, an integer in [0, 2^32), non-zero when p_gait > 0
 *                                4-7    w_none, w_cmd_vel, w_ee_cmd_vel, w_ee_goal   weights of the slot's target command; fixed, >= 0, positive sum
 *                                8-11   cmd_vel_x, cmd_vel_y, cmd_vel_z, cmd_yaw_rate   base frame
 *                                12-14  ee_vx, ee_vy, ee_vz   end-effector velocity, world frame
 *                                15-17  ee_x, ee_y, ee_z      goal position, world frame
 *                                18-21  ee_qx, ee_qy, ee_qz, ee_qw   goal orientation; fixed, unit norm within 1e-9
 *   drawn slot[QMB200_TIMELINE_CMD]  t, tmpl (-1 or a template id), cmd_vel[4] (the quiet NaN 0x7FF8000000000000 unless the kind is cmd_vel), ee_kind (-1,
 *                                QMB200_TARGET_EE_CMD_VEL or QMB200_TARGET_EE_GOAL), ee[7] (zeros; (v, 0, 0, 0, 0) for ee_cmd_vel; position and quaternion for a goal):
 *                                one command of qmb200_gait_dev_set_commands_ee.
 * Every draw of slot j is u = the keyed uniform of the episode draws on a domain constant of its own over (seed, global robot rank * B + b, e, 16 j + c); a box
 * column is fma(u, hi - lo, lo), a fixed column lo itself, byte for byte.  t_0 = draw(t_first) on channel 0, t_j = t_{j-1} + draw(gap) on channel 16 j;
 * c = 1: a gait is inserted when u < p_gait; c = 2: the template is the k-th set bit of gait_set in increasing bit order, k = min(floor(u popcount),
 * popcount - 1); c = 3: the kind is the first of (none, cmd_vel, ee_cmd_vel, ee_goal) whose running sum of weights exceeds u W, W their sum in that order
 * (else the last with a positive weight); c = 4-7 cmd_vel; c = 8-10 the end-effector velocity; c = 11-13 the goal position. */
#define QMB200_TIMELINE 22
#define QMB200_TIMELINE_CMD 14
/* Per-robot ranges lo, hi [B][QMB200_TIMELINE], n_cmd (>= 1) slots per episode and the seed.  NULL lo and hi clear them.  Rejects a non-finite bound,
 * lo > hi, a non-finite hi - lo and the column rules above, naming the field and the robot; on rejection the stored ranges stay unchanged.  Host arrays;
 * synchronous. */
int qmb200_timeline_set_ranges(qmb200_handle* h, int32_t n_cmd, const double* lo /*[B][QMB200_TIMELINE] or NULL*/, const double* hi /*[B][QMB200_TIMELINE] or NULL*/,
                               int64_t seed);
/* The stored n_cmd, ranges and seed (zeros when none are set); is_set = 1 when ranges are set.  Any output may be NULL. */
int qmb200_timeline_get_ranges(const qmb200_handle* h, int32_t* n_cmd, double* lo /*[B][QMB200_TIMELINE]*/, double* hi /*[B][QMB200_TIMELINE]*/, int64_t* seed,
                               int32_t* is_set);
/* One launch, no host work: every robot with mask[b] != 0 draws episode[b]'s n_cmd slots into rows[b] and into the device gait schedule's timeline that
 * qmb200_gait_dev_set_commands(_ee) loaded (its time, template, cmd_vel and, when it has them, end-effector rows), and its cursor goes back to 0.  Robots
 * with mask[b] == 0 are not written.  Fails, writing nothing, when no ranges are set, the device gait schedule is not running, the loaded timeline's width
 * differs from n_cmd, a robot weighs an end-effector kind and the timeline has no end-effector rows, or a gait_set bit lies at or above the template
 * table's size. */
int qmb200_timeline_sample(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* episode /*[B]*/, double* rows /*[B][n_cmd][QMB200_TIMELINE_CMD] in-out*/);
int qmb200_timeline_sample_dev(qmb200_handle* h, const int32_t* mask, const int32_t* episode, double* rows, void* cuda_stream);
/* Host only: the slots [n][n_cmd][QMB200_TIMELINE_CMD] of robots robot[n] (in [0, B)) in episodes episode[n] on the stored ranges and seed, what the
 * sampler draws. */
int qmb200_timeline_draw(const qmb200_handle* h, int32_t n, const int32_t* robot /*[n]*/, const int32_t* episode /*[n]*/, double* rows /*[n][n_cmd][QMB200_TIMELINE_CMD]*/);

/* ---- per-episode end-effector paths (DESIGN.md §4.21): each episode of each robot gets a new end-effector path, drawn on the device right after its
 *      restart into a row of the path table that belongs to the robot, and a pending start of that row (qmb200_gait_dev_command's slot), so that the
 *      path starts on the episode's first MPC tick, after any timeline command due on that tick.
 *   ranges row[QMB200_EE_PATH_RANGES]  0      n_way        waypoint count; fixed (lo == hi), an integer in [1, QMB200_EE_PATH_MAX]
 *                                      1      tau_first    waypoint 0's time after the path starts (s), lo > 0
 *                                      2      gap          time from waypoint i - 1 to waypoint i (s), lo >= T/2 (T the MPC time horizon, as the table's);
 *                                                          tau_first hi + (n_way - 1) gap hi <= 1e300, so that every drawn time is finite
 *                                      3-5    x, y, z      waypoint position in the path's frame (the heading frame at the start for a heading-frame
 *                                                          robot, the world frame otherwise: a table path's frame)
 *                                      6      yaw          turn of the hand about that frame's z axis, bounds in [-pi, pi]
 *                                      7-10   qx, qy, qz, qw   the quaternion it turns; fixed, unit norm within 1e-9
 *   drawn waypoint i  (tau, x, y, z, quaternion xyzw): a row of the path table (qmb200_set_ee_paths' layout).  tau_0 = draw(tau_first), tau_i =
 *                     tau_{i-1} + draw(gap), rounded up where the nearest rounding would leave tau_i - tau_{i-1} under the gap; the position the box drawn per waypoint; the quaternion Rz(draw(yaw)) quat, its half-angle sine and cosine
 *                     from Taylor polynomials in single roundings, so that host and device agree bit for bit.
 * Every draw of waypoint i is u = the keyed uniform of the episode draws on a domain constant of its own over (seed, global robot rank * B + b, e, 8 i + c):
 * c = 0 the time, 1-3 the position, 4 the yaw.  A box column is fma(u, hi - lo, lo), a fixed column lo itself, byte for byte.  Every drawn row passes
 * qmb200_set_ee_paths' check.
 * While ranges are set the device path table holds the P paths of qmb200_set_ee_paths followed by B drawn rows: robot b's is row P + b, an ordinary table
 * index of qmb200_target_trajectories_path.  qmb200_get_ee_paths reports the P paths only, qmb200_set_ee_paths refuses, and commands
 * (qmb200_gait_dev_command, timelines) may still start the P paths only. */
#define QMB200_EE_PATH_RANGES 11
/* Per-robot ranges lo, hi [B][QMB200_EE_PATH_RANGES] and the seed; allocates the B drawn rows of the path table.  NULL lo and hi clear them (the table
 * is the P paths again).  Rejects a non-finite bound, lo > hi, a non-finite hi - lo and the column rules above, naming the field and the robot; on
 * rejection the stored ranges stay unchanged.  Refused while a curriculum is attached to them.  Host arrays; synchronous. */
int qmb200_ee_path_set_ranges(qmb200_handle* h, const double* lo /*[B][QMB200_EE_PATH_RANGES] or NULL*/, const double* hi /*[B][QMB200_EE_PATH_RANGES] or NULL*/,
                              int64_t seed);
/* The stored ranges and seed (zeros when none are set); is_set = 1 when ranges are set.  Any output may be NULL. */
int qmb200_ee_path_get_ranges(const qmb200_handle* h, double* lo /*[B][QMB200_EE_PATH_RANGES]*/, double* hi /*[B][QMB200_EE_PATH_RANGES]*/, int64_t* seed,
                              int32_t* is_set);
/* One launch, no host work: every robot with mask[b] != 0 draws episode[b]'s path into rows[b][0:n_way] and into table row P + b (the waypoints past
 * n_way are not written: no target call reads them), and sets its pending slot to the row qmb200_gait_dev_command writes for (tmpl -1, cmd_vel the quiet NaN, ee_kind QMB200_TARGET_EE_PATH, ee (P + b, 0, ..., 0)).
 * Robots with mask[b] == 0 are not written.  Fails, writing nothing, when no ranges are set or the device gait schedule is not running (its pending
 * slots exist exactly while it runs). */
int qmb200_ee_path_sample(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* episode /*[B]*/, double* rows /*[B][QMB200_EE_PATH_MAX][8] in-out*/);
int qmb200_ee_path_sample_dev(qmb200_handle* h, const int32_t* mask, const int32_t* episode, double* rows, void* cuda_stream);
/* Host only: the paths of robots robot[n] (in [0, B)) in episodes episode[n] on the stored ranges and seed, what the sampler draws: n_way [n] and way
 * [n][QMB200_EE_PATH_MAX][8] (zeros past n_way). */
int qmb200_ee_path_draw(const qmb200_handle* h, int32_t n, const int32_t* robot /*[n]*/, const int32_t* episode /*[n]*/, int32_t* n_way /*[n]*/,
                        double* way /*[n][QMB200_EE_PATH_MAX][8]*/);

/* ---- per-robot curricula (DESIGN.md §4.15): each robot has a level in [0, n_levels) that places the ranges of every attached draw kind (episode,
 *      spawn, timeline, ee path) on the line from an easy box (level 0, the kind's ranges when attached) to a hard box (level n_levels - 1).  When a robot's
 *      episode closes, a device update steps its level from the episode's end code and, optionally, its metrics row, and writes the box of the new level
 *      into the kinds' device ranges, which the unchanged samplers then draw the next episode from.
 *   box at level l, f = l / (n_levels - 1), per column of lo and of hi: base at l = 0, top at l = n_levels - 1, base where base == top, else
 *                                fma(f, top - base, base); the spawn's tile column then floor(x + 0.5).  The timeline's gait_set and ee_q* and the ee path's n_way and
 *                                q* must be equal at both ends.
 *   row[QMB200_CURRICULUM]        0 start_level (an integer in [0, n_levels)), 1 up_after, 2 down_after (integers >= 1), 3-6 threshold[4] (finite)
 *   state[QMB200_CURRICULUM_STATE]  int32: level, pass_run, fail_run, n_updates
 *   rule: n_levels >= 2 and n_cond <= QMB200_CURRICULUM_MAX_COND conditions; condition i compares the closed episode's metrics column column[i]
 *   (QMB200_METRICS) with the robot's threshold[i] by op[i] (QMB200_CURRICULUM_GE: >=, _LE: <=; false when either side is NaN).
 * An update with end 1 or 2 adds one to n_updates; the episode fails when end == 1 or a QMB200_CURRICULUM_FAIL condition holds, else passes when end == 2
 * and every QMB200_CURRICULUM_PASS condition holds, else is neutral.  A pass zeroes fail_run and adds one to pass_run; at up_after the level goes up by
 * one (at most n_levels - 1) and pass_run goes back to 0.  A fail does the same with fail_run, down_after and one level down (at least 0).  End 0 (the
 * run's end) updates nothing.  The start image (qmb200_robot_image_save) does not hold the state: a restore leaves it. */
#define QMB200_CURRICULUM 7
#define QMB200_CURRICULUM_STATE 4
#define QMB200_CURRICULUM_MAX_COND 4
#define QMB200_CURRICULUM_EPISODE 0    /* kinds: the ranges of qmb200_episode_set_ranges, qmb200_spawn_set_ranges, qmb200_timeline_set_ranges, */
#define QMB200_CURRICULUM_SPAWN 1      /* qmb200_ee_path_set_ranges */
#define QMB200_CURRICULUM_TIMELINE 2
#define QMB200_CURRICULUM_EE_PATH 3
#define QMB200_CURRICULUM_GE 0
#define QMB200_CURRICULUM_LE 1
#define QMB200_CURRICULUM_PASS 0
#define QMB200_CURRICULUM_FAIL 1
typedef struct qmb200_curriculum_rule {
  int32_t n_levels, n_cond;
  int32_t column[QMB200_CURRICULUM_MAX_COND], op[QMB200_CURRICULUM_MAX_COND], role[QMB200_CURRICULUM_MAX_COND];
} qmb200_curriculum_rule;
/* The rule and the rows [B][QMB200_CURRICULUM]; every robot's state starts at (start_level, 0, 0, 0).  Rejects an invalid rule or row, naming the field and
 * the robot, and refuses while a kind is attached.  NULL rule and rows clear the curriculum: each attached kind's ranges go back to its base box and
 * the kind is detached.  Host arrays; synchronous. */
int qmb200_curriculum_set(qmb200_handle* h, const qmb200_curriculum_rule* rule, const double* rows /*[B][QMB200_CURRICULUM] or NULL*/);
/* Attaches kind (QMB200_CURRICULUM_*): its ranges in force become level 0, lo_top / hi_top [B][width] level n_levels - 1.  Every level's box must pass the
 * kind's own range check (the spawn's against the tile library in force, the ee path's at the handle's T); the first failure is named with its level, field and robot, and nothing is
 * written.  Then each robot's box at its level is written into the kind's ranges.  While attached, the kind's *_set_ranges refuses.  Synchronous. */
int qmb200_curriculum_attach(qmb200_handle* h, int32_t kind, const double* lo_top /*[B][width]*/, const double* hi_top /*[B][width]*/);
/* One launch, no host work: every robot with mask[b] != 0 and end[b] in {1, 2} updates its state from end[b] and, when the rule has conditions, the closed
 * row rows[b][episode[b]] (rows [B][n_episodes][QMB200_METRICS], qmb200_metrics_close's out), writes its level to level[b] and the box at that level into
 * every attached kind's ranges.  When the rule has conditions and episode[b] lies outside [0, n_episodes), QMB200_ST_OVERFLOW is OR-ed into status[b]
 * and nothing else is written.  A masked end outside {1, 2} and unmasked robots are not written.  Fails, writing nothing, when no curriculum is set, no
 * kind is attached, the rule has conditions and rows is NULL, or n_episodes < 1. */
int qmb200_curriculum_update(qmb200_handle* h, const int32_t* mask /*[B]*/, const int32_t* end /*[B]*/, const int32_t* episode /*[B]*/,
                             const double* rows /*[B][n_episodes][QMB200_METRICS] or NULL*/, int32_t n_episodes, int32_t* level /*[B] in-out*/,
                             int32_t* status /*[B] in-out*/);
int qmb200_curriculum_update_dev(qmb200_handle* h, const int32_t* mask, const int32_t* end, const int32_t* episode, const double* rows, int32_t n_episodes,
                                 int32_t* level, int32_t* status, void* cuda_stream);
/* Synchronous: the state [B][QMB200_CURRICULUM_STATE] (zeros when none is set) after every queued update; is_set = 1 when a curriculum is set.  Any output
 * may be NULL. */
int qmb200_curriculum_get(const qmb200_handle* h, int32_t* state /*[B][QMB200_CURRICULUM_STATE]*/, int32_t* is_set);
/* Host only: the rows of attached kind that its sampler draws for robots robot[n] in episodes episode[n] at levels level[n] (in [0, n_levels)): the
 * kind's *_draw on the box at that level, [n][QMB200_EPISODE], [n][QMB200_SPAWN], [n][n_cmd][QMB200_TIMELINE_CMD] or, for the ee path,
 * [n][1 + QMB200_EE_PATH_MAX * 8]: n_way (as a double), then the waypoints (zeros past n_way). */
int qmb200_curriculum_draw(const qmb200_handle* h, int32_t kind, int32_t n, const int32_t* robot /*[n]*/, const int32_t* episode /*[n]*/,
                           const int32_t* level /*[n]*/, double* rows);

/* The whole QMController::update (QMController.cpp:128-175) on the stored policy: observation update → evaluatePolicy(t_obs) → WbcBase::update
 * (period, t_obs) → safety check + control law.  cmd = the WBC 54-vector, status = WBC status | QMB200_ST_SAFETY. */
int qmb200_update(qmb200_handle* h, const double* rbd /*[B][55]*/, const double* period /*[B]*/, double* t_obs /*[B] in-out*/, double* x_obs /*[B][30] in-out*/, double* joint_cmd /*[B][18][5] in-out*/,
                  double* arm_pos_cmd /*[B][6] in-out*/, double* last_time /*[B] in-out*/, double* cmd /*[B][54]*/, int32_t* status /*[B]*/);
int qmb200_update_dev(qmb200_handle* h, const double* rbd, const double* period, double* t_obs, double* x_obs, double* joint_cmd, double* arm_pos_cmd, double* last_time, double* cmd, int32_t* status, void* cuda_stream);

/* ---- tick pipeline: qmb200_tick / qmb200_tick_dev cut the batch into `chunks` (1..8) robot ranges and run each range's
 *      MPC solve → evaluatePolicy → WbcBase::update chain on its own CUDA stream (forked from / joined into the caller's stream), so
 *      kernels with different bottlenecks overlap on the SMs.  Robots are independent (the reference runs one controller per robot,
 *      QMController.cpp:128-148), so results do not depend on the setting.  Default: 1. */
int qmb200_set_pipeline(qmb200_handle* h, int chunks);

/* measurement support (bench.py): per-kernel device times of the tick [setup, lq, riccati, linesearch, policy_eval, wbc] in ms (mean per call),
 * and the measured fp64 FMA throughput of this GPU */
int qmb200_set_profiling(qmb200_handle* h, int on);
int qmb200_collect_kernel_times(qmb200_handle* h);
int qmb200_get_kernel_times(qmb200_handle* h, double* ms6);
/* the part of ms6[1] (LQ approximation) spent in the thread-per-node flow kernel (kinematics, flow maps, constraint rows); the rest is the warp-per-node projection kernel */
int qmb200_get_flow_kernel_time(qmb200_handle* h, double* ms);
int qmb200_measure_fp64_peak(qmb200_handle* h, double* tflops);

/* diagnostics: the QP step (dx, du) of the last solve and per-robot scalars [armijo, baseline cost, dyn SSE, eq SSE, |dx|, |du|, -, -] */
int qmb200_debug_get_step(qmb200_handle* h, double* dx /*[B][NMAX][30]*/, double* du /*[B][NMAX][30]*/, double* robot /*[B][8]*/);
/* ---- solver variants (SURVEY 8f-3).  QMInterface loads four solver blocks (QMInterface.cpp:69-73: ddp{}, sqp{}, ipm{}, rollout{}); QMController::setupMpc runs
 *      SqpMpc (QMController.cpp:287-288), the handle's default.  The other two blocks select, on the same OCP, LQ model (K2) and backward pass (K3):
 *      IPM  ocs2 IpmSolver with ipm{} (task.info:95-125).  The OCP of qm_interface has no inequality constraint terms (soft constraints + state-input
 *           equalities only, QMInterface.cpp:79-142), so the interior-point iteration carries no barrier / slack / dual variables and its primal step is the
 *           Newton step of the equality-constrained problem - the SQP step; what changes are the iteration count and the filter line-search thresholds
 *           (ipmIteration, deltaTol, g_max = 10, g_min).
 *      DDP  ocs2 GaussNewtonDDP with ddp{} (task.info:33-71) in its discrete-time form (ddp.algorithm ILQR; the file's SLQ integrates a continuous-time Riccati
 *           equation and ODE45 rollouts, which cannot be pinned without a reference run): nominal single-shooting rollout from the measured state, LQ
 *           approximation along it, the discrete Riccati backward pass, rollout line search of the affine controller on merit = cost + penalty * sqrt(ISE of
 *           the state-input equalities) over step lengths maxStepLength * 0.5^j >= minStepLength. */
#define QMB200_SOLVER_SQP 0
#define QMB200_SOLVER_IPM 1
#define QMB200_SOLVER_DDP 2
int qmb200_mpc_set_solver(qmb200_handle* h, int32_t solver);
int qmb200_mpc_get_solver(const qmb200_handle* h, int32_t* solver, int32_t* iterations, double* delta_tol, double* g_max, double* g_min);

/* ---- multi-GPU (SURVEY 8e): robots are independent, rank g owns a contiguous robot range, the only exchange per tick is ONE all-gather of the torque rows.
 *      NCCL is driven from this library (opened with dlopen at the first call: no link-time dependency).  Bootstrap: rank 0 calls qmb200_comm_get_unique_id and
 *      ships the 128 bytes to the other ranks by any means; every rank then calls qmb200_comm_init on its handle (collective, like ncclCommInitRank). */
#define QMB200_COMM_ID_BYTES 128
int qmb200_comm_get_unique_id(void* id128);
int qmb200_comm_init(qmb200_handle* h, int32_t nranks, int32_t rank, const void* id128);
int qmb200_comm_destroy(qmb200_handle* h);                                   /* also done by qmb200_destroy */
int qmb200_comm_info(const qmb200_handle* h, int32_t* nranks, int32_t* rank, int32_t* nccl_version);
/* torque_all[r * B + i][0:18] = torque rows (cmd[.][36:54]) of rank r's robot i, on every rank: one pack kernel + one ncclAllGather on `cuda_stream` (NULL: the
 * handle's stream).  nccl_comm: an ncclComm_t of the caller, or NULL for the handle's communicator (no communicator at all: single rank, plain copy).
 * perm (device, optional): the batch was submitted in gait-binned order, perm[p] = original local index of the robot at position p; the gathered buffer is in
 * ORIGINAL order.  All ranks must hold the same batch size. */
int qmb200_allgather_torque(qmb200_handle* h, void* nccl_comm, const double* cmd_local /*[B][54] device*/, const int32_t* perm /*[B] device or NULL*/,
                            double* torque_all /*[nranks * B][18] device*/, void* cuda_stream);
/* Host helper for mixed-gait batches (BASELINE configs[4]): permutation that sorts the robots by contact phase (stance code at t0, events in the window, time to the
 * next event); perm[p] = original index of the robot at position p. */
int qmb200_gait_bin_permutation(int32_t n, const double* t0, const int32_t* n_events, const double* event_times /*[n][EMAX]*/, const int32_t* modes /*[n][EMAX+1]*/, int32_t* perm /*[n]*/);

/* Host-only (no CUDA device needed): run the constructor chain's parsers (QMInterface::setupModel / setupOptimalControlProblem inputs: task.info, robot.urdf,
 * reference.info, optional gains file — batch / device of cfg are ignored) and copy the resulting model + settings constants (the block replicated to every GPU)
 * into out.  Returns the block size in bytes (also when out is NULL or capacity is too small: nothing is copied then), negative on a parse error
 * (qmb200_last_error(NULL)).  Used to check that two sets of input files define the same problem, bit for bit. */
int64_t qmb200_debug_model_blob(const qmb200_config* cfg, void* out, int64_t capacity);
/* Host-only, like qmb200_debug_model_blob: the SRBD constants [n][QMB200_SRBD] that qmb200_set_model_payload derives for n payload rows [n][8] (NULL: no
 * payload) on the model of cfg.  Returns 0, or negative on a parse error or a rejected payload (qmb200_last_error(NULL)). */
int qmb200_debug_srbd_constants(const qmb200_config* cfg, int32_t n, const double* payload /*[n][8] or NULL*/, double* out /*[n][QMB200_SRBD]*/);

/* number of kernels this library launched since create (bench.py's gpu_launches) */
int64_t qmb200_launch_count(const qmb200_handle* h);
/* stream the handle launches on (cudaStream_t as void*) */
void* qmb200_stream(const qmb200_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* QMB200_H */
