/* include/msckf_b200.h -- C-ABI of the H100 MSCKF measurement-update engine (libmsckf_b200.so).
 *
 * The reference (daniilidis-group/msckf_mono) has no plugin / FFI boundary: its filter is the header-only
 * C++ class template msckf_mono::MSCKF<_S> (include/msckf_mono/msckf.h:31-1512).  This C-ABI is what the
 * replacement class of the same name (include/msckf_mono/msckf.h in THIS repo) binds: each entry point below
 * names the reference member function(s) whose numerics it replaces.  All integer bookkeeping (track lists,
 * clone ids, pruning decisions) stays on the host in the class shim, exactly as in the reference.
 *
 * Conventions: plain pointers and sizes only.  `dtype` selects the scalar type of every `void*` array
 * (MSCKF_B200_F32: float, MSCKF_B200_F64: double) -- the reference's template parameter _S.  Quaternions are
 * (x,y,z,w) (Eigen coeffs() order).  Error-state order: IMU [dtheta, db_g, dv, db_a, dp] then per clone
 * [dtheta_C, dp_C] (msckf.h:885-889, :1376-1390).  Every function returns 0 on success, a negative
 * msckf_b200_status otherwise; there is NO CPU fallback -- a failed device call is a hard error.
 * A handle owns its device buffers and one CUDA stream; calls on one handle must be serialised by the
 * caller (like the reference class), different handles are independent.
 */
#ifndef MSCKF_B200_H_
#define MSCKF_B200_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

enum msckf_b200_dtype { MSCKF_B200_F32 = 0, MSCKF_B200_F64 = 1 };
enum msckf_b200_status {
  MSCKF_B200_OK = 0,
  MSCKF_B200_ERR_CUDA = -1,      /* a CUDA runtime call or kernel failed */
  MSCKF_B200_ERR_CAPACITY = -2,  /* more clones / tracks / observations than msckf_b200_create reserved */
  MSCKF_B200_ERR_ARG = -3,       /* invalid argument (e.g. track longer than 98 observations, msckf.h:91) */
  MSCKF_B200_ERR_NO_DEVICE = -4, /* no CUDA device: the engine never computes on the CPU */
  MSCKF_B200_ERR_STATE = -5,     /* call order violated */
  MSCKF_B200_ERR_NUMERIC = -6    /* the update produced a non-finite delta-x or covariance entry.  The update HAS been applied, like in
                                    the reference (whose only anomaly handling is a print, msckf.h:1405-1409): returned by _fetch
                                    after the report was filled, so the caller decides (the class shim prints and carries on) */
};
enum msckf_b200_mode {
  MSCKF_B200_MARGINALIZE = 0, /* MSCKF::marginalize() msckf.h:336-449: loop A + loop B + measurementUpdate */
  MSCKF_B200_TRIANGULATE = 1, /* checkMotion :980-1025 + initializePosition :1147-1285 only (pruneRedundantStates :488-531) */
  MSCKF_B200_RESIDUALIZE = 2  /* loop B + measurementUpdate at caller-given p_f_G (pruneRedundantStates :545-614) */
};

typedef struct msckf_b200_engine msckf_b200_engine;

typedef struct {
  int dtype;       /* msckf_b200_dtype */
  int device;      /* CUDA device ordinal */
  int max_clones;  /* initial capacity M_max (covariance is (15+6*M_max)^2) */
  int max_tracks;  /* initial capacity of one track batch */
  int max_obs;     /* initial capacity of one batch's total observation count */
} msckf_b200_config;
/* The three capacities are INITIAL sizes: like the reference, whose window and track lists are unbounded std::vectors, the
 * engine grows its device buffers on demand (x2, contents preserved).  Hard limits that remain: 98 observations per track
 * (the reference's chi-square table has 99 entries, msckf.h:91 -- longer tracks index past it there) and the window the
 * tail kernel's shared-memory panels can hold (136 clones; an update of a larger window fails at staging and writes nothing):
 * they fail with MSCKF_B200_ERR_ARG / _CAPACITY.  A track names each clone at most once (MSCKF sees a feature once per
 * image); a track that names one clone twice fails with MSCKF_B200_ERR_ARG.  Such failures come before anything is launched:
 * nothing is written, and in a device batch no member is. */

/* One batch of feature tracks, flat SoA (types.h:102-113 featureTrackToResidualize without the clone copies:
 * the clone poses are device resident and addressed by POSITION in the sliding window, msckf.h:1481). */
typedef struct {
  int n_tracks;
  const int* obs_offset;  /* [n_tracks+1] prefix offsets into obs / clone_index */
  const void* obs;        /* [2*obs_offset[n_tracks]] normalised image coordinates (u,v), dtype scalars */
  const int* clone_index; /* [obs_offset[n_tracks]] positional index of the observing clone, each at most once per track, in
                             any order */
  const void* p_f_G;      /* MSCKF_B200_RESIDUALIZE only: [3*n_tracks] feature positions; else NULL */
} msckf_b200_tracks;

/* Per-track results; every pointer may be NULL (not wanted).  Caller-owned host buffers of n_tracks entries. */
typedef struct {
  int* cm_ok;    /* checkMotion result */
  int* tri_ok;   /* initializePosition validity */
  int* valid;    /* valid_tracks[] of msckf.h:348 */
  int* accepted; /* passed gatingTest */
  void* gamma;   /* Mahalanobis distance, dtype scalars */
  void* p_f_G;   /* [3*n_tracks] triangulated position, dtype scalars */
  int m;         /* out: stacked rows of accepted tracks (stack_counter, msckf.h:443) */
  int rank;      /* out: independent rows kept by the compression */
} msckf_b200_report;
/* (a non-finite result is signalled by _fetch returning MSCKF_B200_ERR_NUMERIC, with the report filled) */

int msckf_b200_create(const msckf_b200_config* cfg, msckf_b200_engine** out);
int msckf_b200_destroy(msckf_b200_engine* e);

/* MSCKF::initialize msckf.h:72-97.
 * camera: q_CI[4], p_C_I[3]; noise: u_var_prime, v_var_prime, Q_imu[144], initial_imu_covar[225] (row-major);
 * params: max_gn_cost_norm, translation_threshold; imu_state: p_I_G[3], v_I_G[3], b_g[3], b_a[3], g[3], q_IG[4]. */
int msckf_b200_initialize(msckf_b200_engine* e, const void* camera, const void* noise, const void* params, const void* imu_state);
/* MSCKF::propagate msckf.h:101-145.  reading: omega[3], a[3], dT */
int msckf_b200_propagate(msckf_b200_engine* e, const void* reading);
/* k consecutive propagate() calls (readings: [k][7] scalars) in one kernel launch per 16 readings; same arithmetic, reading
 * by reading.  The class shim queues the IMU readings that arrive between two images (src/ros_interface.cpp:92-97) */
int msckf_b200_propagate_n(msckf_b200_engine* e, const void* readings, int k);
/* MSCKF::augmentState msckf.h:148-212 (numeric part: clone pose + covariance augmentation) */
int msckf_b200_augment(msckf_b200_engine* e);
/* marginalize / pruneRedundantStates numerics, asynchronous on the handle's stream.  The input arrays are
 * copied to pinned staging before return; results are fetched (and the stream synchronised) by _fetch.
 * A track with a single observation cannot be triangulated or projected (2L - 3 < 1 rows): it is reported as rejected
 * (cm_ok = tri_ok = valid = accepted = 0), not as an error. */
int msckf_b200_update_async(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks);
int msckf_b200_fetch(msckf_b200_engine* e, msckf_b200_report* report);
/* Zero-copy packing: host pointers INTO the engine's pinned input block for a batch of n_tracks tracks / n_obs observations
 * (out->obs_offset, ->obs, ->clone_index, ->p_f_G; out->n_tracks = n_tracks).  The caller fills them and passes the same struct
 * to _update / _update_async / _stage, which then skips its own copy.  Valid until the next call on this handle. */
int msckf_b200_input_buffer(msckf_b200_engine* e, int n_tracks, int n_obs, msckf_b200_tracks* out);
/* update_async split in two: _stage validates and copies the batch into HBM, _launch enqueues the kernels
 * (bench.py times _launch alone: "inputs already resident in HBM") */
int msckf_b200_stage(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks);
int msckf_b200_launch(msckf_b200_engine* e);
/* _launch bracketed by CUDA events on the handle's stream (kernels only); *ms = device time */
int msckf_b200_launch_timed(msckf_b200_engine* e, float* ms);
/* with option key 1 set, per-kernel device times of the last launch (launch order); returns the count */
int msckf_b200_kernel_times(msckf_b200_engine* e, float* ms, const char** names, int cap);
/* with option key 1 set, %globaltimer stamps (ns) taken by the tail kernel at its phase boundaries; 0-terminated */
int msckf_b200_tail_profile(msckf_b200_engine* e, unsigned long long* out, int cap);
/* update_async + fetch */
int msckf_b200_update(msckf_b200_engine* e, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* report);
/* ---- device-side batches of independent filters (SURVEY.md 8e: sequences / Monte-Carlo trials sharing one GPU) ----------
 * A batch groups n engines (same dtype, same device).  One update of the whole group is ONE launch per kernel -- the filter
 * index rides in blockIdx.z, one thread-block cluster per filter runs the serial tail -- replayed as ONE CUDA graph, with ONE
 * packed host->device copy of all track batches and ONE packed device->host copy of all reports.  Results are bit-identical
 * to n separate msckf_b200_update calls.  While a batch exists its engines share the batch's stream (their other calls --
 * propagate, augment, prune, getters -- stay valid and are ordered with the batch's updates); destroying the batch gives
 * every engine its own stream back.  An engine belongs to at most one batch. */
typedef struct msckf_b200_batch msckf_b200_batch;
int msckf_b200_batch_create(msckf_b200_engine** engines, int n, msckf_b200_batch** out);
int msckf_b200_batch_destroy(msckf_b200_batch* b);
/* tracks[n] / reports[n]: one per engine, in the order given to _create; reports may be NULL.  Up to `threads` host threads
 * share the validation and packing of the n track batches (<= 1: the calling thread does all of it); the engine uses fewer
 * for small batches -- one per 8 MB of observations: packing from several cores makes the following host-to-device copy slower
 * than the packing gets faster (measured with scripts/e2e_breakdown.py). */
int msckf_b200_batch_update_async(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, int threads);
int msckf_b200_batch_fetch(msckf_b200_batch* b, msckf_b200_report* reports);
int msckf_b200_batch_update(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* reports, int threads);
/* the same split as _stage / _launch / _launch_timed of a single engine (bench.py: inputs resident in HBM) */
int msckf_b200_batch_stage(msckf_b200_batch* b, int mode, const msckf_b200_tracks* tracks, int threads);
int msckf_b200_batch_launch(msckf_b200_batch* b);
int msckf_b200_batch_launch_timed(msckf_b200_batch* b, float* ms);
/* per-kernel device times of the last batch launch (option key 1 of the FIRST engine set); returns the count */
int msckf_b200_batch_kernel_times(msckf_b200_batch* b, float* ms, const char** names, int cap);
long long msckf_b200_batch_launch_count(const msckf_b200_batch* b);
/* CTAs of the feature kernel (k_jac) resident per SM at the shape of the batch's last launch: the CUDA occupancy calculator's
 * figure for its threads per track and dynamic shared memory (0 before the first launch) */
int msckf_b200_batch_jac_occupancy(const msckf_b200_batch* b);
/* threads per track k_jac ran with at the last update launch of the engine's context (its batch while it belongs to one):
 * option 6's request, widened while a group of the launch's longest track does not fit in shared memory; 0 before any launch */
int msckf_b200_jac_group(msckf_b200_engine* e);
void* msckf_b200_batch_stream(msckf_b200_batch* b);
/* The other device calls of a frame for every member at once (the per-image sequence of datasets/asl_msckf.cpp:233-294 on a
 * batch).  Arrays have one entry per engine, in the order given to _create.  Each call validates every member before it
 * launches anything: a bad argument returns MSCKF_B200_ERR_ARG and a member with an un-fetched update MSCKF_B200_ERR_STATE,
 * and then no member has changed.  Every member computes exactly what its single-engine call computes, bit for bit.
 * Up to 32 members share one launch per kernel; past 32 the members run in consecutive launches of 32.
 * _propagate_n, _augment and _prune are asynchronous like their single-engine forms (arguments travel by value, nothing is
 * synchronised except where _augment grows a member's clone capacity). */
/* msckf_b200_propagate_n for every member (MSCKF::propagate msckf.h:101-145, applied reading by reading):
 * readings[i] = [k[i]][7] scalars; k[i] may be 0 (readings[i] may then be NULL); k = NULL: no member has readings.
 * Launches: for each step of 16 readings, one per 32 members that still have readings in that step
 * (members with at most 16 readings each, at most 32 members: one launch). */
int msckf_b200_batch_propagate_n(msckf_b200_batch* b, const void* const* readings, const int* k);
/* msckf_b200_augment (MSCKF::augmentState msckf.h:148-212) for the members with which[i] != 0 (which = NULL: all) */
int msckf_b200_batch_augment(msckf_b200_batch* b, const int* which);
/* msckf_b200_prune per member (pruneEmptyStates msckf.h:685-761, pruneRedundantStates :616-681): keep[i][0 .. n_keep[i]-1]
 * ascending positions; n_keep[i] < 0 or equal to the member's window: that member is left untouched */
int msckf_b200_batch_prune(msckf_b200_batch* b, const int* const* keep, const int* n_keep);
/* msckf_b200_get_state for every member (imu = NULL, imu[i] = NULL, clone_poses = NULL or clone_poses[i] = NULL: not wanted),
 * with one stream synchronisation for the whole batch */
int msckf_b200_batch_get_state(msckf_b200_batch* b, void* const* imu, void* const* clone_poses);
/* ---- consistency against ground truth (simulation, Monte-Carlo trials) ----------------------------------------------------
 * NEES = e^T P^-1 e of the filter's estimate against a caller-given truth, computed where P lives: one kernel launch (one CTA
 * per filter), one host-to-device copy of the truth, one device-to-host copy of the results, one synchronisation.  Read-only:
 * P, the state, the clone poses, captured graphs and launch counts are untouched.
 * The error state is computed in fp64 for both dtypes, as the exact inverse of the state injection q+ = buildUpdateQuat(dtheta)
 * * q (msckf.h:851-872, :1376-1390): dq = q_true * q_est^-1 (Hamilton product, true inverse conj(q)/|q|^2, dq negated when
 * dq.w < 0), dtheta = -2 vec(dq); every other component is truth - estimate.  In the order [dtheta_I, dp_I, dv, db_g, db_a,
 * clones (dtheta_C, dp_C)...] one fp64 Cholesky factor of P and one forward solve y = L^-1 e give every leading block's NEES
 * as a prefix sum of y^2: orientation (3 dof), IMU pose (6), IMU state (15), whole state (15 + 6M); the position (3) has its
 * own 3 x 3 solve.  If the factorisation meets a pivot <= 0 (P not positive definite), first_bad_pivot is its index in that
 * order and every NEES whose block contains it is NaN; the call still succeeds. */
typedef struct {
  double orientation, position, pose, imu, full;
  int dim_full;        /* 15 + 6M, or 0 without truth poses (full = NaN) */
  int first_bad_pivot; /* -1: positive definite */
} msckf_b200_nees_result;
/* truth_imu: 19 doubles in the layout of msckf_b200_initialize's imu_state (g ignored); truth_poses: [M*7] doubles,
 * p_C_G(3) q_CG(4) in window order (the layout of get_state's clone_poses), or NULL (full = NaN, dim_full = 0).
 * A NULL or non-finite argument or a zero quaternion returns MSCKF_B200_ERR_ARG, an un-fetched update MSCKF_B200_ERR_STATE;
 * then nothing is written. */
int msckf_b200_nees(msckf_b200_engine* e, const double* truth_imu, const double* truth_poses, msckf_b200_nees_result* out);
/* the same for every member of a batch (truth_imu[i], truth_poses = NULL or truth_poses[i] = NULL, out[i]); every member is
 * validated before anything is launched.  One launch per 32 members. */
int msckf_b200_batch_nees(msckf_b200_batch* b, const double* const* truth_imu, const double* const* truth_poses, msckf_b200_nees_result* out);
/* ---- aided measurements (position / pose fixes, zero-velocity updates, caller-linearised constraints) ----------------------
 * One EKF update with residual r (m rows), Jacobian H (m x n, n = 15 + 6M, in the error-state order above) and noise R, fused
 * where P lives: S = H P H^T + R = L L^T, W = L^-1 H P, y = L^-1 r, NIS = y^T y, dx = W^T y, P <- P - W^T W (computed in fp64,
 * rounded to the filter's scalar type once, both halves written: exactly symmetric), then the state injection of the vision
 * update (q_IG <- buildUpdateQuat(dtheta) * q_IG, not renormalised; clone quaternions renormalised; b_g, v, b_a, p additive;
 * the observability copies *_null untouched).  All arithmetic is fp64 for both dtypes.
 * Models (z in doubles; the first four compute r from the resident state, and their H selects state indices):
 *   VELOCITY   z = v_I_G (3) -- zeros: a zero-velocity update        r = z - v          indices 6..8
 *   POSITION   z = p_I_G (3)                                           r = z - p          indices 12..14
 *   POSE       z = p_I_G (3), q_IG xyzw (4)                            r = [dtheta; z_p - p], dtheta of q_z against q_IG in the
 *                                                                      convention of msckf_b200_nees   indices 0..2, 12..14
 *   CLONE_POSE z = p_C_G (3), q_CG xyzw (4) of clone `clone` (window order, get_state's layout)   indices 15+6k .. 20+6k
 *   LINEAR     z = r (m), H = m x n row-major (1 <= m <= 32, n must be the filter's current 15 + 6M)
 * R is m x m row-major; only its lower triangle is read.  For the first four models m and n may be 0 or the model's own values
 * (3, 3, 6, 6 rows).  chi2_max > 0: an update with NIS > chi2_max is not applied (applied = 0; the call succeeds).
 * One launch (one CTA per filter), one host-to-device copy of the inputs, one device-to-host copy of the results, one
 * synchronisation.  P is updated in place: captured update graphs stay valid.  The vision update's bookkeeping (its counters,
 * msckf_b200_last_delta_x, rank pivots) and the launch count are not changed. */
enum msckf_b200_aid_model {
  MSCKF_B200_AID_VELOCITY = 0,
  MSCKF_B200_AID_POSITION = 1,
  MSCKF_B200_AID_POSE = 2,
  MSCKF_B200_AID_CLONE_POSE = 3,
  MSCKF_B200_AID_LINEAR = 4,
  MSCKF_B200_AID_BODY_VELOCITY = 5, /* stacks only (msckf_b200_aid_stack_update) */
  MSCKF_B200_AID_RELATIVE_POSE = 6, /* stacks only */
  MSCKF_B200_AID_ANTENNA_POSITION = 7,       /* stacks only: GNSS */
  MSCKF_B200_AID_CLONE_ANTENNA_POSITION = 8, /* stacks only */
  MSCKF_B200_AID_HEADING = 9,                /* stacks only */
  MSCKF_B200_AID_CLONE_HEADING = 10,         /* stacks only */
  MSCKF_B200_AID_RANGE = 11,                 /* stacks only: radio ranging to a surveyed anchor */
  MSCKF_B200_AID_CLONE_RANGE = 12,           /* stacks only */
  MSCKF_B200_AID_PLANE_RANGE = 13,           /* stacks only: a rangefinder over a level plane */
  MSCKF_B200_AID_CLONE_PLANE_RANGE = 14,     /* stacks only */
  MSCKF_B200_AID_GYRO_AT_REST = 15,          /* stacks only: the mean gyro reading of a standstill */
  MSCKF_B200_AID_ACCEL_AT_REST = 16          /* stacks only: the mean specific force of a standstill */
};
typedef struct {
  int model;          /* msckf_b200_aid_model; in a batch, < 0 leaves that member untouched */
  int clone;          /* CLONE_POSE: the clone's position in the window */
  int m, n;           /* rows and state dimension (LINEAR; 0 or the model's own for the others) */
  const double* z;    /* the measurement (LINEAR: the residual r) */
  const double* H;    /* LINEAR: [m][n]; else ignored */
  const double* R;    /* [m][m], lower triangle read */
  double chi2_max;    /* > 0: NIS gate */
} msckf_b200_aid;
typedef struct {
  double nis;         /* r^T S^-1 r (NaN when S is not positive definite) */
  double dx_norm;     /* |dx| of the applied update (0 when not applied) */
  int dof;            /* m */
  int applied;        /* 1: P and the state were updated */
  int status;         /* 0: applied or gated out (see applied); 1: S not positive definite, nothing written; 2 (stacks
                         only): a HEADING / CLONE_HEADING axis within ~1e-3 rad of vertical (yaw undefined), a RANGE /
                         CLONE_RANGE antenna within 1e-6 m of its anchor, or a PLANE_RANGE / CLONE_PLANE_RANGE beam within
                         ~1e-3 rad of the plane or with the plane behind it; nothing written */
} msckf_b200_aid_result;
/* A bad model, an out-of-window clone, an m / n mismatch, a NULL or non-finite z / H / R or a zero quaternion returns
 * MSCKF_B200_ERR_ARG, an un-fetched update MSCKF_B200_ERR_STATE; then nothing is written.  A non-finite dx or P entry returns
 * MSCKF_B200_ERR_NUMERIC with the result filled: the update has been applied, as _fetch does for the vision update. */
int msckf_b200_aid_update(msckf_b200_engine* e, const msckf_b200_aid* aid, msckf_b200_aid_result* out);
/* the same for every member of a batch (aid[i], out[i]; out[i] is not written for a member with aid[i].model < 0); every
 * member is validated before anything is launched.  One launch per 32 updated members. */
int msckf_b200_batch_aid_update(msckf_b200_batch* b, const msckf_b200_aid* aid, msckf_b200_aid_result* out);
/* ---- stacked aided updates: odometry (wheel speed, non-holonomic constraints, relative motion) with other aids --------------
 * One EKF update of up to 8 items whose rows are stacked (sum of rows m <= 32) with R block-diagonal across items: the update,
 * outcomes and costs of msckf_b200_aid_update, with one NIS and one dof = m for the whole stack and one chi2_max gate.  Every
 * item forms its residual and its Jacobian on the device from the resident state, in fp64 for both dtypes; each row of H has at
 * most 12 non-zeros.  Allowed models: VELOCITY, POSITION, POSE, CLONE_POSE (a = the clone) as in msckf_b200_aid, and
 *   BODY_VELOCITY  z = v_I (3), the IMU velocity in the IMU frame; v^ = C(q_IG) v_I_G, r = z - v^ over the rows selected by the
 *                  mask a (bits 0..2; 0b110 with z = 0: the non-holonomic constraint v_y = v_z = 0; 0b111: full wheel velocity).
 *                  H is non-zero over dtheta (0..2) and dv (6..8) only.
 *   RELATIVE_POSE  clones a != b (window positions): z = p (3), q xyzw (4) of b relative to a in camera frames; predicted
 *                  C^ = C_b C_a^T (q^ = q_b * q_a^-1) and p^ = C_a (p_C_G,b - p_C_G,a); r = [dtheta(q_z, q^); z_p - p^] with the
 *                  dtheta of POSE.  H is non-zero over the two clones' [dtheta, dp].  (Odometry between the IMU state and a
 *                  clone is not a model: convert it to camera frames with q_CI and p_C_I.)
 * GNSS and heading models (satellite navigation, a second antenna, a magnetometer or a compass), with C = C(q_IG) and p = p_I_G,
 * or C = C(q_CG) and p = p_C_G of clone k for the CLONE_ forms -- a fix whose epoch lies behind the IMU's time is fused exactly at
 * the clone of that epoch's image:
 *   ANTENNA_POSITION        a = row mask (1..7), z = p_A_G (3), lever arm l (3) in the IMU frame; p^ = p + C^T l and
 *                           r = z - p^ over the rows of the mask (0b100 with l = 0: an altitude; 0b011: a horizontal fix).
 *                           H is non-zero over dtheta (-C^T [l]x) and dp (12..14).
 *   CLONE_ANTENNA_POSITION  a = clone k, b = row mask; z as above with l in that clone's camera frame; H over its [dtheta, dp].
 *   HEADING                 z = psi (1), axis f (3) in the IMU frame: d = C^T f, psi^ = atan2(d_y, d_x) (yaw of f in G),
 *                           r = z - psi^ wrapped into (-pi, pi]; one row over dtheta.  When d_x^2 + d_y^2 <= 1e-6 |f|^2 (f within
 *                           ~1e-3 rad of vertical) yaw is undefined: the stack writes nothing and reports status 2, NIS NaN.
 *   CLONE_HEADING           a = clone k; z as HEADING with f in that clone's camera frame; one row over its dtheta.
 * Range models (UWB or other radio ranging to surveyed anchors; a laser or sonar rangefinder over the ground or a ceiling), with
 * the same C, p and clone forms; one row each:
 *   RANGE                   z = rho (1), anchor a_G (3), lever arm l (3) in the IMU frame: e = p + C^T l - a_G, rho^ = |e|,
 *                           r = rho - rho^; H over dtheta and dp (12..14).  When rho^ <= 1e-6 m the direction is undefined:
 *                           status 2, NIS NaN, nothing written.
 *   CLONE_RANGE             a = clone k; z as RANGE with l in that clone's camera frame; H over its [dtheta, dp].
 *   PLANE_RANGE             z = rho (1), plane height h (1), lever l (3), beam axis f (3, any non-zero length) in the IMU frame;
 *                           the plane {x : x_z = h} is level in G.  b = C^T f / |f|, rho^ = (h - (p + C^T l)_z) / b_z,
 *                           r = rho - rho^; H over dtheta and dp_z (14).  When b_z^2 <= 1e-6 (the beam within ~1e-3 rad of
 *                           parallel to the plane) or rho^ <= 0 (the plane behind the sensor): status 2, NIS NaN, nothing written.
 *   CLONE_PLANE_RANGE       a = clone k; z as PLANE_RANGE with l and f in that clone's camera frame; H over its [dtheta, dp_z].
 * At-rest models (the IMU readings of a standstill; msckf_b200_standstill_update below forms them), with C = C(q_IG); 3 rows
 * each, a = b = 0:
 *   GYRO_AT_REST            z = the mean gyro reading (3): r = z - b_g; H over db_g (3..5) the identity.
 *   ACCEL_AT_REST           z = the mean specific force (3): h = b_a - C g with the filter's g, r = z - h; H over dtheta -[C g]x
 *                           and over db_a (9..11) the identity.  It observes roll, pitch and b_a, never yaw (H_theta C g = 0).
 *                           Both ignore Earth rotation.
 *   A degenerate item ends its member's whole stack (in a batch the other members are applied).  An anchor's position is taken
 *   as exact, and a range as unbiased; a caller with more than 8 anchors in one epoch makes two calls.
 *   A and b that a model does not use must be 0.  (A lever arm or an axis given in the IMU frame, l_I or f_I, is converted to
 *   camera frames with the engine's q_CI and p_C_I (the camera's position in the IMU frame: p_C_G = p_I_G + C(q_IG)^T p_C_I,
 *   C(q_CG) = C(q_CI) C(q_IG)): l_C = C(q_CI) (l_I - p_C_I), f_C = C(q_CI) f_I.)
 * C(q) is Eigen's toRotationMatrix (C(q_CG) maps G to the camera frame).  LINEAR is not allowed in a stack.  R of an item is its
 * own rows x rows block (3, 3, 6, 6, popcount(mask), 6, popcount(mask), popcount(mask), 1, 1, 1, 1, 1, 1, 3, 3 rows), row-major, lower triangle
 * read; the struct carries no size, so a caller that passes another size is not caught here (the class forms check it). */
typedef struct {
  int model;          /* msckf_b200_aid_model except LINEAR */
  int a;              /* CLONE_POSE, RELATIVE_POSE, CLONE_ANTENNA_POSITION, CLONE_HEADING, CLONE_RANGE, CLONE_PLANE_RANGE: clone
                         position; BODY_VELOCITY, ANTENNA_POSITION: row mask (1..7); else ignored (0 for the GNSS, heading,
                         range and at-rest models) */
  int b;              /* RELATIVE_POSE: the second clone; CLONE_ANTENNA_POSITION: row mask (1..7); else ignored (0 for the
                         GNSS, heading, range and at-rest models) */
  const double* z;    /* 3 (VELOCITY, POSITION, BODY_VELOCITY: all three components; GYRO_AT_REST, ACCEL_AT_REST), 7, 6
                         (antenna), 4 (heading), 7 (range) or 8 (plane range) doubles */
  const double* R;    /* [rows][rows] */
} msckf_b200_aid_item;
/* A bad model, a clone outside the window, a == b, an empty mask, more than 8 items or 32 rows, a NULL or non-finite z / R, a zero
 * quaternion, a zero heading or beam axis, a non-zero unused a / b of a GNSS, heading or range model or a NaN chi2_max returns
 * MSCKF_B200_ERR_ARG, an un-fetched update MSCKF_B200_ERR_STATE; then nothing is written.
 * A non-finite dx or P entry returns MSCKF_B200_ERR_NUMERIC with the result filled and the update applied.  n_items >= 1. */
int msckf_b200_aid_stack_update(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                msckf_b200_aid_result* out);
/* the same for every member of a batch (items[i] [n_items[i]], out[i]; n_items[i] = 0 leaves member i untouched and out[i] not
 * written); every member is validated before anything is launched.  One launch per 32 updated members. */
int msckf_b200_batch_aid_stack_update(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                      double chi2_max, msckf_b200_aid_result* out);
/* ---- fault detection and exclusion (FDE) over a stack's items --------------------------------------------------------------
 * The stacked update with one faulty item (an NLOS range, a GNSS multipath jump, a rangefinder on a table) removed on the device
 * instead of the whole epoch.  A starts as the items that can be linearised; a degenerate item (what ends a plain stack with
 * status 2) is dropped: its state is 2 and it does not count toward max_exclude.  Then, in rounds over the d_A rows of A
 * (S_AA is the principal submatrix of S = H P H^T + R: R is block-diagonal across items):
 *   1. NIS_A = r_A^T S_AA^-1 r_A <= chi2[d_A - 1]: the update is applied with the rows of A; stop.
 *   2. max_exclude items already excluded: rejected (outcome 2).  |A| = 1: rejected (outcome 3).
 *   3. for each j in A, t_j = NIS_A - NIS_{A\j} = y_j^T B_j^-1 y_j with y = S_AA^-1 r_A and B_j = (S_AA^-1)_jj (the block
 *      w-test: chi-square with d_j dof when j is not faulty).
 *   4. j* maximises t_j / chi2[d_j - 1], the lowest item index on a tie; a ratio <= 1 rejects the stack (outcome 3: no single
 *      item explains the failure), else j* leaves A and the next round starts at 1.
 * An applied update is msckf_b200_aid_stack_update on the items of A alone, in their order, without a gate, bit for bit (P,
 * state, NIS, dx_norm); max_exclude = 0 is msckf_b200_aid_stack_update with chi2_max = chi2[m - 1].  S_AA not positive
 * definite in any round: stack.status 1 (outcome -1), nothing written.  No item left: stack.status 2 (outcome -1, dof 0), nothing
 * written.  A rejection writes nothing.  The thresholds come from the caller, e.g. the chi-square quantile 1 - alpha of d dof. */
typedef struct {
  double chi2[32];   /* chi2[d-1], d = 1..32: gate on the NIS of a set of d rows and on an item's t_j of d rows; finite, > 0 */
  int max_exclude;   /* 0 .. 7 */
} msckf_b200_aid_fde;
typedef struct {
  double nis;        /* r_j^T S_jj^-1 r_j: the item alone against the prior P (NaN: degenerate) */
  double test;       /* t_j of the last round the item took part in (NaN: no exclusion round ran) */
  int state;         /* 0 used, 1 excluded, 2 degenerate (dropped), 3 not applied (stack rejected) */
  int round;         /* 0-based round in which it was excluded, else -1 */
} msckf_b200_aid_item_result;
typedef struct {
  msckf_b200_aid_result stack;  /* nis / dof of the last set gated, dx_norm, applied, status 0 / 1 / 2 as above */
  int outcome;                  /* 0 passed, 1 passed after exclusions, 2 rejected at max_exclude, 3 rejected: not identifiable;
                                   -1 with status 1 or 2 */
  int n_excluded;
  msckf_b200_aid_item_result item[8];  /* item[k] for k < n_items; the others have state -1 */
} msckf_b200_aid_fde_result;
/* Refusals (MSCKF_B200_ERR_ARG, nothing written): everything msckf_b200_aid_stack_update refuses, fde NULL, a chi2 entry that
 * is not finite or not > 0, max_exclude outside 0..7; an un-fetched update returns MSCKF_B200_ERR_STATE.  A non-finite dx or P
 * entry returns MSCKF_B200_ERR_NUMERIC with the update applied.  One launch, one copy each way, one synchronisation. */
int msckf_b200_aid_stack_update_fde(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items,
                                    const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out);
/* the same for every member of a batch with one fde (n_items[i] = 0 leaves member i untouched and out[i] not written); every
 * member is validated before anything is launched.  One launch per 32 updated members. */
int msckf_b200_batch_aid_stack_update_fde(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                          const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out);
/* ---- iterated stacked updates (an iterated EKF for the first range or GNSS epoch after drift) ------------------------------
 * One linearisation at the prior leaves a far-off filter overconfident: a range's curvature is of order delta^2 / (2 rho), and
 * the attitude terms of lever arms, BODY_VELOCITY, RELATIVE_POSE, POSE, HEADING and PLANE_RANGE are nonlinear too.  With
 * delta_0 = 0 and the iterate x_i = x^ [+] delta_i (fp64, the injection above on q_IG, v_I_G, p_I_G and on the poses of the clones
 * the items name: q_IG <- buildUpdateQuat(dtheta) * q_IG not renormalised, clone q <- normalise(buildUpdateQuat(dtheta_k) * q),
 * v and p additive), linearisation i forms r_i, H_i of the stack's items at x_i and factors S against the prior P with the
 * residual r_i + H_i delta_i; delta_{i+1} = W^T y = K_i (r_i + H_i delta_i).  It stops when max |delta_{i+1} - delta_i| <= tol
 * (converged; NaN counts as infinite) or after max_iter linearisations; then P <- P - W^T W and one injection of W^T y, both of
 * the last linearisation.  The Jacobian of [+] is not applied.  Linearisation 0 decides the NIS, dof, the chi2_max gate and
 * (FDE) the kept set, every outcome and each item's record; the iteration runs only on an applied stack, over its kept rows.
 * An item of the stack that is degenerate at an iterate (status 2's conditions) stops the iteration and the previous
 * linearisation is applied.  S not positive definite at any linearisation: status 1, nothing written.  max_iter 0 or 1 is the
 * call without _iter bit for bit (P, the state, the NIS, dx_norm).  Still one launch per 32 members, one copy each way and one
 * synchronisation; the iteration runs inside the member's CTA. */
typedef struct {
  int max_iter;          /* linearisations, 0 .. 16 (0 or 1: one) */
  double tol;            /* finite, >= 0: converged when max |delta_{i+1} - delta_i| <= tol */
} msckf_b200_aid_iter;
typedef struct {
  int iterations;        /* linearisations applied (0 when nothing was applied) */
  int converged;         /* 1: the last step was <= tol (always 0 for max_iter <= 1) */
  double step;           /* the last max |delta_{i+1} - delta_i| (0 for max_iter <= 1) */
} msckf_b200_aid_iter_result;
/* Refusals (MSCKF_B200_ERR_ARG, nothing written): everything the call without _iter refuses, iter or iter_out NULL, max_iter
 * outside 0..16, a tol that is not finite and >= 0, a GYRO_AT_REST or ACCEL_AT_REST item (the iterate carries no biases: a
 * standstill's rows are linear in b_g and b_a, and nearly so in the attitude); an un-fetched update returns MSCKF_B200_ERR_STATE.  A non-finite dx or P
 * entry returns MSCKF_B200_ERR_NUMERIC with the update applied. */
int msckf_b200_aid_stack_update_iter(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                     const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out, msckf_b200_aid_iter_result* iter_out);
int msckf_b200_aid_stack_update_fde_iter(msckf_b200_engine* e, const msckf_b200_aid_item* items, int n_items,
                                         const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                         msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out);
/* the same for every member of a batch: iter[i] and iter_out[i] per member (n_items[i] = 0 leaves member i untouched and out[i],
 * iter_out[i] not written, and iter[i] is not read); every member is validated before anything is launched.  One launch per 32
 * updated members. */
int msckf_b200_batch_aid_stack_update_iter(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                           double chi2_max, const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out,
                                           msckf_b200_aid_iter_result* iter_out);
int msckf_b200_batch_aid_stack_update_fde_iter(msckf_b200_batch* b, const msckf_b200_aid_item* const* items, const int* n_items,
                                               const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                               msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out);
/* ---- standstill: detect that the platform is at rest from the IMU, and fuse a zero-motion update (DESIGN.md 4.18) ----------
 * readings: k >= 2 IMU readings [k][7] (omega, a, dT) in msckf_b200_propagate_n's layout and the engine's dtype -- the ones
 * propagated since the previous image.  With R0 the 6 x 6 block diagonal of Q_imu's gyro (rows / columns 0..2) and accelerometer
 * (6..8) blocks, s = noise_scale and T = sum dT_j, the host forms in fp64, in reading order: the dT-weighted means w^ = sum dT_j
 * omega_j / T and a^ = sum dT_j a_j / T, and the scatter sigma = sum_j dT_j (y_j - y^)^T (s^2 R0)^-1 (y_j - y^) of y_j = [omega_j; a_j]
 * (chi-square with 6 (k - 1) dof at rest, whatever the state).  scatter = sigma / (6 (k - 1)) > scatter_max: outcome 1 (moving),
 * nothing is launched or written.  Otherwise the 9-row stack VELOCITY (z = 0, R = sigma_v^2 I), GYRO_AT_REST (z = w^, R = s^2
 * R0_g / T), ACCEL_AT_REST (z = a^, R = s^2 R0_a / T) runs as msckf_b200_aid_stack_update with chi2_max as its gate, bit for bit:
 * outcome 0 applied, 2 gated out (moving: the mean does not fit the state), -1 with stack.status 1 (S not positive definite).
 * The scatter term and the stack's NIS add up to the NIS of the dense update over all 6k reading rows, and the 9-row update
 * equals the dense one: the means are sufficient.  The caller skips the frame's vision work on outcome 0 (INTEGRATION.md).
 * Refusals (MSCKF_B200_ERR_ARG, nothing written): k < 2 or k > 4096, readings NULL, a dT that is not finite and > 0, a
 * non-finite reading, noise_scale < 1 or not finite, a sigma_v, scatter_max or chi2_max that is not finite and > 0, a gyro or
 * accelerometer block of Q_imu that is not positive definite; an un-fetched update returns MSCKF_B200_ERR_STATE.  A non-finite
 * dx or P entry returns MSCKF_B200_ERR_NUMERIC with the result filled and the update applied. */
typedef struct {
  double noise_scale;  /* s >= 1: the IMU noise inflation (vibration) */
  double sigma_v;      /* m/s: the zero-velocity row's standard deviation */
  double scatter_max;  /* > 0: the largest scatter / (6 (k - 1)) taken as at rest */
  double chi2_max;     /* > 0: the gate on the 9-row stack's NIS */
} msckf_b200_standstill;
typedef struct {
  msckf_b200_aid_result stack;  /* the 9-row stack, as msckf_b200_aid_stack_update reports it (outcome 1: NIS NaN, dof 0) */
  double scatter;               /* sigma / (6 (k - 1)) */
  int outcome;                  /* 0 applied; 1 moving (scatter > scatter_max: nothing launched); 2 moving (stack NIS > chi2_max);
                                   -1 stack.status 1 */
} msckf_b200_standstill_result;
int msckf_b200_standstill_update(msckf_b200_engine* e, const void* readings, int k, const msckf_b200_standstill* cfg,
                                 msckf_b200_standstill_result* out);
/* the same for every member of a batch (readings[i] [k[i]][7], out[i]; k[i] = 0 leaves member i untouched and out[i] not
 * written); every member is validated before anything is launched.  One launch per 32 members that pass the scatter test, none
 * when no member does. */
int msckf_b200_batch_standstill_update(msckf_b200_batch* b, const void* const* readings, const int* k, const msckf_b200_standstill* cfg,
                                       msckf_b200_standstill_result* out);
/* ---- mapped landmarks: image observations of landmarks whose position is known (prior map, surveyed marker, relocalisation) --
 * Observation i is (clone[i], z[i] normalised image coordinates, p_L_G[i] landmark position in G).  With C = C(q_CG) and p_C_G of
 * that clone: p_C = C (p_L - p_C_G), z^ = p_C[0:2] / p_C[2], r_i = z_i - z^ (calcResidual, msckf.h:960-978), Jacobian the 2 x 6
 * block [J [p_C]x, -J C] over the clone's [dtheta, dp] (msckf.h:929-936) WITHOUT the observability projection (a known landmark
 * observes global position and yaw) and without a feature null space (the landmark is not estimated; its position is taken as
 * exact -- msckf_b200_map_landmark_update below takes each landmark's map covariance).  Noise R (2 x 2, same for every observation; NULL: diag(u_var', v_var')).
 * Per observation: flag 2 (not used) when p_C[2] <= 0 or z^ is not finite (gamma NaN); else gamma = r^T (X P_kk X^T + R)^-1 r,
 * flag 1 (gated out) when chi2_obs > 0 and gamma > chi2_obs, else flag 0 (used).  The used rows are whitened and compressed per
 * clone by a Householder QR (exact: each row touches one clone), then S = T P T^T + I = L L^T, W = L^-1 T P, y = L^-1 rho,
 * NIS = |y|^2 + the QR leftovers (equal to the NIS of the dense stacked system), dx = W^T y, P <- P - W^T W (fp64, rounded once,
 * both halves written, in place) and the state injection of msckf_b200_aid_update.  All arithmetic is fp64 for both dtypes.
 * Three launches per 32 members with observations, one host-to-device copy, one device-to-host copy, one synchronisation.
 * Caps: 256 observations per clone and 4096 per member and call.  The vision update's bookkeeping and the launch count are
 * not changed.
 * Iterated update (max_iter >= 2, an iterated EKF for relocalisation after drift, where one linearisation is far off): with
 * delta_0 = 0 and the iterate x_i = x^ [+] delta_i on the clone poses (q <- normalise(buildUpdateQuat(dtheta) * q), p <- p + dp,
 * fp64), linearisation i evaluates r_i, H_i at x_i, compresses [X~ | r~ + X~ e_k] per clone as above (e_k: delta_i of clone k)
 * and factors S against the prior P; delta_{i+1} = W^T y = K_i (r_i + H_i delta_i).  It stops when max |delta_{i+1} - delta_i|
 * <= tol (converged) or after max_iter linearisations; then P <- P - W^T W and one injection of W^T y, both of the last
 * linearisation.  The flags, gamma, NIS and dof are linearisation 0's.  A used observation that is behind the camera or not
 * finite at an iterate stops the iteration, and the previous linearisation is applied.  The Jacobian of [+] is not applied
 * (the iterate's error-state Jacobian is taken as I).  The launches per 32 members become clone, gain, (step, clone, gain) x
 * (K - 1), downdate, with K the largest max_iter among them; still one copy each way and one synchronisation.
 * max_iter 0 or 1 is the single linearisation above, bit for bit. */
typedef struct {
  int n_obs;             /* observations; in a batch, 0 leaves the member untouched */
  const int* clone;      /* [n_obs] positions in the window */
  const double* z;       /* [n_obs][2] */
  const double* p_L_G;   /* [n_obs][3] */
  const double* R;       /* [3]: uu, uv, vv (positive definite), or NULL: diag(u_var', v_var') of the filter */
  double chi2_obs;       /* > 0: per-observation gate on gamma */
  double* gamma;         /* [n_obs] out, or NULL */
  int* flag;             /* [n_obs] out (0 used, 1 gated out, 2 behind the camera / not finite, 3 excluded by consensus), or NULL */
  int max_iter;          /* linearisations, 0 .. 16 (0 or 1: one) */
  double tol;            /* finite, >= 0: the iteration has converged when max |delta_{i+1} - delta_i| <= tol */
} msckf_b200_landmarks;
typedef struct {
  double nis;            /* NIS of the used observations (NaN when S is not positive definite) */
  double dx_norm;        /* |dx| of the applied update (0 when not applied) */
  int dof;               /* 2 x used */
  int rows;              /* rows of the compressed system (sum over clones of min(2 a_k, 6)) */
  int used;              /* observations with flag 0 */
  int applied;           /* 1: P and the state were updated */
  int status;            /* 0: applied, or nothing used; 1: S not positive definite (at any linearisation), nothing written */
  int iterations;        /* linearisations applied (1 for the single linearisation; 0 when nothing was applied) */
  int converged;         /* 1: the last step was <= tol (always 0 for max_iter <= 1) */
  double step;           /* the last max |delta_{i+1} - delta_i| (0 for max_iter <= 1) */
} msckf_b200_landmark_result;
/* A clone outside the window, n_obs < 0 or beyond the caps, a NULL or non-finite z / p_L_G / R, an R that is not positive
 * definite, a NaN chi2_obs, max_iter outside 0 .. 16 or a tol that is not finite and >= 0 returns MSCKF_B200_ERR_ARG, an un-fetched update MSCKF_B200_ERR_STATE; then nothing is written.
 * A non-finite dx or P entry returns MSCKF_B200_ERR_NUMERIC with the result filled and the update applied.  n_obs = 0 on a single
 * engine fills out with zeros and launches nothing. */
int msckf_b200_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out);
/* the same for every member of a batch (lm[i], out[i]; out[i] is not written for a member with lm[i].n_obs = 0); every member is
 * validated before anything is launched. */
int msckf_b200_batch_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, msckf_b200_landmark_result* out);
/* ---- mapped landmarks with map uncertainty: the same update with each landmark's position error marginalised -----------
 * Observation i is of landmark landmark[i], whose true position is p_L_G[i] + dp, dp ~ N(0, Sigma_L[landmark[i]]) (p_L_G must be
 * identical for observations of one landmark).  With F_i = J C, the observation's block over dp (= -X_i[:, 3:6]), the gate is
 * gamma_i = r^T (X P_kk X^T + F Sigma F^T + R)^-1 r, and the used observations are fused with the noise R (x) I + F Sigma F^T,
 * which couples the rows of one landmark across the clones that see it: the landmark's error is common to them.  On the device
 * a landmark seen from one clone is whitened by R + F Sigma F^T before its clone's QR; the used rows of a landmark seen from
 * 2 .. 8 clones are stacked under the prior rows [0 | L^-1 | 0] (Sigma = L L^T) and three Householder reflectors on the F
 * columns eliminate dp exactly; the landmarks with one clone set are then compressed together by one Householder QR over their
 * 6c clone columns to min(2 used, 6c) rows.  rows reports the sum of those and of the clones' min(2 a_k, 6); dof = 2 x used and
 * NIS are those of the dense marginal system.  The gain, downdate and injection are the exact-map update's.  Iterated
 * (max_iter >= 2): each linearisation relinearises at the iterate clone poses (F too) with the landmarks kept at p_L_G, so it is
 * an IEKF over the clone poses with the map marginalised, not a joint estimate of the landmarks.  Each call treats the map
 * error as fresh: fusing the same landmarks call after call counts their error more than once (DESIGN.md 4.12).
 * Launches per 32 members when any of them has Sigma_L: clone, set, gain, (step, clone, set, gain) x (K - 1), downdate; still
 * one copy each way and one synchronisation.
 * Caps, each MSCKF_B200_ERR_ARG before anything is launched (nothing written): 8 clones per landmark, 256 observations per
 * clone set, 256 clone sets per member and 1152 rows (6 x 192 clones, the gain's row table) in the worst-case compressed system
 * (the sum over clones of min(2 a_k, 6) and over clone sets of min(2 observations, 6c)).  Also ERR_ARG: landmark NULL or
 * outside 0 .. n_landmarks - 1, a Sigma_L that is not finite or not positive definite, p_L_G differing within a landmark, and one
 * landmark observed twice from one clone. */
typedef struct {
  const int* landmark;   /* [n_obs] landmark of each observation, 0 .. n_landmarks - 1 */
  const double* Sigma_L; /* [n_landmarks][6] lower triangle xx, yx, yy, zx, zy, zz (positive definite), or NULL: the map is exact
                            and the call is msckf_b200_landmark_update's, with its kernels and launches */
  int n_landmarks;
} msckf_b200_landmark_map;
/* map NULL: msckf_b200_landmark_update */
int msckf_b200_map_landmark_update(msckf_b200_engine* e, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                   msckf_b200_landmark_result* out);
/* the same for every member of a batch (lm[i], map[i], out[i]; map NULL: every member exact) */
int msckf_b200_batch_map_landmark_update(msckf_b200_batch* b, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                         msckf_b200_landmark_result* out);
/* ---- mapped landmarks with consensus: which matches to trust, decided on the device before the update (DESIGN.md 4.17) ----
 * Relocalisation matches contain wrong ones, and after drift a per-observation gate against the prior cannot tell them from
 * right ones.  Right matches agree on one common correction of the window; wrong ones do not.  A hypothesis is a 4-dof rigid
 * correction (psi about G's z axis, t) applied to the map: p_L' = Rz(psi)^T (p_L - c - t) + c, c = pivot = the mean p_C_G of the
 * clones the observations name, projected with the filter's clone pose.  Observation i is an inlier of (psi, t) when its depth is
 * > 0 and e_i = (z_i - z^_i)^T R^-1 (z_i - z^_i) <= thresh (R: the call's, or diag(u_var', v_var')).
 * Hypothesis h is fitted to the observations (i, j) drawn from seed by splitmix64 (DESIGN.md 4.17), i != j in input order, by
 * Gauss-Newton from (0, 0): at most 8 steps, stopping at max |step| <= 1e-12.  It is valid when every step's 4 x 4 Cholesky has
 * its pivots > 1e-12 x their diagonal entries, both points stay in front and both are inliers of the result.  The best valid
 * hypothesis has the most inliers (a tie: the lowest h).  A refit (Gauss-Newton over its inliers, from its (psi, t), at most 8
 * steps) is rescored once; the final inliers are the refit's if it succeeded and kept at least as many, else the hypothesis's.
 * Fewer than min_inliers final inliers (no valid hypothesis included): status 1, every observation not flagged 2 gets flag 3
 * and nothing is written (applied 0).  Otherwise the outliers get flag 3 (excluded by consensus, not used) and the update runs
 * on the rest, in every form (exact map or Sigma_L, single or iterated): flag 2 comes before 3, and 3 before the chi2_obs gate.
 * gamma is written as without consensus.  The consensus never seeds the iterate: the update starts from the prior.
 * Two more launches per 32 members with consensus; still one copy each way and one synchronisation. */
typedef struct {
  int hypotheses;             /* 0 .. 1024; 0: no consensus (the plain call, bit for bit) */
  double thresh;              /* finite, > 0 (when hypotheses > 0) */
  int min_inliers;            /* >= 2 (when hypotheses > 0) */
  unsigned long long seed;
  int* scores;                /* [hypotheses] out: each hypothesis's inliers, or -1 when it is not valid; or NULL */
} msckf_b200_landmark_consensus;
typedef struct {
  int status;                 /* 0: a consensus was found; 1: fewer than min_inliers inliers (nothing was written) */
  int inliers;                /* final inliers */
  int best;                   /* the best valid hypothesis, or -1 */
  int valid;                  /* valid hypotheses (0: none) */
  int refit;                  /* 1: the final inliers and (yaw, t) are the refit's */
  double yaw, t[3];           /* the final correction */
  double pivot[3];            /* c */
} msckf_b200_landmark_consensus_result;
/* cons NULL or hypotheses = 0: msckf_b200_map_landmark_update (map NULL: the exact map), bit for bit, and cons_out (if given)
 * gets best = -1 and zeros; cons_out may be NULL.  MSCKF_B200_ERR_ARG before anything is launched: hypotheses outside 0 .. 1024,
 * and with hypotheses > 0 a thresh that is not finite and > 0 or min_inliers < 2; and what the plain call refuses. */
int msckf_b200_landmark_update_consensus(msckf_b200_engine* e, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                         const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_result* out,
                                         msckf_b200_landmark_consensus_result* cons_out);
/* the same for every member of a batch: cons[i] and cons_out[i] (cons NULL: no member runs a consensus); a member's arithmetic
 * depends only on its own inputs, so a batch equals single calls bit for bit */
int msckf_b200_batch_landmark_update_consensus(msckf_b200_batch* b, const msckf_b200_landmarks* lm, const msckf_b200_landmark_map* map,
                                               const msckf_b200_landmark_consensus* cons, msckf_b200_landmark_result* out,
                                               msckf_b200_landmark_consensus_result* cons_out);
/* Convenience: one update on each of n engines through a batch.  If the engines already form a batch (in this order) it is
 * used; otherwise a temporary one is created and destroyed around the call.  Returns the first non-zero status. */
int msckf_b200_update_batch(msckf_b200_engine** engines, int n, int mode, const msckf_b200_tracks* tracks, msckf_b200_report* reports,
                            int threads);
/* covariance / pose gather of pruneEmptyStates msckf.h:685-761 and pruneRedundantStates :616-681:
 * keep[] = ascending positional indices of the clones that survive (n_keep = 0: only the IMU block stays).
 * Asynchronous: keep[] travels as a kernel argument, nothing is synchronised and captured graphs stay valid. */
int msckf_b200_prune(msckf_b200_engine* e, const int* keep, int n_keep);

int msckf_b200_num_clones(msckf_b200_engine* e);
/* imu: p,v,b_g,b_a,g,q_IG, p_null,v_null,q_null (29 scalars); clone_poses: [M*7] p(3) q(4).  Either may be NULL. */
int msckf_b200_get_state(msckf_b200_engine* e, void* imu, void* clone_poses);
/* full (15+6M)^2 covariance, row-major, dtype scalars */
int msckf_b200_get_covariance(msckf_b200_engine* e, void* out);
/* overwrite the covariance (same layout; checkpoint restore, Monte-Carlo initialisation) */
int msckf_b200_set_covariance(msckf_b200_engine* e, const void* in);
/* counters[0..7]: num_feature_tracks_residualized_, pfg_shifted, pfg_oob, n_updates, last m, last rank, 0, 0 */
int msckf_b200_get_counters(msckf_b200_engine* e, long long* counters);
/* last delta-x (fp64), returns its length */
int msckf_b200_last_delta_x(msckf_b200_engine* e, double* out, int cap);
/* diagnostics of the last update's rank decision: for every index of the compressed system, the pivot of the basis Gram matrix
 * relative to its original diagonal (the squared sine against the span of the previous basis vectors) at the moment it was
 * compared with the rank threshold (option 0).  Directions in the null space of H_o show up as rounding noise here; the gap
 * between that noise and the smallest kept pivot is the margin of the decision.  Returns the dimension 15 + 6 M of that update (0 before the first one). */
int msckf_b200_rank_pivots(msckf_b200_engine* e, double* out, int cap);
/* option keys: 0 = rank threshold of the compression (relative pivot of the basis Gram matrix = squared sine to the span of the previous basis vectors, default 1e-9:
 *                  measured pivots of null directions are rounding noise up to ~2e-11, the smallest real pivot of the test windows is > 1e-3,
 *                  see msckf_b200_rank_pivots);
 *              1 = record per-kernel CUDA events in _launch (profiling aid, default off);
 *              2 = replay the update's kernel sequence as a CUDA graph when the batch signature repeats (default on);
 *              3 = fuse the forward substitution into the blocked Cholesky of the tail kernel where the window allows it
 *                  (15 + 6M <= 255; default on; 0 = always run it as a separate sweep -- same results up to rounding);
 *              4 = launch the update's kernels with programmatic dependent launch (default on);
 *              5 = Gram products of the compression on the FP64 tensor-core path (mma.sync m8n8k4 f64, SASS DMMA; default on;
 *                  0 = SIMT DFMA tiles -- same results to fp64 rounding);
 *              6 = threads that work on one track in the feature kernel: 128 (a CTA per track: lowest latency), 64, or 32
 *                  (a warp per track, two tracks per CTA: highest throughput); 0 = by batch size (default: 128 for one
 *                  filter, 32 for a device batch).  The results are bit-identical for every value;
 *              7 = CTAs that run the tail's chains of diagonal blocks: 2 (default where the device accepts clusters of 9: Gamma's
 *                  and S''s chains side by side on two CTAs, seven worker CTAs) or 1 (cluster of 8, both chains on one CTA);
 *                  0 = default.  Same rank decisions; results agree to fp64 rounding;
 *              8 = stop an update after the compression (testing aid, default off): the kernels up to T'', R'', r'' run, nothing
 *                  after them, so P, the state and delta-x are left as they were and the report's rank is 0.  Before the kernels
 *                  every compression workspace of the engine is filled with NaN, so an element no kernel wrote shows up as a NaN
 *                  in msckf_b200_stage_buffer.  A device batch stops only when every member has the option set; a batch whose
 *                  members disagree is refused at stage time (MSCKF_B200_ERR_ARG, nothing written). */
int msckf_b200_set_option(msckf_b200_engine* e, int key, double value);
/* buffers of the last update's compression stage, for msckf_b200_stage_buffer.  n = 15 + 6M, c = 6M, N tracks, O observations */
enum {
  MSCKF_B200_STAGE_T2 = 0,       /* T'' [n][n] fp64 */
  MSCKF_B200_STAGE_R2 = 1,       /* R'' [n][n] fp64 */
  MSCKF_B200_STAGE_R2_RHS = 2,   /* r'' [n] fp64 */
  MSCKF_B200_STAGE_Z = 3,        /* Z = U^T X per track [3N][c] fp64 */
  MSCKF_B200_STAGE_YQ = 4,       /* Yq [3N][c] fp64 */
  MSCKF_B200_STAGE_UR = 5,       /* U^T r [3N] fp64 */
  MSCKF_B200_STAGE_D1 = 6,       /* sum X^T X per clone [M][6][6] fp64 */
  MSCKF_B200_STAGE_D2 = 7,       /* sum X^T D X per clone [M][6][6] fp64 */
  MSCKF_B200_STAGE_BB = 8,       /* sum X^T r per clone [M][6] fp64 */
  MSCKF_B200_STAGE_XG = 9,       /* projected clone Jacobian blocks [O][2][6], the filter's dtype */
  MSCKF_B200_STAGE_RG = 10,      /* residuals [O][2], the filter's dtype */
  MSCKF_B200_STAGE_VG = 11,      /* Householder vectors of H_f, per track [2L][3], the filter's dtype */
  MSCKF_B200_STAGE_TAUG = 12,    /* Householder coefficients [N][3], the filter's dtype */
  MSCKF_B200_STAGE_ACCEPT = 13,  /* gate flags [N] int */
  MSCKF_B200_STAGE_ROW_OFF = 14  /* first stacked row of each track [N + 1] int */
};
/* copy buffer `which` of the last update into out (at most cap elements; out may be NULL when cap is 0) and return its element
 * count.  T'', R'', r'' are the compression's outputs after an update with option 8 set; after a full update the later
 * kernels may have reused them.  0 before an update, or after a stage, window growth or track-capacity growth that followed it;
 * an un-fetched update returns MSCKF_B200_ERR_STATE, an unknown `which` MSCKF_B200_ERR_ARG. */
int msckf_b200_stage_buffer(msckf_b200_engine* e, int which, void* out, int cap);
/* checkpoint / resume: copy the complete filter state of src into dst (same dtype and capacities) */
int msckf_b200_copy_state(msckf_b200_engine* dst, const msckf_b200_engine* src);
/* number of kernels launched by this handle so far (bench.py's gpu_launches) */
long long msckf_b200_launch_count(const msckf_b200_engine* e);
/* the handle's cudaStream_t (for event timing on the launching stream) */
void* msckf_b200_stream(msckf_b200_engine* e);
int msckf_b200_synchronize(msckf_b200_engine* e);
const char* msckf_b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* MSCKF_B200_H_ */
