/* include/msckf_mono_c.h -- C view of the drop-in class msckf_mono::MSCKF<_S> (include/msckf_mono/msckf.h).
 *
 * One function per public member of the reference class (msckf.h:72-848), so that non-C++ hosts (the
 * Python parity tests and bench.py via ctypes) drive exactly the call sequence a C++ caller would.  All
 * scalars cross this view as double (exact widening of the filter's _S = float); the class beneath is
 * instantiated for float or double.  Returns 0 / a count on success, a negative value on failure
 * (msckf_mono_last_error() holds the message).  Exported by libmsckf_b200.so.
 */
#ifndef MSCKF_MONO_C_H_
#define MSCKF_MONO_C_H_
#include <stdint.h>
#include <msckf_b200.h>
#ifdef __cplusplus
extern "C" {
#endif
int msckf_mono_create(int dtype /*0 = float, 1 = double*/, void** out);
void msckf_mono_destroy(void* h);
/* device ordinal and engine capacities (0 = derive from MSCKFParams); call before initialize */
int msckf_mono_set_engine_options(void* h, int device, int max_clones, int max_tracks, int max_obs);
/* camera[12]: c_u,c_v,f_u,f_v,b,q_CI(xyzw),p_C_I; noise[371]: u_var',v_var',Q_imu[144],initial_imu_covar[225];
 * params[8]: max_gn_cost_norm,min_rcond,translation_threshold,redundancy_angle_thresh,redundancy_distance_thresh,
 *            min_track_length,max_track_length,max_cam_states; imu_state[19]: p,v,b_g,b_a,g,q_IG(xyzw)      msckf.h:72 */
int msckf_mono_initialize(void* h, const double* camera, const double* noise, const double* params, const double* imu_state);
int msckf_mono_propagate(void* h, const double* omega_a_dT);                                  /* msckf.h:101 */
int msckf_mono_augment_state(void* h, int state_id, double time);                             /* msckf.h:148 */
int msckf_mono_update(void* h, const double* measurements, const uint64_t* ids, int n);       /* msckf.h:215 */
int msckf_mono_add_features(void* h, const double* features, const uint64_t* ids, int n);     /* msckf.h:302 */
int msckf_mono_marginalize(void* h);                                                          /* msckf.h:336 */
int msckf_mono_prune_redundant_states(void* h);                                               /* msckf.h:453 */
int msckf_mono_prune_empty_states(void* h);                                                   /* msckf.h:685 */
int msckf_mono_finish(void* h);                                                               /* msckf.h:765 */
int msckf_mono_get_num_cam_states(void* h);                                                   /* msckf.h:810 */
int msckf_mono_get_imu_state(void* h, double* out29);                                         /* msckf.h:815 */
int msckf_mono_get_cam_states(void* h, double* poses7, int* ids2, double* times);             /* msckf.h:835 */
int msckf_mono_get_cam_tracked_ids(void* h, int cam, uint64_t* out, int cap);
int msckf_mono_get_covariance(void* h, double* out);
int msckf_mono_get_map(void* h, double* out, int cap);                                        /* msckf.h:820 */
int msckf_mono_get_pruned_states(void* h, double* poses7, int* ids2, int cap);                /* msckf.h:840 */
int msckf_mono_get_tracked_feature_ids(void* h, uint64_t* out, int cap);
/* diagnostics */
int msckf_mono_last_report(void* h, int* flags4 /*cm,valid,accepted,rows*/, double* gamma, double* pfg, int cap);
int msckf_mono_get_counters(void* h, long* out8);
int msckf_mono_set_option(void* h, int key, double value);
int msckf_mono_last_delta_x(void* h, double* out, int cap);
int msckf_mono_queued_tracks(void* h, uint64_t* ids, int* nobs, int cap);
/* the track batch queued by update()/finish() in the engine's flat SoA form (obs as double); returns n_tracks */
int msckf_mono_pack_queued(void* h, int* obs_offset, double* obs, int* clone_index, int cap_tracks, int cap_obs);
/* pipelining helpers: marginalize() = launch + collect */
int msckf_mono_marginalize_launch(void* h);
int msckf_mono_marginalize_collect(void* h);
/* marginalize() on n independent filters of one scalar type as ONE device batch (msckf_mono::MSCKFBatch<_S>: one launch per
 * kernel with the filter index in blockIdx.z, one CUDA graph, one packed copy each way); `threads` host threads share the
 * packing.  Bit-identical to marginalize() on each filter.  _batch_create makes the batch persistent (the filters share its
 * stream while it lives); msckf_mono_marginalize_batch is the one-shot form (temporary batch around one call). */
int msckf_mono_batch_create(void** handles, int n, int threads, void** out);
void msckf_mono_batch_destroy(void* batch);
int msckf_mono_batch_marginalize(void* batch);
/* the rest of the per-image step on every filter of the batch, same meaning as the single-filter calls above; each device
 * operation is one batched call (datasets/asl_msckf.cpp:233-294 for n filters) */
int msckf_mono_batch_propagate(void* batch, int member, const double* omega_a_dT);             /* msckf.h:101, filter `member` */
int msckf_mono_batch_augment_state(void* batch, const int* state_ids, const double* times);    /* msckf.h:148, one per filter */
int msckf_mono_batch_prune_empty_states(void* batch);                                          /* msckf.h:685 */
int msckf_mono_batch_prune_redundant_states(void* batch);                                      /* msckf.h:453 */
int msckf_mono_batch_finish(void* batch);                                                      /* msckf.h:765 */
/* every filter's IMU state and clone poses fetched with one synchronisation (the getters then read the host mirror) */
int msckf_mono_batch_refresh_state(void* batch);
void* msckf_mono_batch_handle(void* batch); /* the msckf_b200_batch* beneath */
int msckf_mono_marginalize_batch(void** handles, int n, int threads);
/* NEES of the estimate against ground truth (MSCKF::nees, msckf_b200_nees): truth_imu[19] p,v,b_g,b_a,g,q_IG(xyzw);
 * truth_poses [M*7] p_C_G,q_CG(xyzw) in window order, or NULL (no whole-state NEES); out7: orientation, position, pose, imu,
 * full, dim_full, first_bad_pivot (-1: positive definite).  _batch_nees: truth_imu[i], truth_poses NULL or [i] per filter,
 * out7 [n][7], one device call for the batch. */
int msckf_mono_nees(void* h, const double* truth_imu, const double* truth_poses, double* out7);
int msckf_mono_batch_nees(void* batch, const double* const* truth_imu, const double* const* truth_poses, double* out7);
/* aided measurement update (MSCKF::aidedUpdate, msckf_b200_aid_update: models, layouts and errors there); the filter's host
 * mirror is refreshed on the next getter.  _batch_aid_update: aid[i] / out[i] per filter (aid[i].model < 0: filter i is left
 * alone), one device call for the batch. */
int msckf_mono_aid_update(void* h, const msckf_b200_aid* aid, msckf_b200_aid_result* out);
int msckf_mono_batch_aid_update(void* batch, const msckf_b200_aid* aid, msckf_b200_aid_result* out);
/* stacked aided update (MSCKF::aidedUpdate(items), msckf_b200_aid_stack_update: models, layouts and errors there): n_items
 * items with clones by window position, one chi2_max.  _batch_aid_stack_update: n_items[i] per filter (0: filter i is left alone
 * and out[i] is not written), the items concatenated in filter order, one device call.  _body_velocity_update: v3 in the IMU
 * frame, mask bits 0..2, R [m][m] over the selected rows.  _relative_pose_update: the pose of image state_id_b relative to
 * image state_id_a (p3, q4 xyzw, R36 [6][6]); an id not in the window fails before any device call. */
int msckf_mono_aid_stack_update(void* h, const msckf_b200_aid_item* items, int n_items, double chi2_max, msckf_b200_aid_result* out);
int msckf_mono_batch_aid_stack_update(void* batch, const int* n_items, const msckf_b200_aid_item* items, double chi2_max,
                                      msckf_b200_aid_result* out);
/* the same stacks with fault detection and exclusion over their items (MSCKF::aidedUpdate(items, fde),
 * msckf_b200_aid_stack_update_fde: rounds, outcomes and errors there); one fde for the batch.  A NULL fde, a chi2 entry that is
 * not finite or not > 0, or max_exclude outside 0..7 fails before any device call. */
int msckf_mono_aid_stack_update_fde(void* h, const msckf_b200_aid_item* items, int n_items, const msckf_b200_aid_fde* fde,
                                    msckf_b200_aid_fde_result* out);
int msckf_mono_batch_aid_stack_update_fde(void* batch, const int* n_items, const msckf_b200_aid_item* items,
                                          const msckf_b200_aid_fde* fde, msckf_b200_aid_fde_result* out);
/* the same stacks iterated (MSCKF::aidedUpdate(items, chi2_max | fde, iter, iter_out), msckf_b200_aid_stack_update_iter /
 * _fde_iter: iteration, results and errors there); the batch forms take iter[i] and fill iter_out[i] per filter (not read or
 * written for a filter left alone).  A NULL iter or iter_out, max_iter outside 0..16 or a tol that is not finite and >= 0
 * fails before any device call. */
int msckf_mono_aid_stack_update_iter(void* h, const msckf_b200_aid_item* items, int n_items, double chi2_max,
                                     const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out, msckf_b200_aid_iter_result* iter_out);
int msckf_mono_aid_stack_update_fde_iter(void* h, const msckf_b200_aid_item* items, int n_items, const msckf_b200_aid_fde* fde,
                                         const msckf_b200_aid_iter* iter, msckf_b200_aid_fde_result* out,
                                         msckf_b200_aid_iter_result* iter_out);
int msckf_mono_batch_aid_stack_update_iter(void* batch, const int* n_items, const msckf_b200_aid_item* items, double chi2_max,
                                           const msckf_b200_aid_iter* iter, msckf_b200_aid_result* out,
                                           msckf_b200_aid_iter_result* iter_out);
int msckf_mono_batch_aid_stack_update_fde_iter(void* batch, const int* n_items, const msckf_b200_aid_item* items,
                                               const msckf_b200_aid_fde* fde, const msckf_b200_aid_iter* iter,
                                               msckf_b200_aid_fde_result* out, msckf_b200_aid_iter_result* iter_out);
int msckf_mono_body_velocity_update(void* h, const double* v3, int mask, const double* R, double chi2_max, msckf_b200_aid_result* out);
int msckf_mono_relative_pose_update(void* h, int state_id_a, int state_id_b, const double* p3, const double* q4, const double* R36,
                                    double chi2_max, msckf_b200_aid_result* out);
/* mapped-landmark update (MSCKF::landmarkUpdate, msckf_b200_landmark_update: model, gate and errors there): n_obs observations,
 * state_ids [n] (the image's state id; an id not in the window fails before any device call), z [n][2], p_L_G [n][3];
 * R3 = uu, uv, vv or NULL (the filter's pixel noise); gamma [n] / flag [n] out, or NULL.  _batch_landmark_update: n_obs[i] per
 * filter (0: filter i is left alone and out[i] is not written), the other arrays concatenated in filter order, one device call. */
int msckf_mono_landmark_update(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                               double chi2_obs, double* gamma, int* flag, msckf_b200_landmark_result* out);
int msckf_mono_batch_landmark_update(void* batch, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G,
                                     const double* R3, double chi2_obs, double* gamma, int* flag, msckf_b200_landmark_result* out);
/* the same, iterated: at most max_iter (0 .. 16) linearisations, converged when max |delta_{i+1} - delta_i| <= tol
 * (MSCKF::landmarkUpdate's max_iter / tol; max_iter 0 or 1 is the calls above) */
int msckf_mono_landmark_update_iter(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G, const double* R3,
                                    double chi2_obs, int max_iter, double tol, double* gamma, int* flag, msckf_b200_landmark_result* out);
int msckf_mono_batch_landmark_update_iter(void* batch, const int* n_obs, const int* state_ids, const double* z, const double* p_L_G,
                                          const double* R3, double chi2_obs, int max_iter, double tol, double* gamma, int* flag,
                                          msckf_b200_landmark_result* out);
/* mapped-landmark update with map uncertainty (MSCKF::landmarkUpdate over mapObservation / mapLandmark,
 * msckf_b200_map_landmark_update: model, gate, caps and errors there): n_obs observations (state_ids [n], landmark [n] indices
 * into this call's landmarks, z [n][2]) of n_landmarks landmarks (p_L_G [L][3], Sigma [L][6] lower triangle xx, yx, yy, zx, zy,
 * zz); R3, chi2_obs, max_iter, tol, gamma, flag as in msckf_mono_landmark_update_iter.  _batch_map_update: n_obs[i] and
 * n_landmarks[i] per filter, every array concatenated over the filters in order; out[i] of a filter with n_obs[i] = 0 is not
 * written. */
int msckf_mono_map_update(void* h, int n_obs, const int* state_ids, const int* landmark, const double* z, int n_landmarks,
                          const double* p_L_G, const double* Sigma, const double* R3, double chi2_obs, int max_iter, double tol,
                          double* gamma, int* flag, msckf_b200_landmark_result* out);
int msckf_mono_batch_map_update(void* batch, const int* n_obs, const int* state_ids, const int* landmark, const double* z,
                                const int* n_landmarks, const double* p_L_G, const double* Sigma, const double* R3, double chi2_obs,
                                int max_iter, double tol, double* gamma, int* flag, msckf_b200_landmark_result* out);
/* mapped-landmark update with a consensus on the matches (MSCKF::landmarkUpdate with a msckf_b200_landmark_consensus,
 * msckf_b200_landmark_update_consensus: model, flag 3, errors there), exact map; the other arguments as in
 * msckf_mono_landmark_update_iter.  _batch_: cons[i] and cons_out[i] per filter, the observation arrays as in
 * msckf_mono_batch_landmark_update_iter.  An invalid consensus fails before any device call. */
int msckf_mono_landmark_update_consensus(void* h, int n_obs, const int* state_ids, const double* z, const double* p_L_G,
                                         const double* R3, double chi2_obs, int max_iter, double tol,
                                         const msckf_b200_landmark_consensus* cons, double* gamma, int* flag,
                                         msckf_b200_landmark_result* out, msckf_b200_landmark_consensus_result* cons_out);
int msckf_mono_batch_landmark_update_consensus(void* batch, const int* n_obs, const int* state_ids, const double* z,
                                               const double* p_L_G, const double* R3, double chi2_obs, int max_iter, double tol,
                                               const msckf_b200_landmark_consensus* cons, double* gamma, int* flag,
                                               msckf_b200_landmark_result* out, msckf_b200_landmark_consensus_result* cons_out);
/* standstill detection and the zero-motion update (MSCKF::standstillUpdate, msckf_b200_standstill_update: statistics, outcomes
 * and errors there): k readings [k][7] omega, a, dT (rounded to the filter's scalar type), the ones propagated since the previous
 * image.  _batch_standstill_update: k[i] per filter (0: filter i is left alone and out[i] is not written), the readings
 * concatenated in filter order, one device call.  Bad readings or a bad cfg fail before any device call. */
int msckf_mono_standstill_update(void* h, const double* readings, int k, const msckf_b200_standstill* cfg, msckf_b200_standstill_result* out);
int msckf_mono_batch_standstill_update(void* batch, const int* k, const double* readings, const msckf_b200_standstill* cfg,
                                       msckf_b200_standstill_result* out);
/* the msckf_b200_engine* beneath (for CUDA-event timing on its stream, launch counts, state copies) */
void* msckf_mono_engine(void* h);
/* copy the complete filter (host bookkeeping + device state) of src into dst; both must be initialised alike */
int msckf_mono_clone_from(void* dst, void* src);
const char* msckf_mono_last_error(void);
#ifdef __cplusplus
}
#endif
#endif
