/*
 * okvis_b200.h -- C-ABI of libokvis_b200.so, the H100-native (sm_90a) hot path of OKVIS.
 *
 * Every entry point is extern "C", takes plain pointers / sizes / POD structs and
 * returns an int status (0 = OKB_OK, <0 = error, see okb_status).  Host buffers are
 * borrowed for the duration of a call only; device memory is owned by the opaque
 * context handle.  No exception ever crosses this boundary.
 *
 * Reference interfaces replaced (paths relative to the OKVIS source tree):
 *   okb_optimize              <- okvis::Estimator::optimize           okvis_ceres/src/Estimator.cpp:843-906
 *                                (Map::solve -> ceres::Solve           okvis_ceres/include/okvis/ceres/Map.hpp:371-373)
 *   okb_window_upload/download<- the graph held by okvis::ceres::Map   okvis_ceres/include/okvis/ceres/Map.hpp:348-402
 *   okb_eval_reprojection     <- ReprojectionError::EvaluateWithMinimalJacobians
 *                                okvis_ceres/include/okvis/ceres/implementation/ReprojectionError.hpp:87-242
 *   okb_eval_imu              <- ImuError::EvaluateWithMinimalJacobians okvis_ceres/src/ImuError.cpp:514-685
 *   okb_imu_propagate         <- ImuError::propagation (static)        okvis_ceres/src/ImuError.cpp:287-504
 *   okb_imu_propagate_batch: no reference counterpart -- okb_imu_propagate for many sessions in one launch
 *   okb_eval_pose_error       <- PoseError::EvaluateWithMinimalJacobians         okvis_ceres/src/PoseError.cpp:86-136
 *   okb_eval_speed_bias_error <- SpeedAndBiasError::EvaluateWithMinimalJacobians okvis_ceres/src/SpeedAndBiasError.cpp:89-116
 *   okb_eval_relative_pose    <- RelativePoseError::EvaluateWithMinimalJacobians okvis_ceres/src/RelativePoseError.cpp:84-162
 *   okb_eval_marginalization  <- MarginalizationError::EvaluateWithMinimalJacobians okvis_ceres/src/MarginalizationError.cpp:893-946
 *   okb_window_marginalize    <- MarginalizationError::addResidualBlock / marginalizeOut / updateErrorComputation
 *                                okvis_ceres/src/MarginalizationError.cpp:127-435, 507-846 (driven by Estimator.cpp:434-773)
 *   okb_window_marginalize_batch: no reference counterpart -- okb_window_marginalize on many resident windows in one launch
 *   okb_hamming_match         <- okvis::DenseMatcher::match            okvis_matcher/include/okvis/implementation/DenseMatcher.hpp:48-225
 *                                + assignbest                          okvis_matcher/src/DenseMatcher.cpp:69-110
 *   okb_hamming_match_gated   <- VioKeyframeWindowMatchingAlgorithm::distance + verifyMatch (hpp:132-144, cpp:304-339),
 *                                ProbabilisticStereoTriangulator::stereoTriangulate (cpp:168-227), triangulateFast
 *   okb_hamming_candidates    <- VioKeyframeWindowMatchingAlgorithm::specificDescriptorDistance
 *                                okvis_frontend/include/okvis/VioKeyframeWindowMatchingAlgorithm.hpp:246-254
 *   okb_track_3d2d_batch      <- the 3D-2D rounds of Frontend::matchToKeyframes / matchToLastFrame (Frontend.cpp:389-411,
 *                                484-494): VioKeyframeWindowMatchingAlgorithm::doSetup + DenseMatcher::match + setBestMatch
 *   okb_stereo_init_batch     <- the 2D-2D match of Frontend::matchStereo (Frontend.cpp:521-546): doSetup + DenseMatcher::
 *                                match + setBestMatch's device half (stereoTriangulate, getUncertainty)
 *   okb_match2d2d_batch       <- the 2D-2D rounds of Frontend::matchToKeyframes / matchToLastFrame (Frontend.cpp:413-452,
 *                                499-509): the same, between an older frame and the current one
 *   okb_keyframe_overlap_batch<- Frontend::doWeNeedANewKeyframe (Frontend.cpp:295-369): cv::convexHull, contourArea and
 *                                pointPolygonTest over the current frame's keypoints, for many sessions in one launch
 *   okb_ransac_3d2d_batch     <- Frontend::runRansac3d2d (Frontend.cpp:575-642): FrameNoncentralAbsoluteAdapter's
 *                                correspondences, FrameAbsolutePoseSacProblem's score; own sampler and generalised P3P
 *   okb_ransac_2d2d_batch     <- Frontend::runRansac2d2d (Frontend.cpp:645-810): FrameRelativeAdapter's correspondences,
 *                                FrameRotationOnly / FrameRelativePoseSacProblem's scores, the decision, outliers and pose
 *                                initialisation; own sampler, two-point rotation and five-point solvers
 *   okb_detect_describe       <- okvis::Frontend::detectAndDescribe    okvis_frontend/src/Frontend.cpp:92-114
 *                                (Frame::detect / Frame::describe      okvis_cv/include/okvis/implementation/Frame.hpp:109-156)
 *   okb_detect_describe_store_batch <- the same for every camera of many sessions' frames, written straight into the
 *                                windows' feature stores
 */
#ifndef OKVIS_B200_H_
#define OKVIS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ status */
typedef enum {
  OKB_OK = 0,
  OKB_ERR_INVALID_ARG = -1,
  OKB_ERR_CUDA = -2,          /* a CUDA runtime call failed; see okb_last_error */
  OKB_ERR_UNSUPPORTED = -3,   /* e.g. non-fixed extrinsics in the device solver */
  OKB_ERR_CAPACITY = -4,      /* window larger than the compiled-in limits */
  OKB_ERR_NO_DEVICE = -5,
  OKB_ERR_NUMERIC = -6,       /* solver failure (all windows report in summary) */
  OKB_ERR_SHARD_TIMEOUT = -7  /* a peer rank of a landmark-sharded window did not arrive at an exchange (status 7) */
} okb_status;

/* --------------------------------------------------------------- basic PODs */

/* Distortion model ids follow okvis_cv/include/okvis/cameras/ (the four Distortion headers) */
enum { OKB_DIST_NONE = 0, OKB_DIST_RADTAN = 1, OKB_DIST_EQUIDISTANT = 2, OKB_DIST_RADTAN8 = 3 };

/* PinholeCamera<DISTORTION>: fu,fv,cu,cv + distortion coefficients
 * (okvis_cv/include/okvis/cameras/PinholeCamera.hpp:60-110). */
typedef struct okb_camera {
  int32_t model;
  int32_t width, height;
  int32_t _pad;
  double fu, fv, cu, cv;
  double dist[8];
} okb_camera;

/* One ReprojectionError residual block (okvis_ceres/include/okvis/implementation/Estimator.hpp:43-90):
 * parameter blocks (pose[pose_idx], landmark[lm_idx], extrinsics[ext_idx]); measurement z (pixels);
 * information = sqrt_info^2 * I2 (sqrt_info = 8/keypoint size); CauchyLoss(1) always attached. */
typedef struct okb_observation {
  uint32_t pose_idx, lm_idx, ext_idx, cam_idx;
  double z[2];
  double sqrt_info;
} okb_observation;

/* okvis::ImuMeasurement with the time stamp as int64 nanoseconds
 * (okvis_common/include/okvis/Measurements.hpp; Time::toSec = sec + 1e-9 nsec). */
typedef struct okb_imu_sample {
  int64_t t_ns;
  double gyro[3];
  double acc[3];
} okb_imu_sample;

/* okvis::ImuParameters (okvis_common/include/okvis/Parameters.hpp:105-120), numeric part. */
typedef struct okb_imu_params {
  double a_max, g_max;
  double sigma_g_c, sigma_a_c;
  double sigma_bg, sigma_ba;
  double sigma_gw_c, sigma_aw_c;
  double tau, g;
  double a0[3];
  int32_t rate;
  int32_t _pad;
} okb_imu_params;

/* One ImuError residual block (okvis_ceres/src/Estimator.cpp:288-306): parameter blocks
 * (pose0, sb0, pose1, sb1); samples [sample_offset, sample_offset+sample_count) of the window's
 * sample array cover [t0,t1] including one sample before t0 and one after t1. */
typedef struct okb_imu_term {
  uint32_t pose0, sb0, pose1, sb1;
  int64_t t0_ns, t1_ns;
  uint32_t sample_offset, sample_count;
} okb_imu_term;

/* PoseError on a T_WS block (okvis_ceres/src/PoseError.cpp:48-136).  sqrt_info is the 6x6
 * (row-major) matrix the reference obtains as LLT(information).matrixL().transpose(); the caller
 * supplies it explicitly because the reference's first-frame prior is singular (SURVEY 8a item 8). */
typedef struct okb_pose_prior {
  uint32_t pose_idx;
  uint32_t _pad;
  double meas[7];          /* [t, q_xyzw] */
  double sqrt_info[36];
} okb_pose_prior;

/* SpeedAndBiasError (okvis_ceres/src/SpeedAndBiasError.cpp:46-116). */
typedef struct okb_sb_prior {
  uint32_t sb_idx;
  uint32_t _pad;
  double meas[9];
  double sqrt_info[81];
} okb_sb_prior;

/* RelativePoseError between two extrinsics blocks (okvis_ceres/src/RelativePoseError.cpp:47-162). */
typedef struct okb_relpose_term {
  uint32_t ext0, ext1;
  double sqrt_info[36];
} okb_relpose_term;

/* Block kinds referenced by the marginalisation prior. */
enum { OKB_BLOCK_POSE = 0, OKB_BLOCK_SPEED_BIAS = 1, OKB_BLOCK_EXTRINSICS = 2 };

/* The linearised prior produced by MarginalizationError::updateErrorComputation
 * (okvis_ceres/src/MarginalizationError.cpp:806-846): e = e0 + J * DeltaChi, J is n x n row-major,
 * DeltaChi stacks minus(x0_i, x_i) of the connected blocks in list order (fixed blocks contribute
 * no columns).  x0 holds the linearisation points, 7 / 9 / 7 doubles per block, concatenated. */
typedef struct okb_marg_prior {
  int32_t n;               /* residual dimension = sum of minimal dims */
  int32_t n_blocks;
  const int32_t* block_kind;   /* [n_blocks] OKB_BLOCK_* */
  const uint32_t* block_idx;   /* [n_blocks] index into poses / speed_bias / extrinsics */
  const double* x0;            /* concatenated linearisation points */
  const double* J;             /* [n][n] row-major */
  const double* e0;            /* [n] */
} okb_marg_prior;

/* A whole keyframe window = what okvis::ceres::Map holds when optimize() is called. */
typedef struct okb_window_desc {
  int32_t n_poses, n_speed_bias, n_extrinsics, n_landmarks;
  int32_t n_cameras, n_obs, n_imu_terms, n_imu_samples;
  int32_t n_pose_priors, n_sb_priors, n_relpose_terms, _pad;
  const double* poses;            /* [n_poses][7]       [t, q_xyzw] (PoseParameterBlock.cpp:68-79) */
  const double* speed_bias;       /* [n_speed_bias][9]  [v_W, b_g, b_a] */
  const double* extrinsics;       /* [n_extrinsics][7]  T_SC */
  const uint8_t* extrinsics_fixed;/* [n_extrinsics] 1 = setParameterBlockConstant (Estimator.cpp:264-267) */
  const double* landmarks;        /* [n_landmarks][4]   homogeneous, w untouched by updates */
  const okb_camera* cameras;      /* [n_cameras] */
  const okb_observation* obs;     /* [n_obs] */
  const okb_imu_term* imu_terms;  /* [n_imu_terms] */
  const okb_imu_sample* imu_samples; /* [n_imu_samples] */
  okb_imu_params imu_params;
  const okb_pose_prior* pose_priors;
  const okb_sb_prior* sb_priors;
  const okb_relpose_term* relpose_terms;
  const okb_marg_prior* marg;     /* NULL if no marginalisation prior */
} okb_window_desc;

/* Solver options = the Ceres 1.9 options Estimator::optimize sets (Estimator.cpp:854-874)
 * plus the time-limit callback (Estimator.cpp:909-929, CeresIterationCallback.hpp:78-87). */
typedef struct okb_solve_options {
  int32_t max_iterations;      /* numIter */
  int32_t min_iterations;      /* CeresIterationCallback::iterationMinimum_ */
  double time_limit_s;         /* <0: no limit */
  int32_t use_cauchy_loss;     /* 1 = CauchyLoss(1) on reprojection blocks (reference default) */
  int32_t _pad;
} okb_solve_options;

/* Per-window result summary (subset of ceres::Solver::Summary). */
enum { OKB_TERM_NO_CONVERGENCE = 0, OKB_TERM_FUNCTION_TOL = 1, OKB_TERM_PARAMETER_TOL = 2,
       OKB_TERM_GRADIENT_TOL = 3, OKB_TERM_MIN_RADIUS = 4, OKB_TERM_TIME_LIMIT = 5,
       OKB_TERM_FAILURE = 6 };
typedef struct okb_summary {
  double initial_cost, final_cost;
  int32_t iterations;          /* accepted + rejected steps, as Ceres counts them */
  int32_t num_successful_steps;
  int32_t termination;
  int32_t imu_redo_count;
  double final_radius;
  double solve_time_s;         /* device time for this optimize call (whole batch) */
} okb_summary;

/* ------------------------------------------------------------ estimator path */
typedef struct okb_ctx okb_ctx;

/* Creates a context on CUDA device `device_id` able to hold `max_windows` resident windows. */
int okb_ctx_create(int device_id, int max_windows, okb_ctx** out);
void okb_ctx_destroy(okb_ctx* ctx);
const char* okb_last_error(const okb_ctx* ctx);   /* ctx may be NULL: returns the creation error */
/* Number of kernels this library has launched on this context since creation. */
int64_t okb_kernel_launches(const okb_ctx* ctx);
/* Raw CUDA stream (cudaStream_t) the context launches on, for event timing by the caller. */
void* okb_stream(const okb_ctx* ctx);

/* Packs and uploads one window into slot `win` (0 <= win < max_windows).  The library stores landmarks internally
 * sorted by observing-frame range; indices and results at this boundary always use the caller's order.  A slot must
 * not be uploaded while an okb_optimize_async on it is still in flight (call okb_optimize_finish first). */
int okb_window_upload(okb_ctx* ctx, int win, const okb_window_desc* desc);
/* Batched form of okb_window_upload (no reference counterpart: one okvis::Estimator owns one window; this serves
 * callers that keep many estimators / sessions on one GPU).  Uploads `count` windows into slots
 * [win_first, win_first+count); descs[i] describes slot win_first+i.
 * The packing of different slots is spread over up to `host_threads` host threads (<= 0: library default).
 * Uploads run on the context's transfer stream: they overlap solver work already launched on OTHER
 * slots, and every later okb_optimize* / okb_window_reset is ordered after them.  Uploads of different slots
 * may also be issued concurrently from several caller threads. */
int okb_window_upload_batch(okb_ctx* ctx, int win_first, int count, const okb_window_desc* descs, int host_threads);
/* ---- resident window: incremental graph updates -------------------------------------------------------------
 * Replace the reference's graph bookkeeping between two optimize() calls -- Estimator::addStates
 * (okvis_ceres/src/Estimator.cpp:110-343), addLandmark (:346-368), addObservation
 * (include/okvis/implementation/Estimator.hpp:43-90), removeObservation (Estimator.cpp:371-413), set_T_WS /
 * setSpeedAndBias / setLandmark (include/okvis/Estimator.hpp:343-409) and the frame / landmark removal part of
 * applyMarginalizationStrategy (Estimator.cpp:434-773) -- so that a window stays resident on the device and only
 * one frame's worth of data crosses PCIe per optimize.  Every call appends a command to the slot's pending stream
 * on the host (no device work); okb_window_commit -- or the next okb_optimize* / okb_window_download* /
 * okb_window_reset of the slot -- ships the stream with one copy and the device applies the commands in order and
 * re-compiles its internal layout.  Index conventions: pose / speed-bias indices are positions in the window
 * (removing position p moves every later frame down by one, exactly like erasing from the reference's ordered
 * statesMap_); landmark indices are stable slots chosen by the caller (0 <= idx < max_landmarks).
 * Indices are validated on the host against the mirrored dimensions (OKB_ERR_INVALID_ARG / OKB_ERR_CAPACITY
 * synchronously); duplicate observations and inconsistent extrinsics are detected by the device and reported by
 * the next okb_optimize_finish / okb_optimize. */

/* Capacities of slot `win` for later incremental growth; call before okb_window_upload of that slot (an upload
 * larger than the reservation simply enlarges it).  max_marg_dim <= 160. */
int okb_window_reserve(okb_ctx* ctx, int win, int max_frames, int max_landmarks, int max_observations,
                       int max_imu_samples, int max_marg_dim);
/* Appends one frame: pose (index n_poses), optionally its speed/bias block (index n_speed_bias; NULL: none) and the
 * ImuError term that links it (Estimator.cpp:288-306; NULL: none).  term->pose0/sb0/pose1/sb1 index the window
 * AFTER the append; term->sample_offset is relative to `samples`. */
int okb_window_add_frame(okb_ctx* ctx, int win, const double* pose /*7*/, const double* speed_bias /*9 or NULL*/,
                         const okb_imu_term* term, const okb_imu_sample* samples, int n_samples);
/* Removes a frame: its pose block, speed/bias block sb_idx (0xffffffff: none), every observation made in it, the IMU
 * terms and priors attached to it.  Later frames move down one position everywhere (observations, IMU terms,
 * priors, marginalisation-prior block list; a prior that still references the removed frame is an error). */
int okb_window_remove_frame(okb_ctx* ctx, int win, uint32_t pose_idx, uint32_t sb_idx);
/* Creates or overwrites landmark slots (Estimator::addLandmark / setLandmark). */
int okb_window_set_landmarks(okb_ctx* ctx, int win, int n, const uint32_t* idx, const double* xyzw /*[n][4]*/);
/* Removes landmarks and all their observations (Estimator::removeObservation loop of Estimator.cpp:625-725). */
int okb_window_remove_landmarks(okb_ctx* ctx, int win, int n, const uint32_t* idx);
int okb_window_add_observations(okb_ctx* ctx, int win, int n, const okb_observation* obs);
typedef struct okb_obs_key { uint32_t pose_idx, lm_idx, cam_idx, _pad; } okb_obs_key;
/* Estimator::removeObservation(landmarkId, poseId, camIdx, keypointIdx) (Estimator.cpp:371-413); unknown keys are ignored. */
int okb_window_remove_observations(okb_ctx* ctx, int win, int n, const okb_obs_key* keys);
/* Estimator::set_T_WS / setSpeedAndBias. */
int okb_window_set_states(okb_ctx* ctx, int win, int n_poses, const uint32_t* pose_idx, const double* poses /*[n][7]*/,
                          int n_sb, const uint32_t* sb_idx, const double* speed_bias /*[n][9]*/);
/* Replaces the pose priors and speed/bias priors; marg != NULL also replaces the marginalisation prior
 * (marg->n == 0 removes it), marg == NULL keeps the current one. */
int okb_window_set_priors(okb_ctx* ctx, int win, int n_pose_priors, const okb_pose_prior* pose_priors, int n_sb_priors,
                          const okb_sb_prior* sb_priors, const okb_marg_prior* marg);
/* Ships the pending commands of slots [win_first, win_first+count) to the device (transfer stream; overlaps solver
 * work on other slots).  Optional: the calls that need the result do it themselves.  On a landmark-sharded context it
 * returns once the commands are applied on the device, and is NOT optional after edits: every rank commits before any
 * rank's okb_optimize*, so that no rank's graph update still queues while its peers' solvers wait on the exchange. */
int okb_window_commit(okb_ctx* ctx, int win_first, int count);

/* Removes speed/bias block sb_idx together with the ImuError terms and SpeedAndBiasError priors attached to it; the
 * pose of that frame stays (the "removeAllButPose" frames of Estimator::applyMarginalizationStrategy,
 * Estimator.cpp:483-554).  Later speed/bias blocks move down one position. */
int okb_window_remove_speed_bias(okb_ctx* ctx, int win, uint32_t sb_idx);

/* ---- device-side marginalisation -----------------------------------------------------------------------------
 * The numeric half of Estimator::applyMarginalizationStrategy (okvis_ceres/src/Estimator.cpp:434-773):
 * MarginalizationError::addResidualBlock (okvis_ceres/src/MarginalizationError.cpp:127-435) for the listed residual
 * blocks -- evaluated at the first-estimate linearisation points, reprojection errors with the Cauchy correction --
 * marginalizeOut (:507-802) of the marked blocks and of the listed landmarks, and updateErrorComputation (:806-846).
 * The window's marginalisation prior is replaced on the device by the result (kept blocks in job order; their
 * linearisation points are kept when block_prev >= 0, else the current estimates become x0).  The bookkeeping half
 * stays with the caller, exactly like the reference: after this call it removes the linearised terms / blocks with
 * okb_window_remove_frame / okb_window_remove_speed_bias / okb_window_remove_landmarks and re-fixes the first pose
 * with okb_window_set_priors (Estimator.cpp:761-770).  H and b0 persist on the device between calls as the
 * reference's H_ / b0_ members do (a prior supplied by the host through okb_window_upload / okb_window_set_priors
 * starts from H = J^T J, b0 = -J^T e0).  Errors found by the device (a residual whose parameter blocks are not all
 * listed, inconsistent block_prev) surface at the next okb_optimize* / okb_window_download_marg. */
typedef struct okb_marg_job {
  int32_t n_blocks;                 /* dense parameter blocks of the linear system, in H order (<= 64) */
  int32_t n_imu_terms, n_sb_priors, n_landmarks;
  const int32_t* block_kind;        /* [n_blocks] OKB_BLOCK_POSE / OKB_BLOCK_SPEED_BIAS */
  const uint32_t* block_idx;        /* [n_blocks] position in the window NOW */
  const int32_t* block_prev;        /* [n_blocks] position in the current prior's block list, -1 = newly connected; every
                                       block of the current prior must appear exactly once */
  const uint8_t* block_marginalize; /* [n_blocks] 1 = marginalise this block out */
  const uint32_t* imu_terms;        /* ImuError terms to linearise (positions in the window's term list) */
  const uint32_t* sb_priors;        /* SpeedAndBiasError terms to linearise */
  const uint32_t* landmarks;        /* landmarks to marginalise: every observation they still have is linearised */
} okb_marg_job;
/* Landmark-sharded windows (okb_shard_*, below): EVERY rank calls okb_window_marginalize* on the window, with the same
 * dense part of the job (block lists, IMU terms, speed/bias priors) and, in `landmarks`, only the marginalised
 * landmarks it holds, as local slots (global slot g lives on rank g % world at local slot g / world).  A rank that
 * holds none of them still calls, with n_landmarks = 0.  Each rank linearises its own landmarks; their Schur terms are
 * summed over the ranks through the shard mailbox in rank order, so the new prior -- J, e0, H / b0, block list, x0,
 * status -- is bit-identical on all ranks.  The calls of all ranks may be issued from one host thread in rank order:
 * no host wait inside the call depends on the peers (buffers the context outgrows are kept until it is destroyed).
 * Device statuses beyond those of an unsharded window (download_marg status[0]):
 *   6 (shard job)     the ranks' dense parts differ (okb_marg_job_fingerprint);
 *   7 (shard timeout) a peer did not arrive within 4 s, or pushed a box of another exchange epoch;
 * and a device error of any one rank (status 1-5, below) is reported by every rank.  A rank reporting any of these
 * abandons the step before the dense marginalisation: its previous prior stays in place, and its next okb_optimize*
 * fails until a full upload.  Statuses 6 and 1-5 are seen by every rank alike; a time-out only by the ranks that timed
 * out (a peer arriving later completes the step), after which the ranks are out of step and the shard contexts must be
 * recreated.  ImuError caches the step had already re-preintegrated keep their new state, as the
 * reference's functor cache does after any evaluation.  Status codes of any window: 1 bad block list, 2 block_prev
 * inconsistent with the current prior, 3 a listed term's blocks are not all listed, 4 a marginalised landmark is
 * observed in a frame that is not listed, 5 dimension mismatch. */
int okb_window_marginalize(okb_ctx* ctx, int win, const okb_marg_job* job);
/* The 64-bit hash landmark-sharded ranks compare before summing: N, the kept dimension, the block lists and the
 * IMU-term / speed/bias-prior lists of `job` (not its landmarks). */
int okb_marg_job_fingerprint(const okb_marg_job* job, uint64_t* out);
/* Batched okb_window_marginalize (no reference counterpart; serves hosts that keep many estimators on one GPU).
 * jobs[i] describes slot win_first+i; jobs[i] == NULL: that slot is not touched (no commit, no wait on its solve, no
 * copy), so its okb_optimize_async may still be running.  Each slot's result -- prior, H / b0, block list, x0, ImuError
 * caches, download_marg status -- is bit-identical to okb_window_marginalize on it.  Every job is checked on the host
 * before any device work: the first failure returns its status, names the slot in okb_last_error and leaves every
 * slot unchanged.  count < 1 or a range outside max_windows: OKB_ERR_INVALID_ARG; all jobs NULL: no-op.  Pending
 * edits of the job slots are committed first; one k_marginalize launch (one CTA per job) then runs on the transfer
 * stream after the solver work already launched on the job slots only, and later calls on those slots are ordered
 * after it.  Errors the device finds stay with their slot and surface as for the single call.  On a landmark-sharded
 * context every rank calls with the same slots, one exchange per slot, under the contract of okb_window_marginalize.
 * Each job occupies one SM while it waits for its peers: ranks that share one device need the sum of their jobs per
 * call to stay at most the device's SM count. */
int okb_window_marginalize_batch(okb_ctx* ctx, int win_first, int count, const okb_marg_job* const* jobs);
/* Reads the window's current marginalisation prior back (tests, host-side persistence): J [n][n], e0 [n], the
 * H / b0 it was factored from, block list, linearisation points.  Any pointer may be NULL; arrays must hold the
 * compiled-in maxima (n <= 160, 64 blocks).  status[4] = {device error code of the last okb_window_marginalize,
 * rank of H, rank of the dense marginalised block, Jacobi sweeps: the larger count of the dense block's and the final H's
 * eigen-decompositions, 40 if either stopped at its sweep cap without converging}. */
int okb_window_download_marg(okb_ctx* ctx, int win, int32_t* n, int32_t* n_blocks, int32_t* block_kind, uint32_t* block_idx,
                             double* x0, double* J, double* e0, double* H, double* b0, int32_t* status);

/* Bytes the last commit (full upload or incremental commands) of this slot copied host -> device (0 if the slot is empty). */
int64_t okb_window_h2d_bytes(const okb_ctx* ctx, int win);
/* Restores the state of the last FULL upload of the slot on the device (no host traffic); used to repeat a solve
 * on resident data.  The window must have the shape (frames, landmarks) it had at that upload. */
int okb_window_reset(okb_ctx* ctx, int win_first, int win_count);
/* Runs the dogleg/Schur solver on windows [win_first, win_first+win_count) in one batch.
 * summaries may be NULL; otherwise [win_count]. */
int okb_optimize(okb_ctx* ctx, int win_first, int win_count, const okb_solve_options* opt,
                 okb_summary* summaries);
/* Same as okb_optimize but does not synchronise or read anything back (for device-side timing);
 * call okb_optimize_finish to collect the summaries.  The context keeps the slot tables of the last 8 launch
 * sequences (each okb_optimize*_async, and each extra round okb_optimize*_finish launches): a 9th waits on the host
 * until the oldest of them has finished on the device. */
int okb_optimize_async(okb_ctx* ctx, int win_first, int win_count, const okb_solve_options* opt);
int okb_optimize_finish(okb_ctx* ctx, int win_first, int win_count, okb_summary* summaries);
/* Runs the solver on the n listed slots in one batch (no reference counterpart; serves hosts that keep many
 * sessions on one GPU and rarely have a contiguous run of them ready at once).  slots[i] are distinct, uploaded
 * slots, in any order; summaries [n] come back in list order (may be NULL).  Per slot the result -- summary,
 * estimates, quality, ImuError caches -- is bit-identical to okb_optimize over a contiguous range that holds the same
 * windows in the same order (the landmark chunking depends on the batch size).  Slots not listed are not committed,
 * waited for, read or written; pending edits of the listed slots are committed once per run of consecutive slots.
 * n < 1, a NULL pointer, a slot out of range, not uploaded or listed twice: OKB_ERR_INVALID_ARG; a landmark-sharded
 * context: OKB_ERR_UNSUPPORTED (sharded windows use okb_optimize); both before any device work.
 * The _async / _finish pair splits the call as okb_optimize_async / okb_optimize_finish do (including the host wait
 * beyond 8 launch sequences in flight); _finish takes the same list. */
int okb_optimize_slots(okb_ctx* ctx, int n, const int32_t* slots, const okb_solve_options* opt, okb_summary* summaries);
int okb_optimize_slots_async(okb_ctx* ctx, int n, const int32_t* slots, const okb_solve_options* opt);
int okb_optimize_slots_finish(okb_ctx* ctx, int n, const int32_t* slots, okb_summary* summaries);
/* Window groups of the batched solve.  A batch is split into groups of consecutive batch positions (sizes differing
 * by at most one), each solved on its own stream and started behind the previous one, so that the latency-bound
 * reduced solve of one group overlaps the landmark kernels of another.  Results are bit-identical for any group count.
 * n = 0 (the default) chooses 4 groups for a batch of at least as many windows as the device has SMs, else one;
 * n = 1..4 forces n groups (at most one per window) for every later okb_optimize* call.  Landmark-sharded contexts
 * always solve in one group.  Other n: OKB_ERR_INVALID_ARG. */
int okb_set_solve_groups(okb_ctx* ctx, int n);
/* Copies the estimates back.  Any pointer may be NULL.  quality[l] = sqrt(lambda_min)/sqrt(lambda_max)
 * of the landmark's 3x3 Hessian block as in Estimator.cpp:880-894 (0 if lambda_min < 1e-12). */
int okb_window_download(okb_ctx* ctx, int win, double* poses, double* speed_bias,
                        double* landmarks, double* quality);
/* Batched form of okb_window_download (no reference counterpart).  Downloads the estimates of `count` slots with one
 * synchronisation.  Each argument is an array of `count`
 * host pointers (or NULL to skip that quantity; individual entries may be NULL too).  Like the uploads this
 * runs on the transfer stream: it waits only for solver work launched on these slots, not for other slots. */
int okb_window_download_batch(okb_ctx* ctx, int win_first, int count, double* const* poses,
                              double* const* speed_bias, double* const* landmarks, double* const* quality);
/* List form of okb_window_download_batch (no reference counterpart; serves hosts whose ready sessions are scattered
 * over the slots).  slots[i] are distinct, uploaded slots in any order; the pointer tables are in list order, with NULL
 * tables or entries allowed as there.  Only the listed slots are touched: their pending edits are committed once per
 * run of consecutive slots, only their solver work is waited for, one D2H copy per slot and one synchronisation.
 * Each slot's outputs are byte-identical to okb_window_download on it.  List errors are those of okb_optimize_slots
 * (OKB_ERR_INVALID_ARG naming the entry, OKB_ERR_UNSUPPORTED on a landmark-sharded context), before any device work. */
int okb_window_download_slots(okb_ctx* ctx, int n, const int32_t* slots, double* const* poses,
                              double* const* speed_bias, double* const* landmarks, double* const* quality);

/* ----------------------------------------------------- landmark-sharded single window (multi-GPU)
 * No reference counterpart (the reference is single-process CPU code); this is the partition SURVEY.md 8(e) row 2 /
 * BASELINE.json configs[4] name: the landmarks (and their observations) of ONE large window are dealt to `world`
 * ranks (lm_idx mod world), every rank holds all poses / speed-bias / IMU / prior blocks.  Per solver round each
 * rank builds the Schur complement of its shard, the partial reduced systems are all-reduced over NVLink peer
 * memory (push into every rank's mailbox + flags, fused into the chunk-reduction kernel and the reduced-solve
 * kernel's prologue), every rank solves the reduced system redundantly and back-substitutes its own landmarks.
 * A context is made a shard member BEFORE its windows are uploaded; every rank then uploads its shard into the
 * same slot and all ranks issue the same okb_optimize* calls.  time_limit_s uses rank 0's clock.
 *   multi-process (one process per GPU): okb_shard_export on every rank, exchange the OKB_SHARD_HANDLE_BYTES-byte
 *     handles out of band (e.g. torch.distributed.all_gather), okb_shard_connect with all `world` handles in rank order.
 *   single process driving several contexts (same or different devices): okb_shard_connect_local.
 * max_frames bounds the keyframes of any sharded window (mailbox sizing).
 *
 * The frontend calls on the feature store (okb_detect_describe_store_batch, okb_track_3d2d_batch, okb_match2d2d_batch,
 * okb_stereo_init_batch, okb_keyframe_overlap_batch, okb_ransac_3d2d_batch, okb_ransac_2d2d_batch) run on a sharded
 * window when the context
 * reserved its global landmark slots with okb_shard_reserve_landmarks before okb_shard_export / okb_shard_connect_local
 * (otherwise they return OKB_ERR_UNSUPPORTED).  The feature store is replicated: every rank reserves it and receives
 * the same store edits (okb_window_reserve_features, okb_window_set_features, okb_window_set_feature_landmarks,
 * okb_window_clear_features), whose landmark slots are GLOBAL slots below max_landmarks.  okb_window_set_landmark_-
 * initialized is landmark state and goes to the owner (rank g mod world) at its local slot g div world, as
 * okb_window_set_landmarks does.  Every rank makes the same call with the same arguments, concurrently (one host thread
 * or process per rank: the calls return only after their device work); track, 2D-2D, stereo initialisation and RANSAC
 * 3D-2D first all-gather the landmark state they read (point, observation count, initialised flag; 40 bytes per global
 * slot, double-buffered) over the mailbox, and return OKB_ERR_SHARD_TIMEOUT (status 7) if a peer does not arrive
 * within the solver's time-out.  Every rank returns the same results as an unsharded context holding the whole
 * window; landmark slots in them are global, and edits derived from them are routed like any other.  A landmark
 * removed on its owner is forgotten by every rank's store at the next exchange. */
#define OKB_SHARD_HANDLE_BYTES 64
/* Global landmark slots of the frontend's landmark replica (0: none, the default); before okb_shard_export /
 * okb_shard_connect_local.  Adds 2 * 40 * max_landmarks bytes to each window's mailbox on every rank. */
int okb_shard_reserve_landmarks(okb_ctx* ctx, int max_landmarks);
/* Mailbox bytes of one window slot on every rank (no context needed): out[0] = offset of the landmark replica,
 * out[1] = its bytes (2 * 40 * max_landmarks), out[2] = the slot's whole mailbox (256-byte aligned). */
int okb_shard_mailbox_layout(int world, int max_frames, int max_landmarks, uint64_t out[3]);
int okb_shard_export(okb_ctx* ctx, int rank, int world, int max_frames, void* handle_out /* OKB_SHARD_HANDLE_BYTES */);
int okb_shard_connect(okb_ctx* ctx, const void* handles /* [world][OKB_SHARD_HANDLE_BYTES] */);
int okb_shard_connect_local(okb_ctx* const* ctxs /* [world], rank order */, int world, int max_frames);
/* After okb_optimize_finish: out[0] = exchange rounds of the last optimize of `win`, out[1] = microseconds this rank
 * spent waiting for and summing the peers' partial systems (device clock), out[2] = 1 if a peer timed out,
 * out[3] = exchange epoch. */
int okb_shard_stats(okb_ctx* ctx, int win, double out[4]);

/* Optional per-kernel device timing: CUDA events on the context stream around every solver kernel
 * launch.  okb_profile_enable(ctx,1) clears the counters; okb_profile_read synchronises and returns
 * out[0] = ms in k_landmarks, out[1] = its launches, out[2] = ms in k_solve, out[3] = launches,
 * out[4] = ms in k_quality, out[5] = launches.  A solve in several window groups (okb_set_solve_groups) counts each
 * round once, and times it from the earliest group's start of the kernels to the latest group's end; the groups run
 * at the same time, so that span also holds other kernels of the other groups and the times are approximate. */
int okb_profile_enable(okb_ctx* ctx, int on);
int okb_profile_read(okb_ctx* ctx, double out[6]);
/* Diagnostics: nanoseconds the reduced-solve kernel spent per internal phase during the last optimize of
 * `win` (dense terms, partial gather, assembly, Cholesky, substitution, back-substitution, dogleg). */
int okb_debug_phase_ns(okb_ctx* ctx, int win, double out[16]);
/* Diagnostics: the Schur-complement kernel's launch shape for an optimize of slots [first, first+count):
 * out[0] = 1 if its accumulators live in shared memory (0: in global memory), out[1] = threads per CTA (256: two
 * CTAs per SM, 512: one), out[2] = dynamic shared memory per CTA in bytes. */
int okb_debug_schur_plan(okb_ctx* ctx, int first, int count, int32_t out[3]);
/* Diagnostics: the mutable preintegration cache of ImuError term `term` (ImuError.hpp:251-276): the bias the
 * preintegration was done at, whether it is valid (0 = redo_), and how often it was redone. */
int okb_debug_imu_cache(okb_ctx* ctx, int win, int term, double sb_ref[9], int32_t* valid, int32_t* redo_count);
/* Diagnostics: what the window's last solver round evaluated for IMU terms [first_term, first_term + n_terms), as
 * OKB_IMU_TERM_OUT doubles per term: the term's 30x30 block J^T J (row-major; J = [J0 J1 J2 J3], the four minimal
 * Jacobians side by side: pose0, speed/bias0, pose1, speed/bias1), then J^T r (30), then the cost 0.5 |r|^2.  After
 * okb_optimize with max_iterations = 0 that is the linearisation at the window's state.  Waits for the solver, commits
 * nothing and launches nothing: after an edit (pending or committed) the output is stale, in the old term numbering,
 * until the next optimize.  A range outside the window's current terms or a NULL `out`: OKB_ERR_INVALID_ARG. */
#define OKB_IMU_TERM_OUT 931
int okb_debug_imu_terms(okb_ctx* ctx, int win, int first_term, int n_terms, double* out);

/* ------------------------------------------------- single-block test hooks
 * Mirror ErrorInterface::EvaluateWithMinimalJacobians (okvis_ceres/include/okvis/ceres/ErrorInterface.hpp:93-95).
 * All run on the device through the same device functions the solver uses.  Jacobians are the
 * MINIMAL ones, row-major.  n = batch size; arrays are [n][...]. */
int okb_eval_reprojection(okb_ctx* ctx, int n, const okb_camera* cam, const double* pose /*[n][7]*/,
                          const double* landmark /*[n][4]*/, const double* extrinsics /*[n][7]*/,
                          const double* z /*[n][2]*/, const double* sqrt_info /*[n]*/,
                          double* r /*[n][2]*/, double* J_pose /*[n][12]*/, double* J_lm /*[n][6]*/,
                          double* J_ext /*[n][12]*/);
int okb_eval_imu(okb_ctx* ctx, const okb_imu_params* params, const okb_imu_sample* samples, int n_samples,
                 int64_t t0_ns, int64_t t1_ns, const double* pose0, const double* sb0,
                 const double* pose1, const double* sb1, const double* sb_ref /* linearisation point or NULL */,
                 double* r /*15*/, double* J0 /*15x6*/, double* J1 /*15x9*/, double* J2 /*15x6*/,
                 double* J3 /*15x9*/, double* sqrt_info_out /*15x15 or NULL*/);
int okb_imu_propagate(okb_ctx* ctx, const okb_imu_params* params, const okb_imu_sample* samples, int n_samples,
                      int64_t t0_ns, int64_t t1_ns, double* pose /*7 in/out*/, double* sb /*9 in/out*/,
                      double* covariance /*15x15 or NULL*/, double* jacobian /*15x15 or NULL*/, int* n_used);

/* One ImuError::propagation of a batch (one session's prediction). */
typedef struct okb_propagate_job {
  const okb_imu_params* params;        /* per job: sessions may have different IMUs */
  const okb_imu_sample* samples;       /* host, n_samples >= 2, as okb_imu_propagate */
  int32_t n_samples, _pad;
  int64_t t0_ns, t1_ns;
  double* pose;                        /* 7, in/out */
  double* speed_bias;                  /* 9, in/out */
  double* covariance;                  /* 15x15 or NULL */
  double* jacobian;                    /* 15x15 or NULL */
  int32_t* n_used;                     /* or NULL */
} okb_propagate_job;
/* Batched okb_imu_propagate (no reference counterpart; serves hosts that keep many sessions on one GPU and predict
 * all of them per camera frame or per IMU sample).  Each job's outputs -- pose, speed/bias, covariance, Jacobian,
 * n_used -- are bit-identical to okb_imu_propagate on the same arguments.  As there, a job whose samples end before
 * t1_ns gets n_used = -1 and its pose, speed/bias, covariance and Jacobian are left untouched; the call still returns
 * OKB_OK.  Every job is checked on the host before any device work, with the single call's checks: the first failure
 * returns OKB_ERR_INVALID_ARG, names the job index in okb_last_error and writes no job's outputs.  n_jobs == 0 is a
 * no-op; n_jobs < 0, or jobs == NULL with n_jobs > 0, is invalid.
 * Each call makes one H2D copy, one launch (one warp per job), one D2H copy and one synchronisation, whatever n_jobs
 * is.  It runs on a stream of its own at the context's greatest priority and is serialised only with other
 * propagation batches, so it never queues behind an okb_optimize_async, an okb_window_marginalize_batch or a frontend
 * batch on the context, and it may run beside the single-block hooks.  okb_imu_propagate itself stays on the solver
 * stream, ordered after solver work already launched.  Pinned and device buffers grow to the largest batch seen and
 * are kept; a call that has to grow them frees the old ones, which waits for all work on the device (an
 * okb_optimize_async in flight included).  Issue one batch of the largest size first to size them. */
int okb_imu_propagate_batch(okb_ctx* ctx, int n_jobs, const okb_propagate_job* jobs);
int okb_eval_pose_error(okb_ctx* ctx, const double* meas /*7*/, const double* sqrt_info /*36*/,
                        const double* pose /*7*/, double* r /*6*/, double* J /*6x6*/);
int okb_eval_speed_bias_error(okb_ctx* ctx, const double* meas /*9*/, const double* sqrt_info /*81*/,
                              const double* sb /*9*/, double* r /*9*/, double* J /*9x9*/);
int okb_eval_relative_pose(okb_ctx* ctx, const double* sqrt_info /*36*/, const double* pose0, const double* pose1,
                           double* r /*6*/, double* J0 /*6x6*/, double* J1 /*6x6*/);
/* x: current block values concatenated like marg->x0; J_eff is the n x n effective minimal Jacobian
 * after Ceres multiplies by the local parameterisation at x (J * lift(x0) * plus(x)). */
int okb_eval_marginalization(okb_ctx* ctx, const okb_marg_prior* marg, const double* x,
                             double* r /*n*/, double* J_eff /*n x n*/);

/* -------------------------------------------------------------- frontend path */
typedef struct okb_keypoint {      /* cv::KeyPoint fields the reference uses */
  float x, y;
  float size;
  float angle;                     /* degrees, set from the gravity direction (Frame.hpp(impl):128-156) */
  float response;
  int32_t octave;
} okb_keypoint;

/* brisk::ScaleSpaceFeatureDetector<HarrisScoreCalculator>(uniformityRadius, octaves=0,
 * absoluteThreshold, maxNumKpt) as constructed at okvis_frontend/src/Frontend.cpp:828-831. */
typedef struct okb_detect_params {
  double uniformity_radius;        /* "detection threshold" in the yaml (40) */
  double absolute_threshold;       /* 800 */
  int32_t max_keypoints;           /* 400 */
  int32_t desc_bytes;              /* 48 (reference) or 64 */
  int32_t rotation_invariance;     /* 1 */
  int32_t _pad;
} okb_detect_params;

int okb_detect_describe(okb_ctx* ctx, int cam_slot, const uint8_t* img, int width, int height, int stride,
                        const okb_camera* cam, const double R_CW[9], const okb_detect_params* params,
                        okb_keypoint* out_kp, uint8_t* out_desc, int max_out, int* n_out);

/* One camera image of a batch (Frontend::detectAndDescribe for one camera of one session). */
typedef struct okb_image_desc {
  const uint8_t* img;              /* host, row stride `stride` bytes */
  int32_t width, height, stride, _pad;
  okb_camera cam;                  /* geometry for the orientation (Frame::describe) */
  double R_CW[9];                  /* as okb_detect_describe */
} okb_image_desc;

/* n_images images (n_images <= 65535), one parameter set.  out_kp [n_images][max_out],
 * out_desc [n_images][max_out][desc_bytes], n_out [n_images].  Per image the result is bit-identical to
 * okb_detect_describe on that image.  Images may differ in size, stride, camera and R_CW.  An image with more NMS
 * candidates than the detector holds gets n_out = -1 and the call returns OKB_ERR_CAPACITY; every other image's
 * outputs are still written.  Arguments are checked per image before any device work (OKB_ERR_INVALID_ARG);
 * n_images == 0 is a no-op.  The batch runs on a stream of its own (not the solver's), blocks until done, and is
 * serialised with other batch calls on the context; it may run beside okb_detect_describe on the camera slots.
 * Device and pinned buffers grow to the largest batch seen and are kept; a call that has to grow them frees the old
 * ones, which waits for all work on the device (an okb_optimize_async in flight included).  Issue one batch of the
 * largest size first to size them.
 * host_threads: host packing threads (<= 0: library default), as okb_window_upload_batch. */
int okb_detect_describe_batch(okb_ctx* ctx, int n_images, const okb_image_desc* images, const okb_detect_params* params,
                              okb_keypoint* out_kp, uint8_t* out_desc, int max_out, int32_t* n_out, int host_threads);

typedef struct okb_pair {          /* DenseMatcher::Pairing */
  int32_t index_a;                 /* -1 = B element unmatched */
  float distance;
} okb_pair;

/* DenseMatcher::match with the plain Hamming MatchingAlgorithm: per-A top-`num_best` lists
 * (out_topk [nA][num_best], may be NULL), greedy mutual assignment in sequential A-ascending order,
 * per-B winners (out_pairs [nB]).  use_ratio / ratio_threshold mirror useDistanceRatioThreshold_.
 * nA == 0 or nB == 0 is legal (no matches: every out_pairs entry is {-1, threshold}), like DenseMatcher::match on an
 * empty MatchingAlgorithm; the same holds for the gated and the candidate-list calls. */
int okb_hamming_match(okb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes,
                      const uint8_t* skipA, const uint8_t* skipB, float threshold, int num_best,
                      int use_ratio, float ratio_threshold, okb_pair* out_topk, okb_pair* out_pairs);

/* ---- geometry-gated matching (SURVEY.md 8f row 2) --------------------------------------------------------------
 * VioKeyframeWindowMatchingAlgorithm::distance (okvis_frontend/include/okvis/VioKeyframeWindowMatchingAlgorithm.hpp:132-144)
 * returns the Hamming distance only if it is below the threshold AND verifyMatch passes
 * (okvis_frontend/src/VioKeyframeWindowMatchingAlgorithm.cpp:304-339), else FLT_MAX; the top-k lists and assignbest of
 * DenseMatcher then run over these gated distances.  okb_hamming_match_gated evaluates the gate on the device inside
 * the list kernel, so no candidate list has to travel back to the host.
 *   OKB_GATE_3D2D : chi-square test of landmark A's projection into frame B against keypoint B (:317-338);
 *                   proj_into_b / proj_uncertainty are what doSetup computes (:159-208)
 *   OKB_GATE_2D2D : ProbabilisticStereoTriangulator::stereoTriangulate (src/ProbabilisticStereoTriangulator.cpp:168-227):
 *                   triangulateFast (src/stereo_triangulation.cpp:51-125) of the two back-projected rays with
 *                   sigma = max(raySigmasA[a], raySigmasB[b]) and the two reprojection checks (:359-384).  The
 *                   bearing vectors are the cameras' backProject() of the keypoints (the caller has the camera
 *                   objects; the reference recomputes them inside every call). */
enum { OKB_GATE_NONE = 0, OKB_GATE_3D2D = 1, OKB_GATE_2D2D = 2 };
typedef struct okb_match_gate {
  int32_t mode, _pad;
  const double* kp_b;              /* [nB][2] keypoint coordinates in B (both modes) */
  const double* kp_size_b;         /* [nB]    keypoint size (both modes) */
  const double* proj_into_b;       /* 3D-2D: [nA][2] projectionsIntoB_ */
  const double* proj_uncertainty;  /* 3D-2D: [nA][4] projectionsIntoBUncertainties_, 2x2 row-major */
  const double* kp_a;              /* 2D-2D: [nA][2] */
  const double* kp_size_a;         /* 2D-2D: [nA] */
  const double* bearing_a;         /* 2D-2D: [nA][3] backProject(kp_a), camera A frame, any length */
  const double* bearing_b;         /* 2D-2D: [nB][3] backProject(kp_b), camera B frame */
  const double* ray_sigma_a;       /* 2D-2D: [nA] raySigmasA_ */
  const double* ray_sigma_b;       /* 2D-2D: [nB] raySigmasB_ */
  okb_camera cam_a, cam_b;         /* 2D-2D: geometries for the reprojection checks */
  double T_AB[7];                  /* 2D-2D: pose of camera B in camera A [t, q_xyzw] */
} okb_match_gate;
int okb_hamming_match_gated(okb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes,
                            const uint8_t* skipA, const uint8_t* skipB, float threshold, int num_best, int use_ratio,
                            float ratio_threshold, const okb_match_gate* gate, okb_pair* out_topk, okb_pair* out_pairs);

/* One DenseMatcher::match of a batch.  gate == NULL: plain Hamming (okb_hamming_match); else as
 * okb_hamming_match_gated.  use_ratio as there (the ratio test itself stays with the caller). */
typedef struct okb_match_job {
  const uint8_t *A, *B, *skipA, *skipB;   /* skip* may be NULL */
  int32_t nA, nB;
  float threshold;
  int32_t num_best, use_ratio, _pad;
  const okb_match_gate* gate;
  okb_pair* out_topk;                     /* [nA][num_best] or NULL */
  okb_pair* out_pairs;                    /* [nB] */
} okb_match_job;
/* n_jobs matches with one descriptor length.  Per job the outputs equal the single call's; plain, 3D-2D and 2D-2D
 * jobs may share a call, and jobs with nA == 0 or nB == 0 are answered on the host.  Arguments are checked per job
 * before any device work.  Runs on the batch stream (see okb_detect_describe_batch), blocking. */
int okb_hamming_match_batch(okb_ctx* ctx, int n_jobs, const okb_match_job* jobs, int desc_bytes);

/* Candidate-list mode for the production (geometry-gated) matching algorithm: for every A, every B
 * with Hamming distance < threshold in ascending B order, CSR layout.  row_ptr [nA+1];
 * col_idx / dist have capacity `cap`; returns OKB_ERR_CAPACITY if more candidates exist
 * (row_ptr[nA] then holds the required capacity). */
int okb_hamming_candidates(okb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes,
                           float threshold, uint32_t* row_ptr, uint32_t* col_idx, uint16_t* dist, int cap);

/* ---- per-window feature store and 3D-2D tracking ------------------------------------------------------------------
 * The keypoints, descriptors and keypoint -> landmark references of the frames of a resident window, kept on the device
 * so that tracking a new frame against its window (the 3D-2D matches of Frontend::matchToKeyframes, Frontend.cpp:389-411,
 * and of Frontend::matchToLastFrame, :484-494) needs no landmark download and no descriptor re-upload.
 * A window's store holds `max_feature_frames` FEATURE SLOTS -- stable indices the caller picks, like landmark slots, and
 * independent of window positions (okb_window_remove_frame never moves the store) -- with, per camera, up to
 * `max_keypoints` keypoints: position and size, descriptor, landmark slot (-1 = none) and an `observed` bit ("the window
 * holds this keypoint's observation").  It also holds one initialised flag per landmark slot (Estimator::
 * setLandmarkInitialized); a slot starts uninitialised and okb_window_remove_landmarks clears it, together with every
 * store reference to the removed slots.  The edit calls below append commands to the slot's pending stream (they
 * need an uploaded window) and are applied in order with the graph edits at commit; a full upload drops the graph edits
 * still pending but keeps the pending store edits, which follow it.  Full uploads and okb_window_reset leave the store
 * as it is.  okb_window_reserve_features allocates the store (a window that never calls it gets none); call it after
 * okb_window_reserve and before the slot's first upload, which then sizes the window's command buffer for one frame's
 * features on top of a full upload (OKB_ERR_CAPACITY if the slot was uploaded without); the initialised flags cover
 * the landmark capacity the slot has then.  Calling it again with other sizes commits what is pending and replaces the
 * store by an empty one (waiting for the device).
 * Landmark-sharded windows (okb_shard_reserve_landmarks): the store is replicated -- every rank reserves it alike and
 * receives the same okb_window_reserve_features / set_features / set_feature_landmarks / clear_features calls, whose
 * landmark slots are GLOBAL slots (below max_landmarks, else OKB_ERR_INVALID_ARG) -- while the initialised flags are
 * landmark state: each rank's cover its own landmarks at their local slots (okb_window_set_landmark_initialized goes
 * to the owner only).  A removal on the owner reaches the other ranks' stores at the next landmark exchange. */
int okb_window_reserve_features(okb_ctx* ctx, int win, int max_feature_frames, int max_cameras, int max_keypoints,
                                int desc_bytes);
/* Replaces the keypoints of (feat_slot, cam): n keypoints (x, y, size are used), their descriptors [n][desc_bytes],
 * landmark slots (NULL: all -1) and observed bits (NULL: all 0). */
int okb_window_set_features(okb_ctx* ctx, int win, int feat_slot, int cam, int n, const okb_keypoint* kp,
                            const uint8_t* desc, const int32_t* lm_slot, const uint8_t* observed);
/* Diagnostic read-back of the committed store entry (feat_slot, cam), after the work queued on the window's store:
 * *n = its keypoint count (-1: none); then, for the first *n keypoints and for each pointer that is not NULL, the
 * keypoints kp [n][2] and sizes size [n] as the store holds them (double), desc [n][desc_bytes], lm_slot [n] and
 * observed [n].  Size the arrays for the store's max_keypoints.  Pending edits are not committed and not seen. */
int okb_debug_features(okb_ctx* ctx, int win, int feat_slot, int cam, int32_t* n, double* kp, double* size, uint8_t* desc,
                       int32_t* lm_slot, uint8_t* observed);
/* Sets the landmark slot and observed bit of keypoints kp_idx[n] of (feat_slot, cam) -- the host-side changes of 2D-2D /
 * stereo initialisation and RANSAC removals. */
int okb_window_set_feature_landmarks(okb_ctx* ctx, int win, int feat_slot, int cam, int n, const int32_t* kp_idx,
                                     const int32_t* lm_slot, const uint8_t* observed);
/* Empties every camera of a feature slot (its frame left the window). */
int okb_window_clear_features(okb_ctx* ctx, int win, int feat_slot);
/* Estimator::setLandmarkInitialized for n landmark slots (flags[i] != 0: initialised). */
int okb_window_set_landmark_initialized(okb_ctx* ctx, int win, int n, const uint32_t* idx, const uint8_t* flags);

/* One VioKeyframeWindowMatchingAlgorithm 3D-2D match of a tracking job: frame A = feature slot feat_slot_a, camera
 * cam_a, against the job's frame B in camera cam_b. */
typedef struct okb_track_round { int32_t feat_slot_a, cam_a, cam_b, _pad; } okb_track_round;
/* An accepted setBestMatch: keypoint kp_b of (B, cam_b) now refers to landmark slot lm_slot. */
typedef struct okb_track_assoc { int32_t round, cam_b, kp_b, lm_slot, uncertain, _pad; } okb_track_assoc;
typedef struct okb_track_job {
  int32_t win;                  /* window slot */
  int32_t pose_b;               /* frame B's position in the window (T_WS of doSetup) */
  int32_t sb_b;                 /* its speed/bias block, -1: frame B is not in the IMU window */
  int32_t feat_slot_b;          /* its feature slot */
  float threshold;              /* briskMatchingThreshold_ (60) */
  int32_t num_best;             /* top-k list length (Frontend's matcher: 4, no ratio test) */
  int32_t n_rounds, _pad;
  const okb_track_round* rounds;  /* [n_rounds], run in order */
  /* outputs; capacities must cover the bounds: assoc_cap >= sum over rounds of B's keypoints in cam_b,
   * uninit_cap >= sum over rounds of A's keypoints */
  okb_track_assoc* assoc; int32_t assoc_cap;
  int32_t* n_assoc;
  int32_t* num_matches;         /* [n_rounds] numMatches_ */
  int32_t* num_uncertain;       /* [n_rounds] numUncertainMatches_ */
  uint32_t* uninit; int32_t uninit_cap;   /* landmark slots doSetup set to uninitialised, in order */
  int32_t* n_uninit;
} okb_track_job;
/* Tracks frame B of each job against its window: per round, in order, VioKeyframeWindowMatchingAlgorithm::doSetup
 * (okvis_frontend/src/VioKeyframeWindowMatchingAlgorithm.cpp:122-215, 238-255) from the store, the landmark estimates,
 * pose, extrinsics and camera of the window and the window's observation counts; DenseMatcher::match with verifyMatch's
 * chi-square gate (:304-339); setBestMatch's 3D-2D branch (:483-526).  Accepted matches are written into B's store
 * entries (landmark slot, observed) and raise the landmark's count for the later rounds; cleared initialised flags are
 * applied on the device.  Results come back in the reference's call order (round, then ascending B); the caller applies
 * them to its own bookkeeping (Estimator::addObservation) -- the call adds no observation to the window.  Results per
 * job are bit-identical to calling it alone.  Every job is checked on the host before any device work (uploaded
 * window, store reserved, feature slots present, ranges of cameras, poses, speed/bias, num_best <= 8, output
 * capacities, one descriptor length per call, a window listed twice, a round of frame B against itself in one
 * camera): the first failure returns OKB_ERR_INVALID_ARG
 * and names the job in okb_last_error.  A landmark-sharded context runs it as described with okb_shard_reserve_landmarks
 * (without that reservation: OKB_ERR_UNSUPPORTED).  Pending edits of the
 * job windows are committed first, one commit per run of consecutive windows; the call then runs on the transfer stream after the solver work already launched on
 * those windows only, with one H2D copy of the job table and one D2H copy of the results, and returns when they are
 * back.  Later solver calls on those windows are ordered after it.  n_jobs == 0 is a no-op. */
int okb_track_3d2d_batch(okb_ctx* ctx, int n_jobs, const okb_track_job* jobs);

/* ---- stereo landmark initialisation (Frontend::matchStereo, Frontend.cpp:521-572) ------------------------------------
 * One job = one VioKeyframeWindowMatchingAlgorithm Match2D2D match as matchStereo issues it: setFrames(mfId, mfId, cam_a,
 * cam_b) with usePoseUncertainty = false, so frames A and B are the job's frame -- one feature slot, two cameras. */
typedef struct okb_stereo_match {   /* one setBestMatch that reached the landmark bookkeeping */
  int32_t kp_a, kp_b;               /* keypoints of (frame, cam_a) / (frame, cam_b) */
  int32_t lm_slot_a, lm_slot_b;     /* their landmark slots in the store (in the graph), -1: none; at most one is set */
  int32_t can_be_initialized, _pad; /* canBeInitialized after stereoTriangulate and getUncertainty */
  double hp_W[4];                   /* T_WCa * hP_Ca, not normalised (what addLandmark / setLandmark receive) */
} okb_stereo_match;
typedef struct okb_stereo_job {
  int32_t win, pose, feat_slot, cam_a, cam_b;  /* window slot, the frame's position (T_WS), its feature slot, cameras */
  float threshold;                             /* briskMatchingThreshold_ (60) */
  int32_t num_best, _pad;                      /* top-k list length (Frontend's matcher: 4) */
  okb_stereo_match* out; int32_t out_cap;      /* out_cap >= keypoints of (feat_slot, cam_b) */
  int32_t* n_out;
} okb_stereo_job;
/* Per job, following the reference line by line and reading only the resident window and its store:
 *   setFrames (VioKeyframeWindowMatchingAlgorithm.cpp:76-111): T_WCa = T_WS T_SCa, T_WCb = T_WS T_SCb,
 *     T_CaCb = T_WCa^-1 T_WCb;
 *   doSetup, 2D-2D branch (:124-146, 216-232, 256-274): UOplus = diag(4e-8 I3, 1e-8 I3), resetFrames' prior H_
 *     (ProbabilisticStereoTriangulator.cpp:117-159), ray sigmas, backProject of every keypoint, and keypoints skipped
 *     whose slot names an initialised landmark of the graph;
 *   DenseMatcher::match with verifyMatch's 2D-2D gate (the matcher kernels of okb_hamming_match_gated);
 *   setBestMatch, 2D-2D branch (:370-481), for every winner below the threshold in ascending B: nothing if both
 *     keypoints name a landmark, else stereoTriangulate (:168-227) and, unless the rays are parallel, getUncertainty
 *     (:253-355), which decides canBeInitialized.
 * The records come back in that order; the caller applies them (addLandmark / setLandmark / setLandmarkInitialized /
 * addObservation, and new landmark ids).  The call changes nothing in the window, its store or its flags.  Every job is
 * checked on the host before any device work (uploaded window, store reserved, the feature slot present for both
 * cameras, cam_a != cam_b in range, pose in range, num_best <= 8, out_cap, one descriptor length per call, a window
 * listed twice): the first failure returns OKB_ERR_INVALID_ARG and names the job in okb_last_error.  A landmark-sharded
 * context runs it as described with okb_shard_reserve_landmarks (landmark exchange first; OKB_ERR_SHARD_TIMEOUT if a
 * peer does not arrive; without that reservation OKB_ERR_UNSUPPORTED).  Pending edits of the job windows are committed
 * first; the call runs on the
 * transfer stream after the solver work already launched on those windows, with one H2D copy of the job table and one
 * D2H copy of the results, and returns when they are back.  n_jobs == 0 is a no-op.  It runs as okb_match2d2d_batch
 * with frame A = frame B. */
int okb_stereo_init_batch(okb_ctx* ctx, int n_jobs, const okb_stereo_job* jobs);

/* ---- 2D-2D landmark initialisation against earlier frames (Frontend::matchToKeyframes :413-452, matchToLastFrame
 * :499-509) -----------------------------------------------------------------------------------------------------------
 * One job = one VioKeyframeWindowMatchingAlgorithm Match2D2D match: setFrames(olderFrameId, currentFrameId, cam_a, cam_b)
 * with usePoseUncertainty = false.  Frame A is the older frame, frame B the current one; each is named by its position in
 * the window (T_WS) and its feature slot.  A job with A = B (same slot and pose, cam_a != cam_b) is a stereo job and
 * returns exactly the records of okb_stereo_init_batch. */
typedef struct okb_match2d2d_job {
  int32_t win;
  int32_t pose_a, feat_slot_a, cam_a;   /* frame A: the older frame (its position in the window, feature slot, camera) */
  int32_t pose_b, feat_slot_b, cam_b;   /* frame B: the current frame */
  int32_t sb_current;                   /* speed/bias block of the window's current frame, -1: not in the IMU window */
  float threshold;                      /* briskMatchingThreshold_ (60) */
  int32_t num_best;                     /* top-k list length (4) */
  okb_stereo_match* out; int32_t out_cap;   /* out_cap >= keypoints of (feat_slot_b, cam_b) */
  int32_t* n_out;
} okb_match2d2d_job;
/* As okb_stereo_init_batch, with two frames:
 *   setFrames: T_WCa = T_WSa T_SCa, T_WCb = T_WSb T_SCb, T_CaCb = T_WCa^-1 T_WCb;
 *   doSetup's prior (:127-142): UOplus = diag(u I3, 1e-8 I3) with u = max(1, |v_current|)^2 * 1e-2 when A and B are
 *     different frames (feat_slot_a != feat_slot_b) and sb_current >= 0, else u = 4e-8;
 *   the rest as above: keypoints skipped whose store slot names an initialised landmark of the graph, the gated match,
 *     and per winner below the threshold, in ascending B, a record unless both store slots name a landmark of the graph.
 * hp_W = T_WCa hP_Ca.  lm_slot_a / lm_slot_b are the store's view: a keypoint that carries a landmark id only on the host
 * (matchStereo names every keypoint, Frontend.cpp:563-571, but most of those ids never enter the graph) has slot -1 and
 * is invisible to the device.  setBestMatch returns early when both keypoints carry an id (:373-375), so the caller drops
 * the records whose two keypoints both carry one.  Host checks, per job and before any device work, each failure
 * returning OKB_ERR_INVALID_ARG and naming the job: uploaded window, store reserved, both feature slots present for their
 * cameras; cameras, poses and sb_current in range; feat_slot_a == feat_slot_b exactly when pose_a == pose_b; no match of
 * one frame against itself in one camera; num_best <= 8; out_cap; one descriptor length per call; a window listed twice.
 * A landmark-sharded context runs it as described with okb_shard_reserve_landmarks (landmark exchange first;
 * OKB_ERR_SHARD_TIMEOUT if a peer does not arrive; without that reservation OKB_ERR_UNSUPPORTED); n_jobs == 0 is a
 * no-op.  The call changes nothing in the window,
 * its store or its flags; commits, stream order and copies are those of okb_stereo_init_batch (four launches, one H2D
 * copy of the job table, one D2H copy of the results). */
int okb_match2d2d_batch(okb_ctx* ctx, int n_jobs, const okb_match2d2d_job* jobs);

/* ---- keyframe decision (Frontend::doWeNeedANewKeyframe, Frontend.cpp:295-369) ---------------------------------------
 * One job = one session's current frame: cameras 0..n_cams-1 of a feature slot of a resident window.  Per camera, as
 * the reference's loop over `im` computes it: the keypoints cast to float; "matched" = store slot >= 0 (landmarkId !=
 * 0); fewer than 3 points or fewer than 3 matched points: skipped; else cv::convexHull of all points and of the matched
 * points (float points, clockwise = false, cv2's vertex order), cv::contourArea of both, the points with
 * cv::pointPolygonTest(matchesHull, p, false) > 0 (counted only when the matched hull has more than 2 vertices),
 * overlap = area_matched / area_all and ratio = n_matched / (double)inside, IEEE results kept (inf, NaN). */
typedef struct okb_keyframe_cam {
  int32_t n_points, n_matched;          /* keypoints of the image, those with a store slot >= 0 */
  int32_t hull_all, hull_matched;       /* vertex counts of the two hulls (0 when skipped) */
  int32_t inside, skipped;              /* points strictly inside the matched hull; 1: the camera changes neither maximum */
  double area_all, area_matched;        /* contourArea of the two hulls */
  double overlap, ratio;                /* overlapArea, matchingRatio */
} okb_keyframe_cam;
typedef struct okb_keyframe_result {
  double overlap, ratio;                /* std::max over the cameras that are not skipped, starting at 0 */
  int32_t need_keyframe, _pad;          /* !(overlap > overlap_threshold && ratio > matching_ratio_threshold) */
} okb_keyframe_result;
typedef struct okb_keyframe_job {
  int32_t win, feat_slot, n_cams;
  float overlap_threshold;              /* keyframeInsertionOverlapThreshold_ (0.6f), compared in double */
  float matching_ratio_threshold;       /* keyframeInsertionMatchingRatioThreshold_ (0.2f) */
  int32_t _pad;
  okb_keyframe_cam* cams;               /* [n_cams] */
  okb_keyframe_result* out;
} okb_keyframe_job;
/* The keyframe decision of every job, one CTA per (job, camera) in one launch; the last CTA of a job takes the maxima
 * in camera order (std::max(value, running): a NaN value wins, a NaN running maximum is replaced) and the decision.
 * Every job is checked on the host before any device work (uploaded window, store reserved, n_cams in 1..the store's
 * cameras, the feature slot present for each of them, cams and out present, a window listed twice): the first failure
 * returns OKB_ERR_INVALID_ARG and names the job in okb_last_error.  A landmark-sharded context runs it as described with
 * okb_shard_reserve_landmarks (landmark exchange first; OKB_ERR_SHARD_TIMEOUT if a peer does not arrive; without that
 * reservation OKB_ERR_UNSUPPORTED).  Pending edits of the job windows are committed first (2D-2D bookkeeping and RANSAC removals
 * arrive as store edits just before the decision); the call runs on the transfer stream after the solver work already
 * launched on those windows, with one H2D copy of the job table and one D2H copy of the results, returns when they are
 * back and changes nothing in the window or its store.  Results per job are bit-identical to calling it alone.
 * n_jobs == 0 is a no-op. */
int okb_keyframe_overlap_batch(okb_ctx* ctx, int n_jobs, const okb_keyframe_job* jobs);

/* ---- 3D-2D outlier rejection (Frontend::runRansac3d2d, Frontend.cpp:575-642) ------------------------------------------
 * One job = one session's current frame: cameras 0..n_cams-1 of a feature slot of a resident window.  Per job:
 *   correspondences as FrameNoncentralAbsoluteAdapter (FrameNoncentralAbsoluteAdapter.cpp:65-160) collects them, cameras
 *     ascending, then keypoints ascending: the store slot names a landmark of the graph, that landmark has at least 2
 *     observations in the window (sqrt_info != 0) and |hp[3]| >= 1e-8; point hp.head<3>() / hp[3], bearing = the
 *     normalised backProject (a failed backProject leaves a NaN bearing: never an inlier, never in a usable sample),
 *     sigmaAngle = sqrt(2) sigma^2 / fu^2 with sigma = 0.8 size / 12;
 *   fewer than 2 frames in the window: ret = 1; fewer than 5 correspondences: ret = n_correspondences; no outliers;
 *   max_iterations hypotheses, each 4 distinct correspondences drawn by a counter-based generator keyed by (seed,
 *     hypothesis, draw) -- independent of the job's position in the batch -- the first 3 solved by a generalised P3P,
 *     the 4th choosing the solution of lowest score; no adaptive stop (DESIGN.md 6f);
 *   score |normalize(C_SC^T (T_WS^-1 X - r_SC)) - bearing|^2 / sigmaAngle (FrameAbsolutePoseSacProblem.hpp:134-160),
 *     inlier iff score < threshold; the most inliers win, ties to the lowest hypothesis;
 *   ret = n_inliers; when n_inliers >= 10 every other correspondence is an outlier record (Frontend.cpp:613-640). */
typedef struct okb_ransac_outlier { int32_t cam, kp, lm_slot; } okb_ransac_outlier;
typedef struct okb_ransac_result {
  int32_t ret;                          /* what runRansac3d2d returns */
  int32_t n_correspondences, n_inliers;
  int32_t best;                         /* winning hypothesis, -1: no hypothesis had a model */
  int32_t n_outliers, _pad;
  double T_WS[7];                       /* the winner's model [t, q_xyzw], zero when best == -1 */
} okb_ransac_result;
typedef struct okb_ransac_job {
  int32_t win, feat_slot, n_cams;
  int32_t max_iterations;               /* hypotheses, 1..64 (the reference: 50) */
  double threshold;                     /* ransac.threshold_ (9) */
  uint64_t seed;
  int32_t* hyp_inliers;                 /* [max_iterations] inliers of every hypothesis, or NULL */
  okb_ransac_outlier* outliers;         /* [outlier_cap], correspondence order */
  int32_t outlier_cap, _pad;            /* >= the keypoints of the frame in cameras 0..n_cams-1 */
  okb_ransac_result* out;
} okb_ransac_job;
/* One CTA per job in one launch.  Every job is checked on the host before any device work (uploaded window, store
 * reserved, n_cams in 1..the store's, the window's extrinsics and cameras (at most 16), the feature slot present for
 * each camera, max_iterations in 1..64, a finite positive threshold, out present, outlier capacity, a window listed
 * twice): the first failure returns OKB_ERR_INVALID_ARG and names the job in okb_last_error.  A landmark-sharded context
 * runs it as described with okb_shard_reserve_landmarks (landmark exchange first; OKB_ERR_SHARD_TIMEOUT if a peer does
 * not arrive; without that reservation OKB_ERR_UNSUPPORTED).  Pending edits of the job windows are committed first
 * (removals from earlier rounds);
 * the call runs on the transfer stream after the solver work already launched on those windows, with one H2D copy of
 * the job table and one D2H copy of the results, returns when they are back and changes nothing in the window or its
 * store: the caller applies the removals.  Results per job are bit-identical to calling it alone.  n_jobs == 0 is a
 * no-op. */
int okb_ransac_3d2d_batch(okb_ctx* ctx, int n_jobs, const okb_ransac_job* jobs);

/* ---- 2D-2D outlier rejection and pose initialisation (Frontend::runRansac2d2d, Frontend.cpp:645-810) -----------------
 * One job = one session's runRansac2d2d(currentFrameId, olderFrameId, initializePose, removeOutliers): frame B (the
 * current frame) and frame A (the older frame), each named by its position in the window (T_WS) and its feature slot,
 * cameras 0..n_cams-1.  Per camera im, ascending, as the reference's loop runs:
 *   correspondences as FrameRelativeAdapter (FrameRelativeAdapter.cpp:139-244) collects them: B's keypoints ascending
 *     whose store slot names a landmark of the graph, the first keypoint per landmark kept (std::map::insert); then A's
 *     keypoints ascending whose store slot names one of those landmarks, matched to B's keypoint for it.  Bearings are
 *     the normalised backProject (a failed backProject leaves a NaN bearing: counted, never an inlier, never in a usable
 *     sample), sigmaAngle = sqrt(2) sigma^2 / fu^2 with sigma = 0.8 size / 12;
 *   fewer than 10 correspondences: the camera is skipped (:670-671);
 *   two RANSACs of max_iterations hypotheses each, drawn by the counter-based generator of okb_ransac_3d2d_batch keyed by
 *     (seed, (2 im + problem) 64 + hypothesis, draw), no adaptive stop (DESIGN.md 6i):
 *     rotation-only (problem 0): 2 correspondences, R from their bearing triads; score
 *       0.5 |R f2 - f1|^2 / sigma1 + 0.5 |R^T f1 - f2|^2 / sigma2 (FrameRotationOnlySacProblem.hpp);
 *     relative pose (problem 1): a five-point solver on 5 correspondences, the 6th choosing among the admissible
 *       solutions; score FrameRelativePoseSacProblem.hpp's, the point triangulated in frame A as the midpoint of the
 *       common perpendicular of the rays l1 f1 and t + l2 R f2;
 *     inlier iff score < threshold; the most inliers win, ties to the lowest hypothesis;
 *   the decision (:709-733): float ratios inliers / correspondences; rotation-only is chosen iff rot_ratio > rel_ratio ||
 *     rot_ratio > 0.8 (rotationOnly = true); more than 10 inliers of the chosen model set that model's success flag;
 *     the flags are not reset between cameras, and the camera is applied when either is set (:735-737), its
 *     correspondences outside the chosen model's inliers becoming outlier records;
 *   with initialize_pose, each applied camera sets T_WS0 = T_WSA T_SCA T_C1C2 T_SC0^-1 (:756-798), T_C1C2 = the
 *     five-point winner when any camera's five-point model succeeded (its unit translation scaled by
 *     max(0, t . r(T_SCA^-1 T_WSA^-1 T_WS0 T_SC0)), T_WS0 as the previous camera left it), else the rotation-only
 *     winner with zero translation; a missing winner leaves T_C1C2 the identity;
 *   ret = the summed inliers of the chosen models of all cameras that were not skipped, or -1 with rotationOnly = true
 *     when no model succeeded (:802-808).
 * One deliberate departure (:735-753): the reference reads and clears multiFrame->landmarkId(im, k) with k the
 * correspondence number and then removes the observation (lmId, current, im, idxB), which clears an unrelated keypoint's
 * id and removes an observation that usually does not exist.  The outlier record names the correspondence's own B
 * keypoint (idxB) and its landmark slot instead, so that the caller reaches okb_ransac_3d2d_batch's end state: the
 * observation removed, the host id 0 and the store slot -1.  A B keypoint that several A keypoints of one landmark
 * matched comes in one record per correspondence; the caller applies the first (Estimator::finishRansac2d2d skips the
 * records whose keypoint no longer carries the landmark). */
typedef struct okb_ransac2d_outlier { int32_t cam, kp_a, kp_b, lm_slot; } okb_ransac2d_outlier;
typedef struct okb_ransac2d_cam {
  int32_t n_correspondences;            /* adapter.getNumberCorrespondences() */
  int32_t rot_inliers, rel_inliers;     /* inliers of each RANSAC's winner (0: skipped or no model) */
  int32_t rot_best, rel_best;           /* winning hypotheses, -1: skipped or no hypothesis had a model */
  int32_t rotation_only;                /* 1: the rotation-only model was chosen */
  int32_t applied;                      /* 1: outliers reported (and, with initialize_pose, the pose set) */
  int32_t n_outliers;
  double R_rot[9];                      /* rotation-only winner, row-major (identity when rot_best == -1) */
  double R_rel[9], t_rel[3];            /* five-point winner T_C1C2 = [R t] (C1: frame A's camera, C2: frame B's), |t| = 1
                                           (identity and zero when rel_best == -1) */
} okb_ransac2d_cam;
typedef struct okb_ransac2d_result {
  int32_t ret;                          /* what runRansac2d2d returns */
  int32_t rotation_only;                /* its rotationOnly */
  int32_t pose_set;                     /* 1: T_WS holds frame B's initialised pose (the caller applies it with set_T_WS) */
  int32_t n_outliers;
  double T_WS[7];                       /* [t, q_xyzw], zero unless pose_set */
} okb_ransac2d_result;
typedef struct okb_ransac2d_job {
  int32_t win;
  int32_t pose_b, feat_slot_b;          /* frame B: the current frame (its position in the window, feature slot) */
  int32_t pose_a, feat_slot_a;          /* frame A: the older frame */
  int32_t n_cams;
  int32_t initialize_pose;              /* initializePose && !isInitialized_ */
  int32_t max_iterations;               /* hypotheses per RANSAC, 1..64 (the reference: 50) */
  double threshold;                     /* threshold_ of both RANSACs (9) */
  uint64_t seed;
  int32_t* hyp_inliers;                 /* [n_cams][2][max_iterations] inliers of every hypothesis (problem 0: rotation-only,
                                           1: five-point), or NULL */
  okb_ransac2d_cam* cams;               /* [n_cams], or NULL */
  okb_ransac2d_outlier* outliers;       /* [outlier_cap], cameras ascending, then correspondence order */
  int32_t outlier_cap, _pad;            /* >= the keypoints of frame A in cameras 0..n_cams-1 */
  okb_ransac2d_result* out;
} okb_ransac2d_job;
/* One CTA per job in one launch.  Every job is checked on the host before any device work (uploaded window, store
 * reserved, both feature slots in range and present for each camera, both poses in range, n_cams in 1..the store's, the
 * window's extrinsics and cameras (at most 16), max_iterations in 1..64, a finite positive threshold, out present,
 * outlier capacity, a window listed twice): the first failure returns OKB_ERR_INVALID_ARG and names the job in
 * okb_last_error.  A landmark-sharded context runs it as described with okb_shard_reserve_landmarks (landmark exchange
 * first; OKB_ERR_SHARD_TIMEOUT if a peer does not arrive; without that reservation OKB_ERR_UNSUPPORTED).  Pending edits of
 * the job windows are committed first; the call runs on the transfer stream after the solver work already launched on
 * those windows, with one H2D copy of the job table and one D2H copy of the results, returns when they are back and
 * changes nothing in the window or its store: the caller applies the removals and the pose.  Results per job are
 * bit-identical to calling it alone.  n_jobs == 0 is a no-op. */
int okb_ransac_2d2d_batch(okb_ctx* ctx, int n_jobs, const okb_ransac2d_job* jobs);

/* ---- detection straight into the feature store (Frontend::detectAndDescribe, Frontend.cpp:92-114, for every camera of
 * a frame whose features the window's store is to hold) ---------------------------------------------------------------
 * One session's frame: images[c] is detected, described and written into camera c of feature slot feat_slot of window
 * win, for c < n_cams (other cameras of the slot are left as they are). */
typedef struct okb_detect_store_job {
  int32_t win, feat_slot, n_cams, _pad;
  const okb_image_desc* images;    /* [n_cams], as okb_detect_describe_batch */
  okb_keypoint* out_kp;            /* [n_cams][max_out] */
  uint8_t* out_desc;               /* [n_cams][max_out][desc_bytes], or NULL */
  int32_t* n_out;                  /* [n_cams] */
} okb_detect_store_job;
/* Per image, n_out / out_kp / out_desc are bit-identical to what okb_detect_describe_batch returns for it with the
 * same parameters, and the store entry (win, feat_slot, camera) then holds what okb_window_set_features(win, feat_slot,
 * camera, n, kp, desc, NULL, NULL) followed by a commit leaves there: x, y and size widened to double, the descriptors,
 * landmark slot -1 and observed 0 for every keypoint, n keypoints.  The host's keypoint counts follow, so later store
 * edits (okb_window_set_feature_landmarks, okb_window_clear_features) apply to the new features.  An image with more NMS
 * candidates than the detector holds gets n_out = -1 and keeps its store entry; every other image is written and the
 * call returns OKB_ERR_CAPACITY.
 * Every job is checked on the host before any device work (uploaded window, store reserved, feat_slot in range, n_cams
 * in 1..the store's cameras, params->desc_bytes = the store's descriptor length, the store's keypoints per image >=
 * min(max_keypoints, max_out), out_kp and n_out present, each image as okb_detect_describe_batch checks it, at most
 * 65535 images in all, a window listed twice): the first failure returns OKB_ERR_INVALID_ARG and names the job in
 * okb_last_error.  A landmark-sharded context runs it as described with okb_shard_reserve_landmarks (every rank
 * detects redundantly into its replicated store; without that reservation OKB_ERR_UNSUPPORTED); n_jobs == 0 is a no-op.
 * Pending edits of the job windows are committed first, and the store writes are ordered after that commit and after
 * the solver work already launched on those windows: a clear of the slot queued before the call does not erase the new
 * features, one queued after it does.  The detection runs as okb_detect_describe_batch over all images of the call (its
 * stream, buffers and serialisation), plus one launch that writes the store; the D2H copy carries the counts and
 * keypoints, and the descriptors only when a job asks for them.  Returns when the store holds the features. */
int okb_detect_describe_store_batch(okb_ctx* ctx, int n_jobs, const okb_detect_store_job* jobs, const okb_detect_params* params,
                                    int max_out, int host_threads);

#ifdef __cplusplus
}
#endif
#endif  /* OKVIS_B200_H_ */
