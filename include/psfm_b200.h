/*
 * psfm_b200.h — C ABI of the H100-native ParticleSfM optimisation hot paths.
 *
 * Two paths, nothing else (SURVEY.md §8):
 *
 *   HP1  dense point-trajectory path-consistency optimiser.
 *        Replaces `particlesfm::optimize_location`
 *        (reference: point_trajectory/optimize/src/trajectory_optimize.cpp:30-96,
 *         declared trajectory_optimize.h:35-42, bound at bindings.cc:31).
 *
 *   HP2  global bundle adjustment.
 *        Replaces `colmap::BundleAdjuster::Solve`
 *        (reference: sfm/gmapper/src/optim/bundle_adjustment.cc:259-320, class at
 *         bundle_adjustment.h:161-198; options bundle_adjustment.h:48-102; called from
 *         sfm/gmapper/src/sfm/global_mapper.cc:438-439).
 *
 * Plain pointers and sizes only; no torch / Eigen / COLMAP types.  Every entry point
 * returns PSFM_OK (0) or a negative psfm_status; there is NO CPU fallback: when no
 * CUDA device is usable the calls return PSFM_ERR_NO_DEVICE / PSFM_ERR_CUDA.
 *
 * Pointers named `h_*` / plain are HOST pointers unless the function name ends in
 * `_device` or the comment says "device pointer".
 */
#ifndef PSFM_B200_H_
#define PSFM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PSFM_ABI_VERSION 2

typedef enum {
  PSFM_OK = 0,
  PSFM_ZERO_RESIDUALS = 1,      /* HP2: problem has no residual (reference returns false,
                                   bundle_adjustment.cc:268-271) */
  PSFM_NO_ROTATIONS = 2,        /* psfm_estimate_global_rotations: no posed pair, or a factorisation failed
                                   (reference returns false, robust_rotation_estimator.cc:101-109, 315-317) */
  PSFM_ERR_INVALID = -1,        /* bad argument / inconsistent sizes */
  PSFM_ERR_NO_DEVICE = -2,      /* no CUDA device: the product has no CPU path */
  PSFM_ERR_CUDA = -3,           /* CUDA runtime error; see psfm_last_error() */
  PSFM_ERR_UNSUPPORTED = -4,    /* e.g. camera model other than SIMPLE_PINHOLE */
  PSFM_ERR_NCCL = -5
} psfm_status;

/* Human-readable text of the last error on this thread ("" if none). */
const char* psfm_last_error(void);
int psfm_abi_version(void);
/* Number of visible CUDA devices (0 when none / driver missing). */
int psfm_device_count(void);
/* Select the CUDA device used by subsequent calls from this process. */
int psfm_set_device(int device);
/* Number of kernel launches issued by this library since process start (for
   bench.py's `gpu_launches`). */
int64_t psfm_launch_count(void);

/* ------------------------------------------------------------------------- */
/* HP1 — path-consistency trajectory optimiser                                */
/* ------------------------------------------------------------------------- */

/* Solver constants of the reference call (trajectory_optimize.cpp:74-79) plus the
   Ceres 2.0.0 defaults it inherits.  Pass NULL to get exactly these. */
typedef struct {
  int32_t max_num_iterations;        /* 200  (trajectory_optimize.cpp:76) */
  double function_tolerance;         /* 1e-6  Ceres default */
  double gradient_tolerance;         /* 1e-10 Ceres default */
  double parameter_tolerance;        /* 1e-8  Ceres default */
  double initial_trust_region_radius;/* 1e4   Ceres default */
  double max_trust_region_radius;    /* 1e16  Ceres default */
  double min_trust_region_radius;    /* 1e-32 Ceres default */
  double min_relative_decrease;      /* 1e-3  Ceres default */
  int32_t max_num_consecutive_invalid_steps; /* 5 Ceres default */
  int32_t jacobi_scaling;            /* 1     Ceres default */
} psfm_traj_options;

typedef struct {
  int32_t num_iterations;            /* iterations executed (successful+unsuccessful+invalid) */
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t termination;               /* psfm_termination */
  double initial_cost;               /* 1/2 sum r^2 */
  double final_cost;
  double solve_ms;                   /* device time of the solver kernel(s) */
  double total_ms;                   /* wall time of the call incl. copies */
} psfm_traj_summary;

typedef enum {
  PSFM_TERM_CONVERGENCE_GRADIENT = 0,
  PSFM_TERM_CONVERGENCE_PARAMETER = 1,
  PSFM_TERM_CONVERGENCE_FUNCTION = 2,
  PSFM_TERM_NO_CONVERGENCE = 3,      /* max iterations */
  PSFM_TERM_FAILURE = 4,             /* too many invalid steps / radius underflow */
  PSFM_TERM_MIN_RADIUS = 5
} psfm_termination;

void psfm_traj_default_options(psfm_traj_options* o);

/*
 * Drop-in for particlesfm.optimize_location (bindings.cc:31).
 *   uv12   [n*4] f64 row-major (x1,y1,x2,y2)       — trajectory_optimize.cpp:31,43-47
 *   ref1   [n*2] f64  x1_ref = x0 + flow01(x0)     — trajectory.py:182
 *   ref2   [n*2] f64  x2_ref = x0 + flow02(x0)     — trajectory.py:183
 *   scale  [n]   f64  weight of the flow02 term    — trajectory.py:179
 *   flow12 [h*w*2] f32 HWC interleaved (u,v)        — the reference force-casts this
 *          f32 map to f64 (py::array_t<double>, trajectory_optimize.h:40); f32->f64 is
 *          exact, so keeping f32 in HBM and widening on load is bit-identical.
 *   out_uv12 [n*4] f64
 * n == 0 is accepted (returns immediately).  Never fails on non-convergence (the
 * reference ignores the Ceres summary, trajectory_optimize.cpp:82).
 */
int psfm_traj_optimize(const double* uv12, const double* ref1, const double* ref2,
                       const double* scale, const float* flow12, int32_t n, int32_t w,
                       int32_t h, const psfm_traj_options* opts, double* out_uv12,
                       psfm_traj_summary* summary);

/* Same, all six array arguments are DEVICE pointers (inputs already resident in HBM);
   runs on `stream` (a cudaStream_t cast to void*) and synchronises it before returning.
   NULL = the library's own non-blocking HP1 stream, which does not wait for work on the
   legacy default stream; pass cudaStreamLegacy for that. */
int psfm_traj_optimize_device(const double* d_uv12, const double* d_ref1,
                              const double* d_ref2, const double* d_scale,
                              const float* d_flow12, int32_t n, int32_t w, int32_t h,
                              const psfm_traj_options* opts, double* d_out_uv12,
                              psfm_traj_summary* summary, void* stream);

/* ------------------------------------------------------------------------- */
/* Tracker stage around HP1 (SURVEY.md 8f row f-1): the float32 sampling,        */
/* survival test and re-seeding of point_trajectory/trajectory.py:25-62,117-194  */
/* and the forward/backward flow check of point_trajectory/utils.py:58-105, bit   */
/* for bit as torch's CPU grid_sample / scipy's distance transform produce them   */
/* (csrc/tracker.cu).  Host buffers in, host buffers out; maps are [H][W][C].      */
/* ------------------------------------------------------------------------- */
/* grid_sample(map, xy) of trajectory.py:25-37: bilinear, zeros padding, align_corners;
   channels 1 or 2; out [n][channels] float32 */
int psfm_grid_sample(const float* map, int32_t h, int32_t w, int32_t channels, const double* xy, int32_t n, float* out);
/* flow_check for one frame pair: err [H][W] (may be NULL), occ [H][W] = err > thres or out of bounds */
int psfm_flow_check(const float* flow_f, const float* flow_b, int32_t h, int32_t w, float thres, float* err, uint8_t* occ);
/* step_forward + the re-seeding mask of extend_all for all live particles:
   next_xy = cur_xy + flow(cur_xy); flags[i] = inside the image and occlusion(cur_xy) <= 0.1;
   reseed_mask [ceil(H/r)][ceil(W/r)] (may be NULL) = distance_transform_edt(1 - occupied) > r on the
   r-strided grid, occupied = the pixels (int(y), int(x)) of the survivors' next positions (needs >= 1 survivor) */
int psfm_tracker_step(const float* flow, const uint8_t* occ, int32_t h, int32_t w, const double* cur_xy, int32_t n,
                      int32_t sample_ratio, double* next_xy, uint8_t* flags, uint8_t* reseed_mask);
/* optimize_buffer's inputs (trajectory.py:171-183): ref1 = x0 + flow01(x0), ref2 = x0 + flow02(x0),
   scale = (1 - occ02(x0)) * (|flow02(x0)| < upper_flow) */
int psfm_tracker_buffer_inputs(const float* flow01, const float* flow02, const uint8_t* occ02, int32_t h, int32_t w,
                               const double* x0, int32_t n, double upper_flow, double* ref1, double* ref2, double* scale);

/* ------------------------------------------------------------------------- */
/* The whole tracker stage resident on the device: point_trajectory/             */
/* track_optimize.py:24-54 from flow maps to the track set.  Maps are DEVICE       */
/* pointers, [H][W][2] float32 flows and [H][W] uint8 (0/1) occlusion maps; the     */
/* particles, their history and HP1's inputs never leave the device.  All work      */
/* runs on `stream` (a cudaStream_t cast to void*, NULL = the legacy default       */
/* stream; HP1 too).  Same results, bit for bit, as the per-op entry points above   */
/* with psfm_traj_optimize as the optimiser.  Once a call on a handle has failed     */
/* for a CUDA reason, every later call on it but psfm_tracker_destroy is refused.   */
/* ------------------------------------------------------------------------- */
typedef struct psfm_tracker psfm_tracker;
/* num_frames = number of images = number of forward flows + 1 */
int psfm_tracker_create(int32_t h, int32_t w, int32_t sample_ratio, int32_t num_frames, void* stream, psfm_tracker** out);
/* One frame t (t = 0, 1, ... in call order) of track_optimize.py:31-50: seed (all grid points at t = 0, else the
   re-seed mask of the previous frame in row-major order), step with flow = flows[t] and occ = occ_maps[t], extend
   (survivors in active order, retired particles ranked in active order, re-seed mask of the survivors' next
   positions), and from t = 1 on select the particles with 3 observations and build HP1's inputs from
   flow_prev = flows[t-1], flow2_prev = flows_f2[t-1], occ2_prev = occ_maps_s2[t-1] (NULL at t = 0).
   counts (may be NULL) [3]: survivors, seeds of the next frame, buffered particles.  When counts[2] > 0 the
   buffered set must be optimised (psfm_tracker_optimize, or psfm_tracker_get_buffer + psfm_tracker_set_buffer)
   before the next frame; `flow` must stay valid until then (it is HP1's flow12). */
int psfm_tracker_advance(psfm_tracker* t, const float* flow, const uint8_t* occ, const float* flow_prev,
                         const float* flow2_prev, const uint8_t* occ2_prev, int32_t* counts);
/* HP1 on the buffered set (opts NULL = defaults), then the optimised x1, x2 written back into the history */
int psfm_tracker_optimize(psfm_tracker* t, const psfm_traj_options* opts, psfm_traj_summary* summary);
/* the buffered set to a host optimiser, in buffer order: uv12 [n][4], ref1 [n][2], ref2 [n][2], scale [n] (host) */
int psfm_tracker_get_buffer(psfm_tracker* t, double* uv12, double* ref1, double* ref2, double* scale);
/* its result, uv12 [n][4] (host), written back as psfm_tracker_optimize does */
int psfm_tracker_set_buffer(psfm_tracker* t, const double* uv12);
/* flow_check for one frame pair on DEVICE buffers, on `stream`, without synchronising: err (may be NULL), occ */
int psfm_flow_check_device(const float* flow_f, const float* flow_b, int32_t h, int32_t w, float thres, float* err,
                           uint8_t* occ, void* stream);
/* clear_active, then the track set in full_trajs order: trajectory id = retire rank, observations in time order,
   trajectories shorter than traj_min_len dropped (ids keep their unfiltered numbering) */
int psfm_tracker_finish(psfm_tracker* t, int32_t traj_min_len, int64_t* num_trajs, int64_t* num_obs);
/* host copies of the finished track set: ids [num_trajs], ptr [num_trajs + 1] (trajectory k owns observations
   ptr[k] .. ptr[k + 1]), frame_ids [num_obs], xy [num_obs][2] */
int psfm_tracker_result(psfm_tracker* t, int64_t* ids, int64_t* ptr, int32_t* frame_ids, double* xy);
void psfm_tracker_destroy(psfm_tracker* t);
/* psfm_tracker_create with the mode: path_consistency 1 is psfm_tracker_create (track_optimize.py:24-54); 0 is
   track.py:24-50, the same tracker without the buffer: psfm_tracker_advance needs only flow and occ on every frame,
   reports 0 buffered and never asks for psfm_tracker_optimize, and a frame without survivors is not an error */
int psfm_tracker_create_mode(int32_t h, int32_t w, int32_t sample_ratio, int32_t num_frames, int32_t path_consistency,
                             void* stream, psfm_tracker** out);

/* ------------------------------------------------------------------------- */
/* track.npy's pickled TrajectorySet state written on the device                */
/* (csrc/track_npy.cu, DESIGN.md 4.13): the body {id: {"frame_ids": [...],        */
/* "locations": [(x, y), ...], "labels": [False, ...]}, ...} as protocol-2 pickle  */
/* opcodes without memo, trajectories in the given order.  The bytes wait in a     */
/* pinned host buffer owned by the handle.                                         */
/* ------------------------------------------------------------------------- */
typedef struct psfm_track_npy psfm_track_npy;
/* host arrays: ids [num_trajs] in [0, 2^31), ptr [num_trajs + 1] monotone from 0 to num_obs, frame_ids [num_obs]
   >= 0, xy [num_obs][2]; anything else is PSFM_ERR_INVALID before the device is used */
int psfm_track_npy_create(const int64_t* ids, const int64_t* ptr, const int32_t* frame_ids, const double* xy, int64_t num_trajs,
                          int64_t num_obs, psfm_track_npy** out, int64_t* nbytes);
/* the finished track set of a tracker (after psfm_tracker_finish), encoded where it lies, on the tracker's stream */
int psfm_tracker_track_npy(psfm_tracker* t, psfm_track_npy** out, int64_t* nbytes);
/* the body's nbytes bytes, valid until psfm_track_npy_destroy */
const uint8_t* psfm_track_npy_data(const psfm_track_npy* h);
void psfm_track_npy_destroy(psfm_track_npy* h);

/* ------------------------------------------------------------------------- */
/* SURVEY.md 8(f) row f-2: track set -> COLMAP keypoints and matches          */
/* (sfm/matches_from_flow.py:51-118, csrc/handoff.cu).  Host buffers in, host   */
/* buffers out; the result stays on the device until it is fetched.  Bit for   */
/* bit what handoff.traj_to_matches returns.                                    */
/* ------------------------------------------------------------------------- */
typedef struct psfm_matches psfm_matches;
/* The kept samples of num_trajs trajectories in the reference's visiting order: trajectory t owns samples
   traj_ptr[t] .. traj_ptr[t + 1] (traj_ptr[0] = 0, non-decreasing, at most 2^31 - 1 samples), frame_ids [..]
   and xy [..][2] per sample.  Every sample becomes a keypoint of its frame (keypoint index = number of earlier
   samples of that frame); a trajectory of n samples matches sample j with every k != j when n <= sample_k,
   otherwise with the targets s * (n / sample_k), s < sample_k, other than j.  Matches are grouped by ordered
   image pair (a, b), in visiting order inside a pair; pairs are listed by a, then by first appearance.
   num_pairs / num_matches receive the result's sizes.  A frame id outside [0, num_images) is PSFM_ERR_INVALID. */
int psfm_matches_create(const int64_t* traj_ptr, int64_t num_trajs, const int64_t* frame_ids, const double* xy,
                        int32_t num_images, int32_t sample_k, psfm_matches** out, int64_t* num_pairs,
                        int64_t* num_matches);
/* host copies of the result: keypoint_ptr [num_images + 1] (image i owns keypoints keypoint_ptr[i] ..
   keypoint_ptr[i + 1]), keypoints [traj_ptr[num_trajs]][2], pair_images [num_pairs][2], pair_ptr [num_pairs + 1]
   (pair p owns matches pair_ptr[p] .. pair_ptr[p + 1]), matches [num_matches][2] (keypoint in a, keypoint in b) */
int psfm_matches_result(const psfm_matches* m, int64_t* keypoint_ptr, double* keypoints, int64_t* pair_images,
                        int64_t* pair_ptr, int64_t* matches);
void psfm_matches_destroy(psfm_matches* m);

/* The COLMAP database's match table, built on the device from a psfm_matches handle (csrc/handoff.cu): bit for bit
   the arrays of handoff.import_keypoints_matches_arrays followed by MatchTables.from_rows, without the int64 host copy.
   image_ids [num_images] is the database id of every frame (distinct, in [0, 2^31 - 1), any permutation).  Images in
   image_id order; keypoints float32(x + 0.5), float32(y + 0.5) (the double sum rounded once to nearest).  Of the two
   ordered pairs (a, b) and (b, a) of one unordered pair the one with the smaller first frame is kept, else the other
   one: the first occurrence in get_image_ids order (import_feature_matches.py:88-99), which is name order because
   SQLite answers that query from the unique index on name.  Its columns are swapped when its first image has the
   larger id.  Pairs in pair_id order, image 1 the smaller id; matches uint32.
   On success the handle's keypoints and int64 matches move into the table and are freed: psfm_matches_result then
   takes NULL keypoints and matches and writes the other arrays only.  num_keypoints / num_pairs / num_matches receive
   the table's sizes.  PSFM_ERR_INVALID before any launch for an id out of range or given twice, a handle whose matches
   were already moved, or an ordered pair of a frame with itself (a trajectory visiting one frame twice). */
/* The psfm_matches handle of a finished tracker's track set (after psfm_tracker_finish), built on the tracker's stream
   from its device arrays without a host copy: the handle psfm_matches_create returns for the host copy of those arrays
   (psfm_tracker_result: ptr as traj_ptr, frame_ids widened to int64, xy), bit for bit.  PSFM_ERR_INVALID for a tracker
   that is not finished, num_images below the tracker's number of frames, or sample_k < 1. */
int psfm_tracker_matches(psfm_tracker* t, int32_t num_images, int32_t sample_k, psfm_matches** out, int64_t* num_pairs,
                         int64_t* num_matches);

typedef struct psfm_match_table psfm_match_table;
int psfm_matches_table(psfm_matches* m, const int32_t* image_ids, psfm_match_table** out, int64_t* num_keypoints,
                       int64_t* num_pairs, int64_t* num_matches);
/* host copies: keypoint_ptr [num_images + 1], keypoints [num_keypoints][2], pair_images [num_pairs][2] image rows,
   match_ptr [num_pairs + 1], matches [num_matches][2] (point2D_idx1, point2D_idx2) */
int psfm_match_table_result(const psfm_match_table* t, int64_t* keypoint_ptr, float* keypoints, int32_t* pair_images,
                            int64_t* match_ptr, uint32_t* matches);
void psfm_match_table_destroy(psfm_match_table* t);

/* ------------------------------------------------------------------------- */
/* SURVEY.md 8(f) row f-4: the RANSAC-free steps that initialise HP2, batched (csrc/init_geometry.cu). */
/* Host buffers in, host buffers out.                                          */
/* ------------------------------------------------------------------------- */
/* BatchOptimizeRelativePositionWithKnownRotation (sfm/gmapper/src/global/known_rotation_util.cc:198-229) for
   num_pairs image pairs at once; per pair OptimizeRelativePositionWithKnownRotation (:107-196): IRLS on the
   epipolar constraints with the two known rotations, sign by the cheirality majority.
   points1 / points2: [pair_ptr[num_pairs]][2] NORMALISED image points (camera.ImageToWorld, :215-221) of the
   correspondences, pair p owns the range pair_ptr[p] .. pair_ptr[p + 1]; qvec1 / qvec2: [num_pairs][4] (w, x, y, z);
   tvec: [num_pairs][3] unit relative positions (pair.tvec); iterations (may be NULL): IRLS iterations run */
int psfm_known_rotation_translations(const double* points1, const double* points2, const int32_t* pair_ptr,
                                     const double* qvec1, const double* qvec2, int32_t num_pairs, double* tvec,
                                     int32_t* iterations);
/* Multi-view DLT of num_tracks tracks at once: COLMAP TriangulateMultiViewPoint, the estimator behind
   IncrementalTriangulator::Create (sfm/incremental_triangulator.cc:463-548) without its RANSAC loop.
   proj_matrices: [track_ptr[num_tracks]][12] row-major 3 x 4 (image.ProjectionMatrix(), :494), points: [..][2]
   normalised image points (:492-493), track t owns the range track_ptr[t] .. track_ptr[t + 1]; xyz: [num_tracks][3] */
int psfm_triangulate_tracks(const double* proj_matrices, const double* points, const int32_t* track_ptr,
                            int32_t num_tracks, double* xyz);
/* TwoViewGeometry::EstimateRelativePose (estimators/two_view_geometry.cc:172-239) of num_pairs verified image pairs
   at once, the step gcolmap's DatabaseCache::Load runs as one ThreadPool task per pair (base/database_cache.cc:206-228)
   (csrc/two_view.cu).  Images: keypoint_ptr [num_images + 1] (image f owns keypoints keypoint_ptr[f] ..
   keypoint_ptr[f + 1]), keypoints [..][2] float32 as stored in the database (COLMAP origin), image_camera
   [num_images] into cameras [num_cameras][3] SIMPLE_PINHOLE (f, cx, cy).  Pairs: pair_images [num_pairs][2] image
   indices (image 1, image 2), config, E / F / H [num_pairs][9] row-major, inlier_ptr [num_pairs + 1] (pair p owns
   inlier_matches [inlier_ptr[p] .. inlier_ptr[p + 1]][2]: keypoint in image 1, keypoint in image 2).
   Per pair: CALIBRATED (2) and UNCALIBRATED (3, E = K2' F K1) decompose E, PLANAR (4), PANORAMIC (5) and
   PLANAR_OR_PANORAMIC (6) decompose H; the candidate with the most correspondences triangulated in front of both
   cameras (CheckCheirality) gives qvec (w, x, y, z), tvec, num_points3D and tri_angle = the median triangulation
   angle of its points (0 without any); PLANAR_OR_PANORAMIC becomes PANORAMIC (tri_angle 0) when |t| = 0, else
   PLANAR.  estimated = 1 for those configs; any other config passes through (estimated 0, config unchanged, zero
   outputs).  Two results the reference leaves undefined are defined here: the four essential candidates are ordered
   (R1, t), (R2, t), (R1, -t), (R2, -t) with t's largest-magnitude component positive and trace R1 >= trace R2, and
   a homography of which no candidate keeps a point (a pure rotation: R = the normalised H, t = 0) gives candidate 0
   with tri_angle 0.  An image, camera or keypoint index out of range is PSFM_ERR_INVALID before anything runs.
   With no pair nothing is launched; with no inlier match only the per-pair kernels run. */
int psfm_two_view_relative_poses(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                 const int32_t* image_camera, const double* cameras, int32_t num_cameras,
                                 int64_t num_pairs, const int32_t* pair_images, const int32_t* config,
                                 const double* E, const double* F, const double* H, const int64_t* inlier_ptr,
                                 const uint32_t* inlier_matches, double* qvec, double* tvec, double* tri_angle,
                                 int32_t* config_out, int64_t* num_points3D, uint8_t* estimated);

/* RobustRotationEstimator::Options (global/robust_rotation_estimator.h:61-89); NULL gives these defaults, which are
   what sfm/main_sfm.py runs.  Check() (robust_rotation_estimator.cc:54-62): every field > 0. */
typedef struct {
  int32_t max_num_l1_iterations;            /* 5: L1 rounds (at most PSFM_ROTATION_MAX_L1_ROUNDS here) */
  double l1_step_convergence_threshold;     /* 0.001 */
  int32_t max_num_irls_iterations;          /* 100 */
  double irls_step_convergence_threshold;   /* 0.001 */
  double irls_loss_parameter_sigma;         /* DegToRad(5.0) */
  double rotation_filter_max_degrees;       /* 5.0 */
} psfm_rotation_options;

/* The ADMM cap doubles every L1 round from 5 (robust_rotation_estimator.cc:164, 179): 16 rounds end at 163,840
   iterations, and the reference's int cap overflows past 28. */
#define PSFM_ROTATION_MAX_L1_ROUNDS 16

typedef struct {
  int32_t num_l1_rounds;                               /* L1Solver::Solve calls */
  int32_t admm_iterations[PSFM_ROTATION_MAX_L1_ROUNDS]; /* ADMM iterations of each round (0 past the last) */
  int32_t num_irls_iterations;
  double l1_final_step;                                /* ComputeAverageStepSize after the last L1 round */
  double irls_final_step;                              /* ... after the last IRLS iteration */
  int32_t gauge_image;                                 /* image index held at the identity (-1: none) */
  int32_t num_images_connected, num_pairs_connected;   /* after the first RemoveDisconnectedViewPairs */
  int32_t num_images_kept, num_pairs_kept;             /* after the rotation filter and the second one */
  int64_t num_launches;                                /* kernels this call launched */
  double host_ms, device_ms;                           /* graph work on the host, device loop (wall, synchronised) */
} psfm_rotation_summary;

void psfm_rotation_default_options(psfm_rotation_options* opts);

/* EstimateGlobalRotations (global/robust_rotation_estimator.cc:310-331), the first step of
   GlobalMapper's reconstruction (controllers/global_mapper.cc:136-184, sfm/global_mapper.cc:89-92)
   (csrc/rotation_averaging.cu).  Pairs: pair_images [num_pairs][2] image indices (image 1, image 2), qvec
   [num_pairs][4] (w, x, y, z) the relative rotation 2_R_1 (world-to-camera orientations: R2 = R12 R1),
   num_correspondences [num_pairs], has_pose [num_pairs] (NULL: all 1).  A pair takes part when has_pose is set and
   its qvec is finite (AllPairs(only_with_pose), base/correspondence_graph.cc:92-100, 148-150).  Steps:
   RemoveDisconnectedViewPairs (global/filter_util.cc:382-431), OrientationsFromMaximumSpanningTree
   (global/orientation_util.cc:102-178), RobustRotationEstimator::EstimateRotations (L1 regression by ADMM, then
   IRLS, robust_rotation_estimator.cc:80-250), FilterViewPairsFromOrientation (filter_util.cc:271-325) and
   RemoveDisconnectedViewPairs again.  Defined here where the reference follows hash order: among equally large
   components the one holding the smallest image index is kept; the gauge image and spanning-tree root is the
   smallest image index of the component (identity orientation); spanning-tree ties go by (-num_correspondences,
   image 1, image 2).
   Out: orientations [num_images][4] (w, x, y, z; zero without one), has_orientation [num_images] (the images of the
   kept component, as the reference keeps them even when the second pruning leaves them no pair), pair_kept
   [num_pairs], summary (nullable).  PSFM_ERR_INVALID before anything runs for an image index out of range, a pair of
   an image with itself, an unordered pair listed twice, or options that fail Check(); PSFM_ERR_UNSUPPORTED for more
   than 8192 images in the kept component (the dense factor) or more than PSFM_ROTATION_MAX_L1_ROUNDS L1 rounds;
   PSFM_NO_ROTATIONS, with nothing launched, when no posed pair exists. */
int psfm_estimate_global_rotations(int32_t num_images, int64_t num_pairs, const int32_t* pair_images,
                                   const double* qvec, const int32_t* num_correspondences, const uint8_t* has_pose,
                                   const psfm_rotation_options* opts, double* orientations, uint8_t* has_orientation,
                                   uint8_t* pair_kept, psfm_rotation_summary* summary);

/* GlobalMapper::OptimizePairwiseTranslations (sfm/global_mapper.cc:106-109 -> BatchOptimizeRelativePositionWithKnownRotation,
   global/known_rotation_util.cc:195-229): every used pair's translation direction re-estimated from all of its inlier
   matches under the image orientations, with psfm_known_rotation_translations' kernel (csrc/init_geometry.cu), the
   keypoints gathered and normalised (SIMPLE_PINHOLE ImageToWorld) on the device.  Images and pairs as
   psfm_two_view_relative_poses takes them; orientations [num_images][4] (w, x, y, z world-to-camera, normally
   psfm_estimate_global_rotations' output), pair_used [num_pairs] (NULL: every pair; normally its pair_kept).
   Out: tvec [num_pairs][3] unit relative positions, iterations [num_pairs] IRLS iterations; an unused pair gets zeros.
   The result is bit-identical to psfm_known_rotation_translations on points normalised as (x - cx) / f in double.
   PSFM_ERR_INVALID before anything runs for an image, camera or keypoint index out of range, or a used pair whose
   image has a zero or non-finite orientation. */
int psfm_optimize_pairwise_translations(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                        const int32_t* image_camera, const double* cameras, int32_t num_cameras,
                                        int64_t num_pairs, const int32_t* pair_images, const int64_t* inlier_ptr,
                                        const uint32_t* inlier_matches, const double* orientations,
                                        const uint8_t* pair_used, double* tvec, int32_t* iterations);

/* theia::ConstrainedL1Solver::Options, which LeastUnsquaredDeviationPositionEstimator constructs with its defaults
   (global/least_unsquared_deviation_position_estimator.cc:161); NULL gives these defaults.  They are recalled, not
   vendored (csrc/position_recalled.cuh).  Check(): max_num_iterations > 0, rho > 0, 0 < alpha < 2, both tolerances
   > 0, all finite.  The reference LUD options max_num_iterations, max_num_reweighted_iterations and
   convergence_criterion never reach the solver there, so they are not mirrored. */
typedef struct {
  int32_t max_num_iterations;   /* 1000 */
  double rho;                   /* 10.0 */
  double alpha;                 /* 1.2 (over-relaxation) */
  double absolute_tolerance;    /* 1e-4 */
  double relative_tolerance;    /* 1e-2 */
} psfm_lud_options;

typedef struct {
  int32_t gauge_image;               /* image index fixed at the origin */
  int32_t num_views;                 /* images of the used pairs */
  int32_t num_pairs_used;
  int32_t admm_iterations;           /* ConstrainedL1Solver iterations run */
  int32_t admm_iterations_queued;    /* iterations launched (in chunks of 32 behind the done flag) */
  int32_t converged;                 /* 1: the stopping test passed; 0: max_num_iterations ran out */
  double primal_residual, primal_tolerance;   /* |A~x - z - b~| and its bound, last iteration */
  double dual_residual, dual_tolerance;       /* |rho A~'(z - z_old)| and its bound, last iteration */
  int64_t num_launches;              /* kernels this call launched: 4 + 4 * admm_iterations_queued */
  double host_ms;                    /* validation and graph work on the host */
  double build_ms, factor_ms, inverse_ms;     /* building S, factoring it, inverting it (CUDA events) */
  double admm_ms;                    /* the ADMM loop with its control reads (wall, synchronised) */
} psfm_position_summary;

void psfm_lud_default_options(psfm_lud_options* opts);

/* GlobalMapper::EstimatePositions (sfm/global_mapper.cc:111-132) with the default method "lud"
   (LeastUnsquaredDeviationPositionEstimator, use_scale_constraints = false, no 1DSfM filter), then the positions'
   part of RegisterAllImages (:140-160), in one call (csrc/position_estimation.cu).  Pairs: pair_images
   [num_pairs][2] (image 1, image 2), pair_tvec [num_pairs][3] the relative translation (psfm_optimize_pairwise_translations),
   pair_used [num_pairs] (NULL: every pair).  Images: orientations [num_images][4] (w, x, y, z world-to-camera),
   has_orientation [num_images] (NULL: all 1).  Solves min sum_k |c1 - c2 - s_k R2' t_k|_1 subject to s_k >= 1 by
   ADMM (theia::ConstrainedL1Solver), with the positions' normal equations reduced to a 3 x 3-block graph Laplacian
   that is factored and inverted once.
   Out: positions [num_images][3] (camera centres), has_position [num_images] (the images of the used pairs), image_tvec
   [num_images][3] = -QuaternionRotatePoint(q, c) (zero without a position), scales [num_pairs] (0 for unused pairs), summary
   (nullable).  Defined here where the reference follows hash order: the gauge is the smallest image index among the
   views, fixed at the origin (any other choice moves every position by one common vector).
   PSFM_ERR_INVALID before anything runs for: no used pair; an image index out of range, a pair of an image with
   itself, an unordered pair listed twice; a used pair touching an image without an orientation; a non-finite
   orientation or pair tvec; used pairs that do not form one connected graph (S singular); options that fail Check().
   PSFM_ERR_UNSUPPORTED before anything runs for 3 (V - 1) > 8190 (more than 2731 views: the dense factor's bound).
   PSFM_ERR_NO_DEVICE without a device (there is no CPU path); PSFM_ERR_INVALID after the launches when S is not
   numerically positive definite. */
int psfm_estimate_global_positions(int32_t num_images, int64_t num_pairs, const int32_t* pair_images,
                                   const double* pair_tvec, const double* orientations, const uint8_t* has_orientation,
                                   const uint8_t* pair_used, const psfm_lud_options* opts, double* positions,
                                   uint8_t* has_position, double* image_tvec, double* scales,
                                   psfm_position_summary* summary);

/* IncrementalTriangulator::Options (sfm/incremental_triangulator.h:46-89): the fields TriangulateImage reads; NULL
   gives these defaults (the bogus-camera thresholds are gcolmap's overrides, controllers/global_mapper.cc:73-79, equal
   to the defaults).  Check() (incremental_triangulator.cc:40-53): max_transitivity >= 0, both angle errors > 0,
   min_angle > 0; both focal ratios > 0, max_extra_param >= 0, all finite. */
typedef struct {
  int32_t max_transitivity;           /* 1 (only 1 is supported) */
  double create_max_angle_error;      /* 2.0 degrees */
  double continue_max_angle_error;    /* 2.0 degrees */
  double min_angle;                   /* 1.5 degrees */
  int32_t ignore_two_view_tracks;     /* 1 */
  double min_focal_length_ratio;      /* 0.1 */
  double max_focal_length_ratio;      /* 10.0 */
  double max_extra_param;             /* 1.0 (SIMPLE_PINHOLE has no extra parameter) */
} psfm_triangulator_options;

typedef struct {
  int64_t num_components;             /* connected components of the graph over registered, non-bogus images */
  int64_t largest_component;          /* observations in the largest one */
  int64_t num_points3D;               /* points created (Create) */
  int64_t num_continued;              /* observations attached to an existing point (Continue) */
  int64_t num_ransac_trials;          /* samples drawn by every EstimateTriangulation */
  int64_t num_local_estimates;        /* multi-view DLTs of the local optimisation */
  int64_t num_launches;               /* kernels this call launched (fixed per call) */
  double host_ms;                     /* validation and per-image tables on the host */
  double graph_ms, components_ms, replay_ms, assembly_ms;   /* CUDA events per phase */
} psfm_triangulation_summary;

void psfm_triangulator_default_options(psfm_triangulator_options* opts);

typedef struct psfm_triangulation psfm_triangulation;
/* GlobalMapper::TriangulateAllPoints (sfm/global_mapper.cc:232-247): IncrementalTriangulator::TriangulateImage
   (sfm/incremental_triangulator.cc:61-119) of every registered image in index order, every Point2D in index order:
   Find, Continue, Create with EstimateTriangulation (LO-RANSAC over CombinationSampler) (csrc/triangulation.cu).
   Images and pairs as psfm_optimize_pairwise_translations takes them, images in ascending image_id; camera_size
   [num_cameras][2] (width, height); pair_used [num_pairs] (NULL: every pair) is the database cache's pair set (at
   least min_num_matches inliers, config not UNDEFINED), which the correspondence graph holds whole; orientations
   [num_images][4] (w, x, y, z) and image_tvec [num_images][3] world-to-camera, registered [num_images].
   The correspondence graph is built as CorrespondenceGraph::AddCorrespondences builds it (a match is dropped when
   either point already has an accepted correspondence into the other image).  Defined here where the reference follows
   hash order: the pairs enter the graph in the order of these arrays (pair_id order from a database).  Angular errors
   are evaluated as atan2(|r1 x r2|, r1 . r2), the reference's acos of the normalised dot product without its loss of
   accuracy near zero.
   Runs everything; num_points3D and num_track_elements receive the result's sizes, psfm_triangulation_result copies
   it.  PSFM_ERR_INVALID before any launch for: an image, camera or keypoint index out of range, a pair of an image
   with itself, an unordered pair listed twice, a registered image with a non-finite pose, a camera size <= 0, options
   that fail Check().  PSFM_ERR_UNSUPPORTED for max_transitivity != 1 or 2^31 - 1 keypoints or more.
   PSFM_ERR_NO_DEVICE without a device. */
int psfm_triangulation_create(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                              const int32_t* image_camera, const double* cameras, int32_t num_cameras,
                              const int32_t* camera_size, int64_t num_pairs, const int32_t* pair_images,
                              const int64_t* inlier_ptr, const uint32_t* inlier_matches, const uint8_t* pair_used,
                              const double* orientations, const double* image_tvec, const uint8_t* registered,
                              const psfm_triangulator_options* opts, psfm_triangulation** out, int64_t* num_points3D,
                              int64_t* num_track_elements);
/* Points in the reference's AddPoint3D order (ids 1, 2, ... are rows 0, 1, ...): xyz [P][3], track_ptr [P + 1], track
   elements [E] (track_image, track_point2D) in the reference's element order (Create's inliers in list order, then
   Continue's appends), point3D_of_keypoint [K] (row of the keypoint's point, -1 without one), summary (nullable).
   Any output pointer may be NULL. */
int psfm_triangulation_result(const psfm_triangulation* h, double* xyz, int64_t* track_ptr, int32_t* track_image,
                              int32_t* track_point2D, int64_t* point3D_of_keypoint, psfm_triangulation_summary* summary);
void psfm_triangulation_destroy(psfm_triangulation* h);

/* TwoViewGeometry::Options with its RANSACOptions, as `colmap matches_importer --match_type pairs` takes them; NULL
   gives what sfm/import_feature_matches.py:106-117 runs.  Check(): max_error > 0, confidence, min_inlier_ratio,
   watermark_min_inlier_ratio and watermark_border_size in [0, 1], 0 <= min_num_trials <= max_num_trials,
   min_num_inliers >= 0, dyn_num_trials_multiplier > 0, max_H_inlier_ratio >= 0, all finite. */
typedef struct {
  double max_error;                    /* 4.0 px */
  double confidence;                   /* 0.999 */
  int32_t max_num_trials;              /* 20000 */
  int32_t min_num_trials;              /* 0 */
  double min_inlier_ratio;             /* 0.1 */
  int32_t min_num_inliers;             /* 15 */
  double dyn_num_trials_multiplier;    /* 3.0 */
  double max_H_inlier_ratio;           /* 0.8 */
  int32_t detect_watermark;            /* 1 */
  double watermark_min_inlier_ratio;   /* 0.7 */
  double watermark_border_size;        /* 0.1 */
  uint64_t random_seed;                /* 0 */
} psfm_verification_options;

/* per estimator kind: [0] F, [1] H, [2] the watermark translation */
typedef struct {
  int64_t num_trials[3];               /* samples the sequential LORANSAC loop draws */
  int64_t num_trials_scored[3];        /* samples the device scored (the same: trials run in sequential order) */
  int64_t num_local_rounds[3];         /* local-optimisation rounds */
  int64_t num_config[8];               /* pairs per config (UNDEFINED 0 .. WATERMARK 7) */
  int64_t num_launches;                /* kernels this call launched: 3 with pairs, 0 without */
  double host_ms;                      /* validation on the host */
  double gather_ms, ransac_ms, compact_ms;   /* CUDA events per phase */
} psfm_verification_summary;

void psfm_verification_default_options(psfm_verification_options* opts);

/* The geometric verification of `colmap matches_importer --match_type pairs` (TwoViewGeometryVerifier ->
   TwoViewGeometry::EstimateUncalibrated) of every image pair at once (csrc/verification.cu): raw matches in, the rows of
   the two_view_geometries table out.  Images as psfm_two_view_relative_poses takes them, camera_size [num_cameras][2]
   (width, height), prior_focal_length [num_cameras] (NULL: none).  Pairs in database orientation: pair_images
   [num_pairs][2] (image 1 = the smaller image_id), match_ptr [num_pairs + 1], matches [M][2] (point2D_idx1,
   point2D_idx2).
   Per pair: fewer than min_num_inliers raw matches gives config UNDEFINED (0), no inliers and zero F / H.  Otherwise
   LORANSAC of the seven-point F (eight-point local step, squared Sampson error) and of the normalised-DLT H (squared
   transfer error), both against max_error^2: DEGENERATE (1) when neither succeeded or both have fewer than
   min_num_inliers inliers, else PLANAR_OR_PANORAMIC (6) when H inliers / F inliers > max_H_inlier_ratio, else
   UNCALIBRATED (3); the inlier matches are F's inliers in match order; with detect_watermark, WATERMARK (7) when
   DetectWatermark finds them translated in the border strip.  E is zero.
   Defined here, the same way in oracle/verification_oracle.py: each trial's sample comes from a SplitMix64 stream keyed
   by (random_seed, pair, kind, trial) (kind 0 F, 1 H, 2 watermark); the seven-point models are ordered by (F00, F01, ...)
   after F22 = 1; stored F and H have unit Frobenius norm with the largest-magnitude entry positive.
   Out: config [num_pairs], F / E / H [num_pairs][9] row-major, inlier_ptr [num_pairs + 1], inlier_matches (room for
   match_ptr[num_pairs] rows; inlier_ptr gives what was written), pair_trials [num_pairs][3] the samples drawn per kind
   (may be NULL), summary (may be NULL).
   PSFM_ERR_INVALID before any launch for an image, camera or keypoint index out of range, a pair of an image with
   itself, an unordered pair listed twice, a camera size <= 0, or options that fail Check().  PSFM_ERR_UNSUPPORTED for a
   pair whose two cameras both have a prior focal length (EstimateCalibrated) or a pair of 2^31 matches or more.
   PSFM_ERR_NO_DEVICE without a device.  With no pair nothing is launched. */
int psfm_verify_two_view_geometries(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                    const int32_t* image_camera, int32_t num_cameras, const int32_t* camera_size,
                                    const uint8_t* prior_focal_length, int64_t num_pairs, const int32_t* pair_images,
                                    const int64_t* match_ptr, const uint32_t* matches,
                                    const psfm_verification_options* opts, int32_t* config, double* F, double* E,
                                    double* H, int64_t* inlier_ptr, uint32_t* inlier_matches, int32_t* pair_trials,
                                    psfm_verification_summary* summary);
/* psfm_verify_two_view_geometries on a resident match table (psfm_matches_table): the same launches and the same
   outputs as the host entry given psfm_match_table_result's arrays.  image_camera [num_images] over num_cameras
   cameras, camera_size, prior_focal_length and opts as there.  The table holds valid keypoint indices and distinct
   pairs by construction; the other checks and statuses are the host entry's. */
int psfm_match_table_verify(const psfm_match_table* t, const int32_t* image_camera, int32_t num_cameras,
                            const int32_t* camera_size, const uint8_t* prior_focal_length,
                            const psfm_verification_options* opts, int32_t* config, double* F, double* E, double* H,
                            int64_t* inlier_ptr, uint32_t* inlier_matches, int32_t* pair_trials,
                            psfm_verification_summary* summary);

/* ------------------------------------------------------------------------- */
/* HP2 — global bundle adjustment                                             */
/* ------------------------------------------------------------------------- */

typedef enum { PSFM_LOSS_TRIVIAL = 0, PSFM_LOSS_SOFT_L1 = 1, PSFM_LOSS_CAUCHY = 2 } psfm_loss_type;

typedef enum {
  /* The reference rule (bundle_adjustment.cc:276-286): <=1000 images -> exact Schur
     step (DENSE_/SPARSE_SCHUR), otherwise ITERATIVE_SCHUR + SCHUR_JACOBI. */
  PSFM_BA_SOLVER_AUTO = 0,
  /* Exact Gauss-Newton/LM step, as DENSE_/SPARSE_SCHUR: the reduced camera system is
     formed explicitly on the device and factorised (banded Cholesky).  When that is not
     possible (principal point refined, or > 4 GB of reduced system) the same PCG is driven
     to `exact_r_tolerance` instead. */
  PSFM_BA_SOLVER_EXACT_SCHUR = 1,
  /* Ceres ITERATIVE_SCHUR + SCHUR_JACOBI semantics: eta forcing, x0 = 0,
     max_linear_solver_iterations. The throughput mode. */
  PSFM_BA_SOLVER_ITERATIVE_SCHUR = 2
} psfm_ba_linear_solver;

/* Mirrors colmap::BundleAdjustmentOptions (bundle_adjustment.h:48-102) and the Ceres
   options the reference sets (controllers/global_mapper.cc:41-71). */
typedef struct {
  int32_t loss_function_type;        /* psfm_loss_type; global BA uses SOFT_L1 (:68-69) */
  double loss_function_scale;        /* 1.0 */
  int32_t refine_focal_length;       /* bundle_adjustment.h:57 */
  int32_t refine_principal_point;    /* :60 */
  int32_t refine_extra_params;       /* :63 (SIMPLE_PINHOLE has none) */
  int32_t refine_extrinsics;         /* :66 */
  int32_t refine_rotation;           /* :69 */
  int32_t print_summary;             /* :72 — prints the PrintSolverSummary block */
  int32_t minimizer_progress_to_stdout;
  double function_tolerance;         /* global BA: 1e-6 (controllers/global_mapper.cc:44) */
  double gradient_tolerance;         /* 1.0  (:45) */
  double parameter_tolerance;        /* 1e-8 (:46) */
  int32_t max_num_iterations;        /* 50   (:47) */
  int32_t max_linear_solver_iterations; /* 100 (:48) */
  int32_t max_num_consecutive_invalid_steps; /* 10 (bundle_adjustment.h:89) */
  int32_t linear_solver;             /* psfm_ba_linear_solver */
  double eta;                        /* 0.1 Ceres default (forcing sequence) */
  double exact_r_tolerance;          /* 1e-10: |r|/|b| target when EXACT_SCHUR has to fall back to PCG (reduced system too
                                        large to factor, principal point refined) */
  int32_t exact_max_iterations;      /* 0 -> min(20000, max(1000, 5 * reduced dimension)) */
  double initial_trust_region_radius;/* 1e4 */
  double max_trust_region_radius;    /* 1e16 */
  double min_trust_region_radius;    /* 1e-32 */
  double min_relative_decrease;      /* 1e-3 */
  double min_lm_diagonal;            /* 1e-6 */
  double max_lm_diagonal;            /* 1e32 */
  int32_t jacobi_scaling;            /* 1 */
  int32_t pcg_check_period;          /* host polls the device termination flag every
                                        this many PCG iterations (0 -> 4) */
} psfm_ba_options;

/*
 * The flattened problem BundleAdjuster::SetUp builds from (Reconstruction, Config)
 * (bundle_adjustment.cc:326-447).  One residual block per observation = one Point2D
 * with a Point3D in an image of the config (:366-411).  Camera model: SIMPLE_PINHOLE
 * (f, cx, cy) — the only one the pipeline creates (sfm/import_feature_matches.py:50-58).
 *
 * qvec/tvec/xyz/cam_params are updated IN PLACE like the reference does through
 * Image::Qvec()/Tvec(), Point3D::XYZ(), Camera::ParamsData() (:357-359,410).
 * All qvecs of images are normalised on entry (:355).
 */
typedef struct {
  int32_t num_images;                /* F */
  int32_t num_points;                /* P */
  int32_t num_observations;          /* M */
  int32_t num_cameras;               /* C */
  double* qvec;                      /* [F*4] w,x,y,z world-to-camera */
  double* tvec;                      /* [F*3] */
  double* xyz;                       /* [P*3] */
  double* cam_params;                /* [C*3] f,cx,cy */
  const int32_t* obs_image;          /* [M] index into images */
  const int32_t* obs_point;          /* [M] index into points */
  const double* obs_xy;              /* [M*2] Point2D::XY() */
  const int32_t* image_camera;       /* [F] index into cameras */
  const uint8_t* pose_constant;      /* [F] BundleAdjustmentConfig::SetConstantPose; may be NULL */
  const uint8_t* tvec_constant_mask; /* [F] bit i set => tvec[i] constant (SetConstantTvec); may be NULL */
  const uint8_t* camera_constant;    /* [C] BundleAdjustmentConfig::SetConstantCamera; may be NULL */
} psfm_ba_problem;

/* Mirrors the fields PrintSolverSummary reads (bundle_adjustment.cc:560-614) plus
   device timings. */
typedef struct {
  int32_t num_residuals_reduced;
  int32_t num_effective_parameters_reduced;
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t num_iterations;            /* LM iterations incl. iteration 0's evaluation excluded */
  int32_t num_linear_iterations;     /* total PCG iterations */
  int32_t termination;               /* psfm_termination */
  double initial_cost;
  double final_cost;
  double total_time_in_seconds;      /* wall time of the solve */
  double device_ms;                  /* CUDA-event time of the LM loop */
  double linearize_ms;               /* summed CUDA-event time of the Jacobian sweep */
  double schur_product_ms;           /* summed time of the implicit S*p kernels */
  int32_t num_linearize;             /* launches of the Jacobian sweep */
  int32_t num_schur_products;        /* applications of S*p */
  int32_t linear_solver_used;        /* psfm_ba_linear_solver actually used */
  int32_t world_size;
  /* explicit (exact) reduced-system path, summed CUDA-event times */
  int32_t num_explicit_solves;
  double schur_w_ms;                 /* per-observation W, W H~ */
  double schur_pairs_ms;             /* image-pair block products */
  double cholesky_ms;                /* assembly + blocked Cholesky + triangular solves */
  /* fused tile path (k_schur_tile): schur_w_ms is its time, schur_pairs_ms stays 0 */
  int64_t num_pair_entries;          /* observation pairs of the Schur complement on this rank */
  int32_t num_pair_tasks;            /* (tile, image pair) runs of those entries */
  int32_t explicit_fused;            /* 1: k_schur_tile, 0: k_schur_w + k_schur_pairs */
  int32_t explicit_dense_tiles;      /* k_schur_tile tiles whose pair blocks are one dense tensor-core
                                        product (the others run the pair loop) */
} psfm_ba_summary;

void psfm_ba_default_options(psfm_ba_options* o);          /* bundle_adjustment.h defaults */
void psfm_ba_global_options(psfm_ba_options* o);           /* controllers/global_mapper.cc:41-71 */

/* Drop-in for BundleAdjuster(options, config).Solve(reconstruction) on HOST buffers:
   uploads, solves on the GPU, writes the refined parameters back.  Returns PSFM_OK for
   any termination (the reference returns true regardless, :306-319),
   PSFM_ZERO_RESIDUALS when M == 0. */
int psfm_ba_solve(psfm_ba_problem* problem, const psfm_ba_options* opts,
                  psfm_ba_summary* summary);

/* Resident-problem API: structure and observations uploaded once, state re-set and
   solved many times (the refinement loop of controllers/global_mapper.cc:253-268, and
   bench.py's device-resident `value`). */
typedef struct psfm_ba_solver psfm_ba_solver;
int psfm_ba_create(const psfm_ba_problem* problem, psfm_ba_solver** out);
/* Host -> device copy of qvec/tvec/xyz/cam_params (any may be NULL = keep). */
int psfm_ba_set_state(psfm_ba_solver* s, const double* qvec, const double* tvec,
                      const double* xyz, const double* cam_params);
int psfm_ba_run(psfm_ba_solver* s, const psfm_ba_options* opts, psfm_ba_summary* summary);
/* Writes the state back (any pointer may be NULL).  xyz: only the points this solver observes
   are written (Ceres never touches a Point3D without a residual either); on a shard of a
   multi-GPU problem those are the shard's own points. */
int psfm_ba_get_state(psfm_ba_solver* s, double* qvec, double* tvec, double* xyz,
                      double* cam_params);
void psfm_ba_destroy(psfm_ba_solver* s);

/* Diagnostics used by the parity tests: evaluate cost / residuals / gradient at the
   current state without stepping.  Any output may be NULL.
     residuals [2*M] loss-corrected, in the caller's observation order
     gradient_cam [6*F + 3*C] tangent-space J^T r (rot3,t3 per image, then f,cx,cy per camera)
     gradient_pts [3*P] */
int psfm_ba_evaluate(psfm_ba_solver* s, const psfm_ba_options* opts, double* cost,
                     double* residuals, double* gradient_cam, double* gradient_pts);

/* One linear solve (iteration-0 linearisation + Jacobi scaling, LM diagonal from
   `radius`, Schur elimination, PCG, back-substitution) without moving the state: writes
   the step in the scaled tangent space, camera slots [6F+3C] and points [3P].  Used by
   the parity tests to compare the PCG step with the oracle's Cholesky step. */
int psfm_ba_linear_step(psfm_ba_solver* s, const psfm_ba_options* opts, double radius,
                        double* step_cam, double* step_pts, int32_t* num_linear_iterations);

/* ------------------------------------------------------------------------- */
/* Refinement loop around the global BA, on the resident solver (the caller's  */
/* observations stay in HBM; filters clear bits of an ALIVE mask and the tile   */
/* structure is re-packed on the device).                                       */
/*   IterativeGlobalRefinement   controllers/global_mapper.cc:245-271           */
/*   AdjustGlobalBundle          sfm/global_mapper.cc:402-448                   */
/*   filters / Normalize         base/reconstruction.cc:373-468,697-729,1321-1434 */
/* All of them act on the solver's current state (psfm_ba_set_state / the       */
/* result of the last psfm_ba_run).  Counts are the reference's num_filtered,   */
/* summed over the ranks of a sharded problem.                                  */
/* ------------------------------------------------------------------------- */
#define PSFM_BA_MAX_REFINEMENTS 8

typedef struct psfm_ba_refine_options {
  int32_t max_refinements;          /* 5      ba_global_max_refinements */
  double max_refinement_change;     /* 5e-4   ba_global_max_refinement_change */
  double filter_max_reproj_error;   /* 4 px   Mapper filter_max_reproj_error */
  double filter_min_tri_angle;      /* 1.5 deg */
  double normalize_extent;          /* 10 */
  double normalize_p0;              /* 0.1 */
  double normalize_p1;              /* 0.9 */
} psfm_ba_refine_options;

typedef struct psfm_ba_refine_report {
  int32_t num_rounds;
  int32_t ba_iterations[PSFM_BA_MAX_REFINEMENTS];
  int32_t ba_termination[PSFM_BA_MAX_REFINEMENTS];
  int64_t num_observations[PSFM_BA_MAX_REFINEMENTS];     /* ComputeNumObservations() before the round */
  int64_t num_negative_depth[PSFM_BA_MAX_REFINEMENTS];   /* FilterObservationsWithNegativeDepth */
  int64_t num_changed[PSFM_BA_MAX_REFINEMENTS];          /* FilterAllPoints3D */
  double changed[PSFM_BA_MAX_REFINEMENTS];               /* num_changed / num_observations */
  double ba_final_cost[PSFM_BA_MAX_REFINEMENTS];
  int64_t final_num_observations;
  double total_time_in_seconds;
} psfm_ba_refine_report;

void psfm_ba_default_refine_options(psfm_ba_refine_options* r);
/* Reconstruction::FilterObservationsWithNegativeDepth */
int psfm_ba_filter_negative_depth(psfm_ba_solver* s, int64_t* num_filtered);
/* Reconstruction::FilterAllPoints3D(max_reproj_error, min_tri_angle [deg]) */
int psfm_ba_filter_points(psfm_ba_solver* s, double max_reproj_error, double min_tri_angle_deg, int64_t* num_filtered);
/* Reconstruction::Normalize(extent, p0, p1, use_images = true); translation [3], scale may be NULL */
int psfm_ba_normalize(psfm_ba_solver* s, double extent, double p0, double p1, double* translation, double* scale);
/* observations still in the problem (all ranks) */
int psfm_ba_num_observations(psfm_ba_solver* s, int64_t* num_alive);
/* alive [M] over the caller's observations: 1 = still in the problem (this rank's shard) */
int psfm_ba_get_observation_mask(psfm_ba_solver* s, uint8_t* alive);
/* Point3D::Error() as the last point filter set it, [P], NaN where not set */
int psfm_ba_get_point_errors(psfm_ba_solver* s, double* error);
/* One IterativeGlobalRefinement pass with `opts` (GlobalBundleAdjustment options with the pass's
   refine_* flags; the "< 10 images" tightening of AdjustGlobalBundle is applied inside). */
int psfm_ba_iterative_refinement(psfm_ba_solver* s, const psfm_ba_options* opts, const psfm_ba_refine_options* ropts,
                                 psfm_ba_refine_report* report);

/* ------------------------------------------------------------------------- */
/* Triangulation -> bundle adjustment -> model, on the device (DESIGN.md §4.9) */
/* ------------------------------------------------------------------------- */
/* The resident problem of a triangulation (psfm_triangulation_create) without its keypoints or point3D_of_keypoint
   leaving the device: the problem ba.flatten builds from Triangulation.to_reconstruction with every registered image
   in the config.  Problem images are the registered images in ascending index, problem cameras the cameras they use
   in ascending index, problem points the triangulation's rows; observations are every keypoint of a registered image
   with a point, images first, keypoints in index order.
     qvec [F][4], tvec [F][3]          poses of the triangulation's F images (rows of unregistered images are ignored)
     cam_params [C][3]                 f, cx, cy of its C cameras
     pose_constant, tvec_constant_mask [F], camera_constant [C]: as in psfm_ba_problem, indexed like the triangulation;
                                       may be NULL
   num_images, num_cameras, num_observations (may be NULL) receive the problem's sizes.  PSFM_ERR_INVALID for a NULL
   argument or no registered image, PSFM_ERR_UNSUPPORTED with a multi-GPU communicator.  The triangulation may be
   destroyed once this returns. */
int psfm_ba_create_from_triangulation(const psfm_triangulation* tri, const double* qvec, const double* tvec,
                                      const double* cam_params, const uint8_t* pose_constant,
                                      const uint8_t* tvec_constant_mask, const uint8_t* camera_constant,
                                      psfm_ba_solver** out, int32_t* num_images, int32_t* num_cameras,
                                      int64_t* num_observations);
/* The refined model of a solver made by psfm_ba_create_from_triangulation, in the triangulation's layout:
     qvec [F][4], tvec [F][3], cam_params [C][3]: the problem's rows are written, the others left as they are
     xyz [P][3]                        every row (a point no observation keeps holds its triangulated position)
     track_ptr [P + 1]                 a point whose observations were all filtered has length 0
     track_image, track_point2D        room for num_observations elements; track_ptr[P] are written: (image index,
                                       point2D_idx) of the alive observations, by point, images ascending within a track
     point3D_of_keypoint [K]           point row of every alive observation's keypoint, -1 elsewhere
   Point errors come from psfm_ba_get_point_errors. */
int psfm_ba_get_model(psfm_ba_solver* s, double* qvec, double* tvec, double* cam_params, double* xyz, int64_t* track_ptr,
                      int32_t* track_image, int32_t* track_point2D, int64_t* point3D_of_keypoint);
/* The observations the solver was created with, in order (any output may be NULL): obs_image [M], obs_point [M],
   obs_xy [M][2], point2D_idx [M] (a solver made by psfm_ba_create_from_triangulation only). */
int psfm_ba_get_observations(psfm_ba_solver* s, int32_t* obs_image, int32_t* obs_point, double* obs_xy,
                             int32_t* point2D_idx);

/* ------------------------------------------------------------------------- */
/* The model -> sparse depth maps and their display images                   */
/* (sfm/convert.py:43-96, csrc/convert.cu).  Host buffers in, host buffers out. */
/* ------------------------------------------------------------------------- */
typedef struct psfm_convert psfm_convert;
typedef struct {
  int32_t num_batches;       /* batches of images the memory budget allowed */
  int32_t pad;
  double upload_ms;          /* create: the model's upload (CUDA events) */
  double kernel_ms;          /* create: the counting pass; result: every batch's kernels, summed */
  double d2h_ms;             /* result: every batch's device-to-pinned copies, summed (they overlap the next batch) */
  double alloc_ms;           /* host wall time of the allocations: create, the model's buffers and the counting slot;
                                result, the two batch slots with their pinned buffers (its first call only) */
  double host_copy_ms;       /* result: host wall time of the copies from the pinned buffers to the caller's */
} psfm_convert_summary;
/* Uploads a model and counts each image's valid pixels (depth > 0 after the last keypoint in keypoint order has
   claimed every pixel).
     cameras     camera_size [num_cameras][2] (width, height), each > 0 and at most 2^31 - 1 pixels
     images      qvec [F][4] (not renormalised), tvec [F][3], image_camera [F], keypoint_ptr [F + 1] over
                 keypoints [K][2] and point_row [K] (row of xyz, -1: no point), K < 2^31
     points      xyz [num_points][3]
     gray_lut    [256] grey level of each colormap entry; a NaN display value is black
     memory_budget  bytes of device memory for the two batch slots (16 B per pixel, 32 B per keypoint each); a batch
                 holds at least one image and at most 65,535
   valid_count [F] receives each image's valid pixels, batch_ptr [F + 1] the batches (batch j holds images
   batch_ptr[j] .. batch_ptr[j + 1], summary->num_batches of them); summary may be NULL.  PSFM_ERR_INVALID before any launch for a
   bad camera size, a camera index or point row out of range, or a bad keypoint_ptr; PSFM_ERR_NO_DEVICE without a
   device. */
int psfm_convert_create(int32_t num_cameras, const int32_t* camera_size, int32_t num_images, const double* qvec,
                        const double* tvec, const int32_t* image_camera, const int64_t* keypoint_ptr,
                        const double* keypoints, const int32_t* point_row, int64_t num_points, const double* xyz,
                        const uint8_t* gray_lut, int64_t memory_budget, psfm_convert** out, int64_t* valid_count,
                        int32_t* batch_ptr, psfm_convert_summary* summary);
/* The maps of the images of batches first_batch .. first_batch + num_batches - 1, images in order, each row-major
   h x w: depth [sum w h] float64, rgba [sum w h][4].  Batch j runs while batch j - 1's maps are copied out.
   PSFM_ERR_INVALID before any launch for a batch out of range or when one of the images has no valid pixel (its
   percentiles do not exist).  The first call allocates the pinned staging buffers the handle keeps. */
int psfm_convert_result(psfm_convert* c, int32_t first_batch, int32_t num_batches, double* depth, uint8_t* rgba,
                        psfm_convert_summary* summary);
void psfm_convert_destroy(psfm_convert* c);

/* ------------------------------------------------------------------------- */
/* The 3D points' colours from the decoded images                            */
/* (Reconstruction::ExtractColorsForAllImages, csrc/colors.cu).              */
/* ------------------------------------------------------------------------- */
typedef struct psfm_colors psfm_colors;
typedef struct {
  int32_t num_batches;       /* psfm_colors_add_images calls that took images */
  int32_t num_images;        /* images added */
  int64_t num_observations;  /* keypoints with a point */
  double setup_ms;           /* create: the observations' upload, the sort and the point lists (CUDA events) */
  double upload_ms;          /* the batches' host-to-device copies, summed (CUDA events) */
  double sample_ms;          /* the batches' k_sample, summed (CUDA events; overlaps the next batch's upload) */
  double mean_ms;            /* result: k_mean (CUDA events) */
  double stage_ms;           /* host wall time of the copies of the caller's pixels into the pinned buffers */
} psfm_colors_summary;
/* Uploads the observations of a model and orders each point's observations by image, then keypoint.
     keypoint_ptr [F + 1] over keypoints [K][2] (x, y in COLMAP's convention: the upper-left pixel's centre is at
     (0.5, 0.5)) and point_of_keypoint [K] (point row in [0, num_points), -1: no point), K < 2^31, num_points < 2^31.
   summary (nullable) receives num_observations and setup_ms.  PSFM_ERR_INVALID before any launch for a bad
   keypoint_ptr or a point row out of range; PSFM_ERR_NO_DEVICE without a device. */
int psfm_colors_create(int32_t num_images, const int64_t* keypoint_ptr, const double* keypoints,
                       const int32_t* point_of_keypoint, int64_t num_points, psfm_colors** out,
                       psfm_colors_summary* summary);
/* Samples the observations of images first .. first + count - 1 in their decoded pixels: width [count],
   height [count], pixels the images one after the other, each top-down rows of w RGB8 triples.  The call copies the
   pixels and returns while the device works; the k-th call runs on stream k % 2.  PSFM_ERR_INVALID before any launch
   for an image index out of range or already added, or a zero width or height.  An image never added contributes
   nothing. */
int psfm_colors_add_images(psfm_colors* c, int32_t first, int32_t count, const int32_t* width, const int32_t* height,
                           const uint8_t* pixels);
/* rgb [num_points][3]: per point the mean of its samples (image ascending, then keypoint; summed in double) rounded
   half away from zero, black without a sample.  summary (nullable) receives the totals. */
int psfm_colors_result(psfm_colors* c, uint8_t* rgb, psfm_colors_summary* summary);
void psfm_colors_destroy(psfm_colors* c);

/* Measured fp64 roof of the current device (bench.py's roofline denominator for the kernels
   that are bounded by the fp64 FMA pipe rather than by HBM): sustained fused multiply-adds
   per second over the whole chip, and the latency in SM cycles of one dependent DFMA. */
int psfm_measure_dfma(double* dfma_per_second, double* dependent_latency_cycles);

/* Diagnostic used by the parity tests: solve one banded(+arrow) SPD system with the
   single-CTA band Cholesky the exact-Schur mode uses (csrc/ba_band_chol.cuh).
     A   [n][n] row-major symmetric, n = nb + 3: A[i][j] == 0 for |i - j| > bw among the
         first nb rows/columns, the last 3 rows/columns are dense (the shared camera)
     b   [n]     x [n] receives the solution.  Returns PSFM_OK, PSFM_ERR_INVALID when the
   matrix is not positive definite, PSFM_ERR_UNSUPPORTED when nb is not a multiple of 6 of at
   least 18, or when the block window (min(bw, nb - 1) + 5) / 6 + 1 exceeds 25 blocks and
   nb / 6 does too. */
int psfm_ba_band_solve(const double* A, const double* b, int32_t nb, int32_t bw, double* x);

/* Test entries of the blocked dense Cholesky (k_chol_blocked, csrc/ba_schur_explicit.cuh) and of the two solvers that
   reuse its factor.  A is [n][n] row-major and symmetric; only its lower triangle is read.  Each returns PSFM_OK,
   PSFM_ERR_INVALID on a bad argument or when a pivot is not positive (psfm_last_error says which), PSFM_ERR_NO_DEVICE
   without a device; argument checks come first.
   psfm_blocked_cholesky_solve: x [ns] = A^-1 b, ns = n, with the bundle adjustment's dense-S launch.  The first nb
     rows form a band, A[i][j] == 0 for i - j > bw there (CholArgs::bw); rows nb .. ns - 1 are dense (the arrow).
     nb = bw = ns is a dense matrix and goes through dense_cholesky_launch.  max_ctas > 0 caps the cooperative grid,
     0 keeps the solver's grid.
   psfm_laplacian_solve: X [n][3] = A^-1 B for three interleaved right-hand sides B [n][3], the rotation averaging's
     factor-then-k_trsv.
   psfm_spd_inverse: X = A^-1 by the position estimation's k_pos_inverse; column j at X + j n. */
int psfm_blocked_cholesky_solve(const double* A, const double* b, int32_t ns, int32_t nb, int32_t bw, int32_t max_ctas,
                                double* x);
int psfm_laplacian_solve(const double* A, const double* B, int32_t n, double* X);
int psfm_spd_inverse(const double* A, int32_t n, double* X);

/* Test entries of the small null-vector solvers of the geometry stages (csrc/dlt.cuh) and of the verification's local
   step.  Each returns PSFM_OK, PSFM_ERR_INVALID on a bad argument (psfm_last_error says which), PSFM_ERR_NO_DEVICE
   without a device; argument checks come first.
   psfm_null_vectors: one solver per thread on `count` (1 .. 2^24) row-major N x N matrices A, its raw outputs in out:
     PSFM_NV_JACOBI_3, _4   one_sided_jacobi<N>: A V [N][N], then V [N][N]
     PSFM_NV_DLT_POINT      dlt_point_4x4 (N = 4): X [3], then the null vector v [4] before hnormalisation
     PSFM_NV_EIGEN_3, _4    smallest_eigenvector<N> of a symmetric A: v [N]
     PSFM_NV_JACOBI_9       one_sided_jacobi_mem on 9 x 9, the local step's solve: A V [9][9], V [9][9], then V's
                            column of the smallest column norm of A V [9]
   psfm_verification_local_model: the local step of the verification's LORANSAC (local_estimate in one 256-thread
     CTA, k_verify's code path) for kind 0 (eight-point F) or 1 (normalised DLT H) on the inliers of `best` [9]
     (residual <= max_squared_error) among n points [n][4] = (x1, y1, x2, y2).  null_vector [9]: the normalised
     solve's null vector (unit norm, any sign); normalization [6]: (s1, c1x, c1y, s2, c2x, c2y), T = [s 0 -s cx;
     0 s -s cy; 0 0 1]; local_model [9]: the denormalised model that k_verify scores next (F after the rank-2 step). */
#define PSFM_NV_JACOBI_3 0
#define PSFM_NV_JACOBI_4 1
#define PSFM_NV_DLT_POINT 2
#define PSFM_NV_EIGEN_3 3
#define PSFM_NV_EIGEN_4 4
#define PSFM_NV_JACOBI_9 5
int psfm_null_vectors(int32_t form, const double* A, int64_t count, double* out);
int psfm_verification_local_model(int32_t kind, const float* points, int64_t n, const double* best,
                                  double max_squared_error, double* null_vector, double* normalization,
                                  double* local_model);

/* ------------------------------------------------------------------------- */
/* RAFT's correlation, lookup, upsampling and flow image on the device          */
/* (csrc/optical_flow.cu, DESIGN.md 4.14).  DEVICE pointers, work enqueued on    */
/* `stream` without synchronising.  Each returns PSFM_OK, PSFM_ERR_INVALID on a  */
/* bad argument (argument checks come first), PSFM_ERR_NO_DEVICE without a      */
/* device.  h x w is the 1/8 grid (8 <= h, w and h w <= 2^20 where a pyramid is  */
/* involved); a pyramid holds, level l = 0 .. 3 after level l - 1, h w images of */
/* (h >> l) x (w >> l) floats: psfm_corr_pyramid_floats(h, w) of them.           */
/* ------------------------------------------------------------------------- */
/* psfm_corr_pyramids: fwd [h w][h w] holds fmap1^T fmap2 (row = pixel of image 1) on entry; on return fwd is the
   forward pyramid (level 0 = the product / 16) and bwd the backward one, built from the transposed product. */
int psfm_corr_pyramids(float* fwd, float* bwd, int32_t h, int32_t w, void* stream);
int64_t psfm_corr_pyramid_floats(int32_t h, int32_t w);
/* psfm_corr_lookup: CorrBlock.__call__ (radius 4) of num_problems pyramids laid end to end: coords [P][2][h][w]
   (x, y at 1/8) -> out [P][324][h][w]; channel l * 81 + a * 9 + b samples level l at (x / 2^l + a - 4,
   y / 2^l + b - 4), zero outside. */
int psfm_corr_lookup(const float* pyramids, int32_t num_problems, int32_t h, int32_t w, const float* coords, float* out,
                     void* stream);
/* psfm_flow_upsample: upsample_flow then InputPadder.unpad: flow [P][2][h][w] (coords1 - coords0), mask [P][576][h][w]
   (the mask head's output before its 0.25 scale), pad [4] = (left, right, top, bottom), each 0 .. 7 ->
   out [P][8 h - top - bottom][8 w - left - right][2]. */
int psfm_flow_upsample(const float* flow, const float* mask, int32_t num_problems, int32_t h, int32_t w, const int32_t* pad,
                       float* out, void* stream);
/* psfm_flow_to_image: flow_to_image(flow, convert_to_bgr=True) of num_maps maps [M][h][w][2] -> bgr [M][h][w][3] */
int psfm_flow_to_image(const float* flow, int32_t num_maps, int32_t h, int32_t w, uint8_t* bgr, void* stream);

/* ------------------------------------------------------------------------- */
/* Monocular depth (MiDaS midas_v21, DESIGN.md §4.16): the steps the reference */
/* runs on the host around the network.  Device pointers, torch's stream.      */
/* ------------------------------------------------------------------------- */
/* psfm_depth_prepare: uint8 RGB frames [n][h][w][3] -> the network input [n][3][net_h][net_w] with channels_last
   strides (memory [n][net_h][net_w][3]), float32 or (half = 1) fp16: / 255, cv2.resize(INTER_CUBIC) in float64,
   (x - ImageNet mean) / std, rounded once to float32 (then to fp16). */
int psfm_depth_prepare(const uint8_t* rgb, int32_t num_frames, int32_t h, int32_t w, int32_t net_h, int32_t net_w,
                       int32_t half, void* out, void* stream);
/* psfm_depth_upsample: the prediction [n][net_h][net_w] (float32, or fp16 with half = 1) -> F.interpolate(bicubic,
   align_corners=False) at h x w, rounded to the prediction's dtype, written as float32 [n][h][w] with the rows
   flipped (the PFM payload); minmax [n][2] receives each frame's minimum and maximum. */
int psfm_depth_upsample(const void* pred, int32_t num_frames, int32_t net_h, int32_t net_w, int32_t half, int32_t h,
                        int32_t w, float* flipped, float* minmax, void* stream);
/* psfm_depth_quantize: write_depth's 16-bit pixels [n][h][w] (frame orientation) from the flipped maps and their
   minmax: (uint16)(65535 * (d - min) / (max - min)) in float32, zeros where max - min <= float64 eps. */
int psfm_depth_quantize(const float* flipped, int32_t num_frames, int32_t h, int32_t w, const float* minmax,
                        uint16_t* pixels, void* stream);

/* ---- trajectory labeller (motion segmentation; DESIGN.md §4.17) ----
   The track set is CSR on the device: trajectory t owns observations ptr[t] .. ptr[t + 1] of frames / xy, its frames
   strictly ascending.  Windows are win_start[w] .. win_start[w] + L - 1. */
/* psfm_seg_max_window: the longest window psfm_seg_encode takes (its per-row state must fit in shared memory). */
int psfm_seg_max_window(void);
/* psfm_seg_hits: hits [num_windows][num_trajs], the number of window frames each trajectory is seen in. */
int psfm_seg_hits(const int64_t* ptr, const int32_t* frames, int32_t num_trajs, const int32_t* win_start,
                  int32_t num_windows, int32_t L, int32_t* hits, void* stream);
/* psfm_seg_shuffle (host): perm [K], the permutation of 0 .. K-1 that std::shuffle with std::mt19937(5489) makes,
   the one TrajectorySet::sample_inside_window applies before cutting an over-full window. */
int psfm_seg_shuffle(int32_t K, int32_t* perm);
/* psfm_seg_windows: for row r (trajectory rows[r] in window row_window[r]) the float64 locations loc [R][L][2] (0
   where the trajectory is not seen) and valid [R][L] (1 where it is). */
int psfm_seg_windows(const int64_t* ptr, const int32_t* frames, const double* xy, const int32_t* rows,
                     const int32_t* row_window, int32_t num_rows, const int32_t* win_start, int32_t L, double* loc,
                     uint8_t* valid, void* stream);
/* psfm_seg_depth_resize: uint16 depth pixels [n][h][w] -> float32 [n][240][424], cv2.resize(INTER_LINEAR) of
   pixels / 65535.0 in float64, then cast. */
int psfm_seg_depth_resize(const uint16_t* pixels, int32_t num_frames, int32_t h, int32_t w, float* out, void* stream);
/* psfm_seg_encode: the encoder features feat [R][16] of the window rows (loc, valid as psfm_seg_windows writes them)
   over the depth maps [num_frames][240][424], frames raw_h x raw_w; weights: the 15881 floats of
   motion_seg.pack_encoder. */
int psfm_seg_encode(const double* loc, const uint8_t* valid, const int32_t* row_window, const int32_t* win_start,
                    int32_t num_windows, int32_t num_rows, int32_t L, const float* depth, int32_t num_frames,
                    int32_t raw_h, int32_t raw_w, const float* weights, float* feat, void* stream);
/* psfm_seg_merge: with row_of [num_windows][num_trajs] (the row of trajectory t in window w, -1 when not sampled) and
   the rows' labels pred [R]: labels [M] (the label of the first window that sampled the trajectory and holds the
   frame, -1 for none) and first_row [num_trajs] (the first row that sampled the trajectory, -1 for none). */
int psfm_seg_merge(const int64_t* ptr, const int32_t* frames, int32_t num_trajs, const int32_t* win_start,
                   int32_t num_windows, int32_t L, const int32_t* row_of, const uint8_t* pred, int8_t* labels,
                   int32_t* first_row, void* stream);
/* psfm_seg_draw: draw_traj_cls's video frames out [L][960][424][3] (BGR) of one window of K rows: the frames
   [L][240][424][3] (BGR), then the labels, the points and the num_draws trajectories draws[], stamped with the pixel
   offsets stamps [(na + nb + nc)][2] (dx, dy) of the three circles; order [L][3][240][424] is scratch. */
int psfm_seg_draw(const uint8_t* frames, const double* loc, const uint8_t* valid, const uint8_t* pred, int32_t K,
                  int32_t L, int32_t raw_h, int32_t raw_w, const int32_t* draws, int32_t num_draws,
                  const int16_t* stamps, int32_t na, int32_t nb, int32_t nc, int32_t* order, uint8_t* out,
                  void* stream);

/* ------------------------------------------------------------------------- */
/* Multi-GPU (HP2): points sharded across ranks, one all-reduce of the         */
/* camera-side vector per PCG step (SURVEY.md §8e).                            */
/* ------------------------------------------------------------------------- */
#define PSFM_NCCL_UNIQUE_ID_BYTES 128
/* rank 0 creates the id; the caller broadcasts the bytes (torch.distributed). */
int psfm_dist_get_unique_id(uint8_t id[PSFM_NCCL_UNIQUE_ID_BYTES]);
int psfm_dist_init(const uint8_t id[PSFM_NCCL_UNIQUE_ID_BYTES], int32_t rank, int32_t world_size);
int psfm_dist_world_size(void);
int psfm_dist_rank(void);
void psfm_dist_finalize(void);
/* When a communicator is initialised, psfm_ba_create expects each rank to pass ITS
   shard of the observations (any subset of points; cameras/images replicated) and
   psfm_ba_run keeps the replicated camera state identical on all ranks. */

#ifdef __cplusplus
}
#endif
#endif /* PSFM_B200_H_ */
