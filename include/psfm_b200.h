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
