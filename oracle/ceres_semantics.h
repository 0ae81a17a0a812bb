/*
 * ceres_semantics.h — every constant of Ceres Solver 2.0.0 (misc/doc/ceres.md:5 pins the
 * version) that the two reference hot paths inherit as a DEFAULT, in one place.
 * TEST INFRASTRUCTURE (oracle).  Recalled from the published Ceres 2.0.0 sources
 * (internal/ceres/{trust_region_minimizer,levenberg_marquardt_strategy,dogleg_strategy,
 * conjugate_gradients_solver,corrector,loss_function}.cc, include/ceres/solver.h);
 * the sources are not in the reference repository — see SURVEY.md Appendix A.
 */
#ifndef PSFM_CERES_SEMANTICS_H_
#define PSFM_CERES_SEMANTICS_H_

/* Solver::Options defaults (solver.h) */
#define CERES_INITIAL_TRUST_REGION_RADIUS 1e4
#define CERES_MAX_TRUST_REGION_RADIUS 1e16
#define CERES_MIN_TRUST_REGION_RADIUS 1e-32
#define CERES_MIN_RELATIVE_DECREASE 1e-3
#define CERES_MIN_LM_DIAGONAL 1e-6
#define CERES_MAX_LM_DIAGONAL 1e32
#define CERES_MAX_NUM_CONSECUTIVE_INVALID_STEPS 5
#define CERES_FUNCTION_TOLERANCE 1e-6
#define CERES_GRADIENT_TOLERANCE 1e-10
#define CERES_PARAMETER_TOLERANCE 1e-8
#define CERES_ETA 1e-1
#define CERES_MIN_LINEAR_SOLVER_ITERATIONS 0

/* LevenbergMarquardtStrategy: radius /= max(1/3, 1 - (2 rho - 1)^3); on reject
   radius /= decrease_factor, decrease_factor *= 2 (reset to 2 on accept). */
#define CERES_LM_MIN_SHRINK (1.0 / 3.0)
#define CERES_LM_DECREASE_FACTOR0 2.0

/* DoglegStrategy (TRADITIONAL_DOGLEG is the default dogleg_type). */
#define CERES_DOGLEG_MIN_MU 1e-8
#define CERES_DOGLEG_MAX_MU 1.0
#define CERES_DOGLEG_MU_INCREASE 10.0
#define CERES_DOGLEG_DECREASE_THRESHOLD 0.25
#define CERES_DOGLEG_INCREASE_THRESHOLD 0.75

/* ConjugateGradientsSolver */
#define CERES_CG_RESIDUAL_RESET_PERIOD 10

#endif
