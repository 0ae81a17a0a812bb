// verification_recalled.cuh — the constants of COLMAP's two-view geometric verification that `colmap matches_importer
// --match_type pairs` runs (TwoViewGeometryVerifier -> TwoViewGeometry::Estimate -> EstimateUncalibrated, the LORANSAC
// loop, InlierSupportMeasurer, RANSAC::ComputeNumTrials, DetectWatermark) but the reference tree does not vendor.  They
// are recalled, not pinned to a source line; oracle/verification_oracle.py keeps the same values in its RECALLED dict.
// A correction is a one-line change on each side.
//
// Order-sensitive details, recalled with the constants:
//   * The trial-bound test (trial >= dyn_max_num_trials && trial >= min_num_trials) runs inside the per-model loop,
//     after the model was scored; once it passes, the remaining models of the sample are not scored.  The trial index
//     is 0-based and the trial count reported is the number of samples drawn.
//   * Support: more inliers, then a strictly smaller residual sum over the inliers; the initial best support has 0
//     inliers and the largest double as its sum, so the first model always becomes the best one.
//   * Local optimisation runs when a model becomes the best with more inliers than the minimal sample and at least as
//     many as the local estimator needs: at most kMaxNumLocalTrials rounds of the local estimator on the best model's
//     inliers; a better local model replaces the best one; the rounds stop as soon as the inlier count did not grow.
//   * ComputeNumTrials(n, m) = ceil(log(1 - confidence) / log(1 - (n / m)^s) * multiplier) with s the estimator's
//     sample size; 1 when the ratio is 1, unbounded when the log is 0.
//   * The RANSAC constructor caps max_num_trials at ComputeNumTrials(min_inlier_ratio * 1e5, 1e5).  The watermark
//     LORANSAC runs with min_inlier_ratio = watermark_min_inlier_ratio (0.7): 18 trials at most.
//   * A pair with fewer raw matches than min_num_inliers is not estimated (config UNDEFINED, no inliers).
#pragma once

namespace psfm {
namespace ver {

constexpr long long kCapNumSamples = 100000;        // RANSAC constructor: the min_inlier_ratio cap's sample count
constexpr int kMaxNumLocalTrials = 10;              // LORANSAC kMaxNumLocalTrials
constexpr int kSevenPointSamples = 7;               // FundamentalMatrixSevenPointEstimator::kMinNumSamples
constexpr int kEightPointSamples = 8;               // FundamentalMatrixEightPointEstimator::kMinNumSamples
constexpr int kHomographySamples = 4;               // HomographyMatrixEstimator::kMinNumSamples
constexpr int kTranslationSamples = 1;              // TranslationTransformEstimator<2>::kMinNumSamples
constexpr double kMinF22 = 1e-10;                   // the seven-point step drops a model with |F(2,2)| below this
constexpr long long kUnbounded = 0x7fffffffffffffffLL;   // ComputeNumTrials when the log is 0

// RANSAC::ComputeNumTrials with `s` samples per model
__host__ __device__ inline long long compute_num_trials(long long num_inliers, long long num_samples, int s,
                                                        double confidence, double multiplier) {
  const double ratio = (double)num_inliers / (double)num_samples;
  const double nom = 1.0 - confidence;
  if (nom <= 0.0) return kUnbounded;
  const double denom = 1.0 - pow(ratio, (double)s);
  if (denom <= 0.0) return 1;
  const double ld = log(denom);
  if (ld == 0.0) return kUnbounded;
  const double n = ceil(log(nom) / ld * multiplier);
  return n >= 9.2e18 ? kUnbounded : (long long)n;
}

}  // namespace ver
}  // namespace psfm
