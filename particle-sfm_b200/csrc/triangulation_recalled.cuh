// triangulation_recalled.cuh — the constants of COLMAP's triangulation estimator that IncrementalTriangulator::Create
// (sfm/incremental_triangulator.cc:463-548) runs but the reference tree does not vendor: EstimateTriangulation, the
// LORANSAC loop, InlierSupportMeasurer, CombinationSampler and RANSAC::ComputeNumTrials.  They are recalled, not pinned
// to a source line; oracle/triangulation_oracle.py keeps the same values in its RECALLED dict.  A correction is a
// one-line change on each side.
//
// Order-sensitive details, recalled with the constants:
//   * CombinationSampler with 2 of m draws (0, 1), (0, 2), ..., (0, m-1), (1, 2), ...; max_num_trials is capped at
//     C(m, 2), so no sample repeats.
//   * The trial-bound test (trial >= dyn_max_num_trials && trial >= min_num_trials) runs inside the per-model loop:
//     a sample that yields no model cannot end the loop.  The trial index it compares is 0-based.
//   * Support: more inliers, then a strictly smaller residual sum (InlierSupportMeasurer::Compare); the initial best
//     support has 0 inliers and the largest double as its sum.
//   * Local optimisation runs when a sample's model becomes the best with more than 2 inliers: at most 10 rounds of
//     the multi-view DLT on the current best model's inliers, a better local model replaces the best one, and the
//     rounds stop as soon as the best inlier count did not grow.
//   * ComputeNumTrials(n, m) = ceil(log(1 - confidence) / log(1 - (n / m)^2) * multiplier); 1 when the ratio is 1.
//     A support without inliers gives log(1) = 0 and -inf, which the reference casts to size_t: unbounded here.
//   * The RANSAC constructor caps max_num_trials at ComputeNumTrials(min_inlier_ratio * 1e5, 1e5) (69,064: no cap at
//     10,000 trials).
#pragma once

namespace psfm {
namespace tri {

constexpr double kConfidence = 0.9999;            // Create's ransac_options.confidence
constexpr double kMinInlierRatio = 0.02;          // Create's ransac_options.min_inlier_ratio
constexpr long long kMaxNumTrials = 10000;        // Create's ransac_options.max_num_trials
constexpr int kExhaustiveSamplingThreshold = 15;  // Create: min_num_trials = C(m, 2) for m <= 15
constexpr double kDynNumTrialsMultiplier = 3.0;   // RANSACOptions::dyn_num_trials_multiplier
constexpr long long kCapNumSamples = 100000;      // RANSAC constructor: the min_inlier_ratio cap's sample count
constexpr int kMaxNumLocalTrials = 10;            // LORANSAC kMaxNumLocalTrials
constexpr int kMinNumSamples = 2;                 // TriangulationEstimator::kMinNumSamples
constexpr double kDepthEpsilon = 2.220446049250313e-16;   // HasPointPositiveDepth: depth >= epsilon
constexpr long long kUnbounded = 0x7fffffffffffffffLL;   // ComputeNumTrials without inliers

// RANSAC::ComputeNumTrials with 2 samples per model
__host__ __device__ inline long long compute_num_trials(long long num_inliers, long long num_samples) {
  const double ratio = (double)num_inliers / (double)num_samples;
  const double nom = 1.0 - kConfidence;
  if (nom <= 0.0) return kUnbounded;
  const double denom = 1.0 - ratio * ratio;
  if (denom <= 0.0) return 1;
  const double ld = log(denom);
  if (ld == 0.0) return kUnbounded;
  const double n = ceil(log(nom) / ld * kDynNumTrialsMultiplier);
  return n >= 9.2e18 ? kUnbounded : (long long)n;
}

}  // namespace tri
}  // namespace psfm
