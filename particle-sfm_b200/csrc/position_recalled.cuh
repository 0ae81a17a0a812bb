// position_recalled.cuh — the defaults of the solver behind the global position estimation that restate a library the
// reference links but does not vendor (Theia's ConstrainedL1Solver::Options, which
// least_unsquared_deviation_position_estimator.cc:161 constructs with its defaults).  They are recalled, not pinned to
// a source line; oracle/position_oracle.py keeps the same values in its RECALLED dict.  A correction is a one-line
// change on each side.
#pragma once

namespace psfm {
namespace pos {

constexpr int kLudMaxIterations = 1000;         // theia::ConstrainedL1Solver::Options::max_num_iterations
constexpr double kLudRho = 10.0;                // theia::ConstrainedL1Solver::Options::rho
constexpr double kLudAlpha = 1.2;               // theia::ConstrainedL1Solver::Options::alpha (over-relaxation)
constexpr double kLudAbsTolerance = 1e-4;       // theia::ConstrainedL1Solver::Options::absolute_tolerance
constexpr double kLudRelTolerance = 1e-2;       // theia::ConstrainedL1Solver::Options::relative_tolerance

}  // namespace pos
}  // namespace psfm
