// rotation_recalled.cuh — the constants of the global rotation averaging that restate libraries the reference links
// but does not vendor (Theia's L1Solver).  They are recalled, not pinned to a source line; oracle/rotation_oracle.py
// keeps the same values in its RECALLED dict.  A correction is a one-line change on each side.
#pragma once

namespace psfm {
namespace rot {

constexpr double kAdmmRho = 1.0;                // theia::L1Solver::Options::rho
constexpr double kAdmmAlpha = 1.0;              // theia::L1Solver::Options::alpha (over-relaxation)
constexpr double kAdmmAbsTolerance = 1e-4;      // theia::L1Solver::Options::absolute_tolerance
constexpr double kAdmmRelTolerance = 1e-2;      // theia::L1Solver::Options::relative_tolerance

}  // namespace rot
}  // namespace psfm
