// DPGO_robust.cpp -- robust cost weights and the GNC mu schedule (host scalar math, not on the GPU path: the
// benchmark configurations run plain least squares).  Behaviour of the reference's src/DPGO_robust.cpp:17-103.
//
// weight(r) is the factor w in the re-weighted least-squares surrogate  w * r^2  of the robust loss rho(r):
//   L2       rho = r^2 / 2                       w = 1
//   L1       rho = |r|                           w = 1 / r
//   Huber    quadratic below c, linear above     w = min(1, c / r)
//   TLS      truncated least squares at c        w = [r < c]
//   GM       Geman-McClure                       w = 1 / (1 + r^2)^2
//   GNC_TLS  graduated non-convexity towards TLS with control parameter mu (Yang et al., eq. 14):
//            w = 0 above (mu+1)/mu * cbar^2, 1 below mu/(mu+1) * cbar^2, cbar sqrt(mu (mu+1)) / r - mu in between;
//            update() multiplies mu by GNCMuStep (the surrogate tightens towards TLS as mu grows).
#include <DPGO/DPGO_robust.h>
#include <DPGO/DPGO_utils.h>

#include <cmath>
#include <cstdio>
#include <stdexcept>

namespace DPGO {

namespace {

inline double huber_weight(double r, double c) { return r < c ? 1.0 : c / r; }

inline double geman_mcclure_weight(double r) {
  const double s = 1.0 + r * r;
  return 1.0 / (s * s);
}

inline double gnc_tls_weight(double r, double mu, double cbar) {
  const double r2 = r * r, c2 = cbar * cbar;
  // the bounds in the reference's order: a different order rounds differently, and the 0 / 1 weights are counted exactly
  if (r2 >= (mu + 1) / mu * c2) return 0.0;     // certainly an outlier at this stage of the schedule
  if (r2 <= mu / (mu + 1) * c2) return 1.0;     // certainly an inlier
  return std::sqrt(c2 * mu * (mu + 1) / r2) - mu;
}

}  // namespace

RobustCost::RobustCost(RobustCostType costType, const RobustCostParameters &params) : mCostType(costType), mParams(params) {
  reset();
}

double RobustCost::weight(double r) {
  switch (mCostType) {
    case L2: return 1.0;
    case L1: return 1.0 / r;
    case Huber: return huber_weight(r, mParams.HuberThreshold);
    case TLS: return r < mParams.TLSThreshold ? 1.0 : 0.0;
    case GM: return geman_mcclure_weight(r);
    case GNC_TLS: return gnc_tls_weight(r, mu, mParams.GNCBarc);
  }
  throw std::runtime_error("RobustCost::weight: unknown cost type");
}

void RobustCost::reset() {
  if (mCostType != GNC_TLS) return;             // only GNC carries state
  mu = mParams.GNCInitMu;
  mGNCIteration = 0;
}

void RobustCost::update() {
  if (mCostType != GNC_TLS) return;
  mGNCIteration += 1;
  if (mGNCIteration > mParams.GNCMaxNumIters) {
    std::printf("GNC: reached maximum iterations.");
    return;                                     // schedule exhausted: mu stays where it is
  }
  mu *= mParams.GNCMuStep;
}

double RobustCost::computeErrorThresholdAtQuantile(double quantile, size_t dimension) {
  // residual threshold t with P(chi2_dof <= t^2) = quantile; dof = dimension of the SE(d) tangent space
  const size_t dof = (dimension == 2) ? 3 : 6;
  return std::sqrt(chi2inv(quantile, dof));
}

}  // namespace DPGO
