// edt_plan.cu -- the later-axis plan (plan_later, edt_passes.cuh) for host code that only needs to
// know which kernel a pass would take, not launch it.  It instantiates no launcher: those live in
// edt_passes_b{1,2,4,8}.cu.
#include "edt_passes.cuh"

namespace edtb200 {
namespace host {

bool later_pass_is_long(const LineGeom& g, PassArith arith, int max_smem_optin) {
  // tile or long-line does not depend on TMA, the CTA count or the integer hull switch
  return plan_later(g, false, arith, max_smem_optin, true, false, false).kernel == 1;
}

bool label_noise_predicted(const DeviceCache& dc) { return noise_predicted(dc); }

BoundedPlan bounded_plan(int ndim, const float w[3], double max_distance, bool sites) {
  int64_t rmax = sites ? EDTB200_BOUNDED_SITES_WINDOW_MAX : EDTB200_BOUNDED_WINDOW_MAX;
  if (const char* env = getenv("EDTB200_BOUNDED_RMAX")) {      // A/B switch for measurements
    rmax = atoll(env);
    if (rmax > kWindowRadiusLimit) rmax = kWindowRadiusLimit;
  }
  return plan_bounded(ndim, w, max_distance, rmax);
}

BoundedPlan window_pass_plan(float w, double max_distance) {
  const float ws[3] = {w, w, w};
  return plan_bounded(1, ws, max_distance, kWindowRadiusLimit);
}

}  // namespace host
}  // namespace edtb200
