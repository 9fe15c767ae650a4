// edt_plan.cu -- the later-axis and label-noise plans (plan_later, plan_noise, edt_passes.cuh) for host
// code that only needs to know what the passes would take, not launch them.  It instantiates no
// launcher: those live in edt_passes_b{1,2,4,8}.cu.
#include "edt_passes.cuh"

namespace edtb200 {
namespace host {

bool later_pass_is_long(const LineGeom& g, PassArith arith, int max_smem_optin) {
  // tile or long-line does not depend on TMA, the CTA count or the integer hull switch
  return plan_later(g, false, arith, max_smem_optin, true, false, false).kernel == 1;
}

NoisePlan noise_plan(const Transform& t, int64_t count, const void* labels, const float* f, const DeviceCache& dc,
                     int noise) {
  // EDTB200_SETTLED_GROUP forces the later passes' group size (A/B switch for measurements)
  static const int forced_group = getenv("EDTB200_SETTLED_GROUP") ? atoi(getenv("EDTB200_SETTLED_GROUP")) : 0;
  return plan_noise(t, count, reinterpret_cast<uintptr_t>(f) % 16 == 0, first_is_vec(labels, t.label_bytes, f, t.n[0]),
                    noise < 0 ? noise_predicted(dc) : noise != 0, no_int_hull(), forced_group, dc.max_smem_optin,
                    dc.sm_count);
}

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
