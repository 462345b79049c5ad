// dojo_b200_cm.cu -- second compilation of the step / gradient kernels with the complete model set of the reference enabled
// (macro DJ_ANY_CONTACT, named after its first use):
//   * every contact model (SURVEY.md 8 f4): NonlinearContact (contacts/nonlinear.jl) as in dojo_b200.cu, plus ImpactContact
//     (contacts/impact.jl) and LinearContact (contacts/linear.jl) from dojo_contact_orthant.cuh;
//   * translational springs / dampers / limits of the joints (SURVEY.md 8 a4 / a6) from dojo_joint_tra.cuh.
//
// Why a second translation unit instead of a run-time branch inside the one kernel: the Newton loop of dojo_step_kernel is ~20 k
// straight-line instructions at 255 registers and is sensitive to instruction-cache footprint and register allocation;
// the benchmarked kernels (all BASELINE models use NonlinearContact) must not change when a contact model is
// added.  The same headers are compiled here under another namespace with DJ_ANY_CONTACT; dojo_create picks this compilation only for
// mechanisms that contain an impact / linear contact or a joint with translational springs / dampers / limits.  The two compilations share the argument block layout (StepArgs, Plan and the
// plan tables are plain data), so the host code in dojo_b200.cu fills one StepArgs and launches whichever kernel the handle holds.
#include <cuda_runtime.h>

#define DJ_ANY_CONTACT 1
#define dj dj_cm
#include "dojo_step_kernel.cuh"
#undef dj

extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_kernel(int grad) {
  return grad ? (const void*)dj_cm::dojo_step_kernel<true> : (const void*)dj_cm::dojo_step_kernel<false>;
}
// the traced forward kernel of this compilation (dojo_step_trace)
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_trace_kernel() {
  return (const void*)dj_cm::dojo_step_kernel<false, false, true>;
}
// the recording rollout kernel of this compilation (dojo_rollout_grad)
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_rec_kernel() {
  return (const void*)dj_cm::dojo_step_kernel<false, false, false, false, true>;
}
// the closed-loop rollout kernel of this compilation (dojo_rollout_feedback)
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_fb_kernel() {
  return (const void*)dj_cm::dojo_step_kernel<false, false, false, false, false, true>;
}
// the adjoint kernel of this compilation (dojo_rollout_vjp)
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_vjp_kernel() {
  return (const void*)dj_cm::dojo_step_kernel<true, false, false, false, false, false, true>;
}
// the closed-loop tape and its adjoint of this compilation (dojo_rollout_feedback_tape / dojo_rollout_feedback_vjp)
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_fbtape_kernel() {
  return (const void*)dj_cm::dojo_step_kernel<false, false, false, false, true, true>;
}
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_fbvjp_kernel() {
  return (const void*)dj_cm::dojo_step_kernel<true, false, false, false, false, true, true>;
}
