// dojo_b200.cu -- C-ABI (include/dojo_b200.h) + kernel entry points of the H100-native (sm_90a) Dojo step.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared -Xcompiler -fPIC  (see build.py)
// There is NO CPU fallback in this library: dojo_create fails with DOJO_ENODEVICE without a CUDA device.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/dojo_b200.h"
#include "dojo_step_kernel.cuh"
#include "dojo_kin.cuh"
#include "dojo_kinjac.cuh"
#include "dojo_envs.cuh"
#include "dojo_storage.cuh"
#include "dojo_lqr.cuh"

using namespace dj;

// ------------------------------------------------------------------------------------------------------------
// Kernels
// ------------------------------------------------------------------------------------------------------------
// dojo_step_kernel<GRAD> (StepArgs): dojo_step_kernel.cuh; the DJ_ANY_CONTACT compilation of the same source lives in
// dojo_b200_cm.cu and is reached through these two entry points
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_kernel(int grad);
// small: the forward kernel may be the one specialised for small mechanisms (small_step_ok)
static const void* step_kernel_fn(bool any_contact, bool grad, bool plan_smem, bool small = false) {
  if (any_contact) return dojo_cm_step_kernel(grad ? 1 : 0);
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) {
    if (!grad && small) return (const void*)dojo_step_kernel<false, true, false, true>;
    return grad ? (const void*)dojo_step_kernel<true, true> : (const void*)dojo_step_kernel<false, true>;
  }
  return grad ? (const void*)dojo_step_kernel<true, false> : (const void*)dojo_step_kernel<false, false>;
}
// the traced forward kernel (dojo_step_trace) of the compilation and plan placement step_kernel_fn picks for the untraced one
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_trace_kernel();
static const void* step_trace_kernel_fn(bool any_contact, bool plan_smem) {
  if (any_contact) return dojo_cm_step_trace_kernel();
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) return (const void*)dojo_step_kernel<false, true, true>;
  return (const void*)dojo_step_kernel<false, false, true>;
}
// the recording rollout kernel (dojo_rollout_grad) of the same compilation and plan placement; generic in the warp count, so that it
// serves every mechanism (the SMALL kernel computes the same step bit for bit)
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_rec_kernel();
static const void* step_rec_kernel_fn(bool any_contact, bool plan_smem) {
  if (any_contact) return dojo_cm_step_rec_kernel();
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) return (const void*)dojo_step_kernel<false, true, false, false, true>;
  return (const void*)dojo_step_kernel<false, false, false, false, true>;
}
// the closed-loop rollout kernel (dojo_rollout_feedback) of the same compilation and plan placement; generic, like the REC kernel
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_fb_kernel();
static const void* step_fb_kernel_fn(bool any_contact, bool plan_smem) {
  if (any_contact) return dojo_cm_step_fb_kernel();
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) return (const void*)dojo_step_kernel<false, true, false, false, false, true>;
  return (const void*)dojo_step_kernel<false, false, false, false, false, true>;
}
// the adjoint kernel (dojo_rollout_vjp): the VJP variant of the gradient kernel of the same compilation and plan placement as k_grad
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_vjp_kernel();
static const void* step_vjp_kernel_fn(bool any_contact, bool plan_smem) {
  if (any_contact) return dojo_cm_step_vjp_kernel();
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) return (const void*)dojo_step_kernel<true, true, false, false, false, false, true>;
  return (const void*)dojo_step_kernel<true, false, false, false, false, false, true>;
}
// the closed-loop tape (REC + FB, dojo_rollout_feedback_tape) and its adjoint (VJP + FB, dojo_rollout_feedback_vjp), placed as the FB and
// the VJP kernel
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_fbtape_kernel();
extern "C" __attribute__((visibility("hidden"))) const void* dojo_cm_step_fbvjp_kernel();
static const void* step_fbtape_kernel_fn(bool any_contact, bool plan_smem) {
  if (any_contact) return dojo_cm_step_fbtape_kernel();
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) return (const void*)dojo_step_kernel<false, true, false, false, true, true>;
  return (const void*)dojo_step_kernel<false, false, false, false, true, true>;
}
static const void* step_fbvjp_kernel_fn(bool any_contact, bool plan_smem) {
  if (any_contact) return dojo_cm_step_fbvjp_kernel();
  if (plan_smem && !getenv("DOJO_B200_GENERIC_PLAN")) return (const void*)dojo_step_kernel<true, true, false, false, false, true, true>;
  return (const void*)dojo_step_kernel<true, false, false, false, false, true, true>;
}

// Order of the work queue.  A per-step launch ends when its slowest environment ends: an environment that stalls (ten line-search
// trials per iteration up to max_iter, ~6 x the median time) and is dequeued late finishes alone.  Which environments stall is not
// predictable with any accuracy (tools/tail_predictor.py: the previous step's iteration count has AUC 0.54; the best physical
// feature, "nearly at rest" -- a degenerate friction cone: zero tangential velocity on a sticking contact -- 0.73), but a weak
// predictor is enough when it is used the other way round: the environments LEAST likely to stall go LAST, so that whatever is
// dequeued in the final millisecond is short.  Key = quantised log2 of sum_bodies |v15|^2 + |w15|^2 of the state the step starts
// from, ascending (at rest first).  List-scheduling simulation on the benchmark batch (592 slots, measured iteration counts):
// makespan 10.4 (index / random / previous-iterations order) -> 8.8; the order never changes a result, only when it is computed.
// (DOJO_B200_LPT=2 keeps round 1's order by the previous call's iteration counts, =3 the energy key alone, =0 the index order.)
__global__ void dojo_risk_key_kernel(const double* __restrict__ Z, int B, int Nb, const int32_t* __restrict__ prev_iters, int32_t* __restrict__ key) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B) return;
  const double* z = Z + (size_t)e * 13 * Nb;
  double k = 0.0;
  for (int b = 0; b < Nb; ++b) {
    const double* p = z + 13 * b;
    k += p[3] * p[3] + p[4] * p[4] + p[5] * p[5] + p[10] * p[10] + p[11] * p[11] + p[12] * p[12];
  }
  // half-octave buckets of the energy between 2^-44 and 2^19 (non-finite or larger: last bucket; they end :failed quickly anyway) ...
  int q = (k > 0.0) ? (int)floor(2.0 * log2(k)) + 88 : 0;
  q = (k == k) ? min(max(q, 0), 127) : 127;
  // ... minus half a bucket per Newton iteration of the previous call: where stalls persist from step to step (quadruped in stance:
  // simulated makespan / ideal 1.157 -> 1.124 with this term, 1.144 without) the environments that were slow go first as well; where
  // they do not (ant: 8.79 with, 8.78 without) the term is noise of the size of one bucket
  const int pi = prev_iters ? min(max(prev_iters[e], 0), 63) : 0;
  key[e] = 2 * q - pi + 64;  // 1 .. 318
}
// Counting sort of the environments by key < 512 (one CTA; the order of equal keys is irrelevant to the results): ascending, or
// descending for the iteration counts of the previous call.
__global__ void dojo_order_kernel(const int32_t* __restrict__ key, int B, int* __restrict__ order, int descending) {
  __shared__ int hist[512], start[512];
  for (int k = threadIdx.x; k < 512; k += blockDim.x) hist[k] = 0;
  __syncthreads();
  for (int e = threadIdx.x; e < B; e += blockDim.x) atomicAdd(&hist[min(max(key[e], 0), 511)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    if (descending) for (int k = 511; k >= 0; --k) { start[k] = acc; acc += hist[k]; }
    else for (int k = 0; k < 512; ++k) { start[k] = acc; acc += hist[k]; }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < B; e += blockDim.x) order[atomicAdd(&start[min(max(key[e], 0), 511)], 1)] = e;
}


// Closes a step of dojo_step_gather_async on the receiving side: returns once every CTA of every rank has counted itself in on this
// rank's counter (dojo_step_kernel signals after its last environment), i.e. once the gathered buffer holds the next states of all
// ranks.  A peer that never arrives (crashed process) must not hang the GPU: after ~10 s the kernel gives up and flags status[0].
__global__ void dojo_gather_wait_kernel(const unsigned long long* flag, unsigned long long target, int32_t* status) {
  if (threadIdx.x != 0) return;
  unsigned long long t0, t1;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
    if (v >= target) break;
    __nanosleep(500);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > 10000000000ull) { if (status) status[0] = DOJO_STATUS_NONFINITE; break; }
  }
  __threadfence_system();
}

struct DojoGather {
  DojoHandle* h = nullptr;
  int world = 1, rank = 0, B = 0;
  double* buf = nullptr;                 // 2 x [nz x B x world] on this device: steps alternate between the two halves (see dojo_gather_buffer)
  size_t half = 0;                       // doubles per half
  int parity = 0, last = 0;              // half the NEXT step writes / half the most recent step wrote
  unsigned long long* flag = nullptr;    // CTAs (of all ranks, all steps so far) that have delivered into buf
  double* peer_buf[DOJO_MAX_GATHER_RANKS] = {};
  unsigned long long* peer_flag[DOJO_MAX_GATHER_RANKS] = {};
  bool opened[DOJO_MAX_GATHER_RANKS] = {};
  bool connected = false;
  unsigned long long expected = 0;       // value of `flag` when every rank has finished the steps issued so far
};

// ------------------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------------------
// [hostemu:handle:begin]
struct DojoHandle {
  int device = 0;
  int max_batch = 0;
  int sm_count = 0;
  int envs_per_sm = 1;      // CTAs per SM (forward kernel)
  int slots = 1, slots_grad = 1;  // environments hosted by one CTA
  Plan plan;  // device pointers inside
  int nw = 4;  // warps per environment
  size_t arena_bytes = 0, grad_bytes = 0;  // per environment
  size_t smem_fwd = 0, smem_grad = 0;     // dynamic shared memory per CTA
  int envs_per_sm_grad = 1;
  double *d_Fz[2] = {nullptr, nullptr}, *d_Fu[2] = {nullptr, nullptr};  // gradient chunk buffers (grad_chunk environments, double buffered)
  cudaEvent_t ev_kernel[2] = {nullptr, nullptr}, ev_copy[2] = {nullptr, nullptr};
  cudaStream_t copy_stream = nullptr;
  int grad_chunk = 0;
  char* d_blob = nullptr;  // plan tables (one contiguous upload)
  int nsteps = 0;  // elimination steps of the block LDU
  int blob_bytes = 0, blob_off[8] = {0, 0, 0, 0, 0, 0, 0, 0}, blob_end[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int plan_smem_off = -1, plan_smem_off_grad = -1;  // doubles; -1: the tables stay in global memory
  int plan_smem_bytes = 0, plan_smem_bytes_grad = 0, plan_smem_mask = 0, plan_smem_mask_grad = 0;  // prefix of the blob kept in shared memory / tables inside it
  int* d_counter = nullptr;
  int* d_kin_order = nullptr;      // joints root -> leaves (minimal -> maximal map)
  double* d_envNorm = nullptr;  // policy rollout: observation mean and standard deviation [2 ns]
  double *d_envS = nullptr, *d_envSn = nullptr, *d_envA = nullptr, *d_envR = nullptr, *d_envS0 = nullptr;  // environment-layer scratch
  int32_t* d_envDone = nullptr;
  double *d_recZ[2] = {nullptr, nullptr}, *d_recS = nullptr, *d_recD = nullptr;  // dojo_simulate_record scratch
  int32_t* d_recAny = nullptr;
  double* d_kjws = nullptr;        // workspace of the map-Jacobian kernel (one slice per CTA)
  int kj_grid = 0;
  int* d_done = nullptr;           // [0] finished count, [1] gradient work queue, [2..] completion-ordered environment list
  bool overlap_grad = true;
  double* d_gsol = nullptr;        // final solutions handed from the forward to the gradient launch [nres x max_batch]
  int32_t* d_gstatus = nullptr;
  int* d_order = nullptr;          // LPT processing order of the next call
  int32_t* d_prev_iters = nullptr;  // iteration counts of the previous call
  bool lpt = true;
  int lpt_mode = 1;                // 1: least-likely-to-stall last (dojo_risk_key_kernel), 2: previous call's iteration counts, 0: index order
  int32_t* d_key = nullptr;        // sort keys of the work-queue order
  unsigned long long* d_prof = nullptr;
  // single-batch scratch of the environment, recording and minimal-coordinate steps, and the staging of dojo_step / dojo_step_trace
  double *d_Z = nullptr, *d_U = nullptr, *d_F = nullptr, *d_Zn = nullptr, *d_sol = nullptr;
  int32_t *d_status = nullptr, *d_iters = nullptr;
  double *p_in = nullptr, *p_out = nullptr;  // pinned, dojo_step / dojo_step_trace only
  char* d_stage = nullptr;  // grow-only staging arena of the other host-pointer calls (HostCall)
  size_t stage_bytes = 0;
  cudaStream_t stream = nullptr;
  // one call in flight per handle: the work queue counter, completion lists, staging and scratch buffers belong to the handle.
  // Calls on DIFFERENT streams are ordered behind each other through this event (enter_call / leave_call), so that an async call
  // on a caller stream followed by a call on another stream (or by a synchronous call, which runs on `stream`) cannot race on them.
  cudaEvent_t ev_last = nullptr;
  cudaStream_t last_stream = nullptr;
  bool has_last = false;
  int64_t launches = 0;
  bool any_contact = false;                       // the mechanism needs the DJ_ANY_CONTACT kernels (dojo_b200_cm.cu): it has ...
  bool orthant_contact = false;                   // ... an ImpactContact / LinearContact
  bool tra_joint = false;                         // ... or translational springs / dampers / limits
  const void *k_fwd = nullptr, *k_grad = nullptr;  // dojo_step_kernel<false> / <true> of the compilation that serves this mechanism
  const void* k_fwd_trace = nullptr;               // its traced variant, set up by the first dojo_step_trace call
  double* d_trace = nullptr;                       // grow-only device buffer of dojo_step_trace (host-pointer calls)
  size_t trace_doubles = 0;
  bool small_step = false;                         // k_fwd is dojo_step_kernel<false, true, false, SMALL = true>
  const void* k_fwd_rec = nullptr;                 // recording rollout kernel (REC), set up by the first dojo_rollout_grad call
  int envs_per_sm_rec = 1;
  // dojo_rollout_grad scratch per (environment, step) pair, grow-only: final solutions [nres x pairs], completion list [2 + pairs]
  // (as d_done), status and iterations [pairs]; the maximal trajectory [nz x B x (T + 1)] of dojo_rollout_minimal_gradients
  double* d_rsol = nullptr;
  int* d_rdone = nullptr;
  int32_t *d_rstatus = nullptr, *d_riters = nullptr;
  size_t rpairs = 0;
  double* d_rZ = nullptr;
  size_t rZ_bytes = 0;
  const void* k_fwd_fb = nullptr;                  // closed-loop rollout kernel (FB), set up by the first dojo_rollout_feedback call
  int envs_per_sm_fb = 1;
  double* d_fbX = nullptr;                         // FB scratch: x_t [2nu x max_batch], then u_t [nu x max_batch] (no U_applied)
  bool lqr_ready = false;                          // dojo_lqr_backward_kernel has the device's shared-memory maximum
  const void* k_vjp = nullptr;                     // adjoint kernel (VJP), set up by the first dojo_rollout_vjp call
  const void* k_fb_tape = nullptr;                 // closed-loop tape (REC + FB), set up by the first dojo_rollout_feedback_tape call
  const void* k_fb_vjp = nullptr;                  // closed-loop adjoint (VJP + FB), set up by the first dojo_rollout_feedback_vjp call
  int envs_per_sm_fb_tape = 1;
  double* d_fbvws = nullptr;                       // closed-loop adjoint scratch of the device-pointer calls (grow-only)
  size_t fbvws_bytes = 0;
  std::string err;
};
// Whether the forward kernel specialised for small mechanisms (dojo_step_kernel.cuh, SMALL) computes this handle's step exactly: the
// NonlinearContact-only compilation, 2 warps per environment, paired line-search trials and joint pairs, and at most 16 nodes in every
// role pass (at 2 warps the passes are the bodies, the contacts and the joints, all of a kind), with the whole plan in shared memory
// (plan_smem_mask: the tables dojo_create places there) read through the shared-memory array (not DOJO_B200_GENERIC_PLAN).
// DOJO_B200_GENERIC_STEP keeps the generic kernel (A/B measurements).
static bool small_step_ok(const DojoHandle* h, int plan_smem_mask) {
  const Plan& P = h->plan;
  return !h->any_contact && h->nw == 2 && P.nw == 2 && P.jpair && P.ls_pair && std::max(P.Nb, std::max(P.Ne, P.Ni)) <= 16 && plan_smem_mask == 0xff &&
         !getenv("DOJO_B200_GENERIC_PLAN") && !getenv("DOJO_B200_GENERIC_STEP");
}
// [hostemu:handle:end]

static std::string g_create_error;

#define CUDA_TRY(h, call)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (call);                                                               \
    if (_e != cudaSuccess) {                                                               \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(_e);                       \
      return DOJO_ECUDA;                                                                   \
    }                                                                                      \
  } while (0)

// Ordering of calls that use the handle's scratch (see DojoHandle::ev_last).  Free when every call uses the same stream.
static void enter_call(DojoHandle* h, cudaStream_t s) {
  if (h->has_last && h->last_stream != s && h->ev_last) cudaStreamWaitEvent(s, h->ev_last, 0);
}
static void leave_call(DojoHandle* h, cudaStream_t s) {
  if (!h->ev_last) return;
  cudaEventRecord(h->ev_last, s);
  h->last_stream = s; h->has_last = true;
}

extern "C" void dojo_default_options(DojoSolverOptions* o) {
  o->rtol = 1.0e-6; o->btol = 1.0e-4; o->ls_scale = 0.5; o->max_iter = 50; o->max_ls = 10;
  o->undercut = INFINITY; o->no_progress_max = 3; o->no_progress_undercut = 10.0; o->verbose = 0;
}

// Gives a kernel function the most dynamic shared memory the device allows (the opt-in maximum minus the kernel's static shared
// memory) and the max-shared carve-out.  The attributes belong to the kernel FUNCTION (per device), not to a handle: several handles
// (ant, pendulum, ...) share the kernel symbols, so they are set to the device's maximum once and for all -- a handle created later
// with a smaller arena must not lower them under the launches of an earlier, larger one
// (tests/test_gpu_parity.py::test_two_handles_share_kernels).
static cudaError_t max_shared_memory(const void* fn, int device) {
  int optin = 0;
  cudaFuncAttributes fa;
  cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fn);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  return e;
}

// [hostemu:padmask:begin]
static void pad_mask(const DojoJointElementDesc& e, double* C, double* A) {
  // joints/joint.jl:56-64 (constraint_mask / nullspace_mask), zero-padded to 3 rows
  std::memset(C, 0, 9 * sizeof(double));
  std::memset(A, 0, 9 * sizeof(double));
  const double* V1 = e.axis_mask; const double* V2 = e.axis_mask + 3; const double* V3_ = e.axis_mask + 6;
  const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  switch (e.nlambda) {
    case 0: std::memcpy(A, I3, sizeof(I3)); break;
    case 1: std::memcpy(C, V3_, 3 * sizeof(double)); std::memcpy(A, V1, 3 * sizeof(double)); std::memcpy(A + 3, V2, 3 * sizeof(double)); break;
    case 2: std::memcpy(C, V1, 3 * sizeof(double)); std::memcpy(C + 3, V2, 3 * sizeof(double)); std::memcpy(A, V3_, 3 * sizeof(double)); break;
    case 3: std::memcpy(C, I3, sizeof(I3)); break;
  }
}

// [hostemu:padmask:end]

extern "C" int dojo_create(const DojoMechanismDesc* d, int device, int max_batch, DojoHandle** out) {
  g_create_error.clear();
  if (!d || !out || max_batch <= 0) { g_create_error = "dojo_create: bad arguments"; return DOJO_EINVAL; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    g_create_error = "dojo_create: no usable CUDA device (this library has no CPU fallback)";
    return DOJO_ENODEVICE;
  }
  // [hostemu:tables:begin]
  const int Nb = d->num_bodies, Ne = d->num_joints, Ni = d->num_contacts;
  auto fail = [&](const char* msg) { g_create_error = std::string("dojo_create: ") + msg; return DOJO_EINVAL; };
  if (Nb < 1 || Nb > 32 || Ne > 32 || Ni > 32) return fail("this build supports up to 32 bodies / 32 joints / 32 contacts per mechanism");
  // ---- topology checks: tree with exactly one parent joint per body
  std::vector<int> parent_joint(Nb, -1);
  for (int j = 0; j < Ne; ++j) {
    const DojoJointDesc& jd = d->joints[j];
    if (jd.child_body < 0 || jd.child_body >= Nb || jd.parent_body < -1 || jd.parent_body >= Nb) return fail("joint body index out of range");
    if (parent_joint[jd.child_body] >= 0) return fail("loop-closure joints are not supported yet (each body needs exactly one parent joint)");
    parent_joint[jd.child_body] = j;
    if (jd.tra.nlimits != 0 && jd.tra.nlimits != 3 - jd.tra.nlambda) return fail("translational limits must cover every free axis");
    if (jd.tra.nlimits != 0 && jd.rot.nlimits != 0) return fail("limits on both the translational and the rotational part of one joint are not supported");
    if (jd.rot.nlimits != 0 && jd.rot.nlimits != 3 - jd.rot.nlambda) return fail("rotational limits must cover every free axis");
  }
  for (int b = 0; b < Nb; ++b) if (parent_joint[b] < 0) return fail("every body needs a parent joint (use a Floating joint to the origin)");
  for (int c = 0; c < Ni; ++c) {
    if (d->contacts[c].type < 0 || d->contacts[c].type > 2) return fail("contact type must be 0 (impact), 1 (linear) or 2 (nonlinear)");
    if (d->contacts[c].parent_body < 0 || d->contacts[c].parent_body >= Nb) return fail("contact body index out of range");
  }

  DojoHandle* h = new DojoHandle();
  h->device = device;
  h->max_batch = max_batch;
  cudaSetDevice(device);

  // ---- solution layout: joints | bodies | contacts (gradients/finite_difference.jl:1-18)
  std::vector<JointDev> joints(Ne);
  std::vector<BodyDev> bodies(Nb);
  std::vector<ContactDev> contacts(Ni);
  int off = 0, uoff = 0;
  for (int j = 0; j < Ne; ++j) {
    const DojoJointDesc& jd = d->joints[j];
    JointDev& J = joints[j];
    std::memset(&J, 0, sizeof(J));
    J.parent = jd.parent_body; J.child = jd.child_body;
    J.nl_t = jd.tra.nlambda; J.nl_r = jd.rot.nlambda; J.nb2_r = jd.rot.nlimits; J.nb_r = 2 * J.nb2_r;
    J.ne = J.nl_t + J.nl_r;
    J.n = J.ne + 2 * J.nb_r;
    J.sol_off = off; off += J.n;
    J.nfree_t = 3 - J.nl_t; J.nfree_r = 3 - J.nl_r;
    J.u_off = uoff; uoff += J.nfree_t + J.nfree_r;
    std::memcpy(J.pa, jd.vertex_parent, sizeof(J.pa));
    std::memcpy(J.pb, jd.vertex_child, sizeof(J.pb));
    std::memcpy(J.qoff, jd.orientation_offset, sizeof(J.qoff));
    pad_mask(jd.tra, J.Ct, J.At);
    pad_mask(jd.rot, J.Cr, J.Ar);
    J.spring_r = (jd.rot.nlambda < 3) ? jd.rot.spring : 0.0;
    J.damper_r = (jd.rot.nlambda < 3) ? jd.rot.damper : 0.0;
    for (int i = 0; i < 3; ++i) { J.spring_off_r[i] = jd.rot.spring_offset[i]; J.lo[i] = jd.rot.limit_lo[i]; J.hi[i] = jd.rot.limit_hi[i]; }
    if (J.nb2_r > 3) { delete h; return fail("too many limited axes"); }
    // translational springs / dampers / limits (joints/translational/springs.jl, dampers.jl, joints/limits.jl): flags + parameters in
    // the unused rows of Ct (dojo_plan.h); such mechanisms run on the DJ_ANY_CONTACT compilation of the kernels
    if (J.nfree_t > 0) {
      if (jd.tra.spring != 0.0) J.flags |= JF_TRA_SPRING;
      if (jd.tra.damper != 0.0) J.flags |= JF_TRA_DAMPER | JF_FULL;
      if (jd.tra.nlimits > 0) {
        J.flags |= JF_LIM_TRA | JF_FULL;
        J.nb2_r = jd.tra.nlimits; J.nb_r = 2 * J.nb2_r;
        J.n = J.ne + 2 * J.nb_r;
        off += 2 * J.nb_r;  // J.sol_off was assigned above with nb_r = 0
        for (int i = 0; i < 3; ++i) { J.lo[i] = jd.tra.limit_lo[i]; J.hi[i] = jd.tra.limit_hi[i]; }
      }
      if (J.flags & (JF_TRA_SPRING | JF_TRA_DAMPER)) {
        double* tp = joint_tra_params(J);
        tp[0] = jd.tra.spring; tp[1] = jd.tra.damper;
        for (int i = 0; i < J.nfree_t; ++i) tp[2 + i] = jd.tra.spring_offset[i];
      }
      if (J.flags) h->any_contact = h->tra_joint = true;
    }
  }
  const int nu = uoff;
  for (int b = 0; b < Nb; ++b) {
    BodyDev& B = bodies[b];
    std::memset(&B, 0, sizeof(B));
    B.mass = d->bodies[b].mass;
    std::memcpy(B.J, d->bodies[b].inertia, sizeof(B.J));
    B.sol_off = off; off += 6;
  }
  for (int c = 0; c < Ni; ++c) {
    const DojoContactDesc& cd = d->contacts[c];
    ContactDev& C = contacts[c];
    std::memset(&C, 0, sizeof(C));
    C.body = cd.parent_body; C.mu = cd.friction_coefficient; C.radius = cd.radius;
    std::memcpy(C.n, cd.normal, sizeof(C.n)); std::memcpy(C.t, cd.tangent, sizeof(C.t));
    std::memcpy(C.o, cd.origin, sizeof(C.o)); std::memcpy(C.off, cd.offset, sizeof(C.off));
    const int nh = cd.type == 0 ? 1 : (cd.type == 1 ? 6 : 4);  // N½: impact.jl:38, linear.jl:46, nonlinear.jl:47
    C.tn = cd.type | (nh << 8);
    if (cd.type != 2) h->any_contact = h->orthant_contact = true;
    C.sol_off = off; off += 2 * nh;
  }
  const int nres = off;

  // ---- warps per environment
  // 2 warps per environment (H100, ant B = 4096 forward: 2 warps 450 k env-steps/s, 1 warp 292 k, 4 warps 283 k).  Mechanisms with more than 16 nodes of a kind
  // (atlas: 31 bodies, 31 joints, 20 contacts) get 4: their arena only lets two environments share an SM (4 of the 8 warps the
  // register file holds), and with every role pass split in two halves of <= 16 nodes they can pair line-search trials on the
  // half-warps and assemble a joint on two lanes like the small mechanisms (round 2; atlas is where the solver stalls most:
  // 7.5 % of its environment-steps run into max_iter with ten line-search trials per iteration).
  int nw = (std::max(Nb, std::max(Ne, Ni)) > 16) ? 4 : 2;
  if (const char* e = getenv("DOJO_B200_WARPS")) nw = atoi(e);
  if (nw != 1 && nw != 2 && nw != 4 && nw != 8) nw = 2;
  h->nw = nw;

  // ---- arena layout: [sol | rhs | sav | reduction scratch | body state | body cst | joint slots | constant blocks |
  //                     re-zeroed region: contact slots, scratch records, matrix blocks]
  Plan& P = h->plan;
  std::memset(&P, 0, sizeof(P));
  P.Nb = Nb; P.Ne = Ne; P.Ni = Ni; P.nres = nres; P.nu = nu; P.nz = 13 * Nb; P.nw = nw;
  P.h = d->timestep; P.input_scaling = d->input_scaling;
  std::memcpy(P.g, d->gravity, sizeof(P.g));
  int a = 0;
  P.sol_off = a; a += nres;
  P.rhs_off = a; a += nres;
  P.sav_off = a; a += nres;
  P.red_off = a; a += 4 * nw + 2;
  for (int b = 0; b < Nb; ++b) { bodies[b].st_off = a; a += 7; }
  for (int b = 0; b < Nb; ++b) { bodies[b].cst_off = a; a += 6; }
  for (int j = 0; j < Ne; ++j) {  // joint contribution slots (also used by the prologue) and constant (per step) blocks
    JointDev& J = joints[j];
    const int slot_len = (J.flags & JF_FULL) ? kSlotC : kSlot;  // full joints: force(3) torque(3) K(6x6), like a contact
    J.slot_c = a; a += slot_len;
    if (J.parent >= 0) { J.slot_p = a; a += slot_len; } else J.slot_p = -1;
    J.Lc_off = a; a += 6 * joint_nq(J);
    if (J.parent >= 0) { J.Gp_off = a; a += 6 * joint_nq(J); } else J.Gp_off = -1;
    J.lim_off = a; a += ((J.flags & JF_FULL) ? 2 * kLim : kLim) * J.nb2_r;  // full: aP(6) aC(6) tP(6) tC(6) per limited axis
  }
  for (int c = 0; c < Ni; ++c) {  // contact records survive the assembly (used by condense / recover)
    ContactDev& C = contacts[c];
    C.slot = a; a += kSlotC;
    C.J_off = a; a += 6 * (C.tn >> 8);   // N½ x 6
    C.G_off = a; a += 6 * (C.tn >> 8);   // 6 x N½
    C.rec_off = a; a += 3;
  }
  P.mat_off = a;
  for (int j = 0; j < Ne; ++j) { if (joints[j].parent >= 0) { joints[j].S_off = a; a += kScratch; } else joints[j].S_off = -1; }
  for (int b = 0; b < Nb; ++b) { bodies[b].D_off = a; a += 36; }
  for (int j = 0; j < Ne; ++j) {
    JointDev& J = joints[j];
    const int nq = joint_nq(J);
    J.D_off = a; a += nq * nq;
    J.Uc_off = a; a += 6 * nq;
    if (J.parent >= 0) {
      J.Up_off = a; a += 6 * nq;
      J.Lp_off = a; a += 6 * nq;
      // body-body coupling exists with dampers and with (condensed) joint limits
      // (rotational terms touch the angular rows only: 3 x 6 and 3 x 3; translational dampers / limits need the full blocks)
      const bool bb_full = (J.flags & JF_FULL) != 0;
      if (J.damper_r != 0.0 || J.nb2_r > 0 || (J.flags & JF_TRA_DAMPER)) { J.BBpc_off = a; a += bb_full ? 36 : 18; J.BBcp_off = a; a += bb_full ? 36 : 9; } else { J.BBpc_off = J.BBcp_off = -1; }
    } else { J.Up_off = J.Lp_off = J.BBpc_off = J.BBcp_off = -1; }
  }
  P.mat_len = a - P.mat_off;
  P.arena_len = a;
  {  // paired line-search trials: shadow of the slot region + a second residual vector inside the (then dead) matrix region
    const int first_slot = Ne > 0 ? joints[0].slot_c : P.mat_off;
    const int span = P.mat_off - first_slot;
    // (every role pass must fit a half-warp: all of a kind on one warp with <= 16 nodes at 2 warps, halves of <= 32 at 4 warps)
    const int per_pass = (nw == 4) ? 32 : 16;
    P.ls_pair = ((nw == 2 || nw == 4) && Nb <= per_pass && Ne <= per_pass && Ni <= per_pass && span + nres <= P.mat_len && !getenv("DOJO_B200_NO_LS_PAIR")) ? 1 : 0;
    // two lanes per joint in set_entries! (eval_joint_pair): mechanisms with NonlinearContact and rotational joint terms only (the kernel
    // also requires <= 16 joints in the pass)
    P.jpair = (!h->any_contact && !getenv("DOJO_B200_NO_JOINT_PAIR")) ? 1 : 0;
    P.ls_assist = getenv("DOJO_B200_NO_LS_ASSIST") ? 0 : 1;
    P.ls_slot_delta = span;
    P.ls_res2_off = P.mat_off + span;
  }
  h->arena_bytes = (size_t)((a + 1) & ~1) * sizeof(double);  // 16-byte multiples: slots and the plan tables follow each other

  // ---- gradient workspace (appended to the arena; only the gradient kernel allocates it)
  std::vector<int> ucol;
  {
    int r = 0;
    for (int j = 0; j < Ne; ++j) { joints[j].r_off = r; r += joint_nq(joints[j]); }
    for (int b = 0; b < Nb; ++b) { bodies[b].r_off = r; r += 6; }
    P.n_red = r;
    P.ncol = 12 * Nb + nu;
    for (int j = 0; j < Ne; ++j)
      for (int k = 0; k < joints[j].nfree_t + joints[j].nfree_r; ++k) { ucol.push_back(j); ucol.push_back(k); }
    // every warp solves ch / nw columns of a chunk (dojo_grad.cuh gradients()), so the chunk never gets narrower than nw
    for (int pass = 0; pass < 4 && (32 >> pass) >= nw; ++pass) {
      P.ch = 32 >> pass;  // 32, 16, 8, 4 columns per chunk
      int g = P.arena_len;
      for (int b = 0; b < Nb; ++b) { bodies[b].gb_off = g; g += 30; }
      for (int c = 0; c < Ni; ++c) { contacts[c].gc_off = g; g += 36; }
      for (int j = 0; j < Ne; ++j) {
        JointDev& J = joints[j];
        J.gj_off = g; g += 12 * joint_nq(J) + 144 + 12 * (J.nfree_t + J.nfree_r);
        if (J.parent >= 0) { J.gv_off = g; g += 6 * P.ch; } else J.gv_off = -1;
      }
      P.gvec_off = g; g += P.n_red * P.ch;
      P.grad_len = g;
      // prefer two environments per SM; large mechanisms (atlas) shrink the chunk until one environment fits
      if ((size_t)g * sizeof(double) <= 113 * 1024) break;
      if (pass >= 1 && (size_t)P.arena_len * sizeof(double) > 100 * 1024 && (size_t)g * sizeof(double) <= 225 * 1024) break;
    }
    h->grad_bytes = (size_t)((P.grad_len + 1) & ~1) * sizeof(double);
  }

  // ---- gather lists (deterministic accumulation order): contacts of b, its parent joint (child side), its child joints
  std::vector<int> ilist;
  for (int b = 0; b < Nb; ++b) {
    bodies[b].g_off = (int)ilist.size();
    for (int c = 0; c < Ni; ++c) if (contacts[c].body == b) ilist.push_back(contacts[c].slot);
    bodies[b].g_ncontact = (int)ilist.size() - bodies[b].g_off;
    // full joints (6 x 6 slots) are marked with bit 30 of the gather entry; only the DJ_ANY_CONTACT kernels ever see such entries
    auto slot_entry = [&](const JointDev& J, int slot) { return (J.flags & JF_FULL) ? (slot | (1 << 30)) : slot; };
    ilist.push_back(slot_entry(joints[parent_joint[b]], joints[parent_joint[b]].slot_c));
    for (int j = 0; j < Ne; ++j) if (joints[j].parent == b) ilist.push_back(slot_entry(joints[j], joints[j].slot_p));
    bodies[b].g_cnt = (int)ilist.size() - bodies[b].g_off;
  }

  for (int b = 0; b < Nb; ++b) {  // adjacency for the gradient pass
    bodies[b].pjoint = parent_joint[b];
    bodies[b].cj_off = (int)ilist.size();
    for (int j = 0; j < Ne; ++j) if (joints[j].parent == b) ilist.push_back(j);
    bodies[b].cj_cnt = (int)ilist.size() - bodies[b].cj_off;
    bodies[b].ct_off = (int)ilist.size();
    for (int c = 0; c < Ni; ++c) if (contacts[c].body == b) ilist.push_back(c);
    bodies[b].ct_cnt = (int)ilist.size() - bodies[b].ct_off;
  }

  // ---- roles: which warp evaluates which nodes (one lane per node)
  std::vector<WarpRole> roles(nw);
  {
    for (auto& r : roles) std::memset(&r, 0, sizeof(r));
    auto add = [&](int w, int type, int first, int count) {
      if (count <= 0) return;
      WarpRole& r = roles[w];
      r.type[r.npass] = type; r.first[r.npass] = first; r.count[r.npass] = count; r.npass++;
    };
    if (nw == 1) { add(0, ROLE_BODY, 0, Nb); add(0, ROLE_CONTACT, 0, Ni); add(0, ROLE_JOINT, 0, Ne); }
    else if (nw == 2) { add(0, ROLE_BODY, 0, Nb); add(0, ROLE_CONTACT, 0, Ni); add(1, ROLE_JOINT, 0, Ne); }
    else if (nw == 4) {  // halves of every kind: bodies + contacts on warps 0 / 1, joints on warps 2 / 3 (every pass <= 16 nodes for <= 32 of a kind)
      const int hb = (Nb + 1) / 2, hc = (Ni + 1) / 2, hj = (Ne + 1) / 2;
      add(0, ROLE_BODY, 0, hb); add(0, ROLE_CONTACT, 0, hc);
      add(1, ROLE_BODY, hb, Nb - hb); add(1, ROLE_CONTACT, hc, Ni - hc);
      add(2, ROLE_JOINT, 0, hj); add(3, ROLE_JOINT, hj, Ne - hj);
    }
    else {
      int hb = (Nb + 1) / 2, hc = (Ni + 1) / 2, qj = (Ne + 3) / 4;
      add(0, ROLE_BODY, 0, hb); add(1, ROLE_BODY, hb, Nb - hb);
      add(2, ROLE_CONTACT, 0, hc); add(3, ROLE_CONTACT, hc, Ni - hc);
      for (int q = 0; q < 4; ++q) add(4 + q, ROLE_JOINT, q * qj, std::max(0, std::min(qj, Ne - q * qj)));
    }
  }

  // ---- elimination steps with heights; a parent body's diagonal / vector updates go to the joint's scratch record
  //      (contacts into bodies, bodies into their parent joint, joints into the parent body: SURVEY.md Appendix C)
  struct HStep { ElimStep s; int height; int group; double cost; };
  std::vector<HStep> hs;
  std::vector<int> body_height(Nb, 0);
  {
    std::vector<char> done(Nb, 0);
    struct Rec {
      std::vector<JointDev>& joints; std::vector<BodyDev>& bodies; std::vector<ContactDev>& contacts;
      const std::vector<int>& pj; std::vector<char>& done; std::vector<HStep>& hs; std::vector<int>& ilist; int Ne, Ni;
      int visit(int b) {  // returns the height of the parent-joint step of b (or of b if the joint has no impulses)
        done[b] = 1;
        int hb = 0;
        std::vector<int> fold, gfold;
        for (int j = 0; j < Ne; ++j)
          if (joints[j].parent == b && !done[joints[j].child]) {
            int hc = visit(joints[j].child);
            hb = std::max(hb, hc + 1);
            fold.push_back(joints[j].S_off);
            gfold.push_back(joints[j].gv_off);
          }
        const BodyDev& B = bodies[b];
        const JointDev& J = joints[pj[b]];
        {  // the body: neighbours = parent joint (if it has impulses) and, with dampers, the parent body
          HStep h; std::memset(&h, 0, sizeof(h));
          ElimStep& s = h.s;
          s.d_off = B.D_off; s.n = 6; s.vec_off = B.sol_off; s.r_off = B.r_off; s.nnb = 0;
          s.fold_off = (int)ilist.size(); s.fold_cnt = (int)fold.size();
          for (int f : fold) ilist.push_back(f);
          s.gfold_off = (int)ilist.size();
          for (int f : gfold) ilist.push_back(f);
          int ij = -1, ip = -1;
          if (joint_nq(J) > 0) {
            ij = s.nnb++;
            s.nb[ij].n = joint_nq(J); s.nb[ij].vec_off = J.sol_off; s.nb[ij].r_off = J.r_off; s.nb[ij].gv_off = -1; s.nb[ij].fwd_abs = -1; s.nb[ij].L_off = J.Uc_off; s.nb[ij].U_off = J.Lc_off; s.nb[ij].U_k = 6; s.nb[ij].U_row = 0;
            s.nb[ij].ld = joint_nq(J); s.nb[ij].row0 = 0;
          }
          int r0 = 0;  // first row of the parent body the coupling reaches: 3 (angular rows only) unless the joint carries full blocks
          if (J.parent >= 0 && J.BBpc_off >= 0) {
            ip = s.nnb++;
            const BodyDev& Pb = bodies[J.parent];
            r0 = (J.flags & JF_FULL) ? 0 : 3;
            s.nb[ip].n = 6 - r0; s.nb[ip].vec_off = Pb.sol_off + r0; s.nb[ip].r_off = Pb.r_off + r0; s.nb[ip].gv_off = J.gv_off; s.nb[ip].fwd_abs = J.S_off + 36 + r0;
            s.nb[ip].L_off = J.BBpc_off; s.nb[ip].U_off = J.BBcp_off; s.nb[ip].U_k = 6 - r0; s.nb[ip].U_row = r0;
            s.nb[ip].ld = 6; s.nb[ip].row0 = r0;
          }
          if (ij >= 0) s.tgt[ij][ij] = J.D_off;
          if (ip >= 0) s.tgt[ip][ip] = J.S_off + 7 * r0;                                  // rows / columns r0.. of the 6 x 6 scratch
          if (ij >= 0 && ip >= 0) { s.tgt[ij][ip] = J.Up_off + r0; s.tgt[ip][ij] = J.Lp_off + r0 * joint_nq(J); }  // columns r0.. of (joint, parent); rows r0.. of (parent, joint)
          h.height = hb; h.group = -1; h.cost = 4.0 + joint_nq(J) * 0.3;
          hs.push_back(h);
        }
        int hj = hb;
        if (joint_nq(J) > 0) {  // the parent joint: neighbour = parent body
          HStep h; std::memset(&h, 0, sizeof(h));
          ElimStep& s = h.s;
          s.d_off = J.D_off; s.n = joint_nq(J); s.vec_off = J.sol_off; s.r_off = J.r_off; s.nnb = 0;
          if (J.parent >= 0) {
            const BodyDev& Pb = bodies[J.parent];
            s.nnb = 1;
            s.nb[0].n = 6; s.nb[0].vec_off = Pb.sol_off; s.nb[0].r_off = Pb.r_off; s.nb[0].gv_off = J.gv_off; s.nb[0].fwd_abs = J.S_off + 36; s.nb[0].L_off = J.Lp_off; s.nb[0].U_off = J.Up_off; s.nb[0].U_k = joint_nq(J); s.nb[0].U_row = 0;
            s.nb[0].ld = 6; s.nb[0].row0 = 0;
            s.tgt[0][0] = J.S_off;
          }
          hj = hb + 1;
          h.height = hj; h.group = -1; h.cost = 2.0 + joint_nq(J) * 0.4;
          hs.push_back(h);
        }
        return hj;
      }
    } rec{joints, bodies, contacts, parent_joint, done, hs, ilist, Ne, Ni};
    for (int j = 0; j < Ne; ++j) if (joints[j].parent < 0 && !done[joints[j].child]) rec.visit(joints[j].child);
    for (int b = 0; b < Nb; ++b) if (!done[b]) { delete h; return fail("mechanism is not a tree rooted at the origin"); }
  }
  // ---- schedule: phase = height; the steps of a phase are independent and are spread over the warps (contacts of one
  //      body stay on one warp, they update the same diagonal block)
  int nphase = 0;
  for (auto& x : hs) nphase = std::max(nphase, x.height + 1);
  std::vector<ElimStep> steps;
  std::vector<int> sched((size_t)nphase * nw * 2, 0);
  for (int ph = 0; ph < nphase; ++ph) {
    std::vector<std::vector<int>> per_warp(nw);
    std::vector<double> load(nw, 0.0);
    std::vector<int> group_warp(Nb, -1);
    for (int i = 0; i < (int)hs.size(); ++i) {
      if (hs[i].height != ph) continue;
      int w;
      if (hs[i].group >= 0 && group_warp[hs[i].group] >= 0) w = group_warp[hs[i].group];
      else {
        w = 0;
        for (int k = 1; k < nw; ++k) if (load[k] < load[w]) w = k;
        if (hs[i].group >= 0) group_warp[hs[i].group] = w;
      }
      per_warp[w].push_back(i);
      load[w] += hs[i].cost;
    }
    for (int w = 0; w < nw; ++w) {
      sched[2 * (ph * nw + w)] = (int)steps.size();
      sched[2 * (ph * nw + w) + 1] = (int)per_warp[w].size();
      for (int i : per_warp[w]) steps.push_back(hs[i].s);
    }
  }
  P.nphase = nphase;
  h->nsteps = (int)steps.size();
  {  // ---- the LDU program (dojo_plan.h LduOp), appended to the schedule table
    std::vector<int> cnt((size_t)nphase * nw), wfirst(nw);
    std::vector<LduOp> ops;
    bool fits = true;  // every offset below kLduNone, every size below 256
    auto u16 = [&](int v) { fits = fits && v >= 0 && v < kLduNone; return v & 0xffff; };
    auto u8 = [&](int v) { fits = fits && v >= 0 && v < 256; return v & 0xff; };
    for (int w = 0; w < nw; ++w) {
      wfirst[w] = (int)ops.size();
      for (int ph = 0; ph < nphase; ++ph) {
        const int s0 = sched[2 * (ph * nw + w)], sn = sched[2 * (ph * nw + w) + 1];
        cnt[ph * nw + w] = sn;
        for (int s = s0; s < s0 + sn; ++s) {
          const ElimStep& st = steps[s];
          int f[kLduFold] = {0, 0, 0};
          for (int k = 0; k < std::min(st.fold_cnt, kLduFold); ++k) f[k] = ilist[st.fold_off + k];
          LduOp op;
          std::memset(&op, 0, sizeof(op));
          op.w[0] = u16(st.d_off) | u16(st.vec_off) << 16;
          op.w[1] = u8(st.n) | u8(st.nnb) << 8 | u16(st.fold_cnt) << 16;
          op.w[2] = u16(st.fold_off) | u16(f[0]) << 16;
          op.w[3] = u16(f[1]) | u16(f[2]) << 16;
          for (int i = 0; i < st.nnb; ++i) {
            const ElimNb& nb = st.nb[i];
            int* q = op.w + 4 * (1 + i);
            q[0] = u16(nb.L_off) | (nb.fwd_abs >= 0 ? u16(nb.fwd_abs) : kLduNone) << 16;
            q[1] = u16(nb.vec_off) | u16(nb.U_off) << 16;
            q[2] = u8(nb.n) | u8(nb.U_row) << 8 | u8(nb.U_k) << 16 | u8(nb.ld) << 24;
            q[3] = u16(st.tgt[i][0]) | (st.nnb > 1 ? u16(st.tgt[i][1]) : 0) << 16;
          }
          ops.push_back(op);
        }
      }
    }
    if (!fits) { delete h; return fail("the block LDU program does not fit its 16-bit offsets"); }
    P.prog_cnt = (int)sched.size();
    sched.insert(sched.end(), cnt.begin(), cnt.end());
    sched.insert(sched.end(), wfirst.begin(), wfirst.end());
    sched.resize((sched.size() + 3) & ~size_t(3), 0);  // the ops start on a 16-byte boundary of the (16-byte aligned) table
    P.prog_ops = (int)sched.size();
    const int* words = reinterpret_cast<const int*>(ops.data());
    sched.insert(sched.end(), words, words + ops.size() * (sizeof(LduOp) / sizeof(int)));
  }
  // [hostemu:tables:end]

  // ---- device resources
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete h; g_create_error = "cudaGetDeviceProperties failed"; return DOJO_ECUDA; }
  h->sm_count = prop.multiProcessorCount;
  if (h->arena_bytes > (size_t)prop.sharedMemPerBlockOptin) {
    delete h;
    g_create_error = "dojo_create: mechanism does not fit the per-environment shared-memory arena";
    return DOJO_ENOMEM;
  }
  auto upload = [&](const void* src, size_t bytes, void** dst) -> bool {
    if (bytes == 0) { *dst = nullptr; return true; }
    if (cudaMalloc(dst, bytes) != cudaSuccess) return false;
    return cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice) == cudaSuccess;
  };
  // [hostemu:blob:begin]
  std::vector<char> blob;
  {
    const void* src[8] = {bodies.data(), joints.data(), contacts.data(), steps.data(), sched.data(), ilist.data(), roles.data(), ucol.data()};
    const size_t len[8] = {sizeof(BodyDev) * Nb, sizeof(JointDev) * Ne, sizeof(ContactDev) * Ni, sizeof(ElimStep) * steps.size(), sizeof(int) * sched.size(),
                           sizeof(int) * ilist.size(), sizeof(WarpRole) * roles.size(), sizeof(int) * ucol.size()};
    // physical order: the tables walked by the serial phases of the solver (schedule with the LDU program, elimination steps, lists,
    // roles) first, the per-node descriptors (read by one lane per node) last, so that a PREFIX of the blob can ride in shared memory
    // when the whole does not fit behind the arenas (atlas: 2 x 102.5 KiB leave 21 KiB, quadruped's gradient pass 2 x 108.4 KiB leave
    // 9.2 KiB)
    const int order[8] = {4, 3, 5, 6, 7, 0, 2, 1};
    for (int q = 0; q < 8; ++q) {
      const int k = order[q];
      h->blob_off[k] = (int)blob.size();
      blob.insert(blob.end(), (const char*)src[k], (const char*)src[k] + len[k]);
      blob.resize((blob.size() + 15) & ~size_t(15), 0);
      h->blob_end[k] = (int)blob.size();
    }
    h->blob_bytes = (int)blob.size();
  }
  // [hostemu:blob:end]
  bool ok = upload(blob.data(), blob.size(), (void**)&h->d_blob);
  {  // joints root -> leaves: a joint is placed once its parent body has been placed (mechanism.root_to_leaves restricted to joints)
    std::vector<int> order;
    std::vector<char> placed(Nb, 0), used(Ne, 0);
    for (bool progress = true; progress && (int)order.size() < Ne;) {
      progress = false;
      for (int j = 0; j < Ne; ++j)
        if (!used[j] && (joints[j].parent < 0 || placed[joints[j].parent])) { order.push_back(j); used[j] = 1; placed[joints[j].child] = 1; progress = true; }
    }
    ok = ok && (int)order.size() == Ne && upload(order.data(), sizeof(int) * Ne, (void**)&h->d_kin_order);
  }
  ok = ok && cudaMalloc((void**)&h->d_counter, sizeof(int)) == cudaSuccess;
  ok = ok && cudaMalloc((void**)&h->d_order, sizeof(int) * max_batch) == cudaSuccess && cudaMalloc((void**)&h->d_prev_iters, sizeof(int32_t) * max_batch) == cudaSuccess &&
       cudaMemset(h->d_prev_iters, 0, sizeof(int32_t) * max_batch) == cudaSuccess;
  if (const char* e = getenv("DOJO_B200_LPT")) { h->lpt = atoi(e) != 0; h->lpt_mode = atoi(e); }
  ok = ok && cudaMalloc((void**)&h->d_key, sizeof(int32_t) * max_batch) == cudaSuccess;
  ok = ok && cudaMalloc((void**)&h->d_prof, (32 + 2 * (size_t)max_batch) * sizeof(unsigned long long)) == cudaSuccess && cudaMemset(h->d_prof, 0, 32 * sizeof(unsigned long long)) == cudaSuccess &&
       cudaMemset(h->d_prof + 31, 0xff, sizeof(unsigned long long)) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&h->ev_last, cudaEventDisableTiming) == cudaSuccess;
  // environments per CTA ("slots"): as many arenas as fit, at most 256 threads (the register file holds 256 threads at 255 registers)
  auto pick_slots = [&](size_t bytes) {
    int g = (int)std::min<size_t>((size_t)prop.sharedMemPerBlockOptin / bytes, (size_t)(256 / (32 * nw)));
    g = std::max(1, std::min(g, 8));
    if (const char* e = getenv("DOJO_B200_SLOTS")) { int v = atoi(e); if (v >= 1 && v <= g) g = v; }
    return g;
  };
  h->slots = pick_slots(h->arena_bytes);
  // the plan tables ride along in shared memory when they fit behind the arenas
  const bool smem_plan = !getenv("DOJO_B200_GLOBAL_PLAN");
  // largest prefix of the blob (whole tables) that fits behind `n` arenas of `bytes` (32 bytes of static shared memory are reserved)
  auto plan_prefix = [&](int n, size_t bytes, int* off, int* pbytes, int* mask) {
    *off = -1; *pbytes = 0; *mask = 0;
    if (!smem_plan) return;
    const size_t room = (size_t)prop.sharedMemPerBlockOptin - 1024 - n * bytes;  // 1 KB: static shared memory of the kernel (mailbox, mbarrier)
    for (int k = 0; k < 8; ++k)
      if ((size_t)h->blob_end[k] <= room) { *mask |= 1 << k; *pbytes = std::max(*pbytes, h->blob_end[k]); }
    for (int k = 0; k < 8; ++k)  // a prefix: drop tables that start beyond the copied bytes (cannot happen with the ordered blob, kept for safety)
      if (((*mask >> k) & 1) && h->blob_end[k] > *pbytes) *mask &= ~(1 << k);
    if (*mask) *off = (int)(n * bytes / sizeof(double));
  };
  plan_prefix(h->slots, h->arena_bytes, &h->plan_smem_off, &h->plan_smem_bytes, &h->plan_smem_mask);
  h->smem_fwd = h->slots * h->arena_bytes + h->plan_smem_bytes;
  h->small_step = small_step_ok(h, h->plan_smem_mask);
  h->k_fwd = step_kernel_fn(h->any_contact, false, h->plan_smem_mask == 0xff, h->small_step);
  h->k_grad = step_kernel_fn(h->any_contact, true, false);  // re-selected below once the gradient configuration is known
  ok = ok && max_shared_memory(h->k_fwd, device) == cudaSuccess;
  const bool grad_fits = h->grad_bytes <= (size_t)prop.sharedMemPerBlockOptin;
  if (grad_fits) {
    h->slots_grad = pick_slots(h->grad_bytes);
    plan_prefix(h->slots_grad, h->grad_bytes, &h->plan_smem_off_grad, &h->plan_smem_bytes_grad, &h->plan_smem_mask_grad);
    h->smem_grad = h->slots_grad * h->grad_bytes + h->plan_smem_bytes_grad;
    h->k_grad = step_kernel_fn(h->any_contact, true, h->plan_smem_mask_grad == 0xff);
    ok = ok && max_shared_memory(h->k_grad, device) == cudaSuccess;
  } else h->grad_bytes = 0;
  if (!ok) { g_create_error = std::string("dojo_create: device allocation failed: ") + cudaGetErrorString(cudaGetLastError()); dojo_destroy(h); return DOJO_ECUDA; }
  // the device code reaches the tables through Ctx (shared-memory copy or this blob); the Plan pointers are kept for debugging
  P.bodies = (const BodyDev*)(h->d_blob + h->blob_off[0]); P.joints = (const JointDev*)(h->d_blob + h->blob_off[1]);
  P.contacts = (const ContactDev*)(h->d_blob + h->blob_off[2]); P.steps = (const ElimStep*)(h->d_blob + h->blob_off[3]);
  P.sched = (const int*)(h->d_blob + h->blob_off[4]); P.ilist = (const int*)(h->d_blob + h->blob_off[5]);
  P.roles = (const WarpRole*)(h->d_blob + h->blob_off[6]); P.ucol = (const int*)(h->d_blob + h->blob_off[7]);
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, h->k_fwd, 32 * h->nw * h->slots, h->smem_fwd);
  h->envs_per_sm = std::max(1, occ);
  if (h->grad_bytes) { occ = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, h->k_grad, 32 * h->nw * h->slots_grad, h->smem_grad); h->envs_per_sm_grad = std::max(1, occ); }
  *out = h;
  return DOJO_OK;
}

extern "C" int dojo_destroy(DojoHandle* h) {
  if (!h) return DOJO_OK;
  cudaSetDevice(h->device);
  cudaFree(h->d_key); cudaFree(h->d_order); cudaFree(h->d_prev_iters); cudaFree(h->d_prof); cudaFree(h->d_blob); cudaFree(h->d_counter); cudaFree(h->d_kin_order); cudaFree(h->d_kjws); cudaFree(h->d_recZ[0]); cudaFree(h->d_recZ[1]); cudaFree(h->d_recS); cudaFree(h->d_recD); cudaFree(h->d_recAny); cudaFree(h->d_envNorm); cudaFree(h->d_envS); cudaFree(h->d_envSn); cudaFree(h->d_envA); cudaFree(h->d_envR); cudaFree(h->d_envS0); cudaFree(h->d_envDone); cudaFree(h->d_gsol); cudaFree(h->d_gstatus); cudaFree(h->d_done); cudaFree(h->d_trace);
  for (int k = 0; k < 2; ++k) { cudaFree(h->d_Fz[k]); cudaFree(h->d_Fu[k]); if (h->ev_kernel[k]) cudaEventDestroy(h->ev_kernel[k]); if (h->ev_copy[k]) cudaEventDestroy(h->ev_copy[k]); }
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  cudaFree(h->d_Z); cudaFree(h->d_U); cudaFree(h->d_F); cudaFree(h->d_Zn); cudaFree(h->d_sol); cudaFree(h->d_status); cudaFree(h->d_iters);
  if (h->p_in) cudaFreeHost(h->p_in);
  if (h->p_out) cudaFreeHost(h->p_out);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->ev_last) cudaEventDestroy(h->ev_last);
  cudaFree(h->d_stage);
  cudaFree(h->d_rsol); cudaFree(h->d_rdone); cudaFree(h->d_rstatus); cudaFree(h->d_riters); cudaFree(h->d_rZ);
  cudaFree(h->d_fbX);
  cudaFree(h->d_fbvws);
  delete h;
  return DOJO_OK;
}

extern "C" const char* dojo_last_error(const DojoHandle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }
extern "C" int dojo_num_state(const DojoHandle* h) { return h->plan.nz; }
extern "C" int dojo_num_input(const DojoHandle* h) { return h->plan.nu; }
extern "C" int dojo_num_residual(const DojoHandle* h) { return h->plan.nres; }
extern "C" int dojo_num_grad_state(const DojoHandle* h) { return 12 * h->plan.Nb; }
extern "C" int dojo_shared_bytes_per_env(const DojoHandle* h) { return (int)h->arena_bytes; }
extern "C" int64_t dojo_launch_count(const DojoHandle* h) { return h->launches; }
// debugging aid (DJ_PROFILE builds): cycle counters accumulated by thread 0 of every CTA; out[5]
// launch configuration chosen by dojo_create (diagnostics: tools/prof_one.py prints it): [slots, slots_grad, gradient chunk width,
// arena bytes, gradient arena bytes, dynamic smem forward, dynamic smem gradient, plan-in-smem mask forward, mask gradient, paired
// line-search trials, elimination phases, elimination steps, plan blob bytes, warps per environment, resident CTAs / SM fwd, grad,
// forward kernel specialised for small mechanisms]
extern "C" int dojo_debug_config(const DojoHandle* h, int* out) {
  if (!h || !out) return DOJO_EINVAL;
  const int v[17] = {h->slots, h->slots_grad, h->plan.ch, (int)h->arena_bytes, (int)h->grad_bytes, (int)h->smem_fwd, (int)h->smem_grad,
                     h->plan_smem_mask, h->plan_smem_mask_grad, h->plan.ls_pair, h->plan.nphase, h->nsteps, h->blob_bytes, h->nw, h->envs_per_sm,
                     h->envs_per_sm_grad, h->small_step ? 1 : 0};
  for (int i = 0; i < 17; ++i) out[i] = v[i];
  return DOJO_OK;
}
extern "C" int dojo_debug_cycles(DojoHandle* h, unsigned long long* out) {
  cudaMemcpy(out, h->d_prof, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
  cudaMemset(h->d_prof, 0, 32 * sizeof(unsigned long long));
  cudaMemset(h->d_prof + 31, 0xff, sizeof(unsigned long long));
  return DOJO_OK;
}
// DJ_PROFILE builds: per-environment (start ns since the first CTA of the launch, duration ns) of the last launch
extern "C" int dojo_debug_env_times(DojoHandle* h, unsigned long long* out, int B) {
  cudaMemcpy(out, h->d_prof + 32, 2 * (size_t)B * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
  return DOJO_OK;
}

// [hostemu:options:begin]
static Options make_options(const DojoSolverOptions* o) {
  DojoSolverOptions d;
  if (!o) { dojo_default_options(&d); o = &d; }
  Options r;
  r.rtol = o->rtol; r.btol = o->btol; r.undercut = o->undercut; r.no_progress_undercut = o->no_progress_undercut;
  r.max_iter = o->max_iter; r.max_ls = o->max_ls; r.no_progress_max = o->no_progress_max;
  return r;
}
// [hostemu:options:end]

// The kernel arguments every launch starts from: all zero, except the plan, the solver options, the batch, one time step, the handle's
// work-queue counter and profile counters, and where the plan tables lie in the forward or (grad) the gradient launch configuration
static StepArgs step_args(const DojoHandle* h, const DojoSolverOptions* opts, int B, bool grad) {
  StepArgs a = {};
  a.plan = h->plan; a.opts = make_options(opts); a.B = B; a.T = 1;
  a.counter = h->d_counter; a.prof = h->d_prof;
  a.slot_stride = (int)((grad ? h->grad_bytes : h->arena_bytes) / sizeof(double));
  a.plan_blob = h->d_blob; a.plan_bytes = h->blob_bytes;
  a.plan_smem_off = grad ? h->plan_smem_off_grad : h->plan_smem_off;
  a.plan_smem_bytes = grad ? h->plan_smem_bytes_grad : h->plan_smem_bytes;
  a.plan_smem_mask = grad ? h->plan_smem_mask_grad : h->plan_smem_mask;
  for (int k = 0; k < 8; ++k) a.plan_off[k] = h->blob_off[k];
  return a;
}

static int launch_forward(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext, double* dZn, double* dsol,
                          double* dsol_raw, int32_t* dstatus, int32_t* diters, uint32_t flags, cudaStream_t s, int* done_count = nullptr, int* done_list = nullptr,
                          DojoGather* g = nullptr, double* dtrace = nullptr) {
  StepArgs a = step_args(h, opts, B, false);
  a.trace = dtrace;  // non-null: the traced kernel (dojo_step_trace_async)
  if (g) {
    if (!g->connected || g->h != h || B != g->B) { h->err = "dojo_step_gather_async: gather not connected / made for another handle / B differs from B_local"; return DOJO_EINVAL; }
    a.n_peers = g->world;
    a.gather_off = (long long)((size_t)g->parity * g->half) + (long long)g->rank * g->B * h->plan.nz;
    g->last = g->parity; g->parity ^= 1;
    for (int r = 0; r < g->world; ++r) { a.peer_buf[r] = g->peer_buf[r]; a.peer_flag[r] = g->peer_flag[r]; }
  }
  a.Z = dZ; a.U = dU; a.Fext = dFext; a.Zn = dZn; a.sol = dsol; a.sol_raw = dsol_raw; a.status = dstatus; a.iters = diters; a.flags = flags;
  a.done_count = done_count; a.done_list = done_list;
  // LPT order from the previous call's iteration counts (only meaningful when the same batch is stepped again, which is what
  // simulation loops do; a stale order is harmless -- it is just an order)
  enter_call(h, s);
  const bool lpt = h->lpt && B <= h->max_batch && B > h->sm_count * h->envs_per_sm * h->slots;
  a.order = lpt ? h->d_order : nullptr;
  a.prev_iters = (h->lpt && B <= h->max_batch) ? h->d_prev_iters : nullptr;
  if (lpt) {
    if (h->lpt_mode == 2) dojo_order_kernel<<<1, 1024, 0, s>>>(h->d_prev_iters, B, h->d_order, 1);
    else {
      dojo_risk_key_kernel<<<(B + 127) / 128, 128, 0, s>>>(dZ, B, h->plan.Nb, h->lpt_mode == 3 ? nullptr : h->d_prev_iters, h->d_key);
      dojo_order_kernel<<<1, 1024, 0, s>>>(h->d_key, B, h->d_order, 0);
      h->launches += 1;
    }
    CUDA_TRY(h, cudaGetLastError());
    h->launches += 1;
  }
  CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  int grid = std::min((B + h->slots - 1) / h->slots, h->sm_count * h->envs_per_sm);
  const void* k = dtrace ? h->k_fwd_trace : h->k_fwd;
  { void* kargs[1] = {(void*)&a}; CUDA_TRY(h, cudaLaunchKernel(k, dim3(grid), dim3(32 * h->nw * h->slots), kargs, h->smem_fwd, s)); }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  if (g) g->expected += (unsigned long long)g->world * (unsigned long long)grid;  // every rank launches the same grid (same B_local, same device type)
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_step_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext,
                               double* dZn, double* dsol, int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream) {
  if (!h || B <= 0 || !dZ || !dZn) { if (h) h->err = "dojo_step_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return launch_forward(h, opts, B, dZ, dU, dFext, dZn, dsol, nullptr, dstatus, diters, flags, (cudaStream_t)cuda_stream);
}

static bool is_device_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// page-locked host memory (cudaMallocHost / cudaHostRegister / torch pin_memory): DMA goes straight from / to the caller's buffer
static bool is_pinned_host_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeHost;
}

// grow-only device buffer; a buffer that is replaced may still be read by the handle's last call
static int grow_buffer(DojoHandle* h, void** buf, size_t* have, size_t need) {
  if (*have >= need) return DOJO_OK;
  CUDA_TRY(h, cudaDeviceSynchronize());
  cudaFree(*buf); *buf = nullptr; *have = 0;
  CUDA_TRY(h, cudaMalloc(buf, need));
  *have = need;
  return DOJO_OK;
}

// The arrays of one synchronous host- or device-pointer entry (every entry but dojo_step / dojo_step_trace).  The pointer kind is
// decided once, from the call's first array; the others are of the same kind.  Device pointers pass through.  With host pointers each
// declared array gets a 256-byte aligned slice of the handle's grow-only staging arena (a null or empty array gets none, and a null
// pointer): bind() points the caller's variables at the slices and copies the inputs in, finish() copies the non-null outputs out, both
// on h->stream and straight from / to the caller's buffers.  finish() ends the call with one synchronisation in either case.
struct HostCall {
  enum { IN = 1, OUT = 2, SCRATCH = 4 };
  struct Array { void* var; const void* host; size_t bytes; int use; size_t off; };
  DojoHandle* h;
  bool dev;
  std::vector<Array> arrays;
  HostCall(DojoHandle* h, const void* first) : h(h), dev(is_device_ptr(first)) {}
  // *p holds the caller's array of n elements; scratch: device memory of host-pointer calls only
  template <class T> void in(T** p, size_t n) { arrays.push_back({(void*)p, (const void*)*p, n * sizeof(T), IN, 0}); }
  template <class T> void out(T** p, size_t n) { arrays.push_back({(void*)p, (const void*)*p, n * sizeof(T), OUT, 0}); }
  template <class T> void inout(T** p, size_t n) { arrays.push_back({(void*)p, (const void*)*p, n * sizeof(T), IN | OUT, 0}); }
  template <class T> void scratch(T** p, size_t n) { arrays.push_back({(void*)p, nullptr, n * sizeof(T), SCRATCH, 0}); }
  int bind() {
    if (dev) return DOJO_OK;
    size_t total = 0;
    for (Array& a : arrays) {
      if (!a.host && a.use != SCRATCH) a.bytes = 0;
      a.off = total;
      total += (a.bytes + 255) & ~size_t(255);
    }
    int rc = grow_buffer(h, (void**)&h->d_stage, &h->stage_bytes, total);
    if (rc != DOJO_OK) return rc;
    for (Array& a : arrays) {
      char* d = a.bytes ? h->d_stage + a.off : nullptr;
      std::memcpy(a.var, &d, sizeof(d));  // the caller's T* variable now points at the slice
      if (a.bytes && (a.use & IN)) CUDA_TRY(h, cudaMemcpyAsync(d, a.host, a.bytes, cudaMemcpyHostToDevice, h->stream));
    }
    return DOJO_OK;
  }
  // rc: the entry's result so far; an error is returned as it is
  int finish(int rc = DOJO_OK) {
    if (rc != DOJO_OK) return rc;
    for (const Array& a : arrays)
      if (!dev && a.bytes && (a.use & OUT)) CUDA_TRY(h, cudaMemcpyAsync((void*)a.host, h->d_stage + a.off, a.bytes, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return DOJO_OK;
  }
};

static int ensure_staging(DojoHandle* h) {
  if (h->d_Z) return DOJO_OK;
  const Plan& P = h->plan;
  size_t B = h->max_batch;
  CUDA_TRY(h, cudaMalloc((void**)&h->d_Z, B * P.nz * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_U, std::max<size_t>(1, B * P.nu) * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_F, B * 6 * P.Nb * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_Zn, B * P.nz * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_sol, B * P.nres * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_status, B * sizeof(int32_t)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_iters, B * sizeof(int32_t)));
  CUDA_TRY(h, cudaMallocHost((void**)&h->p_in, B * (P.nz + P.nu + 6 * P.Nb) * sizeof(double)));
  CUDA_TRY(h, cudaMallocHost((void**)&h->p_out, B * (P.nz + P.nres + 2) * sizeof(double)));
  return DOJO_OK;
}

// ---- traced step! (solver/mehrotra.jl verbose mode): dojo_step + one row per loop-head test of the solver (include/dojo_b200.h)
// The traced kernel is set up on first use, with the shared-memory attributes dojo_create gives k_fwd.
static int ensure_trace_kernel(DojoHandle* h) {
  if (h->k_fwd_trace) return DOJO_OK;
  const void* k = step_trace_kernel_fn(h->any_contact, h->plan_smem_mask == 0xff);
  CUDA_TRY(h, max_shared_memory(k, h->device));
  h->k_fwd_trace = k;
  return DOJO_OK;
}

extern "C" int dojo_step_trace_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext,
                                     double* dZn, double* dsol, int32_t* dstatus, int32_t* diters, double* dtrace, uint32_t flags, void* cuda_stream) {
  if (!h || B <= 0 || !dZ || !dZn || !dtrace) { if (h) h->err = "dojo_step_trace_async: bad arguments (trace is required)"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_trace_kernel(h);
  if (rc != DOJO_OK) return rc;
  return launch_forward(h, opts, B, dZ, dU, dFext, dZn, dsol, nullptr, dstatus, diters, flags, (cudaStream_t)cuda_stream, nullptr, nullptr, nullptr, dtrace);
}

// Host- or device-pointer entry of dojo_step and, with a trace buffer, dojo_step_trace: host buffers are staged through pinned memory,
// copies are part of the call.
static int step_sync(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, const double* Fext, double* Zn,
                     double* sol, int32_t* status, int32_t* iters, double* trace, uint32_t flags) {
  CUDA_TRY(h, cudaSetDevice(h->device));
  const Plan& P = h->plan;
  auto launch = [&](const double* dZ, const double* dU, const double* dF, double* dZn, double* dsol, int32_t* dst, int32_t* dit, double* dtr,
                    cudaStream_t s) {
    return trace ? dojo_step_trace_async(h, opts, B, dZ, dU, dF, dZn, dsol, dst, dit, dtr, flags, s)
                 : dojo_step_async(h, opts, B, dZ, dU, dF, dZn, dsol, dst, dit, flags, s);
  };
  if (is_device_ptr(Z)) {  // resident data: launch on the handle's stream and wait
    int rc = launch(Z, U, Fext, Zn, sol, status, iters, trace, h->stream);
    if (rc != DOJO_OK) return rc;
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return DOJO_OK;
  }
  int rc = ensure_staging(h);
  if (rc != DOJO_OK) return rc;
  const size_t ntr = trace ? (size_t)5 * std::max(0, make_options(opts).max_iter) * B : 0;
  if (trace && std::max<size_t>(ntr, 1) > h->trace_doubles) {  // grow-only device buffer of the trace (never null: max_iter may be 0)
    cudaFree(h->d_trace);
    h->d_trace = nullptr; h->trace_doubles = 0;
    CUDA_TRY(h, cudaMalloc((void**)&h->d_trace, std::max<size_t>(ntr, 1) * sizeof(double)));
    h->trace_doubles = std::max<size_t>(ntr, 1);
  }
  cudaStream_t s = h->stream;
  // inputs: pageable buffers are staged through the handle's pinned buffer, pinned ones are copied from directly
  auto h2d = [&](double* dst, const double* src, double* stage, size_t n) -> cudaError_t {
    if (!is_pinned_host_ptr(src)) { std::memcpy(stage, src, n * sizeof(double)); src = stage; }
    return cudaMemcpyAsync(dst, src, n * sizeof(double), cudaMemcpyHostToDevice, s);
  };
  double* pz = h->p_in;
  double* pu = pz + (size_t)B * P.nz;
  double* pf = pu + (size_t)B * P.nu;
  CUDA_TRY(h, h2d(h->d_Z, Z, pz, (size_t)B * P.nz));
  if (U && P.nu > 0) CUDA_TRY(h, h2d(h->d_U, U, pu, (size_t)B * P.nu));
  if (Fext) CUDA_TRY(h, h2d(h->d_F, Fext, pf, (size_t)B * 6 * P.Nb));
  rc = launch(h->d_Z, (U && P.nu > 0) ? h->d_U : nullptr, Fext ? h->d_F : nullptr, h->d_Zn, sol ? h->d_sol : nullptr, h->d_status, h->d_iters,
              trace ? h->d_trace : nullptr, s);
  if (rc != DOJO_OK) return rc;
  // outputs: one stream synchronisation; pageable destinations receive a host copy out of the pinned staging buffer
  double* po = h->p_out;
  double* ps = po + (size_t)B * P.nz;
  int32_t* pst = (int32_t*)(ps + (size_t)B * P.nres);
  int32_t* pit = pst + B;
  const bool zn_pin = is_pinned_host_ptr(Zn), sol_pin = sol && is_pinned_host_ptr(sol);
  const bool st_pin = status && is_pinned_host_ptr(status), it_pin = iters && is_pinned_host_ptr(iters);
  CUDA_TRY(h, cudaMemcpyAsync(zn_pin ? Zn : po, h->d_Zn, (size_t)B * P.nz * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (sol) CUDA_TRY(h, cudaMemcpyAsync(sol_pin ? sol : ps, h->d_sol, (size_t)B * P.nres * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (status) CUDA_TRY(h, cudaMemcpyAsync(st_pin ? status : pst, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (iters) CUDA_TRY(h, cudaMemcpyAsync(it_pin ? iters : pit, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (ntr) CUDA_TRY(h, cudaMemcpyAsync(trace, h->d_trace, ntr * sizeof(double), cudaMemcpyDeviceToHost, s));  // a diagnostic: no staging
  CUDA_TRY(h, cudaStreamSynchronize(s));
  if (!zn_pin) std::memcpy(Zn, po, (size_t)B * P.nz * sizeof(double));
  if (sol && !sol_pin) std::memcpy(sol, ps, (size_t)B * P.nres * sizeof(double));
  if (status && !st_pin) std::memcpy(status, pst, B * sizeof(int32_t));
  if (iters && !it_pin) std::memcpy(iters, pit, B * sizeof(int32_t));
  return DOJO_OK;
}

extern "C" int dojo_step(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, const double* Fext, double* Zn,
                         double* sol, int32_t* status, int32_t* iters, uint32_t flags) {
  if (!h || B <= 0 || B > h->max_batch || !Z || !Zn) { if (h) h->err = "dojo_step: bad arguments (B must be in 1..max_batch)"; return DOJO_EINVAL; }
  return step_sync(h, opts, B, Z, U, Fext, Zn, sol, status, iters, nullptr, flags);
}

extern "C" int dojo_step_trace(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, const double* Fext, double* Zn,
                               double* sol, int32_t* status, int32_t* iters, double* trace, uint32_t flags) {
  if (!h || B <= 0 || B > h->max_batch || !Z || !Zn || !trace) {
    if (h) h->err = "dojo_step_trace: bad arguments (B must be in 1..max_batch, trace is required)";
    return DOJO_EINVAL;
  }
  return step_sync(h, opts, B, Z, U, Fext, Zn, sol, status, iters, trace, flags);
}

// simulate!: T steps with the state resident on the device (simulation/simulate.jl:16-36).  With dsol_raw, the recording rollout of
// dojo_rollout_grad (k_fwd_rec): per-step solutions, status [B x T] and iterations (diters, nullable) at pair t * B + e, each pair
// published on done_list (nullable), states into dtraj = slab 1 of the trajectory whose slab 0 is dZ0; dZf is not written.
static int launch_rollout(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU, double* dZf, double* dtraj,
                          int32_t* dstatus, cudaStream_t s, int32_t* diters = nullptr, double* dsol_raw = nullptr, int* done_count = nullptr,
                          int* done_list = nullptr) {
  StepArgs a = step_args(h, opts, B, false);
  a.Z = dZ0; a.U = dU; a.Zn = dZf; a.sol_raw = dsol_raw; a.status = dstatus; a.iters = diters;
  a.T = T; a.traj = dtraj; a.done_count = done_count; a.done_list = done_list;
  enter_call(h, s);
  CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  const bool rec = dsol_raw != nullptr;
  int grid = std::min((B + h->slots - 1) / h->slots, h->sm_count * (rec ? h->envs_per_sm_rec : h->envs_per_sm));
  { void* kargs[1] = {(void*)&a}; CUDA_TRY(h, cudaLaunchKernel(rec ? h->k_fwd_rec : h->k_fwd, dim3(grid), dim3(32 * h->nw * h->slots), kargs, h->smem_fwd, s)); }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

// simulate!: T steps fused in ONE launch (simulation/simulate.jl:16-36).  Every environment is advanced through all T
// steps by the CTA that dequeued it, so there is no per-step tail and no per-step launch.  U is [nu x B x T] (step-major).
// Device-pointer variant for resident data (no synchronisation): all pointers are device pointers.
extern "C" int dojo_rollout_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU, double* dZ_final,
                                  double* dZ_traj, int32_t* dstatus_any, void* cuda_stream) {
  if (!h || B <= 0 || T <= 0 || !dZ0 || !dZ_final) { if (h) h->err = "dojo_rollout_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return launch_rollout(h, opts, B, T, dZ0, dU, dZ_final, dZ_traj, dstatus_any, (cudaStream_t)cuda_stream);
}

extern "C" int dojo_rollout(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U, double* Z_final, double* Z_traj,
                            int32_t* status_any) {
  if (!h || B <= 0 || B > h->max_batch || T <= 0 || !Z0 || !Z_final) { if (h) h->err = "dojo_rollout: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t nz = (size_t)B * h->plan.nz;
  const double *dZ0 = Z0, *dU = U;
  double *dZf = Z_final, *dtraj = Z_traj;
  int32_t* dst = status_any;
  HostCall c(h, Z0);
  c.in(&dZ0, nz); c.in(&dU, (size_t)B * h->plan.nu * T); c.out(&dZf, nz); c.out(&dtraj, nz * T); c.out(&dst, B);
  int rc = c.bind();
  if (rc == DOJO_OK) rc = launch_rollout(h, opts, B, T, dZ0, dU, dZf, dtraj, dst, h->stream);
  return c.finish(rc);
}

// gradients: implemented in dojo_grad.cu
// step! + gradients = two launches on the stream: the forward kernel in its own (four slots per CTA) configuration, leaving
// the final solution of every environment in a device buffer, then the gradient kernel (prologue + assembly at that
// solution + IFT solves) in the larger-arena configuration.  Running the Newton loop inside the gradient configuration
// (two slots per CTA) made it twice as slow.  dZn must not alias dZ (the gradient kernel re-reads the input state).
static int step_grad_impl(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext, double* dZn,
                          double* dFz, double* dFu, double* dFc, int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream, DojoGather* g = nullptr);
static int launch_grad(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext, double* dsol_raw,
                       int32_t* dstatus, double* dFz, double* dFu, double* dFc, uint32_t flags, int* done_list, int* counter, cudaStream_t s);
extern "C" int dojo_step_grad_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext,
                                    double* dZn, double* dFz, double* dFu, int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream) {
  return step_grad_impl(h, opts, B, dZ, dU, dFext, dZn, dFz, dFu, nullptr, dstatus, diters, flags, cuda_stream);
}
// + contact-data gradients (get_contact_gradients, gradients/contact.jl:1-55): dFc [12Nb x 5Ni x B], solved as extra columns
extern "C" int dojo_step_grad_contact_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext,
                                            double* dZn, double* dFz, double* dFu, double* dFc, int32_t* dstatus, int32_t* diters, uint32_t flags,
                                            void* cuda_stream) {
  if (h && !dFc) { h->err = "dojo_step_grad_contact_async: Fc is required"; return DOJO_EINVAL; }
  if (h && h->orthant_contact) {  // the reference defines the contact-data blocks for NonlinearContact only (gradients/data.jl:152, :173)
    h->err = "dojo_step_grad_contact: contact-data gradients exist for NonlinearContact only (as in the reference)";
    return DOJO_EINVAL;
  }
  return step_grad_impl(h, opts, B, dZ, dU, dFext, dZn, dFz, dFu, dFc, dstatus, diters, flags, cuda_stream);
}
static int step_grad_impl(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext, double* dZn,
                          double* dFz, double* dFu, double* dFc, int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream, DojoGather* g) {
  if (!h || B <= 0 || B > h->max_batch || !dZ || !dZn || !dFz || !dFu || dZ == dZn) { if (h) h->err = "dojo_step_grad_async: bad arguments (B <= max_batch, dZn != dZ)"; return DOJO_EINVAL; }
  if (!h->grad_bytes) { h->err = "dojo_step_grad_async: the gradient workspace does not fit in shared memory for this mechanism"; return DOJO_ENOMEM; }
  cudaStream_t s = (cudaStream_t)cuda_stream;
  CUDA_TRY(h, cudaSetDevice(h->device));
  enter_call(h, s);
  if (!h->d_gsol) {
    CUDA_TRY(h, cudaMalloc((void**)&h->d_gsol, (size_t)h->max_batch * h->plan.nres * sizeof(double)));
    CUDA_TRY(h, cudaMalloc((void**)&h->d_gstatus, (size_t)h->max_batch * sizeof(int32_t)));
    CUDA_TRY(h, cudaMalloc((void**)&h->d_done, ((size_t)h->max_batch + 2) * sizeof(int)));
    if (getenv("DOJO_B200_NO_GRAD_OVERLAP")) h->overlap_grad = false;
  }
  int32_t* st = dstatus ? dstatus : h->d_gstatus;
  // The gradient kernel is launched programmatically dependent on the forward kernel (same stream): its CTAs start on the
  // SMs the forward kernel's tail leaves idle and consume environments in the order the forward kernel finishes them
  // (done_list), instead of waiting for the whole forward grid.
  const bool overlap = h->overlap_grad;
  int* done_count = overlap ? h->d_done : nullptr;
  int* done_list = overlap ? h->d_done + 2 : nullptr;
  if (overlap) {
    CUDA_TRY(h, cudaMemsetAsync(h->d_done, 0, 2 * sizeof(int), s));                 // [0] finished count, [1] gradient work queue
    CUDA_TRY(h, cudaMemsetAsync(h->d_done + 2, 0xff, (size_t)B * sizeof(int), s));  // -1 = not finished yet
  }
  int rc = launch_forward(h, opts, B, dZ, dU, dFext, dZn, nullptr, h->d_gsol, st, diters, flags, s, done_count, done_list, g);
  if (rc != DOJO_OK) return rc;
  rc = launch_grad(h, opts, B, dZ, dU, dFext, h->d_gsol, st, dFz, dFu, dFc, flags, done_list, overlap ? h->d_done + 1 : nullptr, s);
  if (rc != DOJO_OK) return rc;
  leave_call(h, s);
  return DOJO_OK;
}
// The gradient kernel over B (state, input, final solution) triples.  done_list non-null: launched programmatically dependent on the
// forward launch before it on the stream, consuming done_list in order with `counter` (zeroed by the caller) as its work queue; else
// the handle's work-queue counter, after the forward launch.
static int launch_grad(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext, double* dsol_raw,
                       int32_t* dstatus, double* dFz, double* dFu, double* dFc, uint32_t flags, int* done_list, int* counter, cudaStream_t s) {
  const bool overlap = done_list != nullptr;
  StepArgs a = step_args(h, opts, B, true);
  a.Z = dZ; a.U = dU; a.Fext = dFext; a.sol_raw = dsol_raw; a.status = dstatus; a.flags = flags;
  a.Fz = dFz; a.Fu = dFu; a.Fc = dFc; a.done_list = done_list;
  if (overlap) a.counter = counter;
  else CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  int grid = std::min((B + h->slots_grad - 1) / h->slots_grad, h->sm_count * h->envs_per_sm_grad);
  if (overlap) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(32 * h->nw * h->slots_grad); cfg.dynamicSmemBytes = h->smem_grad; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    void* kargs[1] = {(void*)&a};
    CUDA_TRY(h, cudaLaunchKernelExC(&cfg, h->k_grad, kargs));
  } else {
    void* kargs[1] = {(void*)&a};
    CUDA_TRY(h, cudaLaunchKernel(h->k_grad, dim3(grid), dim3(32 * h->nw * h->slots_grad), kargs, h->smem_grad, s));
  }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  return DOJO_OK;
}

// ------------------------------------------------------------------------------------------------------------
// Multi-GPU exchange of the next states, fused into the step (include/dojo_b200.h; SURVEY.md 8e)
// ------------------------------------------------------------------------------------------------------------
extern "C" int dojo_gather_create(DojoHandle* h, int world, int rank, int B_local, DojoGather** out) {
  if (!h || !out || world < 1 || world > DOJO_MAX_GATHER_RANKS || rank < 0 || rank >= world || B_local <= 0 || B_local > h->max_batch) {
    if (h) h->err = "dojo_gather_create: bad arguments (1 <= world <= 8, B_local <= max_batch)";
    return DOJO_EINVAL;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  DojoGather* g = new DojoGather();
  g->h = h; g->world = world; g->rank = rank; g->B = B_local;
  // Two halves, used alternately: a rank that has closed step t may start step t + 1 -- and write its slice into the other ranks'
  // buffers -- while a slower rank is still READING the gathered states of step t; step t + 1 therefore goes to the other half, and
  // the half of step t is only written again by step t + 2, which no rank starts before every rank has finished step t + 1 (issued
  // behind its readers of step t in stream order).
  g->half = (size_t)world * B_local * h->plan.nz;
  const size_t bytes = 2 * g->half * sizeof(double);
  if (cudaMalloc((void**)&g->buf, bytes) != cudaSuccess || cudaMalloc((void**)&g->flag, sizeof(unsigned long long)) != cudaSuccess ||
      cudaMemset(g->buf, 0, bytes) != cudaSuccess || cudaMemset(g->flag, 0, sizeof(unsigned long long)) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
    h->err = std::string("dojo_gather_create: ") + cudaGetErrorString(cudaGetLastError());
    cudaFree(g->buf); cudaFree(g->flag); delete g;
    return DOJO_ECUDA;
  }
  if (world == 1) { g->peer_buf[0] = g->buf; g->peer_flag[0] = g->flag; g->connected = true; }
  *out = g;
  return DOJO_OK;
}
extern "C" int dojo_gather_export(DojoGather* g, void* handle_out) {
  if (!g || !handle_out) return DOJO_EINVAL;
  static_assert(2 * sizeof(cudaIpcMemHandle_t) <= DOJO_GATHER_HANDLE_BYTES, "descriptor size");
  cudaIpcMemHandle_t hb, hf;
  CUDA_TRY(g->h, cudaSetDevice(g->h->device));
  CUDA_TRY(g->h, cudaIpcGetMemHandle(&hb, g->buf));
  CUDA_TRY(g->h, cudaIpcGetMemHandle(&hf, g->flag));
  std::memset(handle_out, 0, DOJO_GATHER_HANDLE_BYTES);
  std::memcpy(handle_out, &hb, sizeof(hb));
  std::memcpy((char*)handle_out + sizeof(hb), &hf, sizeof(hf));
  return DOJO_OK;
}
extern "C" int dojo_gather_connect(DojoGather* g, const void* all_handles) {
  if (!g || !all_handles) return DOJO_EINVAL;
  CUDA_TRY(g->h, cudaSetDevice(g->h->device));
  for (int r = 0; r < g->world; ++r) {
    if (r == g->rank) { g->peer_buf[r] = g->buf; g->peer_flag[r] = g->flag; continue; }
    cudaIpcMemHandle_t hb, hf;
    const char* src = (const char*)all_handles + (size_t)r * DOJO_GATHER_HANDLE_BYTES;
    std::memcpy(&hb, src, sizeof(hb));
    std::memcpy(&hf, src + sizeof(hb), sizeof(hf));
    CUDA_TRY(g->h, cudaIpcOpenMemHandle((void**)&g->peer_buf[r], hb, cudaIpcMemLazyEnablePeerAccess));
    CUDA_TRY(g->h, cudaIpcOpenMemHandle((void**)&g->peer_flag[r], hf, cudaIpcMemLazyEnablePeerAccess));
    g->opened[r] = true;
  }
  g->connected = true;
  return DOJO_OK;
}
extern "C" double* dojo_gather_buffer(DojoGather* g) { return g ? g->buf + (size_t)g->last * g->half : nullptr; }
extern "C" int dojo_gather_destroy(DojoGather* g) {
  if (!g) return DOJO_OK;
  cudaSetDevice(g->h->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < g->world; ++r)
    if (g->opened[r]) { cudaIpcCloseMemHandle(g->peer_buf[r]); cudaIpcCloseMemHandle(g->peer_flag[r]); }
  cudaFree(g->buf); cudaFree(g->flag);
  delete g;
  return DOJO_OK;
}
static int gather_close_step(DojoHandle* h, DojoGather* g, int32_t* dstatus, cudaStream_t s) {
  dojo_gather_wait_kernel<<<1, 32, 0, s>>>(g->flag, g->expected, dstatus);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}
extern "C" int dojo_step_gather_async(DojoHandle* h, DojoGather* g, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, const double* dFext,
                                      double* dZn, int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream) {
  if (!h || !g || B <= 0 || !dZ || !dZn) { if (h) h->err = "dojo_step_gather_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = launch_forward(h, opts, B, dZ, dU, dFext, dZn, nullptr, nullptr, dstatus, diters, flags, (cudaStream_t)cuda_stream, nullptr, nullptr, g);
  if (rc != DOJO_OK) return rc;
  return gather_close_step(h, g, dstatus, (cudaStream_t)cuda_stream);
}
extern "C" int dojo_step_grad_gather_async(DojoHandle* h, DojoGather* g, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU,
                                           const double* dFext, double* dZn, double* dFz, double* dFu, int32_t* dstatus, int32_t* diters, uint32_t flags,
                                           void* cuda_stream) {
  if (!h || !g) { if (h) h->err = "dojo_step_grad_gather_async: bad arguments"; return DOJO_EINVAL; }
  int rc = step_grad_impl(h, opts, B, dZ, dU, dFext, dZn, dFz, dFu, nullptr, dstatus, diters, flags, cuda_stream, g);
  if (rc != DOJO_OK) return rc;
  return gather_close_step(h, g, dstatus, (cudaStream_t)cuda_stream);
}

// Two chunk buffers of maximal Jacobians (at most 128 MB each, grad_chunk environments or pairs): the kernels of chunk i + 1 run while
// the gradients of chunk i travel to the host.
static int ensure_grad_chunks(DojoHandle* h) {
  if (h->d_Fz[0]) return DOJO_OK;
  const size_t ng = 12 * (size_t)h->plan.Nb, fz = ng * ng, fu = ng * h->plan.nu;
  h->grad_chunk = (int)std::max<size_t>(1, std::min<size_t>(h->max_batch, (size_t(128) << 20) / ((fz + fu) * sizeof(double))));
  for (int k = 0; k < 2; ++k) {
    CUDA_TRY(h, cudaMalloc((void**)&h->d_Fz[k], (size_t)h->grad_chunk * fz * sizeof(double)));
    CUDA_TRY(h, cudaMalloc((void**)&h->d_Fu[k], std::max<size_t>(1, (size_t)h->grad_chunk * fu) * sizeof(double)));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_kernel[k], cudaEventDisableTiming));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_copy[k], cudaEventDisableTiming));
  }
  CUDA_TRY(h, cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
  return DOJO_OK;
}

// Jacobians of `count` environments or pairs to the host through the two chunk buffers: launch(i0, n, k) computes items [i0, i0 + n)
// into d_Fz[k] / d_Fu[k] on h->stream, and their copies to Fz / Fu (fz / fu doubles per item) run on copy_stream while the next chunk
// is computed.  The caller synchronises copy_stream.
template <class Launch>
static int copy_out_chunks(DojoHandle* h, size_t count, double* Fz, size_t fz, double* Fu, size_t fu, Launch launch) {
  cudaStream_t s = h->stream, cs = h->copy_stream;
  int k = 0;
  for (size_t i0 = 0; i0 < count; i0 += h->grad_chunk, k ^= 1) {
    const int n = (int)std::min<size_t>(h->grad_chunk, count - i0);
    if (i0 >= 2 * (size_t)h->grad_chunk) CUDA_TRY(h, cudaStreamWaitEvent(s, h->ev_copy[k], 0));  // buffer k has been drained
    int rc = launch(i0, n, k);
    if (rc != DOJO_OK) return rc;
    CUDA_TRY(h, cudaEventRecord(h->ev_kernel[k], s));
    CUDA_TRY(h, cudaStreamWaitEvent(cs, h->ev_kernel[k], 0));
    CUDA_TRY(h, cudaMemcpyAsync(Fz + i0 * fz, h->d_Fz[k], (size_t)n * fz * sizeof(double), cudaMemcpyDeviceToHost, cs));
    if (fu) CUDA_TRY(h, cudaMemcpyAsync(Fu + i0 * fu, h->d_Fu[k], (size_t)n * fu * sizeof(double), cudaMemcpyDeviceToHost, cs));
    CUDA_TRY(h, cudaEventRecord(h->ev_copy[k], cs));
  }
  return DOJO_OK;
}

// Host- or device-pointer entry.  Host buffers are processed in chunks (the Jacobians are large: (12Nb)^2 doubles per env).
extern "C" int dojo_step_grad(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, const double* Fext, double* Zn,
                              double* Fz, double* Fu, int32_t* status, int32_t* iters, uint32_t flags) {
  if (!h || B <= 0 || B > h->max_batch || !Z || !Zn || !Fz || !Fu) { if (h) h->err = "dojo_step_grad: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  HostCall c(h, Z);
  if (c.dev) return c.finish(dojo_step_grad_async(h, opts, B, Z, U, Fext, Zn, Fz, Fu, status, iters, flags, h->stream));
  int rc = ensure_grad_chunks(h);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t ng = 12 * (size_t)P.Nb, fz = ng * ng, fu = ng * P.nu;
  // whole-batch inputs first (small), per-chunk kernels, gradient copies on the second stream
  const double *dZ = Z, *dU = U, *dF = Fext;
  double* dZn = Zn;
  int32_t *dst = status, *dit = iters;
  c.in(&dZ, (size_t)B * P.nz); c.in(&dU, (size_t)B * P.nu); c.in(&dF, (size_t)B * 6 * P.Nb);
  c.out(&dZn, (size_t)B * P.nz); c.out(&dst, B); c.out(&dit, B);
  rc = c.bind();
  if (rc == DOJO_OK) rc = copy_out_chunks(h, B, Fz, fz, Fu, fu, [&](size_t e0, int nb, int k) {
    return dojo_step_grad_async(h, opts, nb, dZ + e0 * P.nz, dU ? dU + e0 * P.nu : nullptr, dF ? dF + e0 * 6 * P.Nb : nullptr, dZn + e0 * P.nz,
                                h->d_Fz[k], h->d_Fu[k], dst ? dst + e0 : nullptr, dit ? dit + e0 : nullptr, flags, h->stream);
  });
  rc = c.finish(rc);
  if (rc == DOJO_OK) CUDA_TRY(h, cudaStreamSynchronize(h->copy_stream));
  return rc;
}

// ------------------------------------------------------------------------------------------------------------
// minimal <-> maximal coordinate maps and step_minimal_coordinates! (SURVEY.md 8 f1)
// ------------------------------------------------------------------------------------------------------------
extern "C" int dojo_num_minimal(const DojoHandle* h) { return 2 * h->plan.nu; }

static int launch_kin(DojoHandle* h, bool to_maximal, int B, const double* din, double* dout, cudaStream_t s) {
  KinArgs a;
  a.joints = h->plan.joints; a.order = h->d_kin_order;
  a.Ne = h->plan.Ne; a.Nb = h->plan.Nb; a.nu = h->plan.nu; a.B = B; a.h = h->plan.h;
  a.in = din; a.out = dout;
  const int threads = 128, grid = (B + threads - 1) / threads;
  if (to_maximal) dojo_min_to_max_kernel<<<grid, threads, 0, s>>>(a);
  else dojo_max_to_min_kernel<<<grid, threads, 0, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  return DOJO_OK;
}

extern "C" int dojo_minimal_to_maximal_async(DojoHandle* h, int B, const double* dX, double* dZ, void* cuda_stream) {
  if (!h || B <= 0 || !dX || !dZ) { if (h) h->err = "dojo_minimal_to_maximal_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return launch_kin(h, true, B, dX, dZ, (cudaStream_t)cuda_stream);
}
extern "C" int dojo_maximal_to_minimal_async(DojoHandle* h, int B, const double* dZ, double* dX, void* cuda_stream) {
  if (!h || B <= 0 || !dX || !dZ) { if (h) h->err = "dojo_maximal_to_minimal_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return launch_kin(h, false, B, dZ, dX, (cudaStream_t)cuda_stream);
}

// host or device pointers (both arguments of the same kind)
static int kin_sync(DojoHandle* h, bool to_maximal, int B, const double* in, double* out, const char* who) {
  if (!h || B <= 0 || B > h->max_batch || !in || !out) { if (h) h->err = std::string(who) + ": bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t nx = (size_t)B * 2 * h->plan.nu, nz = (size_t)B * h->plan.nz;
  const double* din = in;
  double* dout = out;
  HostCall c(h, in);
  c.in(&din, to_maximal ? nx : nz); c.out(&dout, to_maximal ? nz : nx);
  int rc = c.bind();
  if (rc == DOJO_OK) rc = launch_kin(h, to_maximal, B, din, dout, h->stream);
  return c.finish(rc);
}
extern "C" int dojo_minimal_to_maximal(DojoHandle* h, int B, const double* X, double* Z) { return kin_sync(h, true, B, X, Z, "dojo_minimal_to_maximal"); }
extern "C" int dojo_maximal_to_minimal(DojoHandle* h, int B, const double* Z, double* X) { return kin_sync(h, false, B, Z, X, "dojo_maximal_to_minimal"); }

// step_minimal_coordinates! (simulation/step.jl:42-61): minimal -> maximal, step!, maximal -> minimal; three launches on one
// stream, the maximal states never leave the device.  X, U, X_next: host or device pointers (all of the same kind).
extern "C" int dojo_step_minimal_flags(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U, double* X_next, int32_t* status,
                                       int32_t* iters, uint32_t flags);
extern "C" int dojo_step_minimal(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U, double* X_next, int32_t* status,
                                 int32_t* iters) {
  return dojo_step_minimal_flags(h, opts, B, X, U, X_next, status, iters, 0);
}
extern "C" int dojo_step_minimal_flags(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U, double* X_next, int32_t* status,
                                       int32_t* iters, uint32_t flags) {
  if (!h || B <= 0 || B > h->max_batch || !X || !X_next) { if (h) h->err = "dojo_step_minimal: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  cudaStream_t s = h->stream;
  const size_t nx = (size_t)B * 2 * P.nu;
  const double *dX = X, *dU = U;
  double* dXn = X_next;
  int32_t *dst = status, *dit = iters;
  HostCall c(h, X);
  c.in(&dX, nx); c.in(&dU, (size_t)B * P.nu); c.out(&dXn, nx); c.out(&dst, B); c.out(&dit, B);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_kin(h, true, B, dX, h->d_Z, s);
  if (rc == DOJO_OK) rc = launch_forward(h, opts, B, h->d_Z, dU, nullptr, h->d_Zn, nullptr, nullptr, dst, dit, flags & DOJO_FLAG_Q1_LITERAL_RETURN, s);
  if (rc == DOJO_OK) rc = launch_kin(h, false, B, h->d_Zn, dXn, s);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Jacobians of the coordinate maps and get_minimal_gradients! (SURVEY.md 8 f1; dojo_kinjac.cuh)
// ------------------------------------------------------------------------------------------------------------
static int ensure_kinjac(DojoHandle* h) {
  if (h->d_kjws) return DOJO_OK;
  h->kj_grid = std::max(1, std::min(h->max_batch, h->sm_count * 4));  // 254 registers x 128 threads: two CTAs resident per SM
  CUDA_TRY(h, cudaMalloc((void**)&h->d_kjws, (size_t)h->kj_grid * kinjac_ws_doubles(h->plan.Nb, h->plan.nu) * sizeof(double)));
  return DOJO_OK;
}

// mode 0: M(Z) -> out   1: N(Z) -> out   2: (Z, Zn, Fz, Fu) -> (Gx, Gu)
static int launch_kinjac(DojoHandle* h, int mode, int B, const double* dZ, const double* dZn, const double* dFz, const double* dFu, double* out0,
                         double* out1, cudaStream_t s) {
  int rc = ensure_kinjac(h);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  KinJacArgs a;
  a.joints = P.joints; a.order = h->d_kin_order;
  a.Ne = P.Ne; a.Nb = P.Nb; a.nu = P.nu; a.B = B; a.h = P.h;
  a.Z = dZ; a.Zm = dZn ? dZn : dZ; a.Fz = dFz; a.Fu = dFu;
  a.outM = mode == 0 ? out0 : nullptr; a.outN = mode == 1 ? out0 : nullptr;
  a.Gx = mode == 2 ? out0 : nullptr; a.Gu = mode == 2 ? out1 : nullptr;
  a.ws = h->d_kjws; a.mode = mode;
  enter_call(h, s);
  if (mode == 0) CUDA_TRY(h, cudaMemsetAsync(out0, 0, (size_t)B * 2 * P.nu * 12 * P.Nb * sizeof(double), s));
  dojo_kinjac_kernel<<<std::min(B, h->kj_grid), 128, 0, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_maximal_to_minimal_jacobian_async(DojoHandle* h, int B, const double* dZ, double* dJ, void* cuda_stream) {
  if (!h || B <= 0 || B > h->max_batch || !dZ || !dJ) { if (h) h->err = "dojo_maximal_to_minimal_jacobian_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return launch_kinjac(h, 0, B, dZ, nullptr, nullptr, nullptr, dJ, nullptr, (cudaStream_t)cuda_stream);
}
extern "C" int dojo_minimal_to_maximal_jacobian_async(DojoHandle* h, int B, const double* dZ, double* dJ, void* cuda_stream) {
  if (!h || B <= 0 || B > h->max_batch || !dZ || !dJ) { if (h) h->err = "dojo_minimal_to_maximal_jacobian_async: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return launch_kinjac(h, 1, B, dZ, nullptr, nullptr, nullptr, dJ, nullptr, (cudaStream_t)cuda_stream);
}

static int kinjac_sync(DojoHandle* h, int mode, int B, const double* Z, double* J, const char* who) {
  if (!h || B <= 0 || B > h->max_batch || !Z || !J) { if (h) h->err = std::string(who) + ": bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const Plan& P = h->plan;
  cudaStream_t s = h->stream;
  HostCall c(h, Z);
  if (c.dev) return c.finish(launch_kinjac(h, mode, B, Z, nullptr, nullptr, nullptr, J, nullptr, s));
  const size_t per_env = (size_t)2 * P.nu * 12 * P.Nb;
  const int chunk = (int)std::max<size_t>(1, std::min<size_t>(B, (size_t(256) << 20) / std::max<size_t>(1, per_env * sizeof(double))));
  const double* dZ = Z;
  double* dJ = nullptr;
  c.in(&dZ, (size_t)B * P.nz); c.scratch(&dJ, (size_t)chunk * per_env);
  int rc = c.bind();
  for (int e0 = 0; e0 < B && rc == DOJO_OK; e0 += chunk) {
    const int nb = std::min(chunk, B - e0);
    rc = launch_kinjac(h, mode, nb, dZ + (size_t)e0 * P.nz, nullptr, nullptr, nullptr, dJ, nullptr, s);
    if (rc == DOJO_OK) CUDA_TRY(h, cudaMemcpyAsync(J + (size_t)e0 * per_env, dJ, (size_t)nb * per_env * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  return c.finish(rc);
}
extern "C" int dojo_maximal_to_minimal_jacobian(DojoHandle* h, int B, const double* Z, double* J) { return kinjac_sync(h, 0, B, Z, J, "dojo_maximal_to_minimal_jacobian"); }
extern "C" int dojo_minimal_to_maximal_jacobian(DojoHandle* h, int B, const double* Z, double* J) { return kinjac_sync(h, 1, B, Z, J, "dojo_minimal_to_maximal_jacobian"); }

// ------------------------------------------------------------------------------------------------------------
// Adjoints of the coordinate maps: gZ = M(z)' gX and gX = N(z)' gZ without forming M or N (dojo_kinjac.cuh)
// ------------------------------------------------------------------------------------------------------------
static int map_vjp_check(DojoHandle* h, int n, bool buffers, const char* who) {
  if (!h) return DOJO_EINVAL;
  if (n <= 0 || !buffers || h->plan.nu == 0) { h->err = std::string(who) + ": bad arguments (n >= 1, every buffer, a mechanism with inputs)"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return DOJO_OK;
}

// to_minimal: gZ = M' gX (in = gX, out = gZ);  else gX = N' gZ (in = gZ, out = gX)
static int launch_map_vjp(DojoHandle* h, bool to_minimal, int n, const double* dZ, const double* din, double* dout, cudaStream_t s) {
  const Plan& P = h->plan;
  MapVjpArgs a;
  a.joints = P.joints; a.order = h->d_kin_order;
  a.Ne = P.Ne; a.Nb = P.Nb; a.nu = P.nu; a.n = n; a.h = P.h;
  a.Z = dZ; a.in = din; a.out = dout; a.ws = nullptr;
  if (to_minimal) {
    int G = 1;  // lanes per state: the joints and the bodies each take one lane, up to a warp
    while (G < 32 && (G < P.Ne || G < P.Nb)) G *= 2;
    int per_cta = 128 / G;
    const size_t per_state = (size_t)24 * P.Ne * sizeof(double);
    while (per_cta > 1 && per_cta * per_state > 48 * 1024) per_cta /= 2;
    const size_t smem = per_cta * per_state;
    if (smem > 48 * 1024) CUDA_TRY(h, cudaFuncSetAttribute(dojo_max_to_min_vjp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    enter_call(h, s);
    dojo_max_to_min_vjp_kernel<<<(n + per_cta - 1) / per_cta, per_cta * G, smem, s>>>(a, G);
  } else {
    int rc = ensure_kinjac(h);  // its per-CTA slices hold kinjac_ws_doubles >= min_to_max_vjp_ws_doubles doubles (nu >= 1)
    if (rc != DOJO_OK) return rc;
    a.ws = h->d_kjws;
    enter_call(h, s);
    dojo_min_to_max_vjp_kernel<<<std::min(n, h->kj_grid), 32, 0, s>>>(a);
  }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_maximal_to_minimal_vjp_async(DojoHandle* h, int n, const double* dZ, const double* dgX, double* dgZ, void* cuda_stream) {
  const int rc = map_vjp_check(h, n, dZ && dgX && dgZ, "dojo_maximal_to_minimal_vjp_async");
  return rc != DOJO_OK ? rc : launch_map_vjp(h, true, n, dZ, dgX, dgZ, (cudaStream_t)cuda_stream);
}
extern "C" int dojo_minimal_to_maximal_vjp_async(DojoHandle* h, int n, const double* dZ, const double* dgZ, double* dgX, void* cuda_stream) {
  const int rc = map_vjp_check(h, n, dZ && dgZ && dgX, "dojo_minimal_to_maximal_vjp_async");
  return rc != DOJO_OK ? rc : launch_map_vjp(h, false, n, dZ, dgZ, dgX, (cudaStream_t)cuda_stream);
}

// host or device pointers (all of the same kind); n is not bounded by max_batch: host arrays are staged whole through the arena
static int map_vjp_sync(DojoHandle* h, bool to_minimal, int n, const double* Z, const double* in, double* out, const char* who) {
  int rc = map_vjp_check(h, n, Z && in && out, who);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t nx = (size_t)n * 2 * P.nu, ng = (size_t)n * 12 * P.Nb;
  const double *dZ = Z, *din = in;
  double* dout = out;
  HostCall c(h, Z);
  c.in(&dZ, (size_t)n * P.nz); c.in(&din, to_minimal ? nx : ng); c.out(&dout, to_minimal ? ng : nx);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_map_vjp(h, to_minimal, n, dZ, din, dout, h->stream);
  return c.finish(rc);
}
extern "C" int dojo_maximal_to_minimal_vjp(DojoHandle* h, int n, const double* Z, const double* gX, double* gZ) {
  return map_vjp_sync(h, true, n, Z, gX, gZ, "dojo_maximal_to_minimal_vjp");
}
extern "C" int dojo_minimal_to_maximal_vjp(DojoHandle* h, int n, const double* Z, const double* gZ, double* gX) {
  return map_vjp_sync(h, false, n, Z, gZ, gX, "dojo_minimal_to_maximal_vjp");
}

// get_minimal_gradients! (gradients/state.jl:182-217).  Per chunk of environments, on one stream: minimal -> maximal,
// forward + gradient kernels (dojo_step_grad_async), the map-Jacobian kernel in mode 2, maximal -> minimal of the next state.
extern "C" int dojo_minimal_gradients(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U, double* X_next, double* Gx,
                                      double* Gu, int32_t* status, int32_t* iters) {
  if (!h || B <= 0 || B > h->max_batch || !X || !X_next || !Gx || !Gu) { if (h) h->err = "dojo_minimal_gradients: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);
  if (rc == DOJO_OK) rc = ensure_grad_chunks(h);  // same chunk buffers as the host-pointer path of dojo_step_grad
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  cudaStream_t s = h->stream;
  const size_t nm = 2 * (size_t)P.nu, gx = nm * nm, gu = nm * P.nu;
  const double *dX = X, *dU = (U && P.nu > 0) ? U : nullptr;
  double *dXn = X_next, *dGx = Gx, *dGu = Gu;
  int32_t *dst = status, *dit = iters;
  HostCall c(h, X);
  c.in(&dX, B * nm); c.in(&dU, (size_t)B * P.nu);
  c.out(&dXn, B * nm); c.out(&dGx, B * gx); c.out(&dGu, B * gu); c.out(&dst, B); c.out(&dit, B);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_kin(h, true, B, dX, h->d_Z, s);
  for (int e0 = 0; e0 < B && rc == DOJO_OK; e0 += h->grad_chunk) {
    const int nb = std::min(h->grad_chunk, B - e0);
    rc = dojo_step_grad_async(h, opts, nb, h->d_Z + (size_t)e0 * P.nz, dU ? dU + (size_t)e0 * P.nu : nullptr, nullptr, h->d_Zn + (size_t)e0 * P.nz,
                              h->d_Fz[0], h->d_Fu[0], dst ? dst + e0 : nullptr, dit ? dit + e0 : nullptr, 0, s);
    if (rc == DOJO_OK)
      rc = launch_kinjac(h, 2, nb, h->d_Z + (size_t)e0 * P.nz, h->d_Zn + (size_t)e0 * P.nz, h->d_Fz[0], h->d_Fu[0], dGx + (size_t)e0 * gx,
                         dGu + (size_t)e0 * gu, s);
  }
  if (rc == DOJO_OK) rc = launch_kin(h, false, B, h->d_Zn, dXn, s);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Trajectory Jacobians: simulate! + get_maximal_gradients! / get_minimal_gradients! at every step (include/dojo_b200.h)
// ------------------------------------------------------------------------------------------------------------
// One recording rollout (REC kernel) advances B environments T steps and keeps, per pair p = t * B + e, the final solution, status
// and iterations; the trajectory [nz x B x (T + 1)] holds Z0 in slab 0, so that [feature x B x T] is [feature x pairs] and the unchanged
// gradient kernel runs over the pairs with a.Z = slab 0.
static int ensure_rec_kernel(DojoHandle* h) {
  if (h->k_fwd_rec) return DOJO_OK;
  const void* k = step_rec_kernel_fn(h->any_contact, h->plan_smem_mask == 0xff);
  int occ = 1;
  CUDA_TRY(h, max_shared_memory(k, h->device));
  CUDA_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, 32 * h->nw * h->slots, h->smem_fwd));
  h->envs_per_sm_rec = std::max(1, occ);
  h->k_fwd_rec = k;
  return DOJO_OK;
}

static int ensure_rollout_grad_scratch(DojoHandle* h, size_t pairs) {
  if (h->rpairs >= pairs) return DOJO_OK;
  CUDA_TRY(h, cudaDeviceSynchronize());
  cudaFree(h->d_rsol); cudaFree(h->d_rdone); cudaFree(h->d_rstatus); cudaFree(h->d_riters);
  h->d_rsol = nullptr; h->d_rdone = nullptr; h->d_rstatus = nullptr; h->d_riters = nullptr; h->rpairs = 0;
  CUDA_TRY(h, cudaMalloc((void**)&h->d_rsol, pairs * h->plan.nres * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_rdone, (pairs + 2) * sizeof(int)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_rstatus, pairs * sizeof(int32_t)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_riters, pairs * sizeof(int32_t)));
  h->rpairs = pairs;
  return DOJO_OK;
}

// argument checks shared by the trajectory-gradient, tape and adjoint entries: no launch before every check has passed; `required`
// names the buffers the entry needs
static int trajectory_setup(DojoHandle* h, int B, int T, bool buffers, const char* who, const char* required) {
  if (!h) return DOJO_EINVAL;
  if (B <= 0 || B > h->max_batch || T <= 0 || !buffers || (long long)B * (T + 1) > (long long)INT_MAX - 2) {
    h->err = std::string(who) + ": bad arguments (B in 1..max_batch, T >= 1, B * (T + 1) < 2^31 - 2, " + required + ")";
    return DOJO_EINVAL;
  }
  if (!h->grad_bytes) { h->err = std::string(who) + ": the gradient workspace does not fit in shared memory for this mechanism"; return DOJO_ENOMEM; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return DOJO_OK;
}
static const char* kRollGradBuffers = "state / trajectory / Jacobian buffers required";

extern "C" int dojo_rollout_grad_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU, double* dZ_traj,
                                       double* dFz, double* dFu, int32_t* dstatus, int32_t* diters, void* cuda_stream) {
  int rc = trajectory_setup(h, B, T, dZ0 && dZ_traj && dFz && dFu, "dojo_rollout_grad_async", kRollGradBuffers);
  if (rc == DOJO_OK) rc = ensure_rec_kernel(h);
  if (rc == DOJO_OK) rc = ensure_rollout_grad_scratch(h, (size_t)B * T);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  cudaStream_t s = (cudaStream_t)cuda_stream;
  const int pairs = B * T;
  int32_t* st = dstatus ? dstatus : h->d_rstatus;
  enter_call(h, s);
  if (dZ0 != dZ_traj) CUDA_TRY(h, cudaMemcpyAsync(dZ_traj, dZ0, (size_t)B * P.nz * sizeof(double), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(h, cudaMemsetAsync(h->d_rdone, 0, 2 * sizeof(int), s));                     // [0] finished pairs, [1] gradient work queue
  CUDA_TRY(h, cudaMemsetAsync(h->d_rdone + 2, 0xff, (size_t)pairs * sizeof(int), s));  // -1 = not finished yet
  // the gradients of early steps run on the SMs the rollout's tail leaves idle while later steps are still being solved
  rc = launch_rollout(h, opts, B, T, dZ_traj, dU, nullptr, dZ_traj + (size_t)B * P.nz, st, s, diters, h->d_rsol, h->d_rdone, h->d_rdone + 2);
  if (rc == DOJO_OK) rc = launch_grad(h, opts, pairs, dZ_traj, dU, nullptr, h->d_rsol, st, dFz, dFu, nullptr, 0, h->d_rdone + 2, h->d_rdone + 1, s);
  if (rc != DOJO_OK) return rc;
  leave_call(h, s);
  return DOJO_OK;
}

// Host- or device-pointer entry.  With host buffers the Jacobians (ant: ~212 KB per pair) go to the host in chunks of pairs through the
// two chunk buffers of dojo_step_grad, after one rollout; the gradient kernel of chunk i + 1 runs while chunk i is being copied.
extern "C" int dojo_rollout_grad(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U, double* Z_traj,
                                 double* Fz, double* Fu, int32_t* status, int32_t* iters) {
  int rc = trajectory_setup(h, B, T, Z0 && Z_traj && Fz && Fu, "dojo_rollout_grad", kRollGradBuffers);
  if (rc == DOJO_OK) rc = ensure_rec_kernel(h);
  if (rc == DOJO_OK) rc = ensure_rollout_grad_scratch(h, (size_t)B * T);
  if (rc != DOJO_OK) return rc;
  HostCall c(h, Z0);
  if (c.dev) return c.finish(dojo_rollout_grad_async(h, opts, B, T, Z0, U, Z_traj, Fz, Fu, status, iters, h->stream));
  rc = ensure_grad_chunks(h);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t pairs = (size_t)B * T, ng = 12 * (size_t)P.Nb, fz = ng * ng, fu = ng * P.nu;
  cudaStream_t s = h->stream;
  const double* dU = U;
  double* dtraj = Z_traj;
  int32_t *dst = status, *dit = iters;
  c.in(&dU, pairs * P.nu); c.out(&dtraj, (pairs + B) * P.nz); c.out(&dst, pairs); c.out(&dit, pairs);
  rc = c.bind();
  if (rc != DOJO_OK) return rc;
  int32_t* st = dst ? dst : h->d_rstatus;  // the REC kernel always writes a status
  CUDA_TRY(h, cudaMemcpyAsync(dtraj, Z0, (size_t)B * P.nz * sizeof(double), cudaMemcpyHostToDevice, s));
  rc = launch_rollout(h, opts, B, T, dtraj, dU, nullptr, dtraj + (size_t)B * P.nz, st, s, dit, h->d_rsol);
  if (rc == DOJO_OK) rc = copy_out_chunks(h, pairs, Fz, fz, Fu, fu, [&](size_t p0, int n, int k) {
    enter_call(h, s);
    int rc = launch_grad(h, opts, n, dtraj + p0 * P.nz, dU ? dU + p0 * P.nu : nullptr, nullptr, h->d_rsol + p0 * P.nres, st + p0, h->d_Fz[k],
                         h->d_Fu[k], nullptr, 0, nullptr, nullptr, s);
    if (rc == DOJO_OK) leave_call(h, s);
    return rc;
  });
  rc = c.finish(rc);
  if (rc == DOJO_OK) CUDA_TRY(h, cudaStreamSynchronize(h->copy_stream));
  return rc;
}

// The same in minimal coordinates (get_minimal_gradients! at every step): minimal_to_maximal of X0, the recording rollout, then per
// chunk of pairs the gradient kernel and the map-Jacobian kernel in mode 2 between slabs t and t + 1 (the maximal Jacobians never leave
// the device), and finally maximal_to_minimal of all T + 1 slabs.  Host or device pointers (all of the same kind).
extern "C" int dojo_rollout_minimal_gradients(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* X0, const double* U,
                                              double* X_traj, double* Gx, double* Gu, int32_t* status, int32_t* iters) {
  int rc = trajectory_setup(h, B, T, X0 && X_traj && Gx && Gu, "dojo_rollout_minimal_gradients", kRollGradBuffers);
  if (rc == DOJO_OK) rc = ensure_rec_kernel(h);
  if (rc == DOJO_OK) rc = ensure_rollout_grad_scratch(h, (size_t)B * T);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t pairs = (size_t)B * T, nm = 2 * (size_t)P.nu, gx = nm * nm, gu = nm * P.nu;
  rc = ensure_grad_chunks(h);
  if (rc == DOJO_OK) rc = grow_buffer(h, (void**)&h->d_rZ, &h->rZ_bytes, (pairs + B) * P.nz * sizeof(double));
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = h->stream;
  const double *dX0 = X0, *dU = (U && P.nu > 0) ? U : nullptr;
  double *dXt = X_traj, *cGx = nullptr, *cGu = nullptr;  // cGx, cGu: one chunk of the minimal Jacobians (host pointers)
  int32_t *dst = status, *dit = iters;
  HostCall c(h, X0);
  c.in(&dX0, B * nm); c.in(&dU, pairs * P.nu); c.out(&dXt, (pairs + B) * nm); c.out(&dst, pairs); c.out(&dit, pairs);
  c.scratch(&cGx, h->grad_chunk * gx); c.scratch(&cGu, h->grad_chunk * gu);
  rc = c.bind();
  if (rc != DOJO_OK) return rc;
  int32_t* st = dst ? dst : h->d_rstatus;  // the REC kernel always writes a status
  enter_call(h, s);
  rc = launch_kin(h, true, B, dX0, h->d_rZ, s);
  if (rc == DOJO_OK) rc = launch_rollout(h, opts, B, T, h->d_rZ, dU, nullptr, h->d_rZ + (size_t)B * P.nz, st, s, dit, h->d_rsol);
  for (size_t p0 = 0; p0 < pairs && rc == DOJO_OK; p0 += h->grad_chunk) {
    const int n = (int)std::min<size_t>(h->grad_chunk, pairs - p0);
    double* oGx = c.dev ? Gx + p0 * gx : cGx;
    double* oGu = c.dev ? Gu + p0 * gu : cGu;
    rc = launch_grad(h, opts, n, h->d_rZ + p0 * P.nz, dU ? dU + p0 * P.nu : nullptr, nullptr, h->d_rsol + p0 * P.nres, st + p0, h->d_Fz[0], h->d_Fu[0],
                     nullptr, 0, nullptr, nullptr, s);
    if (rc == DOJO_OK) rc = launch_kinjac(h, 2, n, h->d_rZ + p0 * P.nz, h->d_rZ + (p0 + B) * P.nz, h->d_Fz[0], h->d_Fu[0], oGx, oGu, s);
    if (rc == DOJO_OK && !c.dev) {
      CUDA_TRY(h, cudaMemcpyAsync(Gx + p0 * gx, oGx, (size_t)n * gx * sizeof(double), cudaMemcpyDeviceToHost, s));
      if (gu) CUDA_TRY(h, cudaMemcpyAsync(Gu + p0 * gu, oGu, (size_t)n * gu * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
  }
  if (rc == DOJO_OK) rc = launch_kin(h, false, (int)(pairs + B), h->d_rZ, dXt, s);
  if (rc == DOJO_OK) leave_call(h, s);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Reverse mode through a rollout: the recording rollout without the Jacobians (tape) and its adjoint pass (include/dojo_b200.h)
// ------------------------------------------------------------------------------------------------------------
// the REC launch of dojo_rollout_grad without the gradient kernel and without publishing pairs: the caller's tape is its sol_raw
static int launch_tape(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU, double* dZ_traj, double* dtape,
                       int32_t* dstatus, int32_t* diters, cudaStream_t s) {
  int rc = ensure_rec_kernel(h);
  if (rc == DOJO_OK && !dstatus) rc = ensure_rollout_grad_scratch(h, (size_t)B * T);  // the REC kernel always writes a status
  if (rc != DOJO_OK) return rc;
  enter_call(h, s);
  if (dZ0 != dZ_traj) CUDA_TRY(h, cudaMemcpyAsync(dZ_traj, dZ0, (size_t)B * h->plan.nz * sizeof(double), cudaMemcpyDeviceToDevice, s));
  rc = launch_rollout(h, opts, B, T, dZ_traj, dU, nullptr, dZ_traj + (size_t)B * h->plan.nz, dstatus ? dstatus : h->d_rstatus, s, diters, dtape);
  if (rc == DOJO_OK) leave_call(h, s);
  return rc;
}

static int launch_vjp(DojoHandle* h, int B, int T, const double* dZ_traj, const double* dU, const double* dtape, const double* dgZ, double* dgZ0,
                      double* dgU, int32_t* dstatus, cudaStream_t s) {
  if (!h->k_vjp) {
    const void* k = step_vjp_kernel_fn(h->any_contact, h->plan_smem_mask_grad == 0xff);
    CUDA_TRY(h, max_shared_memory(k, h->device));
    h->k_vjp = k;
  }
  // the adjoint pass reads no solver option: it runs no Newton iteration
  StepArgs a = step_args(h, nullptr, B, true);
  a.Z = dZ_traj; a.U = dU; a.sol_raw = const_cast<double*>(dtape); a.status = dstatus; a.T = T;
  a.vjp_gZ = dgZ; a.vjp_lam = dgZ0; a.vjp_gU = dgU;
  enter_call(h, s);
  CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  // plainly after whatever recorded the tape: step T - 1 is needed first
  const int grid = std::min((B + h->slots_grad - 1) / h->slots_grad, h->sm_count * h->envs_per_sm_grad);
  { void* kargs[1] = {(void*)&a}; CUDA_TRY(h, cudaLaunchKernel(h->k_vjp, dim3(grid), dim3(32 * h->nw * h->slots_grad), kargs, h->smem_grad, s)); }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_rollout_tape_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU, double* dZ_traj,
                                       double* dtape, int32_t* dstatus, int32_t* diters, void* cuda_stream) {
  int rc = trajectory_setup(h, B, T, dZ0 && dZ_traj && dtape, "dojo_rollout_tape_async", "the required buffers");
  if (rc != DOJO_OK) return rc;
  return launch_tape(h, opts, B, T, dZ0, dU, dZ_traj, dtape, dstatus, diters, (cudaStream_t)cuda_stream);
}

extern "C" int dojo_rollout_tape(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U, double* Z_traj,
                                 double* tape, int32_t* status, int32_t* iters) {
  int rc = trajectory_setup(h, B, T, Z0 && Z_traj && tape, "dojo_rollout_tape", "the required buffers");
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t pairs = (size_t)B * T;
  const double *dZ0 = Z0, *dU = U;
  double *dtraj = Z_traj, *dtape = tape;
  int32_t *dst = status, *dit = iters;
  HostCall c(h, Z0);
  c.in(&dZ0, (size_t)B * P.nz); c.in(&dU, pairs * P.nu);
  c.out(&dtraj, (pairs + B) * P.nz); c.out(&dtape, pairs * P.nres); c.out(&dst, pairs); c.out(&dit, pairs);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_tape(h, opts, B, T, dZ0, dU, dtraj, dtape, dst, dit, h->stream);
  return c.finish(rc);
}

extern "C" int dojo_rollout_vjp_async(DojoHandle* h, int B, int T, const double* dZ_traj, const double* dU, const double* dtape, const double* dgZ,
                                      double* dgZ0, double* dgU, int32_t* dstatus, void* cuda_stream) {
  int rc = trajectory_setup(h, B, T, dZ_traj && dtape && dgZ && dgZ0, "dojo_rollout_vjp_async", "the required buffers");
  if (rc != DOJO_OK) return rc;
  return launch_vjp(h, B, T, dZ_traj, dU, dtape, dgZ, dgZ0, dgU, dstatus, (cudaStream_t)cuda_stream);
}

extern "C" int dojo_rollout_vjp(DojoHandle* h, int B, int T, const double* Z_traj, const double* U, const double* tape, const double* gZ, double* gZ0,
                                double* gU, int32_t* status) {
  int rc = trajectory_setup(h, B, T, Z_traj && tape && gZ && gZ0, "dojo_rollout_vjp", "the required buffers");
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t pairs = (size_t)B * T, ng = 12 * (size_t)P.Nb;
  const double *dZt = Z_traj, *dU = U, *dtape = tape, *dgZ = gZ;
  double *dgZ0 = gZ0, *dgU = gU;
  int32_t* dst = status;
  HostCall c(h, Z_traj);
  c.in(&dZt, (pairs + B) * P.nz); c.in(&dtape, pairs * P.nres); c.in(&dU, pairs * P.nu); c.in(&dgZ, (pairs + B) * ng);
  c.out(&dgZ0, B * ng); c.out(&dgU, pairs * P.nu); c.out(&dst, B);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_vjp(h, B, T, dZt, dU, dtape, dgZ, dgZ0, dgU, dst, h->stream);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Closed-loop rollout: simulate! with a linear feedback controller! on the minimal state (include/dojo_b200.h)
// ------------------------------------------------------------------------------------------------------------
// The FB kernel evaluates the law inside the fused rollout, so that a closed loop costs one launch like dojo_rollout instead of three
// launches per step (maximal_to_minimal, the law, dojo_step), each of which waits for its slowest environment.
static int ensure_fb_kernel(DojoHandle* h) {
  if (h->k_fwd_fb) return DOJO_OK;
  const void* k = step_fb_kernel_fn(h->any_contact, h->plan_smem_mask == 0xff);
  int occ = 1;
  CUDA_TRY(h, max_shared_memory(k, h->device));
  CUDA_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, 32 * h->nw * h->slots, h->smem_fwd));
  h->envs_per_sm_fb = std::max(1, occ);
  if (!h->d_fbX) CUDA_TRY(h, cudaMalloc((void**)&h->d_fbX, (size_t)h->max_batch * 3 * h->plan.nu * sizeof(double)));
  h->k_fwd_fb = k;
  return DOJO_OK;
}

// argument checks of the closed-loop entries (dojo_rollout_feedback and its tape / adjoint): no launch before every check has passed
static int feedback_check(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* xi, bool buffers, const char* who) {
  if (!h) return DOJO_EINVAL;
  if (B <= 0 || B > h->max_batch || T <= 0 || !buffers || !fb || !fb->K || (fb->steps != 1 && fb->steps != T) || (fb->envs != 1 && fb->envs != B) ||
      (fb->K_i && !xi) || h->plan.nu == 0) {
    h->err = std::string(who) + ": bad arguments (B in 1..max_batch, T >= 1, Z0 / Z_final / feedback / K required, steps in {1, T}, envs in {1, B}, "
             "xi required with K_i, the mechanism must have inputs)";
    return DOJO_EINVAL;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return DOJO_OK;
}
static int feedback_setup(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* xi, bool buffers, const char* who) {
  int rc = feedback_check(h, B, T, fb, xi, buffers, who);
  return rc == DOJO_OK ? ensure_fb_kernel(h) : rc;
}

// fb's arrays are device pointers here
static int launch_feedback(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const DojoFeedback* fb, double* dxi, double* dZf,
                           double* dtraj, double* dUa, int32_t* dstatus, cudaStream_t s) {
  StepArgs a = step_args(h, opts, B, false);
  a.Z = dZ0; a.Zn = dZf; a.status = dstatus; a.T = T; a.traj = dtraj;
  a.fb_K = fb->K; a.fb_Ki = fb->K_i; a.fb_xref = fb->x_ref; a.fb_uref = fb->u_ref; a.fb_steps = fb->steps; a.fb_envs = fb->envs;
  a.fb_x = h->d_fbX; a.fb_xi = dxi;
  a.fb_u = dUa ? dUa : h->d_fbX + (size_t)h->max_batch * 2 * h->plan.nu; a.fb_u_T = dUa ? 1 : 0;
  enter_call(h, s);
  CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  const int grid = std::min((B + h->slots - 1) / h->slots, h->sm_count * h->envs_per_sm_fb);
  { void* kargs[1] = {(void*)&a}; CUDA_TRY(h, cudaLaunchKernel(h->k_fwd_fb, dim3(grid), dim3(32 * h->nw * h->slots), kargs, h->smem_fwd, s)); }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_rollout_feedback_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const DojoFeedback* fb,
                                           double* dxi, double* dZ_final, double* dZ_traj, double* dU_applied, int32_t* dstatus_any, void* cuda_stream) {
  int rc = feedback_setup(h, B, T, fb, dxi, dZ0 && dZ_final, "dojo_rollout_feedback_async");
  if (rc != DOJO_OK) return rc;
  return launch_feedback(h, opts, B, T, dZ0, fb, dxi, dZ_final, dZ_traj, dU_applied, dstatus_any, (cudaStream_t)cuda_stream);
}

extern "C" int dojo_rollout_feedback(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const DojoFeedback* fb, double* xi,
                                     double* Z_final, double* Z_traj, double* U_applied, int32_t* status_any) {
  int rc = feedback_setup(h, B, T, fb, xi, Z0 && Z_final, "dojo_rollout_feedback");
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t ne = (size_t)fb->steps * fb->envs, nx = 2 * (size_t)P.nu, nk = P.nu * nx * ne;
  DojoFeedback dfb = *fb;
  const double* dZ0 = Z0;
  double *dxi = xi, *dZf = Z_final, *dUa = U_applied, *dtraj = Z_traj;
  int32_t* dst = status_any;
  HostCall c(h, Z0);
  c.in(&dZ0, (size_t)B * P.nz); c.in(&dfb.K, nk); c.in(&dfb.K_i, nk); c.in(&dfb.x_ref, nx * ne); c.in(&dfb.u_ref, P.nu * ne); c.inout(&dxi, nx * B);
  c.out(&dZf, (size_t)B * P.nz); c.out(&dUa, (size_t)P.nu * B * T); c.out(&dtraj, (size_t)P.nz * B * T); c.out(&dst, B);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_feedback(h, opts, B, T, dZ0, &dfb, dxi, dZf, dtraj, dUa, dst, h->stream);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Reverse mode through the closed loop: the feedback tape and its adjoint (include/dojo_b200.h)
// ------------------------------------------------------------------------------------------------------------
// argument checks of both entries (no launch before every check has passed): the feedback rollout's rules and the tape's buffers
static int feedback_tape_setup(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* xi, const double* Xi_traj, bool buffers,
                               const char* who) {
  if (!h) return DOJO_EINVAL;
  if (!fb || (!fb->K_i != !Xi_traj)) {
    h->err = std::string(who) + ": bad arguments (feedback required; Xi_traj is required if and only if K_i is given)";
    return DOJO_EINVAL;
  }
  int rc = trajectory_setup(h, B, T, buffers, who, "Z_traj / X_traj / U_applied / tape required");
  if (rc == DOJO_OK) rc = feedback_check(h, B, T, fb, xi, true, who);
  return rc;
}

static int launch_feedback_tape(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const DojoFeedback* fb, double* dxi,
                                double* dZ_traj, double* dX_traj, double* dXi_traj, double* dUa, double* dtape, int32_t* dstatus, int32_t* diters,
                                cudaStream_t s) {
  if (!h->k_fb_tape) {
    const void* k = step_fbtape_kernel_fn(h->any_contact, h->plan_smem_mask == 0xff);
    int occ = 1;
    CUDA_TRY(h, max_shared_memory(k, h->device));
    CUDA_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, 32 * h->nw * h->slots, h->smem_fwd));
    h->envs_per_sm_fb_tape = std::max(1, occ);
    h->k_fb_tape = k;
  }
  if (!dstatus) {  // the REC kernel always writes a status
    int rc = ensure_rollout_grad_scratch(h, (size_t)B * T);
    if (rc != DOJO_OK) return rc;
  }
  StepArgs a = step_args(h, opts, B, false);
  a.Z = dZ_traj; a.traj = dZ_traj + (size_t)B * h->plan.nz; a.T = T;
  a.sol_raw = dtape; a.status = dstatus ? dstatus : h->d_rstatus; a.iters = diters;
  a.fb_K = fb->K; a.fb_Ki = fb->K_i; a.fb_xref = fb->x_ref; a.fb_uref = fb->u_ref; a.fb_steps = fb->steps; a.fb_envs = fb->envs;
  a.fb_xi = dxi; a.fb_u = dUa; a.fb_u_T = 1; a.fb_xtraj = dX_traj; a.fb_xitraj = dXi_traj;
  enter_call(h, s);
  if (dZ0 != dZ_traj) CUDA_TRY(h, cudaMemcpyAsync(dZ_traj, dZ0, (size_t)B * h->plan.nz * sizeof(double), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  const int grid = std::min((B + h->slots - 1) / h->slots, h->sm_count * h->envs_per_sm_fb_tape);
  { void* kargs[1] = {(void*)&a}; CUDA_TRY(h, cudaLaunchKernel(h->k_fb_tape, dim3(grid), dim3(32 * h->nw * h->slots), kargs, h->smem_fwd, s)); }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_rollout_feedback_tape_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const DojoFeedback* fb,
                                                double* dxi, double* dZ_traj, double* dX_traj, double* dXi_traj, double* dU_applied, double* dtape,
                                                int32_t* dstatus, int32_t* diters, void* cuda_stream) {
  int rc = feedback_tape_setup(h, B, T, fb, dxi, dXi_traj, dZ0 && dZ_traj && dX_traj && dU_applied && dtape, "dojo_rollout_feedback_tape_async");
  if (rc != DOJO_OK) return rc;
  return launch_feedback_tape(h, opts, B, T, dZ0, fb, dxi, dZ_traj, dX_traj, dXi_traj, dU_applied, dtape, dstatus, diters, (cudaStream_t)cuda_stream);
}

extern "C" int dojo_rollout_feedback_tape(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const DojoFeedback* fb, double* xi,
                                          double* Z_traj, double* X_traj, double* Xi_traj, double* U_applied, double* tape, int32_t* status,
                                          int32_t* iters) {
  int rc = feedback_tape_setup(h, B, T, fb, xi, Xi_traj, Z0 && Z_traj && X_traj && U_applied && tape, "dojo_rollout_feedback_tape");
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t pairs = (size_t)B * T, ne = (size_t)fb->steps * fb->envs, nx = 2 * (size_t)P.nu, nk = P.nu * nx * ne;
  DojoFeedback dfb = *fb;
  const double* dZ0 = Z0;
  double *dxi = xi, *dtraj = Z_traj, *dX = X_traj, *dXi = Xi_traj, *dUa = U_applied, *dtape = tape;
  int32_t *dst = status, *dit = iters;
  HostCall c(h, Z0);
  c.in(&dZ0, (size_t)B * P.nz); c.in(&dfb.K, nk); c.in(&dfb.K_i, nk); c.in(&dfb.x_ref, nx * ne); c.in(&dfb.u_ref, P.nu * ne); c.inout(&dxi, nx * B);
  c.out(&dtraj, (pairs + B) * P.nz); c.out(&dX, (pairs + B) * nx); c.out(&dXi, pairs * nx); c.out(&dUa, pairs * P.nu); c.out(&dtape, pairs * P.nres);
  c.out(&dst, pairs); c.out(&dit, pairs);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_feedback_tape(h, opts, B, T, dZ0, &dfb, dxi, dtraj, dX, dXi, dUa, dtape, dst, dit, h->stream);
  return c.finish(rc);
}

// the adjoint's checks: the tape's, the cotangents' and the gradient workspace (which also holds the per-joint contributions of M' w)
static int feedback_vjp_setup(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* Xi_traj, const double* gxi0, bool buffers,
                              const char* who) {
  if (h && fb && fb->K_i && !gxi0) { h->err = std::string(who) + ": bad arguments (gxi0 is required with K_i)"; return DOJO_EINVAL; }
  int rc = feedback_tape_setup(h, B, T, fb, fb && fb->K_i ? gxi0 : nullptr, Xi_traj, buffers, who);
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  if ((size_t)24 * P.Ne > (size_t)P.n_red * P.ch) { h->err = std::string(who) + ": the gradient workspace does not fit for this mechanism"; return DOJO_ENOMEM; }
  return DOJO_OK;
}

static int launch_feedback_vjp(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* dZ_traj, const double* dX_traj, const double* dXi_traj,
                               const double* dUa, const double* dtape, const double* dgZ, const double* dgX, const double* dgUa, const DojoFeedbackGrad* out,
                               double* dgZ0, double* dgxi0, int32_t* dstatus, double* dws, cudaStream_t s) {
  if (!h->k_fb_vjp) {
    const void* k = step_fbvjp_kernel_fn(h->any_contact, h->plan_smem_mask_grad == 0xff);
    CUDA_TRY(h, max_shared_memory(k, h->device));
    h->k_fb_vjp = k;
  }
  StepArgs a = step_args(h, nullptr, B, true);
  a.Z = dZ_traj; a.U = dUa; a.sol_raw = const_cast<double*>(dtape); a.status = dstatus; a.T = T;
  a.vjp_gZ = dgZ; a.vjp_lam = dgZ0;
  a.fb_K = fb->K; a.fb_Ki = fb->K_i; a.fb_xref = fb->x_ref; a.fb_uref = fb->u_ref; a.fb_steps = fb->steps; a.fb_envs = fb->envs; a.fb_xi = dgxi0;
  a.fb_xtraj = const_cast<double*>(dX_traj); a.fb_xitraj = const_cast<double*>(dXi_traj); a.fbv_gX = dgX; a.fbv_gUa = dgUa;
  if (out) { a.fbv_gK = out->K; a.fbv_gKi = fb->K_i ? out->K_i : nullptr; a.fbv_gxref = out->x_ref; a.fbv_guref = out->u_ref; }
  a.fbv_ws = dws;
  enter_call(h, s);
  CUDA_TRY(h, cudaMemsetAsync(h->d_counter, 0, sizeof(int), s));
  const int grid = std::min((B + h->slots_grad - 1) / h->slots_grad, h->sm_count * h->envs_per_sm_grad);
  { void* kargs[1] = {(void*)&a}; CUDA_TRY(h, cudaLaunchKernel(h->k_fb_vjp, dim3(grid), dim3(32 * h->nw * h->slots_grad), kargs, h->smem_grad, s)); }
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}
static size_t feedback_vjp_ws(const Plan& P, int B) { return ((size_t)4 * P.nu + 12 * (size_t)P.Nb) * B; }

extern "C" int dojo_rollout_feedback_vjp_async(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* dZ_traj, const double* dX_traj,
                                               const double* dXi_traj, const double* dU_applied, const double* dtape, const double* dgZ,
                                               const double* dgX, const double* dgUa, const DojoFeedbackGrad* out, double* dgZ0, double* dgxi0,
                                               int32_t* dstatus, void* cuda_stream) {
  int rc = feedback_vjp_setup(h, B, T, fb, dXi_traj, dgxi0, dZ_traj && dX_traj && dU_applied && dtape && dgZ0, "dojo_rollout_feedback_vjp_async");
  if (rc == DOJO_OK) rc = grow_buffer(h, (void**)&h->d_fbvws, &h->fbvws_bytes, feedback_vjp_ws(h->plan, B) * sizeof(double));
  if (rc != DOJO_OK) return rc;
  return launch_feedback_vjp(h, B, T, fb, dZ_traj, dX_traj, dXi_traj, dU_applied, dtape, dgZ, dgX, dgUa, out, dgZ0, dgxi0, dstatus, h->d_fbvws,
                             (cudaStream_t)cuda_stream);
}

extern "C" int dojo_rollout_feedback_vjp(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* Z_traj, const double* X_traj,
                                         const double* Xi_traj, const double* U_applied, const double* tape, const double* gZ, const double* gX,
                                         const double* gUa, const DojoFeedbackGrad* out, double* gZ0, double* gxi0, int32_t* status) {
  int rc = feedback_vjp_setup(h, B, T, fb, Xi_traj, gxi0, Z_traj && X_traj && U_applied && tape && gZ0, "dojo_rollout_feedback_vjp");
  if (rc != DOJO_OK) return rc;
  const Plan& P = h->plan;
  const size_t pairs = (size_t)B * T, ne = (size_t)fb->steps * fb->envs, nx = 2 * (size_t)P.nu, nk = P.nu * nx, ng = 12 * (size_t)P.Nb;
  const size_t no = (size_t)fb->steps * B;  // entries of each gradient output
  DojoFeedback dfb = *fb;
  DojoFeedbackGrad dout = {};
  if (out) dout = *out;
  if (!fb->K_i) dout.K_i = nullptr;
  const double *dZt = Z_traj, *dX = X_traj, *dXi = Xi_traj, *dUa = U_applied, *dtape = tape, *dgZ = gZ, *dgX = gX, *dgUa = gUa;
  double *dgZ0 = gZ0, *dgxi0 = fb->K_i ? gxi0 : nullptr, *dws = nullptr;
  int32_t* dst = status;
  HostCall c(h, Z_traj);
  c.in(&dfb.K, nk * ne); c.in(&dfb.K_i, nk * ne); c.in(&dfb.x_ref, nx * ne); c.in(&dfb.u_ref, P.nu * ne);
  c.in(&dZt, (pairs + B) * P.nz); c.in(&dX, (pairs + B) * nx); c.in(&dXi, pairs * nx); c.in(&dUa, pairs * P.nu); c.in(&dtape, pairs * P.nres);
  c.in(&dgZ, (pairs + B) * ng); c.in(&dgX, (pairs + B) * nx); c.in(&dgUa, pairs * P.nu);
  c.out(&dout.K, nk * no); c.out(&dout.K_i, nk * no); c.out(&dout.x_ref, nx * no); c.out(&dout.u_ref, P.nu * no);
  c.out(&dgZ0, B * ng); c.out(&dgxi0, B * nx); c.out(&dst, B);
  c.scratch(&dws, feedback_vjp_ws(P, B));
  rc = c.bind();
  if (rc == DOJO_OK && c.dev) rc = grow_buffer(h, (void**)&h->d_fbvws, &h->fbvws_bytes, feedback_vjp_ws(P, B) * sizeof(double));
  if (rc == DOJO_OK) rc = launch_feedback_vjp(h, B, T, &dfb, dZt, dX, dXi, dUa, dtape, dgZ, dgX, dgUa, &dout, dgZ0, dgxi0, dst, c.dev ? h->d_fbvws : dws,
                                              h->stream);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Riccati backward pass of iLQR / TVLQR in minimal coordinates (include/dojo_b200.h, dojo_lqr.cuh)
// ------------------------------------------------------------------------------------------------------------
// threads per CTA (one CTA per environment): enough 2 x 2 tiles of the nx x nx products per thread to hide shared-memory latency
static int lqr_threads(int nu) { return nu <= 4 ? 64 : nu <= 16 ? 128 : nu <= 24 ? 256 : 512; }

// argument checks shared by both entries (no launch before every check has passed); fills the kernel arguments but the arrays
static int lqr_setup(DojoHandle* h, int B, int T, const DojoQuadraticCost* c, const int32_t* active, const double* X, const double* U, const double* Gx,
                     const double* Gu, const double* mu, double* K, double* k, double* dV, int32_t* status, LqrArgs* a, const char* who) {
  if (!h) return DOJO_EINVAL;
  const int nu = h->plan.nu;
  int na = 0;
  if (active)
    for (int i = 0; i < nu; ++i) na += active[i] != 0;
  if (B <= 0 || B > h->max_batch || T <= 0 || !X || !Gx || !Gu || !K || !k || !c || !c->Q || !c->R || !c->Q_final || (c->steps != 1 && c->steps != T) ||
      (c->envs != 1 && c->envs != B) || nu == 0 || (active && na == 0)) {
    h->err = std::string(who) + ": bad arguments (B in 1..max_batch, T >= 1, cost / Q / R / Q_final / X_traj / Gx / Gu / K / k required, "
             "steps in {1, T}, envs in {1, B}, the mechanism must have inputs, `active` must have a nonzero entry)";
    return DOJO_EINVAL;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int optin = 0;
  CUDA_TRY(h, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
  if (nu > DJ_LQR_MAX_NU || lqr_smem_bytes(nu) > (size_t)optin) {
    h->err = std::string(who) + ": the Riccati working set of one environment (" + std::to_string(lqr_smem_bytes(nu)) +
             " bytes) exceeds the shared memory of one block";
    return DOJO_ENOMEM;
  }
  if (!h->lqr_ready) {
    CUDA_TRY(h, max_shared_memory((const void*)dojo_lqr_backward_kernel, h->device));
    h->lqr_ready = true;
  }
  *a = LqrArgs{};
  a->nu = nu; a->B = B; a->T = T; a->steps = c->steps; a->envs = c->envs;
  for (int i = 0; i < nu; ++i)
    if (!active || active[i]) a->act[a->na++] = i;
  a->Q = c->Q; a->R = c->R; a->xg = c->x_goal; a->ug = c->u_goal; a->Qf = c->Q_final; a->xgf = c->x_goal_final;
  a->X = X; a->U = U; a->Gx = Gx; a->Gu = Gu; a->mu = mu; a->K = K; a->k = k; a->dV = dV; a->status = status;
  return DOJO_OK;
}

static int launch_lqr(DojoHandle* h, const LqrArgs& a, cudaStream_t s) {
  enter_call(h, s);
  void* kargs[1] = {(void*)&a};
  CUDA_TRY(h, cudaLaunchKernel((const void*)dojo_lqr_backward_kernel, dim3(a.B), dim3(lqr_threads(a.nu)), kargs, lqr_smem_bytes(a.nu), s));
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_lqr_backward_async(DojoHandle* h, int B, int T, const DojoQuadraticCost* cost, const int32_t* active, const double* dX_traj,
                                       const double* dU, const double* dGx, const double* dGu, const double* dmu, double* dK, double* dk, double* ddV,
                                       int32_t* dstatus, void* cuda_stream) {
  LqrArgs a;
  int rc = lqr_setup(h, B, T, cost, active, dX_traj, dU, dGx, dGu, dmu, dK, dk, ddV, dstatus, &a, "dojo_lqr_backward_async");
  if (rc != DOJO_OK) return rc;
  return launch_lqr(h, a, (cudaStream_t)cuda_stream);
}

extern "C" int dojo_lqr_backward(DojoHandle* h, int B, int T, const DojoQuadraticCost* cost, const int32_t* active, const double* X_traj,
                                 const double* U, const double* Gx, const double* Gu, const double* mu, double* K, double* k, double* dV,
                                 int32_t* status) {
  LqrArgs a;
  int rc = lqr_setup(h, B, T, cost, active, X_traj, U, Gx, Gu, mu, K, k, dV, status, &a, "dojo_lqr_backward");
  if (rc != DOJO_OK) return rc;
  const size_t nu = a.nu, nx = 2 * nu, ne = (size_t)cost->steps * cost->envs, pairs = (size_t)B * T;
  HostCall c(h, X_traj);
  c.in(&a.Q, nx * nx * ne); c.in(&a.R, nu * nu * ne); c.in(&a.xg, nx * ne); c.in(&a.ug, nu * ne); c.in(&a.Qf, nx * nx * cost->envs);
  c.in(&a.xgf, nx * cost->envs); c.in(&a.X, nx * (pairs + B)); c.in(&a.U, nu * pairs); c.in(&a.Gx, nx * nx * pairs); c.in(&a.Gu, nx * nu * pairs);
  c.in(&a.mu, B); c.out(&a.K, nu * nx * pairs); c.out(&a.k, nu * pairs); c.out(&a.dV, 2 * (size_t)B); c.out(&a.status, B);
  rc = c.bind();
  if (rc == DOJO_OK) rc = launch_lqr(h, a, h->stream);
  return c.finish(rc);
}

// ------------------------------------------------------------------------------------------------------------
// Batched environment layer (SURVEY.md 8 f2; dojo_envs.cuh)
// ------------------------------------------------------------------------------------------------------------
static bool env_spec_ok(const DojoHandle* h, const DojoEnvSpec* sp) {
  if (!sp) return false;
  const int ns = 2 * h->plan.nu + (sp->contact_obs ? h->plan.Ni : 0);
  return sp->n_unactuated >= 0 && sp->n_unactuated <= h->plan.nu && sp->forward_index < ns && sp->healthy_index < ns && sp->bound_index < ns;
}
static EnvSpec to_dev_spec(const DojoEnvSpec* sp) {
  EnvSpec e;
  e.n_unactuated = sp->n_unactuated; e.contact_obs = sp->contact_obs; e.forward_index = sp->forward_index; e.healthy_index = sp->healthy_index;
  e.bound_index = sp->bound_index; e.w_forward = sp->w_forward; e.w_control = sp->w_control; e.w_contact = sp->w_contact;
  e.survive_reward = sp->survive_reward; e.healthy_min = sp->healthy_min; e.healthy_max = sp->healthy_max; e.bound_abs = sp->bound_abs;
  return e;
}
extern "C" int dojo_env_num_state(const DojoHandle* h, const DojoEnvSpec* spec) { return 2 * h->plan.nu + ((spec && spec->contact_obs) ? h->plan.Ni : 0); }
extern "C" int dojo_env_num_action(const DojoHandle* h, const DojoEnvSpec* spec) { return h->plan.nu - (spec ? spec->n_unactuated : 0); }

static int ensure_env_staging(DojoHandle* h) {
  if (h->d_envS) return DOJO_OK;
  const size_t B = h->max_batch, ns = 2 * (size_t)h->plan.nu + h->plan.Ni;
  CUDA_TRY(h, cudaMalloc((void**)&h->d_envS, B * ns * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_envSn, B * ns * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_envA, std::max<size_t>(1, B * h->plan.nu) * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_envR, B * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_envDone, B * sizeof(int32_t)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_envS0, ns * sizeof(double)));
  return DOJO_OK;
}

static int env_step_impl(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, const double* dS, const double* dA, double* dSn,
                         double* dreward, int32_t* ddone, int32_t* dstatus, int32_t* diters, double* dret, int32_t* ddead, void* cuda_stream);
extern "C" int dojo_env_step_async(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, const double* dS, const double* dA,
                                   double* dSn, double* dreward, int32_t* ddone, int32_t* dstatus, int32_t* diters, void* cuda_stream) {
  return env_step_impl(h, opts, spec, B, dS, dA, dSn, dreward, ddone, dstatus, diters, nullptr, nullptr, cuda_stream);
}
static int env_step_impl(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, const double* dS, const double* dA, double* dSn,
                         double* dreward, int32_t* ddone, int32_t* dstatus, int32_t* diters, double* dret, int32_t* ddead, void* cuda_stream) {
  if (!h || B <= 0 || B > h->max_batch || !dS || !dSn || dS == dSn || !env_spec_ok(h, spec)) {
    if (h) h->err = "dojo_env_step_async: bad arguments (B <= max_batch, S_next != S, indices inside the state)";
    return DOJO_EINVAL;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);  // maximal states, inputs and the solution stay in the handle's device buffers
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = (cudaStream_t)cuda_stream;
  const Plan& P = h->plan;
  EnvArgs a;
  a.joints = P.joints; a.contacts = P.contacts; a.order = h->d_kin_order;
  a.Ne = P.Ne; a.Nb = P.Nb; a.Ni = P.Ni; a.nu = P.nu; a.nres = P.nres; a.B = B; a.h = P.h;
  a.spec = to_dev_spec(spec);
  a.S = dS; a.A = dA; a.Z = h->d_Z; a.U = h->d_U; a.Zn = h->d_Zn; a.sol = h->d_sol; a.Sn = dSn; a.reward = dreward; a.done = ddone;
  a.ret = dret; a.dead = ddead;
  const int threads = 128, grid = (B + threads - 1) / threads;
  enter_call(h, s);
  dojo_env_pre_kernel<<<grid, threads, 0, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  rc = launch_forward(h, opts, B, h->d_Z, P.nu > 0 ? h->d_U : nullptr, nullptr, h->d_Zn, h->d_sol, nullptr, dstatus, diters, 0, s);
  if (rc != DOJO_OK) return rc;
  dojo_env_post_kernel<<<grid, threads, 0, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  leave_call(h, s);
  return DOJO_OK;
}

extern "C" int dojo_env_step(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, const double* S, const double* A, double* Sn,
                             double* reward, int32_t* done, int32_t* status, int32_t* iters) {
  if (!h || B <= 0 || B > h->max_batch || !S || !Sn || !env_spec_ok(h, spec)) { if (h) h->err = "dojo_env_step: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t ns = dojo_env_num_state(h, spec), na = dojo_env_num_action(h, spec);
  const double *dS = S, *dA = A;
  double *dSn = Sn, *dR = reward;
  int32_t *dd = done, *dst = status, *dit = iters;
  HostCall c(h, S);
  c.in(&dS, B * ns); c.in(&dA, B * na); c.out(&dSn, B * ns); c.out(&dR, B); c.out(&dd, B); c.out(&dst, B); c.out(&dit, B);
  int rc = c.bind();
  if (rc == DOJO_OK) rc = dojo_env_step_async(h, opts, spec, B, dS, dA, dSn, dR, dd, dst, dit, h->stream);
  return c.finish(rc);
}

extern "C" int dojo_env_reset(DojoHandle* h, const DojoEnvSpec* spec, int B, const double* s0, const int32_t* mask, double* S) {
  if (!h || B <= 0 || B > h->max_batch || !s0 || !S || !spec) { if (h) h->err = "dojo_env_reset: bad arguments"; return DOJO_EINVAL; }
  const size_t ns = dojo_env_num_state(h, spec);
  if (!is_device_ptr(S)) {  // host buffers: nothing for the device to do
    for (int e = 0; e < B; ++e)
      if (!mask || mask[e]) std::memcpy(S + (size_t)e * ns, s0, ns * sizeof(double));
    return DOJO_OK;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_env_staging(h);
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = h->stream;
  CUDA_TRY(h, cudaMemcpyAsync(h->d_envS0, s0, ns * sizeof(double), cudaMemcpyHostToDevice, s));
  dojo_env_reset_kernel<<<(B + 127) / 128, 128, 0, s>>>((int)ns, B, h->d_envS0, mask, S);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  CUDA_TRY(h, cudaStreamSynchronize(s));
  return DOJO_OK;
}

// ------------------------------------------------------------------------------------------------------------
// Trajectory recording and momentum / energy diagnostics (SURVEY.md 8 f3; dojo_storage.cuh)
// ------------------------------------------------------------------------------------------------------------
static int launch_storage(DojoHandle* h, int B, const double* dZ, const double* dZn, const double* dU, const double* dsol, double* dstorage, double* ddiag,
                          cudaStream_t s) {
  const Plan& P = h->plan;
  StorageArgs a;
  a.bodies = P.bodies; a.joints = P.joints;
  a.Ne = P.Ne; a.Nb = P.Nb; a.nu = P.nu; a.nres = P.nres; a.B = B; a.h = P.h; a.input_scaling = P.input_scaling;
  for (int i = 0; i < 3; ++i) a.g[i] = P.g[i];
  a.Z = dZ; a.Zn = dZn; a.U = dU; a.sol = dsol; a.body_out = dstorage; a.diag = ddiag;
  dojo_storage_kernel<<<(B + 127) / 128, 128, 0, s>>>(a);
  CUDA_TRY(h, cudaGetLastError());
  h->launches += 1;
  return DOJO_OK;
}

__global__ void dojo_status_max_kernel(int B, const int32_t* st, int32_t* any) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < B) any[e] = max(any[e], st[e]);
}

extern "C" int dojo_step_record_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU, double* dZn, double* dstorage,
                                      double* ddiag, int32_t* dstatus, int32_t* diters, void* cuda_stream) {
  if (!h || B <= 0 || B > h->max_batch || !dZ || !dZn || !dstorage || !ddiag || dZ == dZn) {
    if (h) h->err = "dojo_step_record_async: bad arguments (B <= max_batch, Z_next != Z)";
    return DOJO_EINVAL;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);  // the solver solution stays in the handle's device buffer
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = (cudaStream_t)cuda_stream;
  rc = launch_forward(h, opts, B, dZ, dU, nullptr, dZn, h->d_sol, nullptr, dstatus, diters, 0, s);
  if (rc != DOJO_OK) return rc;
  rc = launch_storage(h, B, dZ, dZn, dU, h->d_sol, dstorage, ddiag, s);
  leave_call(h, s);  // the storage kernel reads the handle's solution buffer: later calls on other streams wait for it
  return rc;
}

static int ensure_record_staging(DojoHandle* h) {
  if (h->d_recS) return DOJO_OK;
  const size_t B = h->max_batch;
  for (int k = 0; k < 2; ++k) CUDA_TRY(h, cudaMalloc((void**)&h->d_recZ[k], B * h->plan.nz * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_recS, B * 12 * h->plan.Nb * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_recD, B * 8 * sizeof(double)));
  CUDA_TRY(h, cudaMalloc((void**)&h->d_recAny, B * sizeof(int32_t)));
  return DOJO_OK;
}

extern "C" int dojo_step_record(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, double* Zn, double* storage,
                                double* diag, int32_t* status, int32_t* iters) {
  if (!h || B <= 0 || B > h->max_batch || !Z || !Zn || !storage || !diag) { if (h) h->err = "dojo_step_record: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const Plan& P = h->plan;
  const double *dZ = Z, *dU = U;
  double *dZn = Zn, *dS = storage, *dD = diag;
  int32_t *dst = status, *dit = iters;
  HostCall c(h, Z);
  c.in(&dZ, (size_t)B * P.nz); c.in(&dU, (size_t)B * P.nu);
  c.out(&dZn, (size_t)B * P.nz); c.out(&dS, (size_t)B * 12 * P.Nb); c.out(&dD, (size_t)B * 8); c.out(&dst, B); c.out(&dit, B);
  int rc = c.bind();
  if (rc == DOJO_OK) rc = dojo_step_record_async(h, opts, B, dZ, dU, dZn, dS, dD, dst, dit, h->stream);
  return c.finish(rc);
}

extern "C" int dojo_simulate_record(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U, double* Z_final,
                                    double* Z_traj, double* storage, double* diag, int32_t* status_any) {
  if (!h || B <= 0 || B > h->max_batch || T <= 0 || !Z0 || !Z_final) { if (h) h->err = "dojo_simulate_record: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);
  if (rc == DOJO_OK) rc = ensure_record_staging(h);
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = h->stream;
  const Plan& P = h->plan;
  const double* dU = (U && P.nu > 0) ? U : nullptr;
  HostCall c(h, Z0);
  c.in(&dU, (size_t)P.nu * B * T);
  rc = c.bind();
  if (rc != DOJO_OK) return rc;
  const bool dev = c.dev;
  const cudaMemcpyKind in = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, out = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  const size_t nzb = (size_t)B * P.nz * sizeof(double), nsb = (size_t)B * 12 * P.Nb * sizeof(double), ndb = (size_t)B * 8 * sizeof(double);
  CUDA_TRY(h, cudaMemcpyAsync(h->d_recZ[0], Z0, nzb, in, s));
  CUDA_TRY(h, cudaMemsetAsync(h->d_recAny, 0, (size_t)B * sizeof(int32_t), s));
  int cur = 0;
  for (int k = 0; k < T; ++k, cur ^= 1) {
    // with device pointers the per-step outputs are written in place
    double* dS = (dev && storage) ? storage + (size_t)k * B * 12 * P.Nb : h->d_recS;
    double* dD = (dev && diag) ? diag + (size_t)k * B * 8 : h->d_recD;
    rc = dojo_step_record_async(h, opts, B, h->d_recZ[cur], dU ? dU + (size_t)k * B * P.nu : nullptr, h->d_recZ[cur ^ 1], dS, dD, h->d_status, nullptr, s);
    if (rc != DOJO_OK) return rc;
    dojo_status_max_kernel<<<(B + 255) / 256, 256, 0, s>>>(B, h->d_status, h->d_recAny);
    CUDA_TRY(h, cudaGetLastError());
    h->launches += 1;
    if (Z_traj) CUDA_TRY(h, cudaMemcpyAsync(Z_traj + (size_t)k * B * P.nz, h->d_recZ[cur], nzb, out, s));
    if (!dev && storage) CUDA_TRY(h, cudaMemcpyAsync(storage + (size_t)k * B * 12 * P.Nb, h->d_recS, nsb, cudaMemcpyDeviceToHost, s));
    if (!dev && diag) CUDA_TRY(h, cudaMemcpyAsync(diag + (size_t)k * B * 8, h->d_recD, ndb, cudaMemcpyDeviceToHost, s));
  }
  CUDA_TRY(h, cudaMemcpyAsync(Z_final, h->d_recZ[cur], nzb, out, s));
  if (status_any) CUDA_TRY(h, cudaMemcpyAsync(status_any, h->d_recAny, (size_t)B * sizeof(int32_t), out, s));
  return c.finish();
}

extern "C" int dojo_env_rollout(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, int T, const double* S0, const double* A,
                                double* S_final, double* ret, int32_t* failed) {
  if (!h || B <= 0 || B > h->max_batch || T <= 0 || !S0 || !S_final || !env_spec_ok(h, spec)) { if (h) h->err = "dojo_env_rollout: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);
  if (rc == DOJO_OK) rc = ensure_env_staging(h);
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = h->stream;
  const size_t ns = dojo_env_num_state(h, spec), na = dojo_env_num_action(h, spec);
  const double* dA = (A && na > 0) ? A : nullptr;
  HostCall c(h, S0);
  c.in(&dA, na * B * T);
  rc = c.bind();
  if (rc != DOJO_OK) return rc;
  const cudaMemcpyKind in = c.dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, out = c.dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  double* buf[2] = {h->d_envS, h->d_envSn};
  CUDA_TRY(h, cudaMemcpyAsync(buf[0], S0, (size_t)B * ns * sizeof(double), in, s));
  CUDA_TRY(h, cudaMemsetAsync(h->d_envR, 0, (size_t)B * sizeof(double), s));        // return accumulator
  CUDA_TRY(h, cudaMemsetAsync(h->d_envDone, 0, (size_t)B * sizeof(int32_t), s));    // failure flags
  int cur = 0;
  for (int k = 0; k < T; ++k, cur ^= 1) {
    rc = env_step_impl(h, opts, spec, B, buf[cur], dA ? dA + (size_t)k * B * na : nullptr, buf[cur ^ 1], nullptr, nullptr, h->d_status, nullptr, h->d_envR,
                       h->d_envDone, s);
    if (rc != DOJO_OK) return rc;
  }
  CUDA_TRY(h, cudaMemcpyAsync(S_final, buf[cur], (size_t)B * ns * sizeof(double), out, s));
  if (ret) CUDA_TRY(h, cudaMemcpyAsync(ret, h->d_envR, (size_t)B * sizeof(double), out, s));
  if (failed) CUDA_TRY(h, cudaMemcpyAsync(failed, h->d_envDone, (size_t)B * sizeof(int32_t), out, s));
  return c.finish();
}

// ------------------------------------------------------------------------------------------------------------
// Parameter update (system identification): rebuild the plan tables for the same topology and swap them in place
// ------------------------------------------------------------------------------------------------------------
extern "C" int dojo_update_params(DojoHandle* h, const DojoMechanismDesc* d) {
  if (!h || !d) { if (h) h->err = "dojo_update_params: bad arguments"; return DOJO_EINVAL; }
  DojoHandle* t = nullptr;
  int rc = dojo_create(d, h->device, 1, &t);  // validates the descriptor and builds the tables exactly like a fresh handle
  if (rc != DOJO_OK) { h->err = std::string("dojo_update_params: ") + g_create_error; return rc; }
  const Plan &A = h->plan, &B = t->plan;
  bool same = A.Nb == B.Nb && A.Ne == B.Ne && A.Ni == B.Ni && A.nres == B.nres && A.nu == B.nu && A.nw == B.nw && A.nphase == B.nphase &&
              A.arena_len == B.arena_len && A.grad_len == B.grad_len && A.n_red == B.n_red && h->blob_bytes == t->blob_bytes &&
              h->arena_bytes == t->arena_bytes && (h->grad_bytes == t->grad_bytes);
  for (int k = 0; k < 8; ++k) same = same && h->blob_off[k] == t->blob_off[k];
  // the handle keeps the kernels it was created with: a contact model or a translational spring / damper / limit that needs the other
  // compilation (dojo_b200_cm.cu) cannot be switched on or off by an update
  same = same && h->any_contact == t->any_contact && h->orthant_contact == t->orthant_contact && h->tra_joint == t->tra_joint;
  if (!same) { dojo_destroy(t); h->err = "dojo_update_params: the descriptor has a different topology (use dojo_create)"; return DOJO_EINVAL; }
  cudaError_t e = cudaSetDevice(h->device);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();  // kernels on caller streams may still read the tables
  if (e == cudaSuccess) e = cudaMemcpy(h->d_blob, t->d_blob, (size_t)h->blob_bytes, cudaMemcpyDeviceToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_kin_order, t->d_kin_order, sizeof(int) * A.Ne, cudaMemcpyDeviceToDevice);
  if (e != cudaSuccess) { dojo_destroy(t); h->err = std::string("dojo_update_params: ") + cudaGetErrorString(e); return DOJO_ECUDA; }
  h->plan.h = B.h; h->plan.input_scaling = B.input_scaling;
  for (int i = 0; i < 3; ++i) h->plan.g[i] = B.g[i];
  h->plan.ls_pair = B.ls_pair; h->plan.ls_slot_delta = B.ls_slot_delta; h->plan.ls_res2_off = B.ls_res2_off;
  dojo_destroy(t);
  return DOJO_OK;
}

extern "C" int dojo_env_policy_rollout(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, int T, const double* S0,
                                       const double* Theta, const double* mean, const double* stdev, double* S_final, double* ret, int32_t* failed,
                                       double* S_traj) {
  if (!h || B <= 0 || B > h->max_batch || T <= 0 || !S0 || !Theta || !S_final || !env_spec_ok(h, spec) || ((mean == nullptr) != (stdev == nullptr))) {
    if (h) h->err = "dojo_env_policy_rollout: bad arguments";
    return DOJO_EINVAL;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int rc = ensure_staging(h);
  if (rc == DOJO_OK) rc = ensure_env_staging(h);
  if (rc != DOJO_OK) return rc;
  cudaStream_t s = h->stream;
  const size_t ns = dojo_env_num_state(h, spec), na = dojo_env_num_action(h, spec);
  if (na == 0) { h->err = "dojo_env_policy_rollout: the environment has no actions"; return DOJO_EINVAL; }
  if (!h->d_envNorm) CUDA_TRY(h, cudaMalloc((void**)&h->d_envNorm, 2 * (2 * (size_t)h->plan.nu + h->plan.Ni) * sizeof(double)));
  const double* dTheta = Theta;
  HostCall c(h, S0);
  c.in(&dTheta, B * ns * na);
  rc = c.bind();
  if (rc != DOJO_OK) return rc;
  const cudaMemcpyKind in = c.dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, out = c.dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  if (mean) {
    CUDA_TRY(h, cudaMemcpyAsync(h->d_envNorm, mean, ns * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_TRY(h, cudaMemcpyAsync(h->d_envNorm + ns, stdev, ns * sizeof(double), cudaMemcpyHostToDevice, s));
  }
  double* buf[2] = {h->d_envS, h->d_envSn};
  CUDA_TRY(h, cudaMemcpyAsync(buf[0], S0, (size_t)B * ns * sizeof(double), in, s));
  CUDA_TRY(h, cudaMemsetAsync(h->d_envR, 0, (size_t)B * sizeof(double), s));
  CUDA_TRY(h, cudaMemsetAsync(h->d_envDone, 0, (size_t)B * sizeof(int32_t), s));
  int cur = 0;
  for (int k = 0; k < T; ++k, cur ^= 1) {
    PolicyArgs p;
    p.ns = (int)ns; p.na = (int)na; p.B = B; p.S = buf[cur]; p.Theta = dTheta;
    p.mean = mean ? h->d_envNorm : nullptr; p.stdev = mean ? h->d_envNorm + ns : nullptr; p.A = h->d_envA;
    dojo_env_policy_kernel<<<(B + 127) / 128, 128, 0, s>>>(p);
    CUDA_TRY(h, cudaGetLastError());
    h->launches += 1;
    if (S_traj) CUDA_TRY(h, cudaMemcpyAsync(S_traj + (size_t)k * B * ns, buf[cur], (size_t)B * ns * sizeof(double), out, s));
    rc = env_step_impl(h, opts, spec, B, buf[cur], h->d_envA, buf[cur ^ 1], nullptr, nullptr, h->d_status, nullptr, h->d_envR, h->d_envDone, s);
    if (rc != DOJO_OK) return rc;
  }
  CUDA_TRY(h, cudaMemcpyAsync(S_final, buf[cur], (size_t)B * ns * sizeof(double), out, s));
  if (ret) CUDA_TRY(h, cudaMemcpyAsync(ret, h->d_envR, (size_t)B * sizeof(double), out, s));
  if (failed) CUDA_TRY(h, cudaMemcpyAsync(failed, h->d_envDone, (size_t)B * sizeof(int32_t), out, s));
  return c.finish();
}

// ------------------------------------------------------------------------------------------------------------
// get_contact_gradients (gradients/contact.jl:1-55): host- or device-pointer entry
// ------------------------------------------------------------------------------------------------------------
extern "C" int dojo_num_contact_data(const DojoHandle* h) { return 5 * h->plan.Ni; }

extern "C" int dojo_step_grad_contact(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, double* Zn, double* Fz,
                                      double* Fu, double* Fc, int32_t* status, int32_t* iters) {
  if (!h || B <= 0 || B > h->max_batch || !Z || !Zn || !Fz || !Fu || !Fc) { if (h) h->err = "dojo_step_grad_contact: bad arguments"; return DOJO_EINVAL; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const Plan& P = h->plan;
  cudaStream_t s = h->stream;
  HostCall c(h, Z);
  if (c.dev) return c.finish(dojo_step_grad_contact_async(h, opts, B, Z, U, nullptr, Zn, Fz, Fu, Fc, status, iters, 0, s));
  const size_t ng = 12 * (size_t)P.Nb, fz = ng * ng, fu = ng * P.nu, fc = ng * 5 * P.Ni;
  // chunks of environments whose three Jacobians fit 192 MB of device staging
  const int chunk = (int)std::max<size_t>(1, std::min<size_t>(B, (size_t(192) << 20) / ((fz + fu + fc) * sizeof(double))));
  const double *dZ = Z, *dU = U;
  double *dZn = Zn, *dFz = nullptr;
  int32_t *dst = status, *dit = iters;
  c.in(&dZ, (size_t)B * P.nz); c.in(&dU, (size_t)B * P.nu); c.out(&dZn, (size_t)B * P.nz); c.out(&dst, B); c.out(&dit, B);
  c.scratch(&dFz, (size_t)chunk * (fz + fu + fc));
  int rc = c.bind();
  if (rc != DOJO_OK) return rc;
  double *dFu = dFz + (size_t)chunk * fz, *dFc = dFu + (size_t)chunk * fu;
  for (int e0 = 0; e0 < B && rc == DOJO_OK; e0 += chunk) {
    const int nb = std::min(chunk, B - e0);
    rc = dojo_step_grad_contact_async(h, opts, nb, dZ + (size_t)e0 * P.nz, dU ? dU + (size_t)e0 * P.nu : nullptr, nullptr, dZn + (size_t)e0 * P.nz, dFz, dFu,
                                      dFc, dst ? dst + e0 : nullptr, dit ? dit + e0 : nullptr, 0, s);
    if (rc != DOJO_OK) break;
    CUDA_TRY(h, cudaMemcpyAsync(Fz + (size_t)e0 * fz, dFz, (size_t)nb * fz * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (fu) CUDA_TRY(h, cudaMemcpyAsync(Fu + (size_t)e0 * fu, dFu, (size_t)nb * fu * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (fc) CUDA_TRY(h, cudaMemcpyAsync(Fc + (size_t)e0 * fc, dFc, (size_t)nb * fc * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  return c.finish(rc);
}
