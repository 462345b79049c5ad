// dojo_step_kernel.cuh -- kernel entry point of the per-timestep hot path: dojo_step_kernel<GRAD> and its argument block.
//
// Compiled twice into libdojo_b200.so:
//   * dojo_b200.cu     (namespace dj):    NonlinearContact only -- every BASELINE model; this is the benchmarked kernel
//   * dojo_b200_cm.cu  (namespace dj_cm, DJ_ANY_CONTACT): additionally ImpactContact / LinearContact (SURVEY.md 8 f4) and translational
//     springs / dampers / limits (8 a4 / a6), selected by dojo_create for mechanisms that contain them.  The extra model code never enters the first compilation, whose SASS
//     is bit-identical with and without this split (checked with cuobjdump).
// The `// [hostemu:...]` markers delimit the text that tests/hostemu/gen.py compiles for the CPU emulation of the kernel.
#pragma once
#include "../../include/dojo_b200.h"
#include "dojo_grad.cuh"
#include "dojo_kin.cuh"

namespace dj {

// [hostemu:kernel:begin]
struct StepArgs {
  Plan plan;
  Options opts;
  int B;
  const double* Z;
  const double* U;
  const double* Fext;
  double* Zn;
  double* sol;
  int32_t* status;
  int32_t* iters;
  int* done_count;  // forward kernel: environments finished so far; done_list[k] = k-th finished environment (-1 = not yet).
  int* done_list;   // gradient kernel: consumes done_list in order while the forward kernel is still running (nullable: all ready)
  double* sol_raw;  // nullable [nres x B]: final solution in DEVICE ordering (written by the forward kernel, read by the gradient kernel)
  double* Fz;  // gradients (GRAD kernels): [12Nb x 12Nb x B], [12Nb x nu x B], column-major per environment
  double* Fu;
  double* Fc;  // nullable: contact-data gradients [12Nb x 5Ni x B] (get_contact_gradients)
  uint32_t flags;
  int* counter;  // dynamic work queue over environments
  const int* order;     // processing order (longest-expected first), or nullptr
  int32_t* prev_iters;  // Newton iterations of the previous call per environment (predicts the cost of the next one)
  const char* plan_blob;  // plan tables, one contiguous blob: [bodies | joints | contacts | steps | sched | ilist | roles | ucol]
  int plan_bytes, plan_off[8];
  int plan_smem_off;    // >= 0: doubles from the start of dynamic shared memory where the CTA keeps its copy of the blob ...
  int plan_smem_bytes;  // ... of which the first plan_smem_bytes bytes are copied (the blob starts with the tables of the serial phases:
  int plan_smem_mask;   // steps, sched, ilist, roles); bit k set: table k lies inside that prefix and is read from shared memory
  int slot_stride;      // doubles between the arenas of two slots of a CTA
  int T;                // time steps fused in this launch (rollouts: every environment is advanced T steps by one CTA)
  double* traj;         // nullable [T][B][nz]: state after every step
  unsigned long long* prof;  // DJ_PROFILE builds: cycle counters [eval_jac, eval_ls, factorize, solve, misc, ...] (layout: tools/time_variant.py)
  // Multi-GPU exchange fused into the step (SURVEY.md 8e, dojo_step_gather_async): besides Zn the epilogue writes every environment's
  // next state straight into the gathered buffer of every rank -- peer-mapped memory (CUDA IPC over NVLink / NVSwitch), this rank's
  // slice starts at gather_off doubles -- and every CTA signals the ranks when its share is out.  n_peers = 0: no exchange.
  int n_peers;
  long long gather_off;
  double* peer_buf[DOJO_MAX_GATHER_RANKS];
  unsigned long long* peer_flag[DOJO_MAX_GATHER_RANKS];
  // traced step (TRACE kernels only, T = 1): [5 x max_iter x B], the rows of mehrotra<true> per environment (dojo_kernels.cuh).  Last
  // member, so that the parameter offsets of every other member, and with them the untraced kernels, do not depend on it.
  double* trace;
  // feedback rollout (FB kernels only, dojo_rollout_feedback): before step t the slot maps the state to minimal coordinates x_t and
  // evaluates u_t = u_ref - K (x_t - x_ref) - K_i xi_t, xi_t = xi_{t-1} + h (x_t - x_ref).  Every array holds fb_steps (1 or T) x
  // fb_envs (1 or B) entries, entry (t, e) at index t * fb_envs + e; K / K_i [nu x 2nu] column-major per entry.  After trace, so that
  // no other member moves.
  const double* fb_K;
  const double* fb_Ki;    // nullable: no integral term
  const double* fb_xref;  // nullable: 0
  const double* fb_uref;  // nullable: 0
  int fb_steps, fb_envs;
  double* fb_x;   // [2nu x B] scratch: x_t of the step the slot is about to solve (global memory, L1/L2-resident)
  double* fb_xi;  // [2nu x B] integral state, updated in place (required iff fb_Ki)
  double* fb_u;   // u_t, where prologue reads it: [nu x B x T] (fb_u_T = 1, the applied inputs) or [nu x B] scratch (fb_u_T = 0)
  int fb_u_T;
};

// feedback stage of the FB kernel for environment e before step t from state z (global memory); returns where u_t was written.
// Lanes: one per joint for the map (max_to_min_joint reads only the joint's parent and child), one per entry of xi, one per input.
DJ_DEV const double* feedback(Ctx& c, const StepArgs& a, const double* z, int e, int t) {
  const Plan& P = *c.P;
  const int nu = P.nu, nx = 2 * nu;
  double* x = a.fb_x + (size_t)e * nx;
  for (int j = c.tid; j < P.Ne; j += c.nthreads) max_to_min_joint(c.joints[j], P.h, z, x);
  __threadfence_block();
  slot_sync(c);
  const size_t q = (size_t)(a.fb_steps > 1 ? t : 0) * a.fb_envs + (a.fb_envs > 1 ? e : 0);
  const double* xr = a.fb_xref ? a.fb_xref + q * nx : nullptr;
  double* xi = a.fb_Ki ? a.fb_xi + (size_t)e * nx : nullptr;
  if (xi) {  // the integral is updated before it is used (pendulum_pid.jl)
    for (int k = c.tid; k < nx; k += c.nthreads) xi[k] += P.h * (xr ? x[k] - xr[k] : x[k]);
    __threadfence_block();
    slot_sync(c);
  }
  const double* K = a.fb_K + q * nu * nx;
  const double* Ki = xi ? a.fb_Ki + q * nu * nx : nullptr;
  double* u = a.fb_u + ((size_t)(a.fb_u_T ? t : 0) * a.B + e) * nu;
  for (int i = c.tid; i < nu; i += c.nthreads) {
    double s = 0.0;
    for (int k = 0; k < nx; ++k) s += K[i + (size_t)nu * k] * (xr ? x[k] - xr[k] : x[k]);
    if (Ki)
      for (int k = 0; k < nx; ++k) s += Ki[i + (size_t)nu * k] * xi[k];
    u[i] = (a.fb_uref ? a.fb_uref[q * nu + i] : 0.0) - s;
  }
  __threadfence_block();
  slot_sync(c);
  return u;
}

// epilogue: update_state! + get_next_state (bodies/set.jl:22-36, mechanism/get.jl:126-134).  The default output is the
// mechanism's state after the step, (x3, v25, q3, w25); DOJO_FLAG_Q1_LITERAL_RETURN reproduces step!'s literal return
// value, which advances the configuration a second time (SURVEY.md Q1).
DJ_DEV void epilogue(Ctx& c, double* __restrict__ zn, bool q1_literal, int n_peers = 0, double* const* peer = nullptr, long long peer_off = 0) {
  const Plan& P = *c.P;
  if (c.tid < P.Nb) {
    Kin k = body_kin(c, c.tid, 0.0);
    V3 x3 = k.x3;
    Quat q3 = k.q3;
    if (q1_literal) { x3 = x3 + P.h * k.v; q3 = qmul(q3, qmap(k.w, P.h)); }
    const double v[13] = {x3.x, x3.y, x3.z, k.v.x, k.v.y, k.v.z, q3.s, q3.x, q3.y, q3.z, k.w.x, k.w.y, k.w.z};
    double* o = zn + 13 * c.tid;
#pragma unroll
    for (int i = 0; i < 13; ++i) o[i] = v[i];
    for (int r = 0; r < n_peers; ++r) {  // posted writes into the peers' gathered buffers (this rank's own copy included)
      double* po = peer[r] + peer_off + 13 * c.tid;
#pragma unroll
      for (int i = 0; i < 13; ++i) po[i] = v[i];
    }
  }
}

// register budget: 65536 / (DJ_LB_THREADS * DJ_LB_BLOCKS) registers per thread
#ifndef DJ_LB_THREADS
#define DJ_LB_THREADS 256
#define DJ_LB_BLOCKS 1
#endif
#ifdef DJ_PROFILE
__device__ __forceinline__ unsigned long long k_t0g(unsigned long long* prof) { return *((volatile unsigned long long*)(prof + 31)); }
#endif
// PLAN_SMEM: the launch keeps its copy of the plan tables in shared memory (a.plan_smem_off >= 0), known at compile time, so that
// every table pointer is derived from the shared-memory array and the table reads compile to LDS with immediate offsets instead of
// generic loads (the generic variant, PLAN_SMEM = false, decides at run time and serves mechanisms whose tables do not fit).
// TRACE (forward only): the traced step of dojo_step_trace, which also records the solver's loop heads into a.trace.  A compile-time
// parameter, so that the untraced instantiations are the same code as without it.
// SMALL (forward, PLAN_SMEM, untraced): the launch guarantees nw = 2, Plan::jpair and Plan::ls_pair, at most 16 nodes in every role
// pass and the whole plan in shared memory (dojo_create: small_step_ok).  The Newton loop then decides from constants what the generic
// kernel reads from the plan -- the warp count in the reductions, the elimination schedule and the assist arithmetic, the paired
// line-search branch, the joint pair -- and the one-lane joint assembly eval_joint<true> is not compiled in.  Same floating-point
// operations in the same order as the generic kernel.
// REC (forward, untraced, generic): the recording rollout of dojo_rollout_grad.  After step t of environment e it keeps what the gradient
// kernel needs at pair p = t * B + e -- the final solution in sol_raw [nres x B x T], status [B x T], iters [B x T] (nullable) -- and
// publishes p on done_list (nullable).  a.traj is slab 1 of the [nz x B x (T + 1)] trajectory whose slab 0 is a.Z, so that pair p
// starts from a.Z + p * nz; Zn is not written.  A compile-time parameter, so that the other instantiations are the same code as without it.
// FB (forward, untraced, generic): the closed-loop rollout of dojo_rollout_feedback.  Before the prologue of step t the slot evaluates the
// linear feedback law on the state the step starts from (feedback() above) and the step reads u_t from a.fb_u; a.U is not read.  The step
// itself is dojo_rollout's.  A compile-time parameter, like REC.
template <bool GRAD, bool PLAN_SMEM = false, bool TRACE = false, bool SMALL = false, bool REC = false, bool FB = false>
__global__ void __launch_bounds__(DJ_LB_THREADS, DJ_LB_BLOCKS) dojo_step_kernel(const StepArgs a) {
  static_assert(!SMALL || (!GRAD && PLAN_SMEM && !TRACE), "SMALL is a specialisation of the untraced forward kernel with the plan in shared memory");
  static_assert(!REC || (!GRAD && !TRACE && !SMALL), "REC is a variant of the generic untraced forward kernel");
  static_assert(!FB || (!GRAD && !TRACE && !SMALL && !REC), "FB is a variant of the generic untraced forward kernel");
  extern __shared__ double arena[];
  __shared__ __align__(8) int s_env[128];  // CTA-wide mailbox, layout: dojo_kernels.cuh (cta_align)
  // a CTA hosts a.slots environments at a time; slot k is served by threads [k * 32 nw, (k + 1) * 32 nw)
  const int slot_threads = 32 * (SMALL ? 2 : a.plan.nw);
  const int slot = threadIdx.x / slot_threads;
  Ctx c;
  c.A = arena + (size_t)slot * a.slot_stride;
  c.P = &a.plan;
  c.tid = threadIdx.x - slot * slot_threads;
  c.nthreads = slot_threads;
  c.warp = c.tid >> 5;
  c.lane = c.tid & 31;
  c.bar = 1 + slot;
  c.sd = 0;
  c.mu = 0.0;
  c.slot = slot; c.nslots = blockDim.x / slot_threads; c.slot_stride = a.slot_stride; c.arena0 = arena;
  c.s_int = s_env; c.s_dbl = reinterpret_cast<double*>(s_env + 32);
  c.apar = 0; c.assist = 0;
  {
    const char* gb = a.plan_blob;
    const char* sb = nullptr;
    if (PLAN_SMEM || a.plan_smem_off >= 0) {  // one copy of the plan tables (or of their hot prefix) per CTA, shared by its slots
      int4* dst = reinterpret_cast<int4*>(arena + a.plan_smem_off);
      const int4* src = reinterpret_cast<const int4*>(a.plan_blob);
#ifndef DJ_HOSTEMU
      // TMA bulk staging: ONE thread issues one asynchronous bulk copy global -> shared (cp.async.bulk, 16-byte aligned on both sides, the
      // blob is padded to 16-byte multiples) that completes on an mbarrier; every thread of the CTA then waits on that barrier's phase 0.
      __shared__ __align__(8) unsigned long long s_plan_bar;
      const unsigned bar = (unsigned)__cvta_generic_to_shared(&s_plan_bar);
      if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // make the initialised barrier visible to the async (TMA) proxy
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        const unsigned bytes = (unsigned)a.plan_smem_bytes;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(bytes), "r"(bar) : "memory");
      }
      {
        unsigned done = 0;
        while (!done)
          asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar) : "memory");
      }
#else
      for (int i = threadIdx.x; i < a.plan_smem_bytes / 16; i += blockDim.x) dst[i] = src[i];
      __syncthreads();
#endif
      sb = reinterpret_cast<const char*>(dst);
    }
#define DJ_TABLE(k) ((PLAN_SMEM || (sb && ((a.plan_smem_mask >> (k)) & 1))) ? sb + a.plan_off[k] : gb + a.plan_off[k])
    c.bodies = reinterpret_cast<const BodyDev*>(DJ_TABLE(0));
    c.joints = reinterpret_cast<const JointDev*>(DJ_TABLE(1));
    c.contacts = reinterpret_cast<const ContactDev*>(DJ_TABLE(2));
    c.steps = reinterpret_cast<const ElimStep*>(DJ_TABLE(3));
    c.sched = reinterpret_cast<const int*>(DJ_TABLE(4));
    c.ilist = reinterpret_cast<const int*>(DJ_TABLE(5));
    c.roles = reinterpret_cast<const WarpRole*>(DJ_TABLE(6));
    c.ucol = reinterpret_cast<const int*>(DJ_TABLE(7));
#undef DJ_TABLE
  }
#ifdef DJ_PROFILE
  c.t_eval_jac = c.t_eval_ls = c.t_fact = c.t_solve = c.t_misc = c.t_align = c.t_cone = c.t_center = c.t_rolewait = 0; c.t_last = clock64();
  c.f_fold = c.f_inv = c.f_rm = c.f_schur = c.f_bar = 0;
  c.s_cond = c.s_fwd = c.s_bwd = c.s_rec = c.s_bar = 0;
  long long k_c0 = clock64(); unsigned long long k_t0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(k_t0));
  int k_envs = 0;
  if (c.tid == 0 && a.prof) atomicMin(a.prof + 31, k_t0);
#endif
  // let a programmatically dependent launch (the gradient kernel of dojo_step_grad) start as soon as every CTA of this
  // grid is running; it synchronises per environment through done_list, not through grid completion
  if (!GRAD) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const Plan& P = a.plan;
  for (;;) {
    if (c.tid == 0) {  // dynamic work queue: iteration counts differ between environments
      int q = atomicAdd(a.counter, 1);
      int env = (q < a.B && a.order) ? a.order[q] : q;
      if (GRAD && a.done_list && q < a.B) {  // wait for the q-th environment the forward kernel finishes
        while ((env = ((volatile int*)a.done_list)[q]) < 0) __nanosleep(256);
        __threadfence();
      }
      s_env[slot] = env;
    }
    slot_sync(c);
    const int e = s_env[slot];
    slot_sync(c);
    if (e >= a.B) break;
    DJ_TICK(c, t_misc)
#ifdef DJ_PROFILE
    k_envs++;
    unsigned long long e_t0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(e_t0));
#endif
    const double* z = a.Z + (size_t)e * P.nz;
    int worst = 0, iters = 0, status = 0;
    if (!GRAD) {
      for (int t = 0; t < a.T; ++t) {
        const double* u = a.U ? a.U + ((size_t)t * a.B + e) * P.nu : nullptr;
        if (FB) u = feedback(c, a, z, e, t);
        const double* fx = a.Fext ? a.Fext + (size_t)e * 6 * P.Nb : nullptr;
        prologue(c, z, u, fx, false);
        status = mehrotra<TRACE, SMALL>(c, a.opts, &iters, TRACE ? a.trace + (size_t)e * max(a.opts.max_iter, 0) * 5 : nullptr);
        worst = max(worst, status);
        // state after this step: the trajectory slot if recorded, else the output buffer (re-read by the next step from L2)
        double* zo = (a.traj ? a.traj + ((size_t)t * a.B + e) * P.nz : a.Zn + (size_t)e * P.nz);
        epilogue(c, zo, (a.flags & DOJO_FLAG_Q1_LITERAL_RETURN) != 0, (t + 1 == a.T) ? a.n_peers : 0, a.peer_buf, a.gather_off + (long long)e * P.nz);
        if (REC) {  // pair t * B + e: its solution, status and iterations, visible before the pair appears in done_list
          const size_t p = (size_t)t * a.B + e;
          for (int k = c.tid; k < P.nres; k += c.nthreads) a.sol_raw[p * P.nres + k] = c.A[P.sol_off + k];
          if (c.tid == 0) {
            a.status[p] = status;
            if (a.iters) a.iters[p] = iters;
          }
          if (a.done_list) {
            __threadfence();
            slot_sync(c);
            if (c.tid == 0) {
              const int pos = atomicAdd(a.done_count, 1);
              __threadfence();
              ((volatile int*)a.done_list)[pos] = (int)p;
            }
          }
        }
        if (t + 1 < a.T) { __threadfence_block(); slot_sync(c); z = zo; }
      }
      if (a.traj && !REC) {  // final state also goes to Zn
        slot_sync(c);
        for (int k = c.tid; k < P.nz; k += c.nthreads) a.Zn[(size_t)e * P.nz + k] = a.traj[((size_t)(a.T - 1) * a.B + e) * P.nz + k];
      }
      status = worst;
      if (a.sol_raw && !REC)
        for (int t = c.tid; t < P.nres; t += c.nthreads) a.sol_raw[(size_t)e * P.nres + t] = c.A[P.sol_off + t];
    } else {
      // gradient pass (get_maximal_gradients!, gradients/state.jl:69-126) at the solution the forward launch left in
      // sol_raw: rebuild the step constants and the KKT blocks of the final iterate, then solve for the columns
      const double* u = a.U ? a.U + (size_t)e * P.nu : nullptr;
      const double* fx = a.Fext ? a.Fext + (size_t)e * 6 * P.Nb : nullptr;
      prologue(c, z, u, fx, true);
      for (int t = c.tid; t < P.nres; t += c.nthreads) c.A[P.sol_off + t] = a.sol_raw[(size_t)e * P.nres + t];
      slot_sync(c);
      double rv, bv;
      c.mu = 0.0;
      evaluate<true>(c, 0.0, P.rhs_off, rv, bv);
      if (a.flags & DOJO_FLAG_Q2_LITERAL_GRADIENTS) {
        // get_maximal_gradients! literally (gradients/state.jl:69-76): step! has already run update_state! (bodies/set.jl:22-36)
        // when the data Jacobian is built -- (x2, q2) <- (x3, q3), (v15, w15) <- (v25, w25) -- while the KKT blocks assembled above
        // (the matrix the reference reads back with full_matrix) belong to the unshifted final iterate (SURVEY.md Q2)
        if (c.tid < P.Nb) {
          const BodyDev& bd = c.bodies[c.tid];
          Kin k = body_kin(c, c.tid, 0.0);
          double* stp = c.A + bd.st_off;
          st3(stp, k.x3);
          stp[3] = k.q3.s; stp[4] = k.q3.x; stp[5] = k.q3.y; stp[6] = k.q3.z;
          st3(c.A + bd.gb_off + 27, k.w);
        }
        slot_sync(c);
      }
      status = a.status ? a.status[e] : 0;
      const size_t ng = 12 * (size_t)P.Nb;
      const double* ug = (a.flags & DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN) ? nullptr : u;
      if (!gradients(c, ug, a.Fz + (size_t)e * ng * ng, a.Fu + (size_t)e * ng * P.nu, a.Fc ? a.Fc + (size_t)e * ng * 5 * P.Ni : nullptr) && status == 0) status = 3;
    }
    if (a.sol) {  // reference ordering: joints [tra eq | s | gamma | rot eq] | bodies | contacts (device layout keeps eq rows first)
      double* so = a.sol + (size_t)e * P.nres;
      const int first_body = c.bodies[0].sol_off;
      for (int t = c.tid; t < P.nres; t += c.nthreads)
        if (t >= first_body) so[t] = c.A[P.sol_off + t];
      if (c.tid < P.Ne) {
        const JointDev& jd = c.joints[c.tid];
        const double* src = c.A + P.sol_off + jd.sol_off;
        double* dst = so + jd.sol_off;
#ifdef DJ_ANY_CONTACT
        if (jd.flags & JF_LIM_TRA) {  // translational limits: reference order [tra s | tra gamma | tra eq | rot eq]
          for (int i = 0; i < 2 * jd.nb_r; ++i) dst[i] = src[jd.ne + i];
          for (int i = 0; i < jd.ne; ++i) dst[2 * jd.nb_r + i] = src[i];
        } else
#endif
        {
        for (int i = 0; i < jd.nl_t; ++i) dst[i] = src[i];
        for (int i = 0; i < 2 * jd.nb_r; ++i) dst[jd.nl_t + i] = src[jd.ne + i];
        for (int i = 0; i < jd.nl_r; ++i) dst[jd.nl_t + 2 * jd.nb_r + i] = src[jd.nl_t + i];
        }
      }
    }
    if (c.tid == 0) {
      if (a.status && !REC) a.status[e] = status;
      if (!GRAD && !REC) {
        if (a.iters) a.iters[e] = iters;
        if (a.prev_iters) a.prev_iters[e] = iters;
      }
#ifdef DJ_PROFILE
      if (a.prof) { unsigned long long e_t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(e_t1)); a.prof[32 + 2 * e] = e_t0 - k_t0g(a.prof); a.prof[33 + 2 * e] = e_t1 - e_t0; }
#endif
    }
    if (!GRAD && !REC && a.done_list) {  // publish: results of this environment are visible before its index appears in the list
      __threadfence();
      slot_sync(c);
      if (c.tid == 0) {
        const int pos = atomicAdd(a.done_count, 1);
        __threadfence();
        ((volatile int*)a.done_list)[pos] = e;
      }
    }
    slot_sync(c);
  }
  for (;;) {  // keep the alignment barrier of the Newton loop matched until every slot has drained
    const AlignInfo ai = cta_align(c, false);
    if (ai.n_live == 0) break;
    // one environment left in this CTA: help its line search (same condition as the owner evaluates in mehrotra())
    if (!GRAD && P.ls_assist && ai.n_live == 1 && a.opts.max_ls <= kMaxAssistTrials) ls_assist_loop<SMALL>(c, a.opts, ai.owner, slot < ai.owner ? slot + 1 : slot);
  }
  if (!GRAD && a.n_peers > 0) {
    // every environment of this CTA has been written to the peers: make the writes visible system-wide, then count this CTA in on
    // every rank (the receiving side waits for all CTAs of all ranks, dojo_gather_wait_kernel).  The barrier above orders the other
    // threads' stores before thread 0's fence (fence cumulativity).
    if (threadIdx.x == 0) {
      __threadfence_system();
      for (int r = 0; r < a.n_peers; ++r) atomicAdd_system(a.peer_flag[r], 1ull);
    }
  }
  // a gradient grid that started early (programmatic dependent launch) does not complete before the forward grid has
  if (GRAD) asm volatile("griddepcontrol.wait;" ::: "memory");
#ifdef DJ_PROFILE
  DJ_TICK(c, t_misc)
  if (c.lane == 0 && a.prof) atomicAdd(a.prof + 17 + c.warp, (unsigned long long)c.t_rolewait);
  if (c.tid == 0 && a.prof) {
    atomicAdd(a.prof + 0, (unsigned long long)c.t_eval_jac); atomicAdd(a.prof + 1, (unsigned long long)c.t_eval_ls);
    atomicAdd(a.prof + 2, (unsigned long long)c.t_fact); atomicAdd(a.prof + 3, (unsigned long long)c.t_solve); atomicAdd(a.prof + 4, (unsigned long long)c.t_misc);
    atomicAdd(a.prof + 5, (unsigned long long)c.f_fold); atomicAdd(a.prof + 6, (unsigned long long)c.f_inv); atomicAdd(a.prof + 7, (unsigned long long)c.f_rm);
    atomicAdd(a.prof + 8, (unsigned long long)c.f_schur); atomicAdd(a.prof + 9, (unsigned long long)c.f_bar);
    // solve(): 25 condense + gather, 26 forward sweep, 27 backward sweep, 28 recover, 29 slot barriers (17 + warp: role waits, nw <= 8)
    atomicAdd(a.prof + 25, (unsigned long long)c.s_cond); atomicAdd(a.prof + 26, (unsigned long long)c.s_fwd); atomicAdd(a.prof + 27, (unsigned long long)c.s_bwd);
    atomicAdd(a.prof + 28, (unsigned long long)c.s_rec); atomicAdd(a.prof + 29, (unsigned long long)c.s_bar);
    unsigned long long k_t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(k_t1));
    atomicMax(a.prof + 10, (unsigned long long)(clock64() - k_c0)); atomicMax(a.prof + 11, k_t1 - k_t0);
    atomicMax(a.prof + 12, (unsigned long long)k_envs); atomicAdd(a.prof + 13, (unsigned long long)(clock64() - k_c0));
    atomicAdd(a.prof + 14, (unsigned long long)c.t_align); atomicAdd(a.prof + 15, (unsigned long long)c.t_cone); atomicAdd(a.prof + 16, (unsigned long long)c.t_center);
  }
#endif
}

// [hostemu:kernel:end]

}  // namespace dj
