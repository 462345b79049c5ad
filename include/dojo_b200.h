/*
 * dojo_b200.h -- C-ABI of the H100-native (sm_90a) batched Dojo step.
 *
 * The reference (dojo-sim/Dojo.jl @ be7b518) has no FFI boundary of its own: it is pure Julia.
 * The drop-in boundary is therefore *defined* here at the level of the Julia methods that enter
 * and leave the per-timestep hot path (SURVEY.md §8b).  Each entry point names the reference
 * method it replaces (file:line relative to the reference repository root):
 *
 *   dojo_create / dojo_destroy   <- Mechanism(origin, bodies, joints, contacts; timestep,
 *                                   input_scaling, gravity)        src/mechanism/constructor.jl:46-84
 *                                   (the live Julia Mechanism is flattened into DojoMechanismDesc)
 *   dojo_step                    <- step!(mechanism, z, u; opts)   src/simulation/step.jl:11-30
 *                                   = set_maximal_state! (src/mechanism/set.jl:10-26)
 *                                   + set_input!          (src/mechanism/set.jl:40-53)
 *                                   + mehrotra!           (src/solver/mehrotra.jl:9-73)
 *                                   + update_state!       (src/bodies/set.jl:22-36)
 *                                   + get_next_state      (src/mechanism/get.jl:126-134)
 *   dojo_step_grad               <- get_maximal_gradients!(mechanism, z, u; opts)
 *                                                                  src/gradients/state.jl:69-126
 *   dojo_rollout                 <- simulate!(mechanism, steps, storage, control!)
 *                                                                  src/simulation/simulate.jl:16-36
 *   dojo_rollout_feedback        <- simulate!(mechanism, steps, storage, controller!) with a controller! that reads
 *                                   get_minimal_state and applies a time-varying linear law (examples/control)
 *   dojo_rollout_grad            <- simulate! + get_maximal_gradients! at every step
 *   dojo_rollout_minimal_gradients <- simulate! + get_minimal_gradients! at every step
 *   dojo_rollout_tape + dojo_rollout_vjp <- simulate! + get_maximal_gradients! at every step, contracted with a loss gradient
 *                                   (the vector-Jacobian product, without the Jacobians)
 *   dojo_rollout_feedback_tape + dojo_rollout_feedback_vjp <- the same through dojo_rollout_feedback's closed loop, with the
 *                                   gradients of the law's gains and references (pendulum_pid.jl's gains tuned by gradient)
 *   dojo_lqr_backward            <- the backward pass of IterativeLQR.jl's solve! (iLQR / TVLQR gains
 *                                   from the minimal-coordinate Jacobians and a quadratic cost;
 *                                   docs/src/examples/trajectory_optimization.md)
 *   DojoSolverOptions            <- SolverOptions{T}               src/solver/options.jl:16-26
 *   dojo_minimal_to_maximal      <- minimal_to_maximal(mechanism, x) src/mechanism/state.jl:9-22
 *                                   (set_minimal_coordinates_velocities!, src/joints/minimal.jl:148-203)
 *   dojo_maximal_to_minimal      <- maximal_to_minimal(mechanism, z) src/mechanism/state.jl:44-66
 *   dojo_step_minimal            <- step_minimal_coordinates!(mechanism, x, u; opts)
 *                                                                  src/simulation/step.jl:42-61
 *
 * All arrays are fp64.  Batched arrays are column-major [feature x B] exactly as a Julia
 * Matrix{Float64}(feature, B) is laid out, i.e. environment e owns the contiguous slice
 * [e*feature, (e+1)*feature).  Per body the maximal state is packed as the reference packs it
 * (src/mechanism/get.jl:107-134): [x2(3) v15(3) q2(s,v1,v2,v3) w15(3)].
 * Gradients use the 12-per-body attitude-reduced packing [x(3) v(3) phi(3) w(3)]
 * (src/gradients/state.jl:102-123), column-major [12Nb x 12Nb] and [12Nb x nu] per environment.
 *
 * Buffers passed to the synchronous entries (dojo_step, dojo_step_grad, dojo_rollout, ...) may be
 * HOST or DEVICE pointers, all of one call of the same kind (detected with cudaPointerGetAttributes
 * on the first array); host buffers are copied inside the call.  dojo_step / dojo_step_trace stage
 * pageable buffers through the handle's pinned memory; every other entry copies directly from / to
 * the caller's buffers, through one grow-only device staging arena per handle.  The *_async variants
 * take device pointers only and a cudaStream_t (passed as void*), do not synchronise, and are what a
 * resident-data caller uses.
 *
 * Threading / streams: a handle is not thread-safe (the reference's Mechanism is single-threaded and mutable as well) and
 * has ONE call in flight at a time: the work-queue counter, completion lists, staging and scratch buffers belong to the
 * handle.  Calls issued on different streams (or an *_async call followed by a synchronous one, which runs on the
 * handle's own stream) are therefore ordered behind each other by the library (an event wait on the later stream);
 * use one handle per stream for concurrent batches.
 *
 * Return value: 0 on success, negative DOJO_E* on API misuse / CUDA failure (message via
 * dojo_last_error).  Per-environment solver outcomes never abort the batch; they are reported in
 * status[B]: 0 success, 1 :failed (max_iter reached, src/solver/mehrotra.jl:13,30,72),
 * 2 excessive angular velocity (reserved: the reference throws at src/solver/line_search.jl:18-20, but its test
 *   |w|^2 > 3.91/h^2 comes after candidate_step! has clipped |w|^2 > 3.9/h^2 down to (3.9/h^2)^2/|w|^2 < 3.9/h^2
 *   (src/solver/line_search.jl:141-152), so the branch is unreachable in the reference and no path here produces it),
 * 3 non-finite iterate.
 */
#ifndef DOJO_B200_H
#define DOJO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DOJO_OK 0
#define DOJO_EINVAL (-1)      /* bad argument / unsupported mechanism */
#define DOJO_ECUDA (-2)       /* CUDA runtime failure */
#define DOJO_ENOMEM (-3)      /* mechanism does not fit the per-environment shared-memory budget */
#define DOJO_ENODEVICE (-4)   /* no CUDA device: there is NO CPU fallback in this library */

#define DOJO_STATUS_SUCCESS 0
#define DOJO_STATUS_FAILED 1
#define DOJO_STATUS_EXCESSIVE_OMEGA 2
#define DOJO_STATUS_NONFINITE 3

/* flags */
#define DOJO_FLAG_Q1_LITERAL_RETURN 1u /* reproduce step!'s double-advanced return value (SURVEY Q1) */
/* dojo_step_grad*: reproduce what get_maximal_gradients!(mechanism, z, u) literally returns (SURVEY Q2,
 * src/gradients/state.jl:69-76): step! shifts the state (update_state!, src/bodies/set.jl:22-36: x2 <- x3, q2 <- q3,
 * v15 <- v25, w15 <- w25, input impulses cleared) BEFORE get_maximal_gradients builds the data Jacobian and the
 * integrator chain rule, while `full_matrix(mechanism.system)` still holds the KKT entries of the unshifted final
 * iterate (src/solver/mehrotra.jl:66-69).  Without the flag the consistent implicit-function-theorem gradient is
 * returned (data Jacobian and KKT matrix at the same state), which is what test/data.jl and the documentation pin. */
#define DOJO_FLAG_Q2_LITERAL_GRADIENTS 2u
/* dojo_step_grad*: leave d(input impulse)/d(x2, q2) out of the data Jacobian, as the
 * reference's src/gradients/data.jl does (SURVEY Q17: input_jacobian_configuration of src/joints/{translational,rotational}/
 * input.jl is defined but never called).  Without the flag, Fz is the derivative of the step the library computes, also at
 * nonzero inputs when an actuated joint has a free parent.  Orthogonal to Q2: get_maximal_gradients! literally is Q2 | Q17. */
#define DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN 4u

/* Body: src/bodies/constructor.jl:13-27 (mass, inertia) */
typedef struct {
  double mass;
  double inertia[9]; /* row-major 3x3, body frame */
} DojoBodyDesc;

/* One half of a JointConstraint: Translational / Rotational
 * (src/joints/translational/constructor.jl:19-31, src/joints/rotational/constructor.jl:19-31). */
typedef struct {
  int32_t nlambda;         /* N_lambda: number of constrained axes, 0..3 */
  int32_t nlimits;         /* Nb/2: 0, or 3-nlambda when every free axis is limited (joints/limits.jl) */
  double axis_mask[9];     /* rows V1,V2,V3 (joints/orthogonal.jl:1-12); masks per joints/joint.jl:56-64 */
  double spring, damper;   /* act on the free axes (src/joints/{translational,rotational}/{springs,dampers}.jl); the reference's
                            * set_springs! / set_dampers! (DojoEnvironments/src/utilities.jl:1-39) skip a floating base */
  double spring_offset[3]; /* first 3-nlambda entries used */
  double limit_lo[3], limit_hi[3];
} DojoJointElementDesc;

/* JointConstraint: src/joints/constraints.jl:17-86 */
typedef struct {
  int32_t parent_body;          /* 0-based body index, -1 = origin */
  int32_t child_body;           /* 0-based body index */
  double vertex_parent[3];      /* translational.vertices[1], parent frame */
  double vertex_child[3];       /* translational.vertices[2], child frame */
  double orientation_offset[4]; /* rotational.orientation_offset (s,v1,v2,v3) */
  DojoJointElementDesc tra, rot;
} DojoJointDesc;

/* ContactConstraint{model} + SphereHalfSpaceCollision (src/contacts/constructor.jl:14-43,
 * src/contacts/collisions/sphere_halfspace.jl:11-24); the model is the reference's `contact_type`
 * (src/contacts/constructor.jl:117-128):
 *   2 NonlinearContact{T,8}  second-order friction cone        src/contacts/nonlinear.jl:12-97
 *   1 LinearContact{T,12}    4-sided friction pyramid          src/contacts/linear.jl:10-104
 *   0 ImpactContact{T,2}     no friction (friction_coefficient, tangent unused)  src/contacts/impact.jl:8-146
 * The contact's entry in solution / residual vectors is [s(N/2); gamma(N/2)].  Mechanisms whose contacts are all of type 2
 * (every BASELINE model) run on the benchmarked kernels; any type 0 / 1 contact selects a second compilation of the same
 * kernels with the two orthant models enabled (csrc/dojo_b200_cm.cu).  dojo_step_grad_contact is defined for type 2 only,
 * like the reference's contact-data blocks (src/gradients/data.jl:152, :173). */
typedef struct {
  int32_t type;        /* 0 impact, 1 linear, 2 nonlinear */
  int32_t parent_body; /* 0-based body index; child is always the origin half-space */
  double friction_coefficient;
  double tangent[6];   /* contact_tangent, row-major 2x3 */
  double normal[3];    /* contact_normal */
  double origin[3];    /* contact_origin (body frame) */
  double radius;       /* contact_radius */
  double offset[3];    /* contact_offset */
} DojoContactDesc;

/* Flattened Mechanism.  Node ids follow the reference (src/mechanism/id.jl:5-13):
 * joints 1..Ne, bodies Ne+1..Ne+Nb, contacts after; solution/residual vectors are ordered
 * joints | bodies [v25;w25] | contacts [s;gamma] (src/gradients/finite_difference.jl:1-18).
 * Inputs u are ordered by joint, [tra free axes; rot free axes] each (src/mechanism/set.jl:40-53). */
typedef struct {
  int32_t num_bodies, num_joints, num_contacts;
  double timestep, input_scaling, gravity[3];
  const DojoBodyDesc* bodies;
  const DojoJointDesc* joints;
  const DojoContactDesc* contacts;
} DojoMechanismDesc;

/* SolverOptions: src/solver/options.jl:16-26 (ls_scale is carried but, as in the reference, never read) */
typedef struct {
  double rtol, btol, ls_scale;
  int32_t max_iter, max_ls;
  double undercut;
  int32_t no_progress_max;
  double no_progress_undercut;
  int32_t verbose;
} DojoSolverOptions;

typedef struct DojoHandle DojoHandle;

void dojo_default_options(DojoSolverOptions* opts);

/* device: CUDA device ordinal (>= 0).  max_batch: largest B that will be passed. */
int dojo_create(const DojoMechanismDesc* desc, int device, int max_batch, DojoHandle** out);
int dojo_destroy(DojoHandle* h);
const char* dojo_last_error(const DojoHandle* h); /* h may be NULL: last create error */

/* Parameter update for system identification (examples/system_identification/utilities.jl:41-87 rebuilds the data of a live
 * Mechanism between solves): same topology (bodies, joints, joint types, limits, contacts), new numbers (masses, inertias,
 * vertices, offsets, springs, dampers, limit values, friction coefficients, contact radii / origins, timestep, gravity,
 * input scaling).  The plan tables are rebuilt and swapped in place; device buffers, streams and max_batch are kept.
 * Returns DOJO_EINVAL if the topology differs.  Synchronises the handle's stream. */
int dojo_update_params(DojoHandle* h, const DojoMechanismDesc* desc);

/* sizes derived from the descriptor */
int dojo_num_state(const DojoHandle* h);    /* 13 Nb */
int dojo_num_input(const DojoHandle* h);    /* nu */
int dojo_num_residual(const DojoHandle* h); /* Nres */
int dojo_num_grad_state(const DojoHandle* h); /* 12 Nb */
int dojo_shared_bytes_per_env(const DojoHandle* h);

/* One step! for B environments.  Z [13Nb x B], U [nu x B], Fext nullable [6Nb x B]
 * ([F(3); tau(3)] per body: State.Fext / State.τext), Z_next [13Nb x B],
 * sol nullable [Nres x B] (final solution: joint impulses | v25,w25 | s,gamma),
 * status [B], iters [B] (Newton iterations taken), both nullable. */
int dojo_step(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U,
              const double* Fext, double* Z_next, double* sol, int32_t* status, int32_t* iters,
              uint32_t flags);
int dojo_step_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ,
                    const double* dU, const double* dFext, double* dZ_next, double* dsol,
                    int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream);

/* Traced step!: dojo_step, and the per-iteration record of the interior-point solver that the reference prints with
 * SolverOptions(verbose = true) (src/solver/mehrotra.jl:26-31, 75-98).  Every other argument means what it means for
 * dojo_step / dojo_step_async, and the outputs are bit-identical to theirs.  trace is required: [5 x max_iter x B],
 * environment e's row r at trace[(e * max_iter + r) * 5 + k].  Row r describes the loop head of Newton iteration r + 1:
 *   k = 0  rvio    residual violation tested at this head
 *   k = 1  bvio    bilinear violation tested at this head
 *   k = 2  alpha   the corrected direction's cone-line-search step of the previous iteration (1 in row 0)
 *   k = 3  mu      mutarget of the previous iteration (0 in row 0)
 *   k = 4  trials  line-search trials the previous iteration evaluated up to and including the accepted one (0 in row 0);
 *                  the step taken was alpha / 2^(trials - 1)
 * (alpha and mu at a head belong to the iteration before it, as in the reference's printout).  Rows written: n when the
 * solve converged at head n (iters = n - 1), max_iter when it ended :failed, the heads actually reached when it ended
 * non-finite; the remaining rows are NaN.  The traced kernel is a separate compilation of the same solver loop: the
 * untraced entry points do not pay for it. */
int dojo_step_trace(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U,
                    const double* Fext, double* Z_next, double* sol, int32_t* status, int32_t* iters,
                    double* trace, uint32_t flags);
int dojo_step_trace_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ,
                          const double* dU, const double* dFext, double* dZ_next, double* dsol,
                          int32_t* dstatus, int32_t* diters, double* dtrace, uint32_t flags,
                          void* cuda_stream);

/* step! + consistent IFT gradients at the solution (SURVEY Q2: get_maximal_gradients evaluated
 * right after mehrotra!, before update_state!).  dFz [12Nb x 12Nb x B], dFu [12Nb x nu x B].
 * Two launches on the stream: the forward kernel, then the gradient kernel, which starts on the SMs the
 * forward kernel's tail leaves idle and consumes environments in completion order.  B <= max_batch;
 * the output state buffer must not alias the input state (the gradient kernel re-reads Z). */
int dojo_step_grad(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z,
                   const double* U, const double* Fext, double* Z_next, double* Fz, double* Fu,
                   int32_t* status, int32_t* iters, uint32_t flags);
int dojo_step_grad_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ,
                         const double* dU, const double* dFext, double* dZ_next, double* dFz,
                         double* dFu, int32_t* dstatus, int32_t* diters, uint32_t flags,
                         void* cuda_stream);

/* ---- Multi-GPU: environments shard over the GPUs of a box, one process + one handle per GPU (SURVEY.md 8e) -------------------------
 * The reference is single-process; BASELINE.json's north_star asks for ONE exchange per step: every rank receives the next states
 * of the whole batch.  It is fused into the step kernel: each environment's next state is written, as soon as it is solved, straight
 * into the gathered buffer of every rank (peer memory mapped through CUDA IPC: NVLink / NVSwitch posted writes), so the exchange
 * overlaps the solve and its tail instead of following the kernel as a collective.  No NCCL is involved; a Julia host binds these
 * like every other entry point (INTEGRATION.md).
 *   dojo_gather_create   allocates this rank's gathered buffer [13Nb x B_local x world] (rank r's slice at r * B_local) + a counter
 *   dojo_gather_export   the 128-byte IPC descriptor of this rank (exchange them with any host-side all-gather: MPI, torch.distributed ...)
 *   dojo_gather_connect  maps the buffers of all ranks (descriptors in rank order, world x 128 bytes)
 *   dojo_step_gather_async / dojo_step_grad_gather_async
 *                        dojo_step_async / dojo_step_grad_async + the exchange; on return of the stream work the gathered buffer of THIS
 *                        rank holds the next states of all ranks (a small wait kernel closes the step: it returns once every CTA of
 *                        every rank has signalled; it gives up after ~10 s and reports DOJO_STATUS_NONFINITE in status[0] if a peer died)
 *   dojo_gather_buffer   the gathered states of the MOST RECENT step call.  The buffer has two halves that consecutive steps use
 *                        alternately (a fast rank may already be writing step t + 1 into its peers while a slow rank still reads
 *                        step t): call it after every step; work that reads it must be issued on the step's stream before the next
 *                        step call, and the states of step t stay valid until step t + 2 is issued.
 * All ranks must call with the same B_local and the same sequence of steps. */
#define DOJO_MAX_GATHER_RANKS 8
#define DOJO_GATHER_HANDLE_BYTES 128
typedef struct DojoGather DojoGather;
int dojo_gather_create(DojoHandle* h, int world, int rank, int B_local, DojoGather** out);
int dojo_gather_export(DojoGather* g, void* handle_out /* DOJO_GATHER_HANDLE_BYTES */);
int dojo_gather_connect(DojoGather* g, const void* all_handles /* world x DOJO_GATHER_HANDLE_BYTES, rank order */);
double* dojo_gather_buffer(DojoGather* g); /* device pointer, [13Nb x (world * B_local)] */
int dojo_gather_destroy(DojoGather* g);
int dojo_step_gather_async(DojoHandle* h, DojoGather* g, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU,
                           const double* dFext, double* dZ_next, int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream);
int dojo_step_grad_gather_async(DojoHandle* h, DojoGather* g, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU,
                                const double* dFext, double* dZ_next, double* dFz, double* dFu, int32_t* dstatus, int32_t* diters,
                                uint32_t flags, void* cuda_stream);

/* get_contact_gradients(mechanism) (src/gradients/contact.jl:1-55; data blocks src/gradients/data.jl:152-192): step! and the
 * gradients with respect to the contact data theta_c = [friction_coefficient; contact_radius; contact_origin(3)] of every
 * contact, next to the state / control gradients (the reference returns jacobian_state with jacobian_contact):
 *   Fc [12Nb x 5Ni x B] column-major per environment, columns ordered by contact.
 * The extra 5 Ni columns are solved against the same block-LDU factor in the gradient kernel.  Used with dojo_update_params for
 * system identification (examples/system_identification/utilities.jl:41-87). */
int dojo_num_contact_data(const DojoHandle* h); /* 5 Ni */
int dojo_step_grad_contact(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, double* Z_next,
                           double* Fz, double* Fu, double* Fc, int32_t* status, int32_t* iters);
int dojo_step_grad_contact_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU,
                                 const double* dFext, double* dZ_next, double* dFz, double* dFu, double* dFc,
                                 int32_t* dstatus, int32_t* diters, uint32_t flags, void* cuda_stream);

/* simulate!: T steps with the state resident on the device.  U is [nu x B x T] (step-major) or
 * NULL (zero input); Z_traj nullable [13Nb x B x T] receives the state after every step
 * (Storage, src/simulation/storage.jl:15-42); Z_final [13Nb x B]; status_any [B] = max status.
 * The T steps are fused in ONE kernel launch: the CTA that dequeues an environment advances it through all steps. */
int dojo_rollout(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0,
                 const double* U, double* Z_final, double* Z_traj, int32_t* status_any);

/* device-pointer variant of dojo_rollout: one launch, no synchronisation */
int dojo_rollout_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0,
                       const double* dU, double* dZ_final, double* dZ_traj, int32_t* dstatus_any,
                       void* cuda_stream);

/* Closed-loop rollout: simulate! with a controller! that reads the minimal state at every step and sets a time-varying affine
 * law (examples/control: pendulum_pid.jl, cartpole_lqr.jl; the forward pass of iLQR / DDP / TVLQR).  In the ONE launch of
 * dojo_rollout, before step t of every environment:
 *   x_t  = maximal_to_minimal(z_t)                           (per joint [c_tra; c_rot; v_tra; v_rot], as dojo_maximal_to_minimal)
 *   xi_t = xi_{t-1} + h (x_t - x_ref_t)                      (only with K_i; xi_{-1} = the caller's xi, updated before use)
 *   u_t  = u_ref_t - K_t (x_t - x_ref_t) - K_i,t xi_t
 *   z_{t+1} = step(z_t, u_t)                                 (dojo_rollout's step, bit for bit)
 * Every array of DojoFeedback holds `steps` (1 or T) x `envs` (1 or B) entries, entry (t, e) at t * envs + e: one for all steps or
 * one per step, one for all environments or one per environment.  K and K_i are column-major [nu x 2nu] per entry. */
typedef struct {
  int32_t steps, envs;   /* 1 or T / 1 or B */
  const double* K;       /* [nu x 2nu x envs x steps], required */
  const double* K_i;     /* same shape, nullable: no integral term */
  const double* x_ref;   /* [2nu x envs x steps], nullable: 0 */
  const double* u_ref;   /* [nu x envs x steps], nullable: 0 */
} DojoFeedback;
/* xi [2nu x B]: integral state, in/out (required iff K_i; after the call it holds xi_{T-1}, so that a second call continues it);
 * Z_final [13Nb x B], Z_traj nullable [13Nb x B x T] and status_any [B] as dojo_rollout; U_applied nullable [nu x B x T]: u_t of every
 * step -- dojo_rollout or dojo_rollout_grad driven by it reproduce the trajectory bit for bit.  Host or device pointers (all of one
 * kind; host buffers are staged through grow-only handle buffers); *_async: device pointers, no synchronisation.
 * DOJO_EINVAL, before anything is launched, unless B in 1..max_batch, T >= 1, fb and K given, steps in {1, T}, envs in {1, B},
 * xi given with K_i, and nu > 0.  Flags, external forces and the Q1 literal return are single-step features. */
int dojo_rollout_feedback(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const DojoFeedback* fb,
                          double* xi, double* Z_final, double* Z_traj, double* U_applied, int32_t* status_any);
int dojo_rollout_feedback_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const DojoFeedback* fb,
                                double* dxi, double* dZ_final, double* dZ_traj, double* dU_applied, int32_t* dstatus_any,
                                void* cuda_stream);

/* Riccati backward pass of time-varying LQR / iLQR in minimal coordinates, batched: one launch for all B environments and T steps.
 * Cost per environment:  sum_t 1/2 (x_t - xg_t)' Q_t (x_t - xg_t) + 1/2 (u_t - ug_t)' R_t (u_t - ug_t)  +  1/2 (x_T - xg_T)' Q_f (x_T - xg_T).
 * From the nominal trajectory (X_traj, U) and its Jacobians A_t = Gx[t, e], B_t = Gu[t, e] (the layouts dojo_rollout_minimal_gradients
 * writes), for t = T-1 ... 0 with P_T = Q_f, p_T = Q_f (x_T - xg_T):
 *   Qx = Q_t dx_t + A'p   Qu = R_t du_t + B'p   Qxx = Q_t + A'PA   Quu = R_t + B'PB   Qux = B'PA   (dx = x_t - xg_t, du = u_t - ug_t)
 *   K_t = (Quu + mu_e I)^-1 Qux,   k_t = -(Quu + mu_e I)^-1 Qu          (Cholesky; on the active inputs only)
 *   P = Qxx + K'Quu K - K'Qux - Qux'K (symmetrised),   p = Qx - K'Quu k - K'Qu + Qux'k,   dV += [k'Qu, 1/2 k'Quu k]
 * (the P, p and dV updates use Quu without mu, as Tassa, Erez and Todorov 2012).  The forward law is u = u_bar + alpha k - K (x - x_bar):
 * DojoFeedback with K, x_ref = X_traj, u_ref = U + alpha k, so K goes to dojo_rollout_feedback unchanged.
 * Every array of DojoQuadraticCost holds `steps` (1 or T) x `envs` (1 or B) entries, entry (t, e) at t * envs + e, as DojoFeedback;
 * Q_final and x_goal_final hold `envs` entries.  Matrices are column-major. */
typedef struct {
  int32_t steps, envs;          /* 1 or T / 1 or B */
  const double* Q;              /* [2nu x 2nu x envs x steps], required */
  const double* R;              /* [nu x nu x envs x steps], required */
  const double* x_goal;         /* [2nu x envs x steps], nullable: 0 */
  const double* u_goal;         /* [nu x envs x steps], nullable: 0 */
  const double* Q_final;        /* [2nu x 2nu x envs], required */
  const double* x_goal_final;   /* [2nu x envs], nullable: 0 */
} DojoQuadraticCost;
/* active [nu] (HOST array, nullable = all active): inputs with active = 0 (a floating base, an unactuated joint) get a zero row in K and
 * a zero k, and Quu is factored on the active inputs only.  X_traj [2nu x B x (T+1)], U [nu x B x T] (nullable: 0), Gx [2nu x 2nu x B x T],
 * Gu [2nu x nu x B x T], pair (t, e) at t * B + e.  mu [B] nullable: 0.  Outputs K [nu x 2nu x B x T] (= DojoFeedback.K with
 * envs = B, steps = T), k [nu x B x T], dV [2 x B] nullable (the expected decrease alpha dV[0] + alpha^2 dV[1]), status [B] nullable:
 * 0, or t + 1 when the Cholesky of Quu + mu I failed at step t -- then that environment's K_s and k_s for s <= t and its dV are NaN,
 * and every other environment is unaffected.  Raise mu for it and call again.
 * Host or device pointers (all of one kind; host buffers are staged through grow-only handle buffers); *_async: device pointers, no
 * synchronisation.  DOJO_EINVAL, before anything is launched, unless B in 1..max_batch, T >= 1, cost / Q / R / Q_final / X_traj / Gx /
 * Gu / K / k given, steps in {1, T}, envs in {1, B}, nu > 0 and `active`, if given, has a nonzero entry.  DOJO_ENOMEM when the working
 * set of one environment (about 19 nu^2 doubles) exceeds the device's shared memory per block (nu <= 38 on H100). */
int dojo_lqr_backward(DojoHandle* h, int B, int T, const DojoQuadraticCost* cost, const int32_t* active, const double* X_traj,
                      const double* U, const double* Gx, const double* Gu, const double* mu, double* K, double* k, double* dV,
                      int32_t* status);
int dojo_lqr_backward_async(DojoHandle* h, int B, int T, const DojoQuadraticCost* cost, const int32_t* active, const double* dX_traj,
                            const double* dU, const double* dGx, const double* dGu, const double* dmu, double* dK, double* dk, double* ddV,
                            int32_t* dstatus, void* cuda_stream);

/* Minimal <-> maximal coordinate maps (the step either side of step! for every DojoEnvironments call).
 * Minimal state x = per joint, in joint order, [c_tra; c_rot; v_tra; v_rot] (2 * input_dimension(joint) entries:
 * coordinates along the free translational / rotational axes and their finite-difference velocities);
 * X is [2 nu x B].  Host or device pointers (both of the same kind); *_async: device pointers, no synchronisation. */
int dojo_num_minimal(const DojoHandle* h); /* 2 nu */
int dojo_minimal_to_maximal(DojoHandle* h, int B, const double* X, double* Z);
int dojo_maximal_to_minimal(DojoHandle* h, int B, const double* Z, double* X);
int dojo_minimal_to_maximal_async(DojoHandle* h, int B, const double* dX, double* dZ, void* cuda_stream);
int dojo_maximal_to_minimal_async(DojoHandle* h, int B, const double* dZ, double* dX, void* cuda_stream);

/* step_minimal_coordinates!: minimal -> maximal, step!, maximal -> minimal in three launches on one stream; the maximal
 * states never leave the device.  X [2 nu x B], U [nu x B] (nullable), X_next [2 nu x B]; host or device pointers. */
int dojo_step_minimal(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U,
                      double* X_next, int32_t* status, int32_t* iters);
/* the same with `flags`: DOJO_FLAG_Q1_LITERAL_RETURN maps step!'s LITERAL return value (configuration advanced a second time, SURVEY.md Q1)
 * to minimal coordinates -- what step_minimal_coordinates! of the reference returns, src/simulation/step.jl:42-61 -- instead of the
 * mechanism's state after the step */
int dojo_step_minimal_flags(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U,
                            double* X_next, int32_t* status, int32_t* iters, uint32_t flags);

/* Jacobians of the coordinate maps in attitude-reduced maximal coordinates ([x, v, phi, w] per body, 12 Nb):
 *   dojo_maximal_to_minimal_jacobian   maximal_to_minimal_jacobian(mechanism, z)   src/gradients/state.jl:9-56
 *       J [2 nu x 12 Nb x B] column-major per environment, evaluated at Z [13 Nb x B];
 *   dojo_minimal_to_maximal_jacobian   minimal_to_maximal_jacobian(mechanism, x)   src/gradients/state.jl:136-179
 *       J [12 Nb x 2 nu x B], evaluated at the MAXIMAL state Z (the reference reads the mechanism's stored state; pass
 *       Z = minimal_to_maximal(X)).  The partials are chained root -> leaves, i.e. J is the derivative of
 *       minimal_to_maximal; the reference chains in mechanism.bodies order, which is the same thing whenever parents
 *       precede their children in that list.
 * Host or device pointers (both of the same kind); *_async: device pointers, no synchronisation. */
int dojo_maximal_to_minimal_jacobian(DojoHandle* h, int B, const double* Z, double* J);
int dojo_minimal_to_maximal_jacobian(DojoHandle* h, int B, const double* Z, double* J);
int dojo_maximal_to_minimal_jacobian_async(DojoHandle* h, int B, const double* dZ, double* dJ, void* cuda_stream);
int dojo_minimal_to_maximal_jacobian_async(DojoHandle* h, int B, const double* dZ, double* dJ, void* cuda_stream);

/* Adjoints (vector-Jacobian products) of the two maps, without forming the Jacobians above:
 *   dojo_maximal_to_minimal_vjp   gZ = M(z)' gX   gX [2 nu x n] -> gZ [12 Nb x n]
 *   dojo_minimal_to_maximal_vjp   gX = N(z)' gZ   gZ [12 Nb x n] -> gX [2 nu x n]
 * Z [13 Nb x n] is the maximal state; for dojo_minimal_to_maximal_vjp it is minimal_to_maximal(X), as for
 * dojo_minimal_to_maximal_jacobian.  gZ is in the gradients' packing [x, v, phi, w] per body.  The output is overwritten, not
 * accumulated.  n counts states, not environments, and is not bounded by max_batch: a trajectory [.. x B x (T+1)] goes in one call
 * with n = B (T+1).  Each state's result is one fixed-order sum per entry: it does not depend on n or on the other states.
 * Reverse mode through a rollout in minimal coordinates composes these with the rollout tape and adjoint (INTEGRATION.md):
 *   z0 = minimal_to_maximal(X0), tape, gZ[t] = M(z_t)' gX[t], dojo_rollout_vjp, gX0 = N(z0)' gZ0.
 * DOJO_EINVAL, before anything is launched, for n <= 0, a null buffer or a mechanism without inputs (nu = 0).
 * Host or device pointers (all of the same kind); *_async: device pointers, no synchronisation. */
int dojo_maximal_to_minimal_vjp(DojoHandle* h, int n, const double* Z, const double* gX, double* gZ);
int dojo_maximal_to_minimal_vjp_async(DojoHandle* h, int n, const double* dZ, const double* dgX, double* dgZ, void* cuda_stream);
int dojo_minimal_to_maximal_vjp(DojoHandle* h, int n, const double* Z, const double* gZ, double* gX);
int dojo_minimal_to_maximal_vjp_async(DojoHandle* h, int n, const double* dZ, const double* dgZ, double* dgX, void* cuda_stream);

/* get_minimal_gradients!(mechanism, x, u; opts)  src/gradients/state.jl:182-217: step_minimal_coordinates! and
 *   Gx = M(z') Fz N(z) [2 nu x 2 nu x B],  Gu = M(z') Fu [2 nu x nu x B]   (column-major per environment),
 * with z = minimal_to_maximal(x), (z', Fz, Fu) = dojo_step_grad(z, u) (consistent IFT, SURVEY Q2), M / N the two map
 * Jacobians above.  The maximal states and the 12Nb x 12Nb Jacobians never leave the device (processed in chunks).
 * X [2 nu x B], U [nu x B] (nullable), X_next [2 nu x B]; status / iters nullable; host or device pointers. */
int dojo_minimal_gradients(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* X, const double* U,
                           double* X_next, double* Gx, double* Gu, int32_t* status, int32_t* iters);

/* Trajectory Jacobians: simulate! (src/simulation/simulate.jl:16-36) + get_maximal_gradients! (src/gradients/state.jl:69-126)
 * at every step, i.e. (dz_{t+1}/dz_t, dz_{t+1}/du_t) for t = 0 .. T-1, the Jacobians of dojo_step_grad (consistent IFT, SURVEY Q2)
 * at the states of the fused rollout of dojo_rollout.  Pair (e, t) is at index t*B + e.
 *   Z_traj [13Nb x B x (T+1)]: slab 0 = Z0 on return, slab t+1 = state after step t (slab T = final state);
 *   Fz [12Nb x 12Nb x B x T], Fu [12Nb x nu x B x T], column-major per pair as dojo_step_grad;
 *   U [nu x B x T] nullable (zero input); status / iters [B x T] nullable: status and Newton iterations of every step.
 * B in 1..max_batch, T >= 1 (DOJO_EINVAL otherwise); DOJO_ENOMEM when the gradient workspace does not fit (as dojo_step_grad).
 * dojo_rollout_grad: host or device pointers (all of the same kind); host Jacobians are computed and copied in chunks of pairs.
 * dojo_rollout_grad_async: device pointers, no synchronisation; the gradients of early steps are computed while later steps are
 * still being solved.  Z_traj may hold Z0 in slab 0 already (dZ0 == dZ_traj). */
int dojo_rollout_grad(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U,
                      double* Z_traj, double* Fz, double* Fu, int32_t* status, int32_t* iters);
int dojo_rollout_grad_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU,
                            double* dZ_traj, double* dFz, double* dFu, int32_t* dstatus, int32_t* diters, void* cuda_stream);
/* The same in minimal coordinates: simulate! + get_minimal_gradients! (src/gradients/state.jl:182-217) at every step.  The rollout
 * runs in maximal coordinates from minimal_to_maximal(X0); X_traj [2nu x B x (T+1)] is maximal_to_minimal of its T + 1 slabs,
 * Gx [2nu x 2nu x B x T] = M(z_{t+1}) Fz N(z_t), Gu [2nu x nu x B x T] = M(z_{t+1}) Fu per pair (as dojo_minimal_gradients, whose
 * maximal states never leave the device).  Host or device pointers (all of the same kind). */
int dojo_rollout_minimal_gradients(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* X0, const double* U,
                                   double* X_traj, double* Gx, double* Gu, int32_t* status, int32_t* iters);

/* Reverse mode through a rollout: a loss's vector-Jacobian product without the Jacobians (backpropagation through time, shooting).
 * dojo_rollout_tape is the recording rollout of dojo_rollout_grad without the Jacobians: Z_traj [13Nb x B x (T+1)] (slab 0 = Z0), the
 * TAPE [Nres x B x T] -- the final solver iterate of every pair (t, e) at t*B + e, in the library's internal ordering (opaque; only
 * dojo_rollout_vjp reads it) -- and status / iters [B x T] (nullable), bit for bit those of dojo_rollout_grad.  U [nu x B x T] nullable
 * = zero input.
 * dojo_rollout_vjp is the reverse-mode derivative of the rollout recorded by dojo_rollout_tape (same Z_traj, U, tape):
 *   lambda_T = gZ[T];  for t = T-1 .. 0:  gU[t] = Fu_t' lambda_{t+1},  lambda_t = Fz_t' lambda_{t+1} + gZ[t];   gZ0 = lambda_0
 * with Fz_t, Fu_t exactly the Jacobians dojo_rollout_grad returns (consistent IFT, inputs' configuration derivative included), up to
 * rounding: one transposed solve against each step's KKT factor instead of 12Nb + nu column solves.  Cotangents are in the gradients'
 * attitude-reduced packing [x, v, phi, w] per body: gZ [12Nb x B x (T+1)] (required), gZ0 [12Nb x B] (required), gU [nu x B x T]
 * (nullable), status [B] (nullable): 0, or 3 if a factorisation of the backward pass was not finite (then that environment's gZ0 and gU
 * are NaN; the others are unaffected bit for bit).  An environment's results do not depend on B, the other environments or the launch.
 * It takes no solver options: it runs no Newton iteration.
 * Both: B in 1..max_batch, T >= 1, the required buffers (DOJO_EINVAL otherwise, before anything is launched); DOJO_ENOMEM when the
 * gradient workspace does not fit (as dojo_step_grad).  Host or device pointers, all of one kind (host arrays are staged through
 * grow-only buffers of the handle); the _async forms take device pointers and do not synchronise.  Flags, external forces and the Q1 / Q2
 * literal variants are single-step features, as for dojo_rollout_grad. */
int dojo_rollout_tape(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U, double* Z_traj,
                      double* tape, int32_t* status, int32_t* iters);
int dojo_rollout_tape_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const double* dU, double* dZ_traj,
                            double* dtape, int32_t* dstatus, int32_t* diters, void* cuda_stream);
int dojo_rollout_vjp(DojoHandle* h, int B, int T, const double* Z_traj, const double* U, const double* tape, const double* gZ, double* gZ0,
                     double* gU, int32_t* status);
int dojo_rollout_vjp_async(DojoHandle* h, int B, int T, const double* dZ_traj, const double* dU, const double* dtape, const double* dgZ,
                           double* dgZ0, double* dgU, int32_t* dstatus, void* cuda_stream);

/* Reverse mode through a closed-loop rollout (dojo_rollout_feedback): gradients of a loss with respect to the law's gains, references
 * and the initial state, for fitting a controller by gradient (PID / LQR gain tuning, policies linear in the minimal state).
 * dojo_rollout_feedback_tape is dojo_rollout_feedback recorded like dojo_rollout_tape: Z_traj [13Nb x B x (T+1)] (slab 0 = Z0), the law's
 * minimal states X_traj [2nu x B x (T+1)] (slab T = maximal_to_minimal(z_T)), its integral states Xi_traj [2nu x B x T] (xi_t, required
 * if and only if K_i is given), U_applied [nu x B x T], the tape [Nres x B x T], status / iters [B x T] (nullable), and xi in / out as
 * dojo_rollout_feedback.  Z_traj, U_applied and xi equal dojo_rollout_feedback's bit for bit; Z_traj, the tape, status and iters equal
 * dojo_rollout_tape(Z0, U_applied)'s.
 * dojo_rollout_feedback_vjp is its reverse-mode derivative (same fb, Z_traj, X_traj, Xi_traj, U_applied, tape).  With d_t = x_t - x_ref_t,
 * M_t = dojo_maximal_to_minimal_jacobian at z_t and Fz_t, Fu_t the step Jacobians at the applied inputs (as dojo_rollout_vjp):
 *   lambda_T = gZ[T] + M_T' gX[T],  nu = 0;  for t = T-1 .. 0:
 *     a_t = Fu_t' lambda_{t+1} + gUa[t],  nu -= K_i,t' a_t,  d_bar = -K_t' a_t + h nu,
 *     lambda_t = Fz_t' lambda_{t+1} + gZ[t] + M_t' (d_bar + gX[t]),
 *     du_ref_t = a_t,  dK_t = -a_t d_t',  dK_i,t = -a_t xi_t',  dx_ref_t = -d_bar;
 *   gZ0 = lambda_0 [12Nb x B] (required),  gxi0 = nu [2nu x B] (the cotangent of the caller's xi; required with K_i, else not read).
 * Cotangents, each nullable (= 0): gZ [12Nb x B x (T+1)] in the gradients' packing [x, v, phi, w], gX [2nu x B x (T+1)], gUa [nu x B x T]
 * on the applied inputs.  The law gradients (DojoFeedbackGrad, nullable, each member nullable) are ALWAYS per environment, [.. x B x steps]
 * with the DojoFeedback's steps: entry (t, e) at t * B + e; with steps = 1 the sum over t.  A law array shared by all environments
 * (envs = 1) therefore gets B gradients, which the caller sums: the call has no cross-environment reduction, so every result of an
 * environment is one lane's fixed-order sum and does not depend on B, the other environments or the launch.  status [B] (nullable): 0, or
 * 3 if a factorisation was not finite (then every output of that environment is NaN; the others are unaffected).
 * Both: the checks of dojo_rollout_feedback and of dojo_rollout_tape (DOJO_EINVAL before anything is launched; DOJO_ENOMEM when the
 * gradient workspace does not fit).  Host or device pointers, all of one kind; the _async forms take device pointers and do not
 * synchronise. */
typedef struct {
  double* K;      /* [nu x 2nu x B x steps], nullable */
  double* K_i;    /* same shape, nullable (not written without K_i) */
  double* x_ref;  /* [2nu x B x steps], nullable */
  double* u_ref;  /* [nu x B x steps], nullable */
} DojoFeedbackGrad;
int dojo_rollout_feedback_tape(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const DojoFeedback* fb, double* xi,
                               double* Z_traj, double* X_traj, double* Xi_traj, double* U_applied, double* tape, int32_t* status, int32_t* iters);
int dojo_rollout_feedback_tape_async(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* dZ0, const DojoFeedback* fb,
                                     double* dxi, double* dZ_traj, double* dX_traj, double* dXi_traj, double* dU_applied, double* dtape,
                                     int32_t* dstatus, int32_t* diters, void* cuda_stream);
int dojo_rollout_feedback_vjp(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* Z_traj, const double* X_traj,
                              const double* Xi_traj, const double* U_applied, const double* tape, const double* gZ, const double* gX,
                              const double* gUa, const DojoFeedbackGrad* out, double* gZ0, double* gxi0, int32_t* status);
int dojo_rollout_feedback_vjp_async(DojoHandle* h, int B, int T, const DojoFeedback* fb, const double* dZ_traj, const double* dX_traj,
                                    const double* dXi_traj, const double* dU_applied, const double* dtape, const double* dgZ,
                                    const double* dgX, const double* dgUa, const DojoFeedbackGrad* out, double* dgZ0, double* dgxi0,
                                    int32_t* dstatus, void* cuda_stream);

/* Batched environment layer (DojoEnvironments/src/environments.jl:77-109 and environments/{ant_ars,quadruped_sampling,
 * pendulum}.jl): state_map / input_map / step! / get_state plus the reward and failure test of the learning examples
 * (examples/learning/ant_ars.jl:79-116), fused around the step kernel so that an RL / sampling loop exchanges only
 * (state, action, reward, done) per step.
 *   environment state s = [minimal state (2 nu); clamp(gamma_1, -1, 1) per contact if contact_obs]   (ant_ars.jl:72-79)
 *   state_map(s) = s[1 : 2 nu]; input_map(a) = [zeros(n_unactuated); a]                                (ant_ars.jl:53-61)
 *   reward = w_forward (s'[forward_index] - s[forward_index]) / timestep - w_control a'a
 *            - w_contact sum_c clamp(gamma_1,c)^2 + survive_reward                   (forward_index < 0: no forward term)
 *   done   = !(all finite(s') && healthy_min <= s'[healthy_index] <= healthy_max && |s'[bound_index]| <= bound_abs)
 *            (an index < 0 disables its test)
 * AntARS: {6, 1, 0, 2, -1, 100, 0.05/10, 0.5e-3, 0.05, 0.2, 1.0, 0};  QuadrupedSampling: {6, 0, -1, 2, 0, 0,0,0,0, 0, inf, 1000}. */
typedef struct {
  int32_t n_unactuated, contact_obs, forward_index, healthy_index, bound_index;
  double w_forward, w_control, w_contact, survive_reward, healthy_min, healthy_max, bound_abs;
} DojoEnvSpec;
int dojo_env_num_state(const DojoHandle* h, const DojoEnvSpec* spec);  /* ns = 2 nu + (contact_obs ? Ni : 0) */
int dojo_env_num_action(const DojoHandle* h, const DojoEnvSpec* spec); /* na = nu - n_unactuated */
/* One step!(environment, s, a) for B environments: S [ns x B], A [na x B] (nullable: zero input), S_next [ns x B],
 * reward [B], done [B], status [B], iters [B] (all four nullable).  Three launches on one stream (pre, step, post); the
 * maximal states and the solver solution stay on the device.  Host or device pointers (all of the same kind);
 * _async: device pointers, no synchronisation.  S_next must not alias S. */
int dojo_env_step(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, const double* S,
                  const double* A, double* S_next, double* reward, int32_t* done, int32_t* status, int32_t* iters);
int dojo_env_step_async(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, const double* dS,
                        const double* dA, double* dS_next, double* dreward, int32_t* ddone, int32_t* dstatus,
                        int32_t* diters, void* cuda_stream);
/* Open-loop rollout of T environment steps (the inner loop of sampling-based MPC / ARS evaluation, examples/learning/
 * ant_ars.jl:79-116, quadruped_sampling.jl:66-77) with everything resident on the device: A [na x B x T] (nullable),
 * S_final [ns x B], ret [B] = sum of the rewards up to and including the step at which the failure test fires,
 * failed [B] = 1 if it fired (both nullable).  3 T launches, no host round trip.  Host or device pointers. */
int dojo_env_rollout(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, int T, const double* S0,
                     const double* A, double* S_final, double* ret, int32_t* failed);
/* Closed-loop rollout with one linear policy per environment (ARS evaluation, examples/learning/ant_ars.jl:79-116):
 *   a = Theta_e ((s - mean) ./ std)   Theta [na x ns x B] column-major per environment; mean / std [ns] HOST vectors, frozen for
 *   the call (nullable: no normalisation; the reference updates its Normalizer inside the rollout -- S_traj [ns x B x T],
 *   nullable, returns the state observed before every step so that the caller can update the statistics afterwards).
 * 4 T launches (policy, pre, step, post), nothing leaves the device in between.  Host or device pointers. */
int dojo_env_policy_rollout(DojoHandle* h, const DojoSolverOptions* opts, const DojoEnvSpec* spec, int B, int T,
                            const double* S0, const double* Theta, const double* mean, const double* std, double* S_final,
                            double* ret, int32_t* failed, double* S_traj);
/* reset (initialize!(environment, model), environments.jl:118-120): S[:, e] = s0 for every e with mask[e] != 0 (mask
 * nullable: all).  s0 [ns] is a HOST vector; S / mask host or device pointers of the same kind. */
int dojo_env_reset(DojoHandle* h, const DojoEnvSpec* spec, int B, const double* s0, const int32_t* mask, double* S);

/* Trajectory recording (Storage, src/simulation/storage.jl:15-67) and the diagnostics derived from it
 * (src/mechanics/momentum.jl:17-74, src/mechanics/energy.jl:32-93), computed on the device right after the solve exactly
 * where simulate! calls save_to_storage! (src/simulation/simulate.jl:16-36: after mehrotra!, before update_state!):
 *   storage [12 Nb x B]: per body px(3), pq(3) (momenta, world frame), vl(3) = px / m, wl(3) = J \ R(q2)' pq;
 *   diag    [8 x B]:     total linear momentum(3), angular momentum about the centre of mass(3), kinetic, potential energy.
 * Storage.x / q / v / w of step k are the state BEFORE the k-th solve, i.e. the input Z itself (x2, v15, q2, w15).
 * External forces are taken as zero (simulate! clears them before save_to_storage!).  Host or device pointers (all of the
 * same kind); _async: device pointers, no synchronisation. */
int dojo_step_record(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, double* Z_next,
                     double* storage, double* diag, int32_t* status, int32_t* iters);
int dojo_step_record_async(DojoHandle* h, const DojoSolverOptions* opts, int B, const double* dZ, const double* dU,
                           double* dZ_next, double* dstorage, double* ddiag, int32_t* dstatus, int32_t* diters,
                           void* cuda_stream);
/* simulate!(mechanism, 1:T, storage, control!; record = true) with open-loop inputs U [nu x B x T] (nullable): per step k
 * Z_traj[:, :, k] = state before the k-th solve (Storage.x, q, v, w), storage[:, :, k], diag[:, :, k] as above (each
 * nullable); Z_final [13 Nb x B] = state after the last solve; status_any [B] = max status.  2 T launches. */
int dojo_simulate_record(DojoHandle* h, const DojoSolverOptions* opts, int B, int T, const double* Z0, const double* U,
                         double* Z_final, double* Z_traj, double* storage, double* diag, int32_t* status_any);

/* number of kernel launches issued by this handle so far (bench.py's gpu_launches) */
int64_t dojo_launch_count(const DojoHandle* h);

#ifdef __cplusplus
}
#endif
#endif /* DOJO_B200_H */
