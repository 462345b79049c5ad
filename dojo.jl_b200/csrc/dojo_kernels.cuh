// dojo_kernels.cuh -- the per-timestep hot path as one persistent sm_90a kernel.
//
// A CTA hosts up to four environments ("slots"), each owned by nw warps.  An environment's whole interior-point problem
// (solution vector, residuals, block-sparse KKT matrix) lives in its slot's shared-memory arena for the duration of the step;
// HBM is touched only to read z, u (and Fext) at the start and to write z_next (and status / iters / sol / gradients) at the end.
//
// Reference call stack restated here (file:line relative to the reference's src/):
//   step!                 simulation/step.jl:11-30      -> dojo_step_kernel
//   set_maximal_state!    mechanism/set.jl:10-26        -> prologue()
//   set_input!            mechanism/set.jl:40-53        -> prologue() (input / spring impulses, impulse maps)
//   mehrotra!             solver/mehrotra.jl:9-73       -> mehrotra()
//   set_entries!          solver/linear_system.jl:1-17  -> evaluate<true>()   (residual + KKT blocks)
//   residual_violation / bilinear_violation  solver/violations.jl -> evaluate_ls() (line search, two trials per pass)
//   ldu_factorization! / ldu_backsubstitution! (GraphBasedSystems) -> factorize() / solve()
//   cone_line_search! / centering! / correction! / line_search!   -> same names below
//   update_state! + get_next_state  bodies/set.jl:22-36, mechanism/get.jl:126-134 -> epilogue()
#pragma once
#include "dojo_linalg.cuh"
#include "dojo_plan.h"

namespace dj {

// Gather-list entries (BodyDev::g_off): arena offset of a contribution slot.  In the DJ_ANY_CONTACT compilation bit 30 marks the
// slot of a "full" joint (JF_FULL: 6 x 6 block like a contact slot); the other compilation never sees such entries.
#ifdef DJ_ANY_CONTACT
#define DJ_SLOT_OFF(raw) ((raw) & 0x3fffffff)
#define DJ_SLOT_FULL(raw) (((raw) >> 30) & 1)
#else
#define DJ_SLOT_OFF(raw) (raw)
#endif
#ifdef DJ_ANY_CONTACT  // contact model of a plan entry (ContactDev::tn), see dojo_contact_orthant.cuh
DJ_DEV int contact_type(const ContactDev& cd) { return cd.tn & 0xff; }
DJ_DEV int contact_nh(const ContactDev& cd) { return cd.tn >> 8; }
#endif

DJ_DEV V3 ld3(const double* p) { return V3{p[0], p[1], p[2]}; }
DJ_DEV void st3(double* p, V3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
DJ_DEV void add3(double* p, V3 v) { p[0] += v.x; p[1] += v.y; p[2] += v.z; }
DJ_DEV M33 ldm33(const double* p) {
  M33 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.m[i][j] = p[3 * i + j];
  return r;
}
DJ_DEV void stm33(double* p, const M33& a) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) p[3 * i + j] = a.m[i][j];
}
DJ_DEV Quat ldq(const double* p) { return Quat{p[0], p[1], p[2], p[3]}; }

struct Ctx {
  double* A;  // this environment's arena
  const Plan* P;
  // plan tables (a copy in shared memory when it fits next to the arenas, else the global-memory originals)
  const BodyDev* bodies;
  const JointDev* joints;
  const ContactDev* contacts;
  const ElimStep* steps;
  const int* sched;
  const int* ilist;
  const WarpRole* roles;
  const int* ucol;
  int tid, nthreads, warp, lane;  // thread / warp index inside this environment's slot (nthreads = 32 nw)
  int sd;                         // offset added to contribution-slot addresses (second trial of a paired line-search pass)
  int bar;                        // named barrier of the slot (1 + slot index); barrier 0 is the CTA-wide alignment barrier
  double mu;
  // slots of the CTA: this slot's index, their number, the arena of slot 0 and the distance between arenas; CTA-wide mailbox in
  // static shared memory (s_int / s_dbl, layout below); parity of the next alignment; whether this slot is the OWNER of a
  // line search that the drained slots of the CTA assist (ls_assist_loop)
  int slot, nslots, slot_stride;
  double* arena0;
  int* s_int;
  double* s_dbl;
  int apar, assist;
#ifdef DJ_PROFILE
  long long t_eval_jac, t_eval_ls, t_fact, t_solve, t_misc, t_align, t_cone, t_center, t_rolewait, t_last;
  long long f_fold, f_inv, f_rm, f_schur, f_bar, f_last;
  long long s_cond, s_fwd, s_bwd, s_rec, s_bar;  // solve(): condense + gather, forward sweep, backward sweep, recover, slot barriers
#endif
};
#ifdef DJ_PROFILE
#define DJ_TICK(c, field) { long long _t = clock64(); (c).field += _t - (c).t_last; (c).t_last = _t; }
#define DJ_FTICK(c, field) { long long _t = clock64(); (c).field += _t - (c).f_last; (c).f_last = _t; }
#else
#define DJ_TICK(c, field) {}
#define DJ_FTICK(c, field) {}
#endif

// Barrier over the nw warps that own this environment.  A CTA hosts several environments ("slots"), each with its own
// arena and its own named barrier, so that the slots only meet at the CTA-wide alignment point of the Newton loop.
#ifdef DJ_HOSTEMU  // tests/hostemu runs this code on CPU fibers; the named barrier is provided by its shim
DJ_DEV void slot_sync(const Ctx& c) { hostemu_bar_sync(c.bar, c.nthreads); }
#else
DJ_DEV void slot_sync(const Ctx& c) { asm volatile("bar.sync %0, %1;" ::"r"(c.bar), "r"(c.nthreads) : "memory"); }
#endif

// CTA-wide mailbox (static shared memory of the kernel):
//   s_int[0..7]   environment dequeued by slot k                      s_int[8 + 8 p + k]  slot k is live, alignment parity p
//   s_int[24]     line-search request: 1 = evaluate, 0 = released     s_int[25]           first trial index of the pass
//   s_dbl[0], [1] step length of that first trial, mu                 s_dbl[2 + 2 t], [3 + 2 t]  violations (rv, bv) of trial t < 16
constexpr int kMaxAssistTrials = 16;
struct AlignInfo { int n_live, owner; };
// Every CTA-wide barrier of the Newton loop is THIS instruction: live slots reach it from mehrotra(), drained slots from the loop at the
// end of the kernel, helpers from ls_assist_loop().  Different bar.sync instructions on barrier 0 would match as well (sm_70+ counts
// arrivals per barrier resource, not per instruction), but one shared call site keeps the pattern within what CUDA C++ documents for
// __syncthreads() and what compute-sanitizer's synccheck accepts.
#ifdef DJ_HOSTEMU
DJ_DEV void cta_barrier() { __syncthreads(); }
#else
__device__ __noinline__ void cta_barrier() { __syncthreads(); }
#endif
// CTA-wide alignment barrier (barrier 0): how many slots of the CTA still have work (and the last of them).  Slots that ran out of
// environments keep arriving here (with live = false) until every slot is done.  The flags are double-buffered by the parity of the
// call: a slot can only be two alignments ahead of another one after the barrier in between, which that one passes after its reads.
DJ_DEV AlignInfo cta_align(Ctx& c, bool live) {
  int* fl = c.s_int + 8 + 8 * c.apar;
  c.apar ^= 1;
  if (c.tid == 0) fl[c.slot] = live ? 1 : 0;
  cta_barrier();
  AlignInfo r;
  r.n_live = 0; r.owner = -1;
  for (int q = 0; q < c.nslots; ++q)
    if (fl[q]) { r.n_live++; r.owner = q; }
  return r;
}
// The owner of an assisted line search lets the helpers go (they wait at the CTA barrier for the next request): on every path that
// leaves the Newton iteration, and when a trial has been accepted.
DJ_DEV void assist_release(Ctx& c) {
  if (!c.assist) return;
  if (c.tid == 0) c.s_int[24] = 0;
  cta_barrier();
  c.assist = 0;
}

// SMALL (dojo_step_kernel.cuh): the forward kernel specialised for mechanisms with 2 warps per environment, paired line-search trials
// and joint pairs, at most 16 nodes in every role pass and the whole plan in shared memory.  Every function below that takes it
// decides the same things from constants that the generic code reads from the plan; the floating-point operations and their order
// are the same.  Warps per environment:
template <bool SMALL>
DJ_DEV int slot_warps(const Ctx& c) { return SMALL ? 2 : c.P->nw; }

// slot-wide reductions (deterministic: per-warp shuffles, then a fixed-order combine of the nw partials)
template <bool SMALL = false>
DJ_DEV void block_nanmax2(const Ctx& c, double& a, double& b) {
  double* red = c.A + c.P->red_off;
  a = warp_nanmax(a);
  b = warp_nanmax(b);
  if (slot_warps<SMALL>(c) == 1) return;
  if (c.lane == 0) { red[2 * c.warp] = a; red[2 * c.warp + 1] = b; }
  slot_sync(c);
  a = red[0]; b = red[1];
  for (int w = 1; w < slot_warps<SMALL>(c); ++w) { a = nanmax(a, red[2 * w]); b = nanmax(b, red[2 * w + 1]); }
  slot_sync(c);
}
template <bool SMALL = false>
DJ_DEV double block_min(const Ctx& c, double a) {
  double* red = c.A + c.P->red_off;
  a = warp_min(a);
  if (slot_warps<SMALL>(c) == 1) return a;
  if (c.lane == 0) red[c.warp] = a;
  slot_sync(c);
  a = red[0];
  for (int w = 1; w < slot_warps<SMALL>(c); ++w) a = fmin(a, red[w]);
  slot_sync(c);
  return a;
}
template <bool SMALL = false>
DJ_DEV void block_sum3(const Ctx& c, double& a, double& b, double& d) {
  double* red = c.A + c.P->red_off;
  a = warp_sum(a); b = warp_sum(b); d = warp_sum(d);
  if (slot_warps<SMALL>(c) == 1) return;
  if (c.lane == 0) { red[3 * c.warp] = a; red[3 * c.warp + 1] = b; red[3 * c.warp + 2] = d; }
  slot_sync(c);
  a = red[0]; b = red[1]; d = red[2];
  for (int w = 1; w < slot_warps<SMALL>(c); ++w) { a += red[3 * w]; b += red[3 * w + 1]; d += red[3 * w + 2]; }
  slot_sync(c);
}

// node index handled by this lane for role pass p (or -1)
DJ_DEV int role_item(const WarpRole& r, int p, int lane) { return lane < r.count[p] ? r.first[p] + lane : -1; }

// kinematic state of one body at the candidate solution sol + f * delta
struct Kin {
  V3 x2, v, w, x3;
  Quat q2, q3;
  M33 R3, E;
};

DJ_DEV Kin body_kin(const Ctx& c, int b, double f) {
  Kin k;
  const Plan& P = *c.P;
  if (b < 0) {  // origin: identity pose, zero velocity (bodies/origin.jl)
    k.x2 = k.v = k.w = k.x3 = v3zero();
    k.q2 = k.q3 = Quat{1.0, 0.0, 0.0, 0.0};
    k.R3 = m33ident();
    k.E = m33zero();
    return k;
  }
  const BodyDev& bd = c.bodies[b];
  const double* st = c.A + bd.st_off;
  const double* so = c.A + P.sol_off + bd.sol_off;
  k.x2 = ld3(st);
  k.q2 = ldq(st + 3);
  k.v = ld3(so);
  k.w = ld3(so + 3);
  if (f != 0.0) {  // candidate_step! (solver/line_search.jl:141-152) incl. the angular-velocity clip
    const double* dl = c.A + P.rhs_off + bd.sol_off;
    k.v = k.v + f * ld3(dl);
    k.w = k.w + f * ld3(dl + 3);
    double wmax = 3.9 / (P.h * P.h);
    double wd = dot(k.w, k.w);
    if (wd > wmax) k.w = (wmax / wd) * k.w;
  }
  k.x3 = k.x2 + P.h * k.v;
  k.q3 = qmul(k.q2, qmap(k.w, P.h));
  k.R3 = rotmat(k.q3);
  k.E = attitude_velocity_jacobian(k.w, P.h);
  return k;
}

// ------------------------------------------------------------------------------------------------------------
// Joint geometry shared by the prologue (configuration x2,q2) and the evaluation (configuration x3,q3).
// Attitude-form Jacobians: a body-frame perturbation q (x) (1, d) of the parent / child orientation.
// ------------------------------------------------------------------------------------------------------------
struct JointGeom {
  V3 et;            // translational displacement (parent frame)   translational/minimal.jl:4-12
  M33 Xp, Xc;       // d et / d x_parent, d et / d x_child          :14-30
  M33 Qtp, Qtc;     // d et / d (attitude parent / child)
  Quat qr;          // rotational displacement quaternion            rotational/minimal.jl:4-11
  M33 Qrp, Qrc;     // d vec(qr) / d (attitude parent / child)        :28-40
};

DJ_DEV JointGeom joint_geom(const JointDev& jd, V3 xa, Quat qa, const M33& Ra, V3 xb, Quat qb, const M33& Rb) {
  JointGeom g;
  V3 pa = ld3(jd.pa), pb = ld3(jd.pb);
  V3 dw = xb + Rb * pb - xa - Ra * pa;
  g.et = tmul(Ra, dw);
  M33 Rat = transpose(Ra);
  g.Xc = Rat;
  g.Xp = (-1.0) * Rat;
  g.Qtp = 2.0 * skew(g.et + pa);
  g.Qtc = (-2.0) * (Rat * Rb * skew(pb));
  Quat qoff = ldq(jd.qoff);
  g.qr = qmul(qmul(qinv(qoff), qinv(qa)), qb);
  V3 vr = qvec(g.qr);
  g.Qrc = m33ident(g.qr.s) + skew(vr);
  g.Qrp = (-1.0) * ((m33ident(g.qr.s) - skew(vr)) * transpose(rotmat(qoff)));
  return g;
}

// d rotation_vector(qr) / d attitude (3x3) for the parent / child side
DJ_DEV void rotvec_attitude_jacobians(const JointDev& jd, const JointGeom& g, M33& Tp, M33& Tc) {
  M34 drv = drotation_vector_dq(g.qr);
  V3 vr = qvec(g.qr);
  // child: d qr = [ -vr' ; s I + skew(vr) ] d          parent: d qr = [ vr' Roff' ; -(s I - skew(vr)) Roff' ] d
  M33 Rofft = transpose(rotmat(ldq(jd.qoff)));
  V3 srow_p = vtmul(vr, Rofft);
  V3 srow_c = -vr;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    V3 dv = v3(drv.m[i][1], drv.m[i][2], drv.m[i][3]);
    V3 rc = drv.m[i][0] * srow_c + vtmul(dv, g.Qrc);
    V3 rp = drv.m[i][0] * srow_p + vtmul(dv, g.Qrp);
    Tc.m[i][0] = rc.x; Tc.m[i][1] = rc.y; Tc.m[i][2] = rc.z;
    Tp.m[i][0] = rp.x; Tp.m[i][1] = rp.y; Tp.m[i][2] = rp.z;
  }
}

DJ_DEV void write_slot(double* s, V3 f, V3 t, const M33& K) { st3(s, f); st3(s + 3, t); stm33(s + 6, K); }
// Which side of a limited axis keeps its dual in the joint's node (dojo_plan.h joint_nq), from the current iterate (s, gamma >= 0):
// the smaller REG-shifted slack.  sA, gA: shifted slack / dual of the kept side, sg = +1 (upper) / -1 (lower); kI = gamma'/s' of the
// condensed side.  Evaluated identically by the assembly, the right-hand-side condensation and the recovery of one iteration.
struct LimitSide { bool up; double sA, gA, sg, sI, gI, kI; };
DJ_DEV LimitSide limit_side(double su, double sl, double gu, double gl) {
  LimitSide r;
  const double su1 = su + kReg, sl1 = sl + kReg, gu1 = gu + kReg, gl1 = gl + kReg;
  r.up = su1 <= sl1;
  r.sA = r.up ? su1 : sl1; r.gA = r.up ? gu1 : gl1; r.sg = r.up ? 1.0 : -1.0;
  r.sI = r.up ? sl1 : su1; r.gI = r.up ? gl1 : gu1;
  r.kI = r.gI / r.sI;
  return r;
}

#ifdef DJ_ANY_CONTACT
#include "dojo_joint_tra.cuh"  // translational springs / dampers / limits (only in the compilation that serves such mechanisms)
#endif

// ------------------------------------------------------------------------------------------------------------
// Prologue: set_maximal_state!, set_input!, explicit spring impulses, joint impulse maps (constant over the solve)
// ------------------------------------------------------------------------------------------------------------
DJ_DEV void prologue_joint(Ctx& c, int j, const double* __restrict__ u) {
  const Plan& P = *c.P;
  double* A = c.A;
  const JointDev& jd = c.joints[j];
  V3 cl_p = v3zero(), ca_p = v3zero(), cl_c = v3zero(), ca_c = v3zero();  // [JF2; Jtau2] + spring impulses
  Kin ka = body_kin(c, jd.parent, 0.0), kb = body_kin(c, jd.child, 0.0);
  M33 Ra = rotmat(ka.q2), Rb = rotmat(kb.q2);
  JointGeom g = joint_geom(jd, ka.x2, ka.q2, Ra, kb.x2, kb.q2, Rb);
  M33 Roff = rotmat(ldq(jd.qoff));
  M33 Rrel_t = transpose(Rb) * Ra;  // R(qb^-1 qa)
  // inputs (joints/joint.jl:96-99, translational/input.jl:5-27, rotational/input.jl:5-17)
  if (u) {
    V3 it = v3zero(), ir = v3zero();
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nfree_t) it += u[jd.u_off + i] * ld3(jd.At + 3 * i);
      if (i < jd.nfree_r) ir += u[jd.u_off + jd.nfree_t + i] * ld3(jd.Ar + 3 * i);
    }
    it = P.input_scaling * it;
    ir = P.input_scaling * ir;
    // translational: JF += X' input ; Jtau += (1/2 Q' input) / 2
    cl_p += tmul(g.Xp, it); ca_p += 0.25 * tmul(g.Qtp, it);
    cl_c += tmul(g.Xc, it); ca_c += 0.25 * tmul(g.Qtc, it);
    // rotational: parent -R(qoff) tau, child R(qb^-1 qa qoff) tau
    V3 tp = Roff * ir;
    ca_p -= tp;
    ca_c += Rrel_t * tp;
  }
  // rotational spring (rotational/springs.jl:5-38), explicit at (x2, q2)
  if (jd.spring_r != 0.0 && jd.nfree_r > 0) {
    V3 rv = rotation_vector(g.qr);
    V3 force = v3zero();
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (i < jd.nfree_r) {
        V3 a = ld3(jd.Ar + 3 * i);
        force += (-jd.spring_r * (jd.spring_off_r[i] - dot(a, rv))) * a;
      }
    V3 tp = P.h * (Roff * force);
    ca_p += tp;
    ca_c -= Rrel_t * tp;
  }
#ifdef DJ_ANY_CONTACT
  if (jd.flags) prologue_joint_tra(c, jd, g, cl_p, ca_p, cl_c, ca_c);
#endif
  write_slot(A + jd.slot_c, cl_c, ca_c, m33zero());
  if (jd.parent >= 0) write_slot(A + jd.slot_p, cl_p, ca_p, m33zero());
  // impulse maps at the current configuration (joints/joint.jl:67-93, joints/impulses.jl:4-7): 6 x ne for the equality
  // multipliers; the limit duals act through +-(1/2 Qr' A_i) on the torque rows only (kept per limited axis: tP, tC)
  for (int side = 0; side < 2; ++side) {
    const bool par = (side == 0);
    if (par && jd.parent < 0) continue;
    double* G = A + (par ? jd.Gp_off : jd.Lc_off);
    const double sgn = par ? 1.0 : -1.0;  // the child block stores L = -G directly
    const M33& X = par ? g.Xp : g.Xc;
    const M33& Qt = par ? g.Qtp : g.Qtc;
    const M33& Qr = par ? g.Qrp : g.Qrc;
    const int n = joint_nq(jd);
    for (int q = jd.ne; q < n; ++q)  // columns of the kept limit duals: written at every assembly (the kept side can change)
      for (int r = 0; r < 6; ++r) G[r * n + q] = 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nl_t) {  // translational lambda column i
        V3 ci = ld3(jd.Ct + 3 * i);
        V3 f = tmul(X, ci), t = 0.5 * tmul(Qt, ci);
        int col = i;
        G[0 * n + col] = sgn * f.x; G[1 * n + col] = sgn * f.y; G[2 * n + col] = sgn * f.z;
        G[3 * n + col] = sgn * t.x; G[4 * n + col] = sgn * t.y; G[5 * n + col] = sgn * t.z;
      }
      if (i < jd.nl_r) {  // rotational lambda column i
        V3 ci = ld3(jd.Cr + 3 * i);
        V3 t = 0.5 * tmul(Qr, ci);
        int col = jd.nl_t + i;
        G[0 * n + col] = 0.0; G[1 * n + col] = 0.0; G[2 * n + col] = 0.0;
        G[3 * n + col] = sgn * t.x; G[4 * n + col] = sgn * t.y; G[5 * n + col] = sgn * t.z;
      }
#ifdef DJ_ANY_CONTACT
      if (jd.flags & JF_LIM_TRA) continue;  // translational limits: 6-vectors, written by prologue_joint_tra
#endif
      if (i < jd.nb2_r) {  // G[:, gamma_upper_i] = -[0; t], G[:, gamma_lower_i] = +[0; t],  t = 1/2 Qr' A_i
        V3 t = 0.5 * tmul(Qr, ld3(jd.Ar + 3 * i));
        st3(A + jd.lim_off + kLim * i + (par ? 6 : 9), t);
      }
    }
  }
  // reset! (joints/constraints.jl:440-448): s = gamma = 1, lambda = 0
  double* so = A + P.sol_off + jd.sol_off;
  for (int i = 0; i < jd.ne; ++i) so[i] = 0.0;
  for (int i = 0; i < 2 * jd.nb_r; ++i) so[jd.ne + i] = 1.0;
}

DJ_DEV void prologue(Ctx& c, const double* z, const double* __restrict__ u, const double* __restrict__ fext, const bool grad) {
  const Plan& P = *c.P;
  double* A = c.A;
  const WarpRole& role = c.roles[c.warp];
  // coalesced read of z: [x2(3) v15(3) q2(4) w15(3)] per body (mechanism/set.jl:10-26)
  for (int t = c.tid; t < P.nz; t += c.nthreads) {
    int b = t / 13, k = t - 13 * b;
    double val = z[t];
    const BodyDev& bd = c.bodies[b];
    if (k < 3) A[bd.st_off + k] = val;
    else if (k < 6) A[P.sol_off + bd.sol_off + (k - 3)] = val;
    else if (k < 10) A[bd.st_off + 3 + (k - 6)] = val;
    else A[P.sol_off + bd.sol_off + 3 + (k - 10)] = val;
  }
  slot_sync(c);
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_BODY) {  // constant part of the discrete Euler-Lagrange residual (integrators/constraint.jl:14-25)
      const BodyDev& bd = c.bodies[idx];
      const double* so = A + P.sol_off + bd.sol_off;
      V3 v15 = ld3(so), w15 = ld3(so + 3);
      M33 J = ldm33(bd.J);
      V3 F = v3zero(), tau = v3zero();
      if (fext) { F = ld3(fext + 6 * idx); tau = ld3(fext + 6 * idx + 3); }
      V3 g = ld3(P.g);
      V3 lin = (-bd.mass) * v15 - P.h * (bd.mass * g + F);
      double n0 = 0.5 * P.h * sqrt(4.0 / (P.h * P.h) - dot(w15, w15));
      V3 Jw = J * w15;
      V3 ang = (-1.0) * (n0 * Jw - (0.5 * P.h) * cross(w15, Jw)) - P.h * tau;
      st3(A + bd.cst_off, lin);
      st3(A + bd.cst_off + 3, ang);
      if (grad) st3(A + bd.gb_off + 27, w15);  // gradient pass: the w15 column needs the initial angular velocity
    } else if (role.type[p] == ROLE_JOINT) {
      prologue_joint(c, idx, u);
    } else {  // reset! + initialize! (contacts/constraints.jl:79-86, solver/initialization.jl:7-48)
      double* so = A + P.sol_off + c.contacts[idx].sol_off;
      const double v0 = 1.0 + 0.5 * 1.0 * 1.0 / (1.0 + 1e-20);  // neutral (1,1,0,0) pushed to 1.5 by the Mehrotra-style start
#ifdef DJ_ANY_CONTACT
      if (contact_type(c.contacts[idx]) != 2) {  // impact / linear: neutral = ones(N½), initialize_positive_orthant! (initialization.jl:1-5, :20-33)
        const int n2 = 2 * contact_nh(c.contacts[idx]);
        for (int i = 0; i < n2; ++i) so[i] = v0;
        continue;
      }
#endif
      so[0] = v0; so[1] = v0; so[2] = 0.0; so[3] = 0.0;
      so[4] = v0; so[5] = v0; so[6] = 0.0; so[7] = 0.0;
    }
  }
  slot_sync(c);
  // cst -= [JF2; Jtau2] + spring impulses, gathered per body in a fixed order
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, c.lane);
    if (idx < 0 || role.type[p] != ROLE_BODY) continue;
    const BodyDev& bd = c.bodies[idx];
    double* cst = A + bd.cst_off;
    for (int g = bd.g_ncontact; g < bd.g_cnt; ++g) {  // joint slots only: contacts carry nothing in the prologue
      const double* s = A + DJ_SLOT_OFF(c.ilist[bd.g_off + g]);
      add3(cst, -ld3(s));
      add3(cst + 3, -ld3(s + 3));
    }
  }
  slot_sync(c);
}

// ------------------------------------------------------------------------------------------------------------
// evaluate<JAC>: residuals at sol + f * delta (and, for JAC, every KKT block = set_entries!).
// Residual entries are written to `res` (= rhs when assembling, = sav during the line search, whose saved
// residual is dead at that point).  Returns the residual / bilinear violations (solver/violations.jl).
// ------------------------------------------------------------------------------------------------------------
template <bool JAC>
DJ_DEV void eval_body(Ctx& c, int idx, double f, double* res) {
  const Plan& P = *c.P;
  double* A = c.A;
  const BodyDev& bd = c.bodies[idx];
  Kin k = body_kin(c, idx, f);
  M33 J = ldm33(bd.J);
  const double* cst = A + bd.cst_off;
  double m0 = 0.5 * P.h * sqrt(4.0 / (P.h * P.h) - dot(k.w, k.w));
  V3 Jw = J * k.w;
  V3 dlin = bd.mass * k.v + ld3(cst);
  V3 dang = m0 * Jw + (0.5 * P.h) * cross(k.w, Jw) + ld3(cst + 3);
  st3(res + bd.sol_off, -dlin);
  st3(res + bd.sol_off + 3, -dang);
  if (JAC) {
    double* D = A + bd.D_off;
    D[0] = bd.mass + kReg; D[7] = bd.mass + kReg; D[14] = bd.mass + kReg;
    V3 dm0 = (-(0.25 * P.h * P.h) / m0) * k.w;
    M33 dR = outer(Jw, dm0) + m0 * J + (0.5 * P.h) * (skew(k.w) * J - skew(Jw));
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) D[(3 + i) * 6 + 3 + j] = dR.m[i][j] + (i == j ? kReg : 0.0);
  }
}

// Closed-form solve of the contact diagonal block  D_c y = t  (contacts/nonlinear.jl:78-97), y = [ds(4); dgamma(4)]:
//   rows 0-3 (complementarity): g1' ys1 + s1' yg1 = t0 ;  Arw(g') [ys2 ys3 ys4] + Arw(s') [yg2 yg3 yg4] = t1..t3
//   rows 4-7 (constraint)     : -ys1 = t4 ; mu yg1 - yg2 = t5 ; -ys3 = t6 ; -ys4 = t7
// with the REG-shifted s' = s + REG (1,1,0,0), g' likewise (non-singular while the iterate is strictly inside the cones,
// which the fraction-to-boundary rule maintains).
// This is the elimination of the contact node that the reference's LDU performs first (contacts are the leaves of the
// elimination tree), done per lane in closed form instead of a pivoted 8 x 8 inverse.
struct ContactBlock {
  double s1, s2, s3, s4, g1, g2, g3, g4, mu;  // shifted values
  double r_s1;                                 // 1 / s1'
  double Mi[3][3];                             // inverse of the second-order-cone 3x3 block (adjugate / determinant)
};
// After the trivial rows (ys1 = -t4, ys3 = -t6, ys4 = -t7, yg2 = mu yg1 - t5) and yg1 = (t0 - g1' ys1)/s1', the three
// cone rows read  M [ys2 yg3 yg4]' = b  with  M = [g2' s3 s4; g3 s2' 0; g4 0 s2'].  M is inverted through its adjugate
// (one division by det = s2' (g2' s2' - s3 g3 - s4 g4)): no intermediate growth when s2' is tiny (sticking contact)
// or when g2' is tiny (open contact), which a fixed pivot order would suffer from at tight tolerances.
DJ_DEV ContactBlock contact_block(const double* s, const double* g, double mu) {
  ContactBlock b;
  b.s1 = s[0] + kReg; b.s2 = s[1] + kReg; b.s3 = s[2]; b.s4 = s[3];
  b.g1 = g[0] + kReg; b.g2 = g[1] + kReg; b.g3 = g[2]; b.g4 = g[3];
  b.mu = mu;
  b.r_s1 = 1.0 / b.s1;
  const double det = b.s2 * (b.g2 * b.s2 - b.s3 * b.g3 - b.s4 * b.g4);
  const double rd = 1.0 / det;
  // adj(M) for M = [a b c; d e 0; f 0 e], a = g2', b = s3, c = s4, d = g3, f = g4, e = s2'
  b.Mi[0][0] = (b.s2 * b.s2) * rd;            b.Mi[0][1] = (-b.s3 * b.s2) * rd;                    b.Mi[0][2] = (-b.s4 * b.s2) * rd;
  b.Mi[1][0] = (-b.g3 * b.s2) * rd;           b.Mi[1][1] = (b.g2 * b.s2 - b.s4 * b.g4) * rd;       b.Mi[1][2] = (b.s4 * b.g3) * rd;
  b.Mi[2][0] = (-b.g4 * b.s2) * rd;           b.Mi[2][1] = (b.s3 * b.g4) * rd;                     b.Mi[2][2] = (b.g2 * b.s2 - b.s3 * b.g3) * rd;
  return b;
}
DJ_DEV void contact_solve(const ContactBlock& b, const double* t, double* y) {
  const double ys1 = -t[4], ys3 = -t[6], ys4 = -t[7];
  const double yg1 = (t[0] - b.g1 * ys1) * b.r_s1;
  const double yg2 = b.mu * yg1 - t[5];
  const double b1 = t[1] - b.g3 * ys3 - b.g4 * ys4 - b.s2 * yg2;
  const double b2 = t[2] - b.g2 * ys3 - b.s3 * yg2;
  const double b3 = t[3] - b.g2 * ys4 - b.s4 * yg2;
  y[0] = ys1; y[2] = ys3; y[3] = ys4;
  y[4] = yg1; y[5] = yg2;
  y[1] = b.Mi[0][0] * b1 + b.Mi[0][1] * b2 + b.Mi[0][2] * b3;
  y[6] = b.Mi[1][0] * b1 + b.Mi[1][1] * b2 + b.Mi[1][2] * b3;
  y[7] = b.Mi[2][0] * b1 + b.Mi[2][1] * b2 + b.Mi[2][2] * b3;
}

#ifdef DJ_ANY_CONTACT
#include "dojo_contact_orthant.cuh"  // ImpactContact / LinearContact (only in the translation unit that serves such mechanisms)
#endif

// contacts (contacts/nonlinear.jl:50-97, contacts/contact.jl:37-155, collisions/sphere_halfspace.jl)
template <bool JAC>
DJ_DEV void eval_contact(Ctx& c, int idx, double f, double* res, double& rv, double& bv) {
  const Plan& P = *c.P;
  double* A = c.A;
  const double* sol = A + P.sol_off;
  const double* dl = A + P.rhs_off;
  const ContactDev& cd = c.contacts[idx];
#ifdef DJ_ANY_CONTACT
  if (contact_type(cd) != 2) { eval_contact_orthant<JAC>(c, idx, f, res, rv, bv); return; }
#endif
  Kin k = body_kin(c, cd.body, f);
  double s[4], g[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    s[i] = sol[cd.sol_off + i];
    g[i] = sol[cd.sol_off + 4 + i];
    if (f != 0.0) { s[i] += f * dl[cd.sol_off + i]; g[i] += f * dl[cd.sol_off + 4 + i]; }
  }
  V3 n = ld3(cd.n), t0 = ld3(cd.t), t1 = ld3(cd.t + 3), o = ld3(cd.o), off = ld3(cd.off);
  V3 ow = k.R3 * o;
  V3 rc = ow - off - cd.radius * n;
  double phi = dot(n, k.x3 + ow - off) - cd.radius;
  V3 ww = k.R3 * k.w;
  V3 vc = k.v + cross(ww, rc);
  double r4 = phi - s[0];
  double r5 = cd.mu * g[0] - g[1];
  double r6 = dot(t0, vc) - s[2];
  double r7 = dot(t1, vc) - s[3];
  double c0 = g[0] * s[0];
  double c1 = g[1] * s[1] + g[2] * s[2] + g[3] * s[3];
  double c2 = g[1] * s[2] + s[1] * g[2];
  double c3 = g[1] * s[3] + s[1] * g[3];
  rv = nanmax(rv, nanmax(nanmax(fabs(r4), fabs(r5)), nanmax(fabs(r6), fabs(r7))));
  bv = nanmax(bv, nanmax(nanmax(fabs(c0), fabs(c1)), nanmax(fabs(c2), fabs(c3))));
  double* rr = res + cd.sol_off;
  rr[0] = -(c0 - c.mu); rr[1] = -(c1 - c.mu); rr[2] = -c2; rr[3] = -c3;
  rr[4] = -r4; rr[5] = -r5; rr[6] = -r6; rr[7] = -r7;
  V3 F = g[0] * n + g[2] * t0 + g[3] * t1;       // X gamma, X = [n' 0 t0' t1']
  V3 tau = tmul(k.R3, cross(rc, F));              // R3' (rc x F)
  st3(A + cd.slot + c.sd, F);
  st3(A + cd.slot + c.sd + 3, tau);
  if (JAC) {
    // J (4 x 6): d(constraint rows)/d(v25, w25); rows (phi - s1, mu g1 - g2 [zero], vt1 - s3, vt2 - s4)
    double* Jm = A + cd.J_off;
    M33 R3so = k.R3 * skew(o);
    V3 nphi = (-2.0) * vtmul(n, R3so);  // n' * (-2 R3 skew(o))
    V3 r4w = vtmul(nphi, k.E);
    V3 hn = P.h * n;
    M33 dvc_dw = (-1.0) * (skew(rc) * k.R3);
    M33 dvc_dd = 2.0 * (skew(rc) * (k.R3 * skew(k.w))) - 2.0 * (skew(ww) * R3so);
    M33 W3 = dvc_dw + dvc_dd * k.E;
    V3 r6w = vtmul(t0, W3), r7w = vtmul(t1, W3);
    st3(Jm + 0, hn); st3(Jm + 3, r4w);
    st3(Jm + 6, v3zero()); st3(Jm + 9, v3zero());
    st3(Jm + 12, t0); st3(Jm + 15, r6w);
    st3(Jm + 18, t1); st3(Jm + 21, r7w);
    // G (6 x 4) = [X; R3' skew(rc) X]
    double* Gm = A + cd.G_off;
    V3 qn = tmul(k.R3, cross(rc, n)), q0 = tmul(k.R3, cross(rc, t0)), q1 = tmul(k.R3, cross(rc, t1));
    const double Gc[6][4] = {{n.x, 0.0, t0.x, t1.x}, {n.y, 0.0, t0.y, t1.y}, {n.z, 0.0, t0.z, t1.z},
                             {qn.x, 0.0, q0.x, q1.x}, {qn.y, 0.0, q0.y, q1.y}, {qn.z, 0.0, q0.z, q1.z}};
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) Gm[r * 4 + cc] = Gc[r][cc];
    // condensation onto the body:  dgamma = w0 - W J dv,  W = (D_c^-1)[gamma rows, constraint columns]  =>  D_b += G W J
    ContactBlock cb = contact_block(s, g, cd.mu);
    double Wm[4][4];
#pragma unroll
    for (int kx = 0; kx < 4; ++kx) {
      if (kx == 1) continue;  // J row 1 is zero
      double t[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8];
      t[4 + kx] = 1.0;
      contact_solve(cb, t, y);
#pragma unroll
      for (int r = 0; r < 4; ++r) Wm[r][kx] = y[4 + r];
    }
    const double Jr0[6] = {hn.x, hn.y, hn.z, r4w.x, r4w.y, r4w.z};
    const double Jr2[6] = {t0.x, t0.y, t0.z, r6w.x, r6w.y, r6w.z};
    const double Jr3[6] = {t1.x, t1.y, t1.z, r7w.x, r7w.y, r7w.z};
    double WJ[4][6];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int cc = 0; cc < 6; ++cc) WJ[r][cc] = Wm[r][0] * Jr0[cc] + Wm[r][2] * Jr2[cc] + Wm[r][3] * Jr3[cc];
    // d(G gamma)/d attitude, torque rows only: 2 skew(tau) + 2 R3' skew(F) R3 skew(o)   (impulse_map_jacobian)
    M33 K = 2.0 * skew(tau) + 2.0 * (transpose(k.R3) * (skew(F) * R3so));
    M33 KE = K * k.E;
    double* slotK = A + cd.slot + 6;  // the body does D_b -= slotK:  slotK = KE (angular block) - G W J
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int cc = 0; cc < 6; ++cc) {
        double v = -(Gc[r][0] * WJ[0][cc] + Gc[r][2] * WJ[2][cc] + Gc[r][3] * WJ[3][cc]);
        if (r >= 3 && cc >= 3) v += KE.m[r - 3][cc - 3];
        slotK[r * 6 + cc] = v;
      }
  }
}

// joints (joints/constraints.jl:114-299, joints/joint.jl, joints/limits.jl, rotational/dampers.jl)
// The limit slacks / duals (4 per limited axis) are condensed out analytically:
//   comp:  g' ds + s' dg = rc ;  slack_u: ds_u + a.dw = rs_u ;  slack_l: ds_l - a.dw = rs_l   (a.dw = aP.dw_p + aC.dw_c)
//   =>  dg_u - dg_l = c0 + (k_u + k_l) a.dw,   k = g'/s',  c0 = (rc_u - g_u' rs_u)/s_u' - (rc_l - g_l' rs_l)/s_l'
// and the bodies see  L dgamma = +-t (dg_u - dg_l): a rank-one coupling t (k_u + k_l) a' on the angular blocks.
template <bool JAC>
DJ_DEV void eval_joint(Ctx& c, int idx, double f, double* res, double& rv, double& bv) {
  const Plan& P = *c.P;
  double* A = c.A;
  const double* sol = A + P.sol_off;
  const double* dl = A + P.rhs_off;
  const JointDev& jd = c.joints[idx];
  V3 fl_p = v3zero(), fa_p = v3zero(), fl_c = v3zero(), fa_c = v3zero();  // G * eta (+ damper impulses)
  M33 Kaa = m33zero(), Kcc = m33zero();                                     // D_parent -= Kaa, D_child -= Kcc (angular blocks)
  M33 Bpc = m33zero(), Bcp = m33zero();                                     // (parent,child) / (child,parent) angular blocks
  bool coupled = false;
  Kin ka = body_kin(c, jd.parent, f), kb = body_kin(c, jd.child, f);
  JointGeom g = joint_geom(jd, ka.x3, ka.q3, ka.R3, kb.x3, kb.q3, kb.R3);
  const int n = joint_nq(jd);  // rows of the joint's node: ne equality multipliers + one kept limit dual per limited axis
  double* rr = res + jd.sol_off;
  const double* so = sol + jd.sol_off;
  const double* dd = dl + jd.sol_off;
  double* Uc = A + jd.Uc_off;
  double* Up = (jd.parent >= 0) ? A + jd.Up_off : nullptr;
  double* D = A + jd.D_off;
  M33 QtpE, QtcE, QrpE, QrcE;
  if (JAC) { QtpE = g.Qtp * ka.E; QtcE = g.Qtc * kb.E; QrpE = g.Qrp * ka.E; QrcE = g.Qrc * kb.E; }
  // translational equality rows: C_t e_t
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nl_t) {
      V3 ci = ld3(jd.Ct + 3 * i);
      double gi = dot(ci, g.et);
      rr[i] = -gi;
      rv = nanmax(rv, fabs(gi));
      if (JAC) {
        D[i * n + i] = kReg;
        st3(Uc + i * 6, P.h * vtmul(ci, g.Xc)); st3(Uc + i * 6 + 3, vtmul(ci, QtcE));
        if (Up) { st3(Up + i * 6, P.h * vtmul(ci, g.Xp)); st3(Up + i * 6 + 3, vtmul(ci, QtpE)); }
      }
    }
  }
  // rotational equality rows: C_r vec(qr)
  V3 er = qvec(g.qr);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nl_r) {
      V3 ci = ld3(jd.Cr + 3 * i);
      const int row = jd.nl_t + i;
      double gi = dot(ci, er);
      rr[row] = -gi;
      rv = nanmax(rv, fabs(gi));
      if (JAC) {
        D[row * n + row] = kReg;
        st3(Uc + row * 6, v3zero()); st3(Uc + row * 6 + 3, vtmul(ci, QrcE));
        if (Up) { st3(Up + row * 6, v3zero()); st3(Up + row * 6 + 3, vtmul(ci, QrpE)); }
      }
    }
  }
  // rotational limits: rows [s.gamma - mu (Nb); s_u - (hi - theta); s_l - (theta - lo)]   (joints/limits.jl:1-29)
#ifdef DJ_ANY_CONTACT
  if (jd.nb2_r > 0 && !(jd.flags & JF_LIM_TRA)) {
#else
  if (jd.nb2_r > 0) {
#endif
    V3 rvq = rotation_vector(g.qr);
    M33 Tp, Tc;
    if (JAC) {
      rotvec_attitude_jacobians(jd, g, Tp, Tc);
      Tp = Tp * ka.E;
      Tc = Tc * kb.E;
      coupled = true;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nb2_r) {
        V3 ai = ld3(jd.Ar + 3 * i);
        double th = dot(ai, rvq);
        const int is_u = jd.ne + i, is_l = jd.ne + jd.nb2_r + i;
        const int ig_u = is_u + jd.nb_r, ig_l = is_l + jd.nb_r;
        double su = so[is_u], sl = so[is_l], gu = so[ig_u], gl = so[ig_l];
        if (f != 0.0) { su += f * dd[is_u]; sl += f * dd[is_l]; gu += f * dd[ig_u]; gl += f * dd[ig_l]; }
        bv = nanmax(bv, nanmax(fabs(su * gu), fabs(sl * gl)));
        rr[is_u] = -(su * gu - c.mu);          // complementarity rows
        rr[is_l] = -(sl * gl - c.mu);
        rr[ig_u] = -(su - (jd.hi[i] - th));    // slack rows (stored at the gamma positions)
        rr[ig_l] = -(sl - (th - jd.lo[i]));
        double* lim = A + jd.lim_off + kLim * i;
        V3 tP = ld3(lim + 6), tC = ld3(lim + 9);
        // impulses of the limit duals: G[:, gamma_u] = -t, G[:, gamma_l] = +t
        fa_p += (gl - gu) * tP;
        fa_c += (gl - gu) * tC;
        if (JAC) {
          V3 aP = vtmul(ai, Tp), aC = vtmul(ai, Tc);
          st3(lim, aP); st3(lim + 3, aC);
          // Kept side A = the smaller slack (dojo_plan.h joint_nq): after ds_A = rs_A - sg a.dw its complementarity row reads
          //   s_A' dgamma_A - sg gamma_A' a.dw = rc_A - gamma_A' rs_A          (sg = +1 upper, -1 lower)
          // and is the node's row ne + i; the bodies see dgamma_A through the column sg t.  The other side I is condensed:
          //   dgamma_I = c_I + sg_I k_I a.dw,  k_I = gamma_I'/s_I'  =>  body rows gain  k_I t (aP.dw_p + aC.dw_c).
          const LimitSide ls = limit_side(su, sl, gu, gl);
          Kaa = Kaa - ls.kI * outer(tP, aP);
          Kcc = Kcc - ls.kI * outer(tC, aC);
          Bpc = Bpc + ls.kI * outer(tP, aC);
          Bcp = Bcp + ls.kI * outer(tC, aP);
          const int q = jd.ne + i;
          D[q * n + q] = ls.sA;
          st3(Uc + q * 6, v3zero()); st3(Uc + q * 6 + 3, (-ls.sg * ls.gA) * aC);
          if (Up) { st3(Up + q * 6, v3zero()); st3(Up + q * 6 + 3, (-ls.sg * ls.gA) * aP); }
          double* Lcw = A + jd.Lc_off;
          Lcw[0 * n + q] = 0.0; Lcw[1 * n + q] = 0.0; Lcw[2 * n + q] = 0.0;
          Lcw[3 * n + q] = ls.sg * tC.x; Lcw[4 * n + q] = ls.sg * tC.y; Lcw[5 * n + q] = ls.sg * tC.z;
          if (jd.parent >= 0) {  // pristine parent map G = -L (Lp is refreshed from it below)
            double* Gpw = A + jd.Gp_off;
            Gpw[0 * n + q] = 0.0; Gpw[1 * n + q] = 0.0; Gpw[2 * n + q] = 0.0;
            Gpw[3 * n + q] = -ls.sg * tP.x; Gpw[4 * n + q] = -ls.sg * tP.y; Gpw[5 * n + q] = -ls.sg * tP.z;
          }
        }
      }
    }
  }
#ifdef DJ_ANY_CONTACT
  double K6pp[36], K6cc[36], B6pc[36], B6cp[36];  // translational damper / limits: full 6 x 6 blocks (JF_FULL joints only)
  if (jd.flags & JF_FULL) {
#pragma unroll
    for (int i = 0; i < 36; ++i) { K6pp[i] = 0.0; K6cc[i] = 0.0; B6pc[i] = 0.0; B6cp[i] = 0.0; }
    eval_joint_tra<JAC>(c, jd, f, ka, kb, g, rr, so, dd, bv, fl_p, fa_p, fl_c, fa_c, K6pp, K6cc, B6pc, B6cp);
  }
#endif
  // impulses of the equality multipliers on the two bodies: G * lambda with the pristine maps (child: Lc = -G_c, parent: Gp)
  {
    const double* Lc = A + jd.Lc_off;
    const double* Gp = (jd.parent >= 0) ? A + jd.Gp_off : nullptr;
    double ac[6] = {0, 0, 0, 0, 0, 0}, ap[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < jd.ne; ++i) {  // equality columns only: the limit duals act through (gl - gu) t above
      double e = so[i];
      if (f != 0.0) e += f * dd[i];
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        ac[r] -= Lc[r * n + i] * e;
        if (Gp) ap[r] += Gp[r * n + i] * e;
      }
    }
    fl_c += v3(ac[0], ac[1], ac[2]); fa_c += v3(ac[3], ac[4], ac[5]);
    fl_p += v3(ap[0], ap[1], ap[2]); fa_p += v3(ap[3], ap[4], ap[5]);
    if (JAC && Gp) {  // parent-side lower block is consumed by the factorisation: refresh it from the pristine copy
      double* Lp = A + jd.Lp_off;
      for (int i = 0; i < 6 * n; ++i) Lp[i] = -Gp[i];
    }
  }
  // rotational damper (rotational/dampers.jl:4-27,66-84; rotational/minimal.jl:103-118,151-174)
  if (jd.damper_r != 0.0 && jd.nfree_r > 0) {
    Quat r = qmul(qinv(ka.q2), kb.q2);           // relative orientation at the current step
    Quat ma = qmap(ka.w, P.h), mb = qmap(kb.w, P.h);
    Quat left = qmul(mb, qinv(r));                // w = mb (x) r^-1 (x) conj(ma) (x) r
    Quat rest = qmul(qmul(qinv(r), qconj(ma)), r);
    Quat wq = qmul(mb, rest);
    V3 rvd = rotation_vector(wq);
    M33 AtA = m33zero();
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (i < jd.nfree_r) { V3 a = ld3(jd.Ar + 3 * i); AtA = AtA + outer(a, a); }
    M33 Roff = rotmat(ldq(jd.qoff));
    M33 Rr = rotmat(r);
    M33 B = jd.damper_r * (Roff * AtA);
    V3 ta = B * rvd;
    V3 tb = (-1.0) * tmul(Rr, ta);
    fa_p += ta;  // d -= damper_impulses  =>  res += impulses
    fa_c += tb;
    if (JAC) {
      coupled = true;
      M34 drv = drotation_vector_dq(wq);
      M33 dwa, dwb;  // d rotvec / d w_a, d w_b
      double m0a = ma.s, m0b = mb.s;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        V3 ek = v3(kx == 0 ? 1.0 : 0.0, kx == 1 ? 1.0 : 0.0, kx == 2 ? 1.0 : 0.0);
        Quat dmb = Quat{-(0.25 * P.h * P.h) * comp(kb.w, kx) / m0b, 0.5 * P.h * ek.x, 0.5 * P.h * ek.y, 0.5 * P.h * ek.z};
        Quat dma = Quat{-(0.25 * P.h * P.h) * comp(ka.w, kx) / m0a, 0.5 * P.h * ek.x, 0.5 * P.h * ek.y, 0.5 * P.h * ek.z};
        Quat cb = qmul(dmb, rest);
        Quat ca = qmul(qmul(left, qconj(dma)), r);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          dwb.m[i][kx] = drv.m[i][0] * cb.s + drv.m[i][1] * cb.x + drv.m[i][2] * cb.y + drv.m[i][3] * cb.z;
          dwa.m[i][kx] = drv.m[i][0] * ca.s + drv.m[i][1] * ca.x + drv.m[i][2] * ca.y + drv.m[i][3] * ca.z;
        }
      }
      M33 Ka = B * dwa, Kb = B * dwb;              // d tau_a / d w_a, d tau_a / d w_b
      M33 Rrt = transpose(Rr);
      Kaa = Kaa + Ka;                              // D_parent -= d tau_a / d w_a
      Kcc = Kcc - Rrt * Kb;                        // D_child  -= d tau_b / d w_b = -(Rr' Kb)
      Bpc = Bpc - Kb;                              // (parent,child) = -d tau_a / d w_b
      Bcp = Bcp + Rrt * Ka;                        // (child,parent) = -d tau_b / d w_a = +Rr' Ka
    }
  }
#ifdef DJ_ANY_CONTACT
  if (jd.flags & JF_FULL) {  // 6 x 6 slots and body-body blocks: the translational terms plus the angular 3 x 3 terms from above
    double* sc = A + jd.slot_c + c.sd;
    st3(sc, fl_c); st3(sc + 3, fa_c);
    double* sp = (jd.parent >= 0) ? A + jd.slot_p + c.sd : nullptr;
    if (sp) { st3(sp, fl_p); st3(sp + 3, fa_p); }
    if (JAC) {
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j2 = 0; j2 < 3; ++j2) {
          K6cc[(3 + i) * 6 + 3 + j2] += Kcc.m[i][j2]; K6pp[(3 + i) * 6 + 3 + j2] += Kaa.m[i][j2];
          B6pc[(3 + i) * 6 + 3 + j2] += Bpc.m[i][j2]; B6cp[(3 + i) * 6 + 3 + j2] += Bcp.m[i][j2];
        }
#pragma unroll
      for (int i = 0; i < 36; ++i) { sc[6 + i] = K6cc[i]; if (sp) sp[6 + i] = K6pp[i]; }
      if (jd.parent >= 0 && jd.BBpc_off >= 0) {
        double* Mpc = A + jd.BBpc_off;
        double* Mcp = A + jd.BBcp_off;
#pragma unroll
        for (int i = 0; i < 36; ++i) { Mpc[i] = B6pc[i]; Mcp[i] = B6cp[i]; }
      }
    }
    return;
  }
#endif
  if (JAC && coupled && jd.parent >= 0 && jd.BBpc_off >= 0) {
    // the coupling touches the angular rows / columns only: (parent angular rows, child) is stored 3 x 6, (child angular rows,
    // parent angular columns) 3 x 3 (dojo_plan.h ElimNb::row0); the linear columns of the former stay zero until the factorisation
    double* Mpc = A + jd.BBpc_off;
    double* Mcp = A + jd.BBcp_off;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j2 = 0; j2 < 3; ++j2) {
        Mpc[i * 6 + 3 + j2] = Bpc.m[i][j2];
        Mcp[i * 3 + j2] = Bcp.m[i][j2];
      }
  }
  write_slot(A + jd.slot_c + c.sd, fl_c, fa_c, Kcc);
  if (jd.parent >= 0) write_slot(A + jd.slot_p + c.sd, fl_p, fa_p, Kaa);
}

// ------------------------------------------------------------------------------------------------------------
// set_entries! of one joint on TWO lanes (round 2): lane 2k evaluates the CHILD side of joint k, lane 2k + 1 the PARENT side, with
// one instruction stream -- everything that differs between the sides is data (signs, selected matrices, table offsets), not control
// flow.  The joint pass is the longest lane-serial stretch of the assembly (~3 500 instructions per lane, the other warp waits for
// it half of the time); both lanes still need the kinematics of both bodies and the relative rotation, but each
// forms only ITS body's attitude Jacobian E, products with E, rows of (joint, body), angular blocks and impulse sums.  The two things
// a side needs from the other -- the limit row a' of the other body and the damper block of the other body -- travel through
// pair shuffles.  Same formulas, term by term, as eval_joint<true>(f = 0) (the set of floating-point operations per output is
// unchanged); used when a joint pass has at most 16 joints (ant, quadruped) and the mechanism has only NonlinearContact and rotational
// joint terms (Plan::jpair, set by dojo_create), otherwise one lane per joint as before.
// ------------------------------------------------------------------------------------------------------------
DJ_DEV M33 select33(bool p, const M33& a, const M33& b) {
  M33 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.m[i][j] = p ? a.m[i][j] : b.m[i][j];
  return r;
}
DJ_DEV V3 select3(bool p, V3 a, V3 b) { return V3{p ? a.x : b.x, p ? a.y : b.y, p ? a.z : b.z}; }
DJ_DEV V3 pair_swap3(unsigned pm, V3 v) { return V3{__shfl_xor_sync(pm, v.x, 1), __shfl_xor_sync(pm, v.y, 1), __shfl_xor_sync(pm, v.z, 1)}; }
DJ_DEV M33 pair_swap33(unsigned pm, const M33& a) {
  M33 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.m[i][j] = __shfl_xor_sync(pm, a.m[i][j], 1);
  return r;
}

DJ_DEV void eval_joint_pair(Ctx& c, int idx, const bool par, double* res, double& rv, double& bv) {
  const Plan& P = *c.P;
  double* A = c.A;
  const double* sol = A + P.sol_off;
  const JointDev& jd = c.joints[idx];
  const unsigned pm = 3u << (c.lane & ~1);     // the two lanes of this joint
  const bool act = !(par && jd.parent < 0);    // parent side of a joint to the origin: computes along, stores nothing
  const double sg_x = par ? -1.0 : 1.0;        // X = +-Ra', conj of the velocity-map perturbation, sign of the (., other) damper block
  Kin ka = body_kin(c, jd.parent, 0.0), kb = body_kin(c, jd.child, 0.0);  // (their E members are never read: dead code)
  JointGeom g = joint_geom(jd, ka.x3, ka.q3, ka.R3, kb.x3, kb.q3, kb.R3);
  const V3 wm = select3(par, ka.w, kb.w);
  const M33 E = attitude_velocity_jacobian(wm, P.h);  // of THIS side's body
  const M33 Qt = select33(par, g.Qtp, g.Qtc), Qr = select33(par, g.Qrp, g.Qrc);
  const M33 X = sg_x * g.Xc;  // Xc = Ra', Xp = -Ra'
  const M33 QtE = Qt * E, QrE = Qr * E;
  V3 fl = v3zero(), fa = v3zero();
  M33 K = m33zero(), Bx = m33zero();  // D_mine -= K ; (mine, other) angular block
  bool coupled = false;
  const int n = joint_nq(jd);
  double* rr = res + jd.sol_off;
  const double* so = sol + jd.sol_off;
  const bool pa = par && act;                     // (an inactive parent lane reads the child's tables: harmless, nothing is stored)
  double* U = A + (pa ? jd.Up_off : jd.Uc_off);   // (joint, this body) n x 6
  double* D = A + jd.D_off;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nl_t) {
      V3 ci = ld3(jd.Ct + 3 * i);
      double gi = dot(ci, g.et);
      rv = nanmax(rv, fabs(gi));
      if (!par) { rr[i] = -gi; D[i * n + i] = kReg; }
      if (act) { st3(U + i * 6, P.h * vtmul(ci, X)); st3(U + i * 6 + 3, vtmul(ci, QtE)); }
    }
  }
  V3 er = qvec(g.qr);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nl_r) {
      V3 ci = ld3(jd.Cr + 3 * i);
      const int row = jd.nl_t + i;
      double gi = dot(ci, er);
      rv = nanmax(rv, fabs(gi));
      if (!par) { rr[row] = -gi; D[row * n + row] = kReg; }
      if (act) { st3(U + row * 6, v3zero()); st3(U + row * 6 + 3, vtmul(ci, QrE)); }
    }
  }
  double* mapm = A + (pa ? jd.Gp_off : jd.Lc_off);  // pristine impulse map of this side: parent G_p, child L_c = -G_c
  if (jd.nb2_r > 0) {  // rotational limits (joints/limits.jl:1-29), see eval_joint
    V3 rvq = rotation_vector(g.qr);
    M33 T;  // d rotation_vector(qr) / d attitude of this body (rotvec_attitude_jacobians, one side), times E
    {
      M34 drv = drotation_vector_dq(g.qr);
      V3 vr = qvec(g.qr);
      M33 Rofft = transpose(rotmat(ldq(jd.qoff)));
      V3 srow = select3(par, vtmul(vr, Rofft), -vr);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        V3 dv = v3(drv.m[i][1], drv.m[i][2], drv.m[i][3]);
        V3 r1 = drv.m[i][0] * srow + vtmul(dv, Qr);
        T.m[i][0] = r1.x; T.m[i][1] = r1.y; T.m[i][2] = r1.z;
      }
      T = T * E;
    }
    coupled = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nb2_r) {
        V3 ai = ld3(jd.Ar + 3 * i);
        double th = dot(ai, rvq);
        const int is_u = jd.ne + i, is_l = jd.ne + jd.nb2_r + i;
        const int ig_u = is_u + jd.nb_r, ig_l = is_l + jd.nb_r;
        const double su = so[is_u], sl = so[is_l], gu = so[ig_u], gl = so[ig_l];
        bv = nanmax(bv, nanmax(fabs(su * gu), fabs(sl * gl)));
        if (!par) {
          rr[is_u] = -(su * gu - c.mu);
          rr[is_l] = -(sl * gl - c.mu);
          rr[ig_u] = -(su - (jd.hi[i] - th));
          rr[ig_l] = -(sl - (th - jd.lo[i]));
        }
        double* lim = A + jd.lim_off + kLim * i;
        const V3 tm = ld3(lim + (par ? 6 : 9));  // tP / tC
        fa += (gl - gu) * tm;
        const V3 am = vtmul(ai, T);              // aP / aC
        if (act) st3(lim + (par ? 0 : 3), am);
        const V3 ao = pair_swap3(pm, am);        // the other body's row
        const LimitSide ls = limit_side(su, sl, gu, gl);
        K = K - ls.kI * outer(tm, am);
        Bx = Bx + ls.kI * outer(tm, ao);
        const int q = jd.ne + i;
        if (!par) D[q * n + q] = ls.sA;
        if (act) {
          st3(U + q * 6, v3zero()); st3(U + q * 6 + 3, (-ls.sg * ls.gA) * am);
          const V3 col = (sg_x * ls.sg) * tm;   // L_c column +sg tC, G_p column -sg tP
          mapm[0 * n + q] = 0.0; mapm[1 * n + q] = 0.0; mapm[2 * n + q] = 0.0;
          mapm[3 * n + q] = col.x; mapm[4 * n + q] = col.y; mapm[5 * n + q] = col.z;
        }
      }
    }
  }
  {  // impulses of the equality multipliers on this body: child -L_c lambda, parent +G_p lambda
    double acc[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < jd.ne; ++i) {
      const double e = so[i];
#pragma unroll
      for (int r = 0; r < 6; ++r) acc[r] += mapm[r * n + i] * e;
    }
    fl += (-sg_x) * v3(acc[0], acc[1], acc[2]);
    fa += (-sg_x) * v3(acc[3], acc[4], acc[5]);
    if (jd.parent >= 0) {  // refresh the parent-side lower block from the pristine copy: the two lanes share the copy
      double* Lp = A + jd.Lp_off;
      const double* Gp = A + jd.Gp_off;
      for (int i = (par ? 1 : 0); i < 6 * n; i += 2) Lp[i] = -Gp[i];
    }
  }
  if (jd.damper_r != 0.0 && jd.nfree_r > 0) {  // rotational damper, see eval_joint
    Quat r = qmul(qinv(ka.q2), kb.q2);
    Quat ma = qmap(ka.w, P.h), mb = qmap(kb.w, P.h);
    Quat left = qmul(mb, qinv(r));
    Quat rest = qmul(qmul(qinv(r), qconj(ma)), r);
    Quat wq = qmul(mb, rest);
    V3 rvd = rotation_vector(wq);
    M33 AtA = m33zero();
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (i < jd.nfree_r) { V3 a = ld3(jd.Ar + 3 * i); AtA = AtA + outer(a, a); }
    M33 Roff = rotmat(ldq(jd.qoff));
    M33 Rr = rotmat(r);
    M33 B = jd.damper_r * (Roff * AtA);
    V3 ta = B * rvd;
    V3 tb = (-1.0) * tmul(Rr, ta);
    fa += select3(par, ta, tb);
    coupled = true;
    M34 drv = drotation_vector_dq(wq);
    // d w / d (this body's angular velocity): the perturbed velocity map dm sits between Xq and Yq,
    //   parent: w = left (x) conj(ma) (x) r  ->  left (x) conj(dm) (x) r ;   child: w = mb (x) rest  ->  dm (x) rest
    const double m0 = par ? ma.s : mb.s;
    const Quat Xq = par ? left : Quat{1.0, 0.0, 0.0, 0.0};
    const Quat Yq = par ? r : rest;
    M33 dw;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const double hv = sg_x * 0.5 * P.h;  // conj() flips the vector part on the parent side
      Quat dm = Quat{-(0.25 * P.h * P.h) * comp(wm, kx) / m0, kx == 0 ? hv : 0.0, kx == 1 ? hv : 0.0, kx == 2 ? hv : 0.0};
      Quat cq = qmul(qmul(Xq, dm), Yq);
#pragma unroll
      for (int i = 0; i < 3; ++i) dw.m[i][kx] = drv.m[i][0] * cq.s + drv.m[i][1] * cq.x + drv.m[i][2] * cq.y + drv.m[i][3] * cq.z;
    }
    const M33 Km = B * dw;                  // parent: Ka = d tau_a / d w_a ; child: Kb = d tau_a / d w_b
    const M33 Ko = pair_swap33(pm, Km);     // the other side's block
    const M33 Rrt = transpose(Rr);
    // parent: Kaa += Ka, Bpc -= Kb ;  child: Kcc -= Rr' Kb, Bcp += Rr' Ka
    const M33 N = select33(par, m33ident(), Rrt);
    K = K + (-sg_x) * (N * Km);
    Bx = Bx + sg_x * (N * Ko);
  }
  if (coupled && jd.parent >= 0 && jd.BBpc_off >= 0) {  // (parent angular rows, child) 3 x 6 ; (child angular rows, parent angular columns) 3 x 3
    double* M = A + (par ? jd.BBpc_off + 3 : jd.BBcp_off);
    const int ldm = par ? 6 : 3;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j2 = 0; j2 < 3; ++j2) M[i * ldm + j2] = Bx.m[i][j2];
  }
  if (act) write_slot(A + (par ? jd.slot_p : jd.slot_c), fl, fa, K);
}

// condense_rhs / recover: the per-solve halves of the analytic condensation.  `x` is a right-hand side in solution
// ordering.  condense_rhs writes each node's contribution to its bodies' rows into the slots (gathered by the bodies
// right after); recover overwrites the condensed-out entries of x with the step (ds, dgamma) once dv is known.
DJ_DEV void condense_contact(Ctx& c, int idx, const double* x) {
  const Plan& P = *c.P;
  double* A = c.A;
  const ContactDev& cd = c.contacts[idx];
#ifdef DJ_ANY_CONTACT
  if (contact_type(cd) != 2) { condense_contact_orthant(c, idx, x); return; }
#endif
  const double* so = A + P.sol_off + cd.sol_off;
  ContactBlock cb = contact_block(so, so + 4, cd.mu);
  double y[8];
  contact_solve(cb, x + cd.sol_off, y);  // w0 = y[4:8]:  r_b += G w0
  const double* G = A + cd.G_off;
  double o[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) o[r] = G[r * 4 + 0] * y[4] + G[r * 4 + 2] * y[6] + G[r * 4 + 3] * y[7];
  double* s = A + cd.slot;
#pragma unroll
  for (int r = 0; r < 6; ++r) s[r] = o[r];
}
DJ_DEV void recover_contact(Ctx& c, int idx, double* x) {
  const Plan& P = *c.P;
  double* A = c.A;
  const ContactDev& cd = c.contacts[idx];
#ifdef DJ_ANY_CONTACT
  if (contact_type(cd) != 2) { recover_contact_orthant(c, idx, x); return; }
#endif
  const double* so = A + P.sol_off + cd.sol_off;
  ContactBlock cb = contact_block(so, so + 4, cd.mu);
  const double* J = A + cd.J_off;
  const double* dv = x + c.bodies[cd.body].sol_off;
  double t[8], y[8];
#pragma unroll
  for (int r = 0; r < 4; ++r) t[r] = x[cd.sol_off + r];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) acc += J[r * 6 + k] * dv[k];
    t[4 + r] = x[cd.sol_off + 4 + r] - acc;
  }
  contact_solve(cb, t, y);
#pragma unroll
  for (int r = 0; r < 8; ++r) x[cd.sol_off + r] = y[r];
}
DJ_DEV void condense_joint(Ctx& c, int idx, double* x) {
  const Plan& P = *c.P;
  double* A = c.A;
  const JointDev& jd = c.joints[idx];
#ifdef DJ_ANY_CONTACT
  if (jd.flags & JF_LIM_TRA) { condense_joint_tra(c, jd, x); return; }
#endif
  V3 tp = v3zero(), tc = v3zero();
  const double* so = A + P.sol_off + jd.sol_off;
  double* xr = x + jd.sol_off;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nb2_r) {
      const int is_u = jd.ne + i, is_l = jd.ne + jd.nb2_r + i, ig_u = is_u + jd.nb_r, ig_l = is_l + jd.nb_r;
      const LimitSide ls = limit_side(so[is_u], so[is_l], so[ig_u], so[ig_l]);
      const double rc_u = xr[is_u], rc_l = xr[is_l], rs_u = xr[ig_u], rs_l = xr[ig_l];
      // condensed side I: dgamma_I = c_I + sg_I k_I a.dw;  the body rows carry sg_I t dgamma_I  =>  rhs -= sg_I c_I t
      const double cI = ((ls.up ? rc_l : rc_u) - ls.gI * (ls.up ? rs_l : rs_u)) / ls.sI;
      const double w = ls.sg * cI;  // sg_I = -sg
      const double* lim = A + jd.lim_off + kLim * i;
      tp += w * ld3(lim + 6);
      tc += w * ld3(lim + 9);
      // kept side A: right-hand side of its row (position ne + i of the node); rc of the condensed side is kept at is_l for recover
      xr[is_u] = (ls.up ? rc_u : rc_l) - ls.gA * (ls.up ? rs_u : rs_l);
      if (!ls.up) xr[is_l] = rc_u;
    }
  }
  double* sc = A + jd.slot_c;
  st3(sc, v3zero()); st3(sc + 3, tc);
  if (jd.parent >= 0) { double* sp = A + jd.slot_p; st3(sp, v3zero()); st3(sp + 3, tp); }
}
DJ_DEV void recover_joint(Ctx& c, int idx, double* x) {
  const Plan& P = *c.P;
  double* A = c.A;
  const JointDev& jd = c.joints[idx];
  if (jd.nb2_r == 0) return;
#ifdef DJ_ANY_CONTACT
  if (jd.flags & JF_LIM_TRA) { recover_joint_tra(c, jd, x); return; }
#endif
  const double* so = A + P.sol_off + jd.sol_off;
  double* xr = x + jd.sol_off;
  V3 wp = (jd.parent >= 0) ? ld3(x + c.bodies[jd.parent].sol_off + 3) : v3zero();
  V3 wc = ld3(x + c.bodies[jd.child].sol_off + 3);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nb2_r) {
      const int is_u = jd.ne + i, is_l = jd.ne + jd.nb2_r + i, ig_u = is_u + jd.nb_r, ig_l = is_l + jd.nb_r;
      const LimitSide ls = limit_side(so[is_u], so[is_l], so[ig_u], so[ig_l]);
      const double* lim = A + jd.lim_off + kLim * i;
      const double adw = dot(ld3(lim), wp) + dot(ld3(lim + 3), wc);
      const double dgA = xr[is_u], rcI = xr[is_l], rs_u = xr[ig_u], rs_l = xr[ig_l];
      const double ds_u = rs_u - adw, ds_l = rs_l + adw;
      const double dgI = (rcI - ls.gI * (ls.up ? ds_l : ds_u)) / ls.sI;
      xr[is_u] = ds_u;
      xr[is_l] = ds_l;
      xr[ig_u] = ls.up ? dgA : dgI;
      xr[ig_l] = ls.up ? dgI : dgA;
    }
  }
}

// SMALL: every joint pass takes eval_joint_pair, so that eval_joint<true> is not instantiated.
template <bool JAC, bool SMALL = false>
DJ_DEV void evaluate(Ctx& c, double f, int res_off, double& rvio, double& bvio) {
  const Plan& P = *c.P;
  double* A = c.A;
  double* res = A + res_off;
  const WarpRole& role = c.roles[c.warp];
  double rv = 0.0, bv = 0.0;
  if (JAC) {  // all KKT blocks are rewritten: zero the matrix region cooperatively, then scatter the non-zeros
    for (int t = c.tid; t < P.mat_len; t += c.nthreads) A[P.mat_off + t] = 0.0;
    slot_sync(c);
  }
  for (int p = 0; p < role.npass; ++p) {
    if (JAC && role.type[p] == ROLE_JOINT && (SMALL || (P.jpair && role.count[p] <= 16))) {  // set_entries! of the joints on two lanes each (f = 0)
      if ((c.lane >> 1) < role.count[p]) eval_joint_pair(c, role.first[p] + (c.lane >> 1), (c.lane & 1) != 0, res, rv, bv);
      continue;
    }
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_BODY) eval_body<JAC>(c, idx, f, res);
    else if (role.type[p] == ROLE_CONTACT) eval_contact<JAC>(c, idx, f, res, rv, bv);
    else if (!(SMALL && JAC)) eval_joint<JAC>(c, idx, f, res, rv, bv);
  }
#ifdef DJ_PROFILE
  long long _rw0 = clock64();
#endif
  slot_sync(c);
#ifdef DJ_PROFILE
  c.t_rolewait += clock64() - _rw0;
#endif
  // gather the impulse contributions of the incident joints / contacts into the body rows (fixed order)
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, c.lane);
    if (idx < 0 || role.type[p] != ROLE_BODY) continue;
    const BodyDev& bd = c.bodies[idx];
    double* rb = res + bd.sol_off;
    double* D = A + bd.D_off;
    for (int g = 0; g < bd.g_cnt; ++g) {
      const double* s = A + DJ_SLOT_OFF(c.ilist[bd.g_off + g]);
      add3(rb, ld3(s));
      add3(rb + 3, ld3(s + 3));
      if (JAC) {
#ifdef DJ_ANY_CONTACT
        if (g < bd.g_ncontact || DJ_SLOT_FULL(c.ilist[bd.g_off + g])) {
#else
        if (g < bd.g_ncontact) {
#endif
#pragma unroll
          for (int i = 0; i < 36; ++i) D[i] -= s[6 + i];
        } else {
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) D[(3 + i) * 6 + 3 + j] -= s[6 + 3 * i + j];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) rv = nanmax(rv, fabs(rb[i]));
  }
  block_nanmax2<SMALL>(c, rv, bv);
  rvio = rv;
  bvio = bv;
  slot_sync(c);
}

// Residual-only evaluation for the line search (solver/line_search.jl:1-34) at sol + fk * delta.
// Mechanisms whose role passes have at most 16 nodes (P.ls_pair) run it on the lower half-warps; with `pair` the upper
// half-warps evaluate the NEXT trial (fk / 2) at the same time with the same instruction stream: its residual goes to a
// scratch vector and its contribution slots to a shadow copy, both inside the matrix region, which is dead between the
// solves and the next assembly.  A pass with both halves busy costs about the same as a single trial; an environment that stalls (ten trials per
// iteration) needs five passes instead of ten, one rejection costs no extra pass.
// `W` is the arena that receives everything this evaluation writes (trial residuals, contribution slots, reduction scratch): the
// slot's own arena, or -- when a drained slot evaluates trials of another slot's environment (ls_assist_loop) -- the helper's arena
// while c.A points at the owner's (iterate, direction, per-step constants: read only).
template <bool SMALL = false>
DJ_DEV void evaluate_ls(Ctx& c, double* W, double fk, bool pair, double& rvA, double& bvA, double& rvB, double& bvB) {
  const Plan& P = *c.P;
  double* A = c.A;
  const WarpRole& role = c.roles[c.warp];
  const bool pl = SMALL || P.ls_pair != 0;
  const int half = pl ? (c.lane >> 4) : 0;
  const int ln = pl ? (c.lane & 15) : c.lane;
  const bool on = (half == 0) || pair;
  const double f = half ? 0.5 * fk : fk;
  double* res = W + (half ? P.ls_res2_off : P.sav_off);
  c.sd = (int)(W - A) + (half ? P.ls_slot_delta : 0);
  double rv = 0.0, bv = 0.0;
  for (int p = 0; p < role.npass; ++p) {
    const int idx = on ? role_item(role, p, ln) : -1;
    if (idx < 0) continue;
    if (role.type[p] == ROLE_BODY) eval_body<false>(c, idx, f, res);
    else if (role.type[p] == ROLE_CONTACT) eval_contact<false>(c, idx, f, res, rv, bv);
    else eval_joint<false>(c, idx, f, res, rv, bv);
  }
  slot_sync(c);
  for (int p = 0; p < role.npass; ++p) {  // gather the impulse contributions into the body rows (fixed order)
    const int idx = on ? role_item(role, p, ln) : -1;
    if (idx < 0 || role.type[p] != ROLE_BODY) continue;
    const BodyDev& bd = c.bodies[idx];
    double* rb = res + bd.sol_off;
    for (int g = 0; g < bd.g_cnt; ++g) {
      const double* s = A + DJ_SLOT_OFF(c.ilist[bd.g_off + g]) + c.sd;
      add3(rb, ld3(s));
      add3(rb + 3, ld3(s + 3));
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) rv = nanmax(rv, fabs(rb[i]));
  }
  c.sd = 0;
  // violations per trial: reduce inside the 16-lane halves, then over the warps
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) {
    rv = nanmax(rv, __shfl_xor_sync(0xffffffffu, rv, o));
    bv = nanmax(bv, __shfl_xor_sync(0xffffffffu, bv, o));
  }
  if (!pl) {
    rv = nanmax(rv, __shfl_xor_sync(0xffffffffu, rv, 16));
    bv = nanmax(bv, __shfl_xor_sync(0xffffffffu, bv, 16));
  }
  double* red = W + P.red_off;
  if ((c.lane & 15) == 0) { red[4 * c.warp + 2 * (c.lane >> 4)] = rv; red[4 * c.warp + 2 * (c.lane >> 4) + 1] = bv; }
  slot_sync(c);
  rvA = red[0]; bvA = red[1]; rvB = red[2]; bvB = red[3];
  for (int w = 1; w < slot_warps<SMALL>(c); ++w) {
    rvA = nanmax(rvA, red[4 * w]); bvA = nanmax(bvA, red[4 * w + 1]);
    rvB = nanmax(rvB, red[4 * w + 2]); bvB = nanmax(bvB, red[4 * w + 3]);
  }
  slot_sync(c);
}

// ------------------------------------------------------------------------------------------------------------
// Block LDU (GraphBasedSystems.ldu_factorization! / ldu_backsubstitution!), phase-parallel over the warps
// ------------------------------------------------------------------------------------------------------------
// The LDU program of the plan (dojo_plan.h LduOp): cnt[ph * nw + w] and, after them, wfirst[w]; op k is three 16-byte words
DJ_DEV const int* ldu_cnt(const Ctx& c) { return c.sched + c.P->prog_cnt; }
DJ_DEV const int4* ldu_op(const Ctx& c, int k) { return reinterpret_cast<const int4*>(c.sched + c.P->prog_ops) + 3 * k; }
// arena offset of the j-th scratch record folded into the step of op word 0 `h` (the first kLduFold are inline)
DJ_DEV int ldu_fold(const Ctx& c, int4 h, int j) {
  return j == 0 ? hi16(h.z) : j == 1 ? lo16(h.w) : j == 2 ? hi16(h.w) : c.ilist[lo16(h.z) + j];
}
static_assert(kLduFold == 3, "ldu_fold names three inline fold sources");

template <bool SMALL = false>
DJ_DEV bool factorize(Ctx& c) {
  const Plan& P = *c.P;
  double* A = c.A;
  bool ok = true;
  // the two halves of a warp eliminate two steps of the phase at the same time (blocks are at most 6 x 6: 12 lanes busy)
  const int half = c.lane >> 4, l = c.lane & 15;
  const unsigned mask = 0xffffu << (16 * half);
  const int nw = slot_warps<SMALL>(c);
  const int* cnt = ldu_cnt(c);
  int k = cnt[P.nphase * nw + c.warp];  // this warp's first op of the phase
#ifdef DJ_PROFILE
  c.f_last = clock64();
#endif
  for (int ph = 0; ph < P.nphase; ++ph) {
    const int sn = cnt[ph * nw + c.warp];
    for (int s = half; s < sn; s += 2) {
      const int4* q = ldu_op(c, k + s);
      const int4 h = q[0];
      const int n = byte_of(h.y, 0), nnb = byte_of(h.y, 1), fold_cnt = hi16(h.y);
      double* Dc = A + lo16(h.x);
      if (fold_cnt > 0) {  // fold the children's scratch updates into D_c
        for (int t = l; t < n * n; t += 16) {
          double acc = Dc[t];
          for (int j = 0; j < fold_cnt; ++j) acc += A[ldu_fold(c, h, j) + t];
          Dc[t] = acc;
        }
        __syncwarp(mask);
      }
      DJ_FTICK(c, f_fold)
      ok = block_inverse(Dc, n, n, l, mask) && ok;                                                        // D_c <- D_c^-1
      DJ_FTICK(c, f_inv)
      for (int i = 0; i < nnb; ++i) {                                                                     // L~_ic = M_ic D_c^-1
        const int4 a = q[1 + i];
        right_multiply_inplace(A + lo16(a.x), Dc, byte_of(a.z, 0), n, l, mask);
      }
      DJ_FTICK(c, f_rm)
      for (int i = 0; i < nnb; ++i)
        for (int j = 0; j < nnb; ++j) {                                                                   // M_ij -= L~_ic M_cj
          const int4 ai = q[1 + i], aj = q[1 + j];
          schur_update(A + (j ? hi16(ai.w) : lo16(ai.w)), byte_of(aj.z, 3), A + lo16(ai.x) + byte_of(aj.z, 1), n, A + hi16(aj.y), byte_of(ai.z, 0),
                       byte_of(aj.z, 2), byte_of(aj.z, 0), l, mask);
        }
      DJ_FTICK(c, f_schur)
    }
    k += sn;
    slot_sync(c);
    DJ_FTICK(c, f_bar)
  }
  // all warps of the slot agree on the outcome
  int* flag = (int*)(A + P.red_off);
  const bool wok = __all_sync(0xffffffffu, ok);
  if (c.lane == 0) flag[c.warp] = wok ? 1 : 0;
  slot_sync(c);
  bool all = true;
  for (int w = 0; w < slot_warps<SMALL>(c); ++w) all = all && (flag[w] != 0);
  slot_sync(c);
  return all;
}

// dot product of length n <= 6 (blocks of the condensed system are at most 6 wide): unrolled and predicated, so that the
// twelve shared-memory loads are issued back to back instead of one dependent loop iteration at a time
DJ_DEV double dot6(const double* a, const double* b, int n) {
  double e = 0.0, o = 0.0;  // two interleaved FMA chains
#pragma unroll
  for (int k = 0; k < 6; k += 2) {
    if (k < n) e = fma(a[k], b[k], e);
    if (k + 1 < n) o = fma(a[k + 1], b[k + 1], o);
  }
  return e + o;
}

// x <- KKT^{-1} x for the vector at arena offset vec_off (solution ordering)
template <bool SMALL = false>
DJ_DEV void solve(Ctx& c, int vec_off) {
  const Plan& P = *c.P;
  double* A = c.A;
  double* x = A + vec_off;
  const int lane = c.lane;
  const int half = lane >> 4, l = lane & 15;  // one elimination step per half-warp, as in factorize()
  const int sub = l >> 3, li = l & 7;         // forward substitution: lanes [0,8) of the group serve nb[0], [8,16) nb[1]
  const WarpRole& role = c.roles[c.warp];
#ifdef DJ_PROFILE
  c.f_last = clock64();
#endif
  // condense the right-hand side of the contact / joint-limit rows onto the body rows
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_CONTACT) condense_contact(c, idx, x);
    else if (role.type[p] == ROLE_JOINT) condense_joint(c, idx, x);
  }
  DJ_FTICK(c, s_cond)
  slot_sync(c);
  DJ_FTICK(c, s_bar)
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, lane);
    if (idx < 0 || role.type[p] != ROLE_BODY) continue;
    const BodyDev& bd = c.bodies[idx];
    double* xb = x + bd.sol_off;
    for (int g = 0; g < bd.g_cnt; ++g) {
      const double* s = A + DJ_SLOT_OFF(c.ilist[bd.g_off + g]);
      add3(xb, ld3(s));
      add3(xb + 3, ld3(s + 3));
    }
  }
  DJ_FTICK(c, s_cond)
  slot_sync(c);
  DJ_FTICK(c, s_bar)
  // The two halves of a warp take two steps of a phase with one instruction stream.  Both halves run the same number of loop
  // iterations (a half without a step of its own looks at its partner's and stores nothing), so the warp stays converged and the
  // intra-step synchronisation is the plain full-warp one: a __syncwarp / shuffle whose member mask DIFFERS between the lanes of one
  // instruction (one 16-lane mask per half) is split into groups with MATCH.ANY by the compiler, whose sequences stall the warp.
  // The ops of this warp are walked with a running index k (its first op of the phase): up through the phases, then back down.
  const int nw = slot_warps<SMALL>(c);
  const int* cnt = ldu_cnt(c);
  int k = cnt[P.nphase * nw + c.warp];
  for (int ph = 0; ph < P.nphase; ++ph) {  // forward: z_i -= L~_ic z_c
    const int sn = cnt[ph * nw + c.warp];
    for (int it = 0; 2 * it < sn; ++it) {
      const bool act = 2 * it + half < sn;
      const int4* q = ldu_op(c, k + 2 * it + (act ? half : 0));
      const int4 h = q[0];
      const int n = byte_of(h.y, 0), fold_cnt = hi16(h.y);
      double* xc = x + hi16(h.x);
      if (act && fold_cnt > 0 && l < n) {  // fold (and clear) the children's forward updates of this body
        double acc = xc[l];
        for (int j = 0; j < fold_cnt; ++j) {
          double* v = A + ldu_fold(c, h, j) + 36;
          acc += v[l];
          v[l] = 0.0;
        }
        xc[l] = acc;
      }
      __syncwarp();
      if (act && sub < byte_of(h.y, 1)) {
        const int4 a = q[1 + sub];  // neighbour `sub`
        if (li < byte_of(a.z, 0)) {
          const double* L = A + lo16(a.x) + li * n;
          const double acc = dot6(L, xc, n);
          double* tgt = hi16(a.x) != kLduNone ? A + hi16(a.x) : x + lo16(a.y);
          tgt[li] -= acc;
        }
      }
      __syncwarp();
    }
    k += sn;
    DJ_FTICK(c, s_fwd)
    slot_sync(c);
    DJ_FTICK(c, s_bar)
  }
  for (int ph = P.nphase - 1; ph >= 0; --ph) {  // backward: x_c = D_c^-1 (z_c - sum_j M_cj x_j)
    // same pairing as the forward sweep, last pair first (the steps of one phase are independent)
    const int sn = cnt[ph * nw + c.warp];
    k -= sn;
    for (int it = (sn + 1) / 2 - 1; it >= 0; --it) {
      const bool act = 2 * it + half < sn;
      const int4* q = ldu_op(c, k + 2 * it + (act ? half : 0));
      const int4 h = q[0];
      const int n = byte_of(h.y, 0), nnb = byte_of(h.y, 1);
      const double* Dc = A + lo16(h.x);
      double* xc = x + hi16(h.x);
      if (act && nnb > 0 && l < n) {
        double acc = 0.0;
        for (int j = 0; j < nnb; ++j) {
          const int4 a = q[1 + j];
          const int nn = byte_of(a.z, 0), r = l - byte_of(a.z, 1);
          if (r >= 0 && r < byte_of(a.z, 2)) {
            acc += dot6(A + hi16(a.y) + r * nn, x + lo16(a.y), nn);
          }
        }
        xc[l] -= acc;
      }
      __syncwarp();
      double acc = 0.0;
      if (act && l < n) acc = dot6(Dc + l * n, xc, n);
      __syncwarp();
      if (act && l < n) xc[l] = acc;
      __syncwarp();
    }
    DJ_FTICK(c, s_bwd)
    slot_sync(c);
    DJ_FTICK(c, s_bar)
  }
  // recover the condensed-out steps (ds, dgamma) of the contacts and joint limits
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_CONTACT) recover_contact(c, idx, x);
    else if (role.type[p] == ROLE_JOINT) recover_joint(c, idx, x);
  }
  DJ_FTICK(c, s_rec)
  slot_sync(c);
  DJ_FTICK(c, s_bar)
}

// ------------------------------------------------------------------------------------------------------------
// cone_line_search! (solver/line_search.jl:36-139)
// ------------------------------------------------------------------------------------------------------------
DJ_DEV double ort_step(double lam, double dl, double tau) { return dl < 0.0 ? fmin(1.0, -tau * lam / dl) : 1.0; }
DJ_DEV double soc_step(double l0, double l1, double l2, double d0, double d1, double d2, double tau) {
  const double eps = 1e-14;
  double ll = fmax(l0 * l0 - (l1 * l1 + l2 * l2), 1e-25) + eps;
  double ld = l0 * d0 - (l1 * d1 + l2 * d2) + eps;
  double rs = ld / ll;
  double sq = sqrt(ll);
  double fct = (ld / sq + d0) / (l0 / sq + 1.0);
  double r1 = d1 / sq - fct * l1 / ll;
  double r2 = d2 / sq - fct * l2 / ll;
  double nr = sqrt(r1 * r1 + r2 * r2);
  return (nr - rs > 0.0) ? fmin(1.0, tau / (nr - rs)) : 1.0;
}
template <bool SMALL = false>
DJ_DEV double cone_line_search(Ctx& c, double tau_ort, double tau_soc) {
  const Plan& P = *c.P;
  const double* sol = c.A + P.sol_off;
  const double* dl = c.A + P.rhs_off;
  const WarpRole& role = c.roles[c.warp];
  double a = 1.0;
  for (int p = 0; p < role.npass; ++p) {
#ifndef DJ_ANY_CONTACT
    // NonlinearContact: the slack cone and the dual cone of a contact are two independent (orthant, second-order cone) pairs with the
    // same formulas -- two lanes per contact, lane 2k the slacks, lane 2k + 1 the duals (half the chain of divisions / square roots)
    if (role.type[p] == ROLE_CONTACT && role.count[p] <= 16) {
      const int ci = c.lane >> 1;
      if (ci < role.count[p]) {
        const ContactDev& cd = c.contacts[role.first[p] + ci];
        const int o = cd.sol_off + 4 * (c.lane & 1);
        const double* v = sol + o;
        const double* dv = dl + o;
        a = fmin(a, ort_step(v[0], dv[0], tau_ort));
        a = fmin(a, soc_step(v[1], v[2], v[3], dv[1], dv[2], dv[3], tau_soc));
      }
      continue;
    }
#endif
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_CONTACT) {
      const ContactDev& cd = c.contacts[idx];
      const double* s = sol + cd.sol_off;
#ifdef DJ_ANY_CONTACT
      if (contact_type(cd) != 2) {  // impact / linear: positive orthant only (line_search.jl:71-86)
        const int n2 = 2 * contact_nh(cd);
        for (int i = 0; i < n2; ++i) a = fmin(a, ort_step(s[i], dl[cd.sol_off + i], tau_ort));
        continue;
      }
#endif
      const double* g = s + 4;
      const double* ds = dl + cd.sol_off;
      const double* dg = ds + 4;
      a = fmin(a, ort_step(s[0], ds[0], tau_ort));
      a = fmin(a, ort_step(g[0], dg[0], tau_ort));
      a = fmin(a, soc_step(s[1], s[2], s[3], ds[1], ds[2], ds[3], tau_soc));
      a = fmin(a, soc_step(g[1], g[2], g[3], dg[1], dg[2], dg[3], tau_soc));
    } else if (role.type[p] == ROLE_JOINT) {
      const JointDev& jd = c.joints[idx];
      for (int i = 0; i < 2 * jd.nb_r; ++i) a = fmin(a, ort_step(sol[jd.sol_off + jd.ne + i], dl[jd.sol_off + jd.ne + i], tau_ort));
    }
  }
  return block_min<SMALL>(c, a);
}

// centering! (solver/centering.jl:1-48)
template <bool SMALL = false>
DJ_DEV void centering(Ctx& c, double aaff, double& nu, double& nuaff) {
  const Plan& P = *c.P;
  const double* sol = c.A + P.sol_off;
  const double* dl = c.A + P.rhs_off;
  const WarpRole& role = c.roles[c.warp];
  double sn = 0.0, sa = 0.0, cnt = 0.0;
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_CONTACT) {
      const ContactDev& cd = c.contacts[idx];
#ifdef DJ_ANY_CONTACT
      if (contact_type(cd) != 2) {  // cone_degree = N½ (contact.jl:197)
        const int nh = contact_nh(cd);
        for (int i = 0; i < nh; ++i) {
          double s = sol[cd.sol_off + i], g = sol[cd.sol_off + nh + i];
          sn += s * g;
          sa += (s + aaff * dl[cd.sol_off + i]) * (g + aaff * dl[cd.sol_off + nh + i]);
        }
        cnt += (double)nh;
        continue;
      }
#endif
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        double s = sol[cd.sol_off + i], g = sol[cd.sol_off + 4 + i];
        sn += s * g;
        sa += (s + aaff * dl[cd.sol_off + i]) * (g + aaff * dl[cd.sol_off + 4 + i]);
      }
      cnt += 2.0;  // cone_degree(NonlinearContact) (contacts/nonlinear.jl:101)
    } else if (role.type[p] == ROLE_JOINT) {
      const JointDev& jd = c.joints[idx];
      for (int i = 0; i < jd.nb_r; ++i) {
        int is = jd.sol_off + jd.ne + i, ig = is + jd.nb_r;
        sn += sol[is] * sol[ig];
        sa += (sol[is] + aaff * dl[is]) * (sol[ig] + aaff * dl[ig]);
      }
      cnt += (double)jd.nb_r;
    }
  }
  block_sum3<SMALL>(c, sn, sa, cnt);
  nu = sn / cnt;
  nuaff = sa / cnt;
}

// correction! (solver/correction.jl:1-45): sav += [-ds.dgamma + mu e; 0]
DJ_DEV void correction(Ctx& c) {
  const Plan& P = *c.P;
  const double* dl = c.A + P.rhs_off;
  double* sav = c.A + P.sav_off;
  const WarpRole& role = c.roles[c.warp];
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_CONTACT) {
      const ContactDev& cd = c.contacts[idx];
      const double* ds = dl + cd.sol_off;
#ifdef DJ_ANY_CONTACT
      if (contact_type(cd) != 2) {  // correction.jl:13-19
        const int nh = contact_nh(cd);
        for (int i = 0; i < nh; ++i) sav[cd.sol_off + i] += -ds[i] * ds[nh + i] + c.mu;
        continue;
      }
#endif
      const double* dg = ds + 4;
      double* r = sav + cd.sol_off;
      r[0] += -ds[0] * dg[0] + c.mu;
      r[1] += -(ds[1] * dg[1] + ds[2] * dg[2] + ds[3] * dg[3]) + c.mu;
      r[2] += -(ds[1] * dg[2] + dg[1] * ds[2]);
      r[3] += -(ds[1] * dg[3] + dg[1] * ds[3]);
    } else if (role.type[p] == ROLE_JOINT) {
      const JointDev& jd = c.joints[idx];
      for (int i = 0; i < jd.nb_r; ++i) {
        int is = jd.sol_off + jd.ne + i;
        sav[is] += -dl[is] * dl[is + jd.nb_r] + c.mu;
      }
    }
  }
  slot_sync(c);
}

// ------------------------------------------------------------------------------------------------------------
// mehrotra! (solver/mehrotra.jl:9-73).  Returns the status code; *iters = Newton iterations taken.
// TRACE (the traced step, dojo_step_trace): the slot's thread 0 also writes one row of 5 doubles per loop-head test into
// trace[r * 5 + k], row r = head of iteration r + 1, the heads solver_status prints in verbose mode (solver/mehrotra.jl:26-31,
// 75-98): [rvio, bvio, alpha, mutarget, trials], where alpha (the corrected direction's cone-line-search step), mutarget and
// trials (line-search trials evaluated up to and including the accepted one) belong to the iteration before the head; row 0 is
// [rvio, bvio, 1, 0, 0].  Rows after the last head reached are NaN.  TRACE = false compiles to the untraced loop.
// ------------------------------------------------------------------------------------------------------------
DJ_DEV void trace_row(double* tr, int r, double rvio, double bvio, double alpha, double mu, int trials) {
  double* p = tr + (size_t)r * 5;
  p[0] = rvio; p[1] = bvio; p[2] = alpha; p[3] = mu; p[4] = (double)trials;
}
template <bool TRACE = false, bool SMALL = false>
DJ_DEV int mehrotra(Ctx& c, const Options& o, int* iters, double* trace = nullptr) {
  const Plan& P = *c.P;
  double* A = c.A;
  int status = 1;
  c.mu = 0.0;
  double mutarget = 0.0;
  int no_progress = 0;
  double undercut = o.undercut;
  double rvio = 0.0, bvio = 0.0;
  int ndone = 0;
  // The loop is written so that every large routine (evaluate, factorize, solve, cone_line_search) has exactly ONE call
  // site: the Newton loop is ~20 k straight-line instructions, duplicated inlined bodies cost instruction-fetch bandwidth.
  //   mode 0: set_entries! at the current iterate (first pass: also yields the initial violations)
  //   mode 1: line-search trial at sol + fk * delta
  int mode = 0;
  double fk = 0.0, fsel = 0.0;
  int ls_k = 0;
  bool first = true;
  double alpha_tr = 1.0;  // TRACE: alpha of the current iteration (fk is halved by the line search)
  int rows_tr = 0;        // TRACE: rows written
  for (;;) {
    double rv, bv, rv2 = 0.0, bv2 = 0.0;
    bool pair = false;
    DJ_TICK(c, t_misc)
    if (mode == 0) {
      // alignment point: the environments hosted by this CTA start every Newton iteration together, so that their warps run
      // the same (large, straight-line) code at the same time and share its instruction fetches
      DJ_TICK(c, t_misc)
      {
        // When this is the only slot of the CTA that still has an environment (the tail of a launch), the drained slots evaluate
        // further line-search trials of this iteration at the same time (ls_assist_loop): an environment that stalls needs ten
        // trials per iteration, and it is the latency of such environments that ends a per-step launch.
        const AlignInfo ai = cta_align(c, true);
        c.assist = (P.ls_assist && ai.n_live == 1 && c.nslots > 1 && o.max_ls <= kMaxAssistTrials) ? 1 : 0;
      }
      DJ_TICK(c, t_align)
      evaluate<true, SMALL>(c, 0.0, P.rhs_off, rv, bv);
    } else {
      // trials are evaluated two at a time (k at fk, k + 1 at fk / 2); the second one is used only if the first is rejected
      pair = (SMALL || P.ls_pair != 0) && (ls_k + 1 < o.max_ls);
      if (c.assist) {  // post the pass: the helpers take the trials behind this slot's own
        if (c.tid == 0) { c.s_int[24] = 1; c.s_int[25] = ls_k; c.s_dbl[0] = fk; c.s_dbl[1] = c.mu; }
        cta_barrier();
      }
      evaluate_ls<SMALL>(c, A, fk, pair, rv, bv, rv2, bv2);
      if (c.assist) {
        if (c.tid == 0) {
          c.s_dbl[2 + 2 * ls_k] = rv; c.s_dbl[3 + 2 * ls_k] = bv;
          if (pair) { c.s_dbl[4 + 2 * ls_k] = rv2; c.s_dbl[5 + 2 * ls_k] = bv2; }
        }
        cta_barrier();
      }
    }
    if (mode == 0) { DJ_TICK(c, t_eval_jac) } else { DJ_TICK(c, t_eval_ls) }
    if (mode == 1) {
      // line_search! (solver/line_search.jl:1-34): trial k uses alpha / 2^k, accept unless both violations grow
      if (c.assist) {
        // the pass evaluated the trials ls_k .. ls_k + ntr - 1 (this slot's own and the helpers'): same rule, same order
        const int per = (SMALL || P.ls_pair != 0) ? 2 : 1;
        const int ntr = min(per * c.nslots, o.max_ls - ls_k);
        bool accepted = false;
        for (int j = 0; j < ntr; ++j) {
          rv = c.s_dbl[2 + 2 * ls_k]; bv = c.s_dbl[3 + 2 * ls_k];
          if ((rv > rvio) && (bv > bvio) && (ls_k + 1 < o.max_ls)) { fk *= 0.5; ls_k += 1; continue; }
          accepted = true;
          break;
        }
        if (!accepted) continue;  // next pass
        assist_release(c);
      } else if ((rv > rvio) && (bv > bvio) && (ls_k + 1 < o.max_ls)) {
        fk *= 0.5; ls_k += 1;
        if (!pair) continue;
        rv = rv2; bv = bv2;  // trial k + 1 was evaluated in the same pass
        if ((rv > rvio) && (bv > bvio) && (ls_k + 1 < o.max_ls)) { fk *= 0.5; ls_k += 1; continue; }
      }
      fsel = fk;
      bool made = (!(rv < o.rtol) && (rv < 0.8 * rvio)) || (!(bv < o.btol) && (bv < 0.8 * bvio));
      no_progress = made ? max(no_progress - 1, 0) : no_progress + 1;
      rvio = rv; bvio = bv;
      if (no_progress >= o.no_progress_max) undercut *= o.no_progress_undercut;
      // update! : commit the accepted candidate (with the angular-velocity clip of candidate_step!)
      double* sol = A + P.sol_off;
      const double* dl = A + P.rhs_off;
      if (fsel != 0.0) {
        for (int t = c.tid; t < P.nres; t += c.nthreads) sol[t] += fsel * dl[t];
        slot_sync(c);
        if (c.tid < P.Nb) {
          double* w = sol + c.bodies[c.tid].sol_off + 3;
          double wmax = 3.9 / (P.h * P.h);
          double wd = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
          if (wd > wmax) { double k = wmax / wd; w[0] *= k; w[1] *= k; w[2] *= k; }
        }
        slot_sync(c);
      }
      // The head of the next iteration (mehrotra.jl:26-30) tests exactly these violations (the candidate's, line_search.jl:22-30):
      // decide here, before set_entries! -- the KKT blocks of a final iterate are never used (the gradient pass assembles its own).
      if ((rvio != rvio) || (bvio != bvio)) { status = 3; break; }
      if (ndone >= o.max_iter) break;
      if (TRACE && c.tid == 0) { trace_row(trace, ndone, rvio, bvio, alpha_tr, mutarget, ls_k + 1); rows_tr = ndone + 1; }
      if ((rvio < o.rtol) && (bvio < o.btol)) { status = 0; break; }
      mode = 0; fk = 0.0;
      continue;  // set_entries! at the new iterate (mu = mutarget)
    }
    // mode 0: the system is assembled
    if (first) { rvio = rv; bvio = bv; first = false; }
    if (TRACE && c.tid == 0 && rows_tr == 0 && o.max_iter > 0) { trace_row(trace, 0, rvio, bvio, 1.0, 0.0, 0); rows_tr = 1; }  // the first head
    if ((rvio != rvio) || (bvio != bvio)) { status = 3; assist_release(c); break; }
    // `for n = 1:max_iter` tests convergence at the TOP of an iteration only (solver/mehrotra.jl:26-30): an iterate that meets the
    // tolerances after the last iteration's line search is still :failed
    if (ndone >= o.max_iter) { assist_release(c); break; }
    if ((rvio < o.rtol) && (bvio < o.btol)) { status = 0; assist_release(c); break; }
    ndone += 1;
    for (int t = c.tid; t < P.nres; t += c.nthreads) A[P.sav_off + t] = A[P.rhs_off + t];  // pull_residual!
    slot_sync(c);
    DJ_TICK(c, t_misc)
    if (!factorize<SMALL>(c)) { status = 3; assist_release(c); break; }
    DJ_TICK(c, t_fact)
    double alpha = 1.0;
    for (int pass = 0; pass < 2; ++pass) {  // pass 0: affine direction (Quirk Q3: rhs carries the previous mutarget); pass 1: corrected
      DJ_TICK(c, t_misc)
      solve<SMALL>(c, P.rhs_off);
      DJ_TICK(c, t_solve)
      double mx = fmax(rvio, bvio);
      double tau = (pass == 0) ? 0.95 : fmax(0.95, 1.0 - mx * mx);
      DJ_TICK(c, t_misc)
      alpha = cone_line_search<SMALL>(c, tau, fmin(tau, 0.95));
      DJ_TICK(c, t_cone)
      if (pass == 0) {
        double nu, nuaff;
        centering<SMALL>(c, alpha, nu, nuaff);
        double ratio = nuaff / (nu + 1e-20);
        double sig = (ratio != ratio) ? ratio : fmin(fmax(ratio, 0.0), 1.0);
        sig = sig * sig * sig;
        double sn = sig * nu;
        mutarget = (sn != sn) ? sn : fmax(sn, o.btol / undercut);
        c.mu = mutarget;
        correction(c);
        for (int t = c.tid; t < P.nres; t += c.nthreads) A[P.rhs_off + t] = A[P.sav_off + t];  // push_residual!
        slot_sync(c);
        DJ_TICK(c, t_center)
      }
    }
    mode = 1; fk = alpha; ls_k = 0;
    if (TRACE) alpha_tr = alpha;
  }
  if (TRACE && c.tid == 0)  // NaN padding of the rows after the last head reached
    for (int k = rows_tr * 5; k < o.max_iter * 5; ++k) trace[k] = nan("");
  *iters = ndone;
  return status;
}

// A drained slot of a CTA whose only remaining environment belongs to slot `owner` (the tail of a launch): evaluate line-search trials
// of that environment until the owner releases the iteration.  The owner posts a pass (first trial index, its step length, mu) and
// takes the first `per` trials itself; helper `rank` >= 1 takes the trials k0 + per rank .. with the same halvings of the step length
// the owner would apply (exact: powers of two), reading the owner's arena and writing residuals, contribution slots and reduction
// scratch into its own (evaluate_ls, `W`).  The residual evaluations are the ones the owner would have run in later passes, so the
// accepted trial and its violations -- all the line search hands on -- are bit-identical with and without helpers.
template <bool SMALL = false>
DJ_DEV void ls_assist_loop(Ctx& c, const Options& o, int owner, int rank) {
  const Plan& P = *c.P;
  double* own = c.A;
  const int per = (SMALL || P.ls_pair != 0) ? 2 : 1;
  for (;;) {
    cta_barrier();  // a pass has been posted, or the iteration released
    if (c.s_int[24] == 0) break;
    const int k0 = c.s_int[25] + per * rank;
    if (k0 < o.max_ls) {
      double f = c.s_dbl[0];
      for (int q = 0; q < per * rank; ++q) f *= 0.5;
      c.mu = c.s_dbl[1];
      const bool pair = (per == 2) && (k0 + 1 < o.max_ls);
      double rv, bv, rv2, bv2;
      c.A = c.arena0 + (size_t)owner * c.slot_stride;
      evaluate_ls<SMALL>(c, own, f, pair, rv, bv, rv2, bv2);
      c.A = own;
      if (c.tid == 0) {
        c.s_dbl[2 + 2 * k0] = rv; c.s_dbl[3 + 2 * k0] = bv;
        if (pair) { c.s_dbl[4 + 2 * k0] = rv2; c.s_dbl[5 + 2 * k0] = bv2; }
      }
    }
    cta_barrier();  // results of the pass are in the mailbox
  }
  c.mu = 0.0;
}

}  // namespace dj
