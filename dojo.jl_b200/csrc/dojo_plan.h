// dojo_plan.h -- flattened, device-resident description of one mechanism ("plan").
// Built once on the host in dojo_create() from the DojoMechanismDesc (include/dojo_b200.h), read-only on
// the device.  All *_off fields are offsets (in doubles) into the per-environment shared-memory arena.
//
// Execution model: nw warps own one environment (a CTA hosts several environments, each in its own arena).
//   * assembly / residual evaluation: warps take ROLES (bodies, contacts, joints), one lane per node; per-node
//     contributions to body rows go through 15-double "slots" that the body lanes gather in a fixed order
//     (deterministic floating-point summation order, no atomics);
//   * block LDU: elimination steps are grouped in PHASES by height in the elimination tree; the steps of one
//     phase are independent (updates of a parent body go to a per-joint scratch record that the parent folds in
//     when its own turn comes) and are spread over the half-warps; one slot barrier separates phases.
#pragma once
#include <stdint.h>

namespace dj {

constexpr double kReg = 1.0e-10;  // REG, src/Dojo.jl:4
constexpr int kSlot = 15;         // joint contribution record: force(3) torque(3) K(3x3, angular-angular block)
constexpr int kSlotC = 42;        // contact contribution record: force(3) torque(3) K(6x6)
constexpr int kScratch = 42;      // parent-update scratch record: S(6x6) v(6)
constexpr int kLim = 12;          // per limited axis: aP(3) aC(3) (d theta / d w, assembly) tP(3) tC(3) (impulse map, per step)

enum RoleType { ROLE_BODY = 0, ROLE_CONTACT = 1, ROLE_JOINT = 2 };

struct BodyDev {
  double mass;
  double J[9];
  int sol_off;  // [v25(3); w25(3)] inside the solution vector
  int st_off;   // x2(3), q2(4)
  int cst_off;  // constant part of the dynamics residual for this step (6)
  int D_off;    // 6x6 diagonal block
  int g_off, g_cnt, g_ncontact;  // gather list (Plan::ilist): arena offsets of the slots contributing to this body in a fixed
                                 // order; the first g_ncontact entries are contact slots (kSlotC), the rest joint slots (kSlot)
  // gradient pass (dojo_grad.cuh)
  int pjoint;              // parent joint index
  int cj_off, cj_cnt;      // child joints (Plan::ilist)
  int ct_off, ct_cnt;      // contacts (Plan::ilist)
  int r_off;               // offset of this body's 6 rows in the reduced (condensed) right-hand sides
  int gb_off;              // body record: d(w15 column)(9) Mqq(9) E(9)
};

struct JointDev {
  int parent, child;  // body indices, parent = -1 for the origin
  int n, sol_off;     // impulse dimension / offset inside the solution vector
  int ne;             // equality multipliers nl_t + nl_r; the joint's node in the condensed KKT system has joint_nq() = ne + nb2_r rows
  int nl_t, nl_r, nb2_r, nb_r;  // constrained axes (tra, rot), rotational limits Nb/2 and Nb
  // DEVICE layout of the joint's entries in sol / rhs / sav:  [ tra eq (nl_t) | rot eq (nl_r) | s (nb_r) | gamma (nb_r) ]
  // (the reference orders them [tra eq | s | gamma | rot eq]; the permutation is applied when `sol` is written out)
  int lim_off;        // nb2_r records of kLim doubles
  int nfree_t, nfree_r, u_off;
  int flags;          // JF_* bits below (occupies what used to be alignment padding: the layout the other fields have is unchanged)
  double pa[3], pb[3], qoff[4];
  double Ct[9], At[9], Cr[9], Ar[9];  // constraint / nullspace masks, zero-padded to 3 rows (joints/joint.jl:56-64)
  double spring_r, damper_r, spring_off_r[3], lo[3], hi[3];
  int D_off;                    // nq x nq, nq = joint_nq(): equality rows + one kept limit dual per limited axis
  int Uc_off, Lc_off;           // (joint,child) nq x 6, rewritten every assembly ; (child,joint) 6 x nq = -G_c, constant over the
                                // solve and never written by the factorisation (lives in the constant region of the arena)
  int Up_off, Lp_off, Gp_off;   // same for the parent body (-1 when the parent is the origin); Lp is consumed by the
                                // factorisation and refreshed from the pristine impulse map Gp at every assembly
  int BBpc_off, BBcp_off;       // body-body coupling through rotational limits / dampers, -1 without: (parent angular rows, child) 3 x 6
                                // and (child angular rows, parent angular columns) 3 x 3; JF_FULL joints: full 6 x 6 blocks
  int slot_c, slot_p;           // contribution slots for the child / parent body (slot_p = -1 for the origin)
  int S_off;                    // scratch record receiving this joint's (and its child body's) updates of the parent body
  // gradient pass
  int r_off;                    // offset of the ne equality rows in the reduced right-hand sides
  int gj_off;                   // joint record: RJp(ne x 6) RJc(ne x 6) BPp BPc BCp BCc (6x6 each) Up(6 x nu_j) Uc(6 x nu_j)
  int gv_off;                   // per-column forward scratch v (6 x CH) inside the gradient workspace (-1 for the origin)
};

// JointDev::flags -- translational springs / dampers / limits (joints/translational/{springs,dampers}.jl, joints/limits.jl); only
// the DJ_ANY_CONTACT compilation of the kernels (dojo_b200_cm.cu) reads them, dojo_create routes such mechanisms there
enum JointFlags {
  JF_TRA_SPRING = 1,  // explicit translational spring impulse (prologue)
  JF_TRA_DAMPER = 2,  // implicit translational damper: 6 x 6 velocity Jacobians on and between the two bodies
  JF_LIM_TRA = 4,     // the joint's limits (nb2_r axes, lo / hi) act on the translational coordinates A_t e instead of the rotation vector
  JF_FULL = 8         // contribution slots carry a full 6 x 6 block (kSlotC) and the limit records 6-vectors (2 kLim per axis)
};
// The translational spring / damper parameters [spring, damper, spring_offset(nfree_t)] are kept in the rows nl_t..2 of the
// zero-padded constraint mask Ct, which no kernel reads (every loop over Ct stops at nl_t): JointDev keeps its size.
static_assert(sizeof(JointDev) == 568, "JointDev layout is part of the kernels' addressing");
#if defined(__CUDACC__) || defined(DJ_HOSTEMU)
#define DJ_PLAN_FN __host__ __device__ inline
#else
#define DJ_PLAN_FN inline
#endif
// Size of the joint's node in the condensed KKT system: its ne equality multipliers plus ONE dual per limited axis.  Of the two
// limit sides of an axis (upper / lower) the one nearer to its bound -- the smaller slack, the only one that can be active -- keeps
// its dual as an explicit unknown (a row with diagonal s, like an equality row with diagonal REG); its slack and the whole other side
// are condensed out analytically.  Condensing BOTH sides (division by the active slack s -> 0) put terms of size gamma / s on the body
// rows and lost the dynamics there to rounding (linear residual ~3e-9, no convergence below rtol ~1e-8); the reference eliminates the
// bodies BEFORE the joint node, which is what keeping the active dual in the joint node reproduces (DESIGN.md section 6).
DJ_PLAN_FN int joint_nq(const JointDev& j) { return j.ne + j.nb2_r; }
DJ_PLAN_FN const double* joint_tra_params(const JointDev& j) { return j.Ct + 3 * j.nl_t; }
DJ_PLAN_FN double* joint_tra_params(JointDev& j) { return j.Ct + 3 * j.nl_t; }

struct ContactDev {
  int body, sol_off;  // [s(N½); gamma(N½)] inside the solution vector (NonlinearContact: N½ = 4)
  double mu, radius;
  double n[3], t[6], o[3], off[3];
  int J_off, G_off, rec_off;  // J = d(constraint)/d(v25,w25) 4x6 ; G = impulse map 6x4 ; 3 reciprocals of the closed-form block solve
  int slot;
  int gc_off;                 // gradient pass: condensed body block CB (6x6)
  int tn;                     // contact model: type | N½ << 8 (type 0 impact N½ = 1, 1 linear N½ = 6, 2 nonlinear N½ = 4); the entry is
                              // [s(N½); gamma(N½)], J is N½ x 6, G is 6 x N½.  Occupies what used to be tail padding: the layout the
                              // NonlinearContact kernels see is unchanged
};
static_assert(sizeof(ContactDev) == 168, "ContactDev layout is part of the kernels' addressing");

// One elimination step of the block LDU (GraphBasedSystems ldu_factorization!)
struct ElimNb {
  int n, vec_off;   // neighbour dimension / offset of its entry in the solution-ordered vectors
  int r_off;        // same in the reduced right-hand sides of the gradient pass
  int gv_off;       // >= 0: per-column forward scratch (gradient pass) instead of r_off
  int fwd_abs;      // >= 0: absolute arena offset that receives the forward-substitution update instead of vec_off (scratch v)
  int L_off;        // M_{nb,c}: n_nb x n_c   (overwritten by M_{nb,c} * Dinv_c)
  int U_off, U_k;   // M_{c,nb}: rows [U_row, U_row + U_k) of c, U_k x n_nb (never written by the factorisation)
  int U_row;
  // A neighbour may stand for a SUB-RANGE of rows of its node: the parent body of a joint with rotational limits / dampers couples to
  // the child body through its three angular rows only (round 2: those body-body blocks are stored 3 x 6 / 3 x 3 instead of 6 x 6 with
  // exact zeros).  n, vec_off, r_off, fwd_abs and the tgt offsets below then address the sub-range directly;
  int ld;           // leading dimension of the blocks whose COLUMNS belong to this neighbour's node (its full dimension: 6 for a body)
  int row0;         // first row of the node covered by this neighbour (0, or 3 for the angular rows); only the gradient pass needs it
};
struct ElimStep {
  int d_off, n, vec_off;
  int r_off;               // reduced offset (gradient pass)
  int gfold_off;           // gradient pass: Plan::ilist offsets of the children's per-column scratch v (fold_cnt entries)
  int nnb;
  ElimNb nb[2];
  int tgt[2][2];           // M_{nb_i, nb_j} (the parent body's diagonal is redirected to the joint's scratch record)
  int fold_off, fold_cnt;  // scratch records (Plan::ilist) folded into (D_c, z_c) before c is eliminated
};

// The block LDU of the Newton loop (factorize / solve) reads its steps from a flat PROGRAM instead of walking sched -> ElimStep ->
// ElimNb -> ilist: one LduOp per elimination step with every offset and bound the three passes need already resolved.  A warp's ops
// are contiguous and in phase order, so the address of the next op is a running index that does not wait on a load; the step count
// of (phase, warp) is read next to it.  ElimStep and sched stay for the gradient pass.  Layout (ints, right after sched in the same
// blob table): cnt[nphase][nw] steps of warp w in phase ph and wfirst[nw] first op of warp w from Plan::prog_cnt, padding to
// 16 bytes, then LduOp ops[] from Plan::prog_ops.
// An op is three 16-byte words of 16-bit arena offsets (an arena is < 2^16 doubles) and 8-bit sizes, so that the program costs the
// hot prefix of the blob no table the chain kept in shared memory (quadruped's gradient pass has 9.2 KiB of room for it):
//   word 0:  d_off | vec_off << 16,   n | nnb << 8 | fold_cnt << 16,   fold_off | fold[0] << 16,   fold[1] | fold[2] << 16
//   word 1 + i, neighbour i:  L_off | fwd_abs << 16 (kLduNone: none),   vec_off | U_off << 16,   n | U_row << 8 | U_k << 16 | ld << 24,
//                             tgt[i][0] | tgt[i][1] << 16
// fold[] holds the first kLduFold scratch records folded into the step (arena offsets); the rest stay in Plan::ilist from fold_off.
constexpr int kLduFold = 3;
constexpr int kLduNone = 0xffff;
struct alignas(16) LduOp {
  int w[12];
};
static_assert(sizeof(LduOp) == 48, "LduOp is read as three 16-byte words");
DJ_PLAN_FN int lo16(int v) { return v & 0xffff; }
DJ_PLAN_FN int hi16(int v) { return (int)((unsigned)v >> 16); }
DJ_PLAN_FN int byte_of(int v, int k) { return (v >> (8 * k)) & 0xff; }

struct WarpRole {
  int npass;
  int type[3], first[3], count[3];
};

struct Plan {
  int Nb, Ne, Ni, nres, nu, nz;
  int nw;       // warps per environment
  int nphase;   // elimination phases
  // paired line-search trials (every role pass has <= 16 nodes): the second trial of a pass writes its contribution slots at
  // [slot + ls_slot_delta] and its residual at ls_res2_off, both inside the matrix region
  int ls_pair, ls_slot_delta, ls_res2_off;
  int ls_assist;  // drained slots of a CTA evaluate line-search trials of its last live environment (ls_assist_loop)
  int jpair;    // set_entries! of a joint on two lanes (child side / parent side) when a joint pass has at most 16 joints (eval_joint_pair)
  double h, input_scaling, g[3];
  // arena layout (doubles)
  int sol_off, rhs_off, sav_off, red_off, mat_off, mat_len, arena_len;  // [mat_off, mat_off + mat_len) is re-zeroed at every assembly
  const BodyDev* bodies;
  const JointDev* joints;
  const ContactDev* contacts;
  const ElimStep* steps;
  const int* sched;   // [nphase][nw][2] = (first step, count), followed by the LDU program (LduOp)
  int prog_cnt, prog_ops;  // ints from the start of sched to the program's cnt[] and ops[]
  const int* ilist;   // gather / fold lists
  const WarpRole* roles;  // [nw]
  // gradient pass
  int n_red;            // rows of the condensed system (6 Nb + sum ne)
  int ncol;             // 12 Nb + nu
  int ch;               // columns solved per chunk (one lane per column)
  int gvec_off;         // [n_red][ch] column vectors
  int grad_len;         // arena length with the gradient workspace
  const int* ucol;      // [nu][2] = (joint, dof) of every input column
};

struct Options {
  double rtol, btol, undercut, no_progress_undercut;
  int max_iter, max_ls, no_progress_max;
};

}  // namespace dj
