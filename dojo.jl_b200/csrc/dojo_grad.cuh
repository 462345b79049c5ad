// dojo_grad.cuh -- implicit-function-theorem gradients of the step (K2).
//
// Reference: get_maximal_gradients (gradients/state.jl:78-126) evaluated at the solution right after mehrotra!, before
// update_state! (the consistent variant, SURVEY.md Q2), with the data Jacobian of gradients/data.jl restricted to the
// state / control columns [x2 v15 phi2 w15] per body and the joint inputs (state.jl:92-93).
//
//   d w / d theta = KKT^-1 * d(rhs)/d theta          (state.jl:99 solves the dense system; the reference leaves
//                                                     "use pre-factorization" as a TODO -- here the block-LDU factor
//                                                     of the step's own KKT matrix is reused)
//
// Work split:  (1) roles (one lane per node) write the sparse data-Jacobian blocks, already condensed onto the body /
// joint-equality rows exactly like the right-hand sides of the solver; (2) the factorisation of the final KKT matrix;
// (3) columns are processed in chunks of `ch`, ONE LANE PER COLUMN: each lane builds its right-hand side from the
// blocks, runs the forward / backward substitution for its own column (matrix entries are warp-broadcast reads, the
// column vectors are stored [row][lane], bank-conflict free) and applies the chain rule to (x3, q3) (state.jl:104-123).
// The elimination phases are spread over the warps as in the solver.
//
// Everything is in attitude (body-frame) form: a perturbation q (x) (1, d).  The reference's attjac'd 6x6 blocks
// (joints/*/impulses.jl impulse_transform_jacobian, springs.jl / dampers.jl *_jacobian_configuration, contacts/contact.jl
// impulse_map_jacobian, integrators/integrator.jl integrator_jacobian_configuration) are re-derived in closed form.
// Unlike the reference, the data Jacobian includes d(input impulse)/d(configuration) (SURVEY.md Q17: gradients/data.jl never
// calls input_jacobian_configuration, so its Fz is not the derivative of the step once an actuated joint has a free parent and
// u != 0).  DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN leaves the term out: gradients() is then called without the inputs.
#pragma once
#include "dojo_kernels.cuh"

namespace dj {

DJ_DEV void st_block33(double* B, int ld, int r0, int c0, const M33& m, double sgn = 1.0) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) B[(r0 + i) * ld + c0 + j] = sgn * m.m[i][j];
}
DJ_DEV void add_block33(double* B, int ld, int r0, int c0, const M33& m, double sgn = 1.0) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) B[(r0 + i) * ld + c0 + j] += sgn * m.m[i][j];
}
DJ_DEV M33 transport(V3 w, double h) { return transpose(rotmat(qmap(w, h))); }  // d phi3 / d phi2 = R(m)'

// ---------------------------------------------------------------------------------------------------------
// (1) data-Jacobian blocks
// ---------------------------------------------------------------------------------------------------------
DJ_DEV void grad_body(Ctx& c, int idx) {
  const Plan& P = *c.P;
  double* A = c.A;
  const BodyDev& bd = c.bodies[idx];
  // the v15 / w15 columns need (x1, q1), i.e. the *initial* velocities: recovered from the constant residual part
  // cst is not invertible for that -> the kernel keeps w15 in the body record (written by the prologue)
  double* rec = A + bd.gb_off;
  V3 w15 = ld3(rec + 27);
  M33 J = ldm33(bd.J);
  double n0 = 0.5 * P.h * sqrt(4.0 / (P.h * P.h) - dot(w15, w15));
  V3 Jw = J * w15;
  // -d(D1q)/d w15 = d/dw [ n0 J w - (h/2) w x J w ]       (gradients/data.jl:31-36)
  V3 dn0 = (-(0.25 * P.h * P.h) / n0) * w15;
  M33 dW = outer(Jw, dn0) + n0 * J - (0.5 * P.h) * (skew(w15) * J - skew(Jw));
  stm33(rec, dW);
  Kin k = body_kin(c, idx, 0.0);
  stm33(rec + 9, transport(k.w, P.h));
  stm33(rec + 18, k.E);
}

#ifdef DJ_ANY_CONTACT
// ImpactContact / LinearContact: the data blocks of the state columns are generic over the contact model (gradients/data.jl:126-135,
// :194-205 with constraint_jacobian_configuration of impact.jl:66-75 / contact.jl:9-35); condensed like the solver's right-hand sides
DJ_DEV void grad_contact_orthant(Ctx& c, int idx) {
  const Plan& P = *c.P;
  double* A = c.A;
  const ContactDev& cd = c.contacts[idx];
  const int type = contact_type(cd), nh = contact_nh(cd);
  const double* so = A + P.sol_off + cd.sol_off;
  Kin k = body_kin(c, cd.body, 0.0);
  ContactGeom q = contact_geom(cd, k);
  double s[6], g[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) { s[i] = 1.0; g[i] = 1.0; if (i < nh) { s[i] = so[i]; g[i] = so[nh + i]; } }
  V3 F = orthant_force(type, q, g);
  V3 tau = tmul(k.R3, cross(q.rc, F));
  M33 R3so = k.R3 * skew(q.o);
  M33 Mqq = transport(k.w, P.h);
  V3 nphi = vtmul((-2.0) * vtmul(q.n, R3so), Mqq);
  M33 dvc_dd = (2.0 * (skew(q.rc) * (k.R3 * skew(k.w))) - 2.0 * (skew(q.ww) * R3so)) * Mqq;
  V3 v0 = vtmul(q.t0, dvc_dd), v1 = vtmul(q.t1, dvc_dd);
  const double Zn[6] = {-q.n.x, -q.n.y, -q.n.z, -nphi.x, -nphi.y, -nphi.z};
  const double Z0[6] = {0, 0, 0, -v0.x, -v0.y, -v0.z};
  const double Z1[6] = {0, 0, 0, -v1.x, -v1.y, -v1.z};
  double Zc[6][6];
  orthant_expand(Zn, Z0, Z1, Zc);
  const double* G = A + cd.G_off;
  M33 K = (2.0 * skew(tau) + 2.0 * (transpose(k.R3) * (skew(F) * R3so))) * Mqq;
  double* CB = A + cd.gc_off;
#pragma unroll 1
  for (int cc = 0; cc < 6; ++cc) {
    double t[12], y[12];
#pragma unroll
    for (int i = 0; i < 6; ++i) { t[i] = 0.0; t[6 + i] = 0.0; }
#pragma unroll
    for (int i = 0; i < 6; ++i) if (i < nh) t[nh + i] = Zc[i][cc];
    orthant_solve(type, s, g, cd.mu, t, y);
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      double v = 0.0;
      for (int i = 0; i < nh; ++i) v += G[r * nh + i] * y[nh + i];
      if (r >= 3 && cc >= 3) v += K.m[r - 3][cc - 3];
      CB[r * 6 + cc] = v;
    }
  }
}
#endif

DJ_DEV void grad_contact(Ctx& c, int idx) {
  const Plan& P = *c.P;
  double* A = c.A;
  const ContactDev& cd = c.contacts[idx];
#ifdef DJ_ANY_CONTACT
  if (contact_type(cd) != 2) { grad_contact_orthant(c, idx); return; }
#endif
  const double* so = A + P.sol_off + cd.sol_off;
  Kin k = body_kin(c, cd.body, 0.0);
  V3 n = ld3(cd.n), t0 = ld3(cd.t), t1 = ld3(cd.t + 3), o = ld3(cd.o), off = ld3(cd.off);
  V3 ow = k.R3 * o;
  V3 rc = ow - off - cd.radius * n;
  V3 ww = k.R3 * k.w;
  const double* g = so + 4;
  V3 F = g[0] * n + g[2] * t0 + g[3] * t1;
  V3 tau = tmul(k.R3, cross(rc, F));
  M33 R3so = k.R3 * skew(o);
  M33 Mqq = transport(k.w, P.h);
  // contact rows:  Zc = -d(constraint)/d(x3, phi3) * blkdiag(I, Mqq)   (gradients/data.jl:194-205, contacts/contact.jl:9-35)
  V3 nphi = vtmul((-2.0) * vtmul(n, R3so), Mqq);
  M33 dvc_dd = (2.0 * (skew(rc) * (k.R3 * skew(k.w))) - 2.0 * (skew(ww) * R3so)) * Mqq;
  V3 v0 = vtmul(t0, dvc_dd), v1 = vtmul(t1, dvc_dd);
  const double Zc0[6] = {-n.x, -n.y, -n.z, -nphi.x, -nphi.y, -nphi.z};
  const double Zc2[6] = {0, 0, 0, -v0.x, -v0.y, -v0.z};
  const double Zc3[6] = {0, 0, 0, -v1.x, -v1.y, -v1.z};
  // condensation (as for the solver's right-hand sides): body rows += G W Zc
  ContactBlock cb = contact_block(so, g, cd.mu);
  double Wm[4][4];
#pragma unroll
  for (int kx = 0; kx < 4; ++kx) {
    if (kx == 1) continue;
    double t[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8];
    t[4 + kx] = 1.0;
    contact_solve(cb, t, y);
#pragma unroll
    for (int r = 0; r < 4; ++r) Wm[r][kx] = y[4 + r];
  }
  double WZ[4][6];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int cc = 0; cc < 6; ++cc) WZ[r][cc] = Wm[r][0] * Zc0[cc] + Wm[r][2] * Zc2[cc] + Wm[r][3] * Zc3[cc];
  const double* G = A + cd.G_off;
  // body rows: + d(G gamma)/d(x3, phi3) * blkdiag(I, Mqq): torque rows, attitude columns only   (gradients/data.jl:126-135)
  M33 K = (2.0 * skew(tau) + 2.0 * (transpose(k.R3) * (skew(F) * R3so))) * Mqq;
  double* CB = A + cd.gc_off;
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int cc = 0; cc < 6; ++cc) {
      double v = G[r * 4 + 0] * WZ[0][cc] + G[r * 4 + 2] * WZ[2][cc] + G[r * 4 + 3] * WZ[3][cc];
      if (r >= 3 && cc >= 3) v += K.m[r - 3][cc - 3];
      CB[r * 6 + cc] = v;
    }
}

// Contact-data columns (get_contact_gradients, gradients/contact.jl:1-55; data blocks gradients/data.jl:152-192):
// theta_c = [friction_coefficient; contact_radius; contact_origin(3)].  Column p of contact idx touches only the rows of the
// contact's body after condensation:  v = Q + G W Z,  Z = the four constraint rows [d - s1; mu g1 - g2; vt - s34] of the
// data block, Q = its torque rows.  Computed by the lane that owns the column (no storage).
DJ_DEV void grad_contact_param_rhs(Ctx& c, int idx, int p, double* v) {
  const Plan& P = *c.P;
  double* A = c.A;
  const ContactDev& cd = c.contacts[idx];
  const double* so = A + P.sol_off + cd.sol_off;
  Kin k = body_kin(c, cd.body, 0.0);
  V3 n = ld3(cd.n), t0 = ld3(cd.t), t1 = ld3(cd.t + 3);
  V3 ww = k.R3 * k.w;
  const double* g = so + 4;
  V3 Fb = tmul(k.R3, g[0] * n + g[2] * t0 + g[3] * t1);  // contact force in the body frame
  double Z[4] = {0.0, 0.0, 0.0, 0.0};
  V3 Q = v3zero();
  if (p == 0) {
    Z[1] = -g[0];
  } else if (p == 1) {
    V3 wn = cross(ww, n);
    Z[0] = dot(n, n); Z[2] = dot(t0, wn); Z[3] = dot(t1, wn);
    Q = cross(Fb, tmul(k.R3, n));
  } else {
    const int kk = p - 2;
    V3 ek = v3(kk == 0 ? 1.0 : 0.0, kk == 1 ? 1.0 : 0.0, kk == 2 ? 1.0 : 0.0);
    V3 rk = k.R3 * ek;            // d(contact point) / d(origin_k)
    V3 wr = cross(ww, rk);
    Z[0] = -dot(n, rk); Z[2] = -dot(t0, wr); Z[3] = -dot(t1, wr);
    Q = -1.0 * cross(Fb, ek);
  }
  ContactBlock cb = contact_block(so, g, cd.mu);
  double WZ[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int kx = 0; kx < 4; ++kx) {
    double t[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8];
    t[4 + kx] = 1.0;
    contact_solve(cb, t, y);
#pragma unroll
    for (int r = 0; r < 4; ++r) WZ[r] += y[4 + r] * Z[kx];
  }
  const double* G = A + cd.G_off;
#pragma unroll
  for (int r = 0; r < 6; ++r) v[r] = G[r * 4 + 0] * WZ[0] + G[r * 4 + 2] * WZ[2] + G[r * 4 + 3] * WZ[3];
  v[3] += Q.x; v[4] += Q.y; v[5] += Q.z;
}

#ifdef DJ_ANY_CONTACT
// Translational springs / dampers / limits in the data Jacobian (joints/translational/springs.jl:44-76, dampers.jl:40-98,
// joints/limits.jl with gradients/data.jl:4-14, :67-124).  An impulse h G6(x2, q2) f contributes
//   d(G6) f  -- covered by the caller's derivative of the translational impulse map once f is added to the projected impulse p_t --
//   G6 d(f)  -- added here: f depends on the poses through e(x2, q2) and, for the damper, e(x1, q1) with q1 = q2 (x) m(-w25)
//              (a perturbation d of q2 moves the attitude of q1 by R(m(-w))' d).
// Returns the force to add to p_t.  Limits: the slack rows move with theta = a.e(x3, q3); condensed like the solver's rows.
DJ_DEV V3 grad_joint_tra(Ctx& c, const JointDev& jd, const Kin& ka, const Kin& kb, const JointGeom& g2, const JointGeom& g3, const M33& Ma,
                         const M33& Mb, const double* so, double* BPp, double* BPc, double* BCp, double* BCc, double* RJp, double* RJc) {
  const Plan& P = *c.P;
  double* A = c.A;
  V3 extra = v3zero();
  M33 AtA = m33zero();
#pragma unroll
  for (int i = 0; i < 3; ++i)
    if (i < jd.nfree_t) { V3 a = ld3(jd.At + 3 * i); AtA = AtA + outer(a, a); }
  const bool par = jd.parent >= 0;
  if (jd.flags & JF_TRA_SPRING) {
    const double* tp = joint_tra_params(jd);
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (i < jd.nfree_t) { V3 a = ld3(jd.At + 3 * i); extra += (P.h * tp[0] * (tp[2 + i] - dot(a, g2.et))) * a; }
    const double k = -P.h * tp[0];
    M33 Fxa = k * (AtA * g2.Xp), Fqa = k * (AtA * g2.Qtp), Fxb = k * (AtA * g2.Xc), Fqb = k * (AtA * g2.Qtc);
    g6_accumulate(BCc, g2.Xc, g2.Qtc, Fxb, Fqb, 1.0);
    if (par) {
      g6_accumulate(BPp, g2.Xp, g2.Qtp, Fxa, Fqa, 1.0);
      g6_accumulate(BPc, g2.Xp, g2.Qtp, Fxb, Fqb, 1.0);
      g6_accumulate(BCp, g2.Xc, g2.Qtc, Fxa, Fqa, 1.0);
    }
  }
  if (jd.flags & JF_TRA_DAMPER) {
    const double damper = joint_tra_params(jd)[1];
    V3 xa1 = ka.x2 - P.h * ka.v, xb1 = kb.x2 - P.h * kb.v;
    Quat qa1 = qmul(ka.q2, qmap(-ka.w, P.h)), qb1 = qmul(kb.q2, qmap(-kb.w, P.h));
    M33 Ra1 = rotmat(qa1), Rb1 = rotmat(qb1);
    JointGeom g1 = joint_geom(jd, xa1, qa1, Ra1, xb1, qb1, Rb1);
    extra += (-damper) * (AtA * (g2.et - g1.et));
    M33 Fxa = (-damper) * (AtA * (g2.Xp - g1.Xp)), Fqa = (-damper) * (AtA * (g2.Qtp - g1.Qtp * transport(-ka.w, P.h)));
    M33 Fxb = (-damper) * (AtA * (g2.Xc - g1.Xc)), Fqb = (-damper) * (AtA * (g2.Qtc - g1.Qtc * transport(-kb.w, P.h)));
    g6_accumulate(BCc, g2.Xc, g2.Qtc, Fxb, Fqb, 1.0);
    if (par) {
      g6_accumulate(BPp, g2.Xp, g2.Qtp, Fxa, Fqa, 1.0);
      g6_accumulate(BPc, g2.Xp, g2.Qtp, Fxb, Fqb, 1.0);
      g6_accumulate(BCp, g2.Xc, g2.Qtc, Fxa, Fqa, 1.0);
    }
  }
  if (jd.flags & JF_LIM_TRA) {
    M33 QtpM = g3.Qtp * Ma, QtcM = g3.Qtc * Mb;
    const int ne = jd.ne;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nb2_r) {
        V3 ai = ld3(jd.At + 3 * i);
        const int is_u = ne + i, is_l = ne + jd.nb2_r + i, ig_u = is_u + jd.nb_r, ig_l = is_l + jd.nb_r;
        extra += (so[ig_l] - so[ig_u]) * ai;
        const LimitSide ls = limit_side(so[is_u], so[is_l], so[ig_u], so[ig_l]);  // kept / condensed side as in the solver
        const double kk = ls.kI;
        V3 apx = vtmul(ai, g3.Xp), apq = vtmul(ai, QtpM), acx = vtmul(ai, g3.Xc), acq = vtmul(ai, QtcM);
        const double ap[6] = {apx.x, apx.y, apx.z, apq.x, apq.y, apq.z}, ac[6] = {acx.x, acx.y, acx.z, acq.x, acq.y, acq.z};
        const double* lim = A + jd.lim_off + 2 * kLim * i;
        const int q = ne + i;
#pragma unroll
        for (int r = 0; r < 6; ++r) { RJp[q * 6 + r] = (ls.sg * ls.gA) * ap[r]; RJc[q * 6 + r] = (ls.sg * ls.gA) * ac[r]; }
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            BCc[r * 6 + q] -= kk * lim[18 + r] * ac[q];
            if (par) {
              BPp[r * 6 + q] -= kk * lim[12 + r] * ap[q];
              BPc[r * 6 + q] -= kk * lim[12 + r] * ac[q];
              BCp[r * 6 + q] -= kk * lim[18 + r] * ap[q];
            }
          }
      }
    }
  }
  return extra;
}
#endif

// record layout of a joint (doubles): RJp[nq*6] RJc[nq*6] BPp[36] BPc[36] BCp[36] BCc[36] Up[6*nu] Uc[6*nu]   (nq = joint_nq: the
// node's rows = ne equality rows + one kept limit dual per limited axis)
// u: this environment's inputs, or null to leave the inputs' configuration derivative out (SURVEY.md Q17)
DJ_DEV void grad_joint(Ctx& c, int idx, const double* __restrict__ u) {
  const Plan& P = *c.P;
  double* A = c.A;
  const JointDev& jd = c.joints[idx];
  const int ne = jd.ne, nq = joint_nq(jd), nuj = jd.nfree_t + jd.nfree_r;
  double* RJp = A + jd.gj_off;
  double* RJc = RJp + 6 * nq;
  double* BPp = RJc + 6 * nq;
  double* BPc = BPp + 36;
  double* BCp = BPc + 36;
  double* BCc = BCp + 36;
  double* Up = BCc + 36;
  double* Uc = Up + 6 * nuj;
  for (int i = 0; i < 144; ++i) BPp[i] = 0.0;
  const double* so = A + P.sol_off + jd.sol_off;
  Kin ka = body_kin(c, jd.parent, 0.0), kb = body_kin(c, jd.child, 0.0);
  M33 Ma = (jd.parent >= 0) ? transport(ka.w, P.h) : m33ident();
  M33 Mb = transport(kb.w, P.h);
  // ---- joint rows: -d g / d(x3, phi3) * blkdiag(I, Mqq)        (gradients/data.jl:4-14)
  JointGeom g3 = joint_geom(jd, ka.x3, ka.q3, ka.R3, kb.x3, kb.q3, kb.R3);
  {
    M33 QtpM = g3.Qtp * Ma, QtcM = g3.Qtc * Mb, QrpM = g3.Qrp * Ma, QrcM = g3.Qrc * Mb;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nl_t) {
        V3 ci = ld3(jd.Ct + 3 * i);
        st3(RJp + i * 6, -vtmul(ci, g3.Xp)); st3(RJp + i * 6 + 3, -vtmul(ci, QtpM));
        st3(RJc + i * 6, -vtmul(ci, g3.Xc)); st3(RJc + i * 6 + 3, -vtmul(ci, QtcM));
      }
      if (i < jd.nl_r) {
        V3 ci = ld3(jd.Cr + 3 * i);
        const int row = jd.nl_t + i;
        st3(RJp + row * 6, v3zero()); st3(RJp + row * 6 + 3, -vtmul(ci, QrpM));
        st3(RJc + row * 6, v3zero()); st3(RJc + row * 6 + 3, -vtmul(ci, QrcM));
      }
    }
  }
  // ---- geometry at the current configuration (impulse maps, springs, dampers)
  M33 Ra = rotmat(ka.q2), Rb = rotmat(kb.q2);
  JointGeom g2 = joint_geom(jd, ka.x2, ka.q2, Ra, kb.x2, kb.q2, Rb);
  M33 Roff = rotmat(ldq(jd.qoff));
  V3 vr = qvec(g2.qr);
  const double s0 = g2.qr.s;
  // projected impulses: p_t = C_t' lambda_t ;  p_r = C_r' lambda_r + sum_i (gamma_l - gamma_u) A_i
  V3 pt = v3zero(), pr = v3zero();
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < jd.nl_t) pt += so[i] * ld3(jd.Ct + 3 * i);
    if (i < jd.nl_r) pr += so[jd.nl_t + i] * ld3(jd.Cr + 3 * i);
#ifdef DJ_ANY_CONTACT
    if (jd.flags & JF_LIM_TRA) continue;  // translational limit duals act through p_t (grad_joint_tra)
#endif
    if (i < jd.nb2_r) pr += (so[ne + jd.nb_r + jd.nb2_r + i] - so[ne + jd.nb_r + i]) * ld3(jd.Ar + 3 * i);
  }
#ifdef DJ_ANY_CONTACT
  if (jd.flags) pt += grad_joint_tra(c, jd, ka, kb, g2, g3, Ma, Mb, so, BPp, BPc, BCp, BCc, RJp, RJc);
#endif
  // translational impulses (translational/impulses.jl:9-45):  F_p = -Ra p, F_c = Ra p, tau_p = p x (e + pa), tau_c = pb x (Rb' Ra p)
  // The translational input it (prologue_joint) is such an impulse with only half of its torque (Q16): p = pt + it on the force
  // rows, pt + it / 2 on the torque rows.
  {
    V3 pf = pt, pq = pt;
    if (u && jd.nfree_t > 0) {
      V3 it = v3zero();
#pragma unroll
      for (int i = 0; i < 3; ++i)
        if (i < jd.nfree_t) it += u[jd.u_off + i] * ld3(jd.At + 3 * i);
      it = P.input_scaling * it;
      pf = pt + it;
      pq = pt + 0.5 * it;
    }
    V3 pb = ld3(jd.pb);
    M33 Rasp = Ra * skew(pf);
    add_block33(BPp, 6, 0, 3, Rasp, 2.0);    // dF_p / d phi_a
    add_block33(BCp, 6, 0, 3, Rasp, -2.0);   // dF_c / d phi_a
    M33 sp = skew(pq);
    add_block33(BPp, 6, 3, 0, sp * g2.Xp); add_block33(BPp, 6, 3, 3, sp * g2.Qtp);
    add_block33(BPc, 6, 3, 0, sp * g2.Xc); add_block33(BPc, 6, 3, 3, sp * g2.Qtc);
    M33 RbtRa = transpose(Rb) * Ra;
    add_block33(BCp, 6, 3, 3, skew(pb) * (RbtRa * sp), -2.0);
    add_block33(BCc, 6, 3, 3, skew(pb) * skew(RbtRa * pq), 2.0);
  }
  Quat r = qmul(qinv(ka.q2), kb.q2);
  M33 Rr = rotmat(r), Rrt = transpose(Rr);
  // rotational impulses (rotational/impulses.jl:9-38): tau_c = 1/2 (s p - v x p), tau_p = -1/2 Roff (s p + v x p)
  {
    M33 sp = skew(pr);
    V3 Rv = Roff * vr;
    M33 dc_b = 0.5 * (outer(pr, -vr) + sp * g2.Qrc);       // d tau_c / d phi_b
    M33 dc_a = 0.5 * (outer(pr, Rv) + sp * g2.Qrp);        // d tau_c / d phi_a
    M33 dp_b = (-0.5) * (Roff * (outer(pr, -vr) - sp * g2.Qrc));
    M33 dp_a = (-0.5) * (Roff * (outer(pr, Rv) - sp * g2.Qrp));
    // rotational input (rotational/input.jl:5-17): tau_p = -Roff tau is constant, tau_c = -R(r)' tau_p turns with r
    if (u && jd.nfree_r > 0) {
      V3 ir = v3zero();
#pragma unroll
      for (int i = 0; i < 3; ++i)
        if (i < jd.nfree_r) ir += u[jd.u_off + jd.nfree_t + i] * ld3(jd.Ar + 3 * i);
      V3 tp = (-P.input_scaling) * (Roff * ir);
      dc_a = dc_a + 2.0 * (Rrt * skew(tp));
      dc_b = dc_b + (-2.0) * skew(Rrt * tp);
    }
    add_block33(BCc, 6, 3, 3, dc_b); add_block33(BCp, 6, 3, 3, dc_a);
    add_block33(BPc, 6, 3, 3, dp_b); add_block33(BPp, 6, 3, 3, dp_a);
    (void)s0;
  }
  M33 AtA = m33zero();
#pragma unroll
  for (int i = 0; i < 3; ++i)
    if (i < jd.nfree_r) { V3 a = ld3(jd.Ar + 3 * i); AtA = AtA + outer(a, a); }
  // rotational spring (rotational/springs.jl:44-84): tau_p = h Roff f, f = -k sum (th0_i - a_i.rv) a_i, tau_c = -R(r)' tau_p
  if (jd.spring_r != 0.0 && jd.nfree_r > 0) {
    M33 Tp, Tc;
    rotvec_attitude_jacobians(jd, g2, Tp, Tc);
    V3 rv = rotation_vector(g2.qr);
    V3 force = v3zero();
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (i < jd.nfree_r) { V3 a = ld3(jd.Ar + 3 * i); force += (-jd.spring_r * (jd.spring_off_r[i] - dot(a, rv))) * a; }
    V3 tp = P.h * (Roff * force);
    V3 tc = (-1.0) * (Rrt * tp);
    M33 Bs = (P.h * jd.spring_r) * (Roff * AtA);
    M33 dpa = Bs * Tp, dpb = Bs * Tc;
    add_block33(BPp, 6, 3, 3, dpa); add_block33(BPc, 6, 3, 3, dpb);
    add_block33(BCp, 6, 3, 3, (-1.0) * (Rrt * dpa) + 2.0 * (Rrt * skew(tp)));
    add_block33(BCc, 6, 3, 3, (-1.0) * (Rrt * dpb) + 2.0 * skew(tc));
  }
  // rotational damper (rotational/dampers.jl:33-64): tau_a = c Roff A'A rotvec(w), w = mb r^-1 conj(ma) r, tau_b = -R(r)' tau_a
  if (jd.damper_r != 0.0 && jd.nfree_r > 0) {
    Quat ma = qmap(ka.w, P.h), mb = qmap(kb.w, P.h);
    Quat rinv = qinv(r);
    Quat rest = qmul(qmul(rinv, qconj(ma)), r);
    Quat wq = qmul(mb, rest);
    M33 B = jd.damper_r * (Roff * AtA);
    V3 ta = B * rotation_vector(wq);
    V3 tb = (-1.0) * (Rrt * ta);
    M34 drv = drotation_vector_dq(wq);
    Quat mbr = qmul(mb, rinv);             // mb r^-1
    Quat cmar = qmul(qconj(ma), r);        // conj(ma) r
    M33 dwa, dwb;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      Quat e = Quat{0.0, kx == 0 ? 1.0 : 0.0, kx == 1 ? 1.0 : 0.0, kx == 2 ? 1.0 : 0.0};
      // r -> r (1, d):   dw = -mb (0,d) rest + w (0,d)
      Quat db = Quat{0, 0, 0, 0};
      {
        Quat t1 = qmul(qmul(mb, e), rest), t2 = qmul(wq, e);
        db = Quat{t2.s - t1.s, t2.x - t1.x, t2.y - t1.y, t2.z - t1.z};
      }
      // qa -> qa (1, d): r -> (1,-d) r:  dw = mb r^-1 (0,d) conj(ma) r - mb r^-1 conj(ma) (0,d) r
      Quat da;
      {
        Quat t1 = qmul(qmul(mbr, e), cmar), t2 = qmul(qmul(qmul(mbr, qconj(ma)), e), r);
        da = Quat{t1.s - t2.s, t1.x - t2.x, t1.y - t2.y, t1.z - t2.z};
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        dwb.m[i][kx] = drv.m[i][0] * db.s + drv.m[i][1] * db.x + drv.m[i][2] * db.y + drv.m[i][3] * db.z;
        dwa.m[i][kx] = drv.m[i][0] * da.s + drv.m[i][1] * da.x + drv.m[i][2] * da.y + drv.m[i][3] * da.z;
      }
    }
    M33 dta_a = B * dwa, dta_b = B * dwb;
    add_block33(BPp, 6, 3, 3, dta_a); add_block33(BPc, 6, 3, 3, dta_b);
    add_block33(BCp, 6, 3, 3, (-1.0) * (Rrt * dta_a) + 2.0 * (Rrt * skew(ta)));
    add_block33(BCc, 6, 3, 3, (-1.0) * (Rrt * dta_b) + 2.0 * skew(tb));
  }
  // joint limits, condensed: slack rows -+(A_i Theta Mqq) -> body rows -kk t (abar_p d phi_a + abar_c d phi_b)
#ifdef DJ_ANY_CONTACT
  if (jd.nb2_r > 0 && !(jd.flags & JF_LIM_TRA)) {
#else
  if (jd.nb2_r > 0) {
#endif
    M33 Tp, Tc;
    rotvec_attitude_jacobians(jd, g3, Tp, Tc);
    Tp = Tp * Ma;
    Tc = Tc * Mb;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nb2_r) {
        V3 ai = ld3(jd.Ar + 3 * i);
        V3 ap = vtmul(ai, Tp), ac = vtmul(ai, Tc);
        const int is_u = ne + i, is_l = ne + jd.nb2_r + i, ig_u = is_u + jd.nb_r, ig_l = is_l + jd.nb_r;
        // a data column enters the slack rows with rs = -sg (ap.dphi_a + ac.dphi_b): the condensed side gives -k_I t (.) on the body rows
        // as in the solver, the kept side the right-hand side -gamma_A' rs_A = sg gamma_A' (.) of its own row ne + i (limit_side)
        const LimitSide ls = limit_side(so[is_u], so[is_l], so[ig_u], so[ig_l]);
        const double* lim = A + jd.lim_off + kLim * i;
        V3 tP = ld3(lim + 6), tC = ld3(lim + 9);
        add_block33(BPp, 6, 3, 3, outer(tP, ap), -ls.kI); add_block33(BPc, 6, 3, 3, outer(tP, ac), -ls.kI);
        add_block33(BCp, 6, 3, 3, outer(tC, ap), -ls.kI); add_block33(BCc, 6, 3, 3, outer(tC, ac), -ls.kI);
        const int q = ne + i;
        st3(RJp + q * 6, v3zero()); st3(RJp + q * 6 + 3, (ls.sg * ls.gA) * ap);
        st3(RJc + q * 6, v3zero()); st3(RJc + q * 6 + 3, (ls.sg * ls.gA) * ac);
      }
    }
  }
  // inputs (gradients/data.jl:137-150, translational/input.jl:33-44, rotational/input.jl:23-39)
  {
    int col = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nfree_t) {
        V3 a = P.input_scaling * ld3(jd.At + 3 * i);
        V3 fp = tmul(g2.Xp, a), tp = 0.25 * tmul(g2.Qtp, a), fc = tmul(g2.Xc, a), tc = 0.25 * tmul(g2.Qtc, a);
        Up[0 * nuj + col] = fp.x; Up[1 * nuj + col] = fp.y; Up[2 * nuj + col] = fp.z; Up[3 * nuj + col] = tp.x; Up[4 * nuj + col] = tp.y; Up[5 * nuj + col] = tp.z;
        Uc[0 * nuj + col] = fc.x; Uc[1 * nuj + col] = fc.y; Uc[2 * nuj + col] = fc.z; Uc[3 * nuj + col] = tc.x; Uc[4 * nuj + col] = tc.y; Uc[5 * nuj + col] = tc.z;
        col++;
      }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < jd.nfree_r) {
        V3 a = P.input_scaling * ld3(jd.Ar + 3 * i);
        V3 tp = (-1.0) * (Roff * a);
        V3 tc = Rrt * (Roff * a);
        Up[0 * nuj + col] = 0; Up[1 * nuj + col] = 0; Up[2 * nuj + col] = 0; Up[3 * nuj + col] = tp.x; Up[4 * nuj + col] = tp.y; Up[5 * nuj + col] = tp.z;
        Uc[0 * nuj + col] = 0; Uc[1 * nuj + col] = 0; Uc[2 * nuj + col] = 0; Uc[3 * nuj + col] = tc.x; Uc[4 * nuj + col] = tc.y; Uc[5 * nuj + col] = tc.z;
        col++;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// (3) columns: right-hand side, substitution, chain rule.  One lane per column; `V` = column vectors [n_red][ch].
// ---------------------------------------------------------------------------------------------------------
DJ_DEV void add_col6(double* V, int ch, int lane, int r_off, const double* B, int ld, int col) {
#pragma unroll
  for (int r = 0; r < 6; ++r) V[(r_off + r) * ch + lane] += B[r * ld + col];
}

DJ_DEV void grad_build_rhs(Ctx& c, double* V, int ch, int col, int lane) {
  const Plan& P = *c.P;
  double* A = c.A;
  for (int r = 0; r < P.n_red; ++r) V[r * ch + lane] = 0.0;
  if (col < 12 * P.Nb) {
    const int b = col / 12, k = col - 12 * b;
    const BodyDev& bd = c.bodies[b];
    if (k >= 3 && k < 6) {  // v15 column: m I on the linear rows (gradients/data.jl:30)
      V[(bd.r_off + (k - 3)) * ch + lane] = bd.mass;
    } else if (k >= 9) {    // w15 column
      const double* dW = A + bd.gb_off;
#pragma unroll
      for (int r = 0; r < 3; ++r) V[(bd.r_off + 3 + r) * ch + lane] = dW[r * 3 + (k - 9)];
    } else {                // x2 (k < 3) or phi2 (6 <= k < 9) column
      const int cc = k < 3 ? k : k - 3;
      const JointDev& pj = c.joints[bd.pjoint];
      {  // parent joint: this body is the child
        const int pnq = joint_nq(pj);
        const double* RJc = A + pj.gj_off + 6 * pnq;
        const double* BPc = RJc + 6 * pnq + 36;
        const double* BCc = BPc + 72;
        for (int r = 0; r < pnq; ++r) V[(pj.r_off + r) * ch + lane] += RJc[r * 6 + cc];
        add_col6(V, ch, lane, bd.r_off, BCc, 6, cc);
        if (pj.parent >= 0) add_col6(V, ch, lane, c.bodies[pj.parent].r_off, BPc, 6, cc);
      }
      for (int q = 0; q < bd.cj_cnt; ++q) {  // child joints: this body is the parent
        const JointDev& cj = c.joints[c.ilist[bd.cj_off + q]];
        const int cnq = joint_nq(cj);
        const double* RJp = A + cj.gj_off;
        const double* BPp = RJp + 12 * cnq;
        const double* BCp = BPp + 72;
        for (int r = 0; r < cnq; ++r) V[(cj.r_off + r) * ch + lane] += RJp[r * 6 + cc];
        add_col6(V, ch, lane, bd.r_off, BPp, 6, cc);
        add_col6(V, ch, lane, c.bodies[cj.child].r_off, BCp, 6, cc);
      }
      for (int q = 0; q < bd.ct_cnt; ++q) add_col6(V, ch, lane, bd.r_off, A + c.contacts[c.ilist[bd.ct_off + q]].gc_off, 6, cc);
    }
  } else if (col >= P.ncol) {  // contact-data column
    const int ci = (col - P.ncol) / 5, p = (col - P.ncol) - 5 * ci;
    double v[6];
    grad_contact_param_rhs(c, ci, p, v);
    const BodyDev& bd = c.bodies[c.contacts[ci].body];
#pragma unroll
    for (int r = 0; r < 6; ++r) V[(bd.r_off + r) * ch + lane] = v[r];
  } else {  // input column
    const int ui = col - 12 * P.Nb;
    const JointDev& jd = c.joints[c.ucol[2 * ui]];
    const int dof = c.ucol[2 * ui + 1], nuj = jd.nfree_t + jd.nfree_r;
    const double* Up = A + jd.gj_off + 12 * joint_nq(jd) + 144;
    const double* Uc = Up + 6 * nuj;
    if (jd.parent >= 0) add_col6(V, ch, lane, c.bodies[jd.parent].r_off, Up, nuj, dof);
    add_col6(V, ch, lane, c.bodies[jd.child].r_off, Uc, nuj, dof);
  }
}

// forward / backward substitution of the block LDU, one column per lane.  Every warp owns a chunk of ch <= 32 columns
// (column vectors V [n_red][ch], per-joint forward scratch at +gvo) and runs ALL elimination steps for it, so the sweeps
// need no barrier between the warps; the warp is split in 32 / ch lane groups that take different (independent) steps of
// a phase for the same columns.
DJ_DEV void grad_solve_columns(Ctx& c, double* V, int ch, int gvo, int c0, int ncol) {
  const Plan& P = *c.P;
  double* A = c.A;
  const int groups = 32 / ch, grp = c.lane / ch, lane = c.lane - grp * ch;  // `lane` = column of the chunk
  const bool active = c0 + lane < ncol;
  for (int ph = 0; ph < P.nphase; ++ph) {
    const int s0 = c.sched[2 * (ph * P.nw)], s1 = c.sched[2 * (ph * P.nw + P.nw - 1)] + c.sched[2 * (ph * P.nw + P.nw - 1) + 1];
    for (int s = s0 + grp; s < s1; s += groups) {
      const ElimStep& st = c.steps[s];
      if (!active) continue;
      double zc[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) zc[k] = (k < st.n) ? V[(st.r_off + k) * ch + lane] : 0.0;
      if (st.fold_cnt > 0) {
        for (int q = 0; q < st.fold_cnt; ++q) {
          double* v = A + c.ilist[st.gfold_off + q] + gvo;
#pragma unroll
          for (int k = 0; k < 6; ++k)
            if (k < st.n) { zc[k] += v[k * ch + lane]; v[k * ch + lane] = 0.0; }
        }
#pragma unroll
        for (int k = 0; k < 6; ++k)
          if (k < st.n) V[(st.r_off + k) * ch + lane] = zc[k];
      }
      // the right-hand sides are sparse (a column touches one body and its neighbours): nodes outside the paths from
      // those to the root still hold exact zeros in the forward sweep and have nothing to propagate
      bool nz = false;
#pragma unroll
      for (int k = 0; k < 6; ++k) nz = nz || (zc[k] != 0.0);
      if (!nz) continue;
      for (int j = 0; j < st.nnb; ++j) {
        const ElimNb& nb = st.nb[j];
        const double* L = A + nb.L_off;
        double* tgt = nb.gv_off >= 0 ? A + nb.gv_off + gvo + nb.row0 * ch : V + nb.r_off * ch;  // row0: sub-range of the parent's scratch rows
        for (int i = 0; i < nb.n; ++i) {
          double acc = 0.0;
#pragma unroll
          for (int k = 0; k < 6; ++k)
            if (k < st.n) acc += L[i * st.n + k] * zc[k];
          tgt[i * ch + lane] -= acc;
        }
      }
    }
    __syncwarp();
  }
  for (int ph = P.nphase - 1; ph >= 0; --ph) {
    const int s0 = c.sched[2 * (ph * P.nw)], s1 = c.sched[2 * (ph * P.nw + P.nw - 1)] + c.sched[2 * (ph * P.nw + P.nw - 1) + 1];
    for (int s = s0 + grp; s < s1; s += groups) {
      const ElimStep& st = c.steps[s];
      if (!active) continue;
      double t[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) t[k] = (k < st.n) ? V[(st.r_off + k) * ch + lane] : 0.0;
      for (int j = 0; j < st.nnb; ++j) {
        const ElimNb& nb = st.nb[j];
        const double* U = A + nb.U_off;
        const double* xj = V + nb.r_off * ch;
        if (nb.U_row == 0) {  // M_{c,nb} holds all st.n rows of c
          for (int kk = 0; kk < nb.n; ++kk) {
            double xv = xj[kk * ch + lane];
#pragma unroll
            for (int r = 0; r < 6; ++r)
              if (r < st.n) t[r] -= U[r * nb.n + kk] * xv;
          }
        } else {  // angular coupling only (dojo_plan.h ElimNb::row0): rows 3..5 of c, stored 3 x n_nb
          for (int kk = 0; kk < nb.n; ++kk) {
            double xv = xj[kk * ch + lane];
#pragma unroll
            for (int r = 0; r < 3; ++r) t[3 + r] -= U[r * nb.n + kk] * xv;
          }
        }
      }
      const double* Dc = A + st.d_off;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        if (r < st.n) {
          double acc = 0.0;
#pragma unroll
          for (int k = 0; k < 6; ++k)
            if (k < st.n) acc += Dc[r * st.n + k] * t[k];
          V[(st.r_off + r) * ch + lane] = acc;
        }
      }
    }
    __syncwarp();
  }
}

// chain rule to (x3, v25, phi3, w25) and write the column (gradients/state.jl:104-123)
// (bodies b0, b0 + bstride, ... of the column: the threads of the slot share a column's bodies)
DJ_DEV void grad_write_column(Ctx& c, const double* V, int ch, int col, int lane, int b0, int bstride, double* __restrict__ Fz, double* __restrict__ Fu,
                              double* __restrict__ Fc) {
  const Plan& P = *c.P;
  const double* A = c.A;
  const int ng = 12 * P.Nb;
  double* out = col < ng ? Fz + (size_t)col * ng : (col < P.ncol ? Fu + (size_t)(col - ng) * ng : Fc + (size_t)(col - P.ncol) * ng);
  for (int b = b0; b < P.Nb; b += bstride) {
    const BodyDev& bd = c.bodies[b];
    const double* rec = A + bd.gb_off;
    V3 dv = v3(V[(bd.r_off + 0) * ch + lane], V[(bd.r_off + 1) * ch + lane], V[(bd.r_off + 2) * ch + lane]);
    V3 dw = v3(V[(bd.r_off + 3) * ch + lane], V[(bd.r_off + 4) * ch + lane], V[(bd.r_off + 5) * ch + lane]);
    V3 dx = P.h * dv;
    V3 dphi = ldm33(rec + 18) * dw;  // E dw
    if (col < ng && col / 12 == b) {
      const int k = col - 12 * b;
      if (k < 3) { if (k == 0) dx.x += 1.0; else if (k == 1) dx.y += 1.0; else dx.z += 1.0; }
      else if (k >= 6 && k < 9) {
        const double* M = rec + 9;
        dphi.x += M[0 * 3 + (k - 6)]; dphi.y += M[1 * 3 + (k - 6)]; dphi.z += M[2 * 3 + (k - 6)];
      }
    }
    double* o = out + 12 * b;
    o[0] = dx.x; o[1] = dx.y; o[2] = dx.z;
    o[3] = dv.x; o[4] = dv.y; o[5] = dv.z;
    o[6] = dphi.x; o[7] = dphi.y; o[8] = dphi.z;
    o[9] = dw.x; o[10] = dw.y; o[11] = dw.z;
  }
}

// the whole gradient pass for one environment; the KKT blocks of the final iterate must be assembled (unfactorised)
// Fc (nullable): [12 Nb x 5 Ni] contact-data gradients, solved as extra columns against the same factor
// u (nullable): this environment's inputs; null leaves the inputs' configuration derivative out (SURVEY.md Q17)
DJ_DEV bool gradients(Ctx& c, const double* __restrict__ u, double* __restrict__ Fz, double* __restrict__ Fu, double* __restrict__ Fc) {
  const Plan& P = *c.P;
  double* A = c.A;
  const WarpRole& role = c.roles[c.warp];
  for (int p = 0; p < role.npass; ++p) {
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_BODY) grad_body(c, idx);
    else if (role.type[p] == ROLE_CONTACT) grad_contact(c, idx);
    else grad_joint(c, idx, u);
  }
  // per-column forward scratch must start from zero
  for (int j = c.tid; j < P.Ne; j += c.nthreads)
    if (c.joints[j].gv_off >= 0)
      for (int t = 0; t < 6 * P.ch; ++t) A[c.joints[j].gv_off + t] = 0.0;
  slot_sync(c);
  bool ok = factorize(c);
  // every warp takes its own chunks of chw = ch / nw columns (workspace slice [n_red][chw], forward scratch slice at +gvo)
  const int chw = P.ch / P.nw;
  double* V = A + P.gvec_off + c.warp * P.n_red * chw;
  const int gvo = c.warp * 6 * chw;
  const int parts = 32 / chw, part = c.lane / chw, l = c.lane - part * chw;
  const int ncol = P.ncol + (Fc ? 5 * P.Ni : 0);
  for (int c0 = c.warp * chw; c0 < ncol; c0 += P.ch) {
    if (part == 0 && c0 + l < ncol) grad_build_rhs(c, V, chw, c0 + l, l);
    __syncwarp();
    grad_solve_columns(c, V, chw, gvo, c0, ncol);
    if (c0 + l < ncol) grad_write_column(c, V, chw, c0 + l, l, part, parts, Fz, Fu, Fc);
    __syncwarp();
  }
  slot_sync(c);
  return ok;
}

// ---------------------------------------------------------------------------------------------------------
// (4) adjoint of the step (dojo_rollout_vjp): lambda' Fz and lambda' Fu for ONE cotangent lambda, without the Jacobians.
// ---------------------------------------------------------------------------------------------------------
// Column col of [Fz Fu] is  C K^-1 rhs_col + d_col  (grad_write_column): C maps the body rows of the condensed system to
// (x3, v25, phi3, w25) -- dx = h dv, dphi = E dw -- and d_col is the direct term (e_k on the x2 columns, M e_k on the phi2 columns).
// So  lambda' col = y' rhs_col + lambda' d_col  with  y = K^-T C' lambda:  one transposed solve instead of 12Nb + nu forward ones.
//
// The block LDU of the factorisation is K = L (D + U): L unit lower (L~_{nb,c} at ElimNb::L_off, applied by the forward sweep of
// grad_solve_columns), D the pivots (their inverses at d_off), U the blocks M_{c,nb} at U_off (backward sweep).  K' y = g is solved as
//   (D + U)' w = g   phases in FORWARD order:  w_c = Dinv_c' g_c, then g_nb -= M_{c,nb}' w_c   (the transposed backward sweep)
//   L' y = w         phases in REVERSE order:  y_c = w_c - sum_nb L~_{nb,c}' y_nb              (the transposed forward sweep)
// The first has the forward sweep's access pattern, so it reaches the same targets the same way: updates of a parent body go to the
// per-joint scratch (ElimNb::gv_off, sub-range row0) that the parent folds in (ElimStep::gfold_off) when its own turn comes; the second
// reads its neighbours where the backward sweep does.  One right-hand side: warp 0 runs it, one lane per step of a phase (y and the
// scratch with stride 1: y in the residual region, which the gradient pass no longer needs once the KKT blocks are assembled).
DJ_DEV void vjp_solve(Ctx& c, double* __restrict__ y) {
  const Plan& P = *c.P;
  double* A = c.A;
  for (int ph = 0; ph < P.nphase; ++ph) {
    const int s0 = c.sched[2 * (ph * P.nw)], s1 = c.sched[2 * (ph * P.nw + P.nw - 1)] + c.sched[2 * (ph * P.nw + P.nw - 1) + 1];
    for (int s = s0 + c.lane; s < s1; s += 32) {
      const ElimStep& st = c.steps[s];
      double g[6], w[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) g[k] = (k < st.n) ? y[st.r_off + k] : 0.0;
      for (int q = 0; q < st.fold_cnt; ++q) {
        double* v = A + c.ilist[st.gfold_off + q];
#pragma unroll
        for (int k = 0; k < 6; ++k)
          if (k < st.n) { g[k] += v[k]; v[k] = 0.0; }
      }
      const double* Dc = A + st.d_off;
      bool nz = false;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        w[r] = 0.0;
        if (r < st.n) {
          double acc = 0.0;
#pragma unroll
          for (int k = 0; k < 6; ++k)
            if (k < st.n) acc += Dc[k * st.n + r] * g[k];
          w[r] = acc;
          y[st.r_off + r] = acc;
          nz = nz || (acc != 0.0);
        }
      }
      if (!nz) continue;
      for (int j = 0; j < st.nnb; ++j) {
        const ElimNb& nb = st.nb[j];
        const double* U = A + nb.U_off;
        double* tgt = nb.gv_off >= 0 ? A + nb.gv_off + nb.row0 : y + nb.r_off;
        for (int kk = 0; kk < nb.n; ++kk) {
          double acc = 0.0;
          if (nb.U_row == 0) {  // M_{c,nb} holds all st.n rows of c
#pragma unroll
            for (int r = 0; r < 6; ++r)
              if (r < st.n) acc += U[r * nb.n + kk] * w[r];
          } else {  // angular coupling only: rows 3..5 of c, stored 3 x n_nb
#pragma unroll
            for (int r = 0; r < 3; ++r) acc += U[r * nb.n + kk] * w[3 + r];
          }
          tgt[kk] -= acc;
        }
      }
    }
    __syncwarp();
  }
  for (int ph = P.nphase - 1; ph >= 0; --ph) {
    const int s0 = c.sched[2 * (ph * P.nw)], s1 = c.sched[2 * (ph * P.nw + P.nw - 1)] + c.sched[2 * (ph * P.nw + P.nw - 1) + 1];
    for (int s = s0 + c.lane; s < s1; s += 32) {
      const ElimStep& st = c.steps[s];
      double t[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) t[k] = (k < st.n) ? y[st.r_off + k] : 0.0;
      for (int j = 0; j < st.nnb; ++j) {
        const ElimNb& nb = st.nb[j];
        const double* L = A + nb.L_off;
        const double* xj = y + nb.r_off;
        for (int i = 0; i < nb.n; ++i) {
          const double xv = xj[i];
#pragma unroll
          for (int k = 0; k < 6; ++k)
            if (k < st.n) t[k] -= L[i * st.n + k] * xv;
        }
      }
#pragma unroll
      for (int k = 0; k < 6; ++k)
        if (k < st.n) y[st.r_off + k] = t[k];
    }
    __syncwarp();
  }
}

// One step of the adjoint pass at the final iterate whose KKT blocks are assembled (unfactorised), as gradients() is called:
// on entry lam [12 Nb] (global memory, this slot's only) holds lambda_{t+1}; on return lambda_t = Fz' lambda_{t+1} + gz, and gu [nu]
// (nullable) = Fu' lambda_{t+1}.  u: the step's inputs (their configuration derivative is part of Fz, as in dojo_rollout_grad).
// Every sum runs in a fixed order on one lane.  Returns false when the factorisation is not finite.
DJ_DEV bool vjp_step(Ctx& c, const double* __restrict__ u, double* __restrict__ lam, const double* __restrict__ gz, double* __restrict__ gu) {
  const Plan& P = *c.P;
  double* A = c.A;
  const WarpRole& role = c.roles[c.warp];
  for (int p = 0; p < role.npass; ++p) {  // the data-Jacobian blocks of gradients()
    const int idx = role_item(role, p, c.lane);
    if (idx < 0) continue;
    if (role.type[p] == ROLE_BODY) grad_body(c, idx);
    else if (role.type[p] == ROLE_CONTACT) grad_contact(c, idx);
    else grad_joint(c, idx, u);
  }
  for (int j = c.tid; j < P.Ne; j += c.nthreads)  // the transposed solve's scratch (stride 1) starts from zero
    if (c.joints[j].gv_off >= 0)
      for (int k = 0; k < 6; ++k) A[c.joints[j].gv_off + k] = 0.0;
  double* y = A + P.rhs_off;
  for (int r = c.tid; r < P.n_red; r += c.nthreads) y[r] = 0.0;
  slot_sync(c);
  const bool ok = factorize(c);
  // right-hand side C' lambda on the body rows (zero on the joint rows): dv <- h lambda_x + lambda_v, dw <- E' lambda_phi + lambda_w.
  // The thread of body b then replaces lambda's 12 entries of b by the direct terms (lambda_x on x2, M' lambda_phi on phi2, 0 elsewhere).
  for (int b = c.tid; b < P.Nb; b += c.nthreads) {
    const BodyDev& bd = c.bodies[b];
    const double* rec = A + bd.gb_off;
    double* l = lam + 12 * b;
    const V3 lx = ld3(l), lv = ld3(l + 3), lp = ld3(l + 6), lw = ld3(l + 9);
    st3(y + bd.r_off, P.h * lx + lv);
    st3(y + bd.r_off + 3, tmul(ldm33(rec + 18), lp) + lw);
    st3(l + 3, v3zero());
    st3(l + 6, tmul(ldm33(rec + 9), lp));
    st3(l + 9, v3zero());
  }
  __threadfence_block();
  slot_sync(c);
  if (c.warp == 0) vjp_solve(c, y);
  slot_sync(c);
  // lambda' col = y' rhs_col + (direct term), one lane per column, the columns built by grad_build_rhs in the chunks of gradients()
  const int ng = 12 * P.Nb;
  const int chw = P.ch / P.nw;
  double* V = A + P.gvec_off + c.warp * P.n_red * chw;
  const int part = c.lane / chw, l = c.lane - part * chw;
  for (int c0 = c.warp * chw; c0 < P.ncol; c0 += P.ch) {
    const int col = c0 + l;
    if (part == 0 && col < P.ncol) grad_build_rhs(c, V, chw, col, l);
    __syncwarp();
    if (part == 0 && col < P.ncol) {
      double s = 0.0;
      for (int r = 0; r < P.n_red; ++r) s += y[r] * V[r * chw + l];
      if (col < ng) lam[col] = (s + lam[col]) + gz[col];
      else if (gu) gu[col - ng] = s;
    }
    __syncwarp();
  }
  __threadfence_block();
  slot_sync(c);
  return ok;
}

}  // namespace dj
