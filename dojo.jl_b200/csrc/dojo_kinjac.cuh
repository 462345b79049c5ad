// dojo_kinjac.cuh -- Jacobians of the minimal <-> maximal coordinate maps and the minimal-coordinate gradients on the
// device (SURVEY.md 8 f1, second half):
//
//   maximal_to_minimal_jacobian   gradients/state.jl:9-56    M(z)  [2 nu x 12 Nb]
//   minimal_to_maximal_jacobian   gradients/state.jl:136-179 N(z)  [12 Nb x 2 nu]
//   get_minimal_gradients!        gradients/state.jl:192-217 dx'/dx = M(z') Fz N(z),  dx'/du = M(z') Fu
//
// The reference composes 4x4 / 3x4 quaternion-matrix products (joints/minimal.jl:206-400, translational/minimal.jl:14-193,
// rotational/minimal.jl:13-174).  Here every partial is written directly for body-frame ATTITUDE increments
// q <- q (x) (1, phi) (the reference's attitude Jacobian LV'(q)), with rotation matrices:
//   * a perturbation phi of q2 moves the previous orientation q1 = q2 (x) m(-w) by R(m)' phi, a perturbation of w by
//     -E(-w) dw (E = attitude_velocity_jacobian);
//   * D LV'(q) = -d_s v' + D_v (s I + [v]x),  D RV'(q) = -d_s v' + D_v (s I - [v]x)  for a 3x4 D = [d_s D_v];
//   * d(R p)/dphi = -2 R [p]x.
// Execution model: one CTA per environment (persistent grid), the threads take (i) one joint / one body each for the
// per-node partials, (ii) one output element each for the tree chain and the dense products.  Per-CTA workspace lives in
// global memory (L2 resident: 2 nu x 24 + 288 Nb + 12 Nb x 2 nu + 2 nu x (12 Nb + nu) doubles).  The functions take
// (tid, nthr) and a barrier functor so that tests/hostcheck can run exactly this code with one "thread" on the CPU.
#pragma once
#include "dojo_kin.cuh"

namespace dj {

struct KinJacArgs {
  const JointDev* joints;
  const int* order;  // joints root -> leaves
  int Ne, Nb, nu, B;
  double h;
  const double* Z;    // [13 Nb x B] state at which N (and the partials) are evaluated
  const double* Zm;   // [13 Nb x B] state at which M is evaluated (z' for the minimal gradients)
  const double* Fz;   // [12 Nb x 12 Nb x B] column-major (get_maximal_gradients), mode 2
  const double* Fu;   // [12 Nb x nu x B]
  double* outM;       // mode 0: [2 nu x 12 Nb x B] column-major, zero-filled by the caller
  double* outN;       // mode 1: [12 Nb x 2 nu x B] column-major
  double* Gx;         // mode 2: [2 nu x 2 nu x B] column-major
  double* Gu;         // mode 2: [2 nu x nu x B]
  double* ws;         // per-CTA workspace, kinjac_ws_doubles() each
  int mode;           // 0: M   1: N   2: minimal gradients
};

#ifdef __CUDACC__
__host__ __device__
#endif
inline size_t kinjac_ws_doubles(int Nb, int nu) {
  return (size_t)2 * nu * 24 + (size_t)288 * Nb + (size_t)12 * Nb * 2 * nu + (size_t)2 * nu * (12 * Nb + nu);
}

// ------------------------------------------------------------------------------------------------ small helpers
DJ_DEV M33 sI_plus(double s, V3 v) { return m33ident(s) + skew(v); }
DJ_DEV M33 sI_minus(double s, V3 v) { return m33ident(s) - skew(v); }
DJ_DEV V3 m34_col0(const M34& d) { return v3(d.m[0][0], d.m[1][0], d.m[2][0]); }
DJ_DEV M33 m34_v(const M34& d) {
  M33 r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = d.m[i][1 + j];
  return r;
}
DJ_DEV M33 D_LVt(const M34& d, Quat q) { return m34_v(d) * sI_plus(q.s, qvec(q)) - outer(m34_col0(d), qvec(q)); }   // D LV'(q)
DJ_DEV M33 D_RVt(const M34& d, Quat q) { return m34_v(d) * sI_minus(q.s, qvec(q)) - outer(m34_col0(d), qvec(q)); }  // D RV'(q)
DJ_DEV V3 mask_row(const double* A, int i) { return v3(A[3 * i], A[3 * i + 1], A[3 * i + 2]); }
DJ_DEV void put_row(double* dst, V3 r) { dst[0] = r.x; dst[1] = r.y; dst[2] = r.z; }
DJ_DEV V3 col(const M33& a, int j) { return v3(a.m[0][j], a.m[1][j], a.m[2][j]); }

// attitude Jacobian of q = axis_angle_to_quaternion(x) (orientation/axis_angle.jl:13-40), column k = s dv_k - ds_k v - sgn (v x dv_k):
//   sgn = +1:  vec(conj(q) (x) dq/dx_k), the body-frame increment of q;   sgn = -1:  -vec(q (x) conj(dq/dx_k)), minus that of conj(q)
DJ_DEV M33 att_exp_jacobian(V3 x, double sgn) {
  const double th = sqrt(dot(x, x));
  M33 r;
  if (!(th > 0.0)) return m33ident(0.5);  // q = 1: dv = I / 2, ds = 0
  const double sh = sin(0.5 * th), ch = cos(0.5 * th);
  const V3 u = (1.0 / th) * x, v = sh * u;
  const M33 dv = (0.5 * ch) * outer(u, u) + (sh / th) * (m33ident() - outer(u, u));
  const V3 ds = (-0.5 * sh) * u;
  for (int k = 0; k < 3; ++k) {
    const V3 dvk = col(dv, k);
    const V3 c = ch * dvk - comp(ds, k) * v - sgn * cross(v, dvk);
    r.m[0][k] = c.x; r.m[1][k] = c.y; r.m[2][k] = c.z;
  }
  return r;
}

// ------------------------------------------------------------------------------------------------ M: one joint
// blk: [2 nu_j][24] row-major, columns [parent x v phi w | child x v phi w]; rows [c_tra; c_rot; v_tra; v_rot].
DJ_DEV void max_to_min_block(const JointDev& jd, const BodyState& A, const BodyState& Bc, double h, double* blk) {
  const int nt = jd.nfree_t, nr = jd.nfree_r, nuj = nt + nr;
  for (int i = 0; i < 2 * nuj * 24; ++i) blk[i] = 0.0;
  const double ih = 1.0 / h;
  const V3 pa = v3(jd.pa[0], jd.pa[1], jd.pa[2]), pb = v3(jd.pb[0], jd.pb[1], jd.pb[2]);
  const Quat ma = qmap(-A.w, h), mb = qmap(-Bc.w, h);
  const Quat qa1 = qmul(A.q, ma), qb1 = qmul(Bc.q, mb);
  const M33 RmaT = transpose(rotmat(ma)), RmbT = transpose(rotmat(mb));
  const M33 Ea = attitude_velocity_jacobian(-A.w, h), Eb = attitude_velocity_jacobian(-Bc.w, h);
  if (nt > 0) {  // translational/minimal.jl:57-65, :93-193
    const V3 xa1 = A.x - h * A.v, xb1 = Bc.x - h * Bc.v;
    const M33 Ra = rotmat(A.q), Rb = rotmat(Bc.q), Ra1 = rotmat(qa1), Rb1 = rotmat(qb1);
    const V3 e = tra_displacement(jd, A.x, A.q, Bc.x, Bc.q), e1 = tra_displacement(jd, xa1, qa1, xb1, qb1);
    const M33 RaT = transpose(Ra), Ra1T = transpose(Ra1);
    const M33 c_pa = 2.0 * skew(e + pa);
    const M33 c_pb = (-2.0) * (RaT * Rb * skew(pb));
    const M33 c1_pa0 = 2.0 * skew(e1 + pa);                // w.r.t. the attitude of qa1
    const M33 c1_pb0 = (-2.0) * (Ra1T * Rb1 * skew(pb));   // w.r.t. the attitude of qb1
    const M33 v_xa = ih * (Ra1T - RaT), v_va = (-1.0) * Ra1T, v_pa = ih * (c_pa - c1_pa0 * RmaT), v_wa = ih * (c1_pa0 * Ea);
    const M33 v_xb = ih * (RaT - Ra1T), v_vb = Ra1T, v_pb = ih * (c_pb - c1_pb0 * RmbT), v_wb = ih * (c1_pb0 * Eb);
    for (int i = 0; i < nt; ++i) {
      const V3 a = mask_row(jd.At, i);
      double* rc = blk + (size_t)i * 24;
      double* rv = blk + (size_t)(nuj + i) * 24;
      put_row(rc + 0, -1.0 * tmul(RaT, a));  put_row(rc + 6, tmul(c_pa, a));
      put_row(rc + 12, tmul(RaT, a));        put_row(rc + 18, tmul(c_pb, a));
      put_row(rv + 0, tmul(v_xa, a));  put_row(rv + 3, tmul(v_va, a));  put_row(rv + 6, tmul(v_pa, a));  put_row(rv + 9, tmul(v_wa, a));
      put_row(rv + 12, tmul(v_xb, a)); put_row(rv + 15, tmul(v_vb, a)); put_row(rv + 18, tmul(v_pb, a)); put_row(rv + 21, tmul(v_wb, a));
    }
  }
  if (nr > 0) {  // rotational/minimal.jl:62-80, :103-174
    const Quat qoff = Quat{jd.qoff[0], jd.qoff[1], jd.qoff[2], jd.qoff[3]};
    const Quat qoffi = qinv(qoff);
    const M33 RoffT = transpose(rotmat(qoff));
    const Quat q = qmul(qmul(qoffi, qinv(A.q)), Bc.q);
    const Quat q1 = qmul(qmul(qoffi, qinv(qa1)), qb1);
    const Quat p = qmul(qinv(q1), q);
    const M34 Dq = drotation_vector_dq(q), Dp = drotation_vector_dq(p);
    const M33 c_pb = D_LVt(Dq, q);
    const M33 c_pa = (-1.0) * (D_RVt(Dq, q) * RoffT);
    const M33 DRp = D_RVt(Dp, p);
    const M33 K = DRp * transpose(rotmat(q1)) * RoffT;
    const M33 v_pb = ih * (D_LVt(Dp, p) - DRp * RmbT);
    const M33 v_wb = ih * (DRp * Eb);
    const M33 v_pa = ih * (K * (RmaT - m33ident()));
    const M33 v_wa = (-ih) * (K * Ea);
    for (int i = 0; i < nr; ++i) {
      const V3 a = mask_row(jd.Ar, i);
      double* rc = blk + (size_t)(nt + i) * 24;
      double* rv = blk + (size_t)(nuj + nt + i) * 24;
      put_row(rc + 6, tmul(c_pa, a));  put_row(rc + 18, tmul(c_pb, a));
      put_row(rv + 6, tmul(v_pa, a));  put_row(rv + 9, tmul(v_wa, a));  put_row(rv + 18, tmul(v_pb, a));  put_row(rv + 21, tmul(v_wb, a));
    }
  }
  if (jd.parent < 0)  // the origin is not a variable (state.jl:28-44)
    for (int r = 0; r < 2 * nuj; ++r) for (int c = 0; c < 12; ++c) blk[(size_t)r * 24 + c] = 0.0;
}

// The same block contracted with a cotangent: out[24] = blk' w for w = the joint's 2 nu_j entries of a minimal-state cotangent, without
// forming blk (the adjoint of the closed loop, dojo_step_kernel.cuh: add_max_to_min_vjp).  The partials are max_to_min_block's, each
// applied to the same mask rows; a world parent's 12 entries are zero.
DJ_DEV void max_to_min_vjp_joint(const JointDev& jd, const BodyState& A, const BodyState& Bc, double h, const double* w, double* out) {
  const int nt = jd.nfree_t, nr = jd.nfree_r, nuj = nt + nr;
  for (int i = 0; i < 24; ++i) out[i] = 0.0;
  // out[c0 .. c0 + 2] += w_r (D' a)
  auto acc = [&](int c0, double wr, V3 r) { out[c0] += wr * r.x; out[c0 + 1] += wr * r.y; out[c0 + 2] += wr * r.z; };
  const double ih = 1.0 / h;
  const V3 pa = v3(jd.pa[0], jd.pa[1], jd.pa[2]), pb = v3(jd.pb[0], jd.pb[1], jd.pb[2]);
  const Quat ma = qmap(-A.w, h), mb = qmap(-Bc.w, h);
  const Quat qa1 = qmul(A.q, ma), qb1 = qmul(Bc.q, mb);
  const M33 RmaT = transpose(rotmat(ma)), RmbT = transpose(rotmat(mb));
  const M33 Ea = attitude_velocity_jacobian(-A.w, h), Eb = attitude_velocity_jacobian(-Bc.w, h);
  if (nt > 0) {
    const V3 xa1 = A.x - h * A.v, xb1 = Bc.x - h * Bc.v;
    const M33 Ra = rotmat(A.q), Rb = rotmat(Bc.q), Ra1 = rotmat(qa1), Rb1 = rotmat(qb1);
    const V3 e = tra_displacement(jd, A.x, A.q, Bc.x, Bc.q), e1 = tra_displacement(jd, xa1, qa1, xb1, qb1);
    const M33 RaT = transpose(Ra), Ra1T = transpose(Ra1);
    const M33 c_pa = 2.0 * skew(e + pa);
    const M33 c_pb = (-2.0) * (RaT * Rb * skew(pb));
    const M33 c1_pa0 = 2.0 * skew(e1 + pa);
    const M33 c1_pb0 = (-2.0) * (Ra1T * Rb1 * skew(pb));
    const M33 v_xa = ih * (Ra1T - RaT), v_va = (-1.0) * Ra1T, v_pa = ih * (c_pa - c1_pa0 * RmaT), v_wa = ih * (c1_pa0 * Ea);
    const M33 v_xb = ih * (RaT - Ra1T), v_vb = Ra1T, v_pb = ih * (c_pb - c1_pb0 * RmbT), v_wb = ih * (c1_pb0 * Eb);
    for (int i = 0; i < nt; ++i) {
      const V3 a = mask_row(jd.At, i);
      const double wc = w[i], wv = w[nuj + i];
      acc(0, wc, -1.0 * tmul(RaT, a));  acc(6, wc, tmul(c_pa, a));  acc(12, wc, tmul(RaT, a));  acc(18, wc, tmul(c_pb, a));
      acc(0, wv, tmul(v_xa, a));  acc(3, wv, tmul(v_va, a));  acc(6, wv, tmul(v_pa, a));  acc(9, wv, tmul(v_wa, a));
      acc(12, wv, tmul(v_xb, a)); acc(15, wv, tmul(v_vb, a)); acc(18, wv, tmul(v_pb, a)); acc(21, wv, tmul(v_wb, a));
    }
  }
  if (nr > 0) {
    const Quat qoff = Quat{jd.qoff[0], jd.qoff[1], jd.qoff[2], jd.qoff[3]};
    const Quat qoffi = qinv(qoff);
    const M33 RoffT = transpose(rotmat(qoff));
    const Quat q = qmul(qmul(qoffi, qinv(A.q)), Bc.q);
    const Quat q1 = qmul(qmul(qoffi, qinv(qa1)), qb1);
    const Quat p = qmul(qinv(q1), q);
    const M34 Dq = drotation_vector_dq(q), Dp = drotation_vector_dq(p);
    const M33 c_pb = D_LVt(Dq, q);
    const M33 c_pa = (-1.0) * (D_RVt(Dq, q) * RoffT);
    const M33 DRp = D_RVt(Dp, p);
    const M33 K = DRp * transpose(rotmat(q1)) * RoffT;
    const M33 v_pb = ih * (D_LVt(Dp, p) - DRp * RmbT);
    const M33 v_wb = ih * (DRp * Eb);
    const M33 v_pa = ih * (K * (RmaT - m33ident()));
    const M33 v_wa = (-ih) * (K * Ea);
    for (int i = 0; i < nr; ++i) {
      const V3 a = mask_row(jd.Ar, i);
      const double wc = w[nt + i], wv = w[nuj + nt + i];
      acc(6, wc, tmul(c_pa, a));  acc(18, wc, tmul(c_pb, a));
      acc(6, wv, tmul(v_pa, a));  acc(9, wv, tmul(v_wa, a));  acc(18, wv, tmul(v_pb, a));  acc(21, wv, tmul(v_wb, a));
    }
  }
  if (jd.parent < 0)  // the origin is not a variable
    for (int c = 0; c < 12; ++c) out[c] = 0.0;
}

// body b's 12 entries of M' w from the per-joint contributions contrib [Ne][24] of max_to_min_vjp_joint: the joints b is the parent or
// the child of, in joint order
DJ_DEV void max_to_min_vjp_fold(const JointDev* joints, int Ne, int b, const double* contrib, double* g) {
  for (int k = 0; k < 12; ++k) g[k] = 0.0;
  for (int j = 0; j < Ne; ++j) {
    const JointDev& jd = joints[j];
    if (jd.nfree_t + jd.nfree_r == 0) continue;
    const double* s = contrib + (size_t)24 * j;
    if (jd.parent == b)
      for (int k = 0; k < 12; ++k) g[k] += s[k];
    if (jd.child == b)
      for (int k = 0; k < 12; ++k) g[k] += s[12 + k];
  }
}

// ------------------------------------------------------------------------------------------------ N: one body
// Partials of set_minimal_coordinates_velocities! (joints/minimal.jl:148-203) for the child of joint jd:
//   Pm [12][12] row-major: d(xb, vb, phi_b, wb) / d(Dx, Dtheta, Dv, Dw)  (2 nu_j columns used)   (:314-400)
//   Pp [12][12] row-major: d(xb, vb, phi_b, wb) / d(xa, va, phi_a, wa)                           (:206-312)
// evaluated at the parent state A and the joint's minimal coordinates xm; qb_state is the child's stored orientation, which
// the reference uses for the attitude reduction LV'(qb)' of the orientation rows (:308, :398).
DJ_DEV void put_block(double* P, int r0, int c0, const M33& a) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) P[(r0 + i) * 12 + c0 + j] = a.m[i][j];
}
DJ_DEV void put_col(double* P, int r0, int c, V3 v) { P[(r0 + 0) * 12 + c] = v.x; P[(r0 + 1) * 12 + c] = v.y; P[(r0 + 2) * 12 + c] = v.z; }

DJ_DEV void min_to_max_partials(const JointDev& jd, const BodyState& A, Quat qb_state, const double* xm, double h, double* Pm, double* Pp) {
  const int nt = jd.nfree_t, nr = jd.nfree_r, nuj = nt + nr;
  for (int i = 0; i < 144; ++i) { Pm[i] = 0.0; Pp[i] = 0.0; }
  const double ih = 1.0 / h;
  const V3 pa = v3(jd.pa[0], jd.pa[1], jd.pa[2]), pb = v3(jd.pb[0], jd.pb[1], jd.pb[2]);
  const Quat qoff = Quat{jd.qoff[0], jd.qoff[1], jd.qoff[2], jd.qoff[3]};
  const V3 dx = masked_sum(jd.At, nt, xm), dth = masked_sum(jd.Ar, nr, xm + nt);
  const V3 dv = masked_sum(jd.At, nt, xm + nuj), dw = masked_sum(jd.Ar, nr, xm + nuj + nt);
  // the map itself (joints/minimal.jl:175-197)
  const Quat dq = axis_angle_to_quaternion(dth);
  const Quat S = qmul(qoff, dq);
  const Quat qb = qmul(A.q, S);
  const Quat ma = qmap(-A.w, h);
  const Quat qa1 = qmul(A.q, ma);
  const V3 dx1 = dx - h * dv;
  const Quat W = axis_angle_to_quaternion(h * dw);
  const Quat S1 = qmul(qoff, qmul(dq, qinv(W)));
  const Quat qb1 = qmul(qa1, S1);
  const M33 Ra = rotmat(A.q), Ra1 = rotmat(qa1), Rb = rotmat(qb), Rb1 = rotmat(qb1);
  const M33 RST = transpose(rotmat(S)), RS1T = transpose(rotmat(S1)), RmT = transpose(rotmat(ma));
  const M33 Ea = attitude_velocity_jacobian(-A.w, h);
  const Quat r = qmul(qconj(qb1), qb);   // wb = (2 / h) vec(r)
  const M33 Kp = sI_plus(r.s, qvec(r)), Km = sI_minus(r.s, qvec(r));
  const Quat c = qmul(qconj(qb_state), qb);
  const M33 C = sI_plus(c.s, qvec(c));   // LV'(qb_state)' applied to qb (x) (0, phi)
  const M33 Bx = 2.0 * (Rb * skew(pb)), Bx1 = 2.0 * (Rb1 * skew(pb));  // d(-R pb) / d(attitude)
  if (jd.parent >= 0) {
    const M33 X_pa = (-2.0) * (Ra * skew(pa + dx)) + Bx * RST;
    const M33 X1_pa0 = (-2.0) * (Ra1 * skew(pa + dx1)) + Bx1 * RS1T;  // w.r.t. the attitude of qa1
    put_block(Pp, 0, 0, m33ident());
    put_block(Pp, 0, 6, X_pa);
    put_block(Pp, 3, 3, m33ident());
    put_block(Pp, 3, 6, ih * (X_pa - X1_pa0 * RmT));
    put_block(Pp, 3, 9, ih * (X1_pa0 * Ea));
    put_block(Pp, 6, 6, C * RST);
    put_block(Pp, 9, 6, (2.0 * ih) * (Kp * RST - Km * RS1T * RmT));
    put_block(Pp, 9, 9, (2.0 * ih) * (Km * RS1T * Ea));
  }
  for (int k = 0; k < nt; ++k) {
    const V3 a = mask_row(jd.At, k);
    put_col(Pm, 0, k, Ra * a);
    put_col(Pm, 3, k, ih * (Ra * a - Ra1 * a));
    put_col(Pm, 3, nuj + k, Ra1 * a);
  }
  if (nr > 0) {
    const M33 Th = att_exp_jacobian(dth, 1.0), ThW = att_exp_jacobian(h * dw, -1.0);
    const M33 RW = rotmat(W);
    for (int k = 0; k < nr; ++k) {
      const V3 a = mask_row(jd.Ar, k);
      const V3 pf = Th * a;        // attitude increment of qb per unit Dtheta_k
      const V3 p1 = RW * pf;       // ... of qb1
      put_col(Pm, 0, nt + k, Bx * pf);
      put_col(Pm, 3, nt + k, ih * (Bx * pf - Bx1 * p1));
      put_col(Pm, 6, nt + k, C * pf);
      put_col(Pm, 9, nt + k, (2.0 * ih) * (Kp * pf - Km * p1));
      const V3 pw = (-h) * (ThW * a);  // attitude increment of qb1 per unit Dw_k
      put_col(Pm, 3, nuj + nt + k, (-ih) * (Bx1 * pw));
      put_col(Pm, 9, nuj + nt + k, (-2.0 * ih) * (Km * pw));
    }
  }
}

// minimal coordinates of one joint from the maximal state (mechanism/state.jl:44-66); same arithmetic as max_to_min_env
DJ_DEV void joint_minimal(const JointDev& jd, const BodyState& A, const BodyState& Bc, double h, double* xm) {
  const int nt = jd.nfree_t, nr = jd.nfree_r, nuj = nt + nr;
  const Quat qoffi = qinv(Quat{jd.qoff[0], jd.qoff[1], jd.qoff[2], jd.qoff[3]});
  const V3 xa1 = A.x - h * A.v, xb1 = Bc.x - h * Bc.v;
  const Quat qa1 = next_orientation(A.q, -A.w, h), qb1 = next_orientation(Bc.q, -Bc.w, h);
  const V3 et = tra_displacement(jd, A.x, A.q, Bc.x, Bc.q);
  const V3 et1 = tra_displacement(jd, xa1, qa1, xb1, qb1);
  const Quat q = qmul(qmul(qoffi, qinv(A.q)), Bc.q);
  const Quat q1 = qmul(qmul(qoffi, qinv(qa1)), qb1);
  const V3 th = rotation_vector(q);
  const V3 dth = (1.0 / h) * rotation_vector(qmul(qinv(q1), q));
  const V3 det = (1.0 / h) * (et - et1);
  for (int i = 0; i < nt; ++i) { const V3 ai = mask_row(jd.At, i); xm[i] = dot(ai, et); xm[nuj + i] = dot(ai, det); }
  for (int i = 0; i < nr; ++i) { const V3 ai = mask_row(jd.Ar, i); xm[nt + i] = dot(ai, th); xm[nuj + nt + i] = dot(ai, dth); }
}

// ------------------------------------------------------------------------------------------------ one environment
// Sync: barrier between the phases (__syncthreads on the device, nothing on the host with nthr = 1).
template <class Sync>
DJ_DEV void kinjac_env(const KinJacArgs& a, int e, double* ws, int tid, int nthr, Sync sync) {
  const int Nb = a.Nb, Ne = a.Ne, nu = a.nu, nm = 2 * nu, ns = 12 * Nb, nc = ns + nu;
  double* Mb = ws;                            // [2 nu][24]
  double* Pm = Mb + (size_t)nm * 24;          // [Nb][144]
  double* Pp = Pm + (size_t)144 * Nb;         // [Nb][144]
  double* Nw = Pp + (size_t)144 * Nb;         // [12 Nb x 2 nu] column-major
  double* T = Nw + (size_t)ns * nm;           // [2 nu][12 Nb + nu] row-major
  const double* z = a.Z + (size_t)e * 13 * Nb;
  const double* zm = a.Zm + (size_t)e * 13 * Nb;
  // ---- phase 1: per-joint blocks of M at zm, per-body partials at z
  for (int t = tid; t < 2 * Ne; t += nthr) {
    if (t < Ne) {
      if (a.mode == 1) continue;
      const JointDev& jd = a.joints[t];
      if (jd.nfree_t + jd.nfree_r == 0) continue;
      max_to_min_block(jd, kin_load(zm, jd.parent), kin_load(zm, jd.child), a.h, Mb + (size_t)2 * jd.u_off * 24);
    } else {
      if (a.mode == 0) continue;
      const JointDev& jd = a.joints[t - Ne];
      const BodyState A = kin_load(z, jd.parent), Bc = kin_load(z, jd.child);
      double xm[12];
      joint_minimal(jd, A, Bc, a.h, xm);
      min_to_max_partials(jd, A, Bc.q, xm, a.h, Pm + (size_t)144 * jd.child, Pp + (size_t)144 * jd.child);
    }
  }
  sync();
  if (a.mode == 0) {  // scatter the blocks into the dense (zero-filled) output
    double* out = a.outM + (size_t)e * nm * ns;
    for (int t = tid; t < Ne * 24; t += nthr) {
      const JointDev& jd = a.joints[t / 24];
      const int c = t % 24, nuj = jd.nfree_t + jd.nfree_r;
      const int body = c < 12 ? jd.parent : jd.child;
      if (body < 0) continue;
      for (int r = 0; r < 2 * nuj; ++r) out[(size_t)(12 * body + c % 12) * nm + 2 * jd.u_off + r] = Mb[(size_t)(2 * jd.u_off + r) * 24 + c];
    }
    return;
  }
  // ---- phase 2: chain the partials root -> leaves:  N_i = Pm_i E_j + Pp_i N_parent(i)
  double* N = a.mode == 1 ? a.outN + (size_t)e * ns * nm : Nw;
  for (int k = 0; k < Ne; ++k) {
    const JointDev& jd = a.joints[a.order[k]];
    const int i = jd.child, p = jd.parent, c0 = 2 * jd.u_off, c1 = c0 + 2 * (jd.nfree_t + jd.nfree_r);
    const double* pm = Pm + (size_t)144 * i;
    const double* pp = Pp + (size_t)144 * i;
    for (int t = tid; t < 12 * nm; t += nthr) {
      const int r = t % 12, c = t / 12;
      double acc = (c >= c0 && c < c1) ? pm[r * 12 + (c - c0)] : 0.0;
      if (p >= 0) {
        const double* np = N + (size_t)c * ns + 12 * p;
        for (int q = 0; q < 12; ++q) acc += pp[r * 12 + q] * np[q];
      }
      N[(size_t)c * ns + 12 * i + r] = acc;
    }
    sync();
  }
  if (a.mode == 1) return;
  // ---- phase 3: T = M [Fz Fu]   (M is block sparse: 24 columns per joint)
  const double* Fz = a.Fz + (size_t)e * ns * ns;
  const double* Fu = a.Fu + (size_t)e * ns * nu;
  for (int c = tid; c < nc; c += nthr) {
    const double* f = c < ns ? Fz + (size_t)c * ns : Fu + (size_t)(c - ns) * ns;
    for (int j = 0; j < Ne; ++j) {
      const JointDev& jd = a.joints[j];
      const int nuj = jd.nfree_t + jd.nfree_r;
      if (nuj == 0) continue;
      double fa[12], fb[12];
      for (int q = 0; q < 12; ++q) { fa[q] = jd.parent >= 0 ? f[12 * jd.parent + q] : 0.0; fb[q] = f[12 * jd.child + q]; }
      for (int r = 0; r < 2 * nuj; ++r) {
        const double* m = Mb + (size_t)(2 * jd.u_off + r) * 24;
        double acc = 0.0;
        for (int q = 0; q < 12; ++q) acc += m[q] * fa[q];
        for (int q = 0; q < 12; ++q) acc += m[12 + q] * fb[q];
        T[(size_t)(2 * jd.u_off + r) * nc + c] = acc;
      }
    }
  }
  sync();
  // ---- phase 4: dx'/dx = T[:, :12Nb] N,  dx'/du = T[:, 12Nb:]
  double* Gx = a.Gx + (size_t)e * nm * nm;
  double* Gu = a.Gu + (size_t)e * nm * nu;
  for (int t = tid; t < nm * nc - nm * ns + nm * nm; t += nthr) {
    if (t < nm * nm) {
      const int r = t % nm, c = t / nm;
      const double* tr = T + (size_t)r * nc;
      const double* ncol = Nw + (size_t)c * ns;
      double acc = 0.0;
      for (int q = 0; q < ns; ++q) acc += tr[q] * ncol[q];
      Gx[(size_t)c * nm + r] = acc;
    } else {
      const int t2 = t - nm * nm, r = t2 % nm, c = t2 / nm;
      Gu[(size_t)c * nm + r] = T[(size_t)r * nc + ns + c];
    }
  }
}

// ------------------------------------------------------------------------------------------------ adjoints of the two maps
// Reverse mode through the maps without forming M or N (dojo_maximal_to_minimal_vjp / dojo_minimal_to_maximal_vjp):
//   gZ = M(z)' gX   [12 Nb] <- [2 nu]      gX = N(z)' gZ   [2 nu] <- [12 Nb]
// n states, layouts [feature x n]; every output entry is one lane's sum in a fixed order, so a state's result does not depend on n,
// the grid or the other states.
struct MapVjpArgs {
  const JointDev* joints;
  const int* order;   // joints root -> leaves
  int Ne, Nb, nu, n;
  double h;
  const double* Z;    // [13 Nb x n] the maximal states (for N': minimal_to_maximal(X))
  const double* in;   // M': gX [2 nu x n]    N': gZ [12 Nb x n], packing [x, v, phi, w] per body
  double* out;        // M': gZ [12 Nb x n]   N': gX [2 nu x n]
  double* ws;         // N': per-CTA workspace, min_to_max_vjp_ws_doubles() each
};

#ifdef __CUDACC__
__host__ __device__
#endif
inline size_t min_to_max_vjp_ws_doubles(int Nb) { return (size_t)300 * Nb; }  // Pm, Pp [Nb][144], the accumulators [12 Nb]

// gZ = M(z)' gX for state e: the closed-loop adjoint's two routines (add_max_to_min_vjp), one lane per joint, then one lane per body.
// s: [24 Ne] scratch of this state's lanes.
template <class Sync>
DJ_DEV void max_to_min_vjp_env(const MapVjpArgs& a, int e, double* s, int tid, int nthr, Sync sync) {
  const double* z = a.Z + (size_t)e * 13 * a.Nb;
  const double* w = a.in + (size_t)e * 2 * a.nu;
  for (int j = tid; j < a.Ne; j += nthr) {
    const JointDev& jd = a.joints[j];
    if (jd.nfree_t + jd.nfree_r > 0) max_to_min_vjp_joint(jd, kin_load(z, jd.parent), kin_load(z, jd.child), a.h, w + 2 * jd.u_off, s + (size_t)24 * j);
  }
  sync();
  double* gz = a.out + (size_t)e * 12 * a.Nb;
  for (int b = tid; b < a.Nb; b += nthr) {
    double g[12];
    max_to_min_vjp_fold(a.joints, a.Ne, b, s, g);
    for (int k = 0; k < 12; ++k) gz[12 * b + k] = g[k];
  }
}

// gX = N(z)' gZ for state e: the transpose of kinjac_env's phase-2 chain N_i = Pm_i E_j + Pp_i N_parent(i).  Phase 1 evaluates the
// partials exactly as kinjac_env does; phase 2 walks the joints leaves -> root (the reverse of `order`) with one accumulator per body:
//   gbar_i = gZ_i + sum over the children c of i of Pp_c' gbar_c,    gX[joint of child i] = Pm_i[:, :2 nu_j]' gbar_i.
// A body's accumulator is complete when its own joint is reached, since every joint of which it is the parent comes later in `order`.
// One barrier per joint; lanes take the joint's 2 nu_j + 12 outputs.
template <class Sync>
DJ_DEV void min_to_max_vjp_env(const MapVjpArgs& a, int e, double* ws, int tid, int nthr, Sync sync) {
  const int Nb = a.Nb, Ne = a.Ne;
  double* Pm = ws;                      // [Nb][144]
  double* Pp = Pm + (size_t)144 * Nb;   // [Nb][144]
  double* gb = Pp + (size_t)144 * Nb;   // [12 Nb]
  const double* z = a.Z + (size_t)e * 13 * Nb;
  const double* gz = a.in + (size_t)e * 12 * Nb;
  double* gx = a.out + (size_t)e * 2 * a.nu;
  for (int t = tid; t < Ne; t += nthr) {
    const JointDev& jd = a.joints[t];
    const BodyState A = kin_load(z, jd.parent), Bc = kin_load(z, jd.child);
    double xm[12];
    joint_minimal(jd, A, Bc, a.h, xm);
    min_to_max_partials(jd, A, Bc.q, xm, a.h, Pm + (size_t)144 * jd.child, Pp + (size_t)144 * jd.child);
  }
  for (int k = tid; k < 12 * Nb; k += nthr) gb[k] = gz[k];
  sync();
  for (int k = Ne - 1; k >= 0; --k) {
    const JointDev& jd = a.joints[a.order[k]];
    const int i = jd.child, p = jd.parent, m = 2 * (jd.nfree_t + jd.nfree_r), c0 = 2 * jd.u_off;
    const double* pm = Pm + (size_t)144 * i;
    const double* pp = Pp + (size_t)144 * i;
    const double* gi = gb + 12 * i;
    for (int t = tid; t < m + 12; t += nthr) {
      if (t < m) {
        double acc = 0.0;
        for (int r = 0; r < 12; ++r) acc += pm[r * 12 + t] * gi[r];
        gx[c0 + t] = acc;
      } else if (p >= 0) {
        const int q = t - m;
        double acc = gb[12 * p + q];
        for (int r = 0; r < 12; ++r) acc += pp[r * 12 + q] * gi[r];
        gb[12 * p + q] = acc;
      }
    }
    sync();
  }
}

#if defined(DJ_HOSTEMU) || (defined(__CUDACC__) && !defined(DJ_ANY_CONTACT))  // dojo_b200_cm.cu includes the routines above only
// persistent grid: CTA b takes environments b, b + gridDim.x, ...; workspace slice b
__global__ void __launch_bounds__(128) dojo_kinjac_kernel(const KinJacArgs a) {
  double* ws = a.ws + (size_t)blockIdx.x * kinjac_ws_doubles(a.Nb, a.nu);
  for (int e = blockIdx.x; e < a.B; e += gridDim.x) {
    kinjac_env(a, e, ws, (int)threadIdx.x, (int)blockDim.x, [] { __syncthreads(); });
    __syncthreads();  // the workspace is reused by the next environment
  }
}

// M': a group of G lanes (a power of two <= 32, inside one warp) per state, blockDim.x / G states per CTA, one state per group; the
// dynamic shared memory holds the [24 Ne] scratch of every group.  Groups never wait for each other.
__global__ void __launch_bounds__(128) dojo_max_to_min_vjp_kernel(const MapVjpArgs a, int G) {
#ifdef DJ_HOSTEMU
  double* smem = hostemu_smem();
#else
  extern __shared__ double smem[];
#endif
  const int g = (int)threadIdx.x / G, lane = (int)threadIdx.x % G;
  const int e = (int)blockIdx.x * ((int)blockDim.x / G) + g;
  if (e >= a.n) return;
  const unsigned mask = G == 32 ? 0xffffffffu : ((1u << G) - 1u) << ((threadIdx.x & 31) & ~(unsigned)(G - 1));
  max_to_min_vjp_env(a, e, smem + (size_t)g * 24 * a.Ne, lane, G, [mask] { __syncwarp(mask); });
}

// N': one warp per state, persistent grid: CTA b takes states b, b + gridDim.x, ...; workspace slice b (global memory, L2 resident)
__global__ void __launch_bounds__(32) dojo_min_to_max_vjp_kernel(const MapVjpArgs a) {
  double* ws = a.ws + (size_t)blockIdx.x * min_to_max_vjp_ws_doubles(a.Nb);
  for (int e = blockIdx.x; e < a.n; e += gridDim.x)
    min_to_max_vjp_env(a, e, ws, (int)threadIdx.x, (int)blockDim.x, [] { __syncwarp(); });  // ends with a barrier: ws is free again
}
#endif

}  // namespace dj
