// oracle/dojo_oracle.cpp -- TEST INFRASTRUCTURE: CPU fp64 restatement of the reference hot path.
//
// This file is the *checker* for the CUDA path in dojo.jl_b200/csrc/.  Only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
// It is never linked into, called from, or used as a fallback by the product library.
//
// PARITY STATUS: "parity unpinned".  The reference is pure Julia, Julia is not installed in the
// build image, and the reference ships no golden vectors (SURVEY.md §8c).  The oracle is pinned
// only by the reference's own *property* tests restated in tests/ (finite-difference Jacobians,
// momentum conservation, behaviours) -- see oracle/README.md.
//
// Each function cites the reference file:line it restates (paths relative to the reference's src/).
// The block-LDU follows GraphBasedSystems.jl (external dependency, compat "1.0, 1.2", not vendored):
// in-place block LDU without pivoting across blocks, explicit inverses of the diagonal blocks,
// leaves-to-root elimination (SURVEY.md Appendix C).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>
#include <thread>
#include <vector>

#include "../include/dojo_b200.h"
#include "dojo_math.hpp"

namespace dojo_oracle {

static const double REG = 1.0e-10;  // Dojo.jl:4

// ------------------------------------------------------------------------------------------
// State containers
// ------------------------------------------------------------------------------------------
struct BodyS {  // bodies/state.jl:25-69
  double mass = 0;
  M33 J;
  V3 x1, v15, w15, x2, JF2, Jt2, Fext, text;
  Quat q1, q2;
  V3 vsol[2], wsol[2];
};

struct Elem {  // Translational / Rotational (joints/*/constructor.jl)
  int kind = 0;  // 0 translational, 1 rotational
  int nl = 0, nb2 = 0, nb = 0, n = 0, nfree = 3;
  double C[3][3], A[3][3];  // constraint_mask / nullspace_mask rows (joints/joint.jl:56-64)
  double spring = 0, damper = 0;
  double spring_offset[3] = {0, 0, 0}, lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  V3 input;
};

struct JointS {  // joints/constraints.jl:17-86
  int parent = -1, child = 0;
  V3 pa, pb;
  Quat qoff;
  Elem el[2];
  int n = 0, nu = 0, sol_off = 0, u_off = 0;
  int eoff[2] = {0, 0};
  bool spring = false, damper = false;
  std::vector<double> imp[2];
  V3 applied[2];  // the scaled input of the last set_input: translational force, rotational torque (joint frame)
};

struct ContactS {  // contacts/constructor.jl:14-43 + {nonlinear.jl:12-48, linear.jl:10-47, impact.jl:8-39} + sphere_halfspace.jl:11-24
  int type = 2;    // 0 ImpactContact{T,2}, 1 LinearContact{T,12}, 2 NonlinearContact{T,8}
  int nh = 4;      // N½: impact 1, nonlinear 4, linear 6; the node's entry is [s(nh); γ(nh)]
  int body = 0, sol_off = 0;
  double mu_f = 0, radius = 0;
  Mat<2, 3> t;
  Mat<1, 3> nrm;
  V3 o, off;
  double gam[2][6], s[2][6];
  // neutral_vector: nonlinear [1,1,0,0] (nonlinear.jl:99), impact / linear ones(N½) (contact.jl:196)
  double neutral(int i) const { return type == 2 ? (i < 2 ? 1.0 : 0.0) : 1.0; }
  // cone_degree: nonlinear 2 (nonlinear.jl:101), impact / linear N½ (contact.jl:197)
  int cone_degree() const { return type == 2 ? 2 : nh; }
};
// friction_parameterization of LinearContact (linear.jl:29-34) / NonlinearContact (identity, nonlinear.jl:40-43)
static const double kLinearParam[4][2] = {{0.0, 1.0}, {0.0, -1.0}, {1.0, 0.0}, {-1.0, 0.0}};

struct Cfg {  // (x, v, q, w) of a node; the origin is all-zero / identity (bodies/origin.jl)
  V3 x, v, w;
  Quat q;
};

// variable-height results for one joint element (n <= 12)
struct EVec { int n = 0; double v[12] = {0}; };
struct EJac7 { int n = 0; Mat<12, 7> J; };
struct EMap { int n = 0; Mat<6, 12> G; };

// ------------------------------------------------------------------------------------------
// Integrator (integrators/integrator.jl)
// ------------------------------------------------------------------------------------------
static V3 next_position(const V3& x2, const V3& v25, double h) { return x2 + v25 * h; }  // :14
static Quat next_orientation(const Quat& q2, const V3& w25, double h) {                   // :15
  return q2 * quaternion_map(w25, h) * h / 2.0;
}
static M43 rotational_integrator_jacobian_velocity(const Quat& q2, const V3& w25, double h) {  // :65-67
  return Lmat(q2) * quaternion_map_jacobian(w25, h) * h / 2.0;
}
static M44 rotational_integrator_jacobian_orientation_full(const V3& w25, double h) {  // :58-63 attjac=false
  return Rmat(quaternion_map(w25, h) * h / 2.0);
}
static Mat<7, 6> integrator_jacobian_velocity(const Quat& q2, const V3& w25, double h) {  // :35-39
  Mat<7, 6> m;
  for (int i = 0; i < 3; ++i) m(i, i) = h;
  set_block(m, 3, 3, rotational_integrator_jacobian_velocity(q2, w25, h));
  return m;
}
static Mat<7, 6> integrator_jacobian_configuration_att(const Quat& q2, const V3& w25, double h) {  // :41-48
  Mat<7, 6> m;
  for (int i = 0; i < 3; ++i) m(i, i) = 1.0;
  set_block(m, 3, 3, rotational_integrator_jacobian_orientation_full(w25, h) * LVtmat(q2));
  return m;
}

// ------------------------------------------------------------------------------------------
// Joint element kinematics
// ------------------------------------------------------------------------------------------
struct XQ { M33 X; M34 Q; };

// translational/minimal.jl:4-12
static V3 tra_displacement(const JointS& j, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb, bool rotate = true) {
  V3 d = xb + vector_rotate(j.pb, qb) - (xa + vector_rotate(j.pa, qa));
  return rotate ? vector_rotate(d, inv(qa)) : d;
}
// translational/minimal.jl:14-30
static XQ tra_displacement_jacobian(bool parent, const JointS& j, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb) {
  XQ r;
  if (parent) {
    V3 d = xb + vector_rotate(j.pb, qb) - (xa + vector_rotate(j.pa, qa));
    r.X = -rotation_matrix(inv(qa));
    r.Q = -rotation_matrix(inv(qa)) * drotation_matrix_dq(qa, j.pa);
    r.Q += drotation_matrix_inv_dq(qa, d);
  } else {
    r.X = rotation_matrix(inv(qa));
    r.Q = rotation_matrix(inv(qa)) * drotation_matrix_dq(qb, j.pb);
  }
  return r;
}
// rotational/minimal.jl:4-11
static Quat rot_displacement_q(const JointS& j, const Quat& qa, const Quat& qb) { return inv(j.qoff) * inv(qa) * qb; }
// rotational/minimal.jl:13-26 (vmat=false, attjac=false): 4x4
static M44 rot_displacement_jacobian_q4(bool parent, const JointS& j, const Quat& qa, const Quat& qb) {
  return parent ? Ltmat(j.qoff) * Rmat(qb) * Tmat() : Ltmat(j.qoff) * Ltmat(qa);
}
// rotational/minimal.jl:28-40
static XQ rot_displacement_jacobian(bool parent, const JointS& j, const Quat& qa, const Quat& qb) {
  XQ r;
  r.Q = Vmat() * rot_displacement_jacobian_q4(parent, j, qa, qb);
  return r;
}
static V3 displacement(const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb) {
  return k == 0 ? tra_displacement(j, xa, qa, xb, qb) : Vmat(rot_displacement_q(j, qa, qb));
}
static XQ displacement_jacobian(bool parent, const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb) {
  return k == 0 ? tra_displacement_jacobian(parent, j, xa, qa, xb, qb) : rot_displacement_jacobian(parent, j, qa, qb);
}

// minimal coordinates: translational/minimal.jl:57-59, rotational/minimal.jl:62-67
static void minimal_coordinates(const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb, double* th) {
  const Elem& e = j.el[k];
  V3 d = k == 0 ? tra_displacement(j, xa, qa, xb, qb) : rotation_vector(rot_displacement_q(j, qa, qb));
  for (int i = 0; i < e.nfree; ++i) th[i] = e.A[i][0] * d[0] + e.A[i][1] * d[1] + e.A[i][2] * d[2];
}
// translational/minimal.jl:61-65, rotational/minimal.jl:69-80 (attjac=false): (3-Nλ) x 7 in rows of a 3x7
static Mat<3, 7> minimal_coordinates_jacobian_configuration(bool parent, const JointS& j, int k, const V3& xa, const Quat& qa,
                                                            const V3& xb, const Quat& qb) {
  const Elem& e = j.el[k];
  Mat<3, 7> full;
  if (k == 0) {
    XQ xq = tra_displacement_jacobian(parent, j, xa, qa, xb, qb);
    full = hcat(xq.X, xq.Q);
  } else {
    Quat q = rot_displacement_q(j, qa, qb);
    M34 Q = drotation_vector_dq(vector(q)) * rot_displacement_jacobian_q4(parent, j, qa, qb);
    full = hcat(M33(), Q);
  }
  Mat<3, 7> out;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 7; ++c) out(i, c) = e.A[i][0] * full(0, c) + e.A[i][1] * full(1, c) + e.A[i][2] * full(2, c);
  return out;
}

// joints/joint.jl:9-12, joints/limits.jl:1-17
static EVec element_constraint(const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb,
                               const double* eta, double mu) {
  const Elem& e = j.el[k];
  EVec r;
  r.n = e.n;
  V3 d = displacement(j, k, xa, qa, xb, qb);
  int row = 0;
  if (e.nb > 0) {
    double th[3];
    minimal_coordinates(j, k, xa, qa, xb, qb, th);
    const double* s = eta;
    const double* g = eta + e.nb;
    for (int i = 0; i < e.nb; ++i) r.v[row++] = s[i] * g[i] - mu;
    for (int i = 0; i < e.nb2; ++i) r.v[row++] = s[i] - (e.hi[i] - th[i]);
    for (int i = 0; i < e.nb2; ++i) r.v[row++] = s[e.nb2 + i] - (th[i] - e.lo[i]);
  }
  for (int i = 0; i < e.nl; ++i) r.v[row++] = e.C[i][0] * d[0] + e.C[i][1] * d[1] + e.C[i][2] * d[2];
  return r;
}
// joints/joint.jl:14-19,45-53, joints/limits.jl:19-29  (N x 7)
static EJac7 element_constraint_jacobian_configuration(bool parent, const JointS& j, int k, const V3& xa, const Quat& qa,
                                                       const V3& xb, const Quat& qb) {
  const Elem& e = j.el[k];
  EJac7 r;
  r.n = e.n;
  int row = e.nb;  // ∇comp = 0
  if (e.nb > 0) {
    Mat<3, 7> mc = minimal_coordinates_jacobian_configuration(parent, j, k, xa, qa, xb, qb);
    for (int i = 0; i < e.nb2; ++i, ++row)
      for (int c = 0; c < 7; ++c) r.J(row, c) = mc(i, c);
    for (int i = 0; i < e.nb2; ++i, ++row)
      for (int c = 0; c < 7; ++c) r.J(row, c) = -mc(i, c);
  }
  XQ xq = displacement_jacobian(parent, j, k, xa, qa, xb, qb);
  Mat<3, 7> full = hcat(xq.X, xq.Q);
  for (int i = 0; i < e.nl; ++i, ++row)
    for (int c = 0; c < 7; ++c) r.J(row, c) = e.C[i][0] * full(0, c) + e.C[i][1] * full(1, c) + e.C[i][2] * full(2, c);
  return r;
}
// joints/impulses.jl:4-7: Diagonal([1,1,1,.5,.5,.5]) * [X Q*LVᵀ]ᵀ   (6 x 3)
static Mat<6, 3> impulse_transform(bool parent, const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb) {
  XQ xq = displacement_jacobian(parent, j, k, xa, qa, xb, qb);
  M33 Qa = xq.Q * LVtmat(parent ? qa : qb);
  Mat<6, 3> T;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      T(c, r) = xq.X(r, c);
      T(3 + c, r) = 0.5 * Qa(r, c);
    }
  return T;
}
// joints/joint.jl:87-93: projector (3 x N) = [0(Nb); -A; A; C]ᵀ  (or Cᵀ without limits)
static Mat<3, 12> impulse_projector(const Elem& e) {
  Mat<3, 12> P;
  int col = e.nb;
  if (e.nb > 0) {
    for (int i = 0; i < e.nb2; ++i, ++col)
      for (int r = 0; r < 3; ++r) P(r, col) = -e.A[i][r];
    for (int i = 0; i < e.nb2; ++i, ++col)
      for (int r = 0; r < 3; ++r) P(r, col) = e.A[i][r];
  }
  for (int i = 0; i < e.nl; ++i, ++col)
    for (int r = 0; r < 3; ++r) P(r, col) = e.C[i][r];
  return P;
}
// joints/joint.jl:67-85
static EMap element_impulse_map(bool parent, const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb) {
  EMap r;
  r.n = j.el[k].n;
  r.G = impulse_transform(parent, j, k, xa, qa, xb, qb) * impulse_projector(j.el[k]);
  return r;
}

// ------------------------------------------------------------------------------------------
// minimal velocities (finite difference of minimal coordinates) and their velocity Jacobians
// ------------------------------------------------------------------------------------------
// translational/minimal.jl:93-113, rotational/minimal.jl:103-118
static void minimal_velocities(const JointS& j, int k, const Cfg& a, const Cfg& b, double h, double* dv) {
  const Elem& e = j.el[k];
  Quat qa1 = next_orientation(a.q, -a.w, h), qb1 = next_orientation(b.q, -b.w, h);
  V3 d;
  if (k == 0) {
    V3 xa1 = next_position(a.x, -a.v, h), xb1 = next_position(b.x, -b.v, h);
    d = (tra_displacement(j, a.x, a.q, b.x, b.q) - tra_displacement(j, xa1, qa1, xb1, qb1)) / h;
  } else {
    Quat q = inv(j.qoff) * inv(a.q) * b.q;
    Quat q1 = inv(j.qoff) * inv(qa1) * qb1;
    d = rotation_vector(inv(q1) * q) / h;
  }
  for (int i = 0; i < e.nfree; ++i) dv[i] = e.A[i][0] * d[0] + e.A[i][1] * d[1] + e.A[i][2] * d[2];
}
// translational/minimal.jl:159-193, rotational/minimal.jl:151-174: (3-Nλ) x 6 in the rows of a 3x6
static Mat<3, 6> minimal_velocities_jacobian_velocity(bool parent, const JointS& j, int k, const Cfg& a, const Cfg& b, double h) {
  const Elem& e = j.el[k];
  Quat qa1 = next_orientation(a.q, -a.w, h), qb1 = next_orientation(b.q, -b.w, h);
  Mat<3, 6> full;
  if (k == 0) {
    V3 xa1 = next_position(a.x, -a.v, h), xb1 = next_position(b.x, -b.v, h);
    XQ xq = tra_displacement_jacobian(parent, j, xa1, qa1, xb1, qb1);
    M33 X1 = xq.X * (-h);
    M33 Q1 = xq.Q * (-rotational_integrator_jacobian_velocity(parent ? a.q : b.q, parent ? -a.w : -b.w, h));
    full = (-1.0 / h) * hcat(X1, Q1);
  } else {
    Quat q = inv(j.qoff) * inv(a.q) * b.q;
    Quat q1 = inv(j.qoff) * inv(qa1) * qb1;
    M34 drv = drotation_vector_dq(vector(inv(q1) * q));
    M33 Om;
    if (parent)
      Om = (1.0 / h) * (drv * Rmat(q) * Tmat() * Lmat(inv(j.qoff)) * Rmat(qb1) * Tmat() * (-rotational_integrator_jacobian_velocity(a.q, -a.w, h)));
    else
      Om = (1.0 / h) * (drv * Rmat(q) * Tmat() * Lmat(inv(j.qoff) * inv(qa1)) * (-rotational_integrator_jacobian_velocity(b.q, -b.w, h)));
    full = hcat(M33(), Om);
  }
  Mat<3, 6> out;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 6; ++c) out(i, c) = e.A[i][0] * full(0, c) + e.A[i][1] * full(1, c) + e.A[i][2] * full(2, c);
  return out;
}
// translational/minimal.jl:116-157, rotational/minimal.jl:120-149 (attjac'd): (3-Nλ) x 6
static Mat<3, 6> minimal_velocities_jacobian_configuration(bool parent, const JointS& j, int k, const Cfg& a, const Cfg& b, double h) {
  const Elem& e = j.el[k];
  Quat qa1 = next_orientation(a.q, -a.w, h), qb1 = next_orientation(b.q, -b.w, h);
  Mat<3, 6> full;
  const Quat& qrel = parent ? a.q : b.q;
  const V3& wrel = parent ? a.w : b.w;
  if (k == 0) {
    V3 xa1 = next_position(a.x, -a.v, h), xb1 = next_position(b.x, -b.v, h);
    XQ xq = tra_displacement_jacobian(parent, j, a.x, a.q, b.x, b.q);
    XQ xq1 = tra_displacement_jacobian(parent, j, xa1, qa1, xb1, qb1);
    M33 X1 = -xq1.X;
    M34 Q1 = xq1.Q * (-1.0 * rotational_integrator_jacobian_orientation_full(-wrel, h));
    M33 Qa = xq.Q * LVtmat(qrel);
    M33 Q1a = Q1 * LVtmat(qrel);
    full = (1.0 / h) * hcat(xq.X, Qa) + (1.0 / h) * hcat(X1, Q1a);
  } else {
    Quat q = inv(j.qoff) * inv(a.q) * b.q;
    Quat q1 = inv(j.qoff) * inv(qa1) * qb1;
    M34 drv = drotation_vector_dq(vector(inv(q1) * q));
    M34 Qm;
    if (parent) {
      Qm = (1.0 / h) * (drv * Rmat(q) * Tmat() * Rmat(qb1) * Lmat(inv(j.qoff)) * Tmat() * rotational_integrator_jacobian_orientation_full(-a.w, h));
      Qm += (1.0 / h) * (drv * Lmat(inv(q1)) * Rmat(b.q) * Lmat(inv(j.qoff)) * Tmat());
    } else {
      Qm = (1.0 / h) * (drv * Rmat(q) * Tmat() * Lmat(inv(j.qoff) * inv(qa1)) * rotational_integrator_jacobian_orientation_full(-b.w, h));
      Qm += (1.0 / h) * (drv * Lmat(inv(q1) * inv(j.qoff) * inv(a.q)));
    }
    full = hcat(M33(), Qm * LVtmat(qrel));
  }
  Mat<3, 6> out;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 6; ++c) out(i, c) = e.A[i][0] * full(0, c) + e.A[i][1] * full(1, c) + e.A[i][2] * full(2, c);
  return out;
}
static V3 At_times(const Elem& e, const double* v) {  // Aᵀ v
  V3 r;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 3; ++c) r[c] += e.A[i][c] * v[i];
  return r;
}
static M33 At_times_rows(const Elem& e, const Mat<3, 6>& m, int col0) {  // Aᵀ * m[:, col0:col0+3]
  M33 r;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 3; ++c)
      for (int d = 0; d < 3; ++d) r(c, d) += e.A[i][c] * m(i, col0 + d);
  return r;
}
static Mat<3, 6> At_times_full(const Elem& e, const Mat<3, 6>& m) {  // Aᵀ * m  (3x6)
  Mat<3, 6> r;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 3; ++c)
      for (int d = 0; d < 6; ++d) r(c, d) += e.A[i][c] * m(i, d);
  return r;
}
static Mat<3, 7> At_times_full7(const Elem& e, const Mat<3, 7>& m) {
  Mat<3, 7> r;
  for (int i = 0; i < e.nfree; ++i)
    for (int c = 0; c < 3; ++c)
      for (int d = 0; d < 7; ++d) r(c, d) += e.A[i][c] * m(i, d);
  return r;
}

// ------------------------------------------------------------------------------------------
// Springs (explicit, at x2,q2)
// ------------------------------------------------------------------------------------------
// translational/springs.jl:5-29, rotational/springs.jl:5-38
static V6 spring_impulses(bool parent, const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb, const Quat& qb, double h,
                          bool unitary = false) {
  const Elem& e = j.el[k];
  V6 out;
  if (e.nl == 3) return out;
  double k_s = unitary ? 1.0 : e.spring;
  double th[3], dist[3];
  minimal_coordinates(j, k, xa, qa, xb, qb, th);
  for (int i = 0; i < e.nfree; ++i) dist[i] = e.spring_offset[i] - th[i];
  if (k == 0) {
    V3 force = k_s * At_times(e, dist);
    out = h * (impulse_transform(parent, j, 0, xa, qa, xb, qb) * force);
  } else {
    V3 force = -k_s * At_times(e, dist);
    V3 o = parent ? vector_rotate(force, j.qoff) : vector_rotate(-force, inv(qb) * qa * j.qoff);
    for (int i = 0; i < 3; ++i) out[3 + i] = h * o[i];
  }
  return out;
}

// ------------------------------------------------------------------------------------------
// Dampers (implicit in v25, w25; configuration x2,q2)
// ------------------------------------------------------------------------------------------
// translational/dampers.jl:5-35, rotational/dampers.jl:4-27
static V6 damper_impulses(bool parent, const JointS& j, int k, const Cfg& a, const Cfg& b, double h, bool unitary = false) {
  const Elem& e = j.el[k];
  V6 out;
  if (e.nl == 3) return out;
  double c = unitary ? 1.0 : e.damper;
  double vel[3];
  if (k == 0) {
    minimal_velocities(j, 0, a, b, h, vel);
    V3 input = -c * At_times(e, vel);
    out = h * (impulse_transform(parent, j, 0, a.x, a.q, b.x, b.q) * input);
  } else {
    Cfg a0 = a, b0 = b;  // rotational damper_force passes zero positions / linear velocities
    a0.x = V3(); a0.v = V3(); b0.x = V3(); b0.v = V3();
    minimal_velocities(j, 1, a0, b0, h, vel);
    V3 force = parent ? c * At_times(e, vel) : -c * At_times(e, vel);
    force = parent ? vector_rotate(force, j.qoff) : vector_rotate(force, inv(b.q) * a.q * j.qoff);
    for (int i = 0; i < 3; ++i) out[3 + i] = h * force[i];
  }
  return out;
}
// translational/dampers.jl:57-69,100-123, rotational/dampers.jl:66-84
static M66 damper_jacobian_velocity(bool parent, bool jac_parent, const JointS& j, int k, const Cfg& a, const Cfg& b, double h) {
  const Elem& e = j.el[k];
  M66 out;
  if (e.nl == 3) return out;
  Mat<3, 6> dvel = minimal_velocities_jacobian_velocity(jac_parent, j, k, a, b, h);
  if (k == 0) {
    Mat<3, 6> dinput = (-e.damper) * At_times_full(e, dvel);
    out = h * (impulse_transform(parent, j, 0, a.x, a.q, b.x, b.q) * dinput);
  } else {
    Mat<3, 6> f = At_times_full(e, dvel);
    Mat<3, 6> VO = parent ? rotation_matrix(j.qoff) * (e.damper * f) : rotation_matrix(inv(b.q) * a.q * j.qoff) * ((-e.damper) * f);
    for (int r = 0; r < 3; ++r)
      for (int c2 = 0; c2 < 6; ++c2) out(3 + r, c2) = h * VO(r, c2);
  }
  return out;
}

// ------------------------------------------------------------------------------------------
// Derivatives of the impulse transform w.r.t. configuration (data Jacobians)
// ------------------------------------------------------------------------------------------
// translational/impulses.jl:9-45, rotational/impulses.jl:9-38:  ∂(impulse_transform * p)/∂(x,q)·attjac  (6x6)
static M66 impulse_transform_jacobian(bool parent, bool jac_parent, const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb,
                                      const Quat& qb, const V3& p) {
  M66 out;
  if (k == 0) {
    if (parent) {
      if (jac_parent) {
        M33 Xqa = -drotation_matrix_dq(qa, p) * LVtmat(qa);
        M33 Qxa = dskew_dp(p) * rotation_matrix(inv(qa));
        M33 Qqa = -dskew_dp(p) * drotation_matrix_inv_dq(qa, xb - xa + rotation_matrix(qb) * j.pb) * LVtmat(qa);
        set_block(out, 0, 3, Xqa); set_block(out, 3, 0, Qxa); set_block(out, 3, 3, Qqa);
      } else {
        M33 Qxb = -dskew_dp(p) * rotation_matrix(inv(qa));
        M33 Qqb = -dskew_dp(p) * rotation_matrix(inv(qa)) * drotation_matrix_dq(qb, j.pb) * LVtmat(qb);
        set_block(out, 3, 0, Qxb); set_block(out, 3, 3, Qqb);
      }
    } else {
      V3 cbpb_w = rotation_matrix(qb) * j.pb;
      if (jac_parent) {
        M33 Xqa = drotation_matrix_dq(qa, p) * LVtmat(qa);
        M33 Qqa = rotation_matrix(inv(qb)) * skew(cbpb_w) * drotation_matrix_dq(qa, p) * LVtmat(qa);
        set_block(out, 0, 3, Xqa); set_block(out, 3, 3, Qqa);
      } else {
        M34 Q = drotation_matrix_inv_dq(qb, skew(cbpb_w) * rotation_matrix(qa) * p);
        Q += rotation_matrix(inv(qb)) * dskew_dp(rotation_matrix(qa) * p) * drotation_matrix_dq(qb, j.pb);
        set_block(out, 3, 3, Q * LVtmat(qb));
      }
    }
  } else {
    M33 Q;
    if (parent) {
      if (jac_parent) Q = dVLtmat_dq(Tmat() * Rtmat(qb) * LVtmat(j.qoff) * p) * LVtmat(qa);
      else Q = VLtmat(qa) * Tmat() * dRtmat_dq(LVtmat(j.qoff) * p) * LVtmat(qb);
    } else {
      if (jac_parent) Q = VLtmat(qb) * dLmat_dq(LVtmat(j.qoff) * p) * LVtmat(qa);
      else Q = dVLtmat_dq(Lmat(qa) * LVtmat(j.qoff) * p) * LVtmat(qb);
    }
    set_block(out, 3, 3, 0.5 * Q);
  }
  return out;
}

// ------------------------------------------------------------------------------------------
// dense helpers
// ------------------------------------------------------------------------------------------
// in-place inverse by Gauss-Jordan with partial pivoting (the reference inverts <=~24x24 diagonal blocks
// with StaticArrays/LAPACK `inv`); returns false if singular
static bool invert_inplace(double* M, int n, int ld) {
  std::vector<double> a(n * 2 * n);
  for (int i = 0; i < n; ++i) {
    for (int jx = 0; jx < n; ++jx) a[i * 2 * n + jx] = M[i * ld + jx];
    for (int jx = 0; jx < n; ++jx) a[i * 2 * n + n + jx] = (i == jx) ? 1.0 : 0.0;
  }
  for (int c = 0; c < n; ++c) {
    int p = c;
    double best = std::fabs(a[c * 2 * n + c]);
    for (int r = c + 1; r < n; ++r)
      if (std::fabs(a[r * 2 * n + c]) > best) { best = std::fabs(a[r * 2 * n + c]); p = r; }
    if (!(best > 0.0)) return false;
    if (p != c)
      for (int jx = 0; jx < 2 * n; ++jx) std::swap(a[c * 2 * n + jx], a[p * 2 * n + jx]);
    double piv = 1.0 / a[c * 2 * n + c];
    for (int jx = 0; jx < 2 * n; ++jx) a[c * 2 * n + jx] *= piv;
    for (int r = 0; r < n; ++r) {
      if (r == c) continue;
      double f = a[r * 2 * n + c];
      if (f == 0.0) continue;
      for (int jx = 0; jx < 2 * n; ++jx) a[r * 2 * n + jx] -= f * a[c * 2 * n + jx];
    }
  }
  for (int i = 0; i < n; ++i)
    for (int jx = 0; jx < n; ++jx) M[i * ld + jx] = a[i * 2 * n + n + jx];
  return true;
}

// dense LU with partial pivoting: solves A X = B (A n x n row-major, B n x m row-major), in place on copies
static bool dense_solve(std::vector<double> A, int n, double* B, int m) {
  std::vector<int> perm(n);
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int c = 0; c < n; ++c) {
    int p = c;
    double best = std::fabs(A[c * n + c]);
    for (int r = c + 1; r < n; ++r)
      if (std::fabs(A[r * n + c]) > best) { best = std::fabs(A[r * n + c]); p = r; }
    if (!(best > 0.0)) return false;
    if (p != c) {
      for (int jx = 0; jx < n; ++jx) std::swap(A[c * n + jx], A[p * n + jx]);
      for (int jx = 0; jx < m; ++jx) std::swap(B[c * m + jx], B[p * m + jx]);
    }
    for (int r = c + 1; r < n; ++r) {
      double f = A[r * n + c] / A[c * n + c];
      if (f == 0.0) continue;
      A[r * n + c] = f;
      for (int jx = c + 1; jx < n; ++jx) A[r * n + jx] -= f * A[c * n + jx];
      for (int jx = 0; jx < m; ++jx) B[r * m + jx] -= f * B[c * m + jx];
    }
  }
  for (int r = n - 1; r >= 0; --r) {
    for (int jx = 0; jx < m; ++jx) {
      double s = B[r * m + jx];
      for (int c = r + 1; c < n; ++c) s -= A[r * n + c] * B[c * m + jx];
      B[r * m + jx] = s / A[r * n + r];
    }
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// The mechanism
// ------------------------------------------------------------------------------------------
struct Oracle {
  int Nb = 0, Ne = 0, Ni = 0, nres = 0, nu = 0;
  double h = 0.01, input_scaling = 0.01, mu = 0.0;
  V3 gravity;
  std::vector<BodyS> bodies;
  std::vector<JointS> joints;
  std::vector<ContactS> contacts;
  std::vector<int> body_off;  // solution offset of body b

  // linear system (dense storage, block structure known)
  std::vector<double> A, rhs, res_saved;
  std::vector<int> node_dim, node_off;               // nodes: joints | bodies | contacts
  std::vector<int> elim_order;                       // leaves -> root
  std::vector<std::vector<int>> elim_nbrs;           // later-eliminated neighbours (incl. symbolic fill)
  std::vector<std::pair<int, int>> pattern;          // structurally non-zero (node, node) blocks incl. fill
  bool tree_ok = true;
  int solver_mode = 0;  // 0 block LDU (reference-like), 1 dense partial-pivot LU
  uint32_t grad_flags = 0;  // DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN: the data Jacobian omits d(input impulse)/d(configuration)
  std::vector<double> F;  // factor storage (copy of A)

  // diagnostics of the last mehrotra call
  std::vector<double> trace;  // per iteration: rvio, bvio, alpha, mu

  Cfg cfg_current(int b, int idx) const {  // (x2, vsol[idx], q2, wsol[idx]); origin for b < 0
    Cfg c;
    if (b >= 0) { c.x = bodies[b].x2; c.v = bodies[b].vsol[idx]; c.q = bodies[b].q2; c.w = bodies[b].wsol[idx]; }
    return c;
  }
  Cfg cfg_next(int b) const {  // next_configuration_velocity (integrators/integrator.jl:19)
    Cfg c;
    if (b >= 0) {
      const BodyS& s = bodies[b];
      c.x = next_position(s.x2, s.vsol[1], h);
      c.q = next_orientation(s.q2, s.wsol[1], h);
      c.v = s.vsol[1];
      c.w = s.wsol[1];
    }
    return c;
  }

  // ---------------------------------------------------------------- construction
  explicit Oracle(const DojoMechanismDesc& d) {
    Nb = d.num_bodies; Ne = d.num_joints; Ni = d.num_contacts;
    h = d.timestep; input_scaling = d.input_scaling; gravity = vec3(d.gravity);
    bodies.resize(Nb);
    for (int b = 0; b < Nb; ++b) { bodies[b].mass = d.bodies[b].mass; bodies[b].J = mat33(d.bodies[b].inertia); }
    joints.resize(Ne);
    int off = 0, uoff = 0;
    for (int ji = 0; ji < Ne; ++ji) {
      const DojoJointDesc& jd = d.joints[ji];
      JointS& j = joints[ji];
      j.parent = jd.parent_body; j.child = jd.child_body;
      j.pa = vec3(jd.vertex_parent); j.pb = vec3(jd.vertex_child);
      j.qoff = Quat(jd.orientation_offset[0], jd.orientation_offset[1], jd.orientation_offset[2], jd.orientation_offset[3]);
      const DojoJointElementDesc* eds[2] = {&jd.tra, &jd.rot};
      for (int k = 0; k < 2; ++k) {
        Elem& e = j.el[k];
        const DojoJointElementDesc& ed = *eds[k];
        e.kind = k; e.nl = ed.nlambda; e.nb2 = ed.nlimits; e.nb = 2 * e.nb2; e.n = e.nl + 2 * e.nb; e.nfree = 3 - e.nl;
        const double* V1 = ed.axis_mask; const double* V2 = ed.axis_mask + 3; const double* V3_ = ed.axis_mask + 6;
        std::memset(e.C, 0, sizeof(e.C)); std::memset(e.A, 0, sizeof(e.A));
        auto setrow = [](double (*M)[3], int r, const double* v) { M[r][0] = v[0]; M[r][1] = v[1]; M[r][2] = v[2]; };
        const double I3[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
        switch (e.nl) {  // joints/joint.jl:56-64
          case 0: for (int r = 0; r < 3; ++r) setrow(e.A, r, I3[r]); break;
          case 1: setrow(e.C, 0, V3_); setrow(e.A, 0, V1); setrow(e.A, 1, V2); break;
          case 2: setrow(e.C, 0, V1); setrow(e.C, 1, V2); setrow(e.A, 0, V3_); break;
          case 3: for (int r = 0; r < 3; ++r) setrow(e.C, r, I3[r]); break;
        }
        e.spring = ed.spring; e.damper = ed.damper;
        for (int i = 0; i < 3; ++i) { e.spring_offset[i] = ed.spring_offset[i]; e.lo[i] = ed.limit_lo[i]; e.hi[i] = ed.limit_hi[i]; }
        j.spring = j.spring || (e.spring != 0);
        j.damper = j.damper || (e.damper != 0);
      }
      j.eoff[0] = 0; j.eoff[1] = j.el[0].n;
      j.n = j.el[0].n + j.el[1].n;
      j.nu = j.el[0].nfree + j.el[1].nfree;
      j.sol_off = off; off += j.n;
      j.u_off = uoff; uoff += j.nu;
      j.imp[0].assign(j.n, 0.0); j.imp[1].assign(j.n, 0.0);
    }
    nu = uoff;
    body_off.resize(Nb);
    for (int b = 0; b < Nb; ++b) { body_off[b] = off; off += 6; }
    contacts.resize(Ni);
    for (int c = 0; c < Ni; ++c) {
      const DojoContactDesc& cd = d.contacts[c];
      ContactS& ct = contacts[c];
      ct.body = cd.parent_body; ct.mu_f = cd.friction_coefficient; ct.radius = cd.radius;
      for (int i = 0; i < 6; ++i) ct.t.a[i] = cd.tangent[i];
      for (int i = 0; i < 3; ++i) ct.nrm.a[i] = cd.normal[i];
      ct.o = vec3(cd.origin); ct.off = vec3(cd.offset);
      ct.type = cd.type; ct.nh = (cd.type == 0 ? 1 : (cd.type == 1 ? 6 : 4));
      ct.sol_off = off; off += 2 * ct.nh;
    }
    nres = off;
    A.assign((size_t)nres * nres, 0.0); rhs.assign(nres, 0.0); res_saved.assign(nres, 0.0);
    build_elimination();
  }

  // nodes: joints 0..Ne-1, bodies Ne..Ne+Nb-1, contacts after (mechanism/id.jl:5-13)
  void build_elimination() {
    int N = Ne + Nb + Ni;
    node_dim.resize(N); node_off.resize(N);
    for (int j = 0; j < Ne; ++j) { node_dim[j] = joints[j].n; node_off[j] = joints[j].sol_off; }
    for (int b = 0; b < Nb; ++b) { node_dim[Ne + b] = 6; node_off[Ne + b] = body_off[b]; }
    for (int c = 0; c < Ni; ++c) { node_dim[Ne + Nb + c] = 2 * contacts[c].nh; node_off[Ne + Nb + c] = contacts[c].sol_off; }
    // adjacency (mechanism/system.jl:15-51): joint-parent, joint-child, parent-child bodies, contact-body
    std::vector<std::vector<char>> adj(N, std::vector<char>(N, 0));
    auto link = [&](int a, int b) { adj[a][b] = adj[b][a] = 1; };
    std::vector<int> parent_joint(Nb, -1);
    for (int j = 0; j < Ne; ++j) {
      const JointS& jt = joints[j];
      link(j, Ne + jt.child);
      if (jt.parent >= 0) { link(j, Ne + jt.parent); link(Ne + jt.parent, Ne + jt.child); }
      if (parent_joint[jt.child] >= 0) tree_ok = false;  // loop-closure joint
      else parent_joint[jt.child] = j;
    }
    for (int b = 0; b < Nb; ++b) if (parent_joint[b] < 0) tree_ok = false;
    for (int c = 0; c < Ni; ++c) link(Ne + Nb + c, Ne + contacts[c].body);
    // elimination order: post-order over the body tree: children subtrees, then the body's contacts,
    // the body, and its parent joint ("contacts into bodies, bodies into their parent joint, joints into
    // the parent body", SURVEY.md Appendix C)
    elim_order.clear();
    if (tree_ok) {
      std::vector<char> done(Nb, 0);
      struct Rec { Oracle* o; std::vector<int>& pj; std::vector<char>& done;
        void visit(int b) {
          done[b] = 1;
          for (int j = 0; j < o->Ne; ++j) if (o->joints[j].parent == b && !done[o->joints[j].child]) visit(o->joints[j].child);
          for (int c = 0; c < o->Ni; ++c) if (o->contacts[c].body == b) o->elim_order.push_back(o->Ne + o->Nb + c);
          o->elim_order.push_back(o->Ne + b);
          o->elim_order.push_back(pj[b]);
        } } rec{this, parent_joint, done};
      for (int j = 0; j < Ne; ++j) if (joints[j].parent < 0 && !done[joints[j].child]) rec.visit(joints[j].child);
      if ((int)elim_order.size() != N) tree_ok = false;
    }
    if (!tree_ok) { elim_order.clear(); for (int i = 0; i < N; ++i) elim_order.push_back(i); solver_mode = 1; }
    // symbolic elimination (fill-in)
    std::vector<int> pos(N);
    for (int i = 0; i < N; ++i) pos[elim_order[i]] = i;
    elim_nbrs.assign(N, {});
    for (int step = 0; step < N; ++step) {
      int k = elim_order[step];
      std::vector<int> nb;
      for (int i = 0; i < N; ++i) if (adj[k][i] && pos[i] > step) nb.push_back(i);
      std::sort(nb.begin(), nb.end(), [&](int a, int b) { return pos[a] < pos[b]; });
      for (int a : nb) for (int b : nb) if (a != b) adj[a][b] = 1;
      elim_nbrs[k] = nb;
    }
    pattern.clear();
    for (int a = 0; a < N; ++a) for (int b = 0; b < N; ++b) if (a == b || adj[a][b]) pattern.push_back({a, b});
  }

  // ---------------------------------------------------------------- state in / out
  // mechanism/set.jl:10-26 (set_maximal_state!), bodies/set.jl:1-20
  // ----------------------------------------------------------------------------------------
  // minimal <-> maximal coordinate maps (SURVEY.md 8 f1): mechanism/state.jl:9-22 (minimal_to_maximal), :44-66
  // (maximal_to_minimal), joints/minimal.jl:148-203 (set_minimal_coordinates_velocities!).  Minimal state per joint, in
  // joint order: [c_tra; c_rot; v_tra; v_rot]  (2 * input_dimension(joint) entries).
  // ----------------------------------------------------------------------------------------
  std::vector<int> root_to_leaves_joints() const {  // mechanism.root_to_leaves restricted to joints: parents before children
    std::vector<int> order;
    std::vector<char> placed(Nb, 0);
    bool progress = true;
    while ((int)order.size() < Ne && progress) {
      progress = false;
      for (int j = 0; j < Ne; ++j) {
        const JointS& jt = joints[j];
        bool done = false;
        for (int k : order) done = done || (k == j);
        if (done) continue;
        if (jt.parent < 0 || placed[jt.parent]) { order.push_back(j); placed[jt.child] = 1; progress = true; }
      }
    }
    return order;
  }
  static Quat axis_angle_to_quaternion(const V3& x) {  // orientation/axis_angle.jl:1-11
    double th = std::sqrt(dot(x, x));
    if (th > 0.0) { double s = std::sin(0.5 * th) / th; return Quat(std::cos(0.5 * th), s * x[0], s * x[1], s * x[2]); }
    return Quat(1.0, 0.0, 0.0, 0.0);
  }
  static V3 angular_velocity(const Quat& q1, const Quat& q2, double h) {  // integrators/integrator.jl:22-24
    return (VLtmat(q1) * vector(q2)) * (2.0 / h);
  }
  void minimal_to_maximal(const double* xmin, double* z) const {
    std::vector<Cfg> st(Nb);
    for (int j : root_to_leaves_joints()) {
      const JointS& jt = joints[j];
      const int nt = jt.el[0].nfree, nr = jt.el[1].nfree, nuj = nt + nr;
      const double* xm = xmin + 2 * jt.u_off;
      Cfg a;
      if (jt.parent >= 0) a = st[jt.parent];
      else { a.x = V3(); a.v = V3(); a.w = V3(); a.q = Quat(1.0, 0.0, 0.0, 0.0); }
      V3 dx, dth, dv, dw;  // A' * coordinates
      for (int i = 0; i < nt; ++i) for (int c = 0; c < 3; ++c) { dx[c] += jt.el[0].A[i][c] * xm[i]; dv[c] += jt.el[0].A[i][c] * xm[nuj + i]; }
      for (int i = 0; i < nr; ++i) for (int c = 0; c < 3; ++c) { dth[c] += jt.el[1].A[i][c] * xm[nt + i]; dw[c] += jt.el[1].A[i][c] * xm[nuj + nt + i]; }
      // positions
      Quat dq = axis_angle_to_quaternion(dth);
      Quat qb = a.q * jt.qoff * dq;
      V3 xb = a.x + vector_rotate(jt.pa + dx, a.q) - vector_rotate(jt.pb, qb);
      // previous configuration
      V3 xa1 = next_position(a.x, -a.v, h);
      Quat qa1 = next_orientation(a.q, -a.w, h);
      // finite-difference configuration
      V3 dx1 = dx - dv * h;
      Quat dq1 = dq * inv(axis_angle_to_quaternion(dw * h));
      Quat qb1 = qa1 * jt.qoff * dq1;
      V3 xb1 = xa1 + vector_rotate(jt.pa + dx1, qa1) - vector_rotate(jt.pb, qb1);
      Cfg b;
      b.x = xb; b.q = qb;
      b.v = (xb - xb1) / h;
      b.w = angular_velocity(qb1, qb, h);
      st[jt.child] = b;
    }
    for (int b = 0; b < Nb; ++b) {
      double* zb = z + 13 * b;
      for (int i = 0; i < 3; ++i) { zb[i] = st[b].x[i]; zb[3 + i] = st[b].v[i]; zb[10 + i] = st[b].w[i]; }
      zb[6] = st[b].q.s; zb[7] = st[b].q.v1; zb[8] = st[b].q.v2; zb[9] = st[b].q.v3;
    }
  }
  void maximal_to_minimal(const double* z, double* xmin) const {
    auto unpack = [&](int b) {
      Cfg c;
      if (b < 0) { c.x = V3(); c.v = V3(); c.w = V3(); c.q = Quat(1.0, 0.0, 0.0, 0.0); return c; }
      const double* zb = z + 13 * b;
      for (int i = 0; i < 3; ++i) { c.x[i] = zb[i]; c.v[i] = zb[3 + i]; c.w[i] = zb[10 + i]; }
      c.q = Quat(zb[6], zb[7], zb[8], zb[9]);
      return c;
    };
    for (int j = 0; j < Ne; ++j) {
      const JointS& jt = joints[j];
      const int nt = jt.el[0].nfree, nr = jt.el[1].nfree, nuj = nt + nr;
      double* xm = xmin + 2 * jt.u_off;
      Cfg a = unpack(jt.parent), b = unpack(jt.child);
      minimal_coordinates(jt, 0, a.x, a.q, b.x, b.q, xm);
      minimal_coordinates(jt, 1, a.x, a.q, b.x, b.q, xm + nt);
      minimal_velocities(jt, 0, a, b, h, xm + nuj);
      minimal_velocities(jt, 1, a, b, h, xm + nuj + nt);
    }
  }

  // ---------------------------------------------------------------- Jacobians of the coordinate maps (SURVEY.md 8 f1)
  static M43 daxis_angle_to_quaternion_dx(const V3& x) {  // orientation/axis_angle.jl:13-40
    M43 r;
    double th = std::sqrt(dot(x, x));
    if (th > 0.0) {
      double s = std::sin(0.5 * th), c = std::cos(0.5 * th);
      for (int k = 0; k < 3; ++k) r(0, k) = -0.5 * s * x[k] / th;
      for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k)
          r(1 + i, k) = 0.5 * c * x[k] / th * (x[i] / th) + (i == k ? s / th : 0.0) - s * x[i] / (th * th) * x[k] / th;
    } else {
      for (int i = 0; i < 3; ++i) r(1 + i, i) = 0.5;
    }
    return r;
  }
  static M34 dangular_velocity_dq1(const Quat& q1, const Quat& q2, double h) { return (2.0 / h) * (Vmat() * Rmat(q2) * Tmat()); }  // integrator.jl:26-28
  static M34 dangular_velocity_dq2(const Quat& q1, const Quat& q2, double h) { return (2.0 / h) * (Vmat() * Ltmat(q1)); }         // :30-32
  static Cfg unpack_cfg(const double* z, int b) {  // mechanism/state.jl:68-75; the origin: bodies/origin.jl
    Cfg c;
    if (b < 0) { c.x = V3(); c.v = V3(); c.w = V3(); c.q = Quat(1.0, 0.0, 0.0, 0.0); return c; }
    const double* zb = z + 13 * b;
    for (int i = 0; i < 3; ++i) { c.x[i] = zb[i]; c.v[i] = zb[3 + i]; c.w[i] = zb[10 + i]; }
    c.q = Quat(zb[6], zb[7], zb[8], zb[9]);
    return c;
  }
  static Mat<3, 3> nullspace_t(const Elem& e) {  // zerodimstaticadjoint(nullspace_mask(joint)): 3 x nfree, unused columns zero
    Mat<3, 3> A;
    for (int i = 0; i < e.nfree; ++i) for (int c = 0; c < 3; ++c) A(c, i) = e.A[i][c];
    return A;
  }

  // maximal_to_minimal_jacobian, gradients/state.jl:9-56.  J is (2 nu) x (12 Nb), COLUMN-major; columns per body
  // [x, v, phi, w] (attitude-reduced), rows per joint [c_tra; c_rot; v_tra; v_rot].
  void maximal_to_minimal_jacobian(const double* z, double* J) const {
    const int nr_ = 2 * nu, nc_ = 12 * Nb;
    std::fill(J, J + (size_t)nr_ * nc_, 0.0);
    auto at = [&](int r, int c) -> double& { return J[(size_t)c * nr_ + r]; };
    for (int j = 0; j < Ne; ++j) {
      const JointS& jt = joints[j];
      const int nuj = jt.el[0].nfree + jt.el[1].nfree;
      int c_shift = 0, v_shift = nuj;
      const int row0 = 2 * jt.u_off;
      const Cfg a = unpack_cfg(z, jt.parent), b = unpack_cfg(z, jt.child);
      for (int k = 0; k < 2; ++k) {
        const int ne = jt.el[k].nfree;
        for (int side = 0; side < 2; ++side) {
          const bool parent = (side == 0);
          if (parent && jt.parent < 0) continue;
          const int body = parent ? jt.parent : jt.child;
          const Quat& qrel = parent ? a.q : b.q;
          Mat<3, 7> cj7 = minimal_coordinates_jacobian_configuration(parent, jt, k, a.x, a.q, b.x, b.q);
          M33 cX = block<3, 3>(cj7, 0, 0);
          M33 cQ = block<3, 4>(cj7, 0, 3) * LVtmat(qrel);  // attjac = true (joint.jl:149-161, rotational/minimal.jl:76)
          Mat<3, 6> vc = minimal_velocities_jacobian_configuration(parent, jt, k, a, b, h);
          Mat<3, 6> vv = minimal_velocities_jacobian_velocity(parent, jt, k, a, b, h);
          for (int i = 0; i < ne; ++i)
            for (int c = 0; c < 3; ++c) {
              at(row0 + c_shift + i, 12 * body + c) = cX(i, c);        // x
              at(row0 + c_shift + i, 12 * body + 6 + c) = cQ(i, c);    // phi
              at(row0 + v_shift + i, 12 * body + c) = vc(i, c);        // x
              at(row0 + v_shift + i, 12 * body + 6 + c) = vc(i, 3 + c);
              at(row0 + v_shift + i, 12 * body + 3 + c) = vv(i, c);    // v
              at(row0 + v_shift + i, 12 * body + 9 + c) = vv(i, 3 + c);
            }
        }
        c_shift += ne;
        v_shift += ne;
      }
    }
  }

  // joints/minimal.jl:206-283 (parent: 13 x 13) and :314-383 (minimal: 13 x 2nu_j in a 13 x 12), rows [xb; vb; qb; wb]
  struct MinJac { Mat<13, 13> P; Mat<13, 12> M; };
  MinJac minimal_coordinates_velocities_jacobians(const JointS& jt, const Cfg& a, const double* xm) const {
    const int nt = jt.el[0].nfree, nr = jt.el[1].nfree, nuj = nt + nr;
    const Mat<3, 3> Atra = nullspace_t(jt.el[0]), Arot = nullspace_t(jt.el[1]);
    V3 dx, dth, dv, dw;
    for (int i = 0; i < nt; ++i) for (int c = 0; c < 3; ++c) { dx[c] += Atra(c, i) * xm[i]; dv[c] += Atra(c, i) * xm[nuj + i]; }
    for (int i = 0; i < nr; ++i) for (int c = 0; c < 3; ++c) { dth[c] += Arot(c, i) * xm[nt + i]; dw[c] += Arot(c, i) * xm[nuj + nt + i]; }
    const Quat& qoff = jt.qoff;
    // positions
    Quat dq = axis_angle_to_quaternion(dth);
    Quat qb = a.q * qoff * dq;
    // step backward in time
    Quat qa1 = next_orientation(a.q, -a.w, h);
    V3 dx1 = dx - dv * h;
    Quat dwq = axis_angle_to_quaternion(dw * h);
    Quat dq1 = dq * inv(dwq);
    Quat qb1 = qa1 * qoff * dq1;
    M44 RIO = rotational_integrator_jacobian_orientation_full(-a.w, h);
    M43 RIV = rotational_integrator_jacobian_velocity(a.q, -a.w, h);
    MinJac out;
    {  // parent, :237-276
      Mat<13, 13>& P = out.P;
      M34 dxb_dqa = dvector_rotate_dq(jt.pa + dx, a.q) - dvector_rotate_dq(jt.pb, qb) * Rmat(qoff * dq);
      M44 dqb_dqa = Rmat(qoff * dq);
      M34 dvb_dqa = (1.0 / h) * dvector_rotate_dq(jt.pa + dx, a.q);
      dvb_dqa -= (1.0 / h) * (dvector_rotate_dq(jt.pb, qb) * Rmat(qoff * dq));
      dvb_dqa += (-1.0 / h) * (dvector_rotate_dq(jt.pa + dx1, qa1) * RIO);
      dvb_dqa += (1.0 / h) * (dvector_rotate_dq(jt.pb, qb1) * Rmat(qoff * dq1) * RIO);
      M33 dvb_dwa = (1.0 / h) * (dvector_rotate_dq(jt.pa + dx1, qa1) * RIV);
      dvb_dwa += (-1.0 / h) * (dvector_rotate_dq(jt.pb, qb1) * Rmat(qoff * dq1) * RIV);
      M34 dwb_dqa = dangular_velocity_dq1(qb1, qb, h) * Rmat(qoff * dq1) * RIO;
      dwb_dqa += dangular_velocity_dq2(qb1, qb, h) * Rmat(qoff * dq);
      M33 dwb_dwa = -1.0 * (dangular_velocity_dq1(qb1, qb, h) * Rmat(qoff * dq1) * RIV);
      for (int i = 0; i < 3; ++i) { P(i, i) = 1.0; P(3 + i, 3 + i) = 1.0; }
      set_block(P, 0, 6, dxb_dqa);
      set_block(P, 3, 6, dvb_dqa);
      set_block(P, 3, 10, dvb_dwa);
      set_block(P, 6, 6, dqb_dqa);
      set_block(P, 10, 6, dwb_dqa);
      set_block(P, 10, 10, dwb_dwa);
    }
    {  // minimal, :346-376
      Mat<13, 12>& M = out.M;
      M33 Ra = rotation_matrix(a.q), Ra1 = rotation_matrix(qa1);
      M43 dth_q = daxis_angle_to_quaternion_dx(dth) * Arot;                 // d(dq)/d(theta)  (4 x nr)
      M43 dqb_dth = Lmat(a.q * qoff) * dth_q;
      M43 dqb1_dth = Rmat(inv(dwq)) * Lmat(qa1 * qoff) * dth_q;
      M43 dqb1_dw = Lmat(qa1 * qoff * dq) * Tmat() * daxis_angle_to_quaternion_dx(dw * h) * Arot;  // per unit (dw h)
      M33 dxb_dx = Ra * Atra;
      M33 dxb_dth = -1.0 * (dvector_rotate_dq(jt.pb, qb) * dqb_dth);
      M33 dvb_dx = (1.0 / h) * (Ra * Atra) + (-1.0 / h) * (Ra1 * Atra);
      M33 dvb_dth = (-1.0 / h) * (dvector_rotate_dq(jt.pb, qb) * dqb_dth) + (1.0 / h) * (dvector_rotate_dq(jt.pb, qb1) * dqb1_dth);
      M33 dvb_dv = Ra1 * Atra;
      M33 dvb_dw = dvector_rotate_dq(jt.pb, qb1) * dqb1_dw;
      M33 dwb_dth = dangular_velocity_dq1(qb1, qb, h) * dqb1_dth + dangular_velocity_dq2(qb1, qb, h) * dqb_dth;
      M33 dwb_dw = h * (dangular_velocity_dq1(qb1, qb, h) * dqb1_dw);
      auto put = [&](int r0, int rows, int c0, int cols, auto& blk) {
        for (int r = 0; r < rows; ++r) for (int c = 0; c < cols; ++c) M(r0 + r, c0 + c) = blk(r, c);
      };
      put(0, 3, 0, nt, dxb_dx);          put(0, 3, nt, nr, dxb_dth);
      put(3, 3, 0, nt, dvb_dx);          put(3, 3, nt, nr, dvb_dth);  put(3, 3, nuj, nt, dvb_dv);  put(3, 3, nuj + nt, nr, dvb_dw);
      put(6, 4, nt, nr, dqb_dth);
      put(10, 3, nt, nr, dwb_dth);       put(10, 3, nuj + nt, nr, dwb_dw);
    }
    return out;
  }

  // minimal_to_maximal_jacobian, gradients/state.jl:136-179, evaluated at the maximal state z (the reference reads the
  // mechanism's stored state; its argument x is unused).  J is (12 Nb) x (2 nu), COLUMN-major.
  // body_order_literal: chain the partials in mechanism.bodies order exactly like :170-178 (a child listed before its
  // parent then misses the parent's columns -- the reference's own check is disabled for such models, test/minimal.jl:527,
  // :560); otherwise root -> leaves, the derivative of minimal_to_maximal.
  void minimal_to_maximal_jacobian(const double* z, double* J, bool body_order_literal) const {
    const int nr_ = 12 * Nb, nc_ = 2 * nu;
    std::fill(J, J + (size_t)nr_ * nc_, 0.0);
    auto at = [&](int r, int c) -> double& { return J[(size_t)c * nr_ + r]; };
    std::vector<double> xmin(2 * nu + 1);
    maximal_to_minimal(z, xmin.data());  // minimal_coordinates_velocities(joint, pnode, cnode), joints/minimal.jl:291,390
    std::vector<int> pj(Nb, -1);
    for (int j = 0; j < Ne; ++j) pj[joints[j].child] = j;
    std::vector<int> order;
    if (body_order_literal) for (int b = 0; b < Nb; ++b) order.push_back(b);
    else for (int j : root_to_leaves_joints()) order.push_back(joints[j].child);
    for (int b : order) {
      if (pj[b] < 0) continue;
      const JointS& jt = joints[pj[b]];
      const int nuj = jt.el[0].nfree + jt.el[1].nfree;
      const Cfg a = unpack_cfg(z, jt.parent), cb = unpack_cfg(z, b);
      MinJac mj = minimal_coordinates_velocities_jacobians(jt, a, xmin.data() + 2 * jt.u_off);
      // attitude reduction: cat(I6, LVᵀ(qb)', I3) * J  and  J * cat(I6, LVᵀ(qa), I3)   (joints/minimal.jl:308-310, 398)
      Mat<12, 13> Gb;
      for (int i = 0; i < 6; ++i) Gb(i, i) = 1.0;
      set_block(Gb, 6, 6, tr(LVtmat(cb.q)));
      for (int i = 0; i < 3; ++i) Gb(9 + i, 10 + i) = 1.0;
      Mat<12, 12> Pm = Gb * mj.M;
      if (nuj > 0)
        for (int r = 0; r < 12; ++r) for (int c = 0; c < 2 * nuj; ++c) at(12 * b + r, 2 * jt.u_off + c) += Pm(r, c);
      if (jt.parent < 0) continue;
      Mat<13, 12> Ga;
      for (int i = 0; i < 6; ++i) Ga(i, i) = 1.0;
      set_block(Ga, 6, 6, LVtmat(a.q));
      for (int i = 0; i < 3; ++i) Ga(10 + i, 9 + i) = 1.0;
      Mat<12, 12> Pp = Gb * mj.P * Ga;
      for (int c = 0; c < nc_; ++c)
        for (int r = 0; r < 12; ++r) {
          double acc = 0;
          for (int k = 0; k < 12; ++k) acc += Pp(r, k) * at(12 * jt.parent + k, c);
          at(12 * b + r, c) += acc;
        }
    }
  }

  void set_maximal_state(const double* z) {
    for (int b = 0; b < Nb; ++b) {
      BodyS& s = bodies[b];
      const double* p = z + 13 * b;
      s.x2 = vec3(p); s.v15 = vec3(p + 3); s.q2 = Quat(p[6], p[7], p[8], p[9]); s.w15 = vec3(p + 10);
      s.x1 = next_position(s.x2, -s.v15, h);
      s.q1 = next_orientation(s.q2, -s.w15, h);
      s.JF2 = V3(); s.Jt2 = V3();
      s.vsol[0] = s.vsol[1] = s.v15;
      s.wsol[0] = s.wsol[1] = s.w15;
    }
  }
  // update_state! (bodies/set.jl:22-36)
  void update_state() {
    for (BodyS& s : bodies) {
      s.x1 = s.x2; s.q1 = s.q2;
      s.v15 = s.vsol[1]; s.w15 = s.wsol[1];
      s.x2 = next_position(s.x2, s.vsol[1], h);
      s.q2 = next_orientation(s.q2, s.wsol[1], h);
      s.JF2 = V3(); s.Jt2 = V3();
    }
  }
  void set_external(const double* f) {
    for (int b = 0; b < Nb; ++b) {
      bodies[b].Fext = f ? vec3(f + 6 * b) : V3();
      bodies[b].text = f ? vec3(f + 6 * b + 3) : V3();
    }
  }
  // mechanism/set.jl:40-53, joints/joint.jl:96-99, translational/input.jl:5-27, rotational/input.jl:5-17
  void set_input(const double* u) {
    for (JointS& j : joints) {
      const double* uj = u + j.u_off;
      j.el[0].input = At_times(j.el[0], uj);
      j.el[1].input = At_times(j.el[1], uj + j.el[0].nfree);
    }
    for (JointS& j : joints) {
      Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
      {  // translational
        V3 input = j.el[0].input * input_scaling;
        j.applied[0] = input;
        Mat<6, 3> Ta = impulse_transform(true, j, 0, a.x, a.q, b.x, b.q);
        Mat<6, 3> Tb = impulse_transform(false, j, 0, a.x, a.q, b.x, b.q);
        V6 ia = Ta * input, ib = Tb * input;
        if (j.parent >= 0) for (int i = 0; i < 3; ++i) { bodies[j.parent].JF2[i] += ia[i]; bodies[j.parent].Jt2[i] += ia[3 + i] / 2; }
        for (int i = 0; i < 3; ++i) { bodies[j.child].JF2[i] += ib[i]; bodies[j.child].Jt2[i] += ib[3 + i] / 2; }
        j.el[0].input = V3();
      }
      {  // rotational
        V3 tau = j.el[1].input * input_scaling;
        j.applied[1] = tau;
        if (j.parent >= 0) bodies[j.parent].Jt2 += vector_rotate(-tau, j.qoff);
        bodies[j.child].Jt2 += vector_rotate(tau, inv(b.q) * a.q * j.qoff);
        j.el[1].input = V3();
      }
    }
  }
  // joints/input.jl control Jacobians (translational/input.jl:33-44, rotational/input.jl:23-39) -> 6 x nu_j
  Mat<6, 6> input_jacobian_control(const JointS& j, bool parent) const {
    Mat<6, 6> out;
    Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
    Mat<6, 3> Ta = impulse_transform(parent, j, 0, a.x, a.q, b.x, b.q);
    Mat<6, 3> Bt;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) { Bt(r, c) = Ta(r, c) * input_scaling; Bt(3 + r, c) = 0.5 * Ta(3 + r, c) * input_scaling; }
    Mat<6, 3> Br;
    M33 R = parent ? -rotation_matrix(j.qoff) : rotation_matrix(inv(b.q) * a.q * j.qoff);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) Br(3 + r, c) = R(r, c) * input_scaling;
    int col = 0;
    for (int i = 0; i < j.el[0].nfree; ++i, ++col)
      for (int r = 0; r < 6; ++r) out(r, col) = Bt(r, 0) * j.el[0].A[i][0] + Bt(r, 1) * j.el[0].A[i][1] + Bt(r, 2) * j.el[0].A[i][2];
    for (int i = 0; i < j.el[1].nfree; ++i, ++col)
      for (int r = 0; r < 6; ++r) out(r, col) = Br(r, 0) * j.el[1].A[i][0] + Br(r, 1) * j.el[1].A[i][1] + Br(r, 2) * j.el[1].A[i][2];
    return out;
  }

  // solution vector: joints | bodies [v25; w25] | contacts [s; γ]   (gradients/finite_difference.jl:1-18)
  void get_solution(double* sol, int idx = 1) const {
    for (const JointS& j : joints) for (int i = 0; i < j.n; ++i) sol[j.sol_off + i] = j.imp[idx][i];
    for (int b = 0; b < Nb; ++b) for (int i = 0; i < 3; ++i) { sol[body_off[b] + i] = bodies[b].vsol[idx][i]; sol[body_off[b] + 3 + i] = bodies[b].wsol[idx][i]; }
    for (const ContactS& c : contacts) for (int i = 0; i < c.nh; ++i) { sol[c.sol_off + i] = c.s[idx][i]; sol[c.sol_off + c.nh + i] = c.gam[idx][i]; }
  }
  void set_solution(const double* sol) {
    for (JointS& j : joints) for (int i = 0; i < j.n; ++i) j.imp[0][i] = j.imp[1][i] = sol[j.sol_off + i];
    for (int b = 0; b < Nb; ++b) for (int i = 0; i < 3; ++i) {
      bodies[b].vsol[0][i] = bodies[b].vsol[1][i] = sol[body_off[b] + i];
      bodies[b].wsol[0][i] = bodies[b].wsol[1][i] = sol[body_off[b] + 3 + i];
    }
    for (ContactS& c : contacts) for (int i = 0; i < c.nh; ++i) { c.s[0][i] = c.s[1][i] = sol[c.sol_off + i]; c.gam[0][i] = c.gam[1][i] = sol[c.sol_off + c.nh + i]; }
  }

  // ---------------------------------------------------------------- contacts
  // sphere_halfspace.jl:34-36 / :55-62, velocity.jl:2-38
  V3 contact_point(const ContactS& c, const Cfg& p) const { return p.x + vector_rotate(c.o, p.q) - c.off - tr(c.nrm) * c.radius; }
  // contacts/nonlinear.jl:50-76: [d - s1; μγ1 - γ2; vt - s(3:4)]
  // contacts/impact.jl:41-56:    [d - s1]
  // contacts/linear.jl:72-104:   [d - sγ; μ γ - Σβ - sψ; P vt + ψ 1 - sβ],  γ-vector = [γ; ψ; β(4)], s-vector = [sγ; sψ; sβ(4)]
  // (rows beyond c.nh stay zero)
  Mat<6, 1> contact_constraint(const ContactS& c) const {
    Cfg p = cfg_next(c.body);
    double d = (c.nrm * (p.x + vector_rotate(c.o, p.q) - c.off))[0] - c.radius;
    Mat<6, 1> r;
    r[0] = d - c.s[1][0];
    if (c.type == 0) return r;
    V3 cp = contact_point(c, p);
    V3 vp = p.v + skew(vector_rotate(p.w, p.q)) * (cp - p.x);
    Mat<2, 1> vt = c.t * vp;  // child = origin: zero velocity
    if (c.type == 2) {
      r[1] = c.mu_f * c.gam[1][0] - c.gam[1][1];
      r[2] = vt[0] - c.s[1][2];
      r[3] = vt[1] - c.s[1][3];
    } else {
      r[1] = c.mu_f * c.gam[1][0] - (c.gam[1][2] + c.gam[1][3] + c.gam[1][4] + c.gam[1][5]) - c.s[1][1];
      for (int i = 0; i < 4; ++i) r[2 + i] = (kLinearParam[i][0] * vt[0] + kLinearParam[i][1] * vt[1]) + c.gam[1][1] - c.s[1][2 + i];
    }
    return r;
  }
  // solver/complementarity.jl:16-24: nonlinear [γ1 s1; cone_product(γ(2:4), s(2:4))]  (contacts/cone.jl:2-8); impact / linear γ .* s
  static void contact_complementarity(const ContactS& c, const double* g, const double* s, double* out) {
    if (c.type != 2) { for (int i = 0; i < c.nh; ++i) out[i] = g[i] * s[i]; return; }
    out[0] = g[0] * s[0];
    out[1] = g[1] * s[1] + g[2] * s[2] + g[3] * s[3];
    out[2] = g[1] * s[2] + s[1] * g[2];
    out[3] = g[1] * s[3] + s[1] * g[3];
  }
  // contacts/impact.jl:58-64: [γ s; -1 0];  contacts/linear.jl:49-70: [Diag(γ) Diag(s); -I ∇γ2]   (top-left 2nh x 2nh used)
  Mat<12, 12> contact_constraint_jacobian_orthant(const ContactS& c) const {
    const int nh = c.nh;
    Mat<12, 12> M;
    for (int i = 0; i < nh; ++i) {
      M(i, i) = c.gam[1][i] + REG * c.neutral(i);
      M(i, nh + i) = c.s[1][i] + REG * c.neutral(i);
      M(nh + i, i) = -1.0;
    }
    if (c.type == 1) {
      M(nh + 1, nh + 0) = c.mu_f;
      for (int i = 0; i < 4; ++i) { M(nh + 1, nh + 2 + i) = -1.0; M(nh + 2 + i, nh + 1) = 1.0; }
    }
    return M;
  }
  // contacts/nonlinear.jl:78-97
  Mat<12, 12> contact_constraint_jacobian(const ContactS& c) const {
    if (c.type != 2) return contact_constraint_jacobian_orthant(c);
    Mat<8, 8> M8 = contact_constraint_jacobian_nonlinear(c);
    Mat<12, 12> M;
    for (int r = 0; r < 8; ++r) for (int cc = 0; cc < 8; ++cc) M(r, cc) = M8(r, cc);
    return M;
  }
  Mat<8, 8> contact_constraint_jacobian_nonlinear(const ContactS& c) const {
    double g[4], s[4];
    const double neutral[4] = {1, 1, 0, 0};
    for (int i = 0; i < 4; ++i) { g[i] = c.gam[1][i] + REG * neutral[i]; s[i] = c.s[1][i] + REG * neutral[i]; }
    Mat<8, 8> M;
    auto arrow = [&](int r0, int c0, const double* u) {  // cone_product_jacobian (cone.jl:10-12)
      M(r0, c0) = u[1]; M(r0, c0 + 1) = u[2]; M(r0, c0 + 2) = u[3];
      M(r0 + 1, c0) = u[2]; M(r0 + 1, c0 + 1) = u[1];
      M(r0 + 2, c0) = u[3]; M(r0 + 2, c0 + 2) = u[1];
    };
    M(0, 0) = g[0]; arrow(1, 1, g);          // ∇s rows 1:4
    M(4, 0) = -1; M(6, 2) = -1; M(7, 3) = -1;  // ∇s3 = Diagonal(-1, 0, -1, -1)
    M(0, 4) = s[0]; arrow(1, 5, s);          // ∇γ rows 1:4
    M(5, 4) = c.mu_f; M(5, 5) = -1.0;        // ∇γ3
    return M;
  }
  // Rows of the NonlinearContact pattern [normal; 0; tangent 1; tangent 2] mapped to the model's N½ rows:
  // impact [normal] (impact.jl:66-101), linear [normal; 0; friction_parameterization * tangents] (contact.jl:22-33, :64-74).
  template <int C>
  static Mat<6, C> expand_rows(const ContactS& c, const Mat<4, C>& J4) {
    Mat<6, C> J;
    for (int k = 0; k < C; ++k) J(0, k) = J4(0, k);
    if (c.type == 2) { for (int r = 1; r < 4; ++r) for (int k = 0; k < C; ++k) J(r, k) = J4(r, k); }
    else if (c.type == 1) { for (int i = 0; i < 4; ++i) for (int k = 0; k < C; ++k) J(2 + i, k) = kLinearParam[i][0] * J4(2, k) + kLinearParam[i][1] * J4(3, k); }
    return J;
  }
  Mat<6, 6> contact_constraint_jacobian_velocity(const ContactS& c) const { return expand_rows(c, contact_constraint_jacobian_velocity4(c)); }
  Mat<6, 7> contact_constraint_jacobian_configuration(const ContactS& c) const { return expand_rows(c, contact_constraint_jacobian_configuration4(c)); }
  // contacts/contact.jl:37-77 (relative = :parent): 4 x 6
  Mat<4, 6> contact_constraint_jacobian_velocity4(const ContactS& c) const {
    Cfg p = cfg_next(c.body);
    Mat<1, 3> dddx = c.nrm;
    Mat<1, 4> dddq = c.nrm * dvector_rotate_dq(c.o, p.q);
    V3 cp = contact_point(c, p);
    // velocity.jl:56-104 with the child (origin) terms vanishing
    M34 dcpv_dq = -skew(cp - p.x) * dvector_rotate_dq(p.w, p.q);
    M33 dcpv_dc = skew(vector_rotate(p.w, p.q));
    Mat<2, 4> dvt_dq = c.t * dcpv_dq + c.t * dcpv_dc * dvector_rotate_dq(c.o, p.q);
    Mat<2, 3> dvt_dv = c.t;
    Mat<2, 3> dvt_dw = c.t * (-skew(cp - p.x) * rotation_matrix(p.q));
    // recover current orientation
    Quat q = next_orientation(p.q, -p.w, h);
    M43 dq_dw = rotational_integrator_jacobian_velocity(q, p.w, h);
    Mat<4, 6> J;
    Mat<1, 3> r0 = dddx * h;
    Mat<1, 3> r0w = dddq * dq_dw;
    Mat<2, 3> r2w = dvt_dw + dvt_dq * dq_dw;
    for (int i = 0; i < 3; ++i) {
      J(0, i) = r0[i]; J(0, 3 + i) = r0w[i];
      J(2, i) = dvt_dv(0, i); J(3, i) = dvt_dv(1, i);
      J(2, 3 + i) = r2w(0, i); J(3, 3 + i) = r2w(1, i);
    }
    return J;
  }
  // contacts/contact.jl:9-35 (relative = :parent): 4 x 7, used by the data Jacobian
  Mat<4, 7> contact_constraint_jacobian_configuration4(const ContactS& c) const {
    Cfg p = cfg_next(c.body);
    V3 cp = contact_point(c, p);
    M34 dcpv_dq = -skew(cp - p.x) * dvector_rotate_dq(p.w, p.q);
    M33 dcpv_dc = skew(vector_rotate(p.w, p.q));
    M33 dcpv_dx = -skew(vector_rotate(p.w, p.q));
    Mat<2, 3> dvt_dx = c.t * dcpv_dx + c.t * dcpv_dc;  // ∂contact_point∂x(parent,parent) = I
    Mat<2, 4> dvt_dq = c.t * dcpv_dq + c.t * dcpv_dc * dvector_rotate_dq(c.o, p.q);
    Mat<1, 4> dddq = c.nrm * dvector_rotate_dq(c.o, p.q);
    Mat<4, 7> J;
    for (int i = 0; i < 3; ++i) { J(0, i) = c.nrm[i]; J(2, i) = dvt_dx(0, i); J(3, i) = dvt_dx(1, i); }
    for (int i = 0; i < 4; ++i) { J(0, 3 + i) = dddq[i]; J(2, 3 + i) = dvt_dq(0, i); J(3, 3 + i) = dvt_dq(1, i); }
    return J;
  }
  // contacts/contact.jl:79-100,141-155: [X; Rot(q3)ᵀ skew(c - x3) X], X = [nᵀ 0 tᵀ Pᵀ]  (6 x N½; nonlinear P = I, impact.jl:103-115 X = nᵀ)
  Mat<3, 6> force_mapping(const ContactS& c) const {
    Mat<3, 6> X;
    for (int i = 0; i < 3; ++i) X(i, 0) = c.nrm[i];
    if (c.type == 2) { for (int i = 0; i < 3; ++i) { X(i, 2) = c.t(0, i); X(i, 3) = c.t(1, i); } }
    else if (c.type == 1) { for (int k = 0; k < 4; ++k) for (int i = 0; i < 3; ++i) X(i, 2 + k) = c.t(0, i) * kLinearParam[k][0] + c.t(1, i) * kLinearParam[k][1]; }
    return X;
  }
  Mat<6, 6> contact_impulse_map(const ContactS& c) const {
    Cfg p = cfg_next(c.body);
    Mat<3, 6> X = force_mapping(c);
    V3 r = contact_point(c, p) - p.x;
    Mat<3, 6> Q = rotation_matrix(inv(p.q)) * skew(r) * X;
    return vcat(X, Q);
  }
  // contacts/contact.jl:102-138 (relative = jacobian = :parent; normals/tangents constant): 6 x 7
  Mat<6, 7> contact_impulse_map_jacobian(const ContactS& c) const {
    Cfg p = cfg_next(c.body);
    Mat<3, 6> X = force_mapping(c);
    Mat<6, 1> lam;
    for (int i = 0; i < c.nh; ++i) lam[i] = c.gam[1][i];
    V3 r = contact_point(c, p) - p.x;
    V3 Xl = X * lam;
    M33 Qx = -(rotation_matrix(inv(p.q)) * skew(Xl) * (M33::identity() - M33::identity()));
    M34 Qq = -(rotation_matrix(inv(p.q)) * skew(Xl) * dvector_rotate_dq(c.o, p.q));
    Qq += drotation_matrix_dq(inv(p.q), skew(r) * Xl) * Tmat();
    Mat<6, 7> J;
    set_block(J, 3, 0, Qx);
    set_block(J, 3, 3, Qq);
    return J;
  }

  // ---------------------------------------------------------------- joints
  // joints/constraints.jl:114-120
  void joint_constraint(const JointS& j, double* out) const {
    Cfg a = cfg_next(j.parent), b = cfg_next(j.child);
    for (int k = 0; k < 2; ++k) {
      EVec r = element_constraint(j, k, a.x, a.q, b.x, b.q, j.imp[1].data() + j.eoff[k], mu);
      for (int i = 0; i < r.n; ++i) out[j.eoff[k] + i] = r.v[i];
    }
  }
  // joints/constraints.jl:128-132 + joints/joint.jl:33-43: block diagonal (tra, rot), written into dense A
  void joint_constraint_jacobian(const JointS& j, double* M, int ld) const {
    for (int k = 0; k < 2; ++k) {
      const Elem& e = j.el[k];
      const double* eta = j.imp[1].data() + j.eoff[k];
      int o = j.eoff[k];
      for (int i = 0; i < e.nb; ++i) {
        M[(o + i) * ld + (o + i)] = eta[e.nb + i] + REG;           // Diagonal(γ + reg)
        M[(o + e.nb + i) * ld + (o + i)] = 1.0;                     // Diagonal(ones(Nb))
        M[(o + i) * ld + (o + e.nb + i)] = eta[i] + REG;            // Diagonal(s + reg)
      }
      for (int i = 0; i < e.nl; ++i) M[(o + 2 * e.nb + i) * ld + (o + 2 * e.nb + i)] = REG;
    }
  }
  // joints/constraints.jl:134-148 (at the next configuration): N x 7
  void joint_constraint_jacobian_configuration(const JointS& j, bool parent, Mat<24, 7>& J) const {
    Cfg a = cfg_next(j.parent), b = cfg_next(j.child);
    for (int k = 0; k < 2; ++k) {
      EJac7 r = element_constraint_jacobian_configuration(parent, j, k, a.x, a.q, b.x, b.q);
      for (int i = 0; i < r.n; ++i)
        for (int c = 0; c < 7; ++c) J(j.eoff[k] + i, c) = r.J(i, c);
    }
  }
  // joints/constraints.jl:157-168 (at the current configuration x2,q2): 6 x N
  void joint_impulse_map(const JointS& j, bool parent, Mat<6, 24>& G) const {
    Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
    for (int k = 0; k < 2; ++k) {
      EMap r = element_impulse_map(parent, j, k, a.x, a.q, b.x, b.q);
      for (int i = 0; i < r.n; ++i)
        for (int rr = 0; rr < 6; ++rr) G(rr, j.eoff[k] + i) = r.G(rr, i);
    }
  }

  // ---------------------------------------------------------------- bodies
  // integrators/constraint.jl:1-34 (+ joints/constraints.jl:150-155, contacts/constraints.jl:31-34)
  V6 body_constraint(int bi) const {
    const BodyS& s = bodies[bi];
    V3 x3 = next_position(s.x2, s.vsol[1], h);
    Quat q3 = next_orientation(s.q2, s.wsol[1], h);
    V3 D1x = (-1.0 / h * s.mass) * (s.x2 - s.x1) - 0.5 * h * (s.mass * gravity + s.Fext);
    V3 D2x = (1.0 / h * s.mass) * (x3 - s.x2) - 0.5 * h * (s.mass * gravity + s.Fext);
    V3 D1q = (-2.0 / h) * (tr(LVtmat(s.q2)) * Lmat(s.q1) * Vtmat() * s.J * Vmat() * Ltmat(s.q1) * vector(s.q2)) - 0.5 * h * s.text;
    V3 D2q = (-2.0 / h) * (tr(LVtmat(s.q2)) * Tmat() * Rtmat(q3) * Vtmat() * s.J * Vmat() * Ltmat(s.q2) * vector(q3)) - 0.5 * h * s.text;
    V6 d = vcat(D2x + D1x, D2q + D1q);
    d -= vcat(s.JF2, s.Jt2);
    for (const JointS& j : joints) {
      if (j.parent != bi && j.child != bi) continue;
      bool parent = (j.parent == bi);
      if (j.n > 0) {
        Mat<6, 24> G;
        joint_impulse_map(j, parent, G);
        for (int r = 0; r < 6; ++r) {
          double acc = 0;
          for (int i = 0; i < j.n; ++i) acc += G(r, i) * j.imp[1][i];
          d[r] -= acc;
        }
      }
      Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
      if (j.spring) for (int k = 0; k < 2; ++k) d -= spring_impulses(parent, j, k, a.x, a.q, b.x, b.q, h);
      if (j.damper) for (int k = 0; k < 2; ++k) d -= damper_impulses(parent, j, k, a, b, h);
    }
    for (const ContactS& c : contacts) {
      if (c.body != bi) continue;
      Mat<6, 1> lam;
      for (int i = 0; i < c.nh; ++i) lam[i] = c.gam[1][i];
      d -= contact_impulse_map(c) * lam;
    }
    return d;
  }
  // integrators/constraint.jl:36-66 (+ joints/constraints.jl:184-205, contacts/constraints.jl:53-57)
  M66 body_constraint_jacobian(int bi) const {
    const BodyS& s = bodies[bi];
    Quat q3 = next_orientation(s.q2, s.wsol[1], h);
    M34 dynR = (-2.0 / h) * (tr(LVtmat(s.q2)) * Tmat() *
                             (dRtmat_dq(Vtmat() * s.J * Vmat() * Ltmat(s.q2) * vector(q3)) + Rtmat(q3) * Vtmat() * s.J * Vmat() * Ltmat(s.q2)));
    Mat<6, 7> lhs;
    for (int i = 0; i < 3; ++i) lhs(i, i) = s.mass / h;
    set_block(lhs, 3, 3, dynR);
    Mat<7, 6> ijv = integrator_jacobian_velocity(s.q2, s.wsol[1], h);
    M66 D = lhs * ijv;
    for (int i = 0; i < 6; ++i) D(i, i) += REG;
    for (const JointS& j : joints) {
      if (j.parent != bi && j.child != bi) continue;
      if (!j.damper) continue;  // spring velocity Jacobians are zero
      bool parent = (j.parent == bi);
      Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
      for (int k = 0; k < 2; ++k) D -= damper_jacobian_velocity(parent, parent, j, k, a, b, h);
    }
    for (const ContactS& c : contacts) {
      if (c.body != bi) continue;
      D -= contact_impulse_map_jacobian(c) * ijv;
    }
    return D;
  }

  // ---------------------------------------------------------------- assembly: set_entries! (solver/linear_system.jl:1-17)
  void zero_pattern(std::vector<double>& M) {
    const int n = nres;
    for (auto& pb : pattern) {
      int oa = node_off[pb.first], da = node_dim[pb.first], ob = node_off[pb.second], db = node_dim[pb.second];
      for (int r = 0; r < da; ++r) std::memset(&M[(size_t)(oa + r) * n + ob], 0, sizeof(double) * db);
    }
  }
  void set_entries() {
    zero_pattern(A);  // only the structurally non-zero blocks are ever touched
    const int n = nres;
    // bodies: integrators/constraint.jl:82-85
    for (int b = 0; b < Nb; ++b) {
      M66 D = body_constraint_jacobian(b);
      V6 d = body_constraint(b);
      int o = body_off[b];
      for (int r = 0; r < 6; ++r) {
        rhs[o + r] = -d[r];
        for (int c = 0; c < 6; ++c) A[(size_t)(o + r) * n + o + c] = D(r, c);
      }
    }
    // joints: joints/constraints.jl:296-299, off-diagonals :208-214 and body-body :216-249
    for (const JointS& j : joints) {
      std::vector<double> g(j.n);
      joint_constraint(j, g.data());
      for (int i = 0; i < j.n; ++i) rhs[j.sol_off + i] = -g[i];
      joint_constraint_jacobian(j, &A[(size_t)j.sol_off * n + j.sol_off], n);
      for (int side = 0; side < 2; ++side) {
        bool parent = (side == 0);
        int bi = parent ? j.parent : j.child;
        if (bi < 0) continue;
        const BodyS& s = bodies[bi];
        Mat<24, 7> Jc;
        joint_constraint_jacobian_configuration(j, parent, Jc);
        Mat<24, 6> U = Jc * integrator_jacobian_velocity(s.q2, s.wsol[1], h);
        Mat<6, 24> G;
        joint_impulse_map(j, parent, G);
        int ob = body_off[bi];
        for (int i = 0; i < j.n; ++i)
          for (int c = 0; c < 6; ++c) {
            A[(size_t)(j.sol_off + i) * n + ob + c] = U(i, c);     // joint row, body column
            A[(size_t)(ob + c) * n + j.sol_off + i] = -G(c, i);    // body row, joint column: -impulse_map
          }
      }
      if (j.damper && j.parent >= 0) {
        Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
        M66 Jpc, Jcp;
        for (int k = 0; k < 2; ++k) {
          Jpc -= damper_jacobian_velocity(true, false, j, k, a, b, h);   // ∂(parent impulse)/∂(child velocity)
          Jcp -= damper_jacobian_velocity(false, true, j, k, a, b, h);   // ∂(child impulse)/∂(parent velocity)
        }
        int op = body_off[j.parent], oc = body_off[j.child];
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) {
            A[(size_t)(op + r) * n + oc + c] += Jpc(r, c);
            A[(size_t)(oc + r) * n + op + c] += Jcp(r, c);
          }
      }
    }
    // contacts: contacts/constraints.jl:60-76
    for (const ContactS& c : contacts) {
      const int nh = c.nh;
      Mat<12, 12> Dc = contact_constraint_jacobian(c);
      double comp[6];
      contact_complementarity(c, c.gam[1], c.s[1], comp);
      Mat<6, 1> g = contact_constraint(c);
      for (int i = 0; i < nh; ++i) { rhs[c.sol_off + i] = -(comp[i] - mu * c.neutral(i)); rhs[c.sol_off + nh + i] = -g[i]; }
      for (int r = 0; r < 2 * nh; ++r)
        for (int cc = 0; cc < 2 * nh; ++cc) A[(size_t)(c.sol_off + r) * n + c.sol_off + cc] = Dc(r, cc);
      Mat<6, 6> Jv = contact_constraint_jacobian_velocity(c);
      Mat<6, 6> G = contact_impulse_map(c);
      int ob = body_off[c.body];
      for (int r = 0; r < nh; ++r)
        for (int cc = 0; cc < 6; ++cc) {
          A[(size_t)(c.sol_off + nh + r) * n + ob + cc] = Jv(r, cc);   // [Z; constraint_jacobian_velocity]
          A[(size_t)(ob + cc) * n + c.sol_off + nh + r] = -G(cc, r);   // [Z' -impulse_map]
        }
    }
  }

  // full residual r(w) with the convention rhs = -r (used by the finite-difference tests)
  void evaluate_rhs(double* out) {
    for (int b = 0; b < Nb; ++b) { V6 d = body_constraint(b); for (int r = 0; r < 6; ++r) out[body_off[b] + r] = -d[r]; }
    for (const JointS& j : joints) {
      std::vector<double> g(j.n);
      joint_constraint(j, g.data());
      for (int i = 0; i < j.n; ++i) out[j.sol_off + i] = -g[i];
    }
    for (const ContactS& c : contacts) {
      double comp[6];
      contact_complementarity(c, c.gam[1], c.s[1], comp);
      Mat<6, 1> g = contact_constraint(c);
      for (int i = 0; i < c.nh; ++i) { out[c.sol_off + i] = -(comp[i] - mu * c.neutral(i)); out[c.sol_off + c.nh + i] = -g[i]; }
    }
  }

  // ---------------------------------------------------------------- violations (solver/violations.jl)
  double residual_violation() const {
    double v = 0.0;
    for (const JointS& j : joints) {  // :16-33: equality rows only
      std::vector<double> g(j.n);
      joint_constraint(j, g.data());
      for (int k = 0; k < 2; ++k) {
        const Elem& e = j.el[k];
        for (int i = 0; i < e.nl; ++i) v = std::max(v, std::fabs(g[j.eoff[k] + 2 * e.nb + i]));
      }
    }
    for (int b = 0; b < Nb; ++b) { V6 d = body_constraint(b); for (int r = 0; r < 6; ++r) v = std::max(v, std::fabs(d[r])); }
    for (const ContactS& c : contacts) { Mat<6, 1> g = contact_constraint(c); for (int r = 0; r < c.nh; ++r) v = std::max(v, std::fabs(g[r])); }
    return v;
  }
  double bilinear_violation() const {
    double v = 0.0;
    for (const JointS& j : joints)
      for (int k = 0; k < 2; ++k) {
        const Elem& e = j.el[k];
        const double* eta = j.imp[1].data() + j.eoff[k];
        for (int i = 0; i < e.nb; ++i) v = std::max(v, std::fabs(eta[i] * eta[e.nb + i]));
      }
    for (const ContactS& c : contacts) {
      double comp[6];
      contact_complementarity(c, c.gam[1], c.s[1], comp);
      for (int i = 0; i < c.nh; ++i) v = std::max(v, std::fabs(comp[i]));
    }
    return v;
  }

  // ---------------------------------------------------------------- linear algebra
  // GraphBasedSystems.ldu_factorization! restated on dense storage with known block structure
  bool factorize() {
    const int n = nres;
    if (solver_mode == 1) return true;
    if (F.size() != A.size()) F.assign(A.size(), 0.0);
    for (auto& pb : pattern) {  // copy the structural blocks only
      int oa = node_off[pb.first], da = node_dim[pb.first], ob = node_off[pb.second], db = node_dim[pb.second];
      for (int r = 0; r < da; ++r) std::memcpy(&F[(size_t)(oa + r) * n + ob], &A[(size_t)(oa + r) * n + ob], sizeof(double) * db);
    }
    for (int k : elim_order) {
      int dk = node_dim[k], ok = node_off[k];
      if (dk == 0) continue;
      if (!invert_inplace(&F[(size_t)ok * n + ok], dk, n)) return false;  // D_k <- D_k^{-1}
      const std::vector<int>& nb = elim_nbrs[k];
      // L_ik <- A_ik D_k^{-1}
      std::vector<double> tmp;
      for (int i : nb) {
        int di = node_dim[i], oi = node_off[i];
        tmp.assign((size_t)di * dk, 0.0);
        for (int r = 0; r < di; ++r)
          for (int c = 0; c < dk; ++c) {
            double acc = 0;
            for (int t = 0; t < dk; ++t) acc += F[(size_t)(oi + r) * n + ok + t] * F[(size_t)(ok + t) * n + ok + c];
            tmp[(size_t)r * dk + c] = acc;
          }
        for (int r = 0; r < di; ++r)
          for (int c = 0; c < dk; ++c) F[(size_t)(oi + r) * n + ok + c] = tmp[(size_t)r * dk + c];
      }
      // A_ij -= L_ik A_kj
      for (int i : nb)
        for (int j2 : nb) {
          int di = node_dim[i], oi = node_off[i], dj = node_dim[j2], oj = node_off[j2];
          for (int r = 0; r < di; ++r)
            for (int c = 0; c < dj; ++c) {
              double acc = 0;
              for (int t = 0; t < dk; ++t) acc += F[(size_t)(oi + r) * n + ok + t] * F[(size_t)(ok + t) * n + oj + c];
              F[(size_t)(oi + r) * n + oj + c] -= acc;
            }
        }
    }
    return true;
  }
  // ldu_backsubstitution!: x <- A^{-1} x for m right-hand sides (x is nres x m row-major)
  bool solve(double* x, int m) {
    const int n = nres;
    if (solver_mode == 1) return dense_solve(A, n, x, m);
    std::vector<double> t;
    for (int k : elim_order) {  // forward: b_i -= L_ik b_k
      int dk = node_dim[k], ok = node_off[k];
      for (int i : elim_nbrs[k]) {
        int di = node_dim[i], oi = node_off[i];
        for (int r = 0; r < di; ++r)
          for (int c = 0; c < m; ++c) {
            double acc = 0;
            for (int tt = 0; tt < dk; ++tt) acc += F[(size_t)(oi + r) * n + ok + tt] * x[(size_t)(ok + tt) * m + c];
            x[(size_t)(oi + r) * m + c] -= acc;
          }
      }
    }
    for (int idx = (int)elim_order.size() - 1; idx >= 0; --idx) {  // backward: x_k = D_k^{-1} (b_k - sum A_kj x_j)
      int k = elim_order[idx];
      int dk = node_dim[k], ok = node_off[k];
      if (dk == 0) continue;
      for (int j2 : elim_nbrs[k]) {
        int dj = node_dim[j2], oj = node_off[j2];
        for (int r = 0; r < dk; ++r)
          for (int c = 0; c < m; ++c) {
            double acc = 0;
            for (int tt = 0; tt < dj; ++tt) acc += F[(size_t)(ok + r) * n + oj + tt] * x[(size_t)(oj + tt) * m + c];
            x[(size_t)(ok + r) * m + c] -= acc;
          }
      }
      t.assign((size_t)dk * m, 0.0);
      for (int r = 0; r < dk; ++r)
        for (int c = 0; c < m; ++c) {
          double acc = 0;
          for (int tt = 0; tt < dk; ++tt) acc += F[(size_t)(ok + r) * n + ok + tt] * x[(size_t)(ok + tt) * m + c];
          t[(size_t)r * m + c] = acc;
        }
      for (int r = 0; r < dk; ++r)
        for (int c = 0; c < m; ++c) x[(size_t)(ok + r) * m + c] = t[(size_t)r * m + c];
    }
    return true;
  }

  // ---------------------------------------------------------------- solver pieces
  // solver/line_search.jl:102-113
  static double positive_orthant_step_length(const double* lam, const double* dl, int n, double tau) {
    double a = 1.0;
    for (int i = 0; i < n; ++i) if (dl[i] < 0) a = std::min(a, -tau * lam[i] / dl[i]);
    return a;
  }
  // solver/line_search.jl:115-139
  static double second_order_cone_step_length(const double* lam, const double* dl, double tau) {
    const double eps = 1e-14;
    double l0 = lam[0];
    double ll = std::max(l0 * l0 - (lam[1] * lam[1] + lam[2] * lam[2]), 1e-25);
    ll += eps;
    double ld = l0 * dl[0] - (lam[1] * dl[1] + lam[2] * dl[2]) + eps;
    double rs = ld / ll;
    double sq = std::sqrt(ll);
    double f = (ld / sq + dl[0]) / (l0 / sq + 1.0);
    double rv1 = dl[1] / sq - f * lam[1] / ll;
    double rv2 = dl[2] / sq - f * lam[2] / ll;
    double nrm = std::sqrt(rv1 * rv1 + rv2 * rv2);
    double a = 1.0;
    if (nrm - rs > 0.0) a = std::min(a, tau / (nrm - rs));
    return a;
  }
  // solver/line_search.jl:36-100 (Δ in rhs)
  double cone_line_search(double tau_ort, double tau_soc) const {
    double a = 1.0;
    for (const ContactS& c : contacts) {
      const double* ds = &rhs[c.sol_off];
      const double* dg = &rhs[c.sol_off + c.nh];
      if (c.type != 2) {  // line_search.jl:71-86: impact / linear are orthant-only
        a = std::min(a, std::min(positive_orthant_step_length(c.s[1], ds, c.nh, tau_ort), positive_orthant_step_length(c.gam[1], dg, c.nh, tau_ort)));
        continue;
      }
      double as_ort = positive_orthant_step_length(c.s[1], ds, 1, tau_ort);
      double ag_ort = positive_orthant_step_length(c.gam[1], dg, 1, tau_ort);
      double as_soc = second_order_cone_step_length(c.s[1] + 1, ds + 1, tau_soc);
      double ag_soc = second_order_cone_step_length(c.gam[1] + 1, dg + 1, tau_soc);
      a = std::min(std::min(std::min(a, as_soc), std::min(ag_soc, as_ort)), ag_ort);
    }
    for (const JointS& j : joints)
      for (int k = 0; k < 2; ++k) {
        const Elem& e = j.el[k];
        const double* eta = j.imp[1].data() + j.eoff[k];
        const double* d = &rhs[j.sol_off + j.eoff[k]];
        a = std::min(a, positive_orthant_step_length(eta, d, e.nb, tau_ort));
        a = std::min(a, positive_orthant_step_length(eta + e.nb, d + e.nb, e.nb, tau_ort));
      }
    return a;
  }
  // solver/centering.jl:1-48
  void centering(double aaff, double& nu, double& nuaff) const {
    double sn = 0, sa = 0, cnt = 0;
    for (const ContactS& c : contacts) {
      const double* ds = &rhs[c.sol_off];
      const double* dg = &rhs[c.sol_off + c.nh];
      for (int i = 0; i < c.nh; ++i) { sn += c.s[1][i] * c.gam[1][i]; sa += (c.s[1][i] + aaff * ds[i]) * (c.gam[1][i] + aaff * dg[i]); }
      cnt += c.cone_degree();  // cone_degree(NonlinearContact) = 2 (nonlinear.jl:101), N½ otherwise (contact.jl:197)
    }
    for (const JointS& j : joints)
      for (int k = 0; k < 2; ++k) {
        const Elem& e = j.el[k];
        const double* eta = j.imp[1].data() + j.eoff[k];
        const double* d = &rhs[j.sol_off + j.eoff[k]];
        for (int i = 0; i < e.nb; ++i) { sn += eta[i] * eta[e.nb + i]; sa += (eta[i] + aaff * d[i]) * (eta[e.nb + i] + aaff * d[e.nb + i]); }
        cnt += e.nb;
      }
    nu = sn / cnt;  // 0/0 = NaN when there are no cones, exactly as the reference
    nuaff = sa / cnt;
  }
  // solver/correction.jl:1-45: res_saved += [-Δs∘Δγ + μ e; 0]
  void correction() {
    for (const ContactS& c : contacts) {
      const double* ds = &rhs[c.sol_off];
      const double* dg = &rhs[c.sol_off + c.nh];
      if (c.type != 2) { for (int i = 0; i < c.nh; ++i) res_saved[c.sol_off + i] += -ds[i] * dg[i] + mu; continue; }  // correction.jl:13-19
      res_saved[c.sol_off + 0] += -ds[0] * dg[0] + mu;
      res_saved[c.sol_off + 1] += -(ds[1] * dg[1] + ds[2] * dg[2] + ds[3] * dg[3]) + mu;
      res_saved[c.sol_off + 2] += -(ds[1] * dg[2] + dg[1] * ds[2]);
      res_saved[c.sol_off + 3] += -(ds[1] * dg[3] + dg[1] * ds[3]);
    }
    for (const JointS& j : joints)
      for (int k = 0; k < 2; ++k) {
        const Elem& e = j.el[k];
        int o = j.sol_off + j.eoff[k];
        for (int i = 0; i < e.nb; ++i) res_saved[o + i] += -rhs[o + i] * rhs[o + e.nb + i] + mu;
      }
  }
  // solver/line_search.jl:141-163
  void candidate_step(double alpha, int scale) {
    double f = 1.0 / std::pow(2.0, scale) * alpha;
    for (ContactS& c : contacts)
      for (int i = 0; i < c.nh; ++i) { c.s[1][i] = c.s[0][i] + f * rhs[c.sol_off + i]; c.gam[1][i] = c.gam[0][i] + f * rhs[c.sol_off + c.nh + i]; }
    for (JointS& j : joints)
      for (int i = 0; i < j.n; ++i) j.imp[1][i] = j.imp[0][i] + f * rhs[j.sol_off + i];
    double wmax = 3.9 / (h * h);
    for (int b = 0; b < Nb; ++b) {
      BodyS& s = bodies[b];
      for (int i = 0; i < 3; ++i) { s.vsol[1][i] = s.vsol[0][i] + f * rhs[body_off[b] + i]; s.wsol[1][i] = s.wsol[0][i] + f * rhs[body_off[b] + 3 + i]; }
      double wd = dot(s.wsol[1], s.wsol[1]);
      if (wd > wmax) s.wsol[1] = s.wsol[1] * (wmax / wd);
    }
  }
  bool excessive_omega() const {
    for (const BodyS& s : bodies) if (dot(s.wsol[1], s.wsol[1]) > 3.91 / (h * h)) return true;
    return false;
  }
  // solver/line_search.jl:1-34
  bool line_search(double alpha, double rvio, double bvio, int max_ls, double& rv, double& bv) {
    int scale = 0;
    rv = std::numeric_limits<double>::infinity();
    bv = std::numeric_limits<double>::infinity();
    for (int n = 0; n < max_ls; ++n) {
      candidate_step(alpha, scale);
      if (excessive_omega()) return false;
      rv = residual_violation();
      bv = bilinear_violation();
      if ((rv > rvio) && (bv > bvio)) scale += 1;
      else return true;
    }
    return true;
  }
  // solver/initialization.jl:1-48
  static void initialize_positive_orthant(double& g, double& s) {
    const double eps = 1e-20;
    double ds = std::max(-1.5 * s, 0.0), dg = std::max(-1.5 * g, 0.0);
    double sh = s + ds, gh = g + dg;
    double dhs = 0.5 * sh * gh / (gh + eps), dhg = 0.5 * sh * gh / (sh + eps);
    s = sh + dhs; g = gh + dhg;
  }
  // initialize_positive_orthant! on a vector (initialization.jl:20-33): min / sum over the N½ components
  static void initialize_positive_orthant_n(double* g, double* s, int n) {
    const double eps = 1e-20;
    double smin = s[0], gmin = g[0];
    for (int i = 1; i < n; ++i) { smin = std::min(smin, s[i]); gmin = std::min(gmin, g[i]); }
    double ds = std::max(-1.5 * smin, 0.0), dg = std::max(-1.5 * gmin, 0.0);
    double shg = 0, sums = 0, sumg = 0;
    for (int i = 0; i < n; ++i) { s[i] += ds; g[i] += dg; }
    for (int i = 0; i < n; ++i) { shg += s[i] * g[i]; sums += s[i]; sumg += g[i]; }
    double dhs = 0.5 * shg / (sumg + eps), dhg = 0.5 * shg / (sums + eps);
    for (int i = 0; i < n; ++i) { s[i] += dhs; g[i] += dhg; }
  }
  static void initialize_second_order_cone(double* g, double* s) {
    const double eps = 1e-20;
    double ns = std::sqrt(s[1] * s[1] + s[2] * s[2]), ng = std::sqrt(g[1] * g[1] + g[2] * g[2]);
    double ds = std::max(-1.5 * (s[0] - ns), 0.0), dg = std::max(-1.5 * (g[0] - ng), 0.0);
    double sh0 = s[0] + ds, gh0 = g[0] + dg;
    double shg = sh0 * gh0 + s[1] * g[1] + s[2] * g[2];
    double dhs = 0.5 * shg / ((gh0 + ng) + eps), dhg = 0.5 * shg / ((sh0 + ns) + eps);
    s[0] = sh0 + dhs; g[0] = gh0 + dhg;
  }

  // ---------------------------------------------------------------- mehrotra! (solver/mehrotra.jl:9-73)
  int force_iters = -1;
  int mehrotra(const DojoSolverOptions& opts, int* iters_out) {
    for (ContactS& c : contacts)  // reset! (contacts/constraints.jl:79-86), neutral = [1,1,0,0]
      for (int idx = 0; idx < 2; ++idx) for (int i = 0; i < c.nh; ++i) { c.gam[idx][i] = c.neutral(i); c.s[idx][i] = c.neutral(i); }
    for (JointS& j : joints)      // reset! (joints/constraints.jl:440-448)
      for (int idx = 0; idx < 2; ++idx)
        for (int k = 0; k < 2; ++k) {
          const Elem& e = j.el[k];
          for (int i = 0; i < 2 * e.nb; ++i) j.imp[idx][j.eoff[k] + i] = 1.0;
          for (int i = 0; i < e.nl; ++i) j.imp[idx][j.eoff[k] + 2 * e.nb + i] = 0.0;
        }
    int status = DOJO_STATUS_FAILED;
    mu = 0.0;
    double mutarget = 0.0;
    int no_progress = 0;
    double undercut = opts.undercut;
    double alpha = 1.0;
    for (ContactS& c : contacts)  // initialize! (solver/initialization.jl:7-18)
      for (int idx = 0; idx < 2; ++idx) {
        if (c.type == 2) { initialize_positive_orthant(c.gam[idx][0], c.s[idx][0]); initialize_second_order_cone(c.gam[idx] + 1, c.s[idx] + 1); }
        else initialize_positive_orthant_n(c.gam[idx], c.s[idx], c.nh);  // initialization.jl:1-5
      }
    set_entries();
    double bvio = bilinear_violation();
    double rvio = residual_violation();
    trace.clear();
    int n_done = 0;
    for (int n = 1; n <= opts.max_iter; ++n) {
      trace.push_back(rvio); trace.push_back(bvio); trace.push_back(alpha); trace.push_back(mutarget);
      // force_iters >= 0 (test hook, tests/test_gpu_parity.py): run EXACTLY that many Newton iterations -- the convergence test is skipped
      // before, and taken for granted after -- so that the iterate of a path that stopped one comparison earlier / later can be reproduced
      if (force_iters >= 0 ? (n > force_iters) : ((rvio < opts.rtol) && (bvio < opts.btol))) { status = DOJO_STATUS_SUCCESS; break; }
      n_done = n;
      // affine search direction (Quirk Q3: the rhs carries the previous mutarget)
      res_saved = rhs;                                   // pull_residual!
      if (!factorize() || !solve(rhs.data(), 1)) { status = DOJO_STATUS_NONFINITE; break; }
      double aaff = cone_line_search(0.95, 0.95);
      double nu_, nuaff;
      centering(aaff, nu_, nuaff);
      double ratio = nuaff / (nu_ + 1e-20);
      double sig = std::min(std::max(ratio, 0.0), 1.0);  // clamp (NaN propagates like Julia's clamp)
      if (ratio != ratio) sig = ratio;
      sig = sig * sig * sig;
      // corrected search direction
      mutarget = std::max(sig * nu_, opts.btol / undercut);  // Julia max(NaN, x) = NaN
      if ((sig * nu_) != (sig * nu_)) mutarget = sig * nu_;
      mu = mutarget;
      correction();
      rhs = res_saved;                                   // push_residual!
      if (!solve(rhs.data(), 1)) { status = DOJO_STATUS_NONFINITE; break; }
      double tau = std::max(0.95, 1 - std::max(rvio, bvio) * std::max(rvio, bvio));
      alpha = cone_line_search(tau, std::min(tau, 0.95));
      double rv, bv;
      if (!line_search(alpha, rvio, bvio, opts.max_ls, rv, bv)) { status = DOJO_STATUS_EXCESSIVE_OMEGA; break; }
      bool made_progress = (!(rv < opts.rtol) && (rv < 0.8 * rvio)) || (!(bv < opts.btol) && (bv < 0.8 * bvio));
      if (made_progress) no_progress = std::max(no_progress - 1, 0); else no_progress += 1;
      rvio = rv; bvio = bv;
      if (no_progress >= opts.no_progress_max) undercut *= opts.no_progress_undercut;
      // update! (solver/linear_system.jl:54-69)
      for (BodyS& s : bodies) { s.vsol[0] = s.vsol[1]; s.wsol[0] = s.wsol[1]; }
      for (JointS& j : joints) j.imp[0] = j.imp[1];
      for (ContactS& c : contacts) for (int i = 0; i < c.nh; ++i) { c.s[0][i] = c.s[1][i]; c.gam[0][i] = c.gam[1][i]; }
      set_entries();
      if (!(rvio == rvio) || !(bvio == bvio)) { status = DOJO_STATUS_NONFINITE; break; }
    }
    if (iters_out) *iters_out = n_done;
    return status;
  }

  // ---------------------------------------------------------------- step! (simulation/step.jl:11-30)
  int step(const DojoSolverOptions& opts, const double* z, const double* u, const double* fext, double* z_next, double* sol,
           int* iters, uint32_t flags) {
    set_maximal_state(z);
    set_external(fext);
    set_input(u);
    int status = mehrotra(opts, iters);
    if (sol) get_solution(sol);
    write_next_state(z_next, (flags & DOJO_FLAG_Q1_LITERAL_RETURN) != 0);
    return status;
  }
  // bodies/set.jl:22-36 (update_state!) + mechanism/get.jl:126-134 (get_next_state).  The default returns the
  // true next state (x3, v25, q3, w25) = the mechanism's internal state after update_state!; the Q1-literal flag
  // reproduces step!'s return value, which advances the configuration a second time (SURVEY Q1).
  void write_next_state(double* zn, bool q1_literal) const {
    for (int b = 0; b < Nb; ++b) {
      const BodyS& s = bodies[b];
      V3 x3 = next_position(s.x2, s.vsol[1], h);
      Quat q3 = next_orientation(s.q2, s.wsol[1], h);
      if (q1_literal) { x3 = next_position(x3, s.vsol[1], h); q3 = next_orientation(q3, s.wsol[1], h); }
      double* p = zn + 13 * b;
      for (int i = 0; i < 3; ++i) { p[i] = x3[i]; p[3 + i] = s.vsol[1][i]; p[10 + i] = s.wsol[1][i]; }
      p[6] = q3.s; p[7] = q3.v1; p[8] = q3.v2; p[9] = q3.v3;
    }
  }

  // ---------------------------------------------------------------- gradients
  // Data Jacobian restricted to the state / control columns (gradients/data.jl + gradients/state.jl:92-93):
  // D is nres x (12 Nb + nu), columns = bodies [x2(3) v15(3) φ2(3) ω15(3)] then joint inputs.
  void data_jacobian(std::vector<double>& D) const {
    const int m = 12 * Nb + nu;
    D.assign((size_t)nres * m, 0.0);
    auto add = [&](int row0, int col0, int rows, int cols, auto&& f) {
      for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) D[(size_t)(row0 + r) * m + col0 + c] += f(r, c);
    };
    auto colx = [](int b) { return 12 * b; };
    auto colv = [](int b) { return 12 * b + 3; };
    auto colq = [](int b) { return 12 * b + 6; };
    auto colw = [](int b) { return 12 * b + 9; };
    // joints <- body data (data.jl:4-14): -∂g/∂(x3,q3) * ∂(x3,q3)/∂(x2,q2)
    for (const JointS& j : joints)
      for (int side = 0; side < 2; ++side) {
        bool parent = (side == 0);
        int bi = parent ? j.parent : j.child;
        if (bi < 0) continue;
        const BodyS& s = bodies[bi];
        Mat<24, 7> Jc;
        joint_constraint_jacobian_configuration(j, parent, Jc);
        Mat<24, 6> Z = -(Jc * integrator_jacobian_configuration_att(s.q2, s.wsol[1], h));
        add(j.sol_off, colx(bi), j.n, 3, [&](int r, int c) { return Z(r, c); });
        add(j.sol_off, colq(bi), j.n, 3, [&](int r, int c) { return Z(r, 3 + c); });
      }
    // bodies <- own data (data.jl:16-55): v15, ω15 (z2 block multiplied by zero in the reference)
    for (int b = 0; b < Nb; ++b) {
      const BodyS& s = bodies[b];
      int ob = body_off[b];
      add(ob, colv(b), 3, 3, [&](int r, int c) { return r == c ? s.mass : 0.0; });
      M34 dq1 = (-2.0 / h) * (tr(LVtmat(s.q2)) * dLVtmat_dq(s.J * VLtmat(s.q1) * vector(s.q2)));
      dq1 += (-2.0 / h) * (tr(LVtmat(s.q2)) * LVtmat(s.q1) * s.J * dVLtmat_dq(vector(s.q2)));
      M33 dw15 = dq1 * rotational_integrator_jacobian_velocity(s.q2, -s.w15, h);
      add(ob + 3, colw(b), 3, 3, [&](int r, int c) { return dw15(r, c); });
    }
    // bodies <- neighbour data through joints (data.jl:57-124)
    for (const JointS& j : joints) {
      Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
      for (int side = 0; side < 2; ++side) {
        bool parent = (side == 0);
        int bi = parent ? j.parent : j.child;
        int other = parent ? j.child : j.parent;
        if (bi < 0) continue;
        M66 aa, ab;  // w.r.t. own (x2,q2) and the other body's (x2,q2)
        for (int k = 0; k < 2; ++k) {
          const Elem& e = j.el[k];
          Mat<12, 1> lam;
          for (int i = 0; i < e.n; ++i) lam[i] = j.imp[1][j.eoff[k] + i];
          V3 p = impulse_projector(e) * lam;
          aa += impulse_transform_jacobian(parent, parent, j, k, a.x, a.q, b.x, b.q, p);
          ab += impulse_transform_jacobian(parent, !parent, j, k, a.x, a.q, b.x, b.q, p);
          if (j.spring) {
            aa += spring_jacobian_configuration(parent, parent, j, k, a.x, a.q, b.x, b.q);
            ab += spring_jacobian_configuration(parent, !parent, j, k, a.x, a.q, b.x, b.q);
          }
          if (j.damper) {
            aa += damper_jacobian_configuration(parent, parent, j, k, a, b);
            ab += damper_jacobian_configuration(parent, !parent, j, k, a, b);
          }
        }
        if (!(grad_flags & DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN)) {
          aa += input_jacobian_configuration(parent, parent, j, a, b);
          ab += input_jacobian_configuration(parent, !parent, j, a, b);
        }
        int ob = body_off[bi];
        add(ob, colx(bi), 6, 3, [&](int r, int c) { return aa(r, c); });
        add(ob, colq(bi), 6, 3, [&](int r, int c) { return aa(r, 3 + c); });
        if (other >= 0) {
          add(ob, colx(other), 6, 3, [&](int r, int c) { return ab(r, c); });
          add(ob, colq(other), 6, 3, [&](int r, int c) { return ab(r, 3 + c); });
        }
        // bodies <- joint inputs (data.jl:137-150)
        Mat<6, 6> Bu = input_jacobian_control(j, parent);
        add(ob, 12 * Nb + j.u_off, 6, j.nu, [&](int r, int c) { return Bu(r, c); });
      }
    }
    // contacts (data.jl:126-135, :194-205)
    for (const ContactS& c : contacts) {
      const BodyS& s = bodies[c.body];
      Mat<7, 6> icj = integrator_jacobian_configuration_att(s.q2, s.wsol[1], h);
      Mat<6, 6> Zb = contact_impulse_map_jacobian(c) * icj;
      int ob = body_off[c.body];
      add(ob, colx(c.body), 6, 3, [&](int r, int cc) { return Zb(r, cc); });
      add(ob, colq(c.body), 6, 3, [&](int r, int cc) { return Zb(r, 3 + cc); });
      Mat<6, 6> Zc = -(contact_constraint_jacobian_configuration(c) * icj);
      add(c.sol_off + c.nh, colx(c.body), c.nh, 3, [&](int r, int cc) { return Zc(r, cc); });
      add(c.sol_off + c.nh, colq(c.body), c.nh, 3, [&](int r, int cc) { return Zc(r, 3 + cc); });
    }
  }
  // d(input impulse)/d(x2, φ2) of the impulse set_input applies (SURVEY Q17; the reference's unused input_jacobian_configuration,
  // translational/input.jl:45, rotational/input.jl:41): the translational input acts like a joint impulse with only half of its
  // torque (Q16); the rotational input is a constant joint-frame torque, so only the child's R(qb⁻¹ qa qoff) depends on the poses.
  M66 input_jacobian_configuration(bool parent, bool jac_parent, const JointS& j, const Cfg& a, const Cfg& b) const {
    M66 out = impulse_transform_jacobian(parent, jac_parent, j, 0, a.x, a.q, b.x, b.q, j.applied[0]);
    for (int r = 3; r < 6; ++r)
      for (int c = 0; c < 6; ++c) out(r, c) *= 0.5;
    if (!parent) {
      M33 Q = jac_parent ? M33(rotation_matrix(inv(b.q)) * drotation_matrix_dq(a.q, vector_rotate(j.applied[1], j.qoff)) * LVtmat(a.q))
                         : M33(drotation_matrix_inv_dq(b.q, vector_rotate(j.applied[1], a.q * j.qoff)) * LVtmat(b.q));
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) out(3 + r, 3 + c) += Q(r, c);
    }
    return out;
  }
  // translational/springs.jl:44-60, rotational/springs.jl:44-84 (attjac = true): 6 x 6
  M66 spring_jacobian_configuration(bool parent, bool jac_parent, const JointS& j, int k, const V3& xa, const Quat& qa, const V3& xb,
                                    const Quat& qb) const {
    const Elem& e = j.el[k];
    M66 out;
    if (e.nl == 3) return out;
    const Quat& qj = jac_parent ? qa : qb;
    Mat<3, 7> mc7 = minimal_coordinates_jacobian_configuration(jac_parent, j, k, xa, qa, xb, qb);
    Mat<3, 7> Amc = At_times_full7(e, mc7);  // Aᵀ * ∂θ/∂(x,q)  (3x7)
    Mat<3, 6> Amc6 = hcat(block<3, 3>(Amc, 0, 0), block<3, 4>(Amc, 0, 3) * LVtmat(qj));
    double th[3], dist[3];
    minimal_coordinates(j, k, xa, qa, xb, qb, th);
    for (int i = 0; i < e.nfree; ++i) dist[i] = e.spring_offset[i] - th[i];
    if (k == 0) {
      V3 force = e.spring * At_times(e, dist);
      Mat<6, 6> J1 = impulse_transform(parent, j, 0, xa, qa, xb, qb) * ((-e.spring) * Amc6);
      out = h * (J1 + impulse_transform_jacobian(parent, jac_parent, j, 0, xa, qa, xb, qb, force));
    } else {
      V3 force = -e.spring * At_times(e, dist);  // spring_force(rotate=false) output for :parent; child gets -force
      Mat<3, 6> Jr;
      if (parent) {
        Jr = h * (rotation_matrix(j.qoff) * (e.spring * Amc6));
      } else {
        V3 fchild = -force;
        Quat qrel = inv(qb) * qa * j.qoff;
        Jr = h * (rotation_matrix(qrel) * ((-e.spring) * Amc6));
        M34 Q2;
        if (jac_parent) Q2 = h * (dvector_rotate_dq(fchild, qrel) * Rmat(j.qoff) * Lmat(inv(qb)));
        else Q2 = h * (dvector_rotate_dq(fchild, qrel) * Rmat(qa * j.qoff) * Tmat());
        M33 Q2a = Q2 * LVtmat(qj);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Jr(r, 3 + c) += Q2a(r, c);
      }
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 6; ++c) out(3 + r, c) = Jr(r, c);
    }
    return out;
  }
  // translational/dampers.jl:71-98, rotational/dampers.jl:33-64: 6 x 6
  M66 damper_jacobian_configuration(bool parent, bool jac_parent, const JointS& j, int k, const Cfg& a, const Cfg& b) const {
    const Elem& e = j.el[k];
    M66 out;
    if (e.nl == 3) return out;
    Mat<3, 6> dvel = minimal_velocities_jacobian_configuration(jac_parent, j, k, a, b, h);
    double vel[3];
    if (k == 0) {
      minimal_velocities(j, 0, a, b, h, vel);
      V3 input = -e.damper * At_times(e, vel);
      Mat<3, 6> dinput = (-e.damper) * At_times_full(e, dvel);
      M66 J = impulse_transform(parent, j, 0, a.x, a.q, b.x, b.q) * dinput;
      J += impulse_transform_jacobian(parent, jac_parent, j, 0, a.x, a.q, b.x, b.q, input);
      out = h * J;
    } else {
      Cfg a0 = a, b0 = b;
      a0.x = V3(); a0.v = V3(); b0.x = V3(); b0.v = V3();
      minimal_velocities(j, 1, a0, b0, h, vel);
      V3 force = parent ? e.damper * At_times(e, vel) : -e.damper * At_times(e, vel);  // rotate = false
      M33 dv = At_times_rows(e, dvel, 3);
      M33 Q;
      if (parent) {
        Q = rotation_matrix(j.qoff) * (e.damper * dv);
      } else {
        Q = rotation_matrix(inv(b.q) * a.q * j.qoff) * ((-e.damper) * dv);
        if (jac_parent) Q += rotation_matrix(inv(b.q)) * drotation_matrix_dq(a.q, vector_rotate(force, j.qoff)) * LVtmat(a.q);
        else Q += drotation_matrix_inv_dq(b.q, vector_rotate(force, a.q * j.qoff)) * LVtmat(b.q);
      }
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) out(3 + r, 3 + c) = h * Q(r, c);
    }
    return out;
  }

  // gradients/state.jl:78-126 evaluated at the solution *before* update_state! (SURVEY Q2, consistent IFT).
  // Fz is 12Nb x 12Nb, Fu is 12Nb x nu, both COLUMN-major (Julia layout).
  bool maximal_gradients(double* Fz, double* Fu, bool use_factor) {
    const int m = 12 * Nb + nu, ns = 12 * Nb;
    std::vector<double> D;
    data_jacobian(D);
    bool ok;
    if (use_factor) { ok = factorize() && solve(D.data(), m); }
    else ok = dense_solve(A, nres, D.data(), m);  // solmat \ datamat (state.jl:99)
    if (!ok) return false;
    std::fill(Fz, Fz + (size_t)ns * ns, 0.0);
    std::fill(Fu, Fu + (size_t)ns * nu, 0.0);
    auto out = [&](int row, int col) -> double& { return col < ns ? Fz[(size_t)col * ns + row] : Fu[(size_t)(col - ns) * ns + row]; };
    for (int b = 0; b < Nb; ++b) {
      const BodyS& s = bodies[b];
      int ob = body_off[b];
      Quat q3 = next_orientation(s.q2, s.wsol[1], h);
      M33 Mq = tr(LVtmat(q3)) * rotational_integrator_jacobian_velocity(s.q2, s.wsol[1], h);
      M33 Mqq = tr(LVtmat(q3)) * (rotational_integrator_jacobian_orientation_full(s.wsol[1], h) * LVtmat(s.q2));
      for (int c = 0; c < m; ++c) {
        for (int r = 0; r < 3; ++r) {
          double dv = D[(size_t)(ob + r) * m + c];
          double dw = D[(size_t)(ob + 3 + r) * m + c];
          out(12 * b + 3 + r, c) += dv;
          out(12 * b + 9 + r, c) += dw;
          out(12 * b + r, c) += h * dv;
        }
        for (int r = 0; r < 3; ++r) {
          double acc = 0;
          for (int t = 0; t < 3; ++t) acc += Mq(r, t) * D[(size_t)(ob + 3 + t) * m + c];
          out(12 * b + 6 + r, c) += acc;
        }
      }
      for (int r = 0; r < 3; ++r) {
        out(12 * b + r, 12 * b + r) += 1.0;
        for (int c = 0; c < 3; ++c) out(12 * b + 6 + r, 12 * b + 6 + c) += Mqq(r, c);
      }
    }
    return true;
  }

  // Contact data theta_c = [friction_coefficient; contact_radius; contact_origin(3)] (data_dim = 5, contacts/nonlinear.jl):
  // body rows   body_constraint_jacobian_contact_data     gradients/data.jl:152-171
  // contact rows contact_constraint_jacobian_contact_data gradients/data.jl:173-192
  // D is nres x 5 Ni, row-major.
  void contact_data_jacobian(std::vector<double>& D) const {
    const int m = 5 * Ni;
    D.assign((size_t)nres * m, 0.0);
    for (int ci = 0; ci < Ni; ++ci) {
      const ContactS& c = contacts[ci];
      Cfg p = cfg_next(c.body);  // (x3, v25, q3, w25)
      if (c.type != 2) continue;  // the reference defines the contact-data blocks for NonlinearContact only (gradients/data.jl:152,173)
      Mat<6, 1> gam;
      for (int i = 0; i < 4; ++i) gam[i] = c.gam[1][i];
      Mat<3, 6> X = force_mapping(c);
      V3 Fb = (VRmat(p.q) * LtVtmat(p.q)) * (X * gam);
      M33 dp = -dskew_dp(Fb);                                            // ∇p
      V3 drad = (-dskew_dp(Fb)) * (-(rotation_matrix(inv(p.q)) * tr(c.nrm)));  // ∇contact_radius
      const int ob = body_off[c.body], col0 = 5 * ci;
      for (int r = 0; r < 3; ++r) {  // ∇Q = -[∇friction_coefficient ∇contact_radius ∇p], ∇X = 0
        D[(size_t)(ob + 3 + r) * m + col0 + 1] = -drad[r];
        for (int k = 0; k < 3; ++k) D[(size_t)(ob + 3 + r) * m + col0 + 2 + k] = -dp(r, k);
      }
      V3 ww = vector_rotate(p.w, p.q);
      Mat<4, 3> A43;                       // [-cn; 0; -ct skew(ww)]
      Mat<2, 3> cts = c.t * skew(ww);
      for (int k = 0; k < 3; ++k) { A43(0, k) = -c.nrm[k]; A43(2, k) = -cts(0, k); A43(3, k) = -cts(1, k); }
      Mat<4, 1> g_rad = A43 * tr(c.nrm);
      Mat<4, 3> g_p = (-1.0) * (A43 * rotation_matrix(p.q));   // [cn R; 0; ct skew(ww) R]
      const int oc = c.sol_off + 4;     // rows of g; the complementarity rows get ∇compμ = 0
      D[(size_t)(oc + 1) * m + col0 + 0] = -gam[0];            // -∇friction_coefficient = -[0, γ1, 0, 0]
      for (int r = 0; r < 4; ++r) {
        D[(size_t)(oc + r) * m + col0 + 1] = -g_rad[r];
        for (int k = 0; k < 3; ++k) D[(size_t)(oc + r) * m + col0 + 2 + k] = -g_p(r, k);
      }
    }
  }

  // get_contact_gradients, gradients/contact.jl:1-55 (the jacobian_contact part), consistent variant like maximal_gradients.
  // Fc is 12Nb x 5Ni, COLUMN-major.
  bool contact_gradients(double* Fc, bool use_factor) {
    const int m = 5 * Ni, ns = 12 * Nb;
    std::vector<double> D;
    contact_data_jacobian(D);
    bool ok = true;
    if (m > 0) {
      if (use_factor) ok = factorize() && solve(D.data(), m);
      else ok = dense_solve(A, nres, D.data(), m);
    }
    if (!ok) return false;
    std::fill(Fc, Fc + (size_t)ns * m, 0.0);
    for (int b = 0; b < Nb; ++b) {
      const BodyS& s = bodies[b];
      int ob = body_off[b];
      Quat q3 = next_orientation(s.q2, s.wsol[1], h);
      M33 Mq = tr(LVtmat(q3)) * rotational_integrator_jacobian_velocity(s.q2, s.wsol[1], h);
      for (int c = 0; c < m; ++c) {
        double* o = Fc + (size_t)c * ns + 12 * b;
        for (int r = 0; r < 3; ++r) {
          double dv = D[(size_t)(ob + r) * m + c], dw = D[(size_t)(ob + 3 + r) * m + c];
          o[3 + r] += dv; o[9 + r] += dw; o[r] += h * dv;
        }
        for (int r = 0; r < 3; ++r) {
          double acc = 0;
          for (int t = 0; t < 3; ++t) acc += Mq(r, t) * D[(size_t)(ob + 3 + t) * m + c];
          o[6 + r] += acc;
        }
      }
    }
    return true;
  }

  // ---------------------------------------------------------------- diagnostics (mechanics/momentum.jl:17-86)
  // Momentum of the mechanism evaluated right after mehrotra! (before update_state!), exactly what
  // save_to_storage! records (simulation/storage.jl:50-67).  out6 = [p_linear; p_angular] in the world frame.
  void momentum(double* out6) const {
    std::vector<V3> pl(Nb), pa(Nb);
    for (int bi = 0; bi < Nb; ++bi) {
      const BodyS& s = bodies[bi];
      V3 x3 = next_position(s.x2, s.vsol[1], h);
      Quat q3 = next_orientation(s.q2, s.wsol[1], h);
      V3 D2x = (1.0 / h * s.mass) * (x3 - s.x2) - 0.5 * h * (s.mass * gravity + s.Fext);
      V3 D2q = (-2.0 / h) * (tr(LVtmat(s.q2)) * Tmat() * Rtmat(q3) * Vtmat() * s.J * Vmat() * Ltmat(s.q2) * vector(q3)) - 0.5 * h * s.text;
      V3 p_lin = D2x - 0.5 * s.JF2;
      V3 p_ang = D2q - 0.5 * s.Jt2;
      for (const JointS& j : joints) {
        if (j.parent != bi && j.child != bi) continue;
        bool parent = (j.parent == bi);
        V6 f;
        if (j.n > 0) {
          Mat<6, 24> G;
          joint_impulse_map(j, parent, G);
          for (int r = 0; r < 6; ++r) for (int i = 0; i < j.n; ++i) f[r] += G(r, i) * j.imp[1][i];
        }
        Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
        if (j.spring) for (int k = 0; k < 2; ++k) f += spring_impulses(parent, j, k, a.x, a.q, b.x, b.q, h);
        if (j.damper) for (int k = 0; k < 2; ++k) f += damper_impulses(parent, j, k, a, b, h);
        for (int i = 0; i < 3; ++i) { p_lin[i] -= 0.5 * f[i]; p_ang[i] -= 0.5 * f[3 + i]; }
      }
      pl[bi] = p_lin;
      pa[bi] = vector_rotate(p_ang, s.q2);
    }
    double mass = 0;
    V3 com, P, L;
    for (int bi = 0; bi < Nb; ++bi) { mass += bodies[bi].mass; com += bodies[bi].mass * bodies[bi].x2; P += pl[bi]; }
    com = com / mass;
    V3 vcom = P / mass;
    for (int bi = 0; bi < Nb; ++bi) {
      V3 r = bodies[bi].x2 - com;
      V3 vb = pl[bi] / bodies[bi].mass;
      L += pa[bi] + skew(r) * (bodies[bi].mass * (vb - vcom));
    }
    for (int i = 0; i < 3; ++i) { out6[i] = P[i]; out6[3 + i] = L[i]; }
    last_pl = pl; last_pa = pa;
  }
  mutable std::vector<V3> last_pl, last_pa;

  // save_to_storage! (simulation/storage.jl:50-67) right after mehrotra!: per body [px; pq; vl; wl], and the diagnostics
  // derived from a Storage: momentum (mechanics/momentum.jl:54-74), kinetic_energy (mechanics/energy.jl:32-41),
  // potential_energy (:60-93).  diag = [p_linear(3); p_angular(3); kinetic; potential].
  void storage_record(double* body_out, double* diag) const {
    momentum(diag);
    double ke = 0, pe = 0;
    for (int bi = 0; bi < Nb; ++bi) {
      const BodyS& s = bodies[bi];
      V3 px = last_pl[bi], pq = last_pa[bi];
      V3 vl = px / s.mass;
      V3 rhs = vector_rotate(pq, inv(s.q2));
      double Jm[9], x[3] = {rhs[0], rhs[1], rhs[2]};
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Jm[3 * r + c] = s.J(r, c);
      dense_solve(std::vector<double>(Jm, Jm + 9), 3, x, 1);  // inertia \ (...)
      V3 wl = vec3(x[0], x[1], x[2]);
      double* o = body_out + 12 * bi;
      for (int i = 0; i < 3; ++i) { o[i] = px[i]; o[3 + i] = pq[i]; o[6 + i] = vl[i]; o[9 + i] = wl[i]; }
      ke += 0.5 * s.mass * dot(vl, vl) + 0.5 * dot(wl, s.J * wl);
      pe -= s.mass * dot(gravity, s.x2);
    }
    for (const JointS& j : joints) {
      if (!j.spring) continue;
      for (int k = 0; k < 2; ++k) {
        const Elem& e = j.el[k];
        if (!(e.spring > 0) || e.nl == 3) continue;
        Cfg a = cfg_current(j.parent, 1), b = cfg_current(j.child, 1);
        double th[3], dist[3];
        minimal_coordinates(j, k, a.x, a.q, b.x, b.q, th);
        for (int i = 0; i < e.nfree; ++i) dist[i] = e.spring_offset[i] - th[i];
        V3 force = e.spring * At_times(e, dist);  // |spring_force| (translational/springs.jl:31-52, rotational/springs.jl:40-62)
        pe += 0.5 * dot(force, force) / e.spring;
      }
    }
    diag[6] = ke; diag[7] = pe;
  }
};

}  // namespace dojo_oracle

// ==========================================================================================
// C API (ctypes) -- names are prefixed oracle_ to make it impossible to confuse with the product ABI
// ==========================================================================================
using dojo_oracle::Oracle;

extern "C" {

void* oracle_create(const DojoMechanismDesc* d) { return new Oracle(*d); }
void oracle_destroy(void* h) { delete static_cast<Oracle*>(h); }
int oracle_num_residual(void* h) { return static_cast<Oracle*>(h)->nres; }
int oracle_num_input(void* h) { return static_cast<Oracle*>(h)->nu; }
int oracle_is_tree(void* h) { return static_cast<Oracle*>(h)->tree_ok ? 1 : 0; }
void oracle_set_solver_mode(void* h, int mode) { static_cast<Oracle*>(h)->solver_mode = mode; }
void oracle_set_force_iters(void* h, int n) { static_cast<Oracle*>(h)->force_iters = n; }
void oracle_elimination_order(void* h, int32_t* out) {
  Oracle* o = static_cast<Oracle*>(h);
  for (size_t i = 0; i < o->elim_order.size(); ++i) out[i] = o->elim_order[i];
}

int oracle_step(void* h, const DojoSolverOptions* opts, const double* z, const double* u, const double* fext, double* z_next, double* sol,
                int32_t* iters, uint32_t flags) {
  int it = 0;
  int st = static_cast<Oracle*>(h)->step(*opts, z, u, fext, z_next, sol, &it, flags);
  if (iters) *iters = it;
  return st;
}
// batched convenience (serial loop over environments; column-major [feature x B])
void oracle_step_batch(void* h, const DojoSolverOptions* opts, int B, const double* Z, const double* U, const double* Fext, double* Zn,
                       double* sol, int32_t* status, int32_t* iters, uint32_t flags) {
  Oracle* o = static_cast<Oracle*>(h);
  int nz = 13 * o->Nb;
  for (int e = 0; e < B; ++e) {
    int it = 0;
    int st = o->step(*opts, Z + (size_t)e * nz, U + (size_t)e * o->nu, Fext ? Fext + (size_t)e * 6 * o->Nb : nullptr, Zn + (size_t)e * nz,
                     sol ? sol + (size_t)e * o->nres : nullptr, &it, flags);
    if (status) status[e] = st;
    if (iters) iters[e] = it;
  }
}
// multi-threaded batch: `nthreads` independent mechanism instances (the reference is single-threaded per Mechanism), each
// stepping a contiguous slice of the batch; returns nothing but the outputs.  Used by bench.py as the CPU baseline.
void oracle_step_batch_threads(const DojoMechanismDesc* d, const DojoSolverOptions* opts, int B, const double* Z, const double* U, double* Zn,
                               int32_t* status, int32_t* iters, int nthreads) {
  nthreads = std::max(1, std::min(nthreads, B));
  std::vector<std::thread> pool;
  for (int t = 0; t < nthreads; ++t) {
    pool.emplace_back([=]() {
      Oracle o(*d);
      int lo = (int)((long long)B * t / nthreads), hi = (int)((long long)B * (t + 1) / nthreads);
      int nz = 13 * o.Nb;
      for (int e = lo; e < hi; ++e) {
        int it = 0;
        int st = o.step(*opts, Z + (size_t)e * nz, U + (size_t)e * o.nu, nullptr, Zn + (size_t)e * nz, nullptr, &it, 0);
        if (status) status[e] = st;
        if (iters) iters[e] = it;
      }
    });
  }
  for (auto& th : pool) th.join();
}
// step! + get_maximal_gradients for a batch on `nthreads` threads (bench.py --impl reference --mode grad).  Fz / Fu may be null: the
// Jacobians are then computed into per-thread scratch and dropped (12Nb x 12Nb doubles per environment do not fit a host buffer at
// benchmark batch sizes); use_factor selects the block-LDU back-solve instead of the reference's dense solmat \ datamat.
void oracle_step_grad_batch_threads(const DojoMechanismDesc* d, const DojoSolverOptions* opts, int B, const double* Z, const double* U, double* Zn,
                                    double* Fz, double* Fu, int32_t* status, int32_t* iters, int nthreads, int use_factor, uint32_t flags) {
  nthreads = std::max(1, std::min(nthreads, B));
  std::vector<std::thread> pool;
  for (int t = 0; t < nthreads; ++t) {
    pool.emplace_back([=]() {
      Oracle o(*d);
      int lo = (int)((long long)B * t / nthreads), hi = (int)((long long)B * (t + 1) / nthreads);
      const int nz = 13 * o.Nb;
      const size_t ns = 12 * (size_t)o.Nb;
      std::vector<double> fz(ns * ns), fu(ns * (size_t)o.nu);
      for (int e = lo; e < hi; ++e) {
        int it = 0;
        int st = o.step(*opts, Z + (size_t)e * nz, U + (size_t)e * o.nu, nullptr, Zn + (size_t)e * nz, nullptr, &it, flags);
        if (flags & DOJO_FLAG_Q2_LITERAL_GRADIENTS) o.update_state();
        o.grad_flags = flags;
        double* pz = Fz ? Fz + (size_t)e * ns * ns : fz.data();
        double* pu = Fu ? Fu + (size_t)e * ns * o.nu : fu.data();
        if (!o.maximal_gradients(pz, pu, use_factor != 0) && st == 0) st = DOJO_STATUS_NONFINITE;
        if (status) status[e] = st;
        if (iters) iters[e] = it;
      }
    });
  }
  for (auto& th : pool) th.join();
}
int oracle_step_grad(void* h, const DojoSolverOptions* opts, const double* z, const double* u, const double* fext, double* z_next,
                     double* Fz, double* Fu, int32_t* iters, uint32_t flags, int use_factor) {
  Oracle* o = static_cast<Oracle*>(h);
  int it = 0;
  int st = o->step(*opts, z, u, fext, z_next, nullptr, &it, flags);
  if (iters) *iters = it;
  // DOJO_FLAG_Q2_LITERAL_GRADIENTS: get_maximal_gradients! = step! (incl. update_state!) THEN get_maximal_gradients (gradients/state.jl:69-76);
  // the KKT matrix `A` keeps the entries of the last set_entries! (the unshifted final iterate, solver/mehrotra.jl:66-69)
  if (flags & DOJO_FLAG_Q2_LITERAL_GRADIENTS) o->update_state();
  o->grad_flags = flags;
  if (!o->maximal_gradients(Fz, Fu, use_factor != 0)) return DOJO_STATUS_NONFINITE;
  return st;
}
void oracle_contact_data_jacobian(void* h, double* out) {  // nres x 5Ni row-major
  std::vector<double> D;
  static_cast<Oracle*>(h)->contact_data_jacobian(D);
  std::memcpy(out, D.data(), D.size() * sizeof(double));
}
int oracle_contact_gradients(void* h, double* Fc, int use_factor) { return static_cast<Oracle*>(h)->contact_gradients(Fc, use_factor != 0) ? 0 : 1; }
// --- pieces exposed for the property tests -------------------------------------------------
void oracle_set_state(void* h, const double* z, const double* u, const double* fext) {
  Oracle* o = static_cast<Oracle*>(h);
  o->set_maximal_state(z); o->set_external(fext); o->set_input(u);
}
void oracle_set_solution(void* h, const double* sol, double mu) { Oracle* o = static_cast<Oracle*>(h); o->set_solution(sol); o->mu = mu; }
void oracle_get_solution(void* h, double* sol) { static_cast<Oracle*>(h)->get_solution(sol); }
void oracle_reset_solution(void* h) {  // reset! + initialize! as at the top of mehrotra!
  Oracle* o = static_cast<Oracle*>(h);
  DojoSolverOptions opts; std::memset(&opts, 0, sizeof(opts)); opts.max_iter = 0; opts.undercut = 1;
  int it; o->mehrotra(opts, &it);
}
// assemble: A (nres x nres, row-major) and rhs at the current solution with mechanism.μ = mu
void oracle_assemble(void* h, double mu, double* A, double* rhs) {
  Oracle* o = static_cast<Oracle*>(h);
  o->mu = mu; o->set_entries();
  if (A) std::memcpy(A, o->A.data(), sizeof(double) * o->A.size());
  if (rhs) std::memcpy(rhs, o->rhs.data(), sizeof(double) * o->rhs.size());
}
void oracle_evaluate_rhs(void* h, const double* sol, double mu, double* out) {
  Oracle* o = static_cast<Oracle*>(h);
  o->set_solution(sol); o->mu = mu; o->evaluate_rhs(out);
}
void oracle_violations(void* h, double* rvio, double* bvio) {
  Oracle* o = static_cast<Oracle*>(h);
  *rvio = o->residual_violation(); *bvio = o->bilinear_violation();
}
// solve A x = b with the current assembled matrix; mode 0 block LDU, 1 dense LU
int oracle_linear_solve(void* h, int mode, double* x, int m) {
  Oracle* o = static_cast<Oracle*>(h);
  int old = o->solver_mode; o->solver_mode = mode;
  bool ok = o->factorize() && o->solve(x, m);
  o->solver_mode = old;
  return ok ? 0 : -1;
}
void oracle_data_jacobian(void* h, double* out, uint32_t flags) {  // nres x (12Nb + nu) row-major
  Oracle* o = static_cast<Oracle*>(h);
  o->grad_flags = flags;
  std::vector<double> D; o->data_jacobian(D);
  std::memcpy(out, D.data(), sizeof(double) * D.size());
}
int oracle_trace(void* h, double* out, int cap) {  // rows of (rvio, bvio, alpha, mu)
  Oracle* o = static_cast<Oracle*>(h);
  int n = std::min<int>(cap, (int)o->trace.size());
  std::memcpy(out, o->trace.data(), sizeof(double) * n);
  return (int)o->trace.size() / 4;
}
int oracle_num_minimal(void* h) { return 2 * static_cast<Oracle*>(h)->nu; }
void oracle_minimal_to_maximal(void* h, const double* x, double* z) { static_cast<Oracle*>(h)->minimal_to_maximal(x, z); }
void oracle_maximal_to_minimal(void* h, const double* z, double* x) { static_cast<Oracle*>(h)->maximal_to_minimal(z, x); }
void oracle_maximal_to_minimal_jacobian(void* h, const double* z, double* J) { static_cast<Oracle*>(h)->maximal_to_minimal_jacobian(z, J); }
void oracle_minimal_to_maximal_jacobian(void* h, const double* z, double* J, int body_order_literal) {
  static_cast<Oracle*>(h)->minimal_to_maximal_jacobian(z, J, body_order_literal != 0);
}
void oracle_momentum(void* h, double* out6) { static_cast<Oracle*>(h)->momentum(out6); }
void oracle_storage_record(void* h, double* body_out, double* diag) { static_cast<Oracle*>(h)->storage_record(body_out, diag); }
}
