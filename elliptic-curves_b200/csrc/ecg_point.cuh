// ecg_point.cuh — Jacobian point arithmetic over a field policy F (FpK256 / FpP256).
//
// Replaces (same group law, different coordinates) the reference's homogeneous-projective complete
// formulas: k256/src/arithmetic/projective.rs:96-131 (add), :142-176 (add_mixed), :189-217 (double)
// and primeorder/src/point_arithmetic.rs:222-245, :254-280, :289-318 for a = -3.
// Affine results are canonical, so any coordinate system gives bit-identical output after
// normalisation (the reference itself only compares after to_affine, SURVEY.md fact 3).
//
// Conventions: a Jacobian point (X:Y:Z) is (X/Z^2, Y/Z^3); Z == 0 (mod p) is the identity.
// Jacobian formulas are incomplete, so every exceptional case (identity operands, P == Q, P == -Q) is
// detected and routed through a slow path; in the windowed loops they are unreachable for honest
// inputs (a warp-uniform not-taken branch), but adversarial inputs must still give exact results.
#pragma once
#include "ecg_prim.cuh"

namespace ecg {

// JacN / AffN live in ecg_prim.cuh; the 8-limb names are kept for the secp256k1-only code.  The templates below take
// their types from the field policy (F::FeT, F::JacT, F::AffT), so the same formulas serve 8- and 12-limb fields.
typedef JacN<8> Jac;
typedef AffN<8> Aff;

// a = c ? -a : a  (branch-free: lanes of a warp disagree on c)
template <class F>
ECG_D void fe_cneg(typename F::FeT& a, uint32_t c) {
  typename F::FeT n;
  F::neg(n, a);
#pragma unroll
  for (int i = 0; i < F::NL; i++) a.v[i] = c ? n.v[i] : a.v[i];
}
// r = c ? t : r
template <int NL>
ECG_D void jac_csel(JacN<NL>& r, const JacN<NL>& t, uint32_t c) {
#pragma unroll
  for (int i = 0; i < NL; i++) {
    r.X.v[i] = c ? t.X.v[i] : r.X.v[i];
    r.Y.v[i] = c ? t.Y.v[i] : r.Y.v[i];
    r.Z.v[i] = c ? t.Z.v[i] : r.Z.v[i];
  }
}

// The curve coefficient a is a template mode (named A_IS_MINUS3 for its first two values): 0: a = 0, 1: a = -3
// (EquationAIsMinusThree, primeorder/src/point_arithmetic.rs:212-319), 2: any a, read from F::curve_a
// (EquationAIsGeneric, primeorder/src/point_arithmetic.rs:54-208: brainpoolP256r1 / P384r1, bign-curve256v1).
// Doubling in "halved" form (Z3 = Y*Z, X3 = X3_std/4, Y3 = Y3_std/8): 3M+4S (a=0; 2M+5S with F::SQR_TRADE_DBL) / 4M+4S (a=-3) / 4M+6S (general a),
// 8 cheap linear ops.   L = (3X^2 + a Z^4)/2;  X3 = L^2 - 2XY^2;  Y3 = L(XY^2 - X3) - Y^4.
template <class F, int A_IS_MINUS3>
ECG_D void jac_dbl_body(typename F::JacT& r, const typename F::JacT& p) {
  typedef typename F::FeT Fe;
  Fe A, L, T, D, t, zz;
  F::sqr(A, p.Y);  // Y^2
  if (A_IS_MINUS3 == 1) {
    Fe u, v;
    F::sqr(zz, p.Z);
    F::sub(u, p.X, zz);
    F::add(v, p.X, zz);
    F::mul_d(L, u, v);  // X^2 - Z^4
  } else {
    F::sqr(L, p.X);
  }
  // with F::MUL_SUB, Y^4 is only needed as the subtrahend of Y3, and mul_sub_sqr forms it unreduced there
  constexpr bool Y3_MUL_SUB = A_IS_MINUS3 == 0 && F::MUL_SUB && !F::SQR_TRADE_DBL;
  if constexpr (!Y3_MUL_SUB) F::sqr(D, A);  // Y^4
  if (A_IS_MINUS3 == 0 && F::SQR_TRADE_DBL) {
    // X*Y^2 = ((X + Y^2)^2 - X^2 - Y^4)/2: a squaring (36 products) plus four linear ops instead of a multiplication (64)
    F::add(t, p.X, A);
    F::sqr(T, t);
    F::sub(T, T, L);
    F::sub(T, T, D);
    F::half(T, T);
  } else {
    F::mul_d(T, p.X, A);  // X*Y^2
  }
  if constexpr (A_IS_MINUS3 == 0 && F::HALF3_ADD) {  // 3/2 X^2 = X^2 + X^2/2, no multiplier
    F::half(t, L);
    F::add(L, L, t);
  } else {
    F::mul_small(L, L, 3);
    if constexpr (A_IS_MINUS3 == 2) {  // general a (the field policy of such a curve carries it): L = (3 X^2 + a Z^4) / 2
      Fe z4, ca;
      F::sqr(zz, p.Z);
      F::sqr(z4, zz);
      F::curve_a(ca);
      F::mul_d(z4, z4, ca);
      F::add(L, L, z4);
    }
    F::half(L, L);
  }
  if (A_IS_MINUS3 == 1 && F::DBL_3M5S) {  // Y*Z = ((Y+Z)^2 - Y^2 - Z^2)/2 ; zz was computed for L
    Fe s2;
    F::add(s2, p.Y, p.Z);
    F::sqr(s2, s2);
    F::sub(s2, s2, A);
    F::sub(s2, s2, zz);
    F::half(r.Z, s2);
  } else {
    F::mul_d(r.Z, p.Y, p.Z);
  }
  F::sqr(r.X, L);
  F::add(t, T, T);
  F::sub(r.X, r.X, t);
  F::sub(t, T, r.X);
  if constexpr (Y3_MUL_SUB) {
    F::mul_sub_sqr(r.Y, L, t, A);  // L (T - X3) - (Y^2)^2
  } else {
    F::mul_d(r.Y, L, t);
    F::sub(r.Y, r.Y, D);
  }
}

#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define ECG_NOINLINE_PT __device__ __noinline__
#else
#define ECG_NOINLINE_PT
#endif
template <class F, int A_IS_MINUS3>
ECG_NOINLINE_PT typename F::JacT jac_dbl_call(typename F::JacT p) {
  typename F::JacT r;
  jac_dbl_body<typename F::Inline, A_IS_MINUS3>(r, p);
  return r;
}
template <class F, int A_IS_MINUS3>
ECG_D void jac_dbl(typename F::JacT& r, const typename F::JacT& p) {
  if (F::DBL_CALL)
    r = jac_dbl_call<F, A_IS_MINUS3>(p);
  else
    jac_dbl_body<F, A_IS_MINUS3>(r, p);
}

// 2*(x,y) for an affine input (Z = 1): saves the Z products.
template <class F, int A_IS_MINUS3>
ECG_D void aff_dbl(typename F::JacT& r, const typename F::AffT& p) {
  typename F::JacT j;
  j.X = p.x;
  j.Y = p.y;
  F::set_one(j.Z);  // internal-form one
  jac_dbl<F, A_IS_MINUS3>(r, j);
}

// Slow path of mixed addition: identity accumulator, or H == 0.
template <class F, int A_IS_MINUS3>
#if defined(__CUDA_ARCH__)
__device__ __noinline__
#else
inline
#endif
    void
    jac_madd_slow(typename F::JacT& r, const typename F::JacT& p, const typename F::AffT& q, bool z1zero, bool rzero) {
  if (z1zero) {  // O + Q = Q
    r.X = q.x;
    r.Y = q.y;
    F::set_one(r.Z);
  } else if (rzero) {  // P == Q
    aff_dbl<F, A_IS_MINUS3>(r, q);
  } else {  // P == -Q
    F::set_zero(r.X);
    F::set_one(r.Y);
    F::set_zero(r.Z);
  }
}

// r = p + q, q affine and not the identity.  8M+3S (7M+4S with F::SQR_TRADE_MADD).  If zr != nullptr it receives Z3/Z1 (= H).
template <class F, int A_IS_MINUS3>
ECG_D void jac_madd_body(typename F::JacT& r, const typename F::JacT& p, const typename F::AffT& q, typename F::FeT* zr = nullptr) {
  typedef typename F::FeT Fe;
  Fe zz, u2, s2, H, R, hh, hhh, V, t;
  F::sqr(zz, p.Z);
  F::mul(u2, q.x, zz);
  F::mul(s2, p.Z, zz);
  F::mul(s2, s2, q.y);
  F::sub(H, u2, p.X);
  F::sub(R, s2, p.Y);
  bool z1zero = F::is_zero(p.Z);
  bool hzero = F::is_zero(H);
  if (z1zero | hzero) {
    jac_madd_slow<F, A_IS_MINUS3>(r, p, q, z1zero, F::is_zero(R));
    if (zr) F::set_zero(*zr);
    return;
  }
  F::sqr(hh, H);
  F::mul(hhh, H, hh);
  F::mul(V, p.X, hh);
  if (F::SQR_TRADE_MADD) {  // Z1*H = ((Z1 + H)^2 - Z1^2 - H^2)/2
    F::add(t, p.Z, H);
    F::sqr(t, t);
    F::sub(t, t, zz);
    F::sub(t, t, hh);
    F::half(r.Z, t);
  } else {
    F::mul(r.Z, p.Z, H);
  }
  if (zr) *zr = H;
  F::sqr(t, R);
  F::sub(t, t, hhh);
  F::sub(t, t, V);
  F::sub(r.X, t, V);
  F::sub(t, V, r.X);
  if constexpr (F::MUL_SUB) {
    F::mul_sub(r.Y, t, R, hhh, p.Y);  // (V - X3) R - H^3 Y1
  } else {
    F::mul(t, t, R);
    F::mul(hhh, hhh, p.Y);
    F::sub(r.Y, t, hhh);
  }
}

template <class F, int A_IS_MINUS3>
ECG_NOINLINE_PT typename F::JacT jac_madd_call(typename F::JacT p, typename F::AffT q) {
  typename F::JacT r;
  jac_madd_body<typename F::Inline, A_IS_MINUS3>(r, p, q, nullptr);
  return r;
}
template <class F, int A_IS_MINUS3>
ECG_D void jac_madd(typename F::JacT& r, const typename F::JacT& p, const typename F::AffT& q, typename F::FeT* zr = nullptr) {
  if (F::MADD_CALL && zr == nullptr)
    r = jac_madd_call<F, A_IS_MINUS3>(p, q);
  else
    jac_madd_body<F, A_IS_MINUS3>(r, p, q, zr);
}

// r = p + q, both Jacobian.  12M+4S.
template <class F, int A_IS_MINUS3>
ECG_D void jac_add(typename F::JacT& r, const typename F::JacT& p, const typename F::JacT& q) {
  typedef typename F::FeT Fe;
  bool z1zero = F::is_zero(p.Z), z2zero = F::is_zero(q.Z);
  if (z1zero) {
    r = q;
    return;
  }
  if (z2zero) {
    r = p;
    return;
  }
  Fe z1z1, z2z2, u1, u2, s1, s2, H, R, hh, hhh, V, t;
  F::sqr(z1z1, p.Z);
  F::sqr(z2z2, q.Z);
  F::mul(u1, p.X, z2z2);
  F::mul(u2, q.X, z1z1);
  F::mul(s1, q.Z, z2z2);
  F::mul(s1, s1, p.Y);
  F::mul(s2, p.Z, z1z1);
  F::mul(s2, s2, q.Y);
  F::sub(H, u2, u1);
  F::sub(R, s2, s1);
  if (F::is_zero(H)) {
    if (F::is_zero(R)) {
      jac_dbl<F, A_IS_MINUS3>(r, p);
    } else {
      F::set_zero(r.X);
      F::set_one(r.Y);
      F::set_zero(r.Z);
    }
    return;
  }
  F::sqr(hh, H);
  F::mul(hhh, H, hh);
  F::mul(V, u1, hh);
  F::mul(t, p.Z, q.Z);
  F::mul(r.Z, t, H);
  F::sqr(t, R);
  F::sub(t, t, hhh);
  F::sub(t, t, V);
  F::sub(r.X, t, V);
  F::sub(t, V, r.X);
  F::mul(t, t, R);
  F::mul(hhh, hhh, s1);
  F::sub(r.Y, t, hhh);
}

// y^2 == x^3 + a x + b ?   (AffinePoint::from_coordinates on-curve check, k256/src/arithmetic/affine.rs:134-147)
template <class F, int A_IS_MINUS3>
ECG_D bool aff_on_curve(const typename F::AffT& p, const typename F::FeT& b_internal) {
  typedef typename F::FeT Fe;
  Fe l, r, t;
  F::sqr(l, p.y);
  F::sqr(r, p.x);
  F::mul(r, r, p.x);
  if (A_IS_MINUS3 == 1) {
    F::mul_small(t, p.x, 3);
    F::sub(r, r, t);
  } else if constexpr (A_IS_MINUS3 == 2) {
    Fe ca;
    F::curve_a(ca);
    F::mul(t, p.x, ca);
    F::add(r, r, t);
  }
  F::add(r, r, b_internal);
  F::sub(l, l, r);
  return F::is_zero(l);
}

}  // namespace ecg
