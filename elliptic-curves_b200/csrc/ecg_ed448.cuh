// ecg_ed448.cuh — Ed448 signature verification (RFC 8032 section 5.2.7) over a batch: one thread per signature, the
// Edwards group of ed448-goldilocks on the Curve448 field (ecg_fe_p448.cuh), SHAKE256 from ecg_keccak.cuh.
//
// The contract is the reference's VerifyingKey::from_bytes + verify_inner (ed448-goldilocks/src/sign/verifying_key.rs:
// 187-198, 264-312), verdict for verdict:
//   - S = bytes 57..113 of the signature: byte 56 of S must be 0, S < ell (EdwardsScalar::from_canonical_bytes,
//     edwards/scalar.rs:32-42) and S != 0;
//   - A (the public key) and R (bytes 0..56) decompress as CompressedEdwardsY::decompress (edwards/affine.rs:487-520):
//     y = bytes 0..55 little-endian reduced mod p (y >= p is accepted), the sign of x is bit 7 of byte 56 (bits 0-6 are
//     ignored), x = sqrt((1 - y^2) / (1 - d y^2)) or refusal, and the point must lie in the prime-order subgroup;
//     neither may be the identity;
//   - k = SHAKE256(dom4 || R bytes || A bytes || M, 114) mod ell over the bytes as given (not re-encoded), and
//     [S]B == R + [k]A.
// Everything here is public data (the reference: "not constant-time; it assumes that the public key and signature
// value are public data"), so the code branches on it freely.
//
// Group: a x^2 + y^2 = 1 + d x^2 y^2 with a = 1, d = -39081, in extended coordinates (X : Y : Z : T), T = XY/Z.  d is
// not a square, so the unified addition (Hisil-Wong-Carter-Dawson 2008, "add-2008-hwcd") is complete: no exceptional
// case, no slow path.  Doubling is "dbl-2008-hwcd" (4 M + 4 S; 3 M + 4 S when T is not needed next).
//
// Subgroup test (any method giving the reference's predicate is allowed; the reference uses eprint 2022/1164).  Here
// it is a statement about y alone, as P and -P share it.  E(F_p) = Z/ell x Z/4, so P is in the prime-order subgroup
// iff P lies in 4E.  For y^2 != 1: (i) P lies in 2E iff (1 - d)(1 - d y^2) is a square (2-descent on the birationally
// equivalent Montgomery curve, whose only rational 2-torsion point is (0, 0)); (ii) solving 2Q = P for t = y_Q^2 gives a
// quadratic whose roots are t = num / den with den = d (1 - y^2), num = (N + r)(1 - y) + y den, N = 1 - d y^2 and
// r = +-sqrt((1 - d) N); Q lies in 2E iff t (1 - d t) is not a square, for either root.  So: one square root and one
// quadratic character.  tests/ed448_model.py states it (torsion_free_fast) and the tests compare it with [ell]P == O.
// For y^2 = 1 the point is the identity (refused) or (0, -1) (not in the subgroup): refused either way.
//
// Double scalar multiplication: [S]B + [k](-A), compared with R projectively (no inversion).  Both scalars are made odd
// by adding ell where needed (B and A lie in the prime-order subgroup, so the point does not change) and recoded into
// signed odd digits of fixed width (every window adds, so a warp's threads run the same instruction stream): 4 bits
// for -A from a per-thread table of 8 odd multiples, 7 bits for B from the generated table of 64 odd multiples
// (ecg_ed448_consts.cuh, tools/gen_ed448_consts.py).  444 doublings, 112 + 64 additions.
#pragma once
#include "ecg_ed448_consts.cuh"
#include "ecg_fe_p448.cuh"
#include "ecg_keccak.cuh"

namespace ecg {

// Shipped variant and launch geometry of ed448_verify_kernel (DESIGN.md section 7, "Ed448 verification"): the
// call-based field (mul / sqr as device functions), 128 threads per block, 2 blocks per SM (at 3, ptxas spills).
#ifndef ECG_ED448_OPT
#define ECG_ED448_OPT 2
#endif
#define ED448_BLOCK 128
#ifndef ED448_MINBLK
#define ED448_MINBLK 2
#endif
#define ED448_AW 4    // digit width of the A scalar
#define ED448_AND 112  // its digit count: ceil(447 / 4)
#define ED448_BND 64   // digit count of the B scalar: ceil(447 / ED448_BW)
typedef FpP448T<ECG_ED448_OPT> FpEd448;

static constexpr uint32_t ED448_MINUS_D = 39081;  // d = -39081

template <class F>
struct EdPt {
  typename F::Fe X, Y, Z, T;
};

// a 14-word little-endian integer from 56 bytes (any alignment)
ECG_D void ed448_load56(uint32_t* w, const uint8_t* b) {
#pragma unroll
  for (int i = 0; i < 14; i++)
    w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}

// ---- field helpers ----------------------------------------------------------------------------------------------------
template <class F>
ECG_D void ed_mul_d(typename F::Fe& r, const typename F::Fe& a) {  // r = d a
  F::mul_small(r, a, ED448_MINUS_D);
  F::neg(r, r);
}
template <class F>
ECG_D bool ed_eq(const typename F::Fe& a, const typename F::Fe& b) {
  typename F::Fe x, y;
  F::normalize(x, a);
  F::normalize(y, b);
  uint32_t diff = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) diff |= x.v[i] ^ y.v[i];
  return diff == 0;
}
template <class F>
ECG_D bool ed_is_zero(const typename F::Fe& a) {
  typename F::Fe z;
  F::set_zero(z);
  return ed_eq<F>(a, z);
}
template <class F>
ECG_D bool ed_is_minus_one(const typename F::Fe& a) {  // a == p - 1, the value of a non-square's quadratic character
  typename F::Fe m;
  F::set_one(m);
  F::neg(m, m);
  return ed_eq<F>(a, m);
}
// x222 = a^(2^222 - 1), x223 = a^(2^223 - 1): the common head of the three exponentiations below (228 S + 11 M)
template <class F>
ECG_D void ed_pow_head(typename F::Fe& x222, typename F::Fe& x223, const typename F::Fe& a) {
  typename F::Fe x3, x6, x24, x30, t;
  F::sqr(t, a);
  F::mul(t, t, a);  // x2
  F::sqr(x3, t);
  F::mul(x3, x3, a);
  F::sqr_n(x6, x3, 3);
  F::mul(x6, x6, x3);
  F::sqr_n(t, x6, 6);
  F::mul(t, t, x6);  // x12
  F::sqr_n(x24, t, 12);
  F::mul(x24, x24, t);
  F::sqr_n(x30, x24, 6);
  F::mul(x30, x30, x6);
  F::sqr_n(t, x24, 24);
  F::mul(t, t, x24);  // x48
  F::sqr_n(x6, t, 48);
  F::mul(t, x6, t);  // x96
  F::sqr_n(x6, t, 96);
  F::mul(t, x6, t);  // x192
  F::sqr_n(t, t, 30);
  F::mul(x222, t, x30);
  F::sqr(x223, x222);
  F::mul(x223, x223, a);
}
// a^((p - 3) / 4), (p - 3) / 4 = [223 ones][0][222 ones]
template <class F>
ECG_D void ed_pow_p34(typename F::Fe& r, const typename F::Fe& a) {
  typename F::Fe x222, x223;
  ed_pow_head<F>(x222, x223, a);
  F::sqr_n(r, x223, 223);
  F::mul(r, r, x222);
}
// a^((p + 1) / 4) = [224 ones][222 zeros]: the square root of a square
template <class F>
ECG_D void ed_pow_sqrt(typename F::Fe& r, const typename F::Fe& a) {
  typename F::Fe x222, x223;
  ed_pow_head<F>(x222, x223, a);
  F::sqr(r, x223);
  F::mul(r, r, a);
  F::sqr_n(r, r, 222);
}
// a^((p - 1) / 2) = [223 ones][0][223 ones]: 1 for a non-zero square, p - 1 for a non-square, 0 for 0
template <class F>
ECG_D void ed_pow_chi(typename F::Fe& r, const typename F::Fe& a) {
  typename F::Fe x222, x223;
  ed_pow_head<F>(x222, x223, a);
  F::sqr_n(r, x223, 224);
  F::mul(r, r, x223);
}

// ---- decompression and the subgroup test -------------------------------------------------------------------------------
// CompressedEdwardsY::decompress_unchecked: x, y (canonical) of a 57-byte encoding; returns 1 when x exists
template <class F>
ECG_D uint32_t ed448_decode(typename F::Fe& x, typename F::Fe& y, const uint8_t* b57) {
  typedef typename F::Fe Fe;
  ed448_load56(y.v, b57);
  F::normalize(y, y);  // y mod p: encodings of y >= p are accepted
  const uint32_t sign = b57[56] >> 7;  // bits 0-6 of byte 56 are ignored
  Fe yy, u, v, w, t;
  F::sqr(yy, y);
  F::set_one(t);
  F::sub(u, t, yy);                     // u = 1 - y^2
  F::mul_small(v, yy, ED448_MINUS_D);
  F::add(v, v, t);                      // v = 1 - d y^2 (never 0: 1/d is not a square)
  // x = u v (u v^3)^((p - 3) / 4); a square root of u / v iff v x^2 == u
  F::sqr(t, v);
  F::mul(w, u, v);
  F::mul(t, t, w);                      // u v^3
  ed_pow_p34<F>(t, t);
  F::mul(x, w, t);
  F::normalize(x, x);
  F::sqr(t, x);
  F::mul(t, t, v);
  const uint32_t ok = ed_eq<F>(t, u) ? 1u : 0u;
  if ((x.v[0] & 1u) != sign) {
    F::neg(x, x);
    F::normalize(x, x);
  }
  return ok;
}
// the point with this y lies in the prime-order subgroup and is not the identity (see the header comment)
template <class F>
ECG_D uint32_t ed448_subgroup_not_identity(const typename F::Fe& y) {
  typedef typename F::Fe Fe;
  Fe one, u, n, rr, r, t, den, num;
  F::set_one(one);
  F::sqr(t, y);
  F::sub(u, one, t);                    // 1 - y^2
  if (ed_is_zero<F>(u)) return 0;       // the identity or (0, -1)
  F::mul_small(n, t, ED448_MINUS_D);
  F::add(n, n, one);                    // N = 1 - d y^2
  F::mul_small(rr, n, ED448_MINUS_D + 1);  // (1 - d) N
  ed_pow_sqrt<F>(r, rr);
  F::sqr(t, r);
  if (!ed_eq<F>(t, rr)) return 0;       // P is not in 2E
  ed_mul_d<F>(den, u);                  // den = d (1 - y^2)
  F::add(t, n, r);
  F::sub(num, one, y);
  F::mul(num, t, num);
  F::mul(t, y, den);
  F::add(num, num, t);                  // num = (N + r)(1 - y) + y den
  ed_mul_d<F>(t, num);
  F::sub(t, den, t);                    // den - d num
  F::mul(t, num, t);
  ed_pow_chi<F>(t, t);
  return ed_is_minus_one<F>(t) ? 1u : 0u;
}
// CompressedEdwardsY::decompress followed by the identity refusal of verify_inner: 1 iff the encoding is accepted
template <class F>
ECG_D uint32_t ed448_decompress(typename F::Fe& x, typename F::Fe& y, const uint8_t* b57) {
  if (!ed448_decode<F>(x, y, b57)) return 0;
  return ed448_subgroup_not_identity<F>(y);
}

// ---- scalars mod ell ---------------------------------------------------------------------------------------------------
// s57 is accepted as S: byte 56 zero, 0 < S < ell
ECG_D uint32_t ed448_s_ok(const uint8_t* s57) {
  uint32_t s[14];
  ed448_load56(s, s57);
  uint32_t borrow = 0, nz = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    const uint64_t d = (uint64_t)s[i] - ED448_L[i] - borrow;
    borrow = (uint32_t)(d >> 63);
    nz |= s[i];
  }
  return (s57[56] == 0 && borrow && nz) ? 1u : 0u;
}
// r = h mod ell for a 114-byte little-endian h (EdwardsScalar::from_bytes_mod_order_wide): ell = 2^446 - c, so
// x = lo + 2^446 hi == lo + c hi.  Six folds take 912 bits below 2^446 (912 -> 691 -> 470 -> 448 -> 447 -> 446 bits),
// one conditional subtraction of ell finishes.
#if defined(__CUDACC__)
__device__ __noinline__
#else
inline
#endif
void ed448_mod_l_wide(uint32_t* r, const uint8_t* h) {
  uint32_t x[31];
#pragma unroll 1
  for (int i = 0; i < 31; i++) x[i] = 0;
#pragma unroll 1
  for (int i = 0; i < 114; i++) x[i >> 2] |= (uint32_t)h[i] << (8 * (i & 3));
#pragma unroll 1
  for (int it = 0; it < 6; it++) {
    uint32_t hi[17];
#pragma unroll 1
    for (int j = 0; j < 17; j++) hi[j] = (x[13 + j] >> 30) | (x[14 + j] << 2);
    x[13] &= 0x3FFFFFFFu;
#pragma unroll 1
    for (int j = 14; j < 31; j++) x[j] = 0;
#pragma unroll 1
    for (int i = 0; i < 17; i++) {
      uint64_t carry = 0;
#pragma unroll 1
      for (int j = 0; j < 7; j++) {
        const uint64_t t = (uint64_t)hi[i] * ED448_C[j] + x[i + j] + carry;
        x[i + j] = (uint32_t)t;
        carry = t >> 32;
      }
#pragma unroll 1
      for (int j = i + 7; j < 31 && carry; j++) {
        const uint64_t t = (uint64_t)x[j] + carry;
        x[j] = (uint32_t)t;
        carry = t >> 32;
      }
    }
  }
  // x < 2^446 < 2 ell
  uint32_t t[14], borrow = 0;
#pragma unroll 1
  for (int i = 0; i < 14; i++) {
    const uint64_t d = (uint64_t)x[i] - ED448_L[i] - borrow;
    t[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 63);
  }
#pragma unroll 1
  for (int i = 0; i < 14; i++) r[i] = borrow ? x[i] : t[i];
}
// k (< ell) made odd by adding ell where it is even, then recoded into ND signed odd digits of W bits:
// k = sum dig[i] 2^(W i), dig[i] odd, |dig[i]| < 2^W (regular signed-window recoding)
template <int W, int ND>
ECG_D void ed448_recode(int8_t* dig, const uint32_t* k14) {
  uint32_t t[15];
  const uint32_t even = (k14[0] & 1u) ^ 1u;
  uint64_t carry = 0;
#pragma unroll 1
  for (int i = 0; i < 14; i++) {
    carry += (uint64_t)k14[i] + (even ? ED448_L[i] : 0u);
    t[i] = (uint32_t)carry;
    carry >>= 32;
  }
  t[14] = (uint32_t)carry;
#pragma unroll 1
  for (int i = 0; i < ND - 1; i++) {
    const int d = (int)(t[0] & ((2u << W) - 1)) - (1 << W);
    dig[i] = (int8_t)d;
    // t = (t - d) >> W; t - d is a multiple of 2^W
    int64_t c = -(int64_t)d;
#pragma unroll 1
    for (int j = 0; j < 15; j++) {
      c += (int64_t)t[j];
      t[j] = (uint32_t)c;
      c >>= 32;  // arithmetic: -1, 0 or 1
    }
#pragma unroll 1
    for (int j = 0; j < 14; j++) t[j] = (t[j] >> W) | (t[j + 1] << (32 - W));
    t[14] >>= W;
  }
  dig[ND - 1] = (int8_t)t[0];
}

// ---- the group -------------------------------------------------------------------------------------------------------
// r = 2 p; r.T only when want_t
template <class F>
ECG_D void ed_dbl(EdPt<F>& r, const EdPt<F>& p, bool want_t) {
  typename F::Fe a, b, c, e, g, h;
  F::sqr(a, p.X);
  F::sqr(b, p.Y);
  F::sqr(c, p.Z);
  F::add(c, c, c);      // C = 2 Z^2
  F::add(e, p.X, p.Y);
  F::sqr(e, e);
  F::add(g, a, b);      // G = A + B (a = 1)
  F::sub(e, e, g);      // E = (X + Y)^2 - A - B
  F::sub(h, a, b);      // H = A - B
  F::sub(c, g, c);      // F = G - C
  F::mul(r.X, e, c);
  F::mul(r.Y, g, h);
  F::mul(r.Z, c, g);
  if (want_t) F::mul(r.T, e, h);
}
// r = p + q for q = (x2, y2, z2, d t2) (z2 == nullptr: Z2 = 1, a table entry in affine form); complete for a = 1
template <class F>
ECG_D void ed_add(EdPt<F>& r, const EdPt<F>& p, const typename F::Fe& x2, const typename F::Fe& y2, const typename F::Fe* z2,
                  const typename F::Fe& dt2) {
  typename F::Fe a, b, c, dd, e, t;
  F::mul(a, p.X, x2);
  F::mul(b, p.Y, y2);
  F::mul(c, p.T, dt2);        // C = T1 d T2
  if (z2)
    F::mul(dd, p.Z, *z2);
  else
    dd = p.Z;
  F::add(e, p.X, p.Y);
  F::add(t, x2, y2);
  F::mul(e, e, t);
  F::sub(e, e, a);
  F::sub(e, e, b);            // E = (X1 + Y1)(X2 + Y2) - A - B
  F::sub(t, b, a);            // H = B - a A
  F::sub(b, dd, c);           // F = D - C
  F::add(c, dd, c);           // G = D + C
  F::mul(r.X, e, b);
  F::mul(r.Y, c, t);
  F::mul(r.T, e, t);
  F::mul(r.Z, b, c);
}

// entry |dig| of the base table, negated for a negative digit
template <class F>
ECG_D void ed448_base_entry(typename F::Fe& x, typename F::Fe& y, typename F::Fe& dt, int dig) {
  const int j = (dig < 0 ? -dig : dig) >> 1;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    x.v[i] = ED448_BTAB[j][0][i];
    y.v[i] = ED448_BTAB[j][1][i];
    dt.v[i] = ED448_BTAB[j][2][i];
  }
  if (dig < 0) {
    F::neg(x, x);
    F::neg(dt, dt);
  }
}

// [s]B + [k](-A) == R for A = (ax, ay), R = (rx, ry) affine; s, k < ell as 14 little-endian words
template <class F>
ECG_D uint32_t ed448_check_equation(const uint32_t* s, const uint32_t* k, const typename F::Fe& ax, const typename F::Fe& ay,
                                    const typename F::Fe& rx, const typename F::Fe& ry) {
  typedef typename F::Fe Fe;
  int8_t da[ED448_AND], db[ED448_BND];
  ed448_recode<ED448_AW, ED448_AND>(da, k);
  ed448_recode<ED448_BW, ED448_BND>(db, s);
  // odd multiples 1, 3, ..., 15 of -A as (X, Y, Z, d T)
  EdPt<F> tab[8];
  EdPt<F> a1, a2, q;
  F::neg(a1.X, ax);
  a1.Y = ay;
  F::set_one(a1.Z);
  F::mul(a1.T, a1.X, ay);
  ed_dbl<F>(a2, a1, true);
  Fe da2;
  ed_mul_d<F>(da2, a2.T);
  tab[0] = a1;
#pragma unroll 1
  for (int j = 1; j < 8; j++) ed_add<F>(tab[j], tab[j - 1], a2.X, a2.Y, &a2.Z, da2);
#pragma unroll 1
  for (int j = 0; j < 8; j++) ed_mul_d<F>(tab[j].T, tab[j].T);
  F::set_zero(q.X);
  F::set_one(q.Y);
  F::set_one(q.Z);
  F::set_zero(q.T);
  // positions 444 .. 0: A digits at multiples of 4, B digits at multiples of 7 (uniform across threads)
#pragma unroll 1
  for (int pos = 4 * (ED448_AND - 1); pos >= 0; pos--) {
    const bool at_a = (pos % ED448_AW) == 0, at_b = (pos % ED448_BW) == 0;
    if (pos != 4 * (ED448_AND - 1)) ed_dbl<F>(q, q, at_a || at_b);
    if (at_a) {
      const int d = da[pos / ED448_AW];
      EdPt<F> e = tab[(d < 0 ? -d : d) >> 1];
      if (d < 0) {
        F::neg(e.X, e.X);
        F::neg(e.T, e.T);
      }
      ed_add<F>(q, q, e.X, e.Y, &e.Z, e.T);
    }
    if (at_b) {
      Fe bx, by, bt;
      ed448_base_entry<F>(bx, by, bt, db[pos / ED448_BW]);
      ed_add<F>(q, q, bx, by, nullptr, bt);
    }
  }
  // (X : Y : Z) == (rx, ry)
  Fe t;
  F::mul(t, rx, q.Z);
  if (!ed_eq<F>(t, q.X)) return 0;
  F::mul(t, ry, q.Z);
  return ed_eq<F>(t, q.Y) ? 1u : 0u;
}

// the whole per-signature routine: 1 iff the reference's verify_inner accepts (pk57, sig114) on the message msg[0..mlen)
// under the dom4 prefix dom[0..dom_len) ("SigEd448" || phflag || len(ctx) || ctx)
template <class F>
ECG_D uint8_t ed448_verify_one(const uint8_t* pk57, const uint8_t* sig114, const uint8_t* msg, size_t mlen, const uint8_t* dom,
                               uint32_t dom_len) {
  typedef typename F::Fe Fe;
  if (!ed448_s_ok(sig114 + 57)) return 0;
  Fe ax, ay, rx, ry;
  if (!ed448_decompress<F>(ax, ay, pk57)) return 0;
  if (!ed448_decompress<F>(rx, ry, sig114)) return 0;
  uint8_t h[114];
  {
    Shake256 sh;
    sh.init();
    sh.absorb(dom, dom_len);
    sh.absorb(sig114, 57);
    sh.absorb(pk57, 57);
    sh.absorb(msg, mlen);
    sh.finish<114>(h);
  }
  uint32_t k[14], s[14];
  ed448_mod_l_wide(k, h);
  ed448_load56(s, sig114 + 57);
  return (uint8_t)ed448_check_equation<F>(s, k, ax, ay, rx, ry);
}

// dom4 of a call: "SigEd448" || phflag || len(ctx) || ctx, at most 8 + 2 + 255 bytes; a kernel parameter
struct Ed448Dom {
  uint8_t b[268];
  uint32_t len;
};

#if defined(__CUDACC__)
// one signature per thread: message i is msgs[offs[i] - base .. offs[i + 1] - base)
template <class F, int BLOCK, int MINBLK>
__global__ void __launch_bounds__(BLOCK, MINBLK)
    ed448_verify_kernel(const uint8_t* pk, const uint8_t* sig, const uint8_t* msgs, const uint64_t* offs, uint64_t base, size_t n,
                        Ed448Dom dom, uint8_t* valid) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i >= n) return;
  const uint64_t lo = offs[i], hi = offs[i + 1];
  valid[i] = ed448_verify_one<F>(pk + 57 * i, sig + 114 * i, msgs + (lo - base), (size_t)(hi - lo), dom.b, dom.len);
}
#endif

}  // namespace ecg
