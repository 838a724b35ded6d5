// ecg_fe_p448.cuh — F_p for Curve448 / X448 (RFC 7748), p = 2^448 - 2^224 - 1, on 14 saturated 32-bit limbs.
//
// The reference reads X448 u-coordinates through ed448-goldilocks' FieldElement (a Montgomery form over crypto-bigint,
// ed448-goldilocks/src/field/element.rs).  Representation here: plain integers, little-endian limbs, weakly reduced to
// [0, 2^448).  The generic Montgomery policy (ecg_fe_mont.cuh) would spend 2 * 14^2 + 14 = 406 multiplier slots per
// product; the Solinas shape of p needs none for the reduction:
//
//   c = L + 2^448 H,  H = H_lo + 2^224 H_hi  (L, H: 448 bits; H_lo, H_hi: 224 bits),  2^448 == K = 2^224 + 1 (mod p)
//   c == L + (H_lo + H_hi) + 2^224 (H_lo + 2 H_hi)  (mod p)
//
// which is carry-chain additions on the ALU pipe (the argument of the P-521 Mersenne reduction, DESIGN.md section 4).
// Product: mulNxN<14> (196 IMAD.WIDE); square: sqrN<14> (91 cross products + 14 squares = 105 multiplier slots).
//
// Ranges (tests/test_x448.py checks each on the device and on the host twin):
//   add, sub, neg, mul, sqr, mul_small, inv   any inputs in [0, 2^448)  ->  [0, 2^448), congruent (weakly reduced)
//   normalize, to_canonical, from_bytes       any input in [0, 2^448)  ->  [0, p), the canonical representative
//   cswap                                      exchanges the raw limbs under an all-ones / all-zero mask
// Every operation is straight-line code: no branch and no memory index depends on a limb value.
#pragma once
#include "ecg_prim.cuh"

namespace ecg {

#ifndef ECG_NOINLINE_D
#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define ECG_NOINLINE_D __device__ __noinline__
#else
#define ECG_NOINLINE_D
#endif
#endif

// OPT bit 1: mul / sqr as real device functions (call-based); 0: every operation inlined
template <int OPT>
struct FpP448T {
  static constexpr int NL = 14;
  static constexpr bool LE = true;  // canonical records are little-endian (RFC 7748 encodeUCoordinate)
  static constexpr int FB = 56;     // bytes per canonical record
  typedef FeN<14> FeT;
  typedef FeT Fe;
  static constexpr bool MONT = false;

  ECG_D static void set_zero(Fe& r) {
#pragma unroll
    for (int i = 0; i < 14; i++) r.v[i] = 0;
  }
  ECG_D static void set_one(Fe& r) {
    set_zero(r);
    r.v[0] = 1;
  }
  ECG_D static void set_small(Fe& r, uint32_t v) {
    set_zero(r);
    r.v[0] = v;
  }

  // r (14 limbs) += o*K, K = 2^224 + 1 (o added at limbs 0 and 7 in one chain); returns the carry out of bit 448
  ECG_D static uint32_t add_oK(uint32_t* r, uint32_t o) {
    r[0] = add_cc(r[0], o);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = addc_cc(r[i], 0u);
    r[7] = addc_cc(r[7], o);
#pragma unroll
    for (int i = 8; i < 14; i++) r[i] = addc_cc(r[i], 0u);
    return addc(0u, 0u);
  }
  // r -= c*K for c in {0, 1}; returns the borrow
  ECG_D static uint32_t sub_K(uint32_t* r, uint32_t c) {
    r[0] = sub_cc(r[0], c);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = subc_cc(r[i], 0u);
    r[7] = subc_cc(r[7], c);
#pragma unroll
    for (int i = 8; i < 14; i++) r[i] = subc_cc(r[i], 0u);
    return 0u - subc(0u, 0u);
  }

  // 28-limb c -> r == c (mod p), r in [0, 2^448)
  ECG_D static void reduce28(Fe& r, const uint32_t* c) {
    const uint32_t* Hlo = c + 14;
    const uint32_t* Hhi = c + 21;
    uint32_t s[8], t[8], acc[15];
    // s = H_lo + H_hi (< 2^225), t = s + H_hi = H_lo + 2 H_hi (< 2^226)
    s[0] = add_cc(Hlo[0], Hhi[0]);
#pragma unroll
    for (int i = 1; i < 7; i++) s[i] = addc_cc(Hlo[i], Hhi[i]);
    s[7] = addc(0u, 0u);
    t[0] = add_cc(s[0], Hhi[0]);
#pragma unroll
    for (int i = 1; i < 7; i++) t[i] = addc_cc(s[i], Hhi[i]);
    t[7] = addc(s[7], 0u);
    // acc = L + s
    acc[0] = add_cc(c[0], s[0]);
#pragma unroll
    for (int i = 1; i < 8; i++) acc[i] = addc_cc(c[i], s[i]);
#pragma unroll
    for (int i = 8; i < 14; i++) acc[i] = addc_cc(c[i], 0u);
    acc[14] = addc(0u, 0u);
    // acc += 2^224 t;  acc < 2^448 + 2^225 + 2^450 < 2^451, so the overflow word is below 8
    acc[7] = add_cc(acc[7], t[0]);
#pragma unroll
    for (int i = 1; i < 7; i++) acc[7 + i] = addc_cc(acc[7 + i], t[i]);
    acc[14] = addc(acc[14], t[7]);
    // fold the overflow word o with 2^448 == K; a carry out of that leaves less than o*K + K below 2^448, so a second
    // fold of the carry cannot carry again
    uint32_t c2 = add_oK(acc, acc[14]);
    (void)add_oK(acc, c2);
#pragma unroll
    for (int i = 0; i < 14; i++) r.v[i] = acc[i];
  }

  ECG_D static void mul_body(Fe& r, const Fe& a, const Fe& b) {
    uint32_t t[28];
    mulNxN<14>(t, a.v, b.v);
    reduce28(r, t);
  }
  static ECG_NOINLINE_D Fe mul_call(Fe a, Fe b) {
    Fe r;
    mul_body(r, a, b);
    return r;
  }
  ECG_D static void mul(Fe& r, const Fe& a, const Fe& b) {
    if (OPT & 2)
      r = mul_call(a, b);
    else
      mul_body(r, a, b);
  }
  ECG_D static void sqr_body(Fe& r, const Fe& a) {
    uint32_t t[28];
    sqrN<14>(t, a.v);
    reduce28(r, t);
  }
  static ECG_NOINLINE_D Fe sqr_call(Fe a) {
    Fe r;
    sqr_body(r, a);
    return r;
  }
  ECG_D static void sqr(Fe& r, const Fe& a) {
    if (OPT & 2)
      r = sqr_call(a);
    else
      sqr_body(r, a);
  }

  // a + b < 2^449: one carry folds as K; if that carries too, less than K is left below 2^448 and a second fold cannot
  ECG_D static void add(Fe& r, const Fe& a, const Fe& b) {
    uint32_t c = addN<14>(r.v, a.v, b.v);
    uint32_t c2 = add_oK(r.v, c);
    (void)add_oK(r.v, c2);
  }
  // a - b + 2^448 on a borrow: subtract K; a second borrow leaves at least 2^448 - K, and a third cannot happen
  ECG_D static void sub(Fe& r, const Fe& a, const Fe& b) {
    uint32_t bw = subN<14>(r.v, a.v, b.v);
    uint32_t bw2 = sub_K(r.v, bw);
    (void)sub_K(r.v, bw2);
  }
  ECG_D static void neg(Fe& r, const Fe& a) {
    Fe z;
    set_zero(z);
    sub(r, z, a);
  }
  // r = k*a for a constant k < 2^32 (the ladder's (A + 2)/4 = 39082): 14 IMAD.WIDE, the top word folds as K
  ECG_D static void mul_small(Fe& r, const Fe& a, uint32_t k) {
    uint32_t c = 0;
#pragma unroll
    for (int i = 0; i < 14; i++) {
      uint64_t t = (uint64_t)a.v[i] * k + c;
      r.v[i] = (uint32_t)t;
      c = (uint32_t)(t >> 32);
    }
    uint32_t c2 = add_oK(r.v, c);
    (void)add_oK(r.v, c2);
  }
  // canonical representative: a >= p  <=>  a + K carries out of bit 448, and then a + K - 2^448 = a - p
  ECG_D static void normalize(Fe& r, const Fe& a) {
    uint32_t t[14];
#pragma unroll
    for (int i = 0; i < 14; i++) t[i] = a.v[i];
    const uint32_t m = 0u - add_oK(t, 1u);
#pragma unroll
    for (int i = 0; i < 14; i++) r.v[i] = (t[i] & m) | (a.v[i] & ~m);
  }
  // (a, b) <- (b, a) when mask = ~0, unchanged when mask = 0: the same instructions either way
  ECG_D static void cswap(Fe& a, Fe& b, uint32_t mask) {
#pragma unroll
    for (int i = 0; i < 14; i++) {
      const uint32_t t = (a.v[i] ^ b.v[i]) & mask;
      a.v[i] ^= t;
      b.v[i] ^= t;
    }
  }
  ECG_D static void sqr_n(Fe& r, const Fe& a, int n) {
    r = a;
#pragma unroll 1
    for (int i = 0; i < n; i++) sqr(r, r);
  }
  // a^(p-2), 0 -> 0.  p - 2 = 2^448 - 2^224 - 3 = [223 ones][0][222 ones][0][1] in binary.  x_k = a^(2^k - 1);
  // 453 squarings + 13 multiplications.  (reference: FieldElement::invert, ed448-goldilocks/src/field/element.rs)
  ECG_D static void inv(Fe& r, const Fe& a) {
    Fe x2, x3, x6, x12, x24, x30, x48, t;
    sqr(x2, a);
    mul(x2, x2, a);
    sqr(x3, x2);
    mul(x3, x3, a);
    sqr_n(x6, x3, 3);
    mul(x6, x6, x3);
    sqr_n(x12, x6, 6);
    mul(x12, x12, x6);
    sqr_n(x24, x12, 12);
    mul(x24, x24, x12);
    sqr_n(x30, x24, 6);
    mul(x30, x30, x6);
    sqr_n(x48, x24, 24);
    mul(x48, x48, x24);
    sqr_n(t, x48, 48);
    mul(t, t, x48);      // x96
    sqr_n(x2, t, 96);
    mul(t, x2, t);       // x192
    sqr_n(t, t, 30);
    mul(x30, t, x30);    // x222
    sqr(t, x30);
    mul(t, t, a);        // x223
    sqr_n(t, t, 1 + 222);  // the zero bit, then room for 222 ones
    mul(t, t, x30);
    sqr_n(t, t, 2);      // bits "01"
    mul(r, t, a);
  }
  ECG_D static void to_canonical(Fe& r, const Fe& a) { normalize(r, a); }
};

}  // namespace ecg
