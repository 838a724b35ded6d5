// ecg_fe_p384.cuh — F_p for NIST P-384, p = 2^384 - 2^128 - 2^96 + 2^32 - 1, on 12 saturated 32-bit limbs.
//
// Next curve through the same templates (SURVEY.md section 8(f) rank 4): the reference binds P-384 to the generic
// primeorder code exactly like P-256 (p384/src/arithmetic.rs:43-44: PointArithmetic = EquationAIsMinusThree) over a
// Montgomery field synthesised by fiat-crypto or primefield's generic Montgomery form (p384/src/arithmetic/field.rs:21-77).
// Representation here: plain integers weakly reduced to [0, 2^384) — p == -1 only modulo 2^32, so a multiplier-free
// Montgomery reduction would need twelve dependent one-word rounds (~400 carry-chain instructions); the Solinas / FIPS
// 186-4 D.2.4 word recombination needs ~150 and no domain conversion.  2^384 == K (mod p), K = 2^128 + 2^96 - 2^32 + 1.
// Product: the generic even/odd-accumulator schoolbook mulNxN<12> (144 IMAD.WIDE); squaring: sqrN<12> (66 cross products
// column by column + 12 diagonal squares = 78 multiplier slots).
#pragma once
#include "ecg_prim.cuh"

namespace ecg {

#ifndef ECG_P384_OPT
#define ECG_P384_OPT 2  // bit 1: mul / sqr as real device functions (see ecg_fe_k256.cuh)
#endif
#ifndef ECG_NOINLINE_D
#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define ECG_NOINLINE_D __device__ __noinline__
#else
#define ECG_NOINLINE_D
#endif
#endif

template <int OPT>
struct FpP384T {
  static constexpr int NL = 12;
  static constexpr bool LE = false;  // canonical records are big-endian
  static constexpr int FB = 48;       // bytes per canonical record
  typedef FeN<12> FeT;
  typedef JacN<12> JacT;
  typedef AffN<12> AffT;
  typedef FeT Fe;
  static constexpr bool MONT = false;
  static constexpr bool SQR_TRADE_DBL = false;
  static constexpr bool SQR_TRADE_MADD = false;
  static constexpr bool HALF3_ADD = false, MUL_SUB = false;  // secp256k1-only doubling / Y3 forms (ecg_fe_k256.cuh)
  static constexpr bool DBL_CALL = false;
  static constexpr bool MADD_CALL = false;
  static constexpr bool DBL_3M5S = false;
  typedef FpP384T<0> Inline;

  ECG_D static void set_zero(Fe& r) {
#pragma unroll
    for (int i = 0; i < 12; i++) r.v[i] = 0;
  }
  ECG_D static void set_one(Fe& r) {
    set_zero(r);
    r.v[0] = 1;
  }

  // r (12 limbs) += o*K for 0 <= o < 2^31; returns the carry out of bit 384.
  // o*K = o + (o*2^96 - o*2^32) + o*2^128 = {o, -o, ~0, o-1, o, 0, ...} for o >= 1 (all zero for o = 0)
  ECG_D static uint32_t add_oK(uint32_t* r, uint32_t o) {
    uint32_t m = o ? 0xFFFFFFFFu : 0u;
    r[0] = add_cc(r[0], o);
    r[1] = addc_cc(r[1], 0u - o);
    r[2] = addc_cc(r[2], m);
    r[3] = addc_cc(r[3], (o - 1u) & m);
    r[4] = addc_cc(r[4], o);
#pragma unroll
    for (int i = 5; i < 12; i++) r[i] = addc_cc(r[i], 0u);
    return addc(0u, 0u);
  }
  // r -= c*K for c in {0,1}; returns the borrow.  K = {1, ~0, ~0, 0, 1, 0, ...}
  ECG_D static uint32_t sub_K(uint32_t* r, uint32_t c) {
    uint32_t m = 0u - c;
    r[0] = sub_cc(r[0], c);
    r[1] = subc_cc(r[1], m);
    r[2] = subc_cc(r[2], m);
    r[3] = subc_cc(r[3], 0u);
    r[4] = subc_cc(r[4], c);
#pragma unroll
    for (int i = 5; i < 12; i++) r[i] = subc_cc(r[i], 0u);
    return 0u - subc(0u, 0u);
  }

  // acc (13 limbs: 12 + overflow word) += v / -= v, v a full 12-limb value
  ECG_D static void acc_add(uint32_t* acc, const uint32_t* v) {
    acc[0] = add_cc(acc[0], v[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) acc[i] = addc_cc(acc[i], v[i]);
    acc[12] = addc(acc[12], 0u);
  }
  ECG_D static void acc_sub(uint32_t* acc, const uint32_t* v) {
    acc[0] = sub_cc(acc[0], v[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) acc[i] = subc_cc(acc[i], v[i]);
    acc[12] = subc(acc[12], 0u);
  }

  // 24-limb c -> r = c mod p (weakly reduced).  FIPS 186-4 D.2.4 on 32-bit words:
  //   r = s1 + 2 s2 + s3 + s4 + s5 + s6 + s7 - s8 - s9 - s10   (tuples below are written least significant word first)
  // 4p is added up front so that the running value never goes negative; the overflow word o (< 16) is folded with K.
  ECG_D static void reduce24(Fe& r, const uint32_t* c) {
    uint32_t acc[13], v[12];
    // s1 + 4p;  4p mod 2^384 = {fffffffc, 3, 0, fffffffc, fffffffb, ffffffff x7}, 4p div 2^384 = 3
    acc[0] = add_cc(c[0], 0xFFFFFFFCu);
    acc[1] = addc_cc(c[1], 0x00000003u);
    acc[2] = addc_cc(c[2], 0x00000000u);
    acc[3] = addc_cc(c[3], 0xFFFFFFFCu);
    acc[4] = addc_cc(c[4], 0xFFFFFFFBu);
#pragma unroll
    for (int i = 5; i < 12; i++) acc[i] = addc_cc(c[i], 0xFFFFFFFFu);
    acc[12] = addc(3u, 0u);
    // 2 * s2, s2 = (0,0,0,0, c21,c22,c23, 0,0,0,0,0)
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = 0;
    v[4] = c[21]; v[5] = c[22]; v[6] = c[23];
    acc_add(acc, v);
    acc_add(acc, v);
    // s3 = (c12 .. c23)
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = c[12 + i];
    acc_add(acc, v);
    // s4 = (c21,c22,c23, c12,c13,c14,c15,c16,c17,c18,c19,c20)
    v[0] = c[21]; v[1] = c[22]; v[2] = c[23];
#pragma unroll
    for (int i = 0; i < 9; i++) v[3 + i] = c[12 + i];
    acc_add(acc, v);
    // s5 = (0, c23, 0, c20, c12,c13,c14,c15,c16,c17,c18,c19)
    v[0] = 0; v[1] = c[23]; v[2] = 0; v[3] = c[20];
#pragma unroll
    for (int i = 0; i < 8; i++) v[4 + i] = c[12 + i];
    acc_add(acc, v);
    // s6 = (0,0,0,0, c20,c21,c22,c23, 0,0,0,0)
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = 0;
    v[4] = c[20]; v[5] = c[21]; v[6] = c[22]; v[7] = c[23];
    acc_add(acc, v);
    // s7 = (c20, 0, 0, c21, c22, c23, 0,0,0,0,0,0)
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = 0;
    v[0] = c[20]; v[3] = c[21]; v[4] = c[22]; v[5] = c[23];
    acc_add(acc, v);
    // s8 = (c23, c12,c13,c14,c15,c16,c17,c18,c19,c20,c21,c22)
    v[0] = c[23];
#pragma unroll
    for (int i = 0; i < 11; i++) v[1 + i] = c[12 + i];
    acc_sub(acc, v);
    // s9 = (0, c20, c21, c22, c23, 0,0,0,0,0,0,0)
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = 0;
    v[1] = c[20]; v[2] = c[21]; v[3] = c[22]; v[4] = c[23];
    acc_sub(acc, v);
    // s10 = (0,0,0, c23, c23, 0,0,0,0,0,0,0)
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = 0;
    v[3] = c[23]; v[4] = c[23];
    acc_sub(acc, v);
    // fold the overflow word: value = acc[12] * 2^384 + acc[0..11], acc[12] in [0, 16)
    uint32_t c2 = add_oK(acc, acc[12]);
    uint32_t c3 = add_oK(acc, c2);  // one more wrap at most (the value was below 2^384 + 16 K), and none after it
    (void)c3;
#pragma unroll
    for (int i = 0; i < 12; i++) r.v[i] = acc[i];
  }

  ECG_D static void mul_body(Fe& r, const Fe& a, const Fe& b) {
    uint32_t t[24];
    mulNxN<12>(t, a.v, b.v);
    reduce24(r, t);
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
  ECG_D static void mul_d(Fe& r, const Fe& a, const Fe& b) { mul(r, a, b); }
  ECG_D static void sqr_body(Fe& r, const Fe& a) {
    uint32_t t[24];
    sqrN<12>(t, a.v);
    reduce24(r, t);
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

  ECG_D static void add(Fe& r, const Fe& a, const Fe& b) {
    uint32_t c = addN<12>(r.v, a.v, b.v);
    uint32_t c2 = add_oK(r.v, c);  // 2^384 == K
    (void)add_oK(r.v, c2);         // second wrap only if the first left less than K below 2^384
  }
  ECG_D static void sub(Fe& r, const Fe& a, const Fe& b) {
    uint32_t bw = subN<12>(r.v, a.v, b.v);
    uint32_t bw2 = sub_K(r.v, bw);
    (void)sub_K(r.v, bw2);
  }
  ECG_D static void neg(Fe& r, const Fe& a) {
    Fe z;
    set_zero(z);
    sub(r, z, a);
  }
  // r = k*a for a small constant k (2..16)
  ECG_D static void mul_small(Fe& r, const Fe& a, uint32_t k) {
    uint32_t c = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) {
      uint64_t t = (uint64_t)a.v[i] * k + c;
      r.v[i] = (uint32_t)t;
      c = (uint32_t)(t >> 32);
    }
    uint32_t c2 = add_oK(r.v, c);
    (void)add_oK(r.v, c2);
  }
  // r = a/2 mod p;  p limbs = {~0, 0, 0, ~0, ~0-1, ~0 x7}
  ECG_D static void half(Fe& r, const Fe& a) {
    uint32_t m = 0u - (a.v[0] & 1u);
    uint32_t t[12];
    t[0] = add_cc(a.v[0], m);
    t[1] = addc_cc(a.v[1], 0u);
    t[2] = addc_cc(a.v[2], 0u);
    t[3] = addc_cc(a.v[3], m);
    t[4] = addc_cc(a.v[4], m & 0xFFFFFFFEu);
#pragma unroll
    for (int i = 5; i < 12; i++) t[i] = addc_cc(a.v[i], m);
    uint32_t c = addc(0u, 0u);
#pragma unroll
    for (int i = 0; i < 11; i++) r.v[i] = funnel_r(t[i], t[i + 1], 1);
    r.v[11] = funnel_r(t[11], c, 1);
  }
  // canonical representative: a >= p  <=>  a + K carries out of bit 384
  ECG_D static void normalize(Fe& r, const Fe& a) {
    uint32_t t[12];
#pragma unroll
    for (int i = 0; i < 12; i++) t[i] = a.v[i];
    uint32_t ge = add_oK(t, 1u);
#pragma unroll
    for (int i = 0; i < 12; i++) r.v[i] = ge ? t[i] : a.v[i];
  }
  // a == 0 (mod p)  <=>  a in {0, p}
  ECG_D static bool is_zero(const Fe& a) {
    uint32_t o = 0, hi = 0xFFFFFFFFu;
#pragma unroll
    for (int i = 0; i < 12; i++) o |= a.v[i];
#pragma unroll
    for (int i = 5; i < 12; i++) hi &= a.v[i];
    uint32_t n = ~(a.v[0] & a.v[3] & hi) | a.v[1] | a.v[2] | (a.v[4] ^ 0xFFFFFFFEu);
    return (o == 0) | (n == 0);
  }
  ECG_D static void sqr_n(Fe& r, const Fe& a, int n) {
    r = a;
#pragma unroll 1
    for (int i = 0; i < n; i++) sqr(r, r);
  }
  // a^(p-2): p - 2 = [255 ones][0][32 ones][64 zeros][30 ones][0][1] in binary; 383 squarings + 15 multiplications.
  // 0 -> 0.  (reference: FieldElement::invert through crypto-bigint / fiat divsteps, p384/src/arithmetic/field.rs)
  ECG_D static void inv(Fe& r, const Fe& a) {
    Fe x2, x3, x6, x12, x15, x30, x32, x60, x120, x240, x255, t;
    sqr(x2, a);
    mul(x2, x2, a);
    sqr(x3, x2);
    mul(x3, x3, a);
    sqr_n(x6, x3, 3);
    mul(x6, x6, x3);
    sqr_n(x12, x6, 6);
    mul(x12, x12, x6);
    sqr_n(x15, x12, 3);
    mul(x15, x15, x3);
    sqr_n(x30, x15, 15);
    mul(x30, x30, x15);
    sqr_n(x32, x30, 2);
    mul(x32, x32, x2);
    sqr_n(x60, x30, 30);
    mul(x60, x60, x30);
    sqr_n(x120, x60, 60);
    mul(x120, x120, x60);
    sqr_n(x240, x120, 120);
    mul(x240, x240, x120);
    sqr_n(x255, x240, 15);
    mul(x255, x255, x15);
    sqr_n(t, x255, 1 + 32);  // the zero bit, then room for 32 ones
    mul(t, t, x32);
    sqr_n(t, t, 64 + 30);    // 64 zero bits, then room for 30 ones
    mul(t, t, x30);
    sqr_n(t, t, 2);          // bits "01"
    mul(r, t, a);
  }
  ECG_D static void from_canonical(Fe& r, const Fe& a) { r = a; }
  ECG_D static void to_canonical(Fe& r, const Fe& a) { normalize(r, a); }
};

typedef FpP384T<ECG_P384_OPT> FpP384;

}  // namespace ecg
