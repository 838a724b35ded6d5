// ecg_fe_p256.cuh — F_p for NIST P-256, p = 2^256 - 2^224 + 2^192 + 2^96 - 1, on 8 saturated 32-bit limbs.
//
// Replaces (same values, different representation) the reference's Montgomery-form field
//   p256/src/arithmetic/field.rs:59-118 over p256/src/arithmetic/field/field64.rs:7-144 (add, sub,
//   montgomery_reduce) and primefield/src/monty.rs:319-375.
// Representation (OPT bit 9, the default): the reference's own Montgomery domain, a*R mod p with R = 2^256, weakly
// reduced to [0, 2^256).  p == -1 (mod 2^96), so the Montgomery factor of every 32-bit word is the word itself
// (p' = 1, field64.rs:59-66) and the reduction `redc16` needs no multiplier: three rounds (96 + 96 + 64 bits) of
// "add M * (p + 1) / 2^k" written as 32-bit carry chains — 59 add/sub instructions on the ALU pipe, against ~110 for
// the Solinas / FIPS 186-4 D.2.3 word recombination (`reduce16`, kept behind OPT bit 9 = 0 for comparison in
// tools/kbench.cu), which made the P-256 multiplier ALU-bound in round 1.  Conversions happen only at the boundary
// (from_canonical = multiplication by R^2, to_canonical = one reduction).  2^256 == K (mod p),
// K = 2^224 - 2^192 - 2^96 + 1, folds the carry-out of additions in either representation.
#pragma once
#include "ecg_prim.cuh"

namespace ecg {

#ifndef ECG_P256_OPT
#define ECG_P256_OPT 515  // bit 0: dedicated squaring; bit 1: mul/sqr as real device functions (see ecg_fe_k256.cuh); bit 9: Montgomery domain
#endif
#ifndef ECG_NOINLINE_D
#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define ECG_NOINLINE_D __device__ __noinline__
#else
#define ECG_NOINLINE_D
#endif
#endif

template <int OPT>
struct FpP256T {
  static constexpr int NL = 8;  // 32-bit limbs per field element
  static constexpr bool LE = false;  // canonical records are big-endian
  static constexpr int FB = 32;       // bytes per canonical record
  typedef FeN<8> FeT;
  typedef JacN<8> JacT;
  typedef AffN<8> AffT;
  // the P-256 squaring is bound by its reduction's adds, not by products: no multiplication-for-squaring trades
  static constexpr bool SQR_TRADE_DBL = false;
  static constexpr bool SQR_TRADE_MADD = false;
  static constexpr bool HALF3_ADD = false, MUL_SUB = false;  // secp256k1-only doubling / Y3 forms (ecg_fe_k256.cuh)
  static constexpr bool DBL_CALL = (OPT & 2048) != 0;   // see ecg_fe_k256.cuh
  static constexpr bool MADD_CALL = (OPT & 4096) != 0;
  static constexpr bool DBL_3M5S = (OPT & 1024) != 0;   // a = -3 doubling as 3M+5S (Z3 = ((Y+Z)^2 - Y^2 - Z^2)/2) instead of 4M+4S
  typedef FpP256T<(OPT & (1 | 8 | 16 | 512 | 1024))> Inline;
  ECG_D static void set_zero(Fe& r) {
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = 0;
  }
  static constexpr bool MONT = (OPT & 512) != 0;
  // internal-form one: 1, or R mod p = K in the Montgomery domain
  ECG_D static void set_one(Fe& r) {
    set_zero(r);
    r.v[0] = 1;
    if (MONT) {
      r.v[3] = r.v[4] = r.v[5] = 0xFFFFFFFFu;
      r.v[6] = 0xFFFFFFFEu;
    }
  }

  // r += c*K for c in {0,1}; returns the carry out of bit 256.  K = {1,0,0,~0,~0,~0,~0-1,0}
  ECG_D static uint32_t add_K(uint32_t* r, uint32_t c) {
    uint32_t m = 0u - c;
    r[0] = add_cc(r[0], c);
    r[1] = addc_cc(r[1], 0);
    r[2] = addc_cc(r[2], 0);
    r[3] = addc_cc(r[3], m);
    r[4] = addc_cc(r[4], m);
    r[5] = addc_cc(r[5], m);
    r[6] = addc_cc(r[6], m & 0xFFFFFFFEu);
    r[7] = addc_cc(r[7], 0);
    return addc(0, 0);
  }
  // r -= c*K; returns the borrow
  ECG_D static uint32_t sub_K(uint32_t* r, uint32_t c) {
    uint32_t m = 0u - c;
    r[0] = sub_cc(r[0], c);
    r[1] = subc_cc(r[1], 0);
    r[2] = subc_cc(r[2], 0);
    r[3] = subc_cc(r[3], m);
    r[4] = subc_cc(r[4], m);
    r[5] = subc_cc(r[5], m);
    r[6] = subc_cc(r[6], m & 0xFFFFFFFEu);
    r[7] = subc_cc(r[7], 0);
    return 0u - subc(0, 0);
  }

  // r (8 limbs) += o*K for a small signed o; signed carry propagation; returns the new signed overflow.
  ECG_D static int32_t fold_signed(uint32_t* r, int32_t o) {
    int64_t t = (int64_t)r[0] + o;
    r[0] = (uint32_t)t;
    t >>= 32;
    t += r[1];
    r[1] = (uint32_t)t;
    t >>= 32;
    t += r[2];
    r[2] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)r[3] - o;
    r[3] = (uint32_t)t;
    t >>= 32;
    t += r[4];
    r[4] = (uint32_t)t;
    t >>= 32;
    t += r[5];
    r[5] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)r[6] - o;
    r[6] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)r[7] + o;
    r[7] = (uint32_t)t;
    t >>= 32;
    return (int32_t)t;
  }

  // acc (9 limbs: 8 + overflow word) += v, where v has non-zero limbs lo..7 (limbs below lo are zero)
  template <int LO>
  ECG_D static void acc_add(uint32_t* acc, const uint32_t* v) {
    acc[LO] = add_cc(acc[LO], v[LO]);
#pragma unroll
    for (int i = LO + 1; i < 8; i++) acc[i] = addc_cc(acc[i], v[i]);
    acc[8] = addc(acc[8], 0);
  }
  ECG_D static void acc_sub(uint32_t* acc, const uint32_t* v) {
    acc[0] = sub_cc(acc[0], v[0]);
#pragma unroll
    for (int i = 1; i < 8; i++) acc[i] = subc_cc(acc[i], v[i]);
    acc[8] = subc(acc[8], 0);
  }

  // 16-limb c -> r = c mod p (weakly reduced).  FIPS 186-4 D.2.3: s1 + 2 s2 + 2 s3 + s4 + s5 - s6 - s7 - s8 - s9 on
  // 32-bit words, as 32-bit carry chains only (IADD3.X on the ALU pipe: nothing here competes with the multiplier
  // for the FMA pipe).  5p is added up front so the running value never goes negative; the overflow word o (< 13)
  // is folded with 2^256 == K (mod p).
  ECG_D static void reduce16(Fe& r, const uint32_t* c) {
    uint32_t acc[9], v[8];
    // s1 + 5p            5p = {fffffffb, ffffffff, ffffffff, 4, 0, 0, 5, fffffffb | 4}
    acc[0] = add_cc(c[0], 0xFFFFFFFBu);
    acc[1] = addc_cc(c[1], 0xFFFFFFFFu);
    acc[2] = addc_cc(c[2], 0xFFFFFFFFu);
    acc[3] = addc_cc(c[3], 4u);
    acc[4] = addc_cc(c[4], 0u);
    acc[5] = addc_cc(c[5], 0u);
    acc[6] = addc_cc(c[6], 5u);
    acc[7] = addc_cc(c[7], 0xFFFFFFFBu);
    acc[8] = addc(4u, 0u);
    // t = s2 + s3 = (c15, c14+c15, c13+c14, c12+c13, c11+c12, 0, 0, 0), added twice
    uint32_t t[9];
    t[0] = t[1] = t[2] = 0;
    t[3] = add_cc(c[11], c[12]);
    t[4] = addc_cc(c[12], c[13]);
    t[5] = addc_cc(c[13], c[14]);
    t[6] = addc_cc(c[14], c[15]);
    t[7] = addc_cc(c[15], 0u);
    uint32_t t8 = addc(0u, 0u);
    acc_add<3>(acc, t);
    acc_add<3>(acc, t);
    acc[8] += 2u * t8;
    // s4 = (c15, c14, 0, 0, 0, c10, c9, c8)
    v[0] = c[8]; v[1] = c[9]; v[2] = c[10]; v[3] = 0; v[4] = 0; v[5] = 0; v[6] = c[14]; v[7] = c[15];
    acc_add<0>(acc, v);
    // s5 = (c8, c13, c15, c14, c13, c11, c10, c9)
    v[0] = c[9]; v[1] = c[10]; v[2] = c[11]; v[3] = c[13]; v[4] = c[14]; v[5] = c[15]; v[6] = c[13]; v[7] = c[8];
    acc_add<0>(acc, v);
    // s6 = (c10, c8, 0, 0, 0, c13, c12, c11)
    v[0] = c[11]; v[1] = c[12]; v[2] = c[13]; v[3] = 0; v[4] = 0; v[5] = 0; v[6] = c[8]; v[7] = c[10];
    acc_sub(acc, v);
    // s7 = (c11, c9, 0, 0, c15, c14, c13, c12)
    v[0] = c[12]; v[1] = c[13]; v[2] = c[14]; v[3] = c[15]; v[4] = 0; v[5] = 0; v[6] = c[9]; v[7] = c[11];
    acc_sub(acc, v);
    // s8 = (c12, 0, c10, c9, c8, c15, c14, c13)
    v[0] = c[13]; v[1] = c[14]; v[2] = c[15]; v[3] = c[8]; v[4] = c[9]; v[5] = c[10]; v[6] = 0; v[7] = c[12];
    acc_sub(acc, v);
    // s9 = (c13, 0, c11, c10, c9, 0, c15, c14)
    v[0] = c[14]; v[1] = c[15]; v[2] = 0; v[3] = c[9]; v[4] = c[10]; v[5] = c[11]; v[6] = 0; v[7] = c[13];
    acc_sub(acc, v);
    // fold o = acc[8] in [0, 13):  o*K = {o, 0, 0, -o, ~0, ~0, ~o, o-1}  (o >= 1; all-zero for o = 0)
    uint32_t o = acc[8];
    uint32_t m = o ? 0xFFFFFFFFu : 0u;
    acc[0] = add_cc(acc[0], o);
    acc[1] = addc_cc(acc[1], 0u);
    acc[2] = addc_cc(acc[2], 0u);
    acc[3] = addc_cc(acc[3], 0u - o);
    acc[4] = addc_cc(acc[4], m);
    acc[5] = addc_cc(acc[5], m);
    acc[6] = addc_cc(acc[6], m & ~o);
    acc[7] = addc_cc(acc[7], (o - 1u) & m);
    uint32_t c2 = addc(0u, 0u);
    (void)add_K(acc, c2);  // value was < 2^256 + 13*2^224: one more wrap at most, and none after it
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = acc[i];
  }

  // Alternative reduction (OPT bit 4): the same recombination written per output word on signed 64-bit accumulators;
  // fewer instructions, but nvcc lowers part of it to IMAD/IMAD.MOV on the FMA pipe (measured in tools/kbench.cu).
  ECG_D static void reduce16_cols(Fe& r, const uint32_t* c) {
    int64_t t;
    uint32_t o[8];
    t = (int64_t)c[0] + c[8] + c[9] - c[11] - c[12] - c[13] - c[14];
    o[0] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[1] + c[9] + c[10] - c[12] - c[13] - c[14] - c[15];
    o[1] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[2] + c[10] + c[11] - c[13] - c[14] - c[15];
    o[2] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[3] + 2 * ((int64_t)c[11] + c[12]) + c[13] - c[15] - c[8] - c[9];
    o[3] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[4] + 2 * ((int64_t)c[12] + c[13]) + c[14] - c[9] - c[10];
    o[4] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[5] + 2 * ((int64_t)c[13] + c[14]) + c[15] - c[10] - c[11];
    o[5] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[6] + 3 * (int64_t)c[14] + 2 * (int64_t)c[15] + c[13] - c[8] - c[9];
    o[6] = (uint32_t)t;
    t >>= 32;
    t += (int64_t)c[7] + 3 * (int64_t)c[15] + c[8] - c[10] - c[11] - c[12] - c[13];
    o[7] = (uint32_t)t;
    t >>= 32;
    int32_t ov = (int32_t)t;   // |ov| <= 6
    ov = fold_signed(o, ov);    // now in {-1, 0, 1}
    ov = fold_signed(o, ov);    // now 0
    (void)ov;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = o[i];
  }
  // Montgomery reduction (OPT bit 9): r = t / 2^256 mod p (weakly reduced) for a 16-limb t < 2^512.
  // field64.rs:83-123 does this one 64-bit word at a time with p' = 1; here the words are 32 bits and, because
  // p == -1 (mod 2^96), three words are retired per round: with M = the low 96 bits of the running value,
  //   (t + M*p) / 2^96 = t / 2^96 + M * (2^160 - 2^128 + 2^96 + 1)            [p + 1 = 2^256 - 2^224 + 2^192 + 2^96]
  // and M * (2^64 - 2^32 + 1) < 2^160 is formed by one 3-instruction addition and one 4-instruction subtraction.
  // Rounds: 96 + 96 + 64 bits.  The sum stays below 2^512 + 2^256 p, so the quotient is below 2^256 + p: one
  // conditional fold with K brings it under 2^256.
  ECG_D static void redc16(Fe& r, const uint32_t* t) {
    uint32_t u[16];
    uint32_t x2, x3, x4, n1, n2, n3, n4, ov;
    // round A: M = t[0..2]
    x2 = add_cc(t[2], t[0]);
    x3 = addc_cc(t[1], 0u);
    x4 = addc(t[2], 0u);
    n1 = sub_cc(t[1], t[0]);
    n2 = subc_cc(x2, t[1]);
    n3 = subc_cc(x3, t[2]);
    n4 = subc(x4, 0u);
    u[3] = add_cc(t[3], t[0]);
    u[4] = addc_cc(t[4], t[1]);
    u[5] = addc_cc(t[5], t[2]);
    u[6] = addc_cc(t[6], t[0]);
    u[7] = addc_cc(t[7], n1);
    u[8] = addc_cc(t[8], n2);
    u[9] = addc_cc(t[9], n3);
    u[10] = addc_cc(t[10], n4);
#pragma unroll
    for (int i = 11; i < 16; i++) u[i] = addc_cc(t[i], 0u);
    ov = addc(0u, 0u);
    // round B: M = u[3..5]
    x2 = add_cc(u[5], u[3]);
    x3 = addc_cc(u[4], 0u);
    x4 = addc(u[5], 0u);
    n1 = sub_cc(u[4], u[3]);
    n2 = subc_cc(x2, u[4]);
    n3 = subc_cc(x3, u[5]);
    n4 = subc(x4, 0u);
    uint32_t m0 = u[3], m1 = u[4], m2 = u[5];
    u[6] = add_cc(u[6], m0);
    u[7] = addc_cc(u[7], m1);
    u[8] = addc_cc(u[8], m2);
    u[9] = addc_cc(u[9], m0);
    u[10] = addc_cc(u[10], n1);
    u[11] = addc_cc(u[11], n2);
    u[12] = addc_cc(u[12], n3);
    u[13] = addc_cc(u[13], n4);
    u[14] = addc_cc(u[14], 0u);
    u[15] = addc_cc(u[15], 0u);
    ov = addc(ov, 0u);
    // round C: M = u[6..7] (64 bits): + M * (2^192 - 2^160 + 2^128 + 2^32) at word 8
    m0 = u[6];
    m1 = u[7];
    n1 = sub_cc(m1, m0);
    n2 = subc_cc(m0, m1);
    n3 = subc(m1, 0u);
    r.v[0] = u[8];
    r.v[1] = add_cc(u[9], m0);
    r.v[2] = addc_cc(u[10], m1);
    r.v[3] = addc_cc(u[11], 0u);
    r.v[4] = addc_cc(u[12], m0);
    r.v[5] = addc_cc(u[13], n1);
    r.v[6] = addc_cc(u[14], n2);
    r.v[7] = addc_cc(u[15], n3);
    ov = addc(ov, 0u);
    (void)add_K(r.v, ov);
  }
  ECG_D static void reduce(Fe& r, const uint32_t* t) {
    if (MONT)
      redc16(r, t);
    else if (OPT & 16)
      reduce16_cols(r, t);
    else
      reduce16(r, t);
  }

  ECG_D static void mul_body(Fe& r, const Fe& a, const Fe& b) {
    uint32_t t[16];
    if (OPT & 8)  // OPT bit 3: one-level Karatsuba (48 products + ~60 extra adds) instead of the 64-product schoolbook
      mul8x8_kara(t, a.v, b.v);
    else
      mul8x8(t, a.v, b.v);
    reduce(r, t);
  }
  ECG_D static void sqr_body(Fe& r, const Fe& a) {
    uint32_t t[16];
    if (OPT & 1)
      sqr8(t, a.v);
    else
      mul8x8(t, a.v, a.v);
    reduce(r, t);
  }
  static ECG_NOINLINE_D Fe mul_call(Fe a, Fe b) {
    Fe r;
    mul_body(r, a, b);
    return r;
  }
  static ECG_NOINLINE_D Fe sqr_call(Fe a) {
    Fe r;
    sqr_body(r, a);
    return r;
  }
  // OPT bit 8 (experiment, tools/kbench.cu mode `mem`): operands and result through local memory, see ecg_fe_k256.cuh
  static ECG_NOINLINE_D void mul_call_mem(Fe* r, const Fe* a, const Fe* b) {
    Fe x = *a, y = *b, z;
    mul_body(z, x, y);
    *r = z;
  }
  static ECG_NOINLINE_D void sqr_call_mem(Fe* r, const Fe* a) {
    Fe x = *a, z;
    sqr_body(z, x);
    *r = z;
  }
  ECG_D static void mul(Fe& r, const Fe& a, const Fe& b) {
    if (OPT & 256)
      mul_call_mem(&r, &a, &b);
    else if (OPT & 2)
      r = mul_call(a, b);
    else
      mul_body(r, a, b);
  }
  // multiplication as used inside the doubling formula: OPT bit 5 keeps those three inlined (fewer calls on the
  // hottest path) while the mixed addition still calls
  ECG_D static void mul_d(Fe& r, const Fe& a, const Fe& b) {
    if (OPT & 256)
      mul_call_mem(&r, &a, &b);
    else if ((OPT & 2) && !(OPT & 32))
      r = mul_call(a, b);
    else
      mul_body(r, a, b);
  }
  ECG_D static void sqr(Fe& r, const Fe& a) {
    if ((OPT & 256) && !(OPT & 4))
      sqr_call_mem(&r, &a);
    else if ((OPT & 2) && !(OPT & 4))  // OPT bit 2: keep the (smaller) squaring inlined even when mul is a call
      r = sqr_call(a);
    else
      sqr_body(r, a);
  }
  ECG_D static void add(Fe& r, const Fe& a, const Fe& b) {
    uint32_t c = add8(r.v, a.v, b.v);
    uint32_t c2 = add_K(r.v, c);   // 2^256 == K
    (void)add_K(r.v, c2);          // second wrap only if the first left less than K below 2^256
  }
  ECG_D static void sub(Fe& r, const Fe& a, const Fe& b) {
    uint32_t bw = sub8(r.v, a.v, b.v);
    uint32_t bw2 = sub_K(r.v, bw);
    (void)sub_K(r.v, bw2);
  }
  ECG_D static void neg(Fe& r, const Fe& a) {
    Fe z;
    set_zero(z);
    sub(r, z, a);
  }
  ECG_D static void mul_small(Fe& r, const Fe& a, uint32_t k) {
    uint32_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint64_t t = (uint64_t)a.v[i] * k + c;
      r.v[i] = (uint32_t)t;
      c = (uint32_t)(t >> 32);
    }
    int32_t ov = fold_signed(r.v, (int32_t)c);
    ov = fold_signed(r.v, ov);
    (void)ov;
  }
  // r = a/2 mod p;  p limbs = {~0, ~0, ~0, 0, 0, 0, 1, ~0}
  ECG_D static void half(Fe& r, const Fe& a) {
    uint32_t m = 0u - (a.v[0] & 1u);
    uint32_t t[8];
    t[0] = add_cc(a.v[0], m);
    t[1] = addc_cc(a.v[1], m);
    t[2] = addc_cc(a.v[2], m);
    t[3] = addc_cc(a.v[3], 0);
    t[4] = addc_cc(a.v[4], 0);
    t[5] = addc_cc(a.v[5], 0);
    t[6] = addc_cc(a.v[6], m & 1u);
    t[7] = addc_cc(a.v[7], m);
    uint32_t c = addc(0, 0);
#pragma unroll
    for (int i = 0; i < 7; i++) r.v[i] = funnel_r(t[i], t[i + 1], 1);
    r.v[7] = funnel_r(t[7], c, 1);
  }
  // canonical representative: a >= p  <=>  a + (2^256 - p) carries;  2^256 - p = K
  ECG_D static void normalize(Fe& r, const Fe& a) {
    uint32_t t[8];
#pragma unroll
    for (int i = 0; i < 8; i++) t[i] = a.v[i];
    uint32_t ge = add_K(t, 1u);
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = ge ? t[i] : a.v[i];
  }
  ECG_D static bool is_zero(const Fe& a) {
    uint32_t o = a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7];
    uint32_t n = ~(a.v[0] & a.v[1] & a.v[2] & a.v[7]) | a.v[3] | a.v[4] | a.v[5] | (a.v[6] ^ 1u);
    return (o == 0) | (n == 0);
  }
  ECG_D static void sqr_n(Fe& r, const Fe& a, int n) {
    r = a;
#pragma unroll 1
    for (int i = 0; i < n; i++) sqr(r, r);
  }
  // a^(p-2): p-2 = [32 ones][31 zeros][1][96 zeros][94 ones][0][1]; 255 S + 13 M.  0 -> 0.
  // (reference: FieldElement::invert -> crypto-bigint, p256/src/arithmetic/field.rs:111-118)
  ECG_D static void inv(Fe& r, const Fe& a) {
    Fe x2, x3, x6, x12, x15, x30, x32, t;
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
    sqr_n(t, x32, 32);
    mul(t, t, a);
    sqr_n(t, t, 128);
    mul(t, t, x32);
    sqr_n(t, t, 32);
    mul(t, t, x32);
    sqr_n(t, t, 30);
    mul(t, t, x30);
    sqr_n(t, t, 2);
    mul(r, t, a);
  }
  // boundary encoding: the C ABI speaks canonical integers.  Montgomery domain: in = a * R^2 / R, out = a / R
  // (FieldElement::from_uint_unchecked / to_canonical, p256/src/arithmetic/field.rs:59-64, 94-96).
  ECG_D static void from_canonical(Fe& r, const Fe& a) {
    if (MONT) {
      Fe r2;  // R^2 mod p (p256/src/arithmetic/field.rs:181-186)
      r2.v[0] = 0x00000003u; r2.v[1] = 0x00000000u; r2.v[2] = 0xFFFFFFFFu; r2.v[3] = 0xFFFFFFFBu;
      r2.v[4] = 0xFFFFFFFEu; r2.v[5] = 0xFFFFFFFFu; r2.v[6] = 0xFFFFFFFDu; r2.v[7] = 0x00000004u;
      mul(r, a, r2);
    } else {
      r = a;
    }
  }
  ECG_D static void to_canonical(Fe& r, const Fe& a) {
    if (MONT) {
      uint32_t t[16];
#pragma unroll
      for (int i = 0; i < 8; i++) {
        t[i] = a.v[i];
        t[8 + i] = 0;
      }
      Fe q;
      redc16(q, t);
      normalize(r, q);
    } else {
      normalize(r, a);
    }
  }
};

typedef FpP256T<ECG_P256_OPT> FpP256;

}  // namespace ecg
