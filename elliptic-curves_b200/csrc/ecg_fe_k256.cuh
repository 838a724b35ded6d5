// ecg_fe_k256.cuh — F_p for secp256k1, p = 2^256 - 2^32 - 977, on 8 saturated 32-bit limbs.
//
// Replaces (same values, different representation) the reference's lazily-reduced 5x52 field
//   k256/src/arithmetic/field/field_5x52.rs:240-401 (mul_inner), :122-155 (normalize*), :203-236
//   (negate/add/mul_single) and the wrappers in k256/src/arithmetic/field.rs:116-196.
// Representation: every Fe holds an integer in [0, 2^256) congruent to the field value ("weakly
// reduced": it may exceed p by at most C-1, C = 2^256 - p = 2^32 + 977).  There is no magnitude
// bookkeeping (the reference's `negate(m)` / `normalize_weak` contract disappears); `normalize()`
// produces the canonical representative in [0, p) which is what crosses the C ABI.
#pragma once
#include "ecg_prim.cuh"

namespace ecg {

// OPT bit 0: dedicated squaring (sqr8, 36 products) instead of mul8x8(a, a)
// OPT bit 1: mul / sqr are real (non-inlined) device functions taking and returning Fe by value in registers:
//            the kernels shrink ~3x and fit the instruction cache (ncu: `no_instruction` stalls; DESIGN.md)
#ifndef ECG_K256_OPT
#define ECG_K256_OPT 7
#endif
#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define ECG_NOINLINE_D __device__ __noinline__
#else
#define ECG_NOINLINE_D
#endif

template <int OPT>
struct FpK256T {
  static constexpr int NL = 8;  // 32-bit limbs per field element
  static constexpr bool LE = false;  // canonical records are big-endian
  static constexpr int FB = 32;       // bytes per canonical record
  typedef FeN<8> FeT;
  typedef JacN<8> JacT;
  typedef AffN<8> AffT;
  static constexpr uint32_t C0 = 977u;  // C = 2^32 + 977
  // OPT bits 6/7: the doubling / mixed addition trade one multiplication for a squaring + 4 linear ops
  static constexpr bool SQR_TRADE_DBL = (OPT & 64) != 0;
  static constexpr bool SQR_TRADE_MADD = (OPT & 128) != 0;
  // OPT bits 11/12 (experiments, tools/kbench.cu): the point doubling / the mixed addition is ONE non-inlined function
  // (Jacobian point in registers in and out) whose field operations are all inlined — one call per point operation
  // instead of one per field multiplication, so the call marshalling (IMAD.MOV on the FMA pipe) shrinks accordingly
  static constexpr bool DBL_CALL = (OPT & 2048) != 0;
  static constexpr bool MADD_CALL = (OPT & 4096) != 0;
  static constexpr bool DBL_3M5S = false;
  // OPT bit 13: the window table of k256_mul_thread carries beta*x beside x, so the lambda-half additions read it
  // instead of multiplying in the loop (8 M per table instead of 34 M per scalar)
  static constexpr bool BETA_COLUMN = (OPT & 8192) != 0;
  // OPT bit 14: the a = 0 doubling forms 3/2 X^2 as X^2 + X^2/2 (carry chains) instead of mul_small(3) then half
  static constexpr bool HALF3_ADD = (OPT & 16384) != 0;
  // OPT bit 15: Y3 of the doubling and of the mixed addition is one mul_sub / mul_sub_sqr (two products, one reduction)
  static constexpr bool MUL_SUB = (OPT & 32768) != 0;
  typedef FpK256T<(OPT & (1 | 8 | 64 | 128 | 8192 | 16384 | 32768))> Inline;  // the same field with mul / sqr inlined

  ECG_D static void set_zero(Fe& r) {
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = 0;
  }
  ECG_D static void set_one(Fe& r) {
    set_zero(r);
    r.v[0] = 1;
  }

  // r (8 limbs, already holding the low part) += top * C + e * C^2 where top = t0 + 2^32*t1 <= C, t1 and e in {0,1}
  // (e is bit 512 of a mul_sub intermediate: 2^512 == C^2 = 2^64 + 1954*2^32 + 954529 (mod p); every other caller
  // passes e = 0, which folds away at compile time).  The addend is < 2C^2 < 2^67, so the result is again < 2^256
  // (at most two wrap-arounds, the second confined to limbs 0..3).
  ECG_D static void fold_top(uint32_t* r, uint32_t t0, uint32_t t1, uint32_t e = 0) {
    uint32_t q0, q1;
    mul_wide(q0, q1, t0, C0);                     // t0*977
    uint64_t s0 = (uint64_t)q0 + (e ? 954529u : 0u);  // position-0 column: lo(t0*977) + e*lo(C^2)
    // position-1 column: hi(t0*977) + t0 + t1*977 + e*1954 + carry
    uint64_t s1 = (uint64_t)q1 + t0 + (t1 ? C0 : 0u) + (e ? 1954u : 0u) + (s0 >> 32);
    uint32_t q0s = (uint32_t)s0;
    uint32_t p1 = (uint32_t)s1;
    uint32_t p2 = (uint32_t)(s1 >> 32) + t1 + e;  // position-2 column
    r[0] = add_cc(r[0], q0s);
    r[1] = addc_cc(r[1], p1);
    r[2] = addc_cc(r[2], p2);
#pragma unroll
    for (int i = 3; i < 8; i++) r[i] = addc_cc(r[i], 0);
    uint32_t cf = addc(0, 0);
    // wrapped past 2^256 (rare): the residue is < 2^67, add C once more; cannot wrap again.
    r[0] = add_cc(r[0], cf ? C0 : 0u);
    r[1] = addc_cc(r[1], cf);
    r[2] = addc_cc(r[2], 0);
    r[3] = addc(r[3], 0);
  }

  // 16-limb t (+ e * 2^512, e in {0,1}) -> r = t mod p (weakly reduced).  t_lo + t_hi * C with the even/odd pair
  // trick (any t < 2^512: the sum is < 2^256 (1 + C), so its top is <= C), then fold.
  ECG_D static void reduce16(Fe& r, const uint32_t* t, uint32_t e = 0) {
    uint32_t lo[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      lo[i] = t[i];
      q[i] = t[8 + i];  // q[k] sits at position k+1: the "<<32" half of hi*C
    }
    // even hi limbs * 977 land on positions 0,2,4,6 -> pairs of lo
    mad_wide_cc(lo[0], lo[1], t[8], C0);
    madc_wide_cc(lo[2], lo[3], t[10], C0);
    madc_wide_cc(lo[4], lo[5], t[12], C0);
    madc_wide_cc(lo[6], lo[7], t[14], C0);
    uint32_t e8 = addc(0, 0);
    // odd hi limbs * 977 land on positions 1,3,5,7 -> pairs of q
    mad_wide_cc(q[0], q[1], t[9], C0);
    madc_wide_cc(q[2], q[3], t[11], C0);
    madc_wide_cc(q[4], q[5], t[13], C0);
    madc_wide_cc(q[6], q[7], t[15], C0);
    uint32_t q8 = addc(0, 0);
    // merge
    r.v[0] = lo[0];
    r.v[1] = add_cc(lo[1], q[0]);
#pragma unroll
    for (int k = 2; k < 8; k++) r.v[k] = addc_cc(lo[k], q[k - 1]);
    uint32_t t0 = addc_cc(e8, q[7]);
    uint32_t t1 = addc(q8, 0);  // top = t0 + 2^32*t1 <= C
    fold_top(r.v, t0, t1, e);
  }
  // t (16 limbs) = a*b, u (16 limbs) = c*d, each <= (2^256 - 1)^2 (any operands < 2^256, not only < p)
  //   -> r = (a*b - c*d) mod p, weakly reduced, with one reduction.  t - u lies in (-2^512, 2^512); when it is negative,
  // 2p * 2^256 = 2^513 - 2C * 2^256 (== 0 mod p) is added, giving D in (2^512 - 2C * 2^256, 2^513): D = t' + e * 2^512
  // with t' < 2^512 and e in {0,1}, and reduce16 folds the two together.  t is overwritten.
  ECG_D static void sub_reduce16(Fe& r, uint32_t* t, const uint32_t* u) {
    const uint32_t bw = subN<16>(t, t, u);  // t = a*b - c*d + bw * 2^512
    const uint32_t m = 0u - bw;
    t[8] = sub_cc(t[8], m & 1954u);  // high half -= bw * 2C  (2C = 2^33 + 1954)
    t[9] = subc_cc(t[9], m & 2u);
#pragma unroll
    for (int i = 10; i < 16; i++) t[i] = subc_cc(t[i], 0);
    const uint32_t b2 = 0u - subc(0, 0);  // the 2^512 of the correction was consumed (b2 <= bw: D >= 0)
    reduce16(r, t, bw ^ b2);
  }
  ECG_D static void mul_sub(Fe& r, const Fe& a, const Fe& b, const Fe& c, const Fe& d) {
    uint32_t t[16], u[16];
    if (OPT & 8) {
      mul8x8_kara(u, c.v, d.v);
      mul8x8_kara(t, a.v, b.v);
    } else {
      mul8x8(u, c.v, d.v);
      mul8x8(t, a.v, b.v);
    }
    sub_reduce16(r, t, u);
  }
  // r = (a*b - c^2) mod p, the same way
  ECG_D static void mul_sub_sqr(Fe& r, const Fe& a, const Fe& b, const Fe& c) {
    uint32_t t[16], u[16];
    if (OPT & 1)
      sqr8(u, c.v);
    else
      mul8x8(u, c.v, c.v);
    if (OPT & 8)
      mul8x8_kara(t, a.v, b.v);
    else
      mul8x8(t, a.v, b.v);
    sub_reduce16(r, t, u);
  }

  ECG_D static void mul_body(Fe& r, const Fe& a, const Fe& b) {
    uint32_t t[16];
    if (OPT & 8)  // OPT bit 3: one-level Karatsuba (48 products + ~60 extra adds) instead of the 64-product schoolbook
      mul8x8_kara(t, a.v, b.v);
    else
      mul8x8(t, a.v, b.v);
    reduce16(r, t);
  }
  ECG_D static void sqr_body(Fe& r, const Fe& a) {
    uint32_t t[16];
    if (OPT & 1)
      sqr8(t, a.v);
    else
      mul8x8(t, a.v, a.v);
    reduce16(r, t);
  }
  static ECG_NOINLINE_D Fe mul_call(Fe a, Fe b) {
    Fe r;
    mul_body(r, a, b);
    return r;
  }
  // OPT bit 8 (experiment, tools/kbench.cu): operands and result travel through local memory (LDL/STL on the idle LSU
  // pipe) instead of the register ABI, whose marshalling ptxas emits as IMAD.MOV on the FMA pipe
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
  static ECG_NOINLINE_D Fe sqr_call(Fe a) {
    Fe r;
    sqr_body(r, a);
    return r;
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
    // 2^256 == C (mod p)
    r.v[0] = add_cc(r.v[0], c ? C0 : 0u);
    r.v[1] = addc_cc(r.v[1], c);
#pragma unroll
    for (int i = 2; i < 8; i++) r.v[i] = addc_cc(r.v[i], 0);
    uint32_t c2 = addc(0, 0);  // only if both inputs were >= p
    r.v[0] = add_cc(r.v[0], c2 ? C0 : 0u);
    r.v[1] = addc(r.v[1], c2);
  }
  ECG_D static void sub(Fe& r, const Fe& a, const Fe& b) {
    uint32_t bw = sub8(r.v, a.v, b.v);
    r.v[0] = sub_cc(r.v[0], bw ? C0 : 0u);
    r.v[1] = subc_cc(r.v[1], bw);
#pragma unroll
    for (int i = 2; i < 8; i++) r.v[i] = subc_cc(r.v[i], 0);
    uint32_t bw2 = 0u - subc(0, 0);  // only if a - b + 2^256 < C
    r.v[0] = sub_cc(r.v[0], bw2 ? C0 : 0u);
    r.v[1] = subc(r.v[1], bw2);
  }
  ECG_D static void neg(Fe& r, const Fe& a) {
    Fe z;
    set_zero(z);
    sub(r, z, a);
  }
  // r = k*a for a small constant k (2..16): one dependent IMAD.WIDE chain + fold of the top limb.
  ECG_D static void mul_small(Fe& r, const Fe& a, uint32_t k) {
    uint32_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint64_t t = (uint64_t)a.v[i] * k + c;
      r.v[i] = (uint32_t)t;
      c = (uint32_t)(t >> 32);
    }
    fold_top(r.v, c, 0);
  }
  // r = a/2 mod p
  ECG_D static void half(Fe& r, const Fe& a) {
    uint32_t m = 0u - (a.v[0] & 1u);
    uint32_t t[8];
    t[0] = add_cc(a.v[0], m & 0xFFFFFC2Fu);
    t[1] = addc_cc(a.v[1], m & 0xFFFFFFFEu);
#pragma unroll
    for (int i = 2; i < 8; i++) t[i] = addc_cc(a.v[i], m);
    uint32_t c = addc(0, 0);
#pragma unroll
    for (int i = 0; i < 7; i++) r.v[i] = funnel_r(t[i], t[i + 1], 1);
    r.v[7] = funnel_r(t[7], c, 1);
  }
  // canonical representative in [0, p)
  ECG_D static void normalize(Fe& r, const Fe& a) {
    uint32_t t[8];
    t[0] = add_cc(a.v[0], C0);
    t[1] = addc_cc(a.v[1], 1u);
#pragma unroll
    for (int i = 2; i < 8; i++) t[i] = addc_cc(a.v[i], 0);
    uint32_t ge = addc(0, 0);  // a + C >= 2^256  <=>  a >= p
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = ge ? t[i] : a.v[i];
  }
  // a == 0 (mod p)  <=>  a in {0, p}
  ECG_D static bool is_zero(const Fe& a) {
    uint32_t o = a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7];
    uint32_t n = (a.v[0] ^ 0xFFFFFC2Fu) | (a.v[1] ^ 0xFFFFFFFEu) | ~(a.v[2] & a.v[3] & a.v[4] & a.v[5] & a.v[6] & a.v[7]);
    return (o == 0) | (n == 0);
  }
  // strictly canonical (< p)?  used for input validation (mirrors FieldElement::from_bytes range check,
  // k256/src/arithmetic/field.rs:85-96)
  ECG_D static bool is_canonical(const Fe& a) {
    uint32_t hi = a.v[2] & a.v[3] & a.v[4] & a.v[5] & a.v[6] & a.v[7];
    bool ge = (hi == 0xFFFFFFFFu) && (a.v[1] == 0xFFFFFFFFu || (a.v[1] == 0xFFFFFFFEu && a.v[0] >= 0xFFFFFC2Fu));
    return !ge;
  }
  ECG_D static void sqr_n(Fe& r, const Fe& a, int n) {
    r = a;
#pragma unroll 1
    for (int i = 0; i < n; i++) sqr(r, r);
  }
  // r = a^(p-2) (Fermat).  0 -> 0.  255 squarings + 15 multiplications; the chain is the usual one for
  // p-2 = 2^256 - 2^32 - 979 (blocks of 223 ones, a zero, 22 ones, 0000, 101101).  The reference reaches
  // the same value through crypto-bigint's safegcd (k256/src/arithmetic/field.rs:178-196).
  ECG_D static void inv(Fe& r, const Fe& a) {
    Fe x2, x3, x6, x9, x11, x22, x44, x88, x176, x220, x223, t;
    sqr(x2, a);
    mul(x2, x2, a);
    sqr(x3, x2);
    mul(x3, x3, a);
    sqr_n(x6, x3, 3);
    mul(x6, x6, x3);
    sqr_n(x9, x6, 3);
    mul(x9, x9, x3);
    sqr_n(x11, x9, 2);
    mul(x11, x11, x2);
    sqr_n(x22, x11, 11);
    mul(x22, x22, x11);
    sqr_n(x44, x22, 22);
    mul(x44, x44, x22);
    sqr_n(x88, x44, 44);
    mul(x88, x88, x44);
    sqr_n(x176, x88, 88);
    mul(x176, x176, x88);
    sqr_n(x220, x176, 44);
    mul(x220, x220, x44);
    sqr_n(x223, x220, 3);
    mul(x223, x223, x3);
    sqr_n(t, x223, 23);
    mul(t, t, x22);
    sqr_n(t, t, 5);
    mul(t, t, a);
    sqr_n(t, t, 3);
    mul(t, t, x2);
    sqr_n(t, t, 2);
    mul(r, t, a);
  }
  // boundary encoding: the C ABI speaks canonical integers; this field's internal form is the integer
  // itself, so these are (near) identities.  (P-256 converts to/from the Montgomery domain here.)
  ECG_D static void from_canonical(Fe& r, const Fe& a) { r = a; }
  ECG_D static void to_canonical(Fe& r, const Fe& a) { normalize(r, a); }
};

typedef FpK256T<ECG_K256_OPT> FpK256;
// the policy of k256_varbase_kernel: every field operation inlined, and work moved off the multiplier (OPT bits 13-15):
// beta*x in the window table, 3/2 X^2 by carry chains, Y3 of both point operations with one reduction
typedef FpK256T<1 | 8192 | 16384 | 32768> FpK256Inline;

}  // namespace ecg
