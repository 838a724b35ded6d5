// ecg_kernels.cuh — every __global__ kernel of libecgpu.so except the microbenchmarks (ecg_microbench.cuh) and the
// bucket-method kernels (ecg_msm.cuh).  Host orchestration (contexts, lanes, staging, launches) is in ecgpu.cu.
#pragma once
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#else
// Host build: only tests/sim/sim.cpp, which executes a kernel body once per simulated thread (it supplies threadIdx,
// blockIdx, blockDim, gridDim, the atomics, uint4 and __ldg; ECG_KERNEL / ECG_DEV come from ecg_prim.cuh).  Never
// part of libecgpu.so.
#ifndef ECG_HOST_SIM
#error "ecg_kernels.cuh is CUDA code; a host build exists only for the test simulation (tests/sim/sim.cpp)"
#endif
#endif

#include "../../include/ecgpu.h"
#include "ecg_curves.cuh"
#include "ecg_io.cuh"
#include "ecg_mul.cuh"
#include "ecg_verify.cuh"

using namespace ecg;

// ------------------------------------------------------------------------------------------------
// error flags written by kernels into status[0]; status[1] = smallest offending index
#define ERRF_SCALAR 1u
#define ERRF_POINT 2u
#define ERRF_SKEW 4u /* not an error: the bucket method declined a skewed input (MSM_SKEW_FLAG, ecg_msm.cuh) */

ECG_DEV void report_error(uint32_t* status, uint32_t flag, size_t idx) {
  atomicOr(&status[0], flag);
  atomicMin(&status[1], (uint32_t)(idx > 0xFFFFFFFEull ? 0xFFFFFFFEull : idx));
}

// SoA word-major intermediate layout: word w of element idx at buf[w*n + idx] (coalesced per word)
template <int NW>
ECG_DEV void soa_store(uint32_t* buf, size_t n, size_t idx, const uint32_t* v, int w0) {
#pragma unroll
  for (int w = 0; w < NW; w++) buf[(size_t)(w0 + w) * n + idx] = v[w];
}
template <int NW>
ECG_DEV void soa_load(uint32_t* v, const uint32_t* buf, size_t n, size_t idx, int w0) {
#pragma unroll
  for (int w = 0; w < NW; w++) v[w] = buf[(size_t)(w0 + w) * n + idx];
}

// Load + validate one (scalar, point) pair.  Returns error flags (0 = fine).  On error / identity the
// caller still runs the arithmetic on a harmless substitute (k = 1, P = G) and forces Z = 0 afterwards so
// that warps stay converged.
template <class C>
ECG_DEV uint32_t load_pair(uint32_t* k, typename C::F::AffT& P, bool& inf, const uint8_t* kb,
                                              const uint8_t* pxy, const uint8_t* pinf, size_t idx) {
  typedef typename C::F F;
  typedef typename F::FeT Fe;
  constexpr int NL = F::NL, FB = F::FB;  // limbs and bytes per field element / scalar
  uint32_t err = 0;
  load_fe<F>(k, kb + FB * idx);
  if (!ltN<NL>(k, C::N())) err |= ERRF_SCALAR;
  inf = pinf != nullptr && pinf[idx] != 0;
  Fe x, y;
  load_fe<F>(x.v, pxy + 2 * FB * idx);
  load_fe<F>(y.v, pxy + 2 * FB * idx + FB);
  if (!inf) {
    bool ok = ltN<NL>(x.v, C::P()) && ltN<NL>(y.v, C::P());
    F::from_canonical(P.x, x);
    F::from_canonical(P.y, y);
    if (ok) {
      Fe b;
      C::b_internal(b);
      ok = aff_on_curve<F, C::A_IS_MINUS3>(P, b);
    }
    if (!ok) err |= ERRF_POINT;
  }
  if (inf || err) {
    C::generator(P);
#pragma unroll
    for (int i = 0; i < NL; i++) k[i] = (i == 0);
  }
  return err;
}

// ------------------------------------------------------------------------------------------------
// Per-thread window tables live in global memory, one slot per block: word w of entry e of thread t at
// gtab[blockIdx*BLOCK*EW + (e*WPE + w)*BLOCK + t]  (EW = words per thread: 192 for 8 secp256k1 entries of (x, y, beta*x)
// and for 8 Jacobian P-256 entries).
// A warp's access to one (e, w) of differing e per lane touches 32 distinct 4-byte words spread over at most 8
// rows; the blocks resident at any time on the 132 SMs of an H100 keep 52 MB (secp256k1) to 65 MB (P-256) of tables live
// against its 50 MB L2 (a pair reads ~7 KB of table, so what spills costs little HBM bandwidth).  Shared memory
// was the first home of these tables (512-768 B/thread capped occupancy at 8-12 warps/SM); moving them out lets
// registers set the occupancy (16-20 warps/SM); tools/kbench.cu times both homes.
// secp256k1 slots: 8 affine entries x 24 words (x, y, beta*x) for k256_varbase_kernel; the constant-time and a*G + b*P
// kernels keep 16-word entries (x, y) in the first 128 words of a slot of the same size.
#define K_TAB_WORDS 192
#define P_TAB_WORDS 192  /* 8 Jacobian entries x 24 words */

// secp256k1 variable-base: one pair per thread.
// Field operations fully inlined (FpK256Inline, ecg_fe_k256.cuh: no call marshalling) with a block-wide barrier between the doubling phase
// and the addition phase of every window (k256_mul_thread<.., 1>): all warps of a block then run the same stretch of
// code, so only one phase's instructions have to be resident in the instruction cache at a time — the fully inlined
// body without the barriers thrashes it, the call-based body pays ~21 IMAD.MOV per call on the FMA pipe
// (tools/kbench.cu times the three forms).
// Every thread of a block must reach the barriers: out-of-range threads redo the block's last valid pair and store nothing.
template <int BLOCK, int MINBLK>
ECG_KERNEL(BLOCK, MINBLK)
    k256_varbase_kernel(const uint8_t* __restrict__ kb, const uint8_t* __restrict__ pxy,
                        const uint8_t* __restrict__ pinf, size_t n, uint32_t* __restrict__ jac,
                        uint32_t* __restrict__ gtab, uint32_t* __restrict__ status, size_t base) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  const bool live = idx < n;
  const size_t cidx = live ? idx : n - 1;
  uint32_t k[8];
  Aff P;
  bool inf;
  uint32_t err = load_pair<CurveK256>(k, P, inf, kb, pxy, pinf, cidx);
  if (err && live) report_error(status, err, base + idx);
  K256TabRef<FpK256Inline> tab{gtab + (size_t)blockIdx.x * BLOCK * K_TAB_WORDS + threadIdx.x, (uint32_t)BLOCK};
  Jac r;
  k256_mul_thread<FpK256Inline, 1>(r, k, P, tab);
  if (!live) return;
  if (inf || err) FpK256::set_zero(r.Z);
  soa_store<8>(jac, n, idx, r.X.v, 0);
  soa_store<8>(jac, n, idx, r.Y.v, 8);
  soa_store<8>(jac, n, idx, r.Z.v, 16);
}

// ------------------------------------------------------------------------------------------------
// ECG_FLAG_CONSTTIME kernels: load_pair, or — with pxy == nullptr — the scalar alone with P = G (mul_by_generator through
// the variable-base routine, like the reference's mul_backend::VariableOnly: no table indexed by 16 secret bits)
template <class C>
ECG_DEV uint32_t load_pair_or_generator(uint32_t* k, typename C::F::AffT& P, bool& inf, const uint8_t* kb, const uint8_t* pxy,
                                        const uint8_t* pinf, size_t idx) {
  typedef typename C::F F;
  if (pxy != nullptr) return load_pair<C>(k, P, inf, kb, pxy, pinf, idx);
  inf = false;
  load_fe<F>(k, kb + F::FB * idx);
  C::generator(P);
  if (ltN<F::NL>(k, C::N())) return 0;
#pragma unroll
  for (int i = 0; i < F::NL; i++) k[i] = (i == 0);
  return ERRF_SCALAR;
}

// secp256k1 variable-base with scalar-independent addresses and sign handling (call-based field operations)
template <int BLOCK, int MINBLK>
ECG_KERNEL(BLOCK, MINBLK)
    k256_varbase_ct_kernel(const uint8_t* __restrict__ kb, const uint8_t* __restrict__ pxy, const uint8_t* __restrict__ pinf, size_t n,
                           uint32_t* __restrict__ jac, uint32_t* __restrict__ gtab, uint32_t* __restrict__ status, size_t base) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[8];
  Aff P;
  bool inf;
  uint32_t err = load_pair_or_generator<CurveK256>(k, P, inf, kb, pxy, pinf, idx);
  if (err) report_error(status, err, base + idx);
  TabRef tab{gtab + (size_t)blockIdx.x * BLOCK * K_TAB_WORDS + threadIdx.x, (uint32_t)BLOCK};
  Jac r;
  k256_mul_thread<FpK256, 0, true>(r, k, P, tab);
  if (inf || err) FpK256::set_zero(r.Z);
  soa_store<8>(jac, n, idx, r.X.v, 0);
  soa_store<8>(jac, n, idx, r.Y.v, 8);
  soa_store<8>(jac, n, idx, r.Z.v, 16);
}

// ------------------------------------------------------------------------------------------------
// Generic prime-order curve (P-256) variable-base: Jacobian window table (768 B / thread).
// CT: the ECG_FLAG_CONSTTIME variant (masked table scan; pxy == nullptr selects the generator)
template <class C, int BLOCK, int MINBLK, bool CT = false>
ECG_KERNEL(BLOCK, MINBLK)
    generic_varbase_kernel(const uint8_t* __restrict__ kb, const uint8_t* __restrict__ pxy,
                           const uint8_t* __restrict__ pinf, size_t n, uint32_t* __restrict__ jac,
                           uint32_t* __restrict__ gtab, uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  constexpr int NL = F::NL;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[NL];
  typename F::AffT P;
  bool inf;
  uint32_t err = CT ? load_pair_or_generator<C>(k, P, inf, kb, pxy, pinf, idx) : load_pair<C>(k, P, inf, kb, pxy, pinf, idx);
  if (err) report_error(status, err, base + idx);
  TabRefJN<NL> tab{gtab + (size_t)blockIdx.x * BLOCK * (8 * 3 * NL) + threadIdx.x, (uint32_t)BLOCK};  // 8 Jacobian entries
  typename F::JacT r;
  generic_mul_thread<F, C::A_IS_MINUS3, 0, CT>(r, k, P, tab);
  if (inf || err) F::set_zero(r.Z);
  soa_store<NL>(jac, n, idx, r.X.v, 0);
  soa_store<NL>(jac, n, idx, r.Y.v, NL);
  soa_store<NL>(jac, n, idx, r.Z.v, 2 * NL);
}

// ------------------------------------------------------------------------------------------------
// Fixed-base k*G from a device-resident table of affine odd multiples.
//   table layout: window i (0..FB_WINDOWS-1), entry j (0..2^(FB_W-1)-1) = (2j+1) * 2^(FB_W*i) * G, 16 words
//   (x[8], y[8], internal form); one extra entry at the end = 2^256 * G (the recoding's implicit top digit).
// Replaces BasepointTable (primeorder/src/tables/basepoint.rs:41-125; k256/src/arithmetic/tables.rs:12-22):
// same idea (precomputed multiples of G, only additions at run time), sized for the 50 MB L2 (32 MiB) instead of a
// 30 KiB L1: 16 sixteen-bit windows -> 17 mixed additions and no doubling per scalar.
#define FB_W 16
#define FB_ENTRIES (1u << (FB_W - 1))
// 16-bit windows over an NL-limb scalar: 2*NL windows (16 for the 256-bit curves, 24 for P-384) + the implicit top digit
#define FB_WINDOWS_NL(NL) (2 * (NL))
#define FB_TABLE_POINTS_NL(NL) ((size_t)FB_WINDOWS_NL(NL) * FB_ENTRIES + 1)
#define FB_WINDOWS FB_WINDOWS_NL(8)
#define FB_TABLE_POINTS FB_TABLE_POINTS_NL(8)

template <int NL>
ECG_DEV void fb_load_entry(AffN<NL>& e, const uint32_t* __restrict__ table, size_t point) {
  load_aff_entry<NL>(e, table, point);
}

// acc += k*G (acc Jacobian on the true curve; pass Z = 0 to start from the identity)
template <class C, bool FROM_IDENTITY>
ECG_DEV void fixedbase_accumulate(typename C::F::JacT& acc, const uint32_t* k, const uint32_t* __restrict__ table) {
  typedef typename C::F F;
  constexpr int NL = F::NL, NW = FB_WINDOWS_NL(F::NL);
  FullRecodeN<NL> rc;
  recode_full<NL>(rc, k);
  typename F::AffT e;
  fb_load_entry<NL>(e, table, (size_t)NW * FB_ENTRIES);  // 2^(32 NL) * G
  if (FROM_IDENTITY) {
    acc.X = e.x;
    acc.Y = e.y;
    F::set_one(acc.Z);
  } else {
    jac_madd<F, C::A_IS_MINUS3>(acc, acc, e);
  }
#pragma unroll 1
  for (int i = 0; i < NW; i++) {
    uint32_t w = rc.h[0] & 0xFFFFu;
#pragma unroll
    for (int j = 0; j < NL - 1; j++) rc.h[j] = funnel_r(rc.h[j], rc.h[j + 1], 16);
    rc.h[NL - 1] >>= 16;
    uint32_t pos = w >> (FB_W - 1);
    uint32_t idx = pos ? (w & (FB_ENTRIES - 1)) : (FB_ENTRIES - 1 - w);
    fb_load_entry<NL>(e, table, (size_t)i * FB_ENTRIES + idx);
    fe_cneg<F>(e.y, pos ^ 1u);
    jac_madd<F, C::A_IS_MINUS3>(acc, acc, e);
  }
  // parity correction: subtract G if k was even
  fb_load_entry<NL>(e, table, 0);
  F::neg(e.y, e.y);
  typename F::JacT t;
  jac_madd<F, C::A_IS_MINUS3>(t, acc, e);
  jac_csel(acc, t, rc.even);
}

template <class C>
ECG_KERNEL(128, 4)
    fixedbase_kernel(const uint8_t* __restrict__ kb, size_t n, const uint32_t* __restrict__ table,
                     uint32_t* __restrict__ jac, uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  constexpr int NL = F::NL;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[NL];
  load_fe<F>(k, kb + F::FB * idx);
  bool bad = !ltN<NL>(k, C::N());
  if (bad) {
    report_error(status, ERRF_SCALAR, base + idx);
#pragma unroll
    for (int i = 0; i < NL; i++) k[i] = (i == 0);
  }
  typename F::JacT acc;
  fixedbase_accumulate<C, true>(acc, k, table);
  if (bad) F::set_zero(acc.Z);
  soa_store<NL>(jac, n, idx, acc.X.v, 0);
  soa_store<NL>(jac, n, idx, acc.Y.v, NL);
  soa_store<NL>(jac, n, idx, acc.Z.v, 2 * NL);
}

// a*G + b*P : variable-base thread routine, then the fixed-base accumulation on the same accumulator.
// Replaces mul_by_generator_and_mul_add_vartime (k256/src/arithmetic/mul.rs:303-310, primeorder/src/mul_backend.rs:31-40).
template <class C, int BLOCK, int MINBLK, bool IS_K256>
ECG_KERNEL(BLOCK, MINBLK)
    mul_gen_add_kernel(const uint8_t* __restrict__ ab, const uint8_t* __restrict__ kb,
                       const uint8_t* __restrict__ pxy, const uint8_t* __restrict__ pinf, size_t n,
                       const uint32_t* __restrict__ table, uint32_t* __restrict__ jac, uint32_t* __restrict__ gtab,
                       uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[8], a[8];
  Aff P;
  bool inf;
  uint32_t err = load_pair<C>(k, P, inf, kb, pxy, pinf, idx);
  load_be32(a, ab + 32 * idx);
  if (!lt8(a, C::N())) err |= ERRF_SCALAR;
  if (err) report_error(status, err, base + idx);
  Jac r;
  if (IS_K256) {
    TabRef tab{gtab + (size_t)blockIdx.x * BLOCK * K_TAB_WORDS + threadIdx.x, (uint32_t)BLOCK};
    k256_mul_thread(r, k, P, tab);
  } else {
    TabRefJ tab{gtab + (size_t)blockIdx.x * BLOCK * P_TAB_WORDS + threadIdx.x, (uint32_t)BLOCK};
    generic_mul_thread<F, C::A_IS_MINUS3>(r, k, P, tab);
  }
  if (inf) F::set_zero(r.Z);  // b * O = O, the sum is a*G
  if (err) {
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = (i == 0);
  }
  fixedbase_accumulate<C, false>(r, a, table);
  if (err) F::set_zero(r.Z);
  soa_store<8>(jac, n, idx, r.X.v, 0);
  soa_store<8>(jac, n, idx, r.Y.v, 8);
  soa_store<8>(jac, n, idx, r.Z.v, 16);
}

// ------------------------------------------------------------------------------------------------
// Signature verification front ends (ecg_verify.cuh).  Both reduce to a*G + b*P through mul_gen_add_kernel; the
// kernels here prepare (a, b, P) and judge the result.  Invalid encodings never raise an API error: they are
// marked not-ok, replaced by harmless operands (a = b = 1, P = G) so warps stay converged, and reported as
// valid[i] = 0 — the reference returns Err(Error) per signature, not a batch failure.
ECG_DEV void store_scalar_be(uint8_t* dst, const uint32_t* limbs) { store_be32(dst, limbs); }

#if !defined(ECG_TU) || ECG_TU == 0  // not templates: defined by the translation unit of the 256-bit curves only
// BIP340: pk (x only), 32-byte message, signature r || s.
ECG_KERNEL(128)
    schnorr_prep_kernel(const uint8_t* __restrict__ pk, const uint8_t* __restrict__ msg, const uint8_t* __restrict__ sig, size_t n,
                        uint8_t* __restrict__ pxy, uint8_t* __restrict__ a_out, uint8_t* __restrict__ b_out, uint8_t* __restrict__ ok_out) {
  typedef FpK256 F;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t x[8], r[8], sv[8], e[8];
  load_be32(x, pk + 32 * idx);
  load_be32(r, sig + 64 * idx);
  load_be32(sv, sig + 64 * idx + 32);
  Aff P;
  bool ok = k256_lift_x<F>(P, x);                    // VerifyingKey::from_bytes (schnorr/verifying.rs:36-52)
  ok = ok && lt8(r, K256_P);                           // Signature::try_from: r is a field element,
  ok = ok && lt8(sv, K256_N) && !FnMont<CurveK256>::is_zero(sv);  //   s a non-zero scalar (schnorr.rs:150-170)
  bip340_challenge(e, sig + 64 * idx, pk + 32 * idx, msg + 32 * idx);
  if (!lt8(e, K256_N)) {  // Reduce<FieldBytes>: one conditional subtraction (2^256 < 2n)
    uint32_t t[8];
    sub8(t, e, K256_N);
#pragma unroll
    for (int i = 0; i < 8; i++) e[i] = t[i];
  }
  // b = -e mod n
  uint32_t ne[8];
  if (FnMont<CurveK256>::is_zero(e)) {
#pragma unroll
    for (int i = 0; i < 8; i++) ne[i] = 0;
  } else {
    sub8(ne, K256_N, e);
  }
  if (!ok) {
    CurveK256::generator(P);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      sv[i] = (i == 0);
      ne[i] = (i == 0);
    }
  }
  Fe cx, cy;
  F::to_canonical(cx, P.x);
  F::to_canonical(cy, P.y);
  store_be32(pxy + 64 * idx, cx.v);
  store_be32(pxy + 64 * idx + 32, cy.v);
  store_scalar_be(a_out + 32 * idx, sv);
  store_scalar_be(b_out + 32 * idx, ne);
  ok_out[idx] = ok ? 1 : 0;
}
ECG_KERNEL(256)
    schnorr_check_kernel(const uint8_t* __restrict__ sig, const uint8_t* __restrict__ rxy, const uint8_t* __restrict__ rinf,
                         const uint8_t* __restrict__ ok, size_t n, uint8_t* __restrict__ valid) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const uint32_t* r = reinterpret_cast<const uint32_t*>(sig + 64 * idx);
  const uint32_t* x = reinterpret_cast<const uint32_t*>(rxy + 64 * idx);
  bool same = true;
#pragma unroll
  for (int i = 0; i < 8; i++) same = same && (r[i] == x[i]);
  bool y_even = (rxy[64 * idx + 63] & 1u) == 0;
  valid[idx] = (ok[idx] && !rinf[idx] && y_even && same) ? 1 : 0;  // verifying.rs:94
}

#endif

// ECDSA: z (32-byte hash), signature r || s, public key Q (x || y).  One modular inversion per thread slice
// (Montgomery's trick over s_i, as in normalize_kernel); scr: 8*n words.
template <class C>
ECG_KERNEL(128)
    ecdsa_prep_kernel(const uint8_t* __restrict__ zb, const uint8_t* __restrict__ sig, const uint8_t* __restrict__ qxy, size_t n,
                      int low_s_only, uint32_t* __restrict__ scr, uint8_t* __restrict__ pxy, uint8_t* __restrict__ a_out,
                      uint8_t* __restrict__ b_out, uint8_t* __restrict__ ok_out) {
  typedef typename C::F F;
  typedef FnMont<C> N;
  size_t T = (size_t)gridDim.x * blockDim.x;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  uint32_t acc[8], sm[8];
#pragma unroll
  for (int i = 0; i < 8; i++) acc[i] = C::N_ONE()[i];
  size_t last = t;
  // forward: validate, prefix products of the (Montgomery-form) s_i
  for (size_t idx = t; idx < n; idx += T) {
    uint32_t r[8], sv[8];
    load_be32(r, sig + 64 * idx);
    load_be32(sv, sig + 64 * idx + 32);
    bool ok = lt8(r, C::N()) && !N::is_zero(r) && lt8(sv, C::N()) && !N::is_zero(sv);
    if (ok && low_s_only) {  // EcdsaCurve::NORMALIZE_S (k256/src/ecdsa.rs:104-106): reject s > n/2
      uint32_t twice[8];
      uint32_t c = add8(twice, sv, sv);
      ok = !c && lt8(twice, C::N());
    }
    Aff Q;
    Fe qx, qy;
    load_be32(qx.v, qxy + 64 * idx);
    load_be32(qy.v, qxy + 64 * idx + 32);
    bool qok = lt8(qx.v, C::P()) && lt8(qy.v, C::P());
    F::from_canonical(Q.x, qx);
    F::from_canonical(Q.y, qy);
    if (qok) {
      Fe b;
      C::b_internal(b);
      qok = aff_on_curve<F, C::A_IS_MINUS3>(Q, b);
    }
    ok = ok && qok;
    ok_out[idx] = ok ? 1 : 0;
    if (!ok) {
#pragma unroll
      for (int i = 0; i < 8; i++) sv[i] = (i == 0);
    }
    N::to_mont(sm, sv);
    soa_store<8>(scr, n, idx, acc, 0);
    N::mul(acc, acc, sm);
    last = idx;
  }
  uint32_t inv[8];
  N::inv(inv, acc);
  for (size_t idx = last;; idx -= T) {
    uint32_t r[8], sv[8], z[8], pre[8], w[8], u1[8], u2[8];
    bool ok = ok_out[idx] != 0;
    load_be32(r, sig + 64 * idx);
    load_be32(sv, sig + 64 * idx + 32);
    load_be32(z, zb + 32 * idx);
    if (!ok) {
#pragma unroll
      for (int i = 0; i < 8; i++) sv[i] = (i == 0);
    }
    N::to_mont(sm, sv);
    soa_load<8>(pre, scr, n, idx, 0);
    N::mul(w, inv, pre);   // w = s^-1 (Montgomery form)
    N::mul(inv, inv, sm);
    N::cond_sub_n(z, N::ge_n(z));  // bits2field + reduce for 256-bit curves
    // u1 = z*w, u2 = r*w: mont_mul(plain, mont) = plain product
    N::mul(u1, z, w);
    N::mul(u2, r, w);
    if (!ok) {
#pragma unroll
      for (int i = 0; i < 8; i++) {
        u1[i] = (i == 0);
        u2[i] = (i == 0);
      }
      Aff G;
      C::generator(G);
      Fe gx, gy;
      F::to_canonical(gx, G.x);
      F::to_canonical(gy, G.y);
      store_be32(pxy + 64 * idx, gx.v);
      store_be32(pxy + 64 * idx + 32, gy.v);
    } else {
#pragma unroll
      for (int i = 0; i < 16; i++) reinterpret_cast<uint32_t*>(pxy + 64 * idx)[i] = reinterpret_cast<const uint32_t*>(qxy + 64 * idx)[i];
    }
    store_scalar_be(a_out + 32 * idx, u1);
    store_scalar_be(b_out + 32 * idx, u2);
    if (idx < T) break;
  }
}
template <class C>
ECG_KERNEL(256)
    ecdsa_check_kernel(const uint8_t* __restrict__ sig, const uint8_t* __restrict__ rxy, const uint8_t* __restrict__ rinf,
                       const uint8_t* __restrict__ ok, size_t n, uint8_t* __restrict__ valid) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t r[8], x[8];
  load_be32(r, sig + 64 * idx);
  load_be32(x, rxy + 64 * idx);
  FnMont<C>::cond_sub_n(x, FnMont<C>::ge_n(x));  // x(R) mod n  (p < 2n)
  bool same = true;
#pragma unroll
  for (int i = 0; i < 8; i++) same = same && (r[i] == x[i]);
  valid[idx] = (ok[idx] && !rinf[idx] && same) ? 1 : 0;
}

// Public-key recovery (ecdsa_core::VerifyingKey::recover_from_prehash, the Ethereum `ecrecover` shape; k256/src/ecdsa.rs:45-88,
// vectors :182-262): R = decompress(r [+ n if recid bit 1], y odd = recid bit 0); Q = r^-1 (s R - z G) = u1*G + u2*R with
// u1 = -z r^-1, u2 = s r^-1.  recid: one byte per signature, RecoveryId::to_byte (0..3).
// Two front-end kernels: the square root of the decompression is the expensive part and runs one thread per signature;
// the inversion of the r_i is shared per thread slice (Montgomery's trick) in a second, strided kernel.
template <class C>
ECG_KERNEL(128)
    ecdsa_recover_point_kernel(const uint8_t* __restrict__ sig, const uint8_t* __restrict__ recid, size_t n, int low_s_only,
                               uint8_t* __restrict__ pxy, uint8_t* __restrict__ ok_out) {
  typedef typename C::F F;
  typedef FnMont<C> N;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t r[8], sv[8], x[8];
  load_be32(r, sig + 64 * idx);
  load_be32(sv, sig + 64 * idx + 32);
  const uint32_t id = recid[idx];
  bool ok = id < 4 && lt8(r, C::N()) && !N::is_zero(r) && lt8(sv, C::N()) && !N::is_zero(sv);
  if (ok && low_s_only) {  // the closing verify_prehash of a NORMALIZE_S curve refuses s > n/2
    uint32_t twice[8];
    uint32_t c = add8(twice, sv, sv);
    ok = !c && lt8(twice, C::N());
  }
#pragma unroll
  for (int i = 0; i < 8; i++) x[i] = r[i];
  if (id & 2u) {  // is_x_reduced: the x coordinate of R was r + n (checked_add: no wrap past 2^256; decompress refuses x >= p)
    uint32_t c = add8(x, r, C::N());
    ok = ok && !c;
  }
  Aff R;
  ok = ok && sec1_decompress<C>(R, x, id & 1u);
  Fe cx, cy;
  if (!ok) C::generator(R);  // a harmless stand-in keeps the middle kernel's input checks quiet; the verdict is already 0
  F::to_canonical(cx, R.x);
  F::to_canonical(cy, R.y);
  store_be32(pxy + 64 * idx, cx.v);
  store_be32(pxy + 64 * idx + 32, cy.v);
  ok_out[idx] = ok ? 1 : 0;
}
// scr: 8 * n words
template <class C>
ECG_KERNEL(128)
    ecdsa_recover_prep_kernel(const uint8_t* __restrict__ zb, const uint8_t* __restrict__ sig, const uint8_t* __restrict__ ok_in, size_t n,
                              uint32_t* __restrict__ scr, uint8_t* __restrict__ a_out, uint8_t* __restrict__ b_out) {
  typedef FnMont<C> N;
  size_t T = (size_t)gridDim.x * blockDim.x;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  uint32_t acc[8], rm[8];
#pragma unroll
  for (int i = 0; i < 8; i++) acc[i] = C::N_ONE()[i];
  size_t last = t;
  for (size_t idx = t; idx < n; idx += T) {
    uint32_t r[8];
    load_be32(r, sig + 64 * idx);
    if (!ok_in[idx]) {
#pragma unroll
      for (int i = 0; i < 8; i++) r[i] = (i == 0);
    }
    N::to_mont(rm, r);
    soa_store<8>(scr, n, idx, acc, 0);
    N::mul(acc, acc, rm);
    last = idx;
  }
  uint32_t inv[8];
  N::inv(inv, acc);
  for (size_t idx = last;; idx -= T) {
    uint32_t r[8], sv[8], z[8], pre[8], w[8], u1[8], u2[8];
    bool ok = ok_in[idx] != 0;
    load_be32(r, sig + 64 * idx);
    load_be32(sv, sig + 64 * idx + 32);
    load_be32(z, zb + 32 * idx);
    if (!ok) {
#pragma unroll
      for (int i = 0; i < 8; i++) r[i] = (i == 0);
    }
    N::to_mont(rm, r);
    soa_load<8>(pre, scr, n, idx, 0);
    N::mul(w, inv, pre);  // w = r^-1 (Montgomery form)
    N::mul(inv, inv, rm);
    N::cond_sub_n(z, N::ge_n(z));
    N::mul(u1, z, w);  // z r^-1, then negated mod n
    N::mul(u2, sv, w);
    if (!N::is_zero(u1)) {
      uint32_t neg[8];
      sub8(neg, C::N(), u1);
#pragma unroll
      for (int i = 0; i < 8; i++) u1[i] = neg[i];
    }
    if (!ok) {
#pragma unroll
      for (int i = 0; i < 8; i++) {
        u1[i] = (i == 0);
        u2[i] = (i == 0);
      }
    }
    store_scalar_be(a_out + 32 * idx, u1);
    store_scalar_be(b_out + 32 * idx, u2);
    if (idx < T) break;
  }
}
// after the normalisation wrote x || y and the identity flag: valid = front end ok and Q != O (VerifyingKey::from_affine);
// the flag array becomes the verdict, refused records come back as 64 zero bytes
template <int ECG_ONCE = 0>  // a template only so that several translation units may define it
ECG_KERNEL(256)
    ecdsa_recover_finish_kernel(uint8_t* __restrict__ out_xy, uint8_t* __restrict__ inf_to_valid, const uint8_t* __restrict__ ok, size_t n) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  bool v = ok[idx] && !inf_to_valid[idx];
  if (!v) {
#pragma unroll
    for (int i = 0; i < 16; i++) reinterpret_cast<uint32_t*>(out_xy + 64 * idx)[i] = 0;
  }
  inf_to_valid[idx] = v ? 1 : 0;
}

// ---- the same two entries for every other curve with ECDSA in the reference (p192, p224, p384, p521, brainpoolP256r1/t1,
// brainpoolP384r1/t1: */src/ecdsa.rs) — generic twins over the field policy's limb count, arithmetic mod n through
// ScalarField<C>::T (the Montgomery policy of ecg_fe_mont.cuh instantiated over the group order) ----------------------

// a*G + b*P (MulBackend::mul_by_generator_and_mul_add_vartime, primeorder/src/mul_backend.rs:31-40): the variable-base
// thread routine, then the fixed-base accumulation on the same accumulator
template <class C, int BLOCK, int MINBLK>
ECG_KERNEL(BLOCK, MINBLK)
    mul_gen_add_generic_kernel(const uint8_t* __restrict__ ab, const uint8_t* __restrict__ kb, const uint8_t* __restrict__ pxy,
                               const uint8_t* __restrict__ pinf, size_t n, const uint32_t* __restrict__ table, uint32_t* __restrict__ jac,
                               uint32_t* __restrict__ gtab, uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  constexpr int NL = F::NL;
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[NL], a[NL];
  typename F::AffT P;
  bool inf;
  uint32_t err = load_pair<C>(k, P, inf, kb, pxy, pinf, idx);
  load_fe<F>(a, ab + F::FB * idx);
  if (!ltN<NL>(a, C::N())) err |= ERRF_SCALAR;
  if (err) report_error(status, err, base + idx);
  TabRefJN<NL> tab{gtab + (size_t)blockIdx.x * BLOCK * (8 * 3 * NL) + threadIdx.x, (uint32_t)BLOCK};
  typename F::JacT r;
  generic_mul_thread<F, C::A_IS_MINUS3>(r, k, P, tab);
  if (inf) F::set_zero(r.Z);  // b * O = O, the sum is a*G
  if (err) {
#pragma unroll
    for (int i = 0; i < NL; i++) a[i] = (i == 0);
  }
  fixedbase_accumulate<C, false>(r, a, table);
  if (err) F::set_zero(r.Z);
  soa_store<NL>(jac, n, idx, r.X.v, 0);
  soa_store<NL>(jac, n, idx, r.Y.v, NL);
  soa_store<NL>(jac, n, idx, r.Z.v, 2 * NL);
}

// ECDSA front end: z (FB-byte prehash, already through bits2field), signature r || s (2 FB), public key x || y (2 FB).
// One inversion mod n per thread slice (Montgomery's trick over the s_i); scr: NL * n words.
template <class C>
ECG_KERNEL(128)
    ecdsa_prep_generic_kernel(const uint8_t* __restrict__ zb, const uint8_t* __restrict__ sig, const uint8_t* __restrict__ qxy, size_t n,
                              int low_s_only, uint32_t* __restrict__ scr, uint8_t* __restrict__ pxy, uint8_t* __restrict__ a_out,
                              uint8_t* __restrict__ b_out, uint8_t* __restrict__ ok_out) {
  typedef typename C::F F;
  typedef typename ScalarField<C>::T FN;
  typedef typename FN::FeT Sc;
  constexpr int NL = F::NL, FB = F::FB;
  size_t T = (size_t)gridDim.x * blockDim.x;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  Sc acc, sm;
  FN::set_one(acc);
  size_t last = t;
  // forward: validate, prefix products of the (Montgomery-form) s_i
  for (size_t idx = t; idx < n; idx += T) {
    Sc r, sv;
    load_fe<F>(r.v, sig + 2 * FB * idx);
    load_fe<F>(sv.v, sig + 2 * FB * idx + FB);
    bool ok = ltN<NL>(r.v, C::N()) && !FN::is_zero(r) && ltN<NL>(sv.v, C::N()) && !FN::is_zero(sv);
    if (ok && low_s_only) {  // EcdsaCurve::NORMALIZE_S: reject s > n/2 (false for all these curves in the reference)
      uint32_t twice[NL];
      uint32_t c = addN<NL>(twice, sv.v, sv.v);
      ok = !c && ltN<NL>(twice, C::N());
    }
    typename F::AffT Q;
    typename F::FeT qx, qy;
    load_fe<F>(qx.v, qxy + 2 * FB * idx);
    load_fe<F>(qy.v, qxy + 2 * FB * idx + FB);
    bool qok = ltN<NL>(qx.v, C::P()) && ltN<NL>(qy.v, C::P());
    F::from_canonical(Q.x, qx);
    F::from_canonical(Q.y, qy);
    if (qok) {
      typename F::FeT b;
      C::b_internal(b);
      qok = aff_on_curve<F, C::A_IS_MINUS3>(Q, b);
    }
    ok = ok && qok;
    ok_out[idx] = ok ? 1 : 0;
    if (!ok) {
#pragma unroll
      for (int i = 0; i < NL; i++) sv.v[i] = (i == 0);
    }
    FN::from_canonical(sm, sv);
    soa_store<NL>(scr, n, idx, acc.v, 0);
    FN::mul(acc, acc, sm);
    last = idx;
  }
  Sc inv;
  FN::inv(inv, acc);
  for (size_t idx = last;; idx -= T) {
    Sc r, sv, z, pre, w, u1, u2;
    bool ok = ok_out[idx] != 0;
    load_fe<F>(r.v, sig + 2 * FB * idx);
    load_fe<F>(sv.v, sig + 2 * FB * idx + FB);
    load_fe<F>(z.v, zb + FB * idx);
    if (!ok) {
#pragma unroll
      for (int i = 0; i < NL; i++) {
        sv.v[i] = (i == 0);
        r.v[i] = (i == 0);
      }
    }
    FN::from_canonical(sm, sv);
    soa_load<NL>(pre.v, scr, n, idx, 0);
    FN::mul(w, inv, pre);   // w = s^-1 (Montgomery form)
    FN::mul(inv, inv, sm);
    FN::from_canonical(z, z);  // z * R mod n for ANY z below 2^(32 NL): the reduction of the prehash (Reduce<FieldBytes> for Scalar)
    FN::from_canonical(r, r);
    FN::mul(u1, z, w);
    FN::mul(u2, r, w);
    FN::to_canonical(u1, u1);
    FN::to_canonical(u2, u2);
    if (!ok) {
#pragma unroll
      for (int i = 0; i < NL; i++) {
        u1.v[i] = (i == 0);
        u2.v[i] = (i == 0);
      }
      typename F::AffT G;
      C::generator(G);
      typename F::FeT gx, gy;
      F::to_canonical(gx, G.x);
      F::to_canonical(gy, G.y);
      store_fe<F>(pxy + 2 * FB * idx, gx.v);
      store_fe<F>(pxy + 2 * FB * idx + FB, gy.v);
    } else {
      for (int i = 0; i < 2 * FB; i++) pxy[2 * FB * idx + i] = qxy[2 * FB * idx + i];
    }
    store_fe<F>(a_out + FB * idx, u1.v);
    store_fe<F>(b_out + FB * idx, u2.v);
    if (idx < T) break;
  }
}
template <class C>
ECG_KERNEL(256)
    ecdsa_check_generic_kernel(const uint8_t* __restrict__ sig, const uint8_t* __restrict__ rxy, const uint8_t* __restrict__ rinf,
                               const uint8_t* __restrict__ ok, size_t n, uint8_t* __restrict__ valid) {
  typedef typename C::F F;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t r[NL], x[NL], t[NL];
  load_fe<F>(r, sig + 2 * FB * idx);
  load_fe<F>(x, rxy + 2 * FB * idx);
  uint32_t bw = subN<NL>(t, x, C::N());  // x(R) mod n: x < p < 2n (Hasse), one conditional subtraction
  bool same = true;
#pragma unroll
  for (int i = 0; i < NL; i++) same = same && (r[i] == (bw ? x[i] : t[i]));
  valid[idx] = (ok[idx] && !rinf[idx] && same) ? 1 : 0;
}

// SM2DSA verify_prehash (sm2/src/dsa/verifying.rs:138-175): r, s in [1, n-1]; t = r + s mod n != 0; (x1, y1) = s*G + t*Q;
// valid iff (e + x1) mod n == r.  No inversion: the front end only validates and forms t; the middle is the same a*G + b*P kernel.
template <class C>
ECG_KERNEL(128)
    sm2dsa_prep_kernel(const uint8_t* __restrict__ sig, const uint8_t* __restrict__ qxy, size_t n, uint8_t* __restrict__ pxy,
                       uint8_t* __restrict__ a_out, uint8_t* __restrict__ b_out, uint8_t* __restrict__ ok_out) {
  typedef typename C::F F;
  typedef typename ScalarField<C>::T FN;
  typedef typename FN::FeT Sc;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  Sc r, sv, t;
  load_fe<F>(r.v, sig + 2 * FB * idx);
  load_fe<F>(sv.v, sig + 2 * FB * idx + FB);
  bool ok = ltN<NL>(r.v, C::N()) && !FN::is_zero(r) && ltN<NL>(sv.v, C::N()) && !FN::is_zero(sv);
  if (!ok) {
#pragma unroll
    for (int i = 0; i < NL; i++) r.v[i] = sv.v[i] = (i == 0);
  }
  FN::add(t, r, sv);  // fully reduced operands: the sum is the canonical (r + s) mod n
  ok = ok && !FN::is_zero(t);
  typename F::AffT Q;
  typename F::FeT qx, qy;
  load_fe<F>(qx.v, qxy + 2 * FB * idx);
  load_fe<F>(qy.v, qxy + 2 * FB * idx + FB);
  bool qok = ltN<NL>(qx.v, C::P()) && ltN<NL>(qy.v, C::P());
  F::from_canonical(Q.x, qx);
  F::from_canonical(Q.y, qy);
  if (qok) {
    typename F::FeT b;
    C::b_internal(b);
    qok = aff_on_curve<F, C::A_IS_MINUS3>(Q, b);
  }
  ok = ok && qok;
  ok_out[idx] = ok ? 1 : 0;
  if (!ok) {  // a harmless stand-in (1*G + 1*G) keeps the middle kernel's input checks quiet; the verdict is already 0
#pragma unroll
    for (int i = 0; i < NL; i++) sv.v[i] = t.v[i] = (i == 0);
    typename F::AffT G;
    C::generator(G);
    F::to_canonical(qx, G.x);
    F::to_canonical(qy, G.y);
  }
  store_fe<F>(pxy + 2 * FB * idx, qx.v);
  store_fe<F>(pxy + 2 * FB * idx + FB, qy.v);
  store_fe<F>(a_out + FB * idx, sv.v);
  store_fe<F>(b_out + FB * idx, t.v);
}
template <class C>
ECG_KERNEL(256)
    sm2dsa_check_kernel(const uint8_t* __restrict__ eb, const uint8_t* __restrict__ sig, const uint8_t* __restrict__ rxy,
                        const uint8_t* __restrict__ rinf, const uint8_t* __restrict__ ok, size_t n, uint8_t* __restrict__ valid) {
  typedef typename C::F F;
  typedef typename ScalarField<C>::T FN;
  typedef typename FN::FeT Sc;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  Sc r, x, e, t, sum;
  load_fe<F>(r.v, sig + 2 * FB * idx);
  load_fe<F>(x.v, rxy + 2 * FB * idx);
  load_fe<F>(e.v, eb + FB * idx);
  // Scalar::reduce of a 32-byte value: both e < 2^256 and x < p are below 2n, one conditional subtraction each
  if (!subN<NL>(t.v, x.v, C::N())) x = t;
  if (!subN<NL>(t.v, e.v, C::N())) e = t;
  FN::add(sum, e, x);
  bool same = true;
#pragma unroll
  for (int i = 0; i < NL; i++) same = same && (r.v[i] == sum.v[i]);
  valid[idx] = (ok[idx] && !rinf[idx] && same) ? 1 : 0;
}

// SEC1 compressed points (33 bytes: 02/03 || x; 33 zero bytes = identity) -> affine x || y, identity flag, validity.
template <class C>
ECG_KERNEL(128)
    decompress_kernel(const uint8_t* __restrict__ sec1, size_t n, uint8_t* __restrict__ out_xy, uint8_t* __restrict__ out_inf,
                      uint8_t* __restrict__ valid) {
  typedef typename C::F F;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const uint8_t* rec = sec1 + 33 * idx;
  uint8_t tag = rec[0];
  uint32_t x[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {  // unaligned big-endian words
    const uint8_t* b = rec + 1 + 4 * (7 - i);
    x[i] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | b[3];
  }
  bool zero = (x[0] | x[1] | x[2] | x[3] | x[4] | x[5] | x[6] | x[7]) == 0;
  Aff P;
  bool ok = false, inf = false;
  if (tag == 0 && zero) {
    ok = inf = true;
  } else if (tag == 2 || tag == 3) {
    ok = sec1_decompress<C>(P, x, tag & 1u);
  }
  Fe cx, cy;
  if (ok && !inf) {
    F::to_canonical(cx, P.x);
    F::to_canonical(cy, P.y);
  } else {
    F::set_zero(cx);
    F::set_zero(cy);
  }
  store_be32(out_xy + 64 * idx, cx.v);
  store_be32(out_xy + 64 * idx + 32, cy.v);
  out_inf[idx] = inf ? 1 : 0;
  valid[idx] = ok ? 1 : 0;
}

// ---- SEC1 decompression and the field square root for the other curves with p = 3 (mod 4) (everything except P-224) -----
// r = a^((p+1)/4) by fixed 4-bit windows over the public exponent; E supplies PP14(i), the limbs of (p + 1) / 4
template <class F, class E>
ECG_DEV void sqrt_candidate_generic(typename F::FeT& r, const typename F::FeT& a) {
  typename F::FeT tab[16], acc;
  F::set_one(tab[0]);
  tab[1] = a;
#pragma unroll 1
  for (int i = 2; i < 16; i++) F::mul(tab[i], tab[i - 1], a);
  F::set_one(acc);
#pragma unroll 1
  for (int w = 8 * F::NL - 1; w >= 0; w--) {
    F::sqr_n(acc, acc, 4);
    uint32_t limb = 0;
#pragma unroll
    for (int i = 0; i < F::NL; i++) limb = (w >> 3) == i ? E::PP14(i) : limb;
    F::mul(acc, acc, tab[(limb >> (4 * (w & 7))) & 15u]);
  }
  r = acc;
}
template <int V>
struct ILog2 {
  static constexpr int value = 1 + ILog2<(V >> 1)>::value;
};
template <>
struct ILog2<1> {
  static constexpr int value = 0;
};
// Tonelli-Shanks for a field with p = 1 (mod 4), p - 1 = 2^S (2^K - 1) (P-224: S = 96, K = 128).  Either root may come out:
// the caller checks r^2 == a and (decompression) picks the root by parity, so only "a root when one exists" matters.
// Variable time in a — these are public encodings.
template <class F, class E>
ECG_DEV void sqrt_candidate_ts(typename F::FeT& r, const typename F::FeT& a) {
  typedef typename F::FeT Fe;
  constexpr int NL = F::NL;
  Fe one, w, t, c, b;
  F::set_one(one);
  auto is_one = [&](const Fe& v) {
    uint32_t d = 0;
#pragma unroll
    for (int i = 0; i < NL; i++) d |= v.v[i] ^ one.v[i];
    return d == 0;
  };
  // w = a^(2^(K-1) - 1): x_{2m} = x_m^(2^m) * x_m, x_{2m+1} = x_{2m}^2 * a, over the bits of K - 1 from the top
  w = a;
  int m = 1;
#pragma unroll 1
  for (int bit = ILog2<E::TS_QBITS - 1>::value - 1; bit >= 0; bit--) {
    F::sqr_n(t, w, m);
    F::mul(w, t, w);
    m *= 2;
    if (((E::TS_QBITS - 1) >> bit) & 1) {
      F::sqr(w, w);
      F::mul(w, w, a);
      m++;
    }
  }
  F::mul(r, a, w);  // a^((Q+1)/2)
  F::mul(t, r, w);  // a^Q
#pragma unroll
  for (int i = 0; i < NL; i++) c.v[i] = E::TS_ZQ(i);
  int M = E::TS_S;
#pragma unroll 1
  while (!is_one(t)) {
    if (F::is_zero(t)) return;  // a = 0: r = 0 already
    int i = 0;
    b = t;
#pragma unroll 1
    while (i < M && !is_one(b)) {
      F::sqr(b, b);
      i++;
    }
    if (i == M) return;  // a is not a square; the caller's r^2 == a check fails
    F::sqr_n(b, c, M - i - 1);
    F::mul(r, r, b);
    F::sqr(c, b);
    F::mul(t, t, c);
    M = i;
  }
}
// records: tag (02 / 03; 00 with an all-zero x = the identity) || x, 1 + FB bytes, x in the curve's FieldBytes order (SEC1 2.3.4)
template <class C, class E>
ECG_KERNEL(128)
    decompress_generic_kernel(const uint8_t* __restrict__ sec1, size_t n, uint8_t* __restrict__ out_xy, uint8_t* __restrict__ out_inf,
                              uint8_t* __restrict__ valid) {
  typedef typename C::F F;
  typedef typename F::FeT Fe;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const uint8_t* rec = sec1 + (size_t)(FB + 1) * idx;
  const uint8_t tag = rec[0];
  Fe xc;
  if constexpr (F::LE) {  // bign-curve256v1: FieldBytes are little-endian (from_repr reads them so inside decompress, too)
#pragma unroll
    for (int i = 0; i < NL; i++)
      xc.v[i] = (uint32_t)rec[1 + 4 * i] | ((uint32_t)rec[2 + 4 * i] << 8) | ((uint32_t)rec[3 + 4 * i] << 16) | ((uint32_t)rec[4 + 4 * i] << 24);
  } else {
    load_be_bytes<NL, FB>(xc.v, rec + 1);  // the x bytes are not word-aligned
  }
  uint32_t any = 0;
#pragma unroll
  for (int i = 0; i < NL; i++) any |= xc.v[i];
  bool ok = false, inf = false;
  Fe x, y;
  if (tag == 0 && any == 0) {
    ok = inf = true;
  } else if ((tag == 2 || tag == 3) && ltN<NL>(xc.v, C::P())) {
    Fe rhs, t, b, chk;
    F::from_canonical(x, xc);
    F::sqr(rhs, x);
    F::mul(rhs, rhs, x);
    if (C::A_IS_MINUS3 == 1) {
      F::mul_small(t, x, 3);
      F::sub(rhs, rhs, t);
    } else if constexpr (C::A_IS_MINUS3 == 2) {
      Fe ca;
      F::curve_a(ca);
      F::mul(t, x, ca);
      F::add(rhs, rhs, t);
    }
    C::b_internal(b);
    F::add(rhs, rhs, b);
    if constexpr (E::HAS_SQRT_EXP)
      sqrt_candidate_generic<F, E>(y, rhs);
    else
      sqrt_candidate_ts<F, E>(y, rhs);
    F::sqr(chk, y);
    F::sub(chk, chk, rhs);
    ok = F::is_zero(chk);
    Fe yc;
    F::to_canonical(yc, y);
    if ((yc.v[0] & 1u) != (uint32_t)(tag & 1u)) F::neg(y, y);
  }
  Fe cx, cy;
  if (ok && !inf) {
    F::to_canonical(cx, x);
    F::to_canonical(cy, y);
  } else {
    F::set_zero(cx);
    F::set_zero(cy);
  }
  store_fe<F>(out_xy + 2 * FB * idx, cx.v);
  store_fe<F>(out_xy + 2 * FB * idx + FB, cy.v);
  out_inf[idx] = inf ? 1 : 0;
  valid[idx] = ok ? 1 : 0;
}
template <class C, class E>
ECG_KERNEL(128)
    field_sqrt_generic_kernel(size_t n, const uint8_t* __restrict__ a, uint8_t* __restrict__ out, uint8_t* __restrict__ is_square,
                              uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  typedef typename F::FeT Fe;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  Fe x, r, chk;
  load_fe<F>(x.v, a + FB * idx);
  if (!ltN<NL>(x.v, C::P())) report_error(status, ERRF_POINT, base + idx);
  F::from_canonical(x, x);
  sqrt_candidate_generic<F, E>(r, x);
  F::sqr(chk, r);
  F::sub(chk, chk, x);
  bool ok = F::is_zero(chk);
  F::to_canonical(r, r);
  if (!ok) F::set_zero(r);
  store_fe<F>(out + FB * idx, r.v);
  is_square[idx] = ok ? 1 : 0;
}

// canonical affine big-endian bytes (n * 2FB) -> table words (internal form); used once, when a table is built
template <class C>
ECG_KERNEL(256)
    affine_to_table_kernel(const uint8_t* __restrict__ xy, size_t n, uint32_t* __restrict__ table) {
  typedef typename C::F F;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  typename F::FeT x, y;
  load_fe<F>(x.v, xy + 2 * FB * idx);
  load_fe<F>(y.v, xy + 2 * FB * idx + FB);
  F::from_canonical(x, x);
  F::from_canonical(y, y);
#pragma unroll
  for (int w = 0; w < NL; w++) {
    table[idx * (2 * NL) + w] = x.v[w];
    table[idx * (2 * NL) + NL + w] = y.v[w];
  }
}

// Sum of Jacobian points: thread t adds elements t, t+T, t+2T, ... of `in` (SoA, n_in) and writes partial t of
// `out` (SoA, n_out = T).  Applied repeatedly until one point is left (lincomb's final reduction; SURVEY §8(e)).
template <class C>
ECG_KERNEL(128)
    jac_sum_kernel(const uint32_t* __restrict__ in, size_t n_in, uint32_t* __restrict__ out, size_t n_out) {
  typedef typename C::F F;
  constexpr int NL = F::NL;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_out) return;
  typename F::JacT acc;
  F::set_zero(acc.X);
  F::set_one(acc.Y);
  F::set_zero(acc.Z);
  for (size_t idx = t; idx < n_in; idx += n_out) {
    typename F::JacT p;
    soa_load<NL>(p.X.v, in, n_in, idx, 0);
    soa_load<NL>(p.Y.v, in, n_in, idx, NL);
    soa_load<NL>(p.Z.v, in, n_in, idx, 2 * NL);
    jac_add<F, C::A_IS_MINUS3>(acc, acc, p);
  }
  soa_store<NL>(out, n_out, t, acc.X.v, 0);
  soa_store<NL>(out, n_out, t, acc.Y.v, NL);
  soa_store<NL>(out, n_out, t, acc.Z.v, 2 * NL);
}

// SoA internal Jacobian -> AoS canonical big-endian X||Y||Z (3 FB bytes per point)
template <class C>
ECG_KERNEL(128)
    export_jac_kernel(const uint32_t* __restrict__ jac, size_t n, uint8_t* __restrict__ xyz) {
  typedef typename C::F F;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
#pragma unroll 1
  for (int c = 0; c < 3; c++) {
    typename F::FeT v;
    soa_load<NL>(v.v, jac, n, idx, NL * c);
    F::to_canonical(v, v);
    store_fe<F>(xyz + 3 * FB * idx + FB * c, v.v);
  }
}

// ------------------------------------------------------------------------------------------------
// Jacobian (SoA) -> canonical affine bytes with Montgomery's trick along each thread's strided slice:
// thread t owns elements t, t+T, t+2T, ... ; one field inversion per thread, 7 field multiplications per
// element.  Replaces batch_normalize / BatchInvert (k256/src/arithmetic/projective.rs:367-391,
// k256/src/arithmetic/field.rs:244-291).  scr: NL*n words of scratch (prefix products).
// X_ONLY: write only the x coordinate (FB-byte records): ECDH's SharedSecret is affine.x alone (k256/src/ecdh.rs:56-60),
// which saves the Z^-3 and y products (2 of the 7 multiplications per element) and half of the output bytes.
template <class F, bool X_ONLY = false>
ECG_KERNEL(256)
    normalize_kernel(const uint32_t* __restrict__ jac, size_t n, uint32_t* __restrict__ scr,
                     uint8_t* __restrict__ out_xy, uint8_t* __restrict__ out_inf) {
  typedef typename F::FeT Fe;
  constexpr int NL = F::NL, FB = F::FB;
  size_t T = (size_t)gridDim.x * blockDim.x;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  Fe acc, one;
  F::set_one(one);
  acc = one;
  size_t last = t;
  for (size_t idx = t; idx < n; idx += T) {
    Fe z;
    soa_load<NL>(z.v, jac, n, idx, 2 * NL);
    if (F::is_zero(z)) z = one;
    soa_store<NL>(scr, n, idx, acc.v, 0);
    F::mul(acc, acc, z);
    last = idx;
  }
  Fe inv;
  F::inv(inv, acc);
  for (size_t idx = last;; idx -= T) {
    typename F::JacT p;
    soa_load<NL>(p.Z.v, jac, n, idx, 2 * NL);
    bool inf = F::is_zero(p.Z);
    if (inf) p.Z = one;
    Fe pre, zinv;
    soa_load<NL>(pre.v, scr, n, idx, 0);
    F::mul(zinv, inv, pre);
    F::mul(inv, inv, p.Z);
    soa_load<NL>(p.X.v, jac, n, idx, 0);
    Fe x, y;
    if (X_ONLY) {
      Fe z2;
      F::sqr(z2, zinv);
      F::mul(x, p.X, z2);
      F::to_canonical(x, x);
      if (inf) F::set_zero(x);
      store_fe<F>(out_xy + FB * idx, x.v);
    } else {
      soa_load<NL>(p.Y.v, jac, n, idx, NL);
      jac_to_affine_canonical<F>(x, y, p, zinv);
      if (inf) {
        F::set_zero(x);
        F::set_zero(y);
      }
      store_fe<F>(out_xy + 2 * FB * idx, x.v);
      store_fe<F>(out_xy + 2 * FB * idx + FB, y.v);
    }
    out_inf[idx] = inf ? 1 : 0;
    if (idx < T) break;
  }
}

// AoS big-endian X||Y||Z (n * 3FB bytes, canonical) -> SoA internal form; validates coordinates < p.
// HOM: the input is the reference's own homogeneous projective form (x = X/Z, y = Y/Z, identity (0:1:0):
// k256/src/arithmetic/projective.rs:49-53,64-75; primeorder/src/projective.rs) and is carried over to the Jacobian
// point (X Z : Y Z^2 : Z), which has the same affine image: one squaring and two multiplications per point here, so
// that a reference-side caller can hand its ProjectivePoint coordinates over unchanged.
template <class C, bool HOM = false>
ECG_KERNEL(256)
    import_jac_kernel(const uint8_t* __restrict__ xyz, size_t n, uint32_t* __restrict__ jac,
                      uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  typedef typename F::FeT Fe;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  Fe co[3];
#pragma unroll 1
  for (int c = 0; c < 3; c++) {
    Fe v;
    load_fe<F>(v.v, xyz + 3 * FB * idx + FB * c);
    if (!ltN<NL>(v.v, C::P())) report_error(status, ERRF_POINT, base + idx);
    F::from_canonical(co[c], v);
  }
  if (HOM) {
    Fe zz;
    F::sqr(zz, co[2]);
    F::mul(co[0], co[0], co[2]);
    F::mul(co[1], co[1], zz);
  }
#pragma unroll 1
  for (int c = 0; c < 3; c++) soa_store<NL>(jac, n, idx, co[c].v, NL * c);
}

// out[i] = the square root the reference returns, a^((p+1)/4) (FieldElement::sqrt, k256/src/arithmetic/field.rs:200-235,
// p256/src/arithmetic/field.rs:121-147), is_square[i] = 1; or 32 zero bytes and is_square[i] = 0 (CtOption::none).
template <class C>
ECG_KERNEL(128)
    field_sqrt_kernel(size_t n, const uint8_t* __restrict__ a, uint8_t* __restrict__ out, uint8_t* __restrict__ is_square,
                      uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  Fe x, r, chk;
  load_be32(x.v, a + 32 * idx);
  if (!lt8(x.v, C::P())) report_error(status, ERRF_POINT, base + idx);
  F::from_canonical(x, x);
  if (C::A_IS_MINUS3)
    p256_sqrt_candidate<F>(r, x);
  else
    k256_sqrt_candidate<F>(r, x);
  F::sqr(chk, r);
  F::sub(chk, chk, x);
  bool ok = F::is_zero(chk);
  F::to_canonical(r, r);
  if (!ok) F::set_zero(r);
  store_be32(out + 32 * idx, r.v);
  is_square[idx] = ok ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
template <class C>
ECG_KERNEL(256)
    field_op_kernel(int op, size_t n, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                    uint8_t* __restrict__ out, uint32_t* __restrict__ status, size_t base) {
  typedef typename C::F F;
  constexpr int NL = F::NL, FB = F::FB;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  typename F::FeT x, y, r;
  load_fe<F>(x.v, a + FB * idx);
  if (!ltN<NL>(x.v, C::P())) report_error(status, ERRF_POINT, base + idx);
  F::from_canonical(x, x);
  bool binary = (op == ECG_FOP_ADD || op == ECG_FOP_SUB || op == ECG_FOP_MUL);
  if (binary) {
    load_fe<F>(y.v, b + FB * idx);
    if (!ltN<NL>(y.v, C::P())) report_error(status, ERRF_POINT, base + idx);
    F::from_canonical(y, y);
  } else {
    y = x;
  }
  switch (op) {
    case ECG_FOP_ADD: F::add(r, x, y); break;
    case ECG_FOP_SUB: F::sub(r, x, y); break;
    case ECG_FOP_NEG: F::neg(r, x); break;
    case ECG_FOP_MUL: F::mul(r, x, y); break;
    case ECG_FOP_SQR: F::sqr(r, x); break;
    default: F::inv(r, x); break;
  }
  F::to_canonical(r, r);
  store_fe<F>(out + FB * idx, r.v);
}

