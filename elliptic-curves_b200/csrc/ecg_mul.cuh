// ecg_mul.cuh — one (scalar, point) pair per thread: window table + double-and-add loop.
//
// Replaces the drivers k256 `lincomb`/`mul` (k256/src/arithmetic/mul.rs:112-163, :236-247) and
// primeorder `ProjectivePoint::mul` / `lincomb` (primeorder/src/projective.rs:133-137, :532-557),
// `LookupTable` (primeorder/src/tables/lookup.rs:30-81) and `wnaf_table` (wnaf/src/lib.rs:55-65).
//
// Everything here is per-thread straight-line work on registers plus a per-thread window table behind
// the `TabRef` accessors (a per-block slot of global memory in the kernels — see ecgpu.cu —, a plain array in the
// host simulation).  All threads
// of a warp execute the same operation sequence (fixed windows, every digit non-zero), so there is no
// divergence outside the never-taken exceptional-case branches.
#pragma once
#include "ecg_fe_k256.cuh"
#include "ecg_point.cuh"
#include "ecg_scalar.cuh"

namespace ecg {

// Window-table accessor: entry e (0..7), word w (0..WPE-1: x[0..NL-1], y[0..NL-1], then with WPE = 3 NL a second
// x column, beta*x for secp256k1) lives at base[(e*WPE+w)*stride].
// In the kernels base = slot + threadIdx.x and stride = blockDim.x: the 32 lanes of a warp touch 32 consecutive
// words of each row they select (coalesced when lanes agree on the entry, at worst 8 rows when they do not).
template <int NL, int WPE = 2 * NL>
struct TabRefN {
  uint32_t* base;
  uint32_t stride;
  ECG_D void store(int e, const FeN<NL>& x, const FeN<NL>& y) const {
#pragma unroll
    for (int w = 0; w < NL; w++) {
      base[(e * WPE + w) * stride] = x.v[w];
      base[(e * WPE + NL + w) * stride] = y.v[w];
    }
  }
  ECG_D void store_x2(int e, const FeN<NL>& x2) const {  // the second x column (WPE = 3 NL)
#pragma unroll
    for (int w = 0; w < NL; w++) base[(e * WPE + 2 * NL + w) * stride] = x2.v[w];
  }
  // x from the column starting at word xcol (0, or 2 NL for the second x column), y
  ECG_D void load(int e, FeN<NL>& x, FeN<NL>& y, int xcol = 0) const {
#pragma unroll
    for (int w = 0; w < NL; w++) {
      x.v[w] = base[(e * WPE + xcol + w) * stride];
      y.v[w] = base[(e * WPE + NL + w) * stride];
    }
  }
  // entry `idx` without a secret-dependent address: every entry is read, the wanted one kept by mask
  // (LookupTable::select, primeorder/src/tables/lookup.rs:43-65)
  ECG_D void load_ct(uint32_t idx, FeN<NL>& x, FeN<NL>& y) const {
    static_assert(WPE == 2 * NL, "the masked scan covers the (x, y) layout only");
#pragma unroll
    for (int w = 0; w < NL; w++) x.v[w] = y.v[w] = 0;
#pragma unroll 1
    for (uint32_t e = 0; e < 8; e++) {
      const uint32_t m = 0u - (uint32_t)(e == idx);
#pragma unroll
      for (int w = 0; w < NL; w++) {
        x.v[w] |= base[(e * WPE + w) * stride] & m;
        y.v[w] |= base[(e * WPE + NL + w) * stride] & m;
      }
    }
  }
};
typedef TabRefN<8> TabRef;
// the secp256k1 table of a field policy: (x, y), or (x, y, beta*x) with F::BETA_COLUMN
template <class F>
using K256TabRef = TabRefN<8, F::BETA_COLUMN ? 24 : 16>;
// Same, for Jacobian entries (3*NL words: X, Y, Z).
template <int NL>
struct TabRefJN {
  uint32_t* base;
  uint32_t stride;
  ECG_D void store(int e, const JacN<NL>& p) const {
#pragma unroll
    for (int w = 0; w < NL; w++) {
      base[(e * 3 * NL + w) * stride] = p.X.v[w];
      base[(e * 3 * NL + NL + w) * stride] = p.Y.v[w];
      base[(e * 3 * NL + 2 * NL + w) * stride] = p.Z.v[w];
    }
  }
  ECG_D void load(int e, JacN<NL>& p) const {
#pragma unroll
    for (int w = 0; w < NL; w++) {
      p.X.v[w] = base[(e * 3 * NL + w) * stride];
      p.Y.v[w] = base[(e * 3 * NL + NL + w) * stride];
      p.Z.v[w] = base[(e * 3 * NL + 2 * NL + w) * stride];
    }
  }
  ECG_D void load_ct(uint32_t idx, JacN<NL>& p) const {  // masked scan over all eight entries (see TabRefN::load_ct)
#pragma unroll
    for (int w = 0; w < NL; w++) p.X.v[w] = p.Y.v[w] = p.Z.v[w] = 0;
#pragma unroll 1
    for (uint32_t e = 0; e < 8; e++) {
      const uint32_t m = 0u - (uint32_t)(e == idx);
#pragma unroll
      for (int w = 0; w < NL; w++) {
        p.X.v[w] |= base[(e * 3 * NL + w) * stride] & m;
        p.Y.v[w] |= base[(e * 3 * NL + NL + w) * stride] & m;
        p.Z.v[w] |= base[(e * 3 * NL + 2 * NL + w) * stride] & m;
      }
    }
  }
};
typedef TabRefJN<8> TabRefJ;

ECG_D void k256_beta(Fe& b) {
  // ENDOMORPHISM_BETA, k256/src/arithmetic/projective.rs:32-37
  const uint32_t B[8] = {0x719501EEu, 0xC1396C28u, 0x12F58995u, 0x9CF04975u, 0xAC3434E9u, 0x6E64479Eu, 0x657C0710u, 0x7AE96A2Bu};
#pragma unroll
  for (int i = 0; i < 8; i++) b.v[i] = B[i];
}

// Build the table of odd multiples {1,3,...,15}*P as *affine* points of the curve E' isomorphic to E
// under (x,y) -> (x Zg^2, y Zg^3): the 8 entries share the denominator Zg, which is returned and
// multiplied back into the accumulator's Z once at the end.  Valid for a = 0 only (the a=0 doubling and
// the additions never use the curve constant b, and b is the only coefficient the isomorphism changes).
// Cost: 1 dbl + 7 madd + 35M rescale, no inversion, no block-level synchronisation.  With F::BETA_COLUMN each entry
// also gets beta*x (8M more), the x of the endomorphism image (beta x, y) that the lambda half of the scalar adds.
template <class F>
ECG_D void build_table_iso_a0(const K256TabRef<F>& tab, Fe& Zg, const Aff& P) {
  Jac d, cur;
  aff_dbl<F, false>(d, P);  // 2P = (dX, dY, dZ)
  // On E'' = image under dZ: 2P is affine (dX, dY); P becomes (x dZ^2, y dZ^3).
  Fe z2, z3;
  F::sqr(z2, d.Z);
  F::mul(z3, z2, d.Z);
  F::mul(cur.X, P.x, z2);
  F::mul(cur.Y, P.y, z3);
  F::set_one(cur.Z);
  Aff dd;
  dd.x = d.X;
  dd.y = d.Y;
  Fe zr[8];
  tab.store(0, cur.X, cur.Y);
#pragma unroll 1
  for (int i = 1; i < 8; i++) {
    jac_madd<F, false>(cur, cur, dd, &zr[i]);
    tab.store(i, cur.X, cur.Y);
  }
  // bring entries 0..6 to the denominator of entry 7: scale by zs = Z7/Zi = prod_{j>i} zr[j]
  F::mul(Zg, cur.Z, d.Z);
  Fe zs = zr[7], beta;
  if constexpr (F::BETA_COLUMN) {
    k256_beta(beta);
    F::mul(cur.X, cur.X, beta);
    tab.store_x2(7, cur.X);
  }
#pragma unroll 1
  for (int i = 6; i >= 0; i--) {
    Fe x, y, zz;
    tab.load(i, x, y);
    F::sqr(zz, zs);
    F::mul(x, x, zz);
    F::mul(zz, zz, zs);
    F::mul(y, y, zz);
    tab.store(i, x, y);
    if constexpr (F::BETA_COLUMN) {
      F::mul(x, x, beta);
      tab.store_x2(i, x);
    }
    if (i > 0) F::mul(zs, zs, zr[i]);
  }
}

// secp256k1: r = k*P (Jacobian, true curve).  k: 8 LE limbs, k < n.  P: affine, on curve, not identity.
// GLV split -> two 128-bit halves -> 32 shared windows of (4 dbl + 2 madd); the lambda-half reuses the
// same table through (x,y) -> (beta x, y) (ProjectivePoint::endomorphism, projective.rs:241-247).
// PHASE_SYNC (experiment, tools/kbench.cu): a block-wide barrier between the doubling phase and the addition phase
// keeps all warps of a block in the same stretch of code, so a fully inlined body only needs one phase's
// instructions resident in the instruction cache at a time.
#if defined(__CUDA_ARCH__)
#define ECG_BLOCK_SYNC() __syncthreads()
#else
#define ECG_BLOCK_SYNC() ((void)0)
#endif
// CT (ECG_FLAG_CONSTTIME): window-table entries are fetched by a masked scan over all eight entries and the sign folding
// of the GLV halves is branch-free, so neither addresses nor branches depend on the scalar (what is left: the
// exceptional-case branches of the Jacobian formulas, reachable only for k = 0 and a negligible set of scalars).
template <class F = FpK256, int PHASE_SYNC = 0, bool CT = false>  // PHASE_SYNC: 0 none, 1 per phase (doublings | additions), 2 before every point operation
ECG_D void k256_mul_thread(Jac& r, const uint32_t* k, const Aff& P, const K256TabRef<F>& tab) {
  GlvHalf g1, g2;
  glv_split_k256<CT>(g1, g2, k);
  Fe Zg, beta;
  build_table_iso_a0<F>(tab, Zg, P);
  k256_beta(beta);
  // the lambda half adds (beta x, y): x from the table's beta*x column (word 16 of an entry), or times beta here
  constexpr int BX = F::BETA_COLUMN ? 16 : 0;

  Jac acc;
  Aff e;
  // top digits are both +1: acc = s1*T[0] + s2*lambda*T[0]
  tab.load(0, acc.X, acc.Y);
  fe_cneg<F>(acc.Y, g1.neg);
  F::set_one(acc.Z);
  tab.load(0, e.x, e.y, BX);
  if (!F::BETA_COLUMN) F::mul(e.x, e.x, beta);
  fe_cneg<F>(e.y, g2.neg);
  jac_madd<F, false>(acc, acc, e);

#pragma unroll 1
  for (int i = 0; i < 32; i++) {
    if (PHASE_SYNC == 1) ECG_BLOCK_SYNC();
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
      if (PHASE_SYNC == 2) ECG_BLOCK_SYNC();
      jac_dbl<F, false>(acc, acc);
    }
    if (PHASE_SYNC == 1) ECG_BLOCK_SYNC();
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
      if (PHASE_SYNC == 2) ECG_BLOCK_SYNC();
      uint32_t n = half ? next_window(g2.h) : next_window(g1.h);
      uint32_t sneg = half ? g2.neg : g1.neg;
      uint32_t pos = n >> 3;                       // digit sign: n>=8 -> positive
      uint32_t idx = pos ? (n & 7u) : (7u - n);
      if constexpr (F::BETA_COLUMN) {  // x column chosen by address: no product, no branch
        static_assert(!CT, "the masked scan reads the (x, y) layout");
        tab.load((int)idx, e.x, e.y, half ? BX : 0);
      } else {
        if (CT)
          tab.load_ct(idx, e.x, e.y);
        else
          tab.load((int)idx, e.x, e.y);
        if (half) F::mul(e.x, e.x, beta);
      }
      fe_cneg<F>(e.y, (pos ^ sneg) ^ 1u);              // negative digit XOR negative half-scalar
      jac_madd<F, false>(acc, acc, e);
    }
  }
  // parity corrections: subtract the (signed) base once for every half whose magnitude was even
#pragma unroll 1
  for (int half = 0; half < 2; half++) {
    uint32_t ev = half ? g2.even : g1.even;
    uint32_t sneg = half ? g2.neg : g1.neg;
    tab.load(0, e.x, e.y, half ? BX : 0);
    if (half && !F::BETA_COLUMN) F::mul(e.x, e.x, beta);
    fe_cneg<F>(e.y, sneg ^ 1u);
    Jac t;
    jac_madd<F, false>(t, acc, e);
    jac_csel(acc, t, ev);
  }
  r.X = acc.X;
  r.Y = acc.Y;
  F::mul(r.Z, acc.Z, Zg);
}

// Generic prime-order curve without endomorphism (NIST P-256): r = k*P (Jacobian).
// k: 8 LE limbs, k < n.  P: affine, on curve, not identity.  Signed-odd radix-16 recoding of the full
// 256-bit scalar: implicit top digit +1, then 64 windows of (4 dbl + 1 add) against a table of the eight
// odd multiples kept in Jacobian form (the shared-denominator trick of build_table_iso_a0 needs a = 0).
// Replaces primeorder ProjectivePoint::mul / mul_vartime (primeorder/src/projective.rs:133-144, :532-557).
template <class F, int A_IS_MINUS3, int PHASE_SYNC = 0, bool CT = false>
ECG_D void generic_mul_thread(typename F::JacT& r, const uint32_t* k, const typename F::AffT& P, const TabRefJN<F::NL>& tab) {
  typedef typename F::JacT Jac;
  typedef typename F::AffT Aff;
  FullRecodeN<F::NL> rc;
  recode_full<F::NL>(rc, k);
  Jac d, cur, acc;
  aff_dbl<F, A_IS_MINUS3>(d, P);
  cur.X = P.x;
  cur.Y = P.y;
  F::set_one(cur.Z);
  acc = cur;  // top digit (+1) * P
  tab.store(0, cur);
  jac_madd<F, A_IS_MINUS3>(cur, d, P);  // 3P
  tab.store(1, cur);
#pragma unroll 1
  for (int i = 2; i < 8; i++) {
    jac_add<F, A_IS_MINUS3>(cur, cur, d);
    tab.store(i, cur);
  }
#pragma unroll 1
  for (int i = 0; i < F::NL * 8; i++) {  // one 4-bit window per nibble of the scalar
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
      if (PHASE_SYNC == 2) ECG_BLOCK_SYNC();
      jac_dbl<F, A_IS_MINUS3>(acc, acc);
    }
    if (PHASE_SYNC == 2) ECG_BLOCK_SYNC();
    uint32_t n = next_windowN<F::NL>(rc.h);
    uint32_t pos = n >> 3;
    uint32_t idx = pos ? (n & 7u) : (7u - n);
    Jac e;
    if (CT)
      tab.load_ct(idx, e);
    else
      tab.load((int)idx, e);
    fe_cneg<F>(e.Y, pos ^ 1u);
    jac_add<F, A_IS_MINUS3>(acc, acc, e);
  }
  // parity correction: the loop computed (k+1)*P when k was even
  Aff np;
  np.x = P.x;
  F::neg(np.y, P.y);
  Jac t;
  jac_madd<F, A_IS_MINUS3>(t, acc, np);
  jac_csel(acc, t, rc.even);
  r = acc;
}

}  // namespace ecg
