// ecg_x448.cuh — X448 (RFC 7748 section 5) over a batch: one thread per (scalar, u) pair, a Montgomery ladder over the
// Curve448 field (ecg_fe_p448.cuh).
//
// The reference (x448/src/lib.rs:152-163, ed448-goldilocks/src/montgomery.rs:87-109, 168-219):
//   - the 56 scalar bytes are clamped (k[0] &= 252, k[55] |= 128) and read little-endian WITHOUT reduction mod the
//     group order; the ladder runs over all 448 bits, most significant first;
//   - u is read little-endian and reduced mod p (values in [p, 2^448) are accepted);
//   - each step is Costello-Smith Algorithm 8 (5 M + 4 S + one multiplication by (A + 2)/4 = 39082);
//   - the result is U * W^-1 with 0^-1 = 0, encoded canonically: a result at the identity is 56 zero bytes;
//   - x448::x448 refuses u whose bytes are exactly 0, 1 or p - 1 (MontgomeryPoint::LOW_A / LOW_B / LOW_C); other
//     encodings of those values are not refused.  That check is the `ok` byte here; the ladder runs regardless.
//
// Constant time: the ladder's only data-dependent choice is the conditional swap, done with masks (FpP448T::cswap).  The
// loop bounds, the scalar word read in each outer iteration and every shift amount depend on the loop counters alone;
// the inversion is a fixed addition chain.  No branch and no memory index depends on the scalar or on u.
#pragma once
#include "ecg_fe_p448.cuh"

namespace ecg {

// Shipped variant and launch geometry of x448_kernel (DESIGN.md section 7, "X448"): the call-based field (mul / sqr as
// device functions) at 128 threads per block with at most 168 registers per thread (3 blocks per SM), which ptxas
// meets without spills.
#ifndef ECG_X448_OPT
#define ECG_X448_OPT 2
#endif
#define X448_BLOCK 128
#define X448_MINBLK 3
typedef FpP448T<ECG_X448_OPT> FpP448;

static constexpr uint32_t X448_A24 = 39082;  // (A + 2) / 4, A = 156326

// a 32-bit little-endian word of a 56-byte record (records are 4-byte aligned on the device)
ECG_D uint32_t x448_word(const uint8_t* rec, int w) {
#if defined(__CUDA_ARCH__)
  return reinterpret_cast<const uint32_t*>(rec)[w];
#else
  return (uint32_t)rec[4 * w] | ((uint32_t)rec[4 * w + 1] << 8) | ((uint32_t)rec[4 * w + 2] << 16) | ((uint32_t)rec[4 * w + 3] << 24);
#endif
}
ECG_D void x448_store_word(uint8_t* rec, int w, uint32_t v) {
#if defined(__CUDA_ARCH__)
  reinterpret_cast<uint32_t*>(rec)[w] = v;
#else
  for (int b = 0; b < 4; b++) rec[4 * w + b] = (uint8_t)(v >> (8 * b));
#endif
}

// differential_add_and_double (montgomery.rs:168-204): (x2 : z2) <- 2 (x2 : z2), (x3 : z3) <- (x2 : z2) + (x3 : z3),
// whose difference has affine u-coordinate u.  The comments name the reference's temporaries.
template <class F>
ECG_D void x448_ladder_step(typename F::Fe& x2, typename F::Fe& z2, typename F::Fe& x3, typename F::Fe& z3, const typename F::Fe& u) {
  typename F::Fe a, b, c, d;
  F::add(a, x2, z2);           // t0
  F::sub(b, x2, z2);           // t1
  F::add(c, x3, z3);           // t2
  F::sub(d, x3, z3);           // t3
  F::mul(d, a, d);             // t7 = t0 t3
  F::mul(c, b, c);             // t8 = t1 t2
  F::sqr(a, a);                // t4
  F::sqr(b, b);                // t5
  F::add(x3, d, c);            // t9
  F::sub(z3, d, c);            // t10
  F::sqr(x3, x3);              // t11 = U of the sum
  F::sqr(z3, z3);              // t12
  F::mul(z3, z3, u);           // t17 = W of the sum
  F::sub(c, a, b);             // t6
  F::mul(x2, a, b);            // t14 = U of the double
  F::mul_small(d, c, X448_A24);  // t13
  F::add(d, d, b);             // t15
  F::mul(z2, c, d);            // t16 = W of the double
}

// the reference's low-order check (x448::x448 returns None): 1 unless the 56 bytes are exactly 0, 1 or p - 1
ECG_D uint32_t x448_u_ok(const uint8_t* u56) {
  uint32_t d0 = 0, d1 = 0, d2 = 0;
#pragma unroll
  for (int w = 0; w < 14; w++) {
    const uint32_t v = x448_word(u56, w);
    const uint32_t pm1 = (w == 0 || w == 7) ? 0xFFFFFFFEu : 0xFFFFFFFFu;  // p - 1 = 2^448 - 2^224 - 2
    d0 |= v;
    d1 |= v ^ (w == 0 ? 1u : 0u);
    d2 |= v ^ pm1;
  }
  return (uint32_t)(d0 != 0) & (uint32_t)(d1 != 0) & (uint32_t)(d2 != 0);
}

// out56 = X448(k56, u56); u56 == nullptr: u = 5 (the generator, PublicKey::from).  ok (may be null) = x448_u_ok.
template <class F>
ECG_D void x448_one(const uint8_t* k56, const uint8_t* u56, uint8_t* out56, uint8_t* ok) {
  typedef typename F::Fe Fe;
  Fe u, x2, z2, x3, z3;
  if (u56) {  // a pointer, not data: the same for every element of a call
#pragma unroll
    for (int w = 0; w < 14; w++) u.v[w] = x448_word(u56, w);
    F::normalize(u, u);  // u mod p
  } else {
    F::set_small(u, 5);
  }
  if (ok) *ok = u56 ? (uint8_t)x448_u_ok(u56) : (uint8_t)1;
  F::set_one(x2);
  F::set_zero(z2);
  x3 = u;
  F::set_one(z3);
  uint32_t swap = 0;
  // 448 steps, most significant scalar bit first; one scalar word per outer iteration, clamped as it is read
#pragma unroll 1
  for (int w = 13; w >= 0; w--) {
    uint32_t kw = x448_word(k56, w);
    kw &= (w == 0) ? 0xFFFFFFFCu : 0xFFFFFFFFu;  // k[0] &= 252
    kw |= (w == 13) ? 0x80000000u : 0u;         // k[55] |= 128
#pragma unroll 1
    for (int j = 31; j >= 0; j--) {
      const uint32_t bit = (kw >> j) & 1u;
      swap ^= bit;
      const uint32_t mask = 0u - swap;
      F::cswap(x2, x3, mask);
      F::cswap(z2, z3, mask);
      swap = bit;
      x448_ladder_step<F>(x2, z2, x3, z3, u);
    }
  }
  {
    const uint32_t mask = 0u - swap;  // 0 after the clamp (bit 0 is clear); kept for the RFC's shape
    F::cswap(x2, x3, mask);
    F::cswap(z2, z3, mask);
  }
  F::inv(z2, z2);
  F::mul(x2, x2, z2);
  F::to_canonical(x2, x2);
#pragma unroll
  for (int w = 0; w < 14; w++) x448_store_word(out56, w, x2.v[w]);
}

#if defined(__CUDACC__)
// one pair per thread: k, u (u == nullptr: the generator), out: 56-byte records; ok: one byte per pair (may be null)
template <class F, int BLOCK, int MINBLK>
__global__ void __launch_bounds__(BLOCK, MINBLK) x448_kernel(const uint8_t* k, const uint8_t* u, size_t n, uint8_t* out, uint8_t* ok) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i >= n) return;
  x448_one<F>(k + 56 * i, u ? u + 56 * i : nullptr, out + 56 * i, ok ? ok + i : nullptr);
}
#endif

}  // namespace ecg
