// ecg_ed448_h2c.cuh — Ed448 hash to curve (RFC 9380 edwards448_XOF:SHAKE256_ELL2_RO_ / _NU_) and hash to scalar over a
// batch: GroupDigest for Ed448 and hash_to_scalar::<Ed448, ExpandMsgXof<Shake256>, U84> of ed448-goldilocks, on the
// point layer of ecg_ed448.cuh and the expander of ecg_decaf448.cuh, which are used unchanged.
//
// The contract is the reference's bytes:
//   - hash to field: expand_message_xof with SHAKE256 (k = 28) to 2 x 84 (RO) or 84 (NU) bytes; each 84-byte block is
//     read big-endian mod p (Reduce<Array<u8, U84>>, field/element.rs:76-91);
//   - map: map_to_curve_elligator2 (Z = -1, A = 156326), the 4-isogeny to edwards448 and to_edwards
//     (field/element.rs:195-203, 441-462; edwards/affine.rs:56-63, 75-104);
//   - RO: (map(u0) + map(u1)).clear_cofactor(), NU: map(u0).clear_cofactor(), clear_cofactor = double().double();
//     the output is AffinePoint::compress (57 bytes, the Ed448 group entries' record);
//   - hash to scalar: 84 expanded bytes, big-endian, mod ell, as the 57-byte EdwardsScalar record (byte 56 = 0).
//
// The map, straight-line with one exponentiation: x1 = -A / xd with xd = 1 + t1 (t1 = Z u^2, set to 0 where it is -1)
// stays a fraction; gx1 = gxn / gxd with gxd = xd^3; y1 = gxn gxd (gxn gxd^3)^((p - 3) / 4) satisfies
// y1^2 = chi(gx1) gx1, so e2 = (y1^2 gxd == gxn) is is_square(gx1).  For a non-square gx1, Z = -1 gives x2 = -x1 - A =
// x1 t1 and sqrt(gx2) = sqrt(t1 gx1) = y1 u.  The sign fix y = CMOV(-y, y, e2 xor sgn0(y)) makes the result independent
// of the root found, so it equals the reference's unchecked_sqrt bit for bit.  Every select is masked.
//
// The quirk kept: u in {0, 1, p - 1} gives the Montgomery point (0, 0).  For u = +-1 the reference's t1 = 0 makes
// gx2 = 0 and y = 0, while y1 u is not 0: y is masked to 0 there.  The reference's isogeny then inverts yDen = 0 as 0
// and returns (0, 0) on edwards448, not a curve point; its unified formulas keep X = Y = T = 0 and compress gives 57
// zero bytes, for NU and for RO with either half exceptional.  The isogeny here is homogenised in xd and emits
// (xNum yDen : yNum xDen : xDen yDen : xNum yNum) without an inversion, which is (0 : 0 : 0 : 0) at those u and stays so
// through ed_add and ed_dbl.  The kernel sets Z = 1 where Z = 0 before storing, so the normalisation kernel of
// ecg_ed448_group.cuh (one shared inversion per slice) writes the reference's 57 zero bytes and its slice stays intact.
//
// Output of the point kernels: the SoA extended form of ed448_store_ext, compressed by ed448g_norm_kernel<false>.
#pragma once
#include "ecg_decaf448.cuh"

namespace ecg {

// launch geometry (DESIGN.md section 7, "Ed448 hash to curve"): the tightest bounds without spills
#define ED448H_BLOCK 128
#define ED448H_H2C_MINBLK 2  // hash to curve (RO and NU)
#define ED448H_H2S_MINBLK 6  // hash to scalar

static constexpr uint32_t ED448H_A = 156326;  // the Montgomery coefficient of curve448 (FieldElement::J)

// r == b84 read big-endian (mod p), weakly reduced: v = L + 2^448 H with H < 2^224, and 2^448 == 2^224 + 1, so
// v == L + H + 2^224 H
template <class F>
ECG_D void ed448h_load84(typename F::Fe& r, const uint8_t* b84) {
  typename F::Fe lo, h, h2;
#pragma unroll
  for (int j = 0; j < 14; j++)
    lo.v[j] = (uint32_t)b84[83 - 4 * j] | ((uint32_t)b84[82 - 4 * j] << 8) | ((uint32_t)b84[81 - 4 * j] << 16) |
              ((uint32_t)b84[80 - 4 * j] << 24);
#pragma unroll
  for (int j = 0; j < 7; j++) {
    const int k = 14 + j;
    h.v[j] = (uint32_t)b84[83 - 4 * k] | ((uint32_t)b84[82 - 4 * k] << 8) | ((uint32_t)b84[81 - 4 * k] << 16) |
             ((uint32_t)b84[80 - 4 * k] << 24);
    h.v[7 + j] = 0;
    h2.v[j] = 0;
    h2.v[7 + j] = h.v[j];
  }
  F::add(r, lo, h);
  F::add(r, r, h2);
}

// map_to_curve_elligator2(u).isogeny().to_edwards() as the extended point q (any 14-word u; read mod p)
template <class F>
ECG_D void ed448h_map(EdPt<F>& q, const typename F::Fe& u) {
  typedef typename F::Fe Fe;
  Fe one, t1, xd, d2, gxd, gxn, w, y, t, X, xalt;
  F::set_one(one);
  F::sqr(t1, u);
  F::neg(t1, t1);                                   // t1 = Z u^2
  const uint32_t e1 = 0u - (uint32_t)ed_is_minus_one<F>(t1);
#pragma unroll
  for (int i = 0; i < 14; i++) t1.v[i] &= ~e1;      // t1 = CMOV(t1, 0, e1)
  F::add(xd, one, t1);                              // xd = 1 + t1; x1 = -A / xd
  F::sqr(d2, xd);
  F::mul(gxd, d2, xd);                              // gxd = xd^3
  // gxn = -A^3 + A^3 xd - A xd^2 = -A (xd^2 - A^2 xd + A^2)
  F::set_small(w, ED448H_A);
  F::mul_small(w, w, ED448H_A);                     // A^2
  F::mul_small(t, xd, ED448H_A);
  F::mul_small(t, t, ED448H_A);
  F::sub(gxn, d2, t);
  F::add(gxn, gxn, w);
  F::mul_small(gxn, gxn, ED448H_A);
  F::neg(gxn, gxn);
  // y1 = gxn gxd (gxn gxd^3)^((p - 3) / 4)
  F::sqr(t, gxd);
  F::mul(t, t, gxd);
  F::mul(w, gxn, t);
  ed_pow_p34<F>(w, w);
  F::mul(y, gxn, gxd);
  F::mul(y, y, w);
  F::sqr(t, y);
  F::mul(t, t, gxd);
  const uint32_t e2 = ed_eq<F>(t, gxn) ? 1u : 0u;   // is_square(gx1)
  const uint32_t sq = 0u - e2;
  F::set_small(X, ED448H_A);
  F::neg(X, X);                                     // -A
  F::mul_small(xalt, t1, ED448H_A);
  F::neg(xalt, xalt);                               // x2 = x1 t1 = -A t1 / xd
  F::cswap(X, xalt, ~sq);
  F::mul(t, y, u);                                  // sqrt(gx2) = y1 u
  F::cswap(y, t, ~sq);
#pragma unroll
  for (int i = 0; i < 14; i++) y.v[i] &= ~e1;       // the reference's y = sqrt(t1 gx1) = 0 when t1 was set to 0
  decaf448_cneg<F>(y, y, 0u - (e2 ^ decaf448_is_neg<F>(y)));  // y = CMOV(-y, y, e2 xor sgn0(y))
  // the 4-isogeny at (X / xd, y), homogenised: with a = X^2 - xd^2, b = X^2 + xd^2,
  //   xNum = 4 y a xd^2, xDen = a^2 + 4 y^2 xd^4, yNum = X (4 y^2 xd^4 - a^2), yDen = a^2 X - 2 y^2 b xd^3
  Fe yy, a, b, a2, yd4, xN, xD, yN, yD;
  F::sqr(yy, y);
  F::sqr(t, X);
  F::sub(a, t, d2);
  F::add(b, t, d2);
  F::sqr(a2, a);
  F::sqr(t, d2);
  F::mul(t, t, yy);
  F::mul_small(yd4, t, 4);
  F::mul(t, y, a);
  F::mul(t, t, d2);
  F::mul_small(xN, t, 4);
  F::add(xD, a2, yd4);
  F::sub(t, yd4, a2);
  F::mul(yN, X, t);
  F::mul(t, yy, b);
  F::mul(t, t, gxd);
  F::add(t, t, t);
  F::mul(yD, a2, X);
  F::sub(yD, yD, t);
  F::mul(q.X, xN, yD);
  F::mul(q.Y, yN, xD);
  F::mul(q.Z, xD, yD);
  F::mul(q.T, xN, yN);
}

// ext[i] = the hash-to-curve point of 84 uniform bytes (ONE = true: one map, the NU form) or 168 (two maps added),
// cleared of the cofactor, Z = 1 where it is 0
template <class F, bool ONE>
ECG_D void ed448h_from_uniform(uint32_t* ext, size_t n, size_t i, const uint8_t* u) {
  typename F::Fe fe;
  EdPt<F> q0;
  ed448h_load84<F>(fe, u);
  ed448h_map<F>(q0, fe);
  if (!ONE) {
    EdPt<F> q1;
    ed448h_load84<F>(fe, u + 84);
    ed448h_map<F>(q1, fe);
    ed_mul_d<F>(q1.T, q1.T);
    ed_add<F>(q0, q0, q1.X, q1.Y, &q1.Z, q1.T);
  }
  ed_dbl<F>(q0, q0, false);
  ed_dbl<F>(q0, q0, true);
  typename F::Fe one;
  F::set_one(one);
  F::cswap(q0.Z, one, 0u - (uint32_t)ed_is_zero<F>(q0.Z));
  ed448_store_ext<F>(ext, n, i, q0);
}
// hash to curve of one message into ext[i]: NU = false expands 168 bytes and adds two maps, NU = true expands 84
template <class F, bool NU>
ECG_D void ed448h_h2c_one(uint32_t* ext, size_t n, size_t i, const uint8_t* msg, size_t mlen, const XofSuffix& suffix) {
  uint8_t u[168];
  if (NU)
    expand_message_xof<84>(u, msg, mlen, suffix);
  else
    expand_message_xof<168>(u, msg, mlen, suffix);
  ed448h_from_uniform<F, NU>(ext, n, i, u);
}
// r = b84 read big-endian mod ell: the bytes reversed into the low end of a zero-padded 114-byte little-endian buffer
ECG_D void ed448h_mod_l_84(uint32_t* r, const uint8_t* b84) {
  uint8_t h[114];
#pragma unroll
  for (int i = 0; i < 84; i++) h[i] = b84[83 - i];
#pragma unroll
  for (int i = 84; i < 114; i++) h[i] = 0;
  ed448_mod_l_wide(r, h);
}
ECG_D void ed448h_h2s_one(uint8_t* out57, const uint8_t* msg, size_t mlen, const XofSuffix& suffix) {
  uint8_t u[84];
  expand_message_xof<84>(u, msg, mlen, suffix);
  uint32_t r[14];
  ed448h_mod_l_84(r, u);
#pragma unroll
  for (int i = 0; i < 14; i++) {
    out57[4 * i] = (uint8_t)r[i];
    out57[4 * i + 1] = (uint8_t)(r[i] >> 8);
    out57[4 * i + 2] = (uint8_t)(r[i] >> 16);
    out57[4 * i + 3] = (uint8_t)(r[i] >> 24);
  }
  out57[56] = 0;
}

#if defined(__CUDACC__)
// one message per thread: message i is msgs[offs[i] - base .. offs[i + 1] - base); the extended points go to ext (SoA,
// stride n) for ed448g_norm_kernel<false>
template <class F, bool NU>
__global__ void __launch_bounds__(ED448H_BLOCK, ED448H_H2C_MINBLK)
    ed448h_h2c_kernel(const uint8_t* msgs, const uint64_t* offs, uint64_t base, size_t n, XofSuffix suffix, uint32_t* ext) {
  const size_t i = (size_t)blockIdx.x * ED448H_BLOCK + threadIdx.x;
  if (i >= n) return;
  const uint64_t lo = offs[i], hi = offs[i + 1];
  ed448h_h2c_one<F, NU>(ext, n, i, msgs + (lo - base), (size_t)(hi - lo), suffix);
}
__global__ void __launch_bounds__(ED448H_BLOCK, ED448H_H2S_MINBLK)
    ed448h_h2s_kernel(const uint8_t* msgs, const uint64_t* offs, uint64_t base, size_t n, XofSuffix suffix, uint8_t* out57) {
  const size_t i = (size_t)blockIdx.x * ED448H_BLOCK + threadIdx.x;
  if (i >= n) return;
  const uint64_t lo = offs[i], hi = offs[i + 1];
  ed448h_h2s_one(out57 + 57 * i, msgs + (lo - base), (size_t)(hi - lo), suffix);
}
#endif

}  // namespace ecg
