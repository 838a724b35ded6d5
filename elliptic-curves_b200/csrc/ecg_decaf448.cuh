// ecg_decaf448.cuh — Decaf448 (RFC 9496) over a batch: the prime-order group of ed448-goldilocks (DecafPoint,
// CompressedDecaf, DecafScalar, GroupDigest for Decaf448), built on the Ed448 point layer of ecg_ed448.cuh and the
// variable-base / fixed-base routines of ecg_ed448_group.cuh, which are used unchanged.
//
// The contract is the reference's encodings, verdict for verdict:
//   - a scalar is a 56-byte little-endian record accepted iff DecafScalar::from_canonical_bytes accepts it
//     (decaf/scalar.rs:22-32): byte 55 >> 6 == 0 and the value is < ell; the first follows from the second, so the test
//     is ed448_scalar_ok's (which reads bytes 0..55 only);
//   - a point is a 56-byte record s accepted iff CompressedDecaf::decompress accepts it (decaf/points.rs:555-593):
//     s < p, s even, and the inverse square root exists; all-zero is the identity;
//   - an output is DecafPoint::compress (decaf/points.rs:49-67); the identity is 56 zero bytes.
//
// Representatives.  The reference keeps Decaf points on the twisted curve (a = -1, d = -39082); the point layer here is
// the untwisted Edwards448 curve (a = 1, d = -39081).  decaf448_decode / decaf448_encode are RFC 9496's decaf448
// formulas on the untwisted curve and give the reference's bytes (tests/decaf448_model.py states both and the tests
// compare them).  A decoded representative carries 2-torsion at most ([ell] decode(b) is (0, 1) or (0, -1)), and the
// encoding is invariant under adding (0, -1).  So ed448_mul_var applies as it is: its "add ell when k is even" step
// turns [k]P into [k]P + T with T in E[2], which encodes to the same bytes.  The Ed448 decoder and its subgroup test are
// not used on Decaf records.
//
// The generator: G0 = decode(66..66 33..33) equals [-2]B modulo E[2], B the Ed448 base point.  So [k]G is the encoding
// of [(-2k) mod ell]B, the Ed448 fixed-base kernel's loop over the Ed448 table with one scalar transform
// (decaf448_gen_scalar).  ECG_FLAG_CONSTTIME runs the variable-base routine on G0 instead, as Ed448's k B does.
//
// Hash to group (hash_from_bytes / encode_from_bytes with ExpandMsgXof<Shake256>, k = 28): expand_message_xof, each
// 56-byte half read little-endian mod p, map_to_curve_decaf448 (field/element.rs:466-507) on the twisted curve, one
// twisted addition (curve/twedwards/extended.rs:82-98) and the twisted compress.  Only bytes leave, so the map's output
// never has to move to the untwisted layer.  Hash to scalar: 64 expanded bytes, little-endian, mod ell.
//
// Intermediate points of the group kernels are the Ed448 kernels' SoA extended form (ed448_store_ext / ed448_load_ext).
#pragma once
#include "ecg_ed448_group.cuh"

namespace ecg {

// launch geometry (DESIGN.md section 7, "Decaf448"): the tightest bounds without spills
#define DECAF448_BLOCK 128
#define DECAF448_MINBLK 2      // variable base (k P, lincomb terms, CONSTTIME k G)
#define DECAF448_FB_MINBLK 2   // fixed base (k G)
#define DECAF448_H2C_MINBLK 2  // hash to group
#define DECAF448_H2S_MINBLK 6  // hash to scalar

// sqrt(-d) = 39081^((p + 1) / 4), its inverse, the reference's DECAF_FACTOR (field/element.rs:281-283), and G0 = decode of
// CompressedDecaf::GENERATOR as untwisted (x, y); canonical, 14 little-endian 32-bit limbs (tests/test_decaf448.py
// recomputes them)
ECG_ED448_CONSTANT uint32_t DECAF448_SQRT_MINUS_D[14] = {0xBAA8D8C9u, 0x69BD10F0u, 0x55DF31ADu, 0x9FCC8409u, 0x0291212Du,
                                                          0x7C65990Bu, 0x6973EB45u, 0x9B5D287Eu, 0x5A472AB4u, 0x5E0E5847u,
                                                          0xD05D955Fu, 0xC409728Du, 0x14DB0897u, 0xDD269D04u};
ECG_ED448_CONSTANT uint32_t DECAF448_INV_SQRT_MINUS_D[14] = {0x478797D3u, 0xAC5044A1u, 0x0E616B0Cu, 0x1044DB86u, 0x3DE045EAu,
                                                              0x418F811Du, 0xD759ADE5u, 0x2945A90Du, 0xC5A4D858u, 0xA56F6AF3u,
                                                              0xF43537F8u, 0x6FD41CA5u, 0x1DDD3FA8u, 0x910BF9ADu};
ECG_ED448_CONSTANT uint32_t DECAF448_FACTOR[14] = {0x45572736u, 0x9642EF0Fu, 0xAA20CE52u, 0x60337BF6u, 0xFD6EDED2u,
                                                   0x839A66F4u, 0x968C14BAu, 0x64A2D780u, 0xA5B8D54Bu, 0xA1F1A7B8u,
                                                   0x2FA26AA0u, 0x3BF68D72u, 0xEB24F768u, 0x22D962FBu};
ECG_ED448_CONSTANT uint32_t DECAF448_G0[2][14] = {
    {0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu, 0x55555555u, 0x55555555u,
     0x55555555u, 0x55555555u, 0x55555555u, 0x55555555u, 0x55555555u},
    {0xEA9386EDu, 0xDAEAFBCDu, 0xD1CDA06Bu, 0xBBBCB2BEu, 0x3A2A3098u, 0x0D656583u, 0x8AD8C4B8u, 0xB7E36D72u, 0x35884DD7u,
     0x036ED7A0u, 0x5086C2B0u, 0xB359D620u, 0x4AD7048Du, 0xAE05E963u}};

template <class F>
ECG_D void decaf448_const(typename F::Fe& r, const uint32_t* c) {
#pragma unroll
  for (int i = 0; i < 14; i++) r.v[i] = c[i];
}
// r = |a|: the canonical representative of a or -a, whichever is even; no branch on the value
template <class F>
ECG_D void decaf448_abs(typename F::Fe& r, const typename F::Fe& a) {
  typename F::Fe n;
  F::normalize(r, a);
  F::neg(n, r);
  F::normalize(n, n);
  F::cswap(r, n, 0u - (r.v[0] & 1u));
}
// r = -a where mask = ~0, a where mask = 0 (canonical either way)
template <class F>
ECG_D void decaf448_cneg(typename F::Fe& r, const typename F::Fe& a, uint32_t mask) {
  typename F::Fe n;
  F::normalize(r, a);
  F::neg(n, r);
  F::normalize(n, n);
  F::cswap(r, n, mask);
}
// bit 0 of the canonical representative (FieldElement::is_negative)
template <class F>
ECG_D uint32_t decaf448_is_neg(const typename F::Fe& a) {
  typename F::Fe t;
  F::normalize(t, a);
  return t.v[0] & 1u;
}
// 1 iff a^((p - 3) / 4) = r satisfies r^2 a == 1 (a is a non-zero square): FieldElement::inverse_square_root
template <class F>
ECG_D uint32_t decaf448_isr(typename F::Fe& r, const typename F::Fe& a) {
  typename F::Fe t, one;
  ed_pow_p34<F>(r, a);
  F::sqr(t, r);
  F::mul(t, t, a);
  F::set_one(one);
  return ed_eq<F>(t, one) ? 1u : 0u;
}
template <class F>
ECG_D void decaf448_store56(uint8_t* out56, const typename F::Fe& s) {
#pragma unroll
  for (int i = 0; i < 14; i++) {
    out56[4 * i] = (uint8_t)s.v[i];
    out56[4 * i + 1] = (uint8_t)(s.v[i] >> 8);
    out56[4 * i + 2] = (uint8_t)(s.v[i] >> 16);
    out56[4 * i + 3] = (uint8_t)(s.v[i] >> 24);
  }
}

// ---- the untwisted encoding (RFC 9496 section 5.3) ---------------------------------------------------------------------
// CompressedDecaf::decompress on the untwisted curve: (x, y) of s = b56; 1 iff s < p, s is even and
// I = isr(u2 u1^2) exists (u1 = 1 + s^2, u2 = u1^2 - 4 d s^2); x = |2 s I u1 sqrt(-d)| I u2 / sqrt(-d), y = (1 - s^2) I u1
template <class F>
ECG_D uint32_t decaf448_decode(typename F::Fe& x, typename F::Fe& y, const uint8_t* b56) {
  typedef typename F::Fe Fe;
  Fe s, t, ss, u1, u2, w, I, c;
  ed448_load56(s.v, b56);
  F::normalize(t, s);
  uint32_t diff = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) diff |= t.v[i] ^ s.v[i];  // s >= p changes under normalisation
  const uint32_t canonical = diff == 0, even = (s.v[0] & 1u) ^ 1u;
  F::sqr(ss, s);
  F::set_one(t);
  F::add(u1, t, ss);                      // u1 = 1 + s^2
  F::sub(y, t, ss);                       // 1 - s^2
  F::sqr(u2, u1);
  F::mul_small(t, ss, 4 * ED448_MINUS_D);
  F::add(u2, u2, t);                      // u2 = u1^2 - 4 d s^2
  F::sqr(w, u1);
  F::mul(w, w, u2);
  const uint32_t ok = decaf448_isr<F>(I, w);
  F::add(t, s, s);
  F::mul(t, t, I);
  F::mul(t, t, u1);
  decaf448_const<F>(c, DECAF448_SQRT_MINUS_D);
  F::mul(t, t, c);
  decaf448_abs<F>(t, t);                  // u3
  F::mul(t, t, I);
  F::mul(t, t, u2);
  decaf448_const<F>(c, DECAF448_INV_SQRT_MINUS_D);
  F::mul(x, t, c);
  F::normalize(x, x);
  F::mul(y, y, I);
  F::mul(y, y, u1);
  F::normalize(y, y);
  return canonical & even & ok;
}
// DecafPoint::compress of an untwisted (X : Y : Z : T) (Y is not read): u1 = (X + T)(X - T), I = isr((1 - d) u1 X^2),
// r = |I u1 sqrt(-d)|, u2 = r Z / sqrt(-d) - T, s = |(1 - d) I X u2|.  Branch-free.
template <class F>
ECG_D void decaf448_encode(uint8_t* out56, const EdPt<F>& p) {
  typedef typename F::Fe Fe;
  Fe u1, t, I, c;
  F::add(u1, p.X, p.T);
  F::sub(t, p.X, p.T);
  F::mul(u1, u1, t);
  F::sqr(t, p.X);
  F::mul(t, t, u1);
  F::mul_small(t, t, ED448_MINUS_D + 1);
  ed_pow_p34<F>(I, t);
  F::mul(t, I, u1);
  decaf448_const<F>(c, DECAF448_SQRT_MINUS_D);
  F::mul(t, t, c);
  decaf448_abs<F>(t, t);                  // r
  F::mul(t, t, p.Z);
  decaf448_const<F>(c, DECAF448_INV_SQRT_MINUS_D);
  F::mul(t, t, c);
  F::sub(t, t, p.T);                      // u2
  F::mul(t, t, p.X);
  F::mul(t, t, I);
  F::mul_small(t, t, ED448_MINUS_D + 1);
  decaf448_abs<F>(t, t);
  decaf448_store56<F>(out56, t);
}

// ---- the twisted curve of the reference's hash to group -----------------------------------------------------------------
// FieldElement::map_to_curve_decaf448 of u (any 14-word value; read mod p), twisted extended output
template <class F>
ECG_D void decaf448_tw_map(EdPt<F>& q, const typename F::Fe& u_in) {
  typedef typename F::Fe Fe;
  const uint32_t ONE_MINUS_TWO_D = 2 * ED448_MINUS_D + 1;  // 1 - 2 d = 78163
  Fe u, one, r, a, b, c, n, e, sel;
  F::normalize(u, u_in);
  F::set_one(one);
  F::sqr(r, u);
  F::neg(r, r);                           // r = -u^2
  F::sub(a, r, one);
  F::mul_small(b, a, ED448_MINUS_D);
  F::neg(b, b);                           // b = (r - 1) d
  F::add(a, b, one);
  F::sub(b, b, r);
  F::mul(c, a, b);
  F::add(a, r, one);
  F::mul_small(n, a, ONE_MINUS_TWO_D);
  F::mul(a, c, n);
  const uint32_t square = decaf448_isr<F>(b, a);
  const uint32_t sq_mask = 0u - square;
  c = u;
  F::set_one(sel);
  F::cswap(c, sel, sq_mask);              // c = 1 when square, else u
  F::mul(e, b, c);
  F::mul(a, n, e);
  decaf448_cneg<F>(a, a, 0u - ((decaf448_is_neg<F>(a) ^ 1u) ^ square));
  F::mul_small(c, e, ONE_MINUS_TWO_D);
  F::sqr(b, c);
  F::sub(e, r, one);
  F::mul(c, b, e);
  F::mul(b, c, n);
  decaf448_cneg<F>(b, b, sq_mask);
  F::sub(b, b, one);
  F::sqr(c, a);
  F::add(a, a, a);
  F::add(e, c, one);
  F::mul(q.T, a, e);
  F::mul(q.X, a, b);
  F::sub(a, one, c);
  F::mul(q.Y, e, a);
  F::mul(q.Z, a, b);
}
// r = p + q on the twisted curve (a = -1, d = -39082): ExtendedPoint::add_extended, then to_extended (T = T1 T2)
template <class F>
ECG_D void decaf448_tw_add(EdPt<F>& r, const EdPt<F>& p, const EdPt<F>& q) {
  typename F::Fe A, B, C, D, E, t;
  F::mul(A, p.X, q.X);
  F::mul(B, p.Y, q.Y);
  F::mul(C, p.T, q.T);
  F::mul_small(C, C, ED448_MINUS_D + 1);
  F::neg(C, C);                           // C = T1 T2 d'
  F::mul(D, p.Z, q.Z);
  F::add(E, p.X, p.Y);
  F::add(t, q.X, q.Y);
  F::mul(E, E, t);
  F::sub(E, E, A);
  F::sub(E, E, B);
  F::add(t, B, A);                        // H
  F::sub(B, D, C);                        // F
  F::add(C, D, C);                        // G
  F::mul(r.X, E, B);
  F::mul(r.Y, C, t);
  F::mul(r.Z, B, C);
  F::mul(r.T, E, t);
}
// DecafPoint::compress of a twisted (X : Y : Z : T) (Y is not read)
template <class F>
ECG_D void decaf448_tw_compress(uint8_t* out56, const EdPt<F>& p) {
  typedef typename F::Fe Fe;
  Fe xx_tt, t, I, ratio, c;
  F::add(xx_tt, p.X, p.T);
  F::sub(t, p.X, p.T);
  F::mul(xx_tt, xx_tt, t);
  F::sqr(t, p.X);
  F::mul(t, t, xx_tt);
  F::mul_small(t, t, ED448_MINUS_D);      // NEG_EDWARDS_D = 39081
  ed_pow_p34<F>(I, t);
  F::mul(ratio, I, xx_tt);
  decaf448_const<F>(c, DECAF448_FACTOR);
  F::mul(t, ratio, c);
  decaf448_cneg<F>(ratio, ratio, 0u - decaf448_is_neg<F>(t));
  F::mul(t, ratio, p.Z);
  F::sub(t, t, p.T);                      // k
  F::mul_small(t, t, ED448_MINUS_D);
  F::mul(t, t, I);
  F::mul(t, t, p.X);
  decaf448_abs<F>(t, t);
  decaf448_store56<F>(out56, t);
}

// ---- expand_message_xof (RFC 9380 section 5.3.2) --------------------------------------------------------------------------
// The bytes that follow the message: I2OSP(len_in_bytes, 2) || DST' || I2OSP(len(DST'), 1), prepared by the host (DST' is
// the DST, or for a DST over 255 bytes SHAKE256("H2C-OVERSIZE-DST-" || DST, 2 k / 8)); a kernel parameter
struct XofSuffix {
  uint8_t b[2 + 255 + 1];
  uint32_t len;
};
// out = expand_message_xof(msg, DST, N) with SHAKE256 for the suffix of that DST and N, any N (RFC 9380 bounds it by
// 65535): outputs past the 136-byte rate take one more permutation per block (the edwards448 RO suite reads 2 x 84 bytes)
template <int N>
ECG_D void expand_message_xof(uint8_t* out, const uint8_t* msg, size_t mlen, const XofSuffix& suffix) {
  Shake256 sh;
  sh.init();
  sh.absorb(msg, mlen);
  sh.absorb(suffix.b, suffix.len);
  if constexpr (N <= 136)
    sh.finish<N>(out);
  else
    sh.finish_long<N>(out);
}

// ---- scalars ---------------------------------------------------------------------------------------------------------------
// the Ed448 base-point scalar of [k]G: (-2 k) mod ell, for k < ell (14 words); no branch on k
ECG_D void decaf448_gen_scalar(uint32_t* r, const uint32_t* k) {
  uint32_t t[14], u[14], c = 0, borrow = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {  // t = 2 k < 2 ell < 2^447
    t[i] = (k[i] << 1) | c;
    c = k[i] >> 31;
  }
#pragma unroll
  for (int i = 0; i < 14; i++) {  // u = t - ell; keep it unless it borrowed
    const uint64_t d = (uint64_t)t[i] - ED448_L[i] - borrow;
    u[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 63);
  }
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    t[i] = borrow ? t[i] : u[i];  // 2 k mod ell
    nz |= t[i];
  }
  const uint32_t m = 0u - (uint32_t)(nz != 0);
  borrow = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {  // ell - t, or 0 for t = 0
    const uint64_t d = (uint64_t)(ED448_L[i] & m) - t[i] - borrow;
    r[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 63);
  }
}
// r = h mod ell for 64 little-endian bytes (Reduce<Array<u8, U64>> for DecafScalar): the 114-byte fold of verification
ECG_D void decaf448_mod_l_64(uint32_t* r, const uint8_t* h64) {
  uint8_t h[114];
#pragma unroll
  for (int i = 0; i < 64; i++) h[i] = h64[i];
#pragma unroll
  for (int i = 64; i < 114; i++) h[i] = 0;
  ed448_mod_l_wide(r, h);
}

// ---- the per-element bodies (shared by the kernels and the host twin of tests/dev) -----------------------------------------
// the scalar of element i (zero when refused, after reporting it)
ECG_D void decaf448_load_scalar(uint32_t* k14, const uint8_t* k56, size_t i, size_t base, uint32_t* status) {
  const uint8_t* r = k56 + 56 * i;
  ed448_load56(k14, r);
  if (!ed448_scalar_ok(r)) {
    ed448g_report(status, ED448G_ERR_SCALAR, base + i);
#pragma unroll
    for (int j = 0; j < 14; j++) k14[j] = 0;
  }
}
// ext[i] = [k_i] P_i (p56 == nullptr: P_i = G0); a refused record is reported with its index base + i and computed as
// k = 0 or P = O
template <class F, bool CT>
ECG_D void decaf448_mul_elem(size_t i, const uint8_t* k56, const uint8_t* p56, size_t n, size_t base, uint32_t* ext, uint32_t* status,
                             bool scrub) {
  uint32_t k14[14];
  decaf448_load_scalar(k14, k56, i, base, status);
  typename F::Fe x, y;
  if (p56) {
    if (!decaf448_decode<F>(x, y, p56 + 56 * i)) {
      ed448g_report(status, ED448G_ERR_POINT, base + i);
      F::set_zero(x);
      F::set_one(y);
    }
  } else {
    decaf448_const<F>(x, DECAF448_G0[0]);
    decaf448_const<F>(y, DECAF448_G0[1]);
  }
  EdPt<F> q;
  ed448_mul_var<F, CT>(q, k14, x, y, scrub);
  ed448_store_ext<F>(ext, n, i, q);
}
// ext[i] = [(-2 k_i) mod ell] B from the Ed448 fixed-base table: [k_i]G up to 2-torsion
template <class F>
ECG_D void decaf448_fixed_elem(size_t i, const uint8_t* k56, size_t n, size_t base, const uint32_t* tab, uint32_t* ext, uint32_t* status) {
  uint32_t k14[14], g14[14];
  decaf448_load_scalar(k14, k56, i, base, status);
  decaf448_gen_scalar(g14, k14);
  EdPt<F> q;
  ed448_mul_fixed<F>(q, g14, tab);
  ed448_store_ext<F>(ext, n, i, q);
}
template <class F>
ECG_D void decaf448_encode_elem(size_t i, const uint32_t* ext, size_t n, uint8_t* out56) {
  EdPt<F> p;
  ed448_load_ext<F>(p, ext, n, i);
  decaf448_encode<F>(out56 + 56 * i, p);
}
template <class F>
ECG_D void decaf448_check_elem(size_t i, const uint8_t* p56, uint8_t* ok) {
  typename F::Fe x, y;
  ok[i] = (uint8_t)decaf448_decode<F>(x, y, p56 + 56 * i);
}
// DecafPoint::from_uniform_bytes then compress (decaf/points.rs:79-92) of 56 bytes (ONE = true: a single map, the
// encode_from_bytes form) or 112 bytes (two maps, each half little-endian mod p, added on the twisted curve)
template <class F, bool ONE>
ECG_D void decaf448_from_uniform(uint8_t* out56, const uint8_t* u) {
  typename F::Fe fe;
  EdPt<F> q0;
  ed448_load56(fe.v, u);
  decaf448_tw_map<F>(q0, fe);
  if (!ONE) {
    EdPt<F> q1;
    ed448_load56(fe.v, u + 56);
    decaf448_tw_map<F>(q1, fe);
    decaf448_tw_add<F>(q0, q0, q1);
  }
  decaf448_tw_compress<F>(out56, q0);
}
// hash to group of one message: NU = false reads 112 bytes and adds two maps, NU = true reads 56 bytes and maps once
template <class F, bool NU>
ECG_D void decaf448_h2c_one(uint8_t* out56, const uint8_t* msg, size_t mlen, const XofSuffix& suffix) {
  uint8_t u[112];
  if (NU)
    expand_message_xof<56>(u, msg, mlen, suffix);
  else
    expand_message_xof<112>(u, msg, mlen, suffix);
  decaf448_from_uniform<F, NU>(out56, u);
}
ECG_D void decaf448_h2s_one(uint8_t* out56, const uint8_t* msg, size_t mlen, const XofSuffix& suffix) {
  uint8_t u[64];
  expand_message_xof<64>(u, msg, mlen, suffix);
  uint32_t r[14];
  decaf448_mod_l_64(r, u);
#pragma unroll
  for (int i = 0; i < 14; i++) {
    out56[4 * i] = (uint8_t)r[i];
    out56[4 * i + 1] = (uint8_t)(r[i] >> 8);
    out56[4 * i + 2] = (uint8_t)(r[i] >> 16);
    out56[4 * i + 3] = (uint8_t)(r[i] >> 24);
  }
}

#if defined(__CUDACC__)
template <class F, bool CT>
__global__ void __launch_bounds__(DECAF448_BLOCK, DECAF448_MINBLK)
    decaf448_mul_kernel(const uint8_t* k56, const uint8_t* p56, size_t n, size_t base, uint32_t* ext, uint32_t* status, bool scrub) {
  const size_t i = (size_t)blockIdx.x * DECAF448_BLOCK + threadIdx.x;
  if (i < n) decaf448_mul_elem<F, CT>(i, k56, p56, n, base, ext, status, scrub);
}
template <class F>
__global__ void __launch_bounds__(DECAF448_BLOCK, DECAF448_FB_MINBLK)
    decaf448_fixed_kernel(const uint8_t* k56, size_t n, size_t base, const uint32_t* __restrict__ tab, uint32_t* ext, uint32_t* status) {
  const size_t i = (size_t)blockIdx.x * DECAF448_BLOCK + threadIdx.x;
  if (i < n) decaf448_fixed_elem<F>(i, k56, n, base, tab, ext, status);
}
template <class F>
__global__ void __launch_bounds__(DECAF448_BLOCK) decaf448_encode_kernel(const uint32_t* ext, size_t n, uint8_t* out56) {
  const size_t i = (size_t)blockIdx.x * DECAF448_BLOCK + threadIdx.x;
  if (i < n) decaf448_encode_elem<F>(i, ext, n, out56);
}
template <class F>
__global__ void __launch_bounds__(DECAF448_BLOCK) decaf448_check_kernel(const uint8_t* p56, size_t n, uint8_t* ok) {
  const size_t i = (size_t)blockIdx.x * DECAF448_BLOCK + threadIdx.x;
  if (i < n) decaf448_check_elem<F>(i, p56, ok);
}
// one message per thread: message i is msgs[offs[i] - base .. offs[i + 1] - base)
template <class F, bool NU>
__global__ void __launch_bounds__(DECAF448_BLOCK, DECAF448_H2C_MINBLK)
    decaf448_h2c_kernel(const uint8_t* msgs, const uint64_t* offs, uint64_t base, size_t n, XofSuffix suffix, uint8_t* out56) {
  const size_t i = (size_t)blockIdx.x * DECAF448_BLOCK + threadIdx.x;
  if (i >= n) return;
  const uint64_t lo = offs[i], hi = offs[i + 1];
  decaf448_h2c_one<F, NU>(out56 + 56 * i, msgs + (lo - base), (size_t)(hi - lo), suffix);
}
__global__ void __launch_bounds__(DECAF448_BLOCK, DECAF448_H2S_MINBLK)
    decaf448_h2s_kernel(const uint8_t* msgs, const uint64_t* offs, uint64_t base, size_t n, XofSuffix suffix, uint8_t* out56) {
  const size_t i = (size_t)blockIdx.x * DECAF448_BLOCK + threadIdx.x;
  if (i >= n) return;
  const uint64_t lo = offs[i], hi = offs[i + 1];
  decaf448_h2s_one(out56 + 56 * i, msgs + (lo - base), (size_t)(hi - lo), suffix);
}
// SHAKE256("H2C-OVERSIZE-DST-" || DST, 56) for a DST over 255 bytes (expand_msg.rs:70-97, L = 2 k = 56); one thread
__global__ void xof_oversize_dst_kernel(const uint8_t* dst, size_t dst_len, uint8_t* out56) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  Shake256 sh;
  sh.init();
  const uint8_t salt[17] = {'H', '2', 'C', '-', 'O', 'V', 'E', 'R', 'S', 'I', 'Z', 'E', '-', 'D', 'S', 'T', '-'};
  sh.absorb(salt, 17);
  sh.absorb(dst, dst_len);
  sh.finish<56>(out56);
}
#endif

}  // namespace ecg
