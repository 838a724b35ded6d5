// ecg_ed448_group.cuh — Ed448 group operations over a batch: [k]P, [k]B and sum k_i P_i on the Edwards curve of
// ed448-goldilocks (EdwardsPoint: Mul<&EdwardsScalar>, MulVartime, Group::mul_by_generator, LinearCombination), built
// on the point layer of ecg_ed448.cuh (ed_dbl, ed_add, ed448_decode, ed448_recode, the subgroup test), which is used
// unchanged.
//
// The contract is the reference's encodings, verdict for verdict:
//   - a scalar is a 57-byte little-endian record accepted iff EdwardsScalar::from_canonical_bytes accepts it
//     (edwards/scalar.rs:32-42): its test (byte 56 == 0 | byte 55 >> 6 == 0) & (bytes 0..55 < ell) reduces, as
//     ell < 2^446, to "bytes 0..55 < ell"; byte 56 is ignored;
//   - a point is a 57-byte record accepted iff CompressedEdwardsY::decompress accepts it (edwards/affine.rs:487-520):
//     y = bytes 0..55 reduced mod p, the sign of x is bit 7 of byte 56 (bits 0-6 ignored), on the curve and torsion
//     free.  Unlike verification the identity (0, 1) is accepted, under either sign bit; (0, -1) is refused, and so is
//     the all-zero record (y = 0 is a point of order 4);
//   - an output is AffinePoint::compress (edwards/affine.rs:29-41): canonical y little-endian, byte 56 = (x mod 2) << 7;
//     the identity is 01 00 .. 00.
// The reference's scalar_mul computes [4 (s / 4 mod ell)]P through the 4-isogeny (edwards/extended.rs:357-365), which is
// [s]P on the prime-order subgroup, the only points the encoding lets in; so any correct algorithm gives its bits.
//
// Variable base ([k]P, one thread per pair): k is made odd by adding ell when it is even (P has order ell), recoded into
// 112 signed odd 4-bit digits (ed448_recode), and each of the 112 windows runs 4 doublings and one addition from a
// per-thread table of the odd multiples P, 3P, .., 15P: every window adds, so a warp runs one instruction stream, and the
// complete formulas need no exceptional case (k = 0 becomes [ell]P = O on its own).  The table lives in local memory.
// CT (ECG_FLAG_CONSTTIME): the table is read by a masked scan of all 8 entries, the sign by a masked swap, and ell is
// added under a mask: no branch and no memory address depends on k.  The default path indexes the table by digit.
//
// Fixed base ([k]B): signed odd ED448_FBW-bit digits and one affine table per window, entry (i, j) = (2j + 1) 2^(W i) B
// as (x, y, d x y), one mixed addition per window and no doubling.  The table is built on the device at first use by the
// variable-base kernel and the normalisation kernel below (ecgpu.cu, ensure_ed448_table).
//
// Normalisation: Montgomery's trick along each thread's strided slice (one inversion per slice), then the compressed
// record, or for the fixed-base table the entry (x, y, d x y).
//
// Intermediate points are extended (X, Y, Z, T) in SoA word-major form: word w of element i at buf[w * stride + i].
#pragma once
#include "ecg_ed448.cuh"

namespace ecg {

// launch geometry (DESIGN.md section 7, "Ed448 group operations"): the tightest bounds without spills
#define ED448G_BLOCK 128
#define ED448G_MINBLK 2     // variable base
#define ED448G_FB_MINBLK 2  // fixed base
#define ED448G_NORM_SLICE 32  // elements per thread of the normalisation kernel
#define ED448_FBW 8                                  // fixed-base digit width
#define ED448_FBND ((447 + ED448_FBW - 1) / ED448_FBW)  // fixed-base windows: 56
#define ED448_FBE (1 << (ED448_FBW - 1))             // entries per window: 128
#define ED448_FB_WORDS (ED448_FBND * ED448_FBE * 42)  // the whole table in 32-bit words (1.2 MB)
#define ED448G_ERR_SCALAR 1u  // the ERRF_SCALAR / ERRF_POINT bits that ecgpu.cu's finish() reads
#define ED448G_ERR_POINT 2u

// ---- scalars and points --------------------------------------------------------------------------------------------------
// EdwardsScalar::from_canonical_bytes accepts k57: bytes 0..55 < ell (byte 56 is ignored)
ECG_D uint32_t ed448_scalar_ok(const uint8_t* k57) {
  uint32_t s[14];
  ed448_load56(s, k57);
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    const uint64_t d = (uint64_t)s[i] - ED448_L[i] - borrow;
    borrow = (uint32_t)(d >> 63);
  }
  return borrow;
}
// CompressedEdwardsY::decompress: 1 iff the record decodes to a point of the prime-order subgroup, the identity included
template <class F>
ECG_D uint32_t ed448_group_decompress(typename F::Fe& x, typename F::Fe& y, const uint8_t* b57) {
  if (!ed448_decode<F>(x, y, b57)) return 0;
  typename F::Fe one;
  F::set_one(one);
  if (ed_eq<F>(y, one)) return 1;  // the identity; x = 0 under either sign bit
  return ed448_subgroup_not_identity<F>(y);
}
// r = k, plus ell when k is even, under a mask (k < ell, so r < 2 ell < 2^447 and r is odd)
ECG_D void ed448_make_odd(uint32_t* r, const uint32_t* k) {
  const uint32_t m = (k[0] & 1u) - 1u;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    c += (uint64_t)k[i] + (ED448_L[i] & m);
    r[i] = (uint32_t)c;
    c >>= 32;
  }
}
// odd k (< 2^447) -> ND signed odd digits of W bits, k = sum dig[i] 2^(W i) (ed448_recode for digits wider than int8_t)
template <int W, int ND>
ECG_D void ed448_recode16(int16_t* dig, const uint32_t* k14) {
  uint32_t t[15];
#pragma unroll
  for (int i = 0; i < 14; i++) t[i] = k14[i];
  t[14] = 0;
#pragma unroll 1
  for (int i = 0; i < ND - 1; i++) {
    const int d = (int)(t[0] & ((2u << W) - 1)) - (1 << W);
    dig[i] = (int16_t)d;
    int64_t c = -(int64_t)d;
#pragma unroll 1
    for (int j = 0; j < 15; j++) {
      c += (int64_t)t[j];
      t[j] = (uint32_t)c;
      c >>= 32;
    }
#pragma unroll 1
    for (int j = 0; j < 14; j++) t[j] = (t[j] >> W) | (t[j + 1] << (32 - W));
    t[14] >>= W;
  }
  dig[ND - 1] = (int16_t)t[0];
}

// ---- variable base ---------------------------------------------------------------------------------------------------------
// e = tab[|d| >> 1], negated for d < 0 (tab entries: X, Y, Z, d T).  CT: a masked scan and a masked negation.
template <class F, bool CT>
ECG_D void ed448_pick(EdPt<F>& e, const EdPt<F>* tab, int d) {
  const int32_t s = d >> 31;
  const uint32_t a = (uint32_t)((d ^ s) - s) >> 1;
  if (CT) {
#pragma unroll
    for (int i = 0; i < 14; i++) e.X.v[i] = e.Y.v[i] = e.Z.v[i] = e.T.v[i] = 0;
#pragma unroll 1
    for (uint32_t j = 0; j < 8; j++) {
      const uint32_t m = 0u - (uint32_t)(j == a);
#pragma unroll
      for (int i = 0; i < 14; i++) {
        e.X.v[i] |= tab[j].X.v[i] & m;
        e.Y.v[i] |= tab[j].Y.v[i] & m;
        e.Z.v[i] |= tab[j].Z.v[i] & m;
        e.T.v[i] |= tab[j].T.v[i] & m;
      }
    }
    typename F::Fe nx, nt;
    F::neg(nx, e.X);
    F::neg(nt, e.T);
    F::cswap(e.X, nx, (uint32_t)s);
    F::cswap(e.T, nt, (uint32_t)s);
  } else {
    e = tab[a];
    if (s) {
      F::neg(e.X, e.X);
      F::neg(e.T, e.T);
    }
  }
}
// q = [k] (x, y) for k < ell (14 little-endian words) and (x, y) in the prime-order subgroup.  scrub: overwrite the
// table and the digits (secret-derived, in local memory) before returning.
template <class F, bool CT>
ECG_D void ed448_mul_var(EdPt<F>& q, const uint32_t* k14, const typename F::Fe& x, const typename F::Fe& y, bool scrub) {
  uint32_t ko[14];
  ed448_make_odd(ko, k14);
  int8_t dig[ED448_AND];
  ed448_recode<ED448_AW, ED448_AND>(dig, ko);
  EdPt<F> tab[8], p1, p2, e;
  p1.X = x;
  p1.Y = y;
  F::set_one(p1.Z);
  F::mul(p1.T, x, y);
  ed_dbl<F>(p2, p1, true);
  typename F::Fe dt2;
  ed_mul_d<F>(dt2, p2.T);
  tab[0] = p1;
#pragma unroll 1
  for (int j = 1; j < 8; j++) ed_add<F>(tab[j], tab[j - 1], p2.X, p2.Y, &p2.Z, dt2);
#pragma unroll 1
  for (int j = 0; j < 8; j++) ed_mul_d<F>(tab[j].T, tab[j].T);
  F::set_zero(q.X);
  F::set_one(q.Y);
  F::set_one(q.Z);
  F::set_zero(q.T);
#pragma unroll 1
  for (int w = ED448_AND - 1; w >= 0; w--) {
    if (w != ED448_AND - 1) {
      ed_dbl<F>(q, q, false);
      ed_dbl<F>(q, q, false);
      ed_dbl<F>(q, q, false);
      ed_dbl<F>(q, q, true);
    }
    ed448_pick<F, CT>(e, tab, dig[w]);
    ed_add<F>(q, q, e.X, e.Y, &e.Z, e.T);
  }
  if (scrub) {
    volatile uint32_t* vt = reinterpret_cast<volatile uint32_t*>(tab);
#pragma unroll 1
    for (int i = 0; i < (int)(sizeof tab / 4); i++) vt[i] = 0;
    volatile int8_t* vd = dig;
#pragma unroll 1
    for (int i = 0; i < ED448_AND; i++) vd[i] = 0;
  }
}

// ---- fixed base --------------------------------------------------------------------------------------------------------------
// q = [k] B from the window table (ED448_FB_WORDS words: entry (i, j) at 42 (ED448_FBE i + j)); default path only
template <class F>
ECG_D void ed448_mul_fixed(EdPt<F>& q, const uint32_t* k14, const uint32_t* __restrict__ tab) {
  uint32_t ko[14];
  ed448_make_odd(ko, k14);
  int16_t dig[ED448_FBND];
  ed448_recode16<ED448_FBW, ED448_FBND>(dig, ko);
  F::set_zero(q.X);
  F::set_one(q.Y);
  F::set_one(q.Z);
  F::set_zero(q.T);
#pragma unroll 1
  for (int w = 0; w < ED448_FBND; w++) {
    const int d = dig[w];
    const uint32_t* ent = tab + 42 * (ED448_FBE * w + ((d < 0 ? -d : d) >> 1));
    typename F::Fe ex, ey, edt;
#pragma unroll
    for (int i = 0; i < 14; i++) {
#if defined(__CUDA_ARCH__)
      ex.v[i] = __ldg(ent + i);
      ey.v[i] = __ldg(ent + 14 + i);
      edt.v[i] = __ldg(ent + 28 + i);
#else
      ex.v[i] = ent[i];
      ey.v[i] = ent[14 + i];
      edt.v[i] = ent[28 + i];
#endif
    }
    if (d < 0) {
      F::neg(ex, ex);
      F::neg(edt, edt);
    }
    ed_add<F>(q, q, ex, ey, nullptr, edt);
  }
}

// ---- SoA storage and the per-element bodies (shared by the kernels and the host twin of tests/dev) ------------------------
template <class F>
ECG_D void ed448_store_ext(uint32_t* buf, size_t stride, size_t i, const EdPt<F>& p) {
#pragma unroll
  for (int w = 0; w < 14; w++) {
    buf[(size_t)w * stride + i] = p.X.v[w];
    buf[(size_t)(14 + w) * stride + i] = p.Y.v[w];
    buf[(size_t)(28 + w) * stride + i] = p.Z.v[w];
    buf[(size_t)(42 + w) * stride + i] = p.T.v[w];
  }
}
template <class F>
ECG_D void ed448_load_ext(EdPt<F>& p, const uint32_t* buf, size_t stride, size_t i) {
#pragma unroll
  for (int w = 0; w < 14; w++) {
    p.X.v[w] = buf[(size_t)w * stride + i];
    p.Y.v[w] = buf[(size_t)(14 + w) * stride + i];
    p.Z.v[w] = buf[(size_t)(28 + w) * stride + i];
    p.T.v[w] = buf[(size_t)(42 + w) * stride + i];
  }
}
// status[0] |= flag, status[1] = min(status[1], idx)
ECG_D void ed448g_report(uint32_t* status, uint32_t flag, size_t idx) {
  const uint32_t i32 = (uint32_t)(idx > 0xFFFFFFFEull ? 0xFFFFFFFEull : idx);
#if defined(__CUDA_ARCH__)
  atomicOr(&status[0], flag);
  atomicMin(&status[1], i32);
#else
  status[0] |= flag;
  if (i32 < status[1]) status[1] = i32;
#endif
}
// the scalar of element i (zero when refused, after reporting it)
ECG_D void ed448g_load_scalar(uint32_t* k14, const uint8_t* k57, size_t i, size_t base, uint32_t* status) {
  const uint8_t* r = k57 + 57 * i;
  ed448_load56(k14, r);
  if (!ed448_scalar_ok(r)) {
    ed448g_report(status, ED448G_ERR_SCALAR, base + i);
#pragma unroll
    for (int j = 0; j < 14; j++) k14[j] = 0;
  }
}
// element i of a variable-base batch: ext[i] = [k_i] P_i (P57 == nullptr: P_i = B); a refused record is reported
// with its index base + i and computed as k = 0 or P = O
template <class F, bool CT>
ECG_D void ed448g_mul_elem(size_t i, const uint8_t* k57, const uint8_t* p57, size_t n, size_t base, uint32_t* ext, uint32_t* status,
                           bool scrub) {
  uint32_t k14[14];
  ed448g_load_scalar(k14, k57, i, base, status);
  typename F::Fe x, y;
  if (p57) {
    if (!ed448_group_decompress<F>(x, y, p57 + 57 * i)) {
      ed448g_report(status, ED448G_ERR_POINT, base + i);
      F::set_zero(x);
      F::set_one(y);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 14; j++) {
      x.v[j] = ED448_BTAB[0][0][j];
      y.v[j] = ED448_BTAB[0][1][j];
    }
  }
  EdPt<F> q;
  ed448_mul_var<F, CT>(q, k14, x, y, scrub);
  ed448_store_ext<F>(ext, n, i, q);
}
template <class F>
ECG_D void ed448g_fixed_elem(size_t i, const uint8_t* k57, size_t n, size_t base, const uint32_t* tab, uint32_t* ext, uint32_t* status) {
  uint32_t k14[14];
  ed448g_load_scalar(k14, k57, i, base, status);
  EdPt<F> q;
  ed448_mul_fixed<F>(q, k14, tab);
  ed448_store_ext<F>(ext, n, i, q);
}
// partial t of a sum: elements t, t + n_out, t + 2 n_out, .. of `in` (stride n_in) -> word w at out[w * out_stride + t]
template <class F>
ECG_D void ed448g_sum_elem(size_t t, const uint32_t* in, size_t n_in, uint32_t* out, size_t n_out, size_t out_stride) {
  EdPt<F> acc, p;
  F::set_zero(acc.X);
  F::set_one(acc.Y);
  F::set_one(acc.Z);
  F::set_zero(acc.T);
#pragma unroll 1
  for (size_t i = t; i < n_in; i += n_out) {
    ed448_load_ext<F>(p, in, n_in, i);
    ed_mul_d<F>(p.T, p.T);
    ed_add<F>(acc, acc, p.X, p.Y, &p.Z, p.T);
  }
  ed448_store_ext<F>(out, out_stride, t, acc);
}
// AffinePoint::compress of canonical (x, y)
template <class F>
ECG_D void ed448_compress(uint8_t* out57, const typename F::Fe& x, const typename F::Fe& y) {
#pragma unroll
  for (int i = 0; i < 14; i++) {
    out57[4 * i] = (uint8_t)y.v[i];
    out57[4 * i + 1] = (uint8_t)(y.v[i] >> 8);
    out57[4 * i + 2] = (uint8_t)(y.v[i] >> 16);
    out57[4 * i + 3] = (uint8_t)(y.v[i] >> 24);
  }
  out57[56] = (uint8_t)((x.v[0] & 1u) << 7);
}
// the slice t, t + T, t + 2T, .. of ext (n points) to affine with one inversion (scr: 14 n words of prefix products).
// TABLE = false: out = n compressed 57-byte records; TABLE = true: out = n table entries (x, y, d x y), 42 words each.
template <class F, bool TABLE>
ECG_D void ed448g_norm_slice(size_t t, size_t T, const uint32_t* ext, size_t n, uint32_t* scr, void* out) {
  typedef typename F::Fe Fe;
  Fe acc, z;
  F::set_one(acc);
  size_t last = t;
#pragma unroll 1
  for (size_t i = t; i < n; i += T) {
#pragma unroll
    for (int w = 0; w < 14; w++) {
      z.v[w] = ext[(size_t)(28 + w) * n + i];
      scr[(size_t)w * n + i] = acc.v[w];
    }
    F::mul(acc, acc, z);  // Z is never 0: the formulas are complete
    last = i;
  }
  Fe inv;
  F::inv(inv, acc);
#pragma unroll 1
  for (size_t i = last;; i -= T) {
    Fe pre, zi, x, y;
#pragma unroll
    for (int w = 0; w < 14; w++) {
      z.v[w] = ext[(size_t)(28 + w) * n + i];
      pre.v[w] = scr[(size_t)w * n + i];
      x.v[w] = ext[(size_t)w * n + i];
      y.v[w] = ext[(size_t)(14 + w) * n + i];
    }
    F::mul(zi, inv, pre);
    F::mul(inv, inv, z);
    F::mul(x, x, zi);
    F::mul(y, y, zi);
    F::normalize(x, x);
    F::normalize(y, y);
    if (TABLE) {
      Fe dt;
      F::mul(dt, x, y);
      ed_mul_d<F>(dt, dt);
      F::normalize(dt, dt);
      uint32_t* e = (uint32_t*)out + 42 * i;
#pragma unroll
      for (int w = 0; w < 14; w++) {
        e[w] = x.v[w];
        e[14 + w] = y.v[w];
        e[28 + w] = dt.v[w];
      }
    } else {
      ed448_compress<F>((uint8_t*)out + 57 * i, x, y);
    }
    if (i < T) break;
  }
}

#if defined(__CUDACC__)
template <class F, bool CT>
__global__ void __launch_bounds__(ED448G_BLOCK, ED448G_MINBLK)
    ed448g_mul_kernel(const uint8_t* k57, const uint8_t* p57, size_t n, size_t base, uint32_t* ext, uint32_t* status, bool scrub) {
  const size_t i = (size_t)blockIdx.x * ED448G_BLOCK + threadIdx.x;
  if (i < n) ed448g_mul_elem<F, CT>(i, k57, p57, n, base, ext, status, scrub);
}
template <class F>
__global__ void __launch_bounds__(ED448G_BLOCK, ED448G_FB_MINBLK)
    ed448g_fixed_kernel(const uint8_t* k57, size_t n, size_t base, const uint32_t* __restrict__ tab, uint32_t* ext, uint32_t* status) {
  const size_t i = (size_t)blockIdx.x * ED448G_BLOCK + threadIdx.x;
  if (i < n) ed448g_fixed_elem<F>(i, k57, n, base, tab, ext, status);
}
template <class F>
__global__ void __launch_bounds__(ED448G_BLOCK) ed448g_sum_kernel(const uint32_t* in, size_t n_in, uint32_t* out, size_t n_out, size_t out_stride) {
  const size_t t = (size_t)blockIdx.x * ED448G_BLOCK + threadIdx.x;
  if (t < n_out) ed448g_sum_elem<F>(t, in, n_in, out, n_out, out_stride);
}
template <class F, bool TABLE>
__global__ void __launch_bounds__(ED448G_BLOCK) ed448g_norm_kernel(const uint32_t* ext, size_t n, uint32_t* scr, void* out) {
  const size_t T = (size_t)gridDim.x * ED448G_BLOCK;
  const size_t t = (size_t)blockIdx.x * ED448G_BLOCK + threadIdx.x;
  if (t < n) ed448g_norm_slice<F, TABLE>(t, T, ext, n, scr, out);
}
#endif

}  // namespace ecg
