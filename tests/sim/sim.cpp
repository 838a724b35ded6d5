// tests/sim/sim.cpp — HOST SIMULATION of the device arithmetic (test infrastructure only).
// Compiles the very same .cuh headers the CUDA kernels use, with the PTX carry-chain primitives
// replaced by their C emulation (ecg_prim.cuh, #else branch), so that field / point / scalar-mult logic
// can be checked against the big-integer oracle in a container that has no GPU.  Never linked into
// libecgpu.so; never used as a fallback.
#include <pthread.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

// ---- execution-model shim for the kernel headers (ecg_kernels.cuh, ecg_msm.cuh) -------------------------------
// A kernel is an ordinary function; the launchers below run its body once per simulated thread.  Kernels without
// barriers run their threads one after another (a valid schedule: they share nothing but global memory they own or
// update atomically).  Kernels with __shared__ / __syncthreads() run one block at a time on real threads with a
// pthread barrier.
#define ECG_HOST_SIM 1
struct SimDim {
  unsigned x = 0, y = 0, z = 0;
};
static thread_local SimDim threadIdx, blockIdx, blockDim, gridDim;
static pthread_barrier_t* sim_block_barrier = nullptr;
static inline void __syncthreads() {
  if (sim_block_barrier) pthread_barrier_wait(sim_block_barrier);
}
#define __shared__ static /* one block at a time, so a function-level static is the block's shared memory */
static inline uint32_t atomicOr(uint32_t* p, uint32_t v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t atomicAdd(uint32_t* p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t atomicMin(uint32_t* p, uint32_t v) {
  uint32_t o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v < o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
  }
  return o;
}
static inline uint32_t atomicMax(uint32_t* p, uint32_t v) {
  uint32_t o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v > o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
  }
  return o;
}
struct uint4 {
  uint32_t x, y, z, w;
};
static inline uint4 __ldg(const uint4* p) { return *p; }
struct uint2 {
  uint32_t x, y;
};
static inline uint2 __ldg(const uint2* p) { return *p; }

#include "../../elliptic-curves_b200/csrc/ecg_curves.cuh"
#include "../../elliptic-curves_b200/csrc/ecg_mul.cuh"
#include "../../elliptic-curves_b200/csrc/ecg_io.cuh"
#include "../../elliptic-curves_b200/csrc/ecg_msm.cuh"
#include "../../elliptic-curves_b200/csrc/ecg_verify.cuh"

#include "../../elliptic-curves_b200/csrc/ecg_kernels.cuh"
#include "../../elliptic-curves_b200/csrc/ecg_h2c.cuh"

using namespace ecg;

// grid of ceil(threads / block) blocks, threads executed one after another
template <class Body>
static void sim_launch(size_t threads, unsigned block, Body body) {
  unsigned grid = (unsigned)((threads + block - 1) / block);
  gridDim.x = grid ? grid : 1;
  blockDim.x = block;
  for (unsigned b = 0; b < gridDim.x; b++)
    for (unsigned t = 0; t < block; t++) {
      blockIdx.x = b;
      threadIdx.x = t;
      body();
    }
}
// the same, the blocks shared out over the host's cores: for kernels without __shared__ whose threads write disjoint
// memory or update it atomically (the bucket and reduction kernels over the 2^17-slot windows of the widest geometry)
template <class Body>
static void sim_launch_par(size_t threads, unsigned block, Body body) {
  unsigned grid = (unsigned)((threads + block - 1) / block);
  if (grid == 0) grid = 1;
  unsigned nt = std::max(1u, std::min(grid, std::thread::hardware_concurrency()));
  std::vector<std::thread> th;
  for (unsigned i = 0; i < nt; i++)
    th.emplace_back([=, &body] {
      gridDim.x = grid;
      blockDim.x = block;
      for (unsigned b = i; b < grid; b += nt)
        for (unsigned t = 0; t < block; t++) {
          blockIdx.x = b;
          threadIdx.x = t;
          body();
        }
    });
  for (auto& x : th) x.join();
}
// `grid` blocks of `block` real threads each (kernels that use __shared__ / __syncthreads), one block at a time
template <class Body>
static void sim_launch_blocks(unsigned grid, unsigned block, Body body) {
  for (unsigned b = 0; b < grid; b++) {
    pthread_barrier_t bar;
    pthread_barrier_init(&bar, nullptr, block);
    sim_block_barrier = &bar;
    std::vector<std::thread> th;
    th.reserve(block);
    for (unsigned t = 0; t < block; t++)
      th.emplace_back([=, &body] {
        gridDim.x = grid;
        blockDim.x = block;
        blockIdx.x = b;
        threadIdx.x = t;
        body();
      });
    for (auto& x : th) x.join();
    sim_block_barrier = nullptr;
    pthread_barrier_destroy(&bar);
  }
}

extern "C" {

// op: 0 add 1 sub 2 mul 3 sqr 4 neg 5 half 6 mul3 7 inv 8 normalize 9 mul8   (canonical BE bytes in/out)
int sim_k256_fe_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  typedef FpK256 F;
  Fe x, y, r;
  load_be32(x.v, a);
  load_be32(y.v, b);
  switch (op) {
    case 0: F::add(r, x, y); break;
    case 1: F::sub(r, x, y); break;
    case 2: F::mul(r, x, y); break;
    case 3: F::sqr(r, x); break;
    case 4: F::neg(r, x); break;
    case 5: F::half(r, x); break;
    case 6: F::mul_small(r, x, 3); break;
    case 7: F::inv(r, x); break;
    case 8: r = x; break;
    case 9: F::mul_small(r, x, 8); break;
    default: return -1;
  }
  F::normalize(r, r);
  store_be32(out, r.v);
  return 0;
}

// raw (non-normalised) variant: inputs are arbitrary 256-bit values (exercise the weakly-reduced range)
int sim_k256_fe_op_raw(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  return sim_k256_fe_op(op, a, b, out);
}

int sim_k256_glv(const uint8_t* k_be, uint8_t* out /* h1[16] LE, neg1, even1, h2[16], neg2, even2 */) {
  uint32_t k[8];
  load_be32(k, k_be);
  GlvHalf g1, g2;
  bool ok = glv_split_k256(g1, g2, k);
  memcpy(out, g1.h, 16);
  out[16] = (uint8_t)g1.neg;
  out[17] = (uint8_t)g1.even;
  memcpy(out + 18, g2.h, 16);
  out[34] = (uint8_t)g2.neg;
  out[35] = (uint8_t)g2.even;
  return ok ? 0 : 1;
}

// full per-thread variable-base multiplication + per-point inversion
int sim_k256_mul(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  typedef FpK256 F;
  uint32_t k[8];
  load_be32(k, k_be);
  Aff P;
  load_be32(P.x.v, P_xy);
  load_be32(P.y.v, P_xy + 32);
  std::vector<uint32_t> tabmem(8 * 16);
  TabRef tab{tabmem.data(), 1};
  Jac r;
  k256_mul_thread(r, k, P, tab);
  if (F::is_zero(r.Z)) {
    memset(out_xy, 0, 64);
    *out_inf = 1;
    return 0;
  }
  Fe zinv, x, y;
  F::inv(zinv, r.Z);
  jac_to_affine_canonical<F>(x, y, r, zinv);
  store_be32(out_xy, x.v);
  store_be32(out_xy + 32, y.v);
  *out_inf = 0;
  return 0;
}

int sim_k256_on_curve(const uint8_t* P_xy) {
  typedef FpK256 F;
  Aff P;
  load_be32(P.x.v, P_xy);
  load_be32(P.y.v, P_xy + 32);
  Fe b;
  F::set_zero(b);
  b.v[0] = 7;
  return aff_on_curve<F, false>(P, b) ? 1 : 0;
}

// ---- P-256 -----------------------------------------------------------------------------------
int sim_p256_fe_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  typedef FpP256 F;
  Fe x, y, r;
  load_be32(x.v, a);
  load_be32(y.v, b);
  switch (op) {
    case 0: F::add(r, x, y); break;
    case 1: F::sub(r, x, y); break;
    case 2: F::mul(r, x, y); break;
    case 3: F::sqr(r, x); break;
    case 4: F::neg(r, x); break;
    case 5: F::half(r, x); break;
    case 6: F::mul_small(r, x, 3); break;
    case 7: F::inv(r, x); break;
    case 8: r = x; break;
    case 9: F::mul_small(r, x, 8); break;
    // boundary conversions (canonical in, canonical out): identity round trip, product, inverse
    case 10: F::from_canonical(r, x); F::to_canonical(r, r); store_be32(out, r.v); return 0;
    case 11: F::from_canonical(x, x); F::from_canonical(y, y); F::mul(r, x, y); F::to_canonical(r, r); store_be32(out, r.v); return 0;
    case 12: F::from_canonical(x, x); F::inv(r, x); F::to_canonical(r, r); store_be32(out, r.v); return 0;
    default: return -1;
  }
  F::normalize(r, r);
  store_be32(out, r.v);
  return 0;
}
// 1 when FpP256's internal form is the Montgomery domain (ops 2, 3, 7 of sim_p256_fe_op then carry a factor R^-1 / R^2)
int sim_p256_is_mont(void) { return FpP256::MONT ? 1 : 0; }
}  // extern "C"
template <class F, int AM3>
static int sim_generic_mul(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  constexpr int NL = F::NL, FB = 4 * F::NL;
  uint32_t k[NL];
  load_be<NL>(k, k_be);
  typename F::AffT P;
  load_be<NL>(P.x.v, P_xy);
  load_be<NL>(P.y.v, P_xy + FB);
  F::from_canonical(P.x, P.x);
  F::from_canonical(P.y, P.y);
  std::vector<uint32_t> tabmem(8 * 3 * NL);
  TabRefJN<NL> tab{tabmem.data(), 1};
  typename F::JacT r;
  generic_mul_thread<F, AM3>(r, k, P, tab);
  if (F::is_zero(r.Z)) {
    memset(out_xy, 0, 2 * FB);
    *out_inf = 1;
    return 0;
  }
  typename F::FeT zinv, x, y;
  F::inv(zinv, r.Z);
  jac_to_affine_canonical<F>(x, y, r, zinv);
  store_be<NL>(out_xy, x.v);
  store_be<NL>(out_xy + FB, y.v);
  *out_inf = 0;
  return 0;
}
extern "C" {
int sim_p256_mul(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  return sim_generic_mul<FpP256, true>(k_be, P_xy, out_xy, out_inf);
}
// ---- P-384 (12 limbs) ----
int sim_p384_fe_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  typedef FpP384 F;
  F::Fe x, y, r;
  load_be<12>(x.v, a);
  load_be<12>(y.v, b);
  switch (op) {
    case 0: F::add(r, x, y); break;
    case 1: F::sub(r, x, y); break;
    case 2: F::mul(r, x, y); break;
    case 3: F::sqr(r, x); break;
    case 4: F::neg(r, x); break;
    case 5: F::half(r, x); break;
    case 6: F::mul_small(r, x, 3); break;
    case 7: F::inv(r, x); break;
    case 8: r = x; break;
    case 9: F::mul_small(r, x, 8); break;
    default: return -1;
  }
  F::normalize(r, r);
  store_be<12>(out, r.v);
  return F::is_zero(r) ? 1 : 0;
}
int sim_p384_mul(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  return sim_generic_mul<FpP384, true>(k_be, P_xy, out_xy, out_inf);
}
int sim_p384_on_curve(const uint8_t* P_xy) {
  typedef FpP384 F;
  AffN<12> P;
  load_be<12>(P.x.v, P_xy);
  load_be<12>(P.y.v, P_xy + 48);
  F::Fe b;
  CurveP384::b_internal(b);
  return aff_on_curve<F, true>(P, b) ? 1 : 0;
}
// ---- curves on the generic Montgomery field policy (ecg_fe_mont.cuh / ecg_curves_ext.cuh) ----
// curve ids as in include/ecgpu.h: 3 sm2, 4 brainpoolP256r1, 5 brainpoolP256t1, 6 bign-curve256v1, 7 brainpoolP384r1,
// 8 brainpoolP384t1, 9 P-224, 10 P-192, 11 P-521
}  // extern "C"
#define SIM_FOR_EXT(curve, ...)                         \
  switch (curve) {                                      \
    case 3: { typedef CurveSm2 CV; __VA_ARGS__; } break;      \
    case 4: { typedef CurveBp256r1 CV; __VA_ARGS__; } break;  \
    case 5: { typedef CurveBp256t1 CV; __VA_ARGS__; } break;  \
    case 6: { typedef CurveBignP256 CV; __VA_ARGS__; } break; \
    case 7: { typedef CurveBp384r1 CV; __VA_ARGS__; } break;  \
    case 8: { typedef CurveBp384t1 CV; __VA_ARGS__; } break;  \
    case 9: { typedef CurveP224 CV; __VA_ARGS__; } break;     \
    case 10: { typedef CurveP192 CV; __VA_ARGS__; } break;    \
    case 11: { typedef CurveP521 CV; __VA_ARGS__; } break;    \
    default: break;                                     \
  }
// field operation on canonical records (byte order of the curve); Montgomery conversions at the boundary like the kernels
template <class C>
static int sim_ext_fe_op_t(int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  typedef typename C::F F;
  typename F::FeT x, y, r;
  load_fe<F>(x.v, a);
  load_fe<F>(y.v, b);
  F::from_canonical(x, x);
  F::from_canonical(y, y);
  switch (op) {
    case 0: F::add(r, x, y); break;
    case 1: F::sub(r, x, y); break;
    case 2: F::mul(r, x, y); break;
    case 3: F::sqr(r, x); break;
    case 4: F::neg(r, x); break;
    case 5: F::half(r, x); break;
    case 6: F::mul_small(r, x, 3); break;
    case 7: F::inv(r, x); break;
    case 8: r = x; break;
    case 9: F::mul_small(r, x, 8); break;
    default: return -1;
  }
  F::to_canonical(r, r);
  store_fe<F>(out, r.v);
  return 0;
}
template <class C>
static int sim_ext_mul_t(const uint8_t* kb, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  typedef typename C::F F;
  constexpr int NL = F::NL, FB = F::FB;
  uint32_t k[NL];
  load_fe<F>(k, kb);
  typename F::AffT P;
  load_fe<F>(P.x.v, P_xy);
  load_fe<F>(P.y.v, P_xy + FB);
  F::from_canonical(P.x, P.x);
  F::from_canonical(P.y, P.y);
  typename F::FeT bb;
  C::b_internal(bb);
  if (!aff_on_curve<F, C::A_IS_MINUS3>(P, bb)) return 3;
  std::vector<uint32_t> tabmem(8 * 3 * NL);
  TabRefJN<NL> tab{tabmem.data(), 1};
  typename F::JacT r;
  generic_mul_thread<F, C::A_IS_MINUS3>(r, k, P, tab);
  if (F::is_zero(r.Z)) {
    memset(out_xy, 0, 2 * FB);
    *out_inf = 1;
    return 0;
  }
  typename F::FeT zinv, x, y;
  F::inv(zinv, r.Z);
  jac_to_affine_canonical<F>(x, y, r, zinv);
  store_fe<F>(out_xy, x.v);
  store_fe<F>(out_xy + FB, y.v);
  *out_inf = 0;
  return 0;
}
template <class C>
static int sim_ext_gen_t(uint8_t* out_xy) {  // the generator as the device constants hold it, back in canonical bytes
  typedef typename C::F F;
  typename F::AffT g;
  C::generator(g);
  typename F::FeT x, y;
  F::to_canonical(x, g.x);
  F::to_canonical(y, g.y);
  store_fe<F>(out_xy, x.v);
  store_fe<F>(out_xy + F::FB, y.v);
  return 0;
}
extern "C" {
int sim_ext_fe_op(int curve, int op, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  SIM_FOR_EXT(curve, return sim_ext_fe_op_t<CV>(op, a, b, out));
  return -1;
}
int sim_ext_mul(int curve, const uint8_t* k, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  SIM_FOR_EXT(curve, return sim_ext_mul_t<CV>(k, P_xy, out_xy, out_inf));
  return -1;
}
int sim_ext_generator(int curve, uint8_t* out_xy) {
  SIM_FOR_EXT(curve, return sim_ext_gen_t<CV>(out_xy));
  return -1;
}
// experiment variants measured in tools/kbench.cu: a = -3 doubling as 3M+5S, point-level call structure
int sim_p256_mul_3m5s(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  return sim_generic_mul<FpP256T<515 | 1024 | 2048>, true>(k_be, P_xy, out_xy, out_inf);
}
int sim_k256_mul_ptcalls(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  typedef FpK256T<6151> F;
  uint32_t k[8];
  load_be32(k, k_be);
  Aff P;
  load_be32(P.x.v, P_xy);
  load_be32(P.y.v, P_xy + 32);
  std::vector<uint32_t> tabmem(8 * 16);
  TabRef tab{tabmem.data(), 1};
  Jac r;
  k256_mul_thread<F>(r, k, P, tab);
  if (F::is_zero(r.Z)) {
    memset(out_xy, 0, 64);
    *out_inf = 1;
    return 0;
  }
  Fe zinv, x, y;
  F::inv(zinv, r.Z);
  jac_to_affine_canonical<F>(x, y, r, zinv);
  store_be32(out_xy, x.v);
  store_be32(out_xy + 32, y.v);
  *out_inf = 0;
  return 0;
}
// generic (no-endomorphism) path instantiated for secp256k1 as a cross-check of the shared code
int sim_k256_mul_generic(const uint8_t* k_be, const uint8_t* P_xy, uint8_t* out_xy, uint8_t* out_inf) {
  return sim_generic_mul<FpK256, false>(k_be, P_xy, out_xy, out_inf);
}
int sim_p256_on_curve(const uint8_t* P_xy) {
  typedef FpP256 F;
  Aff P;
  load_be32(P.x.v, P_xy);
  load_be32(P.y.v, P_xy + 32);
  F::from_canonical(P.x, P.x);
  F::from_canonical(P.y, P.y);
  Fe b;
  CurveP256::b_internal(b);
  return aff_on_curve<F, true>(P, b) ? 1 : 0;
}

// Karatsuba variant of the field multiplication (OPT bit 3)
int sim_fe_mul_kara(int curve, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  Fe x, y, r;
  load_be32(x.v, a);
  load_be32(y.v, b);
  if (curve == 0) {
    FpK256T<9>::mul(r, x, y);
    FpK256T<9>::normalize(r, r);
  } else {
    FpP256T<9>::mul(r, x, y);
    FpP256T<9>::normalize(r, r);
    Fe r2;
    FpP256T<17>::mul(r2, x, y);  // column-sum reduction variant must agree
    FpP256T<17>::normalize(r2, r2);
    for (int i = 0; i < 8; i++)
      if (r2.v[i] != r.v[i]) return 1;
  }
  store_be32(out, r.v);
  return 0;
}
// ---- verification front end (ecg_verify.cuh) ----
int sim_bip340_challenge(const uint8_t* r32, const uint8_t* pk32, const uint8_t* m32, uint8_t* e_be) {
  alignas(4) uint8_t rb[32], pb[32], mb[32];
  memcpy(rb, r32, 32);
  memcpy(pb, pk32, 32);
  memcpy(mb, m32, 32);
  uint32_t e[8];
  bip340_challenge(e, rb, pb, mb);
  store_be32(e_be, e);
  return 0;
}
int sim_k256_lift_x(const uint8_t* x_be, uint8_t* y_be) {
  uint32_t x[8];
  load_be32(x, x_be);
  Aff P;
  if (!k256_lift_x<FpK256>(P, x)) return 0;
  Fe y;
  FpK256::normalize(y, P.y);
  store_be32(y_be, y.v);
  return 1;
}
int sim_sec1_decompress(int curve, const uint8_t* x_be, int y_is_odd, uint8_t* y_be) {
  uint32_t x[8];
  load_be32(x, x_be);
  Aff P;
  Fe y;
  if (curve == 0) {
    if (!sec1_decompress<CurveK256>(P, x, (uint32_t)y_is_odd)) return 0;
    FpK256::to_canonical(y, P.y);
  } else {
    if (!sec1_decompress<CurveP256>(P, x, (uint32_t)y_is_odd)) return 0;
    FpP256::to_canonical(y, P.y);
  }
  store_be32(y_be, y.v);
  return 1;
}
// op 0: a*b mod n, op 1: a^-1 mod n   (plain in, plain out; exercises to_mont / mul / inv / from_mont)
int sim_fn_op(int curve, int op, const uint8_t* a_be, const uint8_t* b_be, uint8_t* out_be) {
  uint32_t a[8], b[8], am[8], bm[8], r[8];
  load_be32(a, a_be);
  load_be32(b, b_be);
  if (curve == 0) {
    typedef FnMont<CurveK256> N;
    N::to_mont(am, a);
    N::to_mont(bm, b);
    if (op == 0) N::mul(r, am, bm); else N::inv(r, am);
    N::from_mont(r, r);
  } else {
    typedef FnMont<CurveP256> N;
    N::to_mont(am, a);
    N::to_mont(bm, b);
    if (op == 0) N::mul(r, am, bm); else N::inv(r, am);
    N::from_mont(r, r);
  }
  store_be32(out_be, r);
  return 0;
}
// bucket-method digit recoding (ecg_msm.cuh): m little-endian 36 bytes -> W signed digits
int sim_msm_recode(const uint8_t* m_le36, int c, int nbits, int32_t* out) {
  uint32_t m[9];
  memcpy(m, m_le36, 36);
  MsmGeom g;
  g.c = c;
  g.nbits = nbits;
  g.W = (nbits + c - 1) / c;
  g.nbw = (1u << (c + 1)) + 2;
  msm_recode(out, m, g);
  return g.W;
}
// the same on nm little-endian 32-bit limbs (the prep kernel passes NL + 1: 13 for the 384-bit curves, 18 for P-521)
int sim_msm_recode_n(const uint32_t* m, int nm, int c, int nbits, int32_t* out) {
  MsmGeom g;
  g.c = c;
  g.nbits = nbits;
  g.W = (nbits + c - 1) / c;
  g.nbw = (1u << (c + 1)) + 2;
  msm_recode(out, m, g, nm);
  return g.W;
}
}  // extern "C"

// ------------------------------------------------------------------------------------------------
// Kernel-level simulation: the kernel sequences of ecgpu.cu (run_chunk / launch_varbase / launch_norm), executed on
// the host.  `table` is the fixed-base table in the device layout (simk_affine_to_table of the 16*2^15+1 points).
static const int SIM_BLOCK = 128;

template <class C>
static void simk_normalize(std::vector<uint32_t>& jac, size_t n, uint8_t* out_xy, uint8_t* out_inf) {
  std::vector<uint32_t> scr(C::F::NL * n + 8);
  size_t threads = (n + 31) / 32;  // as launch_norm: slices of up to 32 elements share one inversion
  sim_launch(threads, 256, [&] { normalize_kernel<typename C::F>(jac.data(), n, scr.data(), out_xy, out_inf); });
}

extern "C" int simk_affine_to_table(int curve, size_t n, const uint8_t* xy, uint32_t* table) {
  if (curve == 0)
    sim_launch(n, 256, [&] { affine_to_table_kernel<CurveK256>(xy, n, table); });
  else if (curve == 1)
    sim_launch(n, 256, [&] { affine_to_table_kernel<CurveP256>(xy, n, table); });
  else if (curve == 2)
    sim_launch(n, 256, [&] { affine_to_table_kernel<CurveP384>(xy, n, table); });
  else
    SIM_FOR_EXT(curve, sim_launch(n, 256, [&] { affine_to_table_kernel<CV>(xy, n, table); }));
  return 0;
}

// ecg_mul_batch: status[0] = error flags, status[1] = first offending index
extern "C" int simk_mul_batch(int curve, size_t n, const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, uint8_t* out_xy,
                   uint8_t* out_inf, uint32_t* status) {
  std::vector<uint32_t> jac(24 * n + 24);
  size_t blocks = (n + SIM_BLOCK - 1) / SIM_BLOCK;
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  if (curve == 0) {
    std::vector<uint32_t> gtab(blocks * SIM_BLOCK * K_TAB_WORDS);
    sim_launch(n, SIM_BLOCK, [&] { k256_varbase_kernel<SIM_BLOCK, 4>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    simk_normalize<CurveK256>(jac, n, out_xy, out_inf);
  } else if (curve == 1) {
    std::vector<uint32_t> gtab(blocks * SIM_BLOCK * P_TAB_WORDS);
    sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<CurveP256, SIM_BLOCK, 4>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    simk_normalize<CurveP256>(jac, n, out_xy, out_inf);
  } else if (curve == 2) {
    std::vector<uint32_t> jac12(36 * n + 36), gtab(blocks * SIM_BLOCK * (8 * 36));
    sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<CurveP384, SIM_BLOCK, 4>(k, pxy, pinf, n, jac12.data(), gtab.data(), status, 0); });
    simk_normalize<CurveP384>(jac12, n, out_xy, out_inf);
  } else {
    SIM_FOR_EXT(curve, {
      constexpr size_t NLc = CV::F::NL;
      std::vector<uint32_t> jx(3 * NLc * n + 36), gtab(blocks * SIM_BLOCK * (8 * 3 * NLc));
      sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<CV, SIM_BLOCK, 4>(k, pxy, pinf, n, jx.data(), gtab.data(), status, 0); });
      simk_normalize<CV>(jx, n, out_xy, out_inf);
    });
  }
  return 0;
}

extern "C" int simk_mul_gen_batch(int curve, size_t n, const uint8_t* k, const uint32_t* table, uint8_t* out_xy, uint8_t* out_inf,
                       uint32_t* status) {
  std::vector<uint32_t> jac(36 * n + 36);
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  if (curve == 0) {
    sim_launch(n, 128, [&] { fixedbase_kernel<CurveK256>(k, n, table, jac.data(), status, 0); });
    simk_normalize<CurveK256>(jac, n, out_xy, out_inf);
  } else if (curve == 1) {
    sim_launch(n, 128, [&] { fixedbase_kernel<CurveP256>(k, n, table, jac.data(), status, 0); });
    simk_normalize<CurveP256>(jac, n, out_xy, out_inf);
  } else if (curve == 2) {
    sim_launch(n, 128, [&] { fixedbase_kernel<CurveP384>(k, n, table, jac.data(), status, 0); });
    simk_normalize<CurveP384>(jac, n, out_xy, out_inf);
  } else {
    SIM_FOR_EXT(curve, {
      sim_launch(n, 128, [&] { fixedbase_kernel<CV>(k, n, table, jac.data(), status, 0); });
      simk_normalize<CV>(jac, n, out_xy, out_inf);
    });
  }
  return 0;
}

template <class C, bool IS_K256>
static void simk_mga(size_t n, const uint8_t* a, const uint8_t* b, const uint8_t* pxy, const uint8_t* pinf,
                     const uint32_t* table, uint8_t* out_xy, uint8_t* out_inf, uint32_t* status) {
  std::vector<uint32_t> jac(24 * n + 24);
  size_t blocks = (n + SIM_BLOCK - 1) / SIM_BLOCK;
  std::vector<uint32_t> gtab(blocks * SIM_BLOCK * (IS_K256 ? K_TAB_WORDS : P_TAB_WORDS));
  sim_launch(n, SIM_BLOCK, [&] {
    mul_gen_add_kernel<C, SIM_BLOCK, 4, IS_K256>(a, b, pxy, pinf, n, table, jac.data(), gtab.data(), status, 0);
  });
  simk_normalize<C>(jac, n, out_xy, out_inf);
}

extern "C" int simk_mul_gen_add_batch(int curve, size_t n, const uint8_t* a, const uint8_t* b, const uint8_t* pxy, const uint8_t* pinf,
                           const uint32_t* table, uint8_t* out_xy, uint8_t* out_inf, uint32_t* status) {
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  if (curve == 0)
    simk_mga<CurveK256, true>(n, a, b, pxy, pinf, table, out_xy, out_inf, status);
  else
    simk_mga<CurveP256, false>(n, a, b, pxy, pinf, table, out_xy, out_inf, status);
  return 0;
}

// ecg_ecdsa_verify_batch: prep (range / low-s / on-curve checks, batched s^-1) -> a*G + b*Q -> affine -> verdict
template <class C, bool IS_K256>
static void simk_ecdsa(size_t n, const uint8_t* z, const uint8_t* sig, const uint8_t* q, int low_s, const uint32_t* table,
                       uint8_t* valid) {
  std::vector<uint32_t> scr(8 * n + 8);
  std::vector<uint8_t> vp(64 * n), va(32 * n), vb(32 * n), vok(n), vxy(64 * n), vinf(n);
  uint32_t status[2] = {0, 0xFFFFFFFFu};
  size_t threads = (n + 31) / 32;
  sim_launch(threads, 128, [&] { ecdsa_prep_kernel<C>(z, sig, q, n, low_s, scr.data(), vp.data(), va.data(), vb.data(), vok.data()); });
  simk_mga<C, IS_K256>(n, va.data(), vb.data(), vp.data(), nullptr, table, vxy.data(), vinf.data(), status);
  sim_launch(n, 256, [&] { ecdsa_check_kernel<C>(sig, vxy.data(), vinf.data(), vok.data(), n, valid); });
}

extern "C" int simk_ecdsa_verify_batch(int curve, size_t n, const uint8_t* z, const uint8_t* sig, const uint8_t* q, int low_s,
                            const uint32_t* table, uint8_t* valid) {
  if (curve == 0)
    simk_ecdsa<CurveK256, true>(n, z, sig, q, low_s, table, valid);
  else
    simk_ecdsa<CurveP256, false>(n, z, sig, q, low_s, table, valid);
  return 0;
}

// ecg_schnorr_verify_batch (BIP340)
extern "C" int simk_schnorr_verify_batch(size_t n, const uint8_t* pk, const uint8_t* msg, const uint8_t* sig, const uint32_t* table,
                              uint8_t* valid) {
  std::vector<uint8_t> vp(64 * n), va(32 * n), vb(32 * n), vok(n), vxy(64 * n), vinf(n);
  uint32_t status[2] = {0, 0xFFFFFFFFu};
  sim_launch(n, 128, [&] { schnorr_prep_kernel(pk, msg, sig, n, vp.data(), va.data(), vb.data(), vok.data()); });
  simk_mga<CurveK256, true>(n, va.data(), vb.data(), vp.data(), nullptr, table, vxy.data(), vinf.data(), status);
  sim_launch(n, 256, [&] { schnorr_check_kernel(sig, vxy.data(), vinf.data(), vok.data(), n, valid); });
  return 0;
}

extern "C" int simk_decompress_batch(int curve, size_t n, const uint8_t* sec1, uint8_t* out_xy, uint8_t* out_inf, uint8_t* valid) {
  if (curve == 0)
    sim_launch(n, 128, [&] { decompress_kernel<CurveK256>(sec1, n, out_xy, out_inf, valid); });
  else
    sim_launch(n, 128, [&] { decompress_kernel<CurveP256>(sec1, n, out_xy, out_inf, valid); });
  return 0;
}

// ------------------------------------------------------------------------------------------------
// ecg_lincomb on the host: the kernel sequences of ecgpu.cu's lincomb_shard / msm_run / reduce_points, with
// std::vector buffers in place of the lane arena.  `msm_min_terms` plays MSM_MIN_TERMS (2^13 in the product) so that a
// test can send a few hundred terms through the bucket method.  *path: 0 per-term kernel + tree sum, 1 bucket method,
// 2 bucket method refused the input as too skewed and the per-term path ran instead.
static MsmGeom simk_msm_geometry(int curve, size_t n) {  // = msm_geometry (ecgpu.cu)
  MsmGeom g;
  bool glv = curve == 0;
  size_t nsub = glv ? 2 * n : n;
  int lg = 0;
  while (((size_t)1 << (lg + 1)) <= nsub) lg++;
  g.c = std::min(16, std::max(8, lg - 5));
  static const int ext_bits[] = {256, 256, 256, 256, 384, 384, 224, 192, 544};  // ids 3..11 (32 bits per limb)
  g.nbits = glv ? 128 : (curve == 2 ? 384 : curve >= 3 ? ext_bits[curve - 3] : 256);
  while ((g.nbits + g.c - 1) / g.c > MSM_FINAL_THREADS) g.c++;
  g.W = (g.nbits + g.c - 1) / g.c;
  g.nbw = ((uint32_t)1 << (g.c + 1)) + 2;
  return g;
}
// out = {c, W, nbits, nbw} of simk_msm_geometry
extern "C" int sim_msm_geometry(int curve, size_t n, int* out) {
  MsmGeom g = simk_msm_geometry(curve, n);
  out[0] = g.c;
  out[1] = g.W;
  out[2] = g.nbits;
  out[3] = (int)g.nbw;
  return 0;
}

template <class C>
static std::vector<uint32_t> simk_reduce_points(std::vector<uint32_t> a, size_t n) {  // = reduce_points
  while (n > 1) {
    size_t m = (n + 31) / 32;
    std::vector<uint32_t> b(3 * C::F::NL * m);
    sim_launch(m, 128, [&] { jac_sum_kernel<C>(a.data(), n, b.data(), m); });
    a.swap(b);
    n = m;
  }
  return a;
}

template <class C, bool GLV>
static bool simk_msm_run(const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, size_t n, const MsmGeom& g,
                         uint32_t* status, std::vector<uint32_t>& result, int bucket_k) {  // = msm_run; false = too skewed
  const size_t nsub = GLV ? 2 * n : n;
  const size_t nb = (size_t)g.W * g.nbw;
  std::vector<size_t> lens, nchs;
  size_t len = g.nbw - 1;
  for (;;) {
    const size_t chl = lens.empty() ? MSM_CH0 : MSM_CHU;  // chunk size of this level (ecg_msm.cuh)
    size_t nch = (len + chl - 1) / chl;
    lens.push_back(len);
    nchs.push_back(nch);
    if (nch == 1) break;
    len = nch;
  }
  const int levels = (int)lens.size();
  constexpr size_t NLc = C::F::NL;
  std::vector<uint32_t> pts(nsub * 2 * NLc), count(2 * nb + 4, 0), offset(nb + 1), list(nsub * (size_t)g.W + 1), bkt(nb * 3 * NLc);
  std::vector<int32_t> digits(nsub * (size_t)g.W);
  const unsigned sb = (unsigned)((nb + MSM_SCAN_CHUNK - 1) / MSM_SCAN_CHUNK);
  std::vector<uint32_t> blocksum(sb + 1);
  uint32_t* cursor = count.data() + nb + 1;
  uint32_t* maxcnt = count.data() + 2 * nb + 3;
  sim_launch(n, 128, [&] { msm_prep_kernel<C, GLV>(k, pxy, pinf, n, g, pts.data(), digits.data(), count.data(), status, 0); });
  sim_launch_blocks(sb, MSM_SCAN_BLOCK, [&] { msm_scan_partial_kernel(count.data(), nb, blocksum.data(), maxcnt); });
  sim_launch_blocks(1, 1024, [&] { msm_scan_top_kernel(blocksum.data(), sb, offset.data(), nb); });
  sim_launch_blocks(sb, MSM_SCAN_BLOCK, [&] { msm_scan_final_kernel(count.data(), nb, blocksum.data(), offset.data()); });
  size_t avg = nsub / ((size_t)1 << (g.c - 1)) + 1;
  MsmSkew sk{maxcnt, 4096u, (uint32_t)std::min<size_t>(32 * avg, 0xFFFFFFFFu), status};
  sim_launch(nsub, 256, [&] { msm_scatter_kernel(digits.data(), nsub, g, offset.data(), cursor, list.data()); });
  if (bucket_k == 8)  // ECG_MSM_BUCKETS_PER_THREAD in the product: the warp-balanced variant (shared memory + barriers)
    sim_launch_blocks((unsigned)((nb + MSM_BS_BLOCK * 8 - 1) / (MSM_BS_BLOCK * 8)), MSM_BS_BLOCK,
                      [&] { msm_bucket_sorted_kernel<C, 8>(pts.data(), list.data(), offset.data(), nb, bkt.data(), sk); });
  else if (bucket_k == 4)
    sim_launch_blocks((unsigned)((nb + MSM_BS_BLOCK * 4 - 1) / (MSM_BS_BLOCK * 4)), MSM_BS_BLOCK,
                      [&] { msm_bucket_sorted_kernel<C, 4>(pts.data(), list.data(), offset.data(), nb, bkt.data(), sk); });
  else
  {
    // as msm_run: bucket ids by decreasing population, then one thread per bucket in that order
    std::vector<uint32_t> order(nb), ohist(MSM_ORDER_CLASSES + 1, 0);
    unsigned ob = (unsigned)std::min<size_t>((nb + 255) / 256, 7);
    sim_launch_blocks(ob, 256, [&] { msm_order_hist_kernel(offset.data(), nb, ohist.data()); });
    sim_launch_blocks(1, MSM_ORDER_CLASSES, [&] { msm_order_scan_kernel(ohist.data()); });
    sim_launch_blocks(ob, 256, [&] { msm_order_scatter_kernel(offset.data(), nb, ohist.data(), order.data()); });
    std::vector<uint32_t> seen(nb, 0);
    for (uint32_t b : order) seen[b]++;
    for (size_t b = 0; b < nb; b++)
      if (seen[b] != 1) {
        fprintf(stderr, "msm_order_*: bucket order is not a permutation (bucket %zu seen %u times)\n", b, seen[b]);
        abort();
      }
    sim_launch_par(nb, 128, [&] { msm_bucket_kernel<C>(pts.data(), list.data(), offset.data(), nb, bkt.data(), sk, order.data()); });
  }
  if (status[0] & MSM_SKEW_FLAG) {  // as finish() + the caller in ecgpu.cu: the flag is consumed, the per-term path runs
    status[0] &= ~MSM_SKEW_FLAG;
    return false;
  }
  std::vector<std::vector<uint32_t>> S(levels), X(levels);
  for (int l = 0; l < levels; l++) {
    S[l].assign((size_t)g.W * nchs[l] * 3 * NLc, 0);
    X[l].assign((size_t)g.W * nchs[l] * 3 * NLc, 0);
    const uint32_t* in = l == 0 ? bkt.data() : S[l - 1].data();
    size_t n_in = l == 0 ? nb : (size_t)g.W * nchs[l - 1];
    size_t stride = l == 0 ? g.nbw : nchs[l - 1];
    size_t off = l == 0 ? 1 : 0;
    size_t len_low = ((size_t)1 << (g.c - 1));
    for (int q = 0; q < l; q++) len_low = (len_low + (q == 0 ? MSM_CH0 : MSM_CHU) - 1) / (q == 0 ? MSM_CH0 : MSM_CHU);
    len_low = std::min(len_low, lens[l]);
    sim_launch_par((size_t)g.W * nchs[l], 128, [&] {
      msm_wreduce_kernel<C>(in, n_in, stride, off, lens[l], len_low, g.W, nchs[l], l == 0 ? nullptr : X[l - 1].data(), l, S[l].data(), X[l].data());
    });
  }
  std::vector<uint32_t> Rw((size_t)g.W * 3 * NLc);
  result.assign(3 * NLc, 0);
  sim_launch_blocks(1, MSM_FINAL_THREADS, [&] { msm_final_kernel<C>(X[levels - 1].data(), S[levels - 1].data(), g.W, g.c, levels - 1, Rw.data(), result.data()); });
  return true;
}

template <class C, bool GLV, bool IS_K256>
static void simk_lincomb_t(int curve, size_t n, const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, size_t msm_min_terms,
                           uint8_t* out_xy, uint8_t* out_inf, uint32_t* status, int* path, int bucket_k, int force_c = 0) {
  std::vector<uint32_t> res;
  *path = 0;
  if (n >= msm_min_terms) {
    MsmGeom g = simk_msm_geometry(curve, n);
    if (force_c) {  // a window width the product would pick only for a larger n
      g.c = force_c;
      g.W = (g.nbits + g.c - 1) / g.c;
      g.nbw = ((uint32_t)1 << (g.c + 1)) + 2;
    }
    *path = simk_msm_run<C, GLV>(k, pxy, pinf, n, g, status, res, bucket_k) ? 1 : 2;
  }
  if (*path != 1) {  // per-term kernel + tree sum
    constexpr size_t NLc = C::F::NL;
    std::vector<uint32_t> jac(3 * NLc * n);
    size_t blocks = (n + SIM_BLOCK - 1) / SIM_BLOCK;
    std::vector<uint32_t> gtab(blocks * SIM_BLOCK * (IS_K256 ? K_TAB_WORDS : 8 * 3 * NLc));
    if constexpr (IS_K256)
      sim_launch(n, SIM_BLOCK, [&] { k256_varbase_kernel<SIM_BLOCK, 4>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    else
      sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<C, SIM_BLOCK, 4>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    res = simk_reduce_points<C>(jac, n);
  }
  simk_normalize<C>(res, 1, out_xy, out_inf);
}

extern "C" int simk_lincomb_c(int curve, size_t n, const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, size_t msm_min_terms,
                              uint8_t* out_xy, uint8_t* out_inf, uint32_t* status, int* path, int bucket_k, int force_c) {
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  if (n == 0) {  // empty sum = identity
    memset(out_xy, 0, (curve == 2 || curve == 7 || curve == 8) ? 96 : curve == 9 ? 56 : curve == 10 ? 48 : curve == 11 ? 132 : 64);
    *out_inf = 1;
    *path = 0;
    return 0;
  }
  if (curve == 0)
    simk_lincomb_t<CurveK256, true, true>(curve, n, k, pxy, pinf, msm_min_terms, out_xy, out_inf, status, path, bucket_k, force_c);
  else if (curve == 1)
    simk_lincomb_t<CurveP256, false, false>(curve, n, k, pxy, pinf, msm_min_terms, out_xy, out_inf, status, path, bucket_k, force_c);
  else if (curve == 2)
    simk_lincomb_t<CurveP384, false, false>(curve, n, k, pxy, pinf, msm_min_terms, out_xy, out_inf, status, path, bucket_k, force_c);
  else
    SIM_FOR_EXT(curve, (simk_lincomb_t<CV, false, false>(curve, n, k, pxy, pinf, msm_min_terms, out_xy, out_inf, status, path, bucket_k, force_c)));
  return 0;
}
extern "C" int simk_lincomb_k(int curve, size_t n, const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, size_t msm_min_terms,
                              uint8_t* out_xy, uint8_t* out_inf, uint32_t* status, int* path, int bucket_k) {
  return simk_lincomb_c(curve, n, k, pxy, pinf, msm_min_terms, out_xy, out_inf, status, path, bucket_k, 0);
}
extern "C" int simk_lincomb(int curve, size_t n, const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, size_t msm_min_terms,
                            uint8_t* out_xy, uint8_t* out_inf, uint32_t* status, int* path) {
  return simk_lincomb_k(curve, n, k, pxy, pinf, msm_min_terms, out_xy, out_inf, status, path, 1);
}

// ecg_hash_to_curve_batch / ecg_hash_to_scalar_batch: h2c_kernel (expand_message_xmd, SSWU, isogeny, addition) +
// normalize_kernel, h2s_kernel.  dst_prime = DST || len(DST) as the host side of ecgpu.cu prepares it.
// curve: 0 secp256k1, 1 P-256, 2 P-384, 11 P-521
#define SIM_H2C_SUITE(curve, ...)                                                                  \
  switch (curve) {                                                                                 \
    case 0: { typedef CurveK256 CV; typedef FpMontT<MnK256> FN; __VA_ARGS__; } break;              \
    case 1: { typedef CurveP256 CV; typedef FpMontT<MnP256> FN; __VA_ARGS__; } break;              \
    case 2: { typedef CurveP384 CV; typedef FpMontT<MnP384> FN; __VA_ARGS__; } break;              \
    case 11: { typedef CurveP521 CV; typedef FpMontT<MnP521> FN; __VA_ARGS__; } break;             \
    default: return -1;                                                                            \
  }
extern "C" int simk_hash_to_curve(int curve, size_t n, const uint8_t* msgs, const uint64_t* offsets, const uint8_t* dst_prime,
                                  uint32_t dpl, int nu, uint8_t* out_xy, uint8_t* out_inf) {
  SIM_H2C_SUITE(curve, {
    (void)sizeof(FN);
    std::vector<uint32_t> jac(3 * CV::F::NL * n + 64);
    if (!nu)
      sim_launch(n, 128, [&] { h2c_kernel<CV, false>(msgs, offsets, 0, n, dst_prime, dpl, jac.data()); });
    else
      sim_launch(n, 128, [&] { h2c_kernel<CV, true>(msgs, offsets, 0, n, dst_prime, dpl, jac.data()); });
    simk_normalize<CV>(jac, n, out_xy, out_inf);
  });
  return 0;
}
extern "C" int simk_hash_to_scalar(int curve, size_t n, const uint8_t* msgs, const uint64_t* offsets, const uint8_t* dst_prime,
                                   uint32_t dpl, uint8_t* out) {
  SIM_H2C_SUITE(curve, { sim_launch(n, 128, [&] { h2s_kernel<CV, FN>(msgs, offsets, 0, n, dst_prime, dpl, out); }); });
  return 0;
}

// ECG_FLAG_CONSTTIME kernels: masked table selects, branch-free GLV sign folding; pxy == nullptr: P = G
extern "C" int simk_mul_batch_ct(int curve, size_t n, const uint8_t* k, const uint8_t* pxy, const uint8_t* pinf, uint8_t* out_xy,
                                 uint8_t* out_inf, uint32_t* status) {
  size_t blocks = (n + SIM_BLOCK - 1) / SIM_BLOCK;
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  if (curve == 0) {
    std::vector<uint32_t> jac(24 * n + 24), gtab(blocks * SIM_BLOCK * K_TAB_WORDS);
    sim_launch(n, SIM_BLOCK, [&] { k256_varbase_ct_kernel<SIM_BLOCK, 4>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    simk_normalize<CurveK256>(jac, n, out_xy, out_inf);
  } else if (curve == 1) {
    std::vector<uint32_t> jac(24 * n + 24), gtab(blocks * SIM_BLOCK * P_TAB_WORDS);
    sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<CurveP256, SIM_BLOCK, 4, true>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    simk_normalize<CurveP256>(jac, n, out_xy, out_inf);
  } else if (curve == 2) {
    std::vector<uint32_t> jac(36 * n + 36), gtab(blocks * SIM_BLOCK * (8 * 36));
    sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<CurveP384, SIM_BLOCK, 4, true>(k, pxy, pinf, n, jac.data(), gtab.data(), status, 0); });
    simk_normalize<CurveP384>(jac, n, out_xy, out_inf);
  } else {
    SIM_FOR_EXT(curve, {
      constexpr size_t NLc = CV::F::NL;
      std::vector<uint32_t> jx(3 * NLc * n + 36), gtab(blocks * SIM_BLOCK * (8 * 3 * NLc));
      sim_launch(n, SIM_BLOCK, [&] { generic_varbase_kernel<CV, SIM_BLOCK, 4, true>(k, pxy, pinf, n, jx.data(), gtab.data(), status, 0); });
      simk_normalize<CV>(jx, n, out_xy, out_inf);
    });
  }
  return 0;
}

// ecg_ecdsa_verify_batch / ecg_mul_gen_add_batch for the curves beyond secp256k1 / P-256: the generic twins
// (ecdsa_prep_generic_kernel -> mul_gen_add_generic_kernel -> normalize -> ecdsa_check_generic_kernel), curve ids 2..11
#define SIM_FOR_GENERIC(curve, ...)                        \
  if ((curve) == 2) {                                      \
    typedef CurveP384 CV;                                  \
    __VA_ARGS__;                                           \
  } else {                                                 \
    SIM_FOR_EXT(curve, __VA_ARGS__);                       \
  }
template <class C>
static void simk_mga_generic(size_t n, const uint8_t* a, const uint8_t* b, const uint8_t* pxy, const uint8_t* pinf, const uint32_t* table,
                             uint8_t* out_xy, uint8_t* out_inf, uint32_t* status) {
  constexpr size_t NLc = C::F::NL;
  std::vector<uint32_t> jac(3 * NLc * n + 64);
  size_t blocks = (n + SIM_BLOCK - 1) / SIM_BLOCK;
  std::vector<uint32_t> gtab(blocks * SIM_BLOCK * (8 * 3 * NLc));
  sim_launch(n, SIM_BLOCK, [&] { mul_gen_add_generic_kernel<C, SIM_BLOCK, 4>(a, b, pxy, pinf, n, table, jac.data(), gtab.data(), status, 0); });
  simk_normalize<C>(jac, n, out_xy, out_inf);
}
extern "C" int simk_mul_gen_add_generic(int curve, size_t n, const uint8_t* a, const uint8_t* b, const uint8_t* pxy, const uint8_t* pinf,
                                        const uint32_t* table, uint8_t* out_xy, uint8_t* out_inf, uint32_t* status) {
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  SIM_FOR_GENERIC(curve, simk_mga_generic<CV>(n, a, b, pxy, pinf, table, out_xy, out_inf, status));
  return 0;
}
template <class C>
static void simk_ecdsa_generic(size_t n, const uint8_t* z, const uint8_t* sig, const uint8_t* q, int low_s, const uint32_t* table, uint8_t* valid) {
  constexpr size_t NLc = C::F::NL, FB = C::F::FB;
  std::vector<uint32_t> scr(NLc * n + 8);
  std::vector<uint8_t> vp(2 * FB * n), va(FB * n), vb(FB * n), vok(n), vxy(2 * FB * n), vinf(n);
  uint32_t status[2] = {0, 0xFFFFFFFFu};
  size_t threads = (n + 31) / 32;
  sim_launch(threads, 128, [&] { ecdsa_prep_generic_kernel<C>(z, sig, q, n, low_s, scr.data(), vp.data(), va.data(), vb.data(), vok.data()); });
  simk_mga_generic<C>(n, va.data(), vb.data(), vp.data(), nullptr, table, vxy.data(), vinf.data(), status);
  sim_launch(n, 256, [&] { ecdsa_check_generic_kernel<C>(sig, vxy.data(), vinf.data(), vok.data(), n, valid); });
}
extern "C" int simk_ecdsa_verify_generic(int curve, size_t n, const uint8_t* z, const uint8_t* sig, const uint8_t* q, int low_s,
                                         const uint32_t* table, uint8_t* valid) {
  SIM_FOR_GENERIC(curve, simk_ecdsa_generic<CV>(n, z, sig, q, low_s, table, valid));
  return 0;
}

// ecg_decompress_batch / ecg_field_sqrt_batch for the curves beyond secp256k1 / P-256 (p = 3 mod 4)
extern "C" int simk_decompress_generic(int curve, size_t n, const uint8_t* sec1, uint8_t* out_xy, uint8_t* out_inf, uint8_t* valid) {
  SIM_FOR_GENERIC(curve, sim_launch(n, 128, [&] { decompress_generic_kernel<CV, SqrtExp<CV>::T>(sec1, n, out_xy, out_inf, valid); }));
  return 0;
}
extern "C" int simk_field_sqrt_generic(int curve, size_t n, const uint8_t* a, uint8_t* out, uint8_t* is_square, uint32_t* status) {
  status[0] = 0;
  status[1] = 0xFFFFFFFFu;
  SIM_FOR_GENERIC(curve, sim_launch(n, 128, [&] { field_sqrt_generic_kernel<CV, SqrtExp<CV>::T>(n, a, out, is_square, status, 0); }));
  return 0;
}

// ecg_sm2dsa_verify_batch: SM2DSA front end -> s*G + t*Q -> verdict
extern "C" int simk_sm2dsa_verify(size_t n, const uint8_t* e, const uint8_t* sig, const uint8_t* q, const uint32_t* table, uint8_t* valid) {
  typedef CurveSm2 C;
  constexpr size_t FB = C::F::FB;
  std::vector<uint8_t> vp(2 * FB * n), va(FB * n), vb(FB * n), vok(n), vxy(2 * FB * n), vinf(n);
  uint32_t status[2] = {0, 0xFFFFFFFFu};
  sim_launch(n, 128, [&] { sm2dsa_prep_kernel<C>(sig, q, n, vp.data(), va.data(), vb.data(), vok.data()); });
  simk_mga_generic<C>(n, va.data(), vb.data(), vp.data(), nullptr, table, vxy.data(), vinf.data(), status);
  sim_launch(n, 256, [&] { sm2dsa_check_kernel<C>(e, sig, vxy.data(), vinf.data(), vok.data(), n, valid); });
  return (int)status[0];
}

// ecg_ecdsa_recover_batch: prep (decompress R, batched r^-1) -> u1*G + u2*R -> affine -> key + verdict
template <class C, bool IS_K256>
static int simk_recover(size_t n, const uint8_t* z, const uint8_t* sig, const uint8_t* recid, int low_s, const uint32_t* table, uint8_t* out_xy,
                        uint8_t* valid) {
  std::vector<uint32_t> scr(8 * n + 8);
  std::vector<uint8_t> vp(64 * n), va(32 * n), vb(32 * n), vok(n);
  uint32_t status[2] = {0, 0xFFFFFFFFu};
  size_t threads = (n + 31) / 32;
  sim_launch(n, 128, [&] { ecdsa_recover_point_kernel<C>(sig, recid, n, low_s, vp.data(), vok.data()); });
  sim_launch(threads, 128, [&] { ecdsa_recover_prep_kernel<C>(z, sig, vok.data(), n, scr.data(), va.data(), vb.data()); });
  simk_mga<C, IS_K256>(n, va.data(), vb.data(), vp.data(), nullptr, table, out_xy, valid, status);
  sim_launch(n, 256, [&] { ecdsa_recover_finish_kernel<>(out_xy, valid, vok.data(), n); });
  return (int)status[0];
}
extern "C" int simk_ecdsa_recover_batch(int curve, size_t n, const uint8_t* z, const uint8_t* sig, const uint8_t* recid, int low_s,
                                        const uint32_t* table, uint8_t* out_xy, uint8_t* valid) {
  return curve == 0 ? simk_recover<CurveK256, true>(n, z, sig, recid, low_s, table, out_xy, valid)
                    : simk_recover<CurveP256, false>(n, z, sig, recid, low_s, table, out_xy, valid);
}
