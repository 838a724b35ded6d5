// tests/dev/fe_dev.cu — the field and point layers of the library exactly as its kernels compile them, behind a small C
// ABI for the tests (test infrastructure only; never linked into libecgpu.so).
//
// nvcc builds libecgdev.so: one element per thread, every field policy a production kernel instantiates, each under the
// launch bounds the production kernels use, so that register allocation and spilling match theirs.  The kernels of one
// launch shape form one translation unit (-DDEV_SHAPE=s, s = 0..4; they compile in parallel); the build without
// DEV_SHAPE holds the C entry points, which forward to the unit of the requested shape.  The same file built by g++ (no
// __CUDACC__) is libecgdevsim.so: the identical bodies run in a host loop with the C emulation of the carry primitives,
// which pins the test generators and expected values on a machine without a GPU.
//
// Values travel as raw little-endian 32-bit limbs (NL per element, element-major): no from_canonical and no range check,
// so weakly reduced inputs in [p, 2^(32 NL)) reach the operations of the policies that allow them.
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <type_traits>
#include <vector>

#include "../../elliptic-curves_b200/csrc/ecg_curves.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif
#if defined(__CUDACC__) && !defined(DEV_SHAPE)
#include "../../elliptic-curves_b200/csrc/ecg_kernels.cuh"
#endif

using namespace ecg;

// A = curve coefficient mode of jac_dbl / jac_madd (ecg_point.cuh); -1: a scalar field, no point operations
template <class F_, int A_>
struct Var {
  typedef F_ F;
  static constexpr int A = A_;
};
#define DEV_VARIANTS(X)                                           \
  X(0, "k256", FpK256, 0)                                         \
  X(1, "k256_inl", FpK256T<1>, 0)                                 \
  X(2, "p256", FpP256, 1)                                         \
  X(3, "p256_inl", FpP256T<513>, 1)                               \
  X(4, "p384", FpP384, 1)                                         \
  X(5, "p384_inl", FpP384T<0>, 1)                                 \
  X(6, "sm2", CurveSm2::F, CurveSm2::A_IS_MINUS3)                 \
  X(7, "bp256r1", CurveBp256r1::F, CurveBp256r1::A_IS_MINUS3)     \
  X(8, "bp256t1", CurveBp256t1::F, CurveBp256t1::A_IS_MINUS3)     \
  X(9, "bignp256", CurveBignP256::F, CurveBignP256::A_IS_MINUS3)  \
  X(10, "bp384r1", CurveBp384r1::F, CurveBp384r1::A_IS_MINUS3)    \
  X(11, "bp384t1", CurveBp384t1::F, CurveBp384t1::A_IS_MINUS3)    \
  X(12, "p224", CurveP224::F, CurveP224::A_IS_MINUS3)             \
  X(13, "p192", CurveP192::F, CurveP192::A_IS_MINUS3)             \
  X(14, "p521", CurveP521::F, CurveP521::A_IS_MINUS3)             \
  X(15, "n_k256", ScalarField<CurveK256>::T, -1)                  \
  X(16, "n_p256", ScalarField<CurveP256>::T, -1)                  \
  X(17, "n_p384", ScalarField<CurveP384>::T, -1)                  \
  X(18, "n_sm2", ScalarField<CurveSm2>::T, -1)                    \
  X(19, "n_bp256r1", ScalarField<CurveBp256r1>::T, -1)            \
  X(20, "n_bp256t1", ScalarField<CurveBp256t1>::T, -1)            \
  X(21, "n_bignp256", ScalarField<CurveBignP256>::T, -1)          \
  X(22, "n_bp384r1", ScalarField<CurveBp384r1>::T, -1)            \
  X(23, "n_bp384t1", ScalarField<CurveBp384t1>::T, -1)            \
  X(24, "n_p224", ScalarField<CurveP224>::T, -1)                  \
  X(25, "n_p192", ScalarField<CurveP192>::T, -1)                  \
  X(26, "n_p521", ScalarField<CurveP521>::T, -1)
#define DEV_VARIANT_COUNT 27
// the C entry points; everything else stays inside the library (it is built with hidden visibility, so that no kernel
// handle it shares a name with in libecgpu.so can bind across the two)
#define DEV_API __attribute__((visibility("default")))
// F::MONT where the policy declares it (the secp256k1 field has no Montgomery form)
template <class F, class = void>
struct MontOf {
  static constexpr bool v = false;
};
template <class F>
struct MontOf<F, std::void_t<decltype(F::MONT)>> {
  static constexpr bool v = F::MONT;
};

// ---- per-element bodies ---------------------------------------------------------------------------------------------
template <int NL>
ECG_D void ld(uint32_t* v, const uint32_t* src, size_t i) {
#pragma unroll
  for (int j = 0; j < NL; j++) v[j] = src[i * NL + j];
}
template <int NL>
ECG_D void st(uint32_t* dst, size_t i, const uint32_t* v) {
#pragma unroll
  for (int j = 0; j < NL; j++) dst[i * NL + j] = v[j];
}

// op: 0 add 1 sub 2 mul 3 sqr 4 neg 5 half 6 mul_small 3 7 inv 8 normalize 9 mul_small 8 10 is_zero (sim.cpp numbering)
template <class F>
ECG_D void fe_op_elem(int op, size_t i, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  constexpr int NL = F::NL;
  typename F::FeT x, y, r;
  ld<NL>(x.v, a, i);
  ld<NL>(y.v, b, i);
  switch (op) {
    case 0: F::add(r, x, y); break;
    case 1: F::sub(r, x, y); break;
    case 2: F::mul(r, x, y); break;
    case 3: F::sqr(r, x); break;
    case 4: F::neg(r, x); break;
    case 5: F::half(r, x); break;
    case 6: F::mul_small(r, x, 3); break;
    case 7: F::inv(r, x); break;
    case 8: F::normalize(r, x); break;
    case 9: F::mul_small(r, x, 8); break;
    default:
      F::set_zero(r);
      r.v[0] = F::is_zero(x) ? 1u : 0u;
      st<NL>(out_raw, i, r.v);
      st<NL>(out_norm, i, r.v);
      return;
  }
  st<NL>(out_raw, i, r.v);
  F::normalize(r, r);
  st<NL>(out_norm, i, r.v);
}

// fixedbase_accumulate's shape (ecg_kernels.cuh): the accumulator starts from an affine point with Z = set_one, takes
// L - 1 mixed additions of affine points whose y is conditionally negated by fe_cneg, and the last addition is kept or
// dropped by jac_csel (the parity correction).  start: 2 NL words per element; q: L affine points per element; neg: L
// flags per element; sel: one flag per element; out: Jacobian X, Y, Z (3 NL words per element).
template <class F, int A>
ECG_D void madd_chain_elem(size_t i, int L, const uint32_t* start, const uint32_t* q, const uint8_t* neg, const uint8_t* sel,
                           uint32_t* out) {
  constexpr int NL = F::NL;
  typename F::JacT acc, t;
  typename F::AffT e;
  ld<NL>(acc.X.v, start, 2 * i);
  ld<NL>(acc.Y.v, start, 2 * i + 1);
  F::set_one(acc.Z);
#pragma unroll 1
  for (int s = 0; s < L; s++) {
    const size_t pt = (i * L + s) * 2;
    ld<NL>(e.x.v, q, pt);
    ld<NL>(e.y.v, q, pt + 1);
    fe_cneg<F>(e.y, neg[i * L + s]);
    if (s + 1 < L) {
      jac_madd<F, A>(acc, acc, e);
    } else {
      jac_madd<F, A>(t, acc, e);
      jac_csel(acc, t, sel[i]);
    }
  }
  st<NL>(out, 3 * i, acc.X.v);
  st<NL>(out, 3 * i + 1, acc.Y.v);
  st<NL>(out, 3 * i + 2, acc.Z.v);
}

// op 0: r = 2 P (jac_dbl); 1: r = P + Q (jac_add); 2: r = P + (Q.X, Q.Y) (jac_madd, Q read as affine).  P, Q, out: 3 NL.
template <class F, int A>
ECG_D void jac_op_elem(int op, size_t i, const uint32_t* p, const uint32_t* q, uint32_t* out) {
  constexpr int NL = F::NL;
  typename F::JacT P, Q, r;
  ld<NL>(P.X.v, p, 3 * i);
  ld<NL>(P.Y.v, p, 3 * i + 1);
  ld<NL>(P.Z.v, p, 3 * i + 2);
  ld<NL>(Q.X.v, q, 3 * i);
  ld<NL>(Q.Y.v, q, 3 * i + 1);
  ld<NL>(Q.Z.v, q, 3 * i + 2);
  if (op == 0) {
    jac_dbl<F, A>(r, P);
  } else if (op == 1) {
    jac_add<F, A>(r, P, Q);
  } else {
    typename F::AffT qa;
    qa.x = Q.X;
    qa.y = Q.Y;
    jac_madd<F, A>(r, P, qa);
  }
  st<NL>(out, 3 * i, r.X.v);
  st<NL>(out, 3 * i + 1, r.Y.v);
  st<NL>(out, 3 * i + 2, r.Z.v);
}

// ---- launch shapes: the launch bounds of the production kernels -------------------------------------------------------
// 0: (256) field_op_kernel, normalize / sum kernels; 1: (128, 4) fixedbase_kernel, msm_bucket_kernel, a*G + b*P on
// secp256k1; 2: (256, 2) secp256k1 variable-base; 3: (128, 3) P-384 variable-base; 4: (128, 5) P-256 variable-base
#define DEV_SHAPES(X) X(0, 256) X(1, 128, 4) X(2, 256, 2) X(3, 128, 3) X(4, 128, 5)

#define DEV_DISPATCH(v, call)     \
  switch (v) {                    \
    DEV_VARIANTS(DEV_CASE_##call) \
    default: return -1;           \
  }
#define DEV_CASE_FE(id, nm, F, A) \
  case id: return fe_op_t<Var<F, A>>(op, n, a, b, out_raw, out_norm);
#define DEV_CASE_MADD(id, nm, F, A) \
  case id: return madd_chain_t<Var<F, A>>(n, L, start, q, neg, sel, out);
#define DEV_CASE_JAC(id, nm, F, A) \
  case id: return jac_op_t<Var<F, A>>(op, n, p, q, out);
#define DEV_CAT2(a, b) a##b
#define DEV_CAT(a, b) DEV_CAT2(a, b)

#if defined(__CUDACC__)
// device copies of the host arrays of one call, freed on scope exit
struct DevBufs {
  std::vector<void*> ptrs;
  cudaError_t err = cudaSuccess;
  template <class T>
  T* in(const T* h, size_t count) {
    void* d = nullptr;
    if (err == cudaSuccess) err = cudaMalloc(&d, count * sizeof(T) + 16);
    if (err == cudaSuccess) {
      ptrs.push_back(d);
      err = cudaMemcpy(d, h, count * sizeof(T), cudaMemcpyHostToDevice);
    }
    return (T*)d;
  }
  template <class T>
  T* out(size_t count) {
    void* d = nullptr;
    if (err == cudaSuccess) err = cudaMalloc(&d, count * sizeof(T) + 16);
    if (err == cudaSuccess) {
      ptrs.push_back(d);
      err = cudaMemset(d, 0xA5, count * sizeof(T));  // an element the kernel skips cannot pass for a result
    }
    return (T*)d;
  }
  template <class T>
  void back(T* h, const T* d, size_t count) {
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    if (err == cudaSuccess) err = cudaMemcpy(h, d, count * sizeof(T), cudaMemcpyDeviceToHost);
  }
  ~DevBufs() {
    for (void* p : ptrs) cudaFree(p);
  }
};
#endif

#if defined(__CUDACC__) && defined(DEV_SHAPE)
// ---- one launch shape: kernels and their per-variant launchers -------------------------------------------------------
#if DEV_SHAPE == 0
#define DEV_BOUNDS 256
#define DEV_BLOCK 256
#elif DEV_SHAPE == 1
#define DEV_BOUNDS 128, 4
#define DEV_BLOCK 128
#elif DEV_SHAPE == 2
#define DEV_BOUNDS 256, 2
#define DEV_BLOCK 256
#elif DEV_SHAPE == 3
#define DEV_BOUNDS 128, 3
#define DEV_BLOCK 128
#else
#define DEV_BOUNDS 128, 5
#define DEV_BLOCK 128
#endif

// The kernels of every shape unit share their template names, so each unit keeps its own in an unnamed namespace: a
// kernel's host stub is its launch handle, and one stub registered by several units would launch only one unit's code.
namespace {
template <class F>
__global__ void __launch_bounds__(DEV_BOUNDS)
    fe_op_k(int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* o_raw, uint32_t* o_norm) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) fe_op_elem<F>(op, i, a, b, o_raw, o_norm);
}
template <class F, int A>
__global__ void __launch_bounds__(DEV_BOUNDS) madd_chain_k(size_t n, int L, const uint32_t* start, const uint32_t* q,
                                                          const uint8_t* neg, const uint8_t* sel, uint32_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) madd_chain_elem<F, A>(i, L, start, q, neg, sel, out);
}
template <class F, int A>
__global__ void __launch_bounds__(DEV_BOUNDS) jac_op_k(int op, size_t n, const uint32_t* p, const uint32_t* q, uint32_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) jac_op_elem<F, A>(op, i, p, q, out);
}
static unsigned grid(size_t n) { return (unsigned)((n + DEV_BLOCK - 1) / DEV_BLOCK); }

template <class VT>
static int fe_op_t(int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  typedef typename VT::F F;
  constexpr size_t NL = F::NL;
  DevBufs B;
  const uint32_t* da = B.in(a, n * NL);
  const uint32_t* db = B.in(b, n * NL);
  uint32_t* dr = B.out<uint32_t>(n * NL);
  uint32_t* dn = B.out<uint32_t>(n * NL);
  if (B.err == cudaSuccess && n) fe_op_k<F><<<grid(n), DEV_BLOCK>>>(op, n, da, db, dr, dn);
  B.back(out_raw, dr, n * NL);
  B.back(out_norm, dn, n * NL);
  return (int)B.err;
}
template <class VT>
static int madd_chain_t(size_t n, int L, const uint32_t* start, const uint32_t* q, const uint8_t* neg, const uint8_t* sel,
                        uint32_t* out) {
  typedef typename VT::F F;
  constexpr int A = VT::A;
  constexpr size_t NL = F::NL;
  if constexpr (A < 0) {
    return -1;
  } else {
    DevBufs B;
    const uint32_t* ds = B.in(start, n * 2 * NL);
    const uint32_t* dq = B.in(q, n * L * 2 * NL);
    const uint8_t* dg = B.in(neg, n * L);
    const uint8_t* dl = B.in(sel, n);
    uint32_t* dout = B.out<uint32_t>(n * 3 * NL);
    if (B.err == cudaSuccess && n) madd_chain_k<F, A><<<grid(n), DEV_BLOCK>>>(n, L, ds, dq, dg, dl, dout);
    B.back(out, dout, n * 3 * NL);
    return (int)B.err;
  }
}
template <class VT>
static int jac_op_t(int op, size_t n, const uint32_t* p, const uint32_t* q, uint32_t* out) {
  typedef typename VT::F F;
  constexpr int A = VT::A;
  constexpr size_t NL = F::NL;
  if constexpr (A < 0) {
    return -1;
  } else {
    DevBufs B;
    const uint32_t* dp = B.in(p, n * 3 * NL);
    const uint32_t* dq = B.in(q, n * 3 * NL);
    uint32_t* dout = B.out<uint32_t>(n * 3 * NL);
    if (B.err == cudaSuccess && n) jac_op_k<F, A><<<grid(n), DEV_BLOCK>>>(op, n, dp, dq, dout);
    B.back(out, dout, n * 3 * NL);
    return (int)B.err;
  }
}
}  // namespace

extern "C" {
int DEV_CAT(dev_fe_op_s, DEV_SHAPE)(int v, int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw,
                                    uint32_t* out_norm) {
  DEV_DISPATCH(v, FE)
}
int DEV_CAT(dev_madd_chain_s, DEV_SHAPE)(int v, size_t n, int L, const uint32_t* start, const uint32_t* q, const uint8_t* neg,
                                         const uint8_t* sel, uint32_t* out) {
  DEV_DISPATCH(v, MADD)
}
int DEV_CAT(dev_jac_op_s, DEV_SHAPE)(int v, int op, size_t n, const uint32_t* p, const uint32_t* q, uint32_t* out) {
  DEV_DISPATCH(v, JAC)
}
}  // extern "C"

#else
// ---- the entry points ------------------------------------------------------------------------------------------------
#if defined(__CUDACC__)
extern "C" {
#define DEV_DECL(s, ...)                                                                                                      \
  int dev_fe_op_s##s(int, int, size_t, const uint32_t*, const uint32_t*, uint32_t*, uint32_t*);                               \
  int dev_madd_chain_s##s(int, size_t, int, const uint32_t*, const uint32_t*, const uint8_t*, const uint8_t*, uint32_t*); \
  int dev_jac_op_s##s(int, int, size_t, const uint32_t*, const uint32_t*, uint32_t*);
DEV_SHAPES(DEV_DECL)
#undef DEV_DECL
}
#define DEV_FWD(fn, shape, ...)                        \
  switch (shape) {                                     \
    case 0: return fn##_s0(__VA_ARGS__);               \
    case 1: return fn##_s1(__VA_ARGS__);               \
    case 2: return fn##_s2(__VA_ARGS__);               \
    case 3: return fn##_s3(__VA_ARGS__);               \
    case 4: return fn##_s4(__VA_ARGS__);               \
    default: return -1;                                \
  }
#else
// host: the launch shape does not exist, every shape runs the same loop
template <class VT>
static int fe_op_t(int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  for (size_t i = 0; i < n; i++) fe_op_elem<typename VT::F>(op, i, a, b, out_raw, out_norm);
  return 0;
}
template <class VT>
static int madd_chain_t(size_t n, int L, const uint32_t* start, const uint32_t* q, const uint8_t* neg, const uint8_t* sel,
                        uint32_t* out) {
  if constexpr (VT::A < 0) {
    return -1;
  } else {
    for (size_t i = 0; i < n; i++) madd_chain_elem<typename VT::F, VT::A>(i, L, start, q, neg, sel, out);
    return 0;
  }
}
template <class VT>
static int jac_op_t(int op, size_t n, const uint32_t* p, const uint32_t* q, uint32_t* out) {
  if constexpr (VT::A < 0) {
    return -1;
  } else {
    for (size_t i = 0; i < n; i++) jac_op_elem<typename VT::F, VT::A>(op, i, p, q, out);
    return 0;
  }
}
#endif

extern "C" {

DEV_API int dev_variant_count(void) { return DEV_VARIANT_COUNT; }
DEV_API const char* dev_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}
DEV_API int dev_shape_count(void) { return 5; }
// 1 when this build runs on the GPU (libecgdev.so), 0 for the host build (libecgdevsim.so)
DEV_API int dev_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}

// name, limbs, and the internal form of variant v: mont = 1 when values are a*R mod p (R = 2^(32 NL)); weak = 1 when
// results are only weakly reduced (any NL-limb integer congruent to the value: the hand-written fields, variants 0..5)
// rather than below the modulus; amode = the curve coefficient mode of the point formulas, -1 for a scalar field
DEV_API int dev_variant_info(int v, const char** name, int* nl, int* mont, int* weak, int* amode) {
  switch (v) {
#define DEV_INFO(id, nm, F, A)    \
  case id:                        \
    *name = nm;                   \
    *nl = F::NL;                  \
    *mont = MontOf<F>::v ? 1 : 0; \
    *weak = (id) < 6 ? 1 : 0;     \
    *amode = A;                   \
    return 0;
    DEV_VARIANTS(DEV_INFO)
#undef DEV_INFO
    default: return -1;
  }
}

DEV_API int dev_fe_op(int v, int shape, int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  if (shape < 0 || shape > 4 || op < 0 || op > 10) return -1;
#if defined(__CUDACC__)
  DEV_FWD(dev_fe_op, shape, v, op, n, a, b, out_raw, out_norm)
#else
  DEV_DISPATCH(v, FE)
#endif
}
DEV_API int dev_madd_chain(int v, int shape, size_t n, int L, const uint32_t* start, const uint32_t* q, const uint8_t* neg, const uint8_t* sel,
                   uint32_t* out) {
  if (shape < 0 || shape > 4 || L < 1) return -1;
#if defined(__CUDACC__)
  DEV_FWD(dev_madd_chain, shape, v, n, L, start, q, neg, sel, out)
#else
  DEV_DISPATCH(v, MADD)
#endif
}
DEV_API int dev_jac_op(int v, int shape, int op, size_t n, const uint32_t* p, const uint32_t* q, uint32_t* out) {
  if (shape < 0 || shape > 4 || op < 0 || op > 2) return -1;
#if defined(__CUDACC__)
  DEV_FWD(dev_jac_op, shape, v, op, n, p, q, out)
#else
  DEV_DISPATCH(v, JAC)
#endif
}

// fixedbase_kernel<CurveP384I> (inlined != 0: every field operation inlined, the instantiation P-384 k*G once used) or
// fixedbase_kernel<CurveP384> (call-based field operations) over a caller-built table in the device layout
// (FB_TABLE_POINTS_NL(12) affine points of 24 words).  k: 48-byte big-endian scalars; out: Jacobian (X, Y, Z) per
// element, 36 words, element-major; status: the kernel's two error words.  Host build: -1 (no kernel to run).
DEV_API int dev_fixedbase_p384(int inlined, size_t n, const uint8_t* k, const uint32_t* table, uint32_t* out, uint32_t* status) {
#if defined(__CUDACC__)
  const size_t words = FB_TABLE_POINTS_NL(12) * 24;
  DevBufs B;
  const uint8_t* dk = B.in(k, n * 48);
  const uint32_t* dt = B.in(table, words);
  uint32_t st0[2] = {0, 0xFFFFFFFFu};
  uint32_t* ds = B.in(st0, 2);
  uint32_t* dj = B.out<uint32_t>(n * 36);
  if (B.err == cudaSuccess && n) {
    const unsigned grd = (unsigned)((n + 127) / 128);
    if (inlined)
      fixedbase_kernel<CurveP384I><<<grd, 128>>>(dk, n, dt, dj, ds, 0);
    else
      fixedbase_kernel<CurveP384><<<grd, 128>>>(dk, n, dt, dj, ds, 0);
  }
  std::vector<uint32_t> soa(n * 36);
  B.back(soa.data(), dj, n * 36);
  B.back(status, ds, 2);
  // the kernel stores structure-of-arrays (soa_store: word w of element i at w * n + i); return element-major
  for (size_t i = 0; i < n; i++)
    for (size_t w = 0; w < 36; w++) out[i * 36 + w] = soa[w * n + i];
  return (int)B.err;
#else
  (void)inlined; (void)n; (void)k; (void)table; (void)out; (void)status;
  return -1;
#endif
}

}  // extern "C"
#endif
