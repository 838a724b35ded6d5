// tests/dev/x448_dev.cu — the Curve448 field (ecg_fe_p448.cuh), the ladder step and the X448 kernel exactly as the library
// compiles them, behind a small C ABI for the tests and the variant timing of tools/bench_x448.py (test infrastructure
// only; never linked into libecgpu.so).
//
// nvcc builds libecgx448dev.so: every kernel here carries x448_kernel's production launch bound (X448_BLOCK,
// X448_MINBLK), so register allocation matches the shipped kernel's, and the per-pair entry runs x448_kernel itself.  Two
// field variants: 0 = every operation inlined (FpP448T<0>), 1 = mul / sqr as device functions (FpP448T<2>).  The same
// file built by g++ is libecgx448devsim.so: the identical bodies in a host loop over the C emulation of the carry
// primitives.  Values travel as raw little-endian 32-bit limbs (14 per element), so weakly reduced inputs in [p, 2^448)
// reach the operations.
#include <stddef.h>
#include <stdint.h>

#include "../../elliptic-curves_b200/csrc/ecg_x448.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>

#include <vector>
#endif

using namespace ecg;

#define DEV_API __attribute__((visibility("default")))
#define X448_VARIANTS(X) X(0, FpP448T<0>) X(1, FpP448T<2>)

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

// op: 0 add 1 sub 2 mul 3 sqr 4 neg 5 mul_small 39082 6 inv 7 normalize 8 cswap mask ~0 (r = b) 9 cswap mask 0 (r = a)
template <class F>
ECG_D void fe_op_elem(int op, size_t i, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  typename F::Fe x, y, r;
  ld<14>(x.v, a, i);
  ld<14>(y.v, b, i);
  switch (op) {
    case 0: F::add(r, x, y); break;
    case 1: F::sub(r, x, y); break;
    case 2: F::mul(r, x, y); break;
    case 3: F::sqr(r, x); break;
    case 4: F::neg(r, x); break;
    case 5: F::mul_small(r, x, X448_A24); break;
    case 6: F::inv(r, x); break;
    case 7: F::normalize(r, x); break;
    case 8: F::cswap(x, y, 0xFFFFFFFFu); r = x; break;
    default: F::cswap(x, y, 0u); r = x; break;
  }
  st<14>(out_raw, i, r.v);
  F::normalize(r, r);
  st<14>(out_norm, i, r.v);
}
// one ladder step: in = (x2, z2, x3, z3, u) and out = (x2, z2, x3, z3), 14 words each, element-major
template <class F>
ECG_D void step_elem(size_t i, const uint32_t* in, uint32_t* out) {
  typename F::Fe x2, z2, x3, z3, u;
  ld<14>(x2.v, in, 5 * i);
  ld<14>(z2.v, in, 5 * i + 1);
  ld<14>(x3.v, in, 5 * i + 2);
  ld<14>(z3.v, in, 5 * i + 3);
  ld<14>(u.v, in, 5 * i + 4);
  x448_ladder_step<F>(x2, z2, x3, z3, u);
  st<14>(out, 4 * i, x2.v);
  st<14>(out, 4 * i + 1, z2.v);
  st<14>(out, 4 * i + 2, x3.v);
  st<14>(out, 4 * i + 3, z3.v);
}

#if defined(__CUDACC__)
struct DevBufs {  // device copies of the host arrays of one call, freed on scope exit
  std::vector<void*> ptrs;
  cudaError_t err = cudaSuccess;
  template <class T>
  T* in(const T* h, size_t count) {
    if (!h) return nullptr;
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

template <class F>
__global__ void __launch_bounds__(X448_BLOCK, X448_MINBLK)
    fe_op_k(int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* o_raw, uint32_t* o_norm) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) fe_op_elem<F>(op, i, a, b, o_raw, o_norm);
}
template <class F>
__global__ void __launch_bounds__(X448_BLOCK, X448_MINBLK) step_k(size_t n, const uint32_t* in, uint32_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) step_elem<F>(i, in, out);
}
static unsigned grid(size_t n) { return (unsigned)((n + X448_BLOCK - 1) / X448_BLOCK); }

template <class F>
static int fe_op_t(int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  DevBufs B;
  const uint32_t* da = B.in(a, n * 14);
  const uint32_t* db = B.in(b, n * 14);
  uint32_t* dr = B.out<uint32_t>(n * 14);
  uint32_t* dn = B.out<uint32_t>(n * 14);
  if (B.err == cudaSuccess && n) fe_op_k<F><<<grid(n), X448_BLOCK>>>(op, n, da, db, dr, dn);
  B.back(out_raw, dr, n * 14);
  B.back(out_norm, dn, n * 14);
  return (int)B.err;
}
template <class F>
static int step_t(size_t n, const uint32_t* in, uint32_t* out) {
  DevBufs B;
  const uint32_t* di = B.in(in, n * 70);
  uint32_t* dout = B.out<uint32_t>(n * 56);
  if (B.err == cudaSuccess && n) step_k<F><<<grid(n), X448_BLOCK>>>(n, di, dout);
  B.back(out, dout, n * 56);
  return (int)B.err;
}
// the production kernel template; iters > 0: also time `iters` further launches with CUDA events (ms = the mean)
template <class F>
static int one_t(size_t n, const uint8_t* k, const uint8_t* u, uint8_t* out, uint8_t* ok, int iters, float* ms) {
  DevBufs B;
  const uint8_t* dk = B.in(k, n * 56);
  const uint8_t* du = B.in(u, n * 56);
  uint8_t* dout = B.out<uint8_t>(n * 56);
  uint8_t* dok = B.out<uint8_t>(n + 1);
  if (B.err == cudaSuccess && n) x448_kernel<F, X448_BLOCK, X448_MINBLK><<<grid(n), X448_BLOCK>>>(dk, du, n, dout, dok);
  if (B.err == cudaSuccess && n && iters > 0) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0);
    for (int it = 0; it < iters; it++) x448_kernel<F, X448_BLOCK, X448_MINBLK><<<grid(n), X448_BLOCK>>>(dk, du, n, dout, dok);
    cudaEventRecord(e1);
    B.err = cudaEventSynchronize(e1);
    float t = 0;
    if (B.err == cudaSuccess) B.err = cudaEventElapsedTime(&t, e0, e1);
    if (ms) *ms = t / iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  B.back(out, dout, n * 56);
  if (ok) B.back(ok, dok, n);
  return (int)B.err;
}
#else
// host: one loop, the same bodies
template <class F>
static int fe_op_t(int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  for (size_t i = 0; i < n; i++) fe_op_elem<F>(op, i, a, b, out_raw, out_norm);
  return 0;
}
template <class F>
static int step_t(size_t n, const uint32_t* in, uint32_t* out) {
  for (size_t i = 0; i < n; i++) step_elem<F>(i, in, out);
  return 0;
}
template <class F>
static int one_t(size_t n, const uint8_t* k, const uint8_t* u, uint8_t* out, uint8_t* ok, int iters, float* ms) {
  if (iters > 0) return -1;  // no timing without a device
  (void)ms;
  for (size_t i = 0; i < n; i++) x448_one<F>(k + 56 * i, u ? u + 56 * i : nullptr, out + 56 * i, ok ? ok + i : nullptr);
  return 0;
}
#endif

#define X448_DISPATCH(call)    \
  switch (v) {                 \
    X448_VARIANTS(X448_##call) \
    default: return -1;        \
  }
#define X448_FE(id, F) \
  case id: return fe_op_t<F>(op, n, a, b, out_raw, out_norm);
#define X448_STEP(id, F) \
  case id: return step_t<F>(n, in, out);
#define X448_ONE(id, F) \
  case id: return one_t<F>(n, k, u, out, ok, iters, ms);

extern "C" {

// 1 for libecgx448dev.so, 0 for the host twin
DEV_API int dev_x448_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}
DEV_API const char* dev_x448_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}
// the variant libecgpu.so ships (ECG_X448_OPT) and the launch bound every kernel here carries
DEV_API int dev_x448_shipped_variant(void) { return (ECG_X448_OPT & 2) ? 1 : 0; }
DEV_API void dev_x448_bounds(int* block, int* minblk) {
  *block = X448_BLOCK;
  *minblk = X448_MINBLK;
}
DEV_API int dev_x448_fe_op(int v, int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out_raw, uint32_t* out_norm) {
  if (op < 0 || op > 9) return -1;
  X448_DISPATCH(FE)
}
DEV_API int dev_x448_step(int v, size_t n, const uint32_t* in, uint32_t* out) { X448_DISPATCH(STEP) }
// out = X448(k, u) per pair through x448_kernel (u == NULL: the generator); ok may be NULL
DEV_API int dev_x448_one(int v, size_t n, const uint8_t* k, const uint8_t* u, uint8_t* out, uint8_t* ok) {
  const int iters = 0;
  float* ms = nullptr;
  X448_DISPATCH(ONE)
}
// the same, then `iters` timed launches of the kernel over the same device buffers: *ms = mean milliseconds per launch
DEV_API int dev_x448_time(int v, size_t n, const uint8_t* k, const uint8_t* u, uint8_t* out, int iters, float* ms) {
  uint8_t* ok = nullptr;
  if (iters < 1) return -1;
  X448_DISPATCH(ONE)
}

}  // extern "C"
