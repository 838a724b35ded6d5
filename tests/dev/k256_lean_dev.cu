// tests/dev/k256_lean_dev.cu — the secp256k1 field operations and point formulas of the variable-base kernel's policy
// (FpK256Inline, ecg_fe_k256.cuh) next to those of the plain inlined policy FpK256T<1>, behind a small C ABI for the
// tests (test infrastructure only; never linked into libecgpu.so).
//
// nvcc builds libecgk256leandev.so: kernels under the production launch bound (256, 2).  The same file built by g++ is
// libecgk256leandevsim.so: the identical per-element bodies in a host loop over the C emulation of the carry primitives.
// Field elements travel as 8 little-endian 32-bit limbs; a Jacobian point as X, Y, Z (24 words), an affine one as x, y.
#include <stddef.h>
#include <stdint.h>

#include "../../elliptic-curves_b200/csrc/ecg_mul.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif

using namespace ecg;
typedef FpK256T<1> Plain;

#define DEV_API __attribute__((visibility("default")))

// op 0: a*b - c*d, op 1: a*b - c^2 (d unused)
ECG_D void mul_sub_elem(size_t i, int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* r) {
  Fe x, y, z, w, o;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    x.v[j] = a[8 * i + j];
    y.v[j] = b[8 * i + j];
    z.v[j] = c[8 * i + j];
    w.v[j] = d[8 * i + j];
  }
  if (op == 0)
    FpK256Inline::mul_sub(o, x, y, z, w);
  else
    FpK256Inline::mul_sub_sqr(o, x, y, z);
#pragma unroll
  for (int j = 0; j < 8; j++) r[8 * i + j] = o.v[j];
}

// op 0: 2P, op 1: P + Q (mixed addition, Q affine)
template <class F>
ECG_D void point_elem(size_t i, int op, const uint32_t* jac, const uint32_t* aff, uint32_t* out) {
  Jac p, r;
  Aff q;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    p.X.v[j] = jac[24 * i + j];
    p.Y.v[j] = jac[24 * i + 8 + j];
    p.Z.v[j] = jac[24 * i + 16 + j];
    q.x.v[j] = aff[16 * i + j];
    q.y.v[j] = aff[16 * i + 8 + j];
  }
  if (op == 0)
    jac_dbl<F, 0>(r, p);
  else
    jac_madd<F, 0>(r, p, q);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    out[24 * i + j] = r.X.v[j];
    out[24 * i + 8 + j] = r.Y.v[j];
    out[24 * i + 16 + j] = r.Z.v[j];
  }
}

#if defined(__CUDACC__)
#define BOUND __global__ void __launch_bounds__(256, 2)
BOUND mul_sub_kernel(size_t n, int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* r) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) mul_sub_elem(i, op, a, b, c, d, r);
}
template <class F>
BOUND point_kernel(size_t n, int op, const uint32_t* jac, const uint32_t* aff, uint32_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) point_elem<F>(i, op, jac, aff, out);
}

// copies the inputs to the device, runs `launch`, copies `out` back; returns a cudaError_t
template <class L>
static int on_device(size_t n, const uint32_t* const* in, const size_t* in_words, int n_in, uint32_t* out, size_t out_words, L launch) {
  void* d[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaError_t e = cudaSuccess;
  for (int k = 0; k < n_in && e == cudaSuccess; k++) {
    e = cudaMalloc(&d[k], n * in_words[k] * 4 + 16);
    if (e == cudaSuccess) e = cudaMemcpy(d[k], in[k], n * in_words[k] * 4, cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess) e = cudaMalloc(&d[4], n * out_words * 4 + 16);
  if (e == cudaSuccess) {
    launch((const uint32_t**)d, (uint32_t*)d[4]);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, d[4], n * out_words * 4, cudaMemcpyDeviceToHost);
  for (void* p : d)
    if (p) cudaFree(p);
  return (int)e;
}
static unsigned grid(size_t n) { return (unsigned)((n + 255) / 256); }
#endif

extern "C" {

DEV_API int dev_k256l_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}

DEV_API const char* dev_k256l_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}

// r[i] = (a[i] b[i] - c[i] d[i]) mod p (op 0) or (a[i] b[i] - c[i]^2) mod p (op 1), weakly reduced
DEV_API int dev_k256l_mul_sub(size_t n, int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* r) {
#if defined(__CUDACC__)
  const uint32_t* in[4] = {a, b, c, d};
  const size_t words[4] = {8, 8, 8, 8};
  return on_device(n, in, words, 4, r, 8, [&](const uint32_t** dv, uint32_t* o) {
    mul_sub_kernel<<<grid(n), 256>>>(n, op, dv[0], dv[1], dv[2], dv[3], o);
  });
#else
  for (size_t i = 0; i < n; i++) mul_sub_elem(i, op, a, b, c, d, r);
  return 0;
#endif
}

// out[i] = 2 jac[i] (op 0) or jac[i] + aff[i] (op 1) under FpK256Inline (lean = 1) or FpK256T<1> (lean = 0)
DEV_API int dev_k256l_point(size_t n, int op, int lean, const uint32_t* jac, const uint32_t* aff, uint32_t* out) {
#if defined(__CUDACC__)
  const uint32_t* in[2] = {jac, aff};
  const size_t words[2] = {24, 16};
  return on_device(n, in, words, 2, out, 24, [&](const uint32_t** dv, uint32_t* o) {
    if (lean)
      point_kernel<FpK256Inline><<<grid(n), 256>>>(n, op, dv[0], dv[1], o);
    else
      point_kernel<Plain><<<grid(n), 256>>>(n, op, dv[0], dv[1], o);
  });
#else
  for (size_t i = 0; i < n; i++) {
    if (lean)
      point_elem<FpK256Inline>(i, op, jac, aff, out);
    else
      point_elem<Plain>(i, op, jac, aff, out);
  }
  return 0;
#endif
}

}  // extern "C"
