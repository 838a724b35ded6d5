// tests/dev/ed448_h2c_dev.cu — the Ed448 hash-to-curve routines and kernels (ecg_ed448_h2c.cuh) exactly as the library
// compiles them, behind a small C ABI for the tests (test infrastructure only; never linked into libecgpu.so).
//
// nvcc builds libecged448h2cdev.so: the entries launch the production kernels (ed448h_h2c_kernel, ed448h_h2s_kernel and
// ed448g_norm_kernel<false>) with their launch bounds, and small kernels around the routines they are made of (the
// 84-byte reductions mod p and mod ell, the map with the isogeny, uniform bytes to the extended point).  The same file
// built by g++ is libecged448h2cdevsim.so: the identical per-element bodies in a host loop over the C emulation of the
// carry primitives, with the normalisation run slice by slice as the kernel's threads run it.
// Field values travel as raw little-endian 32-bit limbs (14 per element); extended points as the kernels' SoA form (word
// w of element i at w * n + i).
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../elliptic-curves_b200/csrc/ecg_ed448_h2c.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif

using namespace ecg;
typedef FpEd448 F;
typedef F::Fe FeE;

#define DEV_API __attribute__((visibility("default")))

static unsigned grid(size_t n) { return (unsigned)((n + ED448H_BLOCK - 1) / ED448H_BLOCK); }
// the normalisation kernel's geometry as ecgpu.cu launches it: one thread per ED448G_NORM_SLICE points
static size_t norm_threads(size_t n) { return (n + ED448G_NORM_SLICE - 1) / ED448G_NORM_SLICE; }
static unsigned norm_grid(size_t n) { return (unsigned)((norm_threads(n) + ED448G_BLOCK - 1) / ED448G_BLOCK); }

static XofSuffix make_suffix(const uint8_t* b, uint32_t len) {
  XofSuffix s;
  memset(&s, 0, sizeof s);
  memcpy(s.b, b, len);
  s.len = len;
  return s;
}

ECG_D void load84_elem(size_t i, const uint8_t* b84, uint32_t* out14) {
  FeE r;
  ed448h_load84<F>(r, b84 + 84 * i);
#pragma unroll
  for (int j = 0; j < 14; j++) out14[14 * i + j] = r.v[j];
}
ECG_D void modl84_elem(size_t i, const uint8_t* b84, uint8_t* out57) {
  uint32_t r[14];
  ed448h_mod_l_84(r, b84 + 84 * i);
  for (int j = 0; j < 56; j++) out57[57 * i + j] = (uint8_t)(r[j / 4] >> (8 * (j % 4)));
  out57[57 * i + 56] = 0;
}
// ext = ed448h_map of raw limbs u (14 words per element)
ECG_D void map_elem(size_t i, const uint32_t* u14, size_t n, uint32_t* ext) {
  FeE u;
#pragma unroll
  for (int j = 0; j < 14; j++) u.v[j] = u14[14 * i + j];
  EdPt<F> q;
  ed448h_map<F>(q, u);
  ed448_store_ext<F>(ext, n, i, q);
}
ECG_D void unif_elem(size_t i, const uint8_t* u, int len, size_t n, uint32_t* ext) {
  if (len == 84)
    ed448h_from_uniform<F, true>(ext, n, i, u + 84 * i);
  else
    ed448h_from_uniform<F, false>(ext, n, i, u + 168 * i);
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
#define BOUND __global__ void __launch_bounds__(ED448H_BLOCK, ED448H_H2C_MINBLK)
#define IDX                                                       \
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; \
  if (i >= n) return
BOUND load84_k(size_t n, const uint8_t* b, uint32_t* out) {
  IDX;
  load84_elem(i, b, out);
}
BOUND modl84_k(size_t n, const uint8_t* b, uint8_t* out) {
  IDX;
  modl84_elem(i, b, out);
}
BOUND map_k(size_t n, const uint32_t* u, uint32_t* ext) {
  IDX;
  map_elem(i, u, n, ext);
}
BOUND unif_k(size_t n, const uint8_t* u, int len, uint32_t* ext) {
  IDX;
  unif_elem(i, u, len, n, ext);
}
#define LAUNCH(k, ...) \
  if (B.err == cudaSuccess && n) k<<<grid(n), ED448H_BLOCK>>>(__VA_ARGS__)
#else
// the normalisation as ed448g_norm_kernel<F, false> runs it: threads t < n of a grid of norm_grid(n) blocks, stride T
static void host_norm(const uint32_t* ext, size_t n, uint8_t* out57) {
  std::vector<uint32_t> scr(14 * n + 1);
  const size_t T = (size_t)norm_grid(n) * ED448G_BLOCK;
  for (size_t t = 0; t < T && t < n; t++) ed448g_norm_slice<F, false>(t, T, ext, n, scr.data(), out57);
}
#endif

extern "C" {

DEV_API int dev_edh_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}
DEV_API const char* dev_edh_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}
// out14 = ed448h_load84 of n 84-byte strings (weakly reduced limbs)
DEV_API int dev_edh_load84(size_t n, const uint8_t* b84, uint32_t* out14) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(b84, n * 84);
  uint32_t* dout = B.out<uint32_t>(n * 14);
  LAUNCH(load84_k, n, di, dout);
  B.back(out14, dout, n * 14);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) load84_elem(i, b84, out14);
  return 0;
#endif
}
// out57 = ed448h_mod_l_84 of n 84-byte strings as 57-byte scalar records
DEV_API int dev_edh_mod_l_84(size_t n, const uint8_t* b84, uint8_t* out57) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(b84, n * 84);
  uint8_t* dout = B.out<uint8_t>(n * 57);
  LAUNCH(modl84_k, n, di, dout);
  B.back(out57, dout, n * 57);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) modl84_elem(i, b84, out57);
  return 0;
#endif
}
// ext = ed448h_map of raw limbs (14 words per element): the extended edwards448 point, SoA
DEV_API int dev_edh_map(size_t n, const uint32_t* u14, uint32_t* ext) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint32_t* du = B.in(u14, n * 14);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  LAUNCH(map_k, n, du, dx);
  B.back(ext, dx, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) map_elem(i, u14, n, ext);
  return 0;
#endif
}
// ext = ed448h_from_uniform of n strings of len = 84 (one map) or 168 bytes (two maps), then out57 = the compressed
// points through ed448g_norm_kernel<false> (ext is returned as the hash kernel stored it)
DEV_API int dev_edh_from_uniform(size_t n, const uint8_t* u, int len, uint32_t* ext, uint8_t* out57) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* du = B.in(u, n * (size_t)len);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  uint32_t* dscr = B.out<uint32_t>(n * 14);
  uint8_t* dout = B.out<uint8_t>(n * 57);
  LAUNCH(unif_k, n, du, len, dx);
  if (B.err == cudaSuccess && n) ed448g_norm_kernel<F, false><<<norm_grid(n), ED448G_BLOCK>>>(dx, n, dscr, dout);
  B.back(ext, dx, n * 56);
  B.back(out57, dout, n * 57);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) unif_elem(i, u, len, n, ext);
  if (n) host_norm(ext, n, out57);
  return 0;
#endif
}
// out57 = hash to curve (mode 0: RO, 1: NU) through ed448h_h2c_kernel and ed448g_norm_kernel<false>, or (mode 2) hash to
// scalar through ed448h_h2s_kernel, for the given expand_message_xof suffix (offsets from 0)
DEV_API int dev_edh_hash(size_t n, const uint8_t* msgs, const uint64_t* offs, const uint8_t* sfx, uint32_t slen, int mode, uint8_t* out57) {
  const XofSuffix s = make_suffix(sfx, slen);
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dm = B.in(msgs, (size_t)offs[n] + 1);
  const uint64_t* dofs = B.in(offs, n + 1);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  uint32_t* dscr = B.out<uint32_t>(n * 14);
  uint8_t* dout = B.out<uint8_t>(n * 57);
  if (B.err == cudaSuccess && n) {
    if (mode == 0)
      ed448h_h2c_kernel<F, false><<<grid(n), ED448H_BLOCK>>>(dm, dofs, 0, n, s, dx);
    else if (mode == 1)
      ed448h_h2c_kernel<F, true><<<grid(n), ED448H_BLOCK>>>(dm, dofs, 0, n, s, dx);
    else
      ed448h_h2s_kernel<<<grid(n), ED448H_BLOCK>>>(dm, dofs, 0, n, s, dout);
    if (mode != 2) ed448g_norm_kernel<F, false><<<norm_grid(n), ED448G_BLOCK>>>(dx, n, dscr, dout);
  }
  B.back(out57, dout, n * 57);
  return (int)B.err;
#else
  std::vector<uint32_t> ext(56 * n + 1);
  for (size_t i = 0; i < n; i++) {
    const uint8_t* m = msgs + offs[i];
    const size_t ml = (size_t)(offs[i + 1] - offs[i]);
    if (mode == 0)
      ed448h_h2c_one<F, false>(ext.data(), n, i, m, ml, s);
    else if (mode == 1)
      ed448h_h2c_one<F, true>(ext.data(), n, i, m, ml, s);
    else
      ed448h_h2s_one(out57 + 57 * i, m, ml, s);
  }
  if (mode != 2 && n) host_norm(ext.data(), n, out57);
  return 0;
#endif
}

}  // extern "C"
