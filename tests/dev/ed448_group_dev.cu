// tests/dev/ed448_group_dev.cu — the Ed448 group kernels (ecg_ed448_group.cuh) exactly as the library compiles them,
// behind a small C ABI for the tests (test infrastructure only; never linked into libecgpu.so).
//
// nvcc builds libecged448gdev.so: the entries launch the production kernels themselves (ed448g_mul_kernel,
// ed448g_fixed_kernel, ed448g_sum_kernel, ed448g_norm_kernel) with their launch bounds and the shipped field variant.
// The same file built by g++ is libecged448gdevsim.so: the identical per-element bodies in a host loop over the C
// emulation of the carry primitives.  Field values travel as raw little-endian 32-bit limbs (14 per element); extended
// points as the kernels' SoA form (word w of element i at w * n + i).
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../elliptic-curves_b200/csrc/ecg_ed448_group.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif

using namespace ecg;
typedef FpEd448 F;
typedef F::Fe FeE;

#define DEV_API __attribute__((visibility("default")))

static unsigned grid(size_t n) { return (unsigned)((n + ED448G_BLOCK - 1) / ED448G_BLOCK); }

ECG_D void sok_elem(size_t i, const uint8_t* k57, uint8_t* out) { out[i] = (uint8_t)ed448_scalar_ok(k57 + 57 * i); }
// flags: bit 0 = x exists (decompress_unchecked), bit 1 = accepted by the group decoder; xy = x, y
ECG_D void gdec_elem(size_t i, const uint8_t* b57, uint32_t* xy, uint8_t* flags) {
  FeE x, y;
  const uint32_t dec = ed448_decode<F>(x, y, b57 + 57 * i);
  FeE x2, y2;
  const uint32_t acc = ed448_group_decompress<F>(x2, y2, b57 + 57 * i);
  flags[i] = (uint8_t)(dec | (acc << 1));
#pragma unroll
  for (int j = 0; j < 14; j++) {
    xy[28 * i + j] = x.v[j];
    xy[28 * i + 14 + j] = y.v[j];
  }
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
#define BOUND __global__ void __launch_bounds__(ED448G_BLOCK, ED448G_MINBLK)
BOUND sok_k(size_t n, const uint8_t* in, uint8_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sok_elem(i, in, out);
}
BOUND gdec_k(size_t n, const uint8_t* in, uint32_t* xy, uint8_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) gdec_elem(i, in, xy, flags);
}
#define LAUNCH(k, ...) \
  if (B.err == cudaSuccess && n) k<<<grid(n), ED448G_BLOCK>>>(__VA_ARGS__)
#endif

extern "C" {

DEV_API int dev_ed448g_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}
DEV_API const char* dev_ed448g_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}
// geometry: block, variable-base and fixed-base min blocks, fixed-base digit width, windows, table words
DEV_API void dev_ed448g_geometry(int* g) {
  g[0] = ED448G_BLOCK;
  g[1] = ED448G_MINBLK;
  g[2] = ED448G_FB_MINBLK;
  g[3] = ED448_FBW;
  g[4] = ED448_FBND;
  g[5] = ED448_FB_WORDS;
}
DEV_API int dev_ed448g_scalar_ok(size_t n, const uint8_t* k57, uint8_t* out) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(k57, n * 57);
  uint8_t* dout = B.out<uint8_t>(n);
  LAUNCH(sok_k, n, di, dout);
  B.back(out, dout, n);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) sok_elem(i, k57, out);
  return 0;
#endif
}
DEV_API int dev_ed448g_decompress(size_t n, const uint8_t* b57, uint32_t* xy, uint8_t* flags) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(b57, n * 57);
  uint32_t* dxy = B.out<uint32_t>(n * 28);
  uint8_t* df = B.out<uint8_t>(n);
  LAUNCH(gdec_k, n, di, dxy, df);
  B.back(xy, dxy, n * 28);
  B.back(flags, df, n);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) gdec_elem(i, b57, xy, flags);
  return 0;
#endif
}
// ext (56 n words, SoA) = [k_i] P_i through ed448g_mul_kernel (p57 NULL: B); status = the kernel's two status words
// (error bits, smallest offending index), starting from {0, 0xFFFFFFFF}
DEV_API int dev_ed448g_mul(size_t n, const uint8_t* k57, const uint8_t* p57, int ct, uint32_t* ext, uint32_t* status) {
  const uint32_t st0[2] = {0u, 0xFFFFFFFFu};
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dk = B.in(k57, n * 57);
  const uint8_t* dp = B.in(p57, n * 57);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  uint32_t* ds = B.in(st0, 2);
  if (B.err == cudaSuccess && n) {
    if (ct)
      ed448g_mul_kernel<F, true><<<grid(n), ED448G_BLOCK>>>(dk, dp, n, 0, dx, ds, false);
    else
      ed448g_mul_kernel<F, false><<<grid(n), ED448G_BLOCK>>>(dk, dp, n, 0, dx, ds, true);
  }
  B.back(ext, dx, n * 56);
  B.back(status, ds, 2);
  return (int)B.err;
#else
  status[0] = st0[0];
  status[1] = st0[1];
  for (size_t i = 0; i < n; i++) {
    if (ct)
      ed448g_mul_elem<F, true>(i, k57, p57, n, 0, ext, status, false);
    else
      ed448g_mul_elem<F, false>(i, k57, p57, n, 0, ext, status, true);
  }
  return 0;
#endif
}
// ext = [k_i] B through ed448g_fixed_kernel over the given table (ED448_FB_WORDS words)
DEV_API int dev_ed448g_fixed(size_t n, const uint8_t* k57, const uint32_t* tab, uint32_t* ext, uint32_t* status) {
  const uint32_t st0[2] = {0u, 0xFFFFFFFFu};
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dk = B.in(k57, n * 57);
  const uint32_t* dt = B.in(tab, (size_t)ED448_FB_WORDS);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  uint32_t* ds = B.in(st0, 2);
  if (B.err == cudaSuccess && n) ed448g_fixed_kernel<F><<<grid(n), ED448G_BLOCK>>>(dk, n, 0, dt, dx, ds);
  B.back(ext, dx, n * 56);
  B.back(status, ds, 2);
  return (int)B.err;
#else
  status[0] = st0[0];
  status[1] = st0[1];
  for (size_t i = 0; i < n; i++) ed448g_fixed_elem<F>(i, k57, n, 0, tab, ext, status);
  return 0;
#endif
}
// out (56 n_out words, SoA) = partial sums of in (n_in points) through ed448g_sum_kernel
DEV_API int dev_ed448g_sum(size_t n_in, size_t n_out, const uint32_t* in, uint32_t* out) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint32_t* di = B.in(in, n_in * 56);
  uint32_t* dout = B.out<uint32_t>(n_out * 56);
  if (B.err == cudaSuccess && n_out) ed448g_sum_kernel<F><<<grid(n_out), ED448G_BLOCK>>>(di, n_in, dout, n_out, n_out);
  B.back(out, dout, n_out * 56);
  return (int)B.err;
#else
  for (size_t t = 0; t < n_out; t++) ed448g_sum_elem<F>(t, in, n_in, out, n_out, n_out);
  return 0;
#endif
}
// n points (SoA) -> out through ed448g_norm_kernel with `threads` threads (rounded up to whole blocks: slices of stride
// T = blocks * ED448G_BLOCK): table = 0: 57-byte records; table = 1: entries of 42 words
DEV_API int dev_ed448g_norm(int table, size_t n, size_t threads, const uint32_t* ext, void* out) {
  const size_t T = (size_t)grid(threads) * ED448G_BLOCK;
  const size_t obytes = table ? 168 : 57;
#if defined(__CUDACC__)
  DevBufs B;
  const uint32_t* di = B.in(ext, n * 56);
  uint32_t* scr = B.out<uint32_t>(n * 14);
  uint8_t* dout = B.out<uint8_t>(n * obytes);
  if (B.err == cudaSuccess && n) {
    if (table)
      ed448g_norm_kernel<F, true><<<grid(threads), ED448G_BLOCK>>>(di, n, scr, dout);
    else
      ed448g_norm_kernel<F, false><<<grid(threads), ED448G_BLOCK>>>(di, n, scr, dout);
  }
  B.back((uint8_t*)out, dout, n * obytes);
  return (int)B.err;
#else
  (void)obytes;
  std::vector<uint32_t> scr(n * 14 + 1);
  for (size_t t = 0; t < n && t < T; t++) {
    if (table)
      ed448g_norm_slice<F, true>(t, T, ext, n, scr.data(), out);
    else
      ed448g_norm_slice<F, false>(t, T, ext, n, scr.data(), out);
  }
  return 0;
#endif
}

}  // extern "C"
