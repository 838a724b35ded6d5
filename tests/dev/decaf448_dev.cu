// tests/dev/decaf448_dev.cu — the Decaf448 routines and kernels (ecg_decaf448.cuh) exactly as the library compiles them,
// behind a small C ABI for the tests (test infrastructure only; never linked into libecgpu.so).
//
// nvcc builds libecgdecaf448dev.so: the entries launch the production kernels (decaf448_mul_kernel,
// decaf448_fixed_kernel, decaf448_encode_kernel, decaf448_check_kernel, decaf448_h2c_kernel, decaf448_h2s_kernel) with
// their launch bounds, and small kernels around the routines they are made of (expand_message_xof, the map, the scalar
// transform, the 64-byte reduction, ed448_mul_var on a given (x, y)).  The same file built by g++ is
// libecgdecaf448devsim.so: the identical per-element bodies in a host loop over the C emulation of the carry primitives.
// Field values travel as raw little-endian 32-bit limbs (14 per element); extended points as the kernels' SoA form (word
// w of element i at w * n + i).
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../elliptic-curves_b200/csrc/ecg_decaf448.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif

using namespace ecg;
typedef FpEd448 F;
typedef F::Fe FeE;

#define DEV_API __attribute__((visibility("default")))

static unsigned grid(size_t n) { return (unsigned)((n + DECAF448_BLOCK - 1) / DECAF448_BLOCK); }

static XofSuffix make_suffix(const uint8_t* b, uint32_t len) {
  XofSuffix s;
  memset(&s, 0, sizeof s);
  memcpy(s.b, b, len);
  s.len = len;
  return s;
}

// xy = (x, y) of decaf448_decode, ok = its verdict
ECG_D void dec_elem(size_t i, const uint8_t* b56, uint32_t* xy, uint8_t* ok) {
  FeE x, y;
  ok[i] = (uint8_t)decaf448_decode<F>(x, y, b56 + 56 * i);
#pragma unroll
  for (int j = 0; j < 14; j++) {
    xy[28 * i + j] = x.v[j];
    xy[28 * i + 14 + j] = y.v[j];
  }
}
// ext = [k_i] (x_i, y_i) through ed448_mul_var (default path) for raw (x, y) limbs
ECG_D void mulxy_elem(size_t i, const uint8_t* k56, const uint32_t* xy, size_t n, uint32_t* ext) {
  uint32_t k14[14];
  ed448_load56(k14, k56 + 56 * i);
  FeE x, y;
#pragma unroll
  for (int j = 0; j < 14; j++) {
    x.v[j] = xy[28 * i + j];
    y.v[j] = xy[28 * i + 14 + j];
  }
  EdPt<F> q;
  ed448_mul_var<F, false>(q, k14, x, y, false);
  ed448_store_ext<F>(ext, n, i, q);
}
ECG_D void gens_elem(size_t i, const uint8_t* k56, uint8_t* out56) {
  uint32_t k14[14], r[14];
  ed448_load56(k14, k56 + 56 * i);
  decaf448_gen_scalar(r, k14);
  for (int j = 0; j < 56; j++) out56[56 * i + j] = (uint8_t)(r[j / 4] >> (8 * (j % 4)));
}
ECG_D void modl_elem(size_t i, const uint8_t* h64, uint8_t* out56) {
  uint32_t r[14];
  decaf448_mod_l_64(r, h64 + 64 * i);
  for (int j = 0; j < 56; j++) out56[56 * i + j] = (uint8_t)(r[j / 4] >> (8 * (j % 4)));
}
// ext = map_to_curve_decaf448 of 56-byte u_i (twisted extended, SoA)
ECG_D void map_elem(size_t i, const uint8_t* u56, size_t n, uint32_t* ext) {
  FeE u;
  ed448_load56(u.v, u56 + 56 * i);
  EdPt<F> q;
  decaf448_tw_map<F>(q, u);
  ed448_store_ext<F>(ext, n, i, q);
}
// out = expand_message_xof(msg_i, DST, len) for len = 56, 64, 112 (the Decaf448 entries), 168 (the edwards448 RO suite's
// 2 x 84) or 280 (past two SHAKE256 blocks); out stride XOF_STRIDE
#define XOF_STRIDE 288
ECG_D void xof_elem(size_t i, const uint8_t* msgs, const uint64_t* offs, const XofSuffix& sfx, int len, uint8_t* out) {
  const uint8_t* m = msgs + offs[i];
  const size_t ml = (size_t)(offs[i + 1] - offs[i]);
  uint8_t* o = out + XOF_STRIDE * i;
  if (len == 56)
    expand_message_xof<56>(o, m, ml, sfx);
  else if (len == 64)
    expand_message_xof<64>(o, m, ml, sfx);
  else if (len == 112)
    expand_message_xof<112>(o, m, ml, sfx);
  else if (len == 168)
    expand_message_xof<168>(o, m, ml, sfx);
  else
    expand_message_xof<280>(o, m, ml, sfx);
}
// out56 = DecafPoint::from_uniform_bytes(u112).compress()
ECG_D void unif_elem(size_t i, const uint8_t* u112, uint8_t* out56) { decaf448_from_uniform<F, false>(out56 + 56 * i, u112 + 112 * i); }

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
#define BOUND __global__ void __launch_bounds__(DECAF448_BLOCK, DECAF448_MINBLK)
#define IDX                                                       \
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; \
  if (i >= n) return
BOUND dec_k(size_t n, const uint8_t* b, uint32_t* xy, uint8_t* ok) {
  IDX;
  dec_elem(i, b, xy, ok);
}
BOUND mulxy_k(size_t n, const uint8_t* k, const uint32_t* xy, uint32_t* ext) {
  IDX;
  mulxy_elem(i, k, xy, n, ext);
}
BOUND gens_k(size_t n, const uint8_t* k, uint8_t* out) {
  IDX;
  gens_elem(i, k, out);
}
BOUND modl_k(size_t n, const uint8_t* h, uint8_t* out) {
  IDX;
  modl_elem(i, h, out);
}
BOUND map_k(size_t n, const uint8_t* u, uint32_t* ext) {
  IDX;
  map_elem(i, u, n, ext);
}
BOUND unif_k(size_t n, const uint8_t* u, uint8_t* out) {
  IDX;
  unif_elem(i, u, out);
}
BOUND xof_k(size_t n, const uint8_t* msgs, const uint64_t* offs, XofSuffix sfx, int len, uint8_t* out) {
  IDX;
  xof_elem(i, msgs, offs, sfx, len, out);
}
#define LAUNCH(k, ...) \
  if (B.err == cudaSuccess && n) k<<<grid(n), DECAF448_BLOCK>>>(__VA_ARGS__)
#endif

extern "C" {

DEV_API int dev_decaf_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}
DEV_API const char* dev_decaf_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}
// the constants of the header as 14-word values: sqrt(-d), 1 / sqrt(-d), DECAF_FACTOR, G0 x, G0 y
DEV_API void dev_decaf_constants(uint32_t* out) {
  for (int i = 0; i < 14; i++) {
    out[i] = DECAF448_SQRT_MINUS_D[i];
    out[14 + i] = DECAF448_INV_SQRT_MINUS_D[i];
    out[28 + i] = DECAF448_FACTOR[i];
    out[42 + i] = DECAF448_G0[0][i];
    out[56 + i] = DECAF448_G0[1][i];
  }
}
DEV_API int dev_decaf_decode(size_t n, const uint8_t* b56, uint32_t* xy, uint8_t* ok) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(b56, n * 56);
  uint32_t* dxy = B.out<uint32_t>(n * 28);
  uint8_t* dok = B.out<uint8_t>(n);
  LAUNCH(dec_k, n, di, dxy, dok);
  B.back(xy, dxy, n * 28);
  B.back(ok, dok, n);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) dec_elem(i, b56, xy, ok);
  return 0;
#endif
}
// ok = the verdicts of decaf448_check_kernel
DEV_API int dev_decaf_check(size_t n, const uint8_t* b56, uint8_t* ok) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(b56, n * 56);
  uint8_t* dok = B.out<uint8_t>(n);
  LAUNCH(decaf448_check_kernel<F>, di, n, dok);
  B.back(ok, dok, n);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) decaf448_check_elem<F>(i, b56, ok);
  return 0;
#endif
}
// out56 = decaf448_encode of n untwisted extended points (SoA) through decaf448_encode_kernel
DEV_API int dev_decaf_encode(size_t n, const uint32_t* ext, uint8_t* out56) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint32_t* di = B.in(ext, n * 56);
  uint8_t* dout = B.out<uint8_t>(n * 56);
  LAUNCH(decaf448_encode_kernel<F>, di, n, dout);
  B.back(out56, dout, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) decaf448_encode_elem<F>(i, ext, n, out56);
  return 0;
#endif
}
// ext = [k_i] P_i through decaf448_mul_kernel (p56 NULL: G0); status = its two status words from {0, 0xFFFFFFFF}
DEV_API int dev_decaf_mul(size_t n, const uint8_t* k56, const uint8_t* p56, int ct, uint32_t* ext, uint32_t* status) {
  const uint32_t st0[2] = {0u, 0xFFFFFFFFu};
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dk = B.in(k56, n * 56);
  const uint8_t* dp = B.in(p56, n * 56);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  uint32_t* ds = B.in(st0, 2);
  if (B.err == cudaSuccess && n) {
    if (ct)
      decaf448_mul_kernel<F, true><<<grid(n), DECAF448_BLOCK>>>(dk, dp, n, 0, dx, ds, true);
    else
      decaf448_mul_kernel<F, false><<<grid(n), DECAF448_BLOCK>>>(dk, dp, n, 0, dx, ds, false);
  }
  B.back(ext, dx, n * 56);
  B.back(status, ds, 2);
  return (int)B.err;
#else
  status[0] = st0[0];
  status[1] = st0[1];
  for (size_t i = 0; i < n; i++) {
    if (ct)
      decaf448_mul_elem<F, true>(i, k56, p56, n, 0, ext, status, true);
    else
      decaf448_mul_elem<F, false>(i, k56, p56, n, 0, ext, status, false);
  }
  return 0;
#endif
}
// ext = [k_i] (x_i, y_i) through ed448_mul_var for raw limbs xy (28 words per element)
DEV_API int dev_decaf_mul_xy(size_t n, const uint8_t* k56, const uint32_t* xy, uint32_t* ext) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dk = B.in(k56, n * 56);
  const uint32_t* dxy = B.in(xy, n * 28);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  LAUNCH(mulxy_k, n, dk, dxy, dx);
  B.back(ext, dx, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) mulxy_elem(i, k56, xy, n, ext);
  return 0;
#endif
}
// ext = [(-2 k_i) mod ell] B through decaf448_fixed_kernel over the given Ed448 table (ED448_FB_WORDS words)
DEV_API int dev_decaf_fixed(size_t n, const uint8_t* k56, const uint32_t* tab, uint32_t* ext, uint32_t* status) {
  const uint32_t st0[2] = {0u, 0xFFFFFFFFu};
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dk = B.in(k56, n * 56);
  const uint32_t* dt = B.in(tab, (size_t)ED448_FB_WORDS);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  uint32_t* ds = B.in(st0, 2);
  if (B.err == cudaSuccess && n) decaf448_fixed_kernel<F><<<grid(n), DECAF448_BLOCK>>>(dk, n, 0, dt, dx, ds);
  B.back(ext, dx, n * 56);
  B.back(status, ds, 2);
  return (int)B.err;
#else
  status[0] = st0[0];
  status[1] = st0[1];
  for (size_t i = 0; i < n; i++) decaf448_fixed_elem<F>(i, k56, n, 0, tab, ext, status);
  return 0;
#endif
}
DEV_API int dev_decaf_gen_scalar(size_t n, const uint8_t* k56, uint8_t* out56) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dk = B.in(k56, n * 56);
  uint8_t* dout = B.out<uint8_t>(n * 56);
  LAUNCH(gens_k, n, dk, dout);
  B.back(out56, dout, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) gens_elem(i, k56, out56);
  return 0;
#endif
}
DEV_API int dev_decaf_mod_l_64(size_t n, const uint8_t* h64, uint8_t* out56) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dh = B.in(h64, n * 64);
  uint8_t* dout = B.out<uint8_t>(n * 56);
  LAUNCH(modl_k, n, dh, dout);
  B.back(out56, dout, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) modl_elem(i, h64, out56);
  return 0;
#endif
}
DEV_API int dev_decaf_map(size_t n, const uint8_t* u56, uint32_t* ext) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* du = B.in(u56, n * 56);
  uint32_t* dx = B.out<uint32_t>(n * 56);
  LAUNCH(map_k, n, du, dx);
  B.back(ext, dx, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) map_elem(i, u56, n, ext);
  return 0;
#endif
}
// out (stride XOF_STRIDE) = expand_message_xof(msgs_i, ., len) for the given suffix (offsets from 0)
DEV_API int dev_decaf_xof(size_t n, const uint8_t* msgs, const uint64_t* offs, const uint8_t* sfx, uint32_t slen, int len, uint8_t* out) {
  const XofSuffix s = make_suffix(sfx, slen);
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dm = B.in(msgs, (size_t)offs[n] + 1);
  const uint64_t* dofs = B.in(offs, n + 1);
  uint8_t* dout = B.out<uint8_t>(n * XOF_STRIDE);
  LAUNCH(xof_k, n, dm, dofs, s, len, dout);
  B.back(out, dout, n * XOF_STRIDE);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) xof_elem(i, msgs, offs, s, len, out);
  return 0;
#endif
}
// out56 = from_uniform_bytes of n 112-byte strings (the RO path after expansion: two maps, one addition, compress)
DEV_API int dev_decaf_from_uniform(size_t n, const uint8_t* u112, uint8_t* out56) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* du = B.in(u112, n * 112);
  uint8_t* dout = B.out<uint8_t>(n * 56);
  LAUNCH(unif_k, n, du, dout);
  B.back(out56, dout, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) unif_elem(i, u112, out56);
  return 0;
#endif
}
// out56 = hash to group (nu = 0: RO, 1: NU) or, mode 2, hash to scalar through decaf448_h2c_kernel / decaf448_h2s_kernel
DEV_API int dev_decaf_hash(size_t n, const uint8_t* msgs, const uint64_t* offs, const uint8_t* sfx, uint32_t slen, int mode, uint8_t* out56) {
  const XofSuffix s = make_suffix(sfx, slen);
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dm = B.in(msgs, (size_t)offs[n] + 1);
  const uint64_t* dofs = B.in(offs, n + 1);
  uint8_t* dout = B.out<uint8_t>(n * 56);
  if (B.err == cudaSuccess && n) {
    if (mode == 0)
      decaf448_h2c_kernel<F, false><<<grid(n), DECAF448_BLOCK>>>(dm, dofs, 0, n, s, dout);
    else if (mode == 1)
      decaf448_h2c_kernel<F, true><<<grid(n), DECAF448_BLOCK>>>(dm, dofs, 0, n, s, dout);
    else
      decaf448_h2s_kernel<<<grid(n), DECAF448_BLOCK>>>(dm, dofs, 0, n, s, dout);
  }
  B.back(out56, dout, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) {
    const uint8_t* m = msgs + offs[i];
    const size_t ml = (size_t)(offs[i + 1] - offs[i]);
    if (mode == 0)
      decaf448_h2c_one<F, false>(out56 + 56 * i, m, ml, s);
    else if (mode == 1)
      decaf448_h2c_one<F, true>(out56 + 56 * i, m, ml, s);
    else
      decaf448_h2s_one(out56 + 56 * i, m, ml, s);
  }
  return 0;
#endif
}

}  // extern "C"
