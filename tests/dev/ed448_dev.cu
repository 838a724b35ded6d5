// tests/dev/ed448_dev.cu — the pieces of Ed448 verification (ecg_keccak.cuh, ecg_ed448.cuh) exactly as the library compiles
// them, behind a small C ABI for the tests (test infrastructure only; never linked into libecgpu.so).
//
// nvcc builds libecged448dev.so: every kernel here carries ed448_verify_kernel's production launch bound (ED448_BLOCK,
// ED448_MINBLK) and the shipped field variant (FpEd448), and the per-signature entry runs ed448_verify_kernel itself.
// The same file built by g++ is libecged448devsim.so: the identical bodies in a host loop over the C emulation of the
// carry primitives.  Field values travel as raw little-endian 32-bit limbs (14 per element).
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "../../elliptic-curves_b200/csrc/ecg_ed448.cuh"
#if defined(__CUDACC__)
#include <cuda_runtime.h>

#include <vector>
#endif

using namespace ecg;
typedef FpEd448 F;
typedef F::Fe FeE;

#define DEV_API __attribute__((visibility("default")))

ECG_D void ld14(uint32_t* v, const uint32_t* src, size_t i) {
#pragma unroll
  for (int j = 0; j < 14; j++) v[j] = src[i * 14 + j];
}
ECG_D void st14(uint32_t* dst, size_t i, const uint32_t* v) {
#pragma unroll
  for (int j = 0; j < 14; j++) dst[i * 14 + j] = v[j];
}

// element bodies, shared by the kernels and the host loops
ECG_D void shake_elem(size_t i, const uint8_t* data, const uint64_t* offs, uint8_t* out) {
  Shake256 sh;
  sh.init();
  sh.absorb(data + offs[i], (size_t)(offs[i + 1] - offs[i]));
  sh.finish<114>(out + 114 * i);
}
ECG_D void modl_elem(size_t i, const uint8_t* in, uint32_t* out) {
  uint32_t r[14];
  ed448_mod_l_wide(r, in + 114 * i);
  st14(out, i, r);
}
ECG_D void sok_elem(size_t i, const uint8_t* s57, uint8_t* out) { out[i] = (uint8_t)ed448_s_ok(s57 + 57 * i); }
// flags: bit 0 = x exists (decompress_unchecked), bit 1 = accepted (prime-order subgroup, not the identity); xy = x, y
ECG_D void dec_elem(size_t i, const uint8_t* b57, uint32_t* xy, uint8_t* flags) {
  FeE x, y;
  const uint32_t dec = ed448_decode<F>(x, y, b57 + 57 * i);
  const uint32_t acc = dec ? ed448_subgroup_not_identity<F>(y) : 0u;
  flags[i] = (uint8_t)(dec | (acc << 1));
  st14(xy, 2 * i, x.v);
  st14(xy, 2 * i + 1, y.v);
}
// op 0: r = 2 p (in: X, Y, Z, T); op 1: r = p + q (in: p and q as X, Y, Z, T); out: X, Y, Z, T
ECG_D void point_elem(int op, size_t i, const uint32_t* in, uint32_t* out) {
  EdPt<F> p, r;
  const size_t w = op == 0 ? 4 : 8;
  ld14(p.X.v, in, w * i);
  ld14(p.Y.v, in, w * i + 1);
  ld14(p.Z.v, in, w * i + 2);
  ld14(p.T.v, in, w * i + 3);
  if (op == 0) {
    ed_dbl<F>(r, p, true);
  } else {
    FeE qx, qy, qz, qt;
    ld14(qx.v, in, w * i + 4);
    ld14(qy.v, in, w * i + 5);
    ld14(qz.v, in, w * i + 6);
    ld14(qt.v, in, w * i + 7);
    ed_mul_d<F>(qt, qt);
    ed_add<F>(r, p, qx, qy, &qz, qt);
  }
  st14(out, 4 * i, r.X.v);
  st14(out, 4 * i + 1, r.Y.v);
  st14(out, 4 * i + 2, r.Z.v);
  st14(out, 4 * i + 3, r.T.v);
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
#define BOUND __global__ void __launch_bounds__(ED448_BLOCK, ED448_MINBLK)
BOUND shake_k(size_t n, const uint8_t* d, const uint64_t* o, uint8_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) shake_elem(i, d, o, out);
}
BOUND modl_k(size_t n, const uint8_t* in, uint32_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) modl_elem(i, in, out);
}
BOUND sok_k(size_t n, const uint8_t* in, uint8_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sok_elem(i, in, out);
}
BOUND dec_k(size_t n, const uint8_t* in, uint32_t* xy, uint8_t* flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dec_elem(i, in, xy, flags);
}
BOUND point_k(int op, size_t n, const uint32_t* in, uint32_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) point_elem(op, i, in, out);
}
static unsigned grid(size_t n) { return (unsigned)((n + ED448_BLOCK - 1) / ED448_BLOCK); }
#define LAUNCH(k, ...) \
  if (B.err == cudaSuccess && n) k<<<grid(n), ED448_BLOCK>>>(__VA_ARGS__)
#endif

static Ed448Dom make_dom(const uint8_t* dom, uint32_t len) {
  Ed448Dom d;
  memset(&d, 0, sizeof d);
  memcpy(d.b, dom, len);
  d.len = len;
  return d;
}

extern "C" {

DEV_API int dev_ed448_is_device(void) {
#if defined(__CUDACC__)
  return 1;
#else
  return 0;
#endif
}
DEV_API const char* dev_ed448_error_string(int err) {
#if defined(__CUDACC__)
  return cudaGetErrorString((cudaError_t)err);
#else
  return err ? "error" : "no error";
#endif
}
DEV_API void dev_ed448_bounds(int* block, int* minblk) {
  *block = ED448_BLOCK;
  *minblk = ED448_MINBLK;
}
// out[114 i ..] = SHAKE256(data[offs[i] .. offs[i + 1]), 114)
DEV_API int dev_ed448_shake(size_t n, const uint8_t* data, size_t total, const uint64_t* offs, uint8_t* out) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dd = B.in(data, total + 1);
  const uint64_t* dof = B.in(offs, n + 1);
  uint8_t* dout = B.out<uint8_t>(n * 114);
  LAUNCH(shake_k, n, dd, dof, dout);
  B.back(out, dout, n * 114);
  return (int)B.err;
#else
  (void)total;
  for (size_t i = 0; i < n; i++) shake_elem(i, data, offs, out);
  return 0;
#endif
}
// out (14 words each) = in (114 bytes each) mod ell
DEV_API int dev_ed448_mod_l(size_t n, const uint8_t* in, uint32_t* out) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(in, n * 114);
  uint32_t* dout = B.out<uint32_t>(n * 14);
  LAUNCH(modl_k, n, di, dout);
  B.back(out, dout, n * 14);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) modl_elem(i, in, out);
  return 0;
#endif
}
DEV_API int dev_ed448_s_ok(size_t n, const uint8_t* s57, uint8_t* out) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(s57, n * 57);
  uint8_t* dout = B.out<uint8_t>(n);
  LAUNCH(sok_k, n, di, dout);
  B.back(out, dout, n);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) sok_elem(i, s57, out);
  return 0;
#endif
}
DEV_API int dev_ed448_decompress(size_t n, const uint8_t* b57, uint32_t* xy, uint8_t* flags) {
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* di = B.in(b57, n * 57);
  uint32_t* dxy = B.out<uint32_t>(n * 28);
  uint8_t* df = B.out<uint8_t>(n);
  LAUNCH(dec_k, n, di, dxy, df);
  B.back(xy, dxy, n * 28);
  B.back(flags, df, n);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) dec_elem(i, b57, xy, flags);
  return 0;
#endif
}
DEV_API int dev_ed448_point(int op, size_t n, const uint32_t* in, uint32_t* out) {
  if (op < 0 || op > 1) return -1;
#if defined(__CUDACC__)
  DevBufs B;
  const uint32_t* di = B.in(in, n * 14 * (op == 0 ? 4 : 8));
  uint32_t* dout = B.out<uint32_t>(n * 56);
  LAUNCH(point_k, op, n, di, dout);
  B.back(out, dout, n * 56);
  return (int)B.err;
#else
  for (size_t i = 0; i < n; i++) point_elem(op, i, in, out);
  return 0;
#endif
}
// valid[i] = the whole per-signature routine, through ed448_verify_kernel (dom: the dom4 prefix of the call)
DEV_API int dev_ed448_verify(size_t n, const uint8_t* pk57, const uint8_t* sig114, const uint8_t* msgs, size_t total, const uint64_t* offs,
                             const uint8_t* dom, uint32_t dom_len, uint8_t* valid) {
  if (dom_len > 265) return -1;
  const Ed448Dom d = make_dom(dom, dom_len);
#if defined(__CUDACC__)
  DevBufs B;
  const uint8_t* dpk = B.in(pk57, n * 57);
  const uint8_t* dsig = B.in(sig114, n * 114);
  const uint8_t* dm = B.in(msgs, total + 1);
  const uint64_t* dof = B.in(offs, n + 1);
  uint8_t* dv = B.out<uint8_t>(n);
  if (B.err == cudaSuccess && n)
    ed448_verify_kernel<F, ED448_BLOCK, ED448_MINBLK><<<grid(n), ED448_BLOCK>>>(dpk, dsig, dm, dof, 0, n, d, dv);
  B.back(valid, dv, n);
  return (int)B.err;
#else
  (void)total;
  for (size_t i = 0; i < n; i++)
    valid[i] = ed448_verify_one<F>(pk57 + 57 * i, sig114 + 114 * i, msgs + offs[i], (size_t)(offs[i + 1] - offs[i]), d.b, d.len);
  return 0;
#endif
}

}  // extern "C"
