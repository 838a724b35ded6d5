// tools/kbench.cu — development harness: times kernel variants of the secp256k1 variable-base path on one GPU
// and cross-checks that every variant produces identical Jacobian words.  Not part of the product or of bench.py.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o tools/kbench tools/kbench.cu
//   modes: kbench 20 | kbench 20 lean | kbench 20 trade | kbench 20 shape | kbench 20 mem   (mem: also build with -DECG_FE_ALIGN=16 as tools/kbench_a16)
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <cstring>
#define ECG_K256_OPT 7
#include "../elliptic-curves_b200/csrc/ecg_curves.cuh"
#include "../elliptic-curves_b200/csrc/ecg_io.cuh"
#include "../elliptic-curves_b200/csrc/ecg_mul.cuh"
using namespace ecg;

static uint64_t checksum(const std::vector<uint32_t>& v);
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ void make_inputs(uint32_t* k, Aff& P, size_t idx) {
  // deterministic pseudo-random scalar < 2^255 ; P = G
  uint32_t s = (uint32_t)idx * 2654435761u + 12345u;
  for (int i = 0; i < 8; i++) { s = s * 1664525u + 1013904223u; k[i] = s ^ (s >> 15); }
  k[7] &= 0x7FFFFFFFu;
  CurveK256::generator(P);
}

template <class F, int BLOCK, int MINBLK, bool GLOBAL_TAB>
__global__ void __launch_bounds__(BLOCK, MINBLK) kb_varbase(size_t n, uint32_t* __restrict__ jac, uint32_t* __restrict__ gtab) {
  extern __shared__ uint32_t smem[];
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[8];
  Aff P;
  make_inputs(k, P, idx);
  Jac r;
  if (GLOBAL_TAB) {
    // per-resident-thread table slot in global memory (L2-resident): [entry*16+word][thread] layout per block slot
    size_t slot = ((size_t)blockIdx.x % (132 * 8)) * BLOCK;  // NOTE: timing experiment only (slots may alias across waves)
    TabRef tab{gtab + slot * 128 + threadIdx.x, (uint32_t)BLOCK};
    k256_mul_thread<F>(r, k, P, tab);
  } else {
    TabRef tab{smem + threadIdx.x, (uint32_t)BLOCK};
    k256_mul_thread<F>(r, k, P, tab);
  }
  for (int w = 0; w < 8; w++) {
    jac[(size_t)w * n + idx] = r.X.v[w];
    jac[(size_t)(8 + w) * n + idx] = r.Y.v[w];
    jac[(size_t)(16 + w) * n + idx] = r.Z.v[w];
  }
}

// phase-synchronised variant: every thread of the block stays alive (clamped index) so the barriers are legal
template <class F, int BLOCK, int MINBLK, int LEVEL = 1>
__global__ void __launch_bounds__(BLOCK, MINBLK) kb_varbase_sync(size_t n, uint32_t* __restrict__ jac, uint32_t* __restrict__ gtab) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  size_t cidx = idx < n ? idx : n - 1;
  uint32_t k[8];
  Aff P;
  make_inputs(k, P, cidx);
  Jac r;
  size_t slot = ((size_t)blockIdx.x % (132 * 8)) * BLOCK;
  K256TabRef<F> tab{gtab + slot * (F::BETA_COLUMN ? 192 : 128) + threadIdx.x, (uint32_t)BLOCK};
  k256_mul_thread<F, LEVEL>(r, k, P, tab);
  if (idx >= n) return;
  for (int w = 0; w < 8; w++) {
    jac[(size_t)w * n + idx] = r.X.v[w];
    jac[(size_t)(8 + w) * n + idx] = r.Y.v[w];
    jac[(size_t)(16 + w) * n + idx] = r.Z.v[w];
  }
}
template <class F, int BLOCK, int MINBLK, int LEVEL = 1>
static void run_sync(const char* name, size_t n, uint32_t* jac, uint32_t* gtab) {
  auto kern = kb_varbase_sync<F, BLOCK, MINBLK, LEVEL>;
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, BLOCK, 0));
  unsigned grid = (unsigned)((n + BLOCK - 1) / BLOCK);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 4; rep++) {
    CK(cudaEventRecord(e0));
    kern<<<grid, BLOCK>>>(n, jac, gtab);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  std::vector<uint32_t> h(24 * 4096);
  for (int w = 0; w < 24; w++) CK(cudaMemcpy(&h[w * 4096], jac + (size_t)w * n, 4096 * 4, cudaMemcpyDeviceToHost));
  printf("%-34s regs %3d  blocks/SM %d  warps/SM %2d  %8.3f ms  %.4g mults/s  chk %016llx\n", name, fa.numRegs, occ, occ * BLOCK / 32, best,
         n / (best * 1e-3), (unsigned long long)checksum(h));
}

template <class F, int BLOCK, int MINBLK, bool GLOBAL_TAB>
__global__ void __launch_bounds__(BLOCK, MINBLK) kb_generic(size_t n, uint32_t* __restrict__ jac, uint32_t* __restrict__ gtab) {
  extern __shared__ uint32_t smem[];
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (idx >= n) return;
  uint32_t k[8];
  Aff P;
  make_inputs(k, P, idx);
  CurveP256T<F>::generator(P);
  Jac r;
  if (GLOBAL_TAB) {
    size_t slot = ((size_t)blockIdx.x % (132 * 8)) * BLOCK;
    TabRefJ tab{gtab + slot * 192 + threadIdx.x, (uint32_t)BLOCK};
    generic_mul_thread<F, true>(r, k, P, tab);
  } else {
    TabRefJ tab{smem + threadIdx.x, (uint32_t)BLOCK};
    generic_mul_thread<F, true>(r, k, P, tab);
  }
  for (int w = 0; w < 8; w++) {
    jac[(size_t)w * n + idx] = r.X.v[w];
    jac[(size_t)(8 + w) * n + idx] = r.Y.v[w];
    jac[(size_t)(16 + w) * n + idx] = r.Z.v[w];
  }
}

template <class F>
__global__ void __launch_bounds__(256) kb_fmul(uint32_t* out, int iters, uint32_t seed, int mode) {
  Fe a, b;
  for (int i = 0; i < 8; i++) { a.v[i] = seed * (i + 1) + threadIdx.x; b.v[i] = (seed ^ 0x9E3779B9u) * (i + 3) + blockIdx.x; }
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
    if (mode == 0) { F::mul(a, a, b); F::mul(b, b, a); }
    else { F::sqr(a, a); F::sqr(b, b); }
  }
  uint32_t s = 0;
  for (int i = 0; i < 8; i++) s ^= a.v[i] ^ b.v[i];
  if (s == 0x12345678u) out[0] = s;
}

__global__ void __launch_bounds__(256) kb_dfma(double* out, int iters, double seed) {
  double a = seed + threadIdx.x, b = 1.0000001, c = 0.5;
  double r[8];
  for (int i = 0; i < 8; i++) r[i] = a + i;
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int u = 0; u < 8; u++) {
#pragma unroll
      for (int i = 0; i < 8; i++) r[i] = __fma_rz(r[i], b, c);
    }
  }
  double s = 0;
  for (int i = 0; i < 8; i++) s += r[i];
  if (s == 12345.678) out[0] = s;
}
// DFMA and IMAD.WIDE issued from the same warps: do the FP64 and FMA-heavy pipes overlap?
__global__ void __launch_bounds__(256) kb_mix(double* out, int iters, double seed, uint32_t iseed) {
  double b = 1.0000001, c = 0.5;
  double r[8];
  for (int i = 0; i < 8; i++) r[i] = seed + threadIdx.x + i;
  uint32_t a0 = iseed + threadIdx.x, a1 = a0 * 3 + 1, b0 = iseed ^ 0x9E3779B9u, b1 = b0 + blockIdx.x;
  uint32_t q[16];
  for (int i = 0; i < 16; i++) q[i] = a0 + i;
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      mad_wide_cc(q[0], q[1], a0, b0);
      r[0] = __fma_rz(r[0], b, c); r[1] = __fma_rz(r[1], b, c);
      madc_wide_cc(q[2], q[3], a1, b0);
      r[2] = __fma_rz(r[2], b, c); r[3] = __fma_rz(r[3], b, c);
      madc_wide_cc(q[4], q[5], a0, b1);
      r[4] = __fma_rz(r[4], b, c); r[5] = __fma_rz(r[5], b, c);
      madc_wide_cc(q[6], q[7], a1, b1);
      r[6] = __fma_rz(r[6], b, c); r[7] = __fma_rz(r[7], b, c);
      mad_wide_cc(q[8], q[9], a1, b0);
      r[0] = __fma_rz(r[0], b, c); r[1] = __fma_rz(r[1], b, c);
      madc_wide_cc(q[10], q[11], a0, b1);
      r[2] = __fma_rz(r[2], b, c); r[3] = __fma_rz(r[3], b, c);
      madc_wide_cc(q[12], q[13], a1, b1);
      r[4] = __fma_rz(r[4], b, c); r[5] = __fma_rz(r[5], b, c);
      madc_wide_cc(q[14], q[15], a0, b0);
      r[6] = __fma_rz(r[6], b, c); r[7] = __fma_rz(r[7], b, c);
    }
  }
  double s = 0;
  uint32_t x = 0;
  for (int i = 0; i < 8; i++) s += r[i];
  for (int i = 0; i < 16; i++) x ^= q[i];
  if (s == 12345.678 && x == 77) out[0] = s;
}

// P-256 with a barrier before every point operation (all threads stay alive: clamped index)
template <class F, int BLOCK, int MINBLK, int LEVEL>
__global__ void __launch_bounds__(BLOCK, MINBLK) kb_generic_sync(size_t n, uint32_t* __restrict__ jac, uint32_t* __restrict__ gtab) {
  size_t idx = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  size_t cidx = idx < n ? idx : n - 1;
  uint32_t k[8];
  Aff P;
  make_inputs(k, P, cidx);
  CurveP256T<F>::generator(P);
  Jac r;
  size_t slot = ((size_t)blockIdx.x % (132 * 8)) * BLOCK;
  TabRefJ tab{gtab + slot * 192 + threadIdx.x, (uint32_t)BLOCK};
  generic_mul_thread<F, true, LEVEL>(r, k, P, tab);
  if (idx >= n) return;
  for (int w = 0; w < 8; w++) {
    jac[(size_t)w * n + idx] = r.X.v[w];
    jac[(size_t)(8 + w) * n + idx] = r.Y.v[w];
    jac[(size_t)(16 + w) * n + idx] = r.Z.v[w];
  }
}
template <class F, int BLOCK, int MINBLK, int LEVEL>
static void runp_sync(const char* name, size_t n, uint32_t* jac, uint32_t* gtab) {
  auto kern = kb_generic_sync<F, BLOCK, MINBLK, LEVEL>;
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, BLOCK, 0));
  unsigned grid = (unsigned)((n + BLOCK - 1) / BLOCK);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 3; rep++) {
    CK(cudaEventRecord(e0));
    kern<<<grid, BLOCK>>>(n, jac, gtab);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  std::vector<uint32_t> h(24 * 4096);
  for (int w = 0; w < 24; w++) CK(cudaMemcpy(&h[w * 4096], jac + (size_t)w * n, 4096 * 4, cudaMemcpyDeviceToHost));
  printf("%-34s regs %3d  blocks/SM %d  warps/SM %2d  %8.3f ms  %.4g mults/s  chk %016llx\n", name, fa.numRegs, occ, occ * BLOCK / 32, best,
         n / (best * 1e-3), (unsigned long long)checksum(h));
}

// Ceiling of a double-precision multiplier (52-bit limbs, Emmart-style split): the 25 limb products of a 5x5 schoolbook,
// each as hi = fma_rz(a, b, 2^104), lo = fma_rz(a, b, (2^104 + 2^52) - hi), both halves accumulated into 64-bit integer
// column sums.  No carry resolution, no reduction, no int<->double conversion: if THIS is not well above the integer
// multiplier's 1.1e11 field-mul/s there is nothing to build on.
__global__ void __launch_bounds__(256) kb_dfma_product(unsigned long long* out, int iters, double seed) {
  double a[5], b[5];
  for (int i = 0; i < 5; i++) { a[i] = (double)((threadIdx.x * 7919u + i * 104729u) & 0xFFFFFu) + seed; b[i] = (double)((blockIdx.x * 31u + i * 1299709u) & 0xFFFFFu) + 3.0; }
  const double C1 = 20282409603651670423947251286016.0;       // 2^104
  const double C2 = 20282409603651674927546878656512.0;       // 2^104 + 2^52
  long long col[10];
  for (int i = 0; i < 10; i++) col[i] = 0;
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 5; i++) {
#pragma unroll
      for (int j = 0; j < 5; j++) {
        double hi = __fma_rz(a[i], b[j], C1);
        double lo = __fma_rz(a[i], b[j], C2 - hi);
        col[i + j + 1] += __double_as_longlong(hi);
        col[i + j] += __double_as_longlong(lo);
      }
    }
    // feed something back so that iterations depend on each other without touching the FP64 pipe much
    a[0] = __longlong_as_double((col[3] & 0xFFFFFFFFFll) | 0x4330000000000000ll) - 4503599627370496.0;
  }
  long long s = 0;
  for (int i = 0; i < 10; i++) s ^= col[i];
  if (s == 0x1234567) out[0] = (unsigned long long)s;
}

static uint64_t checksum(const std::vector<uint32_t>& v) {
  uint64_t h = 1469598103934665603ull;
  for (uint32_t x : v) { h ^= x; h *= 1099511628211ull; }
  return h;
}

template <class F, int BLOCK, int MINBLK, bool GLOBAL_TAB>
static void run(const char* name, size_t n, uint32_t* jac, uint32_t* gtab) {
  size_t smem = GLOBAL_TAB ? 0 : (size_t)BLOCK * 128 * 4;
  auto kern = kb_varbase<F, BLOCK, MINBLK, GLOBAL_TAB>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, BLOCK, smem));
  unsigned grid = (unsigned)((n + BLOCK - 1) / BLOCK);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 4; rep++) {
    CK(cudaEventRecord(e0));
    kern<<<grid, BLOCK, smem>>>(n, jac, gtab);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  std::vector<uint32_t> h(24 * 4096);
  // sample: first 4096 elements of each word row
  for (int w = 0; w < 24; w++) CK(cudaMemcpy(&h[w * 4096], jac + (size_t)w * n, 4096 * 4, cudaMemcpyDeviceToHost));
  printf("%-34s regs %3d  blocks/SM %d  warps/SM %2d  %8.3f ms  %.4g mults/s  chk %016llx\n", name, fa.numRegs, occ, occ * BLOCK / 32, best,
         n / (best * 1e-3), (unsigned long long)checksum(h));
}

template <class F, int BLOCK, int MINBLK, bool GLOBAL_TAB>
static void runp(const char* name, size_t n, uint32_t* jac, uint32_t* gtab) {
  size_t smem = GLOBAL_TAB ? 0 : (size_t)BLOCK * 192 * 4;
  auto kern = kb_generic<F, BLOCK, MINBLK, GLOBAL_TAB>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, BLOCK, smem));
  unsigned grid = (unsigned)((n + BLOCK - 1) / BLOCK);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 3; rep++) {
    CK(cudaEventRecord(e0));
    kern<<<grid, BLOCK, smem>>>(n, jac, gtab);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  std::vector<uint32_t> h(24 * 4096);
  for (int w = 0; w < 24; w++) CK(cudaMemcpy(&h[w * 4096], jac + (size_t)w * n, 4096 * 4, cudaMemcpyDeviceToHost));
  printf("%-34s regs %3d  blocks/SM %d  warps/SM %2d  %8.3f ms  %.4g mults/s  chk %016llx\n", name, fa.numRegs, occ, occ * BLOCK / 32, best,
         n / (best * 1e-3), (unsigned long long)checksum(h));
}

template <class F>
static void run_fmul(const char* name) {
  uint32_t* out; CK(cudaMalloc(&out, 256));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int mode = 0; mode < 2; mode++) {
    float best = 1e30f; int iters = 4000; unsigned blocks = 132 * 8;
    for (int rep = 0; rep < 3; rep++) {
      CK(cudaEventRecord(e0));
      kb_fmul<F><<<blocks, 256>>>(out, iters, 777u + rep, mode);
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rep > 0 && ms < best) best = ms;
    }
    printf("%-34s %s: %.4g field-ops/s\n", name, mode ? "sqr" : "mul", (double)blocks * 256 * iters * 2 / (best * 1e-3));
  }
}


// ---- "shape" mode: one measured line for each kernel-shape clause of north_star that the product does not follow ----
// (a) 4 x u64 limbs with mul.lo.u64 / mul.hi.u64 (+ 64-bit carry chains): the 256 x 256 -> 512-bit product only, no reduction
__device__ __forceinline__ void mac3_u64(unsigned long long& c0, unsigned long long& c1, unsigned long long& c2, unsigned long long a,
                                         unsigned long long b) {
  asm volatile("{\n\t.reg .u64 lo, hi;\n\tmul.lo.u64 lo, %3, %4;\n\tmul.hi.u64 hi, %3, %4;\n\tadd.cc.u64 %0, %0, lo;\n\taddc.cc.u64 %1, %1, hi;\n\taddc.u64 %2, %2, 0;\n\t}"
               : "+&l"(c0), "+&l"(c1), "+&l"(c2)
               : "l"(a), "l"(b));
}
__global__ void __launch_bounds__(256) kb_prod_u64(unsigned long long* out, int iters, unsigned long long seed) {
  unsigned long long a[4], b[4], r[8];
  for (int i = 0; i < 4; i++) { a[i] = seed * (2 * i + 1) + threadIdx.x; b[i] = (seed ^ 0x9E3779B97F4A7C15ull) * (2 * i + 3) + blockIdx.x; }
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
    unsigned long long c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int j = k - i;
        if (j >= 0 && j < 4) mac3_u64(c0, c1, c2, a[i], b[j]);
      }
      r[k] = c0; c0 = c1; c1 = c2; c2 = 0;
    }
    r[7] = c0;
    for (int i = 0; i < 4; i++) { a[i] = r[i] ^ r[i + 4]; b[i] += r[7 - i]; }  // keep the chain alive, no modular meaning
  }
  unsigned long long x = 0;
  for (int i = 0; i < 4; i++) x ^= a[i] ^ b[i];
  if (x == 0x1234567812345678ull) out[0] = x;
}
// the same product on 8 x u32 limbs (the product's mul8x8), also without reduction, for the like-for-like comparison
__global__ void __launch_bounds__(256) kb_prod_u32(uint32_t* out, int iters, uint32_t seed) {
  uint32_t a[8], b[8], r[16];
  for (int i = 0; i < 8; i++) { a[i] = seed * (i + 1) + threadIdx.x; b[i] = (seed ^ 0x9E3779B9u) * (i + 3) + blockIdx.x; }
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
    mul8x8(r, a, b);
    for (int i = 0; i < 8; i++) { a[i] = r[i] ^ r[i + 8]; b[i] += r[15 - i]; }
  }
  uint32_t x = 0;
  for (int i = 0; i < 8; i++) x ^= a[i] ^ b[i];
  if (x == 0x12345678u) out[0] = x;
}
// (b) warp-cooperative layout, 8 lanes per field element (4 elements per warp), lane l holds limb l of a and of b.
// Product core only: lane l accumulates column l (products a_i b_(l-i), i <= l) and column l + 8 (a_i b_(l+8-i), i > l):
// 8 products per lane = the same 64 products per element, operands fetched with two shuffles per product; NO carry
// resolution across lanes, no reduction (both would add further shuffle rounds).
__global__ void __launch_bounds__(256) kb_prod_warp8(uint32_t* out, int iters, uint32_t seed) {
  const unsigned lane = threadIdx.x & 31u, l = lane & 7u, base = lane & ~7u;
  uint32_t a = seed * (l + 1) + threadIdx.x, b = (seed ^ 0x9E3779B9u) * (l + 3) + blockIdx.x;
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
    uint32_t s0 = 0, s1 = 0, s2 = 0, t0 = 0, t1 = 0, t2 = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint32_t ai = __shfl_sync(0xFFFFFFFFu, a, base + i);
      uint32_t bj = __shfl_sync(0xFFFFFFFFu, b, base + ((l - i) & 7u));  // b_(l-i) for i <= l, b_(l+8-i) for i > l
      if ((unsigned)i <= l)
        mad_acc3(s0, s1, s2, ai, bj);
      else
        mad_acc3(t0, t1, t2, ai, bj);
    }
    a = s0 ^ t1 ^ s2;
    b += s1 ^ t0 ^ t2;
  }
  if ((a ^ b) == 0x12345678u) out[0] = a;
}
// (c) record loads: 96 bytes per pair (32 k + 64 P) as 24 x 32-bit loads (the product's load_be) vs 6 x 128-bit loads
template <bool VEC>
__global__ void __launch_bounds__(256) kb_record_loads(const uint8_t* __restrict__ kb, const uint8_t* __restrict__ pxy, size_t n, uint32_t* out) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  uint32_t w[24];
  if (VEC) {
    const uint4* k4 = reinterpret_cast<const uint4*>(kb + 32 * idx);
    const uint4* p4 = reinterpret_cast<const uint4*>(pxy + 64 * idx);
#pragma unroll
    for (int q = 0; q < 2; q++) { uint4 v = __ldg(k4 + q); w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w; }
#pragma unroll
    for (int q = 0; q < 4; q++) { uint4 v = __ldg(p4 + q); w[8 + 4 * q] = v.x; w[9 + 4 * q] = v.y; w[10 + 4 * q] = v.z; w[11 + 4 * q] = v.w; }
  } else {
    const uint32_t* k1 = reinterpret_cast<const uint32_t*>(kb + 32 * idx);
    const uint32_t* p1 = reinterpret_cast<const uint32_t*>(pxy + 64 * idx);
#pragma unroll
    for (int q = 0; q < 8; q++) w[q] = __ldg(k1 + q);
#pragma unroll
    for (int q = 0; q < 16; q++) w[8 + q] = __ldg(p1 + q);
  }
  uint32_t x = 0;
#pragma unroll
  for (int q = 0; q < 24; q++) x ^= bswap32(w[q]) + q;
  if (x == 0x12345678u) out[0] = x;
}
template <class K, class... A>
static float time_best(int reps, K launch, A... args) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < reps; rep++) {
    CK(cudaEventRecord(e0));
    launch(args...);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  return best;
}
static void run_shape(size_t n) {
  void* out; CK(cudaMalloc(&out, 256));
  const int iters = 4000; const unsigned blocks = 132 * 8;
  const double units = (double)blocks * 256 * iters;
  float t32 = time_best(4, [&] { kb_prod_u32<<<blocks, 256>>>((uint32_t*)out, iters, 777u); });
  float t64 = time_best(4, [&] { kb_prod_u64<<<blocks, 256>>>((unsigned long long*)out, iters, 777ull); });
  float tw = time_best(4, [&] { kb_prod_warp8<<<blocks, 256>>>((uint32_t*)out, iters, 777u); });
  printf("256x256 product, 8 x u32 limbs, one thread per element (mul8x8, no reduction): %.4g products/s (%.3f ms)\n", units / (t32 * 1e-3), t32);
  printf("256x256 product, 4 x u64 limbs, mul.lo/hi.u64 + 64-bit carry chains (no reduction): %.4g products/s (%.3f ms)  = %.2fx the u32 time\n",
         units / (t64 * 1e-3), t64, t64 / t32);
  printf("256x256 product, warp-cooperative 8 lanes per element (product core only: no carry resolution, no reduction): %.4g products/s (%.3f ms)  = %.2fx the u32 time\n",
         units / 8 / (tw * 1e-3), tw, (tw * 8) / t32);
  uint8_t *kb, *pxy;
  CK(cudaMalloc(&kb, n * 32)); CK(cudaMalloc(&pxy, n * 64));
  CK(cudaMemset(kb, 0x5A, n * 32)); CK(cudaMemset(pxy, 0xA5, n * 64));
  unsigned g = (unsigned)((n + 255) / 256);
  float l32 = time_best(6, [&] { kb_record_loads<false><<<g, 256>>>(kb, pxy, n, (uint32_t*)out); });
  float l128 = time_best(6, [&] { kb_record_loads<true><<<g, 256>>>(kb, pxy, n, (uint32_t*)out); });
  printf("record loads, %zu pairs x 96 B: 24 x LDG.32 per pair %.1f us (%.0f GB/s), 6 x LDG.128 per pair %.1f us (%.0f GB/s); the var-base kernel over the same pairs takes ~17300 us\n",
         n, l32 * 1e3, n * 96.0 / (l32 * 1e-3) / 1e9, l128 * 1e3, n * 96.0 / (l128 * 1e-3) / 1e9);
  cudaFree(kb); cudaFree(pxy); cudaFree(out);
}

int main(int argc, char** argv) {
  size_t n = (size_t)1 << (argc > 1 ? atoi(argv[1]) : 20);
  uint32_t *jac, *gtab;
  CK(cudaMalloc(&jac, n * 96));
  CK(cudaMalloc(&gtab, (size_t)132 * 8 * 640 * 192 * 4));
  printf("n = %zu\n", n);
  if (argc > 2 && !strcmp(argv[2], "shape")) {  // north_star's kernel-shape clauses the product deviates from, one measured line each
    run_shape(n);
    return 0;
  }
  if (argc > 2 && !strcmp(argv[2], "mem")) {  // mul operands through local memory instead of the register ABI (OPT bit 8)
    // build twice: default, and with -DECG_FE_ALIGN=16 (128-bit LDL/STL)
    for (int round = 0; round < 2; round++) {
      run<FpK256T<7>, 128, 4, true>("v7   base                 (128,4)", n, jac, gtab);
      run<FpK256T<263>, 128, 4, true>("v263 mul via memory       (128,4)", n, jac, gtab);
      run<FpK256T<263>, 128, 5, true>("v263 mul via memory       (128,5)", n, jac, gtab);
      run<FpK256T<263>, 128, 6, true>("v263 mul via memory       (128,6)", n, jac, gtab);
      run<FpK256T<263>, 128, 8, true>("v263 mul via memory       (128,8)", n, jac, gtab);
      run<FpK256T<259>, 128, 5, true>("v259 mul+sqr via memory   (128,5)", n, jac, gtab);
      run<FpK256T<259>, 128, 8, true>("v259 mul+sqr via memory   (128,8)", n, jac, gtab);
      runp<FpP256T<3>, 128, 4, true>("p256 v3 Solinas base      (128,4)", n, jac, gtab);
      runp<FpP256T<515>, 128, 4, true>("p256 v515 Montgomery call (128,4)", n, jac, gtab);
      runp<FpP256T<515>, 128, 5, true>("p256 v515 Montgomery call (128,5)", n, jac, gtab);
      runp<FpP256T<519>, 128, 4, true>("p256 v519 Mont, sqr inl   (128,4)", n, jac, gtab);
      runp<FpP256T<513>, 128, 4, true>("p256 v513 Mont, all inl   (128,4)", n, jac, gtab);
      runp<FpP256T<771>, 128, 4, true>("p256 v771 Mont via mem    (128,4)", n, jac, gtab);
      runp<FpP256T<771>, 128, 5, true>("p256 v771 Mont via mem    (128,5)", n, jac, gtab);
      run_fmul<FpP256T<3>>("p256 fmul call Solinas");
      run_fmul<FpP256T<515>>("p256 fmul call Montgomery");
      run_fmul<FpP256T<513>>("p256 fmul inline Montgomery");
      runp<FpP256T<259>, 128, 4, true>("p256 v259 mul+sqr via mem (128,4)", n, jac, gtab);
      runp<FpP256T<259>, 128, 5, true>("p256 v259 mul+sqr via mem (128,5)", n, jac, gtab);
      runp<FpP256T<259>, 128, 6, true>("p256 v259 mul+sqr via mem (128,6)", n, jac, gtab);
      runp<FpP256T<263>, 128, 5, true>("p256 v263 mul via mem     (128,5)", n, jac, gtab);
    }
    return 0;
  }
  if (argc > 2 && !strcmp(argv[2], "r2")) {  // round-2 experiments: point-level calls, barriers per point operation, P-256 doubling, DFMA ceiling
    {
      unsigned long long* dout; CK(cudaMalloc(&dout, 256));
      cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
      float best = 1e30f; int iters = 2000; unsigned blocks = 132 * 8;
      for (int rep = 0; rep < 3; rep++) {
        CK(cudaEventRecord(e0));
        kb_dfma_product<<<blocks, 256>>>(dout, iters, 1.0 + rep);
        CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
      }
      printf("DFMA 5x5 product core (50 DFMA + 25 DADD + 50 IADD64, no carries / reduction): %.4g products/s (%.3f ms)\n",
             (double)blocks * 256 * iters / (best * 1e-3), best);
    }
    for (int round = 0; round < 2; round++) {
      run<FpK256T<7>, 128, 4, true>("v7    base                (128,4)", n, jac, gtab);
      run<FpK256T<2055>, 128, 4, true>("v2055 dbl=call(inl inside)(128,4)", n, jac, gtab);
      run<FpK256T<2055>, 128, 3, true>("v2055 dbl=call(inl inside)(128,3)", n, jac, gtab);
      run<FpK256T<2055>, 256, 2, true>("v2055 dbl=call(inl inside)(256,2)", n, jac, gtab);
      run<FpK256T<6151>, 128, 4, true>("v6151 dbl+madd calls      (128,4)", n, jac, gtab);
      run<FpK256T<6151>, 128, 3, true>("v6151 dbl+madd calls      (128,3)", n, jac, gtab);
      run<FpK256T<6145>, 128, 4, true>("v6145 dbl+madd calls, rest inline(128,4)", n, jac, gtab);
      run_sync<FpK256T<1>, 256, 2, 2>("sync2 inline sqr8 (256,2)", n, jac, gtab);
      run_sync<FpK256T<1>, 512, 1, 2>("sync2 inline sqr8 (512,1)", n, jac, gtab);
      run_sync<FpK256T<1>, 384, 1, 2>("sync2 inline sqr8 (384,1)", n, jac, gtab);
      run_sync<FpK256T<1>, 256, 2, 1>("sync1 inline sqr8 (256,2)", n, jac, gtab);
      run_sync<FpK256T<6145>, 256, 2, 2>("sync2 dbl+madd calls (256,2)", n, jac, gtab);
      run_sync<FpK256T<6145>, 512, 1, 2>("sync2 dbl+madd calls (512,1)", n, jac, gtab);
      runp<FpP256T<515>, 128, 4, true>("p256 v515  Montgomery call (128,4)", n, jac, gtab);
      runp<FpP256T<1539>, 128, 4, true>("p256 v1539 + dbl 3M+5S     (128,4)", n, jac, gtab);
      runp<FpP256T<1539>, 128, 5, true>("p256 v1539 + dbl 3M+5S     (128,5)", n, jac, gtab);
      runp<FpP256T<2563>, 128, 4, true>("p256 v2563 dbl=call        (128,4)", n, jac, gtab);
      runp<FpP256T<3587>, 128, 4, true>("p256 v3587 dbl=call 3M+5S  (128,4)", n, jac, gtab);
      runp<FpP256T<3587>, 128, 3, true>("p256 v3587 dbl=call 3M+5S  (128,3)", n, jac, gtab);
      runp_sync<FpP256T<513>, 256, 2, 2>("p256 sync2 inline (256,2)", n, jac, gtab);
      runp_sync<FpP256T<513>, 512, 1, 2>("p256 sync2 inline (512,1)", n, jac, gtab);
      runp_sync<FpP256T<1537>, 512, 1, 2>("p256 sync2 inline 3M+5S (512,1)", n, jac, gtab);
    }
    return 0;
  }
  if (argc > 2 && !strcmp(argv[2], "lean")) {  // multiplier work removed from the production body (OPT bits 13-15), then the trades
    for (int round = 0; round < 3; round++) {
      run_sync<FpK256T<1>, 256, 2, 1>("v1     parent production (256,2)", n, jac, gtab);
      run_sync<FpK256T<8193>, 256, 2, 1>("v8193  + beta column     (256,2)", n, jac, gtab);
      run_sync<FpK256T<24577>, 256, 2, 1>("v24577 + 3/2 X^2 on ALU  (256,2)", n, jac, gtab);
      run_sync<FpK256T<57345>, 256, 2, 1>("v57345 + Y3 mul_sub      (256,2)", n, jac, gtab);
      run_sync<FpK256T<57409>, 256, 2, 1>("v57409 + dbl 2M+5S       (256,2)", n, jac, gtab);
      run_sync<FpK256T<57473>, 256, 2, 1>("v57473 + madd 7M+4S      (256,2)", n, jac, gtab);
      run_sync<FpK256T<57537>, 256, 2, 1>("v57537 + both trades     (256,2)", n, jac, gtab);
    }
    return 0;
  }
  if (argc > 2 && !strcmp(argv[2], "trade")) {  // multiplication-for-squaring trades in the point formulas (OPT bits 6/7)
    for (int round = 0; round < 2; round++) {
      run<FpK256T<7>, 128, 4, true>("v7   base                (128,4)", n, jac, gtab);
      run<FpK256T<71>, 128, 4, true>("v71  dbl 2M+5S           (128,4)", n, jac, gtab);
      run<FpK256T<135>, 128, 4, true>("v135 madd 7M+4S          (128,4)", n, jac, gtab);
      run<FpK256T<199>, 128, 4, true>("v199 both                (128,4)", n, jac, gtab);
    }
    run<FpK256T<199>, 128, 5, true>("v199 both                (128,5)", n, jac, gtab);
    run<FpK256T<199>, 128, 3, true>("v199 both                (128,3)", n, jac, gtab);
    return 0;
  }
  {
    double* dout; CK(cudaMalloc(&dout, 256));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int which = 0; which < 2; which++) {
      float best = 1e30f; int iters = 4000; unsigned blocks = 132 * 8;
      for (int rep = 0; rep < 3; rep++) {
        CK(cudaEventRecord(e0));
        if (which == 0) kb_dfma<<<blocks, 256>>>(dout, iters, 1.5 + rep); else kb_mix<<<blocks, 256>>>(dout, iters, 1.5 + rep, 99u + rep);
        CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
      }
      if (which == 0) printf("DFMA: %.4g /s (%.3f ms)\n", (double)blocks * 256 * iters * 64 / (best * 1e-3), best);
      else printf("mix: %.4g IMAD.WIDE/s + %.4g DFMA/s concurrently (%.3f ms)\n", (double)blocks * 256 * iters * 32 / (best * 1e-3), (double)blocks * 256 * iters * 64 / (best * 1e-3), best);
    }
  }
  run_fmul<FpK256T<0>>("fmul inline mul8x8");
  run_fmul<FpK256T<1>>("fmul inline sqr8");
  run_fmul<FpK256T<3>>("fmul call sqr8");
  run_fmul<FpK256T<9>>("fmul inline kara");
  run_fmul<FpK256T<11>>("fmul call kara");
  run<FpK256T<0>, 128, 3, false>("v0 inline, sqr=mul   (128,3) smem", n, jac, gtab);
  run<FpK256T<1>, 128, 3, false>("v1 inline, sqr8      (128,3) smem", n, jac, gtab);
  run<FpK256T<2>, 128, 3, false>("v2 call,   sqr=mul   (128,3) smem", n, jac, gtab);
  run<FpK256T<3>, 128, 3, false>("v3 call,   sqr8      (128,3) smem", n, jac, gtab);
  run<FpK256T<3>, 192, 2, false>("v3 call,   sqr8      (192,2) smem", n, jac, gtab);
  run<FpK256T<3>, 96, 4, false>("v3 call,   sqr8      (96,4)  smem", n, jac, gtab);
  run<FpK256T<3>, 64, 7, false>("v3 call,   sqr8      (64,7)  smem", n, jac, gtab);
  run_sync<FpK256T<1>, 512, 1>("sync inline sqr8 (512,1)", n, jac, gtab);
  run_sync<FpK256T<1>, 256, 2>("sync inline sqr8 (256,2)", n, jac, gtab);
  run_sync<FpK256T<1>, 640, 1>("sync inline sqr8 (640,1)", n, jac, gtab);
  run_sync<FpK256T<7>, 512, 1>("sync v7 (512,1)", n, jac, gtab);
  run<FpK256T<39>, 128, 4, true>("v39 dbl inline, madd calls (128,4)", n, jac, gtab);
  run<FpK256T<39>, 128, 3, true>("v39 dbl inline, madd calls (128,3)", n, jac, gtab);
  run<FpK256T<39>, 128, 5, true>("v39 dbl inline, madd calls (128,5)", n, jac, gtab);
  run<FpK256T<11>, 128, 4, true>("v11 kara call, sqr call(128,4) gtab", n, jac, gtab);
  run<FpK256T<11>, 128, 5, true>("v11 kara call, sqr call(128,5) gtab", n, jac, gtab);
  run<FpK256T<7>, 128, 5, true>("v7 mul call, sqr inl (128,5) gtab", n, jac, gtab);
  run<FpK256T<7>, 128, 4, true>("v7 mul call, sqr inl (128,4) gtab", n, jac, gtab);
  run<FpK256T<1>, 128, 5, true>("v1 inline, sqr8      (128,5) gtab", n, jac, gtab);
  run<FpK256T<3>, 128, 5, true>("v3 call,   sqr8      (128,5) gtab", n, jac, gtab);
  run<FpK256T<3>, 256, 2, true>("v3 call,   sqr8      (256,2) gtab", n, jac, gtab);
  run_sync<FpK256T<1>, 512, 1>("sync inline sqr8 (512,1)", n, jac, gtab);
  run_sync<FpK256T<1>, 256, 2>("sync inline sqr8 (256,2)", n, jac, gtab);
  run_sync<FpK256T<1>, 640, 1>("sync inline sqr8 (640,1)", n, jac, gtab);
  run_sync<FpK256T<7>, 512, 1>("sync v7 (512,1)", n, jac, gtab);
  run<FpK256T<39>, 128, 4, true>("v39 dbl inline, madd calls (128,4)", n, jac, gtab);
  run<FpK256T<39>, 128, 3, true>("v39 dbl inline, madd calls (128,3)", n, jac, gtab);
  run<FpK256T<39>, 128, 5, true>("v39 dbl inline, madd calls (128,5)", n, jac, gtab);
  run<FpK256T<11>, 128, 4, true>("v11 kara call, sqr call(128,4) gtab", n, jac, gtab);
  run<FpK256T<11>, 128, 5, true>("v11 kara call, sqr call(128,5) gtab", n, jac, gtab);
  run<FpK256T<7>, 128, 5, true>("v7 mul call, sqr inl (128,5) gtab", n, jac, gtab);
  run<FpK256T<7>, 128, 4, true>("v7 mul call, sqr inl (128,4) gtab", n, jac, gtab);
  run<FpK256T<1>, 128, 5, true>("v1 inline, sqr8      (128,5) gtab", n, jac, gtab);
  run_fmul<FpP256T<1>>("p256 fmul inline");
  run_fmul<FpP256T<3>>("p256 fmul call");
  runp<FpP256T<1>, 128, 2, false>("p256 inline (128,2) smem", n, jac, gtab);
  runp<FpP256T<3>, 128, 2, false>("p256 call   (128,2) smem", n, jac, gtab);
  runp<FpP256T<3>, 128, 3, true>("p256 call   (128,3) gtab", n, jac, gtab);
  runp<FpP256T<3>, 128, 4, true>("p256 call   (128,4) gtab", n, jac, gtab);
  run_fmul<FpP256T<19>>("p256 fmul call cols");
  runp<FpP256T<19>, 128, 4, true>("p256 cols call (128,4) gtab", n, jac, gtab);
  runp<FpP256T<19>, 128, 3, true>("p256 cols call (128,3) gtab", n, jac, gtab);
  runp<FpP256T<23>, 128, 4, true>("p256 cols mulcall sqr-inl (128,4)", n, jac, gtab);
  runp<FpP256T<7>, 128, 4, true>("p256 mul call, sqr inl (128,4) gtab", n, jac, gtab);
  runp<FpP256T<7>, 128, 3, true>("p256 mul call, sqr inl (128,3) gtab", n, jac, gtab);
  return 0;
}
