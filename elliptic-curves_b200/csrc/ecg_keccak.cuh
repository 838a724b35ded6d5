// ecg_keccak.cuh — Keccak-f[1600] and a streaming SHAKE256 (FIPS 202) per thread: rate 136 bytes, domain byte 0x1F.
//
// Ed448 verification (ecg_ed448.cuh) hashes dom4 || R || A || M into 114 bytes (RFC 8032 section 5.2.7); the reference
// uses sha3::Shake256 (ed448-goldilocks/src/sign/verifying_key.rs:292-302).  The state stays in registers (every
// index into it is a compile-time constant); input bytes collect in a 136-byte block buffer, which is XORed into the
// state as 17 lanes when it fills, so absorbing straight from global memory needs no alignment.
#pragma once
#include "ecg_prim.cuh"

namespace ecg {

ECG_D uint64_t keccak_rotl(uint64_t v, int s) { return s ? (v << s) | (v >> (64 - s)) : v; }

// the 24 rounds on the 25 lanes, lane (x, y) at s[x + 5 y]; inlined, so that the lanes stay in registers
ECG_D void keccak_f1600(uint64_t* s) {
  const uint64_t RC[24] = {0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808Aull, 0x8000000080008000ull,
                           0x000000000000808Bull, 0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull,
                           0x000000000000008Aull, 0x0000000000000088ull, 0x0000000080008009ull, 0x000000008000000Aull,
                           0x000000008000808Bull, 0x800000000000008Bull, 0x8000000000008089ull, 0x8000000000008003ull,
                           0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800Aull, 0x800000008000000Aull,
                           0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};
  // rho offsets and the pi permutation along the lane cycle that starts at lane 1
  const int RHO[24] = {1, 3, 6, 10, 15, 21, 28, 36, 45, 55, 2, 14, 27, 41, 56, 8, 25, 43, 62, 18, 39, 61, 20, 44};
  const int PI[24] = {10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};
#pragma unroll 1
  for (int round = 0; round < 24; round++) {
    uint64_t c[5];
#pragma unroll
    for (int x = 0; x < 5; x++) c[x] = s[x] ^ s[x + 5] ^ s[x + 10] ^ s[x + 15] ^ s[x + 20];
#pragma unroll
    for (int x = 0; x < 5; x++) {
      const uint64_t d = c[(x + 4) % 5] ^ keccak_rotl(c[(x + 1) % 5], 1);
#pragma unroll
      for (int y = 0; y < 25; y += 5) s[x + y] ^= d;
    }
    uint64_t t = s[1];
#pragma unroll
    for (int i = 0; i < 24; i++) {
      const uint64_t u = s[PI[i]];
      s[PI[i]] = keccak_rotl(t, RHO[i]);
      t = u;
    }
#pragma unroll
    for (int y = 0; y < 25; y += 5) {
#pragma unroll
      for (int x = 0; x < 5; x++) c[x] = s[y + x];
#pragma unroll
      for (int x = 0; x < 5; x++) s[y + x] = c[x] ^ (~c[(x + 1) % 5] & c[(x + 2) % 5]);
    }
    s[0] ^= RC[round];
  }
}

// SHAKE256: absorb any number of byte strings, then squeeze up to one block (136 bytes) of output
struct Shake256 {
  uint64_t s[25];
  uint8_t buf[136];
  int pos;

  ECG_D void init() {
#pragma unroll
    for (int i = 0; i < 25; i++) s[i] = 0;
    pos = 0;
  }
  ECG_D void absorb_block() {
#pragma unroll
    for (int i = 0; i < 17; i++) {
      uint64_t w = 0;
#pragma unroll
      for (int b = 0; b < 8; b++) w |= (uint64_t)buf[8 * i + b] << (8 * b);
      s[i] ^= w;
    }
    keccak_f1600(s);
    pos = 0;
  }
  ECG_D void absorb(const uint8_t* p, size_t n) {
#pragma unroll 1
    for (size_t i = 0; i < n; i++) {
      buf[pos++] = p[i];
      if (pos == 136) absorb_block();
    }
  }
  // pad (0x1F ... 0x80) and squeeze N <= 136 bytes
  template <int N>
  ECG_D void finish(uint8_t* out) {
    buf[pos++] = 0x1F;
#pragma unroll 1
    while (pos < 136) buf[pos++] = 0;
    buf[135] |= 0x80;
    absorb_block();
#pragma unroll
    for (int i = 0; i < N; i++) out[i] = (uint8_t)(s[i >> 3] >> (8 * (i & 7)));
  }
  // pad (0x1F ... 0x80) and squeeze N bytes of any length: one more permutation before every further 136-byte block
  template <int N>
  ECG_D void finish_long(uint8_t* out) {
    buf[pos++] = 0x1F;
#pragma unroll 1
    while (pos < 136) buf[pos++] = 0;
    buf[135] |= 0x80;
    absorb_block();
#pragma unroll 1
    for (int i = 0; i < N; i++) {
      const int j = i % 136;
      if (i && j == 0) keccak_f1600(s);
      out[i] = (uint8_t)(s[j >> 3] >> (8 * (j & 7)));
    }
  }
};

}  // namespace ecg
