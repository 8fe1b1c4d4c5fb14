// K6 — the encryption layer of PGPMessage.Decrypt (crypto_pgp.go:453-471) on the device.
//
//   K6a rsa_crt_decrypt_kernel   the PKESK's RSA-2048 private-key operation (CRT, two 1024-bit exponentiations) and
//                                PKCS#1 v1.5 type-2 unpadding as Go 1.13's decryptPKCS1v15, then EncryptedKey.Decrypt's
//                                split of the message into cipher byte | key | 16-bit checksum.
//   K6b seipd_decrypt_kernel     OpenPGP CFB without resync (tag 18) under AES-128/192/256: the quick check of every
//                                candidate session key in order, then the whole packet and its SHA-1 MDC.
//
// K6a is constant time in the private key and the padding: the exponent loop has a fixed trip count (256 windows of
// 4 bits over 1024 bits whatever dp / dq are), the window entry is read by scanning the whole table with masks, every
// conditional subtraction is masked (mont_mul<.., CT = true>), and the unpadding scans all 256 bytes with masks.  The
// only data-dependent values that leave the kernel are the ones Go's own control flow reveals (valid or not, the cipher
// byte and the key length).  K6b is not constant time: AES runs from an S-box in shared memory.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "rsa_verify_r32.cuh"
#include "pgp_digest.cuh"

namespace bftq {
namespace k6 {

// One registered private key, radix 2^32 little-endian words.  Lives only in the keyring's dedicated device allocation.
struct RsaPriv32 {
  uint32_t p[32], q[32];
  uint32_t dp[32], dq[32];       // d mod (p-1), d mod (q-1)
  uint32_t r2p[32], r2q[32];     // 2^2048 mod p, mod q
  uint32_t uq[32];               // u * 2^1024 mod q, u = p^-1 mod q (RFC 4880's CRT coefficient) in Montgomery form
  uint32_t n[64];
  uint32_t pn[64];               // p * 2^2048 mod n
  uint32_t p0inv, q0inv, n0inv, pad;
};

// K6a output word per item: status | cipher << 8 | key length << 16.  Key bytes go to a separate per-call array.
constexpr uint32_t kDecNoKey = 0;      // c > n handled on the host; invalid padding: EncryptedKey.Key stays empty
constexpr uint32_t kDecOk = 1;
constexpr uint32_t kDecShort = 2;      // valid padding, message shorter than 3 bytes: the reference panics (b[len(b)-2])

using r32::T;

// out = a + b over the 4-lane group, returns the carry out of the top lane (the same in every lane of the group).
template <int W>
__device__ __forceinline__ uint32_t ct_add(uint32_t (&out)[W], const uint32_t (&a)[W], const uint32_t (&b)[W], const int r, const int gbase) {
  uint32_t g;
  asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(out[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(out[k]) : "r"(a[k]), "r"(b[k]));
  asm volatile("addc.u32 %0, 0, 0;" : "=r"(g));
  uint32_t ones = 1u;
#pragma unroll
  for (int k = 0; k < W; k++) ones &= (uint32_t)(out[k] == 0xffffffffu);
  const uint32_t gb = __ballot_sync(kFull, g != 0u) >> gbase;
  const uint32_t pb = __ballot_sync(kFull, ones != 0u) >> gbase;
  uint32_t ctop;
  const uint32_t ci = r32::lane_carry_in(gb, pb, r, ctop);
  r32::ripple_add(out, ci);
  return ctop;
}
// d = x - n over the group, returns the borrow out of the top lane.
template <int W>
__device__ __forceinline__ uint32_t ct_sub(uint32_t (&d)[W], const uint32_t (&x)[W], const uint32_t (&n)[W], const int r, const int gbase) {
  const uint32_t bo = r32::sub_n(d, x, n);
  uint32_t zeros = 1u;
#pragma unroll
  for (int k = 0; k < W; k++) zeros &= (uint32_t)(d[k] == 0u);
  const uint32_t bgb = __ballot_sync(kFull, bo != 0u) >> gbase;
  const uint32_t bpb = __ballot_sync(kFull, zeros != 0u) >> gbase;
  uint32_t btop;
  const uint32_t bi = r32::lane_carry_in(bgb, bpb, r, btop);
  r32::ripple_sub(d, bi);
  return btop;
}
template <int W>
__device__ __forceinline__ void ct_select(uint32_t (&x)[W], const uint32_t (&y)[W], const uint32_t take_y) {
  const uint32_t m = 0u - take_y;
#pragma unroll
  for (int k = 0; k < W; k++) x[k] = (y[k] & m) | (x[k] & ~m);
}
// x -= n when x >= n, masked.
template <int W>
__device__ __forceinline__ void ct_cond_sub(uint32_t (&x)[W], const uint32_t (&n)[W], const int r, const int gbase) {
  uint32_t d[W];
  const uint32_t bt = ct_sub(d, x, n, r, gbase);
  ct_select(x, d, bt ^ 1u);
}
// A 1024-bit number in the W = 8 layout -> the same number in the W = 16 (2048-bit) layout.
__device__ __forceinline__ void widen(const uint32_t (&a)[8], uint32_t (&o)[16], const int r, const int gbase) {
  const int s0 = gbase + ((2 * r) & 3), s1 = gbase + ((2 * r + 1) & 3);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint32_t x0 = __shfl_sync(kFull, a[j], s0), x1 = __shfl_sync(kFull, a[j], s1);
    o[j] = r < 2 ? x0 : 0u;
    o[8 + j] = r < 2 ? x1 : 0u;
  }
}

template <int W>
__device__ __forceinline__ void mmul(uint32_t (&out)[W], const uint32_t (&a)[W], const uint32_t (&b)[W], const uint32_t (&n)[W], const uint32_t n0inv,
                                     const int r, const int gbase) {
  r32::mont_mul<W, true>(out, a, b, n, n0inv, r, gbase);
}

// The number 1 in the W = 8 layout.  Recomputed from %laneid at each use (volatile asm): kept live across the exponent
// loop it was the one value ptxas spilled to local memory.
__device__ __forceinline__ void make_one(uint32_t (&one)[8]) {
  uint32_t lane;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
#pragma unroll
  for (int j = 0; j < 8; j++) one[j] = (j == 0 && (lane & (T - 1)) == 0) ? 1u : 0u;
}

// c^dexp mod m for one 1024-bit prime; c given as its two 1024-bit halves.  Result fully reduced (< m).
template <int BLOCK>
__device__ __forceinline__ void crt_half(uint32_t (&res)[8], const uint32_t (&c_lo)[8], const uint32_t (&c_hi)[8], const uint32_t* __restrict__ m_g,
                                         const uint32_t* __restrict__ r2_g, const uint32_t* __restrict__ dexp, const uint32_t m0inv,
                                         uint32_t (*tab)[8][BLOCK], const int r, const int gbase) {
  constexpr int W = 8;
  uint32_t m[W], r2[W], s[W], t[W], y[W], one[W];
#pragma unroll
  for (int j = 0; j < W; j++) { m[j] = __ldg(m_g + r * W + j); r2[j] = __ldg(r2_g + r * W + j); }
  make_one(one);
  // c mod m as a value below 2^1024: c_hi * 2^1024 mod m (one product with R^2), + c_lo, minus m while >= 2^1024
  mmul(t, c_hi, r2, m, m0inv, r, gbase);
  uint32_t hi = ct_add(s, t, c_lo, r, gbase);
#pragma unroll
  for (int k = 0; k < 2; k++) {
    uint32_t d[W];
    const uint32_t bt = ct_sub(d, s, m, r, gbase);
    ct_select(s, d, hi);
    hi &= bt ^ 1u;                                // the borrow consumed bit 1024
  }
  uint32_t bm[W];
  mmul(bm, s, r2, m, m0inv, r, gbase);            // Montgomery form of c mod m
  mmul(y, r2, one, m, m0inv, r, gbase);           // Montgomery form of 1
  const int tid = threadIdx.x;
#pragma unroll
  for (int j = 0; j < W; j++) { tab[0][j][tid] = y[j]; tab[1][j][tid] = bm[j]; t[j] = bm[j]; }
#pragma unroll 1
  for (int e = 2; e < 16; e++) {
    uint32_t u[W];
    mmul(u, t, bm, m, m0inv, r, gbase);
#pragma unroll
    for (int j = 0; j < W; j++) { tab[e][j][tid] = u[j]; t[j] = u[j]; }
  }
  // fixed-window exponentiation over all 1024 exponent bits, most significant window first
#pragma unroll 1
  for (int win = 255; win >= 0; win--) {
#pragma unroll 1
    for (int k = 0; k < 4; k++) { mmul(t, y, y, m, m0inv, r, gbase); for (int j = 0; j < W; j++) y[j] = t[j]; }
    const uint32_t w = (__ldg(dexp + (win >> 3)) >> ((win & 7) * 4)) & 15u;
    uint32_t sel[W];
#pragma unroll
    for (int j = 0; j < W; j++) sel[j] = 0u;
#pragma unroll
    for (int e = 0; e < 16; e++) {
      const uint32_t msk = 0u - (uint32_t)((uint32_t)e == w);
#pragma unroll
      for (int j = 0; j < W; j++) sel[j] |= tab[e][j][tid] & msk;
    }
    mmul(t, y, sel, m, m0inv, r, gbase);
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = t[j];
  }
  make_one(one);
  mmul(res, y, one, m, m0inv, r, gbase);          // leaves Montgomery form: <= m
  ct_cond_sub(res, m, r, gbase);
}

// One 4-lane group per item.  c_be: n_items x 256 bytes (the PKESK MPI, left-padded; c <= n checked by the host),
// slot: key slot per item.  out_info: kDec* | cipher << 8 | key length << 16; out_key: n_items x 32 bytes, the first
// min(key length, 32) bytes of the session key, zero beyond.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
rsa_crt_decrypt_kernel(const RsaPriv32* __restrict__ keys, const uint32_t* __restrict__ slot, const uint8_t* __restrict__ c_be, const uint64_t n_items,
                       uint32_t* __restrict__ out_info, uint8_t* __restrict__ out_key) {
  __shared__ uint32_t tab[16][8][BLOCK];
  __shared__ uint8_t em_s[BLOCK / T][256];
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int grp = threadIdx.x / T;
  for (uint64_t base = (uint64_t)blockIdx.x * (BLOCK / T); base < n_items; base += (uint64_t)gridDim.x * (BLOCK / T)) {
    const uint64_t item_raw = base + (uint64_t)grp;
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : n_items - 1;
    const RsaPriv32* __restrict__ key = keys + __ldg(slot + item);
    const uint8_t* cp = c_be + item * 256u;
    uint32_t c_lo[8], c_hi[8], m1[8], m2[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { c_lo[j] = be_word(cp, r * 8 + j); c_hi[j] = be_word(cp, 32 + r * 8 + j); }
    crt_half<BLOCK>(m1, c_lo, c_hi, key->p, key->r2p, key->dp, __ldg(&key->p0inv), tab, r, gbase);
    crt_half<BLOCK>(m2, c_lo, c_hi, key->q, key->r2q, key->dq, __ldg(&key->q0inv), tab, r, gbase);
    // Garner with RFC 4880's u = p^-1 mod q:  h = (m2 - m1) u mod q,  m = m1 + p h  (< n)
    uint32_t q[8], uq[8], a[8], d[8], h[8];
    const uint32_t q0inv = __ldg(&key->q0inv);
#pragma unroll
    for (int j = 0; j < 8; j++) { q[j] = __ldg(key->q + r * 8 + j); uq[j] = __ldg(key->uq + r * 8 + j); a[j] = m1[j]; }
    ct_cond_sub(a, q, r, gbase);                  // m1 < p < 2q
    const uint32_t bt = ct_sub(d, m2, a, r, gbase);
    uint32_t dq_[8];
    ct_add(dq_, d, q, r, gbase);
    ct_select(d, dq_, bt);
    mmul(h, d, uq, q, q0inv, r, gbase);
    ct_cond_sub(h, q, r, gbase);
    uint32_t h16[16], m16[16], nn[16], pn[16], ph[16], mm[16];
    widen(h, h16, r, gbase);
    widen(m1, m16, r, gbase);
#pragma unroll
    for (int j = 0; j < 16; j++) { nn[j] = __ldg(key->n + r * 16 + j); pn[j] = __ldg(key->pn + r * 16 + j); }
    mmul(ph, pn, h16, nn, __ldg(&key->n0inv), r, gbase);   // p h mod n, almost reduced
    ct_cond_sub(ph, nn, r, gbase);
    ct_add(mm, ph, m16, r, gbase);
    // EM = I2OSP(m, 256) into this group's shared bytes
    uint8_t* em = em_s[grp];
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const int off = 256 - 4 - 4 * (r * 16 + j);
      em[off] = (uint8_t)(mm[j] >> 24); em[off + 1] = (uint8_t)(mm[j] >> 16); em[off + 2] = (uint8_t)(mm[j] >> 8); em[off + 3] = (uint8_t)mm[j];
    }
    __syncwarp();
    // decryptPKCS1v15: em[0] == 0, em[1] == 2, the first zero at index >= 10 (all with masks, every byte read)
    uint32_t looking = 1u, index = 0u;
#pragma unroll 8
    for (int i = 2; i < 256; i++) {
      const uint32_t z = (uint32_t)(em[i] == 0);
      const uint32_t take = 0u - (looking & z);
      index = ((uint32_t)i & take) | (index & ~take);
      looking &= z ^ 1u;
    }
    const uint32_t ok = (uint32_t)(em[0] == 0) & (uint32_t)(em[1] == 2) & (looking ^ 1u) & (uint32_t)(index >= 10u);
    const uint32_t len = 255u - index;            // the message is em[index+1 ..]
    const uint32_t keylen = len >= 3u ? len - 3u : 0u;
    // cipher byte (k = 0) and key bytes (k = 1..32): lane r takes k = r, r + 4, ...
    for (int k = r; k < 33; k += T) {
      const uint32_t target = index + 1u + (uint32_t)k;
      uint32_t v = 0u;
#pragma unroll 8
      for (int i = 0; i < 256; i++) v |= (uint32_t)em[i] & (0u - (uint32_t)((uint32_t)i == target));
      const uint32_t keep = 0u - (ok & (uint32_t)(k == 0 || (uint32_t)(k - 1) < keylen));
      v &= keep;
      if (valid) {
        if (k == 0) {
          const uint32_t st = ok ? (len >= 3u ? kDecOk : kDecShort) : kDecNoKey;
          out_info[item_raw] = st | (v << 8) | ((keylen & (0u - ok)) << 16);
        } else {
          out_key[item_raw * 32u + (uint32_t)(k - 1)] = (uint8_t)v;
        }
      }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 64; j++) em[r * 64 + j] = 0;   // no key material left in shared memory: the padded block,
#pragma unroll
    for (int e = 0; e < 16; e++)                       // and the window table (powers of c mod q, which reveal q)
#pragma unroll
      for (int j = 0; j < 8; j++) tab[e][j][threadIdx.x] = 0u;
    __syncwarp();
  }
}

// ---- K6b ------------------------------------------------------------------------------------------------------------
__constant__ uint8_t c_aes_sbox[256] = {
    0x63, 0x7c, 0x77, 0x7b, 0xf2, 0x6b, 0x6f, 0xc5, 0x30, 0x01, 0x67, 0x2b, 0xfe, 0xd7, 0xab, 0x76,
    0xca, 0x82, 0xc9, 0x7d, 0xfa, 0x59, 0x47, 0xf0, 0xad, 0xd4, 0xa2, 0xaf, 0x9c, 0xa4, 0x72, 0xc0,
    0xb7, 0xfd, 0x93, 0x26, 0x36, 0x3f, 0xf7, 0xcc, 0x34, 0xa5, 0xe5, 0xf1, 0x71, 0xd8, 0x31, 0x15,
    0x04, 0xc7, 0x23, 0xc3, 0x18, 0x96, 0x05, 0x9a, 0x07, 0x12, 0x80, 0xe2, 0xeb, 0x27, 0xb2, 0x75,
    0x09, 0x83, 0x2c, 0x1a, 0x1b, 0x6e, 0x5a, 0xa0, 0x52, 0x3b, 0xd6, 0xb3, 0x29, 0xe3, 0x2f, 0x84,
    0x53, 0xd1, 0x00, 0xed, 0x20, 0xfc, 0xb1, 0x5b, 0x6a, 0xcb, 0xbe, 0x39, 0x4a, 0x4c, 0x58, 0xcf,
    0xd0, 0xef, 0xaa, 0xfb, 0x43, 0x4d, 0x33, 0x85, 0x45, 0xf9, 0x02, 0x7f, 0x50, 0x3c, 0x9f, 0xa8,
    0x51, 0xa3, 0x40, 0x8f, 0x92, 0x9d, 0x38, 0xf5, 0xbc, 0xb6, 0xda, 0x21, 0x10, 0xff, 0xf3, 0xd2,
    0xcd, 0x0c, 0x13, 0xec, 0x5f, 0x97, 0x44, 0x17, 0xc4, 0xa7, 0x7e, 0x3d, 0x64, 0x5d, 0x19, 0x73,
    0x60, 0x81, 0x4f, 0xdc, 0x22, 0x2a, 0x90, 0x88, 0x46, 0xee, 0xb8, 0x14, 0xde, 0x5e, 0x0b, 0xdb,
    0xe0, 0x32, 0x3a, 0x0a, 0x49, 0x06, 0x24, 0x5c, 0xc2, 0xd3, 0xac, 0x62, 0x91, 0x95, 0xe4, 0x79,
    0xe7, 0xc8, 0x37, 0x6d, 0x8d, 0xd5, 0x4e, 0xa9, 0x6c, 0x56, 0xf4, 0xea, 0x65, 0x7a, 0xae, 0x08,
    0xba, 0x78, 0x25, 0x2e, 0x1c, 0xa6, 0xb4, 0xc6, 0xe8, 0xdd, 0x74, 0x1f, 0x4b, 0xbd, 0x8b, 0x8a,
    0x70, 0x3e, 0xb5, 0x66, 0x48, 0x03, 0xf6, 0x0e, 0x61, 0x35, 0x57, 0xb9, 0x86, 0xc1, 0x1d, 0x9e,
    0xe1, 0xf8, 0x98, 0x11, 0x69, 0xd9, 0x8e, 0x94, 0x9b, 0x1e, 0x87, 0xe9, 0xce, 0x55, 0x28, 0xdf,
    0x8c, 0xa1, 0x89, 0x0d, 0xbf, 0xe6, 0x42, 0x68, 0x41, 0x99, 0x2d, 0x0f, 0xb0, 0x54, 0xbb, 0x16};

__device__ __forceinline__ uint32_t aes_xt(uint32_t x) { return ((x << 1) ^ ((x & 0x80u) ? 0x1bu : 0u)) & 0xffu; }
__device__ __forceinline__ uint32_t sub_word(uint32_t x, const uint8_t* sb) {
  return ((uint32_t)sb[x >> 24] << 24) | ((uint32_t)sb[(x >> 16) & 0xff] << 16) | ((uint32_t)sb[(x >> 8) & 0xff] << 8) | sb[x & 0xff];
}
// The thread's round keys live in shared memory (rk[i * K6B_BLOCK + tid]), not in registers: 60 live words for AES-256
// next to the SHA-1 state pushed the kernel into local memory.  Zeroed by the kernel before it exits.
constexpr int K6B_BLOCK = 128;
template <int NK>
__device__ __forceinline__ void aes_expand(const uint8_t* __restrict__ key, uint32_t* rk, const uint8_t* sb) {
  const int tid = threadIdx.x;
  uint32_t rcon = 1u;
#pragma unroll 1
  for (int i = 0; i < NK; i++)
    rk[i * K6B_BLOCK + tid] = ((uint32_t)key[4 * i] << 24) | ((uint32_t)key[4 * i + 1] << 16) | ((uint32_t)key[4 * i + 2] << 8) | key[4 * i + 3];
#pragma unroll 1
  for (int i = NK; i < 4 * (NK + 7); i++) {
    uint32_t t = rk[(i - 1) * K6B_BLOCK + tid];
    if (i % NK == 0) { t = sub_word((t << 8) | (t >> 24), sb) ^ (rcon << 24); rcon = aes_xt(rcon); }
    else if (NK > 6 && i % NK == 4) t = sub_word(t, sb);
    rk[i * K6B_BLOCK + tid] = rk[(i - NK) * K6B_BLOCK + tid] ^ t;
  }
}
__device__ __forceinline__ uint32_t sb_col(const uint32_t s0, const uint32_t s1, const uint32_t s2, const uint32_t s3, const uint8_t* sb, const bool mix) {
  const uint32_t a0 = sb[s0 >> 24], a1 = sb[(s1 >> 16) & 0xff], a2 = sb[(s2 >> 8) & 0xff], a3 = sb[s3 & 0xff];
  if (!mix) return (a0 << 24) | (a1 << 16) | (a2 << 8) | a3;
  const uint32_t o0 = aes_xt(a0) ^ aes_xt(a1) ^ a1 ^ a2 ^ a3;
  const uint32_t o1 = a0 ^ aes_xt(a1) ^ aes_xt(a2) ^ a2 ^ a3;
  const uint32_t o2 = a0 ^ a1 ^ aes_xt(a2) ^ aes_xt(a3) ^ a3;
  const uint32_t o3 = aes_xt(a0) ^ a0 ^ a1 ^ a2 ^ aes_xt(a3);
  return (o0 << 24) | (o1 << 16) | (o2 << 8) | o3;
}
template <int NK>
__device__ __forceinline__ void aes_encrypt(const uint32_t* rk, uint32_t& s0, uint32_t& s1, uint32_t& s2, uint32_t& s3, const uint8_t* sb) {
  constexpr int NR = NK + 6;
  const int tid = threadIdx.x;
  s0 ^= rk[0 * K6B_BLOCK + tid]; s1 ^= rk[1 * K6B_BLOCK + tid]; s2 ^= rk[2 * K6B_BLOCK + tid]; s3 ^= rk[3 * K6B_BLOCK + tid];
#pragma unroll 1
  for (int rd = 1; rd <= NR; rd++) {
    const bool mix = rd < NR;
    const uint32_t t0 = sb_col(s0, s1, s2, s3, sb, mix), t1 = sb_col(s1, s2, s3, s0, sb, mix);
    const uint32_t t2 = sb_col(s2, s3, s0, s1, sb, mix), t3 = sb_col(s3, s0, s1, s2, sb, mix);
    s0 = t0 ^ rk[(4 * rd) * K6B_BLOCK + tid]; s1 = t1 ^ rk[(4 * rd + 1) * K6B_BLOCK + tid];
    s2 = t2 ^ rk[(4 * rd + 2) * K6B_BLOCK + tid]; s3 = t3 ^ rk[(4 * rd + 3) * K6B_BLOCK + tid];
  }
}
__device__ __forceinline__ uint32_t load_be32(const uint8_t* p, uint64_t pos, uint64_t len) {
  uint32_t v = 0;
#pragma unroll
  for (int t = 0; t < 4; t++) v = (v << 8) | (pos + t < len ? (uint32_t)p[pos + t] : 0u);
  return v;
}

// OpenPGP's quick check (RFC 4880 §5.13): the last two bytes of the random prefix block repeat in bytes 16, 17.
template <int NK>
__device__ bool quick_check(const uint8_t* __restrict__ key, const uint8_t* __restrict__ ct, uint32_t* rk, const uint8_t* sb) {
  aes_expand<NK>(key, rk, sb);
  uint32_t s0 = 0u, s1 = 0u, s2 = 0u, s3 = 0u;
  aes_encrypt<NK>(rk, s0, s1, s2, s3, sb);
  const uint32_t p3 = load_be32(ct, 12, 16) ^ s3;
  uint32_t c0 = load_be32(ct, 0, 16), c1 = load_be32(ct, 4, 16), c2 = load_be32(ct, 8, 16), c3 = load_be32(ct, 12, 16);
  aes_encrypt<NK>(rk, c0, c1, c2, c3, sb);
  const uint32_t p16 = ct[16] ^ (c0 >> 24), p17 = ct[17] ^ ((c0 >> 16) & 0xff);
  return ((p3 >> 8) & 0xff) == p16 && (p3 & 0xff) == p17;
}

// CFB-decrypts all len bytes (zero IV, no resync: one CFB stream over prefix | data | MDC packet) into pt and checks
// the MDC packet: D3 14 followed by SHA-1(prefix | data | D3 14).
template <int NK>
__device__ bool decrypt_stream(const uint8_t* __restrict__ key, const uint8_t* __restrict__ ct, const uint64_t len, uint8_t* __restrict__ pt,
                               uint32_t* rk, uint32_t* wsh, const uint8_t* sb) {
  aes_expand<NK>(key, rk, sb);
  const uint64_t H = len - 20;                      // hashed bytes
  const uint64_t nblk = (H + 8) / 64 + 1;
  const uint64_t nchunks = max(nblk, (len + 63) / 64);
  uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
  uint32_t f0 = 0u, f1 = 0u, f2 = 0u, f3 = 0u;
  // sha1_compress indexes its message schedule at run time: in registers that array would live in local memory
  uint32_t (&w)[16] = *reinterpret_cast<uint32_t (*)[16]>(wsh);
#pragma unroll 1
  for (uint64_t k = 0; k < nchunks; k++) {
#pragma unroll
    for (int b = 0; b < 4; b++) {
      const uint64_t pos0 = 64 * k + 16 * b;
      uint32_t k0 = f0, k1 = f1, k2 = f2, k3 = f3;
      aes_encrypt<NK>(rk, k0, k1, k2, k3, sb);
      f0 = load_be32(ct, pos0, len); f1 = load_be32(ct, pos0 + 4, len); f2 = load_be32(ct, pos0 + 8, len); f3 = load_be32(ct, pos0 + 12, len);
      const uint32_t pw[4] = {f0 ^ k0, f1 ^ k1, f2 ^ k2, f3 ^ k3};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const uint64_t pos = pos0 + 4 * j;
        uint32_t hw = 0;
#pragma unroll
        for (int t = 0; t < 4; t++) {
          const uint32_t by = (pw[j] >> (24 - 8 * t)) & 0xff;
          if (pos + t < len) pt[pos + t] = (uint8_t)by;
          hw = (hw << 8) | (pos + t < H ? by : (pos + t == H ? 0x80u : 0u));
        }
        w[4 * b + j] = hw;
      }
    }
    if (k == nblk - 1) { w[14] = (uint32_t)((H * 8) >> 32); w[15] = (uint32_t)(H * 8); }
    if (k < nblk) sha1_compress(h, w);
  }
  bool ok = pt[len - 22] == 0xD3 && pt[len - 21] == 0x14;
#pragma unroll
  for (int i = 0; i < 5; i++) ok = ok && load_be32(pt, len - 20 + 4 * i, len) == h[i];
  return ok;
}

__device__ void seipd_item(const uint8_t* __restrict__ ct_blob, const uint64_t* __restrict__ ct_off, const uint32_t* __restrict__ cand_off,
                           const uint32_t* __restrict__ cand_rec, const uint8_t* __restrict__ rec_cipher, const uint8_t* __restrict__ keys,
                           const uint64_t i, uint8_t* __restrict__ pt_blob, uint8_t* __restrict__ out_res, const uint64_t* __restrict__ ct_end,
                           uint32_t* rk, uint32_t* wsh, const uint8_t* sb);

__device__ __forceinline__ int nk_of(uint8_t cipher) { return cipher == 7 ? 4 : (cipher == 8 ? 6 : 8); }

// One thread per message.  ct: the SEIPD body after its version byte, de-chunked, at ct_off[i] (len >= 18); item i's
// candidate session keys are K6a records cand_rec[cand_off[i] .. cand_off[i+1]) with AES cipher ids rec_cipher[].
// out_res[i]: 0 MDC good, 1 MDC bad, 2 no candidate passed the quick check, 3 a candidate passed but the packet is
// too short to hold the MDC packet.  pt (same offsets as ct): the decrypted prefix | data | MDC packet.
// ct_end (nullable): item i spans [ct_off[i], ct_end[i]) instead of [ct_off[i], ct_off[i+1]) — the items need not be
// packed.  cand_off == nullptr: item i's one candidate is record i when rec_cipher[i] != 0, none otherwise (cand_rec
// unused).
__global__ void __launch_bounds__(K6B_BLOCK)
seipd_decrypt_kernel(const uint8_t* __restrict__ ct_blob, const uint64_t* __restrict__ ct_off, const uint32_t* __restrict__ cand_off,
                     const uint32_t* __restrict__ cand_rec, const uint8_t* __restrict__ rec_cipher, const uint8_t* __restrict__ keys,
                     const uint64_t n_items, uint8_t* __restrict__ pt_blob, uint8_t* __restrict__ out_res,
                     const uint64_t* __restrict__ ct_end = nullptr) {
  __shared__ uint8_t sb[256];
  __shared__ uint32_t rk[60 * K6B_BLOCK];
  __shared__ uint32_t wsh[K6B_BLOCK][17];         // SHA-1 schedule per thread, padded against bank conflicts
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sb[i] = c_aes_sbox[i];
  __syncthreads();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_items) seipd_item(ct_blob, ct_off, cand_off, cand_rec, rec_cipher, keys, i, pt_blob, out_res, ct_end, rk, wsh[threadIdx.x], sb);
#pragma unroll 1
  for (int k = 0; k < 60; k++) rk[k * K6B_BLOCK + threadIdx.x] = 0u;    // no key schedule or plaintext left in shared memory
#pragma unroll 1
  for (int k = 0; k < 17; k++) wsh[threadIdx.x][k] = 0u;
}
__device__ void seipd_item(const uint8_t* __restrict__ ct_blob, const uint64_t* __restrict__ ct_off, const uint32_t* __restrict__ cand_off,
                           const uint32_t* __restrict__ cand_rec, const uint8_t* __restrict__ rec_cipher, const uint8_t* __restrict__ keys,
                           const uint64_t i, uint8_t* __restrict__ pt_blob, uint8_t* __restrict__ out_res, const uint64_t* __restrict__ ct_end,
                           uint32_t* rk, uint32_t* wsh, const uint8_t* sb) {
  const uint8_t* ct = ct_blob + ct_off[i];
  const uint64_t len = (ct_end != nullptr ? ct_end[i] : ct_off[i + 1]) - ct_off[i];
  int chosen = -1;
  const uint32_t c0 = cand_off != nullptr ? cand_off[i] : (uint32_t)i;
  const uint32_t c1 = cand_off != nullptr ? cand_off[i + 1] : (uint32_t)i + (rec_cipher[i] != 0 ? 1u : 0u);
  for (uint32_t c = c0; c < c1 && chosen < 0; c++) {
    const uint32_t rec = cand_off != nullptr ? cand_rec[c] : c;
    const uint8_t* key = keys + (uint64_t)rec * 32u;
    const int nk = nk_of(rec_cipher[rec]);
    const bool pass = nk == 4 ? quick_check<4>(key, ct, rk, sb) : (nk == 6 ? quick_check<6>(key, ct, rk, sb) : quick_check<8>(key, ct, rk, sb));
    if (pass) chosen = (int)rec;
  }
  if (chosen < 0) { out_res[i] = 2; return; }
  if (len < 18 + 22) { out_res[i] = 3; return; }
  const uint8_t* key = keys + (uint64_t)chosen * 32u;
  uint8_t* pt = pt_blob + ct_off[i];
  const int nk = nk_of(rec_cipher[chosen]);
  const bool ok = nk == 4 ? decrypt_stream<4>(key, ct, len, pt, rk, wsh, sb) : (nk == 6 ? decrypt_stream<6>(key, ct, len, pt, rk, wsh, sb) : decrypt_stream<8>(key, ct, len, pt, rk, wsh, sb));
  out_res[i] = ok ? 0 : 1;
}


// ---- K6p / K6q: the decryption front stage of the encrypted read path (bftq_read_encrypted_responses_batch) ----------
// K6p decides, per raw answer, whether it has the shape every bftkv answer has on the wire (Message.Encrypt,
// crypto_pgp.go:418-437): exactly one PKESK (new-format header, definite length, v3, RSA, a non-wildcard key id whose
// decryption the host's key loop would hand to exactly one registered private key, an MPI of at most 256 bytes ending the
// packet) followed by one SEIPD v1 (new-format header, definite or partial lengths, ending exactly at the end of the
// message, at least 40 body bytes after the version byte).  Such an answer gets c and its key slot for K6a and its
// de-chunked SEIPD body for K6b; c > n (rsa.decrypt's ErrDecryption) is decided here against the slot's public modulus.
// Every other shape goes to the host path whole: the flag, not a guess, decides.
struct KeySlot { uint64_t key_id; uint32_t slot; uint32_t pad; };
constexpr uint8_t kFrontDevice = 0, kFrontHost = 1, kFrontDecided = 2;
constexpr uint8_t kStDecryptFailed = 10, kStUnsupported = 5, kStHostPlaceholder = 6;

// One thread per answer.  raw_off: absolute offsets, raw_base: the offset of raw[0].  Per answer i (o0 = raw_off[i] -
// raw_base): out_state / out_pre (kFrontDecided: pre is the final status; kFrontHost: pre = a placeholder K0m skips),
// out_slot + out_c (n x 256, c left-padded, zero unless on the device), the de-chunked body at ct_blob + o0 spanning
// [out_ct_beg[i], out_ct_end[i]) (relative to ct_blob), out_inner_end[i] = the absolute end K0m sees when it reads the
// decrypted stream from pt_blob + 18 with the same raw_off.  Stores no secret: it reads the slots' public moduli only.
__global__ void __launch_bounds__(128)
pkesk_seipd_parse_kernel(const uint8_t* __restrict__ raw, const uint64_t* __restrict__ raw_off, const uint64_t raw_base, const uint32_t n_items,
                         const uint8_t* __restrict__ pre_in /* nullable */, const KeySlot* __restrict__ tab, const uint32_t n_tab,
                         const RsaPriv32* __restrict__ keys, uint32_t* __restrict__ out_slot, uint8_t* __restrict__ out_c,
                         uint8_t* __restrict__ ct_blob, uint64_t* __restrict__ out_ct_beg, uint64_t* __restrict__ out_ct_end,
                         uint64_t* __restrict__ out_inner_end, uint8_t* __restrict__ out_state, uint8_t* __restrict__ out_pre,
                         uint8_t* __restrict__ out_cipher) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const uint64_t o0 = raw_off[i] - raw_base, o1 = raw_off[i + 1] - raw_base;
  const uint8_t* m = raw + o0;
  const uint8_t given = pre_in != nullptr ? pre_in[i] : (uint8_t)0;
  uint8_t state = kFrontHost, pre = kStHostPlaceholder;
  uint32_t slot = n_tab ? tab[0].slot : 0u, mpi_at = 0, ml = 0;
  uint64_t L = 0;
  if (given != 0) { state = kFrontDecided; pre = given; }
  else if (o1 - o0 >= 64 && o1 - o0 <= 0x3fffffffull && n_tab) {
    const uint32_t n = (uint32_t)(o1 - o0);
    bool ok = m[0] == 0xC1;
    // ---- PKESK: definite new-format length
    uint32_t p = 1, bl = 0;
    if (ok) {
      const uint8_t o = m[1];
      if (o < 192) { bl = o; p = 2; }
      else if (o < 224) { bl = ((uint32_t)(o - 192) << 8) + m[2] + 192; p = 3; }
      else if (o == 255) { bl = ((uint32_t)m[2] << 24) | ((uint32_t)m[3] << 16) | ((uint32_t)m[4] << 8) | m[5]; p = 6; }
      else ok = false;
      ok = ok && bl <= n - p && bl >= 12;
    }
    uint64_t kid = 0;
    if (ok) {
      const uint8_t* b = m + p;
      for (int k = 1; k < 9; k++) kid = (kid << 8) | b[k];
      ml = ((((uint32_t)b[10] << 8) | b[11]) + 7) / 8;
      ok = b[0] == 3 && kid != 0 && (b[9] == 1 || b[9] == 2) && ml <= 256 && 12 + ml == bl;
      mpi_at = p + 12;
    }
    if (ok) {
      int hit = -1;
      for (uint32_t k = 0; k < n_tab; k++) if (tab[k].key_id == kid) { hit = (int)k; break; }
      ok = hit >= 0;
      if (ok) slot = tab[hit].slot;
    }
    // ---- SEIPD: the rest of the message, de-chunked behind the version byte
    uint32_t q = p + bl;
    ok = ok && q + 2 <= n && m[q] == 0xD2;
    q++;
    bool last = false, first = true;
    uint8_t* ct = ct_blob + o0;
    while (ok && !last) {
      const uint8_t o = m[q];
      uint32_t l;
      if (o < 192) { l = o; q += 1; last = true; }
      else if (o < 224) { if (q + 2 > n) { ok = false; break; } l = ((uint32_t)(o - 192) << 8) + m[q + 1] + 192; q += 2; last = true; }
      else if (o == 255) { if (q + 5 > n) { ok = false; break; } l = ((uint32_t)m[q + 1] << 24) | ((uint32_t)m[q + 2] << 16) | ((uint32_t)m[q + 3] << 8) | m[q + 4]; q += 5; last = true; }
      else { l = 1u << (o & 0x1f); q += 1; }
      if (l > n - q || (!last && q + l >= n)) { ok = false; break; }
      uint32_t k = 0;
      if (first && l > 0) { ok = m[q] == 1; k = 1; first = false; }
      for (; k < l; k++) ct[L++] = m[q + k];
      q += l;
    }
    ok = ok && !first && q == n && L >= 40;
    if (ok) {
      // c left-padded into K6a's layout, then c > n against the slot's modulus (most significant word first)
      uint8_t* c = out_c + (uint64_t)i * 256u;
      for (uint32_t k = 0; k < 256u - ml; k++) c[k] = 0;
      for (uint32_t k = 0; k < ml; k++) c[256u - ml + k] = m[mpi_at + k];
      int cmp = 0;
      for (uint32_t j = 0; j < 256u && cmp == 0; j++) {
        const uint32_t cb = j < 256u - ml ? 0u : m[mpi_at + j - (256u - ml)];
        const uint32_t nb = (__ldg(&keys[slot].n[63 - j / 4]) >> (8 * (3 - j % 4))) & 0xffu;
        cmp = cb > nb ? 1 : (cb < nb ? -1 : 0);
      }
      if (cmp > 0) { state = kFrontDecided; pre = kStDecryptFailed; }
      else { state = kFrontDevice; pre = 0; }
    }
  }
  if (state != kFrontDevice) {
    uint32_t* c = reinterpret_cast<uint32_t*>(out_c + (uint64_t)i * 256u);
    for (int k = 0; k < 64; k++) c[k] = 0u;
    L = 0;
  }
  out_slot[i] = slot;
  out_ct_beg[i] = o0;
  out_ct_end[i] = o0 + L;
  out_inner_end[i] = state == kFrontDevice ? raw_off[i] + L - 40 : raw_off[i];
  out_state[i] = state;
  out_pre[i] = pre;
  out_cipher[i] = 0;
}

// K6q, one thread per answer, between the front stage's kernels.  stage 0 (after K6a): EncryptedKey.Decrypt's outcome
// and FindKey's checks as bftq_message_decrypt_batch applies them to one PKESK — no key (invalid padding, c > n) or a
// message shorter than 3 bytes, an unknown cipher or a wrong key length: ErrDecryptionFailed; 3DES / CAST5: handed back
// (UNSUPPORTED); otherwise the AES cipher id for K6b.  stage 1 (after K6b): the quick check failed -> ErrDecryptionFailed;
// an MDC mismatch goes to the host, which knows whether ReadAll reaches the MDC.
__global__ void __launch_bounds__(256)
front_gate_kernel(const int stage, const uint32_t n_items, const uint32_t* __restrict__ info, const uint8_t* __restrict__ res,
                  uint8_t* __restrict__ state, uint8_t* __restrict__ pre, uint8_t* __restrict__ cipher_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items || state[i] != kFrontDevice) return;
  if (stage == 0) {
    const uint32_t w = info[i], st = w & 0xff, cipher = (w >> 8) & 0xff, klen = w >> 16;
    const uint32_t ks = cipher == 2 || cipher == 8 ? 24u : (cipher == 3 || cipher == 7 ? 16u : (cipher == 9 ? 32u : 0u));
    if (st != kDecOk || ks == 0 || ks != klen) { state[i] = kFrontDecided; pre[i] = kStDecryptFailed; }
    else if (cipher == 2 || cipher == 3) { state[i] = kFrontDecided; pre[i] = kStUnsupported; }
    else cipher_out[i] = (uint8_t)cipher;
  } else {
    const uint8_t r = res[i];
    if (r == 1) { state[i] = kFrontHost; pre[i] = kStHostPlaceholder; }
    else if (r != 0) { state[i] = kFrontDecided; pre[i] = kStDecryptFailed; }
  }
}

}  // namespace k6
}  // namespace bftq
