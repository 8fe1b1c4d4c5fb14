// Host big-number helpers for the per-key constants (up to 4096 bit, 64 x u64 limbs, little-endian).  Plain C++: the
// library includes it, and so does the CPU harness that checks the constants against Python integers.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace bftq {
namespace hostbig {

constexpr int kHL = 64;
struct UBig { uint64_t w[kHL]; };

inline bool ge(const UBig& a, const UBig& b) {
  for (int i = kHL - 1; i >= 0; i--) { if (a.w[i] != b.w[i]) return a.w[i] > b.w[i]; }
  return true;
}
inline void sub(UBig& a, const UBig& b) {
  unsigned __int128 br = 0;
  for (int i = 0; i < kHL; i++) {
    unsigned __int128 d = (unsigned __int128)a.w[i] - b.w[i] - (uint64_t)br;
    a.w[i] = (uint64_t)d;
    br = (d >> 64) & 1;
  }
}
// a = 2a mod n   (a < n on entry)
inline void dbl_mod(UBig& a, const UBig& n) {
  uint64_t top = a.w[kHL - 1] >> 63;
  for (int i = kHL - 1; i > 0; i--) a.w[i] = (a.w[i] << 1) | (a.w[i - 1] >> 63);
  a.w[0] <<= 1;
  if (top || ge(a, n)) sub(a, n);
}
// x * 2^k mod m for x < m
inline UBig shl_mod(UBig x, const UBig& m, int k) {
  for (int i = 0; i < k; i++) dbl_mod(x, m);
  return x;
}
inline int bitlen(const UBig& a) {
  for (int i = kHL - 1; i >= 0; i--) if (a.w[i]) return 64 * i + 64 - __builtin_clzll(a.w[i]);
  return 0;
}
inline void from_be(UBig& a, const uint8_t* be, size_t len) {   // len bytes big-endian, len <= 512
  memset(&a, 0, sizeof(a));
  for (size_t i = 0; i < len; i++) {
    const size_t bi = len - 1 - i;                        // little-endian byte number
    a.w[bi >> 3] |= (uint64_t)be[i] << (8 * (bi & 7));
  }
}
inline void to_words(const UBig& a, uint32_t* w, int nw) {
  for (int i = 0; i < nw; i++) w[i] = (uint32_t)(a.w[i / 2] >> (32 * (i & 1)));
}

// -n^-1 mod 2^32 / 2^64 for odd n (Montgomery's n0inv), by Newton iteration: each step doubles the correct low bits
// (3 -> 96).
inline uint32_t neg_inv32(const uint32_t n0) {
  uint32_t inv = n0;
  for (int i = 0; i < 5; i++) inv *= 2u - n0 * inv;
  return 0u - inv;
}
inline uint64_t neg_inv64(const uint64_t n0) {
  uint64_t inv = n0;
  for (int i = 0; i < 5; i++) inv *= 2u - n0 * inv;
  return 0u - inv;
}

// a * b * 2^-2048 mod n for a, b < n, n odd and below 2^2048; n0inv = -n^-1 mod 2^64.  Word-serial Montgomery product.
inline UBig mont2048(const UBig& a, const UBig& b, const UBig& n, const uint64_t n0inv) {
  constexpr int L = 32;
  uint64_t t[L + 2] = {0};
  for (int i = 0; i < L; i++) {
    unsigned __int128 c = 0;
    for (int j = 0; j < L; j++) {
      c += (unsigned __int128)a.w[j] * b.w[i] + t[j];
      t[j] = (uint64_t)c;
      c >>= 64;
    }
    c += t[L];
    t[L] = (uint64_t)c;
    t[L + 1] = (uint64_t)(c >> 64);
    const uint64_t m = t[0] * n0inv;
    c = ((unsigned __int128)m * n.w[0] + t[0]) >> 64;
    for (int j = 1; j < L; j++) {
      c += (unsigned __int128)m * n.w[j] + t[j];
      t[j - 1] = (uint64_t)c;
      c >>= 64;
    }
    c += t[L];
    t[L - 1] = (uint64_t)c;
    t[L] = t[L + 1] + (uint64_t)(c >> 64);
  }
  UBig r;
  memset(&r, 0, sizeof(r));
  for (int j = 0; j < L; j++) r.w[j] = t[j];
  if (t[L] || ge(r, n)) sub(r, n);                         // t < 2n
  return r;
}

// Constants of the radix-2^32 verification (rsa_verify_r32.cuh) for a modulus of exactly 2048 bits and 1 <= e < 2^32.
// The kernel runs the exponent's square-and-multiply chain on the PLAIN signature s, so it ends at
// Y = s^e * R^-(e-1) mod n with R = 2^2048, and c = R^-(e-1) mod n is the same chain run on s = 1.  The kernel accepts
// iff Y == EM * c (mod n), with EM = H * 2^k + L split at k = 512 (T up to 63 bytes) or k = 1024 (longer T): the top
// part H * 2^k = 00 01 FF..FF 00..00 = 2^2033 - 2^k is the same for every digest, the low part L is built per item.
//   c16 = c * 2^512,  hc16 = (2^2033 - 2^512) * c,  c32 = c * 2^1024,  hc32 = (2^2033 - 2^1024) * c   (all mod n)
struct VerifyConsts { UBig c16, hc16, c32, hc32; };
inline VerifyConsts verify_consts(const UBig& n, const uint32_t e) {
  const uint64_t n0inv = neg_inv64(n.w[0]);
  UBig one;
  memset(&one, 0, sizeof(one));
  one.w[0] = 1;
  UBig c = one;
  for (int bit = 30 - __builtin_clz(e); bit >= 0; bit--) {
    c = mont2048(c, c, n, n0inv);
    if ((e >> bit) & 1u) c = mont2048(c, one, n, n0inv);
  }
  VerifyConsts k;
  k.c16 = shl_mod(c, n, 512);
  k.c32 = shl_mod(k.c16, n, 512);
  const UBig cr = shl_mod(k.c32, n, 1024);                // c * R: a Montgomery product with it is a plain product with c
  auto top = [](int split) {                              // 2^2033 - 2^split < 2^2047 < n
    UBig h, low;
    memset(&h, 0, sizeof(h));
    memset(&low, 0, sizeof(low));
    h.w[2033 / 64] = 1ull << (2033 % 64);
    low.w[split / 64] = 1;
    sub(h, low);
    return h;
  };
  k.hc16 = mont2048(top(512), cr, n, n0inv);
  k.hc32 = mont2048(top(1024), cr, n, n0inv);
  return k;
}

}  // namespace hostbig
}  // namespace bftq
