// K3 — batched Shamir / Lagrange share-combine in Z_m for sm_90a.
//
// Replaces crypto/sss/sss.go:81-107 (SSSProcess.calculateSecret + Lagrange) and
// crypto/threshold/dsa/dsa_core.go:389-403 (calculateS):
//     lambda_i = prod_{j: x_j != x_i} x_j * (x_j - x_i)^-1  mod m,     S = sum_i lambda_i * y_i  mod m
// The reference builds numerator and denominator as unreduced integers and calls big.Int.ModInverse
// once; mathematically that is the product of the per-factor inverses used here, so results are
// bit-identical whenever the reference's inverse exists (when it does not, Go dereferences nil and
// panics; here the item gets status BFTQ_ST_MALFORMED).
//
// One thread per combine, L 32-bit limbs (L = 8 covers the 160-bit DSA q and the P-256 order,
// L = 64 the 2048-bit modulus of sss_test.go).  Every factor (x_j - x_i) is a small integer; products of
// them that still fit 32 bits are inverted together: the inverse of d is  (1 + m*t)/d  with  t = (-m^-1) mod d
// from a 64-bit extended Euclid — no big-number inversion at all.  Products run in Montgomery form (m must be odd); y_i may be >= m (the
// reference's big.Int arithmetic reduces it implicitly) as long as it fits mlen bytes.  HBM-bound: k*(4+mlen)+mlen
// bytes per combine.
// The per-combine code is __host__ __device__ (tests/harness/lagrange_host.cpp builds it with g++); only the kernel
// wrapper needs nvcc.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>
#ifdef __CUDACC__
#include <cuda_runtime.h>
#define BFTQ_LAG_HD __host__ __device__
#define BFTQ_LAG_HD_FI __host__ __device__ __forceinline__
#else
#define BFTQ_LAG_HD
#define BFTQ_LAG_HD_FI inline
#endif
#include "limbs.cuh"
#include "bignum_host.hpp"

namespace bftq {

template <int L>
struct LagrangeMod {
  uint32_t m[L];
  uint32_t r1[L];       // R mod m   (Montgomery one)
  uint32_t r2[L];       // R^2 mod m (plain -> Montgomery form)
  uint32_t m0inv;       // -m^-1 mod 2^32
  uint32_t mlen;        // bytes of m (output width)
};

// r = a*b*R^-1 mod m, fully reduced.  a < m; b < R.
// CT: no branch on the data (K8, thdsa_sign.cuh): b's limbs are picked by a masked scan over a public index, so b may
// live in registers without a local-memory copy, and the final subtraction is always computed and selected with a mask.
template <int L, bool CT = false>
BFTQ_LAG_HD void mont_mul_big(uint32_t* r, const uint32_t* a, const uint32_t* b, const LagrangeMod<L>& M) {
  uint32_t t[L + 2];
#pragma unroll
  for (int i = 0; i < L + 2; i++) t[i] = 0;
#pragma unroll 1
  for (int i = 0; i < L; i++) {
    uint64_t c = 0;
    uint32_t bi;
    if (CT) {
      bi = 0u;
#pragma unroll
      for (int k = 0; k < L; k++) bi |= b[k] & (0u - (uint32_t)(k == i));
    } else {
      bi = b[i];
    }
#pragma unroll
    for (int j = 0; j < L; j++) {
      const uint64_t v = (uint64_t)a[j] * bi + t[j] + c;
      t[j] = (uint32_t)v;
      c = v >> 32;
    }
    uint64_t v = (uint64_t)t[L] + c;
    t[L] = (uint32_t)v;
    t[L + 1] = (uint32_t)(v >> 32);
    const uint32_t q = t[0] * M.m0inv;
    v = (uint64_t)q * M.m[0] + t[0];
    c = v >> 32;
#pragma unroll
    for (int j = 1; j < L; j++) {
      v = (uint64_t)q * M.m[j] + t[j] + c;
      t[j - 1] = (uint32_t)v;
      c = v >> 32;
    }
    v = (uint64_t)t[L] + c;
    t[L - 1] = (uint32_t)v;
    t[L] = t[L + 1] + (uint32_t)(v >> 32);
  }
  if (CT) {
    uint32_t d[L];
    uint32_t br = 0;
#pragma unroll
    for (int i = 0; i < L; i++) { const uint64_t x = (uint64_t)t[i] - M.m[i] - br; d[i] = (uint32_t)x; br = (uint32_t)(x >> 63); }
    const uint32_t take = 0u - ((uint32_t)(t[L] != 0u) | (br ^ 1u));      // t >= m (t < 2m)
#pragma unroll
    for (int i = 0; i < L; i++) t[i] = (d[i] & take) | (t[i] & ~take);
  } else if (t[L] != 0 || limbs::ge<L>(t, M.m)) {
    limbs::sub<L>(t, M.m);
  }
#pragma unroll
  for (int i = 0; i < L; i++) r[i] = t[i];
}

// acc = v^(m-2) R mod m (Montgomery form; v^-1 R when m is prime), v < m plain.  Square-and-multiply over all 32 L bits.
template <int L>
BFTQ_LAG_HD_FI void fermat_pow(uint32_t (&acc)[L], const uint32_t (&v)[L], const LagrangeMod<L>& M) {
  uint32_t e[L], vm[L];
#pragma unroll
  for (int l = 0; l < L; l++) e[l] = M.m[l];
  uint32_t br = 2;                                                  // e = m - 2
#pragma unroll
  for (int l = 0; l < L; l++) { const uint64_t d = (uint64_t)e[l] - br; e[l] = (uint32_t)d; br = (uint32_t)(d >> 63); }
  mont_mul_big<L>(vm, v, M.r2, M);                                  // v R
#pragma unroll
  for (int l = 0; l < L; l++) acc[l] = M.r1[l];                     // 1 R
  for (int bit = 32 * L - 1; bit >= 0; bit--) {
    mont_mul_big<L>(acc, acc, acc, M);
    if ((e[bit >> 5] >> (bit & 31)) & 1u) mont_mul_big<L>(acc, acc, vm, M);
  }
}

// inverse of the small integer d (1 <= d < 2^32) modulo m, as a plain big number.  false if gcd != 1.
template <int L>
BFTQ_LAG_HD bool small_inverse(uint32_t* inv, uint32_t d, const LagrangeMod<L>& M) {
  if (d == 1) {
#pragma unroll
    for (int i = 0; i < L; i++) inv[i] = 0;
    inv[0] = 1;
    // 1 mod m (m > 1 is checked on the host)
    return true;
  }
  uint64_t rem = 0;
#pragma unroll
  for (int i = L - 1; i >= 0; i--) rem = ((rem << 32) | M.m[i]) % d;
  // extended Euclid on (rem, d): find u with rem*u == 1 mod d
  int64_t a0 = (int64_t)rem, a1 = (int64_t)d, u0 = 1, u1 = 0;
  while (a1 != 0) {
    const int64_t qq = a0 / a1;
    int64_t tmp = a0 - qq * a1; a0 = a1; a1 = tmp;
    tmp = u0 - qq * u1; u0 = u1; u1 = tmp;
  }
  if (a0 != 1) return false;
  int64_t u = u0 % (int64_t)d;
  if (u < 0) u += d;                                   // u = m^-1 mod d
  const uint32_t t = (uint32_t)(((int64_t)d - u) % (int64_t)d);     // (-m^-1) mod d
  // P = m*t + 1 (L+1 limbs), inv = P / d exactly
  uint32_t P[L + 1];
  uint64_t c = 1;
#pragma unroll
  for (int i = 0; i < L; i++) {
    const uint64_t v = (uint64_t)M.m[i] * t + c;
    P[i] = (uint32_t)v;
    c = v >> 32;
  }
  P[L] = (uint32_t)c;
  uint64_t r = 0;
#pragma unroll
  for (int i = L; i >= 0; i--) {
    const uint64_t cur = (r << 32) | P[i];
    const uint64_t qd = cur / d;
    r = cur - qd * d;
    if (i < L) inv[i] = (uint32_t)qd;
  }
  return true;
}

// mag mod m as a plain big number (mag < 2^32).
template <int L>
BFTQ_LAG_HD void mag_to_big(uint32_t* out, const uint32_t mag, const LagrangeMod<L>& M) {
#pragma unroll
  for (int i = 0; i < L; i++) out[i] = 0;
  out[0] = mag;
  bool tiny = true;                       // m may be smaller than the chunk
#pragma unroll
  for (int i = 1; i < L; i++) tiny = tiny && (M.m[i] == 0);
  if (tiny) out[0] %= M.m[0];
}

// One combine: item `item` of the batch (k abscissae at xs + item k, k shares of mlen bytes at ys_be + item k mlen) ->
// out_be + item mlen, out_status[item] (0, or 3 when a difference has no inverse mod m) and, when out_lambda is not
// null, the k lambda_i (plain, mlen bytes each) at out_lambda + item k mlen.
template <int L>
BFTQ_LAG_HD_FI void lagrange_item(const LagrangeMod<L>& M, const uint32_t k, const int32_t* __restrict__ xs,
                                  const uint8_t* __restrict__ ys_be, const uint64_t item, uint8_t* __restrict__ out_be,
                                  uint8_t* __restrict__ out_status, uint8_t* __restrict__ out_lambda) {
  const int32_t* x = xs + item * k;
  const uint8_t* yb = ys_be + item * (uint64_t)k * M.mlen;
  uint32_t S[L];                       // running sum (plain)
#pragma unroll
  for (int i = 0; i < L; i++) S[i] = 0;
  bool okay = true;
  for (uint32_t i = 0; i < k; i++) {
    const int32_t xi = limbs::load_i32(x + i);
    uint32_t lam[L];
#pragma unroll
    for (int l = 0; l < L; l++) lam[l] = M.r1[l];               // 1 in Montgomery form
    // Factors are gathered into 32-bit chunks before they touch a big number: numerator chunks |x_j| * |x_j'| * ... and
    // denominator chunks |x_j - x_i| * ..., each flushed (one small-integer inverse / one lift to Montgomery form, one
    // product into lambda) only when the next factor would overflow 2^32.  With node indices as abscissae (1..n, k = 10)
    // that is one or two inversions and about eight Montgomery products per lambda instead of nine and thirty-six.  The
    // value is the same residue: gcd(ab, m) = 1 iff gcd(a, m) = gcd(b, m) = 1, so the "no inverse" decision is too.
    uint32_t numc = 1u, denc = 1u;
    bool neg = false;
    for (uint32_t j = 0; j <= k; j++) {
      const bool last = j == k;
      uint32_t ax = 1u, ad32 = 1u;
      if (!last) {
        const int32_t xj = limbs::load_i32(x + j);
        if (xj == xi) continue;                                  // sss.go:100-102 (also skips duplicates)
        const int64_t d = (int64_t)xj - (int64_t)xi;
        const uint64_t ad = (uint64_t)(d < 0 ? -d : d);
        if (ad >> 32) { okay = false; continue; }
        neg ^= (d < 0) != (xj < 0);
        ax = (uint32_t)(xj < 0 ? -(int64_t)xj : (int64_t)xj);
        ad32 = (uint32_t)ad;
      }
      const uint64_t pn = (uint64_t)numc * ax, pd = (uint64_t)denc * ad32;
      if (last || (pn >> 32)) {                                  // flush the numerator chunk
        if (numc != 1u) {
          uint32_t tmp[L];
          mag_to_big<L>(tmp, numc, M);
          mont_mul_big<L>(tmp, tmp, M.r2, M);
          mont_mul_big<L>(lam, lam, tmp, M);
        }
        numc = ax;
      } else numc = (uint32_t)pn;
      if (last || (pd >> 32)) {                                  // flush the denominator chunk
        if (denc != 1u) {
          uint32_t tmp[L];
          if (!small_inverse<L>(tmp, denc, M)) okay = false;
          else {
            mont_mul_big<L>(tmp, tmp, M.r2, M);
            mont_mul_big<L>(lam, lam, tmp, M);
          }
        }
        denc = ad32;
      } else denc = (uint32_t)pd;
    }
    if (neg) {                                                   // an odd number of negative factors: lambda -> m - lambda
      bool zero = true;
#pragma unroll
      for (int l = 0; l < L; l++) zero = zero && (lam[l] == 0u);
      if (!zero) {
        uint32_t t2[L];
#pragma unroll
        for (int l = 0; l < L; l++) t2[l] = M.m[l];
        limbs::sub<L>(t2, lam);
#pragma unroll
        for (int l = 0; l < L; l++) lam[l] = t2[l];
      }
    }
    if (out_lambda != nullptr) {                                 // lambda_i itself (plain), k x mlen bytes per item
      uint32_t one[L], lp[L];
#pragma unroll
      for (int l = 0; l < L; l++) one[l] = 0;
      one[0] = 1;
      mont_mul_big<L>(lp, lam, one, M);
      uint8_t* lb = out_lambda + (item * k + i) * (uint64_t)M.mlen;
      for (uint32_t p = 0; p < M.mlen; p++) {
        const uint32_t bi = M.mlen - 1 - p;
        lb[p] = okay ? (uint8_t)(lp[bi >> 2] >> (8 * (bi & 3))) : (uint8_t)0;
      }
    }
    // y_i (big-endian, mlen bytes) -> limbs
    uint32_t y[L];
#pragma unroll
    for (int l = 0; l < L; l++) {
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const int pos = (int)M.mlen - 1 - (4 * l + b);
        if (pos >= 0) v |= limbs::load_byte(yb + (uint64_t)i * M.mlen + pos) << (8 * b);
      }
      y[l] = v;
    }
    mont_mul_big<L>(lam, lam, y, M);                             // Montgomery x plain = plain lambda*y mod m
    // S += lam mod m
    uint64_t c = 0;
#pragma unroll
    for (int l = 0; l < L; l++) {
      const uint64_t v = (uint64_t)S[l] + lam[l] + c;
      S[l] = (uint32_t)v;
      c = v >> 32;
    }
    if (c || limbs::ge<L>(S, M.m)) limbs::sub<L>(S, M.m);
  }
  uint8_t* ob = out_be + item * (uint64_t)M.mlen;
  for (uint32_t p = 0; p < M.mlen; p++) {
    const uint32_t byte_index = M.mlen - 1 - p;                  // little-endian byte number
    ob[p] = okay ? (uint8_t)(S[byte_index >> 2] >> (8 * (byte_index & 3))) : (uint8_t)0;
  }
  out_status[item] = okay ? 0 : 3;
}

#ifdef __CUDACC__
template <int L>
__global__ void __launch_bounds__(128)
lagrange_combine_kernel(const LagrangeMod<L> M, const uint32_t k, const int32_t* __restrict__ xs,
                        const uint8_t* __restrict__ ys_be, const uint64_t n_items, uint8_t* __restrict__ out_be,
                        uint8_t* __restrict__ out_status, uint8_t* __restrict__ out_lambda) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  lagrange_item<L>(M, k, xs, ys_be, item, out_be, out_status, out_lambda);
}
#endif

// Host: the LagrangeMod of the mlen-byte big-endian modulus m_be (odd, > 1, mlen <= 4 L).
template <int L>
void make_lagrange_mod(const uint8_t* m_be, uint32_t mlen, LagrangeMod<L>& M) {
  memset(&M, 0, sizeof(M));
  for (uint32_t i = 0; i < mlen; i++) {
    const uint32_t bi = mlen - 1 - i;          // little-endian byte number
    M.m[bi >> 2] |= (uint32_t)m_be[i] << (8 * (bi & 3));
  }
  M.mlen = mlen;
  M.m0inv = hostbig::neg_inv32(M.m[0]);
  // R mod m and R^2 mod m by shift-and-subtract from 1
  std::vector<uint32_t> r(L + 1, 0u);
  r[0] = 1;
  auto ge_m = [&](const std::vector<uint32_t>& v) {
    if (v[L]) return true;
    for (int i = L - 1; i >= 0; i--) if (v[i] != M.m[i]) return v[i] > M.m[i];
    return true;
  };
  auto sub_m = [&](std::vector<uint32_t>& v) {
    uint64_t br = 0;
    for (int i = 0; i < L; i++) { uint64_t d = (uint64_t)v[i] - M.m[i] - br; v[i] = (uint32_t)d; br = (d >> 63) & 1; }
    v[L] -= (uint32_t)br;
  };
  while (ge_m(r)) sub_m(r);
  for (int pass = 0; pass < 2; pass++) {
    for (int b = 0; b < 32 * L; b++) {
      for (int i = L; i > 0; i--) r[i] = (r[i] << 1) | (r[i - 1] >> 31);
      r[0] <<= 1;
      if (ge_m(r)) sub_m(r);
    }
    for (int i = 0; i < L; i++) (pass == 0 ? M.r1 : M.r2)[i] = r[i];
  }
}

}  // namespace bftq
