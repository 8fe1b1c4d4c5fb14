// K7 — the server half of threshold RSA (crypto/threshold/rsa/rsa.go:140-178 rsaContext.Sign) on the device.
//
//   thrsa_modinv_kernel         m^-1 mod N per sign request (m: the public EMSA block), binary extended GCD, one thread per
//                               request.  Variable time: m and N are public.
//   thrsa_partial_sign_kernel   c = base^|d_i| mod N per (request, key id) item, base = m^-1 when the fragment is negative
//                               (and not listed twice in the request, see below), m otherwise.
//
// Each fragment is a full exponentiation with a 2048-bit modulus whose factors the server does not know, so there is no
// CRT; splitKey doubles the exponent length at each tree level (about 4 100 bits at depth 1, 33 000 at depth 4).
// (m^|d|)^-1 = (m^-1)^|d| mod N, so a negative fragment costs the same exponentiation with the other base, chosen by a
// masked select on the fragment's sign, and no secret is ever inverted.
//
// K7 is constant time in the fragment: the trip count is 8 windows per 32-bit word of the fragment's stored length (public:
// the serialized chunk and Go's own Exp reveal it), every window reads the whole 16-entry table with masks, every product
// is mont_mul<16, CT = true>, the sign enters through a mask, and the table (powers of the base) is zeroed before the
// kernel exits.  The host groups items of equal fragment length, so the eight items of a warp share a trip count; a warp
// that still mixes lengths runs its longest, the shorter fragments reading zero windows above their top word.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "rsa_verify_r32.cuh"
#include "modexp.cuh"
#include "msg_decrypt.cuh"

namespace bftq {
namespace k7 {

// The public half of a registered share, at the head of the share's device allocation.  Radix 2^32, little-endian words.
struct ThrsaMod {
  uint32_t n[64];
  uint32_t r2[64];               // 2^4096 mod n
  uint32_t n0inv;                // -n^-1 mod 2^32
  uint32_t pad[3];
};
// A fragment in the same allocation: word 0 its sign (1 negative), then ceil(len / 4) little-endian exponent words.

constexpr int kSignBlock = 32;   // one warp per block: the 16 x 16-word table costs 1 KB of shared memory per thread

using r32::T;

// One 4-lane group per item.  Item i: mod_ptr[i] / frag_ptr[i] (device addresses inside a share's allocation), frag_words[i]
// exponent words, req[i] the sign request whose m (m_be) and m^-1 (minv_be, n_req x 256 bytes each) it uses, dup[i] = 1
// when the request lists the item's key id more than once.  out_be: n_items x 256 bytes, c < N, big-endian.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
thrsa_partial_sign_kernel(const uint64_t* __restrict__ mod_ptr, const uint64_t* __restrict__ frag_ptr, const uint32_t* __restrict__ frag_words,
                          const uint32_t* __restrict__ req, const uint8_t* __restrict__ dup, const uint8_t* __restrict__ m_be,
                          const uint8_t* __restrict__ minv_be, const uint64_t n_items, uint8_t* __restrict__ out_be) {
  constexpr int W = 16;
  __shared__ uint32_t tab[16][W][BLOCK];
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int grp = threadIdx.x / T;
  const int tid = threadIdx.x;
  for (uint64_t base = (uint64_t)blockIdx.x * (BLOCK / T); base < n_items; base += (uint64_t)gridDim.x * (BLOCK / T)) {
    const uint64_t item_raw = base + (uint64_t)grp;
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : n_items - 1;
    const ThrsaMod* __restrict__ M = reinterpret_cast<const ThrsaMod*>(__ldg(mod_ptr + item));
    const uint32_t* __restrict__ fr = reinterpret_cast<const uint32_t*>(__ldg(frag_ptr + item));
    const uint32_t nw = __ldg(frag_words + item);
    uint32_t nd[W], y[W], t[W], x[W];
#pragma unroll
    for (int j = 0; j < W; j++) nd[j] = __ldg(&M->n[r * W + j]);
    const uint32_t n0inv = __ldg(&M->n0inv);
    // base: m^-1 when the fragment is negative and its key id is listed once, m otherwise (Sign's in-place Neg)
    {
      const uint32_t inv = (__ldg(fr) & 1u) & ((uint32_t)__ldg(dup + item) ^ 1u);
      const uint32_t msk = 0u - inv;
      const uint8_t* mp = m_be + (uint64_t)__ldg(req + item) * 256u;
      const uint8_t* ip = minv_be + (uint64_t)__ldg(req + item) * 256u;
#pragma unroll
      for (int j = 0; j < W; j++) x[j] = (be_word(ip, r * W + j) & msk) | (be_word(mp, r * W + j) & ~msk);
    }
    // table: entry e = base^e R mod n (almost reduced)
#pragma unroll
    for (int j = 0; j < W; j++) t[j] = __ldg(&M->r2[r * W + j]);
    uint32_t bm[W];
    r32::mont_mul<W, true>(bm, x, t, nd, n0inv, r, gbase);
#pragma unroll
    for (int j = 0; j < W; j++) x[j] = (r == 0 && j == 0) ? 1u : 0u;
    r32::mont_mul<W, true>(y, t, x, nd, n0inv, r, gbase);        // R mod n: the Montgomery form of 1
#pragma unroll
    for (int j = 0; j < W; j++) { tab[0][j][tid] = y[j]; tab[1][j][tid] = bm[j]; t[j] = bm[j]; }
#pragma unroll 1
    for (int e = 2; e < 16; e++) {
      r32::mont_mul<W, true>(x, t, bm, nd, n0inv, r, gbase);
#pragma unroll
      for (int j = 0; j < W; j++) { tab[e][j][tid] = x[j]; t[j] = x[j]; }
    }
    // the warp's trip count: the longest fragment of its eight items (public lengths only)
    uint32_t nwmax = nw;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) nwmax = max(nwmax, __shfl_xor_sync(kFull, nwmax, o));
#pragma unroll 1
    for (int win = (int)(8u * nwmax) - 1; win >= 0; win--) {
#pragma unroll 1
      for (int k = 0; k < 4; k++) {
        r32::mont_mul<W, true>(t, y, y, nd, n0inv, r, gbase);
#pragma unroll
        for (int j = 0; j < W; j++) y[j] = t[j];
      }
      const uint32_t wi = (uint32_t)win >> 3;
      const uint32_t word = wi < nw ? __ldg(fr + 1 + wi) : 0u;
      const uint32_t w = (word >> ((win & 7) * 4)) & 15u;
#pragma unroll
      for (int j = 0; j < W; j++) x[j] = 0u;
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const uint32_t msk = 0u - (uint32_t)((uint32_t)e == w);
#pragma unroll
        for (int j = 0; j < W; j++) x[j] |= tab[e][j][tid] & msk;
      }
      r32::mont_mul<W, true>(t, y, x, nd, n0inv, r, gbase);
#pragma unroll
      for (int j = 0; j < W; j++) y[j] = t[j];
    }
#pragma unroll
    for (int j = 0; j < W; j++) x[j] = (r == 0 && j == 0) ? 1u : 0u;
    r32::mont_mul<W, true>(t, y, x, nd, n0inv, r, gbase);         // leaves Montgomery form: <= n
    k6::ct_cond_sub<W>(t, nd, r, gbase);
    if (valid) store_be<W>(out_be + item_raw * 256u, 256, t, r);
#pragma unroll
    for (int e = 0; e < 16; e++)                                  // no power of the base left in shared memory
#pragma unroll
      for (int j = 0; j < W; j++) tab[e][j][tid] = 0u;
    __syncwarp();
  }
}

// ---- m^-1 mod N (public operands) ----------------------------------------------------------------------------------
__device__ __forceinline__ bool inv_is_zero(const uint32_t* a) {
  uint32_t o = 0;
  for (int k = 0; k < 64; k++) o |= a[k];
  return o == 0;
}
__device__ __forceinline__ void inv_shr1(uint32_t* a, uint32_t top) {
  for (int k = 0; k < 63; k++) a[k] = (a[k] >> 1) | (a[k + 1] << 31);
  a[63] = (a[63] >> 1) | (top << 31);
}
__device__ __forceinline__ uint32_t inv_add(uint32_t* a, const uint32_t* b) {
  uint64_t c = 0;
  for (int k = 0; k < 64; k++) { c += (uint64_t)a[k] + b[k]; a[k] = (uint32_t)c; c >>= 32; }
  return (uint32_t)c;
}
__device__ __forceinline__ uint32_t inv_sub(uint32_t* a, const uint32_t* b) {
  uint64_t br = 0;
  for (int k = 0; k < 64; k++) { const uint64_t d = (uint64_t)a[k] - b[k] - br; a[k] = (uint32_t)d; br = (d >> 32) & 1u; }
  return (uint32_t)br;
}
__device__ __forceinline__ bool inv_ge(const uint32_t* a, const uint32_t* b) {
  for (int k = 63; k >= 0; k--) if (a[k] != b[k]) return a[k] > b[k];
  return true;
}
// x / 2 mod n (x < n, n odd)
__device__ __forceinline__ void inv_half(uint32_t* x, const uint32_t* n) {
  const uint32_t top = (x[0] & 1u) ? inv_add(x, n) : 0u;
  inv_shr1(x, top);
}

// One thread per request: out = m^-1 mod N, bad = 1 when gcd(m, N) != 1 (out zero then).  m < N (an EMSA block).
// Invariants of the loop: x1 m == u, x2 m == v (mod N).
__global__ void __launch_bounds__(128)
thrsa_modinv_kernel(const uint64_t* __restrict__ mod_ptr, const uint8_t* __restrict__ m_be, const uint64_t n_req, uint8_t* __restrict__ out_be,
                    uint8_t* __restrict__ bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_req) return;
  const ThrsaMod* M = reinterpret_cast<const ThrsaMod*>(mod_ptr[i]);
  uint32_t n[64], u[64], v[64], x1[64], x2[64];
  for (int k = 0; k < 64; k++) {
    n[k] = M->n[k]; v[k] = n[k]; u[k] = be_word(m_be + i * 256u, k);
    x1[k] = k == 0 ? 1u : 0u; x2[k] = 0u;
  }
  bool ok = !inv_is_zero(u);
  while (ok) {
    while (!(u[0] & 1u)) { inv_shr1(u, 0u); inv_half(x1, n); }
    while (!(v[0] & 1u)) { inv_shr1(v, 0u); inv_half(x2, n); }
    if (inv_ge(u, v)) {
      inv_sub(u, v);
      if (inv_sub(x1, x2)) inv_add(x1, n);
      if (inv_is_zero(u)) break;                 // gcd = v
    } else {
      inv_sub(v, u);
      if (inv_sub(x2, x1)) inv_add(x2, n);
    }
  }
  if (ok) {
    uint32_t one = v[0] == 1u;
    for (int k = 1; k < 64; k++) one &= v[k] == 0u;
    ok = one != 0;
  }
  uint8_t* o = out_be + i * 256u;
  for (int k = 0; k < 64; k++) {
    const uint32_t w = ok ? x2[k] : 0u;
    const int off = 256 - 4 - 4 * k;
    o[off] = (uint8_t)(w >> 24); o[off + 1] = (uint8_t)(w >> 16); o[off + 2] = (uint8_t)(w >> 8); o[off + 3] = (uint8_t)w;
  }
  bad[i] = ok ? 0 : 1;
}

}  // namespace k7
}  // namespace bftq
