// K8 — the server half of threshold DSA and ECDSA (crypto/threshold/dsa/dsa_core.go:91-163 dsaContext.Sign) on the device.
//
//   thdsa_zq_kernel         phase 2: k_i, a_i, b_i, c_i = the sums of the decrypted shares' Y mod q, v_i = k_i a_i + b_i;
//                           phase 3: s_i = ((r Y + m) k_i + c_i) mod q.  One thread per item, q <= 256 bits.
//   thdsa_dsa_r_kernel      R_i = g^{a_i} mod p (dsa.go:27-31), p odd with exactly 1024 or 2048 bits: r32::ct_window_pow.
//   thdsa_p256_base_kernel  R_i = elliptic.Marshal(a_i G) on P-256 (ecdsa.go:31-34): p256::base_mul_ct.
//   thdsa_copy_kc_kernel    moves phase 2's (k_i, c_i) into the share's table, device to device.
//
// Every value here but q, p, g, m and r is secret: the long-term share Y, the joint shares and their sums, v_i before it
// is sent.  Constant time means: each trip count depends on public lengths only (the chunk lengths of Y, m, r and of the
// decrypted shares, |q|), every product is mont_mul_big<8, CT = true> / mont_mul<W, true> / fe_mul_ct, every modular
// addition selects its correction with a mask, and every table is read whole with masks.  Secrets stay in registers
// (no local memory: tests/test_threshold_dsa.py checks the SASS), and the host zeroes each per-call buffer after use.
//
// Arbitrary-length values (a Byzantine peer's Y >= q, a client's unreduced m and r) are reduced by Horner's rule over
// their 32-bit words, most significant first: acc = acc 2^32 + w mod q, one Montgomery product with 2^32 R mod q and one
// masked addition per word.  That needs w < q, so q must exceed 2^32 (the host refuses smaller q).
// The per-item cores are __host__ __device__ (tests/harness/thdsa_host.cpp builds them with g++).
#pragma once
#include <cstdint>
#include "lagrange.cuh"
#include "p256.cuh"
#ifdef __CUDACC__
#include "mont_r32.cuh"
#endif

namespace bftq {
namespace k8 {

// The public group of a registered share, at the head of its device allocation; the long-term Y's words follow it.
struct ThdsaGroup {
  LagrangeMod<8> q;              // q (DSA) or N (P-256)
  uint32_t q32[8];               // 2^32 R mod q: one Horner step
  uint32_t p[64];                // DSA: p, radix 2^32, little-endian (p_words of them)
  uint32_t p_r2[64];             // 2^(64 p_words) mod p
  uint32_t gm[64];               // (g mod p) R mod p
  uint32_t p0inv, p_words, q_words, pad;
};

// acc = (acc + w) mod q, acc < q, w < q
BFTQ_LAG_HD_FI void add_mod_ct(uint32_t (&acc)[8], const uint32_t (&w)[8], const LagrangeMod<8>& M) {
  uint32_t s[8], d[8], c = 0, br = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)acc[i] + w[i] + c; s[i] = (uint32_t)v; c = (uint32_t)(v >> 32); }
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)s[i] - M.m[i] - br; d[i] = (uint32_t)v; br = (uint32_t)(v >> 63); }
  const uint32_t take = 0u - (c | (br ^ 1u));
#pragma unroll
  for (int i = 0; i < 8; i++) acc[i] = (d[i] & take) | (s[i] & ~take);
}
// r = a b mod q (plain in, plain out), a < q
BFTQ_LAG_HD_FI void mul_mod_ct(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8], const LagrangeMod<8>& M) {
  uint32_t t[8];
  mont_mul_big<8, true>(t, a, b, M);
  mont_mul_big<8, true>(r, t, M.r2, M);
}
BFTQ_LAG_HD_FI uint32_t load_word(const uint32_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
// acc = (acc + the nw-word little-endian integer at w) mod q, by Horner's rule from the top word
BFTQ_LAG_HD_FI void add_reduced_ct(uint32_t (&acc)[8], const uint32_t* w, uint32_t nw, const ThdsaGroup& G) {
  uint32_t h[8], x[8];
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] = 0u;
  for (uint32_t k = nw; k-- > 0;) {
    mont_mul_big<8, true>(h, h, G.q32, G.q);
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = 0u;
    x[0] = load_word(w + k);
    add_mod_ct(h, x, G.q);
  }
  add_mod_ct(acc, h, G.q);
}

// One value of an item: a device address and a word count (public).
struct Val { uint64_t ptr; uint32_t words, pad; };

// Phase 2 (op 2): vals = 4 per decrypted share (k, a, b, c).  sec = a, k, c (8 words each), pub = v.
// Phase 3 (op 3): vals = Y, m, r; kc = k, c (16 words).  pub = s.
BFTQ_LAG_HD_FI void zq_item(const ThdsaGroup& G, uint32_t op, const Val* vals, uint32_t n_vals, const uint32_t* kc, uint32_t* sec,
                            uint32_t* pub) {
  if (op == 2) {
    uint32_t S[4][8];
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int i = 0; i < 8; i++) S[j][i] = 0u;
    for (uint32_t v = 0; v + 4 <= n_vals; v += 4) {
#pragma unroll
      for (int j = 0; j < 4; j++) add_reduced_ct(S[j], reinterpret_cast<const uint32_t*>(vals[v + j].ptr), vals[v + j].words, G);
    }
    uint32_t ka[8];
    mul_mod_ct(ka, S[0], S[1], G.q);
    add_mod_ct(ka, S[2], G.q);
#pragma unroll
    for (int i = 0; i < 8; i++) { sec[i] = S[1][i]; sec[8 + i] = S[0][i]; sec[16 + i] = S[3][i]; pub[i] = ka[i]; }
  } else {
    uint32_t y[8], m[8], r[8], k[8], c[8], t[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { y[i] = 0u; m[i] = 0u; r[i] = 0u; k[i] = load_word(kc + i); c[i] = load_word(kc + 8 + i); }
    add_reduced_ct(y, reinterpret_cast<const uint32_t*>(vals[0].ptr), vals[0].words, G);
    add_reduced_ct(m, reinterpret_cast<const uint32_t*>(vals[1].ptr), vals[1].words, G);
    add_reduced_ct(r, reinterpret_cast<const uint32_t*>(vals[2].ptr), vals[2].words, G);
    mul_mod_ct(t, r, y, G.q);
    add_mod_ct(t, m, G.q);
    mul_mod_ct(y, t, k, G.q);
    add_mod_ct(y, c, G.q);
#pragma unroll
    for (int i = 0; i < 8; i++) pub[i] = y[i];
  }
}

#ifdef __CUDACC__
// Item i: grp[i] (a share's ThdsaGroup), op[i], its values vals[val_off[i] .. val_off[i+1]), kc[i] (op 3: device address
// of its k, c).  sec: 24 words per item, pub: 8 words per item (little-endian).
__global__ void __launch_bounds__(128)
thdsa_zq_kernel(const uint64_t* __restrict__ grp, const uint8_t* __restrict__ op, const Val* __restrict__ vals,
                const uint32_t* __restrict__ val_off, const uint64_t* __restrict__ kc, const uint64_t n_items, uint32_t* __restrict__ sec,
                uint32_t* __restrict__ pub) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const ThdsaGroup& G = *reinterpret_cast<const ThdsaGroup*>(grp[i]);
  const uint32_t b = val_off[i];
  zq_item(G, op[i], vals + b, val_off[i + 1] - b, reinterpret_cast<const uint32_t*>(kc[i]), sec + i * 24, pub + i * 8);
}

constexpr int kDsaRBlock = 32;   // one warp per block, as K7: the 16-entry window table lives in shared memory

using r32::T;

// R = g^a mod p, one 4-lane group per item; a: item i's 8 words at sec + sec_item[i] * 24 (the a of thdsa_zq_kernel's
// output), q_words of them read.  out_be: n_items x 4 T W bytes, big-endian.
template <int W, int BLOCK>
__global__ void __launch_bounds__(BLOCK)
thdsa_dsa_r_kernel(const uint64_t* __restrict__ grp, const uint32_t* __restrict__ sec_item, const uint32_t* __restrict__ sec,
                   const uint64_t n_items, uint8_t* __restrict__ out_be) {
  __shared__ uint32_t tab[16][W][BLOCK];
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int grp_i = threadIdx.x / T;
  const int tid = threadIdx.x;
  constexpr int PB = 4 * T * W;
  for (uint64_t base = (uint64_t)blockIdx.x * (BLOCK / T); base < n_items; base += (uint64_t)gridDim.x * (BLOCK / T)) {
    const uint64_t item_raw = base + (uint64_t)grp_i;
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : n_items - 1;
    const ThdsaGroup* __restrict__ G = reinterpret_cast<const ThdsaGroup*>(__ldg(grp + item));
    const uint32_t* ea = sec + (uint64_t)__ldg(sec_item + item) * 24u;
    uint32_t nd[W], y[W], t[W], x[W], bm[W];
#pragma unroll
    for (int j = 0; j < W; j++) { nd[j] = __ldg(&G->p[r * W + j]); bm[j] = __ldg(&G->gm[r * W + j]); t[j] = __ldg(&G->p_r2[r * W + j]); }
    const uint32_t n0inv = __ldg(&G->p0inv);
    const uint32_t nw = __ldg(&G->q_words);
#pragma unroll
    for (int j = 0; j < W; j++) x[j] = (r == 0 && j == 0) ? 1u : 0u;
    r32::mont_mul<W, true>(y, t, x, nd, n0inv, r, gbase);        // R mod p: the Montgomery form of 1
    uint32_t nwmax = nw;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) nwmax = max(nwmax, __shfl_xor_sync(kFull, nwmax, o));
    r32::ct_window_pow<W, BLOCK>(y, bm, nd, n0inv, ea, nw, (int)(8u * nwmax), tab, r, gbase);
#pragma unroll
    for (int j = 0; j < W; j++) x[j] = (r == 0 && j == 0) ? 1u : 0u;
    r32::mont_mul<W, true>(t, y, x, nd, n0inv, r, gbase);
    r32::cond_sub<W, true>(t, nd, r, gbase);
    if (valid) store_be<W>(out_be + item_raw * PB, PB, t, r);
#pragma unroll
    for (int e = 0; e < 16; e++)                                  // no power of g left in shared memory
#pragma unroll
      for (int j = 0; j < W; j++) tab[e][j][tid] = 0u;
    __syncwarp();
  }
}

// elliptic.Marshal(a G), one thread per item; table: p256::base_table's words.  out: n_items x 65 bytes.
__global__ void __launch_bounds__(128)
thdsa_p256_base_kernel(const uint32_t* __restrict__ table, const uint32_t* __restrict__ sec_item, const uint32_t* __restrict__ sec,
                       const uint64_t n_items, uint8_t* __restrict__ out65) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const uint32_t* ea = sec + (uint64_t)sec_item[i] * 24u;
  uint32_t a[8];
#pragma unroll
  for (int k = 0; k < 8; k++) a[k] = ea[k];
  p256::base_mul_ct(out65 + i * 65u, a, table);
}

// dst[i][0..15] = k, c of phase-2 item src[i] (sec words 8..23)
__global__ void __launch_bounds__(128)
thdsa_copy_kc_kernel(const uint32_t* __restrict__ src, const uint64_t* __restrict__ dst, const uint64_t n, const uint32_t* __restrict__ sec) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t* d = reinterpret_cast<uint32_t*>(dst[i]);
  const uint32_t* s = sec + (uint64_t)src[i] * 24u + 8u;
#pragma unroll
  for (int k = 0; k < 16; k++) d[k] = s[k];
}
#endif

}  // namespace k8
}  // namespace bftq
