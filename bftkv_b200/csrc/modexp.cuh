// K5 — batched modular exponentiation / product with a shared odd modulus, for the
// "Lagrange in the exponent" steps of the threshold protocols (SURVEY §8f rank 4):
//   crypto/auth/auth.go:386-399            calculateSharedSecret:  prod_i Y_i^lambda_i mod p
//   crypto/threshold/dsa/dsa.go:33-52      CalculateR: (prod_i R_i^lambda_i mod p)^((sum v_i lambda_i)^-1 mod q) mod p mod q
// Reuses K1's lane-distributed radix-2^32 Montgomery product (mont_r32.cuh): a number is
// owned by 4 lanes x W limbs (W = 8: 1024-bit p of DSA L1024; W = 16: the 2048-bit safe prime of
// crypto/auth).  The modulus must have exactly 128*W bits.  Integer-multiplier bound like K1:
// one |q|-bit exponentiation = ~1.5 |q| Montgomery products of 2 (4W)^2 MACs.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "mont_r32.cuh"
#include "lagrange.cuh"

namespace bftq {

template <int W>
struct ModDev {
  uint32_t n[4 * W];
  uint32_t r2[4 * W];          // R^2 mod n, R = 2^(128 W)
  uint32_t n0inv;              // -n^-1 mod 2^32
  uint32_t nbytes;             // 16 W
};

// out[i] = base[i]^exp[i] mod n.  base: N x nbytes (values >= n are reduced, as big.Int.Exp does),
// exp: N x elen bytes big-endian.  One 4-lane group per item.
template <int W, int BLOCK>
__global__ void __launch_bounds__(BLOCK)
modexp_kernel(const ModDev<W> M, const uint8_t* __restrict__ base_be, const uint8_t* __restrict__ exp_be, const uint32_t elen,
              const uint64_t n_items, uint8_t* __restrict__ out_be, const uint32_t n_bases = 0) {
  using namespace r32;
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const uint64_t warp_global = (uint64_t)blockIdx.x * (BLOCK / 32) + (threadIdx.x >> 5);
  const uint64_t warps_total = (uint64_t)gridDim.x * (BLOCK / 32);
  const int nbytes = (int)M.nbytes;
  uint32_t nd[W];
#pragma unroll
  for (int j = 0; j < W; j++) nd[j] = M.n[r * W + j];
  for (uint64_t wbase = warp_global * (32 / T); wbase < n_items; wbase += warps_total * (32 / T)) {
    const uint64_t item_raw = wbase + (uint64_t)(lane / T);
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : (n_items - 1);
    const uint8_t* bp = base_be + (n_bases ? item % n_bases : item) * (uint64_t)nbytes;   // n_bases > 0: shared bases, round robin
    const uint8_t* ep = exp_be + item * (uint64_t)elen;
    uint32_t xm[W], y[W], t[W];
    {
      uint32_t x[W], r2[W];
#pragma unroll
      for (int j = 0; j < W; j++) { x[j] = be_word_dyn(bp, nbytes, r * W + j); r2[j] = M.r2[r * W + j]; }
      r32::mont_mul<W>(xm, x, r2, nd, M.n0inv, r, gbase);               // base * R mod n (almost reduced)
    }
    // highest set bit of the exponent (-1 when the exponent is zero)
    int top = -1;
    for (int b = 0; b < (int)elen; b++) {
      const uint32_t by = __ldg(ep + b);
      if (by) { top = 8 * ((int)elen - 1 - b) + (31 - __clz(by)); break; }
    }
    int topmax = top;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) topmax = max(topmax, __shfl_xor_sync(kFull, topmax, o));
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = xm[j];                       // value after the top bit
#pragma unroll 1
    for (int bit = topmax - 1; bit >= 0; bit--) {
      const bool active = bit < top;
      r32::mont_mul<W>(t, y, y, nd, M.n0inv, r, gbase);
      if (active) {
#pragma unroll
        for (int j = 0; j < W; j++) y[j] = t[j];
      }
      const bool mul = active && ((__ldg(ep + ((int)elen - 1 - (bit >> 3))) >> (bit & 7)) & 1u);
      if (__any_sync(kFull, mul)) {
        r32::mont_mul<W>(t, y, xm, nd, M.n0inv, r, gbase);
        if (mul) {
#pragma unroll
          for (int j = 0; j < W; j++) y[j] = t[j];
        }
      }
    }
    {
      uint32_t one[W];
#pragma unroll
      for (int j = 0; j < W; j++) one[j] = (r == 0 && j == 0) ? 1u : 0u;
      r32::mont_mul<W>(t, y, one, nd, M.n0inv, r, gbase);               // leave Montgomery form
      if (top < 0) {                                               // x^0 = 1
#pragma unroll
        for (int j = 0; j < W; j++) t[j] = one[j];
      }
    }
    r32::cond_sub<W>(t, nd, r, gbase);
    if (valid) store_be<W>(out_be + item_raw * (uint64_t)nbytes, nbytes, t, r);
  }
}

// out[i] = prod_{j<k} vals[i*k + j] mod n.
template <int W, int BLOCK>
__global__ void __launch_bounds__(BLOCK)
modprod_kernel(const ModDev<W> M, const uint8_t* __restrict__ vals_be, const uint32_t k, const uint64_t n_items, uint8_t* __restrict__ out_be) {
  using namespace r32;
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const uint64_t warp_global = (uint64_t)blockIdx.x * (BLOCK / 32) + (threadIdx.x >> 5);
  const uint64_t warps_total = (uint64_t)gridDim.x * (BLOCK / 32);
  const int nbytes = (int)M.nbytes;
  uint32_t nd[W], r2[W];
#pragma unroll
  for (int j = 0; j < W; j++) { nd[j] = M.n[r * W + j]; r2[j] = M.r2[r * W + j]; }
  for (uint64_t wbase = warp_global * (32 / T); wbase < n_items; wbase += warps_total * (32 / T)) {
    const uint64_t item_raw = wbase + (uint64_t)(lane / T);
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : (n_items - 1);
    uint32_t acc[W], t[W], v[W];
#pragma unroll
    for (int j = 0; j < W; j++) acc[j] = be_word_dyn(vals_be + (item * k) * (uint64_t)nbytes, nbytes, r * W + j);
#pragma unroll 1
    for (uint32_t i = 1; i < k; i++) {
#pragma unroll
      for (int j = 0; j < W; j++) v[j] = be_word_dyn(vals_be + (item * k + i) * (uint64_t)nbytes, nbytes, r * W + j);
      r32::mont_mul<W>(t, acc, r2, nd, M.n0inv, r, gbase);              // acc * R
      r32::mont_mul<W>(acc, t, v, nd, M.n0inv, r, gbase);               // (acc R) * v / R = acc * v
    }
    r32::cond_sub<W>(acc, nd, r, gbase);
    r32::cond_sub<W>(acc, nd, r, gbase);                                // k == 1: the input itself may be >= n
    if (valid) store_be<W>(out_be + item_raw * (uint64_t)nbytes, nbytes, acc, r);
  }
}

// Thread-per-item helpers in Z_q (q odd prime, up to 256 bit; L limbs as in lagrange.cuh) -----------
// out = v^(q-2) mod q  (Fermat inverse; v == 0 mod q -> status 3, like big.Int.ModInverse returning nil)
template <int L>
__global__ void __launch_bounds__(128)
fermat_inverse_kernel(const LagrangeMod<L> M, const uint8_t* __restrict__ v_be, const uint64_t n_items, uint8_t* __restrict__ out_be,
                      uint8_t* __restrict__ status) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  uint32_t v[L], acc[L];
  limbs::load_be<L>(v, v_be + item * (uint64_t)M.mlen, (int)M.mlen);
  while (limbs::ge<L>(v, M.m)) limbs::sub<L>(v, M.m);               // v < 2^(8 mlen) <= 256 q: bounded loop
  const bool zero = limbs::is_zero<L>(v);
  fermat_pow<L>(acc, v, M);
  uint32_t one[L];
#pragma unroll
  for (int l = 0; l < L; l++) one[l] = 0;
  one[0] = 1;
  mont_mul_big<L>(acc, acc, one, M);
  limbs::store_be_bytes<L>(out_be + item * (uint64_t)M.mlen, (int)M.mlen, acc);
  if (zero && status) status[item] = 3;
}

// out = big mod q, big: nbytes big-endian (<= 512), out: mlen bytes.  Bitwise shift-subtract.
template <int L>
__global__ void __launch_bounds__(128)
mod_small_kernel(const LagrangeMod<L> M, const uint8_t* __restrict__ big_be, const uint32_t nbytes, const uint64_t n_items,
                 uint8_t* __restrict__ out_be) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  uint32_t r[L];
  limbs::reduce_be<L>(r, big_be + item * (uint64_t)nbytes, nbytes, M.m);
  limbs::store_be_bytes<L>(out_be + item * (uint64_t)M.mlen, (int)M.mlen, r);
}

}  // namespace bftq
