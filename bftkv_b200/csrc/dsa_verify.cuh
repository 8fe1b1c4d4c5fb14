// K1d — DSA signature verification (OpenPGP public-key algorithm 17) on top of K5's lane-distributed
// modular exponentiation.  Follows packet.PublicKey.VerifySignature's DSA arm (x/crypto openpgp/packet/
// public_key.go: digest cut to the subgroup size) and Go crypto/dsa.Verify:
//     0 < r, s < q;  w = s^-1 mod q;  u1 = z w, u2 = r w mod q;  v = (g^u1 y^u2 mod p) mod q;  valid iff v == r
// Three stages per key (p, q, g, y):
//   dsa_prepare_kernel   thread per signature: range checks, w = s^-1 mod q, u1 / u2                 (this file)
//   modexp_kernel        2 items per signature: g^u1, y^u2 (bases broadcast)  +  modprod_kernel      (modexp.cuh)
//   dsa_finish_kernel    thread per signature: (product mod q) == r                                  (this file)
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "lagrange.cuh"
#include "limbs.cuh"
#include "modinv_big.cuh"

namespace bftq {

// r_be / s_be: 32-byte right-aligned values `stride` bytes apart, digest: n x dlen.  u_be: 2n x mlen (u1, u2 interleaved).
// status: BFTQ_ST_OK to continue, 1 when dsa.Verify already says false; a non-zero pre[] entry is copied.
template <int L>
__global__ void __launch_bounds__(128)
dsa_prepare_kernel(const LagrangeMod<L> M, const uint8_t* __restrict__ r_be, const uint8_t* __restrict__ s_be, const uint32_t stride,
                   const uint8_t* __restrict__ digest, const uint32_t dlen,
                   const uint64_t n_items, const uint8_t* __restrict__ pre, uint8_t* __restrict__ u_be, uint8_t* __restrict__ status) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  const int mlen = (int)M.mlen;
  uint8_t* up = u_be + 2 * item * (uint64_t)mlen;
  uint32_t r[L], s[L], z[L], acc[L], t[L];
  limbs::load_be<L>(r, r_be + item * stride, 32);
  limbs::load_be<L>(s, s_be + item * stride, 32);
  bool rz = true, sz = true;
#pragma unroll
  for (int l = 0; l < L; l++) { rz = rz && r[l] == 0; sz = sz && s[l] == 0; }
  uint8_t st = (pre != nullptr) ? pre[item] : 0;
  if (!st && (rz || sz || limbs::ge<L>(r, M.m) || limbs::ge<L>(s, M.m))) st = 1;
  if (st) {
    for (int b = 0; b < 2 * mlen; b++) up[b] = 0;
    status[item] = st;
    return;
  }
  const int take = (int)dlen < mlen ? (int)dlen : mlen;                 // hashBytes[:subgroupSize]
  limbs::load_be<L>(z, digest + item * (uint64_t)dlen, take);
  if (limbs::ge<L>(z, M.m)) limbs::sub<L>(z, M.m);                          // z < 2^(8 mlen) < 2q (q has exactly 8 mlen bits)
  fermat_pow<L>(acc, s, M);
  // acc = s^(q-2) R is s^-1 R only when q is prime, and q is the key holder's choice (nothing checks that it is prime).
  // (w R) s / R == 1 proves w exact (the inverse is unique); otherwise w comes from the extended GCD, and when
  // gcd(s, q) != 1 there is none: dsa.Verify's ModInverse returns nil and the signature is false.
  mont_mul_big<L>(t, acc, s, M);
  bool one = t[0] == 1u;
#pragma unroll
  for (int l = 1; l < L; l++) one = one && t[l] == 0u;
  if (!one) {
    uint32_t w[L];
    if (!modinv_big<L>(w, s, M.m)) {
      for (int b = 0; b < 2 * mlen; b++) up[b] = 0;
      status[item] = 1;
      return;
    }
    mont_mul_big<L>(acc, w, M.r2, M);                                 // w R
  }
  mont_mul_big<L>(t, z, acc, M);                                      // z (w R) / R = z w
  limbs::store_be_bytes<L>(up, mlen, t);
  mont_mul_big<L>(t, r, acc, M);
  limbs::store_be_bytes<L>(up + mlen, mlen, t);
  status[item] = 0;
}

// prod: n x nbytes (g^u1 y^u2 mod p).  status[i] (0 on entry for live items) becomes 0 / 1.
template <int L>
__global__ void __launch_bounds__(128)
dsa_finish_kernel(const LagrangeMod<L> M, const uint8_t* __restrict__ prod_be, const uint32_t nbytes, const uint8_t* __restrict__ r_be,
                  const uint32_t stride,
                  const uint64_t n_items, uint8_t* __restrict__ status) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  if (status[item] != 0) return;
  uint32_t v[L], r[L];
  limbs::reduce_be<L>(v, prod_be + item * (uint64_t)nbytes, nbytes, M.m);
  limbs::load_be<L>(r, r_be + item * stride, 32);
  bool eq = true;
#pragma unroll
  for (int l = 0; l < L; l++) eq = eq && v[l] == r[l];
  status[item] = eq ? 0 : 1;
}

}  // namespace bftq
