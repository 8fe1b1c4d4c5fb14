// a^-1 mod m for an odd modulus m of L 32-bit limbs (little-endian), by the binary extended GCD.  Variable time: the
// operands here are public (DSA's s and a peer's subgroup order q), as in thrsa_modinv_kernel.  Works for any odd m,
// prime or not; returns false when gcd(a, m) != 1, which is when Go's big.Int.ModInverse returns nil.
// __host__ __device__ so that the host build (tests/harness/modinv_host.cpp) checks the same code.
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define BFTQ_MI_HD __host__ __device__ inline
#else
#define BFTQ_MI_HD inline
#endif

namespace bftq {

template <int L>
BFTQ_MI_HD bool mi_is_zero(const uint32_t (&a)[L]) { uint32_t o = 0; for (int k = 0; k < L; k++) o |= a[k]; return o == 0; }
template <int L>
BFTQ_MI_HD bool mi_ge(const uint32_t (&a)[L], const uint32_t (&b)[L]) {
  for (int k = L - 1; k >= 0; k--) if (a[k] != b[k]) return a[k] > b[k];
  return true;
}
template <int L>
BFTQ_MI_HD uint32_t mi_add(uint32_t (&a)[L], const uint32_t (&b)[L]) {
  uint64_t c = 0;
  for (int k = 0; k < L; k++) { c += (uint64_t)a[k] + b[k]; a[k] = (uint32_t)c; c >>= 32; }
  return (uint32_t)c;
}
template <int L>
BFTQ_MI_HD uint32_t mi_sub(uint32_t (&a)[L], const uint32_t (&b)[L]) {
  uint64_t br = 0;
  for (int k = 0; k < L; k++) { const uint64_t d = (uint64_t)a[k] - b[k] - br; a[k] = (uint32_t)d; br = (d >> 32) & 1u; }
  return (uint32_t)br;
}
template <int L>
BFTQ_MI_HD void mi_shr1(uint32_t (&a)[L], uint32_t top) {
  for (int k = 0; k < L - 1; k++) a[k] = (a[k] >> 1) | (a[k + 1] << 31);
  a[L - 1] = (a[L - 1] >> 1) | (top << 31);
}
// x / 2 mod m (x < m, m odd)
template <int L>
BFTQ_MI_HD void mi_half(uint32_t (&x)[L], const uint32_t (&m)[L]) {
  const uint32_t top = (x[0] & 1u) ? mi_add<L>(x, m) : 0u;
  mi_shr1<L>(x, top);
}

// inv = a^-1 mod m for 0 <= a < m, m odd.  Invariants of the loop: x1 a == u, x2 a == v (mod m).
template <int L>
BFTQ_MI_HD bool modinv_big(uint32_t (&inv)[L], const uint32_t (&a)[L], const uint32_t (&m)[L]) {
  uint32_t u[L], v[L], x1[L], x2[L];
  for (int k = 0; k < L; k++) { u[k] = a[k]; v[k] = m[k]; x1[k] = k == 0 ? 1u : 0u; x2[k] = 0u; inv[k] = 0u; }
  if (mi_is_zero<L>(u)) return false;
  while (true) {
    while (!(u[0] & 1u)) { mi_shr1<L>(u, 0u); mi_half<L>(x1, m); }
    while (!(v[0] & 1u)) { mi_shr1<L>(v, 0u); mi_half<L>(x2, m); }
    if (mi_ge<L>(u, v)) {
      mi_sub<L>(u, v);
      if (mi_sub<L>(x1, x2)) mi_add<L>(x1, m);
      if (mi_is_zero<L>(u)) break;                 // gcd = v
    } else {
      mi_sub<L>(v, u);
      if (mi_sub<L>(x2, x1)) mi_add<L>(x2, m);
    }
  }
  bool one = v[0] == 1u;
  for (int k = 1; k < L; k++) one = one && v[k] == 0u;
  if (!one) return false;
  for (int k = 0; k < L; k++) inv[k] = x2[k];
  return true;
}

}  // namespace bftq
