// a^-1 mod m for an odd modulus m of L 32-bit limbs, on the limb library (limbs.cuh).  Variable time: the operands are
// public (DSA's s and a peer's subgroup order q in dsa_prepare_kernel, the EMSA block m and the modulus N in
// thrsa_modinv_kernel).  __host__ __device__, like limbs.cuh, so that tests/harness/modinv_host.cpp checks the same code.
#pragma once
#include <cstdint>
#include "limbs.cuh"

namespace bftq {

// inv = a^-1 mod m for 0 <= a < m, m odd, by the binary extended GCD.  Works for any odd m, prime or not; returns false
// (inv zero) when gcd(a, m) != 1, which is when Go's big.Int.ModInverse returns nil.
// Invariants of the loop: x1 a == u, x2 a == v (mod m).
template <int L>
BFTQ_LIMBS_HD bool modinv_big(uint32_t (&inv)[L], const uint32_t (&a)[L], const uint32_t (&m)[L]) {
  uint32_t u[L], v[L], x1[L], x2[L];
  for (int k = 0; k < L; k++) { u[k] = a[k]; v[k] = m[k]; x1[k] = k == 0 ? 1u : 0u; x2[k] = 0u; inv[k] = 0u; }
  if (limbs::is_zero<L>(u)) return false;
  while (true) {
    while (!(u[0] & 1u)) { limbs::shr1<L>(u, 0u); limbs::half<L>(x1, m); }
    while (!(v[0] & 1u)) { limbs::shr1<L>(v, 0u); limbs::half<L>(x2, m); }
    if (limbs::ge<L>(u, v)) {
      limbs::sub<L>(u, v);
      if (limbs::sub<L>(x1, x2)) limbs::add<L>(x1, m);
      if (limbs::is_zero<L>(u)) break;                 // gcd = v
    } else {
      limbs::sub<L>(v, u);
      if (limbs::sub<L>(x2, x1)) limbs::add<L>(x2, m);
    }
  }
  bool one = v[0] == 1u;
  for (int k = 1; k < L; k++) one = one && v[k] == 0u;
  if (!one) return false;
  for (int k = 0; k < L; k++) inv[k] = x2[k];
  return true;
}

}  // namespace bftq
