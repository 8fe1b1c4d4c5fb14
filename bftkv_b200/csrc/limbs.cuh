// Per-thread big numbers of L 32-bit limbs (little-endian), for the thread-per-item kernels: K3's sums (lagrange.cuh),
// K5's Z_q helpers (modexp.cuh), K1d's final reduction (dsa_verify.cuh) and the extended GCD (modinv_big.cuh).
// Variable time throughout: every operand these kernels pass is public.
// __host__ __device__ so that the host build (tests/harness/modinv_host.cpp) checks the same code the kernels run.
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define BFTQ_LIMBS_HD __host__ __device__ __forceinline__
#else
#define BFTQ_LIMBS_HD inline
#endif

namespace bftq {
namespace limbs {

template <int L>
BFTQ_LIMBS_HD bool is_zero(const uint32_t* a) { uint32_t o = 0; for (int k = 0; k < L; k++) o |= a[k]; return o == 0; }
// a >= b ?
template <int L>
BFTQ_LIMBS_HD bool ge(const uint32_t* a, const uint32_t* b) {
#pragma unroll
  for (int i = L - 1; i >= 0; i--) {
    if (a[i] != b[i]) return a[i] > b[i];
  }
  return true;
}
// a -= b mod 2^(32 L), returns the borrow out (0/1).
template <int L>
BFTQ_LIMBS_HD uint32_t sub(uint32_t* a, const uint32_t* b) {
  uint32_t br = 0;
#pragma unroll
  for (int i = 0; i < L; i++) {
    const uint64_t d = (uint64_t)a[i] - b[i] - br;
    a[i] = (uint32_t)d;
    br = (uint32_t)(d >> 63);
  }
  return br;
}
// a += b mod 2^(32 L), returns the carry out (0/1).
template <int L>
BFTQ_LIMBS_HD uint32_t add(uint32_t* a, const uint32_t* b) {
  uint64_t c = 0;
  for (int k = 0; k < L; k++) { c += (uint64_t)a[k] + b[k]; a[k] = (uint32_t)c; c >>= 32; }
  return (uint32_t)c;
}
// a = (a >> 1) | top << (32 L - 1)
template <int L>
BFTQ_LIMBS_HD void shr1(uint32_t* a, uint32_t top) {
  for (int k = 0; k < L - 1; k++) a[k] = (a[k] >> 1) | (a[k + 1] << 31);
  a[L - 1] = (a[L - 1] >> 1) | (top << 31);
}
// x / 2 mod m (x < m, m odd)
template <int L>
BFTQ_LIMBS_HD void half(uint32_t* x, const uint32_t* m) {
  const uint32_t top = (x[0] & 1u) ? add<L>(x, m) : 0u;
  shr1<L>(x, top);
}

// ---- big-endian byte strings --------------------------------------------------------------------------------------
BFTQ_LIMBS_HD uint32_t load_byte(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
BFTQ_LIMBS_HD int32_t load_i32(const int32_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
// v = the nbytes-long big-endian integer at p (its low 4 L bytes when nbytes is larger).
template <int L>
BFTQ_LIMBS_HD void load_be(uint32_t (&v)[L], const uint8_t* p, int nbytes) {
#pragma unroll
  for (int l = 0; l < L; l++) {
    uint32_t w = 0;
    for (int b = 0; b < 4; b++) { const int pos = nbytes - 1 - (4 * l + b); if (pos >= 0) w |= load_byte(p + pos) << (8 * b); }
    v[l] = w;
  }
}
// The low nbytes bytes of v (nbytes <= 4 L), big-endian, at p.
template <int L>
BFTQ_LIMBS_HD void store_be_bytes(uint8_t* p, int nbytes, const uint32_t (&v)[L]) {
#pragma unroll
  for (int l = 0; l < L; l++) {
    for (int b = 0; b < 4; b++) { const int pos = nbytes - 1 - (4 * l + b); if (pos >= 0) p[pos] = (uint8_t)(v[l] >> (8 * b)); }
  }
}
// out = (the nbytes-long big-endian integer at p) mod m, m > 0, bitwise shift-subtract (the remainder stays below 2m).
template <int L>
BFTQ_LIMBS_HD void reduce_be(uint32_t (&out)[L], const uint8_t* p, uint32_t nbytes, const uint32_t (&m)[L]) {
  uint32_t v[L + 1];
#pragma unroll
  for (int l = 0; l <= L; l++) v[l] = 0;
  for (uint32_t by = 0; by < nbytes; by++) {
    const uint32_t byte = load_byte(p + by);
    for (int bit = 7; bit >= 0; bit--) {
      uint32_t c = (byte >> bit) & 1u;
#pragma unroll
      for (int l = 0; l <= L; l++) { const uint32_t nc = v[l] >> 31; v[l] = (v[l] << 1) | c; c = nc; }
      if (v[L] != 0 || ge<L>(v, m)) v[L] -= sub<L>(v, m);
    }
  }
  for (int l = 0; l < L; l++) out[l] = v[l];
}

}  // namespace limbs
}  // namespace bftq
