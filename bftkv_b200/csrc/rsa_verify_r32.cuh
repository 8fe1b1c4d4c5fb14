// K1 (fast path) — RSA-2048 PKCS#1 v1.5 batch verify, radix 2^32 with IMAD.WIDE.U32.X carry chains.
//
// Same contract as rsa_verify.cuh (the radix-2^28 kernel, kept for moduli of 2041..2047 bits); this
// variant requires the modulus to have exactly 2048 bits, which is what every RSA-2048 key
// generator (gpg, OpenSSL, Go) produces.
//
// Why: on H100 every 64-bit-result integer multiply issues at half the IMAD.LO rate, carry chain or
// not (DESIGN.md §4).  The carry-free radix-2^28 form therefore buys nothing per instruction and
// pays (76/64)^2 = 1.41x more of them.
// Here a signature is owned by 4 lanes x 16 32-bit limbs; mad.lo.cc/madc.hi.cc pairs compile to one
// IMAD.WIDE.U32.X each, and the classic even/odd column split keeps every chain's carry inside the
// instruction stream:
//   E[k] sits at limb position k     (even-aligned pairs (0,1),(2,3),...)
//   O[k] sits at limb position k+1   (odd-aligned pairs (1,2),(3,4),...)
// One round consumes TWO limbs of b (offsets 0 and 1): at offset 0 even limbs of the operand feed E
// and odd ones feed O, at offset 1 it is the other way round, so nothing ever has to be added across
// the two alignments inside a round.  After the round the number is shifted down two limbs, which is
// pure register renaming for E and O; the only cross terms are the 1-bit carry out of position 1
// (fed into the next round's first chain as its carry-in), the upper half of the one O pair the cut
// goes through (kept as a lone pending limb Z at the new position 0) and the two low limbs each lane
// hands to the lane below.  The scheme is checked limb-for-limb by tools/emu_r32.py.  Montgomery products are "almost" reduced (< R = 2^2048): one conditional
// subtraction of n when the result overflowed 2^2048, decided by the carry out of the top lane.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "rsa_verify.cuh"

namespace bftq {
namespace r32 {

constexpr int T = 4;      // lanes per number
// W = 32-bit limbs per lane: 16 for 2048-bit numbers (the RSA kernel), 8 for 1024-bit ones (modexp).

// ---- carry-chain building blocks ----------------------------------------------------------------
// One asm statement per chain (8 mad.lo.cc/madc.hi.cc pairs + the carry limb), so ptxas sees the
// whole chain at once and keeps the carry in a predicate: each pair becomes one IMAD.WIDE.U32.X.
// P(lo,hi) are accumulator limbs, X the operand limbs, m the multiplier.
#define BFTQ_CHAIN8_BODY(first)                                                              \
  first " %0, %18, %26, %0;  madc.hi.cc.u32 %1, %18, %26, %1;"                                \
  "madc.lo.cc.u32 %2, %19, %26, %2;  madc.hi.cc.u32 %3, %19, %26, %3;"                        \
  "madc.lo.cc.u32 %4, %20, %26, %4;  madc.hi.cc.u32 %5, %20, %26, %5;"                        \
  "madc.lo.cc.u32 %6, %21, %26, %6;  madc.hi.cc.u32 %7, %21, %26, %7;"                        \
  "madc.lo.cc.u32 %8, %22, %26, %8;  madc.hi.cc.u32 %9, %22, %26, %9;"                        \
  "madc.lo.cc.u32 %10, %23, %26, %10; madc.hi.cc.u32 %11, %23, %26, %11;"                     \
  "madc.lo.cc.u32 %12, %24, %26, %12; madc.hi.cc.u32 %13, %24, %26, %13;"                     \
  "madc.lo.cc.u32 %14, %25, %26, %14; madc.hi.cc.u32 %15, %25, %26, %15;"                     \
  "addc.cc.u32 %16, %16, 0; addc.u32 %17, %17, 0;"
#define BFTQ_CHAIN8_OPS(p, c0, c1, x)                                                                                     \
  : "+r"(p[0]), "+r"(p[1]), "+r"(p[2]), "+r"(p[3]), "+r"(p[4]), "+r"(p[5]), "+r"(p[6]), "+r"(p[7]), "+r"(p[8]), "+r"(p[9]), \
    "+r"(p[10]), "+r"(p[11]), "+r"(p[12]), "+r"(p[13]), "+r"(p[14]), "+r"(p[15]), "+r"(c0), "+r"(c1)                      \
  : "r"(x[0]), "r"(x[2]), "r"(x[4]), "r"(x[6]), "r"(x[8]), "r"(x[10]), "r"(x[12]), "r"(x[14]), "r"(m)

#define BFTQ_CHAIN4_BODY(first)                                                              \
  first " %0, %10, %14, %0;  madc.hi.cc.u32 %1, %10, %14, %1;"                                \
  "madc.lo.cc.u32 %2, %11, %14, %2;  madc.hi.cc.u32 %3, %11, %14, %3;"                        \
  "madc.lo.cc.u32 %4, %12, %14, %4;  madc.hi.cc.u32 %5, %12, %14, %5;"                        \
  "madc.lo.cc.u32 %6, %13, %14, %6;  madc.hi.cc.u32 %7, %13, %14, %7;"                        \
  "addc.cc.u32 %8, %8, 0; addc.u32 %9, %9, 0;"
#define BFTQ_CHAIN4_OPS(p, c0, c1, x)                                                                                     \
  : "+r"(p[0]), "+r"(p[1]), "+r"(p[2]), "+r"(p[3]), "+r"(p[4]), "+r"(p[5]), "+r"(p[6]), "+r"(p[7]), "+r"(c0), "+r"(c1)      \
  : "r"(x[0]), "r"(x[2]), "r"(x[4]), "r"(x[6]), "r"(m)

// E/O accumulators of one lane: positions 0..W+2 (+1 scratch so every chain has two carry limbs).
template <int W>
struct Acc {
  uint32_t E[W + 4];
  uint32_t O[W + 2];
};

// One carry chain over W/2 (lo,hi) pairs starting at p[0], operand limbs x[0], x[2], ..., carry limbs c0, c1.
template <int W> struct Chain;
template <> struct Chain<16> {
  static __device__ __forceinline__ void run(uint32_t* p, uint32_t& c0, uint32_t& c1, const uint32_t* x, const uint32_t m) {
    asm volatile(BFTQ_CHAIN8_BODY("mad.lo.cc.u32") BFTQ_CHAIN8_OPS(p, c0, c1, x));
  }
  static __device__ __forceinline__ void run_cin(uint32_t* p, uint32_t& c0, uint32_t& c1, const uint32_t* x, const uint32_t m, const uint32_t cin) {
    asm volatile("{ .reg .u32 t; add.cc.u32 t, %27, 0xffffffff;" BFTQ_CHAIN8_BODY("madc.lo.cc.u32") "}"
                 BFTQ_CHAIN8_OPS(p, c0, c1, x), "r"(cin));
  }
};
template <> struct Chain<8> {
  static __device__ __forceinline__ void run(uint32_t* p, uint32_t& c0, uint32_t& c1, const uint32_t* x, const uint32_t m) {
    asm volatile(BFTQ_CHAIN4_BODY("mad.lo.cc.u32") BFTQ_CHAIN4_OPS(p, c0, c1, x));
  }
  static __device__ __forceinline__ void run_cin(uint32_t* p, uint32_t& c0, uint32_t& c1, const uint32_t* x, const uint32_t m, const uint32_t cin) {
    asm volatile("{ .reg .u32 t; add.cc.u32 t, %15, 0xffffffff;" BFTQ_CHAIN4_BODY("madc.lo.cc.u32") "}"
                 BFTQ_CHAIN4_OPS(p, c0, c1, x), "r"(cin));
  }
};

// offset 0: even limbs -> E pairs (k,k+1), odd limbs -> O pairs (O[k-1],O[k]).  `cin` (0/1) enters
// the even chain at position 0.
template <int W>
__device__ __forceinline__ void mac_off0_even(Acc<W>& A, const uint32_t (&x)[W], const uint32_t m, const uint32_t cin) {
  Chain<W>::run_cin(A.E, A.E[W], A.E[W + 1], x, m, cin);
}
template <int W>
__device__ __forceinline__ void mac_off0_even_nocin(Acc<W>& A, const uint32_t (&x)[W], const uint32_t m) {
  Chain<W>::run(A.E, A.E[W], A.E[W + 1], x, m);
}
template <int W>
__device__ __forceinline__ void mac_off0_odd(Acc<W>& A, const uint32_t (&x)[W], const uint32_t m) {
  Chain<W>::run(A.O, A.O[W], A.O[W + 1], x + 1, m);          // x[1], x[3], ...
}
// offset 1: even limbs -> O pairs (O[k],O[k+1]), odd limbs -> E pairs (E[k+1],E[k+2]).
template <int W>
__device__ __forceinline__ void mac_off1_even(Acc<W>& A, const uint32_t (&x)[W], const uint32_t m) {
  Chain<W>::run(A.O, A.O[W], A.O[W + 1], x, m);
}
template <int W>
__device__ __forceinline__ void mac_off1_odd(Acc<W>& A, const uint32_t (&x)[W], const uint32_t m) {
  Chain<W>::run(A.E + 2, A.E[W + 2], A.E[W + 3], x + 1, m);
}

// Ripple-add a 32-bit value into v[0..15]; returns the carry out (0/1).
template <int W>
__device__ __forceinline__ uint32_t ripple_add(uint32_t (&v)[W], const uint32_t x) {
  uint32_t c;
  asm volatile("add.cc.u32 %0, %0, %1;" : "+r"(v[0]) : "r"(x));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("addc.cc.u32 %0, %0, 0;" : "+r"(v[k]));
  asm volatile("addc.u32 %0, 0, 0;" : "=r"(c));
  return c;
}
// v -= x (one limb), returns borrow out (0/1).
template <int W>
__device__ __forceinline__ uint32_t ripple_sub(uint32_t (&v)[W], const uint32_t x) {
  uint32_t b;
  asm volatile("sub.cc.u32 %0, %0, %1;" : "+r"(v[0]) : "r"(x));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("subc.cc.u32 %0, %0, 0;" : "+r"(v[k]));
  asm volatile("subc.u32 %0, 0, 0;" : "=r"(b));
  return b & 1u;
}
// d = v - n (limb-wise with borrow chain), returns borrow out (0/1).
template <int W>
__device__ __forceinline__ uint32_t sub_n(uint32_t (&d)[W], const uint32_t (&v)[W], const uint32_t (&n)[W]) {
  uint32_t b;
  asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(v[0]), "r"(n[0]));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(d[k]) : "r"(v[k]), "r"(n[k]));
  asm volatile("subc.u32 %0, 0, 0;" : "=r"(b));
  return b & 1u;
}

// Carry (or borrow) into each lane of a 4-lane group from per-lane generate / propagate flags:
// in[r] = gen[r-1] | (prop[r-1] & in[r-1]), in[0] = 0.  Returns this lane's carry-in and, in `out`,
// the carry out of the top lane.  gbits/pbits are ballots already shifted to the group's bit 0.
__device__ __forceinline__ uint32_t lane_carry_in(const uint32_t gbits, const uint32_t pbits, const int r, uint32_t& out) {
  const uint32_t c1 = gbits & 1u;
  const uint32_t c2 = ((gbits >> 1) & 1u) | (((pbits >> 1) & 1u) & c1);
  const uint32_t c3 = ((gbits >> 2) & 1u) | (((pbits >> 2) & 1u) & c2);
  out = ((gbits >> 3) & 1u) | (((pbits >> 3) & 1u) & c3);
  return r == 0 ? 0u : (r == 1 ? c1 : (r == 2 ? c2 : c3));
}

// The tail of a Montgomery product: merges the E / O accumulators and the pending carries into W limbs per lane,
// resolves the carries across the four lanes and subtracts n once when the result overflowed 2^(128 W).
// CT: the subtraction is always computed and selected with a mask (no branch on the data: K6a, msg_decrypt.cuh).
template <int W, bool CT = false>
__device__ __forceinline__ void mont_finish(uint32_t (&out)[W], Acc<W>& A, const uint32_t cin, const uint32_t Z, const uint32_t (&n)[W],
                                            const int r, const int gbase) {
  // ---- merge E, O and the pending carry into 16 limbs + overflow ------------------------------
  uint32_t v[W], hi;
  asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(v[0]) : "r"(A.E[0]), "r"(Z));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(v[k]) : "r"(A.E[k]), "r"(A.O[k - 1]));
  asm volatile("addc.u32 %0, %1, %2;" : "=r"(hi) : "r"(A.E[W]), "r"(A.O[W - 1]));
  // the lane's overflow (a few units) belongs to the lane above; the top lane's is bit 2048+
  uint32_t from_below = __shfl_up_sync(kFull, hi, 1, T);
  if (r == 0) from_below = 0u;
  const uint32_t g = ripple_add(v, from_below + cin);
  bool ones = true;
#pragma unroll
  for (int k = 0; k < W; k++) ones = ones && (v[k] == 0xffffffffu);
  const uint32_t gb = __ballot_sync(kFull, g != 0u) >> gbase;
  const uint32_t pb = __ballot_sync(kFull, ones) >> gbase;
  uint32_t ctop;
  const uint32_t ci = lane_carry_in(gb, pb, r, ctop);
  ripple_add(v, ci);
  const uint32_t top_hi = __shfl_sync(kFull, hi, gbase + T - 1);
  const bool overflow = (top_hi + ctop) != 0u;          // result >= 2^2048: subtract n once
  // ---- conditional subtraction ---------------------------------------------------------------
  if (CT || __any_sync(kFull, overflow)) {
    uint32_t d[W];
    const uint32_t bo = sub_n(d, v, n);
    bool zeros = true;
#pragma unroll
    for (int k = 0; k < W; k++) zeros = zeros && (d[k] == 0u);
    const uint32_t bgb = __ballot_sync(kFull, bo != 0u) >> gbase;
    const uint32_t bpb = __ballot_sync(kFull, zeros) >> gbase;
    uint32_t btop;
    const uint32_t bi = lane_carry_in(bgb, bpb, r, btop);
    ripple_sub(d, bi);
    if (CT) {
      const uint32_t m = 0u - (uint32_t)overflow;
#pragma unroll
      for (int k = 0; k < W; k++) v[k] = (d[k] & m) | (v[k] & ~m);
    } else if (overflow) {
#pragma unroll
      for (int k = 0; k < W; k++) v[k] = d[k];
    }
  }
#pragma unroll
  for (int k = 0; k < W; k++) out[k] = v[k];
}

// out = a * b * R^-1 mod n with R = 2^(128 W), out < R ("almost Montgomery").  a, b < R as W limbs/lane.
// owners < T stops after that many owner steps: out == a * b' * 2^(-32 W owners) (mod n) with b' the owners' low lanes of b, out < R
// and, for a < n, out < 2n (K1's final check, one or two owner steps).  All 32 lanes of the warp must call this together.
template <int W, bool CT = false>
__device__ __forceinline__ void mont_mul(uint32_t (&out)[W], const uint32_t (&a)[W], const uint32_t (&b)[W],
                                         const uint32_t (&n)[W], const uint32_t n0inv, const int r, const int gbase,
                                         const int owners = T) {
  Acc<W> A;
#pragma unroll
  for (int k = 0; k < W + 4; k++) A.E[k] = 0u;
#pragma unroll
  for (int k = 0; k < W + 2; k++) A.O[k] = 0u;
  uint32_t cin = 0u;      // 1-bit carry pending at position 0
  uint32_t Z = 0u;        // odd-side limb pending at position 0 (the upper half of the O pair the shift cut)
#pragma unroll 1
  for (int owner = 0; owner < T; owner++) {
    if (owner == owners) break;                 // a constant trip count with an early exit: with the default owners = T (K5, K6a) the test folds away
    const int src = gbase + owner;
#pragma unroll
    for (int jj = 0; jj < W; jj += 2) {
      const uint32_t b0 = __shfl_sync(kFull, b[jj], src);
      const uint32_t b1 = __shfl_sync(kFull, b[jj + 1], src);
      // ---- offset 0 -------------------------------------------------------------------------
      mac_off0_even(A, a, b0, cin);
      uint32_t q0 = (A.E[0] + Z) * n0inv;
      q0 = __shfl_sync(kFull, q0, gbase);
      mac_off0_odd(A, a, b0);
      mac_off1_even(A, a, b1);
      mac_off1_odd(A, a, b1);
      mac_off0_even_nocin(A, n, q0);
      mac_off0_odd(A, n, q0);
      // ---- offset 1 -------------------------------------------------------------------------
      // position 0 = E[0] + Z: zero mod 2^32 in lane 0, its carry moves into position 1
      const uint64_t s0 = (uint64_t)A.E[0] + Z;
      const uint32_t p0 = (uint32_t)s0, c0 = (uint32_t)(s0 >> 32);
      uint32_t q1 = (A.E[1] + A.O[0] + c0) * n0inv;
      q1 = __shfl_sync(kFull, q1, gbase);
      mac_off1_even(A, n, q1);
      mac_off1_odd(A, n, q1);
      // positions 0 and 1 leave the lane: lane 0's are zero, the others' go to the lane below
      const uint64_t s1 = (uint64_t)A.E[1] + A.O[0] + c0;
      const uint32_t p1 = (uint32_t)s1;
      cin = (uint32_t)(s1 >> 32);
      Z = A.O[1];
      uint32_t r0 = __shfl_down_sync(kFull, p0, 1, T);
      uint32_t r1 = __shfl_down_sync(kFull, p1, 1, T);
      if (r == T - 1) { r0 = 0u; r1 = 0u; }
      // shift down two limbs (register renaming)
#pragma unroll
      for (int k = 0; k < W + 2; k++) A.E[k] = A.E[k + 2];
      A.E[W + 2] = 0u; A.E[W + 3] = 0u;
#pragma unroll
      for (int k = 0; k < W; k++) A.O[k] = A.O[k + 2];
      A.O[W] = 0u; A.O[W + 1] = 0u;
      asm volatile("add.cc.u32 %0, %0, %4; addc.cc.u32 %1, %1, %5; addc.cc.u32 %2, %2, 0; addc.u32 %3, %3, 0;"
                   : "+r"(A.E[W - 2]), "+r"(A.E[W - 1]), "+r"(A.E[W]), "+r"(A.E[W + 1]) : "r"(r0), "r"(r1));
    }
  }
  mont_finish<W, CT>(out, A, cin, Z, n, r, gbase);
}

// x >= n ?  (lane-distributed compare)
template <int W>
__device__ __forceinline__ bool group_ge(const uint32_t (&x)[W], const uint32_t (&n)[W], const int gbase) {
  bool gt = false, lt = false;
#pragma unroll
  for (int j = W - 1; j >= 0; j--) {
    if (!gt && !lt) { gt = x[j] > n[j]; lt = x[j] < n[j]; }
  }
  const uint32_t gmask = ((1u << T) - 1u) << gbase;
  const uint32_t gtb = __ballot_sync(kFull, gt) & gmask;
  const uint32_t ltb = __ballot_sync(kFull, lt) & gmask;
  return gtb >= ltb;
}

// d = x - y mod 2^(128 W) over the group's lanes; returns the borrow out of the top lane (the same in all four).
template <int W>
__device__ __forceinline__ uint32_t group_sub(uint32_t (&d)[W], const uint32_t (&x)[W], const uint32_t (&y)[W], const int r, const int gbase) {
  const uint32_t bo = sub_n(d, x, y);
  bool zeros = true;
#pragma unroll
  for (int k = 0; k < W; k++) zeros = zeros && (d[k] == 0u);
  const uint32_t bgb = __ballot_sync(kFull, bo != 0u) >> gbase;
  const uint32_t bpb = __ballot_sync(kFull, zeros) >> gbase;
  uint32_t btop;
  const uint32_t bi = lane_carry_in(bgb, bpb, r, btop);
  ripple_sub(d, bi);
  return btop;
}

// x -= n when x >= n (x < 2n on entry).
template <int W>
__device__ __forceinline__ void cond_sub(uint32_t (&x)[W], const uint32_t (&n)[W], const int r, const int gbase) {
  const bool ge = group_ge(x, n, gbase);
  uint32_t d[W];
  group_sub(d, x, n, r, gbase);
  if (ge) {
#pragma unroll
    for (int k = 0; k < W; k++) x[k] = d[k];
  }
}

}  // namespace r32
}  // namespace bftq
#include "rsa_square_r32.cuh"
namespace bftq {
namespace r32 {

struct RsaKey32 {               // per key, radix 2^32 little-endian words; c = R^-(e-1) mod n, R = 2^2048 (bignum_host.hpp)
  uint32_t n[64];
  uint32_t c16[64];             // c * 2^512 mod n
  uint32_t hc16[64];            // (EM with its low 512 bits cleared) * c mod n, for T of up to 63 bytes
  uint32_t c32[64];             // c * 2^1024 mod n
  uint32_t hc32[64];            // (EM with its low 1024 bits cleared) * c mod n, for longer T (SHA-384, SHA-512)
  uint32_t n0inv;               // -n^-1 mod 2^32
  uint32_t e;
  uint32_t nbits;
  uint32_t pad;
};

// Threads per block and blocks per SM: 4 blocks of 4 warps at 128 registers per thread fill an SM's 64 K registers.
constexpr int kK1Block = 128, kK1MinBlocks = 4;

// The exponentiation never converts s to Montgomery form: it runs the square-and-multiply chain of e on the plain s,
// every 1 bit below the top one a product with the plain s.  A squaring takes y = s^k R^-(k-1) to s^2k R^-(2k-1) and a
// product with s to s^(k+1) R^-k, so the chain ends at Y = s^e c with c = R^-(e-1) mod n: 16 squarings and one product
// for e = 65537.  With EM = H 2^k + L (k = 512, or 1024 for T longer than 63 bytes), s^e == EM (mod n) iff
// Y == c L + hc (mod n); c L is ONE (or two) owner steps of mont_mul with the key's c * 2^k, and hc = H 2^k c mod n is
// a per-key constant because H = 00 01 FF..FF does not depend on the digest (RsaKey32, bignum_host.hpp).
// The squarings go through mont_sqr (rsa_square_r32.cuh).
//
// The four warps of a block meet at a barrier once per task and after every squaring.  Warps that drift apart fetch
// different parts of the hot loop and evict each other from the instruction caches; without the barriers the kernel
// loses 10 % on H100 (DESIGN.md §4).
__global__ void __launch_bounds__(kK1Block, kK1MinBlocks)
rsa_verify_r32_kernel(const RsaKey32* __restrict__ keys, const uint32_t nkeys, const uint32_t* __restrict__ key_idx,
                      const uint8_t* __restrict__ sig, const uint8_t* __restrict__ digest, const uint32_t hash_alg,
                      const uint64_t n_items, const uint32_t flags, const uint8_t* __restrict__ pre_status,
                      uint8_t* __restrict__ status) {
  constexpr int W = 16;
  constexpr int kGroupsPerWarp = 32 / T;
  __shared__ uint32_t y_s[W][kK1Block];
  __shared__ int nbmax_s;
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int plen = c_hash_prefix[hash_alg].len;
  const int dlen = c_hash_prefix[hash_alg].dlen;
  const bool wide = plen + dlen > 63;                        // T and its 00 separator reach above 2^512: split EM at 2^1024
  const int check_owners = wide ? 2 : 1;
  const uint64_t warps_total = (uint64_t)gridDim.x * (kK1Block / 32);
  const uint32_t gmask = ((1u << T) - 1u) << gbase;

  // The trip count is uniform over the block (a warp whose eight signatures lie behind the end computes on clamped items
  // and stores nothing), so the warps of a block may meet at barriers.  Warps that stay in phase fetch the same
  // instructions at the same time (the hot loop is 15 KB).
  for (uint64_t bbase = (uint64_t)blockIdx.x * (kK1Block / 32) * kGroupsPerWarp; bbase < n_items; bbase += warps_total * kGroupsPerWarp) {
    const uint64_t wbase = bbase + (uint64_t)(threadIdx.x >> 5) * kGroupsPerWarp;
    __syncthreads();
    const uint64_t item_raw = wbase + (uint64_t)(lane / T);
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : (n_items - 1);
    uint32_t kidx = __ldg(key_idx + item);
    const bool known = kidx < nkeys;
    if (!known) kidx = 0u;
    const RsaKey32* __restrict__ key = keys + kidx;

    uint32_t nd[W], y[W], t[W];
#pragma unroll
    for (int j = 0; j < W; j++) nd[j] = __ldg(&key->n[r * W + j]);
    const uint32_t n0inv = __ldg(&key->n0inv);
    const uint32_t e = __ldg(&key->e);
    const uint8_t* sp = sig + item * (uint64_t)kRsaBytes;
    const uint8_t* dp = digest + item * (uint64_t)dlen;
    const uint32_t* ck = wide ? key->c32 : key->c16;
    bool s_ge_n;
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = be_word(sp, r * W + j);
    s_ge_n = group_ge(y, nd, gbase);
    const int nb = 32 - __clz(e);
    int nbmax = nb;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) nbmax = max(nbmax, __shfl_xor_sync(kFull, nbmax, o));
    // barriers inside the exponent loop: its trip count must be uniform over the block
    if (threadIdx.x == 0) nbmax_s = 0;
    __syncthreads();
    if (lane == 0) atomicMax(&nbmax_s, nbmax);
    __syncthreads();
    nbmax = nbmax_s;
    // The whole verification as ONE loop over a small program, so that the kernel holds a single instance of the
    // squaring and a single instance of the general product (a straight-line chain followed by the check product holds
    // two; the instruction caches hold 32 KB).
    //   op 1: the squaring of `bit`      op 2: y *= s after the squaring of a 1 bit      op 3: the check product c L
    int bit = nbmax - 2, op = bit >= 0 ? 1 : 3;
#pragma unroll 1
    for (;;) {
      if (op == 1) {
        mont_sqr(t, y, nd, n0inv, r, gbase);
        __syncthreads();                                     // every warp of the block runs nbmax - 1 squarings
        if (bit <= nb - 2) {
#pragma unroll
          for (int j = 0; j < W; j++) y[j] = t[j];
        }
        const bool mul = bit <= nb - 2 && ((e >> bit) & 1u);
        if (__any_sync(kFull, mul)) op = 2;
        else { bit--; op = bit >= 0 ? 1 : 3; }
      } else {
        uint32_t bop[W];
        if (op == 3) {
          // b = EM's words (L in the owner lanes), built by a rolled loop through shared memory: one em_word instance
          // instead of sixteen (2.7 K instructions).  Then Y waits in shared memory while y holds c * 2^k.
#pragma unroll 1
          for (int j = 0; j < W; j++) y_s[j][threadIdx.x] = em_word(r * W + j, dp, plen, dlen, hash_alg);
#pragma unroll
          for (int j = 0; j < W; j++) { bop[j] = y_s[j][threadIdx.x]; y_s[j][threadIdx.x] = y[j]; y[j] = __ldg(&ck[r * W + j]); }
        } else {
#pragma unroll
          for (int j = 0; j < W; j++) bop[j] = be_word(sp, r * W + j);       // the plain s
        }
        mont_mul(t, y, bop, nd, n0inv, r, gbase, op == 2 ? T : check_owners);
        if (op == 3) break;
        if (bit <= nb - 2 && ((e >> bit) & 1u)) {
#pragma unroll
          for (int j = 0; j < W; j++) y[j] = t[j];
        }
        bit--;
        op = bit >= 0 ? 1 : 3;
      }
    }
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = y_s[j][threadIdx.x];
    // y = Y < 2^2048 < 2n and t = Q == c L (mod n), Q < 2n.  With D = (Y mod n) - (Q mod n) mod 2^2048, borrow b, and
    // F = hc - D mod 2^2048:  Y == Q + hc (mod n)  iff  F == 0 (b = 0: D = Y - Q in [0, n))  or  F == n (b = 1: D + n - 2^2048
    // = Y - Q + n in (0, n)).
    cond_sub(y, nd, r, gbase);
    cond_sub(t, nd, r, gbase);
    uint32_t d[W];
    const uint32_t b = group_sub(d, y, t, r, gbase);
    const uint32_t* hk = wide ? key->hc32 : key->hc16;
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = __ldg(&hk[r * W + j]);
    group_sub(t, y, d, r, gbase);
    bool eq = true;
#pragma unroll
    for (int j = 0; j < W; j++) eq = eq && (t[j] == (b ? nd[j] : 0u));
    const uint32_t eqb = __ballot_sync(kFull, eq) & gmask;
    if (valid && r == 0) {
      uint8_t st = (eqb == gmask) ? (uint8_t)0 : (uint8_t)1;
      if ((flags & 1u) && s_ge_n) st = 1;
      if (__ldg(&key->nbits) != 2048u) st = 1;             // not this kernel's key class
      if (!known) st = 4;
      if (pre_status != nullptr) {
        const uint8_t pre = __ldg(pre_status + item_raw);
        if (pre != 0) st = pre;
      }
      status[item_raw] = st;
    }
  }
}

}  // namespace r32
}  // namespace bftq
