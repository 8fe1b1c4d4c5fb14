// Lane-group radix-2^32 Montgomery arithmetic, shared by K1 (rsa_verify_r32.cuh), K5 (modexp.cuh), K6a (msg_decrypt.cuh)
// and K7 (thrsa_sign.cuh).  A number is owned by a group of T = 4 consecutive lanes, W 32-bit limbs per lane (lane r holds
// limbs r W .. r W + W - 1, little-endian); the four lanes of a group, and all 32 lanes of the warp, call every function
// here together.
//
// Why radix 2^32: on H100 every 64-bit-result integer multiply issues at half the IMAD.LO rate, carry chain or not
// (DESIGN.md §4).  The carry-free radix-2^28 form therefore buys nothing per instruction and pays (76/64)^2 = 1.41x more
// of them.
// mad.lo.cc/madc.hi.cc pairs compile to one IMAD.WIDE.U32.X each, and the classic even/odd column split keeps every
// chain's carry inside the instruction stream:
//   E[k] sits at limb position k     (even-aligned pairs (0,1),(2,3),...)
//   O[k] sits at limb position k+1   (odd-aligned pairs (1,2),(3,4),...)
// One round consumes TWO limbs of b (offsets 0 and 1): at offset 0 even limbs of the operand feed E
// and odd ones feed O, at offset 1 it is the other way round, so nothing ever has to be added across
// the two alignments inside a round.  After the round the number is shifted down two limbs, which is
// pure register renaming for E and O; the only cross terms are the 1-bit carry out of position 1
// (fed into the next round's first chain as its carry-in), the upper half of the one O pair the cut
// goes through (kept as a lone pending limb Z at the new position 0) and the two low limbs each lane
// hands to the lane below.  The scheme is checked limb-for-limb by tools/emu_r32.py.  Montgomery products are "almost" reduced (< R = 2^(128 W)): one conditional
// subtraction of n when the result overflowed R, decided by the carry out of the top lane.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace bftq {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kRsaBytes = 256;       // k = 256: RSA-2048 (the class the fast path and the flat API default to)

// ---- lane-distributed big-endian I/O ------------------------------------------------------------------------------

// 32-bit little-endian word k of a KB-byte big-endian integer in global memory.
template <int KB = kRsaBytes>
__device__ __forceinline__ uint32_t be_word(const uint8_t* p, int k) {
  if (k >= KB / 4) return 0u;
  uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(p + (KB - 4) - 4 * k));
  return __byte_perm(v, 0, 0x0123);
}
// little-endian 32-bit word k of an nbytes-long big-endian integer
__device__ __forceinline__ uint32_t be_word_dyn(const uint8_t* p, int nbytes, int k) {
  const int off = nbytes - 4 - 4 * k;
  if (off < 0) return 0u;
  return ((uint32_t)__ldg(p + off) << 24) | ((uint32_t)__ldg(p + off + 1) << 16) | ((uint32_t)__ldg(p + off + 2) << 8) | __ldg(p + off + 3);
}
template <int W>
__device__ __forceinline__ void store_be(uint8_t* p, int nbytes, const uint32_t (&v)[W], int r) {
#pragma unroll
  for (int j = 0; j < W; j++) {
    const int off = nbytes - 4 - 4 * (r * W + j);
    p[off] = (uint8_t)(v[j] >> 24); p[off + 1] = (uint8_t)(v[j] >> 16); p[off + 2] = (uint8_t)(v[j] >> 8); p[off + 3] = (uint8_t)v[j];
  }
}

namespace r32 {

constexpr int T = 4;      // lanes per number
// W = 32-bit limbs per lane: 16 for 2048-bit numbers (K1, K7), 8 for 1024-bit ones (K5 at L1024, K6a's CRT halves).

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

// ---- group add / subtract / select (no branch on the data) -------------------------------------------------------

// out = a + b mod 2^(128 W) over the group's lanes; returns the carry out of the top lane (the same in all four).
template <int W>
__device__ __forceinline__ uint32_t group_add(uint32_t (&out)[W], const uint32_t (&a)[W], const uint32_t (&b)[W], const int r, const int gbase) {
  uint32_t g;
  asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(out[0]) : "r"(a[0]), "r"(b[0]));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(out[k]) : "r"(a[k]), "r"(b[k]));
  asm volatile("addc.u32 %0, 0, 0;" : "=r"(g));
  uint32_t ones = 1u;
#pragma unroll
  for (int k = 0; k < W; k++) ones &= (uint32_t)(out[k] == 0xffffffffu);
  const uint32_t gb = __ballot_sync(kFull, g != 0u) >> gbase;
  const uint32_t pb = __ballot_sync(kFull, ones != 0u) >> gbase;
  uint32_t ctop;
  const uint32_t ci = lane_carry_in(gb, pb, r, ctop);
  ripple_add(out, ci);
  return ctop;
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
// x = take_y ? y : x (take_y 0 / 1), with a mask.
template <int W>
__device__ __forceinline__ void select_mask(uint32_t (&x)[W], const uint32_t (&y)[W], const uint32_t take_y) {
  const uint32_t m = 0u - take_y;
#pragma unroll
  for (int k = 0; k < W; k++) x[k] = (y[k] & m) | (x[k] & ~m);
}

// The tail of a Montgomery product: merges the E / O accumulators and the pending carries into W limbs per lane,
// resolves the carries across the four lanes and subtracts n once when the result overflowed 2^(128 W).
// CT: the subtraction is always computed and selected with a mask (no branch on the data: K6a, K7).
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
    group_sub(d, v, n, r, gbase);
    if (CT) {
      select_mask(v, d, (uint32_t)overflow);
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

// x -= n when x >= n (x < 2n on entry).  CT: the subtraction is always computed and its borrow selects with a mask.
template <int W, bool CT = false>
__device__ __forceinline__ void cond_sub(uint32_t (&x)[W], const uint32_t (&n)[W], const int r, const int gbase) {
  uint32_t d[W];
  if (CT) {
    const uint32_t bt = group_sub(d, x, n, r, gbase);
    select_mask(x, d, bt ^ 1u);
  } else {
    const bool ge = group_ge(x, n, gbase);
    group_sub(d, x, n, r, gbase);
    if (ge) {
#pragma unroll
      for (int k = 0; k < W; k++) x[k] = d[k];
    }
  }
}

// y = y * base^e in Montgomery form, constant time in e and in the base: y enters as 1 R (mod m), bm is base R.  e is
// read as nwin 4-bit windows, most significant first, from the little-endian 32-bit words `words` (words at index >= nw
// read as zero).  The 16-entry table base^i R lives in this thread's column tab[i][.][threadIdx.x]; every window
// squares four times, reads all sixteen entries with masks and multiplies once, and every product is mont_mul<W, true>.
// The table is left filled: the caller zeroes it.  All 32 lanes of the warp must call this together with one nwin.
template <int W, int BLOCK>
__device__ __forceinline__ void ct_window_pow(uint32_t (&y)[W], const uint32_t (&bm)[W], const uint32_t (&m)[W], const uint32_t m0inv,
                                              const uint32_t* __restrict__ words, const uint32_t nw, const int nwin,
                                              uint32_t (*tab)[W][BLOCK], const int r, const int gbase) {
  const int tid = threadIdx.x;
  uint32_t t[W], x[W];
#pragma unroll
  for (int j = 0; j < W; j++) { tab[0][j][tid] = y[j]; tab[1][j][tid] = bm[j]; t[j] = bm[j]; }
#pragma unroll 1
  for (int e = 2; e < 16; e++) {
    mont_mul<W, true>(x, t, bm, m, m0inv, r, gbase);
#pragma unroll
    for (int j = 0; j < W; j++) { tab[e][j][tid] = x[j]; t[j] = x[j]; }
  }
#pragma unroll 1
  for (int win = nwin - 1; win >= 0; win--) {
#pragma unroll 1
    for (int k = 0; k < 4; k++) {
      mont_mul<W, true>(t, y, y, m, m0inv, r, gbase);
#pragma unroll
      for (int j = 0; j < W; j++) y[j] = t[j];
    }
    const uint32_t wi = (uint32_t)win >> 3;
    const uint32_t word = wi < nw ? __ldg(words + wi) : 0u;
    const uint32_t w = (word >> ((win & 7) * 4)) & 15u;
#pragma unroll
    for (int j = 0; j < W; j++) x[j] = 0u;
#pragma unroll
    for (int e = 0; e < 16; e++) {
      const uint32_t msk = 0u - (uint32_t)((uint32_t)e == w);
#pragma unroll
      for (int j = 0; j < W; j++) x[j] |= tab[e][j][tid] & msk;
    }
    mont_mul<W, true>(t, y, x, m, m0inv, r, gbase);
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = t[j];
  }
}

}  // namespace r32
}  // namespace bftq
