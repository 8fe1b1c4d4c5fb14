// K1's dedicated Montgomery SQUARING (radix 2^32, 4 lanes x 16 limbs), on mont_mul's carry chains (mont_r32.cuh).
//
// 16 of the 18 Montgomery products of an e = 65537 verification are squarings, and a square needs only half of the
// limb products a x a of a general product (the n x q half of the CIOS loop stays as it is).  In the lane-distributed
// layout the lanes run the rounds of mont_mul in lock-step, so skipping "the lower triangle" only pays when every lane
// skips the same amount in the same round.  This tiling does that.  Row J = 16*Y + j (owner lane Y broadcasts limb
// a_J); lane X multiplies a_J by
//     X <  Y :  2 * (A_X with limbs <  j zeroed)             the pairs (i in block X, J) with i_loc >= j
//     X >  Y :  2 * (A_X with limbs <= j zeroed)             the pairs (i in block X, J) with i_loc >  j
//     X == Y :  a_j  +  2 * (A_X with limbs <= j zeroed)     the diagonal term once, the rest of the row twice
// so every unordered limb pair {i, J} of different blocks is met exactly once — in row J by the lane that owns i, or
// in row i by the lane that owns J — and in round j EVERY lane multiplies the limbs j..15 of its own block: the
// lock-step rounds shrink together, 136 limb products per lane and step instead of 256 (544 + 1024 IMAD.WIDE per lane
// and squaring instead of 2048; -20.8 % over the whole verification).  A contribution to position p is always made in
// a row <= p, i.e. before the reduction eliminates that position, so the interleaved reduction of mont_mul is kept
// unchanged; no shared memory, no second pass.
// The doubled operand is the lane-local a2 = 2 * A_X (17 limbs, a2[16] = the bit shifted out): a row uses a2[k] for
// k >= j + 2, two patched limbs at k = j and j + 1, and the bit a2[16] as an addend of the chain's first carry limb
// (free).  Unlike mont_mul, a step leaves no pending limb at position 0: the next step's position 0 is folded into one
// limb at once, and the 1-bit carry out of it waits at position 1 and enters with the n x q1 chain.  tools/emu_sq.py
// emulates this file limb for limb.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "mont_r32.cuh"

namespace bftq {
namespace r32 {

// (lo, hi) += x * m + carry, as one IMAD.WIDE.U32(.X): `first` starts a carry chain, the others continue it.
__device__ __forceinline__ void mad_pair_first(uint32_t& lo, uint32_t& hi, const uint32_t x, const uint32_t m) {
  asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(x), "r"(m));
}
__device__ __forceinline__ void mad_pair_next(uint32_t& lo, uint32_t& hi, const uint32_t x, const uint32_t m) {
  asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(x), "r"(m));
}
// N (lo, hi) pairs starting at p[0], operand limbs x[0], x[2], ..., then the carry limbs: c0 += t + carry, c1 += carry.
template <int N>
__device__ __forceinline__ void chain_n(uint32_t* p, uint32_t& c0, uint32_t& c1, const uint32_t* x, const uint32_t m, const uint32_t t) {
  if (N == 0) {
    asm volatile("add.cc.u32 %0, %0, %2; addc.u32 %1, %1, 0;" : "+r"(c0), "+r"(c1) : "r"(t));
    return;
  }
  mad_pair_first(p[0], p[1], x[0], m);
#pragma unroll
  for (int i = 1; i < N; i++) mad_pair_next(p[2 * i], p[2 * i + 1], x[2 * i], m);
  asm volatile("addc.cc.u32 %0, %0, %2; addc.u32 %1, %1, 0;" : "+r"(c0), "+r"(c1) : "r"(t));
}
// The same with one carry limb, for a chain whose carry lands on position 18, which never overflows (see sqr_iter).
template <int N>
__device__ __forceinline__ void chain_n1(uint32_t* p, uint32_t& c, const uint32_t* x, const uint32_t m) {
  mad_pair_first(p[0], p[1], x[0], m);
#pragma unroll
  for (int i = 1; i < N; i++) mad_pair_next(p[2 * i], p[2 * i + 1], x[2 * i], m);
  asm volatile("addc.u32 %0, %0, 0;" : "+r"(c));
}

// One iteration of the squaring loop: the rows JJ and JJ + 1 of owner lane `owner` (JJ even, compile-time), then the
// reduction by two limbs exactly as in mont_mul.
template <int JJ>
__device__ __forceinline__ void sqr_iter(Acc<16>& A, uint32_t& cy1, const uint32_t (&a2)[17], const uint32_t (&n)[16],
                                         const uint32_t n0inv, const int r, const int gbase, const int owner) {
  constexpr int W = 16;
  const uint32_t lt1 = r < owner ? ~1u : 0u, nm = r < owner ? ~0u : ~1u, eqm = r == owner ? ~0u : 0u;
  // this lane's own limbs JJ and JJ + 1 (undoubled); the owner's are the round's multipliers
  const uint32_t aj0 = __funnelshift_r(a2[JJ], a2[JJ + 1], 1);
  const uint32_t aj1 = __funnelshift_r(a2[JJ + 1], a2[JJ + 2], 1);
  const uint32_t b0 = __shfl_sync(kFull, aj0, gbase + owner);
  const uint32_t b1 = __shfl_sync(kFull, aj1, gbase + owner);
  // row operands (window slot k <-> own limb k); only the first two limbs of a row differ from a2
  uint32_t m0[18], m1[18];
#pragma unroll
  for (int k = 0; k < 17; k++) { m0[k] = a2[k]; m1[k] = a2[k]; }
  m0[17] = 0u; m1[17] = 0u;
  // lt1 = lt ? ~1 : 0 (a doubled limb without the bit shifted in from the limb below), nm = lt ? ~0 : ~1, eqm = eq ? ~0 : 0
  m0[JJ] = (a2[JJ] & lt1) | (aj0 & eqm);
  m0[JJ + 1] = a2[JJ + 1] & nm;
  m1[JJ + 1] = (a2[JJ + 1] & lt1) | (aj1 & eqm);
  uint32_t top1 = a2[16];
  if (JJ + 2 < W) m1[JJ + 2] = a2[JJ + 2] & nm;
  else top1 = a2[16] & (lt1 >> 1);                    // row 15: limb 15 is doubled only for the lanes below the owner
  const uint32_t t0 = (0u - a2[16]) & b0;            // a2[16] (0/1) x b: lands on the even chain's first carry limb
  const uint32_t t1 = (0u - top1) & b1;
  // ---- offset 0 ---------------------------------------------------------------------------------------------
  chain_n<(W - JJ) / 2>(A.E + JJ, A.E[W], A.E[W + 1], m0 + JJ, b0, t0);                 // even limbs >= JJ      -> E pairs (k, k+1)
  uint32_t q0 = A.E[0] * n0inv;
  q0 = __shfl_sync(kFull, q0, gbase);
  chain_n<(W - JJ) / 2>(A.O + JJ, A.O[W], A.O[W + 1], m0 + JJ + 1, b0, 0u);             // odd limbs  >= JJ + 1  -> O pairs (k-1, k)
  chain_n<(W - JJ - 2) / 2>(A.O + JJ + 2, A.O[W], A.O[W + 1], m1 + JJ + 2, b1, t1);     // even limbs >= JJ + 2  -> O pairs (k, k+1)
  chain_n1<(W - JJ) / 2>(A.E + JJ + 2, A.O[W + 1], m1 + JJ + 1, b1);                       // odd limbs  >= JJ + 1  -> E pairs (k+1, k+2)
  mac_off0_even_nocin(A, n, q0);
  mac_off0_odd(A, n, q0);
  // ---- offset 1 ---------------------------------------------------------------------------------------------
  uint32_t q1 = (A.E[1] + A.O[0] + cy1) * n0inv;
  q1 = __shfl_sync(kFull, q1, gbase);
  Chain<W>::run_cin(A.O, A.O[W], A.O[W + 1], n, q1, cy1);                              // mac_off1_even, cy1 enters at position 1
  chain_n1<W / 2>(A.E + 2, A.O[W + 1], n + 1, q1);                                      // mac_off1_odd, carry -> O[W + 1]
  // positions 0 and 1 leave the lane (lane 0's are zero, the others' go to the lane below).  Position 2, the next step's
  // position 0, becomes one limb: E[2] + O[1] + the carry out of position 1, whose own carry cy1 waits at position 1.
  const uint32_t p0 = A.E[0];
  uint32_t p1, e0;
  asm("add.cc.u32 %0, %3, %4; addc.cc.u32 %1, %5, %6; addc.u32 %2, 0, 0;"
      : "=r"(p1), "=r"(e0), "=r"(cy1) : "r"(A.E[1]), "r"(A.O[0]), "r"(A.E[2]), "r"(A.O[1]));
  uint32_t r0 = __shfl_down_sync(kFull, p0, 1, T);
  uint32_t r1 = __shfl_down_sync(kFull, p1, 1, T);
  if (r == T - 1) { r0 = 0u; r1 = 0u; }
  // Shift down two limbs.  E and O keep 16 limbs each plus two carry limbs that are zero when a step starts; E[W + 2]
  // and E[W + 3] are never used here.  A lane's accumulated value stays below 2^515 between steps and below 2^579 within
  // one, so position 18 (O[W + 1], where the chains into E[W]..E[W + 1] put their carry, one instruction each) holds a
  // few units and position 19 nothing, and after the shift position 16 (O[W - 1]) takes the carry of the two limbs from
  // the lane above without overflowing (tools/emu_sq.py asserts both).
#pragma unroll
  for (int k = 1; k < W; k++) A.E[k] = A.E[k + 2];
  A.E[0] = e0; A.E[W] = 0u; A.E[W + 1] = 0u;
#pragma unroll
  for (int k = 0; k < W; k++) A.O[k] = A.O[k + 2];
  A.O[W] = 0u; A.O[W + 1] = 0u;
  asm volatile("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, 0;"
               : "+r"(A.E[W - 2]), "+r"(A.E[W - 1]), "+r"(A.O[W - 1]) : "r"(r0), "r"(r1));
}

// out = a * a * R^-1 mod n, out < R ("almost Montgomery"), R = 2^2048.  All 32 lanes of the warp call this together.
__device__ __forceinline__ void mont_sqr(uint32_t (&out)[16], const uint32_t (&a)[16], const uint32_t (&n)[16], const uint32_t n0inv,
                                         const int r, const int gbase) {
  constexpr int W = 16;
  uint32_t a2[17];
  a2[0] = a[0] << 1;
#pragma unroll
  for (int k = 1; k < W; k++) a2[k] = __funnelshift_l(a[k - 1], a[k], 1);
  a2[16] = a[W - 1] >> 31;
  Acc<W> A;
#pragma unroll
  for (int k = 0; k < W + 4; k++) A.E[k] = 0u;
#pragma unroll
  for (int k = 0; k < W + 2; k++) A.O[k] = 0u;
  uint32_t cy1 = 0u;            // 1-bit carry pending at position 1
  // two owner steps per loop body: half the back-edge register moves of one step (2 % faster on H100, DESIGN.md §4)
#pragma unroll 2
  for (int owner = 0; owner < T; owner++) {
    sqr_iter<0>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<2>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<4>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<6>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<8>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<10>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<12>(A, cy1, a2, n, n0inv, r, gbase, owner);
    sqr_iter<14>(A, cy1, a2, n, n0inv, r, gbase, owner);
  }
  // cy1 into O (position 1 on): the value bound keeps the ripple inside O[W - 1]
  asm volatile("add.cc.u32 %0, %0, %1;" : "+r"(A.O[0]) : "r"(cy1));
#pragma unroll
  for (int k = 1; k < W; k++) asm volatile("addc.cc.u32 %0, %0, 0;" : "+r"(A.O[k]));
  mont_finish(out, A, 0u, 0u, n, r, gbase);
}

}  // namespace r32
}  // namespace bftq
