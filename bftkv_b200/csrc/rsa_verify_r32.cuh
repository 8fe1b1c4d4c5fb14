// K1 (fast path) — RSA-2048 PKCS#1 v1.5 batch verify, radix 2^32 with IMAD.WIDE.U32.X carry chains.
//
// Same contract as rsa_verify.cuh (the radix-2^28 kernel, kept for moduli of 2041..2047 bits); this
// variant requires the modulus to have exactly 2048 bits, which is what every RSA-2048 key
// generator (gpg, OpenSSL, Go) produces.
// A signature is owned by 4 lanes x 16 32-bit limbs; the general product is mont_mul (mont_r32.cuh), the squarings
// mont_sqr (rsa_square_r32.cuh).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "rsa_verify.cuh"
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
