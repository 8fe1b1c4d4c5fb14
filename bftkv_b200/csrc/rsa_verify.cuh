// K1 — batched RSA PKCS#1 v1.5 signature verification for sm_90a.
//
// Replaces, for the bftkv hot path, the arithmetic that
//   crypto/pgp/crypto_pgp.go:324,338,454,490  ->  openpgp.CheckDetachedSignature / ReadMessage
//   -> packet.PublicKey.VerifySignature -> rsa.VerifyPKCS1v15 -> big.Int.Exp
// performs on the CPU:  m = s^e mod n,  then EM == 00 01 FF..FF 00 || DigestInfo || digest.
//
// Design (see DESIGN.md §4 K1; the general path beside the radix-2^32 kernel of rsa_verify_r32.cuh):
//  * Big numbers are held in radix 2^28 ("lazy carry"): every partial product is
//    < 2^56 and up to ~2^7 of them are summed in a 64-bit accumulator with plain IMAD.WIDE —
//    no carry flag anywhere in the inner loop.
//  * A signature is owned by a group of T lanes (T = 4 or 8); each lane keeps W digits of the
//    operand, of the modulus and W 64-bit column accumulators in registers.  One Montgomery
//    step = broadcast b_i (SHFL), W MACs, q (1 IMAD + SHFL), W MACs, shift one digit down the
//    group (1 SHFL).  R = 2^(28*T*W) > 2^24 * n, so no conditional subtraction is ever needed
//    between multiplications (Walter's bound), only one canonicalisation at the very end.
//  * e = 65537 costs 1 (to Montgomery form) + 16 squarings + 1 multiply by the PLAIN s (which
//    also leaves Montgomery form) = 18 Montgomery products.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "mont_r32.cuh"

namespace bftq {

constexpr int kDigitBits = 28;
constexpr uint32_t kDigitMask = (1u << kDigitBits) - 1u;
constexpr int kMaxDigits = 152;      // digits kept per key (4096-bit class: 8 lanes x 19)

// Key-size classes: k = modulus bytes (what Go's pub.Size() returns).  Digit layout per class:
//   k=128 (1024 bit): 4 lanes x 10 digits    k=192 (1536): 4 x 14    k=256 (2048): 4 x 19
//   k=384 (3072 bit): 8 lanes x 14 digits    k=512 (4096): 8 x 19
// T*W*28 >= 8k + 24 always, so R > 2^24 n and Montgomery products never need a conditional subtraction.
__host__ __device__ constexpr int class_digits(int kb) {
  return kb == 128 ? 40 : kb == 192 ? 56 : kb == 256 ? 76 : kb == 384 ? 112 : kb == 512 ? 152 : 0;
}
__host__ inline bool class_supported(int kb) { return kb == 128 || kb == 192 || kb == 256 || kb == 384 || kb == 512; }
// Key-size class that carries a modulus of kb = ceil(bits / 8) bytes: the smallest built class that holds it
// (0: larger than any).  A 2056-bit key (k = 257) runs in the 384-byte class: its signatures are left-padded to
// the class stride, the arithmetic is the same Montgomery product with a larger R, and EM is built for k = 257.
__host__ __device__ constexpr int class_of(int kb) { return kb < 1 ? 0 : kb <= 128 ? 128 : kb <= 192 ? 192 : kb <= 256 ? 256 : kb <= 384 ? 384 : kb <= 512 ? 512 : 0; }

// Per-key constants, precomputed on the host at bftq_register_rsa_keys().
struct RsaKeyDev {
  uint32_t n[kMaxDigits];                 // modulus, radix 2^28, little-endian digits, zero padded
  uint32_t r2[kMaxDigits];                // R^2 mod n for R = 2^(28*class_digits(class_of(kbytes)))
  uint32_t n0inv;                         // -n^-1 mod 2^28
  uint32_t e;                             // public exponent (>= 1)
  uint32_t nbits;
  uint32_t kbytes;                        // k = ceil(nbits / 8) = pub.Size(): the length of EM and of a signature
};

// DigestInfo prefixes, identical to Go's crypto/rsa hashPrefixes (and to the copy in the
// reference, crypto/threshold/rsa/rsa.go:345-354), indexed by OpenPGP hash id.
struct HashPrefix { uint8_t len; uint8_t dlen; uint8_t bytes[19]; };
__constant__ HashPrefix c_hash_prefix[12] = {
  {0, 0, {0}},
  {18, 16, {0x30, 0x20, 0x30, 0x0c, 0x06, 0x08, 0x2a, 0x86, 0x48, 0x86, 0xf7, 0x0d, 0x02, 0x05, 0x05, 0x00, 0x04, 0x10}},  // 1 MD5
  {15, 20, {0x30, 0x21, 0x30, 0x09, 0x06, 0x05, 0x2b, 0x0e, 0x03, 0x02, 0x1a, 0x05, 0x00, 0x04, 0x14}},                    // 2 SHA-1
  {14, 20, {0x30, 0x20, 0x30, 0x08, 0x06, 0x06, 0x28, 0xcf, 0x06, 0x03, 0x00, 0x31, 0x04, 0x14}},                          // 3 RIPEMD-160
  {0, 0, {0}}, {0, 0, {0}}, {0, 0, {0}}, {0, 0, {0}},
  {19, 32, {0x30, 0x31, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x01, 0x05, 0x00, 0x04, 0x20}},  // 8 SHA-256
  {19, 48, {0x30, 0x41, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x02, 0x05, 0x00, 0x04, 0x30}},  // 9 SHA-384
  {19, 64, {0x30, 0x51, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x03, 0x05, 0x00, 0x04, 0x40}},  // 10 SHA-512
  {19, 28, {0x30, 0x2d, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x04, 0x05, 0x00, 0x04, 0x1c}},  // 11 SHA-224
};

__host__ inline int host_hash_dlen(uint32_t id) {
  switch (id) { case 1: return 16; case 2: return 20; case 3: return 20; case 8: return 32; case 9: return 48; case 10: return 64; case 11: return 28; default: return 0; }
}

// ---- little helpers --------------------------------------------------------------------------

// Byte i (big-endian position, 0 = most significant) of EMSA-PKCS1-v1_5(digest), k = KB.
// Mirrors the layout rsa.VerifyPKCS1v15 checks: 00 01 FF.. 00 prefix digest.
template <int KB = kRsaBytes>
__device__ __forceinline__ uint32_t em_byte(int i, const uint8_t* digest, int plen, int dlen, uint32_t hash_alg) {
  const int tlen = plen + dlen;
  const int t0 = KB - tlen;
  if (i >= t0) {
    int t = i - t0;
    return t < plen ? (uint32_t)c_hash_prefix[hash_alg].bytes[t] : (uint32_t)__ldg(digest + (t - plen));
  }
  if (i == 0) return 0u;
  if (i == 1) return 1u;
  if (i == t0 - 1) return 0u;
  return 0xFFu;
}
template <int KB = kRsaBytes>
__device__ __forceinline__ uint32_t em_word(int k, const uint8_t* digest, int plen, int dlen, uint32_t hash_alg) {
  if (k >= KB / 4) return 0u;
  const int b = (KB - 4) - 4 * k;
  return (em_byte<KB>(b, digest, plen, dlen, hash_alg) << 24) | (em_byte<KB>(b + 1, digest, plen, dlen, hash_alg) << 16) |
         (em_byte<KB>(b + 2, digest, plen, dlen, hash_alg) << 8) | em_byte<KB>(b + 3, digest, plen, dlen, hash_alg);
}

// The same with the key's own length k (bytes) at run time, for the size-class kernels: byte i of the k-byte EM,
// and the 32-bit little-endian word w of EM read as a number (zero above k bytes).
__device__ __forceinline__ uint32_t em_byte_k(int i, int k, const uint8_t* digest, int plen, int dlen, uint32_t hash_alg) {
  const int t0 = k - (plen + dlen);
  if (i >= t0) {
    const int t = i - t0;
    return t < plen ? (uint32_t)c_hash_prefix[hash_alg].bytes[t] : (uint32_t)__ldg(digest + (t - plen));
  }
  if (i == 0) return 0u;
  if (i == 1) return 1u;
  if (i == t0 - 1) return 0u;
  return 0xFFu;
}
__device__ __forceinline__ uint32_t em_word_k(int w, int k, const uint8_t* digest, int plen, int dlen, uint32_t hash_alg) {
  uint32_t v = 0u;
#pragma unroll
  for (int t = 0; t < 4; t++) {
    const int j = 4 * w + t;                       // byte offset from the least significant end
    if (j < k) v |= em_byte_k(k - 1 - j, k, digest, plen, dlen, hash_alg) << (8 * t);
  }
  return v;
}

// ---- Montgomery product, radix 2^28, T lanes x W digits ---------------------------------------
// out = a * b * R^-1 mod n (value < a*b/R + n), digits "almost normalised" (< 2^28 + 2^10).
// All 32 lanes of the warp must call this together.
template <int T, int W>
__device__ __forceinline__ void mont_mul(uint32_t (&out)[W], const uint32_t (&a)[W], const uint32_t (&b)[W],
                                         const uint32_t (&n)[W], const uint32_t n0inv, const int r, const int gbase) {
  static_assert(W >= 2, "need two digits per lane");
  uint64_t acc[W];
#pragma unroll
  for (int j = 0; j < W; j++) acc[j] = 0ull;

#pragma unroll 1
  for (int owner = 0; owner < T; owner++) {
    const int src = gbase + owner;
#pragma unroll
    for (int jj = 0; jj < W; jj++) {
      const uint32_t bi = __shfl_sync(kFull, b[jj], src);
      acc[0] += (uint64_t)a[0] * bi;
      // Montgomery quotient digit: only lane 0 of the group holds column 0 of the number.
      uint32_t q = ((uint32_t)acc[0] * n0inv) & kDigitMask;
      q = __shfl_sync(kFull, q, gbase);
#pragma unroll
      for (int j = 1; j < W; j++) acc[j] += (uint64_t)a[j] * bi;
#pragma unroll
      for (int j = 0; j < W; j++) acc[j] += (uint64_t)n[j] * q;
      // Shift the whole number one digit down.  Column 0 of lane 0 is now == 0 mod 2^28; for the
      // other lanes its low 28 bits belong to the top column of the lane below, the rest is a
      // carry into the lane's own column 1.
      const uint32_t low = (uint32_t)acc[0] & kDigitMask;
      uint32_t recv = __shfl_down_sync(kFull, low, 1, T);
      if (r == T - 1) recv = 0u;
      acc[1] += acc[0] >> kDigitBits;
#pragma unroll
      for (int j = 0; j < W - 1; j++) acc[j] = acc[j + 1];
      acc[W - 1] = (uint64_t)recv;
    }
  }
  // Local carry ripple, then hand the lane's carry-out to the lane above.
  uint64_t c = 0ull;
#pragma unroll
  for (int j = 0; j < W; j++) {
    const uint64_t v = acc[j] + c;
    out[j] = (uint32_t)v & kDigitMask;
    c = v >> kDigitBits;
  }
  uint32_t clo = __shfl_up_sync(kFull, (uint32_t)c, 1, T);
  uint32_t chi = __shfl_up_sync(kFull, (uint32_t)(c >> 32), 1, T);
  if (r == 0) { clo = 0u; chi = 0u; }
  const uint64_t v0 = (uint64_t)out[0] + (((uint64_t)chi << 32) | clo);
  out[0] = (uint32_t)v0 & kDigitMask;
  out[1] += (uint32_t)(v0 >> kDigitBits);   // <= 2^9: digit stays < 2^28 + 2^10
}

// Make the digits canonical (every digit < 2^28) — carries may ripple through all T lanes.
template <int T, int W>
__device__ __forceinline__ void canonicalise(uint32_t (&y)[W], const int r) {
  uint32_t cout = 0u;
#pragma unroll
  for (int round = 0; round < T; round++) {
    uint32_t c = __shfl_up_sync(kFull, cout, 1, T);
    if (r == 0 || round == 0) c = 0u;
#pragma unroll
    for (int j = 0; j < W; j++) {
      const uint32_t v = y[j] + c;
      y[j] = v & kDigitMask;
      c = v >> kDigitBits;
    }
    cout = c;
  }
}

// ---- the kernel -------------------------------------------------------------------------------
// One group of T lanes per signature; a warp handles 32/T signatures per pass and strides over
// the batch.
template <int T, int W, int BLOCK, int KB>
__global__ void __launch_bounds__(BLOCK)
rsa_verify_kernel(const RsaKeyDev* __restrict__ keys, const uint32_t nkeys, const uint32_t* __restrict__ key_idx,
                  const uint8_t* __restrict__ sig, const uint8_t* __restrict__ digest, const uint32_t hash_alg,
                  const uint64_t n_items, const uint32_t flags, const uint8_t* __restrict__ pre_status,
                  uint8_t* __restrict__ status) {
  static_assert(T * W == class_digits(KB), "digit layout does not match the key-size class");
  static_assert(T * W * kDigitBits >= 8 * KB + 24, "R must exceed 2^24 n");
  constexpr int kGroupsPerWarp = 32 / T;
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int plen = c_hash_prefix[hash_alg].len;
  const int dlen = c_hash_prefix[hash_alg].dlen;
  const uint64_t warp_global = (uint64_t)blockIdx.x * (BLOCK / 32) + (threadIdx.x >> 5);
  const uint64_t warps_total = (uint64_t)gridDim.x * (BLOCK / 32);

  for (uint64_t wbase = warp_global * kGroupsPerWarp; wbase < n_items; wbase += warps_total * kGroupsPerWarp) {
    const uint64_t item_raw = wbase + (uint64_t)(lane / T);
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : (n_items - 1);   // idle groups shadow the last item
    uint32_t kidx = __ldg(key_idx + item);
    const bool known = kidx < nkeys;
    if (!known) kidx = 0u;
    const RsaKeyDev* __restrict__ key = keys + kidx;
    // k = pub.Size().  rsa.VerifyPKCS1v15: "if k < tLen+11 return ErrVerification" and "k != len(sig)" — the
    // signature travels left-padded to the class stride KB >= k, so a non-zero byte above its low k bytes means
    // the caller's signature was longer than k.
    const int kk = (int)__ldg(&key->kbytes);
    bool wrong_class = class_of(kk) != KB || kk < plen + dlen + 11;     // (a key of another class has the wrong R^2)

    uint32_t nd[W], xs[W], xm[W], y[W];
#pragma unroll
    for (int j = 0; j < W; j++) nd[j] = __ldg(&key->n[r * W + j]);
    const uint32_t n0inv = __ldg(&key->n0inv);
    const uint32_t e = __ldg(&key->e);

    // s -> radix 2^28 digits (canonical).
    const uint8_t* sp = sig + item * (uint64_t)KB;
    if (kk < KB) {
      bool longer = false;
      for (int i = r; i < KB - kk; i += T) longer = longer || (__ldg(sp + i) != 0);
      wrong_class = wrong_class || ((__ballot_sync(kFull, longer) >> gbase) & ((T == 32) ? 0xffffffffu : ((1u << T) - 1u))) != 0u;
    }
#pragma unroll
    for (int j = 0; j < W; j++) {
      const int o = kDigitBits * (r * W + j);
      const int wi = o >> 5, sh = o & 31;
      xs[j] = __funnelshift_r(be_word<KB>(sp, wi), be_word<KB>(sp, wi + 1), sh) & kDigitMask;
    }
    // s >= n ?  (lexicographic compare across the group, most significant lane wins)
    bool gt = false, lt = false;
#pragma unroll
    for (int j = W - 1; j >= 0; j--) {
      if (!gt && !lt) { gt = xs[j] > nd[j]; lt = xs[j] < nd[j]; }
    }
    const uint32_t gmask = (T == 32) ? 0xffffffffu : (((1u << T) - 1u) << gbase);
    const uint32_t gtb = __ballot_sync(kFull, gt) & gmask;
    const uint32_t ltb = __ballot_sync(kFull, lt) & gmask;
    const bool s_ge_n = gtb >= ltb;

    // xm = s * R mod n
    {
      uint32_t r2[W];
#pragma unroll
      for (int j = 0; j < W; j++) r2[j] = __ldg(&key->r2[r * W + j]);
      mont_mul<T, W>(xm, xs, r2, nd, n0inv, r, gbase);
    }
    // Left-to-right square and multiply over the bits of e above bit 0.  Control flow is kept
    // warp-uniform (the shuffles inside mont_mul need all lanes); groups whose exponent is
    // shorter simply do not commit the result.
    const int nb = 32 - __clz(e);                       // e >= 1
    int nbmax = nb;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) nbmax = max(nbmax, __shfl_xor_sync(kFull, nbmax, o));
#pragma unroll
    for (int j = 0; j < W; j++) y[j] = xm[j];
#pragma unroll 1
    for (int bit = nbmax - 2; bit >= 1; bit--) {
      const bool active = bit <= nb - 2;
      uint32_t t[W];
      mont_mul<T, W>(t, y, y, nd, n0inv, r, gbase);
      if (active) {
#pragma unroll
        for (int j = 0; j < W; j++) y[j] = t[j];
      }
      const bool mul = active && ((e >> bit) & 1u);
      if (__any_sync(kFull, mul)) {
        mont_mul<T, W>(t, y, xm, nd, n0inv, r, gbase);
        if (mul) {
#pragma unroll
          for (int j = 0; j < W; j++) y[j] = t[j];
        }
      }
    }
    // bit 0: last squaring (if e has more than one bit), then multiply by the PLAIN s (bit 0 set)
    // or by plain 1 (bit 0 clear).  A Montgomery product with a plain operand leaves Montgomery
    // form, so the result is s^e mod n itself.
    {
      uint32_t t[W];
      if (__any_sync(kFull, nb >= 2)) {
        mont_mul<T, W>(t, y, y, nd, n0inv, r, gbase);
        if (nb >= 2) {
#pragma unroll
          for (int j = 0; j < W; j++) y[j] = t[j];
        }
      }
      uint32_t m1[W];
#pragma unroll
      for (int j = 0; j < W; j++) m1[j] = ((e & 1u) && nb >= 2) ? xs[j] : ((r == 0 && j == 0) ? 1u : 0u);   // e == 1: bit 0 is the top bit, already in y
      mont_mul<T, W>(t, y, m1, nd, n0inv, r, gbase);
#pragma unroll
      for (int j = 0; j < W; j++) y[j] = t[j];
    }
    canonicalise<T, W>(y, r);

    // Compare with the expected encoded message.  y < n(1 + 2^-24), and y == EM + n would need EM < 2^-24 n while
    // EM = 00 01 FF.. is at least 2^-16 n for a modulus of k bytes, so a canonical digit compare decides.
    const uint8_t* dp = digest + item * (uint64_t)dlen;
    bool eq = true;
#pragma unroll
    for (int j = 0; j < W; j++) {
      const int o = kDigitBits * (r * W + j);
      const int wi = o >> 5, sh = o & 31;
      const uint32_t lo = em_word_k(wi, kk, dp, plen, dlen, hash_alg);
      const uint32_t hi = em_word_k(wi + 1, kk, dp, plen, dlen, hash_alg);
      const uint32_t emd = __funnelshift_r(lo, hi, sh) & kDigitMask;
      eq = eq && (emd == y[j]);
    }
    const uint32_t eqb = __ballot_sync(kFull, eq) & gmask;
    if (valid && r == 0) {
      uint8_t st = (eqb == gmask) ? (uint8_t)0 : (uint8_t)1;         // BFTQ_ST_OK / BFTQ_ST_BAD_SIGNATURE
      if ((flags & 1u) && s_ge_n) st = 1;                             // BFTQ_F_STRICT_RANGE
      if (wrong_class) st = 1;
      if (!known) st = 4;                                             // BFTQ_ST_UNKNOWN_SIGNER
      if (pre_status != nullptr) {                                    // decided by the packer (missing, malformed ...)
        const uint8_t pre = __ldg(pre_status + item_raw);
        if (pre != 0) st = pre;
      }
      status[item_raw] = st;
    }
  }
}

}  // namespace bftq
