// K10 — the client half of threshold password authentication (crypto/auth/auth.go:239-399 AuthClient: Initiate,
// ProcessResponse's processYi / processBi / processZi, GetCipherKey) on the device, around K9's kernels (auth_server.cuh):
//
//   auth_zq_kernel          dst = A * B mod q, q = (p - 1) / 2, one 4-lane group per item, two mont_mul<16, true> products
//                           and a masked final subtraction.  A and B are 64-word values in device memory, or H =
//                           SHA-256(h1 || h2) computed in the group's lane 0:  PI(pw) = H(pw) * H(pw) (below 2^512 < q, so
//                           the product is exact), e_i = a'_i * H(pw || salt_i) (phase 0), f_i = a * a'_i (phase 1).
//                           `keep` (nullable) receives A: phase 0 stores a'_i in the session's slot this way.
//   auth_words_kernel       256 big-endian bytes -> 64 little-endian words (K5's gs and K9's a^-1 mod q become bases and
//                           exponents of auth_pow_kernel), and sets a flag word.  One thread per item.
//   auth_cipher_key_kernel  GetCipherKey's SHA-256(gs'.Bytes() || pw), gs' = gs^(a^-1) a row of auth_pow_kernel's output.
//   auth_gcm_open_kernel    phase 2: AES-128-GCM(ke).Open(nonce, Zi, aad = Ni): GHASH over Ni and the ciphertext, the tag
//                           compared by ORing the differences of its 16 bytes, and only then the plain text.  One thread
//                           per item; gcm_core is the seal's.
// The exponentiations are auth_pow_kernel's (X = PI^a, Xi = gs^e, Ki = Bi^f, gs^(a^-1) over p; a^(q-2) over q), keySched and
// the MAC auth_kdf_mac_kernel's, and gs = prod Yi^lambda_i is K3 + K5 over public Yi and lambda.
//
// Secrets: pw, a, a^-1, a', si, e, f, gs, Ki, km and ke.  Constant time as K9: every exponent is read as 512 windows of 64
// words, every Z_q product is mont_mul<16, true>, no branch or index depends on a secret.  The trip counts that depend on
// data are SHA-256's over the password's length (and the public salt's), and over the lengths of Ki and gs', which the
// reference leaks the same way (they feed keySched and the hash as minimal encodings).
// No K10 kernel uses local memory (tests/test_auth_client_host.py checks the SASS).
#pragma once
#include <cstdint>
#include "auth_server.cuh"

namespace bftq {
namespace k10 {

using k9::AuthGroup;
using k9::kAuthBytes;

// A session's device allocation: the header, n slots, then the password bytes.  The salt's HMAC key block is public and
// travels with each phase-1 item instead.
struct ClientHeader {
  uint32_t a[64];                        // a, little-endian words (secret)
  uint32_t ainv[64];                     // a^-1 mod q (secret)
  uint32_t gs[64];                       // the shared secret gs (secret)
  uint32_t has_gs;
  uint32_t pw_len;
  uint32_t pad[2];
};
struct ClientSlot {
  uint32_t a2[64];                       // a'_i (secret)
  uint8_t ke[16];                        // phase 1's encryption key (secret) ...
  uint32_t has_ke;                       // ... and whether phase 1 set it
  uint32_t pad[3];
};

#ifdef __CUDACC__
using r32::T;

// dst = A * B mod q.  a, b: 64 little-endian words, or 0 for H = SHA-256(h1 (h1_len bytes) || h2 (h2_len bytes)).
struct ZqItem { uint64_t a, b, dst, keep, h1, h2; uint32_t h1_len, h2_len; };

struct HashSrc {
  const uint8_t* a; uint64_t al; const uint8_t* b;
  __device__ __forceinline__ uint32_t operator()(uint64_t pos) const { return pos < al ? a[pos] : b[pos - al]; }
};

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
auth_zq_kernel(const AuthGroup* __restrict__ Gq, const ZqItem* __restrict__ items, const uint64_t n_items) {
  constexpr int W = 16;
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int grp = threadIdx.x / T;
  for (uint64_t base = (uint64_t)blockIdx.x * (BLOCK / T); base < n_items; base += (uint64_t)gridDim.x * (BLOCK / T)) {
    const uint64_t item_raw = base + (uint64_t)grp;
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : n_items - 1;
    const ZqItem it = items[item];
    uint32_t h[8];
#pragma unroll
    for (int j = 0; j < 8; j++) h[j] = 0u;
    if (r == 0 && (it.a == 0 || it.b == 0)) {
      k9::sha256_init(h);
      k9::sha256_tail(h, HashSrc{reinterpret_cast<const uint8_t*>(it.h1), it.h1_len, reinterpret_cast<const uint8_t*>(it.h2)},
                      (uint64_t)it.h1_len + it.h2_len, 0);
    }
    __syncwarp();
    const uint32_t* aw = reinterpret_cast<const uint32_t*>(it.a);
    const uint32_t* bw = reinterpret_cast<const uint32_t*>(it.b);
    uint32_t A[W], B[W], q[W], r2[W], t[W], o[W];
#pragma unroll
    for (int j = 0; j < W; j++) {
      const uint32_t hj = (r == 0 && j < 8) ? h[7 - j] : 0u;     // H read as a big-endian integer
      A[j] = aw ? aw[r * W + j] : hj;
      B[j] = bw ? bw[r * W + j] : hj;
      q[j] = __ldg(&Gq->p[r * W + j]);
      r2[j] = __ldg(&Gq->r2[r * W + j]);
    }
    const uint32_t n0inv = __ldg(&Gq->n0inv);
    r32::mont_mul<W, true>(t, A, B, q, n0inv, r, gbase);             // A B R^-1, < R
    r32::mont_mul<W, true>(o, t, r2, q, n0inv, r, gbase);            // A B mod q, < 2q
    r32::cond_sub<W, true>(o, q, r, gbase);
    if (valid) {
      uint32_t* dw = reinterpret_cast<uint32_t*>(it.dst);
      uint32_t* kw = reinterpret_cast<uint32_t*>(it.keep);
#pragma unroll
      for (int j = 0; j < W; j++) dw[r * W + j] = o[j];
      if (kw) {
#pragma unroll
        for (int j = 0; j < W; j++) kw[r * W + j] = A[j];
      }
    }
    __syncwarp();
  }
}

// dst (64 words) = the 256 big-endian bytes at src; *flag = 1 when flag != 0.
struct WordsItem { uint64_t src, dst, flag; };

__global__ void __launch_bounds__(128)
auth_words_kernel(const WordsItem* __restrict__ items, const uint64_t n_items) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const WordsItem it = items[i];
  const uint8_t* s = reinterpret_cast<const uint8_t*>(it.src);
  uint32_t* d = reinterpret_cast<uint32_t*>(it.dst);
#pragma unroll 4
  for (int j = 0; j < 64; j++) {
    const uint8_t* w = s + kAuthBytes - 4 - 4 * j;
    d[j] = ((uint32_t)w[0] << 24) | ((uint32_t)w[1] << 16) | ((uint32_t)w[2] << 8) | w[3];
  }
  if (it.flag) *reinterpret_cast<uint32_t*>(it.flag) = 1u;
}

// out (32 bytes) = SHA-256(gs'.Bytes() || pw); gs' is row `row` of auth_pow_kernel's output.
struct KeyItem { uint64_t pw, out; uint32_t pw_len, row; };

__global__ void __launch_bounds__(128)
auth_cipher_key_kernel(const KeyItem* __restrict__ items, const uint64_t n_items, const uint8_t* __restrict__ pow_be,
                       const uint32_t* __restrict__ pow_len) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const KeyItem it = items[i];
  const uint32_t gl = pow_len[it.row];
  uint32_t h[8];
  k9::sha256_init(h);
  k9::sha256_tail(h, HashSrc{pow_be + (uint64_t)it.row * kAuthBytes + (kAuthBytes - gl), gl, reinterpret_cast<const uint8_t*>(it.pw)},
                  (uint64_t)gl + it.pw_len, 0);
  uint8_t* o = reinterpret_cast<uint8_t*>(it.out);
#pragma unroll
  for (int k = 0; k < 8; k++)
#pragma unroll
    for (int b = 0; b < 4; b++) o[4 * k + b] = (uint8_t)(h[k] >> (24 - 8 * b));
}

// Phase 2.  ke / has_ke: the slot's key and flag; aad: Ni (aad_len 32 or 0); ct: Zi, ct_len + 16 bytes (ciphertext ||
// tag); nonce: 12 bytes; out: ct_len bytes of plain text, written only when the tag matches.
struct OpenItem { uint64_t ke, has_ke, aad, ct, nonce, out; uint32_t aad_len, ct_len; };

// ok[i] = 1 when the tag matched (and out holds the plain text), 0 otherwise.
__global__ void __launch_bounds__(k6::K6B_BLOCK)
auth_gcm_open_kernel(const OpenItem* __restrict__ items, const uint64_t n_items, uint8_t* __restrict__ ok) {
  __shared__ uint8_t sb[256];
  __shared__ uint32_t rk[44 * k6::K6B_BLOCK];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sb[i] = k6::c_aes_sbox[i];
  __syncthreads();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_items) {
    const OpenItem it = items[i];
    const uint8_t* ct = reinterpret_cast<const uint8_t*>(it.ct);
    const uint8_t* nn = reinterpret_cast<const uint8_t*>(it.nonce);
    const uint8_t* aad = reinterpret_cast<const uint8_t*>(it.aad);
    const uint32_t n0 = k6::load_be32(nn, 0, 12), n1 = k6::load_be32(nn, 4, 12), n2 = k6::load_be32(nn, 8, 12);
    k6::aes_expand<4>(reinterpret_cast<const uint8_t*>(it.ke), rk, sb);
    uint8_t tag[16];
    k9::gcm_core(k9::AesEnc{rk, sb}, n0, n1, n2, aad, it.aad_len, ct, it.ct_len, nullptr, false, tag);
    uint32_t diff = *reinterpret_cast<const uint32_t*>(it.has_ke) ^ 1u;
#pragma unroll
    for (int b = 0; b < 16; b++) diff |= (uint32_t)(tag[b] ^ ct[it.ct_len + b]);
    const bool good = diff == 0u;
    if (good) k9::gcm_core(k9::AesEnc{rk, sb}, n0, n1, n2, aad, it.aad_len, ct, it.ct_len, reinterpret_cast<uint8_t*>(it.out), false, tag);
    ok[i] = good ? 1 : 0;
  }
#pragma unroll 1
  for (int k = 0; k < 44; k++) rk[k * k6::K6B_BLOCK + threadIdx.x] = 0u;       // no key schedule left in shared memory
}
#endif

}  // namespace k10
}  // namespace bftq
