// K9 — the server half of threshold password authentication (crypto/auth/auth.go:168-237 AuthServer.MakeResponse) on
// the device.
//
//   auth_pow_kernel        out = base^e mod p over the fixed 2048-bit safe prime of crypto/auth: phase 0's Yi = X^y, and
//                          phase 1's Bi = v^b and Ki = Xi^b.  One 4-lane group per item, r32::ct_window_pow.
//   auth_kdf_mac_kernel    phase 1: keySched (HKDF-SHA256, salt as the extract key, Ki.Bytes() as the input key material,
//                          nil info; km = OKM[0:16], ke = OKM[16:32]) and the MAC HMAC-SHA256(km, Xi || Bi.Bytes()).
//                          One thread per item; writes ke and the MAC where the item says: the server's allocation, or
//                          for the client half (auth_client.cuh) the session's slot and the per-call buffer.
//   auth_gcm_seal_kernel   phase 2: the MAC check (constant time) and AES-128-GCM(ke).Seal(nonce, proof, aad = mac).
//                          One thread per item; wipes the server's phase-1 state whatever the outcome.
//
// Secrets: y, v, b, Ki, km, ke and the MAC.  Constant time means:
//  - every exponentiation reads 512 four-bit windows of a 64-word exponent, whatever the length of y or b, reads the
//    whole window table with masks, and every product is mont_mul<16, true>; the table is zeroed before the kernel exits;
//  - public bases of any length (X, Xi) are reduced mod p by Horner's rule over 2048-bit chunks; the trip count is the
//    chunk count of the warp's longest base (public);
//  - the minimal length of Ki is found with a masked scan; that length is the one value the reference also leaks
//    (Ki.Bytes() feeds keySched), and it sets the trip count of HKDF's extract.  Nothing else depends on Ki's value;
//  - HMAC and HKDF run sha256_compress over trip counts set by the lengths of Xi, Bi.Bytes() and Ki.Bytes();
//  - GHASH is a masked bit-serial carry-less multiply: no table indexed by anything derived from H;
//  - the MAC comparison ORs the differences of all 32 bytes.
// AES itself is K6b's (msg_decrypt.cuh), with the S-box in shared memory: the symmetric layer has the timing of the
// existing decrypt path.
// No K9 kernel uses local memory (tests/test_auth_host.py checks the SASS).
//
// The HMAC / HKDF, GHASH and GCM cores are __host__ __device__: tests/harness/auth_host.cpp builds them with g++.
#pragma once
#include <cstdint>
#include "sha256.cuh"
#ifdef __CUDACC__
#include "mont_r32.cuh"
#include "msg_decrypt.cuh"
#endif

namespace bftq {
namespace k9 {

constexpr int kAuthBytes = 256;          // |p| = 2048 bits
constexpr int kSaltKeyMax = 64;          // HMAC's block: a longer salt is hashed first (host)

// The server's registered parameters and its phase-1 state, at the head of its device allocation; the proof follows.
struct AuthState {
  uint32_t y[64];                        // y, little-endian words (secret)
  uint32_t v[64];                        // v mod p, little-endian words (secret)
  uint32_t salt_key[16];                 // HMAC key block of the salt: big-endian words, zero-padded to 64 bytes
  uint8_t ke[16];                        // phase-1 state (secret): the encryption key ...
  uint8_t mac[32];                       // ... the MAC the client must echo ...
  uint32_t has_p1;                       // ... and whether a phase 1 ran since the last phase 2
  uint32_t proof_len;
  uint32_t pad[2];
};

// p, 2^4096 mod p and -p^-1 mod 2^32, radix 2^32 little-endian; built once per engine.
struct AuthGroup {
  uint32_t p[64];
  uint32_t r2[64];
  uint32_t n0inv;
  uint32_t pad[3];
};

BFTQ_SHA_HD_FI void sha256_init(uint32_t (&h)[8]) {
  h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
  h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
}

// Compresses len message bytes src(0 .. len) and SHA-256's padding, after `done` bytes already compressed (a multiple
// of 64).  The trip count depends on len only.
template <class Src>
BFTQ_SHA_HD_FI void sha256_tail(uint32_t (&h)[8], const Src& src, const uint64_t len, const uint64_t done) {
  const uint64_t nblocks = (len + 9 + 63) / 64, total = (done + len) * 8;
  for (uint64_t blk = 0; blk < nblocks; blk++) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) {
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const uint64_t pos = blk * 64 + 4 * i + b;
        v = (v << 8) | (pos < len ? (uint32_t)src(pos) : (pos == len ? 0x80u : 0u));
      }
      w[i] = v;
    }
    if (blk == nblocks - 1) { w[14] = (uint32_t)(total >> 32); w[15] = (uint32_t)total; }
    sha256_compress(h, w);
  }
}

// HMAC-SHA256 with a key of at most 64 bytes given as its zero-padded block k (big-endian words).
template <class Src>
BFTQ_SHA_HD_FI void hmac_sha256(uint32_t (&out)[8], const uint32_t (&k)[16], const Src& src, const uint64_t len) {
  uint32_t w[16], h[8];
  sha256_init(h);
#pragma unroll
  for (int i = 0; i < 16; i++) w[i] = k[i] ^ 0x36363636u;
  sha256_compress(h, w);
  sha256_tail(h, src, len, 64);
  uint32_t o[8];
  sha256_init(o);
#pragma unroll
  for (int i = 0; i < 16; i++) w[i] = k[i] ^ 0x5c5c5c5cu;
  sha256_compress(o, w);
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = h[i];
  w[8] = 0x80000000u;
#pragma unroll
  for (int i = 9; i < 15; i++) w[i] = 0u;
  w[15] = (64 + 32) * 8;
  sha256_compress(o, w);
#pragma unroll
  for (int i = 0; i < 8; i++) out[i] = o[i];
}

struct OneByte {
  BFTQ_SHA_HD_FI uint32_t operator()(uint64_t) const { return 0x01u; }
};

// keySched: HKDF-SHA256(ikm, salt, nil info), 32 bytes of output as km (t[0..3]) and ke (t[4..7]), big-endian words.
template <class Src>
BFTQ_SHA_HD_FI void hkdf_sha256_32(uint32_t (&t)[8], const uint32_t (&salt_key)[16], const Src& ikm, const uint64_t ikm_len) {
  uint32_t prk[8], k[16];
  hmac_sha256(prk, salt_key, ikm, ikm_len);
#pragma unroll
  for (int i = 0; i < 16; i++) k[i] = i < 8 ? prk[i] : 0u;
  hmac_sha256(t, k, OneByte{}, 1);
}

// calculateMac: HMAC-SHA256(km, Xi || Bi)
struct TwoPart {
  const uint8_t* a; uint64_t al; const uint8_t* b;
  BFTQ_SHA_HD_FI uint32_t operator()(uint64_t pos) const { return pos < al ? a[pos] : b[pos - al]; }
};
BFTQ_SHA_HD_FI void auth_mac(uint32_t (&mac)[8], const uint32_t (&km)[4], const uint8_t* xi, const uint64_t xl, const uint8_t* bi, const uint64_t bl) {
  uint32_t k[16];
#pragma unroll
  for (int i = 0; i < 16; i++) k[i] = i < 4 ? km[i] : 0u;
  hmac_sha256(mac, k, TwoPart{xi, xl, bi}, xl + bl);
}

// x = x * h in GCM's GF(2^128) (NIST SP 800-38D, algorithm 1); each value is two big-endian 64-bit halves.  Bit-serial,
// every step a masked xor: the trip count and the memory accesses depend on nothing.
BFTQ_SHA_HD_FI void gf128_mul(uint64_t& xh, uint64_t& xl, const uint64_t hh, const uint64_t hl) {
  uint64_t zh = 0, zl = 0, vh = hh, vl = hl;
#pragma unroll 1
  for (int i = 0; i < 128; i++) {
    const uint64_t bit = i < 64 ? (xh >> (63 - i)) & 1u : (xl >> (127 - i)) & 1u;
    const uint64_t m = 0ull - bit;
    zh ^= vh & m; zl ^= vl & m;
    const uint64_t lsb = 0ull - (vl & 1u);
    vl = (vl >> 1) | (vh << 63);
    vh = (vh >> 1) ^ (0xe100000000000000ull & lsb);
  }
  xh = zh; xl = zl;
}

BFTQ_SHA_HD_FI void gcm_block(uint64_t& xh, uint64_t& xl, const uint32_t s0, const uint32_t s1, const uint32_t s2, const uint32_t s3,
                              const uint64_t hh, const uint64_t hl) {
  xh ^= ((uint64_t)s0 << 32) | s1;
  xl ^= ((uint64_t)s2 << 32) | s3;
  gf128_mul(xh, xl, hh, hl);
}

// Big-endian word j of the 16-byte block `blk` of p (len bytes), zero past the end.
BFTQ_SHA_HD_FI uint32_t gcm_word(const uint8_t* p, const uint64_t len, const uint64_t blk, const int j) {
  uint32_t v = 0;
  for (int b = 0; b < 4; b++) {
    const uint64_t pos = blk * 16 + 4 * j + b;
    v = (v << 8) | (pos < len ? (uint32_t)p[pos] : 0u);
  }
  return v;
}

// AES-GCM with a 12-byte nonce (n0, n1, n2: its big-endian words; NIST SP 800-38D): H = E(0), J0 = nonce || 1, block b of
// src (len bytes) is xored with E(inc32(J0) + b).  dst (nullable) receives src xor the key stream.  GHASH runs over aad
// (aad_len bytes) and the ciphertext, which is what dst receives when `seal`, else src; tag = GHASH xor E(J0).
// enc(s0, s1, s2, s3) encrypts one block in place under the key.  Trip counts depend on aad_len and len only.
template <class Enc>
BFTQ_SHA_HD_FI void gcm_core(const Enc& enc, const uint32_t n0, const uint32_t n1, const uint32_t n2, const uint8_t* aad, const uint64_t aad_len,
                             const uint8_t* src, const uint64_t len, uint8_t* dst, const bool seal, uint8_t (&tag)[16]) {
  uint32_t h0 = 0u, h1 = 0u, h2 = 0u, h3 = 0u;
  enc(h0, h1, h2, h3);
  const uint64_t hh = ((uint64_t)h0 << 32) | h1, hl = ((uint64_t)h2 << 32) | h3;
  uint64_t xh = 0, xl = 0;
#pragma unroll 1
  for (uint64_t blk = 0; blk * 16 < aad_len; blk++)
    gcm_block(xh, xl, gcm_word(aad, aad_len, blk, 0), gcm_word(aad, aad_len, blk, 1), gcm_word(aad, aad_len, blk, 2), gcm_word(aad, aad_len, blk, 3), hh, hl);
#pragma unroll 1
  for (uint64_t blk = 0; blk * 16 < len; blk++) {
    uint32_t k[4] = {n0, n1, n2, (uint32_t)(blk + 2)};                   // inc32(J0) + blk
    enc(k[0], k[1], k[2], k[3]);
    uint32_t c[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const uint64_t pos = blk * 16 + 4 * j + b;
        const uint32_t in = pos < len ? (uint32_t)src[pos] : 0u;
        const uint32_t by = pos < len ? (in ^ (uint8_t)(k[j] >> (24 - 8 * b))) : 0u;
        if (dst && pos < len) dst[pos] = (uint8_t)by;
        v = (v << 8) | (seal ? by : in);
      }
      c[j] = v;
    }
    gcm_block(xh, xl, c[0], c[1], c[2], c[3], hh, hl);
  }
  gcm_block(xh, xl, (uint32_t)((aad_len * 8) >> 32), (uint32_t)(aad_len * 8), (uint32_t)((len * 8) >> 32), (uint32_t)(len * 8), hh, hl);
  uint32_t s0 = n0, s1 = n1, s2 = n2, s3 = 1u;                               // J0
  enc(s0, s1, s2, s3);
  const uint64_t th = xh ^ (((uint64_t)s0 << 32) | s1), tl = xl ^ (((uint64_t)s2 << 32) | s3);
#pragma unroll
  for (int b = 0; b < 8; b++) { tag[b] = (uint8_t)(th >> (56 - 8 * b)); tag[8 + b] = (uint8_t)(tl >> (56 - 8 * b)); }
}

#ifdef __CUDACC__
using r32::T;
using k6::K6B_BLOCK;
using k6::c_aes_sbox;
using k6::aes_expand;
using k6::aes_encrypt;
using k6::load_be32;

constexpr int kPowBlock = 32;            // one warp per block, as K7: the 16-entry window table lives in shared memory

// One exponentiation: base (little-endian words, any count), exp (64 little-endian words).
struct PowItem { uint64_t base; uint64_t exp; uint32_t base_words, pad; };

// out_be[i]: base^e mod p, 256 bytes big-endian; out_len[i]: the length of its minimal encoding (big.Int.Bytes()).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK)
auth_pow_kernel(const AuthGroup* __restrict__ G, const PowItem* __restrict__ items, const uint64_t n_items, uint8_t* __restrict__ out_be,
                uint32_t* __restrict__ out_len) {
  constexpr int W = 16;
  __shared__ uint32_t tab[16][W][BLOCK];
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int grp = threadIdx.x / T;
  const int tid = threadIdx.x;
  for (uint64_t base = (uint64_t)blockIdx.x * (BLOCK / T); base < n_items; base += (uint64_t)gridDim.x * (BLOCK / T)) {
    const uint64_t item_raw = base + (uint64_t)grp;
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : n_items - 1;
    const uint32_t* __restrict__ bw = reinterpret_cast<const uint32_t*>(__ldg(&items[item].base));
    const uint32_t* __restrict__ ew = reinterpret_cast<const uint32_t*>(__ldg(&items[item].exp));
    const uint32_t nw = __ldg(&items[item].base_words);
    uint32_t nd[W], r2[W], acc[W], t[W], c[W], d[W];
#pragma unroll
    for (int j = 0; j < W; j++) { nd[j] = __ldg(&G->p[r * W + j]); r2[j] = __ldg(&G->r2[r * W + j]); acc[j] = 0u; }
    const uint32_t n0inv = __ldg(&G->n0inv);
    // base mod p by Horner's rule over 2048-bit chunks, most significant first: acc = acc 2^2048 + chunk mod p
    uint32_t nch = (nw + 63) / 64;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) nch = max(nch, __shfl_xor_sync(kFull, nch, o));
#pragma unroll 1
    for (uint32_t k = nch; k-- > 0;) {
      r32::mont_mul<W, true>(t, acc, r2, nd, n0inv, r, gbase);      // acc R mod p, < 2p
      r32::cond_sub<W, true>(t, nd, r, gbase);
#pragma unroll
      for (int j = 0; j < W; j++) {
        const uint32_t at = 64u * k + (uint32_t)(r * W + j);
        c[j] = at < nw ? __ldg(bw + at) : 0u;
      }
      r32::cond_sub<W, true>(c, nd, r, gbase);                      // chunk < 2^2048 < 2p
      const uint32_t carry = r32::group_add(acc, t, c, r, gbase);
      const uint32_t bo = r32::group_sub(d, acc, nd, r, gbase);
      r32::select_mask(acc, d, carry | (bo ^ 1u));
    }
    uint32_t y[W], bm[W];
    r32::mont_mul<W, true>(bm, acc, r2, nd, n0inv, r, gbase);        // Montgomery form of the base
#pragma unroll
    for (int j = 0; j < W; j++) c[j] = (r == 0 && j == 0) ? 1u : 0u;
    r32::mont_mul<W, true>(y, r2, c, nd, n0inv, r, gbase);          // R mod p: the Montgomery form of 1
    r32::ct_window_pow<W, BLOCK>(y, bm, nd, n0inv, ew, 64, 512, tab, r, gbase);
    r32::mont_mul<W, true>(t, y, c, nd, n0inv, r, gbase);           // leaves Montgomery form: <= p
    r32::cond_sub<W, true>(t, nd, r, gbase);
    uint8_t* o = out_be + item_raw * kAuthBytes;
    if (valid) store_be<W>(o, kAuthBytes, t, r);
    __syncwarp();
    if (valid && r == 0) {                                         // leading zero bytes, by a masked scan of all 256
      uint32_t seen = 0u, lz = 0u;
#pragma unroll 1
      for (int b = 0; b < kAuthBytes; b++) { seen |= (uint32_t)(o[b] != 0); lz += seen ^ 1u; }
      out_len[item_raw] = (uint32_t)kAuthBytes - lz;
    }
#pragma unroll
    for (int e = 0; e < 16; e++)                                     // no power of a base left in shared memory
#pragma unroll
      for (int j = 0; j < W; j++) tab[e][j][tid] = 0u;
    __syncwarp();
  }
}

// Phase 1's keys and MAC.  Ki is a row of auth_pow_kernel's output; Bi is that too (bi == 0: row bi_row, the server's own
// Bi) or bi_len bytes at bi (the client's, as received).  salt_key: the salt's HMAC key block; ke (16 bytes), mac (32
// bytes) and flag (set to 1) are where the results go.
struct KdfItem { uint64_t salt_key, ke, mac, flag, xi, bi; uint32_t xi_len, bi_len, ki_row, bi_row; };

struct KiBytes {
  const uint8_t* p;
  __device__ __forceinline__ uint32_t operator()(uint64_t pos) const { return p[pos]; }
};

__global__ void __launch_bounds__(128)
auth_kdf_mac_kernel(const KdfItem* __restrict__ items, const uint64_t n_items, const uint8_t* __restrict__ pow_be,
                    const uint32_t* __restrict__ pow_len) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const KdfItem it = items[i];
  const uint32_t* salt_key = reinterpret_cast<const uint32_t*>(it.salt_key);
  uint8_t* ke = reinterpret_cast<uint8_t*>(it.ke);
  uint8_t* mo = reinterpret_cast<uint8_t*>(it.mac);
  uint32_t sk[16], t[8], km[4], mac[8];
#pragma unroll
  for (int k = 0; k < 16; k++) sk[k] = salt_key[k];
  const uint32_t kl = pow_len[it.ki_row];
  hkdf_sha256_32(t, sk, KiBytes{pow_be + (uint64_t)it.ki_row * kAuthBytes + (kAuthBytes - kl)}, kl);
#pragma unroll
  for (int k = 0; k < 4; k++) km[k] = t[k];
  const uint32_t bl = it.bi ? it.bi_len : pow_len[it.bi_row];
  const uint8_t* bi = it.bi ? reinterpret_cast<const uint8_t*>(it.bi) : pow_be + (uint64_t)it.bi_row * kAuthBytes + (kAuthBytes - bl);
  auth_mac(mac, km, reinterpret_cast<const uint8_t*>(it.xi), it.xi_len, bi, bl);
#pragma unroll
  for (int k = 0; k < 4; k++)
#pragma unroll
    for (int b = 0; b < 4; b++) ke[4 * k + b] = (uint8_t)(t[4 + k] >> (24 - 8 * b));
#pragma unroll
  for (int k = 0; k < 8; k++)
#pragma unroll
    for (int b = 0; b < 4; b++) mo[4 * k + b] = (uint8_t)(mac[k] >> (24 - 8 * b));
  *reinterpret_cast<uint32_t*>(it.flag) = 1u;
}

// One AES-128 block under the key schedule rk (K6b's, S-box sb in shared memory): gcm_core's block cipher.
struct AesEnc {
  const uint32_t* rk; const uint8_t* sb;
  __device__ __forceinline__ void operator()(uint32_t& s0, uint32_t& s1, uint32_t& s2, uint32_t& s3) const { aes_encrypt<4>(rk, s0, s1, s2, s3, sb); }
};

// Phase 2.  ni: the request (ni_len bytes), nonce: 12 bytes, out: proof_len + 16 bytes (ciphertext || tag).
struct SealItem { uint64_t state; uint64_t ni; uint64_t nonce; uint64_t out; uint32_t ni_len, pad; };

// ok[i] = 1 when the item's MAC matched and out holds the sealed proof, 0 otherwise.
__global__ void __launch_bounds__(K6B_BLOCK)
auth_gcm_seal_kernel(const SealItem* __restrict__ items, const uint64_t n_items, uint8_t* __restrict__ ok) {
  __shared__ uint8_t sb[256];
  __shared__ uint32_t rk[44 * K6B_BLOCK];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sb[i] = c_aes_sbox[i];
  __syncthreads();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_items) {
    const SealItem it = items[i];
    AuthState* S = reinterpret_cast<AuthState*>(it.state);
    const uint8_t* ni = reinterpret_cast<const uint8_t*>(it.ni);
    uint32_t diff = it.ni_len ^ 32u;
#pragma unroll 1
    for (int b = 0; b < 32; b++) diff |= (uint32_t)((b < (int)it.ni_len ? ni[b] : 0u) ^ S->mac[b]);
    const bool good = diff == 0u && S->has_p1 == 1u;
    if (good) {
      aes_expand<4>(S->ke, rk, sb);
      const uint8_t* nn = reinterpret_cast<const uint8_t*>(it.nonce);
      const uint64_t len = S->proof_len;
      const uint8_t* pf = reinterpret_cast<const uint8_t*>(S) + sizeof(AuthState);
      uint8_t* out = reinterpret_cast<uint8_t*>(it.out);
      uint8_t tag[16];
      gcm_core(AesEnc{rk, sb}, load_be32(nn, 0, 12), load_be32(nn, 4, 12), load_be32(nn, 8, 12), S->mac, 32, pf, len, out, true, tag);
#pragma unroll
      for (int b = 0; b < 16; b++) out[len + b] = tag[b];
    }
    ok[i] = good ? 1 : 0;
#pragma unroll
    for (int b = 0; b < 16; b++) S->ke[b] = 0;                              // server.go drops the session after phase 2
#pragma unroll
    for (int b = 0; b < 32; b++) S->mac[b] = 0;
    S->has_p1 = 0u;
  }
#pragma unroll 1
  for (int k = 0; k < 44; k++) rk[k * K6B_BLOCK + threadIdx.x] = 0u;       // no key schedule left in shared memory
}
#endif

}  // namespace k9
}  // namespace bftq
