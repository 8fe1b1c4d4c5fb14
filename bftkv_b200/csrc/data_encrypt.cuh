// K11 — DataEncryption (crypto_pgp.go:532-554) on the device: OpenPGP passphrase encryption as x/crypto's
// SymmetricallyEncrypt writes it, and the symmetric half of ReadMessage.
//
//   s2k_kernel          one thread per (item, SKESK): RFC 4880 §3.7.1 S2K modes 0, 1 and 3 over SHA-256, then the
//                       SKESK's encrypted session key unwrapped (AES-CFB, zero IV, over cipher byte | key).  Writes a
//                       K6a-style record: 32 key bytes and an AES cipher id, 0 when the unwrap gives no AES key.
//   data_cand_kernel    one block: each item's records with a non-zero cipher id, in SKESK order, as K6b's candidate
//                       list (cand_off / cand_rec).  A failed unwrap must not be a candidate: nk_of(0) reads it as AES-256.
//   data_encrypt_kernel one thread per item: the SKESK with its wrapped session key, then the SEIPD packet with the OCFB
//                       prefix (no resync), the literal packet and the SHA-1 MDC in one CFB pass, with Go's partial-length
//                       framing written directly into the output.  The framing comes from a per-item list of writes the
//                       host computes (data_layout.hpp); the kernel only follows it.
// Decryption then runs K6b's seipd_decrypt_kernel unchanged.
//
// Timing: the S2K trip count depends on the count byte and the passphrase length only; the unwrap and every AES use
// K6b's S-box in shared memory, which is not constant time (DESIGN.md, K11).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "msg_decrypt.cuh"
#include "sha256.cuh"
#include "data_layout.hpp"

namespace bftq {
namespace k11 {

using k6::K6B_BLOCK;

// One S2K and its unwrap.  The passphrase is at key_off in the call's key blob.
struct S2kJob {
  uint64_t key_off;
  uint32_t key_len;
  uint32_t count;                 // bytes to hash (mode 3: the decoded count byte)
  uint8_t salt[8];
  uint8_t mode;                   // 0, 1 or 3
  uint8_t cipher;                 // the SKESK's key-encryption cipher: 7, 8 or 9
  uint8_t esk_len;                // 0 (the S2K output is the session key) .. 63
  uint8_t pad;
  uint8_t esk[64];
};

__device__ __forceinline__ int nk_of_cipher(uint32_t c) { return c == 7 ? 4 : (c == 8 ? 6 : (c == 9 ? 8 : 0)); }

// Message words of one S2K block from the byte stream (salt | key) repeated: pos counts bytes of the stream, idx is pos
// modulo the combined length; the bytes past total are SHA-256's padding.
__device__ __forceinline__ void s2k_block_bytes(const S2kJob& j, const uint8_t* __restrict__ key, const uint32_t slen, const uint32_t clen,
                                                const uint64_t total, uint64_t& pos, uint32_t& idx, uint32_t (&w)[16]) {
#pragma unroll
  for (int k = 0; k < 16; k++) {
    uint32_t v = 0;
#pragma unroll
    for (int t = 0; t < 4; t++) {
      uint32_t by = 0;
      if (pos < total) {
        by = idx < slen ? j.salt[idx] : key[idx - slen];
        idx = idx + 1 == clen ? 0u : idx + 1;
      } else if (pos == total) {
        by = 0x80u;
      }
      pos++;
      v = (v << 8) | by;
    }
    w[k] = v;
  }
}

// The S2K tables hold up to kS2kTabBlocks distinct full blocks per thread: with bftkv's 32-byte keys the combined string is
// 40 bytes and the block pattern repeats every 5 blocks.
constexpr uint32_t kS2kTabBlocks = 5;

// SHA-256 over the first max(count, len) bytes (mode 3; mode 0 / 1: exactly len) of (salt | key) repeated, where mode 0
// has no salt.  When the full blocks repeat within kS2kTabBlocks blocks, their words come from the thread's table `tab`
// (tab[q * K6B_BLOCK + tid], shared memory); the other blocks are assembled byte by byte.  The trip count depends on the
// count and the key length only.
__device__ void s2k_sha256(const S2kJob& j, const uint8_t* __restrict__ key, uint32_t* tab, uint32_t (&h)[8]) {
  const uint32_t slen = j.mode == 0 ? 0u : 8u;
  const uint32_t clen = slen + j.key_len;
  const uint64_t total = j.mode == 3 ? max((uint64_t)j.count, (uint64_t)clen) : (uint64_t)clen;
  const uint64_t nblk = (total + 8) / 64 + 1;
  h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
  h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
  const int tid = threadIdx.x;
  uint32_t period = 0;                            // clen / gcd(64, clen): blocks until the pattern repeats
  if (clen) { uint32_t g = clen & (0u - clen); g = g > 64 ? 64 : g; period = clen / g; }
  const uint64_t nfull = period && period <= kS2kTabBlocks ? total / 64 : 0;
  uint32_t idx = 0;
  uint64_t pos = 0;
  if (nfull) {
    for (uint32_t q = 0; q < period * 16; q++) {
      uint32_t v = 0;
      for (int t = 0; t < 4; t++) {
        v = (v << 8) | (idx < slen ? j.salt[idx] : key[idx - slen]);
        idx = idx + 1 == clen ? 0u : idx + 1;
      }
      tab[q * K6B_BLOCK + tid] = v;
    }
    uint32_t ph = 0;
#pragma unroll 1
    for (uint64_t b = 0; b < nfull; b++) {
      uint32_t w[16];
#pragma unroll
      for (int k = 0; k < 16; k++) w[k] = tab[(ph * 16 + k) * K6B_BLOCK + tid];
      ph = ph + 1 == period ? 0u : ph + 1;
      sha256_compress(h, w);
    }
    pos = nfull * 64;
    idx = (uint32_t)(pos % clen);
  }
#pragma unroll 1
  for (uint64_t b = nfull; b < nblk; b++) {
    uint32_t w[16];
    s2k_block_bytes(j, key, slen, clen, total, pos, idx, w);
    if (b == nblk - 1) { w[14] = (uint32_t)((total * 8) >> 32); w[15] = (uint32_t)(total * 8); }
    sha256_compress(h, w);
  }
}

// One AES-CFB keystream block under the thread's round keys: s <- E(s).
__device__ __forceinline__ void aes_block(const int nk, const uint32_t* rk, uint32_t (&s)[4], const uint8_t* sb) {
  if (nk == 4) k6::aes_encrypt<4>(rk, s[0], s[1], s[2], s[3], sb);
  else if (nk == 6) k6::aes_encrypt<6>(rk, s[0], s[1], s[2], s[3], sb);
  else k6::aes_encrypt<8>(rk, s[0], s[1], s[2], s[3], sb);
}
__device__ __forceinline__ void aes_setup(const int nk, const uint8_t* key, uint32_t* rk, const uint8_t* sb) {
  if (nk == 4) k6::aes_expand<4>(key, rk, sb);
  else if (nk == 6) k6::aes_expand<6>(key, rk, sb);
  else k6::aes_expand<8>(key, rk, sb);
}
__device__ __forceinline__ uint32_t byte_of(const uint32_t (&s)[4], const int i) {
  const uint32_t w = i < 4 ? s[0] : (i < 8 ? s[1] : (i < 12 ? s[2] : s[3]));
  return (w >> (24 - 8 * (i & 3))) & 0xffu;
}

// out_key: n_jobs x 32 bytes, out_cipher: n_jobs.  keys: the passphrases (secret), jobs: public.
__global__ void __launch_bounds__(K6B_BLOCK)
s2k_kernel(const S2kJob* __restrict__ jobs, const uint8_t* __restrict__ keys, const uint64_t n_jobs, uint8_t* __restrict__ out_key,
           uint8_t* __restrict__ out_cipher) {
  __shared__ uint8_t sb[256];
  __shared__ uint32_t tab[kS2kTabBlocks * 16 * K6B_BLOCK];   // the S2K table, then the unwrap's round keys
  __shared__ uint8_t kek[K6B_BLOCK][33];
  uint32_t* rk = tab;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sb[i] = k6::c_aes_sbox[i];
  __syncthreads();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_jobs) {
    const S2kJob& j = jobs[i];
    uint32_t h[8];
    s2k_sha256(j, keys + j.key_off, tab, h);
    const int knk = nk_of_cipher(j.cipher);
    const uint32_t ks = 4u * (uint32_t)knk;
    uint8_t* rec = out_key + i * 32u;
    uint8_t* kk = kek[threadIdx.x];
#pragma unroll
    for (int k = 0; k < 32; k++) kk[k] = (uint8_t)(h[k >> 2] >> (24 - 8 * (k & 3)));
#pragma unroll
    for (int k = 0; k < 8; k++) h[k] = 0u;
    uint32_t cipher = j.cipher;
    if (j.esk_len == 0) {
      for (uint32_t k = 0; k < 32; k++) rec[k] = k < ks ? kk[k] : 0u;
    } else {
      // CFB decryption with a zero IV: keystream block b is E(ciphertext block b - 1).
      aes_setup(knk, kk, rk, sb);
      uint32_t s[4] = {0u, 0u, 0u, 0u};
      const uint32_t n = j.esk_len;
      cipher = 0;
      for (uint32_t b = 0; b * 16 < n; b++) {
        aes_block(knk, rk, s, sb);
        uint32_t c[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int t = 0; t < 16; t++) {
          const uint32_t p = b * 16 + t;
          const uint32_t cb = p < n ? j.esk[p] : 0u;
          c[t >> 2] |= cb << (24 - 8 * (t & 3));
          const uint32_t pb = (cb ^ byte_of(s, t)) & 0xffu;
          if (p == 0) cipher = pb;
          else if (p < n && p <= 32) kk[p - 1] = (uint8_t)pb;
        }
#pragma unroll
        for (int t = 0; t < 4; t++) s[t] = c[t];
      }
      const int unk = nk_of_cipher(cipher);
      if (unk == 0 || n - 1 != 4u * (uint32_t)unk) cipher = 0;     // unknown, 3DES / CAST5, or the wrong key length
      const uint32_t ul = cipher ? n - 1 : 0u;
      for (uint32_t k = 0; k < 32; k++) rec[k] = k < ul ? kk[k] : 0u;
      s[0] = s[1] = s[2] = s[3] = 0u;
    }
    out_cipher[i] = (uint8_t)cipher;
  }
#pragma unroll 1
  for (int k = 0; k < (int)kS2kTabBlocks * 16; k++) tab[k * K6B_BLOCK + threadIdx.x] = 0u;   // no key, S2K table or key
#pragma unroll 1                                                                             // schedule left in shared memory
  for (int k = 0; k < 33; k++) kek[threadIdx.x][k] = 0u;
}

// One block of 1024 threads.  job_off[i] .. job_off[i+1]: item i's records in SKESK order.  cand_off (n + 1) and cand_rec
// as seipd_decrypt_kernel reads them.  The ids it reads are public in the sense Go's control flow is: which SKESK unwrapped.
constexpr int kCandBlock = 1024;
__global__ void __launch_bounds__(kCandBlock)
data_cand_kernel(const uint32_t* __restrict__ job_off, const uint8_t* __restrict__ rec_cipher, const uint64_t n_items,
                 uint32_t* __restrict__ cand_off, uint32_t* __restrict__ cand_rec) {
  __shared__ uint32_t warp_sum[kCandBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t base = 0;
  for (uint64_t t0 = 0; t0 < n_items; t0 += kCandBlock) {
    const uint64_t i = t0 + threadIdx.x;
    uint32_t cnt = 0;
    if (i < n_items) for (uint32_t r = job_off[i]; r < job_off[i + 1]; r++) cnt += rec_cipher[r] != 0;
    uint32_t x = cnt;                              // inclusive scan within the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint32_t s = warp_sum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += y; }
      warp_sum[lane] = s;
    }
    __syncthreads();
    const uint32_t excl = base + (warp ? warp_sum[warp - 1] : 0u) + x - cnt;
    if (i < n_items) {
      cand_off[i] = excl;
      uint32_t c = excl;
      for (uint32_t r = job_off[i]; r < job_off[i + 1]; r++) if (rec_cipher[r] != 0) cand_rec[c++] = r;
    }
    base += warp_sum[kCandBlock / 32 - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) cand_off[n_items] = base;
  if (threadIdx.x < kCandBlock / 32) warp_sum[threadIdx.x] = 0u;
}

// The CFB stream of one message (zero IV, no resync): the prefix, the encrypted writes and the MDC, with the SHA-1 MDC
// hash over the plain bytes before the digest.
struct CfbMdc {
  uint32_t ks[4];                 // keystream block; byte `used` is next
  uint32_t ct[4];                 // ciphertext block being collected
  uint32_t used;
  uint32_t h[5];
  uint64_t hashed;
};
__device__ __forceinline__ void shl8(uint32_t (&s)[4], const uint32_t in) {
  s[0] = (s[0] << 8) | (s[1] >> 24); s[1] = (s[1] << 8) | (s[2] >> 24); s[2] = (s[2] << 8) | (s[3] >> 24); s[3] = (s[3] << 8) | in;
}
// Encrypts one plain byte (hashing it first when `hash`) and returns the cipher byte.
__device__ __forceinline__ uint32_t cfb_byte(CfbMdc& st, const uint32_t p, const bool hash, const uint32_t* rk, uint32_t* w, const uint8_t* sb) {
  if (hash) {
    const uint32_t at = (uint32_t)(st.hashed & 63);
    w[at >> 2] = (at & 3) ? (w[at >> 2] | (p << (24 - 8 * (at & 3)))) : (p << 24);
    st.hashed++;
    if ((st.hashed & 63) == 0) sha1_compress(st.h, *reinterpret_cast<uint32_t (*)[16]>(w));
  }
  if (st.used == 16) {
    st.ks[0] = st.ct[0]; st.ks[1] = st.ct[1]; st.ks[2] = st.ct[2]; st.ks[3] = st.ct[3];
    k6::aes_encrypt<4>(rk, st.ks[0], st.ks[1], st.ks[2], st.ks[3], sb);
    st.used = 0;
  }
  const uint32_t c = (p ^ (st.ks[0] >> 24)) & 0xffu;
  shl8(st.ks, 0u);
  shl8(st.ct, c);
  st.used++;
  return c;
}

// One thread per item, AES-128 (Go's default cipher).  kek: the S2K records (16 bytes used), rand: 40 bytes per item (salt,
// session key, IV, in the order Go reads them), plain at plain_off, writes at wr_off (data_layout.hpp), output at out_off.
// lit_head: the six bytes that open the literal body ('t', an empty name, time 0), most significant byte first.
__global__ void __launch_bounds__(K6B_BLOCK)
data_encrypt_kernel(const uint8_t* __restrict__ kek, const uint8_t* __restrict__ rand, const uint8_t* __restrict__ plain,
                    const uint64_t* __restrict__ plain_off, const uint32_t* __restrict__ wr, const uint64_t* __restrict__ wr_off,
                    const uint64_t n_items, const uint64_t lit_head, uint8_t* __restrict__ out, const uint64_t* __restrict__ out_off) {
  __shared__ uint8_t sb[256];
  __shared__ uint32_t rk[60 * K6B_BLOCK];
  __shared__ uint32_t wsh[K6B_BLOCK][17];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sb[i] = k6::c_aes_sbox[i];
  __syncthreads();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t* w = wsh[threadIdx.x];
  if (i < n_items) {
    const uint8_t* rnd = rand + i * 40u;
    uint8_t* o = out + out_off[i];
    // ---- SKESK: C3 1E | 04 07 | 03 08 salt 60 | CFB_kek(07 | session key)
    k6::aes_expand<4>(kek + i * 32u, rk, sb);
    const uint8_t head[6] = {0xC3, 0x1E, 0x04, 0x07, 0x03, 0x08};
    for (int k = 0; k < 6; k++) o[k] = head[k];
    for (int k = 0; k < 8; k++) o[6 + k] = rnd[k];
    o[14] = 0x60;
    uint32_t s[4] = {0u, 0u, 0u, 0u};
    k6::aes_encrypt<4>(rk, s[0], s[1], s[2], s[3], sb);
    uint32_t c[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int t = 0; t < 16; t++) {
      const uint32_t cb = ((t == 0 ? 7u : (uint32_t)rnd[8 + t - 1]) ^ byte_of(s, t)) & 0xffu;
      o[15 + t] = (uint8_t)cb;
      c[t >> 2] |= cb << (24 - 8 * (t & 3));
    }
    k6::aes_encrypt<4>(rk, c[0], c[1], c[2], c[3], sb);
    o[31] = (uint8_t)((rnd[8 + 15] ^ (c[0] >> 24)) & 0xffu);
    o[32] = 0xD2;
    s[0] = s[1] = s[2] = s[3] = 0u; c[0] = c[1] = c[2] = c[3] = 0u;
    // ---- SEIPD under the session key: the writes of the cascade, each framed by Go's partialLengthWriter
    k6::aes_expand<4>(rnd + 8, rk, sb);
    CfbMdc st;
    st.ks[0] = st.ks[1] = st.ks[2] = st.ks[3] = 0u;
    st.ct[0] = st.ct[1] = st.ct[2] = st.ct[3] = 0u;
    st.used = 16;
    st.h[0] = 0x67452301u; st.h[1] = 0xEFCDAB89u; st.h[2] = 0x98BADCFEu; st.h[3] = 0x10325476u; st.h[4] = 0xC3D2E1F0u;
    st.hashed = 0;
    const uint8_t* pl = plain + plain_off[i];
    uint64_t q = 33, body = 0;                      // output position, position in the literal body stream
    uint32_t pre = 0, mdc = 0;                      // bytes of the prefix / MDC packet produced
#pragma unroll 1
    for (uint64_t e = wr_off[i]; e < wr_off[i + 1]; e++) {
      const uint32_t d = wr[e], kind = d >> 24, cb = (d >> 16) & 0xffu;
      uint32_t rem = d & 0xffffu;
#pragma unroll 1
      while (rem) {
        uint32_t pw = 14;
        while ((1u << pw) > rem) pw--;
        o[q++] = (uint8_t)(224 + pw);
        rem -= 1u << pw;
#pragma unroll 1
        for (uint32_t k = 0; k < (1u << pw); k++) {
          uint32_t outb;
          if (kind == kLayoutRaw) {
            outb = cb;
          } else if (kind == kLayoutPrefix) {           // IV | IV[14..16]
            const uint32_t at = pre < 16 ? pre : pre - 2;
            outb = cfb_byte(st, rnd[24 + at], true, rk, w, sb);
            pre++;
          } else if (kind == kLayoutByte) {
            outb = cfb_byte(st, cb, true, rk, w, sb);
          } else if (kind == kLayoutBody) {
            const uint32_t b = body < 6 ? (uint32_t)(lit_head >> (40 - 8 * body)) & 0xffu : pl[body - 6];
            outb = cfb_byte(st, b, true, rk, w, sb);
            body++;
          } else {                                  // D3 14, then SHA-1 of everything hashed so far
            uint32_t b;
            if (mdc < 2) {
              b = mdc == 0 ? 0xD3u : 0x14u;
              outb = cfb_byte(st, b, true, rk, w, sb);
              if (mdc == 1) {                       // SHA-1 padding of the hashed stream
                const uint64_t bits = st.hashed * 8;
                uint32_t at = (uint32_t)(st.hashed & 63);
                w[at >> 2] = (at & 3) ? (w[at >> 2] | (0x80u << (24 - 8 * (at & 3)))) : 0x80000000u;
                for (uint32_t z = (at >> 2) + 1; z < 16; z++) w[z] = 0u;
                if (at >= 56) { sha1_compress(st.h, *reinterpret_cast<uint32_t (*)[16]>(w)); for (int z = 0; z < 16; z++) w[z] = 0u; }
                w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
                sha1_compress(st.h, *reinterpret_cast<uint32_t (*)[16]>(w));
              }
            } else {
              const uint32_t at = mdc - 2;
              const uint32_t hv = at < 4 ? st.h[0] : (at < 8 ? st.h[1] : (at < 12 ? st.h[2] : (at < 16 ? st.h[3] : st.h[4])));
              outb = cfb_byte(st, (hv >> (24 - 8 * (at & 3))) & 0xffu, false, rk, w, sb);
            }
            mdc++;
          }
          o[q++] = (uint8_t)outb;
        }
      }
    }
    o[q] = 0x00;                                    // the outer partialLengthWriter's Close
    st.ks[0] = st.ks[1] = st.ks[2] = st.ks[3] = 0u;
    st.h[0] = st.h[1] = st.h[2] = st.h[3] = st.h[4] = 0u;
  }
#pragma unroll 1
  for (int k = 0; k < 60; k++) rk[k * K6B_BLOCK + threadIdx.x] = 0u;   // no key schedule or plain text left in shared memory
#pragma unroll 1
  for (int k = 0; k < 17; k++) w[k] = 0u;
}

}  // namespace k11
}  // namespace bftq
