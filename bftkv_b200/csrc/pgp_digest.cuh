// K4 — batched OpenPGP v4 signature digest (SHA-1 / SHA-224 / SHA-256 / SHA-384 / SHA-512) for sm_90a.
//
// Replaces the hashing half of openpgp.CheckDetachedSignature as reached from
// crypto/pgp/crypto_pgp.go:324,338,490:  h = hashForSignature(sig.Hash, sig.SigType);
// io.Copy(h, signed); h.Write(sig.HashSuffix); digest = h.Sum(nil); digest[0:2] must equal the
// packet's 16-bit hash tag (checked by the caller against out_digest).  `signed` is
// packet.TBS / packet.TBSS output (packet/packet.go:156-190) and is shared by all signatures of
// one collective signature, hence the (data_idx -> data_off) indirection.
//
// One thread per digest; messages are 30..300 B (1..6 blocks), so this is latency/LSU-bound and
// small next to K1; it exists so the host does not have to hash 10^7 messages per second.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "sha256.cuh"

namespace bftq {

__constant__ uint64_t c_k512[80] = {
    0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull, 0x59f111f1b605d019ull,
    0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull, 0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull,
    0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull, 0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull,
    0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull, 0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull,
    0x983e5152ee66dfabull, 0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,
    0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull, 0x53380d139d95b3dfull,
    0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull, 0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull,
    0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull, 0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull,
    0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull, 0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull,
    0x5b9cca4f7763e373ull, 0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
    0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull, 0xd186b8c721c0c207ull,
    0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull, 0x113f9804bef90daeull, 0x1b710b35131c471bull,
    0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull, 0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull,
    0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull};

__device__ __forceinline__ uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

__device__ __forceinline__ void sha512_compress(uint64_t (&h)[8], uint64_t (&w)[16]) {
  uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
  for (int i = 0; i < 80; i++) {
    uint64_t wi;
    if (i < 16) {
      wi = w[i];
    } else {
      const uint64_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
      const uint64_t s0 = rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7);
      const uint64_t s1 = rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6);
      wi = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
      w[i & 15] = wi;
    }
    const uint64_t t1 = hh + (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41)) + ((e & f) ^ (~e & g)) + c_k512[i] + wi;
    const uint64_t t2 = (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

__device__ __forceinline__ void sha1_compress(uint32_t (&h)[5], uint32_t (&w)[16]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
#pragma unroll 1
  for (int i = 0; i < 80; i++) {
    uint32_t wi;
    if (i < 16) {
      wi = w[i];
    } else {
      const uint32_t x = w[(i - 3) & 15] ^ w[(i - 8) & 15] ^ w[(i - 14) & 15] ^ w[i & 15];
      wi = __funnelshift_l(x, x, 1);
      w[i & 15] = wi;
    }
    uint32_t f, k;
    if (i < 20) { f = (b & c) | (~b & d); k = 0x5A827999u; }
    else if (i < 40) { f = b ^ c ^ d; k = 0x6ED9EBA1u; }
    else if (i < 60) { f = (b & c) | (b & d) | (c & d); k = 0x8F1BBCDCu; }
    else { f = b ^ c ^ d; k = 0xCA62C1D6u; }
    const uint32_t t = __funnelshift_l(a, a, 5) + f + e + k + wi;
    e = d; d = c; c = __funnelshift_l(b, b, 30); b = a; a = t;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}

__constant__ uint32_t c_md5_k[64] = {
  0xd76aa478u, 0xe8c7b756u, 0x242070dbu, 0xc1bdceeeu, 0xf57c0fafu, 0x4787c62au, 0xa8304613u, 0xfd469501u, 0x698098d8u, 0x8b44f7afu, 0xffff5bb1u,
  0x895cd7beu, 0x6b901122u, 0xfd987193u, 0xa679438eu, 0x49b40821u, 0xf61e2562u, 0xc040b340u, 0x265e5a51u, 0xe9b6c7aau, 0xd62f105du, 0x02441453u,
  0xd8a1e681u, 0xe7d3fbc8u, 0x21e1cde6u, 0xc33707d6u, 0xf4d50d87u, 0x455a14edu, 0xa9e3e905u, 0xfcefa3f8u, 0x676f02d9u, 0x8d2a4c8au, 0xfffa3942u,
  0x8771f681u, 0x6d9d6122u, 0xfde5380cu, 0xa4beea44u, 0x4bdecfa9u, 0xf6bb4b60u, 0xbebfbc70u, 0x289b7ec6u, 0xeaa127fau, 0xd4ef3085u, 0x04881d05u,
  0xd9d4d039u, 0xe6db99e5u, 0x1fa27cf8u, 0xc4ac5665u, 0xf4292244u, 0x432aff97u, 0xab9423a7u, 0xfc93a039u, 0x655b59c3u, 0x8f0ccc92u, 0xffeff47du,
  0x85845dd1u, 0x6fa87e4fu, 0xfe2ce6e0u, 0xa3014314u, 0x4e0811a1u, 0xf7537e82u, 0xbd3af235u, 0x2ad7d2bbu, 0xeb86d391u};
__constant__ uint8_t c_md5_s[64] = {7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 5, 9, 14, 20, 5, 9, 14, 20, 5, 9, 14, 20, 5, 9, 14, 20,
                                    4, 11, 16, 23, 4, 11, 16, 23, 4, 11, 16, 23, 4, 11, 16, 23, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21};

// MD5 (RFC 1321): x/crypto links crypto/md5 (v3 key fingerprints), so hash id 1 is "available" to
// hashForSignature and a foreign MD5 signature is verified, not refused.
__device__ __forceinline__ void md5_compress(uint32_t (&h)[4], const uint32_t (&w)[16]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3];
#pragma unroll 1
  for (int i = 0; i < 64; i++) {
    uint32_t f; int g;
    if (i < 16) { f = (b & c) | (~b & d); g = i; }
    else if (i < 32) { f = (d & b) | (~d & c); g = (5 * i + 1) & 15; }
    else if (i < 48) { f = b ^ c ^ d; g = (3 * i + 5) & 15; }
    else { f = c ^ (b | ~d); g = (7 * i) & 15; }
    uint32_t wg = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) wg = (k == g) ? w[k] : wg;       // register file, no local-memory indexing
    const uint32_t tmp = d;
    d = c; c = b;
    const uint32_t x = a + f + c_md5_k[i] + wg;
    b = b + __funnelshift_l(x, x, c_md5_s[i]);
    a = tmp;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d;
}

struct DigestSrc {
  const uint8_t* dp; const uint8_t* sp; uint64_t dlen, total;
  __device__ __forceinline__ uint32_t byte(uint64_t pos) const {
    if (pos < dlen) return __ldg(dp + pos);
    if (pos < total) return __ldg(sp + (pos - dlen));
    return pos == total ? 0x80u : 0u;
  }
};

// ALG = OpenPGP hash id: 1 MD5, 2 SHA-1, 8 SHA-256, 9 SHA-384, 10 SHA-512, 11 SHA-224.  out stride = digest length.
template <int ALG>
__global__ void __launch_bounds__(128)
pgp_digest_kernel(const uint8_t* __restrict__ data_blob, const uint64_t* __restrict__ data_off,
                  const uint32_t* __restrict__ data_idx, const uint8_t* __restrict__ suffix_blob,
                  const uint64_t* __restrict__ suffix_off, const uint64_t n_items, uint8_t* __restrict__ out_digest,
                  const uint16_t* __restrict__ hash_tag, uint8_t* __restrict__ pre_status) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  const uint32_t di = data_idx ? __ldg(data_idx + item) : (uint32_t)item;
  const uint64_t d0 = __ldg(data_off + di), d1 = __ldg(data_off + di + 1);
  const uint64_t s0 = __ldg(suffix_off + item), s1 = __ldg(suffix_off + item + 1);
  DigestSrc src{data_blob + d0, suffix_blob + s0, d1 - d0, (d1 - d0) + (s1 - s0)};
  constexpr int kOutLen = ALG == 1 ? 16 : ALG == 2 ? 20 : ALG == 8 ? 32 : ALG == 9 ? 48 : ALG == 10 ? 64 : 28;
  uint8_t* o = out_digest + item * kOutLen;
  uint32_t first16;
  if constexpr (ALG == 9 || ALG == 10) {
    uint64_t h[8];
    if (ALG == 10) { h[0] = 0x6a09e667f3bcc908ull; h[1] = 0xbb67ae8584caa73bull; h[2] = 0x3c6ef372fe94f82bull; h[3] = 0xa54ff53a5f1d36f1ull;
                     h[4] = 0x510e527fade682d1ull; h[5] = 0x9b05688c2b3e6c1full; h[6] = 0x1f83d9abfb41bd6bull; h[7] = 0x5be0cd19137e2179ull; }
    else { h[0] = 0xcbbb9d5dc1059ed8ull; h[1] = 0x629a292a367cd507ull; h[2] = 0x9159015a3070dd17ull; h[3] = 0x152fecd8f70e5939ull;
           h[4] = 0x67332667ffc00b31ull; h[5] = 0x8eb44a8768581511ull; h[6] = 0xdb0c2e0d64f98fa7ull; h[7] = 0x47b5481dbefa4fa4ull; }
    const uint64_t nblocks = (src.total + 17 + 127) / 128;
    for (uint64_t blk = 0; blk < nblocks; blk++) {
      uint64_t w[16];
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint64_t v = 0;
#pragma unroll
        for (int b = 0; b < 8; b++) v = (v << 8) | src.byte(blk * 128 + 8 * i + b);
        w[i] = v;
      }
      if (blk == nblocks - 1) { w[14] = 0; w[15] = src.total * 8; }
      sha512_compress(h, w);
    }
    for (int i = 0; i < kOutLen / 8; i++)
      for (int b = 0; b < 8; b++) o[8 * i + b] = (uint8_t)(h[i] >> (56 - 8 * b));
    first16 = (uint32_t)(h[0] >> 48);
  } else if constexpr (ALG == 1) {
    uint32_t h[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};
    const uint64_t nblocks = (src.total + 9 + 63) / 64;
    for (uint64_t blk = 0; blk < nblocks; blk++) {
      uint32_t w[16];
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t v = 0;
#pragma unroll
        for (int b = 0; b < 4; b++) v |= src.byte(blk * 64 + 4 * i + b) << (8 * b);       // little-endian words
        w[i] = v;
      }
      if (blk == nblocks - 1) { w[14] = (uint32_t)(src.total * 8); w[15] = (uint32_t)((src.total * 8) >> 32); }
      md5_compress(h, w);
    }
    for (int i = 0; i < 4; i++)
      for (int b = 0; b < 4; b++) o[4 * i + b] = (uint8_t)(h[i] >> (8 * b));
    first16 = ((h[0] & 0xffu) << 8) | ((h[0] >> 8) & 0xffu);
  } else if constexpr (ALG == 2) {
    uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
    const uint64_t nblocks = (src.total + 9 + 63) / 64;
    for (uint64_t blk = 0; blk < nblocks; blk++) {
      uint32_t w[16];
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t v = 0;
#pragma unroll
        for (int b = 0; b < 4; b++) v = (v << 8) | src.byte(blk * 64 + 4 * i + b);
        w[i] = v;
      }
      if (blk == nblocks - 1) { w[14] = (uint32_t)((src.total * 8) >> 32); w[15] = (uint32_t)(src.total * 8); }
      sha1_compress(h, w);
    }
    for (int i = 0; i < 5; i++)
      for (int b = 0; b < 4; b++) o[4 * i + b] = (uint8_t)(h[i] >> (24 - 8 * b));
    first16 = h[0] >> 16;
  } else {
    uint32_t h[8];
    if (ALG == 8) { h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au; h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u; }
    else { h[0] = 0xc1059ed8u; h[1] = 0x367cd507u; h[2] = 0x3070dd17u; h[3] = 0xf70e5939u; h[4] = 0xffc00b31u; h[5] = 0x68581511u; h[6] = 0x64f98fa7u; h[7] = 0xbefa4fa4u; }
    const uint64_t nblocks = (src.total + 9 + 63) / 64;
    for (uint64_t blk = 0; blk < nblocks; blk++) {
      uint32_t w[16];
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t v = 0;
#pragma unroll
        for (int b = 0; b < 4; b++) v = (v << 8) | src.byte(blk * 64 + 4 * i + b);
        w[i] = v;
      }
      if (blk == nblocks - 1) { w[14] = (uint32_t)((src.total * 8) >> 32); w[15] = (uint32_t)(src.total * 8); }
      sha256_compress(h, w);
    }
    for (int i = 0; i < kOutLen / 4; i++)
      for (int b = 0; b < 4; b++) o[4 * i + b] = (uint8_t)(h[i] >> (24 - 8 * b));
    first16 = h[0] >> 16;
  }
  // x/crypto's 16-bit quick check ("hash tag doesn't match") before any RSA work.
  if (hash_tag != nullptr && pre_status != nullptr) {
    const uint16_t tag = __ldg(hash_tag + item);                  // big-endian: first digest byte in the high half
    if ((uint16_t)first16 != tag && pre_status[item] == 0) pre_status[item] = 2;   // BFTQ_ST_HASH_TAG
  }
}

using PgpDigestKernel = void (*)(const uint8_t*, const uint64_t*, const uint32_t*, const uint8_t*, const uint64_t*, uint64_t, uint8_t*,
                                 const uint16_t*, uint8_t*);
// The digest kernel of an OpenPGP hash id, or null when the device does not compute that digest.
inline PgpDigestKernel pgp_digest_kernel_for(uint32_t hash_alg) {
  switch (hash_alg) {
    case 1: return pgp_digest_kernel<1>;
    case 2: return pgp_digest_kernel<2>;
    case 8: return pgp_digest_kernel<8>;
    case 9: return pgp_digest_kernel<9>;
    case 10: return pgp_digest_kernel<10>;
    case 11: return pgp_digest_kernel<11>;
    default: return nullptr;
  }
}
inline bool digest_on_device(uint32_t hash_alg) { return pgp_digest_kernel_for(hash_alg) != nullptr; }

}  // namespace bftq
