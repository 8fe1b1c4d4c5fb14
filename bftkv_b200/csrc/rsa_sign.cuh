// K12 — the private-key operation of PGPSignature.Sign (crypto_pgp.go:346-371) on the device: rsa.SignPKCS1v15 with
// SHA-256 over the digest K4 (pgp_digest_kernel<8>) computed, written out as x/crypto's whole signature packet
// (sign_packet.hpp has the layout).  Go's decryptAndCheck, s^e == EM mod n, runs after it on K1 (rsa_verify_r32_kernel).
//
// One 4-lane group per item, as K6a, with the same CRT body (k6::rsa_crt) and so the same constant-time properties:
// fixed trip counts over all exponent bits, a table scan with masks for every window entry, masked conditional
// subtractions.  EM is public (it is fixed by the digest); the window table, which holds powers of EM mod p and mod q,
// is zeroed before the kernel exits.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "msg_decrypt.cuh"
#include "rsa_verify.cuh"
#include "sign_packet.hpp"

namespace bftq {
namespace k12 {

// key: the signer's slot in the keyring's private-key table; digest: n_items x 32 bytes; suffix: n_items x kSuffixBytes
// (sign_suffix).  out_s: n_items x 256 bytes, s for K1; out_packet: n_items x BFTQ_SIGN_PACKET_BYTES.
// Six blocks of 64 per SM, K6a's occupancy (168 registers, no spills): without the minimum ptxas gives the kernel 229
// registers, and four blocks fit.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 6)
rsa_crt_sign_kernel(const k6::RsaPriv32* __restrict__ key, const uint8_t* __restrict__ digest, const uint8_t* __restrict__ suffix,
                    const uint64_t n_items, uint8_t* __restrict__ out_s, uint8_t* __restrict__ out_packet) {
  using r32::T;
  __shared__ uint32_t tab[16][8][BLOCK];
  const int lane = threadIdx.x & 31;
  const int r = lane & (T - 1);
  const int gbase = lane & ~(T - 1);
  const int grp = threadIdx.x / T;
  const int plen = c_hash_prefix[BFTQ_HASH_SHA256].len, dlen = c_hash_prefix[BFTQ_HASH_SHA256].dlen;
  for (uint64_t base = (uint64_t)blockIdx.x * (BLOCK / T); base < n_items; base += (uint64_t)gridDim.x * (BLOCK / T)) {
    const uint64_t item_raw = base + (uint64_t)grp;
    const bool valid = item_raw < n_items;
    const uint64_t item = valid ? item_raw : n_items - 1;
    const uint8_t* dp = digest + item * 32u;
    // EM = 00 01 FF .. FF 00 || DigestInfo(SHA-256) || digest, as its low and high 1024-bit halves
    uint32_t c_lo[8], c_hi[8], s[16];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      c_lo[j] = em_word(r * 8 + j, dp, plen, dlen, BFTQ_HASH_SHA256);
      c_hi[j] = em_word(32 + r * 8 + j, dp, plen, dlen, BFTQ_HASH_SHA256);
    }
    k6::rsa_crt<BLOCK>(s, c_lo, c_hi, key, tab, r, gbase);
    if (valid) {
      uint8_t* so = out_s + item_raw * 256u;
      uint8_t* po = out_packet + item_raw * (uint64_t)BFTQ_SIGN_PACKET_BYTES;
#pragma unroll
      for (int j = 0; j < 16; j++) {
        const int off = 256 - 4 - 4 * (r * 16 + j);
        for (int b = 0; b < 4; b++) {
          const uint8_t v = (uint8_t)(s[j] >> (24 - 8 * b));
          so[off + b] = v;
          po[kSigAt + off + b] = v;
        }
      }
      if (r == 0) {
        const uint8_t* sp = suffix + item_raw * kSuffixBytes;
        po[0] = 0xC2; po[1] = 0xC0; po[2] = 0x5C;
        for (int i = 0; i < (int)kHashedBytes; i++) po[kPacketHead + i] = __ldg(sp + i);
        po[kPacketHead + kHashedBytes] = 0; po[kPacketHead + kHashedBytes + 1] = 0;          // no unhashed subpackets
        po[kPacketHead + kHashedBytes + 2] = __ldg(dp); po[kPacketHead + kHashedBytes + 3] = __ldg(dp + 1);
        po[kSigAt - 2] = 0x08; po[kSigAt - 1] = 0x00;
      }
    }
    __syncwarp();
#pragma unroll
    for (int e = 0; e < 16; e++)                       // the window table: powers of EM mod p and mod q, which reveal them
#pragma unroll
      for (int j = 0; j < 8; j++) tab[e][j][threadIdx.x] = 0u;
    __syncwarp();
  }
}

}  // namespace k12
}  // namespace bftq
