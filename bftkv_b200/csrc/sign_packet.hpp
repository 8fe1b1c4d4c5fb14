// The host half of K12's signature packets (PGPSignature.Sign, crypto_pgp.go:346-371).  Plain C++: the library builds
// every call with it, and tests/harness/sign_host.cpp checks it against tests/signature_sign_oracle.py.
//
// x/crypto @53104e6ec876's DetachSign with a nil config signs with the entity's primary RSA key: SigType 0 (binary),
// SHA-256, and buildSubpackets puts creation time (type 2) and issuer (type 16) in the hashed area, nothing unhashed.
// The digest is SHA-256(tbs || suffix) with the suffix below; the packet is
//   C2 C0 5C | suffix[0 .. 22) | 00 00 | digest[0 .. 2) | 08 00 | s, left-padded to 256 bytes
// (the MPI header is 08 00 for every s: Signature.Sign sets bitLength = 8 * len(SignPKCS1v15's output)).
#pragma once
#include <cstdint>
#include <cstring>
#include "../../include/bftq.h"

namespace bftq {
namespace k12 {

constexpr uint64_t kSuffixBytes = 28;
constexpr uint64_t kPacketHead = 3;             // C2 C0 5C: new-format tag 2, two-octet length 284
constexpr uint64_t kHashedBytes = 22;           // version .. end of the hashed area: what the packet repeats of the suffix
constexpr uint64_t kSigAt = BFTQ_SIGN_PACKET_BYTES - 256;

// Signature.HashSuffix: 04 00 01 08 | 00 10 | 05 02 ctime | 09 10 key id | 04 FF 00 00 00 16 (the trailer's length is the
// 22 bytes before it).
inline void sign_suffix(uint32_t ctime, uint64_t key_id, uint8_t out[kSuffixBytes]) {
  static const uint8_t head[6] = {4, 0, 1, 8, 0, 16};
  memcpy(out, head, 6);
  out[6] = 5; out[7] = 2;
  for (int i = 0; i < 4; i++) out[8 + i] = (uint8_t)(ctime >> (24 - 8 * i));
  out[12] = 9; out[13] = 16;
  for (int i = 0; i < 8; i++) out[14 + i] = (uint8_t)(key_id >> (56 - 8 * i));
  static const uint8_t trailer[6] = {4, 0xFF, 0, 0, 0, (uint8_t)kHashedBytes};
  memcpy(out + 22, trailer, 6);
}

// Go's decryptAndCheck verdict per item: status[i] is K1's (0: s^e == EMSA-PKCS1-v1_5(digest) mod n).  A failed item's
// packet is zeroed and its code is BFTQ_ERR_SIGNING_FAILED, so no unchecked signature leaves the call.
inline void sign_release(const uint8_t* status, uint64_t n_items, uint8_t* packets, int32_t* out_err) {
  for (uint64_t i = 0; i < n_items; i++) {
    out_err[i] = status[i] == 0 ? BFTQ_OK : BFTQ_ERR_SIGNING_FAILED;
    if (status[i] != 0) memset(packets + i * BFTQ_SIGN_PACKET_BYTES, 0, BFTQ_SIGN_PACKET_BYTES);
  }
}

}  // namespace k12
}  // namespace bftq
