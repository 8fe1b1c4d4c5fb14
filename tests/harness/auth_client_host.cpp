// Host build of the AES-GCM core that K9's seal and K10's open share (gcm_core in bftkv_b200/csrc/auth_server.cuh), over
// libcrypto's AES block function instead of K6b's device AES.
#include <openssl/aes.h>

#include <cstring>
#include "../../bftkv_b200/csrc/auth_server.cuh"
using namespace bftq;

namespace {
struct HostAes {
  AES_KEY k;
  void operator()(uint32_t& s0, uint32_t& s1, uint32_t& s2, uint32_t& s3) const {
    uint8_t b[16];
    uint32_t* w[4] = {&s0, &s1, &s2, &s3};
    for (int i = 0; i < 16; i++) b[i] = (uint8_t)(*w[i / 4] >> (24 - 8 * (i % 4)));
    AES_encrypt(b, b, &k);
    for (int i = 0; i < 4; i++) *w[i] = ((uint32_t)b[4 * i] << 24) | ((uint32_t)b[4 * i + 1] << 16) | ((uint32_t)b[4 * i + 2] << 8) | b[4 * i + 3];
  }
};
uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
}  // namespace

extern "C" {
// seal: dst = src xor key stream (the ciphertext), ghash over it; open: ghash over src, dst (nullable) = plain text.
// tag16 receives the tag either way.
void auth_gcm_core_host(const uint8_t* key16, const uint8_t* nonce12, const uint8_t* aad, uint64_t aad_len, const uint8_t* src, uint64_t len,
                        uint8_t* dst, int seal, uint8_t* tag16) {
  HostAes enc;
  AES_set_encrypt_key(key16, 128, &enc.k);
  uint8_t tag[16];
  k9::gcm_core(enc, be32(nonce12), be32(nonce12 + 4), be32(nonce12 + 8), aad, aad_len, src, len, dst, seal != 0, tag);
  memcpy(tag16, tag, 16);
}
}
