// Host build of K9's __host__ __device__ cores (bftkv_b200/csrc/auth_server.cuh over sha256.cuh): GHASH's masked
// multiply, HMAC-SHA256 and keySched's HKDF-SHA256.
#include <cstring>
#include "../../bftkv_b200/csrc/auth_server.cuh"
using namespace bftq;

namespace {
struct Bytes {
  const uint8_t* p;
  uint32_t operator()(uint64_t pos) const { return p[pos]; }
};
void key_block(uint32_t (&k)[16], const uint8_t* key, uint32_t len) {      // len <= 64
  uint8_t b[64] = {0};
  memcpy(b, key, len);
  for (int i = 0; i < 16; i++) k[i] = ((uint32_t)b[4 * i] << 24) | ((uint32_t)b[4 * i + 1] << 16) | ((uint32_t)b[4 * i + 2] << 8) | b[4 * i + 3];
}
void put(uint8_t* out, const uint32_t* w, int n) {
  for (int i = 0; i < 4 * n; i++) out[i] = (uint8_t)(w[i / 4] >> (24 - 8 * (i % 4)));
}
}  // namespace

extern "C" {
// x = x * h in GF(2^128), 16-byte blocks
void auth_gf128_mul_host(uint8_t* x16, const uint8_t* h16) {
  uint64_t xh = 0, xl = 0, hh = 0, hl = 0;
  for (int i = 0; i < 8; i++) { xh = xh << 8 | x16[i]; xl = xl << 8 | x16[8 + i]; hh = hh << 8 | h16[i]; hl = hl << 8 | h16[8 + i]; }
  k9::gf128_mul(xh, xl, hh, hl);
  for (int i = 0; i < 8; i++) { x16[i] = (uint8_t)(xh >> (56 - 8 * i)); x16[8 + i] = (uint8_t)(xl >> (56 - 8 * i)); }
}
// HMAC-SHA256(key, msg), key <= 64 bytes
void auth_hmac_host(const uint8_t* key, uint32_t klen, const uint8_t* msg, uint64_t mlen, uint8_t* out32) {
  uint32_t k[16], o[8];
  key_block(k, key, klen);
  k9::hmac_sha256(o, k, Bytes{msg}, mlen);
  put(out32, o, 8);
}
// keySched(ikm, salt): km || ke.  A salt longer than 64 bytes is hashed first, as bftq_auth_server_create does.
void auth_hkdf_host(const uint8_t* salt, uint32_t slen, const uint8_t* ikm, uint64_t ilen, uint8_t* out32) {
  uint32_t k[16], t[8];
  if (slen > (uint32_t)k9::kSaltKeyMax) {
    uint32_t h[8];
    uint8_t d[32];
    k9::sha256_init(h);
    k9::sha256_tail(h, Bytes{salt}, slen, 0);
    put(d, h, 8);
    key_block(k, d, 32);
  } else {
    key_block(k, salt, slen);
  }
  k9::hkdf_sha256_32(t, k, Bytes{ikm}, ilen);
  put(out32, t, 8);
}
// calculateMac(km, xi, bi)
void auth_mac_host(const uint8_t* km16, const uint8_t* xi, uint64_t xl, const uint8_t* bi, uint64_t bl, uint8_t* out32) {
  uint32_t km[4], o[8];
  for (int i = 0; i < 4; i++) km[i] = ((uint32_t)km16[4 * i] << 24) | ((uint32_t)km16[4 * i + 1] << 16) | ((uint32_t)km16[4 * i + 2] << 8) | km16[4 * i + 3];
  k9::auth_mac(o, km, xi, xl, bi, bl);
  put(out32, o, 8);
}
}
