// Host build of bftkv_b200/csrc/modinv_big.cuh (the same __host__ __device__ code dsa_prepare_kernel runs).
#include "../../bftkv_b200/csrc/modinv_big.cuh"
extern "C" {
// out = a^-1 mod m (32-byte big-endian operands, m odd, a < m); returns 1, or 0 when gcd(a, m) != 1 (out zero then)
int modinv_host(const uint8_t* a_be, const uint8_t* m_be, uint8_t* out_be) {
  uint32_t a[8], m[8], inv[8];
  for (int i = 0; i < 8; i++) {
    a[i] = ((uint32_t)a_be[28 - 4 * i] << 24) | ((uint32_t)a_be[29 - 4 * i] << 16) | ((uint32_t)a_be[30 - 4 * i] << 8) | a_be[31 - 4 * i];
    m[i] = ((uint32_t)m_be[28 - 4 * i] << 24) | ((uint32_t)m_be[29 - 4 * i] << 16) | ((uint32_t)m_be[30 - 4 * i] << 8) | m_be[31 - 4 * i];
  }
  const bool ok = bftq::modinv_big<8>(inv, a, m);
  for (int i = 0; i < 8; i++) { out_be[28 - 4 * i] = (uint8_t)(inv[i] >> 24); out_be[29 - 4 * i] = (uint8_t)(inv[i] >> 16); out_be[30 - 4 * i] = (uint8_t)(inv[i] >> 8); out_be[31 - 4 * i] = (uint8_t)inv[i]; }
  return ok ? 1 : 0;
}
}
