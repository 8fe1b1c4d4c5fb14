// Host build of bftkv_b200/csrc/modinv_big.cuh and limbs.cuh (the same __host__ __device__ code dsa_prepare_kernel and
// thrsa_modinv_kernel run).
#include "../../bftkv_b200/csrc/modinv_big.cuh"

template <int L>
static int modinv_host_l(const uint8_t* a_be, const uint8_t* m_be, uint8_t* out_be) {
  uint32_t a[L], m[L], inv[L];
  bftq::limbs::load_be<L>(a, a_be, 4 * L);
  bftq::limbs::load_be<L>(m, m_be, 4 * L);
  const bool ok = bftq::modinv_big<L>(inv, a, m);
  bftq::limbs::store_be_bytes<L>(out_be, 4 * L, inv);
  return ok ? 1 : 0;
}

extern "C" {
// out = a^-1 mod m (m odd, a < m); returns 1, or 0 when gcd(a, m) != 1 (out zero then).
// modinv_host: 32-byte big-endian operands (modinv_big<8>, K1d's s^-1 mod q); modinv_host64: 256-byte operands
// (modinv_big<64>, K7's m^-1 mod N).
int modinv_host(const uint8_t* a_be, const uint8_t* m_be, uint8_t* out_be) { return modinv_host_l<8>(a_be, m_be, out_be); }
int modinv_host64(const uint8_t* a_be, const uint8_t* m_be, uint8_t* out_be) { return modinv_host_l<64>(a_be, m_be, out_be); }
}
