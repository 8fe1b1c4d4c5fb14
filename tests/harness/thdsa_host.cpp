// Host build of K8's __host__ __device__ cores (bftkv_b200/csrc/thdsa_sign.cuh, p256.cuh's constant-time half).
#include <cstring>
#include <vector>
#include "../../bftkv_b200/csrc/thdsa_sign.cuh"
using namespace bftq;
using namespace bftq::p256;

namespace {
const uint32_t* table() {
  static std::vector<uint32_t> t;
  if (t.empty()) { t.resize(kBaseTableWords); base_table(t.data()); }
  return t.data();
}
k8::ThdsaGroup group(const uint8_t* q_be, uint32_t qlen) {
  k8::ThdsaGroup G;
  memset(&G, 0, sizeof(G));
  make_lagrange_mod<8>(q_be, qlen, G.q);
  const uint32_t c32[8] = {0, 1, 0, 0, 0, 0, 0, 0};
  mont_mul_big<8>(G.q32, G.q.r2, c32, G.q);
  return G;
}
void to_ppt(ppt& p, const uint8_t* a65) {               // 00 first byte: the identity
  const uint32_t R1[8] = BFTQ_P256_R1;
  if (a65[0] == 0) { for (int i = 0; i < 8; i++) { p.X[i] = 0; p.Y[i] = R1[i]; p.Z[i] = 0; } return; }
  uint32_t x[8], y[8];
  be_to_limbs(x, a65 + 1); be_to_limbs(y, a65 + 33);
  fe_to_mont(p.X, x); fe_to_mont(p.Y, y); fe_set(p.Z, R1);
}
}  // namespace

extern "C" {
void thdsa_base_mul_host(const uint8_t* a_be, uint8_t* out65) {
  uint32_t a[8];
  be_to_limbs(a, a_be);
  base_mul_ct(out65, a, table());
}
// complete addition; out65 = 04 || x || y, or 04 || 0^64 for the identity
void thdsa_add_host(const uint8_t* a65, const uint8_t* b65, uint8_t* out65) {
  ppt p, q, r;
  to_ppt(p, a65); to_ppt(q, b65);
  ppt_add_ct(r, p, q);
  fe zi, x, y;
  const uint32_t one[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  fe_inv_ct(zi, r.Z);
  fe_mul_ct(x, r.X, zi); fe_mul_ct(y, r.Y, zi);
  fe_mul_ct(x, x, one); fe_mul_ct(y, y, one);
  out65[0] = 4; limbs_to_be(out65 + 1, x); limbs_to_be(out65 + 33, y);
}
// out = (v mod q) for an arbitrary-length big-endian v (Horner), and out2 = (a b) mod q for a < q, b < 2^256
void thdsa_zq_host(const uint8_t* q_be, uint32_t qlen, const uint8_t* v_be, uint32_t vlen, const uint8_t* a_be, const uint8_t* b_be,
                   uint8_t* out32, uint8_t* out2_32) {
  const k8::ThdsaGroup G = group(q_be, qlen);
  std::vector<uint32_t> w((vlen + 3) / 4 + 1, 0);
  for (uint32_t b = 0; b < vlen; b++) { const uint32_t bit = vlen - 1 - b; w[bit / 4] |= (uint32_t)v_be[b] << (8 * (bit % 4)); }
  uint32_t acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  k8::add_reduced_ct(acc, w.data(), (vlen + 3) / 4, G);
  limbs::store_be_bytes<8>(out32, 32, acc);
  uint32_t a[8], b[8], r[8];
  limbs::load_be<8>(a, a_be, 32); limbs::load_be<8>(b, b_be, 32);
  k8::mul_mod_ct(r, a, b, G.q);
  limbs::store_be_bytes<8>(out2_32, 32, r);
}
}
