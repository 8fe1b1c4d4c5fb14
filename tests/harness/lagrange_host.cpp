// Host build of bftkv_b200/csrc/lagrange.cuh and limbs.cuh: the same __host__ __device__ code lagrange_combine_kernel<L>
// (K3), fermat_inverse_kernel and mod_small_kernel (K5's Z_q helpers) run, with the modulus set up by the library's
// own make_lagrange_mod.
#include "../../bftkv_b200/csrc/lagrange.cuh"

template <int L>
static void combine_l(const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* xs, const uint8_t* ys_be, uint64_t n,
                      uint8_t* out_be, uint8_t* status, uint8_t* lambda_be) {
  bftq::LagrangeMod<L> M;
  bftq::make_lagrange_mod<L>(m_be, mlen, M);
  for (uint64_t item = 0; item < n; item++) bftq::lagrange_item<L>(M, k, xs, ys_be, item, out_be, status, lambda_be);
}

// acc = v^(m-2) mod m as fermat_inverse_kernel computes it: fermat_pow, then out of Montgomery form.
template <int L>
static void fermat_l(const uint8_t* m_be, uint32_t mlen, const uint8_t* v_be, uint8_t* out_be) {
  bftq::LagrangeMod<L> M;
  bftq::make_lagrange_mod<L>(m_be, mlen, M);
  uint32_t v[L], acc[L], one[L];
  bftq::limbs::load_be<L>(v, v_be, (int)mlen);
  bftq::fermat_pow<L>(acc, v, M);
  for (int l = 0; l < L; l++) one[l] = 0;
  one[0] = 1;
  bftq::mont_mul_big<L>(acc, acc, one, M);
  bftq::limbs::store_be_bytes<L>(out_be, (int)mlen, acc);
}

template <int L>
static void reduce_l(const uint8_t* m_be, uint32_t mlen, const uint8_t* big_be, uint32_t nbytes, uint8_t* out_be) {
  uint32_t m[L], r[L];
  bftq::limbs::load_be<L>(m, m_be, (int)mlen);
  bftq::limbs::reduce_be<L>(r, big_be, nbytes, m);
  bftq::limbs::store_be_bytes<L>(out_be, (int)mlen, r);
}

extern "C" {
// The limb class launch_lagrange_any picks for an mlen-byte modulus.
int lagrange_class(uint32_t mlen) { return mlen <= 32 ? 8 : mlen <= 64 ? 16 : mlen <= 128 ? 32 : 64; }

// n combines of k shares each (the batch layout of bftq_lagrange_combine_batch); lambda_be may be null.
void lagrange_combine_host(const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* xs, const uint8_t* ys_be, uint64_t n,
                           uint8_t* out_be, uint8_t* status, uint8_t* lambda_be) {
  switch (lagrange_class(mlen)) {
    case 8: combine_l<8>(m_be, mlen, k, xs, ys_be, n, out_be, status, lambda_be); break;
    case 16: combine_l<16>(m_be, mlen, k, xs, ys_be, n, out_be, status, lambda_be); break;
    case 32: combine_l<32>(m_be, mlen, k, xs, ys_be, n, out_be, status, lambda_be); break;
    default: combine_l<64>(m_be, mlen, k, xs, ys_be, n, out_be, status, lambda_be); break;
  }
}

// out = v^(m-2) mod m (v < m, mlen bytes each), at the limb class of mlen.
void fermat_pow_host(const uint8_t* m_be, uint32_t mlen, const uint8_t* v_be, uint8_t* out_be) {
  switch (lagrange_class(mlen)) {
    case 8: fermat_l<8>(m_be, mlen, v_be, out_be); break;
    case 16: fermat_l<16>(m_be, mlen, v_be, out_be); break;
    case 32: fermat_l<32>(m_be, mlen, v_be, out_be); break;
    default: fermat_l<64>(m_be, mlen, v_be, out_be); break;
  }
}

// out = (nbytes-long big-endian big_be) mod m, mlen bytes; limbs::reduce_be at 8 limbs (mod_small_kernel's class).
void reduce_be_host(const uint8_t* m_be, uint32_t mlen, const uint8_t* big_be, uint32_t nbytes, uint8_t* out_be) {
  reduce_l<8>(m_be, mlen, big_be, nbytes, out_be);
}
}
