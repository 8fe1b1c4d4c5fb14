// K1b — batched Ed25519 signature verification (RFC 8032, pure Ed25519) for sm_90a.
//
// BASELINE config 4 ("Ed25519 PGP keys").  NOTE: the reference itself cannot do this — its OpenPGP
// library (golang.org/x/crypto/openpgp @53104e6ec876) has no EdDSA (public-key algorithm 22) and
// skips such keys (SURVEY F5), so there is no reference behaviour to be bit-identical with.  The
// semantics here are RFC 8032 §5.1.7 as Go's crypto/ed25519 / ref10 / OpenSSL implement it:
//   reject S >= L;  decode A as edwards25519.Point.SetBytes does: y = the low 255 bits reduced mod p (y >= p is
//   accepted), reject only when (y^2 - 1) / (d y^2 + 1) is not a square, x = 0 with the sign bit set is accepted;
//   k = SHA-512(R || A || M) mod L over the caller's raw 32 key bytes;  accept iff  encode([S]B - [k]A) == R (byte
//   compare: R is never decoded, so a non-canonical R never matches).  No cofactor: small-order and mixed-order A and R
//   are decided by this equation alone.  libsodium is stricter (it rejects small-order A and R and non-canonical A).
// In OpenPGP (RFC 4880bis / GnuPG) M is the 32-byte v4 signature digest, so messages are a fixed 32
// bytes here.  Parity oracle for this kernel: a restatement of Go's Verify (oracle/ed25519_oracle.py) and OpenSSL
// (`cryptography`); libsodium (pynacl) wherever it is not stricter.
//
// This file: the table-free kernel (batches with few signatures per key) and the shared field / group / scalar code;
// ed25519_fast.cuh holds the cached-window-table path every large batch takes.
// One thread per signature; field elements are 10 limbs in radix 2^25.5 (26/25-bit alternating,
// signed) so that every product is one 32x32->64 IMAD.WIDE and ten of them are summed without
// carries — the same lazy-carry idea as K1's radix-2^28 kernel, in the form curve25519 code has
// used since ref10.  Double-scalar multiplication is Shamir's trick over the table {B, -A, B-A}
// (253 doublings + ~190 additions, ~3.7 k field multiplications, ~0.4 M MACs per verify).
// Everything below is __host__ __device__ so the arithmetic is unit-tested on the CPU as well.
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define BFTQ_HD __host__ __device__ inline
#define BFTQ_HD_NOINLINE __host__ __device__ __noinline__
#define BFTQ_ED_CONST __device__ __constant__ const
#else
#define BFTQ_HD inline
#define BFTQ_HD_NOINLINE inline
#define BFTQ_ED_CONST static const
#endif

namespace bftq { namespace ed {

typedef int32_t fe[10];

// constants (tools/gen_ed25519_consts.py)
#ifdef __CUDA_ARCH__
#define BFTQ_ED_TAB(name) d_##name
#else
#define BFTQ_ED_TAB(name) h_##name
#endif
#define BFTQ_ED_DEF(name, ...)                                      \
  static const int32_t h_##name[10] = __VA_ARGS__;                  \
  BFTQ_ED_DEVCONST(name, __VA_ARGS__)
#ifdef __CUDACC__
#define BFTQ_ED_DEVCONST(name, ...) __device__ __constant__ const int32_t d_##name[10] = __VA_ARGS__;
#else
#define BFTQ_ED_DEVCONST(name, ...)
#endif
BFTQ_ED_DEF(kD, {56195235, 13857412, 51736253, 6949390, 114729, 24766616, 60832955, 30306712, 48412415, 21499315})
BFTQ_ED_DEF(kD2, {45281625, 27714825, 36363642, 13898781, 229458, 15978800, 54557047, 27058993, 29715967, 9444199})
BFTQ_ED_DEF(kSqrtM1, {34513072, 25610706, 9377949, 3500415, 12389472, 33281959, 41962654, 31548777, 326685, 11406482})
BFTQ_ED_DEF(kBx, {52811034, 25909283, 16144682, 17082669, 27570973, 30858332, 40966398, 8378388, 20764389, 8758491})
BFTQ_ED_DEF(kBy, {40265304, 26843545, 13421772, 20132659, 26843545, 6710886, 53687091, 13421772, 40265318, 26843545})
BFTQ_ED_DEF(kBt, {28827043, 27438313, 39759291, 244362, 8635006, 11264893, 19351346, 13413597, 16611511, 27139452})
// group order L = 2^252 + 27742317777372353535851937790883648493, little-endian 32-bit words
#define BFTQ_ED_L {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0x0u, 0x0u, 0x0u, 0x10000000u}

// ---- field arithmetic mod p = 2^255 - 19 -------------------------------------------------------
BFTQ_HD void fe_copy(fe h, const fe f) { for (int i = 0; i < 10; i++) h[i] = f[i]; }
BFTQ_HD void fe_0(fe h) { for (int i = 0; i < 10; i++) h[i] = 0; }
BFTQ_HD void fe_1(fe h) { fe_0(h); h[0] = 1; }
BFTQ_HD void fe_add(fe h, const fe f, const fe g) { for (int i = 0; i < 10; i++) h[i] = f[i] + g[i]; }
BFTQ_HD void fe_sub(fe h, const fe f, const fe g) { for (int i = 0; i < 10; i++) h[i] = f[i] - g[i]; }
BFTQ_HD void fe_neg(fe h, const fe f) { for (int i = 0; i < 10; i++) h[i] = -f[i]; }

// Signed carry chain: brings every limb back to |h_even| <= 2^25, |h_odd| <= 2^24 (two passes: the
// first pass feeds 19*carry9 into limb 0).
BFTQ_HD void fe_carry(fe h, int64_t (&t)[10]) {
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
#pragma unroll
    for (int i = 0; i < 10; i++) {
      const int b = (i & 1) ? 25 : 26;
      const int64_t c = (t[i] + ((int64_t)1 << (b - 1))) >> b;
      t[i] -= c * ((int64_t)1 << b);
      if (i < 9) t[i + 1] += c; else t[0] += 19 * c;
    }
  }
  // limb 0 may have picked up 19 * (tiny carry): one more step 0 -> 1 keeps the bound
  const int64_t c0 = (t[0] + ((int64_t)1 << 25)) >> 26;
  t[0] -= c0 * ((int64_t)1 << 26);
  t[1] += c0;
#pragma unroll
  for (int i = 0; i < 10; i++) h[i] = (int32_t)t[i];
}

// h = f * g.  Inputs bounded by ~2^27 per limb (a few additions of carried elements).
BFTQ_HD_NOINLINE void fe_mul(fe h, const fe f, const fe g) {
  int32_t g19[10], f2[10];
#pragma unroll
  for (int i = 0; i < 10; i++) { g19[i] = 19 * g[i]; f2[i] = 2 * f[i]; }
  int64_t t[10];
#pragma unroll
  for (int k = 0; k < 10; k++) t[k] = 0;
#pragma unroll
  for (int i = 0; i < 10; i++) {
#pragma unroll
    for (int j = 0; j < 10; j++) {
      const int32_t fi = ((i & 1) && (j & 1)) ? f2[i] : f[i];
      const int k = i + j;
      if (k < 10) t[k] += (int64_t)fi * g[j];
      else t[k - 10] += (int64_t)fi * g19[j];
    }
  }
  fe_carry(h, t);
}
BFTQ_HD void fe_sq(fe h, const fe f) { fe_mul(h, f, f); }

// Canonical 32-byte little-endian encoding.
BFTQ_HD_NOINLINE void fe_tobytes(uint8_t* s, const fe hin) {
  int64_t t[10];
  for (int i = 0; i < 10; i++) t[i] = hin[i];
  fe hh;
  fe_carry(hh, t);
  int32_t h[10];
  for (int i = 0; i < 10; i++) h[i] = hh[i];
  // q = floor((h + 19) / 2^255) in {-1?,0,1}: compute as ref10 does
  int32_t q = (19 * h[9] + (1 << 24)) >> 25;
  for (int i = 0; i < 10; i++) q = (h[i] + q) >> ((i & 1) ? 25 : 26);
  h[0] += 19 * q;
  for (int i = 0; i < 10; i++) {
    const int b = (i & 1) ? 25 : 26;
    const int32_t c = h[i] >> b;
    if (i < 9) h[i + 1] += c;
    h[i] -= c * (1 << b);
  }
  // pack 26/25-bit limbs
  uint32_t w[8];
  uint64_t acc = 0; int bits = 0, wi = 0;
  for (int i = 0; i < 10; i++) {
    acc |= (uint64_t)(uint32_t)h[i] << bits;
    bits += (i & 1) ? 25 : 26;
    while (bits >= 32 && wi < 8) { w[wi++] = (uint32_t)acc; acc >>= 32; bits -= 32; }
  }
  if (wi < 8) w[wi++] = (uint32_t)acc;
  for (int i = 0; i < 8; i++) { s[4 * i] = (uint8_t)w[i]; s[4 * i + 1] = (uint8_t)(w[i] >> 8); s[4 * i + 2] = (uint8_t)(w[i] >> 16); s[4 * i + 3] = (uint8_t)(w[i] >> 24); }
}
// Loads 255 bits (the top bit is ignored); values in [p, 2^255) stay as they are, a valid representative of value - p.
// Returns false when the value is >= p (non-canonical).
BFTQ_HD bool fe_frombytes(fe h, const uint8_t* s) {
  uint32_t w[8];
  for (int i = 0; i < 8; i++) w[i] = (uint32_t)s[4 * i] | ((uint32_t)s[4 * i + 1] << 8) | ((uint32_t)s[4 * i + 2] << 16) | ((uint32_t)s[4 * i + 3] << 24);
  w[7] &= 0x7fffffffu;
  bool ge_p = w[7] == 0x7fffffffu && w[6] == 0xffffffffu && w[5] == 0xffffffffu && w[4] == 0xffffffffu && w[3] == 0xffffffffu &&
              w[2] == 0xffffffffu && w[1] == 0xffffffffu && w[0] >= 0xffffffedu;
  int pos = 0;
  for (int i = 0; i < 10; i++) {
    const int b = (i & 1) ? 25 : 26;
    const int wi = pos >> 5, sh = pos & 31;
    uint64_t v = w[wi];
    if (wi + 1 < 8) v |= (uint64_t)w[wi + 1] << 32;
    h[i] = (int32_t)((v >> sh) & (((uint64_t)1 << b) - 1));
    pos += b;
  }
  return !ge_p;
}
BFTQ_HD bool fe_isnegative(const fe f) { uint8_t s[32]; fe_tobytes(s, f); return s[0] & 1; }
BFTQ_HD bool fe_iszero(const fe f) { uint8_t s[32]; fe_tobytes(s, f); uint8_t r = 0; for (int i = 0; i < 32; i++) r |= s[i]; return r == 0; }

// z^(2^252 - 3) = z^((p-5)/8)
BFTQ_HD_NOINLINE void fe_pow22523(fe out, const fe z) {
  fe t0, t1, t2;
  fe_sq(t0, z);
  fe_sq(t1, t0); fe_sq(t1, t1);
  fe_mul(t1, z, t1);
  fe_mul(t0, t0, t1);
  fe_sq(t0, t0);
  fe_mul(t0, t1, t0);                                   // z^31 = z^(2^5 - 1)
  fe_sq(t1, t0); for (int i = 1; i < 5; i++) fe_sq(t1, t1);
  fe_mul(t0, t1, t0);                                   // 2^10 - 1
  fe_sq(t1, t0); for (int i = 1; i < 10; i++) fe_sq(t1, t1);
  fe_mul(t1, t1, t0);                                   // 2^20 - 1
  fe_sq(t2, t1); for (int i = 1; i < 20; i++) fe_sq(t2, t2);
  fe_mul(t1, t2, t1);                                   // 2^40 - 1
  fe_sq(t1, t1); for (int i = 1; i < 10; i++) fe_sq(t1, t1);
  fe_mul(t0, t1, t0);                                   // 2^50 - 1
  fe_sq(t1, t0); for (int i = 1; i < 50; i++) fe_sq(t1, t1);
  fe_mul(t1, t1, t0);                                   // 2^100 - 1
  fe_sq(t2, t1); for (int i = 1; i < 100; i++) fe_sq(t2, t2);
  fe_mul(t1, t2, t1);                                   // 2^200 - 1
  fe_sq(t1, t1); for (int i = 1; i < 50; i++) fe_sq(t1, t1);
  fe_mul(t0, t1, t0);                                   // 2^250 - 1
  fe_sq(t0, t0); fe_sq(t0, t0);                         // 2^252 - 4
  fe_mul(out, t0, z);                                   // 2^252 - 3
}
// z^(p-2) = z^(2^255 - 21)
BFTQ_HD_NOINLINE void fe_invert(fe out, const fe z) {
  fe t0, t1, t2, t3;
  fe_sq(t0, z);                                         // 2
  fe_sq(t1, t0); fe_sq(t1, t1);                         // 8
  fe_mul(t1, z, t1);                                    // 9
  fe_mul(t0, t0, t1);                                   // 11
  fe_sq(t2, t0);                                        // 22
  fe_mul(t1, t1, t2);                                   // 31 = 2^5 - 1
  fe_sq(t2, t1); for (int i = 1; i < 5; i++) fe_sq(t2, t2);
  fe_mul(t1, t2, t1);                                   // 2^10 - 1
  fe_sq(t2, t1); for (int i = 1; i < 10; i++) fe_sq(t2, t2);
  fe_mul(t2, t2, t1);                                   // 2^20 - 1
  fe_sq(t3, t2); for (int i = 1; i < 20; i++) fe_sq(t3, t3);
  fe_mul(t2, t3, t2);                                   // 2^40 - 1
  fe_sq(t2, t2); for (int i = 1; i < 10; i++) fe_sq(t2, t2);
  fe_mul(t1, t2, t1);                                   // 2^50 - 1
  fe_sq(t2, t1); for (int i = 1; i < 50; i++) fe_sq(t2, t2);
  fe_mul(t2, t2, t1);                                   // 2^100 - 1
  fe_sq(t3, t2); for (int i = 1; i < 100; i++) fe_sq(t3, t3);
  fe_mul(t2, t3, t2);                                   // 2^200 - 1
  fe_sq(t2, t2); for (int i = 1; i < 50; i++) fe_sq(t2, t2);
  fe_mul(t1, t2, t1);                                   // 2^250 - 1
  fe_sq(t1, t1); for (int i = 1; i < 5; i++) fe_sq(t1, t1);   // 2^255 - 32
  fe_mul(out, t1, t0);                                  // 2^255 - 21
}

// ---- group: extended twisted Edwards coordinates (X:Y:Z:T), a = -1 ------------------------------
struct ge { fe X, Y, Z, T; };

BFTQ_HD void ge_identity(ge& p) { fe_0(p.X); fe_1(p.Y); fe_1(p.Z); fe_0(p.T); }
BFTQ_HD void ge_neg(ge& r, const ge& p) { fe_neg(r.X, p.X); fe_copy(r.Y, p.Y); fe_copy(r.Z, p.Z); fe_neg(r.T, p.T); }

// RFC 8032 §5.1.4 addition (unified).
BFTQ_HD_NOINLINE void ge_add(ge& r, const ge& p, const ge& q) {
  fe a, b, c, d, e, f, g, h, t;
  fe_sub(a, p.Y, p.X); fe_sub(t, q.Y, q.X); fe_mul(a, a, t);
  fe_add(b, p.Y, p.X); fe_add(t, q.Y, q.X); fe_mul(b, b, t);
  fe_mul(c, p.T, q.T); fe_mul(c, c, BFTQ_ED_TAB(kD2));
  fe_mul(d, p.Z, q.Z); fe_add(d, d, d);
  fe_sub(e, b, a); fe_sub(f, d, c); fe_add(g, d, c); fe_add(h, b, a);
  fe_mul(r.X, e, f); fe_mul(r.Y, g, h); fe_mul(r.T, e, h); fe_mul(r.Z, f, g);
}
// RFC 8032 §5.1.4 doubling.
BFTQ_HD_NOINLINE void ge_dbl(ge& r, const ge& p) {
  fe a, b, c, e, f, g, h, t;
  fe_sq(a, p.X); fe_sq(b, p.Y);
  fe_sq(c, p.Z); fe_add(c, c, c);
  fe_add(h, a, b);
  fe_add(t, p.X, p.Y); fe_sq(t, t); fe_sub(e, h, t);
  fe_sub(g, a, b);
  fe_add(f, c, g);
  // f = c + g can reach 2^27 per limb: keep it the FIRST operand (the second one is pre-multiplied by 19 in 32 bits)
  fe_mul(r.X, f, e); fe_mul(r.Y, g, h); fe_mul(r.T, e, h); fe_mul(r.Z, f, g);
}
// Point decoding as Go's edwards25519.Point.SetBytes and OpenSSL do it: RFC 8032 §5.1.3 except that y >= p is taken mod p
// and x = 0 with the sign bit set is accepted (x stays 0).  false = (y^2 - 1) / (d y^2 + 1) has no square root.
BFTQ_HD bool ge_frombytes(ge& p, const uint8_t* s) {
  const int sign = s[31] >> 7;
  fe_frombytes(p.Y, s);                    // y >= p: the limbs hold y, which is y - p mod p
  fe u, v, v3, x, vxx, chk;
  fe_1(p.Z);
  fe_sq(u, p.Y);
  fe_mul(v, u, BFTQ_ED_TAB(kD));
  fe_sub(u, u, p.Z);                       // u = y^2 - 1
  fe_add(v, v, p.Z);                       // v = d y^2 + 1
  fe_sq(v3, v); fe_mul(v3, v3, v);         // v^3
  fe_sq(x, v3); fe_mul(x, x, v); fe_mul(x, x, u);   // u v^7
  fe_pow22523(x, x);
  fe_mul(x, x, v3); fe_mul(x, x, u);       // x = u v^3 (u v^7)^((p-5)/8)
  fe_sq(vxx, x); fe_mul(vxx, vxx, v);
  fe_sub(chk, vxx, u);
  if (!fe_iszero(chk)) {
    fe_add(chk, vxx, u);
    if (!fe_iszero(chk)) return false;
    fe_mul(x, x, BFTQ_ED_TAB(kSqrtM1));
  }
  if ((int)fe_isnegative(x) != sign) fe_neg(x, x);   // x = 0: -0 = 0
  fe_copy(p.X, x);
  fe_mul(p.T, p.X, p.Y);
  return true;
}
BFTQ_HD void ge_tobytes(uint8_t* s, const ge& p) {
  fe zi, x, y;
  fe_invert(zi, p.Z);
  fe_mul(x, p.X, zi); fe_mul(y, p.Y, zi);
  fe_tobytes(s, y);
  s[31] ^= (uint8_t)(fe_isnegative(x) << 7);
}

// ---- scalars mod L ------------------------------------------------------------------------------
// ---- scalars: Barrett reduction mod L (HAC 14.42 with b = 2^32, k = 8) -----------------------------------------------
// out = x mod L for the 512-bit x given as 16 little-endian words.
BFTQ_HD_NOINLINE void sc_reduce512(uint32_t (&out)[8], const uint32_t (&x)[16]) {
  const uint32_t Lw[9] = {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0x0u, 0x0u, 0x0u, 0x10000000u, 0u};
  const uint32_t mu[9] = {0x0a2c131bu, 0xed9ce5a3u, 0x086329a7u, 0x2106215du, 0xffffffebu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xfu};  // floor(2^512 / L)
  uint32_t q2[18];
#pragma unroll
  for (int i = 0; i < 18; i++) q2[i] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {                              // q2 = floor(x / b^7) * mu
    uint64_t carry = 0;
    const uint32_t qi = x[7 + i];
#pragma unroll
    for (int j = 0; j < 9; j++) {
      const uint64_t acc = (uint64_t)q2[i + j] + (uint64_t)qi * mu[j] + carry;
      q2[i + j] = (uint32_t)acc; carry = acc >> 32;
    }
    q2[i + 9] = (uint32_t)carry;
  }
  uint32_t r2[9];                                            // r2 = (floor(q2 / b^9) * L) mod b^9
#pragma unroll
  for (int i = 0; i < 9; i++) r2[i] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    uint64_t carry = 0;
    const uint32_t qi = q2[9 + i];
#pragma unroll
    for (int j = 0; j < 9; j++) {
      if (j + i >= 9) continue;
      const uint64_t acc = (uint64_t)r2[i + j] + (uint64_t)qi * Lw[j] + carry;
      r2[i + j] = (uint32_t)acc; carry = acc >> 32;
    }
  }
  uint32_t r[9];                                             // r = (x mod b^9) - r2 mod b^9, then at most two subtractions of L
  uint32_t br = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) { const uint64_t d = (uint64_t)x[i] - r2[i] - br; r[i] = (uint32_t)d; br = (uint32_t)(d >> 63); }
  for (int pass = 0; pass < 2; pass++) {
    bool ge = true, decided = false;                         // r >= L ?
#pragma unroll
    for (int i = 8; i >= 0; i--) { if (!decided && r[i] != Lw[i]) { ge = r[i] > Lw[i]; decided = true; } }
    if (ge) {
      uint32_t b2 = 0;
#pragma unroll
      for (int i = 0; i < 9; i++) { const uint64_t d = (uint64_t)r[i] - Lw[i] - b2; r[i] = (uint32_t)d; b2 = (uint32_t)(d >> 63); }
    }
  }
  for (int i = 0; i < 8; i++) out[i] = r[i];
}
// out (8 words) = the 64-byte little-endian value `in` mod L.
BFTQ_HD void sc_reduce64(uint32_t (&out)[8], const uint8_t* in) {
  uint32_t x[16];
  for (int i = 0; i < 16; i++) x[i] = (uint32_t)in[4 * i] | ((uint32_t)in[4 * i + 1] << 8) | ((uint32_t)in[4 * i + 2] << 16) | ((uint32_t)in[4 * i + 3] << 24);
  sc_reduce512(out, x);
}
// s (32 bytes little-endian) < L ?
BFTQ_HD bool sc_is_canonical(const uint8_t* s, uint32_t (&w)[8]) {
  const uint32_t Lw[8] = BFTQ_ED_L;
  for (int i = 0; i < 8; i++) w[i] = (uint32_t)s[4 * i] | ((uint32_t)s[4 * i + 1] << 8) | ((uint32_t)s[4 * i + 2] << 16) | ((uint32_t)s[4 * i + 3] << 24);
  for (int i = 7; i >= 0; i--) { if (w[i] != Lw[i]) return w[i] < Lw[i]; }
  return false;
}

// ---- verification given k = H(R || A || M) already reduced mod L --------------------------------
// sig = R (32) || S (32);  pk = A (32).  Returns true iff encode([S]B - [k]A) == R.
BFTQ_HD bool verify_core(const uint8_t* sig, const uint8_t* pk, const uint32_t (&k)[8]) {
  uint32_t s[8];
  if (!sc_is_canonical(sig + 32, s)) return false;                 // S >= L
  ge tab[3];                                                        // B, -A, B - A
  if (!ge_frombytes(tab[1], pk)) return false;
  ge_neg(tab[1], tab[1]);
  fe_copy(tab[0].X, BFTQ_ED_TAB(kBx)); fe_copy(tab[0].Y, BFTQ_ED_TAB(kBy)); fe_1(tab[0].Z); fe_copy(tab[0].T, BFTQ_ED_TAB(kBt));
  ge_add(tab[2], tab[0], tab[1]);
  ge p;
  ge_identity(p);
  for (int bit = 252; bit >= 0; bit--) {
    ge_dbl(p, p);
    const int idx = (int)((s[bit >> 5] >> (bit & 31)) & 1u) | (int)(((k[bit >> 5] >> (bit & 31)) & 1u) << 1);
    if (idx) { ge q; ge_add(q, p, tab[idx - 1]); p = q; }
  }
  uint8_t enc[32];
  ge_tobytes(enc, p);
  uint8_t diff = 0;
  for (int i = 0; i < 32; i++) diff |= enc[i] ^ sig[i];
  return diff == 0;
}


}}  // namespace bftq::ed
