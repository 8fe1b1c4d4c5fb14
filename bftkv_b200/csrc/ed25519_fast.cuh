// K1b fast path (round 2) — Ed25519 batch verification against cached per-key window tables.
//
// What changed against the first K1b (ed25519.cuh, kept for batches with few signatures per key):
//   * field products are forced inline with every limb in a register (the first version passed `fe` arrays to
//     __noinline__ functions, i.e. through local memory), a dedicated squaring (55 instead of 100 limb products) and
//     the interleaved 12-step carry chain curve25519 code has used since ref10;
//   * [S]B - [k]A is at most 48 MIXED additions (7 field products each) against window tables in affine "precomputed"
//     form (y+x, y-x, 2dxy; 128 bytes per entry): table[i][j-1] = j * 2^(W i) * P with signed radix-2^W digits.  The base
//     point has ONE radix-2^12 table per engine (22 windows x 2048 multiples = 5.8 MB), every key a radix-2^10 table of -A
//     (26 windows x 512 multiples = 1.7 MB) in a per-engine cache keyed by the 32 key bytes, so a
//     key pays its 250 doublings once per engine, not once per batch;
//   * the final X/Z, Y/Z needs ONE inversion per eight signatures: kernel 2 (`ed25519_finish_kernel`) runs Montgomery's
//     simultaneous inversion over eight results per thread;
//   * k = SHA-512(R || A || M) mod L is a Barrett reduction (81 + 45 word products) instead of 512 shift-subtract steps.
// Per verification: ~47.9 * 7 = 335 field products in kernel 1 + ~25 in kernel 2 (about 36 000 32x32->64 multiplies)
// instead of ~1 230 (135 000).  Semantics are those of ed25519.cuh (RFC 8032 §5.1.7 as Go's crypto/ed25519 / OpenSSL
// implement it: S < L; A decoded as edwards25519.Point.SetBytes does, y reduced mod p and x = 0 with the sign bit allowed;
// k over the raw key bytes; byte compare of the encoding of [S]B - [k]A with R; no cofactor).
// Everything is __host__ __device__: tests/harness/ed25519_host.cpp runs the same code on the CPU against OpenSSL,
// libsodium and the RFC 8032 vectors.
#pragma once
#include "ed25519.cuh"

#ifndef BFTQ_ED_PIN
#define BFTQ_ED_PIN 1
#endif
#ifdef __CUDACC__
#define BFTQ_HDI __host__ __device__ __forceinline__
#else
#define BFTQ_HDI inline
#endif

namespace bftq { namespace ed {

// ---- field: inlined products ---------------------------------------------------------------------------------------
// Interleaved carry chain (two chains of six steps run side by side; the order is ref10's).  Input: column sums of a
// product, |t| < 2^62.  Output: |h_even| <= 1.01 * 2^25, |h_odd| <= 1.01 * 2^24.
#define BFTQ_FX_STEP(i, j, b)                                                \
  { const int64_t c = (t[i] + ((int64_t)1 << ((b) - 1))) >> (b); t[j] += c; t[i] -= c * ((int64_t)1 << (b)); }
BFTQ_HDI void fex_carry(int32_t (&h)[10], int64_t (&t)[10]) {
  BFTQ_FX_STEP(0, 1, 26) BFTQ_FX_STEP(4, 5, 26)
  BFTQ_FX_STEP(1, 2, 25) BFTQ_FX_STEP(5, 6, 25)
  BFTQ_FX_STEP(2, 3, 26) BFTQ_FX_STEP(6, 7, 26)
  BFTQ_FX_STEP(3, 4, 25) BFTQ_FX_STEP(7, 8, 25)
  BFTQ_FX_STEP(4, 5, 26) BFTQ_FX_STEP(8, 9, 26)
  { const int64_t c = (t[9] + ((int64_t)1 << 24)) >> 25; t[0] += 19 * c; t[9] -= c * ((int64_t)1 << 25); }
  BFTQ_FX_STEP(0, 1, 26)
#pragma unroll
  for (int i = 0; i < 10; i++) {
    h[i] = (int32_t)t[i];
#if defined(__CUDA_ARCH__) && BFTQ_ED_PIN
    // Pin the limb in a 32-bit register.  Otherwise the compiler keeps "sign-extend the low half of the 64-bit column" as a
    // 64-bit value and the next product that takes the limb as its first operand becomes ten 64 x 64-bit multiplies
    // (IMAD.WIDE.U32 + two IMAD + a sign word each) instead of ten IMAD.WIDE: measured in SASS, 115 of 700 per mixed addition.
    asm("" : "+r"(h[i]));
#endif
  }
}
// h = f * g.  |f| <= 3.1 * 2^25 per limb, |g| <= 3.1 * 2^25 (g is multiplied by 19 in 32 bits: 19 |g| < 2^31).
BFTQ_HDI void fex_mul(int32_t (&h)[10], const int32_t (&f)[10], const int32_t (&g)[10]) {
  // The pre-scalings are done in UNSIGNED 32-bit arithmetic on purpose: with signed (no-signed-wrap) multiplies the
  // compiler widens sext(2 f_i) * sext(19 g_j) into 38 * f_i * g_j as a 64 x 64-bit product (IMAD.WIDE.U32 + two IMAD + a
  // sign extension instead of one IMAD.WIDE) for the 15 odd-odd wrapped terms of every product.
  int32_t g19[10], f2[10];
#pragma unroll
  for (int i = 0; i < 10; i++) { g19[i] = (int32_t)(19u * (uint32_t)g[i]); f2[i] = (int32_t)(2u * (uint32_t)f[i]); }
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
  fex_carry(h, t);
}
// h = f^2: 55 limb products.  |f| <= 1.65 * 2^26 (even limbs), 1.65 * 2^25 (odd limbs) — any sum of two carried elements.
BFTQ_HDI void fex_sq(int32_t (&h)[10], const int32_t (&f)[10]) {
  int32_t f2[10], fw[10];           // f2 = 2 f;  fw[j] = f[j] * 19 (j even) or * 38 (j odd): the wrapped partner
#pragma unroll
  for (int i = 0; i < 10; i++) { f2[i] = (int32_t)(2u * (uint32_t)f[i]); fw[i] = (int32_t)(((i & 1) ? 38u : 19u) * (uint32_t)f[i]); }    // unsigned: see fex_mul
  int64_t t[10];
#pragma unroll
  for (int k = 0; k < 10; k++) t[k] = 0;
#pragma unroll
  for (int i = 0; i < 10; i++) {
#pragma unroll
    for (int j = i; j < 10; j++) {
      // coefficient of f_i f_j in column i + j: (i != j ? 2 : 1) * (both odd ? 2 : 1) * (i + j >= 10 ? 19 : 1)
      const bool wrap = i + j >= 10, odd2 = (i & 1) && (j & 1);
      const int32_t a = (i != j) ? f2[i] : f[i];
      // partner: plain f_j, 2 f_j (both odd), 19 f_j (wrap, j even => i even... or i odd), 38 f_j (wrap and both odd)
      int32_t b;
      if (!wrap) b = odd2 ? f2[j] : f[j];
      else if (j & 1) b = odd2 ? fw[j] : (int32_t)(19u * (uint32_t)f[j]);      // j odd: fw = 38 f_j; with i even only 19 f_j is needed
      else b = fw[j];                                                // j even: 19 f_j (both-odd impossible)
      const int k = wrap ? i + j - 10 : i + j;
      t[k] += (int64_t)a * b;
    }
  }
  fex_carry(h, t);
}
BFTQ_HDI void fex_add(int32_t (&h)[10], const int32_t (&f)[10], const int32_t (&g)[10]) {
#pragma unroll
  for (int i = 0; i < 10; i++) h[i] = f[i] + g[i];
}
BFTQ_HDI void fex_sub(int32_t (&h)[10], const int32_t (&f)[10], const int32_t (&g)[10]) {
#pragma unroll
  for (int i = 0; i < 10; i++) h[i] = f[i] - g[i];
}
BFTQ_HDI void fex_copy(int32_t (&h)[10], const int32_t (&f)[10]) {
#pragma unroll
  for (int i = 0; i < 10; i++) h[i] = f[i];
}

// z^(2^255 - 21) (inverse, `inverse` = true) or z^(2^252 - 3) (the square-root exponent (p - 5) / 8) by ONE addition
// chain run as a small program: a single squaring and a single product instance in the code.
// Saved values: 0 z, 1 z^2, 2 z^9, 3 z^11, 4 z^(2^5-1), 5 z^(2^10-1), 6 z^(2^20-1), 7 z^(2^50-1), 8 z^(2^100-1).
BFTQ_HD_NOINLINE void fex_pow_chain(int32_t (&out)[10], const int32_t (&z)[10], const bool inverse) {
  //                     sq  mul store
  const int8_t prog[12][3] = {{1, -1, 1}, {2, 0, 2}, {0, 1, 3}, {1, 2, 4}, {5, 4, 5}, {10, 5, 6}, {20, 6, -1}, {10, 5, 7},
                              {50, 7, 8}, {100, 8, -1}, {50, 7, -1}, {5, 3, -1}};
  int32_t saved[9][10];
  int32_t t[10];
  for (int i = 0; i < 10; i++) { t[i] = z[i]; saved[0][i] = z[i]; }
#pragma unroll 1
  for (int s = 0; s < 12; s++) {
    int nsq = prog[s][0], mul = prog[s][1];
    const int store = prog[s][2];
    if (s == 11 && !inverse) { nsq = 2; mul = 0; }          // z^(2^250-1) -> ^4 * z = z^(2^252-3)
#pragma unroll 1
    for (int n = 0; n < nsq; n++) { int32_t u[10]; fex_sq(u, t); fex_copy(t, u); }
    if (mul >= 0) {
      int32_t m[10], u[10];
      for (int i = 0; i < 10; i++) m[i] = saved[mul][i];
      fex_mul(u, t, m);
      fex_copy(t, u);
    }
    if (store >= 0) for (int i = 0; i < 10; i++) saved[store][i] = t[i];
  }
  fex_copy(out, t);
}

// Canonical little-endian words of a field element (|limbs| within fex_mul's input bounds).
BFTQ_HDI void fex_towords(uint32_t (&w)[8], const int32_t (&hin)[10]) {
  int32_t h[10];
#pragma unroll
  for (int i = 0; i < 10; i++) h[i] = hin[i];
  int32_t q = (19 * h[9] + (1 << 24)) >> 25;
#pragma unroll
  for (int i = 0; i < 10; i++) q = (h[i] + q) >> ((i & 1) ? 25 : 26);
  h[0] += 19 * q;
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const int b = (i & 1) ? 25 : 26;
    const int32_t c = h[i] >> b;
    if (i < 9) h[i + 1] += c;
    h[i] -= c * (1 << b);
  }
  // limb i starts at bit 0, 26, 51, 77, 102, 128, 153, 179, 204, 230
  w[0] = (uint32_t)h[0] | ((uint32_t)h[1] << 26);
  w[1] = ((uint32_t)h[1] >> 6) | ((uint32_t)h[2] << 19);
  w[2] = ((uint32_t)h[2] >> 13) | ((uint32_t)h[3] << 13);
  w[3] = ((uint32_t)h[3] >> 19) | ((uint32_t)h[4] << 6);
  w[4] = (uint32_t)h[5] | ((uint32_t)h[6] << 25);
  w[5] = ((uint32_t)h[6] >> 7) | ((uint32_t)h[7] << 19);
  w[6] = ((uint32_t)h[7] >> 13) | ((uint32_t)h[8] << 12);
  w[7] = ((uint32_t)h[8] >> 20) | ((uint32_t)h[9] << 6);
}

// ---- group ---------------------------------------------------------------------------------------------------------
struct gea { int32_t ypx[10], ymx[10], xy2d[10], pad[2]; };       // affine (y+x, y-x, 2dxy), carried limbs; 128 bytes
static_assert(sizeof(gea) == 128, "table entry is one 128-byte line");
// Window geometry for a signed radix-2^W recoding of a scalar < 2^253: W * windows >= 254, so the top digit never carries out.
template <int W> struct FxWin {
  static constexpr int bits = W;
  static constexpr int windows = (253 + W) / W;                    // 8 -> 32, 10 -> 26, 12 -> 22
  static constexpr int multiples = 1 << (W - 1);                   // j = 1 .. 2^(W-1): digits in [-2^(W-1), 2^(W-1) - 1]
  static constexpr int entries = windows * multiples;
};
constexpr int kFxWB = 12;                                          // the base point: ONE table per engine, 22 x 2048 entries = 5.8 MB
constexpr int kFxWA = 10;                                          // a key: 26 x 512 entries = 1.7 MB
typedef FxWin<kFxWB> FxB;
typedef FxWin<kFxWA> FxA;
constexpr int kFxChunk = 8;                                        // table entries (and results) per simultaneous inversion
constexpr int kFxScalarWords = 9;                                  // a scalar travels as 8 words + one zero word (a window may straddle the top)

struct gex { int32_t X[10], Y[10], Z[10], T[10]; };

// p += q (neg: p -= q), q affine-precomputed: 7 products.  Every coordinate of p stays carried.
BFTQ_HDI void gex_madd(gex& p, const int32_t (&q_ypx)[10], const int32_t (&q_ymx)[10], const int32_t (&q_xy2d)[10], const bool neg) {
  int32_t a[10], b[10], c[10], u[10], v[10], s1[10], s2[10], s3[10];
#pragma unroll
  for (int i = 0; i < 10; i++) {
    u[i] = p.Y[i] - p.X[i]; v[i] = p.Y[i] + p.X[i];
    s1[i] = neg ? q_ypx[i] : q_ymx[i];
    s2[i] = neg ? q_ymx[i] : q_ypx[i];
    s3[i] = neg ? -q_xy2d[i] : q_xy2d[i];
  }
  fex_mul(a, u, s1);                      // A = (Y1 - X1)(y2 - x2)
  fex_mul(b, v, s2);                      // B = (Y1 + X1)(y2 + x2)
  fex_mul(c, p.T, s3);                    // C = T1 * 2d x2 y2
  int32_t e[10], f[10], g[10], h[10];
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const int32_t d = 2 * p.Z[i];
    e[i] = b[i] - a[i]; h[i] = b[i] + a[i]; f[i] = d - c[i]; g[i] = d + c[i];
  }
  fex_mul(p.X, e, f); fex_mul(p.Y, g, h); fex_mul(p.T, e, h); fex_mul(p.Z, g, f);
}
// r = p + q, both extended (RFC 8032 §5.1.4): 9 products.  r may alias p or q.
BFTQ_HD_NOINLINE void gex_add(gex& r, const gex& p, const gex& q) {
  int32_t a[10], b[10], c[10], d[10], u[10], v[10], kd2[10];
  for (int i = 0; i < 10; i++) kd2[i] = BFTQ_ED_TAB(kD2)[i];
  fex_sub(u, p.Y, p.X); fex_sub(v, q.Y, q.X); fex_mul(a, u, v);
  fex_add(u, p.Y, p.X); fex_add(v, q.Y, q.X); fex_mul(b, u, v);
  fex_mul(c, p.T, q.T); fex_mul(u, c, kd2);
  fex_mul(d, p.Z, q.Z);
  int32_t e[10], f[10], g[10], h[10];
  for (int i = 0; i < 10; i++) { const int32_t dd = 2 * d[i]; e[i] = b[i] - a[i]; h[i] = b[i] + a[i]; f[i] = dd - u[i]; g[i] = dd + u[i]; }
  fex_mul(r.X, e, f); fex_mul(r.Y, g, h); fex_mul(r.T, e, h); fex_mul(r.Z, g, f);
}
// r = 2 p (RFC 8032 §5.1.4): 4 squarings + 4 products.  r may alias p.
BFTQ_HD_NOINLINE void gex_dbl(gex& r, const gex& p) {
  int32_t a[10], b[10], c[10], t[10], u[10];
  fex_sq(a, p.X); fex_sq(b, p.Y); fex_sq(c, p.Z);
  fex_add(u, p.X, p.Y); fex_sq(t, u);
  int32_t e[10], f[10], g[10], h[10], hc[10];
  for (int i = 0; i < 10; i++) { h[i] = a[i] + b[i]; g[i] = a[i] - b[i]; }
  for (int i = 0; i < 10; i++) { e[i] = h[i] - t[i]; f[i] = 2 * c[i] + g[i]; }      // |e| <= 3 * 2^25, |f| <= 4 * 2^25
  // f can reach 4.04 * 2^25: it is only ever the FIRST operand (the second one is multiplied by 19 in 32 bits)
  fex_copy(hc, h);
  fex_mul(r.X, f, e); fex_mul(r.Y, g, hc); fex_mul(r.T, e, hc); fex_mul(r.Z, f, g);
}
BFTQ_HDI void gex_identity(gex& p) {
#pragma unroll
  for (int i = 0; i < 10; i++) { p.X[i] = 0; p.Y[i] = (i == 0); p.Z[i] = (i == 0); p.T[i] = 0; }
}
BFTQ_HD void gex_basepoint(gex& b) {
  for (int i = 0; i < 10; i++) { b.X[i] = BFTQ_ED_TAB(kBx)[i]; b.Y[i] = BFTQ_ED_TAB(kBy)[i]; b.Z[i] = (i == 0); b.T[i] = BFTQ_ED_TAB(kBt)[i]; }
}
// Point decoding with the inlined field, the same decisions as ge_frombytes: y >= p is taken mod p, x = 0 with the sign bit
// set is accepted; false only when x^2 has no square root.  Two encodings of one point are two cache slots.
BFTQ_HD_NOINLINE bool gex_frombytes(gex& p, const uint8_t* s) {
  const int sign = s[31] >> 7;
  fe_frombytes(p.Y, s);                    // y >= p: the limbs hold y, which is y - p mod p
  int32_t u[10], v[10], v3[10], x[10], t[10], vxx[10], chk[10], one[10], kd[10], ksm1[10];
  for (int i = 0; i < 10; i++) { one[i] = (i == 0); kd[i] = BFTQ_ED_TAB(kD)[i]; ksm1[i] = BFTQ_ED_TAB(kSqrtM1)[i]; }
  fex_copy(p.Z, one);
  fex_sq(u, p.Y);
  fex_mul(v, u, kd);
  fex_sub(u, u, one);                      // u = y^2 - 1
  fex_add(v, v, one);                      // v = d y^2 + 1
  fex_sq(t, v); fex_mul(v3, t, v);         // v^3
  fex_sq(t, v3); fex_mul(x, t, v); fex_mul(t, x, u);     // u v^7
  fex_pow_chain(x, t, false);
  fex_mul(t, x, v3); fex_mul(x, t, u);     // x = u v^3 (u v^7)^((p-5)/8)
  fex_sq(t, x); fex_mul(vxx, t, v);
  fex_sub(chk, vxx, u);
  if (!fe_iszero(chk)) {
    fex_add(chk, vxx, u);
    if (!fe_iszero(chk)) return false;
    fex_mul(t, x, ksm1); fex_copy(x, t);
  }
  if ((int)fe_isnegative(x) != sign) { for (int i = 0; i < 10; i++) x[i] = -x[i]; }   // x = 0: -0 = 0
  fex_copy(p.X, x);
  fex_mul(p.T, p.X, p.Y);
  return true;
}

// ---- scalars ----------------------------------------------------------------------------------------------------------
// S < L ?  (words little-endian)
BFTQ_HDI bool sc_words_canonical(const uint32_t (&w)[8]) {
  const uint32_t Lw[8] = BFTQ_ED_L;
  bool lt = false, decided = false;
#pragma unroll
  for (int i = 7; i >= 0; i--) { if (!decided && w[i] != Lw[i]) { lt = w[i] < Lw[i]; decided = true; } }
  return lt;
}
// Signed radix-2^W digit i of a scalar (< 2^253, kFxScalarWords words, word w at sw[w * stride]): d in [-2^(W-1), 2^(W-1) - 1],
// the carry chained upwards through `carry` (digits must be taken in ascending order).
template <int W>
BFTQ_HDI int sc_digit(const uint32_t* sw, const int stride, const int i, uint32_t& carry) {
  const int bit = W * i, wi = bit >> 5, sh = bit & 31;
  uint32_t v = sw[wi * stride] >> sh;
  if (sh + W > 32) v |= sw[(wi + 1) * stride] << (32 - sh);
  const uint32_t d = (v & ((1u << W) - 1u)) + carry;
  carry = (d + (1u << (W - 1))) >> W;
  return (int)d - (int)(carry << W);
}

// ---- table construction ----------------------------------------------------------------------------------------------
// Step 1 (one thread per point): window bases 2^(w i) * P, i = 0..nw-1, as extended points with carried limbs.
BFTQ_HD void fx_window_bases(gex* bases, const gex& P, const int nw, const int w) {
  gex b = P;
  for (int i = 0; i < nw; i++) {
    bases[i] = b;
    if (i + 1 < nw) for (int t = 0; t < w; t++) gex_dbl(b, b);
  }
}
// Step 2 (one thread per (point, window, chunk of 8 multiples)): entries (8c+1 .. 8c+8) * base in affine precomputed form,
// one inversion for the eight (Montgomery's trick).
BFTQ_HD void fx_window_chunk(gea* out, const gex& base, const int chunk) {
  gex m[kFxChunk];
  // m[0] = (8 chunk + 1) * base by double-and-add from the top bit
  const int first = kFxChunk * chunk + 1;
  gex acc = base;
  int top = 0;
  for (int b = 12; b >= 0; b--) if ((first >> b) & 1) { top = b; break; }
  for (int b = top - 1; b >= 0; b--) { gex_dbl(acc, acc); if ((first >> b) & 1) gex_add(acc, acc, base); }
  m[0] = acc;
  for (int j = 1; j < kFxChunk; j++) gex_add(m[j], m[j - 1], base);
  // simultaneous inversion of the eight Z
  int32_t pre[kFxChunk][10];
  fex_copy(pre[0], m[0].Z);
  for (int j = 1; j < kFxChunk; j++) fex_mul(pre[j], pre[j - 1], m[j].Z);
  int32_t inv[10], kd2[10];
  fex_pow_chain(inv, pre[kFxChunk - 1], true);
  for (int i = 0; i < 10; i++) kd2[i] = BFTQ_ED_TAB(kD2)[i];
  for (int j = kFxChunk - 1; j >= 0; j--) {
    int32_t zi[10], t[10];
    if (j > 0) { fex_mul(zi, inv, pre[j - 1]); fex_mul(t, inv, m[j].Z); fex_copy(inv, t); }
    else fex_copy(zi, inv);
    int32_t x[10], y[10], xy[10];
    fex_mul(x, m[j].X, zi); fex_mul(y, m[j].Y, zi); fex_mul(xy, x, y);
    gea e;
    int64_t s[10];
    for (int i = 0; i < 10; i++) s[i] = (int64_t)y[i] + x[i];
    fex_carry(e.ypx, s);
    for (int i = 0; i < 10; i++) s[i] = (int64_t)y[i] - x[i];
    fex_carry(e.ymx, s);
    fex_mul(e.xy2d, xy, kd2);
    e.pad[0] = 0; e.pad[1] = 0;
    out[j] = e;
  }
}

// ---- verification ----------------------------------------------------------------------------------------------------
// One table entry into registers (device: eight 16-byte read-only loads of the 128-byte line).
BFTQ_HDI void fx_load_entry(int32_t (&ypx)[10], int32_t (&ymx)[10], int32_t (&xy2d)[10], const gea* q) {
#ifdef __CUDA_ARCH__
  const int4* v = reinterpret_cast<const int4*>(q);
  int32_t w[32];
#pragma unroll
  for (int i = 0; i < 8; i++) { const int4 x = __ldg(v + i); w[4 * i] = x.x; w[4 * i + 1] = x.y; w[4 * i + 2] = x.z; w[4 * i + 3] = x.w; }
#pragma unroll
  for (int i = 0; i < 10; i++) { ypx[i] = w[i]; ymx[i] = w[10 + i]; xy2d[i] = w[20 + i]; }
#else
  for (int i = 0; i < 10; i++) { ypx[i] = q->ypx[i]; ymx[i] = q->ymx[i]; xy2d[i] = q->xy2d[i]; }
#endif
}
// [S]B - [k]A as an extended point: at most 22 + 26 = 48 mixed additions.  tabB: the base point's radix-2^12 table, tabNegA:
// -A's radix-2^10 table; the scalars are kFxScalarWords words each, word w of S at s[w * stride] (the kernel keeps them in
// shared memory, one column per thread).  The caller has checked S < L and that A decodes.
BFTQ_HDI void fx_accumulate(gex& p, const uint32_t* s, const uint32_t* k, const int stride, const gea* tabB, const gea* tabNegA) {
  gex_identity(p);
  uint32_t cs = 0, ck = 0;
#pragma unroll 1
  for (int it = 0; it < FxB::windows + FxA::windows; it++) {
    const bool which = it >= FxB::windows;
    const int i = which ? it - FxB::windows : it;
    int dig;
    const gea* q;
    if (which) { dig = sc_digit<kFxWA>(k, stride, i, ck); q = tabNegA + i * FxA::multiples; }
    else { dig = sc_digit<kFxWB>(s, stride, i, cs); q = tabB + i * FxB::multiples; }
    if (dig != 0) {
      const int mag = dig < 0 ? -dig : dig;
      int32_t ypx[10], ymx[10], xy2d[10];
      fx_load_entry(ypx, ymx, xy2d, q + (mag - 1));
      gex_madd(p, ypx, ymx, xy2d, dig < 0);
    }
  }
}
// encode(X/Z, Y/Z) == R ?  given zinv = 1/Z.  r = the signature's first 32 bytes as little-endian words.
BFTQ_HDI bool fx_encodes_to(const int32_t (&X)[10], const int32_t (&Y)[10], const int32_t (&zinv)[10], const uint32_t (&r)[8]) {
  int32_t x[10], y[10];
  fex_mul(x, X, zinv); fex_mul(y, Y, zinv);
  uint32_t wx[8], wy[8];
  fex_towords(wx, x); fex_towords(wy, y);
  wy[7] ^= (wx[0] & 1u) << 31;
  uint32_t diff = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) diff |= wy[i] ^ r[i];
  return diff == 0;
}

// ---- table-free verification (batches that bring many new keys): Shamir's trick over {B, -A, B - A} ------------------------
// 253 doublings + ~190 additions on the inlined field; same decisions as verify_core (ed25519.cuh), which stays as the
// host-side cross-check.  k = H(R || A || M) mod L.
BFTQ_HD bool verify_core_fast(const uint8_t* sig, const uint8_t* pk, const uint32_t (&k)[8]) {
  uint32_t s[8], r[8];
  for (int i = 0; i < 8; i++) {
    r[i] = (uint32_t)sig[4 * i] | ((uint32_t)sig[4 * i + 1] << 8) | ((uint32_t)sig[4 * i + 2] << 16) | ((uint32_t)sig[4 * i + 3] << 24);
    s[i] = (uint32_t)sig[32 + 4 * i] | ((uint32_t)sig[32 + 4 * i + 1] << 8) | ((uint32_t)sig[32 + 4 * i + 2] << 16) | ((uint32_t)sig[32 + 4 * i + 3] << 24);
  }
  if (!sc_words_canonical(s)) return false;                        // S >= L
  gex tab[3];                                                       // B, -A, B - A
  if (!gex_frombytes(tab[1], pk)) return false;
  for (int i = 0; i < 10; i++) { tab[1].X[i] = -tab[1].X[i]; tab[1].T[i] = -tab[1].T[i]; }
  gex_basepoint(tab[0]);
  gex_add(tab[2], tab[0], tab[1]);
  gex p;
  gex_identity(p);
  for (int bit = 252; bit >= 0; bit--) {
    gex_dbl(p, p);
    const int idx = (int)((s[bit >> 5] >> (bit & 31)) & 1u) | (int)(((k[bit >> 5] >> (bit & 31)) & 1u) << 1);
    if (idx) gex_add(p, p, tab[idx - 1]);
  }
  int32_t zi[10];
  fex_pow_chain(zi, p.Z, true);
  return fx_encodes_to(p.X, p.Y, zi, r);
}

}}  // namespace bftq::ed

#ifdef __CUDACC__
#include "pgp_digest.cuh"
namespace bftq {

// ---- table-free kernel: one thread per signature (ed::verify_core_fast).  status: 0 valid, 1 invalid, 4 key index out of range.
__global__ void __launch_bounds__(128)
ed25519_verify_kernel(const uint8_t* __restrict__ pubkeys, const uint32_t n_keys, const uint32_t* __restrict__ key_idx,
                      const uint8_t* __restrict__ sig, const uint8_t* __restrict__ msg, const uint64_t n_items,
                      uint8_t* __restrict__ status) {
  const uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  const uint32_t kidx = __ldg(key_idx + item);
  if (kidx >= n_keys) { status[item] = 4; return; }
  uint8_t s[64], a[32];
  for (int i = 0; i < 64; i++) s[i] = __ldg(sig + item * 64 + i);
  for (int i = 0; i < 32; i++) a[i] = __ldg(pubkeys + (uint64_t)kidx * 32 + i);
  // k = SHA-512(R || A || M): 96 bytes = one padded block
  uint64_t w[16];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    uint64_t r = 0, aa = 0, m = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) {
      r = (r << 8) | s[8 * i + b];
      aa = (aa << 8) | a[8 * i + b];
      m = (m << 8) | (uint64_t)__ldg(msg + item * 32 + 8 * i + b);
    }
    w[i] = r; w[4 + i] = aa; w[8 + i] = m;
  }
  w[12] = 0x8000000000000000ull; w[13] = 0; w[14] = 0;
  w[15] = 96 * 8;
  uint64_t h[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                   0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
  sha512_compress(h, w);
  uint8_t dg[64];
  for (int i = 0; i < 8; i++) for (int b = 0; b < 8; b++) dg[8 * i + b] = (uint8_t)(h[i] >> (56 - 8 * b));
  uint32_t k[8];
  ed::sc_reduce64(k, dg);
  status[item] = ed::verify_core_fast(s, a, k) ? 0 : 1;
}


struct EdSlotHdr { uint8_t key[32]; uint32_t ok; uint32_t pad[7]; };       // one per cache slot: the key bytes and "A decodes"
static_assert(sizeof(EdSlotHdr) == 64, "slot header");

// ---- table construction (runs once per key and engine) ---------------------------------------------------------------
// Step 1: thread = one point: decodes key number first_slot + t from its header (base_point: the one base point instead)
// and stores the nw window bases of -A (of B).
__global__ void __launch_bounds__(32)
ed25519_bases_kernel(EdSlotHdr* __restrict__ hdr, const uint32_t first_slot, const uint32_t n_points, ed::gex* __restrict__ bases,
                     const int nw, const int wbits, const int base_point) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_points) return;
  ed::gex P;
  if (base_point) ed::gex_basepoint(P);
  else {
    const uint32_t slot = first_slot + t;
    uint8_t a[32];
    for (int i = 0; i < 32; i++) a[i] = hdr[slot].key[i];
    const bool ok = ed::gex_frombytes(P, a);
    hdr[slot].ok = ok ? 1u : 0u;
    if (!ok) ed::gex_identity(P);                              // the table is never read (every signature under the key is invalid)
    for (int i = 0; i < 10; i++) { P.X[i] = -P.X[i]; P.T[i] = -P.T[i]; }
  }
  ed::fx_window_bases(bases + (size_t)t * nw, P, nw, wbits);
}
// Step 2: thread = (point, window, chunk of eight multiples); `tab` = the first point's table, `multiples` entries per window.
__global__ void __launch_bounds__(64)
ed25519_multiples_kernel(const ed::gex* __restrict__ bases, const uint32_t n_points, const int nw, const int multiples, ed::gea* __restrict__ tab) {
  const int chunks = multiples / ed::kFxChunk;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_points * nw * chunks) return;
  const uint32_t chunk = (uint32_t)(t % chunks), window = (uint32_t)((t / chunks) % nw), s = (uint32_t)(t / ((uint64_t)chunks * nw));
  const ed::gex base = bases[(size_t)s * nw + window];
  ed::fx_window_chunk(tab + ((size_t)s * nw + window) * multiples + chunk * ed::kFxChunk, base, (int)chunk);
}

// ---- kernel 1: one thread per signature, [S]B - [k]A ------------------------------------------------------------------
// Writes the projective result (X, Y, Z: 30 limbs, structure of arrays over n_pad items) and a preliminary status
// (0 = compare the encoding, else final: 1 invalid, 4 key index out of range).
#ifndef BFTQ_ED_ACC_BLOCK
#define BFTQ_ED_ACC_BLOCK 128
#endif
#ifndef BFTQ_ED_ACC_MINB
#define BFTQ_ED_ACC_MINB 3
#endif
constexpr int kEdAccBlock = BFTQ_ED_ACC_BLOCK;
__global__ void __launch_bounds__(kEdAccBlock, BFTQ_ED_ACC_MINB)
ed25519_accumulate_kernel(const ed::gea* __restrict__ tabB, const ed::gea* __restrict__ tab, const EdSlotHdr* __restrict__ hdr, const uint32_t* __restrict__ slot_of_key,
                          const uint32_t n_keys, const uint32_t* __restrict__ key_idx, const uint8_t* __restrict__ sig,
                          const uint8_t* __restrict__ msg, const uint64_t n_items, const uint64_t n_pad,
                          int32_t* __restrict__ xyz, uint8_t* __restrict__ pre_status) {
  __shared__ uint32_t sc[2][ed::kFxScalarWords][kEdAccBlock];    // the two scalars (+ a zero word each), one column per thread
  const uint64_t item = (uint64_t)blockIdx.x * kEdAccBlock + threadIdx.x;
  if (item >= n_items) return;
  uint8_t st = 0;
  const uint32_t kidx = __ldg(key_idx + item);
  uint32_t slot = 0;
  if (kidx >= n_keys) st = 4;
  else { slot = __ldg(slot_of_key + kidx); if (__ldg(&hdr[slot].ok) == 0u) st = 1; }
  uint32_t sw[16];                                             // R (8 words) || S (8 words), little-endian
  const uint8_t* sp = sig + item * 64;
  if ((reinterpret_cast<uintptr_t>(sig) & 15u) == 0) {
#pragma unroll
    for (int i = 0; i < 4; i++) { const uint4 v = __ldg(reinterpret_cast<const uint4*>(sp) + i); sw[4 * i] = v.x; sw[4 * i + 1] = v.y; sw[4 * i + 2] = v.z; sw[4 * i + 3] = v.w; }
  } else {
#pragma unroll
    for (int i = 0; i < 16; i++) sw[i] = (uint32_t)__ldg(sp + 4 * i) | ((uint32_t)__ldg(sp + 4 * i + 1) << 8) | ((uint32_t)__ldg(sp + 4 * i + 2) << 16) | ((uint32_t)__ldg(sp + 4 * i + 3) << 24);
  }
  uint32_t s[8];
#pragma unroll
  for (int i = 0; i < 8; i++) s[i] = sw[8 + i];
  if (st == 0 && !ed::sc_words_canonical(s)) st = 1;           // S >= L
  ed::gex p;
  ed::gex_identity(p);
  if (st == 0) {
    // k = SHA-512(R || A || M) mod L: 96 bytes = one padded block
    uint64_t w[16];
    const uint8_t* mp = msg + item * 32;
    const uint8_t* ap = hdr[slot].key;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      w[i] = ((uint64_t)__byte_perm(sw[2 * i], 0, 0x0123) << 32) | __byte_perm(sw[2 * i + 1], 0, 0x0123);
      uint64_t aa = 0, mm = 0;
#pragma unroll
      for (int b = 0; b < 8; b++) { aa = (aa << 8) | (uint64_t)__ldg(ap + 8 * i + b); mm = (mm << 8) | (uint64_t)__ldg(mp + 8 * i + b); }
      w[4 + i] = aa; w[8 + i] = mm;
    }
    w[12] = 0x8000000000000000ull; w[13] = 0; w[14] = 0; w[15] = 96 * 8;
    uint64_t h[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                     0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    sha512_compress(h, w);
    uint32_t x[16], k[8];                                      // the digest as a little-endian integer
#pragma unroll
    for (int i = 0; i < 8; i++) { x[2 * i] = __byte_perm((uint32_t)(h[i] >> 32), 0, 0x0123); x[2 * i + 1] = __byte_perm((uint32_t)h[i], 0, 0x0123); }
    ed::sc_reduce512(k, x);
#pragma unroll
    for (int i = 0; i < 8; i++) { sc[0][i][threadIdx.x] = s[i]; sc[1][i][threadIdx.x] = k[i]; }
    sc[0][8][threadIdx.x] = 0u; sc[1][8][threadIdx.x] = 0u;
    ed::fx_accumulate(p, &sc[0][0][threadIdx.x], &sc[1][0][threadIdx.x], kEdAccBlock, tabB, tab + (size_t)slot * ed::FxA::entries);
  }
#pragma unroll
  for (int i = 0; i < 10; i++) { xyz[(size_t)i * n_pad + item] = p.X[i]; xyz[(size_t)(10 + i) * n_pad + item] = p.Y[i]; xyz[(size_t)(20 + i) * n_pad + item] = p.Z[i]; }
  pre_status[item] = st;
}

// ---- kernel 2: eight results per thread share one inversion; encode and compare with R ---------------------------------
constexpr int kEdFinBlock = 64;
__global__ void __launch_bounds__(kEdFinBlock)
ed25519_finish_kernel(const int32_t* __restrict__ xyz, const uint8_t* __restrict__ pre_status, const uint8_t* __restrict__ sig,
                      const uint64_t n_items, const uint64_t n_pad, uint8_t* __restrict__ status) {
  const uint64_t threads = n_pad / ed::kFxChunk;               // n_pad is a multiple of 8 * kEdFinBlock
  const uint64_t t = (uint64_t)blockIdx.x * kEdFinBlock + threadIdx.x;
  if (t >= threads || t >= n_items) return;
  int32_t pre[ed::kFxChunk][10];                               // prefix products of the Z (items past the end count as 1)
#pragma unroll
  for (int j = 0; j < ed::kFxChunk; j++) {
    const uint64_t item = t + (uint64_t)j * threads;
    int32_t z[10];
#pragma unroll
    for (int i = 0; i < 10; i++) z[i] = item < n_items ? xyz[(size_t)(20 + i) * n_pad + item] : (i == 0);
    if (j == 0) ed::fex_copy(pre[0], z); else ed::fex_mul(pre[j], pre[j - 1], z);
  }
  int32_t inv[10];
  ed::fex_pow_chain(inv, pre[ed::kFxChunk - 1], true);
#pragma unroll
  for (int j = ed::kFxChunk - 1; j >= 0; j--) {
    const uint64_t item = t + (uint64_t)j * threads;
    int32_t zi[10];
    if (j > 0) {
      int32_t z[10], u[10];
#pragma unroll
      for (int i = 0; i < 10; i++) z[i] = item < n_items ? xyz[(size_t)(20 + i) * n_pad + item] : (i == 0);
      ed::fex_mul(zi, inv, pre[j - 1]); ed::fex_mul(u, inv, z); ed::fex_copy(inv, u);
    } else ed::fex_copy(zi, inv);
    if (item < n_items) {
      const uint8_t ps = pre_status[item];
      uint8_t out = ps;
      if (ps == 0) {
        int32_t X[10], Y[10];
#pragma unroll
        for (int i = 0; i < 10; i++) { X[i] = xyz[(size_t)i * n_pad + item]; Y[i] = xyz[(size_t)(10 + i) * n_pad + item]; }
        uint32_t r[8];
        const uint8_t* sp = sig + item * 64;
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = (uint32_t)__ldg(sp + 4 * i) | ((uint32_t)__ldg(sp + 4 * i + 1) << 8) | ((uint32_t)__ldg(sp + 4 * i + 2) << 16) | ((uint32_t)__ldg(sp + 4 * i + 3) << 24);
        out = ed::fx_encodes_to(X, Y, zi, r) ? 0 : 1;
      }
      status[item] = out;
    }
  }
}

}  // namespace bftq
#endif
