// NIST P-256 point arithmetic, one thread per point, for the ECDSA half of row a12:
//   crypto/threshold/ecdsa/ecdsa.go:36-59  ecdsaGroupOperations.CalculateR
//     R = (sum_i lambda_i * R_i) * v^-1,  v = sum_i v_i lambda_i mod N,  r = R.x mod N
// (Go: elliptic.P256().ScalarMult / Add / Unmarshal).  Field elements are 8 x 32-bit limbs in
// Montgomery form mod p; points are Jacobian with a = -3; scalar multiplication is plain
// double-and-add (the batches here are tiny: 2t+1 scalar multiplications per signing session).
// __host__ __device__ throughout so the arithmetic is unit-tested on the CPU.
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define BFTQ_P_HD __host__ __device__ inline
#define BFTQ_P_HD_NOINLINE __host__ __device__ __noinline__
#else
#define BFTQ_P_HD inline
#define BFTQ_P_HD_NOINLINE inline
#endif

namespace bftq { namespace p256 {

typedef uint32_t fe[8];   // little-endian limbs

// p = 2^256 - 2^224 + 2^192 + 2^96 - 1
#define BFTQ_P256_P {0xffffffffu, 0xffffffffu, 0xffffffffu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000001u, 0xffffffffu}
// R mod p and R^2 mod p for R = 2^256;  -p^-1 mod 2^32 = 1
#define BFTQ_P256_R1 {0x00000001u, 0x00000000u, 0x00000000u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xfffffffeu, 0x00000000u}
#define BFTQ_P256_R2 {0x00000003u, 0x00000000u, 0xffffffffu, 0xfffffffbu, 0xfffffffeu, 0xffffffffu, 0xfffffffdu, 0x00000004u}
// curve coefficient b in Montgomery form
#define BFTQ_P256_BM {0x29c4bddfu, 0xd89cdf62u, 0x78843090u, 0xacf005cdu, 0xf7212ed6u, 0xe5a220abu, 0x04874834u, 0xdc30061du}

BFTQ_P_HD bool fe_ge(const fe a, const uint32_t (&p)[8]) { for (int i = 7; i >= 0; i--) { if (a[i] != p[i]) return a[i] > p[i]; } return true; }
BFTQ_P_HD void fe_set(fe r, const fe a) { for (int i = 0; i < 8; i++) r[i] = a[i]; }
BFTQ_P_HD bool fe_is_zero(const fe a) { uint32_t x = 0; for (int i = 0; i < 8; i++) x |= a[i]; return x == 0; }
BFTQ_P_HD bool fe_eq(const fe a, const fe b) { uint32_t x = 0; for (int i = 0; i < 8; i++) x |= a[i] ^ b[i]; return x == 0; }

BFTQ_P_HD void fe_add(fe r, const fe a, const fe b) {
  const uint32_t P[8] = BFTQ_P256_P;
  uint64_t c = 0; uint32_t t[8];
  for (int i = 0; i < 8; i++) { c += (uint64_t)a[i] + b[i]; t[i] = (uint32_t)c; c >>= 32; }
  if (c || fe_ge(t, P)) { uint64_t br = 0; for (int i = 0; i < 8; i++) { const uint64_t d = (uint64_t)t[i] - P[i] - br; t[i] = (uint32_t)d; br = (d >> 63) & 1; } }
  for (int i = 0; i < 8; i++) r[i] = t[i];
}
BFTQ_P_HD void fe_sub(fe r, const fe a, const fe b) {
  const uint32_t P[8] = BFTQ_P256_P;
  uint64_t br = 0; uint32_t t[8];
  for (int i = 0; i < 8; i++) { const uint64_t d = (uint64_t)a[i] - b[i] - br; t[i] = (uint32_t)d; br = (d >> 63) & 1; }
  if (br) { uint64_t c = 0; for (int i = 0; i < 8; i++) { c += (uint64_t)t[i] + P[i]; t[i] = (uint32_t)c; c >>= 32; } }
  for (int i = 0; i < 8; i++) r[i] = t[i];
}
// Field elements cross every non-inlined call BY VALUE (struct of 8 words: registers in, registers out).
// The first version passed uint32_t* into __noinline__ functions; nvcc 12.9 then coloured two live result
// buffers of the caller into one stack slot (visible in PTX: both calls got the same destination), which made
// the on-curve check fail on the device only.  By-value cores leave no address-taken temporaries to colour,
// and save the local-memory round trip per product.
struct fe_v { uint32_t v[8]; };
// Montgomery product a*b/R mod p (CIOS; -p^-1 mod 2^32 == 1 so q = t0)
BFTQ_P_HD_NOINLINE fe_v fe_mul_v(const fe_v a, const fe_v b) {
  const uint32_t P[8] = BFTQ_P256_P;
  uint32_t t[10];
  for (int i = 0; i < 10; i++) t[i] = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t c = 0;
    for (int j = 0; j < 8; j++) { const uint64_t v = (uint64_t)a.v[j] * b.v[i] + t[j] + c; t[j] = (uint32_t)v; c = v >> 32; }
    uint64_t v = (uint64_t)t[8] + c; t[8] = (uint32_t)v; t[9] = (uint32_t)(v >> 32);
    const uint32_t q = t[0];
    v = (uint64_t)q * P[0] + t[0]; c = v >> 32;
    for (int j = 1; j < 8; j++) { v = (uint64_t)q * P[j] + t[j] + c; t[j - 1] = (uint32_t)v; c = v >> 32; }
    v = (uint64_t)t[8] + c; t[7] = (uint32_t)v; t[8] = t[9] + (uint32_t)(v >> 32);
  }
  bool ge = t[8] != 0;
  if (!ge) { ge = true; for (int i = 7; i >= 0; i--) { if (t[i] != P[i]) { ge = t[i] > P[i]; break; } } }
  if (ge) { uint64_t br = 0; for (int i = 0; i < 8; i++) { const uint64_t d = (uint64_t)t[i] - P[i] - br; t[i] = (uint32_t)d; br = (d >> 63) & 1; } }
  fe_v r;
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
  return r;
}
BFTQ_P_HD void fe_mul(fe r, const fe a, const fe b) {
  fe_v x, y;
  for (int i = 0; i < 8; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  const fe_v z = fe_mul_v(x, y);
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
}
BFTQ_P_HD void fe_sq(fe r, const fe a) { fe_mul(r, a, a); }
BFTQ_P_HD void fe_to_mont(fe r, const fe a) { const uint32_t R2[8] = BFTQ_P256_R2; fe_mul(r, a, R2); }
BFTQ_P_HD void fe_from_mont(fe r, const fe a) { const uint32_t one[8] = {1, 0, 0, 0, 0, 0, 0, 0}; fe_mul(r, a, one); }
// a^(p-2) (Montgomery form in, Montgomery form out)
BFTQ_P_HD_NOINLINE fe_v fe_inv_v(const fe_v av) {
  const uint32_t P[8] = BFTQ_P256_P;
  fe a; for (int i = 0; i < 8; i++) a[i] = av.v[i];
  const uint32_t R1[8] = BFTQ_P256_R1;
  uint32_t e[8];
  for (int i = 0; i < 8; i++) e[i] = P[i];
  e[0] -= 2;                                              // p - 2 (no borrow: low limb is 0xffffffff)
  fe acc; fe_set(acc, R1);
  for (int bit = 255; bit >= 0; bit--) {
    fe_sq(acc, acc);
    if ((e[bit >> 5] >> (bit & 31)) & 1u) fe_mul(acc, acc, a);
  }
  fe_v r; for (int i = 0; i < 8; i++) r.v[i] = acc[i];
  return r;
}
BFTQ_P_HD void fe_inv(fe r, const fe a) {
  fe_v x; for (int i = 0; i < 8; i++) x.v[i] = a[i];
  const fe_v z = fe_inv_v(x);
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
}

struct pt { fe X, Y, Z; };        // Jacobian, Montgomery form; Z == 0 <=> point at infinity

BFTQ_P_HD void pt_inf(pt& p) { const uint32_t R1[8] = BFTQ_P256_R1; fe_set(p.X, R1); fe_set(p.Y, R1); for (int i = 0; i < 8; i++) p.Z[i] = 0; }
BFTQ_P_HD bool pt_is_inf(const pt& p) { return fe_is_zero(p.Z); }

// dbl-2001-b (a = -3)
BFTQ_P_HD_NOINLINE pt pt_dbl_v(const pt p) {
  pt r;
  if (pt_is_inf(p)) { r = p; return r; }
  fe delta, gamma, beta, alpha, t0, t1;
  fe_sq(delta, p.Z); fe_sq(gamma, p.Y); fe_mul(beta, p.X, gamma);
  fe_sub(t0, p.X, delta); fe_add(t1, p.X, delta); fe_mul(alpha, t0, t1);
  fe_add(t0, alpha, alpha); fe_add(alpha, t0, alpha);                 // 3 (X - delta)(X + delta)
  fe X3, Y3, Z3;
  fe_sq(X3, alpha); fe_add(t0, beta, beta); fe_add(t0, t0, t0); fe_add(t1, t0, t0);   // t0 = 4 beta, t1 = 8 beta
  fe_sub(X3, X3, t1);
  fe_add(Z3, p.Y, p.Z); fe_sq(Z3, Z3); fe_sub(Z3, Z3, gamma); fe_sub(Z3, Z3, delta);
  fe_sub(Y3, t0, X3); fe_mul(Y3, alpha, Y3);
  fe_sq(t1, gamma); fe_add(t1, t1, t1); fe_add(t1, t1, t1); fe_add(t1, t1, t1);       // 8 gamma^2
  fe_sub(Y3, Y3, t1);
  fe_set(r.X, X3); fe_set(r.Y, Y3); fe_set(r.Z, Z3);
  return r;
}
BFTQ_P_HD void pt_dbl(pt& r, const pt& p) { r = pt_dbl_v(p); }
// add-2007-bl with the special cases handled (infinity, P == Q, P == -Q)
BFTQ_P_HD_NOINLINE pt pt_add_v(const pt p, const pt q) {
  pt r;
  if (pt_is_inf(p)) { r = q; return r; }
  if (pt_is_inf(q)) { r = p; return r; }
  fe z1z1, z2z2, u1, u2, s1, s2, h, i, j, rr, v, t;
  fe_sq(z1z1, p.Z); fe_sq(z2z2, q.Z);
  fe_mul(u1, p.X, z2z2); fe_mul(u2, q.X, z1z1);
  fe_mul(s1, p.Y, q.Z); fe_mul(s1, s1, z2z2);
  fe_mul(s2, q.Y, p.Z); fe_mul(s2, s2, z1z1);
  fe_sub(h, u2, u1);
  fe_sub(rr, s2, s1);
  if (fe_is_zero(h)) {
    if (fe_is_zero(rr)) { r = pt_dbl_v(p); return r; }
    pt_inf(r); return r;
  }
  fe_add(rr, rr, rr);
  fe_add(i, h, h); fe_sq(i, i);
  fe_mul(j, h, i);
  fe_mul(v, u1, i);
  fe X3, Y3, Z3;
  fe_sq(X3, rr); fe_sub(X3, X3, j); fe_sub(X3, X3, v); fe_sub(X3, X3, v);
  fe_sub(t, v, X3); fe_mul(Y3, rr, t);
  fe_mul(t, s1, j); fe_add(t, t, t); fe_sub(Y3, Y3, t);
  fe_add(Z3, p.Z, q.Z); fe_sq(Z3, Z3); fe_sub(Z3, Z3, z1z1); fe_sub(Z3, Z3, z2z2); fe_mul(Z3, Z3, h);
  fe_set(r.X, X3); fe_set(r.Y, Y3); fe_set(r.Z, Z3);
  return r;
}
BFTQ_P_HD void pt_add(pt& r, const pt& p, const pt& q) { r = pt_add_v(p, q); }
// r = k * p, k: 8 little-endian words
BFTQ_P_HD_NOINLINE pt pt_mul_v(const pt p, const fe_v k) {
  pt acc; pt_inf(acc);
  for (int bit = 255; bit >= 0; bit--) {
    acc = pt_dbl_v(acc);
    if ((k.v[bit >> 5] >> (bit & 31)) & 1u) acc = pt_add_v(acc, p);
  }
  return acc;
}
BFTQ_P_HD void pt_mul(pt& r, const pt& p, const uint32_t (&k)[8]) {
  fe_v kv; for (int i = 0; i < 8; i++) kv.v[i] = k[i];
  r = pt_mul_v(p, kv);
}
// 32-byte big-endian <-> limbs
BFTQ_P_HD void be_to_limbs(uint32_t (&w)[8], const uint8_t* b) { for (int i = 0; i < 8; i++) w[i] = ((uint32_t)b[28 - 4 * i] << 24) | ((uint32_t)b[29 - 4 * i] << 16) | ((uint32_t)b[30 - 4 * i] << 8) | b[31 - 4 * i]; }
BFTQ_P_HD void limbs_to_be(uint8_t* b, const uint32_t (&w)[8]) { for (int i = 0; i < 8; i++) { b[28 - 4 * i] = (uint8_t)(w[i] >> 24); b[29 - 4 * i] = (uint8_t)(w[i] >> 16); b[30 - 4 * i] = (uint8_t)(w[i] >> 8); b[31 - 4 * i] = (uint8_t)w[i]; } }

// elliptic.Unmarshal: 65 bytes 04 || X || Y; false when not on the curve / coordinates >= p.
BFTQ_P_HD bool pt_from_xy(pt& p, const uint8_t* x_be, const uint8_t* y_be) {
  const uint32_t P[8] = BFTQ_P256_P;
  const uint32_t R1[8] = BFTQ_P256_R1;
  const uint32_t BM[8] = BFTQ_P256_BM;
  uint32_t x[8], y[8];
  be_to_limbs(x, x_be); be_to_limbs(y, y_be);
  if (fe_ge(x, P) || fe_ge(y, P)) return false;
  fe_to_mont(p.X, x); fe_to_mont(p.Y, y); fe_set(p.Z, R1);
  fe lhs, rhs, t;                                             // y^2 == x^3 - 3x + b
  fe_sq(lhs, p.Y);
  fe_sq(rhs, p.X); fe_mul(rhs, rhs, p.X);
  fe_add(t, p.X, p.X); fe_add(t, t, p.X); fe_sub(rhs, rhs, t); fe_add(rhs, rhs, BM);
  return fe_eq(lhs, rhs);
}
BFTQ_P_HD bool pt_from_uncompressed(pt& p, const uint8_t* s) { return s[0] == 4 && pt_from_xy(p, s + 1, s + 33); }
// affine coordinates (plain, big-endian); false for the point at infinity
BFTQ_P_HD bool pt_to_affine(uint8_t* x_be, uint8_t* y_be, const pt& p) {
  if (pt_is_inf(p)) return false;
  fe zi, zi2, zi3, ax, ay; uint32_t o[8];
  fe_inv(zi, p.Z); fe_sq(zi2, zi); fe_mul(zi3, zi2, zi);
  fe_mul(ax, p.X, zi2); fe_mul(ay, p.Y, zi3);
  fe_from_mont(o, ax); limbs_to_be(x_be, o);
  if (y_be) { fe_from_mont(o, ay); limbs_to_be(y_be, o); }
  return true;
}

// ---- arithmetic modulo the group order N (for ECDSA verification) ---------------------------------
#define BFTQ_P256_N {0xfc632551u, 0xf3b9cac2u, 0xa7179e84u, 0xbce6faadu, 0xffffffffu, 0xffffffffu, 0x00000000u, 0xffffffffu}
#define BFTQ_P256_NR1 {0x039cdaafu, 0x0c46353du, 0x58e8617bu, 0x43190552u, 0x00000000u, 0x00000000u, 0xffffffffu, 0x00000000u}
#define BFTQ_P256_NR2 {0xbe79eea2u, 0x83244c95u, 0x49bd6fa6u, 0x4699799cu, 0x2b6bec59u, 0x2845b239u, 0xf3d95620u, 0x66e12d94u}
#define BFTQ_P256_N0INV 0xee00bc4fu
#define BFTQ_P256_GXM {0x18a9143cu, 0x79e730d4u, 0x5fedb601u, 0x75ba95fcu, 0x77622510u, 0x79fb732bu, 0xa53755c6u, 0x18905f76u}
#define BFTQ_P256_GYM {0xce95560au, 0xddf25357u, 0xba19e45cu, 0x8b4ab8e4u, 0xdd21f325u, 0xd2e88688u, 0x25885d85u, 0x8571ff18u}

// Montgomery product modulo N
BFTQ_P_HD_NOINLINE fe_v sc_mul_v(const fe_v av, const fe_v bv) {
  const uint32_t M[8] = BFTQ_P256_N;
  const uint32_t* a = av.v; const uint32_t* b = bv.v;
  uint32_t t[10];
  for (int i = 0; i < 10; i++) t[i] = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t c = 0;
    for (int j = 0; j < 8; j++) { const uint64_t v = (uint64_t)a[j] * b[i] + t[j] + c; t[j] = (uint32_t)v; c = v >> 32; }
    uint64_t v = (uint64_t)t[8] + c; t[8] = (uint32_t)v; t[9] = (uint32_t)(v >> 32);
    const uint32_t q = t[0] * BFTQ_P256_N0INV;
    v = (uint64_t)q * M[0] + t[0]; c = v >> 32;
    for (int j = 1; j < 8; j++) { v = (uint64_t)q * M[j] + t[j] + c; t[j - 1] = (uint32_t)v; c = v >> 32; }
    v = (uint64_t)t[8] + c; t[7] = (uint32_t)v; t[8] = t[9] + (uint32_t)(v >> 32);
  }
  if (t[8] || fe_ge(t, M)) { uint64_t br = 0; for (int i = 0; i < 8; i++) { const uint64_t d = (uint64_t)t[i] - M[i] - br; t[i] = (uint32_t)d; br = (d >> 63) & 1; } }
  fe_v r; for (int i = 0; i < 8; i++) r.v[i] = t[i];
  return r;
}
BFTQ_P_HD void sc_mul(fe r, const fe a, const fe b) {
  fe_v x, y;
  for (int i = 0; i < 8; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  const fe_v z = sc_mul_v(x, y);
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
}
// ecdsa.Verify (Go crypto/ecdsa, as x/crypto's PublicKey.VerifySignature calls it for algorithm 19):
//   0 < r, s < N;  e = leftmost min(len, 32) bytes of the digest;  w = s^-1;  (x, y) = (e w) G + (r w) Q;
//   accept iff the point is finite and x mod N == r.   q: the public key (Montgomery/Jacobian, Z = 1).
BFTQ_P_HD bool ecdsa_verify_core(const pt& q, const uint32_t (&r)[8], const uint32_t (&s)[8], const uint8_t* digest, int dlen) {
  const uint32_t Nw[8] = BFTQ_P256_N;
  const uint32_t NR1[8] = BFTQ_P256_NR1;
  const uint32_t NR2[8] = BFTQ_P256_NR2;
  if (fe_is_zero(r) || fe_is_zero(s) || fe_ge(r, Nw) || fe_ge(s, Nw)) return false;
  const int take = dlen < 32 ? dlen : 32;           // hashToInt: leftmost 32 bytes, right-aligned
  uint32_t z[8];
  for (int i = 0; i < 8; i++) {
    uint32_t w = 0;
    for (int b = 0; b < 4; b++) { const int pos = take - 1 - (4 * i + b); if (pos >= 0) w |= (uint32_t)digest[pos] << (8 * b); }
    z[i] = w;
  }
  // w = s^(N-2) mod N (Montgomery domain), u1 = z w, u2 = r w (plain)
  fe sm, acc, zm, rm, u1, u2;
  sc_mul(sm, s, NR2);
  fe_set(acc, NR1);
  uint32_t e[8];
  for (int i = 0; i < 8; i++) e[i] = Nw[i];
  e[0] -= 2;
  for (int bit = 255; bit >= 0; bit--) {
    sc_mul(acc, acc, acc);
    if ((e[bit >> 5] >> (bit & 31)) & 1u) sc_mul(acc, acc, sm);
  }
  // z may exceed N: reduce by Montgomery round trip (z R2 / R = z R mod N; times plain w... ) -> use (zm * accM)/R = z w mod N
  sc_mul(zm, z, NR2);                 // z R mod N (z < 2^256 < 2N is fine for CIOS with one conditional subtraction)
  sc_mul(rm, r, NR2);
  sc_mul(u1, zm, acc);                // (zR)(wR)/R = z w R
  sc_mul(u2, rm, acc);
  const uint32_t one[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  sc_mul(u1, u1, one);                // leave Montgomery form
  sc_mul(u2, u2, one);
  // Shamir: table {G, Q, G + Q}
  const uint32_t R1[8] = BFTQ_P256_R1;
  const uint32_t GX[8] = BFTQ_P256_GXM;
  const uint32_t GY[8] = BFTQ_P256_GYM;
  pt tg, tgq;
  fe_set(tg.X, GX); fe_set(tg.Y, GY); fe_set(tg.Z, R1);
  tgq = pt_add_v(tg, q);
  pt p; pt_inf(p);
  for (int bit = 255; bit >= 0; bit--) {
    p = pt_dbl_v(p);
    const int idx = (int)((u1[bit >> 5] >> (bit & 31)) & 1u) | (int)(((u2[bit >> 5] >> (bit & 31)) & 1u) << 1);
    if (idx) {
      pt sel;                                       // word-wise select: no dynamically indexed table in local memory
      for (int w = 0; w < 8; w++) {
        sel.X[w] = idx == 1 ? tg.X[w] : (idx == 2 ? q.X[w] : tgq.X[w]);
        sel.Y[w] = idx == 1 ? tg.Y[w] : (idx == 2 ? q.Y[w] : tgq.Y[w]);
        sel.Z[w] = idx == 1 ? tg.Z[w] : (idx == 2 ? q.Z[w] : tgq.Z[w]);
      }
      p = pt_add_v(p, sel);
    }
  }
  if (pt_is_inf(p)) return false;
  uint32_t x[8];
  {
    fe zi, zi2, ax;
    fe_inv(zi, p.Z); fe_sq(zi2, zi); fe_mul(ax, p.X, zi2);
    fe_from_mont(x, ax);
  }
  if (fe_ge(x, Nw)) { uint64_t br = 0; for (int i = 0; i < 8; i++) { const uint64_t d = (uint64_t)x[i] - Nw[i] - br; x[i] = (uint32_t)d; br = (d >> 63) & 1; } }
  return fe_eq(x, r);
}

// ---- constant time: a * G for a secret a (K8, thdsa_sign.cuh) -------------------------------------
// Masked variants of fe_add / fe_sub / fe_mul: the final correction is always computed and selected with a mask, every
// loop has a fixed trip count, and everything is forced inline so no field element is ever addressed in local memory.
#ifdef __CUDACC__
#define BFTQ_P_CT __host__ __device__ __forceinline__
#else
#define BFTQ_P_CT inline
#endif

BFTQ_P_CT void fe_select(fe r, const fe a, const uint32_t take_a) {     // r = take_a ? a : r  (take_a 0 / 1)
  const uint32_t m = 0u - take_a;
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = (a[i] & m) | (r[i] & ~m);
}
BFTQ_P_CT void fe_add_ct(fe r, const fe a, const fe b) {
  const uint32_t P[8] = BFTQ_P256_P;
  uint32_t t[8], d[8], c = 0, br = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)a[i] + b[i] + c; t[i] = (uint32_t)v; c = (uint32_t)(v >> 32); }
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)t[i] - P[i] - br; d[i] = (uint32_t)v; br = (uint32_t)(v >> 63); }
  const uint32_t take = 0u - (c | (br ^ 1u));                    // a + b >= p
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = (d[i] & take) | (t[i] & ~take);
}
BFTQ_P_CT void fe_sub_ct(fe r, const fe a, const fe b) {
  const uint32_t P[8] = BFTQ_P256_P;
  uint32_t t[8], br = 0, c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)a[i] - b[i] - br; t[i] = (uint32_t)v; br = (uint32_t)(v >> 63); }
  const uint32_t m = 0u - br;                                    // a < b: add p back
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)t[i] + (P[i] & m) + c; r[i] = (uint32_t)v; c = (uint32_t)(v >> 32); }
}
// Montgomery product a*b/R mod p as fe_mul_v, with the final subtraction masked
BFTQ_P_CT void fe_mul_ct(fe r, const fe a, const fe b) {
  const uint32_t P[8] = BFTQ_P256_P;
  uint32_t t[10];
#pragma unroll
  for (int i = 0; i < 10; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { const uint64_t v = (uint64_t)a[j] * b[i] + t[j] + c; t[j] = (uint32_t)v; c = v >> 32; }
    uint64_t v = (uint64_t)t[8] + c; t[8] = (uint32_t)v; t[9] = (uint32_t)(v >> 32);
    const uint32_t q = t[0];
    v = (uint64_t)q * P[0] + t[0]; c = v >> 32;
#pragma unroll
    for (int j = 1; j < 8; j++) { v = (uint64_t)q * P[j] + t[j] + c; t[j - 1] = (uint32_t)v; c = v >> 32; }
    v = (uint64_t)t[8] + c; t[7] = (uint32_t)v; t[8] = t[9] + (uint32_t)(v >> 32);
  }
  uint32_t d[8], br = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) { const uint64_t v = (uint64_t)t[i] - P[i] - br; d[i] = (uint32_t)v; br = (uint32_t)(v >> 63); }
  const uint32_t take = 0u - ((uint32_t)(t[8] != 0u) | (br ^ 1u));
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = (d[i] & take) | (t[i] & ~take);
}
// a^(p-2): the exponent is the public constant p - 2, so the square-and-multiply pattern reveals nothing; 0 maps to 0.
BFTQ_P_CT void fe_inv_ct(fe r, const fe a) {
  const uint32_t R1[8] = BFTQ_P256_R1;
  fe acc;
#pragma unroll
  for (int i = 0; i < 8; i++) acc[i] = R1[i];
#pragma unroll 1
  for (int bit = 255; bit >= 0; bit--) {
    fe_mul_ct(acc, acc, acc);
    const int wi = bit >> 5;                                     // word wi of p - 2, without an indexed array
    const uint32_t e = (wi == 7 || wi == 2 || wi == 1) ? 0xffffffffu : wi == 6 ? 1u : wi == 0 ? 0xfffffffdu : 0u;
    if ((e >> (bit & 31)) & 1u) fe_mul_ct(acc, acc, a);
  }
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = acc[i];
}

// Homogeneous projective point (X : Y : Z), x = X / Z, y = Y / Z, Montgomery form; the identity is (0 : 1 : 0).
struct ppt { fe X, Y, Z; };

// Complete addition for a = -3 (Renes, Costello, Batina, "Complete addition formulas for prime order elliptic curves",
// EUROCRYPT 2016, Algorithm 4): one straight-line sequence for every pair of inputs, doublings and the identity included.
BFTQ_P_CT void ppt_add_ct(ppt& o, const ppt& p, const ppt& q) {
  const uint32_t BM[8] = BFTQ_P256_BM;
  fe t0, t1, t2, t3, t4, X3, Y3, Z3;
  fe_mul_ct(t0, p.X, q.X); fe_mul_ct(t1, p.Y, q.Y); fe_mul_ct(t2, p.Z, q.Z);
  fe_add_ct(t3, p.X, p.Y); fe_add_ct(t4, q.X, q.Y); fe_mul_ct(t3, t3, t4);
  fe_add_ct(t4, t0, t1); fe_sub_ct(t3, t3, t4); fe_add_ct(t4, p.Y, p.Z);
  fe_add_ct(X3, q.Y, q.Z); fe_mul_ct(t4, t4, X3); fe_add_ct(X3, t1, t2);
  fe_sub_ct(t4, t4, X3); fe_add_ct(X3, p.X, p.Z); fe_add_ct(Y3, q.X, q.Z);
  fe_mul_ct(X3, X3, Y3); fe_add_ct(Y3, t0, t2); fe_sub_ct(Y3, X3, Y3);
  fe_mul_ct(Z3, BM, t2); fe_sub_ct(X3, Y3, Z3); fe_add_ct(Z3, X3, X3);
  fe_add_ct(X3, X3, Z3); fe_sub_ct(Z3, t1, X3); fe_add_ct(X3, t1, X3);
  fe_mul_ct(Y3, BM, Y3); fe_add_ct(t1, t2, t2); fe_add_ct(t2, t1, t2);
  fe_sub_ct(Y3, Y3, t2); fe_sub_ct(Y3, Y3, t0); fe_add_ct(t1, Y3, Y3);
  fe_add_ct(Y3, t1, Y3); fe_add_ct(t1, t0, t0); fe_add_ct(t0, t1, t0);
  fe_sub_ct(t0, t0, t2); fe_mul_ct(t1, t4, Y3); fe_mul_ct(t2, t0, Y3);
  fe_mul_ct(Y3, X3, Z3); fe_add_ct(Y3, Y3, t2); fe_mul_ct(X3, t3, X3);
  fe_sub_ct(X3, X3, t1); fe_mul_ct(Z3, t4, Z3); fe_mul_ct(t1, t3, t0);
  fe_add_ct(Z3, Z3, t1);
#pragma unroll
  for (int i = 0; i < 8; i++) { o.X[i] = X3[i]; o.Y[i] = Y3[i]; o.Z[i] = Z3[i]; }
}

// The fixed-base table: entry (i, j) = (j + 1) 16^i G for window i = 0..63 and digit j + 1 = 1..15, affine X then Y in
// Montgomery form, 16 words per entry.  Public data, built once per engine by p256_base_table.
constexpr int kBaseWindows = 64, kBaseDigits = 15, kBaseEntryWords = 16;
constexpr int kBaseTableWords = kBaseWindows * kBaseDigits * kBaseEntryWords;

BFTQ_P_CT uint32_t base_tab_word(const uint32_t* tab, int k) {
#ifdef __CUDA_ARCH__
  return __ldg(tab + k);
#else
  return tab[k];
#endif
}

// out65 = elliptic.Marshal(a G) for a scalar a < 2^256 (8 little-endian words): 04 || x || y, and 04 || 0^64 when a G is
// the identity (a = 0 mod N).  One complete addition per 4-bit window, each reading all fifteen entries of its row with
// masks; the affine conversion inverts Z with the fixed exponent p - 2, which maps Z = 0 to 0 and so the identity to
// (0, 0) without a branch.
BFTQ_P_CT void base_mul_ct(uint8_t* out65, const uint32_t (&a)[8], const uint32_t* tab) {
  const uint32_t R1[8] = BFTQ_P256_R1;
  ppt acc;
#pragma unroll
  for (int i = 0; i < 8; i++) { acc.X[i] = 0u; acc.Y[i] = R1[i]; acc.Z[i] = 0u; }
#pragma unroll 1
  for (int w = 0; w < kBaseWindows; w++) {
    uint32_t word = 0u;                                          // a's word w / 8, by a masked scan (a stays in registers)
#pragma unroll
    for (int k = 0; k < 8; k++) word |= a[k] & (0u - (uint32_t)(k == (w >> 3)));
    const uint32_t d = (word >> (4 * (w & 7))) & 15u;
    ppt s;
#pragma unroll
    for (int i = 0; i < 8; i++) { s.X[i] = 0u; s.Y[i] = 0u; }
    const uint32_t* row = tab + w * kBaseDigits * kBaseEntryWords;
#pragma unroll 1
    for (int j = 0; j < kBaseDigits; j++) {
      const uint32_t m = 0u - (uint32_t)((uint32_t)(j + 1) == d);
#pragma unroll
      for (int i = 0; i < 8; i++) {
        s.X[i] |= base_tab_word(row, j * kBaseEntryWords + i) & m;
        s.Y[i] |= base_tab_word(row, j * kBaseEntryWords + 8 + i) & m;
      }
    }
    const uint32_t zero = 0u - (uint32_t)(d == 0u);              // digit 0: the identity (0 : 1 : 0)
#pragma unroll
    for (int i = 0; i < 8; i++) { s.Y[i] |= R1[i] & zero; s.Z[i] = R1[i] & ~zero; }
    ppt t;
    ppt_add_ct(t, acc, s);
    acc = t;
  }
  fe zi, x, y;
  const uint32_t one[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  fe_inv_ct(zi, acc.Z);
  fe_mul_ct(x, acc.X, zi); fe_mul_ct(y, acc.Y, zi);
  fe_mul_ct(x, x, one); fe_mul_ct(y, y, one);
  out65[0] = 4;
  limbs_to_be(out65 + 1, x);
  limbs_to_be(out65 + 33, y);
}

// Host: the table base_mul_ct reads (kBaseTableWords words), with the variable-time arithmetic above: G is public.
inline void base_table(uint32_t* tab) {
  const uint32_t R1[8] = BFTQ_P256_R1;
  const uint32_t GX[8] = BFTQ_P256_GXM;
  const uint32_t GY[8] = BFTQ_P256_GYM;
  pt b;                                                          // 16^i G
  fe_set(b.X, GX); fe_set(b.Y, GY); fe_set(b.Z, R1);
  for (int w = 0; w < kBaseWindows; w++) {
    pt m = b;
    for (int j = 0; j < kBaseDigits; j++) {
      uint8_t xb[32], yb[32];
      uint32_t xw[8], yw[8];
      pt_to_affine(xb, yb, m);
      be_to_limbs(xw, xb); be_to_limbs(yw, yb);
      uint32_t* e = tab + (w * kBaseDigits + j) * kBaseEntryWords;
      fe_to_mont(e, xw); fe_to_mont(e + 8, yw);
      pt_add(m, m, b);
    }
    for (int k = 0; k < 4; k++) pt_dbl(b, b);
  }
}

}}  // namespace bftq::p256

#ifdef __CUDACC__
namespace bftq {
// stage 1: one thread per (session, share): out[i] = lambda_i * R_i as a Jacobian point (24 words); ok[i] = 0 when R_i is
// not a curve point (elliptic.Unmarshal returns nil there and the reference then dereferences it).
__global__ void __launch_bounds__(128)
p256_scalar_mul_kernel(const uint8_t* __restrict__ points65, const uint8_t* __restrict__ scalars_be, const uint64_t n, uint32_t* __restrict__ out_jac,
                       uint8_t* __restrict__ ok) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t pb[65], kb[32];
  for (int b = 0; b < 65; b++) pb[b] = __ldg(points65 + i * 65 + b);
  for (int b = 0; b < 32; b++) kb[b] = __ldg(scalars_be + i * 32 + b);
  p256::pt p, r;
  const bool good = p256::pt_from_uncompressed(p, pb);
  uint32_t k[8];
  p256::be_to_limbs(k, kb);
  if (good) p256::pt_mul(r, p, k); else p256::pt_inf(r);
  for (int w = 0; w < 8; w++) { out_jac[i * 24 + w] = r.X[w]; out_jac[i * 24 + 8 + w] = r.Y[w]; out_jac[i * 24 + 16 + w] = r.Z[w]; }
  ok[i] = good ? 1 : 0;
}
// stage 2: one thread per session: P = sum of its k points; R = vinv * P; r = R.x mod N (ecdsa.go:55-58).
// status: 0 ok, 3 malformed input point / result at infinity.
__global__ void __launch_bounds__(128)
p256_sum_mul_kernel(const uint32_t* __restrict__ jac, const uint8_t* __restrict__ ok, const uint32_t k, const uint8_t* __restrict__ vinv_be,
                    const uint64_t n, uint8_t* __restrict__ out_r, uint8_t* __restrict__ status) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  p256::pt acc; p256::pt_inf(acc);
  bool good = true;
  for (uint32_t j = 0; j < k; j++) {
    p256::pt q, t;
    const uint64_t o = (i * k + j) * 24;
    for (int w = 0; w < 8; w++) { q.X[w] = __ldg(jac + o + w); q.Y[w] = __ldg(jac + o + 8 + w); q.Z[w] = __ldg(jac + o + 16 + w); }
    good = good && __ldg(ok + i * k + j);
    p256::pt_add(t, acc, q); acc = t;
  }
  uint8_t vb[32];
  for (int b = 0; b < 32; b++) vb[b] = __ldg(vinv_be + i * 32 + b);
  uint32_t v[8];
  p256::be_to_limbs(v, vb);
  p256::pt r;
  p256::pt_mul(r, acc, v);
  uint8_t xb[32];
  const bool finite = p256::pt_to_affine(xb, nullptr, r);
  // x mod N  (x < p < 2N: at most one subtraction)
  const uint32_t N[8] = {0xfc632551u, 0xf3b9cac2u, 0xa7179e84u, 0xbce6faadu, 0xffffffffu, 0xffffffffu, 0x00000000u, 0xffffffffu};
  uint32_t x[8];
  p256::be_to_limbs(x, xb);
  if (finite && p256::fe_ge(x, N)) { uint64_t br = 0; for (int w = 0; w < 8; w++) { const uint64_t d = (uint64_t)x[w] - N[w] - br; x[w] = (uint32_t)d; br = (d >> 63) & 1; } }
  if (!finite) for (int w = 0; w < 8; w++) x[w] = 0;
  p256::limbs_to_be(xb, x);
  for (int b = 0; b < 32; b++) out_r[i * 32 + b] = xb[b];
  status[i] = (good && finite) ? 0 : 3;
}

// ECDSA P-256 verification, one thread per signature.  keys: n_keys x 64 bytes (X || Y), r/s: n x 32 bytes big-endian
// (MPIs left-padded), digest: n x dlen.  status: 0 valid, 1 invalid, 3 key not on the curve, 4 key index out of range.
__global__ void __launch_bounds__(128)
ecdsa_p256_verify_kernel(const uint8_t* __restrict__ keys, const uint32_t n_keys, const uint32_t* __restrict__ key_idx,
                         const uint8_t* __restrict__ r_be, const uint8_t* __restrict__ s_be, const uint8_t* __restrict__ digest,
                         const uint32_t dlen, const uint64_t n, const uint8_t* __restrict__ pre_status, uint8_t* __restrict__ status) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (pre_status != nullptr && pre_status[i] != 0) { status[i] = pre_status[i]; return; }
  const uint8_t *kp, *rp, *sp;
  if (key_idx == nullptr) {          // packer layout: 128-byte records r || s || X || Y (keys = base of the records)
    rp = keys + i * 128; sp = rp + 32; kp = rp + 64;
  } else {
    const uint32_t kidx = __ldg(key_idx + i);
    if (kidx >= n_keys) { status[i] = 4; return; }
    kp = keys + (uint64_t)kidx * 64; rp = r_be + i * 32; sp = s_be + i * 32;
  }
  p256::pt q;
  if (!p256::pt_from_xy(q, kp, kp + 32)) { status[i] = 3; return; }
  uint32_t r[8], s[8];
  p256::be_to_limbs(r, rp); p256::be_to_limbs(s, sp);
  status[i] = p256::ecdsa_verify_core(q, r, s, digest + i * (uint64_t)dlen, (int)dlen) ? 0 : 1;
}
}  // namespace bftq
#endif
