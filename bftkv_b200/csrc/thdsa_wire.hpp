// Threshold DSA / ECDSA wire format on the host (crypto/threshold/dsa/dsa_core.go, dsa.go, ecdsa.go): P-256's group
// constants, the client's answer parsers (parseJointShare, parsePartialSignature), the two requests it writes
// (serializeSignRequest), OS2I and formatDSA.  Plain C++: bftq.cu includes it (thdsa_host.inc, thdsa_proc_host.inc), and
// tests/harness/thdsa_proc_host.cpp builds it with g++.
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <utility>
#include <vector>
#include "wire_host.hpp"

namespace {

// P-256's CurveParams as ecdsa.go serializes them
const uint8_t kP256P[32] = {0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x01, 0, 0, 0, 0, 0, 0, 0, 0,
                            0, 0, 0, 0, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff};
const uint8_t kP256N[32] = {0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x00, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                            0xbc, 0xe6, 0xfa, 0xad, 0xa7, 0x17, 0x9e, 0x84, 0xf3, 0xb9, 0xca, 0xc2, 0xfc, 0x63, 0x25, 0x51};
const uint8_t kP256B[32] = {0x5a, 0xc6, 0x35, 0xd8, 0xaa, 0x3a, 0x93, 0xe7, 0xb3, 0xeb, 0xbd, 0x55, 0x76, 0x98, 0x86, 0xbc,
                            0x65, 0x1d, 0x06, 0xb0, 0xcc, 0x53, 0xb0, 0xf6, 0x3b, 0xce, 0x3c, 0x3e, 0x27, 0xd2, 0x60, 0x4b};
const uint8_t kP256Gx[32] = {0x6b, 0x17, 0xd1, 0xf2, 0xe1, 0x2c, 0x42, 0x47, 0xf8, 0xbc, 0xe6, 0xe5, 0x63, 0xa4, 0x40, 0xf2,
                             0x77, 0x03, 0x7d, 0x81, 0x2d, 0xeb, 0x33, 0xa0, 0xf4, 0xa1, 0x39, 0x45, 0xd8, 0x98, 0xc2, 0x96};
const uint8_t kP256Gy[32] = {0x4f, 0xe3, 0x42, 0xe2, 0xfe, 0x1a, 0x7f, 0x9b, 0x8e, 0xe7, 0xeb, 0x4a, 0x7c, 0x0f, 0x9e, 0x16,
                             0x2b, 0xce, 0x33, 0x57, 0x6b, 0x31, 0x5e, 0xce, 0xcb, 0xb6, 0x40, 0x68, 0x37, 0xbf, 0x51, 0xf5};

// parseJointShare: u16 n, then n x (chunk, u64 node id); false on a framing error (nothing is kept then, as in Go).
bool thdsa_parse_joint_share(const uint8_t* d, uint64_t dl, std::vector<std::pair<const uint8_t*, uint64_t>>& cs, std::vector<uint64_t>& ids) {
  ThReader r{d, dl};
  uint16_t n;
  if (!r.u16(n)) return false;
  for (uint32_t k = 0; k < n; k++) {
    const uint8_t* c; uint64_t l; uint32_t hi, lo;
    if (!r.chunk(c, l) || !r.u32(hi) || !r.u32(lo)) return false;
    cs.push_back({c, l});
    ids.push_back(((uint64_t)hi << 32) | lo);
  }
  return true;
}

// parsePartialSignature: u64 x, chunk(s), chunk(v), the group (ParseParams: DSA chunks p, q, g; ECDSA chunks P, N, B, Gx,
// Gy and a u32 BitSize), the group's chunks without leading zeros.  Trailing bytes are ignored, as bytes.Reader leaves them.
struct ThdsaPartial { uint64_t x; const uint8_t *s, *v, *c[5]; uint64_t sl, vl, l[5]; uint32_t bits; };
bool thdsa_parse_partial(bool dsa, const uint8_t* d, uint64_t dl, ThdsaPartial& P) {
  ThReader r{d, dl};
  uint32_t hi, lo;
  if (!r.u32(hi) || !r.u32(lo) || !r.chunk(P.s, P.sl) || !r.chunk(P.v, P.vl)) return false;
  P.x = ((uint64_t)hi << 32) | lo;
  P.bits = 0;
  const int nc = dsa ? 3 : 5;
  for (int k = 0; k < nc; k++) {
    if (!r.chunk(P.c[k], P.l[k])) return false;
    th_strip(P.c[k], P.l[k]);
  }
  return dsa || r.u32(P.bits);
}

// The groups the device runs: DSA with p odd of exactly 1024 / 2048 bits and q odd, 1 < q < 2^256; exactly P-256.
bool thdsa_group_built(bool dsa, const ThdsaPartial& P) {
  if (!dsa)
    return th_eq(P.c[0], P.l[0], kP256P) && th_eq(P.c[1], P.l[1], kP256N) && th_eq(P.c[2], P.l[2], kP256B) && th_eq(P.c[3], P.l[3], kP256Gx) &&
           th_eq(P.c[4], P.l[4], kP256Gy) && P.bits == 256;
  const uint8_t *p = P.c[0], *q = P.c[1];
  const uint64_t pl = P.l[0], ql = P.l[1];
  return (pl == 128 || pl == 256) && (p[0] & 0x80) && (p[pl - 1] & 1) && ql >= 1 && ql <= 32 && (q[ql - 1] & 1) && (ql > 1 || q[0] > 1);
}

// big.Int.Bytes() of big-endian bytes
void thdsa_minimal(std::vector<uint8_t>& o, const uint8_t* b, uint64_t l) {
  while (l && !*b) { b++; l--; }
  o.assign(b, b + l);
}

// OS2I(dgst) for the order q (no leading zeros): dgst[:(|q| + 7) / 8] as m, shifted right by the excess bits on a curve
// (none for P-256's N, and DSA does not shift).  false where Go slices past the digest and panics.
bool thdsa_os2i(const std::vector<uint8_t>& dgst, const uint8_t* q, uint64_t ql, std::vector<uint8_t>& m) {
  if (dgst.size() < ql) return false;
  thdsa_minimal(m, dgst.data(), ql);
  return true;
}

// serializeSignRequest(nil, nil, kmap), the ids in `order` (one legal order of Go's map); the counts are Go's uint16 casts
void thdsa_request1(std::vector<uint8_t>& o, const std::vector<uint64_t>& order, const std::map<uint64_t, std::vector<std::vector<uint8_t>>>& kmap) {
  o.push_back(0);
  th_put_u16(o, (uint32_t)order.size());
  for (uint64_t id : order) {
    const auto& v = kmap.at(id);
    th_put_u32(o, (uint32_t)(id >> 32)); th_put_u32(o, (uint32_t)id);
    th_put_u16(o, (uint32_t)v.size());
    for (const auto& c : v) th_put_chunk(o, c.data(), c.size());
  }
}

// serializeSignRequest(m, r, nil): 01 || WriteBigInt(m) || WriteBigInt(r), m and r minimal
void thdsa_request2(std::vector<uint8_t>& o, const std::vector<uint8_t>& m, const std::vector<uint8_t>& r) {
  o.push_back(1);
  th_put_chunk(o, m.data(), m.size());
  th_put_chunk(o, r.data(), r.size());
}

// formatDSA(r, s, q): r and s left-padded to n = |q| bytes each; false where Go panics (r or s longer than n)
bool thdsa_format(const std::vector<uint8_t>& r, const uint8_t* s, uint64_t sl, uint32_t n, std::vector<uint8_t>& out) {
  while (sl && !*s) { s++; sl--; }
  if (r.size() > n || sl > n) return false;
  out.assign(2 * (size_t)n, 0);
  std::copy(r.begin(), r.end(), out.begin() + (n - r.size()));
  std::copy(s, s + sl, out.begin() + (2 * n - sl));
  return true;
}

}  // namespace
