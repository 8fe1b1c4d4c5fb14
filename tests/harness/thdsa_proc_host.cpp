// Host build of the threshold-DSA client's wire code (bftkv_b200/csrc/thdsa_wire.hpp) and the reduction of Byzantine
// sizes (bignum_host.hpp's be_mod).  Each entry writes a canonical form of its result for tests/test_thdsa_proc_host.py:
// -1 where the library reports a framing error or a Go panic.
#include <cstring>
#include <map>
#include <vector>
#include "../../bftkv_b200/csrc/bignum_host.hpp"
#include "../../bftkv_b200/csrc/thdsa_wire.hpp"
using namespace bftq::hostbig;

namespace {
int64_t put(const std::vector<uint8_t>& v, uint8_t* out, uint64_t cap) {
  if (v.size() > cap) return -2;
  memcpy(out, v.data(), v.size());
  return (int64_t)v.size();
}
}  // namespace

extern "C" {
// parseJointShare: count | (u64 id | chunk) per share
int64_t thdsa_joint_host(const uint8_t* d, uint64_t dl, uint8_t* out, uint64_t cap) {
  std::vector<std::pair<const uint8_t*, uint64_t>> cs;
  std::vector<uint64_t> ids;
  if (!thdsa_parse_joint_share(d, dl, cs, ids)) return -1;
  std::vector<uint8_t> o;
  th_put_u32(o, (uint32_t)cs.size());
  for (size_t k = 0; k < cs.size(); k++) {
    th_put_u32(o, (uint32_t)(ids[k] >> 32)); th_put_u32(o, (uint32_t)ids[k]);
    th_put_chunk(o, cs[k].first, cs[k].second);
  }
  return put(o, out, cap);
}
// parsePartialSignature: u64 x | chunk(s) | chunk(v minimal) | the group's chunks (minimal) | u32 BitSize | u8 built
int64_t thdsa_partial_host(int dsa, const uint8_t* d, uint64_t dl, uint8_t* out, uint64_t cap) {
  ThdsaPartial P;
  if (!thdsa_parse_partial(dsa != 0, d, dl, P)) return -1;
  std::vector<uint8_t> o;
  th_put_u32(o, (uint32_t)(P.x >> 32)); th_put_u32(o, (uint32_t)P.x);
  th_put_chunk(o, P.s, P.sl);
  th_put_minimal_chunk(o, P.v, P.vl);
  for (int k = 0; k < (dsa ? 3 : 5); k++) th_put_chunk(o, P.c[k], P.l[k]);
  th_put_u32(o, P.bits);
  o.push_back(thdsa_group_built(dsa != 0, P) ? 1 : 0);
  return put(o, out, cap);
}
// phase-1 request from the shares (ids[i], chunks c_off[i] .. c_off[i+1]) inserted in order
int64_t thdsa_request1_host(const uint64_t* ids, const uint8_t* c, const uint64_t* c_off, uint64_t n, uint8_t* out, uint64_t cap) {
  std::vector<uint64_t> order;
  std::map<uint64_t, std::vector<std::vector<uint8_t>>> kmap;
  for (uint64_t i = 0; i < n; i++) {
    if (!kmap.count(ids[i])) order.push_back(ids[i]);
    kmap[ids[i]].emplace_back(c + c_off[i], c + c_off[i + 1]);
  }
  std::vector<uint8_t> o;
  thdsa_request1(o, order, kmap);
  return put(o, out, cap);
}
// OS2I with the order q, then the phase-2 request with r
int64_t thdsa_request2_host(const uint8_t* dgst, uint64_t dlen, const uint8_t* q, uint64_t ql, const uint8_t* r, uint64_t rl, uint8_t* out,
                            uint64_t cap) {
  std::vector<uint8_t> m, rm, o;
  th_strip(q, ql);
  if (!thdsa_os2i(std::vector<uint8_t>(dgst, dgst + dlen), q, ql, m)) return -1;
  thdsa_minimal(rm, r, rl);
  thdsa_request2(o, m, rm);
  return put(o, out, cap);
}
// formatDSA(r, s, q) for n = |q| bytes
int64_t thdsa_format_host(const uint8_t* r, uint64_t rl, const uint8_t* s, uint64_t sl, uint32_t n, uint8_t* out, uint64_t cap) {
  std::vector<uint8_t> rm, o;
  thdsa_minimal(rm, r, rl);
  if (!thdsa_format(rm, s, sl, n, o)) return -1;
  return put(o, out, cap);
}
// b mod m, mlen bytes
void thdsa_be_mod_host(const uint8_t* b, uint64_t l, const uint8_t* m, uint32_t mlen, uint8_t* out) {
  const std::vector<uint8_t> v = be_mod(b, l, m, mlen);
  memcpy(out, v.data(), mlen);
}
}  // extern "C"
