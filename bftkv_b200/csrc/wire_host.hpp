// The reference's wire format on the host, shared by thrsa_host.inc, thdsa_host.inc and auth_host.inc: the reader and
// writers below, and big-endian bytes as the little-endian words the kernels read.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

// bytes.Reader over a serialized structure (encoding/binary big-endian, packet.ReadChunk's u64-length chunks)
struct ThReader {
  const uint8_t* p; uint64_t len, pos = 0;
  bool u8(uint8_t& v) { if (len - pos < 1) return false; v = p[pos++]; return true; }
  bool u16(uint16_t& v) { if (len - pos < 2) return false; v = (uint16_t)((p[pos] << 8) | p[pos + 1]); pos += 2; return true; }
  bool u32(uint32_t& v) {
    if (len - pos < 4) return false;
    v = ((uint32_t)p[pos] << 24) | ((uint32_t)p[pos + 1] << 16) | ((uint32_t)p[pos + 2] << 8) | p[pos + 3];
    pos += 4;
    return true;
  }
  bool chunk(const uint8_t*& c, uint64_t& l) {
    if (len - pos < 8) return false;
    l = 0;
    for (int k = 0; k < 8; k++) l = (l << 8) | p[pos + k];
    pos += 8;
    if (l > len - pos) return false;                 // io.ReadFull: unexpected EOF
    c = p + pos;
    pos += l;
    return true;
  }
};
void th_put_u16(std::vector<uint8_t>& o, uint32_t v) { o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
void th_put_u32(std::vector<uint8_t>& o, uint32_t v) { for (int s = 24; s >= 0; s -= 8) o.push_back((uint8_t)(v >> s)); }
void th_put_chunk(std::vector<uint8_t>& o, const uint8_t* c, uint64_t l) {
  for (int s = 56; s >= 0; s -= 8) o.push_back((uint8_t)(l >> s));
  o.insert(o.end(), c, c + l);
}
// big.Int.Bytes(): the minimal big-endian form (empty for zero)
void th_put_minimal_chunk(std::vector<uint8_t>& o, const uint8_t* be, uint64_t l) {
  while (l && *be == 0) { be++; l--; }
  th_put_chunk(o, be, l);
}

void th_strip(const uint8_t*& c, uint64_t& l) { while (l && *c == 0) { c++; l--; } }
bool th_eq(const uint8_t* c, uint64_t l, const uint8_t (&v)[32]) { th_strip(c, l); return l == 32 && memcmp(c, v, 32) == 0; }
// big-endian bytes -> little-endian words, ceil(l / 4) of them appended to w (a word vector with any allocator)
template <class V> void th_words(V& w, const uint8_t* c, uint64_t l) {
  const uint64_t nw = (l + 3) / 4, at = w.size();
  w.resize(at + nw, 0);
  for (uint64_t b = 0; b < l; b++) {
    const uint64_t bit = l - 1 - b;
    w[at + bit / 4] |= (uint32_t)c[b] << (8 * (bit % 4));
  }
}

}  // namespace
