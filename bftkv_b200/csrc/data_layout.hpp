// The byte layout of DataEncryption.Encrypt's output (x/crypto @53104e6ec876: SymmetricallyEncrypt(w, key, nil, nil),
// one Write(plain), Close) as a function of the value's length.  Plain C++: the library plans K11's encrypt calls with it,
// and tests/harness/data_host.cpp checks it against the Python restatement.
//
// Every Write in x/crypto's writer cascade reaches the outer partialLengthWriter as its own Write, which frames it as a run
// of power-of-two chunks (at most 2^14 bytes each).  In order:
//   the version byte (plain) | the 18-byte OCFB prefix | CB (the literal packet's stream header) | per Write into the
//   literal packet's own partialLengthWriter (74 00, the four time bytes, then the value): each of its chunks as two
//   Writes, length byte then data | that writer's closing 00 | the 22-byte MDC packet.
// Around them: the SKESK (32 bytes), D2 before and the outer writer's closing 00 after.
#pragma once
#include <cstdint>
#include <vector>

namespace bftq {
namespace k11 {

constexpr uint32_t kLayoutRaw = 0, kLayoutByte = 1, kLayoutPrefix = 2, kLayoutBody = 3, kLayoutMdc = 4;
constexpr uint64_t kSkeskBytes = 32;
// 't' (text mode), an empty file name, time 0: the literal body stream opens with these six bytes.
constexpr uint64_t kLiteralHead = 0x740000000000ull;

inline uint32_t layout_entry(uint32_t kind, uint32_t len, uint32_t byte = 0) { return kind << 24 | byte << 16 | len; }

// Bytes one Write of n bytes takes behind partialLengthWriter: a length byte per chunk.
inline uint64_t partial_bytes(uint64_t n) {
  uint64_t chunks = n >> 14, r = n & 0x3fff;
  while (r) { chunks += r & 1; r >>= 1; }
  return n + chunks;
}

// The Writes that reach the outer partialLengthWriter for a value of `len` bytes (appended to *writes when non-null, as
// layout_entry words), and the length of the whole message.
inline uint64_t data_layout(uint64_t len, std::vector<uint32_t>* writes) {
  uint64_t total = kSkeskBytes + 1 + 1;           // SKESK, D2, the closing 00
  auto put = [&](uint32_t kind, uint32_t n, uint32_t byte) {
    total += partial_bytes(n);
    if (writes) writes->push_back(layout_entry(kind, n, byte));
  };
  put(kLayoutRaw, 1, 0x01);                       // SEIPD version
  put(kLayoutPrefix, 18, 0);
  put(kLayoutByte, 1, 0xCB);                      // literal data, new format, partial lengths follow
  auto inner = [&](uint64_t n) {                  // one Write into the literal packet's partialLengthWriter
    while (n) {
      uint32_t p = 14;
      while ((1ull << p) > n) p--;
      put(kLayoutByte, 1, 224 + p);
      put(kLayoutBody, 1u << p, 0);
      n -= 1ull << p;
    }
  };
  inner(2);                                       // 't', name length 0
  inner(4);                                       // time
  inner(len);
  put(kLayoutByte, 1, 0x00);                      // the literal writer's Close
  put(kLayoutMdc, 22, 0);
  return total;
}

}  // namespace k11
}  // namespace bftq
