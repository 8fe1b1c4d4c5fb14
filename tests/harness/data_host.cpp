// Host build of DataEncryption's output layout (bftkv_b200/csrc/data_layout.hpp) for tests/test_data_encryption.py.
#include <cstring>
#include <vector>
#include "../../bftkv_b200/csrc/data_layout.hpp"

extern "C" {
// The message length for a value of `len` bytes; the layout words go to writes (up to cap), their count to *n_writes.
uint64_t data_layout_host(uint64_t len, uint32_t* writes, uint64_t cap, uint64_t* n_writes) {
  std::vector<uint32_t> w;
  const uint64_t total = bftq::k11::data_layout(len, &w);
  *n_writes = w.size();
  if (w.size() <= cap) memcpy(writes, w.data(), w.size() * 4);
  return total;
}
}
