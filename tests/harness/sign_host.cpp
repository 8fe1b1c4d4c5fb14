// Host build of K12's packet helpers (bftkv_b200/csrc/sign_packet.hpp) for tests/test_signature_sign.py.
#include "../../bftkv_b200/csrc/sign_packet.hpp"

extern "C" {
void sign_suffix_host(uint32_t ctime, uint64_t key_id, uint8_t* out) { bftq::k12::sign_suffix(ctime, key_id, out); }
void sign_release_host(const uint8_t* status, uint64_t n_items, uint8_t* packets, int32_t* out_err) {
  bftq::k12::sign_release(status, n_items, packets, out_err);
}
}
