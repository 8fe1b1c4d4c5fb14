// K0m / K2m — the read path from raw transport answers: packets in, Client.Read's decision out.
//
// What protocol/client.go:250-268 does per read operation, once the host has removed the encryption layer of every
// answer (RSA private-key operation + AES-CFB / MDC stay on the host): for each response
//   transport.Multicast (transport/transport.go:116-126)  tr.Decrypt -> PGPMessage.Decrypt (crypto_pgp.go:453-471):
//       readSignedMessage + signatureCheckReader — hash the literal body, verify the trailing signature with the key the
//       one-pass packet names (an unknown signer is NOT an error) — then the nonce in the literal FileName must equal the
//       nonce the request carried (ErrTransportNonceMismatch)
//   Client.processResponse (client.go:207-230)            packet.Parse(res.Data) -> bucket (t, value)
// and per operation the arrival-order decision of bftq_read_decide_batch.
//
// K0m, one thread per response, takes the message bytes as the caller handed them over and, when the message has the
// one shape every bftkv answer has — one-pass signature (v3, binary, SHA-256, last), literal data in any framing Go or
// GnuPG emit (definite, or partial-length chunks), ONE v4 RSA signature packet to the end, signer with exactly one usable
// 2048-bit RSA key or no key at all — de-chunks the literal body into a scratch buffer, base64-decodes the FileName and
// compares it with the expected nonce, parses the body as a bftkv packet (bftkv_packet.hpp), hashes body || hashed area
// || trailer, applies the hash-tag check and lays out K1's inputs.  Every other shape is flagged and goes through the
// host packer (plan_message) afterwards: a fallback is always safe, the flag — not a guess — decides.
// K2m, one warp per operation, finalises the statuses (signature verdict from K1, then nonce, then packet.Parse), groups
// equal values by exact byte comparison and takes the decision.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "bftkv_packet.hpp"
#include "pgp_digest.cuh"
#include "pgp_fastparse.hpp"
#include "pgp_parse.cuh"
#include "tally.cuh"

namespace bftq {

constexpr uint8_t kAuxNonceMismatch = 0x01, kAuxPacketError = 0x02, kAuxNonceCorrupt = 0x04;
constexpr uint8_t kStUnverifiedSigner = 8;      // BFTQ_ST_UNVERIFIED_SIGNER
constexpr uint8_t kStNonceMismatch = 7;         // BFTQ_ST_NONCE_MISMATCH
constexpr int kMaxFastName = 32, kMaxNonce = 24;

// Sequential reader over a literal data packet's body: one definite-length run, or Go's / GnuPG's partial-length chunks.
struct LitReader {
  const uint8_t* m; uint32_t n;      // the whole message
  uint32_t pos;                      // next byte
  uint32_t rem;                      // bytes left in the current chunk
  bool last, bad;                    // current chunk is the final one / framing ran off the message
  __device__ __forceinline__ void next_len() {            // new-format length octet(s) at pos
    if (pos >= n) { bad = true; rem = 0; last = true; return; }
    const uint8_t o = m[pos];
    if (o < 192) { rem = o; pos += 1; last = true; }
    else if (o < 224) { if (pos + 2 > n) { bad = true; last = true; rem = 0; return; } rem = ((uint32_t)(o - 192) << 8) + m[pos + 1] + 192; pos += 2; last = true; }
    else if (o == 255) { if (pos + 5 > n) { bad = true; last = true; rem = 0; return; } rem = ((uint32_t)m[pos + 1] << 24) | ((uint32_t)m[pos + 2] << 16) | ((uint32_t)m[pos + 3] << 8) | m[pos + 4]; pos += 5; last = true; }
    else { rem = 1u << (o & 0x1f); pos += 1; last = false; }
    if (rem > n - pos) { bad = true; rem = 0; last = true; }
  }
  // false at the end of the packet
  __device__ __forceinline__ bool get(uint8_t& b) {
    while (rem == 0) { if (last) return false; next_len(); }
    b = m[pos++]; rem--;
    return true;
  }
};

__device__ __forceinline__ int b64val(uint8_t c) {
  if (c >= 'A' && c <= 'Z') return c - 'A';
  if (c >= 'a' && c <= 'z') return c - 'a' + 26;
  if (c >= '0' && c <= '9') return c - '0' + 52;
  if (c == '+') return 62;
  if (c == '/') return 63;
  return -1;
}

__global__ void __launch_bounds__(128)
msg_parse_digest_kernel(const uint8_t* __restrict__ msg_blob, const uint64_t* __restrict__ msg_off, const uint64_t msg_base, const uint32_t n_items,
                        const IssuerEntry* __restrict__ issuers, const uint32_t n_issuers, const uint8_t* __restrict__ pre_in /* nullable */,
                        const uint8_t* __restrict__ nonce_blob, const uint32_t nonce_len, uint8_t* __restrict__ plain_blob,
                        uint32_t* __restrict__ out_key_idx, uint8_t* __restrict__ out_sig /* n x 256 */, uint8_t* __restrict__ out_digest /* n x 32 */,
                        uint8_t* __restrict__ out_pre, uint8_t* __restrict__ out_where, uint8_t* __restrict__ out_aux, uint64_t* __restrict__ out_ts,
                        uint32_t* __restrict__ out_voff, uint32_t* __restrict__ out_vlen, uint32_t* __restrict__ out_plen,
                        uint64_t* __restrict__ out_signed_by, const uint64_t* __restrict__ msg_end = nullptr /* item i ends at msg_end[i], not msg_off[i+1] */) {
  // the SHA-256 message block of every thread lives in shared memory (word-major: conflict-free), so the byte stream can be
  // absorbed with a dynamic word index without spilling sixteen registers to local memory
  __shared__ uint32_t w_s[16][128];
  const uint32_t item_raw = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = item_raw < n_items;
  const uint32_t item = live ? item_raw : n_items - 1;
  const int lane = threadIdx.x & 31;
  const uint64_t o0 = msg_off[item] - msg_base, o1 = (msg_end != nullptr ? msg_end[item] : msg_off[item + 1]) - msg_base;
  const uint8_t* m = msg_blob + o0;
  uint8_t* plain = plain_blob + ((o0 + 3) & ~(uint64_t)3);        // 4-byte aligned inside the item's span (the fast path stores words)
  uint8_t where = kParseDecided, pre = 0, aux = 0;
  uint32_t kidx = 0, plen = 0, voff = 0, vlen = 0;
  uint64_t ts = 0, signed_by = 0;
  bool copy = false;
  fastparse::FastSig f;
  f.mpi_off = 0; f.mpi_len = 0; f.hashed_off = 0; f.hashed_len = 0; f.tag = 0;
  uint32_t sig_at = 0;
  const uint8_t given = pre_in != nullptr ? pre_in[item] : (uint8_t)0;
  if (given != 0) pre = given;                                   // the transport failed before this point: nothing to look at
  else if (o1 - o0 < 18 || o1 - o0 > 0x3fffffffull) where = kParseHost;
  else {
    const uint32_t n = (uint32_t)(o1 - o0);
    // ---- one-pass signature: new-format C4 0D or old-format 90 0D, 13 bytes: 03 type hash pkalgo keyid[8] last
    if (!((m[0] == 0xC4 || m[0] == 0x90) && m[1] == 13 && m[2] == 3 && m[3] == 0x00 && m[4] == 8 && m[14] != 0)) where = kParseHost;
    else {
      for (int i = 0; i < 8; i++) signed_by = (signed_by << 8) | m[6 + i];
      LitReader r{m, n, 15, 0, true, false};
      const uint8_t hdr = m[15];
      r.pos = 16;
      if (hdr == 0xCB) r.next_len();                             // new format: any length form
      else if ((hdr & 0xFC) == 0xAC && (hdr & 3) != 3) {         // old format tag 11, definite length
        const uint32_t nl = 1u << (hdr & 3);
        if (16 + nl > n) r.bad = true;
        else { uint32_t l = 0; for (uint32_t i = 0; i < nl; i++) l = (l << 8) | m[16 + i]; r.pos = 16 + nl; r.rem = l; r.last = true; if (l > n - r.pos) r.bad = true; }
      } else r.bad = true;
      // ---- literal header: format, name length, name, time
      uint8_t b, name[kMaxFastName];
      uint32_t name_len = 0;
      bool okh = !r.bad && r.get(b);                             // format byte ('b' / 't' / 'u': the one-pass type decides the hashing)
      okh = okh && r.get(b);
      if (okh) { name_len = b; if (name_len > (uint32_t)kMaxFastName) okh = false; }
      for (uint32_t i = 0; okh && i < name_len; i++) { okh = r.get(b); name[i] = b; }
      for (int i = 0; okh && i < 4; i++) okh = r.get(b);
      if (!okh || r.bad) where = kParseHost;
      else {
        // ---- ONE loop over the hashed byte stream: the literal body (de-chunked into the scratch as it passes), then — once the
        // signature packet behind it has been parsed and its signer found — the packet's hashed area, the v4 trailer and the
        // SHA-256 padding.  A single absorb / compress site keeps the kernel small.
        uint32_t h[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
        uint32_t cur = 0, tot = 0, spos = 0, msg_bytes = 0;
        int phase = 0, pad_state = 0, pad_k = 0;                 // 0 body, 1 suffix, 2 padding
        const uint8_t* suf = nullptr;
        bool done = false, hashing = true;
        while (!done) {
          // ---- fast path: a whole 64-byte block of the body inside one chunk, at a block boundary of the hash — seventeen
          // independent aligned word loads (latency overlapped), funnel-shifted to the stream's alignment, one compress, sixteen
          // word stores into the scratch.  Everything else (chunk headers, the tail, the suffix, the padding) takes the byte loop.
          while (phase == 0 && (tot & 63u) == 0u && r.rem >= 64u) {
            const uintptr_t a = reinterpret_cast<uintptr_t>(m + r.pos);
            const uint32_t sh = (uint32_t)(a & 3u) * 8u;
            const uint32_t* aw = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
            uint32_t x[17];
#pragma unroll
            for (int i = 0; i < 17; i++) x[i] = __ldg(aw + i);        // x[16] may lie up to 3 bytes behind the message: inside the buffer's slack
            uint32_t w[16];
            uint32_t* pw = reinterpret_cast<uint32_t*>(plain + plen);
#pragma unroll
            for (int i = 0; i < 16; i++) {
              const uint32_t le = __funnelshift_r(x[i], x[i + 1], sh);
              pw[i] = le;
              w[i] = __byte_perm(le, 0, 0x0123);
            }
            sha256_compress(h, w);
            r.pos += 64u; r.rem -= 64u; tot += 64u; plen += 64u;
          }
          if (phase == 0) {
            if (r.get(b)) plain[plen++] = b;
            else {
              // ---- the body has ended: everything that decides whether (and against which key) the digest is needed
              hashing = false;
              if (r.bad) { where = kParseHost; break; }
              sig_at = r.pos;
              if (sig_at >= n || fastparse::parse(m + sig_at, (size_t)(n - sig_at), f) != fastparse::kFast || f.hash_id != 8) { where = kParseHost; break; }
              int hit = -1;                                      // md.SignedBy = first key of KeysByIdUsage(one-pass key id, sign)
              for (uint32_t i = 0; i < n_issuers; i++) if (issuers[i].key_id == signed_by) { hit = (int)i; break; }
              if (hit < 0) pre = kStUnverifiedSigner;            // unknown signer: SignatureError stays nil, nothing is verified
              else {
                const IssuerEntry en = issuers[hit];
                if (en.kind != 0) { where = kParseHost; break; }
                kidx = en.key_idx;
                hashing = true;
                if (en.algo != f.pk_algo) pre = 1;
                if (f.mpi_len > en.kbytes) { if (!pre) pre = 1; }
                else copy = true;
              }
              // ---- nonce: base64.StdEncoding.DecodeString(FileName) == the request's nonce (CR / LF skipped, padding mandatory)
              {
                uint8_t dec[kMaxNonce]; uint32_t nd = 0; uint8_t q[4] = {0, 0, 0, 0}; int nq = 0; bool closed = false, corrupt = false;
                for (uint32_t i = 0; i < name_len && !corrupt; i++) {
                  const uint8_t c = name[i];
                  if (c == '\r' || c == '\n') continue;
                  if (closed) { corrupt = true; break; }
                  if (c == '=') {
                    if (nq < 2) { corrupt = true; break; }
                    if (nq == 2) {
                      uint32_t j = i + 1;
                      while (j < name_len && (name[j] == '\r' || name[j] == '\n')) j++;
                      if (j >= name_len || name[j] != '=') { corrupt = true; break; }
                      i = j;
                    }
                    const int v0 = b64val(q[0]), v1 = b64val(q[1]), v2 = nq > 2 ? b64val(q[2]) : 0;
                    if (nd + 2 > (uint32_t)kMaxNonce) { corrupt = true; break; }
                    dec[nd++] = (uint8_t)((v0 << 2) | (v1 >> 4));
                    if (nq > 2) dec[nd++] = (uint8_t)(((v1 & 15) << 4) | (v2 >> 2));
                    nq = 0; closed = true;
                    continue;
                  }
                  if (b64val(c) < 0) { corrupt = true; break; }
                  q[nq++] = c;
                  if (nq == 4) {
                    if (nd + 3 > (uint32_t)kMaxNonce) { corrupt = true; break; }
                    const int v0 = b64val(q[0]), v1 = b64val(q[1]), v2 = b64val(q[2]), v3 = b64val(q[3]);
                    dec[nd++] = (uint8_t)((v0 << 2) | (v1 >> 4)); dec[nd++] = (uint8_t)(((v1 & 15) << 4) | (v2 >> 2)); dec[nd++] = (uint8_t)(((v2 & 3) << 6) | v3);
                    nq = 0;
                  }
                }
                if (nq != 0) corrupt = true;
                if (corrupt) aux |= kAuxNonceCorrupt;              // Decrypt returns the base64 error BEFORE looking at SignatureError
                else {
                  bool same = nd == nonce_len;
                  for (uint32_t i = 0; same && i < nonce_len; i++) same = dec[i] == nonce_blob[(size_t)item * nonce_len + i];
                  if (!same) aux |= kAuxNonceMismatch;
                }
              }
              // ---- processResponse: packet.Parse of a non-empty answer
              if (plen > 0) {
                const pkt::View v = pkt::parse(plain, plen);
                if (v.err) aux |= kAuxPacketError;
                else { ts = v.t; voff = v.value_off; vlen = v.value_len; }
              }
              if (!hashing || (pre != 0 && pre != 1)) { hashing = false; break; }
              suf = m + sig_at + f.hashed_off;
              phase = 1;
              continue;
            }
          } else if (phase == 1) {
            const uint32_t hl = f.hashed_len;
            if (spos < hl) b = suf[spos];
            else if (spos < hl + 6) { const uint32_t q = spos - hl; b = q == 0 ? 0x04 : q == 1 ? 0xff : (uint8_t)((hl >> (8 * (5 - q))) & 0xffu); }
            else { phase = 2; msg_bytes = tot; continue; }
            spos++;
          } else {
            if (pad_state == 0) { b = 0x80; pad_state = 1; }
            else if (pad_state == 1) { if ((tot & 63u) != 56u) b = 0; else { pad_state = 2; continue; } }
            else { const uint64_t bits = (uint64_t)msg_bytes * 8ull; b = (uint8_t)(bits >> (8 * (7 - pad_k))); pad_k++; if (pad_k == 8) done = true; }
          }
          // ---- absorb one byte; every fourth completes a word, every 64th a block
          cur = (cur << 8) | b;
          tot++;
          if ((tot & 3u) == 0u) {
            w_s[((tot - 1u) >> 2) & 15u][threadIdx.x] = cur;
            if ((tot & 63u) == 0u) {
              uint32_t w[16];
#pragma unroll
              for (int i = 0; i < 16; i++) w[i] = w_s[i][threadIdx.x];
              sha256_compress(h, w);
            }
          }
        }
        if (where == kParseDecided && hashing) {
          uint32_t* o = reinterpret_cast<uint32_t*>(out_digest + (size_t)item * 32);
#pragma unroll
          for (int i = 0; i < 8; i++) o[i] = __byte_perm(h[i], 0, 0x0123);
          if (!pre && (uint16_t)(h[0] >> 16) != f.tag) pre = 2;     // BFTQ_ST_HASH_TAG
        }
      }
    }
  }
  if (where == kParseHost) { pre = 6; copy = false; aux = 0; }    // K1 leaves the item alone; the host packer decides it
  if (!live) copy = false;
  // ---- per warp: left-pad the signature MPIs into K1's layout, coalesced (as K0)
  const uint64_t src_pos = o0 + sig_at + f.mpi_off;
  for (int j = 0; j < 32; j++) {
    if (!__shfl_sync(0xffffffffu, (int)copy, j)) continue;
    const uint32_t it = __shfl_sync(0xffffffffu, item, j);
    const uint32_t len = __shfl_sync(0xffffffffu, f.mpi_len, j);
    const uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)src_pos, j), hi = __shfl_sync(0xffffffffu, (uint32_t)(src_pos >> 32), j);
    const uint8_t* src = msg_blob + (((uint64_t)hi << 32) | lo);
    const uint32_t padn = 256u - len;
    uint32_t* dst = reinterpret_cast<uint32_t*>(out_sig + (size_t)it * 256);
#pragma unroll
    for (int t = 0; t < 2; t++) {
      const uint32_t b0 = (uint32_t)(t * 32 + lane) * 4u;
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const uint32_t idx = b0 + b;
        const uint32_t byte = idx >= padn ? (uint32_t)__ldg(src + (idx - padn)) : 0u;
        v |= byte << (8 * b);
      }
      dst[t * 32 + lane] = v;
    }
  }
  if (live) {
    out_key_idx[item] = kidx; out_pre[item] = pre; out_where[item] = where; out_aux[item] = aux;
    out_ts[item] = ts; out_voff[item] = voff; out_vlen[item] = vlen; out_plen[item] = plen;
    if (out_signed_by != nullptr) out_signed_by[item] = signed_by;
  }
}

// The plain text of every good answer (status OK / UNVERIFIED_SIGNER), one warp per answer: plain_len[i] bytes from
// plain_ptr[i] to out + (off[i] - base), the rest of the answer's span zeroed; out_len[i] = that length (0 otherwise).
__global__ void __launch_bounds__(256)
plain_gather_kernel(const uint8_t* __restrict__ status, const uint64_t* __restrict__ plain_ptr, const uint32_t* __restrict__ plain_len,
                    const uint64_t* __restrict__ off, const uint64_t base, const uint32_t n_items, uint8_t* __restrict__ out, uint32_t* __restrict__ out_len) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n_items) return;
  const uint64_t o0 = off[i] - base, span = off[i + 1] - off[i];
  const uint8_t st = status[i];
  const uint32_t len = (st == 0 || st == kStUnverifiedSigner) ? plain_len[i] : 0u;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(plain_ptr[i]);
  for (uint64_t k = lane; k < span; k += 32) out[o0 + k] = k < len ? src[k] : (uint8_t)0;
  if (lane == 0) out_len[i] = len;
}

// K2m: one warp per operation (<= 32 responders).  status[] holds K1's verdicts (or the host packer's for the flagged
// items, with aux cleared); this kernel applies the nonce and packet.Parse checks, writes the final status back, assigns
// value ids by exact byte comparison and decides as read_tally_kernel does.
__global__ void __launch_bounds__(256)
read_responses_kernel(const QuorumDev q, const uint32_t* __restrict__ op_off, const uint32_t* __restrict__ peer_idx, uint8_t* __restrict__ status,
                      const uint8_t* __restrict__ aux, const uint64_t* __restrict__ ts, const uint32_t* __restrict__ voff, const uint32_t* __restrict__ vlen,
                      const uint64_t* __restrict__ plain_ptr, const uint64_t n_ops, uint8_t* __restrict__ out_decision, uint32_t* __restrict__ out_winner,
                      uint32_t* __restrict__ out_decided_at) {
  const int lane = threadIdx.x & 31;
  const uint64_t warp = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t op = warp; op < n_ops; op += nwarps) {
    const uint32_t lo = __ldg(op_off + op), hi = __ldg(op_off + op + 1);
    const uint32_t p = lo + lane;
    const bool have = p < hi;
    const uint32_t k = have ? __ldg(peer_idx + p) : 0xffffffffu;
    uint8_t st = have ? status[p] : (uint8_t)6;
    if (have) {
      const uint8_t a = aux[p];
      if (st == 0 || st == kStUnverifiedSigner) {
        if (a & kAuxNonceCorrupt) st = 3;                         // the base64 error: BFTQ_ST_MALFORMED
        else if (a & kAuxNonceMismatch) st = kStNonceMismatch;    // ErrTransportNonceMismatch
        else if (a & kAuxPacketError) st = 3;                     // packet.Parse failed: processResponse returns the error
      } else if (a & kAuxNonceCorrupt) st = 3;
      status[p] = st;
    }
    const bool ok = have && (st == 0 || st == kStUnverifiedSigner);
    const uint64_t t = ok ? ts[p] : 0ull;
    const uint32_t my_len = ok ? vlen[p] : 0u;
    const uint8_t* my_val = ok ? reinterpret_cast<const uint8_t*>(plain_ptr[p]) + voff[p] : nullptr;
    // value ids: the lowest lane whose value bytes equal this lane's (exact comparison, as Go's map keyed by string(val))
    const uint32_t okmask = __ballot_sync(0xffffffffu, ok);
    uint32_t v = 0xffffffffu;
    uint32_t pending = okmask;
    while (pending) {
      const int rep = __ffs(pending) - 1;
      const uint32_t rlen = __shfl_sync(0xffffffffu, my_len, rep);
      const uint64_t rptr = __shfl_sync(0xffffffffu, (unsigned long long)my_val, rep);
      bool same = ok && v == 0xffffffffu && my_len == rlen;
      if (same && lane != rep) {
        const uint8_t* rv = reinterpret_cast<const uint8_t*>(rptr);
        for (uint32_t i = 0; i < rlen; i++) if (my_val[i] != rv[i]) { same = false; break; }
      }
      if (same) v = (uint32_t)rep;
      pending &= ~__ballot_sync(0xffffffffu, same);
    }
    // ---- the arrival-order decision (see read_tally_kernel)
    const uint32_t upto = 0xffffffffu >> (31 - lane);
    uint64_t pmax = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t other = __shfl_up_sync(0xffffffffu, pmax, o);
      if (lane >= o && other > pmax) pmax = other;
    }
    const uint32_t same_t = __match_any_sync(0xffffffffu, t);
    const uint32_t same_v = __match_any_sync(0xffffffffu, v);
    const uint32_t bucket = same_t & same_v & okmask & upto;
    bool dv = ok && t == pmax && q.nqc > 0, dr = have && !ok;
#pragma unroll
    for (int c = 0; c < kMaxQc; c++) {
      if (c < q.nqc) {
        const uint32_t mm = __ballot_sync(0xffffffffu, have && is_member(q, c, k));
        if (q.threshold[c] > 0 && __popc(bucket & mm) < q.threshold[c]) dv = false;
        const int bad = __popc(mm & ~okmask & upto);
        if (q.f[c] == 0 || bad <= q.f[c]) dr = false;
      }
    }
    const uint32_t dvm = __ballot_sync(0xffffffffu, dv), drm = __ballot_sync(0xffffffffu, dr);
    const uint32_t any = dvm | drm;
    const int d = any ? __ffs(any) - 1 : 0;
    const uint32_t bucket_d = __shfl_sync(0xffffffffu, bucket, d);
    if (lane == 0) {
      uint8_t dec = 2; uint32_t w = 0xffffffffu, at = hi - lo;
      if (any) {
        at = (uint32_t)d + 1;
        if ((dvm >> d) & 1u) { dec = 0; w = (uint32_t)(__ffs(bucket_d) - 1); } else dec = 1;
      }
      out_decision[op] = dec;
      out_decided_at[op] = at;
      out_winner[op] = w;
    }
  }
}

}  // namespace bftq
