/*
 * bftq.h — C ABI of libbftq.so, the H100-native batched Byzantine-quorum verification engine.
 *
 * This is the drop-in boundary for ONE hot path of yahoo/bftkv: the per-response OpenPGP
 * signature check (crypto/pgp), the web-of-trust quorum tally (quorum/wotqs) and the threshold
 * share-combine (crypto/sss, crypto/threshold).  bftkv is pure Go and has no FFI of its own; the
 * entry points below are what a cgo shim behind bftkv's crypto.Signature /
 * crypto.CollectiveSignature / quorum.Quorum interfaces binds (INTEGRATION.md shows the shim).
 * Each entry point cites the reference interface it replaces (file:line relative to the
 * reference tree).
 *
 * Conventions
 *   - plain pointers and sizes only; caller owns every buffer; nothing is retained after return
 *     (cgo pointer rules), except data explicitly registered (keys, quorums).
 *   - every function returns 0 (BFTQ_OK) or a negative BFTQ_ERR_* code; per-item results go to a
 *     caller-provided status array.
 *   - big integers are big-endian byte strings, exactly as Go's big.Int.Bytes()/SetBytes() and
 *     OpenPGP MPIs carry them; fixed-width fields are left-padded with zeros.
 *   - all *_batch functions are thread-safe and re-entrant (bftkv calls Message.Decrypt from one
 *     goroutine per peer, transport/transport.go:110-127).
 *   - there is NO CPU fallback: if no CUDA device is usable, bftq_init fails with
 *     BFTQ_ERR_NO_DEVICE and nothing else can be called.
 */
#ifndef BFTQ_H
#define BFTQ_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BFTQ_VERSION 1

/* ---- error codes --------------------------------------------------------------------------- */
#define BFTQ_OK                     0
#define BFTQ_ERR_NO_DEVICE         -1   /* no CUDA device / driver: the engine cannot exist      */
#define BFTQ_ERR_CUDA              -2   /* a CUDA call failed; bftq_last_error() has the text    */
#define BFTQ_ERR_INVALID_ARG       -3
#define BFTQ_ERR_UNSUPPORTED_KEY   -4   /* modulus size / exponent outside what is built         */
#define BFTQ_ERR_NOMEM             -5
#define BFTQ_ERR_INVALID_SIGNATURE -6   /* crypto.ErrInvalidSignature (crypto/crypto.go)         */
#define BFTQ_ERR_INSUFFICIENT_SIGS -7   /* crypto.ErrInsufficientNumberOfSignatures              */
#define BFTQ_ERR_MALFORMED         -8
#define BFTQ_ERR_NOT_SIGNED        -9   /* crypto.ErrInvalidTransportSecurityData (crypto_pgp.go:458-460)  */
#define BFTQ_ERR_MESSAGE_BODY     -10   /* the literal body ends early / FileName is not base64: Decrypt returns that error as is */
#define BFTQ_ERR_UNSUPPORTED      -11   /* a form the reference's library handles and this build does not (compressed data)       */
#define BFTQ_ERR_MDC             -12   /* the SEIPD packet's modification detection code does not match: ReadAll's error, returned as is */
#define BFTQ_ERR_INVALID_INPUT   -13   /* crypto.ErrInvalidInput (threshold RSA: the hash info leaves less than 3 padding bytes) */
#define BFTQ_ERR_SHARE_NOT_FOUND -14   /* crypto.ErrShareNotFound (threshold DSA: no joint share for this node, or a stale nonce) */
#define BFTQ_ERR_KEY_NOT_FOUND   -15   /* crypto.ErrKeyNotFound (threshold DSA: phase 3 without a phase 2 for the peer) */
#define BFTQ_ERR_AUTH_FAILURE    -16   /* bftkv.ErrAuthenticationFailure (password authentication: Ni does not match) */
#define BFTQ_ERR_NO_AUTH_DATA    -17   /* crypto.ErrNoAuthenticationData (password authentication: no secret for the peer) */
#define BFTQ_ERR_DECRYPTION_FAILED -18 /* crypto.ErrDecryptionFailed (password authentication: Zi does not open) */
#define BFTQ_ERR_INSUFFICIENT_SECRETS -19 /* crypto.ErrInsufficientNumberOfSecrets (GetCipherKey before k secrets) */

/* ---- per-item status bytes (SURVEY §8b "Errors") --------------------------------------------
 * The reference collapses every failure to ErrInvalidSignature (crypto_pgp.go:325-327); the shim
 * maps any non-zero status to that sentinel.  The richer codes exist for statistics only. */
#define BFTQ_ST_OK              0
#define BFTQ_ST_BAD_SIGNATURE   1   /* s^e mod n != EMSA-PKCS1-v1_5(digest)                      */
#define BFTQ_ST_HASH_TAG        2   /* OpenPGP 16-bit hash-tag pre-check failed                  */
#define BFTQ_ST_MALFORMED       3
#define BFTQ_ST_UNKNOWN_SIGNER  4   /* key index out of range / issuer not in keyring            */
#define BFTQ_ST_UNSUPPORTED     5   /* algorithm the reference's library cannot verify either    */
#define BFTQ_ST_MISSING         6   /* no response from this replica (tally input only)          */
#define BFTQ_ST_NOT_BUILT       9   /* a key size / curve / DSA domain the reference's library verifies and this build does not
                                       (RSA > 4096 bit, DSA p other than 1024 / 2048 bit or q > 256 bit, ECDSA P-384 / P-521): the item is
                                       reported as BFTQ_ERR_UNSUPPORTED and the shim re-runs it on crypto/pgp                         */
#define BFTQ_ST_NONCE_MISMATCH  7   /* transport.ErrTransportNonceMismatch (transport.go:121-124)  */
#define BFTQ_ST_UNVERIFIED_SIGNER 8 /* ACCEPTED, as the reference accepts it: the message's signer is not in the keyring, so
                                       openpgp.ReadMessage leaves SignedBy nil and never checks the signature (read path only) */
#define BFTQ_ST_DECRYPT_FAILED 10  /* Decrypt returned crypto.ErrDecryptionFailed (ReadMessage failed: no PKESK key decrypts,
                                      quick check, SEIPD framing, inner-stream framing) or ReadAll's MDC error (encrypted read path only) */

/* ---- hash algorithm ids = OpenPGP ids (RFC 4880 §9.4), as sig.Hash in x/crypto ---------------*/
#define BFTQ_HASH_MD5        1
#define BFTQ_HASH_SHA1       2
#define BFTQ_HASH_RIPEMD160  3
#define BFTQ_HASH_SHA256     8
#define BFTQ_HASH_SHA384     9
#define BFTQ_HASH_SHA512    10
#define BFTQ_HASH_SHA224    11

/* ---- flags --------------------------------------------------------------------------------- */
#define BFTQ_F_STRICT_RANGE  0x1u  /* reject s >= n.  Default (0) matches Go 1.13's
                                      rsa.VerifyPKCS1v15, which computes s^e mod n for any
                                      k-byte s (no range check before Go 1.20).                  */

typedef struct bftq_engine bftq_engine;

/* ---- engine life cycle --------------------------------------------------------------------- */
/* One engine per GPU.  Wired where the reference calls pgp.New() (cmd/bftkv/main.go:66,
 * api/api.go:37).  device = CUDA ordinal. */
int  bftq_init(int device, bftq_engine** out);
void bftq_shutdown(bftq_engine* e);
const char* bftq_last_error(void);          /* thread-local text of the last failure */

/* Page-locked host memory for the shim's C-side blobs (SURVEY §8b "Ownership": "host shim pins/copies into
 * page-locked staging").  Go memory cannot be handed to the DMA engine, so the shim's aggregator appends every
 * request's (tbs, sig) to a blob anyway; when that blob comes from bftq_host_alloc the *_batch calls DMA it in place
 * instead of copying it through the library's own staging first.  The block is allocated on the NUMA node the
 * engine's GPU hangs off.  Pageable buffers remain valid inputs everywhere (they are staged). */
int  bftq_host_alloc(bftq_engine* e, uint64_t bytes, void** out);
int  bftq_host_free(bftq_engine* e, void* p);
/* Binds the CALLING thread to the CPUs of the GPU's NUMA node (the library's own worker threads are bound already).
 * Returns the node number, or -1 when the node is unknown / binding is disabled (BFTQ_NUMA_BIND=0). */
int  bftq_bind_thread(bftq_engine* e);
int  bftq_version(void);
int  bftq_device_sm_count(bftq_engine* e);
/* BFTQ_F_* flags the packet-level entry points (Signature / CollectiveSignature / Message / read path) pass to K1.  Default 0
 * = Go 1.13 (the version go.mod pins): rsa.VerifyPKCS1v15 computes s^e mod n for any k-byte s.  A deployment built with
 * Go >= 1.20 (the reference's Dockerfile is `FROM golang`) rejects s >= n: set BFTQ_F_STRICT_RANGE (or env
 * BFTQ_STRICT_RANGE=1 at bftq_init). */
int  bftq_engine_set_verify_flags(bftq_engine* e, uint32_t flags);

/* ---- key table ------------------------------------------------------------------------------
 * Replaces the keyring lookup inside openpgp.CheckDetachedSignature (EntityList.KeysByIdUsage),
 * reached from crypto/pgp/crypto_pgp.go:324,338,490.  Registers `count` RSA public keys:
 * n_be = count x 256 bytes (big-endian modulus, left-padded), e = count public exponents.
 * Precomputes the per-key Montgomery constants once.  Keys are appended; *first_index receives
 * the index of the first new key (indices are what key_idx[] refers to).  Any odd modulus of up to
 * 4096 bits is accepted; a key of k = ceil(bits/8) bytes (Go's pub.Size()) travels in the smallest
 * size class that holds it — 128, 192, 256, 384 or 512 bytes — and its EM is built for its own k.
 * Exactly-2048-bit moduli (what gpg --quick-gen-key rsa2048 produces) take the radix-2^32 fast path. */
int bftq_register_rsa_keys(bftq_engine* e, const uint8_t* n_be, const uint32_t* exps,
                           uint32_t count, uint32_t* first_index);
/* Same with moduli of up to 512 bytes: n_be = count x stride bytes, each left-padded. */
int bftq_register_rsa_keys_k(bftq_engine* e, const uint8_t* n_be, uint32_t stride, const uint32_t* exps,
                             uint32_t count, uint32_t* first_index);
int bftq_key_count(bftq_engine* e);

/* ---- K1: batched RSA PKCS#1 v1.5 verify ------------------------------------------------------
 * Replaces x/crypto packet.PublicKey.VerifySignature -> rsa.VerifyPKCS1v15 (Go 1.13) as reached
 * from crypto_pgp.go:324 (Signature.Verify), :338 (VerifyWithCertificate), :490
 * (CollectiveSignature.Verify) and :454 (Message.Decrypt's m.SignatureError).
 *   key_idx[i]      index into the key table (>= key count -> BFTQ_ST_UNKNOWN_SIGNER)
 *   sig_be          n_items x 256 bytes, the signature MPI left-padded to the key size
 *                   (what x/crypto's padToKeySize hands to rsa.VerifyPKCS1v15)
 *   digest          n_items x digest_len(hash_alg) bytes, the OpenPGP v4 signature digest
 *   out_status[i]   BFTQ_ST_*
 * Host buffers; the call stages them through pinned memory, runs the kernel and copies the
 * status bytes back before returning. */
int bftq_rsa_verify_batch(bftq_engine* e, const uint32_t* key_idx, const uint8_t* sig_be,
                          const uint8_t* digest, uint32_t hash_alg, uint64_t n_items,
                          uint32_t flags, uint8_t* out_status);

/* Same, but every pointer is a DEVICE pointer and the work is enqueued on `cuda_stream`
 * (a cudaStream_t, may be NULL for the default stream) without synchronising. */
int bftq_rsa_verify_batch_dev(bftq_engine* e, const uint32_t* d_key_idx, const uint8_t* d_sig_be,
                              const uint8_t* d_digest, uint32_t hash_alg, uint64_t n_items,
                              uint32_t flags, uint8_t* d_status, void* cuda_stream);

/* Key-size-class forms: every signature of the batch is stored in key_bytes bytes (128/192/256/384/512),
 * left-padded, and must refer to keys of that class (k <= key_bytes, no smaller class holds k).  A key of
 * another class, or non-zero bytes above the key's own k, give BFTQ_ST_BAD_SIGNATURE, as
 * rsa.VerifyPKCS1v15 rejects len(sig) != k. */
int bftq_rsa_verify_batch_k(bftq_engine* e, uint32_t key_bytes, const uint32_t* key_idx, const uint8_t* sig_be,
                            const uint8_t* digest, uint32_t hash_alg, uint64_t n_items, uint32_t flags,
                            uint8_t* out_status);
int bftq_rsa_verify_batch_dev_k(bftq_engine* e, uint32_t key_bytes, const uint32_t* d_key_idx, const uint8_t* d_sig_be,
                                const uint8_t* d_digest, uint32_t hash_alg, uint64_t n_items, uint32_t flags,
                                uint8_t* d_status, void* cuda_stream);

/* ---- K1b: batched Ed25519 verify (BASELINE config 4) ------------------------------------------
 * NOT a replacement of anything in the reference: golang.org/x/crypto/openpgp @53104e6ec876 has no
 * EdDSA (algorithm 22) and skips such keys.  RFC 8032 pure Ed25519 as GnuPG uses it in OpenPGP: the
 * signed "message" is the 32-byte v4 signature digest.  pubkeys: n_keys x 32 (compressed A),
 * sig: n_items x 64 (R || S), msg: n_items x 32.  out_status: BFTQ_ST_OK / _BAD_SIGNATURE /
 * _UNKNOWN_SIGNER.  Decides as Go's crypto/ed25519 (1.17 and later) and OpenSSL do: rejects S >= L; decodes A as
 * edwards25519.Point.SetBytes does (y >= p is reduced mod p, x = 0 with the sign bit set is accepted, an A with no
 * square root is rejected); hashes the raw 32 key bytes; compares the encoding of [S]B - [k]A with R's bytes; no
 * cofactor.  libsodium is stricter: it also rejects small-order A and R and non-canonical A.
 * Keys are metadata, like the RSA key table: `pubkeys` is HOST memory in both forms (the _dev form takes the bulk arrays
 * key_idx / sig / msg / status in device memory).  Batches run against window tables that the engine caches: one for
 * the base point (5.8 MB) and one per key (1.7 MB each, built on first sight of the 32 key bytes, bounded by
 * BFTQ_ED25519_CACHE_SLOTS = 256 slots); a batch that would bring more than one new key per 32 signatures uses the
 * table-free double-and-add kernel. */
int bftq_ed25519_verify_batch(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, const uint32_t* key_idx,
                              const uint8_t* sig, const uint8_t* msg, uint64_t n_items, uint8_t* out_status);
int bftq_ed25519_verify_batch_dev(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, const uint32_t* d_key_idx,
                                  const uint8_t* d_sig, const uint8_t* d_msg, uint64_t n_items, uint8_t* d_status,
                                  void* cuda_stream);

/* ---- K1c: batched ECDSA P-256 verify -----------------------------------------------------------
 * Replaces the PubKeyAlgoECDSA arm of packet.PublicKey.VerifySignature (x/crypto openpgp/packet/
 * public_key.go, reached from crypto/pgp/pgp.go:593 via CheckDetachedSignature) = Go crypto/ecdsa.Verify:
 * 0 < r, s < N, e = leftmost min(len, 32) digest bytes, (x, y) = (e/s) G + (r/s) Q, valid iff finite and
 * x mod N == r (no low-s rule).  pubkeys: n_keys x 64 (X || Y), r_be / s_be: n_items x 32 (MPIs left-
 * padded), digest: n_items x digest_len (<= 64).  out_status: BFTQ_ST_OK / _BAD_SIGNATURE / _MALFORMED
 * (key not on the curve) / _UNKNOWN_SIGNER (key index out of range). */
int bftq_ecdsa_p256_verify_batch(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, const uint32_t* key_idx,
                                 const uint8_t* r_be, const uint8_t* s_be, const uint8_t* digest, uint32_t digest_len,
                                 uint64_t n_items, uint8_t* out_status);

/* ---- K1d: batched DSA verify (one key per call) -------------------------------------------------
 * Replaces the PubKeyAlgoDSA arm of packet.PublicKey.VerifySignature (digest cut to the subgroup size) =
 * Go crypto/dsa.Verify: 0 < r, s < q, w = s^-1 mod q, v = (g^(z w) y^(r w) mod p) mod q, valid iff v == r;
 * false for every signature when q's bit length is not a multiple of 8.  p_be/g_be/y_be: plen bytes
 * (plen 128 or 256, p odd with exactly 8*plen bits), q_be: qlen <= 32 bytes, q an odd PRIME (the inverse is
 * taken by Fermat).  r_be / s_be: n_items x 32 (MPIs left-padded), digest: n_items x digest_len (<= 64).
 * out_status: BFTQ_ST_OK / _BAD_SIGNATURE.  Other domain sizes: BFTQ_ERR_UNSUPPORTED_KEY. */
int bftq_dsa_verify_batch(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, const uint8_t* g_be,
                          const uint8_t* y_be, const uint8_t* r_be, const uint8_t* s_be, const uint8_t* digest, uint32_t digest_len,
                          uint64_t n_items, uint8_t* out_status);

/* ---- K2: batched wotqs quorum tally ---------------------------------------------------------
 * A quorum descriptor is what wotqs.getQuorumFrom builds (quorum/wotqs/wotqs.go:95-115): a list of
 * quorum cliques qc{nodes,f,min,threshold,suff} (wotqs.go:16-22, values from newQC :36-70).
 * Members are given as KEY-TABLE INDICES (the shim maps node.Id() -> index once per keyring
 * version); member_key_idx[member_off .. member_off+member_cnt) belongs to clique i. */
typedef struct {
  int32_t f, min, threshold, suff;
  uint32_t member_off, member_cnt;
} bftq_qc_t;
typedef struct bftq_quorum bftq_quorum;
int  bftq_quorum_create(bftq_engine* e, const bftq_qc_t* qcs, uint32_t n_qc, const uint32_t* member_key_idx,
                        uint32_t n_members, bftq_quorum** out);
void bftq_quorum_destroy(bftq_engine* e, bftq_quorum* q);

/* Tally bits written per operation */
#define BFTQ_TALLY_IS_QUORUM      0x01  /* wotqs.go:144-155 */
#define BFTQ_TALLY_IS_THRESHOLD   0x02  /* wotqs.go:157-167 */
#define BFTQ_TALLY_IS_SUFFICIENT  0x04  /* wotqs.go:169-176 */
#define BFTQ_TALLY_REJECT         0x08  /* wotqs.go:178-185, evaluated over the FAILED responders */
#define BFTQ_NO_WINNER            0xffffffffu

/* Replaces Quorum.IsQuorum/IsThreshold/IsSufficient/Reject (quorum/quorum.go:18-25) as the
 * multicast callbacks call them after every response (protocol/client.go:74,77,111,113,153).
 * Operation i owns responders [op_off[i], op_off[i+1]); responder p = (key_idx[p], status[p]).
 * status 0 = verified response -> counted in the `nodes` list; any other status -> `failure`
 * list.  Duplicated responders count as often as they occur (wotqs.go:195-206).  Host buffers. */
int bftq_tally_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                     const uint8_t* status, uint64_t n_ops, uint8_t* out_bits);

/* Replaces Client.maxTimestampedValue + isThreshold (protocol/client.go:181-205) over the
 * buckets processResponse builds (:207-230): ts[p] = packet timestamp, value_id[p] = index of
 * the distinct value inside the operation (the packer compares value bytes exactly; < 2^31).
 * out_winner[i] = responder index (0-based inside the op) of the first member of the winning
 * (max t, value) bucket or BFTQ_NO_WINNER (errInProgress); out_bits[i] = IS_THRESHOLD|REJECT.
 * At most 32 responders per operation. */
int bftq_read_tally_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                          const uint8_t* status, const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops,
                          uint32_t* out_winner, uint8_t* out_bits);

/* Client.Read's decision (protocol/client.go:250-268) exactly as the multicast callback reaches it.  The responders of
 * an operation are taken IN THE ORDER GIVEN (= arrival order): a response with status 0 is bucketed by (ts, value_id)
 * (processResponse :207-230) and maxTimestampedValue (:189-205) is asked — only the buckets of the maximum t so far,
 * IsThreshold over the bucket's responders; any other status joins `failure` and q.Reject(failure) is asked.  The
 * first decisive response fixes the result, later ones are collected but decide nothing (ch = nil):
 *   out_decision[i]    BFTQ_READ_VALUE      out_winner[i] = responder index (inside the op) of the first member of
 *                                           the winning bucket: its value / t are Read's result
 *                      BFTQ_READ_REJECTED   majorityError(errs, ErrInsufficientNumberOfValidResponses)
 *                      BFTQ_READ_EXHAUSTED  ErrInsufficientNumberOfResponses (:267)
 *   out_decided_at[i]  number of responses consumed when the decision fell (1-based; the count for EXHAUSTED)
 * At most 32 responders per operation. */
#define BFTQ_READ_VALUE      0
#define BFTQ_READ_REJECTED   1
#define BFTQ_READ_EXHAUSTED  2
int bftq_read_decide_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                           const uint8_t* status, const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops,
                           uint8_t* out_decision, uint32_t* out_winner, uint32_t* out_decided_at);
/* K1 + the read decision in one call: every tuple is verified (pre_status as in bftq_verify_tally_batch), then each
 * operation is decided as bftq_read_decide_batch does.  Host buffers of any size: the operations travel in chunks
 * through a ring of staging slots, copies overlapping the kernels; bftq_host_alloc memory is DMA'd in place. */
int bftq_verify_read_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                           const uint8_t* sig_be, const uint8_t* digest, uint32_t hash_alg, const uint8_t* pre_status,
                           const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops, uint32_t flags,
                           uint8_t* out_status, uint8_t* out_decision, uint32_t* out_winner, uint32_t* out_decided_at);
int bftq_verify_read_batch_dev(bftq_engine* e, const bftq_quorum* q, const uint32_t* d_op_off, const uint32_t* d_key_idx,
                               const uint8_t* d_sig_be, const uint8_t* d_digest, uint32_t hash_alg, const uint8_t* d_pre_status,
                               const uint64_t* d_ts, const uint32_t* d_value_id, uint64_t n_ops, uint64_t n_items, uint32_t flags,
                               uint8_t* d_status, uint8_t* d_bits, uint8_t* d_decision, uint32_t* d_winner, uint32_t* d_decided_at,
                               void* cuda_stream);

/* K1 + K2 in one call (BASELINE configs 3 and 5: "read ops x R-replica quorum, verify + wotqs
 * tally"): verifies all tuples, then tallies per operation on the same stream.  pre_status
 * (nullable) carries per-tuple results decided by the packer (BFTQ_ST_MISSING, _MALFORMED,
 * _HASH_TAG ...): non-zero entries are not verified and keep their status.  ts/value_id nullable:
 * when given, the read tally is produced as in bftq_read_tally_batch, otherwise out_winner is
 * not touched.  Host buffers of any size (chunked and pipelined like bftq_verify_read_batch). */
int bftq_verify_tally_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                            const uint8_t* sig_be, const uint8_t* digest, uint32_t hash_alg, const uint8_t* pre_status,
                            const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops, uint32_t flags,
                            uint8_t* out_status, uint8_t* out_bits, uint32_t* out_winner);
/* Device-pointer form on a caller stream (no synchronisation); n_items = op_off[n_ops]. */
int bftq_verify_tally_batch_dev(bftq_engine* e, const bftq_quorum* q, const uint32_t* d_op_off, const uint32_t* d_key_idx,
                                const uint8_t* d_sig_be, const uint8_t* d_digest, uint32_t hash_alg,
                                const uint8_t* d_pre_status, const uint64_t* d_ts, const uint32_t* d_value_id,
                                uint64_t n_ops, uint64_t n_items, uint32_t flags, uint8_t* d_status, uint8_t* d_bits,
                                uint32_t* d_winner, void* cuda_stream);

/* ---- K3: batched Lagrange share-combine in Z_m ----------------------------------------------
 * Replaces sss.SSSProcess.calculateSecret / sss.Lagrange (crypto/sss/sss.go:81-107) and
 * calculateS (crypto/threshold/dsa/dsa_core.go:389-403):  S = sum_i lambda_i(x) * y_i mod m.
 * m_be: modulus (mlen bytes, big-endian, odd, > 1, <= 256 bytes), shared by the batch;
 * x: n_items x k share abscissae (Coordinate.X); y_be: n_items x k x mlen share values;
 * out_be: n_items x mlen (left-padded; the shim strips zeros where the reference returns
 * big.Int.Bytes()); out_status: 0, or BFTQ_ST_MALFORMED when some (x_j - x_i) is not invertible
 * mod m (the reference panics there). */
int bftq_lagrange_combine_batch(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* x,
                                const uint8_t* y_be, uint64_t n_items, uint8_t* out_be, uint8_t* out_status);
/* Same with DEVICE pointers for x / y / out / status (m_be stays a host pointer), enqueued on `cuda_stream` without
 * synchronising. */
int bftq_lagrange_combine_batch_dev(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* d_x,
                                    const uint8_t* d_y_be, uint64_t n_items, uint8_t* d_out_be, uint8_t* d_status, void* cuda_stream);

/* ---- K5: Lagrange in the exponent (SURVEY §8f rank 4) -------------------------------------------
 * out[i] = base[i]^exp[i] mod m: big.Int.Exp with a shared odd modulus of exactly 1024 or 2048 bits
 * (mlen = 128 / 256); base: n_items x mlen, exp: n_items x elen bytes, all big-endian. */
int bftq_modexp_batch(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, const uint8_t* base_be, const uint8_t* exp_be,
                      uint32_t elen, uint64_t n_items, uint8_t* out_be);
/* Threshold-RSA combine (crypto/threshold/rsa/rsa.go:244-251,318-329 calculateSignature): the product of the
 * k partial signatures at the leaves of a completed signature tree, out[i] = prod_j vals[i][j] mod N, left-padded
 * to len(N) like I2OS (rsa.go:380-393).  N: exactly 1024 or 2048 bits; vals: n_items x k x mlen. */
int bftq_modprod_batch(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const uint8_t* vals_be, uint64_t n_items,
                       uint8_t* out_be);
/* ---- K7: threshold-RSA partial signing (crypto/threshold/rsa/rsa.go) ----------------------------
 * A share is rsaContext's saved parameter: the bytes of ThresholdInstance's secret after its algo byte (TH_RSA only),
 * serializePartialParam's framing (rsa.go:409-485): u16 count, per fragment u32 key index, a sign byte and a u64-length
 * chunk (big-endian magnitude; an empty chunk is the fragment 0), then the N chunk, u32 id, u8 n.  Registration is opt-in:
 * the fragments go to one device allocation per share, zeroed before it is freed (bftq_thrsa_share_destroy,
 * bftq_shutdown); the host copies are wiped after upload and no key material reaches stats or error texts.
 *   BFTQ_ERR_MALFORMED        framing error (truncated share)
 *   BFTQ_ERR_UNSUPPORTED_KEY  N not odd with exactly 2048 bits, or a fragment longer than 8192 bytes (splitKey's depth
 *                             n - k <= 4): the shim keeps such a share on the Go path */
typedef struct bftq_thrsa_share bftq_thrsa_share;
int bftq_thrsa_share_create(bftq_engine* e, const uint8_t* sec, uint64_t len, bftq_thrsa_share** out);
void bftq_thrsa_share_destroy(bftq_thrsa_share* s);
/* rsaContext.Sign (rsa.go:140-178) over n_items (share, serialized sign request) pairs: item i signs request
 * req_blob[req_off[i] .. req_off[i+1]) with shares[share_idx[i]] (share_idx[i] < n_shares).  Output: item i's
 * serializePartialSignature bytes at out_blob[out_off[i] .. out_off[i+1]), packed; u16 count, per distinct index
 * kid * n + id + 1 (uint32 arithmetic) a u32 index and the chunk of the partial signature's minimal big-endian bytes,
 * then the N chunk.  Go writes the entries in map order (random); here they follow the order in which the request
 * first lists their index.  A request listing the same key id twice with a negative fragment yields m^|d| for it, as
 * the reference's in-place Neg does.  out_cap must hold the sum over items of  2 + kids (12 + 256) + 8 + 256  bytes
 * (kids: the request's key-id count), else BFTQ_ERR_INVALID_ARG before any work.
 *   out_err[i]  0 (an item whose request names no key id of the share: length 0, Sign's (nil, nil)) |
 *               BFTQ_ERR_MALFORMED (request framing) | BFTQ_ERR_INVALID_INPUT (emsaEncode's padlen < 3) |
 *               BFTQ_ERR_UNSUPPORTED (m is not invertible mod N: only with a factor of N) */
int bftq_thrsa_sign_batch(bftq_engine* e, bftq_thrsa_share* const* shares, uint32_t n_shares, const uint32_t* share_idx,
                          const uint8_t* req_blob, const uint64_t* req_off, uint64_t n_items, int32_t* out_err, uint8_t* out_blob,
                          uint64_t out_cap, uint64_t* out_off);
/* rsaProc.ProcessResponse (rsa.go:235-338) replayed, statelessly, over each process's responses in arrival order:
 * process p's responses are r = proc_off[p] .. proc_off[p+1]), response r at resp_blob[resp_off[r] .. resp_off[r+1]).
 * n (>= 2) and k are the Threshold's.  Processing stops at the first response that yields a signature or an error, as
 * the DistSign callback does; out_at[p] is its index within the process (the response count when none did).  The
 * first partial signature registered at an index wins; a response's entries register in the order it lists them (Go:
 * map order); N is the completing response's.  Completed products run on the device (K5 modprod, one launch per N).
 *   out_state[p]  BFTQ_THRSA_SIGNED: out_sig[p * 256 ..] = I2OS(s, 256) | BFTQ_THRSA_FAILED: out_err[p] = BFTQ_ERR_MALFORMED
 *                 (a response does not parse) or BFTQ_ERR_UNSUPPORTED_KEY (the completing N is not odd 2048-bit, or a
 *                 partial signature exceeds 512 bytes: the shim combines on big.Int) | BFTQ_THRSA_INCOMPLETE: the
 *                 missingKeys list for the next MakeRequest at out_missing[out_missing_off[p] .. out_missing_off[p+1])
 *                 (empty: MakeRequest returns no request, ErrInsufficientNumberOfThresholdSignatures).
 * missing_cap: capacity of out_missing in entries (BFTQ_ERR_INVALID_ARG when the lists do not fit). */
#define BFTQ_THRSA_INCOMPLETE 0
#define BFTQ_THRSA_SIGNED     1
#define BFTQ_THRSA_FAILED     2
int bftq_thrsa_process_batch(bftq_engine* e, uint32_t n, uint32_t k, const uint8_t* resp_blob, const uint64_t* resp_off,
                             const uint64_t* proc_off, uint64_t n_procs, int32_t* out_state, int32_t* out_err, uint64_t* out_at,
                             uint8_t* out_sig, uint32_t* out_missing, uint64_t missing_cap, uint64_t* out_missing_off);
/* ---- K8: threshold DSA / ECDSA partial signing (crypto/threshold/dsa/dsa_core.go:91-163 dsaContext.Sign) ------------
 * A share is dsaContext's saved parameter: the bytes of ThresholdInstance's secret after its algo byte, whose value
 * (crypto.TH_DSA = 2, TH_ECDSA = 3) is `algo`.  serializePartialParam's framing: the group (DSA: chunks p, q, g; ECDSA:
 * chunks P, N, B, Gx, Gy and a u32 BitSize), then u64 X, the chunk Y, u16 t and the nodes' OpenPGP entity stream.
 * Registration is opt-in: Y goes to one device allocation per share, zeroed before it is freed (bftq_thdsa_share_destroy,
 * bftq_shutdown), and the host copy is wiped after upload.  The entity stream is read leniently (it serves phase 1 only):
 * a stream Go's ParseStream rejects does not fail registration here.
 *   BFTQ_ERR_MALFORMED        framing error (truncated share)
 *   BFTQ_ERR_UNSUPPORTED_KEY  DSA without p odd of exactly 1024 / 2048 bits and q odd of 33..256 bits, or an ECDSA group
 *                             that is not exactly P-256 (P, N, B, Gx, Gy, BitSize 256): the shim keeps such a share on Go */
#define BFTQ_THDSA_DSA   2
#define BFTQ_THDSA_ECDSA 3
typedef struct bftq_thdsa_share bftq_thdsa_share;
typedef struct bftq_keyring bftq_keyring;          /* the packet-level keyring, below */
int bftq_thdsa_share_create(bftq_engine* e, uint32_t algo, const uint8_t* sec, uint64_t len, bftq_thdsa_share** out);
void bftq_thdsa_share_destroy(bftq_thdsa_share* s);
/* The most bytes one item signed with this share can write: 8 + (8 + |p| or 65) + (8 + 32) + the group's serialized length. */
uint64_t bftq_thdsa_share_out_bound(const bftq_thdsa_share* s);
/* dsaContext.Sign's phases 2 and 3 over n_items requests.  Item i: request req_blob[req_off[i] .. req_off[i+1]) for share
 * shares[share_idx[i]] from client peer_id[i]; self_id is this server's node id.  has_nonce[i] / nonce_blob[nonce_off[i] ..
 * nonce_off[i+1]): the nonce phase 1 (on Go) stored for peer_id[i], ctx.nonces[peerId].  The items behave as if they ran one
 * after another in item order: a phase-3 item uses the (k_i, c_i) of the latest earlier phase-2 item for the same (share,
 * peer), in this call or an earlier one; the share's table of them grows as Go's map does and is never evicted.  Every
 * encrypted share of every phase-2 item is decrypted in ONE bftq_message_decrypt_batch on `kr`, which holds this server's
 * private key and the nodes' certificates.
 * Output: item i's serializePartialSignature bytes at out_blob[out_off[i] .. out_off[i+1]), packed.  Phase 2: u64 x,
 * chunk(R_i), chunk(v_i), the group; phase 3: u64 X, chunk(s_i), an empty chunk, the group.  R_i: DSA g^{a_i} mod p minimal
 * (01 for a_i = 0), ECDSA elliptic.Marshal(a_i G) (04 || 0^64 for a_i = 0).  out_cap must hold the sum over items of
 * bftq_thdsa_share_out_bound(their share), else BFTQ_ERR_INVALID_ARG before any work.
 *   out_err[i]  0 | BFTQ_ERR_MALFORMED (request framing; a share message's framing; a share whose signer key id is not the
 *               primary key id of an entity in the keyring, where GetCertById returns nil and Go panics on signer.Id(); or,
 *               as bftq_message_decrypt_batch reports it, a share message ReadMessage cannot read, which Go returns as
 *               crypto.ErrDecryptionFailed: the code does not tell these apart) | BFTQ_ERR_SHARE_NOT_FOUND (no entry for self_id,
 *               no self-signed share, or its nonce differs from / lacks the stored one) | BFTQ_ERR_INVALID_INPUT (the four
 *               X of a share differ from the first share's X, or the entry for self_id holds no share) |
 *               BFTQ_ERR_KEY_NOT_FOUND (phase 3 without a phase 2) | a code of bftq_message_decrypt_batch for the first share
 *               that fails, as Message.Decrypt returns it; BFTQ_ERR_UNSUPPORTED there means: run this Sign on Go, and route
 *               the (share, peer)'s phase 3 to Go too.  A failed item stores nothing. */
int bftq_thdsa_sign_batch(bftq_keyring* kr, bftq_thdsa_share* const* shares, uint32_t n_shares, const uint32_t* share_idx,
                          const uint8_t* req_blob, const uint64_t* req_off, const uint64_t* peer_id, uint64_t self_id,
                          const uint8_t* nonce_blob, const uint64_t* nonce_off, const uint8_t* has_nonce, uint64_t n_items,
                          int32_t* out_err, uint8_t* out_blob, uint64_t out_cap, uint64_t* out_off);
/* ---- K8, client half: dsaProc (crypto/threshold/dsa/dsa_core.go:269-403) -----------------------------------------------
 * bftq_thdsa_proc_create is dsaContext.NewProcess: algo = BFTQ_THDSA_DSA / _ECDSA, dgst = hash(tbs) as Go computes it, t and
 * node_ids the context's (ctx.t, ctx.nodes: what the first MakeRequest returns).  2t > 255 is BFTQ_ERR_UNSUPPORTED_KEY.  A
 * process holds public state only (the digest, t, the node list, the kmap, the partial signatures, m, r, the phase and the
 * result), in host memory: no key material, no device allocation, no engine.  One process must not be used by two calls at
 * once, as Go's dsaProc. */
typedef struct bftq_thdsa_proc bftq_thdsa_proc;
int  bftq_thdsa_proc_create(uint32_t algo, const uint8_t* dgst, uint64_t dgst_len, uint32_t t, const uint64_t* node_ids, uint32_t n_nodes,
                            bftq_thdsa_proc** out);
void bftq_thdsa_proc_destroy(bftq_thdsa_proc* p);

#define BFTQ_THDSA_REQUEST   (-1)   /* MakeRequest                      */
#define BFTQ_THDSA_RESPONSE  0      /* ProcessResponse(data, peer_id)   */
#define BFTQ_THDSA_PENDING   0      /* out_state: (nil, nil)            */
#define BFTQ_THDSA_CONTINUE  1      /*            crypto.ErrContinue    */
#define BFTQ_THDSA_SIGNED    2      /*            the r || s result     */
#define BFTQ_THDSA_FAILED    3      /*            out_err[i]            */
/* The calls a Go client makes one at a time, batched: item i applies op[i] to procs[proc_idx[i]], a RESPONSE with the answer
 * data_blob[data_off[i] .. data_off[i+1]) of peer_id[i].  The result equals the same calls made one after another in item
 * order; items of different processes are independent.  Item i's output is at out_blob[out_off[i] .. out_off[i+1]).
 *   REQUEST   u32 count | count x u64 node id (the node list, which then resets), then the request: phase 1
 *             serializeSignRequest(nil, nil, kmap) with the ids in first-insertion order (one legal order of Go's map), phase 2
 *             01 || chunk(m) || chunk(r), else nothing (Go's nil).
 *   RESPONSE  out_state; SIGNED writes formatDSA(r, s, q).  The peer joins the node list before any parsing.
 *             phase 0  parseJointShare; the phase advances when the count of the last-listed id reaches 2t.
 *             phase 1  the 2t-th partial signature runs CalculateR and OS2I with its own group (DSA OS2I: dgst[:|q| bytes]).
 *             phase 2  the 2t-th runs calculateS mod its own q, then formatDSA; every later RESPONSE returns the same result.
 *             x is Go's int(u64); equal abscissae are skipped in the Lagrange coefficients.  v.ModInverse(v, q) is Go's:
 *             v^-1 when gcd(v, q) = 1, else v itself (DSA r = 1 for v = 0); ECDSA r = 0 for v = 0 or a sum at infinity.
 *   out_err[i]  0 | BFTQ_ERR_MALFORMED (framing: the item changes the node list only; or where Go panics: an R_i that
 *               elliptic.Unmarshal rejects, a Lagrange denominator with no inverse mod q, a digest shorter than the order, an r
 *               longer than the phase-2 q) | BFTQ_ERR_UNSUPPORTED_KEY (an x outside int32, or a completing answer whose group
 *               is neither DSA with p odd of exactly 1024 / 2048 bits and q odd, 1 < q < 2^256, nor exactly P-256: the item
 *               changes nothing, and the shim replays the process on Go).  A completion that fails leaves the process failed:
 *               it and every later item of the process return the same code.
 * *out_need (bytes the outputs may take, from public sizes) is set on every return; out_cap below it is BFTQ_ERR_INVALID_ARG
 * before any work, with nothing changed, as are a bad index or op.  A BFTQ_ERR_CUDA / BFTQ_ERR_NOMEM return can leave the
 * call's processes advanced past what any output shows: destroy them. */
int bftq_thdsa_process_batch(bftq_engine* e, bftq_thdsa_proc* const* procs, uint32_t n_procs, const uint32_t* proc_idx,
                             const int32_t* op, const uint64_t* peer_id, const uint8_t* data_blob, const uint64_t* data_off,
                             uint64_t n_items, int32_t* out_state, int32_t* out_err, uint8_t* out_blob, uint64_t out_cap,
                             uint64_t* out_off, uint64_t* out_need);
/* AuthClient.calculateSharedSecret (crypto/auth/auth.go:386-399) and the first half of CalculateR:
 * out[i] = prod_j y[i][j]^lambda_j mod p,  lambda_j = sss.Lagrange(x[i][j], x[i][*], q).
 * p: plen = 128/256 bytes; q: any odd modulus up to 256 bytes (auth uses q = (p-1)/2). */
int bftq_lagrange_exp_product_batch(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen,
                                    uint32_t k, const int32_t* x, const uint8_t* y_be, uint64_t n_items, uint8_t* out_be,
                                    uint8_t* out_status);
/* dsaGroupOperations.CalculateR (crypto/threshold/dsa/dsa.go:33-52):
 * r = (prod R_i^lambda_i mod p)^((sum v_i lambda_i)^-1 mod q) mod p mod q, per item over its k
 * partial results (x_i, R_i, v_i); q prime, <= 256 bits.  out_r_be: n_items x qlen (left-padded, as
 * formatDSA lays r out, dsa_core.go:375-387). */
int bftq_dsa_calculate_r_batch(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, uint32_t k,
                               const int32_t* x, const uint8_t* ri_be, const uint8_t* vi_be, uint64_t n_items,
                               uint8_t* out_r_be, uint8_t* out_status);

/* ecdsaGroupOperations.CalculateR on P-256 (crypto/threshold/ecdsa/ecdsa.go:36-59):
 * R = (sum_i lambda_i * R_i) * v^-1 with v = sum_i v_i lambda_i mod N, r = R.x mod N.
 * ri: n_items x k x 65 bytes (elliptic.Marshal: 04 || X || Y), vi: n_items x k x 32, out_r: n_items x 32. */
int bftq_ecdsa_p256_calculate_r_batch(bftq_engine* e, uint32_t k, const int32_t* x, const uint8_t* ri, const uint8_t* vi_be,
                                      uint64_t n_items, uint8_t* out_r_be, uint8_t* out_status);

/* ---- K4: batched OpenPGP v4 signature digest --------------------------------------------------
 * Replaces hashForSignature + the hash-suffix step of packet.PublicKey.VerifySignature
 * (x/crypto, reached from crypto_pgp.go:324,338,490): digest_i = H(data[data_idx[i]] || suffix_i).
 * data blobs are the TBS/TBSS byte strings (packet/packet.go:156-190), shared by all signatures of
 * one collective signature; suffix_i = sigpacket[0 : 6+hashedLen] || 04 FF || be32(6+hashedLen).
 * data_off has n_data+1 entries, suffix_off n_items+1; data_idx may be NULL (identity).
 * hash_alg: SHA-256 (what bftkv's own signer emits, crypto_pgp.go:353 with nil config), SHA-1,
 * SHA-224, SHA-384 or SHA-512 (what foreign gpg keys may carry); MD5 / RIPEMD-160 are not built.
 * out_digest: n_items x digest_len(hash_alg). */
int bftq_pgp_digest_batch(bftq_engine* e, const uint8_t* data_blob, const uint64_t* data_off, uint32_t n_data,
                          const uint32_t* data_idx, const uint8_t* suffix_blob, const uint64_t* suffix_off,
                          uint32_t hash_alg, uint64_t n_items, uint8_t* out_digest);

/* ---- host packer: the reference-facing operator interface -----------------------------------
 * These entry points take exactly what bftkv passes to crypto.Signature /
 * crypto.CollectiveSignature — the signed bytes and SignaturePacket.Data (raw concatenated OpenPGP
 * signature packets, packet/packet.go:25-31) — parse them on the host, run digest + tag check +
 * RSA verify (+ tally) on the GPU in one stream, and fold the per-tuple results back into the
 * reference's decisions.  Blobs are concatenations with (count+1) offsets.
 *
 * Keyring: mirrors crypto/pgp PGPKeyring (crypto_pgp.go:115-223).  Entities are parsed from
 * serialized OpenPGP public-key blocks (what PGPCertificate.Parse/ParseStream consume, :225-251);
 * priv != 0 registers into the secring, which getKeyring() searches first (:195-197).  An entity
 * whose primary key id is already present is replaced (replace(), :124-140).  RSA keys of
 * 2041..2048 bits are also entered in the engine's key table. */
typedef struct bftq_keyring bftq_keyring;
int  bftq_keyring_create(bftq_engine* e, bftq_keyring** out);
void bftq_keyring_destroy(bftq_keyring* kr);
int  bftq_keyring_add(bftq_keyring* kr, const uint8_t* key_blocks, uint64_t len, int priv, uint32_t* n_entities);
int  bftq_keyring_remove(bftq_keyring* kr, const uint64_t* key_ids, uint32_t n);      /* PGPKeyring.Remove :160-177 */
/* node.Id() of every entity, secring first then keyring (getKeyring order); *n = count. */
int  bftq_keyring_ids(bftq_keyring* kr, uint64_t* out_ids, uint32_t cap, uint32_t* n);
/* PGPCertificateInstance.Signers (crypto_pgp.go:80-88): issuer ids of the third-party
 * certifications on entity `key_id` (the trust-graph edges node/graph/graph.go:61-71 reads). */
int  bftq_keyring_certifiers(bftq_keyring* kr, uint64_t key_id, uint64_t* out_ids, uint32_t cap, uint32_t* n);

/* PGPSignature.Verify (crypto_pgp.go:319-330), batched over n_items independent (tbs, sig.Data)
 * pairs: out_err[i] = 0 (nil), BFTQ_ERR_INVALID_SIGNATURE, or BFTQ_ERR_UNSUPPORTED when the item fails while one of its
 * packets uses an algorithm / key size the reference's library verifies and this build does not (RSA > 4096 bit,
 * DSA beyond 1024/2048-bit p or 256-bit q, ECDSA P-384 / P-521, RIPEMD-160): the shim re-runs exactly those items on
 * crypto/pgp (bftq_stats counts them in unsupported_items).  Every signature packet of the
 * stream must verify, empty data is invalid, unknown issuers are skipped unless they end the
 * stream — exactly the reference's loop over openpgp.CheckDetachedSignature. */
int bftq_signature_verify_batch(bftq_keyring* kr, const uint8_t* tbs_blob, const uint64_t* tbs_off,
                                const uint8_t* sig_blob, const uint64_t* sig_off, uint64_t n_items, int32_t* out_err);
/* PGPSignature.VerifyWithCertificate (crypto_pgp.go:332-344): the keyring of item i is the FIRST
 * entity of cert i (Issuer(), :396-405); items with no parseable entity are invalid. */
int bftq_signature_verify_with_cert_batch(bftq_keyring* kr, const uint8_t* tbs_blob, const uint64_t* tbs_off,
                                          const uint8_t* sig_blob, const uint64_t* sig_off, const uint8_t* cert_blob,
                                          const uint64_t* cert_off, uint64_t n_items, int32_t* out_err);
/* Diagnostic: runs ONLY the host half of bftq_signature_verify_batch (packet parsing, keyring lookup,
 * tuple composition; `threads` = 0 picks the library default, BFTQ_HOST_THREADS) and reports the number
 * of (signature, candidate key) tuples it would send to the GPU and the wall time.  No verification
 * happens and no result is produced; works on a parse-only keyring.  Used to size the host side of the
 * path against the kernels (bench.py `packer`). */
int bftq_signature_plan_measure(bftq_keyring* kr, const uint8_t* tbs_blob, const uint64_t* tbs_off, const uint8_t* sig_blob,
                                const uint64_t* sig_off, uint64_t n_items, uint32_t threads, uint64_t* n_tuples, double* seconds);

/* PGPSignature.Signers (crypto_pgp.go:373-390) for one SignaturePacket.Data: key ids of the
 * issuers present in the keyring (primary ids via getCertById), duplicates kept, in packet order. */
int bftq_signature_signers(bftq_keyring* kr, const uint8_t* sig, uint64_t sig_len, uint64_t* out_ids, uint32_t cap, uint32_t* n);

/* PGPMessage.Decrypt's signature half (crypto_pgp.go:453-471; the per-response check of every multicast,
 * transport/transport.go:116-126), batched.  Item i is the packet stream the message's SymmetricallyEncrypted packet
 * decrypts to — [compressed] one-pass signature, literal data, signature — the host keeps the private-key operation and
 * the AES-CFB / MDC layer.  openpgp.ReadMessage's readSignedMessage + signatureCheckReader are restated packet for
 * packet (old / new framing, partial-length literal bodies as Go's own writer emits them, v3 and v4 signatures, text
 * mode): the literal body is hashed with the ONE-PASS packet's algorithm and signature type, the packet behind it is
 * verified with the FIRST key KeysByIdUsage(one-pass key id, sign) yields, and a message whose signer is not in the
 * keyring is NOT an error (m.SignedBy == nil: SignatureError stays nil, the reference returns peer = nil).
 *   out_err[i]        0 | BFTQ_ERR_INVALID_SIGNATURE (m.SignatureError != nil) | BFTQ_ERR_MALFORMED (ReadMessage failed:
 *                     crypto.ErrDecryptionFailed) | BFTQ_ERR_NOT_SIGNED | BFTQ_ERR_MESSAGE_BODY | BFTQ_ERR_UNSUPPORTED,
 *                     in the precedence Decrypt applies them
 *   out_signed_by[i]  m.SignedByKeyId (the shim maps it with GetCertById: the peer may be nil)
 *   out_flags[i]      BFTQ_MSG_SIGNER_KNOWN (m.SignedBy != nil) | BFTQ_MSG_BINARY (literal format 'b')
 *   out_plain_blob    (nullable) item i's plain text — the de-chunked literal body — at out_plain_blob + msg_off[i],
 *                     out_plain_len[i] bytes: the blob needs msg_off[n_items] bytes, a plain text is never longer than its
 *                     message
 *   out_nonce_blob    (nullable) base64-decoded FileName likewise at out_nonce_blob + msg_off[i], out_nonce_len[i] bytes */
#define BFTQ_MSG_SIGNER_KNOWN 0x01
#define BFTQ_MSG_BINARY       0x02
int bftq_message_verify_batch(bftq_keyring* kr, const uint8_t* msg_blob, const uint64_t* msg_off, uint64_t n_items, int32_t* out_err,
                              uint64_t* out_signed_by, uint8_t* out_flags, uint8_t* out_plain_blob, uint32_t* out_plain_len,
                              uint8_t* out_nonce_blob, uint32_t* out_nonce_len);

/* ---- the encryption layer (K6): opt-in private keys on the device --------------------------------------------------
 * Registers the private halves of RSA keys for decryption: a stream of OpenPGP secret-key packets (tag 5 / 7, v4, S2K usage
 * 0), as gpg --export-secret-keys writes them for an unprotected key, or as x/crypto's packet.PrivateKey.Serialize writes the
 * entity's primary key and each subkey.  Keys are matched by key id (fingerprint of the public part); an entity registered
 * with bftq_keyring_add(priv = 1) uses them.  Nothing secret reaches the device unless it is registered here.  Each key is
 * checked (2-byte checksum, p q == n, n of exactly 2048 bits with 1024-bit p and q) and must pass one encrypt / decrypt round
 * trip on the device.  Keys that fail are not registered: BFTQ_ERR_UNSUPPORTED_KEY (protected, not RSA, other sizes,
 * inconsistent) or BFTQ_ERR_MALFORMED (framing, checksum) is returned after the other keys of the stream were processed;
 * *n_keys = keys registered.  The private halves live in one device allocation per keyring, zeroed before it is freed
 * (bftq_keyring_remove of the owning entity, bftq_keyring_destroy); host copies are wiped after upload. */
int bftq_keyring_add_private(bftq_keyring* kr, const uint8_t* packets, uint64_t len, uint32_t* n_keys);

/* The whole of PGPMessage.Decrypt (crypto_pgp.go:453-471) on raw transport messages: openpgp.ReadMessage's PKESK loop
 * (each PKESK in order, KeysById over secring ++ keyring, keys without a private half skipped), the RSA-CRT session-key
 * recovery (K6a), the quick check of each candidate in order and the AES-CFB / SHA-1 MDC layer (K6b), then the signature
 * half of bftq_message_verify_batch on the decrypted packet stream.  Outputs as bftq_message_verify_batch, at raw_off.
 *   out_err[i]  0 | BFTQ_ERR_INVALID_SIGNATURE | BFTQ_ERR_MALFORMED (ReadMessage failed: no key decrypts, bad framing, unknown
 *               cipher, wrong key length, a session-key message shorter than 3 bytes — where the reference panics) |
 *               BFTQ_ERR_NOT_SIGNED (also: the message is not encrypted) | BFTQ_ERR_MESSAGE_BODY | BFTQ_ERR_MDC |
 *               BFTQ_ERR_UNSUPPORTED: the shim re-runs the item on crypto/pgp — compressed inner streams, CAST5 / 3DES,
 *               tag 9 without MDC, tag 3, ElGamal PKESKs, wildcard key id 0, a secring key without a registered private half,
 *               several private candidates for one PKESK, packets behind the encrypted packet. */
int bftq_message_decrypt_batch(bftq_keyring* kr, const uint8_t* raw_blob, const uint64_t* raw_off, uint64_t n_items, int32_t* out_err,
                               uint64_t* out_signed_by, uint8_t* out_flags, uint8_t* out_plain_blob, uint32_t* out_plain_len,
                               uint8_t* out_nonce_blob, uint32_t* out_nonce_len);

/* Batching aggregator: bftkv calls Signature.Verify one (tbs, sig) at a time from many goroutines
 * (one per peer in transport.Multicast, transport/transport.go:110-127; one per HTTP request on the
 * servers).  bftq_aggregator_verify blocks its caller until the batch it was coalesced into has been
 * verified: a batch is flushed when it reaches max_batch items or max_wait_us after its first item.
 * This is where "tens of thousands of tuples" come from without touching bftkv's call sites.
 * cert == NULL selects Verify; a non-NULL cert selects VerifyWithCertificate with that key block — also when cert_len is 0
 * (an empty certificate fails, it never falls back to the shared keyring).
 * Returns 0 (valid), BFTQ_ERR_INVALID_SIGNATURE, or a BFTQ_ERR_* infrastructure error. */
typedef struct bftq_aggregator bftq_aggregator;
int  bftq_aggregator_create(bftq_keyring* kr, uint32_t max_batch, uint32_t max_wait_us, bftq_aggregator** out);
void bftq_aggregator_destroy(bftq_aggregator* a);
int  bftq_aggregator_verify(bftq_aggregator* a, const uint8_t* tbs, uint64_t tbs_len, const uint8_t* sig, uint64_t sig_len,
                            const uint8_t* cert, uint64_t cert_len);
/* batches flushed / items verified since creation */
int  bftq_aggregator_stats(bftq_aggregator* a, uint64_t* n_batches, uint64_t* n_items);

/* Parse-only inspection of one SignaturePacket.Data stream against the keyring (host only, no GPU):
 * how the reference's loop over openpgp.CheckDetachedSignature would walk it.  collective = 0:
 * Signature.Verify's strict walk (stops at the first structural error / unknown-issuer tail, *failed = 1);
 * collective != 0: CollectiveSignature.Verify's tolerant walk.  Writes, per call that reached a
 * known-issuer signature packet, the issuer key id and the OpenPGP hash id (up to cap entries). */
int bftq_signature_parse(bftq_keyring* kr, const uint8_t* sig, uint64_t sig_len, int collective, uint64_t* out_issuers,
                         uint8_t* out_hash_ids, uint32_t cap, uint32_t* n_calls, int32_t* failed);

/* Quorum descriptor by node id, for the collective-signature calls (members are node.Id()s). */
typedef struct {
  int32_t f, min, threshold, suff;
  uint32_t member_off, member_cnt;      /* into member_ids[] */
} bftq_qc_ids_t;
/* PGPCollectiveSignature.Verify (crypto_pgp.go:485-500), batched: valid packets append their
 * signer (no dedupe), invalid / unknown ones are ignored, success as soon as q.IsSufficient
 * (monotone, so the decision equals IsSufficient over all valid signers).  out_err[i] = 0,
 * BFTQ_ERR_INSUFFICIENT_SIGS, or BFTQ_ERR_UNSUPPORTED (insufficient while a packet could not be judged here, see
 * bftq_signature_verify_batch); on success the shim sets ss.Completed = true (:494).  The tally runs
 * on the GPU (K2) over the verified signers. */
int bftq_collective_verify_batch(bftq_keyring* kr, const bftq_qc_ids_t* qcs, uint32_t n_qc, const uint64_t* member_ids,
                                 uint32_t n_members, const uint8_t* tbs_blob, const uint64_t* tbs_off,
                                 const uint8_t* ss_blob, const uint64_t* ss_off, uint64_t n_items, int32_t* out_err);
/* PGPCollectiveSignature.Combine's decision (crypto_pgp.go:506-515) for ss.Data ++ s.Data already
 * concatenated by the shim: q.IsSufficient(Signers(ss)) — packet parse only, no crypto. *out = 0/1. */
int bftq_collective_combine_sufficient(bftq_keyring* kr, const bftq_qc_ids_t* qcs, uint32_t n_qc, const uint64_t* member_ids,
                                       uint32_t n_members, const uint8_t* ss, uint64_t ss_len, int32_t* out);

/* The read path from raw answers: what Client.Read (protocol/client.go:250-268) does with the R answers of each of n_ops
 * read operations, once the host has removed the encryption layer of every answer — packets in, decisions out.
 * Response p (operation i owns [op_off[i], op_off[i+1]), in ARRIVAL order, at most 32) is
 *   peer_ids[p]     the node the request went to (res.Peer: what the quorum predicates count; the message's signer is NOT
 *                   compared with it — transport.Multicast ignores Decrypt's peer, transport/transport.go:119)
 *   msg p           the packet stream its answer decrypts to (as bftq_message_verify_batch takes it)
 *   pre_status[p]   (nullable) non-zero: the transport failed earlier (no answer, HTTP error, decryption failed) — a failure
 *   nonce p         nonce_len bytes at nonce_blob + p * nonce_len: the nonce the request carried (transport.go:103,121)
 * Per response: Message.Decrypt's signature half, then the nonce comparison, then packet.Parse of a non-empty answer
 * (client.go:207-230; an empty answer buckets as ("", 0)); per operation: the arrival-order decision of
 * bftq_read_decide_batch, values compared byte for byte.  K0m parses, de-chunks, hashes and lays out K1's inputs on the
 * GPU for the shape every bftkv answer has; anything else goes through the host packer and is patched in.
 *   out_status[p]     BFTQ_ST_OK / BFTQ_ST_UNVERIFIED_SIGNER (both count as good answers) or the failure kind
 *   out_ts / out_value_off / out_value_len (nullable)  timestamp and value span inside the answer's plain text
 *   out_decision / out_winner / out_decided_at          as bftq_read_decide_batch */
int bftq_read_responses_batch(bftq_keyring* kr, const bftq_qc_ids_t* qcs, uint32_t n_qc, const uint64_t* member_ids, uint32_t n_members,
                              const uint32_t* op_off, uint64_t n_ops, const uint64_t* peer_ids, const uint8_t* msg_blob, const uint64_t* msg_off,
                              const uint8_t* pre_status, const uint8_t* nonce_blob, uint32_t nonce_len, uint8_t* out_status, uint64_t* out_ts,
                              uint32_t* out_value_off, uint32_t* out_value_len, uint8_t* out_decision, uint32_t* out_winner, uint32_t* out_decided_at);

/* The read path from the raw wire answers: bftq_read_responses_batch with PGPMessage.Decrypt's encryption layer in front.
 * Arguments, limits and argument errors are those of bftq_read_responses_batch; response p is the raw answer as
 * transport.Multicast receives it (PKESK(s) + SEIPD, what Message.Encrypt writes), at raw_blob + raw_off[p].  The client's
 * private key must have been registered with bftq_keyring_add_private.  The status of an answer follows the code
 * bftq_message_decrypt_batch returns for the same bytes: pre_status non-zero is kept; 0 -> OK / UNVERIFIED_SIGNER, then
 * NONCE_MISMATCH, then MALFORMED when packet.Parse fails (as bftq_read_responses_batch); BFTQ_ERR_INVALID_SIGNATURE ->
 * BAD_SIGNATURE or HASH_TAG; BFTQ_ERR_MALFORMED, BFTQ_ERR_MDC -> BFTQ_ST_DECRYPT_FAILED; BFTQ_ERR_NOT_SIGNED,
 * BFTQ_ERR_MESSAGE_BODY -> MALFORMED (so a signed but unencrypted answer fails here); BFTQ_ERR_UNSUPPORTED -> UNSUPPORTED.
 * On the device (K6p parse -> K6a RSA-CRT -> K6b AES-CFB / MDC -> K0m -> K1 -> K2m) for the shape every bftkv answer has:
 * one PKESK v3 to a key with exactly one registered private half, one SEIPD v1 to the end of the message.  Every other
 * answer, and every one whose MDC does not match, runs whole through bftq_message_decrypt_batch and is patched in.
 *   out_plain_blob / out_plain_len (nullable pair)  each good answer's plain text (what Decrypt returns) at
 *                     out_plain_blob + raw_off[p], out_plain_len[p] bytes (0 for the other answers, whose span is zeroed);
 *                     out_value_off is relative to it.
 * Decrypted plain text left in the library's device scratch is not scrubbed (as bftq_message_decrypt_batch); session keys
 * live in a per-call allocation zeroed before the call returns. */
int bftq_read_encrypted_responses_batch(bftq_keyring* kr, const bftq_qc_ids_t* qcs, uint32_t n_qc, const uint64_t* member_ids, uint32_t n_members,
                                        const uint32_t* op_off, uint64_t n_ops, const uint64_t* peer_ids, const uint8_t* raw_blob, const uint64_t* raw_off,
                                        const uint8_t* pre_status, const uint8_t* nonce_blob, uint32_t nonce_len,
                                        uint8_t* out_status, uint64_t* out_ts, uint32_t* out_value_off, uint32_t* out_value_len,
                                        uint8_t* out_plain_blob, uint32_t* out_plain_len,
                                        uint8_t* out_decision, uint32_t* out_winner, uint32_t* out_decided_at);

/* ---- threshold password authentication, server half (crypto/auth/auth.go:168-237, K9) ---------------------------
 * bftq_auth_server_create is NewServer(params, proof): params as serializeParams writes them (int32 x, then chunks y, v
 * and salt, each a u64 big-endian length and its bytes).  y, v, the salt's HMAC key block and the proof go to one device
 * allocation per server, zeroed before it is freed (bftq_auth_server_destroy, bftq_shutdown); the host copies of y and v
 * are wiped.  Returns
 *   BFTQ_ERR_MALFORMED        truncated framing
 *   BFTQ_ERR_UNSUPPORTED_KEY  y or v longer than 256 bytes (setAuth stores params unverified: keep that session on Go)
 * No secret reaches an error text or the statistics. */
typedef struct bftq_auth_server bftq_auth_server;
int bftq_auth_server_create(bftq_engine* e, const uint8_t* params, uint64_t params_len, const uint8_t* proof, uint64_t proof_len,
                            bftq_auth_server** out);
void bftq_auth_server_destroy(bftq_auth_server* s);
/* The largest answer of one item: phase 0: 4 + 8 + 256 + 8 + |salt|; phase 1: 8 + 256; phase 2: 8 + |proof| + 16 + 8 + 12;
 * any other phase: 0. */
uint64_t bftq_auth_server_out_bound(const bftq_auth_server* s, int32_t phase);
/* One scheduling tick of MakeResponse(phase[i], req[i]) on handles[handle_idx[i]], phases mixed.  req: the adata as
 * received (X, Xi or Ni); rand: the randomness Go drew (phase 1: b, exactly 256 big-endian bytes; phase 2: the 12-byte
 * GCM nonce; ignored otherwise).  A wrong rand length, a server listed twice, or out_cap below the sum of
 * bftq_auth_server_out_bound(server, phase) over the items is BFTQ_ERR_INVALID_ARG before any work.
 *   phase 0  out = int32 x | chunk(Yi.Bytes()) | chunk(salt), Yi = X^y mod p
 *   phase 1  out = chunk(Bi.Bytes()), Bi = v^b mod p; stores keySched(Ki.Bytes(), salt)'s ke and the MAC
 *            HMAC-SHA256(km, Xi || Bi.Bytes()) on the device (Ki = Xi^b mod p); a repeated phase 1 overwrites them
 *   phase 2  out = chunk(AES-128-GCM(ke).Seal(nonce, proof, mac) || tag) | chunk(nonce) when Ni equals the MAC (constant
 *            time), else out_err[i] = BFTQ_ERR_AUTH_FAILURE.  Either way the server's phase-1 state is zeroed.
 *            Divergence: a server with no phase-1 state fails here.  The reference compares Ni against a nil MAC, so
 *            an empty Ni passes and the proof is sealed under an all-zero key.
 *   other    empty answer, out_err[i] = 0, no state change.
 * out_off[i] .. out_off[i+1]: item i's answer in out_blob.  Per-call device and host buffers that held b or Ki are
 * zeroed before the call returns.  The attempts counter, its delay and ErrAuthTooManyAttempts, request framing and the
 * per-variable session map stay in Go (INTEGRATION.md). */
int bftq_auth_server_respond_batch(bftq_engine* e, bftq_auth_server* const* handles, uint32_t n_handles, const uint32_t* handle_idx,
                                   const int32_t* phase, const uint8_t* req_blob, const uint64_t* req_off, const uint8_t* rand_blob,
                                   const uint64_t* rand_off, uint64_t n_items, int32_t* out_err, uint8_t* out_blob, uint64_t out_cap,
                                   uint64_t* out_off);

/* ---- threshold password authentication, client half (crypto/auth/auth.go:239-399, K10) ---------------------------
 * bftq_auth_client_create is auth.NewClient(cred, n, k), 1 <= k <= n <= 255.  The password goes to the session's device
 * allocation (header: a, a^-1 mod q, gs; n slots: a'_i, ke and its flag; then the password), zeroed before it
 * is freed (bftq_auth_client_destroy, bftq_shutdown).  The host keeps public values only: per peer its id, x, Yi, salt,
 * Xi, Ni and Pi.  The salt's HMAC key block is public and travels with each phase-1 item. */
typedef struct bftq_auth_client bftq_auth_client;
int  bftq_auth_client_create(bftq_engine* e, const uint8_t* cred, uint64_t cred_len, uint32_t n, uint32_t k, bftq_auth_client** out);
void bftq_auth_client_destroy(bftq_auth_client* c);

#define BFTQ_AUTH_INITIATE   (-1)   /* generateX: rand = a, 256 big-endian bytes           -> out = X.Bytes()              */
                                    /* 0, 1, 2: ProcessResponse(phase, data, peer_id)      -> out = the returned map, if any */
#define BFTQ_AUTH_CIPHER_KEY (-2)   /* GetCipherKey                                         -> out = 32 bytes               */

/* The calls a Go client makes one at a time, batched: item i applies op[i] to handles[handle_idx[i]] with data
 * data_blob[data_off[i] .. data_off[i+1]) (the answer of peer_id[i]) and randomness rand_blob[rand_off[i] .. rand_off[i+1]).
 * The result equals the same calls made one after another in item order; items of different sessions are independent.
 *   INITIATE     rand = a (256 bytes, as rand.Int(rand.Reader, q)); out = X.Bytes().  A second INITIATE replaces a and keeps
 *                the secrets, gs and the response counter.
 *   phase 0      processYi.  An item that leaves at least k secrets completes: gs = prod Yi^lambda_i over every secret, a
 *                fresh a' per secret from rand (m x 256 bytes, one per secret in first-arrival order, m >= the secrets
 *                the item leaves; extra bytes are ignored, as is the rand of an item that does not complete), and
 *                out = the map {peer: Xi}.  A repeated peer replaces its secret (and drops its keys, Ni and Pi).
 *   phase 1      processBi: Ki = Bi^(a a' mod q), keySched, Ni = MAC(km, Xi, Bi.Bytes()) of the received Bi; every answer
 *                counts, repeated ones too; the answer that brings the count to the number of secrets returns {peer: Ni}
 *                (an empty Ni for a peer that never answered) and resets the count.
 *   phase 2      processZi: Pi = AES-128-GCM(ke).Open(nonce, Zi, Ni); a failure does not count and, as Go's
 *                `secret.Pi, err = decrypt(...)`, leaves the peer with no Pi (an empty map entry); the count reaching the
 *                number of secrets returns {peer: Pi}.
 *   CIPHER_KEY   SHA-256((gs^(a^-1) mod p).Bytes() || pw), 32 bytes.
 *   other ops    nothing (ProcessResponse's other phases).
 * A map is u32 count | count x (u64 peer id | u64 length | bytes), big-endian, in the order the secrets first arrived (one
 * legal order of Go's map); out_has_map[i] = 1 tells Go's non-nil map from nil.  Item i's output is at out_blob[out_off[i] ..
 * out_off[i+1]).
 *   out_err[i]   0 | BFTQ_ERR_MALFORMED (parseYi / parseBi / parseZi) | BFTQ_ERR_NO_AUTH_DATA (phase 1 or 2 from a peer with no
 *                secret) | BFTQ_ERR_DECRYPTION_FAILED | BFTQ_ERR_INSUFFICIENT_SECRETS (CIPHER_KEY before gs).  A failed item
 *                changes nothing, except that BFTQ_ERR_DECRYPTION_FAILED drops the peer's Pi, as Go does.
 * BFTQ_ERR_INVALID_ARG before any work, with nothing changed: items of one session with different ops, INITIATE or CIPHER_KEY
 * twice for one session, a rand of the wrong length, a = 0 mod q (ModInverse fails), more than n distinct phase-0 peers, a
 * phase 1 or CIPHER_KEY on a session with no a or a phase 1 on a secret with no a' (Go dereferences nil there), or out_cap
 * below *out_need.  *out_need (the bytes the outputs may take, from public data) is set on every return.
 * Divergences: phase 2 for a peer whose keys phase 1 never set fails with BFTQ_ERR_DECRYPTION_FAILED (Go opens under an
 * all-zero key); a nonce that is not 12 bytes fails with BFTQ_ERR_DECRYPTION_FAILED (Go's aead.Open panics); the (n+1)-th
 * distinct peer is rejected (protocol/client.go multicasts to n nodes only).  Per-call buffers that held a, a', e, f or Ki
 * are zeroed before the call returns.  A BFTQ_ERR_CUDA / BFTQ_ERR_NOMEM return after the device work began can leave the
 * device half of the call's sessions partly updated while their host half is not: destroy those sessions. */
int bftq_auth_client_process_batch(bftq_engine* e, bftq_auth_client* const* handles, uint32_t n_handles, const uint32_t* handle_idx,
                                   const int32_t* op, const uint64_t* peer_id, const uint8_t* data_blob, const uint64_t* data_off,
                                   const uint8_t* rand_blob, const uint64_t* rand_off, uint64_t n_items,
                                   int32_t* out_err, uint8_t* out_has_map, uint8_t* out_blob, uint64_t out_cap, uint64_t* out_off,
                                   uint64_t* out_need);

/* ---- DataEncryption (K11: crypto_pgp.go:532-554) ---------------------------------------------------------------------
 * Passphrase encryption of stored values, batched.  Item i's key is key_blob[key_off[i] .. key_off[i+1]) (any length).
 *
 * bftq_data_encrypt_batch: Encrypt(key, plain) as x/crypto's SymmetricallyEncrypt(w, key, nil, nil) + Write(plain) + Close
 * write it, byte for byte: an SKESK (v4, AES-128, iterated-and-salted S2K over SHA-256 with count byte 0x60, the session
 * key wrapped under the S2K key) and a SEIPD packet holding a text literal packet (empty name, time 0) and the MDC, with
 * Go's partial-length chunks.  rand: rand_len = 40 x n bytes, item i's at rand[40 i ..]: salt (8), session key (16),
 * IV (16), in the order Go reads its random source.  Item i's message goes to out_blob[out_off[i] .. out_off[i+1]); its
 * length is a function of the plain text's length only.  out_err[i] is 0.
 *
 * bftq_data_decrypt_batch: Decrypt(key, cipher) as ReadMessage's symmetric half + ReadAll.  The plain text goes to
 * out_blob[out_off[i] .. out_off[i+1]) (empty unless out_err[i] is 0).
 *   out_err[i]  0 | BFTQ_ERR_DECRYPTION_FAILED (no SKESK gives a key that passes the quick check: Go's prompt is asked
 *               forever) | BFTQ_ERR_MDC (the MDC packet is missing or does not match) | BFTQ_ERR_MESSAGE_BODY (the literal
 *               body ends early) | BFTQ_ERR_MALFORMED (framing, no SKESK, no SEIPD, a stream too short for the prefix or
 *               the MDC: Go panics on the nil message; divergence: a SEIPD body cut short, where Go returns ReadAll's
 *               read error) | BFTQ_ERR_UNSUPPORTED (compressed or signed inner data, tag 9, a
 *               PKESK, S2K modes other than 0 / 1 / 3 or hashes other than SHA-256, a SKESK that is not v4 AES, a 3DES or
 *               CAST5 key-encryption cipher, more than 16 SKESKs, packets after the SEIPD: the shim runs Go).
 *   A SKESK whose unwrapped cipher byte is unknown or has the wrong key length is skipped, as in Go.  Divergence: an
 *   unwrapped 3DES or CAST5 key is skipped too, where Go would try it.
 *
 * Both: every BFTQ_ERR_INVALID_ARG (NULL arguments, bad offsets, a rand of the wrong length, a key of 2^32 bytes or more,
 * out_cap below *out_need) is returned before any device work, with no output written.  *out_need (the exact output
 * length for encrypt, a bound for decrypt, from lengths only) is set on every return.  The keys, the S2K outputs, the
 * session keys and the plain texts are on the device only in a per-call buffer zeroed before the call returns. */
int bftq_data_encrypt_batch(bftq_engine* e, const uint8_t* key_blob, const uint64_t* key_off, const uint8_t* plain_blob,
                            const uint64_t* plain_off, const uint8_t* rand, uint64_t rand_len, uint64_t n_items, uint8_t* out_blob,
                            uint64_t out_cap, uint64_t* out_off, uint64_t* out_need, int32_t* out_err);
int bftq_data_decrypt_batch(bftq_engine* e, const uint8_t* key_blob, const uint64_t* key_off, const uint8_t* cipher_blob,
                            const uint64_t* cipher_off, uint64_t n_items, uint8_t* out_blob, uint64_t out_cap, uint64_t* out_off,
                            uint64_t* out_need, int32_t* out_err);

/* ---- quorum-descriptor builder (host only; no GPU needed) --------------------------------------
 * The step before the tally: wotqs.ChooseQuorum over the PGP trust graph
 * (quorum/wotqs/wotqs.go:36-127, node/graph/graph.go:46-75,117-125,279-393,420-438).  The shim
 * mirrors graph.AddNodes / SetSelfNodes / RemoveNodes / Revoke into it (node ids + the issuer ids of
 * each node's certifications, crypto_pgp.go:80-88 = bftq_keyring_certifiers) and caches the
 * descriptor per (rw, graph version) instead of recomputing it on every call as the reference
 * does.  rw = OR of BFTQ_RW_* (quorum/quorum.go:10-16). */
#define BFTQ_RW_READ  0x01
#define BFTQ_RW_WRITE 0x02
#define BFTQ_RW_AUTH  0x04
#define BFTQ_RW_CERT  0x08
#define BFTQ_RW_PEER  0x10
typedef struct bftq_graph bftq_graph;
int  bftq_graph_create(bftq_graph** out);
void bftq_graph_destroy(bftq_graph* g);
int  bftq_graph_add_node(bftq_graph* g, uint64_t id, const uint64_t* signer_ids, uint32_t n_signers);   /* graph.go:46-75 */
int  bftq_graph_set_self(bftq_graph* g, uint64_t id);                                                   /* graph.go:77-88 */
int  bftq_graph_remove_node(bftq_graph* g, uint64_t id);                                                /* graph.go:90-108 */
int  bftq_graph_revoke(bftq_graph* g, uint64_t id);                                                     /* graph.go:131-140 */
/* The graph's version (advanced by every mutation above) and the descriptor cache's counters: descriptors are cached
 * per rw and rebuilt only when the version moved — the reference recomputes them on every call. */
int  bftq_graph_version(bftq_graph* g, uint64_t* version, uint64_t* cache_hits, uint64_t* cache_builds);
/* wotqs.ChooseQuorum(rw): writes up to cap_qc cliques and cap_members member ids; *n_qc / *n_members
 * receive the required counts (call with caps 0 to size the buffers). */
int  bftq_graph_choose_quorum(bftq_graph* g, int rw, bftq_qc_ids_t* out_qcs, uint32_t cap_qc, uint32_t* n_qc,
                              uint64_t* out_members, uint32_t cap_members, uint32_t* n_members);

/* Client.revoke's equivocation scan (protocol/client.go:304-346; server side protocol/server.go:354-373), batched: for
 * every operation the signers that signed two DIFFERENT values at the same timestamp — "same signer, same t, different
 * value".  Response p of operation i (op_off as everywhere; status 0 = a good response, others are skipped; t == 0 is
 * skipped as the reference does) carries value_id[p] and the signers of its collective signature,
 * signer_ids[signer_off[p] .. signer_off[p+1]) (= CollectiveSignature.Signers(ss): bftq_signature_signers).  The ids to
 * revoke for operation i go to out_ids[out_off[i] .. out_off[i+1]), each once, in responder order (the reference's order
 * follows Go map iteration and is unspecified); *n_ids = total (call with cap_ids 0 to size out_ids).  Host-side
 * bookkeeping on ids — no crypto — so it needs no engine. */
int bftq_equivocation_scan_batch(const uint32_t* op_off, uint64_t n_ops, const uint8_t* status, const uint64_t* ts, const uint32_t* value_id,
                                 const uint32_t* signer_off, const uint64_t* signer_ids, uint32_t* out_off, uint64_t* out_ids, uint64_t cap_ids,
                                 uint64_t* n_ids);

/* ---- statistics ------------------------------------------------------------------------------
 * Counters since bftq_init (SURVEY §5 "metrics"): items verified, kernel launches. */
typedef struct {
  uint64_t items;          /* tuples pushed through bftq_rsa_verify_batch*            */
  uint64_t launches;       /* CUDA kernel launches issued by this engine              */
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  /* host half of the packet-level entry points, summed over their worker threads (nanoseconds) */
  uint64_t packer_chunks;    /* plans (chunks of a batch call) sent to the device                     */
  uint64_t packer_parse_ns;  /* OpenPGP parsing + keyring lookup + tuple composition                  */
  uint64_t packer_stage_ns;  /* composing the flat inputs in pinned staging + enqueueing copies/kernels */
  uint64_t packer_wait_ns;   /* waiting for a chunk's results                                          */
  int32_t  numa_node;        /* NUMA node of the engine's GPU (-1 unknown)                             */
  uint32_t numa_cpus;        /* CPUs the library's worker threads are bound to (0 = not bound)         */
  uint64_t msg_gpu_items;    /* transport answers decided on the GPU by bftq_read_responses_batch (K0m) and
                                bftq_read_encrypted_responses_batch (K6p .. K0m)                                  */
  uint64_t msg_host_items;   /* ... and the ones those kernels flagged, decided through the host packer / decrypt path */
  uint64_t unsupported_items;/* tuples answered BFTQ_ST_NOT_BUILT by the packer: key sizes / curves the reference's
                                library can verify and this build cannot (INTEGRATION.md "fallback")              */
} bftq_stats_t;
int bftq_stats(bftq_engine* e, bftq_stats_t* out);

/* ---- integer-pipe peak (roofline denominator) -----------------------------------------------
 * Runs independent carry chains of mad.lo.cc/madc.hi.cc pairs (the IMAD.WIDE.U32.X form the RSA kernel
 * executes) on the engine's device and returns the measured rate in 32x32->64 multiply-accumulates per second (SURVEY §8d: "measure
 * an unrolled mad.lo.u32 microbenchmark on the box; do not hard-code a datasheet number"). */
int bftq_measure_int_peak(bftq_engine* e, double* macs_per_second);

#ifdef __cplusplus
}
#endif
#endif /* BFTQ_H */
