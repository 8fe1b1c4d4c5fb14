"""Host-side mirror of the reference's operator interfaces for the hot path, over libbftq.so.

Names and argument meaning follow the reference (so tests read like the reference's own):
  crypto.Keyring              crypto/crypto.go:35-41      -> Keyring.register / remove / get_keyring
  crypto.Signature            crypto/crypto.go:50-58      -> Signature.sign / verify / verify_with_certificate / signers
  crypto.CollectiveSignature  crypto/crypto.go:66-71      -> CollectiveSignature.verify / combine / signers
  quorum.Quorum               quorum/quorum.go:18-25      -> Quorum.is_quorum / is_threshold / is_sufficient / reject
Errors are the reference's sentinels (crypto/crypto.go:13-33): every verification failure is
ErrInvalidSignature, a collective signature without enough valid signers is
ErrInsufficientNumberOfSignatures.  Each call is a batch of one; the *_batch variants are what a
batching aggregator (the Go shim's coalescer, INTEGRATION.md) feeds.
"""
import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .engine import Engine, QC, TALLY_IS_QUORUM, TALLY_IS_SUFFICIENT, TALLY_IS_THRESHOLD, TALLY_REJECT

ErrInvalidSignature = "crypto: invalid signature"
ErrInsufficientNumberOfSignatures = "crypto: insufficient number of signatures"
ErrDecryptionFailed = "crypto: decryption failed"
ErrInvalidTransportSecurityData = "crypto: invalid transport security data"
ErrMessageBody = "message body / nonce error"
ErrMessageUnsupported = "unsupported message form (compressed data)"
ErrNotBuilt = "gpu: key size / curve not built into libbftq (the shim re-runs the item on crypto/pgp)"
ErrMDC = "openpgp: invalid signature: hash mismatch"        # seMDCReader.Close's SignatureError, returned by ReadAll as is
ErrCertificateNotFound = "crypto: certifiate not found"            # the reference's spelling (crypto/crypto.go)
ErrSigningFailed = "crypto: failed to sign"
SIGN_PACKET_BYTES = 287                                     # BFTQ_SIGN_PACKET_BYTES
_ERR = {0: None, -6: ErrInvalidSignature, -7: ErrInsufficientNumberOfSignatures, -8: ErrDecryptionFailed, -9: ErrInvalidTransportSecurityData,
        -10: ErrMessageBody, -11: ErrMessageUnsupported, -12: ErrMDC}
_ERR_SIG = dict(_ERR)
_ERR_SIG[-11] = ErrNotBuilt


def _blob(items: Sequence[bytes]):
    off = np.zeros(len(items) + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in items])
    blob = np.frombuffer(b"".join(items) or b"\0", np.uint8).copy()
    return blob, off


class QCIds(C.Structure):
    _fields_ = [("f", C.c_int32), ("min", C.c_int32), ("threshold", C.c_int32), ("suff", C.c_int32),
                ("member_off", C.c_uint32), ("member_cnt", C.c_uint32)]


class Quorum:
    """A wotqs quorum (quorum/wotqs/wotqs.go:24-26): list of (f, min, threshold, suff, [node ids])."""

    def __init__(self, engine: Engine, qcs: Sequence[Tuple[int, int, int, int, Sequence[int]]]):
        self.engine, self.qcs = engine, [(f, mn, th, sf, list(m)) for f, mn, th, sf, m in qcs]
        ids = sorted({i for q in self.qcs for i in q[4]})
        self._dense = {nid: k for k, nid in enumerate(ids)}
        self._h = engine.quorum_create([(f, mn, th, sf, [self._dense[i] for i in m]) for f, mn, th, sf, m in self.qcs])

    def _c_desc(self):
        arr = (QCIds * max(1, len(self.qcs)))()
        members, off = [], 0
        for i, (f, mn, th, sf, m) in enumerate(self.qcs):
            arr[i] = QCIds(f, mn, th, sf, off, len(m))
            members += m
            off += len(m)
        return arr, np.asarray(members if members else [0], np.uint64), len(members)

    def _bits(self, nodes: Sequence[int], failed=False) -> int:
        unknown = len(self._dense)
        idx = np.asarray([self._dense.get(n, unknown) for n in nodes] or [0], np.uint32)
        st = np.full(len(idx), 1 if failed else 0, np.uint8)
        off = np.asarray([0, len(nodes)], np.uint32)
        return int(self.engine.tally_batch(self._h, off, idx, st)[0])

    def nodes(self) -> List[int]:
        return [i for q in self.qcs for i in q[4]]

    def is_quorum(self, nodes) -> bool:
        return bool(self._bits(nodes) & TALLY_IS_QUORUM)

    def is_threshold(self, nodes) -> bool:
        return bool(self._bits(nodes) & TALLY_IS_THRESHOLD)

    def is_sufficient(self, nodes) -> bool:
        return bool(self._bits(nodes) & TALLY_IS_SUFFICIENT)

    def reject(self, nodes) -> bool:
        return bool(self._bits(nodes, failed=True) & TALLY_REJECT)

    def get_threshold(self) -> int:
        return sum(q[2] for q in self.qcs)


class Keyring:
    """crypto/pgp PGPKeyring (crypto_pgp.go:115-223) over bftq_keyring."""

    def __init__(self, engine: Optional[Engine]):
        """engine=None gives a parse-only keyring (host side only: parse / signers / certifiers)."""
        self.engine, self._lib = engine, _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.bftq_keyring_create(engine._h if engine is not None else None, C.byref(h)))
        self._h = h

    def register(self, key_blocks: bytes, priv: bool = False) -> int:
        buf = np.frombuffer(key_blocks or b"\0", np.uint8).copy()
        n = C.c_uint32()
        _lib.check(self._lib.bftq_keyring_add(self._h, C.c_void_p(buf.ctypes.data), len(key_blocks), int(priv), C.byref(n)))
        return n.value

    def register_private(self, packets: bytes) -> int:
        """bftq_keyring_add_private: OpenPGP secret-key packets (unprotected RSA-2048) -> keys registered on the device."""
        buf = np.frombuffer(packets or b"\0", np.uint8).copy()
        n = C.c_uint32()
        rc = self._lib.bftq_keyring_add_private(self._h, C.c_void_p(buf.ctypes.data), len(packets), C.byref(n))
        buf[:] = 0
        _lib.check(rc)
        return n.value

    def remove(self, ids: Sequence[int]):
        a = np.asarray(list(ids) or [0], np.uint64)
        _lib.check(self._lib.bftq_keyring_remove(self._h, C.c_void_p(a.ctypes.data), len(ids)))

    def get_keyring(self) -> List[int]:
        n = C.c_uint32()
        _lib.check(self._lib.bftq_keyring_ids(self._h, None, 0, C.byref(n)))
        out = np.zeros(max(1, n.value), np.uint64)
        _lib.check(self._lib.bftq_keyring_ids(self._h, C.c_void_p(out.ctypes.data), n.value, C.byref(n)))
        return [int(x) for x in out[:n.value]]

    def certifiers(self, key_id: int) -> List[int]:
        n = C.c_uint32()
        _lib.check(self._lib.bftq_keyring_certifiers(self._h, key_id, None, 0, C.byref(n)))
        out = np.zeros(max(1, n.value), np.uint64)
        _lib.check(self._lib.bftq_keyring_certifiers(self._h, key_id, C.c_void_p(out.ctypes.data), n.value, C.byref(n)))
        return [int(x) for x in out[:n.value]]

    def close(self):
        if self._h:
            self._lib.bftq_keyring_destroy(self._h)
            self._h = None


class Signature:
    """crypto.Signature (crypto_pgp.go:319-390): signing with the keyring's private key, and verification."""

    def __init__(self, keyring: Keyring):
        self.keyring, self._lib = keyring, _lib.load()

    def sign_batch(self, tbs: Sequence[bytes], ctimes: Sequence[int]):
        """PGPSignature.Sign over many tbs (bftq_signature_sign_batch): secring[0]'s primary key signs item i with creation
        time ctimes[i].  -> (errs, packets): errs[i] None or ErrSigningFailed, packets[i] the signature packet
        (SignaturePacket.Data) or None.  A call-level error (ErrCertificateNotFound's code -20, BFTQ_ERR_UNSUPPORTED: the
        shim signs on crypto/pgp) raises BftqError."""
        n = len(tbs)
        if len(ctimes) != n:
            raise ValueError("sign_batch: one creation time per tbs")
        tb, to = _blob(tbs)
        ct = np.asarray(list(ctimes) or [0], np.uint32)
        out = np.zeros(max(n, 1) * SIGN_PACKET_BYTES, np.uint8)
        err = np.zeros(max(n, 1), np.int32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        _lib.check(self._lib.bftq_signature_sign_batch(self.keyring._h, p(tb), p(to), p(ct), n, p(out), p(err)))
        errs = [None if e == 0 else ErrSigningFailed for e in err[:n]]
        packets = [bytes(out[i * SIGN_PACKET_BYTES:(i + 1) * SIGN_PACKET_BYTES]) if e is None else None for i, e in enumerate(errs)]
        return errs, packets

    def sign(self, tbs: bytes, ctime: Optional[int] = None):
        """Go's Sign: -> (packet, err), with time.Now()'s seconds as the default creation time."""
        import time
        try:
            errs, packets = self.sign_batch([tbs], [int(time.time()) if ctime is None else ctime])
        except _lib.BftqError as ex:
            if ex.code == -20:
                return None, ErrCertificateNotFound
            raise
        return packets[0], errs[0]

    def verify_batch(self, tbs: Sequence[bytes], sig_data: Sequence[bytes], certs: Optional[Sequence[bytes]] = None):
        n = len(tbs)
        tb, to = _blob(tbs)
        sb, so = _blob(sig_data)
        err = np.zeros(max(n, 1), np.int32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        if certs is None:
            _lib.check(self._lib.bftq_signature_verify_batch(self.keyring._h, p(tb), p(to), p(sb), p(so), n, p(err)))
        else:
            cb, co = _blob(certs)
            _lib.check(self._lib.bftq_signature_verify_with_cert_batch(self.keyring._h, p(tb), p(to), p(sb), p(so), p(cb), p(co), n, p(err)))
        return [_ERR_SIG[int(e)] for e in err[:n]]

    def verify(self, tbs: bytes, sig_data: bytes) -> Optional[str]:
        return self.verify_batch([tbs], [sig_data])[0]

    def verify_with_certificate(self, tbs: bytes, sig_data: bytes, cert: bytes) -> Optional[str]:
        return self.verify_batch([tbs], [sig_data], [cert])[0]

    def parse(self, sig_data: bytes, collective: bool = False):
        """Host-only walk of a SignaturePacket.Data stream: ([(issuer id, hash id), ...], failed)."""
        buf = np.frombuffer(sig_data or b"\0", np.uint8).copy()
        iss, hid = np.zeros(1024, np.uint64), np.zeros(1024, np.uint8)
        n, failed = C.c_uint32(), C.c_int32()
        _lib.check(self._lib.bftq_signature_parse(self.keyring._h, C.c_void_p(buf.ctypes.data), len(sig_data), int(collective),
                                                  C.c_void_p(iss.ctypes.data), C.c_void_p(hid.ctypes.data), 1024, C.byref(n), C.byref(failed)))
        return [(int(iss[i]), int(hid[i])) for i in range(min(n.value, 1024))], bool(failed.value)

    def signers(self, sig_data: bytes) -> List[int]:
        buf = np.frombuffer(sig_data or b"\0", np.uint8).copy()
        out = np.zeros(256, np.uint64)
        n = C.c_uint32()
        _lib.check(self._lib.bftq_signature_signers(self.keyring._h, C.c_void_p(buf.ctypes.data), len(sig_data),
                                                    C.c_void_p(out.ctypes.data), 256, C.byref(n)))
        return [int(x) for x in out[:n.value]]


class BatchingSignature:
    """crypto.Signature whose single-item Verify calls, issued concurrently from many threads (bftkv:
    goroutines), are coalesced into GPU batches by libbftq's aggregator (bftq_aggregator_*)."""

    def __init__(self, keyring: Keyring, max_batch: int = 16384, max_wait_us: int = 200):
        self.keyring, self._lib = keyring, _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.bftq_aggregator_create(keyring._h, max_batch, max_wait_us, C.byref(h)))
        self._h = h

    def _call(self, tbs: bytes, sig: bytes, cert: bytes):
        rc = self._lib.bftq_aggregator_verify(self._h, tbs, len(tbs), sig, len(sig), cert or None, len(cert or b""))
        if rc not in _ERR:
            _lib.check(rc)
        return _ERR[rc]

    def verify(self, tbs: bytes, sig_data: bytes) -> Optional[str]:
        return self._call(tbs, sig_data, b"")

    def verify_with_certificate(self, tbs: bytes, sig_data: bytes, cert: bytes) -> Optional[str]:
        return self._call(tbs, sig_data, cert)

    def stats(self):
        b, n = C.c_uint64(), C.c_uint64()
        _lib.check(self._lib.bftq_aggregator_stats(self._h, C.byref(b), C.byref(n)))
        return {"batches": b.value, "items": n.value}

    def close(self):
        if self._h:
            self._lib.bftq_aggregator_destroy(self._h)
            self._h = None


class CollectiveSignature:
    """crypto.CollectiveSignature (crypto_pgp.go:485-515)."""

    def __init__(self, signature: Signature):
        self.signature, self._lib = signature, _lib.load()

    def verify_batch(self, tbs: Sequence[bytes], ss_data: Sequence[bytes], q: Quorum):
        n = len(tbs)
        tb, to = _blob(tbs)
        sb, so = _blob(ss_data)
        arr, members, nm = q._c_desc()
        err = np.zeros(max(n, 1), np.int32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        _lib.check(self._lib.bftq_collective_verify_batch(self.signature.keyring._h, C.cast(arr, C.c_void_p), len(q.qcs), p(members), nm,
                                                          p(tb), p(to), p(sb), p(so), n, p(err)))
        return [_ERR_SIG[int(e)] for e in err[:n]]

    def verify(self, tbs: bytes, ss_data: bytes, q: Quorum):
        """Returns (error, completed) — the reference sets ss.Completed = true on success."""
        e = self.verify_batch([tbs], [ss_data], q)[0]
        return e, e is None

    def combine(self, ss_type: int, ss_data: bytes, s_type: int, s_data: bytes, q: Quorum):
        """Returns (sufficient, new_type, new_data) — crypto_pgp.go:506-515."""
        if ss_type == 0:
            ss_type = s_type
        elif ss_type != s_type:
            return False, ss_type, ss_data
        ss_data = (ss_data or b"") + (s_data or b"")
        buf = np.frombuffer(ss_data or b"\0", np.uint8).copy()
        arr, members, nm = q._c_desc()
        out = C.c_int32()
        _lib.check(self._lib.bftq_collective_combine_sufficient(self.signature.keyring._h, C.cast(arr, C.c_void_p), len(q.qcs),
                                                                C.c_void_p(members.ctypes.data), nm, C.c_void_p(buf.ctypes.data),
                                                                len(ss_data), C.byref(out)))
        return bool(out.value), ss_type, ss_data

    def signers(self, ss_data: bytes) -> List[int]:
        return self.signature.signers(ss_data)


READ, WRITE, AUTH, CERT, PEER = 0x01, 0x02, 0x04, 0x08, 0x10     # quorum/quorum.go:10-16


class QuorumSystem:
    """quorum.QuorumSystem (quorum/quorum.go:27-29) over the trust graph: mirrors graph.AddNodes /
    SetSelfNodes / RemoveNodes / Revoke (node/graph/graph.go) and wotqs.ChooseQuorum.  Host only."""

    def __init__(self):
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.bftq_graph_create(C.byref(h)))
        self._h = h

    def add_node(self, node_id: int, signers: Sequence[int] = ()):
        a = np.asarray(list(signers) or [0], np.uint64)
        _lib.check(self._lib.bftq_graph_add_node(self._h, node_id, C.c_void_p(a.ctypes.data), len(signers)))

    def set_self(self, node_id: int):
        _lib.check(self._lib.bftq_graph_set_self(self._h, node_id))

    def remove_node(self, node_id: int):
        _lib.check(self._lib.bftq_graph_remove_node(self._h, node_id))

    def revoke(self, node_id: int):
        _lib.check(self._lib.bftq_graph_revoke(self._h, node_id))

    def choose_quorum_desc(self, rw: int):
        """wotqs.ChooseQuorum(rw) as a descriptor: list of (f, min, threshold, suff, [node ids])."""
        nq, nm = C.c_uint32(), C.c_uint32()
        _lib.check(self._lib.bftq_graph_choose_quorum(self._h, rw, None, 0, C.byref(nq), None, 0, C.byref(nm)))
        arr = (QCIds * max(1, nq.value))()
        mem = np.zeros(max(1, nm.value), np.uint64)
        _lib.check(self._lib.bftq_graph_choose_quorum(self._h, rw, C.cast(arr, C.c_void_p), nq.value, C.byref(nq),
                                                      C.c_void_p(mem.ctypes.data), nm.value, C.byref(nm)))
        return [(arr[i].f, arr[i].min, arr[i].threshold, arr[i].suff,
                 [int(x) for x in mem[arr[i].member_off:arr[i].member_off + arr[i].member_cnt]]) for i in range(nq.value)]

    def choose_quorum(self, rw: int, engine: Engine) -> Quorum:
        return Quorum(engine, self.choose_quorum_desc(rw))

    def close(self):
        if self._h:
            self._lib.bftq_graph_destroy(self._h)
            self._h = None


class Message:
    """crypto.Message's Decrypt (crypto/crypto.go:60-64, crypto_pgp.go:453-471), signature half: the host has already
    removed the encryption layer; each item is the packet stream inside (one-pass signature, literal data, signature)."""

    def __init__(self, keyring: "Keyring"):
        self.kr = keyring

    def decrypt_verify_batch(self, streams: Sequence[bytes]):
        """-> list of dict(err, plain, nonce, signed_by_key_id, signer_known, binary)."""
        n = len(streams)
        if n == 0:
            return []
        blob, off = _blob(streams)
        total = int(off[-1])
        err = np.zeros(n, np.int32)
        by = np.zeros(n, np.uint64)
        flags = np.zeros(n, np.uint8)
        plain, nonce = np.zeros(max(total, 1), np.uint8), np.zeros(max(total, 1), np.uint8)
        plen, nlen = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        _lib.check(self.kr._lib.bftq_message_verify_batch(self.kr._h, p(blob), p(off), n, p(err), p(by), p(flags), p(plain), p(plen), p(nonce), p(nlen)))
        out = []
        for i in range(n):
            o = int(off[i])
            ok_body = int(err[i]) in (0, -6)
            out.append({"err": _ERR[int(err[i])], "plain": bytes(plain[o:o + int(plen[i])]) if ok_body else None,
                        "nonce": bytes(nonce[o:o + int(nlen[i])]) if ok_body else None, "signed_by_key_id": int(by[i]),
                        "signer_known": bool(flags[i] & 1), "binary": bool(flags[i] & 2)})
        return out

    def decrypt_verify(self, stream: bytes):
        return self.decrypt_verify_batch([stream])[0]

    def decrypt_batch(self, raws: Sequence[bytes]):
        """PGPMessage.Decrypt on raw encrypted transport messages (bftq_message_decrypt_batch): the session key is recovered
        with the private key registered by Keyring.register_private.  -> list of dicts as decrypt_verify_batch, plus
        "code" (the BFTQ_ERR_* value)."""
        n = len(raws)
        if n == 0:
            return []
        blob, off = _blob(raws)
        total = int(off[-1])
        err = np.zeros(n, np.int32)
        by = np.zeros(n, np.uint64)
        flags = np.zeros(n, np.uint8)
        plain, nonce = np.zeros(max(total, 1), np.uint8), np.zeros(max(total, 1), np.uint8)
        plen, nlen = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        _lib.check(self.kr._lib.bftq_message_decrypt_batch(self.kr._h, p(blob), p(off), n, p(err), p(by), p(flags), p(plain), p(plen), p(nonce), p(nlen)))
        out = []
        for i in range(n):
            o = int(off[i])
            ok_body = int(err[i]) in (0, -6)
            out.append({"code": int(err[i]), "err": _ERR[int(err[i])], "plain": bytes(plain[o:o + int(plen[i])]) if ok_body else None,
                        "nonce": bytes(nonce[o:o + int(nlen[i])]) if ok_body else None, "signed_by_key_id": int(by[i]),
                        "signer_known": bool(flags[i] & 1), "binary": bool(flags[i] & 2)})
        return out


def _read_args(qcs, op_off, peer_ids, msgs, nonces, pre_status, blobs):
    op_off = np.ascontiguousarray(op_off, np.uint32)
    n_ops, n = len(op_off) - 1, int(op_off[-1])
    arr = (QCIds * max(1, len(qcs)))()
    members, off = [], 0
    for i, (f, mn, th, sf, m) in enumerate(qcs):
        arr[i] = QCIds(f, mn, th, sf, off, len(m))
        members += list(m)
        off += len(m)
    mem = np.asarray(members if members else [0], np.uint64)
    blob, moff = blobs if blobs is not None else _blob(msgs)
    nonces = np.ascontiguousarray(nonces, np.uint8)
    pre = None if pre_status is None else np.ascontiguousarray(pre_status, np.uint8)
    out = {"status": np.zeros(max(n, 1), np.uint8), "ts": np.zeros(max(n, 1), np.uint64), "value_off": np.zeros(max(n, 1), np.uint32),
           "value_len": np.zeros(max(n, 1), np.uint32), "decision": np.zeros(n_ops, np.uint8), "winner": np.zeros(n_ops, np.uint32),
           "decided_at": np.zeros(n_ops, np.uint32)}
    return op_off, n_ops, n, arr, mem, len(members), blob, moff, np.ascontiguousarray(peer_ids, np.uint64), nonces, pre, out


def read_encrypted_responses_batch(kr: "Keyring", qcs, op_off, peer_ids, raws: Sequence[bytes], nonces, pre_status=None, blobs=None, want_plain=True):
    """Client.Read from the raw wire answers (bftq_read_encrypted_responses_batch): as read_responses_batch, but each answer
    is the encrypted transport message (PKESK + SEIPD) and the client's private key must be registered
    (Keyring.register_private).  With want_plain the result also holds "plain": the good answers' plain texts (bytes, b""
    for the others)."""
    op_off, n_ops, n, arr, mem, n_mem, blob, moff, peer_ids, nonces, pre, out = _read_args(qcs, op_off, peer_ids, raws, nonces, pre_status, blobs)
    pblob = np.zeros(max(int(moff[-1]) if len(moff) else 0, 1), np.uint8) if want_plain else None
    plen = np.zeros(max(n, 1), np.uint32) if want_plain else None
    p = lambda a: C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)
    _lib.check(kr._lib.bftq_read_encrypted_responses_batch(kr._h, C.cast(arr, C.c_void_p), len(qcs), p(mem), n_mem, p(op_off), n_ops, p(peer_ids), p(blob),
                                                           p(moff), p(pre), p(nonces), int(nonces.shape[1]), p(out["status"]), p(out["ts"]),
                                                           p(out["value_off"]), p(out["value_len"]), p(pblob), p(plen), p(out["decision"]),
                                                           p(out["winner"]), p(out["decided_at"])))
    for k in ("status", "ts", "value_off", "value_len"):
        out[k] = out[k][:n]
    if want_plain:
        out["plain_len"] = plen[:n]
        out["plain"] = [bytes(pblob[int(moff[i]):int(moff[i]) + int(plen[i])]) for i in range(n)]
    return out


def read_responses_batch(kr: "Keyring", qcs, op_off, peer_ids, msgs: Sequence[bytes], nonces, pre_status=None, blobs=None):
    """Client.Read from raw answers (bftq_read_responses_batch).  qcs: [(f, min, threshold, suff, [node ids])]; op_off (n_ops+1)
    uint32; peer_ids (N) uint64; msgs: N decrypted answers; nonces (N, nonce_len) uint8 — the nonces the requests carried.
    blobs: (msg_blob, msg_off) arrays to use instead of joining `msgs` (e.g. page-locked ones).
    Returns dict(status, ts, value_off, value_len, decision, winner, decided_at)."""
    op_off, n_ops, n, arr, mem, n_mem, blob, moff, peer_ids, nonces, pre, out = _read_args(qcs, op_off, peer_ids, msgs, nonces, pre_status, blobs)
    p = lambda a: C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)
    _lib.check(kr._lib.bftq_read_responses_batch(kr._h, C.cast(arr, C.c_void_p), len(qcs), p(mem), n_mem, p(op_off), n_ops, p(peer_ids), p(blob), p(moff),
                                                 p(pre), p(nonces), int(nonces.shape[1]), p(out["status"]), p(out["ts"]), p(out["value_off"]), p(out["value_len"]),
                                                 p(out["decision"]), p(out["winner"]), p(out["decided_at"])))
    for k in ("status", "ts", "value_off", "value_len"):
        out[k] = out[k][:n]
    return out


ErrInvalidInput = "crypto: invalid input"
ErrInsufficientNumberOfThresholdSignatures = "crypto: insufficient number of threshold signatures"


class ThresholdRSA:
    """crypto.Threshold for TH_RSA (crypto/threshold/rsa/rsa.go): the server's Sign over registered shares and the client's
    ProcessResponse, both batched.  A share is the saved parameter (ThresholdInstance's secret without its algo byte)."""

    def __init__(self, engine: Engine):
        self.engine = engine
        self._shares = {}

    def register(self, sec: bytes):
        """Uploads a share once (opt-in: its fragments then live on the device until close())."""
        if sec not in self._shares:
            self._shares[sec] = self.engine.thrsa_share_create(sec)
        return self._shares[sec]

    def sign_batch(self, secs: Sequence[bytes], reqs: Sequence[bytes]):
        """[(serialized partial signature or None, error or None)], as Sign(sec, req) returns them."""
        handles, idx, pos = [], [], {}
        for s in secs:
            h = self.register(s)
            if h.value not in pos:
                pos[h.value] = len(handles)
                handles.append(h)
            idx.append(pos[h.value])
        err, outs = self.engine.thrsa_sign_batch(handles, idx, list(reqs))
        res = []
        for e, o in zip(err, outs):
            if e == 0:
                res.append((o if o else None, None))
            else:
                res.append((None, {-13: ErrInvalidInput, -8: "threshold rsa: malformed request"}.get(int(e), ErrNotBuilt)))
        return res

    def sign(self, sec: bytes, req: bytes):
        return self.sign_batch([sec], [req])[0]

    def process(self, n: int, k: int, responses: Sequence[bytes]):
        """ProcessResponse over the responses so far (arrival order): (signature or None, error or None, index of the deciding
        response or None, missing keys for the next MakeRequest)."""
        state, err, at, sig, missing = self.engine.thrsa_process_batch(n, k, [list(responses)])[0]
        if state == 1:
            return sig, None, at, []
        if state == 2:
            return None, ({-8: "threshold rsa: malformed response"}.get(err, ErrNotBuilt)), at, []
        return None, (None if missing else ErrInsufficientNumberOfThresholdSignatures), None, missing

    def close(self):
        for h in self._shares.values():
            self.engine.thrsa_share_destroy(h)
        self._shares = {}


ErrShareNotFound = "crypto: share not found"
ErrKeyNotFound = "crypto: key not found"
TH_DSA, TH_ECDSA = 2, 3


class ThresholdDSA:
    """The server half of crypto.Threshold for TH_DSA / TH_ECDSA (crypto/threshold/dsa/dsa_core.go dsaContext.Sign):
    phases 2 and 3 over registered shares, batched.  Phase 1 (random joint shares, Message.Encrypt) stays on Go, which
    passes the nonce it kept for the peer.  curve: "dsa" or "p256".  keyring: the server's Keyring (its private key and
    the nodes' certificates), which decrypts the joint shares."""

    _ERRS = {-8: "threshold dsa: malformed request or share", -13: ErrInvalidInput, -14: ErrShareNotFound, -15: ErrKeyNotFound,
             -6: ErrInvalidSignature, -9: ErrInvalidTransportSecurityData, -10: ErrMessageBody, -12: ErrMDC, -11: ErrNotBuilt}

    def __init__(self, engine: Engine, curve: str = "dsa"):
        self.engine = engine
        self.algo = {"dsa": TH_DSA, "p256": TH_ECDSA}[curve]
        self._shares = {}

    def register(self, sec: bytes):
        """Uploads a share once (opt-in: Y and the (k, c) table then live on the device until close())."""
        if sec not in self._shares:
            self._shares[sec] = self.engine.thdsa_share_create(self.algo, sec)
        return self._shares[sec]

    def sign_batch(self, keyring: "Keyring", secs: Sequence[bytes], reqs: Sequence[bytes], peer_ids: Sequence[int], self_id: int,
                   nonces: Sequence[Optional[bytes]]):
        """[(serialized partial signature or None, error or None)], as Sign(sec, req, peerId, selfId) returns them, in order."""
        handles, idx, pos = [], [], {}
        for s in secs:
            h = self.register(s)
            if h.value not in pos:
                pos[h.value] = len(handles)
                handles.append(h)
            idx.append(pos[h.value])
        err, outs = self.engine.thdsa_sign_batch(keyring._h, handles, idx, list(reqs), list(peer_ids), self_id, list(nonces))
        return [(o, None) if e == 0 else (None, self._ERRS.get(int(e), ErrDecryptionFailed)) for e, o in zip(err, outs)]

    def sign(self, keyring, sec: bytes, req: bytes, peer_id: int, self_id: int, nonce: Optional[bytes]):
        return self.sign_batch(keyring, [sec], [req], [peer_id], self_id, [nonce])[0]

    def close(self):
        for h in self._shares.values():
            self.engine.thdsa_share_destroy(h)
        self._shares = {}


ErrContinue = "crypto: continue"
THDSA_REQUEST, THDSA_RESPONSE = -1, 0
THDSA_PENDING, THDSA_CONTINUE, THDSA_SIGNED, THDSA_FAILED = 0, 1, 2, 3


class ThresholdDSAProcess:
    """The client half of crypto.Threshold for TH_DSA / TH_ECDSA (dsa_core.go dsaProc): MakeRequest and ProcessResponse
    over a process whose CalculateR and calculateS run on the device.  The process holds public state only.  dgst is
    hash(tbs) as NewProcess computes it; t and node_ids are the context's.  ErrContinue is returned as a sentinel string."""

    _ERRS = {-8: "threshold dsa: malformed response", -4: ErrNotBuilt}

    def __init__(self, engine: Engine, curve: str, dgst: bytes, t: int, node_ids: Sequence[int]):
        self.engine = engine
        self._h = engine.thdsa_proc_create({"dsa": TH_DSA, "p256": TH_ECDSA}[curve], dgst, t, list(node_ids))

    @classmethod
    def process_batch(cls, engine: Engine, procs: Sequence["ThresholdDSAProcess"], ops: Sequence[int], datas: Sequence[bytes],
                      peer_ids: Sequence[int]):
        """Items (procs[i], ops[i], datas[i], peer_ids[i]) in one call, applied as if one at a time in order.  A REQUEST gives
        ((node ids, request bytes or None), None); a RESPONSE (result or None, None / ErrContinue / an error)."""
        tab = list({id(p): p for p in procs}.values())
        pos = {id(p): j for j, p in enumerate(tab)}
        state, err, outs = engine.thdsa_process_batch([p._h for p in tab], [pos[id(p)] for p in procs], list(ops), list(peer_ids), list(datas))
        res = []
        for op, st, e, o in zip(ops, state, err, outs):
            if st == THDSA_FAILED:
                res.append((None, cls._ERRS.get(int(e), int(e))))
            elif op == THDSA_REQUEST:
                cnt = int.from_bytes(o[:4], "big")
                ids = [int.from_bytes(o[4 + 8 * j:12 + 8 * j], "big") for j in range(cnt)]
                req = o[4 + 8 * cnt:]
                res.append(((ids, req or None), None))
            elif st == THDSA_SIGNED:
                res.append((o, None))
            else:
                res.append((None, ErrContinue if st == THDSA_CONTINUE else None))
        return res

    def make_request(self):
        """MakeRequest(): ((node ids, request or None), err)."""
        return self.process_batch(self.engine, [self], [THDSA_REQUEST], [b""], [0])[0]

    def process_response(self, data: bytes, peer_id: int):
        """ProcessResponse(data, peer): (result or None, err)."""
        return self.process_batch(self.engine, [self], [THDSA_RESPONSE], [data], [peer_id])[0]

    def close(self):
        if self._h is not None:
            self.engine.thdsa_proc_destroy(self._h)
            self._h = None


ErrAuthenticationFailure = "authentication failure"
ErrAuthTooManyAttempts = "crypto: too many attempts"
AUTH_RETRY_LIMIT = 10
AUTH_DELAY_RATE = 1.0                  # seconds of delay per earlier phase-0 attempt (auth.go AUTH_DELAY_RATE)
# p of crypto/auth (auth.go:81-115)
AUTH_P = int("b0a67d9f5cebc0ffe81690e7b2670ab05f9fa4c2e73639f660c0408a2d9a4a8b454a9893fd7d4e8fa399cfc9c9ba05b080f903e33bcdcbefaed40915"
             "e51d46f58d1a5bd204db20fa3fe9db71f0b8e0aa87b5771406f25fad59e7f10fe52556447588"
             "72ea2dec1f6dcd11be905de59a044f6c2ea3982b2235acc9021a196fc4ce0b19f6b312ee9cfc5997dc5f7ce2f386131294a56ba93a41a3b60e27e03956039f51"
             "ae73b89c795c5ae7d841e9b455c37341c052404e8fe9fe4f0d52bc162a41f1eeb9ef292c66a9d6a619aa548807eb1187ee22bd62e20e26c3c08c22ecef12d3"
             "b2304a010ed1f50a68e0261afe1a0bdddf7ab8a61774d3af3f1cce2b95dad3", 16)


class AuthServer:
    """The server half of crypto/auth (threshold password authentication): NewServer / MakeResponse over a server
    registered on the device.  Phase 0 answers Yi, phase 1 Bi (and keeps ke and the MAC on the device), phase 2 seals the
    proof.  The attempts counter and its delay stay here, as in auth.go; `delay` is the sleep function (injectable, so
    tests do not sleep).  One divergence: phase 2 before any phase 1 is ErrAuthenticationFailure (the reference seals the
    proof under an all-zero key there)."""

    def __init__(self, engine: Engine, params: bytes, proof: bytes, delay=None):
        import time
        self.engine = engine
        self.attempts = 0
        self._delay = delay if delay is not None else time.sleep
        self._h = engine.auth_server_create(params, proof)

    @staticmethod
    def draw(phase: int) -> bytes:
        """The randomness MakeResponse draws: b = rand.Int(rand.Reader, p) for phase 1, a 12-byte nonce for phase 2."""
        import secrets
        if phase == 1:
            return secrets.randbelow(AUTH_P).to_bytes(256, "big")
        return secrets.token_bytes(12) if phase == 2 else b""

    @classmethod
    def respond_batch(cls, engine: Engine, servers: Sequence["AuthServer"], phases: Sequence[int], reqs: Sequence[bytes],
                      rands: Optional[Sequence[bytes]] = None):
        """MakeResponse over distinct servers in one call: [(res, done, err)] in order.  rands: the randomness per item
        (None: drawn here)."""
        if rands is None:
            rands = [cls.draw(p) for p in phases]
        err, outs = engine.auth_server_respond_batch([s._h for s in servers], list(range(len(servers))), list(phases), list(reqs), list(rands))
        res = []
        for s, ph, e, o in zip(servers, phases, err, outs):
            if ph == 0:
                delay = s.attempts * AUTH_DELAY_RATE
                if delay > 0:
                    s._delay(delay)
                s.attempts += 1
                res.append((o, False, ErrAuthTooManyAttempts if s.attempts >= AUTH_RETRY_LIMIT else None))
            elif ph == 1:
                res.append((o, False, None))
            elif ph == 2:
                res.append((o, True, None) if e == 0 else (None, True, ErrAuthenticationFailure))
            else:
                res.append((None, False, None))
        return res

    def make_response(self, phase: int, req: bytes, rand: Optional[bytes] = None):
        """(res, done, err) as AuthServer.MakeResponse returns them."""
        return self.respond_batch(self.engine, [self], [phase], [req], None if rand is None else [rand])[0]

    def close(self):
        if self._h is not None:
            self.engine.auth_server_destroy(self._h)
            self._h = None


ErrNoAuthenticationData = "crypto: no authentication data"
ErrInsufficientNumberOfSecrets = "crypto: insufficient number of secrets"
AUTH_Q = (AUTH_P - 1) // 2
AUTH_INITIATE, AUTH_CIPHER_KEY = -1, -2
_AUTH_CLIENT_ERRORS = {-8: "malformed answer", -17: ErrNoAuthenticationData, -18: ErrDecryptionFailed, -19: ErrInsufficientNumberOfSecrets}


class AuthClient:
    """The client half of crypto/auth: NewClient / Initiate / ProcessResponse / Done / GetCipherKey over a session
    registered on the device.  The password, a, a' and gs stay on the device.  `rand(n)` draws an integer below n (default
    secrets.randbelow, injectable for tests): a = rand(q) at Initiate, and a' = rand(q) per secret when a phase-0 answer
    completes the set, in the order the secrets first arrived.  Maps are dicts in that order; None is Go's nil map."""

    def __init__(self, engine: Engine, password: bytes, n: int, k: int, rand=None):
        import secrets
        self.engine = engine
        self.n, self.k = n, k
        self._rand = rand if rand is not None else secrets.randbelow
        self._peers = []                        # distinct phase-0 peers so far: how many a' a completing answer needs
        self._h = engine.auth_client_create(password, n, k)

    def _rand_for(self, op: int, peer_id: int) -> bytes:
        if op == AUTH_INITIATE:
            return self._rand(AUTH_Q).to_bytes(256, "big")
        if op == 0:
            m = len(self._peers) + (peer_id not in self._peers)
            if m >= self.k:
                return b"".join(self._rand(AUTH_Q).to_bytes(256, "big") for _ in range(m))
        return b""

    @staticmethod
    def _parse_map(b: bytes) -> dict:
        import struct
        cnt, pos, out = struct.unpack(">I", b[:4])[0], 4, {}
        for _ in range(cnt):
            pid, ln = struct.unpack(">QQ", b[pos:pos + 16])
            out[pid] = b[pos + 16:pos + 16 + ln]
            pos += 16 + ln
        return out

    @classmethod
    def process_batch(cls, engine: Engine, clients: Sequence["AuthClient"], ops: Sequence[int], datas: Sequence[bytes],
                      peer_ids: Sequence[int], rands: Optional[Sequence[bytes]] = None):
        """Items (clients[i], ops[i], datas[i], peer_ids[i]) in one call, applied as if one at a time in order:
        [(result, err)].  Initiate's result is X, a phase's the returned map (or None), GetCipherKey's the 32-byte key.
        rands: the randomness per item (None: drawn here)."""
        tab = list({id(c): c for c in clients}.values())
        pos = {id(c): j for j, c in enumerate(tab)}
        if rands is None:
            rands = []
            for c, op, pid in zip(clients, ops, peer_ids):
                rands.append(c._rand_for(op, pid))
                if op == 0 and pid not in c._peers:
                    c._peers.append(pid)
        err, has, outs = engine.auth_client_process_batch([c._h for c in tab], [pos[id(c)] for c in clients], list(ops), list(peer_ids),
                                                          list(datas), list(rands))
        res = []
        for c, op, pid, e, hm, o in zip(clients, ops, peer_ids, err, has, outs):
            if op == 0 and e == 0 and pid not in c._peers:
                c._peers.append(pid)
            if e != 0:
                res.append((None, _AUTH_CLIENT_ERRORS.get(int(e), int(e))))
            elif op in (AUTH_INITIATE, AUTH_CIPHER_KEY):
                res.append((o, None))
            else:
                res.append((cls._parse_map(o) if hm else None, None))
        return res

    def initiate(self, nodes: Sequence[int]) -> dict:
        """Initiate(nodes): {node id: X}."""
        X, _ = self.process_batch(self.engine, [self], [AUTH_INITIATE], [b""], [0])[0]
        return {nid: X for nid in nodes}

    def process_response(self, phase: int, data: bytes, peer_id: int):
        """ProcessResponse(phase, data, peer): (map or None, err)."""
        return self.process_batch(self.engine, [self], [phase], [data], [peer_id])[0]

    @staticmethod
    def done(phase: int) -> bool:
        return phase > 2

    def get_cipher_key(self):
        """GetCipherKey(): (key, err)."""
        return self.process_batch(self.engine, [self], [AUTH_CIPHER_KEY], [b""], [0])[0]

    def close(self):
        if self._h is not None:
            self.engine.auth_client_destroy(self._h)
            self._h = None


ErrUnexpectedEOF = "unexpected EOF"                        # io.ErrUnexpectedEOF: the literal body ends early
ErrMalformedMessage = "openpgp: malformed message (the reference's Decrypt panics on it, or fails reading a cut-short body)"
_DATA_ERRORS = {-8: ErrMalformedMessage, -10: ErrUnexpectedEOF, -11: ErrMessageUnsupported, -12: ErrMDC, -18: ErrDecryptionFailed}


class DataEncryption:
    """crypto.DataEncryption (crypto/crypto.go:73-76, crypto_pgp.go:525-554) on the device: Encrypt is x/crypto's
    SymmetricallyEncrypt byte for byte, Decrypt its ReadMessage.  `rand(n)` supplies Go's random bytes (default
    os.urandom, injectable for tests): 40 per Encrypt, salt, session key and IV.  Results are (value, err) pairs with the
    reference's errors; where Go would never return (a wrong key) the error is ErrDecryptionFailed, and where it would
    panic (a malformed message) ErrMalformedMessage, which also stands for a SEIPD body cut short (Go: ReadAll's read
    error)."""

    def __init__(self, engine: Engine, rand=None):
        import os
        self.engine = engine
        self._rand = rand if rand is not None else os.urandom

    def encrypt_batch(self, keys: Sequence[bytes], plains: Sequence[bytes]):
        rands = [self._rand(40) for _ in plains]
        err, outs = self.engine.data_encrypt_batch(list(keys), list(plains), rands)
        return [(o, None) if e == 0 else (None, _DATA_ERRORS.get(int(e), int(e))) for e, o in zip(err, outs)]

    def decrypt_batch(self, keys: Sequence[bytes], ciphers: Sequence[bytes]):
        err, outs = self.engine.data_decrypt_batch(list(keys), list(ciphers))
        return [(o, None) if e == 0 else (None, _DATA_ERRORS.get(int(e), int(e))) for e, o in zip(err, outs)]

    def encrypt(self, key: bytes, plain: bytes):
        return self.encrypt_batch([key], [plain])[0]

    def decrypt(self, key: bytes, cipher: bytes):
        return self.decrypt_batch([key], [cipher])[0]
