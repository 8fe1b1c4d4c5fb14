"""Thin host-side handle on a libbftq engine (one per GPU).  numpy arrays / raw pointers in,
numpy arrays out; all arithmetic happens in the CUDA kernels behind the C ABI."""
import ctypes as C
import numpy as np
from . import _lib

HASH_SHA256 = 8
F_STRICT_RANGE = 1
ST_OK, ST_BAD_SIGNATURE, ST_HASH_TAG, ST_MALFORMED, ST_UNKNOWN_SIGNER, ST_UNSUPPORTED, ST_MISSING = range(7)
DIGEST_LEN = {1: 16, 2: 20, 3: 20, 8: 32, 9: 48, 10: 64, 11: 28}


class QC(C.Structure):
    _fields_ = [("f", C.c_int32), ("min", C.c_int32), ("threshold", C.c_int32), ("suff", C.c_int32),
                ("member_off", C.c_uint32), ("member_cnt", C.c_uint32)]


TALLY_IS_QUORUM, TALLY_IS_THRESHOLD, TALLY_IS_SUFFICIENT, TALLY_REJECT = 1, 2, 4, 8
NO_WINNER = 0xFFFFFFFF
READ_VALUE, READ_REJECTED, READ_EXHAUSTED = 0, 1, 2


def _ptr(a):
    if a is None:
        return C.c_void_p(0)
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return C.c_void_p(a.ctypes.data)
    if isinstance(a, int):
        return C.c_void_p(a)
    if hasattr(a, "data_ptr"):           # torch tensor (host pinned or device)
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


class Engine:
    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.bftq_init(device, C.byref(h)))
        self._h = h
        self.device = device

    def close(self):
        if self._h:
            self._lib.bftq_shutdown(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def sm_count(self):
        return self._lib.bftq_device_sm_count(self._h)

    @property
    def key_count(self):
        return self._lib.bftq_key_count(self._h)

    def register_rsa_keys(self, moduli, exps) -> int:
        """moduli: iterable of Python ints of up to 4096 bits (or a (K,stride) uint8 big-endian array);
        returns the index of the first new key."""
        if not isinstance(moduli, np.ndarray):
            moduli = [int(n) for n in moduli]
            stride = 256 if all(n.bit_length() <= 2048 for n in moduli) else 512
            moduli = np.frombuffer(b"".join(n.to_bytes(stride, "big") for n in moduli), dtype=np.uint8).reshape(-1, stride)
        moduli = np.ascontiguousarray(moduli, dtype=np.uint8)
        exps = np.ascontiguousarray(np.asarray(exps, dtype=np.uint32))
        assert exps.shape[0] == moduli.shape[0]
        first = C.c_uint32()
        _lib.check(self._lib.bftq_register_rsa_keys_k(self._h, _ptr(moduli), moduli.shape[1], _ptr(exps), moduli.shape[0], C.byref(first)))
        return first.value

    def rsa_verify_batch(self, key_idx, sig_be, digest, hash_alg=HASH_SHA256, flags=0, out=None, key_bytes=256):
        """Host buffers (numpy or pinned torch tensors).  Returns uint8 status per item.
        key_bytes: size class of the batch (128/192/256/384/512); sig_be is (N, key_bytes)."""
        n = int(key_idx.shape[0])
        if out is None:
            out = np.empty(n, dtype=np.uint8)
        _lib.check(self._lib.bftq_rsa_verify_batch_k(self._h, key_bytes, _ptr(key_idx), _ptr(sig_be), _ptr(digest),
                                                     hash_alg, n, flags, _ptr(out)))
        return out

    def rsa_verify_batch_dev(self, d_key_idx, d_sig, d_digest, n, d_status, hash_alg=HASH_SHA256, flags=0, stream=0):
        _lib.check(self._lib.bftq_rsa_verify_batch_dev(self._h, _ptr(d_key_idx), _ptr(d_sig), _ptr(d_digest),
                                                       hash_alg, n, flags, _ptr(d_status), C.c_void_p(stream)))

    # ---- K2 ----
    def quorum_create(self, qcs):
        """qcs: list of (f, min, threshold, suff, [member key indices]).  Returns an opaque handle."""
        arr = (QC * max(1, len(qcs)))()
        members, off = [], 0
        for i, (f, mn, th, sf, mem) in enumerate(qcs):
            arr[i] = QC(f, mn, th, sf, off, len(mem))
            members += list(mem)
            off += len(mem)
        m = np.asarray(members if members else [0], dtype=np.uint32)
        h = C.c_void_p()
        _lib.check(self._lib.bftq_quorum_create(self._h, C.cast(arr, C.c_void_p), len(qcs), _ptr(m), len(members), C.byref(h)))
        return h

    def quorum_destroy(self, q):
        self._lib.bftq_quorum_destroy(self._h, q)

    def tally_batch(self, q, op_off, key_idx, status):
        n_ops = int(op_off.shape[0]) - 1
        out = np.empty(n_ops, np.uint8)
        _lib.check(self._lib.bftq_tally_batch(self._h, q, _ptr(op_off), _ptr(key_idx), _ptr(status), n_ops, _ptr(out)))
        return out

    def read_tally_batch(self, q, op_off, key_idx, status, ts, value_id):
        n_ops = int(op_off.shape[0]) - 1
        win, bits = np.empty(n_ops, np.uint32), np.empty(n_ops, np.uint8)
        _lib.check(self._lib.bftq_read_tally_batch(self._h, q, _ptr(op_off), _ptr(key_idx), _ptr(status), _ptr(ts), _ptr(value_id),
                                                   n_ops, _ptr(win), _ptr(bits)))
        return win, bits

    def verify_tally_batch(self, q, op_off, key_idx, sig_be, digest, pre_status=None, ts=None, value_id=None,
                           hash_alg=HASH_SHA256, flags=0, out_status=None, out_bits=None, out_winner=None):
        n_ops = int(op_off.shape[0]) - 1
        n_items = int(key_idx.shape[0])
        st = out_status if out_status is not None else np.empty(max(n_items, 1), np.uint8)
        bits = out_bits if out_bits is not None else np.empty(n_ops, np.uint8)
        win = out_winner if out_winner is not None else (np.empty(n_ops, np.uint32) if ts is not None else None)
        _lib.check(self._lib.bftq_verify_tally_batch(self._h, q, _ptr(op_off), _ptr(key_idx), _ptr(sig_be), _ptr(digest), hash_alg,
                                                     _ptr(pre_status), _ptr(ts), _ptr(value_id), n_ops, flags, _ptr(st), _ptr(bits),
                                                     _ptr(win)))
        return (st[:n_items] if out_status is None else st), bits, win

    def verify_tally_batch_dev(self, q, d_op_off, d_key_idx, d_sig, d_digest, n_ops, n_items, d_status, d_bits, d_pre=None,
                               d_ts=None, d_value_id=None, d_winner=None, hash_alg=HASH_SHA256, flags=0, stream=0):
        _lib.check(self._lib.bftq_verify_tally_batch_dev(self._h, q, _ptr(d_op_off), _ptr(d_key_idx), _ptr(d_sig), _ptr(d_digest),
                                                         hash_alg, _ptr(d_pre), _ptr(d_ts), _ptr(d_value_id), n_ops, n_items, flags,
                                                         _ptr(d_status), _ptr(d_bits), _ptr(d_winner), C.c_void_p(stream)))

    def read_decide_batch(self, q, op_off, key_idx, status, ts, value_id):
        """Client.Read's decision per operation, responders in arrival order -> (decision, winner, decided_at)."""
        n_ops = int(op_off.shape[0]) - 1
        dec, win, at = np.empty(n_ops, np.uint8), np.empty(n_ops, np.uint32), np.empty(n_ops, np.uint32)
        _lib.check(self._lib.bftq_read_decide_batch(self._h, q, _ptr(op_off), _ptr(key_idx), _ptr(status), _ptr(ts), _ptr(value_id), n_ops,
                                                    _ptr(dec), _ptr(win), _ptr(at)))
        return dec, win, at

    def verify_read_batch(self, q, op_off, key_idx, sig_be, digest, ts, value_id, pre_status=None, hash_alg=HASH_SHA256, flags=0,
                          out_status=None, out_decision=None, out_winner=None, out_decided_at=None):
        """K1 + Client.Read's decision, host buffers of any size (chunked inside the library).
        Returns (status, decision, winner, decided_at)."""
        n_ops = int(op_off.shape[0]) - 1
        n_items = int(key_idx.shape[0])
        st = out_status if out_status is not None else np.empty(max(n_items, 1), np.uint8)
        dec = out_decision if out_decision is not None else np.empty(n_ops, np.uint8)
        win = out_winner if out_winner is not None else np.empty(n_ops, np.uint32)
        at = out_decided_at if out_decided_at is not None else np.empty(n_ops, np.uint32)
        _lib.check(self._lib.bftq_verify_read_batch(self._h, q, _ptr(op_off), _ptr(key_idx), _ptr(sig_be), _ptr(digest), hash_alg,
                                                    _ptr(pre_status), _ptr(ts), _ptr(value_id), n_ops, flags, _ptr(st), _ptr(dec), _ptr(win),
                                                    _ptr(at)))
        return (st[:n_items] if out_status is None else st), dec, win, at

    def verify_read_batch_dev(self, q, d_op_off, d_key_idx, d_sig, d_digest, d_ts, d_value_id, n_ops, n_items, d_status, d_bits, d_decision,
                              d_winner, d_decided_at, d_pre=None, hash_alg=HASH_SHA256, flags=0, stream=0):
        _lib.check(self._lib.bftq_verify_read_batch_dev(self._h, q, _ptr(d_op_off), _ptr(d_key_idx), _ptr(d_sig), _ptr(d_digest), hash_alg,
                                                        _ptr(d_pre), _ptr(d_ts), _ptr(d_value_id), n_ops, n_items, flags, _ptr(d_status),
                                                        _ptr(d_bits), _ptr(d_decision), _ptr(d_winner), _ptr(d_decided_at), C.c_void_p(stream)))

    # ---- page-locked host memory on the GPU's NUMA node ----
    def host_alloc(self, shape, dtype=np.uint8):
        """numpy array over a bftq_host_alloc block (DMA'd in place by the *_batch calls).  Free with host_free(arr)."""
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        nbytes = int(np.prod(shape, dtype=np.int64)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        _lib.check(self._lib.bftq_host_alloc(self._h, max(nbytes, 1), C.byref(p)))
        buf = (C.c_uint8 * max(nbytes, 1)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape, dtype=np.int64))).reshape(shape)
        self._host_blocks = getattr(self, "_host_blocks", {})
        self._host_blocks[arr.ctypes.data] = p.value
        return arr

    def host_copy(self, a):
        """A page-locked copy of array `a` (what the shim does when it appends a request to its blob)."""
        a = np.ascontiguousarray(a)
        out = self.host_alloc(a.shape, a.dtype)
        out[...] = a
        return out

    def host_free(self, arr):
        p = getattr(self, "_host_blocks", {}).pop(arr.ctypes.data, None)
        if p is not None:
            _lib.check(self._lib.bftq_host_free(self._h, C.c_void_p(p)))

    def bind_thread(self) -> int:
        return self._lib.bftq_bind_thread(self._h)

    # ---- K3 ----
    def lagrange_combine_batch(self, m: int, x, y_be):
        """m: odd modulus (int); x: (B,k) int32; y_be: (B,k,mlen) uint8 big-endian.  Returns (out (B,mlen), status (B,))."""
        mlen = (m.bit_length() + 7) // 8
        x = np.ascontiguousarray(x, np.int32)
        y_be = np.ascontiguousarray(y_be, np.uint8)
        B, k = x.shape
        assert y_be.shape == (B, k, mlen)
        mb = np.frombuffer(m.to_bytes(mlen, "big"), np.uint8).copy()
        out, st = np.empty((B, mlen), np.uint8), np.empty(B, np.uint8)
        _lib.check(self._lib.bftq_lagrange_combine_batch(self._h, _ptr(mb), mlen, k, _ptr(x), _ptr(y_be), B, _ptr(out), _ptr(st)))
        return out, st

    # ---- K1b ----
    def ed25519_verify_batch(self, pubkeys, key_idx, sig, msg):
        """pubkeys (K,32), key_idx (N,), sig (N,64), msg (N,32) uint8/uint32 arrays -> status (N,)."""
        pubkeys = np.ascontiguousarray(pubkeys, np.uint8)
        n = int(key_idx.shape[0])
        out = np.empty(n, np.uint8)
        _lib.check(self._lib.bftq_ed25519_verify_batch(self._h, _ptr(pubkeys), pubkeys.shape[0], _ptr(key_idx), _ptr(sig), _ptr(msg), n, _ptr(out)))
        return out

    # ---- K1c ----
    def ecdsa_p256_verify_batch(self, pubkeys, key_idx, r_be, s_be, digest):
        """pubkeys (K,64) X||Y, key_idx (N,) uint32, r_be/s_be (N,32), digest (N,dlen) uint8 -> status (N,)."""
        pubkeys = np.ascontiguousarray(pubkeys, np.uint8)
        key_idx = np.ascontiguousarray(key_idx, np.uint32)
        r_be = np.ascontiguousarray(r_be, np.uint8)
        s_be = np.ascontiguousarray(s_be, np.uint8)
        digest = np.ascontiguousarray(digest, np.uint8)
        n = int(key_idx.shape[0])
        out = np.empty(n, np.uint8)
        _lib.check(self._lib.bftq_ecdsa_p256_verify_batch(self._h, _ptr(pubkeys), pubkeys.shape[0], _ptr(key_idx), _ptr(r_be),
                                                          _ptr(s_be), _ptr(digest), digest.shape[1] if n else 32, n, _ptr(out)))
        return out

    # ---- K1d ----
    def dsa_verify_batch(self, p: int, q: int, g: int, y: int, r_be, s_be, digest):
        """One DSA key (p, q, g, y); r_be/s_be (N,32), digest (N,dlen) uint8 -> status (N,)."""
        plen, qlen = (p.bit_length() + 7) // 8, (q.bit_length() + 7) // 8
        pb, qb = self._be([p], plen), self._be([q], qlen)
        gb, yb = self._be([g % p], plen), self._be([y % p], plen)
        r_be = np.ascontiguousarray(r_be, np.uint8)
        s_be = np.ascontiguousarray(s_be, np.uint8)
        digest = np.ascontiguousarray(digest, np.uint8)
        n = int(r_be.shape[0])
        out = np.empty(n, np.uint8)
        _lib.check(self._lib.bftq_dsa_verify_batch(self._h, _ptr(pb), plen, _ptr(qb), qlen, _ptr(gb), _ptr(yb), _ptr(r_be), _ptr(s_be),
                                                   _ptr(digest), digest.shape[1] if n else 32, n, _ptr(out)))
        return out

    # ---- K5 ----
    @staticmethod
    def _be(vals, width):
        return np.frombuffer(b"".join(int(v).to_bytes(width, "big") for v in vals), np.uint8).copy()

    def modexp_batch(self, m: int, bases, exps, elen=None):
        """[pow(b, e, m)] for a shared odd modulus of exactly 1024 or 2048 bits."""
        mlen = (m.bit_length() + 7) // 8
        elen = elen or max(1, max((int(e).bit_length() + 7) // 8 for e in exps))
        n = len(bases)
        out = np.empty((n, mlen), np.uint8)
        mb, bb, eb = self._be([m], mlen), self._be(bases, mlen), self._be(exps, elen)      # keep the buffers alive across the call
        _lib.check(self._lib.bftq_modexp_batch(self._h, _ptr(mb), mlen, _ptr(bb), _ptr(eb), elen, n, _ptr(out)))
        return [int.from_bytes(bytes(o), "big") for o in out]

    def modprod_batch(self, m: int, vals):
        """Threshold-RSA combine: [prod(row) mod m for row in vals] (rows of equal length)."""
        mlen = (m.bit_length() + 7) // 8
        B, k = len(vals), len(vals[0])
        mb, vb = self._be([m], mlen), self._be([v for row in vals for v in row], mlen)
        out = np.empty((B, mlen), np.uint8)
        _lib.check(self._lib.bftq_modprod_batch(self._h, _ptr(mb), mlen, k, _ptr(vb), B, _ptr(out)))
        return [bytes(o) for o in out]

    # ---- K7: threshold-RSA partial signing and the client's combine (crypto/threshold/rsa/rsa.go) ----
    def thrsa_share_create(self, sec: bytes):
        """Registers one share (rsaContext's saved parameter) on the device; returns its handle."""
        h = C.c_void_p()
        buf = np.frombuffer(sec, np.uint8) if sec else np.zeros(1, np.uint8)
        _lib.check(self._lib.bftq_thrsa_share_create(self._h, _ptr(buf), len(sec), C.byref(h)))
        return h

    def thrsa_share_destroy(self, share):
        self._lib.bftq_thrsa_share_destroy(share)

    @staticmethod
    def _blob(items):
        off = np.zeros(len(items) + 1, np.uint64)
        off[1:] = np.cumsum([len(b) for b in items], dtype=np.uint64) if items else []
        blob = np.frombuffer(b"".join(items), np.uint8) if off[-1] else np.zeros(1, np.uint8)
        return blob, off

    def thrsa_sign_batch(self, shares, share_idx, requests):
        """rsaContext.Sign over (shares[share_idx[i]], requests[i]): (out_err int32[n], [serialized partial signatures])."""
        n = len(requests)
        blob, off = self._blob(list(requests))
        tab = (C.c_void_p * max(1, len(shares)))(*[s.value for s in shares])
        idx = np.ascontiguousarray(share_idx, np.uint32)
        kids = [int.from_bytes(r[:2], "big") if len(r) >= 2 else 0 for r in requests]
        cap = sum(2 + k * (12 + 256) + 8 + 256 for k in kids)
        out = np.zeros(max(1, cap), np.uint8)
        out_off = np.zeros(n + 1, np.uint64)
        err = np.zeros(max(1, n), np.int32)
        _lib.check(self._lib.bftq_thrsa_sign_batch(self._h, tab, len(shares), _ptr(idx), _ptr(blob), _ptr(off), n, _ptr(err),
                                                   _ptr(out), cap, _ptr(out_off)))
        return err[:n], [bytes(out[out_off[i]:out_off[i + 1]]) for i in range(n)]

    def thrsa_process_batch(self, n: int, k: int, procs):
        """rsaProc.ProcessResponse replayed over each process's responses (lists of bytes, arrival order).  Per process:
        (state, err, at, signature bytes or None, missing key list)."""
        P = len(procs)
        flat = [r for rs in procs for r in rs]
        blob, off = self._blob(flat)
        poff = np.zeros(P + 1, np.uint64)
        poff[1:] = np.cumsum([len(rs) for rs in procs], dtype=np.uint64) if procs else []
        state, err = np.zeros(max(1, P), np.int32), np.zeros(max(1, P), np.int32)
        at = np.zeros(max(1, P), np.uint64)
        sig = np.zeros((max(1, P), 256), np.uint8)
        moff = np.zeros(P + 1, np.uint64)
        cap = 1 << 16
        while True:
            miss = np.zeros(cap, np.uint32)
            rc = self._lib.bftq_thrsa_process_batch(self._h, n, k, _ptr(blob), _ptr(off), _ptr(poff), P, _ptr(state), _ptr(err), _ptr(at),
                                                    _ptr(sig), _ptr(miss), cap, _ptr(moff))
            if rc == -3 and moff[P] > cap:
                cap = int(moff[P])
                continue
            _lib.check(rc)
            break
        return [(int(state[p]), int(err[p]), int(at[p]), bytes(sig[p]) if state[p] == 1 else None,
                 [int(x) for x in miss[moff[p]:moff[p + 1]]]) for p in range(P)]

    # ---- K8: threshold DSA / ECDSA partial signing (crypto/threshold/dsa/dsa_core.go) ----
    def thdsa_share_create(self, algo: int, sec: bytes):
        """Registers one share (dsaContext's saved parameter; algo 2 = TH_DSA, 3 = TH_ECDSA) on the device; returns its handle."""
        h = C.c_void_p()
        buf = np.frombuffer(sec, np.uint8) if sec else np.zeros(1, np.uint8)
        _lib.check(self._lib.bftq_thdsa_share_create(self._h, algo, _ptr(buf), len(sec), C.byref(h)))
        return h

    def thdsa_share_destroy(self, share):
        self._lib.bftq_thdsa_share_destroy(share)

    def thdsa_sign_batch(self, keyring, shares, share_idx, requests, peer_ids, self_id: int, nonces):
        """dsaContext.Sign phases 2 / 3 over (shares[share_idx[i]], requests[i], peer_ids[i]); nonces[i]: the phase-1 nonce
        stored for the peer, or None.  keyring: a crypto_gpu.Keyring handle.  (out_err int32[n], [serialized outputs])."""
        n = len(requests)
        blob, off = self._blob(list(requests))
        nblob, noff = self._blob([x or b"" for x in nonces])
        has = np.array([x is not None for x in nonces] or [0], np.uint8)
        tab = (C.c_void_p * max(1, len(shares)))(*[s.value for s in shares])
        idx = np.ascontiguousarray(share_idx, np.uint32)
        peers = np.ascontiguousarray(peer_ids, np.uint64) if n else np.zeros(1, np.uint64)
        cap = sum(int(self._lib.bftq_thdsa_share_out_bound(shares[i])) for i in share_idx)
        out = np.zeros(max(1, cap), np.uint8)
        out_off = np.zeros(n + 1, np.uint64)
        err = np.zeros(max(1, n), np.int32)
        _lib.check(self._lib.bftq_thdsa_sign_batch(keyring, tab, len(shares), _ptr(idx), _ptr(blob), _ptr(off), _ptr(peers), self_id,
                                                   _ptr(nblob), _ptr(noff), _ptr(has), n, _ptr(err), _ptr(out), cap, _ptr(out_off)))
        return err[:n], [bytes(out[out_off[i]:out_off[i + 1]]) for i in range(n)]

    def thdsa_proc_create(self, algo: int, dgst: bytes, t: int, node_ids):
        """A threshold-DSA client process (dsaContext.NewProcess; algo 2 = TH_DSA, 3 = TH_ECDSA), host memory only."""
        h = C.c_void_p()
        db = np.frombuffer(dgst, np.uint8) if dgst else np.zeros(1, np.uint8)
        ids = np.ascontiguousarray(list(node_ids) or [0], np.uint64)
        _lib.check(self._lib.bftq_thdsa_proc_create(algo, _ptr(db), len(dgst), t, _ptr(ids), len(node_ids), C.byref(h)))
        return h

    def thdsa_proc_destroy(self, proc):
        self._lib.bftq_thdsa_proc_destroy(proc)

    def thdsa_process_batch(self, procs, proc_idx, ops, peer_ids, datas):
        """MakeRequest (op -1) and ProcessResponse(datas[i], peer_ids[i]) (op 0) on procs[proc_idx[i]], one call.
        (out_state int32[n], out_err int32[n], [outputs]); the output buffer is sized from the library's out_need."""
        n = len(ops)
        blob, off = self._blob(list(datas))
        tab = (C.c_void_p * max(1, len(procs)))(*[p.value for p in procs])
        idx = np.ascontiguousarray(proc_idx, np.uint32) if n else np.zeros(1, np.uint32)
        op = np.ascontiguousarray(ops, np.int32) if n else np.zeros(1, np.int32)
        peers = np.ascontiguousarray(peer_ids, np.uint64) if n else np.zeros(1, np.uint64)
        out_off = np.zeros(n + 1, np.uint64)
        state = np.zeros(max(1, n), np.int32)
        err = np.zeros(max(1, n), np.int32)
        need = C.c_uint64(0)
        cap = 0
        while True:
            out = np.zeros(max(1, cap), np.uint8)
            rc = self._lib.bftq_thdsa_process_batch(self._h, tab, len(procs), _ptr(idx), _ptr(op), _ptr(peers), _ptr(blob), _ptr(off), n,
                                                    _ptr(state), _ptr(err), _ptr(out), cap, _ptr(out_off), C.byref(need))
            if rc == -3 and need.value > cap:
                cap = need.value
                continue
            _lib.check(rc)
            break
        return state[:n], err[:n], [bytes(out[out_off[i]:out_off[i + 1]]) for i in range(n)]

    def auth_server_create(self, params: bytes, proof: bytes):
        """Registers one password-authentication server (auth.NewServer(params, proof)) on the device; returns its handle."""
        h = C.c_void_p()
        pb = np.frombuffer(params, np.uint8) if params else np.zeros(1, np.uint8)
        fb = np.frombuffer(proof, np.uint8) if proof else np.zeros(1, np.uint8)
        _lib.check(self._lib.bftq_auth_server_create(self._h, _ptr(pb), len(params), _ptr(fb), len(proof), C.byref(h)))
        return h

    def auth_server_destroy(self, server):
        self._lib.bftq_auth_server_destroy(server)

    def auth_server_respond_batch(self, servers, server_idx, phases, requests, rands):
        """AuthServer.MakeResponse(phases[i], requests[i]) on servers[server_idx[i]], one call; rands[i]: b (256 bytes,
        phase 1), the GCM nonce (12 bytes, phase 2), else b"".  (out_err int32[n], [answers])."""
        n = len(requests)
        blob, off = self._blob(list(requests))
        rblob, roff = self._blob(list(rands))
        tab = (C.c_void_p * max(1, len(servers)))(*[s.value for s in servers])
        idx = np.ascontiguousarray(server_idx, np.uint32) if n else np.zeros(1, np.uint32)
        ph = np.ascontiguousarray(phases, np.int32) if n else np.zeros(1, np.int32)
        cap = sum(int(self._lib.bftq_auth_server_out_bound(servers[i], int(p))) for i, p in zip(server_idx, phases))
        out = np.zeros(max(1, cap), np.uint8)
        out_off = np.zeros(n + 1, np.uint64)
        err = np.zeros(max(1, n), np.int32)
        _lib.check(self._lib.bftq_auth_server_respond_batch(self._h, tab, len(servers), _ptr(idx), _ptr(ph), _ptr(blob), _ptr(off),
                                                            _ptr(rblob), _ptr(roff), n, _ptr(err), _ptr(out), cap, _ptr(out_off)))
        return err[:n], [bytes(out[out_off[i]:out_off[i + 1]]) for i in range(n)]

    def auth_client_create(self, password: bytes, n: int, k: int):
        """Registers one password-authentication client session (auth.NewClient(cred, n, k)) on the device; returns its handle."""
        h = C.c_void_p()
        pb = np.frombuffer(password, np.uint8) if password else np.zeros(1, np.uint8)
        _lib.check(self._lib.bftq_auth_client_create(self._h, _ptr(pb), len(password), n, k, C.byref(h)))
        return h

    def auth_client_destroy(self, client):
        self._lib.bftq_auth_client_destroy(client)

    def auth_client_process_batch(self, clients, client_idx, ops, peer_ids, datas, rands):
        """Initiate (op -1), ProcessResponse(op, datas[i], peer_ids[i]) (ops 0..2) and GetCipherKey (op -2) on
        clients[client_idx[i]], one call.  rands[i]: a (256 bytes, Initiate), the a' values of a completing phase-0 item, else
        b"".  (out_err int32[n], has_map uint8[n], [outputs]); the output buffer is sized from the library's out_need."""
        n = len(ops)
        blob, off = self._blob(list(datas))
        rblob, roff = self._blob(list(rands))
        tab = (C.c_void_p * max(1, len(clients)))(*[c.value for c in clients])
        idx = np.ascontiguousarray(client_idx, np.uint32) if n else np.zeros(1, np.uint32)
        op = np.ascontiguousarray(ops, np.int32) if n else np.zeros(1, np.int32)
        peers = np.ascontiguousarray(peer_ids, np.uint64) if n else np.zeros(1, np.uint64)
        out_off = np.zeros(n + 1, np.uint64)
        err = np.zeros(max(1, n), np.int32)
        has = np.zeros(max(1, n), np.uint8)
        need = C.c_uint64(0)
        cap = 0
        while True:
            out = np.zeros(max(1, cap), np.uint8)
            rc = self._lib.bftq_auth_client_process_batch(self._h, tab, len(clients), _ptr(idx), _ptr(op), _ptr(peers), _ptr(blob), _ptr(off),
                                                          _ptr(rblob), _ptr(roff), n, _ptr(err), _ptr(has), _ptr(out), cap, _ptr(out_off),
                                                          C.byref(need))
            if rc == -3 and need.value > cap:
                cap = need.value
                continue
            _lib.check(rc)
            break
        return err[:n], has[:n], [bytes(out[out_off[i]:out_off[i + 1]]) for i in range(n)]

    def lagrange_exp_product_batch(self, p: int, q: int, x, ys):
        """auth.calculateSharedSecret: prod_j ys[i][j]^lambda_j mod p.  x: (B,k) ints, ys: B lists of k ints."""
        plen, qlen = (p.bit_length() + 7) // 8, (q.bit_length() + 7) // 8
        x = np.ascontiguousarray(x, np.int32)
        B, k = x.shape
        yb = self._be([v for row in ys for v in row], plen)
        out, st = np.empty((B, plen), np.uint8), np.empty(B, np.uint8)
        pb, qb = self._be([p], plen), self._be([q], qlen)
        _lib.check(self._lib.bftq_lagrange_exp_product_batch(self._h, _ptr(pb), plen, _ptr(qb), qlen, k,
                                                             _ptr(x), _ptr(yb), B, _ptr(out), _ptr(st)))
        return [int.from_bytes(bytes(o), "big") for o in out], st

    def dsa_calculate_r_batch(self, p: int, q: int, x, ris, vis):
        """dsa.CalculateR per item over k partial results (x_i, R_i, v_i)."""
        plen, qlen = (p.bit_length() + 7) // 8, (q.bit_length() + 7) // 8
        x = np.ascontiguousarray(x, np.int32)
        B, k = x.shape
        rb = self._be([v for row in ris for v in row], plen)
        vb = self._be([v for row in vis for v in row], qlen)
        out, st = np.empty((B, qlen), np.uint8), np.empty(B, np.uint8)
        pb, qb = self._be([p], plen), self._be([q], qlen)
        _lib.check(self._lib.bftq_dsa_calculate_r_batch(self._h, _ptr(pb), plen, _ptr(qb), qlen, k,
                                                        _ptr(x), _ptr(rb), _ptr(vb), B, _ptr(out), _ptr(st)))
        return [int.from_bytes(bytes(o), "big") for o in out], st

    def ecdsa_p256_calculate_r_batch(self, x, ris, vis):
        """ecdsa.CalculateR: x (B,k) ints, ris: B lists of k 65-byte uncompressed points, vis: B lists of k ints."""
        x = np.ascontiguousarray(x, np.int32)
        B, k = x.shape
        rb = np.frombuffer(b"".join(p for row in ris for p in row), np.uint8).copy()
        vb = self._be([v for row in vis for v in row], 32)
        out, st = np.empty((B, 32), np.uint8), np.empty(B, np.uint8)
        _lib.check(self._lib.bftq_ecdsa_p256_calculate_r_batch(self._h, k, _ptr(x), _ptr(rb), _ptr(vb), B, _ptr(out), _ptr(st)))
        return [int.from_bytes(bytes(o), "big") for o in out], st

    # ---- K4 ----
    def pgp_digest_batch(self, datas, suffixes, data_idx=None, hash_alg=HASH_SHA256):
        """datas: list of bytes (TBS strings); suffixes: list of bytes (one per signature)."""
        n = len(suffixes)
        doff = np.zeros(len(datas) + 1, np.uint64)
        doff[1:] = np.cumsum([len(d) for d in datas])
        soff = np.zeros(n + 1, np.uint64)
        soff[1:] = np.cumsum([len(s) for s in suffixes])
        dblob = np.frombuffer(b"".join(datas) or b"\0", np.uint8).copy()
        sblob = np.frombuffer(b"".join(suffixes) or b"\0", np.uint8).copy()
        didx = None if data_idx is None else np.ascontiguousarray(data_idx, np.uint32)
        out = np.empty((n, DIGEST_LEN[hash_alg]), np.uint8)
        _lib.check(self._lib.bftq_pgp_digest_batch(self._h, _ptr(dblob), _ptr(doff), len(datas), _ptr(didx), _ptr(sblob), _ptr(soff),
                                                   hash_alg, n, _ptr(out)))
        return out

    def stats(self):
        s = _lib.Stats()
        _lib.check(self._lib.bftq_stats(self._h, C.byref(s)))
        return {"items": s.items, "launches": s.launches, "h2d_bytes": s.h2d_bytes, "d2h_bytes": s.d2h_bytes,
                "packer_chunks": s.packer_chunks, "packer_parse_ns": s.packer_parse_ns, "packer_stage_ns": s.packer_stage_ns,
                "packer_wait_ns": s.packer_wait_ns, "numa_node": s.numa_node, "numa_cpus": s.numa_cpus,
                "msg_gpu_items": s.msg_gpu_items, "msg_host_items": s.msg_host_items, "unsupported_items": s.unsupported_items}

    def measure_int_peak(self) -> float:
        v = C.c_double()
        _lib.check(self._lib.bftq_measure_int_peak(self._h, C.byref(v)))
        return v.value
