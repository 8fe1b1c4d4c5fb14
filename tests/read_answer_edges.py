"""Raw read answers at the edges of the device parse (K0m / K2m in bftkv_b200/csrc/msg_parse.cuh): every literal framing
Go and GnuPG write, SHA-256 block boundaries of the hashed stream, FileName nonces of every base64 shape, one-pass and
signature packet variants, and read operations whose decision hangs on exact value grouping.

build() is seeded and deterministic: the same rows, byte for byte, on every run.  Each row is a dict
  msg     the decrypted transport answer (one-pass signature, literal data, signature)
  nonce   the nonce the request carried
  pre     pre_status (non-zero: the transport failed before the answer)
  family  "A" .. "E"
  name    what the row exercises
  route   "device" (K0m decides it) or "host" (K0m flags it for the host packer)
  want    the status class pgp_oracle.read_response_status gives it (ST_OK / ST_UNVERIFIED / ST_INVALID / ST_NONCE / ST_OTHER)
and family E rows also `op` (index of their read operation) and `peer` (index into Edges.peer_ids).

The transport signature covers the literal body and the signature's hashed area, not the framing, so one signature per
(signer, body, hashed area) serves every framing of that body.  Every row whose signature verifies and whose answer is
good has a tampered twin ("<name>/tampered": one flipped bit in the body or in the signature MPI) that is ST_INVALID."""
import base64
import hashlib
import random
import struct

from bftkv_b200 import workload as W
from oracle import packet_oracle, pgp_oracle as pgp

ST_OK, ST_INVALID, ST_OTHER, ST_NONCE, ST_UNVERIFIED = pgp.ST_OK, pgp.ST_INVALID, pgp.ST_OTHER, pgp.ST_NONCE, pgp.ST_UNVERIFIED
NONCE_LENS = (1, 2, 3, 8, 23, 24)        # family C runs once per length (the nonce length is per call)
X = b"the variable"
CTIME = 0x5F000000
N_SIGNERS = 4                            # keys 0 .. 3: in the keyring, the quorum of families A - D
OUTSIDER, SUB_PRIMARY, SUB_KEY = 4, 5, 6 # a signer outside the keyring; an entity whose subkey may only encrypt
N_PEERS = 32                             # family E: a full warp of responders


# ---- keys ------------------------------------------------------------------------------------------------------------
def _is_prime(n, rng):
    for p in (3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41, 43, 47, 53, 59, 61, 67, 71, 73, 79, 83, 89, 97):
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d //= 2; s += 1
    for _ in range(8):
        x = pow(rng.randrange(2, n - 1), d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = pow(x, 2, n)
            if x == n - 1:
                break
        else:
            return False
    return True


def rsa3072_key(seed=0xBF7C3072):
    """A deterministic RSA-3072 key (e = 65537): seeded candidates + Miller-Rabin, as tests/golden/make_rsa_keys.py."""
    rng = random.Random(seed)

    def prime():
        while True:
            c = rng.getrandbits(1536) | (3 << 1534) | 1
            if (c - 1) % 65537 and _is_prime(c, rng):
                return c
    p, q = prime(), prime()
    n, e = p * q, 65537
    assert n.bit_length() == 3072
    return {"p": p, "q": q, "n": n, "e": e, "d": pow(e, -1, (p - 1) * (q - 1))}


def rsa_sign(k, digest: bytes) -> int:
    """EMSA-PKCS1-v1_5 / SHA-256 signature, by CRT (the same value as workload.raw_rsa_sign)."""
    t = W.SHA256_PREFIX + digest
    klen = (k["n"].bit_length() + 7) // 8
    m = int.from_bytes(b"\x00\x01" + b"\xff" * (klen - len(t) - 3) + b"\x00" + t, "big")
    p, q = k["p"], k["q"]
    sp, sq = pow(m, k["d"] % (p - 1), p), pow(m, k["d"] % (q - 1), q)
    return sq + q * ((sp - sq) * pow(q, -1, p) % p)


def subkey_block(k, sub, uid: bytes, ctime: int = 0x5E000000):
    """pgp_public_key_block of k plus one RSA subkey `sub` bound with key flags encrypt-only (0x0C).  -> (block, subkey id)."""
    block, kid = W.pgp_public_key_block(k, W._private_key(k), uid, ctime)
    body = bytes([4]) + struct.pack(">I", ctime) + bytes([1]) + W._mpi(k["n"]) + W._mpi(k["e"])
    sub_body = bytes([4]) + struct.pack(">I", ctime) + bytes([1]) + W._mpi(sub["n"]) + W._mpi(sub["e"])
    prefix = b"\x99" + struct.pack(">H", len(body)) + body + b"\x99" + struct.pack(">H", len(sub_body)) + sub_body
    binding = W._v4_sig_packet(W._private_key(k), kid, 0x18, prefix, ctime, extra_hashed=bytes([2, 27, 0x0C]))
    return block + W._old_packet(14, sub_body) + binding, W.pgp_key_id(sub_body)


# ---- packets ---------------------------------------------------------------------------------------------------------
def new_len(n: int, form: int) -> bytes:
    """A new-format definite length in the 1-, 2- or 5-octet form (the 5-octet form may be non-minimal)."""
    if form == 1:
        assert n < 192
        return bytes([n])
    if form == 2:
        assert 192 <= n < 8384
        return bytes([((n - 192) >> 8) + 192, (n - 192) & 0xFF])
    return b"\xff" + struct.pack(">I", n)


def sub(typ: int, data: bytes) -> bytes:
    """A signature subpacket with its length in the shortest form."""
    n = len(data) + 1
    ln = bytes([n]) if n < 192 else new_len(n, 2) if n < 8384 else new_len(n, 5)
    return ln + bytes([typ]) + data


def literal_body(name: bytes, plain: bytes) -> bytes:
    return b"b" + bytes([len(name)]) + name + b"\x00" * 4 + plain


def partial(body: bytes, exps, final_form: int = 1) -> bytes:
    """Literal data in partial-length chunks of 2^e for e in exps, then the rest as the final chunk in `final_form`."""
    out, p = bytearray([0xCB]), 0
    for e in exps:
        out.append(224 + e)
        out += body[p:p + (1 << e)]
        p += 1 << e
    assert p <= len(body)
    return bytes(out) + new_len(len(body) - p, final_form) + body[p:]


def pow2_split(n: int):
    """Exponents of the powers of two that add up to n, largest first."""
    return [e for e in range(14, -1, -1) if n >> e & 1]


class Signed:
    """A v4 RSA / SHA-256 signature over `plain` with a chosen hashed area; serialised in any header and MPI form."""

    def __init__(self, k, plain: bytes, hashed: bytes, unhashed: bytes = b"", sig_type: int = 0):
        self.head = bytes([4, sig_type, 1, 8]) + struct.pack(">H", len(hashed)) + hashed
        self.unhashed = unhashed
        signed = W.canonical_text(plain) if sig_type == 1 else plain
        self.digest = hashlib.sha256(signed + self.head + b"\x04\xff" + struct.pack(">I", len(self.head))).digest()
        self.s = rsa_sign(k, self.digest)

    def packet(self, old: bool = False, tag: bytes = None, mpi: bytes = None, flip_mpi: bool = False) -> bytes:
        m = bytearray(mpi if mpi is not None else W._mpi(self.s))
        if flip_mpi:
            m[-1] ^= 0x01
        body = self.head + struct.pack(">H", len(self.unhashed)) + self.unhashed + (tag if tag is not None else self.digest[:2]) + bytes(m)
        return W._old_packet(2, body) if old else W._new_packet(2, body)


def go_hashed(kid: int) -> bytes:
    """x/crypto's hashed area: creation time and issuer."""
    return sub(2, struct.pack(">I", CTIME)) + sub(16, struct.pack(">Q", kid))


def one_pass(kid: int, old: bool = False, sig_type: int = 0, hash_id: int = 8, is_last: int = 1) -> bytes:
    body = bytes([3, sig_type, hash_id, 1]) + struct.pack(">Q", kid) + bytes([is_last])
    return (b"\x90\x0d" if old else b"\xc4\x0d") + body


# ---- the builder -----------------------------------------------------------------------------------------------------
class Edges:
    def __init__(self, seed: int = 0xBF7C00E0):
        self.rng = random.Random(seed)
        self.keys = W.load_keys(N_PEERS)
        blocks, self.kids = [], []
        for i in range(SUB_KEY + 1):
            b, kid = W.pgp_public_key_block(self.keys[i], W._private_key(self.keys[i]), b"e%02d <e%02d@bftq.test>" % (i, i))
            blocks.append(b); self.kids.append(kid)
        for i in range(SUB_KEY + 1, N_PEERS):        # family E's other responders: ids only (signers come from keys 0 .. 3)
            self.kids.append(W.pgp_key_id(bytes([4]) + struct.pack(">I", 0x5E000000) + bytes([1]) + W._mpi(self.keys[i]["n"]) + W._mpi(self.keys[i]["e"])))
        sub_block, self.sub_kid = subkey_block(self.keys[SUB_PRIMARY], self.keys[SUB_KEY], b"sub <sub@bftq.test>")
        self.big = rsa3072_key()
        big_block, self.big_kid = W.pgp_public_key_block(self.big, W._private_key(self.big), b"big <big@bftq.test>")
        self.keyring = b"".join(blocks[:N_SIGNERS]) + sub_block + big_block
        self.peer_ids = list(self.kids)
        self.rows = []
        self._sigs = {}
        self.family_a(); self.family_b(); self.family_c(); self.family_d(); self.family_e()

    # -- helpers
    def nonce(self, n: int = 8) -> bytes:
        return bytes(self.rng.randrange(256) for _ in range(n))

    def signed(self, signer, plain: bytes, hashed: bytes = None, unhashed: bytes = b"") -> Signed:
        k, kid = self.signer_key(signer)
        hashed = go_hashed(kid) if hashed is None else hashed
        key = (signer, plain, hashed, unhashed)
        if key not in self._sigs:
            self._sigs[key] = Signed(k, plain, hashed, unhashed)
        return self._sigs[key]

    def signer_key(self, signer):
        if signer == "big":
            return self.big, self.big_kid
        if signer == "sub":
            return self.keys[SUB_KEY], self.sub_kid
        return self.keys[signer], self.kids[signer]

    def add(self, family, name, route, want, msg, nonce, pre=0, **kw):
        self.rows.append(dict(family=family, name=name, route=route, want=want, msg=bytes(msg), nonce=nonce, pre=pre, **kw))

    def answer(self, family, name, plain, frame=lambda L: b"\xcb" + new_len(len(L), 5) + L, signer=0, route="device", want=ST_OK,
               nonce=None, file_name=None, ops=None, sig=None, sig_kw=None, tail=b"", twin=True, **kw):
        """One answer (and its tampered twin when `twin` and the answer is good): one-pass | frame(literal body) | signature | tail."""
        nonce = self.nonce() if nonce is None else nonce
        file_name = base64.b64encode(nonce) if file_name is None else file_name
        kid = self.signer_key(signer)[1]
        ops = one_pass(kid) if ops is None else ops
        sig = self.signed(signer, plain) if sig is None else sig
        sk = sig_kw or {}
        msg = ops + frame(literal_body(file_name, plain)) + sig.packet(**sk) + tail
        self.add(family, name, route, want, msg, nonce, **kw)
        if twin and want == ST_OK:
            if plain and self.rng.random() < 0.5:
                bad = bytearray(plain)
                bad[self.rng.randrange(len(bad))] ^= 1 << self.rng.randrange(8)
                msg = ops + frame(literal_body(file_name, bytes(bad))) + sig.packet(**sk) + tail
            else:
                msg = ops + frame(literal_body(file_name, plain)) + sig.packet(flip_mpi=True, **sk) + tail
            self.add(family, name + "/tampered", route, ST_INVALID, msg, nonce, **kw)

    def value(self, n: int) -> bytes:
        return bytes(self.rng.randrange(256) for _ in range(n))

    # -- A: literal framing
    def family_a(self):
        small = packet_oracle.serialize(X, self.value(40), 11)            # literal body < 192
        mid = packet_oracle.serialize(X, self.value(700), 12)             # 2-octet lengths
        big = packet_oracle.serialize(X, self.value(33000), 13)           # above 2^15: room for every chunk size
        hl = 2 + 12 + 4                                                   # format, name length, 12 name bytes, time
        for i, (plain, form) in enumerate([(small, 1), (mid, 2), (big, 5), (small, 5)]):
            self.answer("A", "new-definite/%d-octet%s" % (form, "/non-minimal" if i == 3 else ""), plain,
                        lambda L, f=form: b"\xcb" + new_len(len(L), f) + L, signer=i % N_SIGNERS)
        for plain, nl, name in [(small, 1, "0xAC"), (mid, 2, "0xAD"), (big, 4, "0xAE"), (small, 4, "0xAE/non-minimal")]:
            self.answer("A", "old-definite/" + name, plain, lambda L, nl=nl: bytes([0xAC | {1: 0, 2: 1, 4: 2}[nl]]) + len(L).to_bytes(nl, "big") + L)
        self.answer("A", "old-indeterminate/0xAF", small, lambda L: b"\xaf" + L, route="host", want=ST_INVALID)
        # with an unknown signer nothing behind the literal is read: the signature packet ends up in the body, and packet.Parse fails
        self.answer("A", "old-indeterminate/0xAF/unknown-signer", small, lambda L: b"\xaf" + L, signer=OUTSIDER, route="host", want=ST_OTHER)
        # partial chunks of every size 2^0 .. 2^14, rising and falling, and Go's writer shape
        self.answer("A", "partial/rising-2^0..2^14", big, lambda L: partial(L, list(range(15)), 2))
        self.answer("A", "partial/falling-2^14..2^0", big, lambda L: partial(L, list(range(14, -1, -1)), 5))
        self.answer("A", "partial/go-writer", mid, lambda L: b"\xcb" + W.go_partial_write(L) + b"\x00")
        # the literal header split at every byte: 1-byte chunks up to the split, then the rest
        for s in range(1, hl + 1):
            self.answer("A", "partial/header-split-%02d" % s, mid, lambda L, s=s: partial(L, [0] * s + [9], 2))
        # a chunk of >= 128 bytes starting at every offset 1 .. 63 of a hash block: the fast path re-enters inside it
        for r in range(1, 64):
            self.answer("A", "partial/fast-path-reentry-%02d" % r, mid,
                        lambda L, r=r: partial(L, pow2_split(hl + r) + [7 + (r & 1)], 2), signer=r % N_SIGNERS, twin=r % 8 == 1)
        # the final chunk: empty, 1-, 2- and 5-octet lengths
        self.answer("A", "partial/final-empty", mid, lambda L: partial(L, pow2_split(len(L)), 1))
        self.answer("A", "partial/final-1-octet", mid, lambda L: partial(L, [9, 7], 1))
        self.answer("A", "partial/final-2-octet", mid, lambda L: partial(L, [8], 2))
        self.answer("A", "partial/final-5-octet", mid, lambda L: partial(L, [8, 6], 5))
        self.answer("A", "partial/final-5-octet-empty", mid, lambda L: partial(L, pow2_split(len(L)), 5))
        # the body at every alignment mod 4 inside the answer: CR / LF in the FileName lengthen the header
        for extra in range(4):
            n = self.nonce()
            name = base64.b64encode(n) + b"\r\n\n"[:extra]
            for fr, frame in [("new", lambda L: b"\xcb" + new_len(len(L), 2) + L), ("old", lambda L: b"\xad" + len(L).to_bytes(2, "big") + L),
                              ("partial", lambda L: partial(L, [9], 2))]:
                self.answer("A", "align/%s/+%d" % (fr, extra), mid, frame, nonce=n, file_name=name)
        # framing that runs off the message
        ops, lit = one_pass(self.kids[0]), partial(literal_body(base64.b64encode(bytes(8)), mid), [9], 2)
        self.add("A", "off-end/partial-chunk-longer-than-rest", "host", ST_OTHER, ops + lit[:300], bytes(8))
        at = len(ops) + 1 + 512 + 1                                      # CB, E9, 512 bytes: the final chunk's 2-octet length
        self.add("A", "off-end/cut-in-2-octet-length", "host", ST_OTHER, (ops + lit)[:at + 1], bytes(8))
        cut5 = ops + partial(literal_body(base64.b64encode(bytes(8)), mid), [9], 5)
        for j in range(1, 5):
            self.add("A", "off-end/cut-in-5-octet-length-%d" % j, "host", ST_OTHER, cut5[:at + j], bytes(8))
        self.add("A", "off-end/old-definite-longer-than-rest", "host", ST_OTHER, ops + b"\xad\x40\x00" + literal_body(base64.b64encode(bytes(8)), mid), bytes(8))
        for signer, want in [(0, ST_INVALID), (OUTSIDER, ST_UNVERIFIED)]:
            n = self.nonce()
            kid = self.kids[signer]
            for fr, frame in [("new", lambda L: b"\xcb" + new_len(len(L), 2) + L), ("partial", lambda L: partial(L, [9], 2))]:
                self.add("A", "off-end/no-signature/%s/%s" % (fr, "known" if signer == 0 else "unknown"), "host", want,
                         one_pass(kid) + frame(literal_body(base64.b64encode(n), mid)), n)
        # the transport failed before the answer: K0m passes pre_status through
        self.add("A", "pre-status/empty", "device", ST_OTHER, b"", bytes(8), pre=6)
        n = self.nonce()
        good = one_pass(self.kids[1]) + b"\xcb" + new_len(len(literal_body(base64.b64encode(n), small)), 1) + literal_body(base64.b64encode(n), small) + self.signed(1, small).packet()
        self.add("A", "pre-status/good-answer", "device", ST_OTHER, good, n, pre=6)

    # -- B: hash-block boundaries
    def family_b(self):
        # body + hashed area + 6: the go_hashed area is 22 bytes with the version octets, so the stream is 64 + len(v) long
        base = self.value(100 + 63)
        for r in range(64):
            v = base[:100 + r]
            plain = packet_oracle.serialize(X, v, 100 + r)
            self.answer("B", "residue-%02d/fast" % ((len(plain) + 28) % 64), plain, signer=r % N_SIGNERS, twin=r % 4 == 0)
            self.answer("B", "residue-%02d/no-fast" % ((len(plain) + 28) % 64), plain, lambda L: partial(L, [5] * (len(L) // 32), 1),
                        signer=r % N_SIGNERS, twin=r % 4 == 2)
        for n in (0, 1, 63, 64, 65, 4095, 4096, 4097, 16 * 1024 + 300):
            plain = b"" if n == 0 else b"\x00" if n == 1 else packet_oracle.serialize(b"", self.value(n - 24), n)
            assert len(plain) == n
            self.answer("B", "body-%d" % n, plain, want=ST_OTHER if n == 1 else ST_OK, signer=n % N_SIGNERS)
        plain = packet_oracle.serialize(X, self.value(200), 21)
        for extra in (20, 41, 42, 43, 58, 64, 100, 190, 191, 300, 1000):
            hashed = go_hashed(self.kids[extra % N_SIGNERS]) + sub(100, self.value(extra))
            sig = self.signed(extra % N_SIGNERS, plain, hashed)
            self.answer("B", "long-hashed-area-%d" % extra, plain, signer=extra % N_SIGNERS, sig=sig)
            self.answer("B", "long-hashed-area-%d/no-fast" % extra, plain, lambda L: partial(L, [5] * (len(L) // 32), 1),
                        signer=extra % N_SIGNERS, sig=sig, twin=False)

    # -- C: the FileName nonce, once per nonce length
    def family_c(self):
        plain = packet_oracle.serialize(X, self.value(60), 31)
        for nl in NONCE_LENS:

            def row(name, file_name, want, nonce, route=None, **kw):
                route = route or ("device" if len(file_name) <= 32 else "host")
                self.answer("C", "n%d/%s" % (nl, name), plain, nonce=nonce, file_name=file_name, want=want, route=route,
                            signer=len(self.rows) % N_SIGNERS, nonce_len=nl, **kw)
            n = self.nonce(nl)
            b = base64.b64encode(n)
            row("plain", b, ST_OK, n)
            row("name-empty", b"", ST_NONCE, n)
            pad32 = b + b"\n" * (32 - len(b))
            row("name-32", pad32, ST_OK, n)
            row("name-33", pad32 + b"\r", ST_OK, n)
            for i in range(len(b) + 1):
                row("crlf-at-%02d" % i, b[:i] + (b"\r" if i % 2 else b"\n") + b[i:], ST_OK, n, twin=i % 5 == 0)
            row("crlf-everywhere", b"\r\n".join(bytes([c]) for c in b), ST_OK, n)
            row("bad-char", b[:-1] + b"*" if not b.endswith(b"=") else b"*" + b[1:], ST_OTHER, n)
            row("bad-char-dot", b[:1] + b"." + b[2:], ST_OTHER, n)
            q0 = len(b) - 4
            row("eq-at-quad-0", b[:q0] + b"====", ST_OTHER, n)
            row("eq-at-quad-1", b[:q0] + b[q0:q0 + 1] + b"===", ST_OTHER, n)
            row("data-after-padding", b + b"AA==" if b.endswith(b"=") else b + b"=", ST_OTHER, n)
            row("bare-quad-after-padding", b + b"AAAA", ST_OTHER if b.endswith(b"=") else ST_NONCE, n)
            row("unpadded-tail", b.rstrip(b"=") if b.endswith(b"=") else b[:-1], ST_OTHER, n)
            row("unpadded-tail-crlf", (b.rstrip(b"=") if b.endswith(b"=") else b[:-1]) + b"\r\n", ST_OTHER, n)
            if b.endswith(b"==") :
                row("xx=-then-A", b[:-1] + b"A", ST_OTHER, n)
                row("xx=-then-crlf-then-A", b[:-1] + b"\r\nA", ST_OTHER, n)
                row("xx=-crlf-=", b[:-1] + b"\r\n=", ST_OK, n)
                row("xx=-at-end", b[:-1], ST_OTHER, n)
            if b.endswith(b"="):
                row("padding-then-crlf", b + b"\n\r", ST_OK, n)
            # the bits a padded tail leaves unused: Go does not check them
            if nl % 3:
                j = len(b) - (3 if nl % 3 == 1 else 2)
                c = pgp._B64[(pgp._B64.index(b[j:j + 1]) | (15 if nl % 3 == 1 else 3))]
                row("trailing-bits", b[:j] + bytes([c]) + b[j + 1:], ST_OK, n)
            other = n[:-1] if nl > 1 else n + b"\x00"
            row("wrong-length", base64.b64encode(other), ST_NONCE, n)
            row("wrong-bytes", base64.b64encode(bytes([n[0] ^ 1]) + n[1:]), ST_NONCE, n)
            # which error wins: the base64 error before the signature verdict, the signature verdict before the nonce
            sig_kw = {"flip_mpi": True}
            row("corrupt-and-bad-signature", b"*" + b[1:], ST_OTHER, n, sig_kw=sig_kw)
            row("mismatch-and-bad-signature", base64.b64encode(other), ST_INVALID, n, sig_kw=sig_kw)
            row("mismatch-unknown-signer", base64.b64encode(other), ST_NONCE, n, ops=one_pass(self.kids[OUTSIDER]))

    # -- D: one-pass and signature packets
    def family_d(self):
        plain = packet_oracle.serialize(X, self.value(80), 41)
        s = self.signed(0, plain)
        self.answer("D", "one-pass-old-format", plain, ops=one_pass(self.kids[0], old=True))
        self.answer("D", "one-pass-not-last", plain, ops=one_pass(self.kids[0], is_last=0), route="host", want=ST_OTHER, twin=False)
        text = packet_oracle.serialize(X, b"line one\nline two\r\n", 41)
        ts = Signed(self.keys[0], text, go_hashed(self.kids[0]), sig_type=1)
        self.answer("D", "one-pass-text-mode", text, ops=one_pass(self.kids[0], sig_type=1), sig=ts, route="host", want=ST_OK, twin=False)
        self.answer("D", "one-pass-hash-sha512", plain, ops=one_pass(self.kids[0], hash_id=10), route="host", want=ST_INVALID)
        self.answer("D", "one-pass-hash-sha224", plain, ops=one_pass(self.kids[0], hash_id=11), route="host", want=ST_INVALID)
        self.answer("D", "signature-old-format", plain, sig_kw={"old": True})
        sig = self.signed(1, plain, sub(2, struct.pack(">I", CTIME)), sub(16, struct.pack(">Q", self.kids[1])))
        self.answer("D", "issuer-unhashed-only", plain, signer=1, sig=sig)
        sig = self.signed(2, plain, sub(2, struct.pack(">I", CTIME)))
        self.answer("D", "no-issuer", plain, signer=2, sig=sig, route="host", want=ST_OK, twin=False)
        # a signature MPI shorter than the key: grind the creation time until s < 2^2040
        for t in range(CTIME, CTIME + 100000):
            sg = self.signed(3, plain, sub(2, struct.pack(">I", t)) + sub(16, struct.pack(">Q", self.kids[3])))
            if sg.s < 1 << 2040:
                break
            del self._sigs[(3, plain, sub(2, struct.pack(">I", t)) + sub(16, struct.pack(">Q", self.kids[3])), b"")]
        assert len(W._mpi(sg.s)) <= 2 + 255
        self.answer("D", "short-mpi", plain, signer=3, sig=sg)
        self.answer("D", "mpi-longer-than-key", plain, sig=s, sig_kw={"mpi": struct.pack(">H", 2056) + b"\x00" + s.s.to_bytes(256, "big")}, want=ST_INVALID)
        self.answer("D", "hash-tag-mismatch", plain, sig=s, sig_kw={"tag": bytes([s.digest[0] ^ 0x80, s.digest[1]])}, want=ST_INVALID)
        self.answer("D", "trailing-bytes", plain, tail=b"\x00\x01", route="host")
        self.answer("D", "unknown-packet-before-signature", plain, frame=lambda L: b"\xcb" + new_len(len(L), 5) + L + b"\xfc\x03abc", route="host")
        self.answer("D", "signer-unknown", plain, signer=OUTSIDER, want=ST_UNVERIFIED)
        self.answer("D", "signer-encryption-only-subkey", plain, signer="sub", want=ST_UNVERIFIED)
        self.answer("D", "signer-rsa-3072", plain, signer="big", route="host")

    # -- E: K2m's grouping and decision; rows carry their operation and responder
    def family_e(self):
        self.e_ops = 0

        def op(responses):
            """responses: (peer index, body, signer, literal framing or None, route, bytes after the signature)"""
            for peer, plain, signer, frame, route, tail in responses:
                want = ST_OTHER if not parses(plain) else ST_OK if signer != OUTSIDER else ST_UNVERIFIED
                if frame is None:
                    frame = lambda L: b"\xcb" + new_len(len(L), 5) + L
                self.answer("E", "op%02d/%02d" % (self.e_ops, peer), plain, frame, signer=signer, route=route, want=want, tail=tail,
                            twin=False, op=self.e_ops, peer=peer)
            self.e_ops += 1
        v = self.value(48)
        A, B, C = (packet_oracle.serialize(X, v + bytes([i]), 50) for i in range(3))
        # 32 responders: ten each of three values that differ only in their last byte, one failure, then the eleventh A
        seq = [A, B, C] * 10
        fail = packet_oracle.serialize(X, v, 50)[:-1]                  # packet.Parse fails
        resp = [(i, p, i % N_SIGNERS, None, "device", b"") for i, p in enumerate(seq)] + [(30, fail, 2, None, "device", b""), (31, A, 3, None, "device", b"")]
        op(resp)
        op([])                                                            # no responders
        # an empty value and a packet that ends before its value bucket together as ("", 0)
        empty, short = packet_oracle.serialize(X, b"", 0), packet_oracle.serialize(X)
        op([(i, empty if i % 2 else short, i % N_SIGNERS, None, "device", b"") for i in range(11)])
        # the same value at two timestamps: no bucket reaches the threshold
        v1, v2 = packet_oracle.serialize(X, v, 60), packet_oracle.serialize(X, v, 61)
        op([(i, v1 if i % 2 else v2, i % N_SIGNERS, None, "device", b"") for i in range(20)])
        # t = 0 and t = 2^64 - 1
        lo, hi = packet_oracle.serialize(X, v, 0), packet_oracle.serialize(X, v, (1 << 64) - 1)
        op([(i, lo, i % N_SIGNERS, None, "device", b"") for i in range(5)] + [(i, hi, i % N_SIGNERS, None, "device", b"") for i in range(5, 16)])
        op([(i, hi if i < 6 else lo, i % N_SIGNERS, None, "device", b"") for i in range(17)])
        # one value from host-route and device-route answers alike (two value buffers behind the pointers)
        same = packet_oracle.serialize(X, self.value(300), 70)
        op([(i, same, i % N_SIGNERS, None, "host" if i % 2 else "device", b"\x00" if i % 2 else b"") for i in range(11)])
        op([(i, same, OUTSIDER if i % 3 == 0 else i % N_SIGNERS, lambda L: partial(L, [5] * (len(L) // 32), 1) if i % 2 else None,
             "host" if i % 4 == 1 else "device", b"\x00" if i % 4 == 1 else b"") for i in range(12)])
        # unknown signers alone decide
        op([(i, A, OUTSIDER, None, "device", b"") for i in range(11)])

    # -- views
    def family_rows(self, family, nonce_len=None):
        return [r for r in self.rows if r["family"] == family and (nonce_len is None or r.get("nonce_len", 8) == nonce_len)]


def parses(plain: bytes) -> bool:
    """processResponse accepts the body: empty, or packet.Parse succeeds."""
    try:
        return not plain or packet_oracle.parse(plain) is not None
    except (EOFError, ValueError, struct.error):
        return False


_CACHE = {}


def build(seed: int = 0xBF7C00E0) -> Edges:
    if seed not in _CACHE:
        _CACHE[seed] = Edges(seed)
    return _CACHE[seed]
