"""Encrypted transport messages at the edges of the decryption layer (K6a rsa_crt_decrypt_kernel, K6b seipd_decrypt_kernel
and the read path's front stage K6p / K6q in bftkv_b200/csrc/msg_decrypt.cuh).

build() is seeded and deterministic.  Each row is a dict
  family  "A" K6a arithmetic, "B" unpadding and split, "C" SEIPD lengths and framing, "D" candidate order
  name    what the row exercises
  raw     the encrypted message
  want    the BFTQ_ERR_* code Go's PGPMessage.Decrypt ends with (pgp_encrypt_ref.message_decrypt restates it), or None
          when the row's code is by definition that of row `same_as` (a wrong session key taken: the code of its garbage)
  preds   [(statement, bool)]: the property the row exists for, evaluated on the construction
  plain, nonce   what a code-0 row decrypts to (from the construction)
  inner   the signed stream inside the SEIPD (None where there is none)
  shape   exactly one PKESK and one SEIPD of at least 40 body bytes: the shape the encrypted read path takes on the device
  host    the encrypted read path hands the answer to the host: K6b finds its MDC wrong, or K0m cannot parse its inner stream
Every key of families A and B is one of KEYS: fixture keys 0 (p < q) and 5 (p > q), and the fixture keys L (p / q ~ 1/2) and
H (p / q ~ 2) of tests/golden/decrypt_edges.json."""
import base64
import hashlib
import json
import os
import random
import struct

from bftkv_b200 import workload as W
from oracle import packet_oracle
import pgp_encrypt_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "decrypt_edges.json")
KEYS = ("0", "5", "L", "H")
SIGNER = 1                                   # fixture key 1 signs every inner stream
X = b"the variable"
CTIME = 0x5F000000
KS = {7: 16, 8: 24, 9: 32}
TOP = 1 << 2032                              # a type-2 block lies in [2 TOP, 3 TOP)


def load_fixture():
    d = json.load(open(FIXTURE))
    keys = {}
    for name, k in d["keys"].items():
        p, q = int(k["p"], 16), int(k["q"], 16)
        keys[name] = {"p": p, "q": q, "n": p * q, "e": d["e"], "d": pow(d["e"], -1, (p - 1) * (q - 1))}
    coll = [{"cipher": c["cipher"], "key": bytes.fromhex(c["key"]), "prefix": bytes.fromhex(c["prefix"]), "wrong": bytes.fromhex(c["wrong"])}
            for c in d["collisions"]]
    return keys, coll


def secret_key_packet(k, tag: int = 5, u: int = None, ctime: int = 0x5E000000) -> bytes:
    """An unprotected RSA secret-key packet (tag 5 or 7) with the CRT coefficient `u` (default p^-1 mod q) and a correct
    checksum."""
    pub = bytes([4]) + struct.pack(">I", ctime) + bytes([1]) + W._mpi(k["n"]) + W._mpi(k["e"])
    sec = W._mpi(k["d"]) + W._mpi(k["p"]) + W._mpi(k["q"]) + W._mpi(pow(k["p"], -1, k["q"]) if u is None else u)
    return W._new_packet(tag, pub + bytes([0]) + sec + struct.pack(">H", sum(sec) & 0xFFFF))


# ---- packets ---------------------------------------------------------------------------------------------------------
def pkesk_c(kid: int, c: int, mpi: bytes = None) -> bytes:
    return W._new_packet(1, bytes([3]) + struct.pack(">Q", kid) + bytes([1]) + (W._mpi(c) if mpi is None else mpi))


def enc(k, em: bytes) -> int:
    return pow(int.from_bytes(em, "big"), k["e"], k["n"])


def definite(n: int, form: int) -> bytes:
    if form == 1:
        return bytes([n])
    if form == 2:
        return bytes([((n - 192) >> 8) + 192, (n - 192) & 0xFF])
    return b"\xff" + struct.pack(">I", n)


def seipd_body(key: bytes, inner: bytes, prefix: bytes) -> bytes:
    """The SEIPD body after its version byte: CFB over prefix | its last two bytes | inner | MDC packet."""
    pre = prefix + prefix[14:16]
    return R.cfb_encrypt(key, pre + inner + b"\xd3\x14" + hashlib.sha1(pre + inner + b"\xd3\x14").digest())


def seipd_packet(ct: bytes, form: int = 0) -> bytes:
    """Tag 18 around version 1 | ct: Go's partial lengths (form 0) or a definite length in the 1-, 2- or 5-octet form."""
    data = b"\x01" + ct
    if form == 0:
        return b"\xd2" + W.go_partial_write(data) + b"\x00"
    return b"\xd2" + definite(len(data), form) + data


def session_block(cipher: int, key: bytes, bad_sum: bool = False) -> bytes:
    return bytes([cipher]) + key + struct.pack(">H", (sum(key) ^ bad_sum) & 0xFFFF)


def type2(rng, msg: bytes) -> bytes:
    return R.pkcs1_type2(rng, msg)


def block_with_residue(rng, prime: int, r: int, tail: bytes) -> bytes:
    """A valid type-2 block ending in `tail` (the zero separator and the message) whose integer m has m = r mod prime.  CRT
    of m = tail mod 2^(8 len(tail)) and m = r mod prime gives x; m = x + j 2^(8 len(tail)) prime for a random j that puts m
    in [2 TOP, 3 TOP), redrawn until the padding bytes are all non-zero (about 40 % of draws are)."""
    M = 1 << (8 * len(tail))
    t = int.from_bytes(tail, "big")
    x = t + M * ((r - t) * pow(M, -1, prime) % prime)
    step = M * prime
    j0 = (2 * TOP - x + step - 1) // step
    while True:
        m = x + step * (j0 + rng.randrange(TOP // step - 1))
        assert 2 * TOP <= m < 3 * TOP
        em = m.to_bytes(256, "big")
        if 0 not in em[2:256 - len(tail)]:
            return em


# ---- the builder -----------------------------------------------------------------------------------------------------
class Edges:
    def __init__(self, seed: int = 0xBF7C06E0):
        self.rng = random.Random(seed)
        fix = W.load_keys(6)
        extra, self.collisions = load_fixture()
        self.keys = {"0": fix[0], "5": fix[5], "L": extra["L"], "H": extra["H"]}
        self.blocks, self.ids = {}, {}
        for name, k in self.keys.items():
            self.blocks[name], self.ids[name] = W.pgp_public_key_block(k, W._private_key(k), b"edge-%s <%s@bftq.test>" % (name.encode(), name.encode()))
        self.signer = fix[SIGNER]
        self.signer_block, self.signer_id = W.pgp_public_key_block(self.signer, W._private_key(self.signer), b"signer <s@bftq.test>")
        self.rows = []
        self.inners = [self.inner(140 + 37 * i) for i in range(6)]
        self.family_a(); self.family_b(); self.family_c(); self.family_d()

    # -- helpers
    def inner(self, vlen: int):
        """(inner stream, plain, nonce): a signed transport message around a bftkv value of vlen bytes.  The literal packet
        has a 2-octet definite length, so the stream's length grows by one with each value byte."""
        plain = packet_oracle.serialize(X, self.rng.randbytes(vlen), 7)
        nonce = self.rng.randbytes(8)
        name = base64.b64encode(nonce)
        lit = W._new_packet(11, b"b" + bytes([len(name)]) + name + bytes(4) + plain)
        assert 192 <= len(lit) - 3 < 8384
        s = W.one_pass_packet(0, 8, 1, self.signer_id) + lit + W.go_signature_packet(self.signer, self.signer_id, 8, plain, CTIME)
        return s, plain, nonce

    def add(self, family, name, raw, want, preds=(), inner=None, shape=False, host=False, same_as=None):
        self.rows.append(dict(family=family, name=name, raw=bytes(raw), want=want, preds=list(preds),
                              plain=inner[1] if inner and want == 0 else None, nonce=inner[2] if inner and want == 0 else None,
                              inner=inner[0] if inner else None, shape=shape, host=host, same_as=same_as))

    def session(self, cipher):
        return self.rng.randbytes(KS[cipher])

    def message(self, key, inner, pkesks, form=0):
        return b"".join(pkesks) + seipd_packet(seipd_body(key, inner[0], self.rng.randbytes(16)), form)

    def pick(self):
        return self.inners[self.rng.randrange(len(self.inners))]

    # -- A: K6a's arithmetic.  Code 0 with the exact plain text shows that every key byte came back.
    def family_a(self):
        for kn in KEYS:
            k, kid = self.keys[kn], self.ids[kn]
            p, q, n = k["p"], k["q"], k["n"]

            def good(name, em, cipher, key, preds, mpi=None):
                c = enc(k, em)
                inner = self.pick()
                self.add("A", "%s/%s/aes%d" % (kn, name, KS[cipher] * 8), self.message(key, inner, [pkesk_c(kid, c, mpi)]), 0, preds, inner,
                         shape=True)
            for cipher in (7, 8, 9):
                key = self.session(cipher)
                tail = b"\x00" + session_block(cipher, key)
                for pn, prime in (("p", p), ("q", q)):
                    for r, rn in ((0, "0"), (prime - 1, "-1")):
                        em = block_with_residue(self.rng, prime, r, tail)
                        good("m=%s-mod-%s" % (rn, pn), em, cipher, key, [("m %% %s == %s" % (pn, rn), int.from_bytes(em, "big") % prime == r)])
            if p > q:                                  # Garner's a = m1 - q
                for i in range(8):
                    cipher = (7, 8, 9)[i % 3]
                    key = self.session(cipher)
                    em = block_with_residue(self.rng, p, q + self.rng.randrange(p - q), b"\x00" + session_block(cipher, key))
                    good("m-mod-p>=q/%d" % i, em, cipher, key, [("(m % p) >= q", int.from_bytes(em, "big") % p >= q)])
            for want_lt in (True, False):
                while True:
                    cipher = self.rng.choice((7, 8, 9))
                    key = self.session(cipher)
                    em = type2(self.rng, session_block(cipher, key))
                    m = int.from_bytes(em, "big")
                    if (m % q < m % p) == want_lt:
                        break
                good("m-mod-q<m-mod-p" if want_lt else "m-mod-q>=m-mod-p", em, cipher, key,
                     [("(m % q) < (m % p)" if want_lt else "(m % q) >= (m % p)", (m % q < m % p) == want_lt)])
            while True:                                # c < 2^2040: an MPI shorter than the modulus
                cipher = self.rng.choice((7, 8, 9))
                key = self.session(cipher)
                em = type2(self.rng, session_block(cipher, key))
                c = enc(k, em)
                if c < 1 << 2040:
                    break
            good("short-mpi", em, cipher, key, [("c < 2^2040", c < 1 << 2040)])
            mpi = struct.pack(">H", 2048) + c.to_bytes(256, "big")
            good("mpi-leading-zero-byte", em, cipher, key, [("MPI bit count 2048 over a leading zero byte", mpi[2] == 0)], mpi=mpi)
            # statuses only: these blocks are not valid type-2 blocks (or c > n), so no key comes back
            for name, c in (("0", 0), ("1", 1), ("n-1", n - 1), ("n", n), ("n+1", n + 1), ("p", p), ("q", q), ("2p", 2 * p),
                            ("m=2", pow(2, k["e"], n))):
                m = pow(c, k["d"], n) if c <= n else None
                key = self.session(7)
                self.add("A", "%s/c=%s" % (kn, name), self.message(key, self.pick(), [pkesk_c(kid, c)]), -8,
                         [("c > n or m is no type-2 block", m is None or m >> 2032 != 2)], shape=True)

    # -- B: decryptPKCS1v15's checks and EncryptedKey.Decrypt's split.  Each edge block is followed by a good PKESK to
    # the same key: a block the unpadding rejects is passed over (code 0), one it accepts decides the message.
    def family_b(self):
        for kn in KEYS:
            k, kid = self.keys[kn], self.ids[kn]
            inner = self.pick()

            def row(name, em, want, preds, right_key=None):
                cipher = 7
                key = right_key or self.session(cipher)
                right = pkesk_c(kid, enc(k, type2(self.rng, session_block(cipher, key))))
                self.add("B", "%s/%s" % (kn, name), self.message(key, inner, [pkesk_c(kid, enc(k, em)), right]), want, preds, inner)

            def nz(n):
                return bytes(self.rng.randrange(1, 256) for _ in range(n))

            def sep_at(i, msg=None, head=b"\x00\x02"):
                msg = nz(255 - i) if msg is None else msg
                return head + nz(i - 2) + b"\x00" + msg
            for i in (2, 9, 10, 11):
                em = sep_at(i)
                row("separator-at-%d" % i, em, 0 if i < 10 else -8, [("first zero after em[1] at %d" % i, em.index(0, 2) == i)])
            em = b"\x00\x02" + nz(254)
            row("no-separator", em, 0, [("no zero after em[1]", 0 not in em[2:])])
            for h in (b"\x01\x02", b"\x00\x01", b"\x00\x03"):
                em = sep_at(20, head=h)
                row("em[0:2]=%s" % h.hex(), em, 0, [("em[0:2] == %s" % h.hex(), em[:2] == h)])
            for ln in (0, 1, 2, 3):
                em = sep_at(255 - ln)
                row("message-length-%d" % ln, em, -8, [("len(message) == %d" % ln, len(em) - 1 - em.index(0, 2) == ln)])
            for cipher in (7, 8, 9):
                key = self.session(cipher)
                for cb in (7, 8, 9):
                    em = type2(self.rng, session_block(cb, key))
                    # a matching block is taken: its key must be the SEIPD's, so the good PKESK carries the same key
                    row("cipher-%d-key-%d" % (cb, len(key)), em, 0 if cb == cipher else -8,
                        [("key length %d, cipher %d" % (len(key), cb), len(em) - em.index(0, 2) - 4 == len(key))], right_key=key)
            for cb, kl in ((2, 24), (3, 16)):
                em = type2(self.rng, session_block(cb, self.rng.randbytes(kl)))
                row("cipher-%d-3des-cast5" % cb, em, -11, [("cipher byte %d" % cb, em[em.index(0, 2) + 1] == cb)])
            for kl in (33, 34, 242):
                em = type2(self.rng, session_block(9, nz(kl)))
                row("cipher-9-key-%d" % kl, em, -8, [("key length %d" % kl, len(em) - em.index(0, 2) - 4 == kl)])
            key = self.session(7)
            em = type2(self.rng, session_block(7, key, bad_sum=True))
            row("bad-checksum", em, 0, [("checksum != sum(key)", struct.unpack(">H", em[-2:])[0] != sum(key) & 0xFFFF)], right_key=key)

    # -- C: K6b over every hashed length mod 64 (SHA-1's padding spills into an extra block at 56), every CFB residue,
    # the shortest bodies and every framing of the SEIPD packet
    def family_c(self):
        kn = "H"
        k, kid = self.keys[kn], self.ids[kn]
        sweep, seen, base = [], set(), 0
        for v in range(200, 400):                                   # each value byte adds one, a short signature MPI takes one
            s = self.inner(v)
            base = max(base, len(s[0]) - (v - 200))
            if (len(s[0]) + 20) % 64 not in seen:
                seen.add((len(s[0]) + 20) % 64)
                sweep.append(s)
            if len(seen) == 64:
                break
        assert len(seen) == 64
        for cipher in (7, 8, 9):
            for s in sweep:
                key = self.session(cipher)
                H = 18 + len(s[0]) + 2                    # prefix | inner | D3 14: what the MDC hashes
                raw = pkesk_c(kid, enc(k, type2(self.rng, session_block(cipher, key)))) + seipd_packet(seipd_body(key, s[0], self.rng.randbytes(16)))
                self.add("C", "aes%d/H-mod-64=%02d" % (KS[cipher] * 8, H % 64), raw, 0, [("H mod 64 == %d" % (H % 64), True)], s, shape=True)
        # bodies after the version byte of 17 .. 41 bytes, every one with a quick check that passes
        for L in (17, 18, 39, 40, 41):
            key = self.session(7)
            prefix = self.rng.randbytes(16)
            if L >= 40:
                ct = seipd_body(key, self.rng.randbytes(L - 40), prefix)
            else:
                ct = R.cfb_encrypt(key, prefix + prefix[14:16] + self.rng.randbytes(max(0, L - 18)))[:L]
            raw = pkesk_c(kid, enc(k, type2(self.rng, session_block(7, key)))) + seipd_packet(ct, 1)
            pt = R.cfb_decrypt(key, ct)
            self.add("C", "body-%d" % L, raw, -8, [("body of %d bytes" % L, len(ct) == L), ("quick check passes", L < 18 or pt[14:16] == pt[16:18])],
                     shape=L >= 40, host=L >= 40)
        # Go's partial-length writer at its chunk boundaries: version byte + body of 2^k - 1, 2^k and 2^k + 1 bytes
        for total in (1023, 1024, 1025, 2047, 2048, 2049):
            s = self.inner(200 + total - 41 - base)
            while 1 + 18 + len(s[0]) + 22 != total:                   # a signature MPI one byte short
                s = self.inner(200 + total - 41 - base)
            key = self.session(9)
            raw = pkesk_c(kid, enc(k, type2(self.rng, session_block(9, key)))) + seipd_packet(seipd_body(key, s[0], self.rng.randbytes(16)))
            self.add("C", "go-partial/%d" % total, raw, 0, [("SEIPD data of %d bytes" % total, 1 + 18 + len(s[0]) + 22 == total)], s, shape=True)
        # the remaining outcomes of the layer: an MDC mismatch, a bad signature inside, no encryption at all
        s = self.pick()
        key = self.session(7)
        ct = bytearray(seipd_body(key, s[0], self.rng.randbytes(16)))
        ct[-1] ^= 1
        self.add("C", "mdc-flipped", pkesk_c(kid, enc(k, type2(self.rng, session_block(7, key)))) + seipd_packet(bytes(ct)), -12,
                 [("MDC differs", True)], s, shape=True, host=True)
        bad = bytearray(s[0])
        bad[-5] ^= 1                                                   # inside the signature MPI
        bs = (bytes(bad), s[1], s[2])
        key = self.session(7)
        self.add("C", "bad-signature", self.message(key, bs, [pkesk_c(kid, enc(k, type2(self.rng, session_block(7, key))))]), -6,
                 [("signature MPI changed", bad != s[0])], shape=True)
        self.rows[-1]["plain"], self.rows[-1]["nonce"] = s[1], s[2]
        self.add("C", "not-encrypted", s[0], -9, [("no PKESK", s[0][0] != 0xC1)])
        # definite lengths: the 1-octet form only fits a stream too short to be signed (ReadMessage fails on it)
        for form in (1, 2, 5):
            s = (b"", None, None) if form == 1 else self.pick()
            key = self.session(8)
            head = pkesk_c(kid, enc(k, type2(self.rng, session_block(8, key))))
            se = seipd_packet(seipd_body(key, s[0], self.rng.randbytes(16)), form)
            self.add("C", "definite-%d-octet" % form, head + se, -8 if form == 1 else 0,
                     [("%d-octet length" % form, {1: se[1] < 192, 2: 192 <= se[1] < 224, 5: se[1] == 255}[form])], s, shape=True, host=form == 1)

    # -- D: the order of candidate session keys.  ReadMessage takes the first key whose quick check passes; a wrong key
    # that passes it decrypts the message to garbage.
    def family_d(self):
        k0, kid0 = self.keys["0"], self.ids["0"]
        for col in self.collisions:
            cipher, key, wrong = col["cipher"], col["key"], col["wrong"]
            inner = self.pick()
            se = seipd_packet(seipd_body(key, inner[0], col["prefix"]))
            pt = R.cfb_decrypt(wrong, seipd_body(key, inner[0], col["prefix"])[:18])
            passes = [("the wrong key passes the quick check", pt[14:16] == pt[16:18])]

            def pk(kk, kid, blk):
                return pkesk_c(kid, enc(kk, type2(self.rng, blk)))
            right, bad = pk(k0, kid0, session_block(cipher, key)), pk(k0, kid0, session_block(cipher, wrong))
            while True:
                other = self.rng.randbytes(KS[cipher])
                po = R.cfb_decrypt(other, seipd_body(key, inner[0], col["prefix"])[:18])
                if po[14:16] != po[16:18]:
                    break
            failing = pk(k0, kid0, session_block(cipher, other))
            invalid = pkesk_c(kid0, enc(k0, b"\x00\x02" + bytes(self.rng.randrange(1, 256) for _ in range(7)) + b"\x00" +
                                        b"\x00" * (246 - len(session_block(cipher, key))) + session_block(cipher, key)))
            tag = "aes%d" % (KS[cipher] * 8)
            alone = "%s/wrong-alone" % tag
            self.add("D", alone, bad + se, None, passes, inner, shape=True, host=True, same_as=None)
            self.add("D", "%s/wrong,right" % tag, bad + right + se, None, passes, inner, same_as=alone)
            self.add("D", "%s/right,wrong" % tag, right + bad + se, 0, passes, inner)
            self.add("D", "%s/failing,wrong,right" % tag, failing + bad + right + se, None, passes + [("the third key fails it", True)], inner, same_as=alone)
            self.add("D", "%s/invalid(separator-at-9),right" % tag, invalid + right + se, 0, passes, inner)
        # three PKESKs to three registered keys: a failing quick check, an invalid block, then the right one
        inner = self.pick()
        key = self.session(9)
        ct = seipd_body(key, inner[0], self.rng.randbytes(16))
        k5, kL, kH = self.keys["5"], self.keys["L"], self.keys["H"]
        while True:
            other = self.session(9)
            po = R.cfb_decrypt(other, ct[:18])
            if po[14:16] != po[16:18]:
                break
        rows = [pkesk_c(self.ids["5"], enc(k5, type2(self.rng, session_block(9, other)))),
                pkesk_c(self.ids["L"], enc(kL, b"\x00\x03" + bytes(self.rng.randrange(1, 256) for _ in range(254)))),
                pkesk_c(self.ids["H"], enc(kH, type2(self.rng, session_block(9, key))))]
        self.add("D", "three-keys", b"".join(rows) + seipd_packet(ct), 0,
                 [("three key ids", len({self.ids[x] for x in ("5", "L", "H")}) == 3), ("the first key fails the quick check", True)], inner)

    # -- views
    def family(self, f):
        return [r for r in self.rows if r["family"] == f]

    def by_name(self, name):
        return next(r for r in self.rows if r["name"] == name)

    def keyring_blocks(self):
        """(secring blocks: the four keys, keyring blocks: the signer)."""
        return b"".join(self.blocks[n] for n in KEYS), self.signer_block

    def oracle(self, raws, priv=None, sec_ids=None, pub_ids=None, ring=None):
        """pgp_encrypt_ref.message_decrypt over this keyring: every key of KEYS registered with its private half."""
        from oracle import pgp_oracle as O
        sec, pub = self.keyring_blocks()
        ring = ring if ring is not None else O.read_entities(sec + pub)
        priv = priv if priv is not None else {self.ids[n]: self.keys[n] for n in KEYS}
        sec_ids = sec_ids if sec_ids is not None else set(priv)
        pub_ids = pub_ids if pub_ids is not None else {self.signer_id}
        return [R.message_decrypt(raw, priv, sec_ids, pub_ids, ring) for raw in raws]


_CACHE = {}


def build(seed: int = 0xBF7C06E0) -> Edges:
    if seed not in _CACHE:
        _CACHE[seed] = Edges(seed)
    return _CACHE[seed]
