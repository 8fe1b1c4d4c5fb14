"""Encrypted transport messages as Go's openpgp.Encrypt writes them (crypto_pgp.go:418-451), restated with Python ints and
`cryptography`'s AES block primitive, plus the secret-key packets of the fixture keys.  Used by the decryption tests: one
PKESK v3 to the recipient key, SEIPD v1 in partial-length chunks (packet.serializeStreamHeader), OpenPGP CFB without resync
(RFC 4880 §13.9: zero IV over prefix | data | MDC packet), the SHA-1 MDC packet."""
import hashlib
import random
import struct

from bftkv_b200 import workload as W


def _aes_ecb(key: bytes, block: bytes) -> bytes:
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
    e = Cipher(algorithms.AES(key), modes.ECB()).encryptor()
    return e.update(block) + e.finalize()


def cfb_encrypt(key: bytes, data: bytes) -> bytes:
    """CFB with a zero IV, built by hand from the block primitive."""
    out, fb = bytearray(), bytes(16)
    for o in range(0, len(data), 16):
        ks = _aes_ecb(key, fb)
        c = bytes(a ^ b for a, b in zip(data[o:o + 16], ks))
        out += c
        fb = c if len(c) == 16 else fb
    return bytes(out)


def cfb_decrypt(key: bytes, data: bytes) -> bytes:
    out, fb = bytearray(), bytes(16)
    for o in range(0, len(data), 16):
        ks = _aes_ecb(key, fb)
        c = data[o:o + 16]
        out += bytes(a ^ b for a, b in zip(c, ks))
        fb = c
    return bytes(out)


def secret_key_packet(k, ctime: int = 0x5E000000, protected: bool = False, algo: int = 1) -> bytes:
    """RFC 4880 §5.5.3 secret-key packet (tag 5), v4, S2K usage 0 (or 254 when `protected`)."""
    pub = bytes([4]) + struct.pack(">I", ctime) + bytes([algo]) + W._mpi(k["n"]) + W._mpi(k["e"])
    u = pow(k["p"], -1, k["q"])
    sec = W._mpi(k["d"]) + W._mpi(k["p"]) + W._mpi(k["q"]) + W._mpi(u)
    if protected:
        body = pub + bytes([254, 7, 0, 2]) + bytes(8) + sec      # usage 254, AES-128, simple S2K (contents unreadable without a passphrase)
    else:
        body = pub + bytes([0]) + sec + struct.pack(">H", sum(sec) & 0xFFFF)
    return W._new_packet(5, body)


def pkcs1_type2(rng: random.Random, msg: bytes, k: int = 256) -> bytes:
    ps = bytes(rng.randrange(1, 256) for _ in range(k - 3 - len(msg)))
    return b"\x00\x02" + ps + b"\x00" + msg


def pkesk(key_id: int, k, em: bytes) -> bytes:
    c = pow(int.from_bytes(em, "big"), k["e"], k["n"])
    return W._new_packet(1, bytes([3]) + struct.pack(">Q", key_id) + bytes([1]) + W._mpi(c))


def session_block(cipher: int, key: bytes) -> bytes:
    return bytes([cipher]) + key + struct.pack(">H", sum(key) & 0xFFFF)


def seipd(key: bytes, inner: bytes, rng: random.Random, flip_mdc: bool = False, bad_quick: bool = False) -> bytes:
    prefix = bytes(rng.randrange(256) for _ in range(16))
    prefix += prefix[14:16] if not bad_quick else bytes([prefix[14] ^ 1, prefix[15]])
    mdc = hashlib.sha1(prefix + inner + b"\xd3\x14").digest()
    if flip_mdc:
        mdc = bytes([mdc[0] ^ 1]) + mdc[1:]
    ct = cfb_encrypt(key, prefix + inner + b"\xd3\x14" + mdc)
    return bytes([0xC0 | 18]) + W.go_partial_write(bytes([1]) + ct) + b"\x00"


def encrypt(rng: random.Random, recipient, recipient_id: int, inner: bytes, cipher: int = 7, **kw) -> bytes:
    """One message: PKESK to recipient_id + SEIPD over `inner` (the signed packet stream)."""
    key = bytes(rng.randrange(256) for _ in range({7: 16, 8: 24, 9: 32}[cipher]))
    return pkesk(recipient_id, recipient, pkcs1_type2(rng, session_block(cipher, key))) + seipd(key, inner, rng, **kw)


# ---- reference decryption: openpgp.ReadMessage's encryption half over Python ints -------------------------------------
# Restated from RFC 4880 and the published x/crypto/openpgp (read.go ReadMessage, packet/encrypted_key.go,
# packet/symmetrically_encrypted.go) and Go 1.13 crypto/rsa decryptPKCS1v15; the signature half is oracle/pgp_oracle.py's
# message_verify.  Codes are BFTQ_ERR_* values; shapes the library hands back to crypto/pgp are -11.
def _code(err):
    from oracle import pgp_oracle as O
    return {None: 0, O.ERR_INVALID_SIGNATURE: -6, O.ERR_DECRYPTION_FAILED: -8, O.ERR_TRANSPORT_SECURITY: -9,
            O.ERR_MESSAGE_BODY: -10, O.ERR_MESSAGE_UNSUPPORTED: -11}[err]


def _mdc_reached(keyring, inner, res) -> bool:
    """Is seMDCReader.Close reached?  At the literal's EOF with an unknown signer (checkReader), after a signature packet
    with a known one (signatureCheckReader); never when ReadMessage failed, the message is unsigned or the body is short."""
    from oracle import pgp_oracle as O
    if res.err in (O.ERR_DECRYPTION_FAILED, O.ERR_TRANSPORT_SECURITY, O.ERR_MESSAGE_UNSUPPORTED):
        return False
    r = O.Reader(inner)
    try:
        while True:
            pk = O.read_packet(r)
            if pk is None:
                return False
            if pk[0] == 11:
                break
    except O.PGPError:
        return False                                # the literal body ends early: ReadAll fails before the MDC
    if not res.signer_known:
        return True
    try:
        while True:
            pk = O.read_packet(r)
            if pk is None:
                return False
            if pk[0] in O.KNOWN_TAGS:
                break
        if pk[0] != 2:
            return False
        O.parse_signature(pk[1])
        return True
    except O.PGPError:
        return False


def message_decrypt(raw: bytes, priv: dict, sec_ids: set, pub_ids: set, keyring):
    """-> (code, plain, nonce).  priv: key id -> fixture key dict (the registered private halves); sec_ids / pub_ids: key
    ids (primary and subkeys) of the secring / keyring entities; keyring: oracle entities for the signature half."""
    from oracle import pgp_oracle as O
    r = O.Reader(raw)
    pairs, any_keys = [], False
    try:
        while True:
            at = r.pos
            pk = O.read_packet(r)
            if pk is None:
                return -8, None, None                      # io.EOF before the encrypted packet
            tag, body = pk
            if tag not in O.KNOWN_TAGS:
                continue
            if tag == 1:
                if len(body) < 10 or body[0] != 3:
                    return -8, None, None
                kid, algo = int.from_bytes(body[1:9], "big"), body[9]
                if algo == 16 or kid == 0:
                    return -11, None, None                 # ElGamal, wildcard key id
                if algo not in (1, 2):
                    continue
                c, _, _ = O.read_mpi(body, 10)
                any_keys = any_keys or kid in sec_ids or kid in pub_ids
                if kid in sec_ids:
                    if kid not in priv:
                        return -11, None, None
                    pairs.append((kid, c))
                continue
            if tag == 18:
                if len(body) < 1 or body[0] != 1:
                    return -8, None, None
                if r.pos < len(raw):
                    return -11, None, None
                se = body[1:]
                break
            if tag in (8, 11, 4):
                if any_keys:
                    return -8, None, None                  # key material not followed by encrypted message
                res = O.message_verify(keyring, raw[at:])
                return {O.ERR_DECRYPTION_FAILED: -8, O.ERR_MESSAGE_UNSUPPORTED: -11}.get(res.err, -9), None, None
            return -11, None, None                         # tag 3, tag 9, other packets
    except O.PGPError:
        return -8, None, None
    for kid, c in pairs:
        k = priv[kid]
        if c > k["n"]:
            continue                                       # ErrDecryption: EncryptedKey.Key stays empty
        em = pow(c, k["d"], k["n"]).to_bytes(256, "big")
        if em[0] != 0 or em[1] != 2 or 0 not in em[2:] or em.index(0, 2) < 10:
            continue
        b = em[em.index(0, 2) + 1:]
        if len(b) < 3:
            return -8, None, None                          # the reference panics on b[len(b)-2]
        cipher, key = b[0], b[1:-2]                        # a checksum mismatch leaves the key in place
        ks = {2: 24, 3: 16, 7: 16, 8: 24, 9: 32}.get(cipher, 0)
        if ks == 0 or len(key) != ks or len(se) < 18:
            return -8, None, None
        if cipher in (2, 3):
            return -11, None, None
        pre = cfb_decrypt(key, se[:18])
        if pre[14:16] != pre[16:18]:
            continue                                       # ErrKeyIncorrect: the next candidate
        if len(se) < 40:
            return -8, None, None
        pt = cfb_decrypt(key, se)
        inner = pt[18:-22]
        res = O.message_verify(keyring, inner)
        mdc_ok = pt[-22:-20] == b"\xd3\x14" and hashlib.sha1(pt[:-20]).digest() == pt[-20:]
        if not mdc_ok and _mdc_reached(keyring, inner, res):
            return -12, None, None
        return _code(res.err), res.plain, res.nonce
    return -8, None, None
