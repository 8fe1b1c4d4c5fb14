"""PGPSignature.Sign (crypto_pgp.go:346-371) restated in Python: what bftq_signature_sign_batch must write, byte for byte.

Sign calls openpgp.DetachSign(&w, secring[0], tbs, nil) of golang.org/x/crypto @53104e6ec876 (not in the reference tree;
restated here from the published code, by function):
  openpgp/write.go detachSign   signer = the entity's PrimaryKey / PrivateKey (never a subkey); SigType 0x00, PubKeyAlgo the
                                signer's, Hash = config.Hash() = SHA-256 for a nil config, CreationTime = config.Now(),
                                IssuerKeyId = the primary key id; tbs hashed, then sig.Sign, then sig.Serialize
  packet/signature.go buildSubpackets   creation time (type 2, 4 bytes) then issuer (type 16, 8 bytes), both hashed;
                                nothing unhashed
  packet/signature.go signPrepareHash   HashSuffix = 04 | SigType | PubKeyAlgo | Hash | u16 len | hashed subpackets, then
                                the trailer 04 FF | u32 len(the HashSuffix before it); digest = SHA-256(tbs || all that)
  packet/signature.go Sign      RSASignature.bytes = rsa.SignPKCS1v15(.., SHA-256, digest), and bitLength = 8 * len(bytes):
                                the MPI header is 08 00 whatever s is, and a short s keeps its leading zero bytes
  Go 1.13 crypto/rsa SignPKCS1v15   EM = 00 01 FF .. FF 00 || DigestInfo(SHA-256) || digest, s = EM^d mod n (CRT with
                                blinding, then decryptAndCheck), copyWithLeftPad to 256 bytes; deterministic
  packet/signature.go Serialize  a new-format header: C2, then the two-octet length of the 284-byte body
"""
import hashlib
import struct

from bftkv_b200 import workload as W

PACKET_BYTES = 287
SHA256_PREFIX = bytes.fromhex("3031300d060960864801650304020105000420")


def hashed_area(ctime: int, key_id: int) -> bytes:
    return bytes([5, 2]) + struct.pack(">I", ctime) + bytes([9, 16]) + struct.pack(">Q", key_id)


def suffix(ctime: int, key_id: int) -> bytes:
    """HashSuffix and trailer: the 28 bytes hashed after tbs."""
    head = bytes([4, 0, 1, 8]) + struct.pack(">H", 16) + hashed_area(ctime, key_id)
    return head + b"\x04\xff" + struct.pack(">I", len(head))


def digest(tbs: bytes, ctime: int, key_id: int) -> bytes:
    return hashlib.sha256(tbs + suffix(ctime, key_id)).digest()


def em(dg: bytes) -> int:
    t = SHA256_PREFIX + dg
    return int.from_bytes(b"\x00\x01" + b"\xff" * (256 - len(t) - 3) + b"\x00" + t, "big")


def sign_s(k, dg: bytes) -> int:
    """s = EM^d mod n: the value SignPKCS1v15 returns (blinding does not change it).  Computed by CRT, for speed."""
    m, p, q = em(dg), k["p"], k["q"]
    sp, sq = pow(m, k["d"] % (p - 1), p), pow(m, k["d"] % (q - 1), q)
    return sq + q * ((sp - sq) * pow(q, -1, p) % p)


def packet(k, key_id: int, tbs: bytes, ctime: int, s_of=sign_s) -> bytes:
    """The signature packet.  s_of(k, digest) -> s: sign_s, or a faster signer that agrees with it (cryptography_s)."""
    dg = digest(tbs, ctime, key_id)
    body = suffix(ctime, key_id)[:22] + b"\x00\x00" + dg[:2] + b"\x08\x00" + s_of(k, dg).to_bytes(256, "big")
    assert len(body) == 284
    return b"\xc2\xc0\x5c" + body


def cryptography_s(k, dg: bytes) -> int:
    """sign_s by OpenSSL through `cryptography` (RSA PKCS#1 v1.5 of a prehashed SHA-256 digest): equal to sign_s on every
    fixture case (tests/golden/make_signature_sign.py checks it), and fast enough for tests that sign many thousands."""
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding
    from cryptography.hazmat.primitives.asymmetric.utils import Prehashed
    if "_priv" not in k:
        k["_priv"] = W._private_key(k)
    return int.from_bytes(k["_priv"].sign(dg, padding.PKCS1v15(), Prehashed(hashes.SHA256())), "big")


def key_block(k, uid: bytes = b"signer <signer@bftq.test>"):
    """(transferable public key, primary key id) as the tests register it."""
    return W.pgp_public_key_block(k, W._private_key(k), uid)
