"""DataEncryption (crypto_pgp.go:532-554) restated in Python: the test oracle of K11.

encrypt() is x/crypto @53104e6ec876's SymmetricallyEncrypt(w, key, nil, nil) followed by one Write(plain) and Close,
with the 40 random bytes Go reads (salt 8, session key 16, IV 16) given by the caller.  Every Write in its writer cascade
reaches the outer partialLengthWriter as its own Write (workload.go_partial_write).  decrypt() is ReadMessage's symmetric
half plus ReadAll, answering with the device's error codes where Go would hang or panic.  hashlib and the `cryptography`
AES block only."""
import hashlib

from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes

from bftkv_b200.workload import go_partial_write

OK, MALFORMED, MESSAGE_BODY, UNSUPPORTED, MDC, DECRYPTION_FAILED = 0, -8, -10, -11, -12, -18
KEY_SIZE = {2: 24, 3: 16, 7: 16, 8: 24, 9: 32}            # packet.CipherFunction.KeySize
AES = (7, 8, 9)


def fixture_value(n: int, seed: int) -> bytes:
    """The n-byte value of tests/golden/data_encryption.json's case `seed` (no CR byte: GnuPG rewrites CR LF in text mode)."""
    out, k = bytearray(), 0
    while len(out) < n:
        out += hashlib.sha256(b"%d/%d" % (seed, k)).digest()
        k += 1
    return bytes(out[:n]).replace(b"\r", b"\n")


def count_of(c: int) -> int:
    return (16 + (c & 15)) << ((c >> 4) + 6)


def s2k(mode: int, salt: bytes, count: int, key: bytes, size: int) -> bytes:
    """s2k.Simple / Salted / Iterated over SHA-256 (size <= 32: one hash context)."""
    data = key if mode == 0 else salt + key
    if mode == 3:
        n = max(count, len(data))
        data = (data * (n // max(1, len(data)) + 1))[:n] if data else b""
    return hashlib.sha256(data).digest()[:size]


def _ecb(key: bytes, block: bytes) -> bytes:
    e = Cipher(algorithms.AES(key), modes.ECB()).encryptor()
    return e.update(block) + e.finalize()


def cfb_encrypt(key: bytes, data: bytes) -> bytes:
    """OpenPGP CFB with a zero IV and no resync, as one stream."""
    out, prev = bytearray(), bytes(16)
    for k in range(0, len(data), 16):
        ks = _ecb(key, prev)
        c = bytes(a ^ b for a, b in zip(data[k:k + 16], ks))
        out += c
        prev = c if len(c) == 16 else prev
    return bytes(out)


def cfb_decrypt(key: bytes, data: bytes) -> bytes:
    out, prev = bytearray(), bytes(16)
    for k in range(0, len(data), 16):
        c = data[k:k + 16]
        out += bytes(a ^ b for a, b in zip(c, _ecb(key, prev)))
        prev = c
    return bytes(out)


def writes(n: int):
    """The Writes that reach the outer partialLengthWriter for a value of n bytes: (kind, length) in order, kind one of
    'raw' (the version byte), 'prefix', 'byte' (one encrypted framing byte), 'body', 'mdc'."""
    out = [("raw", 1), ("prefix", 18), ("byte", 1)]
    for w in (2, 4, n):
        while w:
            p = max(k for k in range(15) if (1 << k) <= w)
            out += [("byte", 1), ("body", 1 << p)]
            w -= 1 << p
    return out + [("byte", 1), ("mdc", 22)]


def encrypted_len(n: int) -> int:
    return 32 + 1 + sum(len(go_partial_write(bytes(w))) for _, w in writes(n)) + 1


def encrypt(key: bytes, plain: bytes, rand: bytes) -> bytes:
    assert len(rand) == 40
    salt, sk, iv = rand[:8], rand[8:24], rand[24:40]
    kek = s2k(3, salt, 65536, key, 16)
    skesk = bytes([0xC3, 0x1E, 4, 7, 3, 8]) + salt + b"\x60" + cfb_encrypt(kek, b"\x07" + sk)
    # the plain stream, cut into the cascade's Writes
    body = b"t\x00" + bytes(4) + plain
    prefix = iv + iv[14:16]
    pieces, pos = [], 0
    inner = [224 + max(k for k in range(15) if (1 << k) <= w) for kind, w in writes(len(plain)) if kind == "body"]
    framing = iter([0xCB] + [x for x in inner] + [0x00])
    for kind, w in writes(len(plain)):
        if kind == "raw":
            pieces.append(("raw", b"\x01"))
        elif kind == "prefix":
            pieces.append(("enc", prefix))
        elif kind == "byte":
            pieces.append(("enc", bytes([next(framing)])))
        elif kind == "body":
            pieces.append(("enc", body[pos:pos + w]))
            pos += w
        else:
            hashed = b"".join(p for k, p in pieces if k == "enc") + b"\xD3\x14"
            pieces.append(("enc", b"\xD3\x14" + hashlib.sha1(hashed).digest()))
    stream = cfb_encrypt(sk, b"".join(p for k, p in pieces if k == "enc"))
    out, at = bytearray(skesk + b"\xD2"), 0
    for k, p in pieces:
        if k == "raw":
            out += go_partial_write(p)
        else:
            out += go_partial_write(stream[at:at + len(p)])
            at += len(p)
    return bytes(out + b"\x00")


class _Short(Exception):
    pass


def _packet(m: bytes, p: int):
    """(tag, body, next position) of the packet at p, partial lengths de-chunked; _Short on framing errors."""
    if p >= len(m) or not m[p] & 0x80:
        raise _Short
    h = m[p]
    p += 1
    if not h & 0x40:
        tag, lt = (h & 0x3F) >> 2, h & 3
        if lt == 3:
            return tag, m[p:], len(m)
        nl = 1 << lt
        if p + nl > len(m):
            raise _Short
        n = int.from_bytes(m[p:p + nl], "big")
        p += nl
        if n > len(m) - p:
            raise _Short
        return tag, m[p:p + n], p + n
    tag, body = h & 0x3F, bytearray()
    while True:
        if p >= len(m):
            raise _Short
        o = m[p]
        partial = False
        if o < 192:
            n, p = o, p + 1
        elif o < 224:
            if p + 2 > len(m):
                raise _Short
            n, p = ((o - 192) << 8) + m[p + 1] + 192, p + 2
        elif o == 255:
            if p + 5 > len(m):
                raise _Short
            n, p = int.from_bytes(m[p + 1:p + 5], "big"), p + 5
        else:
            n, p, partial = 1 << (o & 0x1F), p + 1, True
        if n > len(m) - p:
            raise _Short
        body += m[p:p + n]
        p += n
        if not partial:
            return tag, bytes(body), p


KNOWN_TAGS = {1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 13, 14, 17, 18}


def _literal(d: bytes):
    """(code, body) of the first literal packet of the inner stream d, read as far as d goes."""
    p = 0
    while True:
        if p >= len(d) or not d[p] & 0x80:
            return MALFORMED, None
        h = d[p]
        tag = h & 0x3F if h & 0x40 else (h & 0x3F) >> 2
        if tag != 11:
            try:
                t, _, p = _packet(d, p)
            except _Short:
                return MALFORMED, None
            if t in KNOWN_TAGS:
                return UNSUPPORTED, None
            continue
        p += 1
        lit, short = bytearray(), False
        if not h & 0x40:
            lt = h & 3
            if lt == 3:
                lit += d[p:]
            else:
                nl = 1 << lt
                if p + nl > len(d):
                    return MALFORMED, None
                n = int.from_bytes(d[p:p + nl], "big")
                p += nl
                short = n > len(d) - p
                lit += d[p:p + n]
        else:
            first = True
            while True:
                if p >= len(d):
                    if first:
                        return MALFORMED, None
                    short = True
                    break
                o = d[p]
                hl = 1 if o < 192 else 2 if o < 224 else 5 if o == 255 else 1
                if p + hl > len(d):
                    if first:
                        return MALFORMED, None
                    short = True
                    break
                if o < 192:
                    n = o
                elif o < 224:
                    n = ((o - 192) << 8) + d[p + 1] + 192
                elif o == 255:
                    n = int.from_bytes(d[p + 1:p + 5], "big")
                else:
                    n = 1 << (o & 0x1F)
                p += hl
                first = False
                take = d[p:p + n]
                lit += take
                p += len(take)
                if len(take) < n:
                    short = True
                    break
                if not (224 <= o < 255):
                    break
        if len(lit) < 2 or len(lit) < 6 + lit[1]:
            return MALFORMED, None
        return (MESSAGE_BODY, None) if short else (OK, bytes(lit[6 + lit[1]:]))


def unwrap(sk_packet: dict, key: bytes):
    """SymmetricKeyEncrypted.Decrypt: (cipher, session key), or None when Go's Decrypt returns an error (and, the
    documented divergence, for an unwrapped 3DES or CAST5 key)."""
    c = sk_packet["cipher"]
    kek = s2k(sk_packet["mode"], sk_packet["salt"], sk_packet["count"], key, KEY_SIZE[c])
    esk = sk_packet["esk"]
    if not esk:
        return c, kek
    pt = cfb_decrypt(kek, esk)
    if pt[0] not in AES or len(pt) - 1 != KEY_SIZE[pt[0]]:
        return None
    return pt[0], pt[1:]


def decrypt(key: bytes, msg: bytes):
    """(code, plain text or None)."""
    p, sks = 0, []
    while True:
        try:
            tag, b, p = _packet(msg, p)
        except _Short:
            return MALFORMED, None
        if tag not in KNOWN_TAGS:
            continue
        if tag == 3:
            if len(sks) == 16:
                return UNSUPPORTED, None
            if len(b) < 4:
                return MALFORMED, None
            if b[0] != 4 or b[1] not in AES or b[3] != 8:
                return UNSUPPORTED, None
            mode, q = b[2], 4
            if mode not in (0, 1, 3):
                return UNSUPPORTED, None
            salt, count = b"", 0
            if mode in (1, 3):
                need = 8 if mode == 1 else 9
                if len(b) - q < need:
                    return MALFORMED, None
                salt = b[q:q + 8]
                count = count_of(b[q + 8]) if mode == 3 else 0
                q += need
            if len(b) - q >= 64:
                return UNSUPPORTED, None
            sks.append({"cipher": b[1], "mode": mode, "salt": salt, "count": count, "esk": b[q:]})
            continue
        if tag == 18:
            if len(b) < 1 or b[0] != 1:
                return MALFORMED, None
            if p < len(msg):
                return UNSUPPORTED, None
            if not sks or len(b) - 1 < 18:
                return MALFORMED, None
            ct = b[1:]
            break
        if tag in (8, 11, 4) and sks:
            return MALFORMED, None
        return UNSUPPORTED, None
    for s in sks:
        u = unwrap(s, key)
        if u is None:
            continue
        cipher, sk = u
        pt = cfb_decrypt(sk, ct)
        if pt[14:16] != pt[16:18]:                               # the quick check
            continue
        if len(ct) < 40:
            return MALFORMED, None
        code, body = _literal(pt[18:-22])
        if code != OK:
            return code, None
        trailer = pt[-22:]
        if trailer[:2] != b"\xD3\x14" or hashlib.sha1(pt[:-20]).digest() != trailer[2:]:
            return MDC, None
        return OK, body
    return DECRYPTION_FAILED, None
