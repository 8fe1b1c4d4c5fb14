"""crypto/auth (threshold password authentication, auth.go) restated in Python integers, hashlib / hmac and
`cryptography`: GeneratePartialAuthenticationParams, PI, every serializer, the server (NewServer / MakeResponse) and the
client (Initiate / ProcessResponse / GetCipherKey).  Randomness is injectable: every draw goes through an `rng` with
randbelow(n) and randbytes(k) (random.Random works; seed it for reproducible rounds).

HKDF, HMAC and the GCM seal are written out here (GCM on AES-ECB from `cryptography` and a bit-serial GHASH), so that
tests can check them against `cryptography`'s own HKDF and AESGCM."""
import hashlib
import hmac as _hmac
import struct

from oracle import sss_oracle as sss

# p of crypto/auth (auth.go:81-115), a 2048-bit safe prime, and q = (p - 1) / 2
P = int("b0a67d9f5cebc0ffe81690e7b2670ab05f9fa4c2e73639f660c0408a2d9a4a8b454a9893fd7d4e8fa399cfc9c9ba05b080f903e33bcdcbefaed40915"
        "e51d46f58d1a5bd204db20fa3fe9db71f0b8e0aa87b5771406f25fad59e7f10fe52556447588"
        "72ea2dec1f6dcd11be905de59a044f6c2ea3982b2235acc9021a196fc4ce0b19f6b312ee9cfc5997dc5f7ce2f386131294a56ba93a41a3b60e27e03956039f51"
        "ae73b89c795c5ae7d841e9b455c37341c052404e8fe9fe4f0d52bc162a41f1eeb9ef292c66a9d6a619aa548807eb1187ee22bd62e20e26c3c08c22ecef12d3"
        "b2304a010ed1f50a68e0261afe1a0bdddf7ab8a61774d3af3f1cce2b95dad3", 16)
Q = (P - 1) // 2
AUTH_RETRY_LIMIT = 10


class AuthenticationFailure(Exception):
    """bftkv.ErrAuthenticationFailure"""


class DecryptionFailed(Exception):
    """crypto.ErrDecryptionFailed"""


# ---- framing ---------------------------------------------------------------------------------------------------------
def i2b(v: int) -> bytes:                                      # big.Int.Bytes(): minimal, empty for 0
    return v.to_bytes((v.bit_length() + 7) // 8, "big")


def chunk(b: bytes) -> bytes:                                  # packet.WriteChunk
    return struct.pack(">Q", len(b)) + b


class Reader:
    def __init__(self, b: bytes):
        self.b, self.pos = b, 0

    def int32(self) -> int:
        if len(self.b) - self.pos < 4:
            raise ValueError("EOF")
        v = struct.unpack(">i", self.b[self.pos:self.pos + 4])[0]
        self.pos += 4
        return v

    def chunk(self) -> bytes:                                  # packet.ReadChunk (nil for length 0)
        if len(self.b) - self.pos < 8:
            raise ValueError("EOF")
        n = struct.unpack(">Q", self.b[self.pos:self.pos + 8])[0]
        self.pos += 8
        if n == 0:
            return b""
        if len(self.b) - self.pos < n:
            raise ValueError("unexpected EOF")
        c = self.b[self.pos:self.pos + n]
        self.pos += n
        return c


def serialize_params(x: int, y: int, v: int, salt: bytes) -> bytes:
    return struct.pack(">i", x) + chunk(i2b(y)) + chunk(i2b(v)) + chunk(salt)


def parse_params(b: bytes):
    r = Reader(b)
    return r.int32(), int.from_bytes(r.chunk(), "big"), int.from_bytes(r.chunk(), "big"), r.chunk()


def serialize_yi(x: int, yi: int, salt: bytes) -> bytes:
    return struct.pack(">i", x) + chunk(i2b(yi)) + chunk(salt)


def parse_yi(b: bytes):
    r = Reader(b)
    return r.int32(), int.from_bytes(r.chunk(), "big"), r.chunk()


def serialize_bi(bi: int) -> bytes:
    return chunk(i2b(bi))


def parse_bi(b: bytes) -> int:
    return int.from_bytes(Reader(b).chunk(), "big")


def serialize_zi(zi: bytes, nonce: bytes) -> bytes:
    return chunk(zi) + chunk(nonce)


def parse_zi(b: bytes):
    r = Reader(b)
    return r.chunk(), r.chunk()


# ---- symmetric layer -------------------------------------------------------------------------------------------------
def h(*args: bytes) -> bytes:                                  # auth.go hash()
    s = hashlib.sha256()
    for a in args:
        s.update(a)
    return s.digest()


def hmac_sha256(key: bytes, msg: bytes) -> bytes:
    return _hmac.new(key, msg, hashlib.sha256).digest()


def hkdf_sha256(ikm: bytes, salt: bytes, info: bytes = b"", n: int = 32) -> bytes:    # RFC 5869
    prk = hmac_sha256(salt if salt else bytes(32), ikm)
    out, t, i = b"", b"", 1
    while len(out) < n:
        t = hmac_sha256(prk, t + info + bytes([i]))
        out += t
        i += 1
    return out[:n]


def key_sched(ki: bytes, salt: bytes):                         # keySched: (km, ke)
    okm = hkdf_sha256(ki, salt)
    return okm[:16], okm[16:32]


def calculate_mac(km: bytes, xi: bytes, bi: bytes) -> bytes:
    return hmac_sha256(km, xi + bi)


def gf128_mul(x: int, y: int) -> int:
    """GCM's GF(2^128) product of two 128-bit blocks read big-endian (bit 0 = the block's first bit)."""
    R = 0xE1 << 120
    z, v = 0, y
    for i in range(128):
        if (x >> (127 - i)) & 1:
            z ^= v
        v = (v >> 1) ^ R if v & 1 else v >> 1
    return z


def _aes_ecb(key: bytes, block: bytes) -> bytes:
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
    e = Cipher(algorithms.AES(key), modes.ECB()).encryptor()
    return e.update(block) + e.finalize()


def ghash(hk: int, aad: bytes, ct: bytes) -> int:
    x = 0
    for data in (aad, ct):
        for i in range(0, len(data), 16):
            x = gf128_mul(x ^ int.from_bytes(data[i:i + 16].ljust(16, b"\0"), "big"), hk)
    return gf128_mul(x ^ ((len(aad) * 8) << 64 | len(ct) * 8), hk)


def gcm_seal(key: bytes, nonce: bytes, pt: bytes, aad: bytes) -> bytes:
    """AES-GCM with a 12-byte nonce and a 16-byte tag: ciphertext || tag (cipher.AEAD.Seal)."""
    hk = int.from_bytes(_aes_ecb(key, bytes(16)), "big")
    ct = bytearray()
    for j in range(0, len(pt), 16):
        ks = _aes_ecb(key, nonce + struct.pack(">I", 2 + j // 16))
        ct += bytes(a ^ b for a, b in zip(pt[j:j + 16], ks))
    s = int.from_bytes(_aes_ecb(key, nonce + struct.pack(">I", 1)), "big")
    return bytes(ct) + (ghash(hk, aad, bytes(ct)) ^ s).to_bytes(16, "big")


def gcm_open(key: bytes, nonce: bytes, ct: bytes, aad: bytes) -> bytes:
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    try:
        return AESGCM(key).decrypt(nonce, ct, aad)
    except Exception as exc:
        raise DecryptionFailed() from exc


# ---- the protocol ----------------------------------------------------------------------------------------------------
def PI(password: bytes) -> int:
    t = int.from_bytes(h(password), "big")
    return t * t % Q


def generate_params(cred: bytes, n: int, k: int, rng):
    """GeneratePartialAuthenticationParams: n serialized parameter sets."""
    s = rng.randbelow(Q)
    coords = sss.distribute(s, [rng.randbelow(Q) for _ in range(k - 1)], n, Q)
    pi = PI(cred)
    salt = rng.randbytes(16)
    res = []
    for i, (x, y) in enumerate(coords):
        psalt = h(salt, bytes([i & 0xff]))
        si = int.from_bytes(h(cred, psalt), "big") * s % Q
        res.append(serialize_params(x, y, pow(pi, si, P), psalt))
    return res


class Server:
    """AuthServer.  make_response takes the randomness Go would draw (b for phase 1, the nonce for phase 2).

    reference_zero_key_quirk (default True, as auth.go): a server that never ran phase 1 has mac = nil, so an empty Ni
    passes ConstantTimeCompare and the proof is sealed under an all-zero key.  False: such a phase 2 fails, as the device
    path does."""

    def __init__(self, params: bytes, proof: bytes, reference_zero_key_quirk: bool = True):
        self.x, self.y, self.v, self.salt = parse_params(params)
        self.proof = proof
        self.attempts = 0
        self.km, self.ke = bytes(16), bytes(16)
        self.mac = None
        self.quirk = reference_zero_key_quirk

    def make_yi(self, X: bytes) -> bytes:
        return serialize_yi(self.x, pow(int.from_bytes(X, "big"), self.y, P), self.salt)

    def make_bi(self, Xi: bytes, b: int) -> bytes:
        bi = pow(self.v, b, P)
        ki = pow(int.from_bytes(Xi, "big"), b, P)
        self.km, self.ke = key_sched(i2b(ki), self.salt)
        self.mac = calculate_mac(self.km, Xi, i2b(bi))
        return serialize_bi(bi)

    def make_zi(self, Ni: bytes, nonce: bytes) -> bytes:
        if self.mac is None and not self.quirk:
            raise AuthenticationFailure()
        if not _hmac.compare_digest(Ni, self.mac or b""):
            raise AuthenticationFailure()
        return serialize_zi(gcm_seal(self.ke, nonce, self.proof, self.mac or b""), nonce)

    def make_response(self, phase: int, req: bytes, rand: bytes = b""):
        """(res, done, err) without the retry delay."""
        if phase == 0:
            res = self.make_yi(req)
            self.attempts += 1
            return res, False, ("too many attempts" if self.attempts >= AUTH_RETRY_LIMIT else None)
        if phase == 1:
            return self.make_bi(req, int.from_bytes(rand, "big")), False, None
        if phase == 2:
            try:
                return self.make_zi(req, rand), True, None
            except AuthenticationFailure:
                return None, True, "authentication failure"
        return None, False, None


class Client:
    def __init__(self, password: bytes, n: int, k: int, rng):
        self.password, self.n, self.k, self.rng = password, n, k, rng
        self.secrets = {}
        self.gs = None
        self.nresponses = 0

    def generate_x(self) -> bytes:
        self.a = self.rng.randbelow(Q)
        return i2b(pow(PI(self.password), self.a, P))

    def calculate_shared_secret(self) -> int:
        xs = [s["x"] for s in self.secrets.values()]
        gs = 1
        for s in self.secrets.values():
            gs = gs * pow(s["Y"], sss.lagrange(s["x"], xs, Q), P) % P
        return gs

    def process_yi(self, res: bytes, pid: int):
        x, yi, salt = parse_yi(res)
        self.secrets[pid] = {"x": x, "Y": yi, "salt": salt}
        if len(self.secrets) < self.k:
            return None
        self.gs = self.calculate_shared_secret()
        out = {}
        for i, s in self.secrets.items():
            s["a2"] = self.rng.randbelow(Q)
            si = int.from_bytes(h(self.password, s["salt"]), "big")
            s["Xi"] = i2b(pow(self.gs, s["a2"] * si % Q, P))
            out[i] = s["Xi"]
        self.nresponses = 0
        return out

    def process_bi(self, res: bytes, pid: int):
        bi = parse_bi(res)
        s = self.secrets[pid]
        ki = pow(bi, self.a * s["a2"] % Q, P)
        s["km"], s["ke"] = key_sched(i2b(ki), s["salt"])
        s["Ni"] = calculate_mac(s["km"], s["Xi"], i2b(bi))
        self.nresponses += 1
        if self.nresponses >= len(self.secrets):
            self.nresponses = 0
            return {i: t["Ni"] for i, t in self.secrets.items()}
        return None

    def process_zi(self, res: bytes, pid: int):
        zi, nonce = parse_zi(res)
        s = self.secrets[pid]
        s["Pi"] = gcm_open(s["ke"], nonce, zi, s["Ni"])
        self.nresponses += 1
        if self.nresponses >= len(self.secrets):
            return {i: t["Pi"] for i, t in self.secrets.items()}
        return None

    def get_cipher_key(self) -> bytes:
        ainv = pow(self.a, -1, Q)
        return h(i2b(pow(self.gs, ainv, P)), self.password)


class Rng:
    """A seeded source for every draw the protocol makes (rand.Int and rand.Read)."""

    def __init__(self, seed):
        import random
        self.r = random.Random(seed)

    def randbelow(self, n: int) -> int:
        return self.r.randrange(n)

    def randbytes(self, k: int) -> bytes:
        return self.r.randbytes(k)


def run_round(password: bytes, proof: bytes, n: int, k: int, rng, make_servers=None, respond=None):
    """TestAuth's testAuth: servers answer phases 0, 1 and 2 for a client until it has k proofs.  respond(servers, ids,
    phase, reqs, rands) -> answers replaces the oracle servers' make_response (a device run passes its own).  Returns
    (client, {id: Pi})."""
    params = generate_params(password, n, k, rng)
    servers = make_servers(params, proof) if make_servers else [Server(p, proof) for p in params]
    if respond is None:
        def respond(srv, ids, phase, reqs, rands):
            return [srv[i].make_response(phase, q, r)[0] for i, q, r in zip(ids, reqs, rands)]
    c = Client(password, n, k, rng)
    X = c.generate_x()
    xis = None
    for i in range(n):
        (yi,) = respond(servers, [i], 0, [X], [b""])
        xis = c.process_yi(yi, i)
        if xis is not None:
            break
    assert xis is not None
    ids = sorted(xis)
    bis = respond(servers, ids, 1, [xis[i] for i in ids], [rng.randbelow(P).to_bytes(256, "big") for _ in ids])
    nis = None
    for i, bi in zip(ids, bis):
        nis = c.process_bi(bi, i)
    assert nis is not None
    ids = sorted(nis)
    zis = respond(servers, ids, 2, [nis[i] for i in ids], [rng.randbytes(12) for _ in ids])
    pis = None
    for i, zi in zip(ids, zis):
        pis = c.process_zi(zi, i)
    return c, pis
