"""Threshold DSA / ECDSA (crypto/threshold/dsa/dsa_core.go, dsa.go, ecdsa.go) restated in Python ints: the share and
message serializers, sss.Distribute-style joint shares, the server's phases 2 and 3 (dsaContext.Sign), and the client's
CalculateR, calculateS and formatDSA."""
import random
import struct

P256 = dict(P=2**256 - 2**224 + 2**192 + 2**96 - 1,
            N=0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551,
            B=0x5ac635d8aa3a93e7b3ebbd55769886bc651d06b0cc53b0f63bce3c3e27d2604b,
            Gx=0x6b17d1f2e12c4247f8bce6e563a440f277037d812deb33a0f4a13945d898c296,
            Gy=0x4fe342e2fe1a7f9b8ee7eb4a7c0f9e162bce33576b315ececbb6406837bf51f5, BitSize=256)


def bts(v: int) -> bytes:                      # big.Int.Bytes()
    return v.to_bytes((v.bit_length() + 7) // 8, "big")


def chunk(b: bytes) -> bytes:                  # packet.WriteChunk
    return struct.pack(">Q", len(b)) + b


def group_ser(g) -> bytes:
    if g["kind"] == "dsa":
        return chunk(bts(g["p"])) + chunk(bts(g["q"])) + chunk(bts(g["g"]))
    return b"".join(chunk(bts(P256[k])) for k in ("P", "N", "B", "Gx", "Gy")) + struct.pack(">I", P256["BitSize"])


def order(g) -> int:
    return g["q"] if g["kind"] == "dsa" else P256["N"]


def share_secret(g, x: int, y: bytes, t: int, nodes: bytes = b"") -> bytes:   # serializePartialParam (y: the Y chunk as is)
    return group_ser(g) + struct.pack(">Q", x) + chunk(y) + struct.pack(">H", t) + nodes


def distribute(rng, s: int, n: int, t: int, q: int):
    """A degree t - 1 polynomial with constant s, evaluated at x = 1..n."""
    co = [s] + [rng.randrange(q) for _ in range(t - 1)]
    return [(x, sum(c * x ** i for i, c in enumerate(co)) % q) for x in range(1, n + 1)]


def share_plain(coords) -> bytes:              # serializeShare(k, a, b, c): four (u64 X, chunk(Y.Bytes()))
    return b"".join(struct.pack(">Q", x) + chunk(y if isinstance(y, bytes) else bts(y)) for x, y in coords)


def phase2_request(kmap) -> bytes:             # serializeSignRequest(nil, nil, kmap): [(id, [encrypted share bytes])]
    out = b"\x00" + struct.pack(">H", len(kmap))
    for nid, shares in kmap:
        out += struct.pack(">QH", nid, len(shares)) + b"".join(chunk(s) for s in shares)
    return out


def phase3_request(m: int, r: int) -> bytes:
    return b"\x01" + chunk(bts(m)) + chunk(bts(r))


def partial_r(g, a: int) -> bytes:             # CalculatePartialR
    if g["kind"] == "dsa":
        return bts(pow(g["g"], a, g["p"]))
    if a % P256["N"] == 0:
        return b"\x04" + bytes(64)
    from cryptography.hazmat.primitives.asymmetric import ec
    pn = ec.derive_private_key(a, ec.SECP256R1()).public_key().public_numbers()
    return b"\x04" + pn.x.to_bytes(32, "big") + pn.y.to_bytes(32, "big")


def phase2(g, plains):
    """Sign's phase 2 over the decrypted shares (plain texts, in request order): (x, k, c, serialized output)."""
    q = order(g)
    x, S = None, [0, 0, 0, 0]
    for pl in plains:
        pos = 0
        for j in range(4):
            cx = struct.unpack(">Q", pl[pos:pos + 8])[0]
            ln = struct.unpack(">Q", pl[pos + 8:pos + 16])[0]
            y = int.from_bytes(pl[pos + 16:pos + 16 + ln], "big")
            pos += 16 + ln
            x = cx if x is None else x
            assert cx == x
            S[j] = (S[j] + y) % q
    k, a, b, c = S
    v = (k * a % q + b) % q
    return x, k, c, struct.pack(">Q", x) + chunk(partial_r(g, a)) + chunk(bts(v)) + group_ser(g)


def phase3(g, X: int, Y: int, m: int, r: int, k: int, c: int) -> bytes:
    q = order(g)
    s = ((r * Y % q + m) % q * k % q + c) % q
    return struct.pack(">Q", X) + chunk(bts(s)) + chunk(b"") + group_ser(g)


def lagrange(xi: int, xs, q: int) -> int:
    num, den = 1, 1
    for xj in xs:
        if xj != xi:
            num, den = num * xj, den * (xj - xi)
    return num * pow(den % q, -1, q) % q


def parse_partial(g, data: bytes):
    x = struct.unpack(">Q", data[:8])[0]
    ln = struct.unpack(">Q", data[8:16])[0]
    s = data[16:16 + ln]
    ln2 = struct.unpack(">Q", data[16 + ln:24 + ln])[0]
    v = int.from_bytes(data[24 + ln:24 + ln + ln2], "big")
    return x, s, v


def calculate_r(g, parts) -> int:              # parts: [(x, R bytes, v)]
    q = order(g)
    xs = [p[0] for p in parts]
    v = sum(vi * lagrange(x, xs, q) for x, _, vi in parts) % q
    vinv = pow(v, -1, q)
    if g["kind"] == "dsa":
        R = 1
        for x, Ri, _ in parts:
            R = R * pow(int.from_bytes(Ri, "big"), lagrange(x, xs, q), g["p"]) % g["p"]
        return pow(R, vinv, g["p"]) % q
    from oracle import sss_oracle as S
    acc = None
    for x, Ri, _ in parts:
        pt = S.p256_mul(lagrange(x, xs, q), (int.from_bytes(Ri[1:33], "big"), int.from_bytes(Ri[33:], "big")))
        acc = pt if acc is None else S.p256_add(acc, pt)
    return S.p256_mul(vinv, acc)[0] % q


def calculate_s(g, parts) -> int:              # parts: [(x, s)]
    q = order(g)
    xs = [p[0] for p in parts]
    return sum(s * lagrange(x, xs, q) for x, s in parts) % q


def format_dsa(r: int, s: int, q: int) -> bytes:
    n = (q.bit_length() + 7) // 8
    return r.to_bytes(n, "big") + s.to_bytes(n, "big")


def _probable_prime(n: int, rng: random.Random) -> bool:
    if n < 2 or any(n % s == 0 for s in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)):
        return n in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)
    d, r = n - 1, 0
    while d % 2 == 0:
        d, r = d // 2, r + 1
    for _ in range(32):
        x = pow(rng.randrange(2, n - 1), d, n)
        if x in (1, n - 1):
            continue
        for _ in range(r - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def dsa_group(pbits=2048, qbits=256, seed=1):
    """A seeded DSA domain: q prime of qbits, p = k q + 1 prime of exactly pbits, g = h^((p - 1) / q) != 1."""
    rng = random.Random(0xD5A0000 + 1000 * pbits + qbits + seed)
    while True:
        q = rng.getrandbits(qbits) | (1 << (qbits - 1)) | 1
        if _probable_prime(q, rng):
            break
    small = [x for x in range(3, 2000, 2) if all(x % y for y in range(3, int(x ** 0.5) + 1, 2))]
    while True:
        k = (rng.getrandbits(pbits - qbits) | (1 << (pbits - qbits - 1))) & ~1
        p = k * q + 1
        if p.bit_length() == pbits and all(p % s for s in small) and _probable_prime(p, rng):
            break
    h = 2
    while pow(h, (p - 1) // q, p) == 1:
        h += 1
    return dict(kind="dsa", p=p, q=q, g=pow(h, (p - 1) // q, p))


def golden_key():
    """The reference's crypto/threshold/dsa/test.pkcs8 (tests/golden/thdsa_key.json): its group and private x."""
    import json
    import os
    d = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "thdsa_key.json")))
    return dict(kind="dsa", p=int(d["p"], 16), q=int(d["q"], 16), g=int(d["g"], 16)), int(d["x"], 16)


def deal(rng: random.Random, g, n: int, t: int, x: int = None):
    """Distribute: the key x (random unless given) and its n shares (X, Y)."""
    q = order(g)
    x = rng.randrange(1, q) if x is None else x
    return x, distribute(rng, x, n, t, q)


def joint_shares(rng: random.Random, g, n: int, t: int):
    """One server's phase 1: k, a (random, degree t - 1) and b, c (zero, degree 2t - 1) shares per node."""
    q = order(g)
    k = distribute(rng, rng.randrange(q), n, t, q)
    a = distribute(rng, rng.randrange(q), n, t, q)
    b = distribute(rng, 0, n, 2 * t, q)
    c = distribute(rng, 0, n, 2 * t, q)
    return [[k[i], a[i], b[i], c[i]] for i in range(n)]
