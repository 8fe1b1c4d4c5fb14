"""The client of threshold DSA / ECDSA (crypto/threshold/dsa/dsa_core.go:269-403 dsaProc, dsa.go:33-52, ecdsa.go:36-59)
restated in Python ints on threshold_dsa_oracle's helpers, with the reference's edge behaviour:
  - phase 0 advances when the count of the LAST-listed id of a response reaches 2t (th is overwritten per share);
  - the 2t-th phase-1 answer runs CalculateR and OS2I with its own group, the 2t-th phase-2 answer calculateS mod its q;
  - v.ModInverse(v, q) returns nil and leaves v alone when gcd(v, q) != 1, so DSA's exponent is v itself (r = 1 at v = 0);
  - ECDSA: (0, 0) stands for the point at infinity in CurveParams' Add and ScalarMult, so r = 0 for v = 0 or a sum at
    infinity.  Equal points are doubled (the group law; the duplicate-x case leans on it);
  - where Go panics (Unmarshal's nil point, a Lagrange denominator with no inverse, a short digest, formatDSA's overflow)
    the oracle raises Panic; a framing error raises ParseError, after the peer joined the node list.
step() maps a call to the (state, err, output) the device call reports, a Panic leaving the process failed."""
import math
import struct

import threshold_dsa_oracle as O

PENDING, CONTINUE, SIGNED, FAILED = 0, 1, 2, 3
MALFORMED = -8


class Panic(Exception):
    pass


class ParseError(Exception):
    pass


class Reader:
    def __init__(self, b: bytes):
        self.b, self.pos = b, 0

    def take(self, n: int) -> bytes:
        if len(self.b) - self.pos < n:
            raise ParseError("truncated")
        out = self.b[self.pos:self.pos + n]
        self.pos += n
        return out

    def uint(self, n: int) -> int:
        return int.from_bytes(self.take(n), "big")

    def chunk(self) -> bytes:                  # packet.ReadChunk
        return self.take(self.uint(8))


def joint_share_response(shares) -> bytes:     # serializeJointShare: [(coords bytes, node id)]
    return struct.pack(">H", len(shares)) + b"".join(O.chunk(c) + struct.pack(">Q", nid) for c, nid in shares)


def parse_group(kind: str, r: Reader):
    if kind == "dsa":
        p, q, g = (int.from_bytes(r.chunk(), "big") for _ in range(3))
        return dict(kind="dsa", p=p, q=q, g=g)
    vals = [int.from_bytes(r.chunk(), "big") for _ in range(5)]
    return dict(kind="p256", P=vals[0], N=vals[1], B=vals[2], Gx=vals[3], Gy=vals[4], BitSize=r.uint(4))


def parse_partial(kind: str, data: bytes):     # parsePartialSignature: (group, x, s, v)
    r = Reader(data)
    x = r.uint(8)
    x = x - (1 << 64) if x >> 63 else x        # Go's int(u64)
    s = r.chunk()
    v = int.from_bytes(r.chunk(), "big")
    return parse_group(kind, r), x, s, v


def order(g) -> int:
    return g["q"] if g["kind"] == "dsa" else g["N"]


def lagrange(x: int, xs, q: int) -> int:       # sss.Lagrange: b.ModInverse(b, q) nil -> a.Mul(a, nil) panics
    a, b = 1, 1
    for xj in xs:
        if xj != x:
            a, b = a * xj, b * (xj - x)
    if math.gcd(b % q, q) != 1:
        raise Panic("Lagrange: no inverse")
    return a * pow(b % q, -1, q) % q


def go_mod_inverse(v: int, q: int) -> int:     # v.ModInverse(v, q): nil leaves v unchanged
    return pow(v, -1, q) if math.gcd(v, q) == 1 else v


def unmarshal(b: bytes):                       # elliptic.Unmarshal on P-256
    from oracle import sss_oracle as S
    if len(b) != 65 or b[0] != 4:
        return None
    x, y = int.from_bytes(b[1:33], "big"), int.from_bytes(b[33:], "big")
    if x >= S.P256_P or y >= S.P256_P or (y * y - x ** 3 + 3 * x - S.P256_B) % S.P256_P:
        return None
    return x, y


def calculate_r(g, parts) -> int:              # parts: [(x, R bytes, v)]
    q = order(g)
    xs = [x for x, _, _ in parts]
    v = 0
    if g["kind"] == "dsa":
        r = 1
        for x, Ri, vi in parts:
            lam = lagrange(x, xs, q)
            r = r * pow(int.from_bytes(Ri, "big"), lam, g["p"]) % g["p"]
            v = (v + vi * lam % q) % q
        return pow(r, go_mod_inverse(v, q), g["p"]) % q
    from oracle import sss_oracle as S
    acc = None                                 # None: (0, 0), the point at infinity
    for x, Ri, vi in parts:
        lam = lagrange(x, xs, q)
        pt = unmarshal(Ri)
        if pt is None:
            raise Panic("Unmarshal: nil point")
        acc = S.p256_add(acc, S.p256_mul(lam, pt))
        v = (v + vi * lam % q) % q
    R = S.p256_mul(go_mod_inverse(v, q), acc)
    return 0 if R is None else R[0] % q


def os2i(g, dgst: bytes) -> int:
    q = order(g)
    size = (q.bit_length() + 7) // 8
    if len(dgst) < size:
        raise Panic("OS2I: slice bounds out of range")
    m = int.from_bytes(dgst[:size], "big")
    excess = size * 8 - q.bit_length()
    return m >> excess if g["kind"] == "p256" and excess > 0 else m


def format_dsa(r: int, s: int, q: int) -> bytes:
    n = (q.bit_length() + 7) // 8
    if (r.bit_length() + 7) // 8 > n or (s.bit_length() + 7) // 8 > n:
        raise Panic("formatDSA: the size of the order")
    return r.to_bytes(n, "big") + s.to_bytes(n, "big")


class Proc:
    def __init__(self, kind: str, dgst: bytes, t: int, nodes):
        self.kind, self.dgst, self.t = kind, dgst, t
        self.nodes = list(nodes)
        self.kmap = {}                         # insertion order: the order the device writes
        self.ri, self.si = [], []
        self.phase = 0
        self.m = self.r = self.result = None
        self.failed = None

    def make_request(self):
        if self.phase == 1:
            req = b"\x00" + struct.pack(">H", len(self.kmap) & 0xffff)
            for nid, cs in self.kmap.items():
                req += struct.pack(">QH", nid, len(cs) & 0xffff) + b"".join(O.chunk(c) for c in cs)
        elif self.phase == 2:
            req = b"\x01" + O.chunk(O.bts(self.m)) + O.chunk(O.bts(self.r))
        else:
            req = None
        nodes, self.nodes = self.nodes, []
        return nodes, req

    def process_response(self, data: bytes, peer: int):
        """(result, continue): the result bytes or None, and whether Go returns ErrContinue."""
        self.nodes.append(peer)
        if self.phase == 0:
            r = Reader(data)
            shares = []
            for _ in range(r.uint(2)):
                c = r.chunk()
                shares.append((c, r.uint(8)))
            th = 0
            for c, nid in shares:
                self.kmap.setdefault(nid, []).append(c)
                th = len(self.kmap[nid])
            if th >= 2 * self.t:
                self.phase = 1
                return None, True
            return None, False
        if self.phase == 1:
            g, x, ri, vi = parse_partial(self.kind, data)
            self.ri.append((x, ri, vi))
            if len(self.ri) >= 2 * self.t:
                self.r = calculate_r(g, self.ri)
                self.m = os2i(g, self.dgst)
                self.phase = 2
                return None, True
            return None, False
        if self.phase == 2:
            g, x, si, _ = parse_partial(self.kind, data)
            self.si.append((x, int.from_bytes(si, "big")))
            if len(self.si) >= 2 * self.t:
                q = order(g)
                xs = [x for x, _ in self.si]
                s = 0
                for x, y in self.si:
                    s = (s + y * lagrange(x, xs, q) % q) % q
                self.result = format_dsa(self.r, s, q)
                self.phase = 3
                return self.result, False
            return None, False
        return self.result, False


def step(proc: Proc, op: int, data: bytes = b"", peer: int = 0):
    """One item as the device call reports it: (state, err, output bytes)."""
    if proc.failed is not None:
        return FAILED, proc.failed, b""
    if op == -1:
        nodes, req = proc.make_request()
        return PENDING, 0, struct.pack(">I", len(nodes)) + b"".join(struct.pack(">Q", n) for n in nodes) + (req or b"")
    try:
        res, cont = proc.process_response(data, peer)
    except ParseError:
        return FAILED, MALFORMED, b""
    except Panic:
        proc.failed = MALFORMED
        return FAILED, MALFORMED, b""
    if res is not None:
        return SIGNED, 0, res
    return (CONTINUE if cont else PENDING), 0, b""
