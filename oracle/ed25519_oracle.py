"""Ed25519 verification as Go's crypto/ed25519.Verify (Go 1.17 and later) decides it, in plain big-integer arithmetic.

    reject S >= L;
    decode A as edwards25519.Point.SetBytes does: y is the low 255 bits reduced mod p (so y in [p, 2^255) is accepted),
        x = +-sqrt((y^2 - 1) / (d y^2 + 1)) picked by the sign bit, and x = 0 with the sign bit set is accepted (x stays 0);
    k = SHA-512(R || A || M) mod L over the caller's raw key bytes;
    accept iff the canonical encoding of [S]B - [k]A equals R's 32 bytes (R itself is never decoded).

OpenSSL decides the same way.  libsodium is stricter: it also rejects small-order A and R and non-canonical A.
Verification is cofactorless: nothing is multiplied by 8.  TEST ORACLE ONLY."""
import hashlib

P = 2 ** 255 - 19
L = 2 ** 252 + 27742317777372353535851937790883648493
D = -121665 * pow(121666, -1, P) % P
SQRT_M1 = pow(2, (P - 1) // 4, P)
IDENTITY = (0, 1)


def add(p, q):
    """Affine Edwards addition (complete on edwards25519: d is not a square)."""
    (x1, y1), (x2, y2) = p, q
    t = D * x1 * x2 * y1 * y2 % P
    return ((x1 * y2 + x2 * y1) * pow(1 + t, -1, P) % P, (y1 * y2 + x1 * x2) * pow(1 - t, -1, P) % P)


def neg(p):
    return (-p[0] % P, p[1])


def mul(k, p):
    """[k] p for k >= 0, in extended coordinates (X : Y : Z : T), x = X/Z, y = Y/Z, xy = T/Z."""
    def ext_add(a, b):
        X1, Y1, Z1, T1 = a
        X2, Y2, Z2, T2 = b
        A = (Y1 - X1) * (Y2 - X2) % P
        B_ = (Y1 + X1) * (Y2 + X2) % P
        C = 2 * D * T1 * T2 % P
        D_ = 2 * Z1 * Z2 % P
        E, F, G, H = B_ - A, D_ - C, D_ + C, B_ + A
        return (E * F % P, G * H % P, F * G % P, E * H % P)
    r = (0, 1, 1, 0)
    q = (p[0], p[1], 1, p[0] * p[1] % P)
    while k:
        if k & 1:
            r = ext_add(r, q)
        q = ext_add(q, q)
        k >>= 1
    zi = pow(r[2], -1, P)
    return (r[0] * zi % P, r[1] * zi % P)


def encode(p):
    """Canonical RFC 8032 encoding: y < p, sign bit = x mod 2."""
    x, y = p
    return (y | ((x & 1) << 255)).to_bytes(32, "little")


def x_of(y, sign):
    """x with x^2 = (y^2 - 1) / (d y^2 + 1) and x mod 2 == sign (x = 0 whatever the sign); None if there is no root."""
    u, v = (y * y - 1) % P, (D * y * y + 1) % P
    x2 = u * pow(v, -1, P) % P
    x = pow(x2, (P + 3) // 8, P)
    if (x * x - x2) % P:
        x = x * SQRT_M1 % P
    if (x * x - x2) % P:
        return None
    if x & 1 != sign:
        x = -x % P
    return x


def decode_go(b):
    """edwards25519.Point.SetBytes: the point, or None."""
    assert len(b) == 32
    y = (int.from_bytes(b, "little") & ((1 << 255) - 1)) % P
    x = x_of(y, b[31] >> 7)
    return None if x is None else (x, y)


def decode_strict(b):
    """RFC 8032 §5.1.3 decoding: also rejects y >= p and x = 0 with the sign bit set."""
    v = int.from_bytes(b, "little")
    y, sign = v & ((1 << 255) - 1), v >> 255
    if y >= P:
        return None
    x = x_of(y, sign)
    if x is None or (x == 0 and sign):
        return None
    return (x, y)


BASE = (x_of(4 * pow(5, -1, P) % P, 0), 4 * pow(5, -1, P) % P)


def challenge(r32, a32, msg):
    return int.from_bytes(hashlib.sha512(r32 + a32 + msg).digest(), "little") % L


def verify(a32, sig, msg):
    """crypto/ed25519.Verify(A, M, sig)."""
    if len(a32) != 32 or len(sig) != 64:
        return False
    S = int.from_bytes(sig[32:], "little")
    if S >= L:
        return False
    A = decode_go(a32)
    if A is None:
        return False
    k = challenge(sig[:32], a32, msg)
    return encode(add(mul(S, BASE), neg(mul(k, A)))) == sig[:32]


def order(p):
    """Order of a point of small order (1, 2, 4 or 8), or None for any other point."""
    for o in (1, 2, 4, 8):
        if mul(o, p) == IDENTITY:
            return o
    return None


def torsion8():
    """A fixed point of order 8: [L] Q for the first y = 2, 3, ... that decodes to a Q whose [L] Q has order 8."""
    y = 2
    while True:
        x = x_of(y, 0)
        if x is not None:
            T = mul(L, (x, y))
            if mul(4, T) != IDENTITY:
                return T
        y += 1


def signed_digits(s, w, nw):
    """The signed radix-2^w recoding the device's window tables use: digits in [-2^(w-1), 2^(w-1) - 1], carries upwards."""
    out, carry = [], 0
    for i in range(nw):
        d = ((s >> (w * i)) & ((1 << w) - 1)) + carry
        carry = (d + (1 << (w - 1))) >> w
        out.append(d - (carry << w))
    return out
