#!/usr/bin/env python3
"""Adversarial ECDSA P-256 and DSA vectors for K1c (p256.cuh), K1d (dsa_verify.cuh) and ECDSA CalculateR, seed 0xBF7C51A0.
Output committed as tests/golden/sig_adversarial.json; the tests read it and generate no domains.

A Byzantine peer picks its own key, digest and signature, so every vector here is built from the verifier's side:

ECDSA (key substitution).  Verification never needs the private key.  For target scalars (u1, u2) and a key Q = c G:
    R = (u1 + c u2) G,  r = R.x mod N,  s = r u2^-1,  e = u1 s        =>  e s^-1 = u1,  r s^-1 = u2.
When R is fixed first (a point of unknown logarithm, or R = k G), Q = u2^-1 (R - u1 G).  The Shamir ladder of
ecdsa_verify_core holds a_i = (u1 >> i) + c (u2 >> i) after bit i, so at bit i the add doubles when
2 a_{i+1} = b1 + c b2 and gives infinity when 2 a_{i+1} = -(b1 + c b2); both are solved for c from a small prefix.
Each vector names the branch it was built for (`tag`); `expect` is the verdict by construction, `status` what
ecdsa_p256_verify_batch returns (3: key not on the curve / non-canonical).  Every vector has a tampered twin.

DSA.  p = m q + 1 and g = h^((p-1)/q), so any q gets a key with known x: composite q = q1 q2 (where w = s^(q-2) is
not s^-1), prime q of 8, 64, 160, 224 and 256 bits with 1024- and 2048-bit p, and a q whose bit length is not a
multiple of 8.  `fermat` marks the signatures made so that the Fermat form of w accepts what dsa.Verify rejects.
Rows with g / y overridden (`g`, `y`: hex, possibly >= p) must go through the raw ABI.

CalculateR.  k partial points R_i whose weighted running sum doubles, passes through infinity, or ends at infinity.
TEST FIXTURE ONLY."""
import json
import os
import random
import sys
from math import gcd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import sss_oracle as so  # noqa: E402

SEED = 0xBF7C51A0
rng = random.Random(SEED)
N, P, G, B = so.P256_N, so.P256_P, so.P256_G, so.P256_B
SMALL = [p for p in range(3, 5000, 2) if all(p % q for q in range(3, int(p ** 0.5) + 1, 2))]


# ---- number theory -------------------------------------------------------------------------------------------------
def is_prime(n):
    if n < 2:
        return False
    for p in SMALL:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d //= 2; s += 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41, 43, 47, 53):
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def rand_prime(bits, top=1):
    """A random prime of exactly `bits` bits whose `top` leading bits are set."""
    while True:
        v = rng.getrandbits(bits) | (((1 << top) - 1) << (bits - top)) | 1
        if is_prime(v):
            return v


def lcm(a, b):
    return a // gcd(a, b) * b


# ---- P-256 ---------------------------------------------------------------------------------------------------------
def mul(k, pt=G):
    return so.p256_mul(k % N, pt)


def add(a, b):
    return so.p256_add(a, b)


def neg(a):
    return None if a is None else (a[0], (-a[1]) % P)


def lift_x(x):
    """A point with abscissa x (x mod p on the curve), or None.  p = 3 mod 4: y = rhs^((p+1)/4)."""
    xr = x % P
    rhs = (xr ** 3 - 3 * xr + B) % P
    y = pow(rhs, (P + 1) // 4, P)
    return (xr, y) if y * y % P == rhs else None


def be32(v):
    return "%064x" % v


def ec_row(tag, Q, r, s, digest, expect, status=None, c=None):
    return {"tag": tag, "qx": be32(Q[0]), "qy": be32(Q[1]), "r": be32(r), "s": be32(s), "digest": digest.hex(),
            "expect": bool(expect), "status": (0 if expect else 1) if status is None else status,
            **({"c": be32(c)} if c is not None else {})}


def sign_subst(u1, u2, c, dlen=32):
    """Key substitution with known c: (Q, r, s, digest) with e s^-1 = u1, r s^-1 = u2; None when R is infinity."""
    R = mul(u1 + c * u2)
    if R is None or R[0] % N == 0:
        return None
    r = R[0] % N
    s = r * pow(u2, -1, N) % N
    e = u1 * s % N
    return mul(c), r, s, digest_of(e, dlen)


def digest_of(e, dlen):
    """A dlen-byte digest whose leftmost min(dlen, 32) bytes read as e (e must fit)."""
    take = min(dlen, 32)
    assert e < 1 << (8 * take)
    return e.to_bytes(take, "big") + bytes(rng.randrange(256) for _ in range(dlen - take))


def sign_with_point(R, u1, u2, r=None, dlen=32, e=None):
    """R fixed first: Q = u2^-1 (R - u1 G), r = R.x mod N (or the given r), s = r u2^-1, digest = e (or u1 s)."""
    Q = mul(pow(u2, -1, N), add(R, neg(mul(u1))))
    r = R[0] % N if r is None else r
    s = r * pow(u2, -1, N) % N
    return Q, r, s, digest_of(u1 * s % N if e is None else e, dlen)


def sign_for_key(Q, u1, u2, dlen=32):
    """Any key, no private key: R = u1 G + u2 Q, r = R.x mod N, s = r u2^-1, e = u1 s."""
    R = add(mul(u1), mul(u2, Q))
    r = R[0] % N
    s = r * pow(u2, -1, N) % N
    return r, s, digest_of(u1 * s % N, dlen)


def tamper(row):
    d = bytearray(bytes.fromhex(row["digest"]))
    take = min(len(d), 32)
    d[rng.randrange(take)] ^= 1 << rng.randrange(8)
    t = dict(row, tag=row["tag"] + "+tampered", digest=bytes(d).hex(), expect=False)
    t.pop("c", None)
    if t["status"] == 0:
        t["status"] = 1
    return t


def ladder_prefix_case(i, idx, sigma):
    """(u1, u2, c) such that the add at bit i of the ladder meets sigma * addend (sigma = +1: doubling, -1: infinity),
    addend = G, Q or G + Q (idx 1, 2, 3)."""
    b1, b2 = idx & 1, idx >> 1
    top = 256 - (i + 1)                                  # prefix bits available above bit i
    for _ in range(64):
        P1 = rng.randrange(1, 1 << min(top, 8)) if top < 8 else rng.randrange(1, 256)
        P2 = rng.randrange(1, 1 << min(top, 8)) if top < 8 else rng.randrange(1, 256)
        den = (2 * P2 - sigma * b2) % N
        if not den:
            continue
        c = (sigma * b1 - 2 * P1) * pow(den, -1, N) % N
        u1 = (P1 << (i + 1)) | (b1 << i) | rng.getrandbits(i) if i else (P1 << 1) | b1
        u2 = (P2 << (i + 1)) | (b2 << i) | rng.getrandbits(i) if i else (P2 << 1) | b2
        if c not in (0, 1, N - 1) and u1 < N and 0 < u2 < N:       # Q = +-G would turn it into a table case
            return u1, u2, c
    return None                                          # at bit 254 the only prefix (1, 1) forces Q = -G for G + Q


def ecdsa_vectors():
    rows = []

    def push(row, twin=True):
        rows.append(row)
        if twin:
            rows.append(tamper(row))

    # in-loop doubling / infinity against each addend, at several bit positions
    for i in (254, 200, 129, 64, 31, 1, 0):
        for idx in (1, 2, 3):
            for sigma, tag in ((1, "loop_double"), (-1, "loop_infinity")):
                case = ladder_prefix_case(i, idx, sigma)
                out = case and sign_subst(*case)
                if out is None:
                    continue
                Q, r, s, d = out
                push(ec_row("%s/%s@%d" % (tag, "G Q GQ".split()[idx - 1], i), Q, r, s, d, True, c=case[2]))
    # the accumulator back at infinity mid-loop and then added to: a_{i} = 0 for a prefix, with more bits below
    for i in (180, 90, 12):
        case = ladder_prefix_case(i, 3, -1)
        Q, r, s, d = sign_subst(*case)
        push(ec_row("acc_inf_mid@%d" % i, Q, r, s, d, True, c=case[2]))
    # the table entry G + Q: Q = G doubles, Q = -G gives infinity (then every idx = 3 step adds infinity)
    for c, tag in ((1, "table_double"), (N - 1, "table_infinity")):
        for _ in range(3):
            out = sign_subst(rng.randrange(1, N), rng.randrange(1, N), c)
            if out:
                Q, r, s, d = out
                push(ec_row(tag, Q, r, s, d, True, c=c))
    # u1 = u2
    for _ in range(2):
        u = rng.randrange(1, N)
        c = rng.randrange(2, N)
        Q, r, s, d = sign_subst(u, u, c)
        push(ec_row("u1_eq_u2", Q, r, s, d, True, c=c))
    # u1 = 0: the digest is all zeros, or reads exactly N
    for e, dig in ((0, bytes(32)), (0, N.to_bytes(32, "big"))):
        k = rng.randrange(1, N)
        Q, r, s, _ = sign_with_point(mul(k), 0, rng.randrange(1, N), e=0)
        push(ec_row("u1_zero" if dig == bytes(32) else "u1_zero/z_eq_n", Q, r, s, dig, True))
    # u1 / u2 with many leading zero bits
    for bits1, bits2 in ((40, 256), (256, 40), (8, 8), (1, 200)):
        u1 = rng.getrandbits(bits1) | 1
        u2 = rng.getrandbits(bits2) | 1
        u1 %= N; u2 %= N
        c = rng.randrange(2, N)
        out = sign_subst(u1, u2, c)
        if out:
            Q, r, s, d = out
            push(ec_row("short_scalars/%d_%d" % (bits1, bits2), Q, r, s, d, True, c=c))
    # a result at infinity: u1 + c u2 = 0; rejected whatever r is
    for _ in range(3):
        u2, c = rng.randrange(1, N), rng.randrange(2, N)
        u1 = (-c * u2) % N
        r = rng.randrange(1, N)
        s = r * pow(u2, -1, N) % N
        push(ec_row("result_inf", mul(c), r, s, digest_of(u1 * s % N, 32), False, c=c))
    # e >= N: the same e plus N (fits 32 bytes only when e < 2^256 - N)
    for _ in range(3):
        e = rng.randrange(1, (1 << 256) - N)
        k = rng.randrange(1, N)
        sv = rng.randrange(1, N)
        R = mul(k)
        r = R[0] % N
        u1, u2 = e * pow(sv, -1, N) % N, r * pow(sv, -1, N) % N
        Q, r, s, _ = sign_with_point(R, u1, u2)
        assert s == sv
        push(ec_row("z_ge_n", Q, r, s, (e + N).to_bytes(32, "big"), True))
        push(ec_row("z_lt_n", Q, r, s, e.to_bytes(32, "big"), True), twin=False)
    # digest lengths 20, 28, 32, 48, 64 (hashToInt: leftmost 32 bytes)
    for dlen in (20, 28, 32, 48, 64):
        for _ in range(2):
            e = rng.getrandbits(8 * min(dlen, 32)) % N
            k, sv = rng.randrange(1, N), rng.randrange(1, N)
            R = mul(k)
            r = R[0] % N
            Q, r, s, d = sign_with_point(R, e * pow(sv, -1, N) % N, r * pow(sv, -1, N) % N, dlen=dlen, e=e)
            push(ec_row("dlen_%d" % dlen, Q, r, s, d, True))
    # R.x in [N, p): r = t is valid, r = t + 1 is not, r = x fails the range check
    t = 0
    found = 0
    while found < 3:
        R = lift_x(N + t)
        if R is not None:
            for sgn in (R, neg(R)) if found == 0 else (R,):
                u1, u2 = rng.randrange(1, N), rng.randrange(1, N)
                Q, r, s, d = sign_with_point(sgn, u1, u2)
                assert r == t
                push(ec_row("x_ge_n/t=%d" % t, Q, r, s, d, True))
                for rr, tag in ((t + 1, "x_ge_n/r=t+1"), (N + t, "x_ge_n/r=x")):
                    s2 = rr * pow(u2, -1, N) % N
                    rows.append(ec_row(tag, Q, rr, s2, digest_of(u1 * s2 % N, 32), False))
            found += 1
        t += 1
    # r or s equal to 1 or N - 1
    for sv in (1, N - 1):
        k = rng.randrange(1, N)
        R = mul(k)
        r = R[0] % N
        u1 = rng.randrange(1, N)
        Q, r, s, d = sign_with_point(R, u1, r * pow(sv, -1, N) % N)
        assert s == sv
        push(ec_row("s=%s" % ("1" if sv == 1 else "N-1"), Q, r, s, d, True))
    for rv, xs in ((1, (1, N + 1)), (N - 1, (N - 1,))):
        for x in xs:
            R = lift_x(x)
            if R is None:
                continue
            u1, u2 = rng.randrange(1, N), rng.randrange(1, N)
            Q, r, s, d = sign_with_point(R, u1, u2)
            assert r == rv
            push(ec_row("r=%s/x=%s" % ("1" if rv == 1 else "N-1", "N+1" if x == N + 1 else ("1" if x == 1 else "N-1")), Q, r, s, d, True))
    # a key whose X >= p is on the curve once reduced: non-canonical, status 3 (elliptic.Unmarshal refuses it)
    x0 = 1
    while lift_x(x0) is None:
        x0 += 1
    Q0 = lift_x(x0)
    r, s, d = sign_for_key(Q0, rng.randrange(1, N), rng.randrange(1, N))
    rows.append(ec_row("key_x_ge_p", (Q0[0] + P, Q0[1]), r, s, d, False, status=3))
    push(ec_row("key_x_ge_p/reduced", Q0, r, s, d, True))                  # the same key written canonically
    return rows


# ---- CalculateR ----------------------------------------------------------------------------------------------------
def calc_r_rows():
    rows = []
    xs3 = [1, 2, 3]
    xs2 = [2, 5]

    def lam(x, xs):
        return so.lagrange(x, xs, N)

    def row(tag, xs, pts, vis):
        acc = None
        for x, R in zip(xs, pts):
            acc = add(acc, mul(lam(x, xs), R))
        v = sum(vi * lam(x, xs) for x, vi in zip(xs, vis)) % N
        Rf = mul(pow(v, -1, N), acc) if acc is not None else None
        return {"tag": tag, "x": xs, "points": [so.p256_marshal(p).hex() for p in pts], "v": [be32(vi) for vi in vis],
                "status": 0 if Rf is not None else 3, "r": be32(Rf[0] % N if Rf is not None else 0)}

    for _ in range(2):
        R0 = mul(rng.randrange(1, N))
        l0, l1 = lam(xs2[0], xs2), lam(xs2[1], xs2)
        R1 = mul(l0 * pow(l1, -1, N), R0)                     # l1 R1 = l0 R0: the running sum doubles
        rows.append(row("sum_double", xs2, [R0, R1], [rng.randrange(1, N) for _ in xs2]))
        R1n = neg(R1)                                          # l1 R1 = -l0 R0: the sum ends at infinity
        rows.append(row("sum_inf_end", xs2, [R0, R1n], [rng.randrange(1, N) for _ in xs2]))
        m0, m1 = lam(xs3[0], xs3), lam(xs3[1], xs3)
        Ra = mul(rng.randrange(1, N))
        Rb = neg(mul(m0 * pow(m1, -1, N), Ra))                 # infinity after two terms, then a third
        rows.append(row("sum_inf_mid", xs3, [Ra, Rb, mul(rng.randrange(1, N))], [rng.randrange(1, N) for _ in xs3]))
        Rc = mul(m0 * pow(m1, -1, N), Ra)                      # doubling, then a third term equal to the doubled sum
        m2 = lam(xs3[2], xs3)
        Rd = mul(2 * m0 * pow(m2, -1, N), Ra)
        rows.append(row("sum_double_twice", xs3, [Ra, Rc, Rd], [rng.randrange(1, N) for _ in xs3]))
    return rows


# ---- DSA -----------------------------------------------------------------------------------------------------------
def dsa_domain(name, q, pbits, factors=None):
    """p = m q + 1 prime of exactly pbits bits, g of order q (checked on every prime factor of q)."""
    qf = factors or [q]
    while True:
        m = rng.getrandbits(pbits - q.bit_length()) | (1 << (pbits - q.bit_length() - 1))
        m -= m % 2
        p = m * q + 1
        if p.bit_length() != pbits:
            continue
        if any(p % sp == 0 for sp in SMALL):
            continue
        if is_prime(p):
            break
    h = 2
    while True:                                   # g + p and y + p still fit plen bytes (the g, y >= p rows)
        g = pow(h, (p - 1) // q, p)
        if g != 1 and g + p < 1 << pbits and all(pow(g, q // f, p) != 1 for f in qf):
            break
        h += 1
    while True:
        x = rng.randrange(1, q)
        if pow(g, x, p) + p < 1 << pbits:
            break
    return {"name": name, "p": p, "q": q, "g": g, "x": x, "y": pow(g, x, p), "factors": qf}


def composite_q(bits):
    """q = q1 q2 with |q| = bits and gcd(q - 2, lambda(q)) = 1, so the Fermat form can be steered."""
    while True:
        q1 = rand_prime(bits // 2, top=2)
        q2 = rand_prime(bits // 2, top=2)
        q = q1 * q2
        if q1 != q2 and q.bit_length() == bits and gcd(q - 2, lcm(q1 - 1, q2 - 1)) == 1:
            return q, [q1, q2]


def dsa_sign(D, z, k=None):
    """(r, s) with r = (g^k mod p) mod q, s = k^-1 (z + x r) mod q; k, r, s all invertible."""
    p, q, g, x = D["p"], D["q"], D["g"], D["x"]
    while True:
        kk = k if k is not None else rng.randrange(1, q)
        r = pow(g, kk, p) % q
        t = (z + x * r) % q
        if r and gcd(kk, q) == 1 and gcd(t, q) == 1:
            return kk, r, pow(kk, -1, q) * t % q
        if k is not None:
            return None


def zval(D, digest):
    sub = (D["q"].bit_length() + 7) // 8
    return int.from_bytes(digest[:sub], "big")


def dsa_vectors():
    doms = []
    for qbits in (160, 256):
        q, f = composite_q(qbits)
        for pbits in (1024, 2048):
            doms.append(dsa_domain("comp%d_p%d" % (qbits, pbits), q, pbits, f))
    for name, qbits, pbits in (("q8_p1024", 8, 1024), ("q64_p1024", 64, 1024), ("q224_p2048", 224, 2048),
                               ("q160_p2048", 160, 2048), ("q256_p1024", 256, 1024), ("q160_p1024", 160, 1024)):
        q = 251 if qbits == 8 else rand_prime(qbits)
        doms.append(dsa_domain(name, q, pbits))
    doms.append(dsa_domain("q159_p1024", rand_prime(159), 1024))          # bit length not a multiple of 8
    rows = []

    def rowd(D, tag, digest, r, s, expect, twin=True, **kw):
        row = {"domain": D["name"], "tag": tag, "digest": digest.hex(), "r": be32(r), "s": be32(s), "expect": bool(expect), **kw}
        rows.append(row)
        if twin:
            gg, yy = int(kw.get("g", "%x" % D["g"]), 16), int(kw.get("y", "%x" % D["y"]), 16)
            while True:                                            # a small q can accept a tampered digest by chance
                d = bytearray(digest)
                sub = min(len(d), (D["q"].bit_length() + 7) // 8)
                d[rng.randrange(sub)] ^= 1 << rng.randrange(8)
                if not dsa_verify_int(D["p"], D["q"], gg, yy, bytes(d), r, s):
                    break
            rows.append(dict(row, tag=tag + "+tampered", digest=bytes(d).hex(), expect=False))

    def rdig(n):
        return bytes(rng.randrange(256) for _ in range(n))

    for D in doms:
        p, q, g, y, x = D["p"], D["q"], D["g"], D["y"], D["x"]
        qlen = (q.bit_length() + 7) // 8
        ok = q.bit_length() % 8 == 0
        dl = 20 if qlen <= 20 else 32
        for _ in range(3):
            d = rdig(dl)
            _, r, s = dsa_sign(D, zval(D, d))
            rowd(D, "honest", d, r, s, ok)
        if len(D["factors"]) > 1:
            q1, q2 = D["factors"]
            lam = lcm(q1 - 1, q2 - 1)
            ei = pow(q - 2, -1, lam)
            n_craft = 0
            while n_craft < 3:
                d = rdig(dl)
                z = zval(D, d)
                k = rng.randrange(1, q)
                r = pow(g, k, p) % q
                t = (z + x * r) % q
                if not r or gcd(t, q) != 1 or gcd(k, q) != 1:
                    continue
                wf = k * pow(t, -1, q) % q                         # the w that makes g^(z w) y^(r w) = g^k
                s = pow(wf, ei, q)                                 # s^(q-2) = wf: accepted by the Fermat form
                assert pow(s, q - 2, q) == wf
                rowd(D, "fermat_crafted", d, r, s, False, fermat=True)
                n_craft += 1
            for f in (q1, q2):
                s = f * rng.randrange(1, q // f)                   # gcd(s, q) > 1: ModInverse returns nil
                rowd(D, "s_not_invertible", rdig(dl), rng.randrange(1, q), s, False, twin=False)
            s = q1                                                 # the factor itself, with a verdict-steering r
            rowd(D, "s_eq_factor", rdig(dl), pow(g, 5, p) % q or 1, s, False, twin=False)
        # digests: z >= q after truncation, z = 0 mod q, z = 0, short (20 bytes) and long (64 bytes)
        dff = b"\xff" * max(dl, qlen)
        _, r, s = dsa_sign(D, zval(D, dff))
        rowd(D, "z_ge_q", dff, r, s, ok)
        dq = q.to_bytes(qlen, "big") + rdig(max(dl, qlen) - qlen)
        _, r, s = dsa_sign(D, 0)
        rowd(D, "z_eq_q", dq, r, s, ok)
        rowd(D, "z_zero", bytes(max(dl, qlen)), r, s, ok)
        for n in (20, 64):
            d = rdig(n)
            _, r, s = dsa_sign(D, zval(D, d))
            rowd(D, "dlen_%d" % n, d, r, s, ok)
        # r and s at q - 1 and 1 (s steered through the digest: z = s k - x r)
        k = rng.randrange(1, q)
        r0 = pow(g, k, p) % q
        for sv in (1, q - 1):
            z = (sv * k - x * r0) % q
            d = z.to_bytes(qlen, "big") + rdig(dl - qlen)
            good = gcd(sv, q) == 1 and r0 != 0
            rowd(D, "s=%s" % ("1" if sv == 1 else "q-1"), d, r0, sv, ok and good)
        for rv in (1, q - 1):
            d = rdig(dl)
            s = rng.randrange(1, q)
            while dsa_verify_int(p, q, g, y, d, rv, s):
                s = rng.randrange(1, q)
            rowd(D, "r=%s" % ("1" if rv == 1 else "q-1"), d, rv, s, False, twin=False)
        # r or s >= q with bytes above qlen set (q shorter than 32 bytes)
        if qlen < 32:
            d = rdig(dl)
            _, r, s = dsa_sign(D, zval(D, d))
            rowd(D, "r_high_bytes", d, r + (1 << (8 * qlen)), s, False, twin=False)
            rowd(D, "s_high_bytes", d, r, s + (1 << (8 * qlen)), False, twin=False)
            rowd(D, "r_plus_q", d, r + q, s, False, twin=False)
        # g = 1, y = 1, y = p - 1 (public values a peer can choose), and g / y >= p written in plen bytes
        plen = (p.bit_length() + 7) // 8
        d = rdig(dl)
        _, r, s = dsa_sign(D, zval(D, d))
        for tag, gg, yy in (("g=1", 1, y), ("y=1", g, 1), ("y=p-1", g, p - 1)):
            rowd(D, tag, d, r, s, None, twin=False, g="%x" % gg, y="%x" % yy)
        rowd(D, "g_ge_p", d, r, s, ok, g="%x" % (g + p), y="%x" % y, raw=True)
        rowd(D, "y_ge_p", d, r, s, ok, g="%x" % g, y="%x" % (y + p), raw=True)
        rowd(D, "y_all_ones", d, r, s, None, twin=False, g="%x" % g, y="%x" % ((1 << (8 * plen)) - 1), raw=True)
    out_doms = [{"name": D["name"], **{k: "%x" % D[k] for k in ("p", "q", "g", "x", "y")},
                 "factors": ["%x" % f for f in D["factors"]]} for D in doms]
    # expect None: decided by the group law, not by construction; fill it from dsa.Verify restated in integers
    byname = {D["name"]: D for D in doms}
    for row in rows:
        if row["expect"] is None:
            D = byname[row["domain"]]
            row["expect"] = dsa_verify_int(D["p"], D["q"], int(row.get("g", "%x" % D["g"]), 16), int(row.get("y", "%x" % D["y"]), 16),
                                           bytes.fromhex(row["digest"]), int(row["r"], 16), int(row["s"], 16))
            row["by"] = "restated"
    return out_doms, rows


def dsa_verify_int(p, q, g, y, digest, r, s):
    """Go crypto/dsa.Verify after x/crypto's digest cut, in plain integers (extended Euclid for ModInverse)."""
    digest = digest[:(q.bit_length() + 7) // 8]
    if not (0 < r < q and 0 < s < q):
        return False
    a, b, u, v = s, q, 1, 0
    while b:
        t = a // b
        a, b, u, v = b, a - t * b, v, u - t * v
    if a != 1 or q.bit_length() % 8:
        return False
    w = u % q
    z = int.from_bytes(digest, "big")
    return pow(g, z * w % q, p) * pow(y, r * w % q, p) % p % q == r


def main():
    ec = ecdsa_vectors()
    cr = calc_r_rows()
    doms, dsa = dsa_vectors()
    out = {"seed": "0x%X" % SEED, "ecdsa": ec, "calc_r": cr, "dsa_domains": doms, "dsa": dsa}
    path = os.path.join(HERE, "sig_adversarial.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", path, len(ec), "ECDSA,", len(cr), "CalculateR,", len(dsa), "DSA rows")


if __name__ == "__main__":
    main()
