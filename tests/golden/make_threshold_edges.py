#!/usr/bin/env python3
"""Edge vectors for the share-combine arithmetic, seed 0xBF7C7E00.  Output committed as tests/golden/threshold_edges.json.

K3 (lagrange_combine_kernel<L>, lagrange.cuh): Shamir combines S = sum_i lambda_i y_i mod m with lambda_i from
oracle/sss_oracle.py, which restates Go's sss.Lagrange (unreduced numerator and denominator, ModInverse of a possibly
negative denominator).  A combine whose denominator has no inverse (Go: nil, then a panic) is status 3, out zero.
  moduli      one per limb class and at each class boundary (mlen 1, 4, 5, 31..33, 63..65, 127..129, 255, 256),
              2^(32 j) +- c, odd m < 2^32, and composite m (small primes, and a product of two primes that only one
              32-bit denominator chunk covers as a whole);
  abscissae   node indices, large positive and negative values, 0, INT32_MIN with INT32_MAX, duplicates;
  shapes      k = 1, 2, 10, 255; y = 0, m - 1 and y >= m (still mlen bytes).
K5 (modexp_kernel<W> / modprod_kernel<W>, modexp.cuh): W = 8 and 16 moduli at 2^(128 W - 1) + c and 2^(128 W) - c;
bases 0, 1, n - 1, n, 2^(128 W) - 1; exponents 0, 1, all-ones, a single top bit, elen 1, 3, 21, 33, 129, 256; warps of
eight items that mix exponent lengths; products with k = 1 and 2 on inputs >= n.
lagrange_exp_product: prod y_i^lambda_i mod p with q in each K3 limb class.
dsa.CalculateR on L1024/N160 (dsa_test.go's domain), and generated L2048/N224 and L2048/N256 domains, with items whose
sum v_i lambda_i is 0 mod q (Go: ModInverse returns nil and r = 1; the device: status 3).
Operands are tokens and outputs a digest per record (tests/threshold_edges.py decodes them); the tests recompute every
output with sss_oracle / pow and check it against the digest.
TEST FIXTURE ONLY."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
from oracle import sss_oracle as so  # noqa: E402
import threshold_edges as te  # noqa: E402

SEED = 0xBF7C7E00
rng = random.Random(SEED)
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
SMALL = [p for p in range(3, 2000, 2) if all(p % q for q in range(3, int(p ** 0.5) + 1, 2))]


def is_prime(n):
    if n < 2:
        return False
    for p in SMALL:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d //= 2; s += 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
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


def rand_prime(bits):
    while True:
        v = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
        if is_prime(v):
            return v


def h(v):
    return format(v, "x")


def combine(m, xs, ys):
    """(out, status) as the device reports them."""
    try:
        return so.calculate_secret(list(zip(xs, ys)), m), 0
    except ValueError:
        return 0, 3


def abscissae(kind, k):
    if kind == "node":
        return rng.sample(range(1, max(k, 15) + 1), k)
    if kind == "large":
        return [rng.choice((1, -1)) * rng.randrange(1 << 30, 1 << 31) for _ in range(k)]
    if kind == "int32":
        return [rng.randrange(I32_MIN, I32_MAX + 1) for _ in range(k)]
    if kind == "zero":
        xs = [rng.randrange(-1000, 1000) for _ in range(k)]
        xs[rng.randrange(k)] = 0
        return xs
    if kind == "extremes":
        xs = [I32_MIN, I32_MAX] + [rng.choice((I32_MIN + 1, I32_MAX - 1, -1, 1, rng.randrange(I32_MIN, I32_MAX))) for _ in range(k - 2)]
        rng.shuffle(xs)
        return xs
    if kind == "dups":
        base = [rng.randrange(-50000, 50000) for _ in range(max(1, k // 2))]
        return [rng.choice(base) for _ in range(k)]
    if kind == "small_signed":
        return rng.sample(range(-20, 21), k) if k <= 41 else [rng.randrange(-300, 301) for _ in range(k)]
    raise ValueError(kind)


def share_tokens(k, mode):
    """"edges": each share one of 0, 1, m - 1, m, 2^(8 mlen) - 1, >= m, random; "small": three edges, then below 2^48."""
    return "".join(rng.choice("01-nTGrr") if (mode == "edges" or i < 3) else "s" for i in range(k))


K3_GROUPS, MODULI = [], {}


def k3_group(tag, m, k, rows):
    """rows: [(xs, share tokens)].  The modulus goes to MODULI once, by name."""
    name = next((nm for nm, v in MODULI.items() if v == h(m)), None)
    if name is None:
        name = "m%d" % len(MODULI)
        MODULI[name] = h(m)
    g = {"tag": tag, "m": name, "k": k, "items": [{"x": xs, "y": y} for xs, y in rows]}
    _, _, items = te.k3_items(g, MODULI)
    res = [combine(m, xs, ys) for xs, ys in items]
    g["status"] = [st for _, st in res]
    g["digest"] = te.digest(g["status"], [o for o, _ in res], te.mlen_of(m))
    K3_GROUPS.append(g)


def k3_kinds(tag, m, k, kinds, mode="edges"):
    k3_group(tag, m, k, [(abscissae(kind, k), share_tokens(k, mode)) for kind in kinds])


def k3_vectors():
    moduli = []
    for ml in (1, 4, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256):            # random odd, and primes
        bits = 8 * ml
        moduli.append(("rand%d" % ml, (rng.getrandbits(bits) | (1 << (bits - 1)) | 1) if ml > 1 else 0xC3))
        if ml in (4, 32, 33, 64, 65, 128, 256):
            moduli.append(("prime%d" % ml, rand_prime(bits)))
    for j in (1, 2, 8, 16, 32, 64):                                                      # 2^(32 j) +- c
        c = rng.randrange(1, 1 << 16) | 1
        moduli.append(("pow2_%d_minus" % j, (1 << (32 * j)) - c))
        moduli.append(("pow2_%d_plus" % j, (1 << (32 * j)) + c) if j < 64 else ("pow2_%d_minus1" % j, (1 << (32 * j)) - 1))
    moduli.append(("pow2_1_minus1", (1 << 32) - 1))
    for m in (3, 5, 1237, (1 << 31) - 1, (1 << 32) - 5):                                # odd m < 2^32
        moduli.append(("small%d" % m, m))
    moduli += [("comp15", 15), ("comp15015", 3 * 5 * 7 * 11 * 13), ("comp9x25", 9 * 25 * 49),
               ("comp_p31xq", 2147483647 * rand_prime(100)), ("comp_2p", 65537 * 65539 * rand_prime(160))]
    for tag, m in moduli:
        k3_kinds(tag + "_k1", m, 1, ["int32"])
        k3_kinds(tag + "_k2", m, 2, ["int32", "extremes", "zero"])
        k3_kinds(tag + "_k10", m, 10, ["node", "large", "int32", "zero", "extremes", "dups", "small_signed"])
    # k = 255 in every limb class (small shares after three edges)
    for tag, m, kinds in [("k255_prime4", rand_prime(32), ["node", "int32"]), ("k255_p256n", so.P256_N, ["node", "large"]),
                          ("k255_prime33", rand_prime(264), ["node"]), ("k255_prime65", rand_prime(520), ["node"]),
                          ("k255_m256", [m for t, m in moduli if t == "prime256"][0], ["node", "int32"]),
                          ("k255_small1237", 1237, ["small_signed"])]:
        k3_kinds(tag, m, 255, kinds, mode="small")
    # chunk flushes at chosen places: numerator chunk 65535 * 65537 = 2^32 - 1 (no flush), then a third factor (flush);
    # denominators 2^32 - 1 (INT32_MIN vs INT32_MAX) and 2^31 (INT32_MIN vs 0)
    crafted = [[65535, 65537, 3, -3], [I32_MIN, I32_MAX, 0], [I32_MIN, 0, 1], [I32_MAX, -1, 1, 2],
               [1 << 16, -(1 << 16), 1 << 15, -(1 << 15), 1], [I32_MIN, I32_MIN + 1, I32_MAX, I32_MAX - 1]]
    for tag, m in [("crafted_p256n", so.P256_N), ("crafted_2p31m1", (1 << 31) - 1), ("crafted_1237", 1237),
                   ("crafted_comp", 65537 * 65539 * 7)]:
        for xs in crafted:
            k3_group("%s_%d" % (tag, len(xs)), m, len(xs), [(xs, "r" * len(xs))])
    # composite m = 77 q: a denominator chunk whose factors carry 7 and 11 separately (the chunk is 0 mod 77)
    m = 77 * rand_prime(64)
    for i, xs in enumerate(([0, 7, 18], [1, 8, 12], [1, 8, 19], [100, 107, 111])):
        k3_group("chunk_gcd_77_%d" % i, m, 3, [(xs, "rrr")])


MODEXP, MODPROD = [], []


def k5_vectors():
    moduli = []
    for W in (8, 16):
        bits = 128 * W
        c = rng.randrange(1, 1 << 20) | 1
        moduli += [("W%d_low_%d" % (W, c), W, (1 << (bits - 1)) + c), ("W%d_high_1" % W, W, (1 << bits) - 1)]
        if W == 8:
            moduli += [("W%d_low_1" % W, W, (1 << (bits - 1)) + 1), ("W%d_high_%d" % (W, c), W, (1 << bits) - c)]
    for tag, W, n in moduli:
        bases_edge, exps_edge = "01-nTrG2", "01TBf23h"
        for elen in (1, 3, 21, 33, 129, 256) if W == 8 else (1, 3, 33, 256):
            # warp 1: every edge base next to exponents of every length class, zeros among them; warp 2 (W = 8): one
            # random base, every exponent; warp 3: all-ones exponents next to zero exponents
            bases = bases_edge + ("r" * 8 if W == 8 else "") + "".join(bases_edge[(i + 3) % 8] for i in range(8))
            exps = "".join(exps_edge[(i * 3) % 8] for i in range(8)) + (exps_edge if W == 8 else "") + "0T" * 4
            r = {"tag": "%s_e%d" % (tag, elen), "n": h(n), "elen": elen, "base": bases, "exp": exps}
            _, bs, es = te.modexp_operands(r)
            r["digest"] = te.digest([0] * len(bs), [pow(b, e, n) for b, e in zip(bs, es)], 16 * W)
            MODEXP.append(r)
        for k, rows in ((1, ["0", "1", "-", "n", "+", "T", "G", "r"]), (2, ["TT", "nT", "--", "+-", "0T", "1T", "T1", "rT"])):
            r = {"tag": "%s_k%d" % (tag, k), "n": h(n), "k": k, "vals": rows}
            _, vals = te.modprod_rows(r)
            outs = [(row[0] * (row[1] if k == 2 else 1)) % n for row in vals]
            r["digest"] = te.digest([0] * len(outs), outs, 16 * W)
            MODPROD.append(r)


EXP_PRODUCT, DSA = [], []


def dsa_domain(lbits, nbits):
    q = rand_prime(nbits)
    while True:
        r = rng.getrandbits(lbits - nbits) | (1 << (lbits - nbits - 1))
        p = q * r * 2 + 1
        if p.bit_length() == lbits and is_prime(p):
            break
    while True:
        g = pow(rng.randrange(2, p - 1), (p - 1) // q, p)
        if g != 1:
            return p, q, g


def exp_product_vectors(golden_p1024):
    p2048 = rand_prime(2048)
    for p in (golden_p1024, p2048):
        for qbytes in (20, 33, 64, 65, 128, 129, 256):
            if qbytes > te.mlen_of(p):
                continue
            q = rand_prime(8 * qbytes) if qbytes <= 65 else (rng.getrandbits(8 * qbytes) | (1 << (8 * qbytes - 1)) | 1)
            rows = [{"x": abscissae(kind, k), "y": "".join(rng.choice("01-nrr") for _ in range(k))}
                    for kind, k in (("node", 5), ("int32", 3), ("large", 4), ("zero", 3), ("dups", 4), ("node", 1))]
            r = {"tag": "p%d_q%d" % (p.bit_length(), qbytes), "p": h(p), "q": h(q), "rows": rows}
            outs, sts = [], []
            for xs, ys in te.exp_product_rows(r)[2]:
                try:
                    out = 1
                    for y, l in zip(ys, [so.lagrange(x, xs, q) for x in xs]):
                        out = out * pow(y, l, p) % p
                    outs.append(out); sts.append(0)
                except ValueError:
                    outs.append(0); sts.append(3)
            r["status"], r["digest"] = sts, te.digest(sts, outs, te.mlen_of(p))
            EXP_PRODUCT.append(r)


def dsa_vectors(name, p, q, g):
    d = {"domain": name, "p": h(p), "q": h(q), "g": h(g), "items": []}
    zero_v = []
    for case in range(14):
        k = [8, 8, 3, 2, 1, 8, 5, 8, 4, 8, 8, 3, 6, 2][case]
        kind = ["node", "node", "large", "int32", "node", "extremes", "zero", "node", "small_signed", "dups", "node", "int32",
                "node", "node"][case]
        R = ("nT" + "g" * (k - 2)) if case == 1 else "g" * k                      # R_i >= p is reduced, like big.Int.Exp
        d["items"].append({"x": abscissae(kind, k), "R": R, "v": "r" * k})
        zero_v.append(case in (7, 10, 11))
    # solve one v_j per zero_v item so that sum v_i lambda_i == 0 mod q (a Byzantine last share)
    for it, (xs, _, vs), z in zip(d["items"], dsa_items_(d), zero_v):
        if z:
            lams = [so.lagrange(x, xs, q) for x in xs]
            j = next(i for i, l in enumerate(lams) if l % q)
            rest = sum(v * l for i, (v, l) in enumerate(zip(vs, lams)) if i != j) % q
            it["v"] = ["r"] * len(xs)
            it["v"][j] = "x" + h((-rest * pow(lams[j], -1, q)) % q)
    outs, sts = [], []
    for (xs, Rs, vs), z in zip(dsa_items_(d), zero_v):
        try:
            outs.append(so.dsa_calculate_r(list(zip(xs, Rs, vs)), p, q)); sts.append(0)
        except ValueError:
            outs.append(0); sts.append(3)
        assert (sts[-1] == 3) == z
    d["status"], d["zero_v"], d["digest"] = sts, [int(z) for z in zero_v], te.digest(sts, outs, te.mlen_of(q))
    DSA.append(d)


def dsa_items_(d):
    return te.dsa_items(d)[2]


FERMAT, REDUCE = [], []


def host_vectors():
    """fermat_pow (v^(m-2) mod m) and limbs::reduce_be (v mod m); the tests compute the reference with pow and %."""
    for m in (3, 5, 1237, (1 << 31) - 1, (1 << 32) - 5, rand_prime(64), rand_prime(160), rand_prime(224), so.P256_N,
              (1 << 255) - 19, (1 << 256) - 189, rand_prime(264), rand_prime(512), 15015, (1 << 256) - 1,
              rng.getrandbits(1024) | (1 << 1023) | 1, rng.getrandbits(2048) | (1 << 2047) | 1):
        FERMAT.append({"m": h(m), "v": "012-=rs" if m > 5 else "012-"})
    for m in (3, 1237, (1 << 32) - 5, (1 << 32) + 15, rand_prime(160), rand_prime(224), so.P256_N, (1 << 256) - 1):
        for nbytes in (1, 4, 20, 31, 32, 33, 128, 256) + ((512,) if m.bit_length() in (160, 256) else ()):
            top = (1 << (8 * nbytes)) - 1
            toks = "0Tf" + "".join(t for t, v in (("n", m), ("-", m - 1), ("D", 2 * m), ("M", m), ("L", m)) if v <= top)
            REDUCE.append({"m": h(m), "nbytes": nbytes, "v": toks})


def main():
    golden = json.load(open(os.path.join(HERE, "golden.json")))
    dp, dq, dg = (int(golden["dsa_test"][k], 16) for k in "PQG")
    k3_vectors()
    k5_vectors()
    exp_product_vectors(dp)
    dsa_vectors("L1024N160", dp, dq, dg)
    dsa_vectors("L2048N224", *dsa_domain(2048, 224))
    dsa_vectors("L2048N256", *dsa_domain(2048, 256))
    host_vectors()
    doc = {"seed": SEED, "k3_moduli": MODULI, "k3": K3_GROUPS, "modexp": MODEXP, "modprod": MODPROD, "exp_product": EXP_PRODUCT, "dsa": DSA,
           "fermat": FERMAT, "reduce": REDUCE}
    with open(os.path.join(HERE, "threshold_edges.json"), "w") as f:
        f.write("{\n")
        f.write(",\n".join("%s: [\n%s\n]" % (json.dumps(k), ",\n".join(json.dumps(r, separators=(",", ":")) for r in v))
                           if isinstance(v, list) else "%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in doc.items()))
        f.write("\n}\n")


if __name__ == "__main__":
    main()
