#!/usr/bin/env python3
"""Boundary moduli and directed operands for the radix-2^32 Montgomery arithmetic (rsa_verify_r32.cuh), seed 0xBF7C0032.
Output committed as tests/golden/r32_boundary.json; the tests read it and search for no primes.

Moduli, at 1024 and 2048 bits (and 2047 bits, the radix-2^28 class of K1):
    low_c       the least prime 2^(b-1) + c                       (c below)
    high_c      the greatest prime 2^b - c
    n0inv_max   a prime n = 1 (mod 2^32): -n^-1 mod 2^32 = 2^32 - 1
    n0inv_one   a prime n = -1 (mod 2^32): -n^-1 mod 2^32 = 1
    lane1_ones  a prime whose lane 1 (bits 32W .. 64W - 1, W = b / 128) is all ones
    lane2_zeros a prime whose lane 2 is all zeros
    top_bit     p q with p, q primes that have only their top bit forced, q the least such prime with p q >= 2^(b-1),
                so n lies just above 2^(b-1)
Every prime p here has p = 2 (mod 3) and p != 1 (mod 65537), so e = 3 and e = 65537 are invertible mod lambda(n).

Directed operands of K5's modprod (modexp.cuh) at W = 8 (1024-bit moduli) and W = 16 (2048-bit moduli).  A case is
kept only when the limb emulation (tools/emu_r32.py) reports that it took the path it was made for:
    finish_carry_prop   k = 2, 3: the last product's target X = prod mod n has lanes 0 .. r zero
    finish_overflow     k = 2, 3: X in [R - n, n), so the product can reach R + X - n ... R + n
    finish_borrow_prop  k = 2, 3: such an X with lane r all ones (the subtraction of n borrows through lane r)
    cond_*, ge_*        k = 1: x in [n, R) equal to n in chosen lanes (ties in group_ge, borrows through equal lanes)
Each case records every path the emulation took (`paths`) and whether its last product subtracted n (`overflow`).
TEST FIXTURE ONLY."""
import json
import os
import random
import sys
from collections import Counter

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "tools"))
from emu_r32 import T, modprod_emu, n0inv_of  # noqa: E402

SEED = 0xBF7C0032
rng = random.Random(SEED)
SMALL = [p for p in range(3, 2000, 2) if all(p % q for q in range(3, int(p ** 0.5) + 1, 2))]


def is_prime(n):
    for p in SMALL:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d //= 2; s += 1
    for _ in range(16):
        x = pow(rng.randrange(2, n - 1), d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def good_prime(p):
    return p % 3 == 2 and (p - 1) % 65537 != 0 and is_prime(p)


def search(start, step):
    p = start
    while not good_prime(p):
        p += step
    return p


def moduli(b):
    W = b // 128
    lane = 32 * W
    out = {}
    p = search((1 << (b - 1)) + 1, 2)
    out["low_c"] = {"c": p - (1 << (b - 1)), "factors": [p]}
    p = search((1 << b) - 1, -2)
    out["high_c"] = {"c": (1 << b) - p, "factors": [p]}
    p = search((1 << (b - 1)) | (rng.getrandbits(b - 34) << 32) | 1, 1 << 32)
    out["n0inv_max"] = {"factors": [p]}
    p = search((1 << (b - 1)) | (rng.getrandbits(b - 34) << 32) | 0xFFFFFFFF, 1 << 32)
    out["n0inv_one"] = {"factors": [p]}
    if b % 128 == 0:
        while True:
            p = rng.getrandbits(b) | (1 << (b - 1)) | 1 | (((1 << lane) - 1) << lane)
            if good_prime(p):
                break
        out["lane1_ones"] = {"factors": [p]}
        while True:
            p = (rng.getrandbits(b) | (1 << (b - 1)) | 1) & ~(((1 << lane) - 1) << (2 * lane))
            if good_prime(p):
                break
        out["lane2_zeros"] = {"factors": [p]}
    h = b // 2
    while True:
        p = rng.getrandbits(h) | (1 << (h - 1)) | 1
        if good_prime(p):
            break
    q0 = -(-(1 << (b - 1)) // p)
    q = search(q0 | 1, 2)
    assert (p * q).bit_length() == b
    out["top_bit"] = {"factors": [p, q]}
    for v in out.values():
        n = 1
        for f in v["factors"]:
            n *= f
        assert n.bit_length() == b and n % 2
        v["n"] = n
    return out


def lanes_set(x, W, r, val):
    m = ((1 << (32 * W)) - 1) << (32 * W * r)
    return (x & ~m) | (val << (32 * W * r))


def trace_case(vals, n, W):
    tr = Counter()
    got = modprod_emu(vals, n, W, tr)
    want = 1
    for v in vals:
        want = want * v % n
    assert got == want
    return tr


def product_cases(n, W, path, lane, make_target, quota, tries):
    """k = 2 and k = 3 rows whose last product has residue X = make_target(); kept when (path, lane) was taken"""
    out = []
    for k in (2, 3):
        got = 0
        for _ in range(tries):
            X = make_target()
            if X is None:
                break
            head = [rng.randrange(1, n) for _ in range(k - 1)]
            acc = 1
            for v in head:
                acc = acc * v % n
            if acc == 0:
                continue
            vals = head + [X * pow(acc, -1, n) % n]
            tr = trace_case(vals, n, W)
            if tr[(path, lane)]:
                out.append((path, lane, vals, tr))
                got += 1
                if got == quota:
                    break
    return out


def directed(n, W):
    b = 128 * W
    R = 1 << b
    L = 32 * W
    ones = (1 << L) - 1
    nl = [(n >> (L * r)) & ones for r in range(T)]
    cases = []

    def zeros_below(r):
        return lambda: rng.randrange(n) & ~((1 << (L * (r + 1))) - 1)

    def high():
        return rng.randrange(R - n, n)

    def high_ones(r):
        def f():
            for _ in range(64):
                X = lanes_set(rng.randrange(R - n, n), W, r, ones)
                if R - n <= X < n:
                    return X
            return None
        return f

    for r in (1, 2):
        cases += product_cases(n, W, "finish_carry_prop", r, zeros_below(r), 2, 12)
    cases += product_cases(n, W, "finish_overflow", None, high, 2, 12)
    for r in (1, 2):
        cases += product_cases(n, W, "finish_borrow_prop", r, high_ones(r), 2, 24)
    # k = 1: x in [n, R) that ties n in chosen lanes; cond_sub runs twice on it
    ks = [("ge_equal", None, n)]
    for r in range(T - 1):
        for d in (1, -1):
            v = nl[r] + d
            if 0 <= v <= ones:
                ks.append(("ge_below_top", r, lanes_set(n, W, r, v)))
    for r in (1, 2):
        for h in range(r + 1, T):
            if nl[h] < ones and nl[r - 1] > 0:
                ks.append(("cond_borrow_prop", r, lanes_set(lanes_set(n, W, h, nl[h] + 1), W, r - 1, nl[r - 1] - 1)))
    ks.append(("cond_sub_taken", None, R - 1))
    ks.append(("cond_sub_skipped", None, n - 1))
    for path, lane, x in ks:
        tr = trace_case([x], n, W)
        if tr[(path, lane)]:
            cases.append((path, lane, [x], tr))
    return [{"path": p, "lane": ln, "vals": ["%x" % v for v in vals],
             "overflow": bool(tr[("finish_overflow", None)]),
             "paths": sorted({e for (e, _) in tr})} for p, ln, vals, tr in cases]


def main():
    out = {"seed": "0x%X" % SEED, "moduli": {}, "directed": {}}
    for b in (1024, 2048, 2047):
        for name, v in moduli(b).items():
            n = v["n"]
            key = "%d_%s" % (b, name)
            out["moduli"][key] = {"bits": b, "n": "%x" % n, "n0inv": n0inv_of(n),
                                  "factors": ["%x" % f for f in v["factors"]], **({"c": v["c"]} if "c" in v else {})}
            if b % 128 == 0:
                out["directed"][key] = directed(n, b // 128)
                print(key, len(out["directed"][key]), "cases", flush=True)
    path = os.path.join(HERE, "r32_boundary.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", path)


if __name__ == "__main__":
    main()
