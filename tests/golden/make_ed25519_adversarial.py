#!/usr/bin/env python3
"""Adversarial Ed25519 vectors for K1b (ed25519.cuh, ed25519_fast.cuh), seed 0xBF7CED25.
Output committed as tests/golden/ed25519_adversarial.json; running this again reproduces it byte for byte.

A Byzantine peer picks its own key, message and signature, so every row is built from the verifier's side with
big-integer Edwards arithmetic (oracle/ed25519_oracle.py).  Keys of known discrete logarithm are [a]B, the eight
torsion points [j]T8 and their sums [a]B + [j]T8.  Where a verdict depends on k = H(R || A || M) mod ord(T), the
message is ground until k has the residue wanted; every accepted row sits next to a rejected twin.

Each row: `tag` (the case), `a` (32-byte key), `sig` (R || S), `msg` (32 bytes), `expect` (Go's crypto/ed25519.Verify,
which the generator checks against the verdict the row was built for) and `note`.

Tags:
  small_order_A   A = [j]T8 canonically encoded; R = [r]B, S = r: valid iff k = 0 mod ord(A)
  noncanon_A      y in [p, 2^255) with both sign bits, and the "-0" forms of (0, 1) and (0, -1): Go and OpenSSL reduce
                  y mod p and allow -0.  The small-order ones get valid signatures, the order-8L ones can only be rejected
  mixed_A         A = [a]B + [j]T8, honest S = r + k a: valid iff k = 0 mod ord([j]T8)
  small_order_R   R = [j]T8 under a torsion key, built so that the cofactorless equation holds (or only a cofactored one does)
  mixed_R         R = [r]B + [j]T8 likewise
  noncanon_R      the right point R encoded as y + p or as -0 (rejected: R is compared as bytes) next to its canonical twin
  S_edge          S in {0, 1, L - 1} under the identity key (valid); S >= L, S + L and S + 2^255 (invalid)
  digit_edge      S whose signed radix-2^12 / 2^10 digits sit at -2^(W-1) or 2^(W-1) - 1 or carry through every window;
                  honest signatures whose k has digits at the ends of the key's radix-2^10 table
  undecodable_A   y with no square root, below p and at or above p
TEST FIXTURE ONLY."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import ed25519_oracle as eo  # noqa: E402

SEED = 0xBF7CED25
P, L, B, ID = eo.P, eo.L, eo.BASE, eo.IDENTITY
OUT = os.path.join(HERE, "ed25519_adversarial.json")


def le(v):
    return v.to_bytes(32, "little")


class Gen:
    def __init__(self):
        self.rng = random.Random(SEED)
        self.rows = []
        self.T8 = eo.torsion8()
        self.T = [eo.mul(j, self.T8) for j in range(8)]           # T[j] = [j] T8; T[0] = identity, T[4] = (0, -1)

    def msg(self):
        return bytes(self.rng.randrange(256) for _ in range(32))

    def scalar(self):
        return self.rng.randrange(1, L)

    def push(self, tag, a32, r32, S, msg, expect, note):
        sig = r32 + S.to_bytes(32, "little")
        got = eo.verify(a32, sig, msg)
        assert got == expect, (tag, note, a32.hex(), sig.hex())
        self.rows.append({"tag": tag, "a": a32.hex(), "sig": sig.hex(), "msg": msg.hex(), "expect": expect, "note": note})

    def grind(self, r32, a32, want):
        """A message whose k = H(R || A || M) mod L satisfies want(k)."""
        while True:
            m = self.msg()
            k = eo.challenge(r32, a32, m)
            if want(k):
                return m, k

    def signed_pair(self, tag, a32, tors, note, a_log=0, r=None):
        """Key a32 = [a_log]B + tors (tors of small order o): R = [r]B, S = r + k a_log, once with k = 0 mod o (valid)
        and once with k != 0 mod o (invalid; for o = 1, S + 1 instead)."""
        o = eo.order(tors)
        r = r if r is not None else self.scalar()
        R = eo.encode(eo.mul(r, B))
        m, k = self.grind(R, a32, lambda k: k % o == 0)
        self.push(tag, a32, R, (r + k * a_log) % L, m, True, f"{note}; k = 0 mod {o}")
        if o == 1:
            self.push(tag, a32, R, (r + k * a_log + 1) % L, m, False, f"{note}; S + 1")
        else:
            m, k = self.grind(R, a32, lambda k: k % o != 0)
            self.push(tag, a32, R, (r + k * a_log) % L, m, False, f"{note}; k = {k % o} mod {o}")

    # ---- cases ---------------------------------------------------------------------------------------------------------
    def small_order_A(self):
        for j in range(8):
            self.signed_pair("small_order_A", eo.encode(self.T[j]), self.T[j], f"A = [{j}]T8")

    def noncanon_A(self):
        for t in range(19):                                            # y = p + t: every value in [p, 2^255)
            for sign in (0, 1):
                a32 = le((P + t) | (sign << 255))
                A = eo.decode_go(a32)
                if A is None:
                    continue
                assert eo.decode_strict(a32) is None
                o = eo.order(A)
                if o is not None:
                    self.signed_pair("noncanon_A", a32, A, f"y = p + {t}, sign {sign}, order {o}")
                else:                                                  # order 8L, unknown logarithm: decodes, never valid
                    assert eo.mul(8 * L, A) == ID
                    r = self.scalar()
                    R = eo.encode(eo.mul(r, B))
                    m = self.msg()
                    self.push("noncanon_A", a32, R, r, m, False, f"y = p + {t}, sign {sign}, order 8L")
                    self.push("noncanon_A", a32, eo.encode(eo.add(eo.mul(r, B), eo.neg(eo.mul(eo.challenge(R, a32, m), A)))), r, m, False,
                              f"y = p + {t}, sign {sign}, order 8L; R = [S]B - [k']A for another k'")
        for y, name in ((1, "(0, 1)"), (P - 1, "(0, -1)")):            # -0: x = 0 with the sign bit set
            a32 = le(y | (1 << 255))
            assert eo.decode_strict(a32) is None and eo.decode_go(a32) == (0, y)
            self.signed_pair("noncanon_A", a32, (0, y), f"-0 form of {name}")

    def mixed_A(self):
        for j in range(1, 8):
            a = self.scalar()
            A = eo.add(eo.mul(a, B), self.T[j])
            self.signed_pair("mixed_A", eo.encode(A), self.T[j], f"A = [a]B + [{j}]T8", a_log=a)

    def small_and_mixed_R(self):
        # A = [i]T8, S = 0: [S]B - [k]A = [-k i]T8.  R = [j]T8 holds iff -k i = j mod 8.
        for i, j in ((1, 3), (1, 4), (3, 7), (2, 6), (4, 4), (5, 1)):
            a32 = eo.encode(self.T[i])
            R = eo.encode(self.T[j])
            m, _ = self.grind(R, a32, lambda k: (-k * i - j) % 8 == 0)
            self.push("small_order_R", a32, R, 0, m, True, f"A = [{i}]T8, R = [{j}]T8, S = 0, -k {i} = {j} mod 8")
            m, _ = self.grind(R, a32, lambda k: (-k * i - j) % 8 != 0)
            self.push("small_order_R", a32, R, 0, m, False, f"A = [{i}]T8, R = [{j}]T8, S = 0, -k {i} != {j} mod 8")
        # honest key: R = identity with S = k a holds; R = [j]T8 with S = k a only holds times the cofactor
        a = self.scalar()
        a32 = eo.encode(eo.mul(a, B))
        for j in range(8):
            R = eo.encode(self.T[j])
            m = self.msg()
            k = eo.challenge(R, a32, m)
            self.push("small_order_R", a32, R, k * a % L, m, j == 0, f"honest A, R = [{j}]T8, S = k a" + ("" if j == 0 else ": cofactored only"))
        # mixed R = [r]B + [j]T8 under A = [a]B + T8, S = r + k a: holds iff -k = j mod 8
        a = self.scalar()
        a32 = eo.encode(eo.add(eo.mul(a, B), self.T8))
        for j in (1, 2, 4, 7):
            r = self.scalar()
            R = eo.encode(eo.add(eo.mul(r, B), self.T[j]))
            m, k = self.grind(R, a32, lambda k: (k + j) % 8 == 0)
            self.push("mixed_R", a32, R, (r + k * a) % L, m, True, f"A = [a]B + T8, R = [r]B + [{j}]T8, -k = {j} mod 8")
            m, k = self.grind(R, a32, lambda k: (k + j) % 8 != 0)
            self.push("mixed_R", a32, R, (r + k * a) % L, m, False, f"A = [a]B + T8, R = [r]B + [{j}]T8, -k != {j} mod 8: cofactored only")
        # honest A, R = [r]B + [j]T8, S = r + k a: only a cofactored verifier accepts
        a = self.scalar()
        a32 = eo.encode(eo.mul(a, B))
        for j in (1, 4):
            r = self.scalar()
            R = eo.encode(eo.add(eo.mul(r, B), self.T[j]))
            m = self.msg()
            self.push("mixed_R", a32, R, (r + eo.challenge(R, a32, m) * a) % L, m, False, f"honest A, R = [r]B + [{j}]T8: cofactored only")

    def noncanon_R(self):
        # R = identity under an honest key (S = k a): canonical 01 00..00 vs y = p + 1, -0, and both
        a = self.scalar()
        a32 = eo.encode(eo.mul(a, B))
        for enc, name in ((le(1), "canonical"), (le(P + 1), "y = p + 1"), (le(1 | (1 << 255)), "-0"), (le((P + 1) | (1 << 255)), "y = p + 1, -0")):
            m = self.msg()
            self.push("noncanon_R", a32, enc, eo.challenge(enc, a32, m) * a % L, m, name == "canonical", f"R = identity, {name}")
        # R = (0, -1) = [4]T8 under A = [4]T8, S = 0: -[k]A = R iff k odd.  Canonical vs -0.
        a32 = eo.encode(self.T[4])
        for enc, name in ((le(P - 1), "canonical"), (le((P - 1) | (1 << 255)), "-0")):
            m, _ = self.grind(enc, a32, lambda k: k % 2 == 1)
            self.push("noncanon_R", a32, enc, 0, m, name == "canonical", f"R = (0, -1), {name}, k odd")
        # R = [2]T8 or [6]T8 (y = 0) under A = [2]T8, S = 0: canonical y = 0 vs y = p with the same sign
        a32 = eo.encode(self.T[2])
        for j in (2, 6):
            x = self.T[j][0]
            for enc, name in ((le((x & 1) << 255), "canonical"), (le(P | ((x & 1) << 255)), "y = p")):
                m, _ = self.grind(enc, a32, lambda k: (-2 * k - j) % 8 == 0)
                self.push("noncanon_R", a32, enc, 0, m, name == "canonical", f"R = [{j}]T8, {name}")

    def s_edges(self):
        a32 = le(1)                                                    # the identity: any S < L is valid with R = enc([S]B)
        for S in (0, 1, L - 1):
            R = eo.encode(eo.mul(S, B))
            m = self.msg()
            self.push("S_edge", a32, R, S, m, True, f"identity key, S = {S if S < 2 else 'L - 1'}")
            self.push("S_edge", a32, eo.encode(eo.mul(S + 1, B)), S, m, False, "identity key, R = enc([S + 1]B)")
        for S, name in ((L, "L"), (L + 1, "L + 1"), (2 ** 253 - 1, "2^253 - 1"), (2 ** 256 - 1, "2^256 - 1")):
            self.push("S_edge", a32, eo.encode(eo.mul(S % L, B)), S, self.msg(), False, f"identity key, S = {name}")
        a = self.scalar()
        a32 = eo.encode(eo.mul(a, B))
        r = self.scalar()
        R = eo.encode(eo.mul(r, B))
        m, k = self.grind(R, a32, lambda k: (r + k * a) % L < 2 ** 253 - L)     # S + L still fits below 2^253
        S = (r + k * a) % L
        self.push("S_edge", a32, R, S, m, True, "honest")
        self.push("S_edge", a32, R, S + L, m, False, "honest S + L")
        self.push("S_edge", a32, R, S + (1 << 255), m, False, "honest S with bit 255 set")

    def digit_edges(self):
        a32 = le(1)
        picks = []
        for w, nw in ((12, 22), (10, 26)):
            h = 1 << (w - 1)
            picks += [(h - 1) * sum(1 << (w * i) for i in range(nw - 1)),             # every digit 2^(W-1) - 1
                      h + sum((h - 1) << (w * i) for i in range(1, nw - 1)),           # every digit -2^(W-1), carries throughout
                      h * sum(1 << (w * i) for i in range(nw - 1)),                   # alternating carries
                      (1 << (w * (nw - 1))) - 1]                                       # all ones: -1 digits, carry to the top window
        picks += [(1 << 252) - 1, 1 << 252, L - 2, (L - 1) >> 1, int("80" * 31, 16)]
        for S in picks:
            S %= L
            ds = eo.signed_digits(S, 12, 22)
            assert sum(d << (12 * i) for i, d in enumerate(ds)) == S
            ends = sum(d in (-2048, 2047) for d in ds), sum(d in (-512, 511) for d in eo.signed_digits(S, 10, 26))
            m = self.msg()
            self.push("digit_edge", a32, eo.encode(eo.mul(S, B)), S, m, True, f"identity key, S = {S:#x}; digits at the ends: {ends[0]} (2^12), {ends[1]} (2^10)")
            self.push("digit_edge", a32, eo.encode(eo.mul(S, B)), (S + 1) % L, m, False, "identity key, S + 1")
        # honest key: k's radix-2^10 digits at -512 (the last entry of the key's table) in some window
        a = self.scalar()
        a32 = eo.encode(eo.mul(a, B))
        for _ in range(3):
            r = self.scalar()
            R = eo.encode(eo.mul(r, B))
            m, k = self.grind(R, a32, lambda k: sum(d == -512 for d in eo.signed_digits(k, 10, 26)) >= 2)
            self.push("digit_edge", a32, R, (r + k * a) % L, m, True, "honest key, k has two radix-2^10 digits of -512")
            self.push("digit_edge", a32, R, (r + k * a + 1) % L, m, False, "honest key, S + 1")

    def undecodable_A(self):
        r = self.scalar()
        R = eo.encode(eo.mul(r, B))
        found = 0
        for y in range(2, 40):                                         # below p
            if eo.x_of(y, 0) is None:
                for sign in (0, 1):
                    self.push("undecodable_A", le(y | (sign << 255)), R, r, self.msg(), False, f"y = {y}, no root")
                found += 1
                if found == 3:
                    break
        for t in range(19):                                            # at or above p
            if eo.x_of(t, 0) is None:
                for sign in (0, 1):
                    self.push("undecodable_A", le((P + t) | (sign << 255)), R, r, self.msg(), False, f"y = p + {t}, no root")


def main(out=OUT):
    g = Gen()
    g.small_order_A()
    g.noncanon_A()
    g.mixed_A()
    g.small_and_mixed_R()
    g.noncanon_R()
    g.s_edges()
    g.digit_edges()
    g.undecodable_A()
    with open(out, "w") as f:
        json.dump({"seed": hex(SEED), "T8": eo.encode(g.T8).hex(), "rows": g.rows}, f, indent=0)
        f.write("\n")
    return g.rows


if __name__ == "__main__":
    rows = main(sys.argv[1] if len(sys.argv) > 1 else OUT)
    from collections import Counter
    print(len(rows), dict(Counter(r["tag"] for r in rows)))
