"""Shared by test_r32_boundary.py (CPU, limb emulation) and test_r32_boundary_gpu.py (K1, K5 on the device): the boundary
moduli and directed operands of tests/golden/r32_boundary.json (made by make_r32_boundary.py) and the K1 inputs built
from them, so that both suites check exactly the same inputs."""
import json
import math
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from emu_verify import em_int  # noqa: E402
from oracle.pgp_oracle import DIGEST_PREFIX  # noqa: E402

R2048 = 1 << 2048
DLEN = {1: 16, 2: 20, 3: 20, 8: 32, 9: 48, 10: 64, 11: 28}      # the seven hash algorithms K1 takes (OpenPGP ids)
EDGE_S = ("0", "1", "n-1", "n", "s+n", "2^2048-1")

# Paths of the lane-distributed arithmetic (tools/emu_r32.py) every width must reach, and how many directed cases must
# take each one at W = 8 and at W = 16.
REQUIRED_PATHS = {"finish_carry_gen": 20, "finish_carry_prop": 8, "finish_overflow": 10, "finish_borrow_gen": 10,
                  "finish_borrow_prop": 8, "cond_borrow_gen": 20, "cond_borrow_prop": 8, "cond_sub_taken": 20,
                  "cond_sub_skipped": 20, "ge_below_top": 20, "ge_equal": 5}


def load():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "r32_boundary.json")))


def moduli(fx, bits):
    """{name: (n, factors)} of one size"""
    out = {}
    for name, m in fx["moduli"].items():
        if m["bits"] == bits:
            out[name] = (int(m["n"], 16), [int(f, 16) for f in m["factors"]])
    return out


def directed(fx, name):
    """[(case, [vals as ints])] of one modulus"""
    return [(c, [int(v, 16) for v in c["vals"]]) for c in fx["directed"][name]]


def private_exponent(factors, e):
    lam = 1
    for f in factors:
        lam = math.lcm(lam, f - 1)
    return pow(e, -1, lam)


def k1_cases(n, factors, e, alg, seed):
    """(label, s, digest, EM) for one key, exponent and hash algorithm: a valid signature, the same with one bit flipped,
    the valid signature on another digest, and the edge values of s (EDGE_S)"""
    rng = random.Random(seed)
    d = private_exponent(factors, e)
    dig = bytes(rng.getrandbits(8) for _ in range(DLEN[alg]))
    em = em_int(DIGEST_PREFIX[alg], dig)
    s = pow(em, d, n)
    assert pow(s, e, n) == em
    other = bytes(b ^ 0x5A for b in dig)
    out = [("valid", s, dig, em), ("flip", s ^ (1 << rng.randrange(2048 if n.bit_length() == 2048 else 2040)), dig, em),
           ("other digest", s, other, em_int(DIGEST_PREFIX[alg], other))]
    for label, v in zip(EDGE_S, (0, 1, n - 1, n, s + n, R2048 - 1)):
        if v < R2048:
            out.append((label, v, dig, em))
    return out


def expect_ok(n, e, s, em, strict):
    return pow(s, e, n) == em and (not strict or s < n)


def warp_layout(cases, branch):
    """Each case at every slot of a warp's eight lane groups (slot = item index mod 8), the other seven slots holding
    cases whose `branch` differs from its own where there are such.  Returns the list of rows."""
    rows = []
    for i, (c, vals) in enumerate(cases):
        others = [v for c2, v in cases if branch(c2) != branch(c)] or [v for _, v in cases]
        for slot in range(8):
            warp = [others[(i + 3 * j) % len(others)] for j in range(8)]
            warp[slot] = vals
            rows += warp
    return rows
