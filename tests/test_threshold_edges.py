"""The share-combine arithmetic on the CPU: K3's per-combine code (lagrange_item<L>, small_inverse, mag_to_big,
mont_mul_big), fermat_pow and limbs::reduce_be from csrc/lagrange.cuh and limbs.cuh, built with g++
(tests/harness/lagrange_host.cpp), against Python integers through oracle/sss_oracle.py (Go's sss.Lagrange restated).
Vectors: tests/golden/threshold_edges.json (make_threshold_edges.py, decoded by threshold_edges.py), plus a seeded
random sweep per limb class."""
import ctypes
import os
import random
import subprocess
import time
from collections import Counter
from math import gcd

import numpy as np
import pytest

from oracle import sss_oracle as sss
import threshold_edges as te

HERE = os.path.dirname(os.path.abspath(__file__))
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
mlen_of, limb_class = te.mlen_of, te.limb_class


@pytest.fixture(scope="module")
def vec():
    return te.load()


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so_path = tmp_path_factory.mktemp("lagrange") / "liblagrange.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-o", str(so_path), os.path.join(HERE, "harness", "lagrange_host.cpp")], check=True)
    return ctypes.CDLL(str(so_path))


def host_combine(lib, m, xs, ys):
    """xs: (B, k) ints, ys: B lists of k ints -> (outs, status, lambdas) from the host build of lagrange_item."""
    mlen = mlen_of(m)
    x = np.ascontiguousarray(xs, np.int32)
    B, k = x.shape
    yb = np.frombuffer(b"".join(int(v).to_bytes(mlen, "big") for row in ys for v in row), np.uint8).copy()
    out = np.zeros((B, mlen), np.uint8)
    st = np.full(B, 0xEE, np.uint8)
    lam = np.zeros((B, k, mlen), np.uint8)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)    # noqa: E731
    lib.lagrange_combine_host(m.to_bytes(mlen, "big"), ctypes.c_uint32(mlen), ctypes.c_uint32(k), p(x), p(yb), ctypes.c_uint64(B),
                              p(out), p(st), p(lam))
    outs = [int.from_bytes(bytes(o), "big") for o in out]
    lams = [[int.from_bytes(bytes(lam[b, i]), "big") for i in range(k)] for b in range(B)]
    return outs, st.tolist(), lams


def expected(m, xs, ys):
    """(out, status, lambdas): Go's calculateSecret; status 3 (out 0) where ModInverse has no answer."""
    try:
        lams = [sss.lagrange(x, xs, m) for x in xs]
    except ValueError:
        return 0, 3, None
    return sss.calculate_secret(list(zip(xs, ys)), m), 0, lams


def test_vectors_are_consistent_with_the_oracle(vec):
    """The committed statuses and output digests are what sss_oracle computes, and the vectors reach what they are for:
    every limb class at both outcomes, INT32_MIN with INT32_MAX, x = 0, duplicates, k = 255, y >= m, m < 2^32 with a
    numerator chunk >= m (mag_to_big's reduction)."""
    classes, flags = Counter(), Counter()
    for g in vec["k3"]:
        m, k, items = te.k3_items(g, vec["k3_moduli"])
        res = [expected(m, xs, ys) for xs, ys in items]
        assert g["status"] == [st for _, st, _ in res], g["tag"]
        assert g["digest"] == te.digest(g["status"], [o for o, _, _ in res], mlen_of(m)), g["tag"]
        for (xs, ys), (_, st, _) in zip(items, res):
            classes[(limb_class(mlen_of(m)), st)] += 1
            flags["min_max"] += I32_MIN in xs and I32_MAX in xs
            flags["zero"] += 0 in xs and st == 0 and k > 1
            flags["dups"] += len(set(xs)) < len(xs)
            flags["k255"] += k == 255
            flags["y_ge_m"] += any(y >= m for y in ys)
            flags["tiny_chunk_ge_m"] += m < (1 << 32) and st == 0 and any(abs(a) >= m for a in xs)
            flags["neg"] += st == 0 and any(a < 0 for a in xs) and any(a > 0 for a in xs)
    for L in (8, 16, 32, 64):
        assert classes[(L, 0)] >= 30 and classes[(L, 3)] >= 15, (L, classes)
    for f in ("min_max", "zero", "dups", "k255", "y_ge_m", "tiny_chunk_ge_m", "neg"):
        assert flags[f] >= 5, (f, flags)
    mlens = {mlen_of(int(m, 16)) for m in vec["k3_moduli"].values()}
    assert {1, 4, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256} <= mlens


def test_host_combine_matches_oracle_on_vectors(vec, lib):
    """Out and status on every committed K3 vector equal the oracle's (and the frozen digest), and so does each
    lambda_i where the combine succeeds."""
    n = 0
    for g in vec["k3"]:
        m, k, items = te.k3_items(g, vec["k3_moduli"])
        outs, st, lams = host_combine(lib, m, [xs for xs, _ in items], [ys for _, ys in items])
        assert st == g["status"] and te.digest(st, outs, mlen_of(m)) == g["digest"], g["tag"]
        for b, (xs, ys) in enumerate(items):
            out, s, lam = expected(m, xs, ys)
            assert (st[b], outs[b]) == (s, out), (g["tag"], b)
            if s == 0 and k <= 10:
                assert lams[b] == lam, (g["tag"], b)
            n += 1
    assert n > 500


def random_modulus(rng, L):
    lo = {8: 1, 16: 33, 32: 65, 64: 129}[L]
    hi = {8: 32, 16: 64, 32: 128, 64: 256}[L]
    mlen = rng.choice([lo, hi, rng.randint(lo, hi)])
    bits = 8 * mlen
    kind = rng.randrange(4)
    if kind == 0 and bits > 8:                                     # odd m times a product of small primes
        sm = rng.choice([s for s in (3, 5, 7, 15, 21, 105, 3 * 5 * 7 * 11 * 13, 9, 25, 65537 * 3) if s.bit_length() + 2 < bits])
        return (rng.getrandbits(bits - sm.bit_length()) | (1 << (bits - sm.bit_length() - 1)) | 1) * sm
    if kind == 1 and L == 8:                                       # m below 2^32
        return rng.getrandbits(rng.randint(2, 32)) | 1 | 2
    m = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
    return m


def test_host_combine_random_sweep(lib):
    """About 10^5 seeded combines over the whole int32 abscissa range and random odd moduli (prime or composite) of
    every limb class: out, status and lambda_i equal Python's; status 3 exactly when pow(b % m, -1, m) raises."""
    rng = random.Random(0xBF7C7E01)
    t0 = time.time()
    total, statuses = 0, Counter()
    plan = {8: (2400, 32), 16: (800, 20), 32: (400, 16), 64: (200, 10)}     # (batches, items per batch), k 1..6
    for L, (batches, per) in plan.items():
        for _ in range(batches):
            m = random_modulus(rng, L)
            k = rng.choice([1, 2, 2, 3, 3, 4, 5, 6])
            xs, ys = [], []
            for _ in range(per):
                kind = rng.randrange(4)
                if kind == 0:
                    row = [rng.randrange(I32_MIN, I32_MAX + 1) for _ in range(k)]
                elif kind == 1:
                    row = [rng.choice([I32_MIN, I32_MAX, 0, -1, 1, rng.randrange(-40, 41)]) for _ in range(k)]
                elif kind == 2:
                    row = [rng.choice((1, -1)) * rng.randrange(1 << 20, 1 << 31) for _ in range(k)]
                else:
                    row = rng.sample(range(1, 16), k)
                xs.append(row)
                ys.append([rng.getrandbits(8 * mlen_of(m)) for _ in range(k)])
            outs, st, lams = host_combine(lib, m, xs, ys)
            for b in range(per):
                out, s, lam = expected(m, xs[b], ys[b])
                assert (st[b], outs[b]) == (s, out), (m, xs[b], ys[b])
                if s == 0:
                    assert lams[b] == lam, (m, xs[b])
                statuses[(L, s)] += 1
            total += per
    assert total >= 90000
    for L in plan:
        assert statuses[(L, 0)] > 500 and statuses[(L, 3)] > 100, statuses
    print("sweep: %d combines in %.1f s; %s" % (total, time.time() - t0, dict(sorted(statuses.items()))))


def test_status_3_exactly_when_the_inverse_does_not_exist(lib):
    """One denominator pair per combine, swept over composite m: status 3 iff gcd(x_j - x_i, m) != 1, including
    differences whose shared prime sits in a chunk of two factors (x_j - x_i = 7 * 11 for m = 77 q)."""
    rng = random.Random(0xBF7C7E02)
    for m in [15, 77 * 1000003, 3 * 5 * 7 * 11 * 13 * 17 * 19 * 23, 9 * 2147483647, (1 << 32) - 1, (1 << 64) - 1, 3 ** 40]:
        xs, ys = [], []
        for _ in range(300):
            a = rng.randrange(-1000, 1000)
            d = rng.choice([rng.randrange(1, 200), 77, 7 * 11 * 13, 3, 9, rng.randrange(1, 1 << 31)])
            b = max(I32_MIN, min(I32_MAX, a + rng.choice((1, -1)) * d))
            third = rng.randrange(-5000, 5000)
            xs.append([a, b, third]); ys.append([rng.randrange(m) for _ in range(3)])
        outs, st, _ = host_combine(lib, m, xs, ys)
        for row, s in zip(xs, st):
            ok = all(gcd(row[j] - row[i], m) == 1 for i in range(3) for j in range(3) if row[i] != row[j])
            assert s == (0 if ok else 3), (m, row)


def test_fermat_pow_and_reduce_be_on_edges(vec, lib):
    """fermat_pow (acc = v^(m-2), out of Montgomery form, as fermat_inverse_kernel does) at every limb class, and
    limbs::reduce_be (mod_small_kernel, dsa_finish_kernel) on operands of 1..512 bytes around multiples of m."""
    for i, r in enumerate(vec["fermat"]):
        m = int(r["m"], 16)
        mlen = mlen_of(m)
        for v in te.values(r["v"], m, mlen, "fermat/%d" % i):
            out = ctypes.create_string_buffer(mlen)
            lib.fermat_pow_host(m.to_bytes(mlen, "big"), ctypes.c_uint32(mlen), v.to_bytes(mlen, "big"), out)
            assert int.from_bytes(out.raw, "big") == pow(v, m - 2, m), (hex(m), hex(v))
    assert {limb_class(mlen_of(int(r["m"], 16))) for r in vec["fermat"]} == {8, 16, 32, 64}
    for i, r in enumerate(vec["reduce"]):
        m, nb = int(r["m"], 16), r["nbytes"]
        mlen = mlen_of(m)
        for v in te.values(r["v"], m, nb, "reduce/%d" % i):
            out = ctypes.create_string_buffer(mlen)
            lib.reduce_be_host(m.to_bytes(mlen, "big"), ctypes.c_uint32(mlen), v.to_bytes(nb, "big"), ctypes.c_uint32(nb), out)
            assert int.from_bytes(out.raw, "big") == v % m, (hex(m), nb, hex(v))
    assert {r["nbytes"] for r in vec["reduce"]} >= {1, 32, 33, 128, 256, 512}
