"""CPU suite: the radix-2^32 lane-distributed Montgomery arithmetic (rsa_verify_r32.cuh: mont_mul, mont_sqr, mont_finish,
group_ge, group_sub, cond_sub) on the carry and borrow paths random operands never reach, through its limb emulation
(tools/emu_r32.py, tools/emu_sq.py, tools/emu_verify.py) at both limb widths, W = 8 (1024-bit numbers: K5, K6a) and
W = 16 (2048-bit numbers: K1, K5).

A carry crosses a lane boundary by propagation only when the whole lane is all ones (mont_finish) or all zeros (the
subtractions): 2^-256 or 2^-512 per random operand.  The directed operands of tests/golden/r32_boundary.json are solved
for such lanes on boundary moduli; each records the paths the emulation took, and these tests check that it still takes
them and that every path is reached often enough at each width.  test_r32_boundary_gpu.py runs the same inputs on K1
and K5."""
import os
import sys
from collections import Counter

import pytest

import r32_boundary as rb

sys.path.insert(0, os.path.join(rb.ROOT, "tools"))
import emu_r32  # noqa: E402
import emu_sq  # noqa: E402
from emu_verify import verify_emu  # noqa: E402


@pytest.fixture(scope="module")
def fx():
    return rb.load()


def test_emulator_random_and_adversarial_loops():
    """the emulators' own loops (random operands, R - 1, alternating and single-bit limbs, modulus R - 1), bounded"""
    emu_r32.check_random(W=8, iters=200, seed=8)
    emu_r32.check_random(W=16, iters=80, seed=16)
    assert emu_sq.check_random(iters=80, seed=2) == 544


def test_boundary_moduli(fx):
    """each modulus is the product of its factors and has the shape its name states"""
    seen = Counter()
    for key, m in fx["moduli"].items():
        b = m["bits"]
        n, fs = int(m["n"], 16), [int(f, 16) for f in m["factors"]]
        assert n == fs[0] * (fs[1] if len(fs) > 1 else 1) and n.bit_length() == b and n % 2, key
        for f in fs:
            assert f % 3 == 2 and (f - 1) % 65537 and pow(3, f - 1, f) == 1 and pow(5, f - 1, f) == 1, key
        assert m["n0inv"] == (-pow(n, -1, 1 << 32)) % (1 << 32)
        name = key.split("_", 1)[1]
        L = b // 4
        lane = [(n >> (L * r)) & ((1 << L) - 1) for r in range(4)]
        assert {"low_c": n - (1 << (b - 1)) == m.get("c") and m["c"] < 1 << 16,
                "high_c": (1 << b) - n == m.get("c") and m["c"] < 1 << 16,
                "n0inv_max": n % (1 << 32) == 1 and m["n0inv"] == 0xFFFFFFFF,
                "n0inv_one": n % (1 << 32) == 0xFFFFFFFF and m["n0inv"] == 1,
                "lane1_ones": lane[1] == (1 << L) - 1,
                "lane2_zeros": lane[2] == 0,
                "top_bit": len(fs) == 2 and n - (1 << (b - 1)) < 1 << (b // 2 + 20)}[name], key
        seen[b] += 1
    assert seen == {1024: 7, 2048: 7, 2047: 5}


@pytest.mark.parametrize("bits", [1024, 2048])
def test_directed_operands_take_their_paths(fx, bits):
    """every directed modprod row against Python integers, limb for limb through the emulation of modprod_kernel; the row
    must still take the path it was made for, and every path of REQUIRED_PATHS must be taken often enough"""
    W = bits // 128
    counts = Counter()
    ncases = 0
    for name, (n, _) in rb.moduli(fx, bits).items():
        for c, vals in rb.directed(fx, name):
            tr = Counter()
            want = 1
            for v in vals:
                want = want * v % n
            assert emu_r32.modprod_emu(vals, n, W, tr) == want, (name, c["path"], c["lane"])
            assert tr[(c["path"], c["lane"])], (name, c["path"], c["lane"])
            assert sorted({e for e, _ in tr}) == c["paths"], (name, c["path"])
            assert bool(tr[("finish_overflow", None)]) == c["overflow"]
            for e in {e for e, _ in tr}:
                counts[e] += 1
            ncases += 1
    print("\nW = %d: %d directed cases; cases per path:" % (W, ncases))
    for p in sorted(set(counts) | set(rb.REQUIRED_PATHS)):
        print("  %-20s %4d" % (p, counts[p]))
    for p, least in rb.REQUIRED_PATHS.items():
        assert counts[p] >= least, (W, p, counts[p])


def test_squaring_finish_on_boundary_moduli(fx):
    """K1's squarings end in the same mont_finish: squarings of the directed targets on the 2048-bit boundary moduli
    against Python integers, and the carry paths they take"""
    counts = Counter()
    for name, (n, _) in rb.moduli(fx, 2048).items():
        R = 1 << 2048
        for c, vals in rb.directed(fx, name)[::2]:
            a = vals[-1]
            tr = Counter()
            t = emu_sq.mont_sqr_emu(a, n, tr)
            assert t < R and t % n == a * a * pow(R, -1, n) % n, name
            counts.update({e for e, _ in tr})
        for a in (R - 1, n - 1, n, (R - 1) // 3):
            t = emu_sq.mont_sqr_emu(a, n)
            assert t < R and t % n == a * a * pow(R, -1, n) % n, name
    print("\nmont_sqr on the directed targets, cases per path:", dict(counts))
    assert counts["finish_carry_gen"] and counts["finish_overflow"]


def test_verify_emu_on_boundary_keys(fx):
    """the emulated K1 verification (tools/emu_verify.py) on the 2048-bit boundary keys, for exactly the inputs
    test_r32_boundary_gpu.py gives the kernel: its decision must be pow(s, e, n) == EM"""
    ncase = 0
    for name, (n, fs) in rb.moduli(fx, 2048).items():
        for e in (3, 65537):
            for alg in rb.DLEN:
                for label, s, dig, em in rb.k1_cases(n, fs, e, alg, "%s %d %d" % (name, e, alg)):
                    if s >= rb.R2048:
                        continue
                    if e == 65537 and alg not in (8, 10) and label != "valid":
                        continue                      # e = 65537 in full for one short and one long DigestInfo
                    tlen = len(rb.DIGEST_PREFIX[alg]) + rb.DLEN[alg]
                    assert verify_emu(n, e, s, em, tlen) == rb.expect_ok(n, e, s, em, False), (name, e, alg, label)
                    ncase += 1
    assert ncase > 250
