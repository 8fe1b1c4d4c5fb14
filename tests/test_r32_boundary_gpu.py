"""GPU suite: K5 (modexp_kernel, modprod_kernel) and K1 (rsa_verify_r32_kernel, and the radix-2^28 kernel for 2041..2047-bit
keys) on the boundary moduli and directed operands of tests/golden/r32_boundary.json, byte for byte against Python
integers.  test_r32_boundary.py checks that the same inputs take the cross-lane carry and borrow paths they were made
for in the limb emulation; here they run on the device.

mont_finish subtracts n under __any_sync(overflow): every directed row sits at each of the eight lane-group slots of a
warp, next to rows whose last product took the other branch."""
import itertools
import random

import numpy as np
import pytest

import r32_boundary as rb
from bftkv_b200 import Engine

pytestmark = pytest.mark.gpu
F_STRICT_RANGE = 1


@pytest.fixture(scope="module")
def fx():
    return rb.load()


def prod_mod(vals, n):
    out = 1
    for v in vals:
        out = out * v % n
    return out


def mlen_of(bits):
    return (bits + 7) // 8


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("bits", [1024, 2048])
def test_modprod_directed(engine, fx, bits, k):
    mlen = bits // 8
    nrows = 0
    for name, (n, _) in rb.moduli(fx, bits).items():
        cases = [(c, v) for c, v in rb.directed(fx, name) if len(v) == k]
        if k == 1:     # the other branch of k = 1 is cond_sub's: x < n next to x >= n
            rows = rb.warp_layout(cases, lambda c: "cond_sub_taken" in c["paths"])
        else:
            rows = rb.warp_layout(cases, lambda c: c["overflow"])
        assert cases and len(rows) == 64 * len(cases)
        want = [prod_mod(r, n).to_bytes(mlen, "big") for r in rows]
        assert engine.modprod_batch(n, rows) == want, (name, k)
        for cut in (1, 5, 13, len(rows) - 3):               # ragged batches: the last warp is partly empty
            assert engine.modprod_batch(n, rows[:cut]) == want[:cut], (name, k, cut)
        nrows += len(rows)
    assert nrows >= 64 * 7


@pytest.mark.parametrize("bits", [1024, 2048])
def test_modexp_directed(engine, fx, bits):
    """the directed targets as bases (exponent 1 ends in the product whose residue they were solved for), with exponents
    0, 1, 2, random and full length mixed in every warp"""
    rng = random.Random(bits)
    for name, (n, _) in rb.moduli(fx, bits).items():
        R = 1 << bits
        bases = [prod_mod(v, n) for _, v in rb.directed(fx, name)] + [v[0] for c, v in rb.directed(fx, name) if len(v) == 1]
        bases += [0, 1, n - 1, n, n + 1, R - 1]
        exps_of = [lambda: 0, lambda: 1, lambda: 2, lambda: rng.getrandbits(160), lambda: rng.getrandbits(bits) | 1 << (bits - 1)]
        items = [(b, exps_of[(i + j) % 5]()) for i, b in enumerate(bases) for j in range(5)]
        items = items[:len(items) - 3] if len(items) % 8 == 0 else items
        got = engine.modexp_batch(n, [b for b, _ in items], [e for _, e in items], elen=mlen_of(bits))
        assert got == [pow(b, e, n) for b, e in items], name


def k1_batch(mods, alg, es=(3, 65537)):
    """keys to register as (n, e) and the items (key, label, s, digest, EM): every key once per exponent, the items of
    its exponents interleaved so that each warp mixes them"""
    keys, items = [], []
    for name, (n, fs) in mods.items():
        per_e = []
        for e in es:
            keys.append((n, e))
            per_e.append([(len(keys) - 1,) + c for c in rb.k1_cases(n, fs, e, alg, "%s %d %d" % (name, e, alg))])
        for group in itertools.zip_longest(*per_e):
            items += [it for it in group if it is not None]
    return keys, items


def run_k1(eng, first, keys, items, alg, flags):
    kidx = np.array([first + i for i, *_ in items], np.uint32)
    sig = np.frombuffer(b"".join(s.to_bytes(256, "big") for _, _, s, _, _ in items), np.uint8).reshape(-1, 256).copy()
    dig = np.frombuffer(b"".join(d for *_, d, _ in items), np.uint8).reshape(-1, rb.DLEN[alg]).copy()
    return eng.rsa_verify_batch(kidx, sig, dig, hash_alg=alg, flags=flags)


@pytest.mark.parametrize("alg", sorted(rb.DLEN))
def test_k1_boundary_keys(built, fx, alg):
    """K1 on the 2048-bit boundary keys, e = 3 and e = 65537 in every warp: valid and tampered signatures and the edge
    values of s, without and with BFTQ_F_STRICT_RANGE; status 0 iff pow(s, e, n) == EM (and s < n when strict)"""
    mods = rb.moduli(fx, 2048)
    keys, items = k1_batch(mods, alg)
    eng = Engine(0)                       # only exactly-2048-bit keys: the radix-2^32 kernel
    try:
        first = eng.register_rsa_keys([n for n, _ in keys], [e for _, e in keys])
        for flags in (0, F_STRICT_RANGE):
            st = run_k1(eng, first, keys, items, alg, flags)
            want = [0 if rb.expect_ok(keys[i][0], keys[i][1], s, em, flags) else 1 for i, _, s, _, em in items]
            bad = [(items[j][0], items[j][1]) for j in range(len(items)) if st[j] != want[j]]
            assert not bad, (alg, flags, bad[:8])
            assert sum(w == 0 for w in want) >= len(keys)          # at least every valid signature
    finally:
        eng.close()


@pytest.mark.parametrize("alg", [8, 10])
def test_k1_radix28_2047_bit_keys(built, fx, alg):
    """the 2041..2047-bit class (radix-2^28 kernel) on 2^2046 + c, 2^2047 - c, n = +-1 mod 2^32 and a product just
    above 2^2046"""
    mods = rb.moduli(fx, 2047)
    keys, items = k1_batch(mods, alg)
    eng = Engine(0)
    try:
        first = eng.register_rsa_keys([n for n, _ in keys], [e for _, e in keys])
        for flags in (0, F_STRICT_RANGE):
            st = run_k1(eng, first, keys, items, alg, flags)
            want = [0 if rb.expect_ok(keys[i][0], keys[i][1], s, em, flags) else 1 for i, _, s, _, em in items]
            bad = [(items[j][0], items[j][1]) for j in range(len(items)) if st[j] != want[j]]
            assert not bad, (alg, flags, bad[:8])
    finally:
        eng.close()
