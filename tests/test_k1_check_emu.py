"""CPU suite: K1's verification without a conversion to Montgomery form (rsa_verify_r32.cuh).

* The per-key constants of bignum_host.hpp, compiled into a small C++ harness, against their definition with Python
  integers: c = R^-(e-1) mod n (R = 2^2048), c16 = c 2^512, hc16 = (2^2033 - 2^512) c, c32 = c 2^1024,
  hc32 = (2^2033 - 2^1024) c, all mod n.
* The limb-level emulation of the whole verification (tools/emu_verify.py) against pow(s, e, n) == EM, for exponents
  with and without interior 1 bits, even ones and e = 1, edge signatures and all seven hash algorithms (the short
  DigestInfos split EM at 2^512, SHA-384 / SHA-512 at 2^1024)."""
import hashlib
import math
import os
import random
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from emu_verify import R, em_int, key_consts, verify_emu  # noqa: E402
from oracle.pgp_oracle import DIGEST_PREFIX  # noqa: E402

EXPONENTS = [1, 2, 3, 17, 65536, 65537, 2**32 - 1]
HASHES = {1: "md5", 2: "sha1", 3: "ripemd160", 8: "sha256", 9: "sha384", 10: "sha512", 11: "sha224"}
SMALL_PRIMES = [p for p in range(3, 2000, 2) if all(p % q for q in range(3, int(p ** 0.5) + 1, 2))]

HARNESS = r"""
#include <cstdio>
#include <cstdlib>
#include "bignum_host.hpp"
using namespace bftq::hostbig;
static void put(const UBig& a) { for (int i = 31; i >= 0; i--) printf("%016llx", (unsigned long long)a.w[i]); printf("\n"); }
int main(int argc, char** argv) {
  uint8_t be[256];
  for (int i = 0; i < 256; i++) { unsigned v; sscanf(argv[1] + 2 * i, "%2x", &v); be[i] = (uint8_t)v; }
  UBig n;
  from_be(n, be, 256);
  for (int i = 2; i < argc; i++) {
    const VerifyConsts k = verify_consts(n, (uint32_t)strtoul(argv[i], nullptr, 10));
    put(k.c16); put(k.hc16); put(k.c32); put(k.hc32);
  }
  return 0;
}
"""


def is_probable_prime(x, rng):
    if any(x % p == 0 for p in SMALL_PRIMES):
        return False
    d, s = x - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for _ in range(24):
        y = pow(rng.randrange(2, x - 1), d, x)
        if y in (1, x - 1):
            continue
        for _ in range(s - 1):
            y = y * y % x
            if y == x - 1:
                break
        else:
            return False
    return True


def blum_prime(rng):
    """p = 3 mod 4, 1024 bits (top two set), with (p - 1) / 2 prime to 3, 5, 17, 257, 65537: every odd exponent of the
    list is invertible mod (p - 1), and squaring permutes the quadratic residues."""
    while True:
        p = rng.getrandbits(1024) | (3 << 1022) | 3
        if all(((p - 1) // 2) % f for f in (3, 5, 17, 257, 65537)) and is_probable_prime(p, rng):
            return p


@pytest.fixture(scope="module")
def key():
    rng = random.Random(0xBF7C00E1)
    p, q = blum_prime(rng), blum_prime(rng)
    n = p * q
    assert n.bit_length() == 2048
    return p, q, n


def sign(p, q, e, em):
    """s with s^e = em (mod n), for em a quadratic residue when e is even."""
    lam = math.lcm((p - 1) // 2, (q - 1) // 2) if e % 2 == 0 else math.lcm(p - 1, q - 1)
    s = pow(em, pow(e, -1, lam), p * q)
    assert pow(s, e, p * q) == em
    return s


def residue_digest(p, q, alg, even, tag):
    """a digest whose EM has e-th roots (a quadratic residue mod p and q when e is even)"""
    for i in range(1000):
        d = hashlib.new(HASHES[alg], b"%s %d" % (tag, i)).digest()
        em = em_int(DIGEST_PREFIX[alg], d)
        if not even or (pow(em, (p - 1) // 2, p) == 1 and pow(em, (q - 1) // 2, q) == 1):
            return d, em
    raise AssertionError("no residue found")


def test_host_constants_match_definition(key, tmp_path):
    _, _, n = key
    src = tmp_path / "consts.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "consts"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "bftkv_b200", "csrc"),
                           "-o", str(exe), str(src)])
    from bftkv_b200 import workload
    mods = [n] + [k["n"] for k in workload.load_keys(3)]
    for m in mods:
        out = subprocess.run([str(exe), m.to_bytes(256, "big").hex()] + [str(e) for e in EXPONENTS], capture_output=True,
                             text=True, check=True).stdout.split()
        assert len(out) == 4 * len(EXPONENTS)
        for i, e in enumerate(EXPONENTS):
            c = pow(2, -2048 * (e - 1), m)
            want = [c * 2**512 % m, (2**2033 - 2**512) * c % m, c * 2**1024 % m, (2**2033 - 2**1024) * c % m]
            assert [int(h, 16) for h in out[4 * i:4 * i + 4]] == want, (hex(m)[:18], e)
            assert key_consts(m, e) == dict(zip(("c16", "hc16", "c32", "hc32"), want))


@pytest.mark.parametrize("e", EXPONENTS)
def test_emulated_verification_matches_pow(key, e):
    p, q, n = key
    consts = key_consts(n, e)
    for alg in HASHES:
        tlen = len(DIGEST_PREFIX[alg]) + hashlib.new(HASHES[alg]).digest_size
        d, em = residue_digest(p, q, alg, e % 2 == 0, b"k1 %d" % e)
        s = sign(p, q, e, em)
        assert verify_emu(n, e, s, em, tlen, consts), (e, alg)
        assert not verify_emu(n, e, s ^ (1 << (alg * 97 % 2048)), em, tlen, consts), (e, alg)
        other = em_int(DIGEST_PREFIX[alg], bytes(b ^ 0x40 for b in d))
        assert not verify_emu(n, e, s, other, tlen, consts), (e, alg)
        if alg in (8, 10):            # the edge signatures, with one split of EM each
            for sv in (0, 1, n - 1, n, n + s, R - 1):
                if sv < R:
                    assert verify_emu(n, e, sv, em, tlen, consts) == (pow(sv, e, n) == em), (e, alg, hex(sv)[:10])


def test_lane_with_shorter_exponent_than_its_block(key):
    """a lane of e = 1 or 3 in a block that runs 65537's 16 squarings: the extra squarings are not applied"""
    p, q, n = key
    em = em_int(DIGEST_PREFIX[8], hashlib.sha256(b"mixed").digest())
    for e in (1, 3):
        s = sign(p, q, e, em)
        assert verify_emu(n, e, s, em, 51, nbmax=17)
        assert not verify_emu(n, e, s + 1, em, 51, nbmax=17)
