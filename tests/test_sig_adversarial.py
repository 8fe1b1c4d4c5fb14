"""ECDSA P-256 (K1c) and DSA (K1d) on keys and signatures a Byzantine peer builds (tests/golden/sig_adversarial.json).

CPU only.  The oracle's restatements of Go crypto/ecdsa.Verify and crypto/dsa.Verify are pinned against OpenSSL and a
plain integer restatement; a Python model of ecdsa_verify_core's Shamir ladder shows that each vector reaches the
branch of pt_add_v it was built for; the host build of the P-256 core (the kernel's own __host__ __device__ code) must
give the oracle's verdict on every vector; and the host build of modinv_big (dsa_prepare_kernel's s^-1 when q is not
prime, thrsa_modinv_kernel's m^-1 mod N) must agree with pow(s, -1, q)."""
import ctypes
import json
import os
import random
import subprocess
from collections import Counter
from math import gcd

import pytest

from oracle import pgp_oracle as pgp, sss_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
N, P, G = so.P256_N, so.P256_P, so.P256_G


@pytest.fixture(scope="module")
def vec():
    return json.load(open(os.path.join(HERE, "golden", "sig_adversarial.json")))


def _h(v):
    return int(v, 16)


def ec_args(row):
    return (_h(row["qx"]), _h(row["qy"])), bytes.fromhex(row["digest"]), _h(row["r"]), _h(row["s"])


def dsa_dom(vec, row):
    D = [d for d in vec["dsa_domains"] if d["name"] == row["domain"]][0]
    g = _h(row["g"]) if "g" in row else _h(D["g"])
    y = _h(row["y"]) if "y" in row else _h(D["y"])
    return _h(D["p"]), _h(D["q"]), g, y, D


def dsa_args(vec, row):
    p, q, g, y, _ = dsa_dom(vec, row)
    return p, q, g, y, bytes.fromhex(row["digest"]), _h(row["r"]), _h(row["s"])


def dsa_restated(p, q, g, y, digest, r, s):
    """crypto/dsa.Verify after x/crypto's cut of the digest to the subgroup size, with ModInverse by extended Euclid."""
    digest = digest[:(q.bit_length() + 7) // 8]
    if p == 0 or not (0 < r < q) or not (0 < s < q):
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


def dsa_fermat(p, q, g, y, digest, r, s):
    """The same with w = s^(q-2) mod q, as dsa_prepare_kernel computed it before it checked w s == 1."""
    digest = digest[:(q.bit_length() + 7) // 8]
    if not (0 < r < q) or not (0 < s < q) or q.bit_length() % 8:
        return False
    w = pow(s, q - 2, q)
    z = int.from_bytes(digest, "big")
    return pow(g, z * w % q, p) * pow(y, r * w % q, p) % p % q == r


# ---- oracle pinned ------------------------------------------------------------------------------------------------
_HASH_OF = {20: "SHA1", 28: "SHA224", 32: "SHA256", 48: "SHA384", 64: "SHA512"}


def test_ecdsa_oracle_matches_openssl_and_construction(vec):
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    n_ok = n_bad = 0
    for row in vec["ecdsa"]:
        q, d, r, s = ec_args(row)
        got = pgp.ecdsa_p256_verify(q, d, r, s)
        assert got == row["expect"], row["tag"]
        try:
            pub = ec.EllipticCurvePublicNumbers(q[0], q[1], ec.SECP256R1()).public_key()
        except ValueError:
            assert row["status"] == 3 and not got, row["tag"]          # the non-canonical key: elliptic.Unmarshal refuses it too
            continue
        if not (0 < r < 2 ** 256 and 0 < s < 2 ** 256):
            assert not got
            continue
        try:
            pub.verify(utils.encode_dss_signature(r, s), d, ec.ECDSA(utils.Prehashed(getattr(hashes, _HASH_OF[len(d)])())))
            ossl = True
        except InvalidSignature:
            ossl = False
        if row["status"] == 3:
            # OpenSSL reduces X mod p and accepts; Go's elliptic.Unmarshal refuses a coordinate >= p, so the key is void
            assert ossl and not got, row["tag"]
            continue
        assert ossl == got, row["tag"]
        n_ok += got
        n_bad += not got
    assert n_ok >= 60 and n_bad >= 60


def test_dsa_oracle_matches_openssl_and_restatement(vec):
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import dsa, utils
    n_ossl = 0
    for row in vec["dsa"]:
        p, q, g, y, d, r, s = dsa_args(vec, row)
        got = pgp.dsa_verify(p, q, g, y, d, r, s)
        assert got == row["expect"] == dsa_restated(p, q, g, y, d, r, s), (row["domain"], row["tag"])
        if q.bit_length() not in (160, 224, 256) or p.bit_length() not in (1024, 2048) or not (1 < g < p) or not (1 < y < p):
            continue
        try:
            pub = dsa.DSAPublicNumbers(y, dsa.DSAParameterNumbers(p, q, g)).public_key()
        except ValueError:
            continue
        if r >= 2 ** 256 or s >= 2 ** 256:
            continue
        try:
            pub.verify(utils.encode_dss_signature(r, s), d, utils.Prehashed(getattr(hashes, _HASH_OF[len(d)])()))
            ossl = True
        except InvalidSignature:
            ossl = False
        assert ossl == got, (row["domain"], row["tag"])
        n_ossl += 1
    assert n_ossl >= 150


def test_composite_q_rows_separate_fermat_from_modinverse(vec):
    """With q composite, w = s^(q-2) is not s^-1: honest signatures (which dsa.Verify accepts) fail the Fermat form,
    and the crafted ones (which it rejects) pass it.  These are the rows that catch the Fermat inverse."""
    comp = {d["name"] for d in vec["dsa_domains"] if len(d["factors"]) > 1}
    assert len(comp) == 4
    honest = crafted = noinv = 0
    for row in vec["dsa"]:
        if row["domain"] not in comp:
            continue
        a = dsa_args(vec, row)
        good, ferm = pgp.dsa_verify(*a), dsa_fermat(*a)
        if row["tag"] == "honest":
            assert good and not ferm
            honest += 1
        if row.get("fermat") and not row["tag"].endswith("tampered"):
            assert ferm and not good
            crafted += 1
        if row["tag"] in ("s_not_invertible", "s_eq_factor"):
            assert gcd(a[-1], a[1]) > 1 and not good
            noinv += 1
    assert honest >= 12 and crafted >= 12 and noinv >= 12


def test_dsa_rows_cover_the_edges(vec):
    tags = Counter((row["domain"], row["tag"]) for row in vec["dsa"])
    names = {d["name"] for d in vec["dsa_domains"]}
    assert {"q8_p1024", "q64_p1024", "q224_p2048", "q160_p2048", "q256_p1024", "q159_p1024"} <= names
    for t in ("z_ge_q", "z_eq_q", "z_zero", "dlen_20", "dlen_64", "s=1", "s=q-1", "r=1", "r=q-1", "g=1", "y=1", "y=p-1",
              "g_ge_p", "y_ge_p"):
        assert sum(v for (dn, tg), v in tags.items() if tg == t) >= len(names) - 1, t
    assert all(not row["expect"] for row in vec["dsa"] if row["domain"] == "q159_p1024")
    for row in vec["dsa"]:
        if row.get("raw"):
            p, q, g, y, _ = dsa_dom(vec, row)
            assert g >= p or y >= p


# ---- the Shamir ladder of ecdsa_verify_core, modelled on affine points ------------------------------------------------
def _neg(a):
    return None if a is None else (a[0], (-a[1]) % P)


def ladder_branches(q, digest, r, s):
    """Replays ecdsa_verify_core's table build and Shamir loop on exact points; returns the set of pt_add_v branches
    taken and the verdict.  Branches: table_double / table_infinity (G + Q), loop_double / loop_infinity (an add whose
    operands are equal / opposite), acc_inf_mid (an add into an accumulator that had been finite and returned to
    infinity), addend_inf (the table entry G + Q at infinity is added), result_inf, x_ge_n, z_ge_n."""
    br = set()
    if not (0 < r < N and 0 < s < N):
        return br, False
    e = int.from_bytes(digest[:32], "big")
    if e >= N:
        br.add("z_ge_n")
    w = pow(s, -1, N)
    u1, u2 = e * w % N, r * w % N
    if q == G:
        br.add("table_double")
    elif q == _neg(G):
        br.add("table_infinity")
    tab = [None, G, q, so.p256_add(G, q)]
    acc, was_finite = None, False
    for bit in range(255, -1, -1):
        acc = so.p256_add(acc, acc)
        idx = ((u1 >> bit) & 1) | (((u2 >> bit) & 1) << 1)
        if not idx:
            continue
        a = tab[idx]
        if acc is None:
            if was_finite:
                br.add("acc_inf_mid")
        elif a is None:
            br.add("addend_inf")
        elif acc == a:
            br.add("loop_double")
        elif acc == _neg(a):
            br.add("loop_infinity")
        acc = so.p256_add(acc, a)
        was_finite = was_finite or acc is not None
    if acc is None:
        br.add("result_inf")
        return br, False
    if acc[0] >= N:
        br.add("x_ge_n")
    return br, acc[0] % N == r


def _branch_of(tag):
    if tag == "x_ge_n/r=x":
        return None                                                   # r >= N: refused before the ladder
    base = tag.split("/")[0].split("@")[0]
    return {"loop_double": "loop_double", "loop_infinity": "loop_infinity", "acc_inf_mid": "acc_inf_mid",
            "table_double": "table_double", "table_infinity": "addend_inf", "result_inf": "result_inf",
            "x_ge_n": "x_ge_n", "z_ge_n": "z_ge_n", "u1_zero": None}.get(base)


MIN_BRANCH = {"loop_double": 12, "loop_infinity": 12, "acc_inf_mid": 12, "table_double": 3, "table_infinity": 3,
              "addend_inf": 3, "result_inf": 3, "x_ge_n": 3, "z_ge_n": 4}


def test_vectors_take_their_branches(vec):
    counts = Counter()
    for row in vec["ecdsa"]:
        if row["status"] == 3:
            continue
        q, d, r, s = ec_args(row)
        br, ok = ladder_branches(q, d, r, s)
        assert ok == row["expect"] == pgp.ecdsa_p256_verify(q, d, r, s), row["tag"]
        if "tampered" in row["tag"]:
            continue
        want = _branch_of(row["tag"])
        if want:
            assert want in br, (row["tag"], br)
        if row["tag"].startswith("x_ge_n/t="):
            assert "x_ge_n" in br
        if row["tag"] == "u1_zero/z_eq_n":
            assert "z_ge_n" in br
        counts.update(br)
    print("ladder branches reached:", dict(sorted(counts.items())))
    for b, m in MIN_BRANCH.items():
        assert counts[b] >= m, (b, counts[b])


# ---- host builds of the kernels' code ------------------------------------------------------------------------------
def _build(tmp_path, name, src):
    so_path = tmp_path / name
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-o", str(so_path), os.path.join(HERE, "harness", src)], check=True)
    return ctypes.CDLL(str(so_path))


def test_p256_core_on_host_matches_oracle(vec, tmp_path):
    """ecdsa_verify_core from csrc/p256.cuh, compiled with g++: status 1 / 0 as the oracle says, -1 (the kernel's status
    3) for the non-canonical key."""
    lib = _build(tmp_path, "libp256adv.so", "p256_host.cpp")
    for row in vec["ecdsa"]:
        q, d, r, s = ec_args(row)
        pub = b"\x04" + q[0].to_bytes(32, "big") + q[1].to_bytes(32, "big")
        got = lib.p256_ecdsa_verify_host(pub, r.to_bytes(32, "big"), s.to_bytes(32, "big"), d, len(d))
        want = -1 if row["status"] == 3 else int(pgp.ecdsa_p256_verify(q, d, r, s))
        assert got == want, row["tag"]


def test_modinv_on_host(vec, tmp_path):
    """modinv_big from csrc/modinv_big.cuh against pow(s, -1, q): random odd moduli of 3..256 bits, prime and
    composite, operands sharing a factor with them, and every s of the composite-q DSA rows; and at 64 limbs (K7's
    m^-1 mod N) random odd 2048-bit moduli and an RSA modulus p q with 0, 1, N - 1 and multiples of p and of q."""
    lib = _build(tmp_path, "libmodinv.so", "modinv_host.cpp")
    out = ctypes.create_string_buffer(32)

    def check(a, m):
        rc = lib.modinv_host(a.to_bytes(32, "big"), m.to_bytes(32, "big"), out)
        if gcd(a, m) == 1:
            assert rc == 1 and int.from_bytes(out.raw, "big") == pow(a, -1, m), (a, m)
        else:
            assert rc == 0 and out.raw == bytes(32), (a, m)

    rng = random.Random(0xBF7C51A1)
    n = 0
    for bits in [3, 8, 31, 32, 33, 63, 64, 65, 160, 224, 255, 256] * 8:
        m = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
        for a in (0, 1, 2, m - 1, m - 2, rng.randrange(m), rng.randrange(m) & ~0xffff, 1 << (bits - 2)):
            check(a % m, m)
            n += 1
        f = 3 if m % 3 == 0 else (5 if m % 5 == 0 else None)
        if f:
            check(f * rng.randrange(m // f) % m, m)
    for row in vec["dsa"]:
        p, q, g, y, D = dsa_dom(vec, row)
        s = _h(row["s"])
        if s < q:
            check(s, q)
            n += 1
    for m in (2 ** 256 - 189, N, P, 3):
        check(rng.randrange(1, m), m)
    assert n > 1000

    # modinv_big<64>: thrsa_modinv_kernel's m^-1 mod N on 2048-bit moduli, random odd ones and the RSA modulus of the
    # threshold key with operands that share its factor p
    out64 = ctypes.create_string_buffer(256)

    def check64(a, m):
        rc = lib.modinv_host64(a.to_bytes(256, "big"), m.to_bytes(256, "big"), out64)
        if gcd(a, m) == 1:
            assert rc == 1 and int.from_bytes(out64.raw, "big") == pow(a, -1, m), (a, m)
        else:
            assert rc == 0 and out64.raw == bytes(256), (a, m)

    key = json.load(open(os.path.join(HERE, "golden", "thrsa_key.json")))
    p, q = _h(key["p"]), _h(key["q"])
    assert p * q == _h(key["n"]) and (p * q).bit_length() == 2048
    moduli = [rng.getrandbits(2048) | (1 << 2047) | 1 for _ in range(6)] + [p * q]
    for m in moduli:
        for a in (0, 1, 2, m - 1, m - 2, rng.randrange(m), 1 << 2046):
            check64(a, m)
    for _ in range(4):
        check64(p * rng.randrange(1, q), p * q)
        check64(q * rng.randrange(1, p), p * q)
