"""CPU suite for threshold DSA / ECDSA: the oracle's full rounds produce signatures `cryptography` verifies (the property
the reference's TestThreshold asserts), and K8's kernels keep every secret out of local memory."""
import os
import random
import subprocess

import pytest

import threshold_dsa_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _verify(g, x: int, digest: bytes, sig: bytes) -> None:
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import dsa, ec, utils
    q = O.order(g)
    n = (q.bit_length() + 7) // 8
    der = utils.encode_dss_signature(int.from_bytes(sig[:n], "big"), int.from_bytes(sig[n:], "big"))
    if g["kind"] == "dsa":
        pn = dsa.DSAParameterNumbers(g["p"], g["q"], g["g"])
        pub = dsa.DSAPublicNumbers(pow(g["g"], x, g["p"]), pn).public_key()
        pub.verify(der, digest, utils.Prehashed(hashes.SHA256()) if len(digest) == 32 else hashes.SHA256())
    else:
        pub = ec.derive_private_key(x, ec.SECP256R1()).public_key()
        pub.verify(der, digest, ec.ECDSA(utils.Prehashed(hashes.SHA256())))


def round_trip(g, n: int, seed: int, key: int = None):
    """Distribute, phase 1 on every server, phase 2 / 3 on the first 2t, CalculateR, calculateS, formatDSA."""
    rng = random.Random(seed)
    t = n // 2
    x, coords = O.deal(rng, g, n, t, key)
    q = O.order(g)
    joint = [O.joint_shares(rng, g, n, t) for _ in range(n)]           # joint[j][i]: server j's shares for node i
    parts, kc = [], {}
    for i in range(2 * t):
        X, k, c, out = O.phase2(g, [O.share_plain(joint[j][i]) for j in range(n)])
        kc[i] = (k, c)
        parts.append(O.parse_partial(g, out))
    import hashlib
    digest = hashlib.sha256(b"tbs %d" % seed).digest()
    m = int.from_bytes(digest[:(q.bit_length() + 7) // 8], "big")
    if len(digest) * 8 > q.bit_length():
        m >>= 8 * ((q.bit_length() + 7) // 8) - q.bit_length()
    r = O.calculate_r(g, [(px, ri, vi) for px, ri, vi in parts])
    sparts = []
    for i in range(2 * t):
        X, Y = coords[i]
        out = O.phase3(g, X, Y, m, r, *kc[i])
        px, s, _ = O.parse_partial(g, out)
        sparts.append((px, int.from_bytes(s, "big")))
    s = O.calculate_s(g, sparts)
    # TestDSA's arithmetic (dsa_test.go:222-330): r = g^(k^-1) mod p mod q (ECDSA: (k^-1 G).x mod N), s = k (m + x r) mod q
    kk = O.calculate_s(g, [(i + 1, kc[i][0]) for i in range(2 * t)])
    if g["kind"] == "dsa":
        assert r == pow(g["g"], pow(kk, -1, q), g["p"]) % q
    else:
        from oracle import sss_oracle as S
        assert r == S.p256_mul(pow(kk, -1, q), S.P256_G)[0] % q
    assert s == kk * (m + x * r) % q
    return x, digest, O.format_dsa(r, s, q)


@pytest.mark.parametrize("n", [4, 7, 10])
def test_oracle_round_verifies_p256(n):
    g = dict(kind="p256")
    x, digest, sig = round_trip(g, n, 0xD5A0 + n)
    _verify(g, x, digest, sig)


@pytest.mark.parametrize("n", [4, 7, 10])
def test_oracle_round_verifies_reference_dsa_key(n):
    g, key = O.golden_key()
    assert pow(g["g"], g["q"], g["p"]) == 1 and g["p"].bit_length() == 1024 and g["q"].bit_length() == 160
    x, digest, sig = round_trip(g, n, 0xD5A1 + n, key)
    _verify(g, x, digest, sig)


@pytest.mark.parametrize("qbits,n", [(224, 4), (256, 7), (256, 10)])
def test_oracle_round_verifies_dsa(qbits, n):
    g = O.dsa_group(2048, qbits)
    x, digest, sig = round_trip(g, n, 0xD5A1 + n)
    _verify(g, x, digest, sig)


def test_k8_kernels_use_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    fns = {b.split("\n", 1)[0].strip(): b for b in sass.split("Function :")[1:]}
    for kernel in ("thdsa_zq_kernel", "thdsa_dsa_r_kernel", "thdsa_p256_base_kernel", "thdsa_copy_kc_kernel"):
        bodies = [b for name, b in fns.items() if kernel in name]
        assert bodies, kernel
        for b in bodies:
            assert "LDL" not in b and "STL" not in b, f"{kernel} uses local memory"
