"""K8's constant-time cores on the CPU (tests/harness/thdsa_host.cpp builds thdsa_sign.cuh with g++): the fixed-base a G
against the oracle and `cryptography`, the complete addition on doublings, inverses and the identity, and the Z_q
Horner reduction and products at the limb-class edges of the threshold fixtures."""
import ctypes
import json
import os
import random
import subprocess

import pytest

from oracle import sss_oracle as sss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, G, P = sss.P256_N, sss.P256_G, sss.P256_P


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libthdsahost.so")
    src = os.path.join(ROOT, "tests", "harness", "thdsa_host.cpp")
    deps = [src] + [os.path.join(ROOT, "bftkv_b200", "csrc", f) for f in ("thdsa_sign.cuh", "p256.cuh", "lagrange.cuh", "limbs.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def marshal(pt):
    return b"\x04" + bytes(64) if pt is None else sss.p256_marshal(pt)


def test_base_mul(host):
    from cryptography.hazmat.primitives.asymmetric import ec
    rng = random.Random(0xD5A6)
    out = ctypes.create_string_buffer(65)
    for a in [0, 1, 2, N - 2, N - 1, N, 2 ** 255, 2 ** 256 - 1] + [rng.randrange(N) for _ in range(20)]:
        host.thdsa_base_mul_host(a.to_bytes(32, "big"), out)
        assert out.raw == marshal(sss.p256_mul(a, G)), hex(a)
        if 0 < a < N:
            pn = ec.derive_private_key(a, ec.SECP256R1()).public_key().public_numbers()
            assert out.raw == b"\x04" + pn.x.to_bytes(32, "big") + pn.y.to_bytes(32, "big")


def test_complete_addition(host):
    rng = random.Random(0xD5A7)
    out = ctypes.create_string_buffer(65)
    inf = b"\x00" * 65
    for _ in range(10):
        Pt = sss.p256_mul(rng.randrange(1, N), G)
        Q = sss.p256_mul(rng.randrange(1, N), G)
        neg = (Pt[0], P - Pt[1])
        for a, b, want in [(Pt, Q, sss.p256_add(Pt, Q)), (Pt, Pt, sss.p256_add(Pt, Pt)), (Pt, neg, None)]:
            host.thdsa_add_host(sss.p256_marshal(a), sss.p256_marshal(b), out)
            assert out.raw == marshal(want)
        host.thdsa_add_host(inf, sss.p256_marshal(Pt), out)
        assert out.raw == sss.p256_marshal(Pt)
        host.thdsa_add_host(sss.p256_marshal(Pt), inf, out)
        assert out.raw == sss.p256_marshal(Pt)
    host.thdsa_add_host(inf, inf, out)
    assert out.raw == marshal(None)


def test_zq_edges(host):
    edges = json.load(open(os.path.join(ROOT, "tests", "golden", "threshold_edges.json")))
    rng = random.Random(0xD5A8)
    qs = [N, (1 << 159) + 7, (1 << 255) - 19, (1 << 33) + 1]
    for h in edges["k3_moduli"].values():                      # the K3 limb-class moduli that K8 accepts (33..256 bits)
        m = int(h, 16)
        if (1 << 32) < m < (1 << 256) and m & 1:
            qs.append(m)
    assert len(qs) > 6
    out, out2 = ctypes.create_string_buffer(32), ctypes.create_string_buffer(32)
    for q in qs:
        qb = q.to_bytes((q.bit_length() + 7) // 8, "big")
        for v in [0, 1, q - 1, q, q + 1, 2 * q - 1, (1 << 32) - 1, 1 << 32, (1 << 256) - 1, (1 << 600) + q, rng.getrandbits(1000)]:
            vb = v.to_bytes(max(1, (v.bit_length() + 7) // 8), "big")
            a, b = rng.randrange(q), rng.getrandbits(256)
            host.thdsa_zq_host(qb, len(qb), vb, len(vb), a.to_bytes(32, "big"), b.to_bytes(32, "big"), out, out2)
            assert int.from_bytes(out.raw, "big") == v % q
            assert int.from_bytes(out2.raw, "big") == a * b % q
