"""K9's symmetric cores on the CPU (tests/harness/auth_host.cpp builds auth_server.cuh and sha256.cuh with g++): the GHASH
multiply against a bit-serial GF(2^128) product, HMAC-SHA256 and keySched's HKDF against `cryptography` at the salt and
key-material lengths that change the block count, and the SASS check that no K9 kernel uses local memory."""
import ctypes
import os
import random
import subprocess

import pytest

import auth_oracle as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libauthhost.so")
    src = os.path.join(ROOT, "tests", "harness", "auth_host.cpp")
    deps = [src] + [os.path.join(ROOT, "bftkv_b200", "csrc", f) for f in ("auth_server.cuh", "sha256.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def test_gf128_mul(host):
    rng = random.Random(0x6A5)
    R = 0xE1 << 120
    edges = [0, 1, 1 << 127, 1 << 120, R, R | 1, (1 << 128) - 1, 0x80, 1 << 64, (1 << 64) - 1]
    vals = edges + [rng.getrandbits(128) for _ in range(40)]
    buf = ctypes.create_string_buffer(16)
    for h in vals:
        for x in vals[:12] + [rng.getrandbits(128) for _ in range(4)]:
            buf.raw = x.to_bytes(16, "big")
            host.auth_gf128_mul_host(buf, h.to_bytes(16, "big"))
            assert int.from_bytes(buf.raw, "big") == A.gf128_mul(x, h), (hex(x), hex(h))


@pytest.mark.parametrize("salt_len", [0, 1, 32, 64, 65, 200])
@pytest.mark.parametrize("ikm_len", [0, 1, 55, 56, 64, 255, 256])
def test_hkdf_and_hmac(host, salt_len, ikm_len):
    from cryptography.hazmat.primitives import hashes, hmac
    from cryptography.hazmat.primitives.kdf.hkdf import HKDF
    rng = random.Random(salt_len * 977 + ikm_len)
    salt, ikm = rng.randbytes(salt_len), rng.randbytes(ikm_len)
    out = ctypes.create_string_buffer(32)
    host.auth_hkdf_host(salt, len(salt), ikm, len(ikm), out)
    assert out.raw == HKDF(hashes.SHA256(), 32, salt or None, None).derive(ikm)
    km = out.raw[:16]
    xi, bi = rng.randbytes(ikm_len), rng.randbytes(salt_len)
    host.auth_mac_host(km, xi, len(xi), bi, len(bi), out)
    m = hmac.HMAC(km, hashes.SHA256())
    m.update(xi + bi)
    assert out.raw == m.finalize()
    if salt_len <= 64:
        host.auth_hmac_host(salt, len(salt), ikm, len(ikm), out)
        m = hmac.HMAC(salt, hashes.SHA256())
        m.update(ikm)
        assert out.raw == m.finalize()


def test_k9_kernels_use_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    fns = {b.split("\n", 1)[0].strip(): b for b in sass.split("Function :")[1:]}
    for kernel in ("auth_pow_kernel", "auth_kdf_mac_kernel", "auth_gcm_seal_kernel"):
        bodies = [b for name, b in fns.items() if kernel in name]
        assert bodies, kernel
        for b in bodies:
            assert "LDL" not in b and "STL" not in b, f"{kernel} uses local memory"
