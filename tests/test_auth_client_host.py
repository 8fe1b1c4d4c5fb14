"""The client half of crypto/auth (K10) on the CPU: the oracle client checked on its own terms, the AES-GCM core K9's seal
and K10's open share (tests/harness/auth_client_host.cpp builds it with g++ over libcrypto's AES) against
`cryptography`'s AESGCM, and the SASS check that no K10 kernel uses local memory."""
import ctypes
import os
import random
import subprocess

import pytest

import auth_oracle as A
from oracle import sss_oracle as sss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n,k", [(4, 3), (10, 7)])
def test_oracle_cipher_key_is_the_password_secret(n, k):
    """A full round's key is H((PI^s).Bytes(), pw) with s interpolated from generate_params' y values: the oracle client
    derives the one key the password and the registered parameters define, whatever a and a' were."""
    rng = A.Rng(0x5EC + n)
    pw, proof = b"hunter2", b"the proof"
    params = A.generate_params(pw, n, k, A.Rng(0x5EC + n))
    c, pis = A.run_round(pw, proof, n, k, rng, make_servers=lambda ps, pf: [A.Server(p, pf) for p in params])
    assert pis is not None and set(pis.values()) == {proof}
    shares = [(x, y) for x, y, _, _ in (A.parse_params(p) for p in params[:k])]
    s = sss.calculate_secret(shares, A.Q)
    assert c.get_cipher_key() == A.h(A.i2b(pow(A.PI(pw), s, A.P)), pw)


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libauthclienthost.so")
    src = os.path.join(ROOT, "tests", "harness", "auth_client_host.cpp")
    deps = [src] + [os.path.join(ROOT, "bftkv_b200", "csrc", f) for f in ("auth_server.cuh", "sha256.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-deprecated-declarations", "-o", so, src, "-lcrypto"])
    return ctypes.CDLL(so)


def _core(host, key, nonce, aad, src, seal):
    dst = ctypes.create_string_buffer(max(1, len(src)))
    tag = ctypes.create_string_buffer(16)
    host.auth_gcm_core_host(key, nonce, aad, ctypes.c_uint64(len(aad)), src, ctypes.c_uint64(len(src)), dst, int(seal), tag)
    return dst.raw[:len(src)], tag.raw


@pytest.mark.parametrize("aad_len", [0, 32])
@pytest.mark.parametrize("length", [0, 1, 15, 16, 17, 255])
def test_gcm_core_against_aesgcm(host, aad_len, length):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    rng = random.Random(aad_len * 1000 + length)
    key, nonce, aad, pt = rng.randbytes(16), rng.randbytes(12), rng.randbytes(aad_len), rng.randbytes(length)
    ref = AESGCM(key).encrypt(nonce, pt, aad)
    ct, tag = _core(host, key, nonce, aad, pt, True)
    assert ct + tag == ref
    out, tag2 = _core(host, key, nonce, aad, ct, False)                      # open: the same tag over the ciphertext
    assert (out, tag2) == (pt, tag)
    # open over a changed ciphertext, aad or nonce: the tag it computes is the one AESGCM seals the resulting plain text
    # under, so the kernel's compare against the received tag fails exactly when AESGCM.decrypt would
    cases = [(ct, aad, nonce[:5] + bytes([nonce[5] ^ 0x10]) + nonce[6:])]
    if length:
        at = rng.randrange(length)
        cases.append((ct[:at] + bytes([ct[at] ^ 1 << rng.randrange(8)]) + ct[at + 1:], aad, nonce))
    if aad_len:
        cases.append((ct, aad[:-1] + bytes([aad[-1] ^ 0x80]), nonce))
    for c2, a2, n2 in cases:
        out2, tag3 = _core(host, key, n2, a2, c2, False)
        assert AESGCM(key).encrypt(n2, out2, a2) == c2 + tag3
        assert tag3 != tag


def test_k10_kernels_use_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    fns = {b.split("\n", 1)[0].strip(): b for b in sass.split("Function :")[1:]}
    for kernel in ("auth_zq_kernel", "auth_words_kernel", "auth_cipher_key_kernel", "auth_gcm_open_kernel", "auth_kdf_mac_kernel",
                   "auth_gcm_seal_kernel"):
        bodies = [b for name, b in fns.items() if kernel in name]
        assert bodies, kernel
        for b in bodies:
            assert "LDL" not in b and "STL" not in b, f"{kernel} uses local memory"
