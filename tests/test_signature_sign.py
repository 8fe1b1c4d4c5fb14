"""PGPSignature.Sign on the CPU: the oracle (tests/signature_sign_oracle.py) against every packet of
tests/golden/signature_sign.json, the packet helpers the library signs with (sign_packet.hpp, built with g++ by
tests/harness/sign_host.cpp) against the oracle, the release step with failing checks, and K12's local-memory shape."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import signature_sign_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_signature_sign as G  # noqa: E402

FIXTURE = json.load(open(os.path.join(ROOT, "tests", "golden", "signature_sign.json")))
SIGNING_FAILED = -21


@pytest.fixture(scope="module")
def keys():
    return {name: (k, O.key_block(k)[1]) for name, k in G.keys().items()}


def test_oracle_reproduces_every_fixture_packet(keys):
    for c in FIXTURE["cases"]:
        k, kid = keys[c["key"]]
        assert "%016x" % kid == c["key_id"]
        got = O.packet(k, kid, G.tbs_bytes(c["tbs_len"], c["tbs_index"]), c["ctime"])
        assert got.hex() == c["packet"], (c["key"], c["tbs_len"], c["ctime"])
        assert len(got) == O.PACKET_BYTES and got[-258:-256] == b"\x08\x00"
        assert int.from_bytes(got[-256:], "big").bit_length() == c["s_bits"]
        assert c["gnupg_ok"] == (c["ctime"] > 1)              # GnuPG refuses only signatures older than the key


def test_fixture_covers_the_edges():
    cs = FIXTURE["cases"]
    assert {c["key"] for c in cs} == set(G.KEYS)
    for name in G.KEYS:
        mine = [c for c in cs if c["key"] == name]
        assert {c["tbs_len"] for c in mine} >= set(G.LENGTHS)
        assert {c["ctime"] for c in mine} >= set(G.CTIMES)
        assert any(c["s_bits"] < 2048 for c in mine)
        assert any(c["s_bits"] <= 2040 and bytes.fromhex(c["packet"])[-256] == 0 for c in mine)
    # with the 28 suffix bytes these end the hashed stream on both sides of 55 / 56 and 119 / 120 bytes
    assert len(O.suffix(0, 0)) == 28 and {27 + 28, 28 + 28, 91 + 28, 92 + 28} == {55, 56, 119, 120}


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libsignhost.so")
    src = os.path.join(ROOT, "tests", "harness", "sign_host.cpp")
    deps = [src, os.path.join(ROOT, "bftkv_b200", "csrc", "sign_packet.hpp"), os.path.join(ROOT, "include", "bftq.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.sign_suffix_host.argtypes = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p]
    lib.sign_release_host.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def test_suffix_matches_the_oracle(host):
    buf = (ctypes.c_uint8 * 28)()
    for ct in (0, 1, 0x5F000000, 1 << 31, (1 << 32) - 1):
        for kid in (0, 1, 0x470F1BF15EE422E6, (1 << 64) - 1):
            host.sign_suffix_host(ct, kid, buf)
            assert bytes(buf) == O.suffix(ct, kid)


def test_release_zeroes_failed_items(host):
    rng = np.random.default_rng(12)
    n = 257
    packets = rng.integers(0, 256, n * O.PACKET_BYTES, dtype=np.uint8)
    before = packets.copy()
    status = np.zeros(n, np.uint8)
    status[[0, 5, 100, n - 1]] = [1, 2, 4, 1]                  # K1's failing statuses: bad signature, hash tag, unknown key
    err = np.full(n, 99, np.int32)
    host.sign_release_host(status.ctypes.data, n, packets.ctypes.data, err.ctypes.data)
    pk, bf = packets.reshape(n, -1), before.reshape(n, -1)
    for i in range(n):
        if status[i]:
            assert err[i] == SIGNING_FAILED and not pk[i].any()
        else:
            assert err[i] == 0 and np.array_equal(pk[i], bf[i])


def test_k12_uses_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    bodies = [b for b in sass.split("Function :")[1:] if "rsa_crt_sign_kernel" in b.split("\n", 1)[0]]
    assert bodies
    for b in bodies:
        assert "LDL" not in b and "STL" not in b, "rsa_crt_sign_kernel spills to local memory"
    usage = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout.split("\n")
    seen = 0
    for i, line in enumerate(usage):
        if "rsa_crt_sign_kernel" in line:
            assert "STACK:0 " in usage[i + 1] and "LOCAL:0 " in usage[i + 1], usage[i + 1]
            seen += 1
    assert seen == 1


def test_sign_batch_needs_one_ctime_per_tbs(built):
    from bftkv_b200.crypto_gpu import Keyring, Signature
    kr = Keyring(None)                                 # parse-only: the length check comes before the library call
    with pytest.raises(ValueError):
        Signature(kr).sign_batch([b"a", b"b"], [1])
    kr.close()
