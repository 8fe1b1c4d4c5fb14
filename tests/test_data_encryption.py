"""DataEncryption's oracle and host layout on the CPU: the oracle (tests/data_encryption_oracle.py) against every GnuPG
verdict in tests/golden/data_encryption.json and its own Go-shaped entries byte for byte, the layout function the
library plans encrypt calls with (data_layout.hpp, built with g++ by tests/harness/data_host.cpp) against the oracle's
writer cascade, and the K11 kernels' register and local-memory shape."""
import base64
import ctypes
import hashlib
import json
import os
import subprocess

import pytest

import data_encryption_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = json.load(open(os.path.join(ROOT, "tests", "golden", "data_encryption.json")))
KIND = {"raw": 0, "byte": 1, "prefix": 2, "body": 3, "mdc": 4}


@pytest.mark.parametrize("case", FIXTURE["cases"], ids=lambda c: c["name"])
def test_oracle_agrees_with_gnupg(case):
    msg = base64.b64decode(case["message"])
    code, plain = O.decrypt(case["passphrase"].encode(), msg)
    assert code == case["code"]
    if code == O.OK:
        assert case["gnupg_ok"] and hashlib.sha256(plain).hexdigest() == case["gnupg_plain_sha256"]
        assert plain == O.fixture_value(case["plain_len"], case["seed"])
    else:
        assert not case["gnupg_ok"] or code == O.UNSUPPORTED
    if case["source"] == "go":
        assert O.encrypt(case["passphrase"].encode(), plain, bytes.fromhex(case["rand"])) == msg
        assert len(msg) == O.encrypted_len(len(plain))


def test_oracle_wrong_key_and_divergences():
    rand = bytes(range(40))
    msg = O.encrypt(b"k" * 32, b"value", rand)
    assert O.decrypt(b"k" * 32, msg) == (O.OK, b"value")
    assert O.decrypt(b"k" * 31, msg) == (O.DECRYPTION_FAILED, None)
    assert O.decrypt(b"k" * 32, msg[:-1]) == (O.MALFORMED, None)         # the outer writer's closing 00 is missing


@pytest.fixture(scope="module")
def layout():
    so = os.path.join(ROOT, "tests", "harness", "libdatahost.so")
    src = os.path.join(ROOT, "tests", "harness", "data_host.cpp")
    deps = [src, os.path.join(ROOT, "bftkv_b200", "csrc", "data_layout.hpp")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.data_layout_host.restype = ctypes.c_uint64
    lib.data_layout_host.argtypes = [ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]
    buf = (ctypes.c_uint32 * 4096)()
    nw = ctypes.c_uint64()

    def call(n):
        total = lib.data_layout_host(n, buf, 4096, ctypes.byref(nw))
        return total, list(buf[:nw.value])
    return call


def _want(n):
    """The oracle's cascade as layout words: kind << 24 | framing byte << 16 | length."""
    ws = O.writes(n)
    inner = [224 + w.bit_length() - 1 for k, w in ws if k == "body"]
    framing = iter([0xCB] + inner + [0x00])
    out = []
    for k, w in ws:
        b = 0x01 if k == "raw" else next(framing) if k == "byte" else 0
        out.append(KIND[k] << 24 | b << 16 | w)
    return out


def test_layout_matches_the_oracle(layout):
    lengths = list(range(0, 20001)) + sorted({(1 << k) + d for k in range(15, 21) for d in (-1, 0, 1)})
    for n in lengths:
        total, words = layout(n)
        assert total == O.encrypted_len(n), n
        assert words == _want(n), n


def test_k11_kernels_use_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    fns = {b.split("\n", 1)[0].strip(): b for b in sass.split("Function :")[1:]}
    for kernel in ("s2k_kernel", "data_cand_kernel", "data_encrypt_kernel"):
        bodies = [b for name, b in fns.items() if kernel in name]
        assert bodies, kernel
        for b in bodies:
            assert "LDL" not in b and "STL" not in b, f"{kernel} spills to local memory"
    usage = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout.split("\n")
    seen = 0
    for i, line in enumerate(usage):
        if any(k in line for k in ("s2k_kernel", "data_cand_kernel", "data_encrypt_kernel")):
            assert "STACK:0 " in usage[i + 1] and "LOCAL:0 " in usage[i + 1], usage[i + 1]
            seen += 1
    assert seen == 3
