"""K1b Ed25519 on keys and signatures a Byzantine peer builds (tests/golden/ed25519_adversarial.json): small-order,
mixed-order and non-canonically encoded keys, small-order and mixed-order R, non-canonical R, S at and past L, scalars
whose window digits sit at the ends of the tables.  The verdict is Go's crypto/ed25519.Verify (oracle/ed25519_oracle.py),
which decodes A as edwards25519.Point.SetBytes does: y is reduced mod p and x = 0 may carry the sign bit.  OpenSSL must
agree on every row; libsodium is stricter on small-order and non-canonical points, and only there.  CPU tests run the
kernels' own __host__ __device__ code (tests/harness/ed25519_host.cpp)."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys
from collections import Counter

import pytest

from oracle import ed25519_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ed25519_adversarial.json")
P, L = eo.P, eo.L
# rows where libsodium may say no although Go and OpenSSL say yes: it rejects small-order A and R and non-canonical A
SODIUM_STRICTER = {"small_order_A", "small_order_R", "noncanon_A"}
MIN_ROWS = {"small_order_A": 16, "noncanon_A": 40, "mixed_A": 14, "small_order_R": 16, "mixed_R": 8, "noncanon_R": 8,
            "S_edge": 12, "digit_edge": 24, "undecodable_A": 8}


@pytest.fixture(scope="module")
def rows():
    return json.load(open(GOLDEN))["rows"]


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libedhost.so")
    src = os.path.join(ROOT, "tests", "harness", "ed25519_host.cpp")
    deps = [src] + [os.path.join(ROOT, "bftkv_b200", "csrc", h) for h in ("ed25519.cuh", "ed25519_fast.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def _unpack(row):
    return bytes.fromhex(row["a"]), bytes.fromhex(row["sig"]), bytes.fromhex(row["msg"])


def _openssl(a, sig, m):
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PublicKey
    try:
        Ed25519PublicKey.from_public_bytes(a).verify(sig, m)
        return True
    except Exception:
        return False


def _sodium(a, sig, m):
    import nacl.exceptions
    import nacl.signing
    try:
        nacl.signing.VerifyKey(a).verify(m, sig)
        return True
    except (nacl.exceptions.BadSignatureError, nacl.exceptions.ValueError):
        return False


def test_generator_reproduces_the_vectors(tmp_path):
    out = tmp_path / "ed.json"
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tests", "golden", "make_ed25519_adversarial.py"), str(out)],
                          stdout=subprocess.DEVNULL)
    assert out.read_bytes() == open(GOLDEN, "rb").read()


def test_row_counts_and_twins(rows):
    n = Counter(r["tag"] for r in rows)
    for tag, lo in MIN_ROWS.items():
        assert n[tag] >= lo, (tag, n[tag])
    assert set(n) == set(MIN_ROWS)
    # every accepted row is followed by a rejected twin (the same tag)
    for i, r in enumerate(rows):
        if r["expect"]:
            assert not rows[i + 1]["expect"] and rows[i + 1]["tag"] == r["tag"], i
    acc = Counter(r["tag"] for r in rows if r["expect"])
    for tag in ("small_order_A", "noncanon_A", "mixed_A", "small_order_R", "mixed_R", "noncanon_R", "S_edge", "digit_edge"):
        assert acc[tag] >= 3, tag
    # the non-canonical keys that carry valid signatures: y = p (order 4), y = p + 1 (the identity), -0 forms
    ok_keys = {r["a"] for r in rows if r["tag"] == "noncanon_A" and r["expect"]}
    assert {(P + 1).to_bytes(32, "little").hex(), ((P + 1) | 1 << 255).to_bytes(32, "little").hex(),
            (1 | 1 << 255).to_bytes(32, "little").hex(), ((P - 1) | 1 << 255).to_bytes(32, "little").hex()} <= ok_keys
    assert len(ok_keys) == 6


def test_oracle_is_go_semantics(rows):
    """The restatement decides every row as the vectors say, and agrees with RFC 8032 test vector 1."""
    for r in rows:
        assert eo.verify(*_unpack(r)) == r["expect"], r["note"]
    pk = bytes.fromhex("d75a980182b10ab7d54bfed3c964073a0ee172f3daa62325af021a68f707511a")
    sig = bytes.fromhex("e5564300c360ac729086e2cc806e828a84877f1eb8e5d974d873e065224901555fb8821590a33bacc61e39701cf9b46bd25bf5f0595bbe24655141438e7a100b")
    assert eo.verify(pk, sig, b"") and not eo.verify(pk, sig[:63] + b"\x0a", b"")
    # the decoders: loose (Go) and strict (RFC 8032) differ exactly on y >= p and on -0
    for y in (0, 1, P - 1, P, P + 1, P + 3, 2 ** 255 - 1):
        for sign in (0, 1):
            b = ((y | sign << 255) & (2 ** 256 - 1)).to_bytes(32, "little")
            loose, strict = eo.decode_go(b), eo.decode_strict(b)
            if strict is not None:
                assert loose == strict
            elif loose is not None:
                assert y >= P or loose[0] == 0


def test_openssl_agrees_on_every_row(rows):
    bad = [r["note"] for r in rows if _openssl(*_unpack(r)) != r["expect"]]
    assert not bad, bad


def test_libsodium_is_stricter_only_where_known(rows):
    """libsodium rejects small-order A and R and non-canonical A.  It never accepts what Go rejects, and it rejects
    what Go accepts only on rows of those tags and on rows of other tags whose A or R is of small order (the S and
    digit edges run under the identity key; a valid non-canonical R is a small-order point)."""
    def small(b):
        pt = eo.decode_go(b)
        return pt is not None and eo.order(pt) is not None
    differ = Counter()
    for r in rows:
        a, sig, m = _unpack(r)
        if _sodium(a, sig, m) != r["expect"]:
            assert r["expect"], r["note"]
            assert r["tag"] in SODIUM_STRICTER or small(a) or small(sig[:32]), r["note"]
            differ[r["tag"]] += 1
    assert SODIUM_STRICTER <= set(differ), differ
    assert not {"mixed_A", "mixed_R", "undecodable_A"} & set(differ), differ


@pytest.mark.parametrize("core", ["ed_verify_core_host", "ed_verify_fast_host", "ed_verify_core_fast_host"])
def test_host_cores_match_the_vectors(host, rows, core):
    """The classic core (ed25519.cuh), the window-table path (accumulate + finish) and the table-free fast core each
    decide every row as Go does."""
    f = getattr(host, core)
    bad = []
    for r in rows:
        a, sig, m = _unpack(r)
        got = f(sig, a, hashlib.sha512(sig[:32] + a + m).digest())
        if got != int(r["expect"]):
            bad.append((r["tag"], r["note"]))
    assert not bad, f"{len(bad)} rows: {bad}"


def test_table_entries_of_adversarial_keys(host, rows):
    """Window-table entries j * 2^(10 w) * A of small-order, mixed-order and non-canonically encoded keys (the tables the
    cache builds for them) against big-integer arithmetic on the point Go decodes."""
    T8 = bytes.fromhex(json.load(open(GOLDEN))["T8"])
    mixed = [bytes.fromhex(r["a"]) for r in rows if r["tag"] == "mixed_A"][::2][:3]
    keys = [T8, eo.encode(eo.mul(2, eo.decode_go(T8))), (P - 1).to_bytes(32, "little"), (1).to_bytes(32, "little")] + mixed + \
           [((P + t) | s << 255).to_bytes(32, "little") for t, s in ((0, 0), (0, 1), (1, 0), (1, 1), (3, 0), (9, 1), (18, 1))] + \
           [(1 | 1 << 255).to_bytes(32, "little"), ((P - 1) | 1 << 255).to_bytes(32, "little")]
    e1, e2, e3 = (ctypes.create_string_buffer(32) for _ in range(3))
    for a32 in keys:
        A = eo.decode_go(a32)
        assert A is not None
        for w, j in ((0, 1), (0, 2), (0, 8), (0, 512), (1, 3), (13, 511), (25, 1), (25, 512)):
            assert host.ed_fx_table_entry_host(a32, 0, w, j, e1, e2, e3) == 1, (a32.hex(), w, j)
            x, y = eo.mul(j << (10 * w), A)
            assert int.from_bytes(e1.raw, "little") == (y + x) % P and int.from_bytes(e2.raw, "little") == (y - x) % P, (a32.hex(), w, j)
            assert int.from_bytes(e3.raw, "little") == 2 * eo.D * x * y % P, (a32.hex(), w, j)
