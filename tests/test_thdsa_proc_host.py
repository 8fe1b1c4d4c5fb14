"""The threshold-DSA client's host wire code on the CPU (tests/harness/thdsa_proc_host.cpp builds thdsa_wire.hpp and
bignum_host.hpp's be_mod with g++) against the client oracle (tests/threshold_dsa_proc_oracle.py): parseJointShare and
parsePartialSignature at every truncation point of one answer of each phase, both requests, OS2I, formatDSA and the
reduction of Byzantine sizes."""
import ctypes
import hashlib
import os
import random
import struct
import subprocess

import pytest

import threshold_dsa_oracle as O
import threshold_dsa_proc_oracle as P
from test_threshold_dsa_proc import Round

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libthdsaprochost.so")
    src = os.path.join(ROOT, "tests", "harness", "thdsa_proc_host.cpp")
    deps = [src] + [os.path.join(ROOT, "bftkv_b200", "csrc", f) for f in ("thdsa_wire.hpp", "wire_host.hpp", "bignum_host.hpp")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    for f in ("thdsa_joint_host", "thdsa_partial_host", "thdsa_request1_host", "thdsa_request2_host", "thdsa_format_host"):
        getattr(lib, f).restype = ctypes.c_int64
    return lib


def call(fn, *args):
    out = ctypes.create_string_buffer(1 << 16)
    n = fn(*args, out, ctypes.c_uint64(len(out)))
    return None if n == -1 else out.raw[:n]


def want_joint(data: bytes):
    r = P.Reader(data)
    try:
        shares = [(r.chunk(), r.uint(8)) for _ in range(r.uint(2))]
    except P.ParseError:
        return None
    return struct.pack(">I", len(shares)) + b"".join(struct.pack(">Q", nid) + O.chunk(c) for c, nid in shares)


def want_partial(kind: str, data: bytes):
    try:
        g, x, s, v = P.parse_partial(kind, data)
    except P.ParseError:
        return None
    if kind == "dsa":
        vals, bits = [g["p"], g["q"], g["g"]], 0
        built = g["p"].bit_length() in (1024, 2048) and g["p"] & 1 and g["q"] & 1 and 1 < g["q"] < 2 ** 256
    else:
        vals, bits = [g[k] for k in ("P", "N", "B", "Gx", "Gy")], g["BitSize"]
        built = all(g[k] == O.P256[k] for k in ("P", "N", "B", "Gx", "Gy", "BitSize"))
    return (struct.pack(">Q", x % 2 ** 64) + O.chunk(s) + O.chunk(O.bts(v)) + b"".join(O.chunk(O.bts(c)) for c in vals) +
            struct.pack(">I", bits) + bytes([1 if built else 0]))


@pytest.mark.parametrize("name", ["1024/160", "p256"])
def test_every_truncation(host, name):
    g = dict(kind="p256") if name == "p256" else O.golden_key()[0]
    kind = "p256" if name == "p256" else "dsa"
    rd = Round(g, 4, 0xD5F8)
    p0 = rd.phase0(0)
    proc = P.Proc(kind, rd.dgst, rd.t, rd.ids)
    for j in range(2 * rd.t):
        P.step(proc, 0, rd.phase0(j), rd.ids[j])
    req1 = proc.make_request()[1]
    p1 = rd.phase1(0, req1)
    p2 = O.phase3(g, rd.coords[0][0], rd.coords[0][1], 5, 7, *rd.kc[0])
    for c in range(len(p0) + 1):
        assert call(host.thdsa_joint_host, p0[:c], ctypes.c_uint64(c)) == want_joint(p0[:c]), c
    for ans in (p1, p2, p1 + b"trailing"):
        for c in range(len(ans) + 1):
            assert call(host.thdsa_partial_host, int(kind == "dsa"), ans[:c], ctypes.c_uint64(c)) == want_partial(kind, ans[:c]), c


def test_groups_and_odd_x(host):
    gk = O.golden_key()[0]
    cases = [("dsa", gk), ("dsa", dict(kind="dsa", p=(1 << 1535) + 1, q=gk["q"], g=2)), ("dsa", dict(kind="dsa", p=gk["p"], q=1, g=2)),
             ("dsa", dict(kind="dsa", p=gk["p"], q=(1 << 256) + 1, g=2)), ("dsa", dict(kind="dsa", p=gk["p"], q=gk["q"] + 1, g=2)),
             ("p256", dict(kind="p256"))]
    for kind, g in cases:
        for x in (0, 1, 2 ** 31 - 1, 2 ** 63, 2 ** 64 - 1):
            ans = struct.pack(">Q", x) + O.chunk(b"\x00\x05") + O.chunk(b"\x00" * 3 + b"\x07") + O.group_ser(g)
            assert call(host.thdsa_partial_host, int(kind == "dsa"), ans, ctypes.c_uint64(len(ans))) == want_partial(kind, ans)
    bad = O.group_ser(dict(kind="p256"))[:-4] + struct.pack(">I", 384)
    ans = struct.pack(">Q", 1) + O.chunk(b"") + O.chunk(b"") + bad
    assert call(host.thdsa_partial_host, 0, ans, ctypes.c_uint64(len(ans)))[-1] == 0


def test_requests(host):
    rng = random.Random(0xD5F9)
    proc = P.Proc("dsa", bytes(32), 3, [])
    ids, chunks = [], []
    for j in range(5):
        shares = [(bytes(rng.randrange(256) for _ in range(rng.randrange(0, 40))), rng.choice([7, 9, 2 ** 63 + 5, 11])) for _ in range(rng.randrange(0, 4))]
        P.step(proc, 0, P.joint_share_response(shares), j)
        ids += [nid for _, nid in shares]
        chunks += [c for c, _ in shares]
    proc.phase = 1
    want = proc.make_request()[1]
    off = [0]
    for c in chunks:
        off.append(off[-1] + len(c))
    arr = (ctypes.c_uint64 * max(1, len(ids)))(*ids)
    offs = (ctypes.c_uint64 * len(off))(*off)
    assert call(host.thdsa_request1_host, arr, b"".join(chunks), offs, ctypes.c_uint64(len(ids))) == want
    gk = O.golden_key()[0]
    for g in (gk, O.dsa_group(2048, 256), dict(kind="p256", **O.P256)):
        q = P.order(g)
        for dgst in (hashlib.sha256(b"m").digest(), bytes(32), b"\x00\x01" + bytes(30), hashlib.sha512(b"m").digest(), bytes(19), bytes(31)):
            for r in (0, 1, q - 1):
                qb, rb = O.bts(q), O.bts(r)
                try:
                    want = b"\x01" + O.chunk(O.bts(P.os2i(g, dgst))) + O.chunk(rb)
                except P.Panic:
                    want = None
                assert call(host.thdsa_request2_host, dgst, ctypes.c_uint64(len(dgst)), qb, ctypes.c_uint64(len(qb)), b"\x00" + rb,
                            ctypes.c_uint64(len(rb) + 1)) == want


def test_format_and_reduction(host):
    rng = random.Random(0xD5FA)
    for q in (O.golden_key()[0]["q"], P.order(dict(kind="p256", **O.P256)), 3 * 5 * 7 * 1000003):
        n = (q.bit_length() + 7) // 8
        for r, s in [(0, 0), (1, q - 1), (q - 1, 5), (1 << (8 * n), 1), (rng.randrange(q), rng.randrange(q))]:
            try:
                want = P.format_dsa(r, s, q)
            except P.Panic:
                want = None
            rb, sb = O.bts(r), s.to_bytes(n, "big")
            assert call(host.thdsa_format_host, rb, ctypes.c_uint64(len(rb)), sb, ctypes.c_uint64(len(sb)), ctypes.c_uint32(n)) == want
    gk = O.golden_key()[0]
    out = ctypes.create_string_buffer(256)
    for m in (gk["p"], gk["q"], P.order(dict(kind="p256", **O.P256)), 3):
        mb = O.bts(m)
        for v in (0, 1, m - 1, m, m + 1, 5 * m + 3, (1 << 2400) + 17, rng.getrandbits(700)):
            vb = b"\x00\x00" + O.bts(v)
            host.thdsa_be_mod_host(vb, ctypes.c_uint64(len(vb)), mb, ctypes.c_uint32(len(mb)), out)
            assert out.raw[:len(mb)] == (v % m).to_bytes(len(mb), "big"), (m, v)
