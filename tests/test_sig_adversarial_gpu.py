"""ECDSA P-256 (K1c), DSA (K1d) and ECDSA CalculateR on the device, over the adversarial vectors of
tests/golden/sig_adversarial.json, element by element against the oracle.  DSA includes composite subgroup orders,
where the device's s^-1 must be the true inverse (and absent when gcd(s, q) != 1), as Go's ModInverse has it."""
import hashlib
import json
import os
import random
import struct
from collections import defaultdict
from math import gcd

import numpy as np
import pytest

from oracle import pgp_oracle as pgp, sss_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
N, G = so.P256_N, so.P256_G
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vec():
    return json.load(open(os.path.join(HERE, "golden", "sig_adversarial.json")))


def _h(v):
    return int(v, 16)


def _rows32(vals):
    return np.frombuffer(b"".join(v.to_bytes(32, "big") for v in vals), np.uint8).reshape(-1, 32)


def _ecdsa_batch(engine, rows):
    keys = sorted({(row["qx"], row["qy"]) for row in rows})
    kix = {k: i for i, k in enumerate(keys)}
    pub = np.frombuffer(b"".join(bytes.fromhex(x) + bytes.fromhex(y) for x, y in keys), np.uint8).reshape(-1, 64)
    by_len = defaultdict(list)
    for i, row in enumerate(rows):
        by_len[len(row["digest"]) // 2].append(i)
    got = [None] * len(rows)
    for dlen, idx in sorted(by_len.items()):
        sel = [rows[i] for i in idx]
        st = engine.ecdsa_p256_verify_batch(pub, np.array([kix[(r["qx"], r["qy"])] for r in sel], np.uint32),
                                            _rows32([_h(r["r"]) for r in sel]), _rows32([_h(r["s"]) for r in sel]),
                                            np.frombuffer(b"".join(bytes.fromhex(r["digest"]) for r in sel), np.uint8).reshape(-1, dlen))
        for i, s in zip(idx, st.tolist()):
            got[i] = s
    return got


def _ecdsa_ref(row):
    if row["status"] == 3:
        return 3
    q = (_h(row["qx"]), _h(row["qy"]))
    return 0 if pgp.ecdsa_p256_verify(q, bytes.fromhex(row["digest"]), _h(row["r"]), _h(row["s"])) else 1


def test_ecdsa_vectors_mixed_keys(engine, vec):
    rows = vec["ecdsa"]
    ref = [_ecdsa_ref(r) for r in rows]
    assert ref == [r["status"] for r in rows]
    assert _ecdsa_batch(engine, rows) == ref


def test_ecdsa_every_vector_in_every_block_position(engine, vec):
    """128 x V items of 32-byte digests: block b holds vector (b + lane) mod V at each lane, so every vector runs in
    every lane of a 128-thread block next to vectors that take other branches."""
    rows = [r for r in vec["ecdsa"] if len(r["digest"]) == 64]
    V = len(rows)
    assert V >= 128
    order = [(b + lane) % V for b in range(V) for lane in range(128)]
    got = _ecdsa_batch(engine, [rows[i] for i in order])
    assert got == [rows[i]["status"] for i in order]


def _dsa_groups(vec):
    doms = {d["name"]: d for d in vec["dsa_domains"]}
    groups = defaultdict(list)
    for row in vec["dsa"]:
        D = doms[row["domain"]]
        groups[(row["domain"], row.get("g", D["g"]), row.get("y", D["y"]), len(row["digest"]) // 2, bool(row.get("raw")))].append(row)
    return doms, groups


def _dsa_raw(engine, p, q, g, y, rb, sb, dg):
    """bftq_dsa_verify_batch with g and y written as given in plen bytes (Engine.dsa_verify_batch reduces them mod p)."""
    from bftkv_b200 import _lib
    from bftkv_b200.engine import _ptr
    plen, qlen = (p.bit_length() + 7) // 8, (q.bit_length() + 7) // 8
    pb, qb, gb, yb = (np.frombuffer(v.to_bytes(n, "big"), np.uint8).copy() for v, n in ((p, plen), (q, qlen), (g, plen), (y, plen)))
    out = np.empty(rb.shape[0], np.uint8)
    _lib.check(engine._lib.bftq_dsa_verify_batch(engine._h, _ptr(pb), plen, _ptr(qb), qlen, _ptr(gb), _ptr(yb), _ptr(rb), _ptr(sb),
                                                 _ptr(dg), dg.shape[1], rb.shape[0], _ptr(out)))
    return out


def test_dsa_vectors(engine, vec):
    """Every DSA row, one launch per (domain, g, y, digest length), against dsa.Verify.  Composite q: honest signatures
    are accepted and the Fermat-crafted ones and non-invertible s refused."""
    doms, groups = _dsa_groups(vec)
    mismatches, n = [], 0
    for (name, gh, yh, dlen, raw), rows in sorted(groups.items()):
        D = doms[name]
        p, q, g, y = _h(D["p"]), _h(D["q"]), _h(gh), _h(yh)
        rb, sb = _rows32([_h(r["r"]) for r in rows]), _rows32([_h(r["s"]) for r in rows])
        dg = np.frombuffer(b"".join(bytes.fromhex(r["digest"]) for r in rows), np.uint8).reshape(-1, dlen)
        st = _dsa_raw(engine, p, q, g, y, rb, sb, dg) if raw else engine.dsa_verify_batch(p, q, g, y, rb, sb, dg)
        for row, got in zip(rows, st.tolist()):
            want = 0 if pgp.dsa_verify(p, q, g, y, bytes.fromhex(row["digest"]), _h(row["r"]), _h(row["s"])) else 1
            assert want == (0 if row["expect"] else 1)
            if got != want:
                mismatches.append((name, row["tag"], got, want))
            n += 1
    assert not mismatches, mismatches
    assert n == len(vec["dsa"])


def test_dsa_composite_q_in_both_directions(engine, vec):
    """The composite-q rows alone, one domain at a time: what Go accepts, the device accepts, and what it rejects
    (signatures steered so that w = s^(q-2) would pass), the device rejects."""
    comp = [d for d in vec["dsa_domains"] if len(d["factors"]) > 1]
    for D in comp:
        p, q, g, y = _h(D["p"]), _h(D["q"]), _h(D["g"]), _h(D["y"])
        rows = [r for r in vec["dsa"] if r["domain"] == D["name"] and r["tag"] in ("honest", "fermat_crafted", "s_not_invertible", "s_eq_factor")]
        assert sum(r["tag"] == "honest" for r in rows) == 3 and sum(r["tag"] == "fermat_crafted" for r in rows) == 3
        dlen = len(rows[0]["digest"]) // 2
        st = engine.dsa_verify_batch(p, q, g, y, _rows32([_h(r["r"]) for r in rows]), _rows32([_h(r["s"]) for r in rows]),
                                     np.frombuffer(b"".join(bytes.fromhex(r["digest"]) for r in rows), np.uint8).reshape(-1, dlen))
        got = {(r["tag"], i): s for i, (r, s) in enumerate(zip(rows, st.tolist()))}
        assert [s for (t, _), s in got.items() if t == "honest"] == [0, 0, 0], D["name"]
        assert [s for (t, _), s in got.items() if t == "fermat_crafted"] == [1, 1, 1], D["name"]
        assert all(s == 1 for (t, _), s in got.items() if t in ("s_not_invertible", "s_eq_factor")), D["name"]


def test_ecdsa_calculate_r_adversarial_sums(engine, vec):
    rows = vec["calc_r"]
    for k in sorted({len(r["x"]) for r in rows}):
        sel = [r for r in rows if len(r["x"]) == k]
        got, st = engine.ecdsa_p256_calculate_r_batch(np.array([r["x"] for r in sel], np.int32),
                                                      [[bytes.fromhex(p) for p in r["points"]] for r in sel],
                                                      [[_h(v) for v in r["v"]] for r in sel])
        assert st.tolist() == [r["status"] for r in sel]
        assert got == [_h(r["r"]) for r in sel]
    assert {r["tag"] for r in rows} >= {"sum_double", "sum_inf_end", "sum_inf_mid"}
    assert any(r["status"] == 3 for r in rows) and any(r["status"] == 0 for r in rows)


# ---- the packer: Signature.Verify over keys a peer writes itself ----------------------------------------------------
def _mpi(x):
    return struct.pack(">H", x.bit_length()) + x.to_bytes((x.bit_length() + 7) // 8, "big")


def _packet(tag, body):
    return bytes([0x80 | (tag << 2) | 1]) + struct.pack(">H", len(body)) + body


def _key_id(body):
    return int.from_bytes(hashlib.sha1(b"\x99" + struct.pack(">H", len(body)) + body).digest()[12:], "big")


P256_OID = bytes([0x2A, 0x86, 0x48, 0xCE, 0x3D, 0x03, 0x01, 0x07])


def _ecdsa_body(Q):
    pt = int.from_bytes(b"\x04" + Q[0].to_bytes(32, "big") + Q[1].to_bytes(32, "big"), "big")
    return bytes([4]) + struct.pack(">I", 0x5E000000) + bytes([19, len(P256_OID)]) + P256_OID + _mpi(pt)


def _dsa_body(p, q, g, y):
    return bytes([4]) + struct.pack(">I", 0x5E000000) + bytes([17]) + _mpi(p) + _mpi(q) + _mpi(g) + _mpi(y)


def _sig_packet(algo, kid, sig_type, prefix, sign, extra_hashed=b""):
    """v4 signature over `prefix`, SHA-256; sign(digest) -> (r, s)."""
    hashed = bytes([5, 2]) + struct.pack(">I", 0x5E000001) + extra_hashed
    head = bytes([4, sig_type, algo, 8]) + struct.pack(">H", len(hashed)) + hashed
    digest = hashlib.sha256(prefix + head + b"\x04\xff" + struct.pack(">I", len(head))).digest()
    r, s = sign(digest)
    unhashed = bytes([9, 16]) + struct.pack(">Q", kid)
    return _packet(2, head + struct.pack(">H", len(unhashed)) + unhashed + digest[:2] + _mpi(r) + _mpi(s))


def _key_block(body, algo, sign, uid):
    kid = _key_id(body)
    prefix = b"\x99" + struct.pack(">H", len(body)) + body + b"\xb4" + struct.pack(">I", len(uid)) + uid
    return _packet(6, body) + bytes([0xb4, len(uid)]) + uid + _sig_packet(algo, kid, 0x13, prefix, sign, bytes([2, 27, 0x03])), kid


def test_packer_peer_written_keys(engine, vec):
    """A P-256 key Q = -G (its table entry G + Q is infinity) and a composite-q DSA key, registered from key blocks
    written here; Signature.Verify over honest, tampered and steered signatures must equal crypto/pgp's verdicts.
    Registration parses the self-signature for its flags only; it verifies no signature on the device."""
    from bftkv_b200.crypto_gpu import Keyring, Signature
    rng = random.Random(0xBF7C51A2)
    c = N - 1

    def ec_sign(dg):
        e = int.from_bytes(dg, "big") % N
        k = rng.randrange(1, N)
        r = so.p256_mul(k, G)[0] % N
        return r, pow(k, -1, N) * (e + c * r) % N

    D = [d for d in vec["dsa_domains"] if d["name"] == "comp160_p1024"][0]
    p, q, g, y, x = (_h(D[k]) for k in ("p", "q", "g", "y", "x"))
    q1, q2 = (_h(f) for f in D["factors"])
    lam = (q1 - 1) * (q2 - 1) // gcd(q1 - 1, q2 - 1)

    def dsa_sign(dg, mode="honest"):
        z = int.from_bytes(dg[:20], "big")
        while True:
            k = rng.randrange(1, q)
            r = pow(g, k, p) % q
            t = (z + x * r) % q
            if r and gcd(k, q) == 1 and gcd(t, q) == 1:
                break
        if mode == "honest":
            return r, pow(k, -1, q) * t % q
        if mode == "fermat":
            return r, pow(k * pow(t, -1, q) % q, pow(q - 2, -1, lam), q)
        return r, q1 * rng.randrange(1, q2)                                  # s with no inverse mod q

    ec_block, ec_kid = _key_block(_ecdsa_body(so.p256_mul(c, G)), 19, ec_sign, b"peer-ec <ec@bftq.test>")
    ds_block, ds_kid = _key_block(_dsa_body(p, q, g, y), 17, dsa_sign, b"peer-dsa <dsa@bftq.test>")
    kr = Keyring(engine)
    assert kr.register(ec_block) == 1 and kr.register(ds_block) == 1
    ents = pgp.read_entities(ec_block) + pgp.read_entities(ds_block)
    tbs, sigs = [], []
    for i in range(6):
        t = b"tbs-%d" % i + bytes(rng.randrange(256) for _ in range(40))
        tbs += [t] * 6 + [t + b"x"] * 2
        sigs += [_sig_packet(19, ec_kid, 0, t, ec_sign),
                 _sig_packet(19, ec_kid, 0, t, lambda dg: (int.from_bytes(dg, "big") % N or 1, rng.randrange(1, N))),   # u1 = u2: result at infinity
                 _sig_packet(17, ds_kid, 0, t, dsa_sign),
                 _sig_packet(17, ds_kid, 0, t, lambda dg: dsa_sign(dg, "fermat")),
                 _sig_packet(17, ds_kid, 0, t, lambda dg: dsa_sign(dg, "noinv")),
                 _sig_packet(19, ec_kid, 0, t, ec_sign) + _sig_packet(17, ds_kid, 0, t, dsa_sign),
                 _sig_packet(19, ec_kid, 0, t, ec_sign),
                 _sig_packet(17, ds_kid, 0, t, dsa_sign)]
    got = Signature(kr).verify_batch(tbs, sigs)
    ref = [pgp.signature_verify(ents, t, s) for t, s in zip(tbs, sigs)]
    assert got == ref
    assert [r is None for r in ref[:8]] == [True, False, True, False, False, True, False, False]
    kr.close()
