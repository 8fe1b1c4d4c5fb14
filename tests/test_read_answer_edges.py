"""CPU half of the read-answer edge suite: the rows of read_answer_edges.py decode under the oracle to the status class
each was built for, every family reaches both routes and every status class it is meant to, the shared bftkv packet
parser agrees with the oracle on the bodies of families B and E, and the oracle agrees with GnuPG on answers GnuPG wrote."""
import ctypes as C
import hashlib
import json
import os
import subprocess
from collections import Counter

import pytest

import read_answer_edges as E
from oracle import packet_oracle, pgp_oracle as pgp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "read_answers_gnupg.json")

# per family: (least device-route rows, least host-route rows, status classes that must occur)
MINIMUM = {
    "A": (120, 10, {E.ST_OK, E.ST_INVALID, E.ST_OTHER, E.ST_UNVERIFIED}),
    "B": (200, 0, {E.ST_OK, E.ST_INVALID, E.ST_OTHER}),
    "C": (150, 60, {E.ST_OK, E.ST_INVALID, E.ST_OTHER, E.ST_NONCE}),
    "D": (10, 8, {E.ST_OK, E.ST_INVALID, E.ST_OTHER, E.ST_UNVERIFIED}),
    "E": (100, 6, {E.ST_OK, E.ST_OTHER, E.ST_UNVERIFIED}),
}


@pytest.fixture(scope="module")
def edges():
    return E.build()


def test_rows_decode_to_their_intended_class(edges):
    ents = pgp.read_entities(edges.keyring)
    bad = []
    for r in edges.rows:
        st, _, _ = pgp.read_response_status(ents, r["msg"], r["nonce"], r["pre"])
        if st != r["want"]:
            bad.append((r["family"], r["name"], st, r["want"]))
    assert not bad, bad


def test_every_family_reaches_both_routes_and_its_classes(edges):
    for fam, (dev, host, classes) in MINIMUM.items():
        rows = edges.family_rows(fam)
        routes = Counter(r["route"] for r in rows)
        print("family %s: %d device-route rows, %d host-route rows" % (fam, routes["device"], routes["host"]))
        assert routes["device"] >= dev and routes["host"] >= host, (fam, routes)
        assert {r["want"] for r in rows} >= classes, (fam, {r["want"] for r in rows})
    names = Counter(r["name"] for r in edges.rows)
    assert max(names.values()) == 1
    for nl in E.NONCE_LENS:
        rows = edges.family_rows("C", nl)
        assert rows and all(len(r["nonce"]) == nl for r in rows)
        assert Counter(r["route"] for r in rows)["device"] >= 12, nl
    # every good answer with a known signer has a tampered twin that is a bad signature
    names = {r["name"]: r for r in edges.rows}
    twins = [r for r in edges.rows if r["name"].endswith("/tampered")]
    assert len(twins) >= 150
    for t in twins:
        assert t["want"] == E.ST_INVALID and names[t["name"][:-len("/tampered")]]["want"] == E.ST_OK


def test_hashed_stream_covers_every_residue(edges):
    """Family B: body + hashed area + trailer takes every length mod 64, with the fast path and without."""
    for kind in ("fast", "no-fast"):
        res = {int(r["name"].split("/")[0][len("residue-"):]) for r in edges.family_rows("B") if r["name"].startswith("residue-") and r["name"].endswith("/" + kind)}
        assert res == set(range(64)), kind


def test_rows_are_deterministic(edges):
    again = E.Edges()
    assert len(again.rows) == len(edges.rows)
    for a, b in zip(again.rows, edges.rows):
        assert a == b, a["name"]
    digest = hashlib.sha256(b"".join(r["msg"] + r["nonce"] for r in edges.rows)).hexdigest()
    assert digest == hashlib.sha256(b"".join(r["msg"] + r["nonce"] for r in again.rows)).hexdigest()


# ---- bftkv_packet.hpp's host build against packet_oracle.parse -------------------------------------------------------
_SRC = r"""
#include "bftkv_packet.hpp"
extern "C" int pkt_parse(const unsigned char* p, unsigned long long n, unsigned long long* t, unsigned int* off, unsigned int* len) {
  const bftq::pkt::View v = bftq::pkt::parse(p, n);
  *t = v.t; *off = v.value_off; *len = v.value_len;
  return v.err ? 1 : 0;
}
"""


@pytest.fixture(scope="module")
def pkt_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("pkt")
    src, so = d / "pkt.cpp", d / "pkt.so"
    src.write_text(_SRC)
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "bftkv_b200", "csrc"), "-o", str(so), str(src)], check=True)
    return C.CDLL(str(so))


def _bodies(edges):
    """The literal bodies of families B and E, as the oracle de-chunks them, and every prefix of a few of them."""
    ents = pgp.read_entities(edges.keyring)
    out = []
    for r in edges.family_rows("B") + edges.family_rows("E"):
        res = pgp.message_verify(ents, r["msg"])
        if res.plain is not None:
            out.append(res.plain)
    small = sorted(set(out), key=len)[:6]
    return out + [b[:i] for b in small for i in range(len(b))]


def test_packet_parser_host_build_against_oracle(edges, pkt_lib):
    n_ok = n_err = 0
    for body in _bodies(edges):
        if not body:
            continue
        t, off, ln = C.c_ulonglong(), C.c_uint(), C.c_uint()
        err = pkt_lib.pkt_parse(body, len(body), C.byref(t), C.byref(off), C.byref(ln))
        try:
            _, value, want_t, _, _, _ = packet_oracle.parse(body)
        except (EOFError, ValueError):
            assert err == 1, body.hex()
            n_err += 1
            continue
        assert err == 0, body.hex()
        assert t.value == want_t and body[off.value:off.value + ln.value] == (value or b""), body.hex()
        n_ok += 1
    assert n_ok >= 200 and n_err >= 20, (n_ok, n_err)


# ---- GnuPG-written answers -------------------------------------------------------------------------------------------
def test_oracle_agrees_with_gnupg():
    g = json.load(open(GOLDEN))
    ents = pgp.read_entities(bytes.fromhex(g["keyring"]))
    kinds = Counter()
    for c in g["cases"]:
        st, t, v = pgp.read_response_status(ents, bytes.fromhex(c["msg"]), bytes.fromhex(c["nonce"]))
        good = st in (pgp.ST_OK, pgp.ST_UNVERIFIED)
        assert good == c["gpg_good"], c["name"]
        if good:
            assert st == pgp.ST_OK and (hashlib.sha256(v).hexdigest(), t) == (c["value_sha256"], c["t"]), c["name"]
        kinds[(c["framing"], c["gpg_good"])] += 1
    assert set(kinds) == {(f, g) for f in ("old-definite", "new-definite", "partial") for g in (True, False)}, kinds
