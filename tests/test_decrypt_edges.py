"""The decryption edge cases (tests/decrypt_edges.py) on the CPU: the fixture regenerates byte for byte, every row has the
property it exists for, and the reference decryption (pgp_encrypt_ref.message_decrypt) gives every row its intended code."""
import os
import subprocess
import sys

import pytest

import decrypt_edges as D

HERE = os.path.dirname(os.path.abspath(__file__))


def test_fixture_regenerates(tmp_path):
    out = tmp_path / "decrypt_edges.json"
    subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_decrypt_edges.py"), str(out)], check=True)
    assert out.read_bytes() == open(D.FIXTURE, "rb").read()


def test_fixture_keys():
    keys, coll = D.load_fixture()
    assert 0.49 < keys["L"]["p"] / keys["L"]["q"] < 0.52 and 1.9 < keys["H"]["p"] / keys["H"]["q"] < 2.05
    for k in keys.values():
        assert k["n"].bit_length() == 2048 and k["p"].bit_length() == k["q"].bit_length() == 1024
    import pgp_encrypt_ref as R
    for c in coll:
        pre = R.cfb_decrypt(c["wrong"], D.seipd_body(c["key"], b"", c["prefix"])[:18])
        assert len(c["key"]) == len(c["wrong"]) == D.KS[c["cipher"]] and c["key"] != c["wrong"]
        assert pre[14:16] == pre[16:18]


@pytest.fixture(scope="module")
def edges():
    return D.build()


def test_rows_have_their_property(edges):
    assert {r["family"] for r in edges.rows} == set("ABCD")
    for r in edges.rows:
        assert r["preds"], r["name"]
        for what, ok in r["preds"]:
            assert ok, (r["name"], what)
    for kn in ("5", "H"):
        assert sum(r["name"].startswith(kn + "/m-mod-p>=q/") for r in edges.rows) >= 8
    h = {r["name"].split("=")[-1] for r in edges.family("C") if "/H-mod-64=" in r["name"]}
    assert len(h) == 64


def test_oracle_gives_intended_codes(edges):
    got = edges.oracle([r["raw"] for r in edges.rows])
    code_of = {r["name"]: g[0] for r, g in zip(edges.rows, got)}
    for r, (code, plain, nonce) in zip(edges.rows, got):
        if r["want"] is None:                         # a wrong session key is taken: the code of its garbage, never 0
            assert code != 0 and (r["same_as"] is None or code == code_of[r["same_as"]]), r["name"]
        else:
            assert code == r["want"], (r["name"], code, r["want"])
        if code in (0, -6):
            assert (plain, nonce) == (r["plain"], r["nonce"]), r["name"]
    assert {0, -6, -8, -9, -11, -12} <= set(code_of.values())
