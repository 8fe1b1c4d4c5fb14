"""GPU half of the read-answer edge suite: every row of read_answer_edges.py through bftq_read_responses_batch (K0m, K1,
the host packer for the flagged shapes, K2m), compared element by element with pgp_oracle.read_response_status and
wotqs_oracle.read_decide: status class, timestamp and value bytes per answer; decision, winner and decided_at per
operation.  Each family also runs alone, so the engine's device / host item counters must equal the routes the rows
were built for; edge rows sit at every lane of a warp between rows of the other route; batch sizes straddle K0m's
128-thread blocks; a subprocess with tiny pieces and super-chunks must give identical outputs; GnuPG's answers take the
same path; and families A - C, sealed as encrypted transport messages, go through the encrypted read path, where K0m
reads the decrypted stream 18 bytes into the plain text and stops at the MDC."""
import json
import os
import pickle
import random
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import pgp_encrypt_ref as R
import read_answer_edges as E
from bftkv_b200 import workload as W
from oracle import pgp_oracle as pgp, wotqs_oracle as wq

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLIENT = 7                                     # the client's key for the encrypted path (not a signer)
OUTPUT_KEYS = ("status", "ts", "value_off", "value_len", "decision", "winner", "decided_at")


def status_class(st):
    return {0: pgp.ST_OK, 8: pgp.ST_UNVERIFIED, 7: pgp.ST_NONCE, 1: pgp.ST_INVALID, 2: pgp.ST_INVALID}.get(int(st), pgp.ST_OTHER)


@pytest.fixture(scope="module")
def edges():
    return E.build()


@pytest.fixture(scope="module")
def ents(edges):
    return pgp.read_entities(edges.keyring)


@pytest.fixture(scope="module")
def kr(engine, edges):
    from bftkv_b200.crypto_gpu import Keyring
    k = Keyring(engine)
    k.register(edges.keyring)
    yield k
    k.close()


class Oracle:
    """read_response_status (+ the plain text) per row, computed once per distinct (message, nonce, pre)."""

    def __init__(self, ents):
        self.ents, self.memo = ents, {}

    def __call__(self, msg, nonce, pre):
        key = (msg, nonce, pre)
        if key not in self.memo:
            st, t, v = pgp.read_response_status(self.ents, msg, nonce, pre)
            plain = pgp.message_verify(self.ents, msg).plain if st in (pgp.ST_OK, pgp.ST_UNVERIFIED) else None
            self.memo[key] = (st, t, v, plain)
        return self.memo[key]


@pytest.fixture(scope="module")
def oracle(ents):
    return Oracle(ents)


def small_quorum(edges):
    """Families A - D: operations of four responders over a clique of the four signers (f = 1, threshold 2)."""
    ids = edges.peer_ids[:E.N_SIGNERS]
    return [(1, 4, 2, 3, ids)], wq.Quorum([wq.QC([wq.Node(i) for i in ids], 1, 4, 2, 3)])


def e_quorum(edges):
    """Family E: one clique of all 32 responders, f = 10, threshold 11."""
    ids = edges.peer_ids[:E.N_PEERS]
    return [(10, 31, 11, 21, ids)], wq.Quorum([wq.QC([wq.Node(i) for i in ids], 10, 31, 11, 21)])


def in_fours(edges, rows):
    """-> (op_off, peer ids): consecutive rows in operations of four, responders 0 .. 3 in turn."""
    n = len(rows)
    op_off = np.array(list(range(0, n, 4)) + [n], np.uint32)
    return op_off, np.array([edges.peer_ids[i % 4] for i in range(n)], np.uint64)


def e_layout(edges):
    rows = edges.family_rows("E")
    ops = max(r["op"] for r in rows) + 1
    op_off = np.searchsorted(np.array([r["op"] for r in rows]), np.arange(ops + 1)).astype(np.uint32)
    assert all(rows[i]["op"] <= rows[i + 1]["op"] for i in range(len(rows) - 1))
    return rows, op_off, np.array([edges.peer_ids[r["peer"]] for r in rows], np.uint64)


def call(kr, rows, op_off, peers, qcs, encrypted=None):
    from bftkv_b200.crypto_gpu import read_encrypted_responses_batch, read_responses_batch
    nonces = np.frombuffer(b"".join(r["nonce"] for r in rows), np.uint8).reshape(len(rows), -1) if rows else np.zeros((0, 8), np.uint8)
    pre = np.array([r["pre"] for r in rows], np.uint8)
    if encrypted is None:
        return read_responses_batch(kr, qcs, op_off, peers, [r["msg"] for r in rows], nonces, pre_status=pre)
    return read_encrypted_responses_batch(kr, qcs, op_off, peers, encrypted, nonces, pre_status=pre)


def check(rows, op_off, peers, quorum, got, want):
    """want[p] = (class, t, value, plain) per row; compares every answer and every operation."""
    for p, r in enumerate(rows):
        st, t, v, plain = want[p]
        assert status_class(got["status"][p]) == st, (p, r["family"], r["name"], int(got["status"][p]), st)
        if st in (pgp.ST_OK, pgp.ST_UNVERIFIED):
            vo, vl = int(got["value_off"][p]), int(got["value_len"][p])
            assert int(got["ts"][p]) == t and plain[vo:vo + vl] == v, (p, r["name"], int(got["ts"][p]), t, vo, vl)
            if "plain" in got:
                assert got["plain"][p] == plain, (p, r["name"])
    decs = Counter()
    for op in range(len(op_off) - 1):
        resp = []
        for p in range(op_off[op], op_off[op + 1]):
            st, t, v, _ = want[p]
            good = st in (pgp.ST_OK, pgp.ST_UNVERIFIED)
            resp.append((wq.Node(int(peers[p])), not good, t, v))
        kind, at, value, t = wq.read_decide(resp, quorum)
        assert (int(got["decision"][op]), int(got["decided_at"][op])) == (kind, at), (op, [rows[p]["name"] for p in range(op_off[op], op_off[op + 1])], kind, at)
        if kind == wq.READ_VALUE:
            wi = int(got["winner"][op])
            assert resp[wi][2] == t and resp[wi][3] == value and not resp[wi][1], op
            assert not any(not r2[1] and r2[2] == t and r2[3] == value for r2 in resp[:wi]), op
        else:
            assert got["winner"][op] == 0xFFFFFFFF, op
        decs[kind] += 1
    return decs


def run_and_check(engine, kr, oracle, rows, op_off, peers, qcs, quorum):
    s0 = engine.stats()
    got = call(kr, rows, op_off, peers, qcs)
    s1 = engine.stats()
    want = [oracle(r["msg"], r["nonce"], r["pre"]) for r in rows]
    decs = check(rows, op_off, peers, quorum, got, want)
    return got, decs, (s1["msg_gpu_items"] - s0["msg_gpu_items"], s1["msg_host_items"] - s0["msg_host_items"])


# ---- each family in a call of its own: outputs against the oracle, counters against the routes -----------------------
@pytest.mark.parametrize("family", ["A", "B", "C", "D", "E"])
def test_family_alone(engine, kr, oracle, edges, family):
    calls = []
    if family == "E":
        rows, op_off, peers = e_layout(edges)
        calls.append((rows, op_off, peers) + e_quorum(edges))
    elif family == "C":
        for nl in E.NONCE_LENS:
            rows = edges.family_rows("C", nl)
            calls.append((rows,) + in_fours(edges, rows) + small_quorum(edges))
    else:
        rows = edges.family_rows(family)
        calls.append((rows,) + in_fours(edges, rows) + small_quorum(edges))
    total, decs = Counter(), Counter()
    for rows, op_off, peers, qcs, quorum in calls:
        got, d, (on_gpu, on_host) = run_and_check(engine, kr, oracle, rows, op_off, peers, qcs, quorum)
        routes = Counter(r["route"] for r in rows)
        assert (on_gpu, on_host) == (routes["device"], routes["host"]), (family, on_gpu, on_host, routes)
        total += routes
        decs += d
        if family == "A":
            # the body of the alignment rows starts at every address mod 4
            blob_off = np.concatenate([[0], np.cumsum([len(r["msg"]) for r in rows])])
            al = {(int(blob_off[p]) + r["msg"].find(oracle(r["msg"], r["nonce"], r["pre"])[3][:64])) % 4 for p, r in enumerate(rows)
                  if r["name"].startswith("align/") and not r["name"].endswith("/tampered")}
            assert al == {0, 1, 2, 3}, al
    print("family %s: %d device-route rows, %d host-route rows; decisions %s" % (family, total["device"], total["host"], dict(decs)))
    assert total["device"] > 0
    if family == "E":
        assert set(decs) == {wq.READ_VALUE, wq.READ_EXHAUSTED}, decs


def test_full_warp_op_decides_at_its_last_responder(engine, kr, oracle, edges):
    """Family E's first operation: 32 responders, three values equal but for their last byte, decided by the 32nd."""
    rows, op_off, peers = e_layout(edges)
    got = call(kr, rows, op_off, peers, e_quorum(edges)[0])
    assert int(op_off[1]) == 32 and int(op_off[2]) == 32                 # and the next operation has no responder
    assert (int(got["decision"][0]), int(got["decided_at"][0]), int(got["winner"][0])) == (wq.READ_VALUE, 32, 0)
    assert (int(got["decision"][1]), int(got["decided_at"][1]), int(got["winner"][1])) == (wq.READ_EXHAUSTED, 0, 0xFFFFFFFF)


# ---- every edge row at every lane, between rows of the other route ----------------------------------------------------
def lane_sweep(edges):
    """Device-route and host-route rows of families A - D (nonce length 8) alternating, the sequence made odd in length
    and repeated 32 times: row j of the sequence lands on lane (k * len + j) mod 32 in round k, i.e. on every lane."""
    base = [r for f in "ABCD" for r in edges.family_rows(f, 8)]
    dev, host = [r for r in base if r["route"] == "device"], [r for r in base if r["route"] == "host"]
    seq = []
    for i, r in enumerate(dev):
        seq += [r, host[i % len(host)]]
    if len(seq) % 2 == 0:
        seq.append(dev[0])
    return seq * 32


@pytest.fixture(scope="module")
def sweep(edges):
    return lane_sweep(edges)


@pytest.mark.parametrize("n", [1, 127, 128, 129, 4097, None])
def test_every_lane_and_batch_size(engine, kr, oracle, edges, sweep, n):
    rows = sweep if n is None else sweep[:n]
    op_off, peers = in_fours(edges, rows)
    qcs, quorum = small_quorum(edges)
    got, decs, (on_gpu, on_host) = run_and_check(engine, kr, oracle, rows, op_off, peers, qcs, quorum)
    routes = Counter(r["route"] for r in rows)
    assert (on_gpu, on_host) == (routes["device"], routes["host"])
    if n is None:
        assert set(decs) == {wq.READ_VALUE, wq.READ_REJECTED, wq.READ_EXHAUSTED}, decs


def _dump(rows_path, out_path):
    """Subprocess body: the same lane-sweep call under the caller's environment, outputs to out_path."""
    from bftkv_b200 import Engine
    from bftkv_b200.crypto_gpu import Keyring
    with open(rows_path, "rb") as f:
        keyring, rows, op_off, peers, qcs = pickle.load(f)
    eng = Engine(0)
    k = Keyring(eng)
    k.register(keyring)
    got = call(k, rows, op_off, peers, qcs)
    np.savez(out_path, **{key: got[key] for key in OUTPUT_KEYS})
    k.close()
    eng.close()


def test_small_pieces_and_super_chunks_agree(kr, edges, sweep, tmp_path):
    rows = sweep[:4097]
    op_off, peers = in_fours(edges, rows)
    qcs = small_quorum(edges)[0]
    got = call(kr, rows, op_off, peers, qcs)
    rows_path, out_path = str(tmp_path / "rows.pkl"), str(tmp_path / "small.npz")
    with open(rows_path, "wb") as f:
        pickle.dump((edges.keyring, rows, op_off, peers, qcs), f)
    env = dict(os.environ, BFTQ_READ_PIECE="37", BFTQ_READ_SUPER="500")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_read_answer_edges_gpu as T; T._dump(%r, %r)" % (ROOT, os.path.join(ROOT, "tests"), rows_path, out_path)
    subprocess.run([sys.executable, "-c", code], env=env, check=True, cwd=ROOT)
    small = np.load(out_path)
    for key in OUTPUT_KEYS:
        assert np.array_equal(small[key], got[key]), key


# ---- GnuPG's answers ---------------------------------------------------------------------------------------------------
def test_gnupg_answers(engine):
    from bftkv_b200.crypto_gpu import Keyring
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "read_answers_gnupg.json")))
    ring = bytes.fromhex(g["keyring"])
    ents = pgp.read_entities(ring)
    k = Keyring(engine)
    k.register(ring)
    rows = [dict(family="G", name=c["name"], msg=bytes.fromhex(c["msg"]), nonce=bytes.fromhex(c["nonce"]), pre=0) for c in g["cases"]]
    ids = [ents[0].primary_key.key_id, 11, 12, 13]
    qcs = [(1, 4, 2, 3, ids)]
    quorum = wq.Quorum([wq.QC([wq.Node(i) for i in ids], 1, 4, 2, 3)])
    op_off = np.array(list(range(0, len(rows), 4)) + [len(rows)], np.uint32)
    peers = np.array([ids[i % 4] for i in range(len(rows))], np.uint64)
    got = call(k, rows, op_off, peers, qcs)
    o = Oracle(ents)
    want = [o(r["msg"], r["nonce"], 0) for r in rows]
    check(rows, op_off, peers, quorum, got, want)
    for c, w in zip(g["cases"], want):
        assert (w[0] == pgp.ST_OK) == c["gpg_good"], c["name"]
    k.close()


# ---- the encrypted path: families A - C sealed to the client ----------------------------------------------------------
@pytest.mark.parametrize("nonce_len", [None] + list(E.NONCE_LENS))
def test_encrypted_path(engine, edges, nonce_len):
    from bftkv_b200.crypto_gpu import Keyring
    if nonce_len is None:
        rows = [r for f in "AB" for r in edges.family_rows(f)]
    else:
        rows = edges.family_rows("C", nonce_len)
    rows = [r for r in rows if r["msg"] and not r["pre"]]
    keys = edges.keys
    cli_block, cli_id = W.pgp_public_key_block(keys[CLIENT], W._private_key(keys[CLIENT]), b"client <c@bftq.test>")
    k = Keyring(engine)
    k.register(cli_block, priv=True)
    k.register(edges.keyring)
    assert k.register_private(W.secret_key_packet(keys[CLIENT])) == 1
    rng = random.Random(0xBF7C00E1 + (nonce_len or 0))
    raws = [R.encrypt(rng, keys[CLIENT], cli_id, r["msg"]) for r in rows]
    op_off, peers = in_fours(edges, rows)
    qcs, quorum = small_quorum(edges)
    got = call(k, rows, op_off, peers, qcs, encrypted=raws)
    ring = pgp.read_entities(cli_block + edges.keyring)
    pub_ids = {e.primary_key.key_id for e in ring} | {s.public_key.key_id for e in ring for s in e.subkeys}
    o = Oracle(ring)
    want = []
    for r, raw in zip(rows, raws):
        code, plain, _ = R.message_decrypt(raw, {cli_id: keys[CLIENT]}, {cli_id}, pub_ids, ring)
        if code == 0:
            want.append(o(r["msg"], r["nonce"], 0))
        else:
            want.append((pgp.ST_INVALID if code == -6 else pgp.ST_OTHER, 0, b"", None))
        assert want[-1][0] == r["want"], r["name"]
    check(rows, op_off, peers, quorum, got, want)
    k.close()
