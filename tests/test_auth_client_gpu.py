"""GPU suite: the client half of crypto/auth on the device (K10) against the oracle client, byte for byte given the same
a and a' values: full rounds against oracle servers and K9 device servers, arrival orders, repeated and unknown peers,
edge values of every public input, every phase-2 failure, the argument errors, mixed and concurrent calls, and handles
that outlive their engine."""
import random
import struct
import threading

import pytest

import auth_oracle as A
from auth_client_oracle import Insufficient, NoAuthData, OracleClient, wire_map
from bftkv_b200 import Engine, _lib
from bftkv_b200.crypto_gpu import AuthClient, ErrInsufficientNumberOfSecrets, ErrNoAuthenticationData

pytestmark = pytest.mark.gpu
INIT, KEY = -1, -2
INVALID_ARG, MALFORMED, NO_AUTH_DATA, DECRYPTION_FAILED, INSUFFICIENT = -3, -8, -17, -18, -19


def a_bytes(v: int) -> bytes:
    return v.to_bytes(256, "big")


class Session:
    """A device session and the oracle client it must match."""

    def __init__(self, engine, password, n, k):
        self.h = engine.auth_client_create(password, n, k)
        self.o = OracleClient(password, n, k)
        self.seen = []

    def rand(self, op, pid, rng):
        if op == INIT:
            return a_bytes(rng.randrange(1, A.Q))
        if op == 0:
            m = len(self.seen) + (pid not in self.seen)
            if pid not in self.seen:
                self.seen.append(pid)
            if m >= self.o.k:
                return b"".join(a_bytes(rng.randrange(A.Q)) for _ in range(m))
        return b""

    def oracle(self, op, data, pid, rand):
        """(err, has_map, out) of one item on the oracle."""
        try:
            if op == INIT:
                return 0, 0, self.o.initiate(int.from_bytes(rand, "big"))
            if op == KEY:
                return 0, 0, self.o.cipher_key()
            if op in (0, 1, 2):
                a2s = [int.from_bytes(rand[256 * j:256 * j + 256], "big") for j in range(len(rand) // 256)]
                m = self.o.yi(data, pid, a2s) if op == 0 else self.o.bi(data, pid) if op == 1 else self.o.zi(data, pid)
                return (0, 1, wire_map(m)) if m is not None else (0, 0, b"")
            return 0, 0, b""
        except ValueError:
            return MALFORMED, 0, b""
        except NoAuthData:
            return NO_AUTH_DATA, 0, b""
        except A.DecryptionFailed:
            return DECRYPTION_FAILED, 0, b""
        except Insufficient:
            return INSUFFICIENT, 0, b""


def run(engine, items, check=True):
    """items: (session, op, data, peer id, rand).  One device call; every item checked against its oracle in order."""
    tab = list({id(s): s for s, *_ in items}.values())
    pos = {id(s): j for j, s in enumerate(tab)}
    err, has, outs = engine.auth_client_process_batch([s.h for s in tab], [pos[id(s)] for s, *_ in items], [it[1] for it in items],
                                                      [it[3] for it in items], [it[2] for it in items], [it[4] for it in items])
    got = list(zip([int(e) for e in err], [int(h) for h in has], outs))
    if check:
        for (s, op, data, pid, rand), g in zip(items, got):
            assert g == s.oracle(op, data, pid, rand), (op, pid)
    return got


@pytest.fixture
def sessions(engine):
    made = []

    def make(password, n, k):
        s = Session(engine, password, n, k)
        made.append(s)
        return s
    yield make
    for s in made:
        engine.auth_client_destroy(s.h)


def setup(rng, password, n, k, proof=b"proof"):
    params = A.generate_params(password, n, k, rng)
    return [A.Server(p, proof, reference_zero_key_quirk=False) for p in params]


def login(engine, s, servers, rng, ids=None, shuffle=True):
    """A whole round one item per call: X to every server, phase-0 answers until the set completes, then phases 1 and 2
    over the completing map.  Returns the cipher key."""
    ids = list(range(len(servers))) if ids is None else ids
    X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])[0][2]
    order = list(ids)
    if shuffle:
        rng.shuffle(order)
    xis = None
    for i in order:
        yi = servers[i].make_yi(X)
        e, hm, out = run(engine, [(s, 0, yi, i, s.rand(0, i, rng))])[0]
        if hm:
            xis = AuthClient._parse_map(out)
            break
    assert xis is not None
    nis = None
    for i in xis:
        bi = servers[i].make_bi(xis[i], rng.randrange(A.P))
        e, hm, out = run(engine, [(s, 1, bi, i, b"")])[0]
        if hm:
            nis = AuthClient._parse_map(out)
    assert nis is not None
    pis = None
    for i in nis:
        zi = servers[i].make_zi(nis[i], rng.randbytes(12))
        e, hm, out = run(engine, [(s, 2, zi, i, b"")])[0]
        if hm:
            pis = AuthClient._parse_map(out)
    assert pis is not None and all(p == servers[i].proof for i, p in pis.items())
    e, _, key = run(engine, [(s, KEY, b"", 0, b"")])[0]
    assert e == 0
    return key


@pytest.mark.parametrize("n,k", [(4, 3), (10, 7), (31, 21)])
def test_full_rounds_against_oracle_servers(engine, sessions, n, k):
    rng = random.Random(0xC1 + n)
    pw = rng.randbytes(8)
    servers = setup(A.Rng(n), pw, n, k)
    s = sessions(pw, n, k)
    key = login(engine, s, servers, rng)
    assert key == s.o.get_cipher_key()
    # the password-derived key is the same whichever k servers answered
    s2 = sessions(pw, n, k)
    assert login(engine, s2, servers, rng) == key


def test_full_round_against_device_servers(engine, sessions):
    """K9 servers on the device answer K10's requests; the key matches the oracle client run on the oracle servers."""
    rng = random.Random(0xD5)
    pw, n, k = b"correct horse", 10, 7
    params = A.generate_params(pw, n, k, A.Rng(0xD5))
    srv = [engine.auth_server_create(p, b"the proof %d" % i) for i, p in enumerate(params)]
    try:
        s = sessions(pw, n, k)
        X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])[0][2]
        _, yis = engine.auth_server_respond_batch(srv, list(range(n)), [0] * n, [X] * n, [b""] * n)
        got = run(engine, [(s, 0, yis[i], i, s.rand(0, i, rng)) for i in range(n)])
        xis = AuthClient._parse_map(got[-1][2])
        ids = list(xis)
        _, bis = engine.auth_server_respond_batch(srv, ids, [1] * len(ids), [xis[i] for i in ids], [a_bytes(rng.randrange(A.P)) for _ in ids])
        got = run(engine, [(s, 1, b, i, b"") for i, b in zip(ids, bis)])
        nis = AuthClient._parse_map(got[-1][2])
        err, zis = engine.auth_server_respond_batch(srv, ids, [2] * len(ids), [nis[i] for i in ids], [rng.randbytes(12) for _ in ids])
        assert not any(err)
        got = run(engine, [(s, 2, z, i, b"") for i, z in zip(ids, zis)])
        assert AuthClient._parse_map(got[-1][2]) == {i: b"the proof %d" % i for i in ids}
        key = run(engine, [(s, KEY, b"", 0, b"")])[0][2]
        # the same password against the same parameters on the oracle side gives the same key
        o = OracleClient(pw, n, k)
        o.a = int.from_bytes(a_bytes(rng.randrange(1, A.Q)), "big")
        o.initiate(o.a)
        for i in range(k):
            o.yi(A.Server(params[i], b"").make_yi(A.i2b(pow(A.PI(pw), o.a, A.P))), i, [1] * k)
        assert key == o.get_cipher_key()
    finally:
        for h in srv:
            engine.auth_server_destroy(h)


def test_arrival_orders_repeats_and_unknown_peers(engine, sessions):
    rng = random.Random(0xA7)
    pw, n, k = b"pw", 6, 3
    servers = setup(A.Rng(7), pw, n, k)
    s = sessions(pw, n, k)
    X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])[0][2]
    ys = [srv.make_yi(X) for srv in servers]
    # a repeated phase-0 peer before and after the k-th, answers after the k-th (each recomputes gs and a fresh Xi map)
    run(engine, [(s, 0, ys[4], 4, s.rand(0, 4, rng)), (s, 0, ys[4], 4, s.rand(0, 4, rng)), (s, 0, ys[1], 1, s.rand(0, 1, rng))])
    run(engine, [(s, 0, ys[2], 2, s.rand(0, 2, rng)), (s, 0, ys[2], 2, s.rand(0, 2, rng)), (s, 0, ys[0], 0, s.rand(0, 0, rng))])
    xis = s.o.secrets
    ids = list(xis)
    # phase 1: an unknown peer, a repeated answer (counted again: the map holds an empty Ni for a silent peer)
    bis = {i: servers[i].make_bi(xis[i]["Xi"], rng.randrange(A.P)) for i in ids}
    run(engine, [(s, 1, bis[ids[0]], 5, b""), (s, 1, bis[ids[0]], ids[0], b""), (s, 1, bis[ids[0]], ids[0], b"")])
    run(engine, [(s, 1, bis[i], i, b"") for i in ids[1:]])
    nis = {i: t.get("Ni", b"") for i, t in s.o.secrets.items()}
    # phase 2: unknown peer, a peer with keys, the silent-but-listed peers fail closed, repeats count
    zis = {i: servers[i].make_zi(nis[i], rng.randbytes(12)) for i in ids if nis[i] and servers[i].mac is not None}
    items = [(s, 2, next(iter(zis.values())), 5, b"")]
    for i, z in zis.items():
        items += [(s, 2, z, i, b""), (s, 2, z, i, b"")]
    run(engine, items)
    run(engine, [(s, KEY, b"", 0, b"")])
    # a second Initiate keeps the secrets, gs and the counter; a new a changes the key
    run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])
    run(engine, [(s, KEY, b"", 0, b"")])
    run(engine, [(s, 0, ys[3], 3, s.rand(0, 3, rng))])
    run(engine, [(s, KEY, b"", 0, b"")])


def _yi(x, y, salt):
    return struct.pack(">i", x) + A.chunk(y) + A.chunk(salt)


def test_edge_public_values(engine, sessions):
    rng = random.Random(0xED)
    pw, n, k = b"edge", 8, 3
    pb = A.P.to_bytes(256, "big")
    edges = [b"", b"\x01", (A.P - 1).to_bytes(256, "big"), pb, (A.P + 5).to_bytes(256, "big"), (1 << 2048).to_bytes(257, "big"),
             rng.randbytes(300), b"\x00\x00" + rng.randbytes(100), b"\xff" * 256]
    for j in range(0, len(edges), 2):
        s = sessions(pw, n, k)
        run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])
        ys = [edges[j], edges[(j + 1) % len(edges)], rng.randbytes(256), edges[(j + 3) % len(edges)]]
        xs = [-5, 0, 7, 7]
        salts = [b"", rng.randbytes(64), rng.randbytes(65), rng.randbytes(200)]
        run(engine, [(s, 0, _yi(x, y, sl), i, s.rand(0, i, rng)) for i, (x, y, sl) in enumerate(zip(xs, ys, salts))])
        ids = list(s.o.secrets)
        run(engine, [(s, 1, A.chunk(edges[(j + t) % len(edges)]), i, b"") for t, i in enumerate(ids)])
        run(engine, [(s, KEY, b"", 0, b"")])
        # phase 2 with the keys phase 1 derived: seal with the oracle's own keys
        items = []
        for i in ids:
            t = s.o.secrets[i]
            nonce = rng.randbytes(12)
            items.append((s, 2, A.serialize_zi(A.gcm_seal(t["ke"], nonce, rng.randbytes(i * 7), t["Ni"]), nonce), i, b""))
        run(engine, items)


@pytest.mark.parametrize("pwlen", [0, 55, 56, 64, 1500])
def test_passwords_and_extreme_randomness(engine, sessions, pwlen):
    rng = random.Random(pwlen)
    pw = rng.randbytes(pwlen)
    servers = setup(A.Rng(pwlen), pw, 4, 3)
    for a, a2 in [(1, 0), (A.Q - 1, A.Q - 1), (rng.randrange(A.Q), 1)]:
        s = sessions(pw, 4, 3)
        X = run(engine, [(s, INIT, b"", 0, a_bytes(a))])[0][2]
        run(engine, [(s, 0, servers[i].make_yi(X), i, a_bytes(a2) * 3) for i in range(3)])
        ids = list(s.o.secrets)
        run(engine, [(s, 1, servers[i].make_bi(s.o.secrets[i]["Xi"], rng.randrange(A.P)), i, b"") for i in ids])
        run(engine, [(s, 2, servers[i].make_zi(s.o.secrets[i]["Ni"], rng.randbytes(12)), i, b"") for i in ids])
        key = run(engine, [(s, KEY, b"", 0, b"")])[0][2]
        assert len(key) == 32


def test_phase2_failures(engine, sessions):
    rng = random.Random(0x22)
    pw = b"tamper"
    for proof in (b"", rng.randbytes(100)):
        servers = setup(A.Rng(0x22), pw, 5, 3, proof)
        s = sessions(pw, 5, 3)
        X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])[0][2]
        run(engine, [(s, 0, servers[i].make_yi(X), i, s.rand(0, i, rng)) for i in range(4)])
        ids = list(s.o.secrets)
        run(engine, [(s, 1, servers[i].make_bi(s.o.secrets[i]["Xi"], rng.randrange(A.P)), i, b"") for i in ids[:3]])
        nonce = rng.randbytes(12)
        good = {i: servers[i].make_zi(s.o.secrets[i]["Ni"], nonce) for i in ids[:3]}
        zi, nc = A.parse_zi(good[ids[0]])
        flip = lambda b, at: b[:at] + bytes([b[at] ^ 1]) + b[at + 1:]
        bad = [A.serialize_zi(flip(zi, len(zi) - 1), nc),                    # tag
               A.serialize_zi(flip(zi, 0), nc) if len(zi) > 16 else A.serialize_zi(zi, flip(nc, 0)),
               A.serialize_zi(zi, flip(nc, 3)),                             # nonce
               A.serialize_zi(zi[:15], nc),                                 # shorter than a tag
               A.serialize_zi(zi, nc + b"\0"),                              # a 13-byte nonce
               A.serialize_zi(zi, nc[:8]),
               A.chunk(zi),                                                 # framing
               b"\0" * 3]
        items = [(s, 2, b, ids[0], b"") for b in bad]
        items.append((s, 2, good[ids[1]], ids[3], b""))                     # a peer with no phase-1 keys
        items += [(s, 2, good[i], i, b"") for i in ids[:3]]
        # a proof sealed under the right key over another Ni (aad) does not open
        t = s.o.secrets[ids[2]]
        items.append((s, 2, A.serialize_zi(A.gcm_seal(t["ke"], nonce, proof, b"\x55" * 32), nonce), ids[2], b""))
        run(engine, items)


def test_cipher_key_before_gs_and_phase_errors(engine, sessions):
    rng = random.Random(0x33)
    s = sessions(b"x", 4, 3)
    run(engine, [(s, KEY, b"", 0, b"")])
    run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])
    run(engine, [(s, KEY, b"", 0, b"")])
    run(engine, [(s, 1, A.chunk(b"\1"), 3, b""), (s, 1, b"\0\0", 3, b"")])
    run(engine, [(s, 2, A.serialize_zi(b"z" * 20, b"n" * 12), 3, b""), (s, 2, b"", 3, b"")])
    run(engine, [(s, 0, b"\0\0\0", 1, b""), (s, 0, _yi(1, b"\2", b"s"), 1, b"")])
    run(engine, [(s, 7, b"", 1, b""), (s, 7, b"", 2, b"")])


def test_invalid_arg_changes_nothing(engine, sessions):
    """Every refused call is followed by a checked step of the same session: a refused call that had written a, gs, a'
    or the public state would show up as a difference from the oracle there."""
    import ctypes as C
    import numpy as np
    rng = random.Random(0x44)
    pw, n, k = b"inv", 4, 2
    servers = setup(A.Rng(0x44), pw, n, k)
    s, t = sessions(pw, n, k), sessions(pw, n, k)
    h = [s.h, t.h]

    def bad(idx, ops, pids, datas, rands):
        with pytest.raises(_lib.BftqError) as ei:
            engine.auth_client_process_batch(h, idx, ops, pids, datas, rands)
        assert ei.value.code == INVALID_ARG

    def key(sess):                                          # read-only: the key depends on a, a^-1 and gs
        run(engine, [(sess, KEY, b"", 0, b"")])

    X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])[0][2]
    ys = [srv.make_yi(X) for srv in servers]
    run(engine, [(s, 0, ys[0], 0, s.rand(0, 0, rng))])
    bad([0], [1], [0], [A.chunk(b"\1")], [b""])             # phase 1 on a secret with no a'
    bad([0], [0], [1], [ys[1]], [a_bytes(1)])               # 2 secrets need 2 a' values
    run(engine, [(s, 0, ys[1], 1, s.rand(0, 1, rng))])       # continues: completes with the a of the first INITIATE
    key(s)
    refused = [([0, 0], [INIT, INIT], [0, 0], [b"", b""], [a_bytes(5), a_bytes(6)]),
               ([0, 0], [INIT, 0], [0, 2], [b"", ys[2]], [a_bytes(5), a_bytes(7) * 3]),
               ([0], [INIT], [0], [b""], [b"\1" * 255]),
               ([0], [INIT], [0], [b""], [a_bytes(0)]),
               ([0], [INIT], [0], [b""], [a_bytes(A.Q)]),
               ([0], [INIT], [0], [b""], [a_bytes(2 * A.Q)]),
               ([0, 0], [KEY, KEY], [0, 0], [b"", b""], [b"", b""]),
               ([0], [0], [2], [ys[2]], [a_bytes(1) * 2]),                                  # 3 secrets need 3 a' values
               ([0, 0, 0], [0, 0, 0], [2, 3, 9], [ys[2], ys[3], ys[0]], [a_bytes(1) * 5] * 3)]   # n + 1 distinct peers
    for call in refused:
        bad(*call)
        key(s)
    # out_cap below the need: refused, and *out_need says how much the call takes (peer 2 completes with 3 secrets)
    tab = (C.c_void_p * 1)(s.h.value)
    need = C.c_uint64(0)
    arrs = [np.zeros(1, np.uint32), np.zeros(1, np.int32), np.array([2], np.uint64), np.frombuffer(ys[2], np.uint8).copy(),
            np.array([0, len(ys[2])], np.uint64), np.frombuffer(a_bytes(3) * 3, np.uint8).copy(), np.array([0, 768], np.uint64),
            np.zeros(1, np.int32), np.zeros(1, np.uint8), np.zeros(8, np.uint8), np.zeros(2, np.uint64)]
    ptr = [x.ctypes.data for x in arrs]
    rc = _lib.load().bftq_auth_client_process_batch(engine._h, tab, 1, ptr[0], ptr[1], ptr[2], ptr[3], ptr[4], ptr[5], ptr[6], 1, ptr[7], ptr[8],
                                                    ptr[9], 8, ptr[10], C.byref(need))
    assert rc == INVALID_ARG and need.value == 4 + 3 * (16 + 256)
    key(s)
    # t completes its set without an INITIATE: phase 1 and CIPHER_KEY are refused, then t continues
    run(engine, [(t, 0, ys[0], 0, t.rand(0, 0, rng)), (t, 0, ys[1], 1, t.rand(0, 1, rng))])
    bad([1], [1], [0], [A.chunk(b"\1")], [b""])             # phase 1 before Initiate
    bad([1], [KEY], [0], [b""], [b""])                      # CIPHER_KEY before Initiate
    run(engine, [(t, INIT, b"", 0, t.rand(INIT, 0, rng))])
    key(t)
    run(engine, [(t, 1, A.chunk(b"\x05" * 40), i, b"") for i in list(t.o.secrets)])
    # s finishes its login as if none of the refused calls happened
    run(engine, [(s, 0, ys[2], 2, s.rand(0, 2, rng))])
    ids = list(s.o.secrets)
    run(engine, [(s, 1, servers[i].make_bi(s.o.secrets[i]["Xi"], rng.randrange(A.P)), i, b"") for i in ids])
    run(engine, [(s, 2, servers[i].make_zi(s.o.secrets[i]["Ni"], rng.randbytes(12)), i, b"") for i in ids])
    key(s)


def test_failed_open_drops_the_proof(engine, sessions):
    """processZi assigns decrypt's result whatever it is: a good answer followed by a bad one from the same peer leaves
    that peer with no proof, and the map that completes later carries an empty entry for it."""
    rng = random.Random(0x2F)
    pw = b"drop"
    servers = setup(A.Rng(0x2F), pw, 3, 3, b"the proof")
    flip = lambda b, at: b[:at] + bytes([b[at] ^ 1]) + b[at + 1:]     # noqa: E731
    for variant in range(4):
        s = sessions(pw, 3, 3)
        X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))])[0][2]
        run(engine, [(s, 0, servers[i].make_yi(X), i, s.rand(0, i, rng)) for i in range(3)])
        run(engine, [(s, 1, servers[i].make_bi(s.o.secrets[i]["Xi"], rng.randrange(A.P)), i, b"") for i in range(3)])
        good = [servers[i].make_zi(s.o.secrets[i]["Ni"], rng.randbytes(12)) for i in range(3)]
        zi, nc = A.parse_zi(good[0])
        bad = [A.serialize_zi(flip(zi, len(zi) - 1), nc),          # tag mismatch
               A.serialize_zi(zi[:15], nc),                        # shorter than a tag
               A.serialize_zi(zi, nc + b"\0"),                     # a nonce that is not 12 bytes
               A.serialize_zi(flip(zi, 0), nc)][variant]           # ciphertext
        items = [(s, 2, good[0], 0, b""), (s, 2, bad, 0, b""), (s, 2, good[1], 1, b"")]
        got = run(engine, items)
        assert [g[0] for g in got] == [0, DECRYPTION_FAILED, 0]
        got = run(engine, [(s, 2, good[2], 2, b"")])[0]
        assert got[1] == 1 and AuthClient._parse_map(got[2]) == {0: b"", 1: b"the proof", 2: b"the proof"}
        # in one call too: the failure sits between the two successes of the other peers
        s2 = sessions(pw, 3, 3)
        X = run(engine, [(s2, INIT, b"", 0, s2.rand(INIT, 0, rng))])[0][2]
        run(engine, [(s2, 0, servers[i].make_yi(X), i, s2.rand(0, i, rng)) for i in range(3)])
        run(engine, [(s2, 1, servers[i].make_bi(s2.o.secrets[i]["Xi"], rng.randrange(A.P)), i, b"") for i in range(3)])
        good = [servers[i].make_zi(s2.o.secrets[i]["Ni"], rng.randbytes(12)) for i in range(3)]
        zi, nc = A.parse_zi(good[1])
        got = run(engine, [(s2, 2, good[1], 1, b""), (s2, 2, good[0], 0, b""), (s2, 2, A.serialize_zi(flip(zi, len(zi) - 1), nc), 1, b""),
                           (s2, 2, good[2], 2, b""), (s2, 2, good[0], 0, b"")])
        assert AuthClient._parse_map(got[4][2]) == {0: b"the proof", 1: b"", 2: b"the proof"}


def _mixed_sessions(engine, sessions, rng, count):
    """count sessions at every stage of a login: (session, next item) pairs, and the servers of each."""
    pw = b"mixed"
    servers = setup(A.Rng(0x256), pw, 5, 3)
    out = []
    for j in range(count):
        s = sessions(pw + bytes([j % 7]), 5, 3)
        stage = j % 5
        if stage >= 1:
            X = run(engine, [(s, INIT, b"", 0, s.rand(INIT, 0, rng))], check=True)[0][2]
            s.ys = [srv.make_yi(X) for srv in servers]
        if stage >= 2:
            run(engine, [(s, 0, s.ys[i], i, s.rand(0, i, rng)) for i in range(3)])
        if stage >= 3:
            run(engine, [(s, 1, servers[i].make_bi(s.o.secrets[i]["Xi"], 99 + i), i, b"") for i in range(3)])
        out.append((s, stage))
    return servers, out


def test_mixed_call_equals_sequential_replay(engine, sessions):
    rng = random.Random(0x256)
    servers, ss = _mixed_sessions(engine, sessions, rng, 256)
    items = []
    for s, stage in ss:
        if stage == 0:
            items.append((s, INIT, b"", 0, s.rand(INIT, 0, rng)))
        elif stage == 1:
            # a' for every peer the session can have: enough whichever of its items completes after the shuffle
            items += [(s, 0, s.ys[i], i, b"".join(a_bytes(rng.randrange(A.Q)) for _ in range(5))) for i in (2, 0, 1, 1, 4)]
        elif stage == 2:
            items += [(s, 1, servers[i].make_bi(s.o.secrets[i]["Xi"], 7 + i), i, b"") for i in (1, 0, 2)]
        elif stage == 3:
            for i in (0, 1, 2):                         # sealed as server i would seal it after this session's phase 1
                t = s.o.secrets[i]
                items.append((s, 2, A.serialize_zi(A.gcm_seal(t["ke"], bytes(12), b"proof", t["Ni"]), bytes(12)), i, b""))
        else:
            items.append((s, KEY, b"", 0, b""))
    rng.shuffle(items)
    run(engine, items)


def test_threads_on_disjoint_sessions(engine, sessions):
    params = A.generate_params(b"thr", 4, 3, A.Rng(0x88))
    ss = [[sessions(b"thr", 4, 3) for _ in range(2)] for _ in range(8)]
    errors = []

    def work(t):
        try:
            rng = random.Random(t)
            servers = [A.Server(p, b"proof", reference_zero_key_quirk=False) for p in params]
            for s in ss[t]:
                login(engine, s, servers, rng)
        except Exception as exc:                    # noqa: BLE001
            errors.append(exc)
    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


def test_destroy_and_handle_outliving_engine(built):
    eng = Engine(0)
    rng = random.Random(0x99)
    servers = setup(A.Rng(0x99), b"life", 4, 3)
    s = Session(eng, b"life", 4, 3)
    login(eng, s, servers, rng)
    c = AuthClient(eng, b"life", 4, 3, rand=rng.randrange)
    X = c.initiate([0, 1, 2, 3])[0]
    res = None
    for i in range(3):
        res, err = c.process_response(0, servers[i].make_yi(X), i)
        assert err is None
    assert set(res) == {0, 1, 2}
    assert c.get_cipher_key()[1] is None
    c.close()
    c.close()
    eng.close()
    eng.auth_client_destroy(s.h)


def test_wrapper_errors(engine):
    rng = random.Random(0x5)
    c = AuthClient(engine, b"w", 4, 2, rand=rng.randrange)
    try:
        assert c.get_cipher_key() == (None, ErrInsufficientNumberOfSecrets)
        assert c.process_response(1, A.chunk(b"\1"), 3) == (None, ErrNoAuthenticationData)
        c.initiate([0])
        assert c.process_response(2, A.serialize_zi(b"z" * 20, b"n" * 12), 3) == (None, ErrNoAuthenticationData)
        assert c.done(3) and not c.done(2)
    finally:
        c.close()
