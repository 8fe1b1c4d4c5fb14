"""GPU suite: the server half of crypto/auth on the device (K9) against the oracle (tests/auth_oracle.py), byte for byte
given the same b and nonce: full TestAuth rounds, edge bases, exponents and parameters, every phase-2 case, mixed and
concurrent calls, and the one divergence (phase 2 before phase 1 fails instead of sealing under a zero key)."""
import json
import os
import random
import threading

import pytest

import auth_oracle as A
from bftkv_b200 import _lib
from bftkv_b200.crypto_gpu import AuthServer, ErrAuthTooManyAttempts, ErrAuthenticationFailure

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTH_FAILURE, INVALID_ARG, MALFORMED, UNSUPPORTED_KEY = -16, -3, -8, -4


class Pair:
    """A device server and the oracle server it must match (the oracle with the device's fail-closed phase 2)."""

    def __init__(self, engine, params, proof):
        self.h = engine.auth_server_create(params, proof)
        self.o = A.Server(params, proof, reference_zero_key_quirk=False)

    def oracle(self, phase, req, rand):
        if phase == 0:
            return 0, self.o.make_yi(req)
        if phase == 1:
            return 0, self.o.make_bi(req, int.from_bytes(rand, "big"))
        if phase == 2:
            try:
                return 0, self.o.make_zi(req, rand)
            except A.AuthenticationFailure:
                return AUTH_FAILURE, b""
            finally:                                    # server.go drops the session after phase 2
                self.o.mac, self.o.ke = None, bytes(16)
        return 0, b""


def call(engine, pairs, phases, reqs, rands, check=True):
    err, outs = engine.auth_server_respond_batch([p.h for p in pairs], list(range(len(pairs))), phases, reqs, rands)
    if check:
        for p, ph, q, r, e, o in zip(pairs, phases, reqs, rands, err, outs):
            we, wo = p.oracle(ph, q, r)
            assert (int(e), o) == (we, wo), (ph, len(q))
    return err, outs


def rand_for(phase, rng):
    return rng.randbelow(A.P).to_bytes(256, "big") if phase == 1 else rng.randbytes(12) if phase == 2 else b""


@pytest.fixture
def new_pairs(engine):
    made = []

    def make(params_list, proof):
        ps = [Pair(engine, p, proof) for p in params_list]
        made.extend(ps)
        return ps
    yield make
    for p in made:
        engine.auth_server_destroy(p.h)


def _collective_signature():
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "golden.json")))
    return b"".join(bytes.fromhex(c["sig"]) for c in g["cases"][:4])


@pytest.mark.parametrize("n,k,rounds,proof", [(10, 7, 3, None), (4, 3, 2, None), (4, 3, 1, "sig")])
def test_full_rounds(engine, new_pairs, n, k, rounds, proof):
    rng = A.Rng(0x9A17 + n + rounds)
    for _ in range(rounds):
        password = rng.randbytes(8)
        pf = _collective_signature() if proof == "sig" else rng.randbytes(16)

        def respond(pairs, ids, phase, reqs, rands):
            return call(engine, [pairs[i] for i in ids], [phase] * len(ids), reqs, rands)[1]
        c, pis = A.run_round(password, pf, n, k, rng, make_servers=new_pairs, respond=respond)
        assert pis is not None and len(pis) >= k and all(p == pf for p in pis.values())


def _params(rng, y=None, v=None, salt=None):
    return A.serialize_params(rng.randbelow(100), rng.randbelow(A.Q) if y is None else y, rng.randbelow(A.P) if v is None else v,
                              rng.randbytes(32) if salt is None else salt)


def test_edge_bases(engine, new_pairs):
    rng = A.Rng(0xE1)
    P = A.P
    xs = [b"", b"\0", b"\1", A.i2b(P - 1), A.i2b(P), A.i2b(P + 1), A.i2b(2 * P), b"\0\0\0" + A.i2b(P - 5), b"\0" * 300,
          rng.randbytes(300), rng.randbytes(4096), b"\0" * 17 + rng.randbytes(256)]
    pairs = new_pairs([_params(rng) for _ in xs], b"proof")
    call(engine, pairs, [0] * len(xs), xs, [b""] * len(xs))
    rands = [rand_for(1, rng) for _ in xs]
    call(engine, pairs, [1] * len(xs), xs, rands)
    nis = [p.o.mac for p in pairs]
    call(engine, pairs, [2] * len(xs), nis, [rand_for(2, rng) for _ in xs])


def test_edge_exponents_and_params(engine, new_pairs):
    rng = A.Rng(0xE2)
    P, Q = A.P, A.Q
    params = [_params(rng, y=0), _params(rng, y=Q - 1), _params(rng, v=0), _params(rng, v=1), _params(rng, salt=b""),
              _params(rng, salt=rng.randbytes(65)), _params(rng, salt=rng.randbytes(200)), _params(rng, v=P - 1, salt=rng.randbytes(64)),
              A.serialize_params(-5, 2 ** 2048 - 1, 2 ** 2048 - 1, b"s")]                      # v >= p: reduced on registration
    pairs = new_pairs(params, rng.randbytes(33))
    X = A.i2b(pow(A.PI(b"pw"), rng.randbelow(Q), P))
    call(engine, pairs, [0] * len(pairs), [X] * len(pairs), [b""] * len(pairs))
    for b in (0, 1, P - 1, rng.randbelow(P)):
        call(engine, pairs, [1] * len(pairs), [X] * len(pairs), [b.to_bytes(256, "big")] * len(pairs))
        call(engine, pairs, [2] * len(pairs), [p.o.mac for p in pairs], [rand_for(2, rng) for _ in pairs])


def test_minimal_encodings_with_leading_zeros(engine, new_pairs):
    """Seeded searches for b whose Bi or Ki has leading zero bytes, and for Bi and Ki = 0 (empty encodings)."""
    rng = A.Rng(0xE3)
    v = rng.randbelow(A.P)
    pair, = new_pairs([_params(rng, v=v)], b"p" * 20)
    xi = A.i2b(rng.randbelow(A.P))
    found_bi = found_ki = 0
    for _ in range(3000):
        b = rng.randbelow(A.P)
        bi, ki = pow(v, b, A.P), pow(int.from_bytes(xi, "big"), b, A.P)
        if bi < 1 << 2040 or ki < 1 << 2040:
            found_bi += bi < 1 << 2040
            found_ki += ki < 1 << 2040
            call(engine, [pair], [1], [xi], [b.to_bytes(256, "big")])
            call(engine, [pair], [2], [pair.o.mac], [rand_for(2, rng)])
        if found_bi and found_ki:
            break
    assert found_bi and found_ki
    zero, = new_pairs([_params(rng, v=0)], b"z")
    b = rng.randbelow(A.P).to_bytes(256, "big")
    for x in (b"", A.i2b(A.P), A.i2b(3 * A.P)):                      # Ki = 0 and Bi = 0: both empty
        _, (out,) = call(engine, [zero], [1], [x], [b])
        assert out == bytes(8)
        call(engine, [zero], [2], [zero.o.mac], [rand_for(2, rng)])


def test_phase_two_cases(engine, new_pairs):
    rng = A.Rng(0xE4)
    pairs = new_pairs([_params(rng) for _ in range(8)], b"the proof")
    xi = A.i2b(rng.randbelow(A.P))
    # phase 2 before any phase 1: the divergence, even with an empty Ni
    err, outs = call(engine, pairs[:2], [2, 2], [b"", bytes(32)], [rand_for(2, rng)] * 2)
    assert list(err) == [AUTH_FAILURE] * 2 and outs == [b"", b""]
    assert A.Server(A.serialize_params(1, 2, 3, b"s"), b"the proof").make_response(2, b"", bytes(12))[2] is None   # the reference leaks
    call(engine, pairs, [1] * 8, [xi] * 8, [rand_for(1, rng) for _ in range(8)])
    mac = [p.o.mac for p in pairs]
    flipped = bytes([mac[1][0] ^ 0x10]) + mac[1][1:]
    nis = [mac[0], flipped, mac[2][:16], mac[3][:31], mac[4] + b"\0", b"", mac[6], mac[7]]
    # pairs 6 and 7: a repeated phase 1 (the latest wins) and a phase 0 in between (keeps the state)
    call(engine, pairs[6:7], [1], [xi], [rand_for(1, rng)])
    call(engine, pairs[7:8], [0], [xi], [b""])
    nis[6] = pairs[6].o.mac
    err, _ = call(engine, pairs, [2] * 8, nis, [rand_for(2, rng) for _ in range(8)])
    assert list(err) == [0, AUTH_FAILURE, AUTH_FAILURE, AUTH_FAILURE, AUTH_FAILURE, AUTH_FAILURE, 0, 0]
    # phase 2 twice: the state was wiped by the first
    err, _ = call(engine, pairs[:1], [2], [mac[0]], [rand_for(2, rng)])
    assert list(err) == [AUTH_FAILURE]
    # phase >= 3: empty, no error, no state change
    call(engine, pairs[:2], [1, 1], [xi, xi], [rand_for(1, rng)] * 2)
    err, outs = call(engine, pairs[:2], [3, 7], [b"x", b""], [b"", b""])
    assert list(err) == [0, 0] and outs == [b"", b""]
    call(engine, pairs[:2], [2, 2], [pairs[0].o.mac, pairs[1].o.mac], [rand_for(2, rng)] * 2)


def test_mixed_call_over_many_servers(engine, new_pairs):
    rng = A.Rng(0xE5)
    n = 96
    pairs = new_pairs([_params(rng, salt=rng.randbytes(rng.randbelow(90))) for _ in range(n)], rng.randbytes(rng.randbelow(2000)))
    xs = [A.i2b(rng.randbelow(A.P)) for _ in range(n)]
    call(engine, pairs[: n // 2], [1] * (n // 2), xs[: n // 2], [rand_for(1, rng) for _ in range(n // 2)])
    phases = [rng.randbelow(4) for _ in range(n)]
    order = list(range(n))
    rng.r.shuffle(order)
    sel = [pairs[i] for i in order]
    ph = [phases[i] for i in order]
    reqs = [p.o.mac if (f == 2 and p.o.mac) else xs[i] for p, f, i in zip(sel, ph, order)]
    err, _ = call(engine, sel, ph, reqs, [rand_for(f, rng) for f in ph])
    assert 0 in list(err)


def test_duplicate_handle_and_bad_arguments_change_nothing(engine, new_pairs):
    rng = A.Rng(0xE6)
    pairs = new_pairs([_params(rng) for _ in range(2)], b"proof")
    xi = A.i2b(rng.randbelow(A.P))
    call(engine, pairs, [1, 1], [xi, xi], [rand_for(1, rng)] * 2)
    for idx, phases, rands in [([0, 0], [2, 2], [bytes(12)] * 2),          # the same server twice
                               ([0, 1], [1, 2], [bytes(255), bytes(12)]),  # b of the wrong length
                               ([0, 1], [2, 2], [bytes(12), bytes(16)])]:  # a nonce of the wrong length
        with pytest.raises(_lib.BftqError) as ei:
            engine.auth_server_respond_batch([p.h for p in pairs], idx, phases, [pairs[0].o.mac] * 2, rands)
        assert ei.value.code == INVALID_ARG
    call(engine, pairs, [2, 2], [pairs[0].o.mac, pairs[1].o.mac], [rand_for(2, rng)] * 2)       # the state survived
    assert [p.o.mac for p in pairs] == [None, None]


def test_registration_errors(engine):
    good = A.serialize_params(1, 5, 7, b"salt")
    for bad in (b"", good[:3], good[:4 + 8 + 1], good[:-1]):
        with pytest.raises(_lib.BftqError) as ei:
            engine.auth_server_create(bad, b"p")
        assert ei.value.code == MALFORMED
    for y, v in ((1 << 2048, 1), (1, 1 << 2048)):
        with pytest.raises(_lib.BftqError) as ei:
            engine.auth_server_create(A.serialize_params(1, y, v, b"s"), b"p")
        assert ei.value.code == UNSUPPORTED_KEY


def test_eight_threads_disjoint_servers(engine, new_pairs):
    rng = A.Rng(0xE7)
    groups = [new_pairs([_params(rng) for _ in range(6)], rng.randbytes(40)) for _ in range(8)]
    plans = []
    for g in groups:
        xi = A.i2b(rng.randbelow(A.P))
        plans.append((g, xi, [rand_for(1, rng) for _ in g], [rand_for(2, rng) for _ in g]))
    errors = []

    def work(g, xi, r1, r2):
        try:
            for _ in range(3):
                call(engine, g, [0] * len(g), [xi] * len(g), [b""] * len(g))
                call(engine, g, [1] * len(g), [xi] * len(g), r1)
                call(engine, g, [2] * len(g), [p.o.mac for p in g], r2)
        except Exception as exc:                         # noqa: BLE001 (reported below)
            errors.append(exc)
    ts = [threading.Thread(target=work, args=pl) for pl in plans]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_auth_server_class_attempts_and_delay(engine):
    rng = A.Rng(0xE8)
    params = A.generate_params(b"pw", 4, 3, rng)
    delays = []
    s = AuthServer(engine, params[0], b"proof", delay=delays.append)
    o = A.Server(params[0], b"proof")
    X = A.i2b(pow(A.PI(b"pw"), 12345, A.P))
    for i in range(10):
        res, done, err = s.make_response(0, X)
        assert res == o.make_yi(X) and not done
        assert err == (ErrAuthTooManyAttempts if i == 9 else None)
    assert delays == [float(i) for i in range(1, 10)]
    res, done, err = s.make_response(2, b"")
    assert (res, done, err) == (None, True, ErrAuthenticationFailure)
    b = rng.randbelow(A.P).to_bytes(256, "big")
    assert s.make_response(1, X, b) == (o.make_bi(X, int.from_bytes(b, "big")), False, None)
    res, done, err = s.make_response(2, o.mac)
    zi, nonce = A.parse_zi(res)
    assert done and err is None and A.gcm_open(o.ke, nonce, zi, o.mac) == b"proof"
    s.close()
