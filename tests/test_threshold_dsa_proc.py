"""The threshold DSA / ECDSA client oracle (tests/threshold_dsa_proc_oracle.py) through whole rounds against the oracle
servers (threshold_dsa_oracle.phase2 / phase3, the joint shares travelling unencrypted), every signature checked by
`cryptography`; and its edge rules on hand-built answers.  The device client is checked against it in
test_threshold_dsa_proc_gpu.py."""
import hashlib
import math
import random
import struct

import pytest

import threshold_dsa_oracle as O
import threshold_dsa_proc_oracle as P
from test_threshold_dsa import _verify

REQUEST, RESPONSE = -1, 0


def shares_for(req: bytes, nid: int):
    """parseJointShareById over a phase-1 request."""
    r = P.Reader(req)
    assert r.uint(1) == 0
    for _ in range(r.uint(2)):
        i = r.uint(8)
        cs = [r.chunk() for _ in range(r.uint(2))]
        if i == nid:
            return cs
    return None


def parse_final(req: bytes):
    r = P.Reader(req)
    assert r.uint(1) == 1
    return int.from_bytes(r.chunk(), "big"), int.from_bytes(r.chunk(), "big")


def split_request(out: bytes):
    cnt = struct.unpack(">I", out[:4])[0]
    return [struct.unpack(">Q", out[4 + 8 * j:12 + 8 * j])[0] for j in range(cnt)], out[4 + 8 * cnt:]


class Round:
    """One signing round's servers (the oracle's phases 2 and 3 over plain joint shares) for a client driven by `call`,
    a function from [(op, data, peer)] to [(state, err, out)]."""

    def __init__(self, g, n: int, seed: int, tbs: bytes = b"tbs"):
        self.g, self.n, self.t = g, n, n // 2
        self.rng = random.Random(seed)
        self.x, self.coords = O.deal(self.rng, g, n, self.t)
        self.ids = [0x1000 + 17 * i for i in range(n)]
        self.joint = [O.joint_shares(self.rng, g, n, self.t) for _ in range(n)]       # joint[j][i]
        self.dgst = hashlib.sha256(tbs).digest()
        self.kc = {}

    def phase0(self, j: int) -> bytes:
        return P.joint_share_response([(O.share_plain(self.joint[j][i]), self.ids[i]) for i in range(self.n)])

    def phase1(self, i: int, req: bytes) -> bytes:
        X, k, c, out = O.phase2(self.g, shares_for(req, self.ids[i]))
        self.kc[i] = (k, c)
        return out

    def phase2(self, i: int, req: bytes) -> bytes:
        m, r = parse_final(req)
        return O.phase3(self.g, self.coords[i][0], self.coords[i][1], m, r, *self.kc[i])

    def run(self, call):
        """Drives the client one call per step; returns the signature and every output the client gave."""
        t2 = 2 * self.t
        log = []
        log += call([(REQUEST, b"", 0)])
        assert split_request(log[-1][2]) == (self.ids, b"")
        got = call([(RESPONSE, self.phase0(j), self.ids[j]) for j in range(t2)])
        assert [s for s, _, _ in got] == [P.PENDING] * (t2 - 1) + [P.CONTINUE]
        log += got
        (st, err, out), = call([(REQUEST, b"", 0)])
        nodes, req1 = split_request(out)
        assert nodes == self.ids[:t2]
        log.append((st, err, out))
        got = call([(RESPONSE, self.phase1(i, req1), self.ids[i]) for i in range(t2)])
        assert [s for s, _, _ in got] == [P.PENDING] * (t2 - 1) + [P.CONTINUE], got
        log += got
        (st, err, out), = call([(REQUEST, b"", 0)])
        log.append((st, err, out))
        _, req2 = split_request(out)
        got = call([(RESPONSE, self.phase2(i, req2), self.ids[i]) for i in range(t2)])
        assert [s for s, _, _ in got] == [P.PENDING] * (t2 - 1) + [P.SIGNED]
        log += got
        return got[-1][2], log


def oracle_call(proc):
    return lambda items: [P.step(proc, op, d, peer) for op, d, peer in items]


@pytest.mark.parametrize("name", ["1024/160", "2048/256", "p256"])
@pytest.mark.parametrize("n", [4, 7, 10])
def test_oracle_rounds_verify(name, n):
    g = dict(kind="p256") if name == "p256" else O.golden_key()[0] if name == "1024/160" else O.dsa_group(2048, 256)
    rd = Round(g, n, 0xD5B0 + n)
    proc = P.Proc("p256" if name == "p256" else "dsa", rd.dgst, rd.t, rd.ids)
    sig, _ = rd.run(oracle_call(proc))
    _verify(g, rd.x, rd.dgst, sig)
    assert P.step(proc, RESPONSE, b"anything", 5) == (P.SIGNED, 0, sig)          # the default branch: the same result


def test_phase0_last_listed():
    proc = P.Proc("dsa", bytes(32), 1, [])
    # th is the count of the LAST-listed id: 2 here (id 9 twice) although id 8 has one share
    assert P.step(proc, RESPONSE, P.joint_share_response([(b"a", 9), (b"b", 8)]), 1)[0] == P.PENDING
    assert P.step(proc, RESPONSE, P.joint_share_response([(b"c", 8), (b"d", 9)]), 2)[0] == P.CONTINUE
    assert proc.kmap == {9: [b"a", b"d"], 8: [b"b", b"c"]}
    proc = P.Proc("dsa", bytes(32), 1, [])
    assert P.step(proc, RESPONSE, P.joint_share_response([(b"a", 9), (b"c", 8)]), 1)[0] == P.PENDING
    assert P.step(proc, RESPONSE, P.joint_share_response([(b"d", 9), (b"e", 7)]), 2)[0] == P.PENDING
    assert P.step(proc, RESPONSE, struct.pack(">H", 0), 3)[0] == P.PENDING      # no shares: th = 0
    assert P.step(proc, RESPONSE, P.joint_share_response([(b"f", 7)]), 4)[0] == P.CONTINUE


def test_go_inverse_rules():
    g = O.golden_key()[0]
    q = g["q"]
    # v = 0: ModInverse nil, exponent 0, r = 1
    parts = [(1, O.bts(pow(g["g"], 5, g["p"])), 0), (2, O.bts(pow(g["g"], 7, g["p"])), 0)]
    assert P.calculate_r(g, parts) == 1
    # a composite odd q: gcd(v, q) = 3 makes the exponent v itself, gcd(v, q) = 1 its inverse; Fermat's power gives neither
    gc = dict(kind="dsa", p=g["p"], q=3 * 5 * 7 * 11 * 13 * 1000003, g=g["g"])
    qc = gc["q"]
    lam = [P.lagrange(x, [1, 2], qc) for x in (1, 2)]
    rp = pow(5, lam[0], g["p"]) * pow(7, lam[1], g["p"]) % g["p"]
    for v2, gcd, e in ((9, 3, lambda v: v), (4, 1, lambda v: pow(v, -1, qc))):
        v = (3 * lam[0] + v2 * lam[1]) % qc
        assert v != 0 and math.gcd(v, qc) == gcd
        want = pow(rp, e(v), g["p"]) % qc
        assert want != pow(rp, pow(v, qc - 2, qc), g["p"]) % qc
        assert P.calculate_r(gc, [(1, b"\x05", 3), (2, b"\x07", v2)]) == want
    # no inverse of the Lagrange denominator: Go panics
    with pytest.raises(P.Panic):
        P.lagrange(1, [1, 4], 3)


def test_ecdsa_infinity_and_bad_point():
    from oracle import sss_oracle as S
    g = dict(kind="p256", **O.P256)
    pt = S.p256_marshal(S.p256_mul(5, S.P256_G))
    neg = S.p256_mul(5, S.P256_G)
    negm = b"\x04" + neg[0].to_bytes(32, "big") + (S.P256_P - neg[1]).to_bytes(32, "big")
    # lambda = (2, -1) at x = (1, 2): 2 R - R' with R' = 2 R sums to infinity -> r = 0
    two = S.p256_marshal(S.p256_mul(10, S.P256_G))
    assert P.calculate_r(g, [(1, pt, 1), (2, two, 1)]) == 0
    assert P.calculate_r(g, [(1, pt, 0), (2, negm, 0)]) == 0                    # v = 0
    with pytest.raises(P.Panic):
        P.calculate_r(g, [(1, pt, 1), (2, b"\x04" + bytes(64), 1)])
