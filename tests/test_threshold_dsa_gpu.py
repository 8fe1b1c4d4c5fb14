"""K8 (thdsa_sign.cuh, bftq_thdsa_sign_batch): dsaContext.Sign's phases 2 and 3 on the device, byte-equal to the oracle
(tests/threshold_dsa_oracle.py).  The rounds run end to end on the device: the joint shares through the device's decrypt,
phase 2, the existing CalculateR (bftq_dsa_calculate_r_batch / bftq_ecdsa_p256_calculate_r_batch), phase 3 and the
existing calculateS (bftq_lagrange_combine_batch); the signature is checked by `cryptography` and by the device's own
DSA / ECDSA verification (K1c / K1d).  Also: the quirks of the reference's decrypt loop on both group kinds, mixed shares
in one call, and calls from 8 host threads."""
import numpy as np
import hashlib
import random
import threading

import pytest

from bftkv_b200 import workload as W
from bftkv_b200.crypto_gpu import Keyring, ThresholdDSA
import pgp_encrypt_ref as R
import threshold_dsa_oracle as O
from test_threshold_dsa import _verify

pytestmark = pytest.mark.gpu

_GROUPS = {}


def group(name):
    if name not in _GROUPS:
        # 1024/160: the reference's own key (crypto/threshold/dsa/test.pkcs8); the 2048-bit domains are seeded
        _GROUPS[name] = dict(kind="p256") if name == "p256" else O.golden_key()[0] if name == "1024/160" else \
            O.dsa_group(2048, int(name.split("/")[1]))
    return _GROUPS[name]


class Net:
    """n nodes with RSA-2048 PGP keys; node s's keyring holds its private key and every node's certificate."""

    def __init__(self, engine, n):
        self.keys = W.load_keys(n)
        privs = [W._private_key(k) for k in self.keys]
        self.blocks = [W.pgp_public_key_block(k, pv, b"node%d" % i) for i, (k, pv) in enumerate(zip(self.keys, privs))]
        self.ids = [b[1] for b in self.blocks]
        self.rings = []
        for s in range(n):
            kr = Keyring(engine)
            kr.register(self.blocks[s][0], priv=True)
            for j in range(n):
                if j != s:
                    kr.register(self.blocks[j][0])
            assert kr.register_private(R.secret_key_packet(self.keys[s])) == 1
            self.rings.append(kr)

    def message(self, rng, sender, recipient, plain, nonce):
        inner = W.make_transport_message(self.keys[sender], self.ids[sender], plain, nonce)
        return R.encrypt(rng, self.keys[recipient], self.ids[recipient], inner)


def setup_round(engine, name, n, seed):
    g = group(name)
    rng = random.Random(seed)
    t = n // 2
    net = Net(engine, n)
    x, coords = O.deal(rng, g, n, t)
    secs = [O.share_secret(g, X, O.bts(Y), t) for X, Y in coords]
    joint = [O.joint_shares(rng, g, n, t) for _ in range(n)]
    nonces = [bytes(rng.randrange(256) for _ in range(16)) for _ in range(n)]       # each server's nonce for this client
    # the phase-2 request: for every node id, the encrypted shares of every responder, in response order
    kmap = [(net.ids[i], [net.message(rng, j, i, O.share_plain(joint[j][i]), nonces[j]) for j in range(n)]) for i in range(n)]
    return g, rng, t, net, x, coords, secs, joint, nonces, kmap


def device_verify(engine, g, x: int, digest: bytes, sig: bytes) -> int:
    q = O.order(g)
    n = (q.bit_length() + 7) // 8
    r_be = np.frombuffer(sig[:n].rjust(32, b"\0"), np.uint8).reshape(1, 32)
    s_be = np.frombuffer(sig[n:].rjust(32, b"\0"), np.uint8).reshape(1, 32)
    d = np.frombuffer(digest, np.uint8).reshape(1, -1)
    if g["kind"] == "dsa":
        return int(engine.dsa_verify_batch(g["p"], q, g["g"], pow(g["g"], x, g["p"]), r_be, s_be, d)[0])
    from oracle import sss_oracle as S
    X, Y = S.p256_mul(x, S.P256_G)
    pub = np.frombuffer(X.to_bytes(32, "big") + Y.to_bytes(32, "big"), np.uint8).reshape(1, 64)
    return int(engine.ecdsa_p256_verify_batch(pub, np.zeros(1, np.uint32), r_be, s_be, d)[0])


@pytest.mark.parametrize("name,n", [("1024/160", 4), ("2048/224", 4), ("2048/256", 4), ("1024/160", 10), ("p256", 4), ("p256", 7),
                                    ("p256", 10)])
def test_round_end_to_end(engine, name, n):
    g, rng, t, net, x, coords, secs, joint, nonces, kmap = setup_round(engine, name, n, 0xD5A2 + n)
    req2 = O.phase2_request(kmap)
    th = ThresholdDSA(engine, "p256" if name == "p256" else "dsa")
    client = 0x51
    parts, kc = [], {}
    for i in range(2 * t):
        got = th.sign(net.rings[i], secs[i], req2, client, net.ids[i], nonces[i])
        X, k, c, want = O.phase2(g, [O.share_plain(joint[j][i]) for j in range(n)])
        assert got == (want, None), (name, i)
        kc[i] = (k, c)
        parts.append(O.parse_partial(g, got[0]))
    q = O.order(g)
    digest = hashlib.sha256(b"tbs").digest()
    m = int.from_bytes(digest[:(q.bit_length() + 7) // 8], "big")                 # OS2I: q is byte-aligned here
    xs = [[p[0] for p in parts]]
    if g["kind"] == "dsa":                                                          # the existing device CalculateR
        rs, st = engine.dsa_calculate_r_batch(g["p"], q, xs, [[int.from_bytes(p[1], "big") for p in parts]], [[p[2] for p in parts]])
    else:
        rs, st = engine.ecdsa_p256_calculate_r_batch(xs, [[p[1] for p in parts]], [[p[2] for p in parts]])
    assert st[0] == 0 and rs[0] == O.calculate_r(g, parts)
    r = rs[0]
    req3 = O.phase3_request(m, r)
    sparts = []
    for i in range(2 * t):
        got, err = th.sign(net.rings[i], secs[i], req3, client, net.ids[i], None)
        want = O.phase3(g, coords[i][0], coords[i][1], m, r, *kc[i])
        assert (got, err) == (want, None)
        px, s, _ = O.parse_partial(g, got)
        sparts.append((px, int.from_bytes(s, "big")))
    qlen = (q.bit_length() + 7) // 8                                                # the existing device calculateS
    ys = np.frombuffer(b"".join(v.to_bytes(qlen, "big") for _, v in sparts), np.uint8).reshape(1, len(sparts), qlen)
    out, st = engine.lagrange_combine_batch(q, np.array([[p[0] for p in sparts]], np.int32), ys)
    assert st[0] == 0 and int.from_bytes(bytes(out[0]), "big") == O.calculate_s(g, sparts)
    sig = O.format_dsa(r, int.from_bytes(bytes(out[0]), "big"), q)
    _verify(g, x, digest, sig)
    assert device_verify(engine, g, x, digest, sig) == 0
    bad = sig[:-1] + bytes([sig[-1] ^ 1])
    assert device_verify(engine, g, x, digest, bad) != 0
    th.close()


@pytest.mark.parametrize("name", ["p256", "1024/160", "2048/256"])
def test_quirks(engine, name):
    g, rng, t, net, x, coords, secs, joint, nonces, kmap = setup_round(engine, name, 4, 0xD5A3)
    th = ThresholdDSA(engine, "p256" if name == "p256" else "dsa")
    kr, me = net.rings[0], net.ids[0]
    req2 = O.phase2_request(kmap)
    B = lambda reqs, nn, peers=None: th.sign_batch(kr, [secs[0]] * len(reqs), reqs, peers or [7] * len(reqs), me, nn)
    # absent / wrong nonce, no entry for self, phase 3 first, an entry with zero shares, truncation
    res = B([req2, req2, O.phase2_request(kmap[1:]), O.phase3_request(5, 6), O.phase2_request([(me, [])]), O.phase2_request(kmap[:1])[:-3]],
            [None, b"x" * 16, nonces[0], None, nonces[0], nonces[0]], [7, 7, 7, 99, 7, 7])
    assert [e for _, e in res] == ["crypto: share not found"] * 3 + ["crypto: key not found", "crypto: invalid input",
                                                                     "threshold dsa: malformed request or share"]
    # no self share among the encrypted ones -> share not found; an unknown signer -> malformed (Go panics)
    no_self = [(me, kmap[0][1][1:])]
    stranger = W.load_keys(6)[5]
    inner = W.make_transport_message(stranger, 0x0102030405060708, O.share_plain(joint[1][0]), nonces[1])
    alien = R.encrypt(rng, net.keys[0], me, inner)
    bad_x = list(joint[1][0]); bad_x[2] = (bad_x[2][0] + 1, bad_x[2][1])
    tampered = bytearray(W.make_transport_message(net.keys[1], net.ids[1], O.share_plain(joint[1][0]), nonces[1]))
    tampered[-5] ^= 1                                                              # a byte of the signature packet
    tampered = R.encrypt(rng, net.keys[0], me, bytes(tampered))
    res = B([O.phase2_request(no_self), O.phase2_request([(me, [kmap[0][1][0], alien])]),
             O.phase2_request([(me, [kmap[0][1][0], net.message(rng, 1, 0, O.share_plain(bad_x), nonces[1])])]),
             O.phase2_request([(me, [kmap[0][1][0], tampered] + kmap[0][1][2:])])],
            [nonces[0]] * 4)
    assert [e for _, e in res] == ["crypto: share not found", "threshold dsa: malformed request or share", "crypto: invalid input",
                                   "crypto: invalid signature"]
    # two phase-2s before a phase 3, within one call: the later wins; Y, m, r >= q and long
    q = O.order(g)
    j2 = [O.joint_shares(rng, g, 4, 2) for _ in range(4)]             # j2[j][0]: server j's shares for node 0
    kmap2 = [(me, [net.message(rng, j, 0, O.share_plain(j2[j][0] if j else joint[0][0]), nonces[j]) for j in range(4)])]
    req_b = O.phase2_request(kmap2)
    big = (1 << 600) + 3 * q
    res = B([req2, req_b, O.phase3_request(big + 5, big + 11)], [nonces[0]] * 2 + [None])
    _, k, c, want2 = O.phase2(g, [O.share_plain(j2[j][0] if j else joint[0][0]) for j in range(4)])
    assert res[1] == (want2, None)
    assert res[2] == (O.phase3(g, coords[0][0], coords[0][1], big + 5, big + 11, k, c), None)
    # ... and across calls: a later call's phase 2 replaces the stored (k, c)
    assert B([req2], [nonces[0]]) == [(O.phase2(g, [O.share_plain(joint[j][0]) for j in range(4)])[3], None)]
    _, k1, c1, _ = O.phase2(g, [O.share_plain(joint[j][0]) for j in range(4)])
    assert B([O.phase3_request(3, 4)], [None]) == [(O.phase3(g, coords[0][0], coords[0][1], 3, 4, k1, c1), None)]
    # a Byzantine peer's joint share with Y >= q in a long chunk: reduced like big.Int's sums
    q = O.order(g)
    long_j = [(X_, (Y_ + 3 * q).to_bytes(90, "big")) for X_, Y_ in joint[1][0]]
    kmap3 = [(me, [kmap[0][1][0], net.message(rng, 1, 0, O.share_plain(long_j), nonces[1])] + kmap[0][1][2:])]
    want3 = O.phase2(g, [O.share_plain(joint[0][0]), O.share_plain(long_j)] + [O.share_plain(joint[j][0]) for j in range(2, 4)])[3]
    assert B([O.phase2_request(kmap3)], [nonces[0]], [9]) == [(want3, None)]
    long_y = O.share_secret(g, coords[0][0], (coords[0][1] + 5 * q).to_bytes(80, "big"), 2)
    r3 = th.sign_batch(kr, [long_y, long_y], [req_b, O.phase3_request(1, 2)], [8, 8], me, [nonces[0], None])
    assert r3[1] == (O.phase3(g, coords[0][0], coords[0][1], 1, 2, k, c), None)
    th.close()


def test_a_zero(engine):
    """a_i = 0 mod q: R_i is 04 || 0^64 on P-256 and 01 in DSA."""
    for name in ("p256", "1024/160"):
        g = group(name)
        rng = random.Random(0xD5A4)
        net = Net(engine, 2)
        q = O.order(g)
        sh = [[(1, rng.randrange(q)), (1, 0 if j == 0 else q), (1, 0), (1, rng.randrange(q))] for j in range(2)]
        nonce = bytes(16)
        req = O.phase2_request([(net.ids[0], [net.message(rng, j, 0, O.share_plain(sh[j]), nonce) for j in range(2)])])
        th = ThresholdDSA(engine, "p256" if name == "p256" else "dsa")
        got, err = th.sign(net.rings[0], O.share_secret(g, 1, b"\x05", 1), req, 3, net.ids[0], nonce)
        assert err is None and got == O.phase2(g, [O.share_plain(s) for s in sh])[3]
        assert (b"\x04" + bytes(64)) in got if name == "p256" else got[8:17] == b"\x00" * 7 + b"\x01\x01"
        th.close()


@pytest.mark.parametrize("sec_kind", ["p384", "bits", "even", "3072"])
def test_unsupported_groups(engine, sec_kind):
    from bftkv_b200._lib import BftqError
    if sec_kind in ("p384", "bits"):
        g = dict(kind="p256")
        sec = O.share_secret(g, 1, b"\x01", 1)
        if sec_kind == "bits":
            sec = sec[:len(O.group_ser(g)) - 4] + (384).to_bytes(4, "big") + sec[len(O.group_ser(g)):]
        else:
            sec = O.chunk(O.bts((1 << 384) - (1 << 128) - (1 << 96) + (1 << 32) - 1)) + sec[8 + 32:]
        algo = 3
    else:
        p = {"even": (1 << 1023) + 2, "3072": (1 << 3071) + 1}[sec_kind]
        sec = O.share_secret(dict(kind="dsa", p=p, q=(1 << 159) + 7, g=2), 1, b"\x01", 1)
        algo = 2
    with pytest.raises(BftqError) as ei:
        engine.thdsa_share_create(algo, sec)
    assert ei.value.code == -4


def test_threads(engine):
    g, rng, t, net, x, coords, secs, joint, nonces, kmap = setup_round(engine, "1024/160", 4, 0xD5A5)
    req2 = O.phase2_request(kmap)
    want = O.phase2(g, [O.share_plain(joint[j][0]) for j in range(4)])[3]
    th = ThresholdDSA(engine, "dsa")
    th.register(secs[0])
    out = [None] * 8

    def work(i):
        out[i] = th.sign_batch(net.rings[0], [secs[0]] * 4, [req2] * 4, [100 + i] * 4, net.ids[0], [nonces[0]] * 4)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    [x.start() for x in ts]
    [x.join() for x in ts]
    assert all(r == [(want, None)] * 4 for r in out)
    th.close()


def test_mixed_shares_one_call(engine):
    """Shares of 1024/160, 2048/224, 2048/256 and P-256 in one call, phase-2 and phase-3 items interleaved: every R kernel,
    the warp's trip count over q of different lengths, and the (k, c) rows across shares."""
    rng = random.Random(0xD5AA)
    n, t = 4, 2
    net = Net(engine, n)
    me = net.ids[0]
    names = ["1024/160", "2048/224", "2048/256", "p256"]
    nonce = bytes(range(16))
    case = {}
    for name in names:
        g = group(name)
        x, coords = O.deal(rng, g, n, t)
        joint = [O.joint_shares(rng, g, n, t) for _ in range(n)]
        req2 = O.phase2_request([(me, [net.message(rng, j, 0, O.share_plain(joint[j][0]), nonce) for j in range(n)])])
        _, k, c, want2 = O.phase2(g, [O.share_plain(joint[j][0]) for j in range(n)])
        q = O.order(g)
        m, r = rng.randrange(q), rng.randrange(q)
        case[name] = (O.share_secret(g, coords[0][0], O.bts(coords[0][1]), t), req2, want2,
                      O.phase3_request(m, r), O.phase3(g, coords[0][0], coords[0][1], m, r, k, c))
    th_d, th_e = ThresholdDSA(engine, "dsa"), ThresholdDSA(engine, "p256")
    for name in names:
        (th_e if name == "p256" else th_d).register(case[name][0])
    order = [(0, 2), (1, 2), (0, 3), (3, 2), (2, 2), (1, 3), (3, 3), (2, 3)]           # (group, phase)
    reqs = [case[names[gi]][1 if ph == 2 else 3] for gi, ph in order]
    want = [(case[names[gi]][2 if ph == 2 else 4], None) for gi, ph in order]
    handles = [(th_e if names[gi] == "p256" else th_d).register(case[names[gi]][0]) for gi, _ in order]
    uniq = []
    for h in handles:
        if h.value not in [u.value for u in uniq]:
            uniq.append(h)
    idx = [[u.value for u in uniq].index(h.value) for h in handles]
    err, outs = engine.thdsa_sign_batch(net.rings[0]._h, uniq, idx, reqs, [5] * len(order), me,
                                        [nonce if ph == 2 else None for _, ph in order])
    assert list(err) == [0] * len(order)
    assert [(o, None) for o in outs] == want
    th_d.close()
    th_e.close()
