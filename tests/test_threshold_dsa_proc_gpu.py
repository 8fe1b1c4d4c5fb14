"""K8's client half (bftq_thdsa_process_batch): dsaProc's MakeRequest and ProcessResponse with CalculateR and calculateS on
the device, byte-equal to the client oracle (tests/threshold_dsa_proc_oracle.py) item by item: whole rounds (against the
oracle servers and against K8's device servers), any interleaving and split of many processes over calls, the reference's
quirks, every failure, and calls from 8 host threads."""
import hashlib
import random
import struct
import threading

import pytest

from bftkv_b200 import _lib
from bftkv_b200.crypto_gpu import ThresholdDSA, ThresholdDSAProcess, ErrContinue
import threshold_dsa_oracle as O
import threshold_dsa_proc_oracle as P
from test_threshold_dsa import _verify
from test_threshold_dsa_proc import REQUEST, RESPONSE, Round, oracle_call, split_request, shares_for
from test_threshold_dsa_gpu import device_verify, group, setup_round

pytestmark = pytest.mark.gpu

KIND = lambda name: "p256" if name == "p256" else "dsa"
ALGO = {"dsa": 2, "p256": 3}


def device_run(engine, procs, items):
    """items: [(proc index, op, data, peer)] in one call -> [(state, err, out)]."""
    st, err, outs = engine.thdsa_process_batch(procs, [i for i, _, _, _ in items], [op for _, op, _, _ in items],
                                               [p for _, _, _, p in items], [d for _, _, d, _ in items])
    return [(int(s), int(e), o) for s, e, o in zip(st, err, outs)]


def device_call(engine, h):
    return lambda items: device_run(engine, [h], [(0, op, d, p) for op, d, p in items])


def both(engine, kind, dgst, t, nodes, items):
    """The same items on the oracle and on the device (one call): both result lists, asserted equal."""
    proc = P.Proc(kind, dgst, t, nodes)
    want = [P.step(proc, op, d, p) for op, d, p in items]
    h = engine.thdsa_proc_create(ALGO[kind], dgst, t, nodes)
    got = device_call(engine, h)(items)
    engine.thdsa_proc_destroy(h)
    assert got == want
    return got


def partial(g, x: int, s: bytes, v: int) -> bytes:                       # serializePartialSignature
    return struct.pack(">Q", x & (2 ** 64 - 1)) + O.chunk(s) + O.chunk(O.bts(v) if isinstance(v, int) else v) + O.group_ser(g)


@pytest.mark.parametrize("name", ["1024/160", "2048/224", "2048/256", "p256"])
@pytest.mark.parametrize("n", [4, 7, 10])
def test_rounds_against_oracle(engine, name, n):
    g = group(name)
    rd_o, rd_d = Round(g, n, 0xD5C0 + n), Round(g, n, 0xD5C0 + n)
    proc = P.Proc(KIND(name), rd_o.dgst, rd_o.t, rd_o.ids)
    sig_o, log_o = rd_o.run(oracle_call(proc))
    h = engine.thdsa_proc_create(ALGO[KIND(name)], rd_d.dgst, rd_d.t, rd_d.ids)
    sig, log = rd_d.run(device_call(engine, h))
    assert log == log_o and sig == sig_o
    _verify(g, rd_d.x, rd_d.dgst, sig)
    assert device_verify(engine, g, rd_d.x, rd_d.dgst, sig) == 0
    assert device_verify(engine, g, rd_d.x, rd_d.dgst, sig[:-1] + bytes([sig[-1] ^ 1])) != 0
    assert device_call(engine, h)([(RESPONSE, b"late", 77)]) == [(P.SIGNED, 0, sig)]
    engine.thdsa_proc_destroy(h)


@pytest.mark.parametrize("name", ["1024/160", "2048/224", "2048/256", "p256"])
@pytest.mark.parametrize("n", [4, 7, 10])
def test_round_with_device_servers(engine, name, n):
    """Server phases 2 and 3 through bftq_thdsa_sign_batch (real encrypted joint shares), the client through the new call."""
    g, rng, t, net, x, coords, secs, joint, nonces, kmap = setup_round(engine, name, n, 0xD5C9 + n)
    th = ThresholdDSA(engine, KIND(name))
    dgst = hashlib.sha256(b"device servers").digest()
    cl = ThresholdDSAProcess(engine, KIND(name), dgst, t, net.ids)
    oc = P.Proc(KIND(name), dgst, t, net.ids)
    client = 0x51
    assert cl.make_request() == ((net.ids, None), None)
    oc.make_request()
    for j in range(2 * t):                                                   # phase 0: server j's encrypted shares for every node
        resp = P.joint_share_response([(kmap[i][1][j], net.ids[i]) for i in range(n)])
        want = P.step(oc, RESPONSE, resp, net.ids[j])
        assert cl.process_response(resp, net.ids[j]) == (None, ErrContinue if want[0] == P.CONTINUE else None)
    (nodes, req1), _ = cl.make_request()
    assert struct.pack(">I", len(nodes)) + b"".join(struct.pack(">Q", v) for v in nodes) + req1 == P.step(oc, REQUEST)[2]
    for i in range(2 * t):
        (ans, err), = th.sign_batch(net.rings[i], [secs[i]], [req1], [client], net.ids[i], [nonces[i]])
        assert err is None
        want = P.step(oc, RESPONSE, ans, net.ids[i])
        assert cl.process_response(ans, net.ids[i]) == (None, ErrContinue if want[0] == P.CONTINUE else None)
    (nodes, req2), _ = cl.make_request()
    assert req2 == P.step(oc, REQUEST)[2][4 + 8 * len(nodes):]
    for i in range(2 * t):
        (ans, err), = th.sign_batch(net.rings[i], [secs[i]], [req2], [client], net.ids[i], [None])
        res = cl.process_response(ans, net.ids[i])
        want = P.step(oc, RESPONSE, ans, net.ids[i])
        assert res == ((want[2], None) if want[0] == P.SIGNED else (None, None))
    sig = res[0]
    _verify(g, x, dgst, sig)
    assert device_verify(engine, g, x, dgst, sig) == 0
    cl.close()
    th.close()


def _scripts(n_procs, seed):
    """Per process: its group kind, create arguments and item list (from the oracle run), and the oracle's outputs."""
    rng = random.Random(seed)
    names = ["1024/160", "2048/224", "2048/256", "p256"]
    out = []
    for k in range(n_procs):
        name = names[k % 4]
        n = rng.choice([4, 5, 6])
        rd = Round(group(name), n, seed * 1000 + k)
        items = []
        proc = P.Proc(KIND(name), rd.dgst, rd.t, rd.ids)

        def call(its):
            res = [P.step(proc, op, d, p) for op, d, p in its]
            items.extend(its)
            if its[-1][0] == RESPONSE and rng.random() < 0.3:              # a truncated answer: MALFORMED, the node joins
                items.append((RESPONSE, its[-1][1][:rng.randrange(1, 8)], 999))
            return res
        rd.run(call)
        items += [(RESPONSE, b"", 5), (REQUEST, b"", 0)]
        replay = P.Proc(KIND(name), rd.dgst, rd.t, rd.ids)                 # the malformed answers change the node lists only
        want = [P.step(replay, op, d, p) for op, d, p in items]
        out.append((KIND(name), (rd.dgst, rd.t, rd.ids), items, want))
    return out


@pytest.mark.parametrize("split", ["one", "several", "each"])
def test_sequential_equivalence(engine, split):
    scripts = _scripts(16, 0xD5D0)
    rng = random.Random(0xD5D1)
    queue = [(p, j) for p, s in enumerate(scripts) for j in range(len(s[2]))]
    order, heads = [], [0] * len(scripts)                                   # a random interleaving keeping each process's order
    while len(order) < len(queue):
        p = rng.choice([q for q in range(len(scripts)) if heads[q] < len(scripts[q][2])])
        order.append((p, heads[p]))
        heads[p] += 1
    hs = [engine.thdsa_proc_create(ALGO[k], *args) for k, args, _, _ in scripts]
    flat = [(p, scripts[p][2][j][0], scripts[p][2][j][1], scripts[p][2][j][2]) for p, j in order]
    cuts = {"one": [0, len(flat)], "several": sorted({0, len(flat)} | set(rng.sample(range(1, len(flat)), 6))),
            "each": list(range(len(flat) + 1))}[split]
    got = []
    for a, b in zip(cuts, cuts[1:]):
        got += device_run(engine, hs, flat[a:b])
    for (p, j), g in zip(order, got):
        assert g == scripts[p][3][j], (p, j)
    for h in hs:
        engine.thdsa_proc_destroy(h)


def test_quirks(engine):
    from oracle import sss_oracle as S
    d = hashlib.sha256(b"q").digest()
    # phase-0 th from the last-listed id
    both(engine, "dsa", d, 1, [1], [(RESPONSE, P.joint_share_response([(b"a", 9), (b"b", 8)]), 1),
                                    (RESPONSE, P.joint_share_response([(b"c", 8), (b"d", 9)]), 2), (REQUEST, b"", 0)])
    both(engine, "dsa", d, 1, [], [(RESPONSE, struct.pack(">H", 0), 3), (RESPONSE, P.joint_share_response([(b"", 7)]), 4),
                                   (RESPONSE, P.joint_share_response([(b"x", 7)]), 4), (REQUEST, b"", 0)])
    p0 = [(RESPONSE, P.joint_share_response([(b"s", 1)]), 1), (RESPONSE, P.joint_share_response([(b"s", 1)]), 2)]
    gk = group("1024/160")
    q = gk["q"]
    Rs = [O.bts(pow(gk["g"], a, gk["p"])) for a in (3, 5, 7, 11)]
    # duplicate x in phase 1 and phase 2; R_i >= p, longer than p, empty; v_i and s_i >= q in long chunks
    for p1 in ([partial(gk, 1, Rs[0], 4), partial(gk, 1, Rs[1], 6)],
               [partial(gk, 1, (int.from_bytes(Rs[0], "big") + gk["p"]).to_bytes(200, "big"), (5 + 3 * q).to_bytes(90, "big")),
                partial(gk, 2, b"", 7)],
               [partial(gk, 2, Rs[2], 0), partial(gk, 3, Rs[3], 0)]):                       # v = 0: r = 1
        p2 = [partial(gk, 1, O.bts(10 + q), 0), partial(gk, 1, (3 * q + 4).to_bytes(70, "big"), 0)]
        both(engine, "dsa", d, 1, [], p0 + [(REQUEST, b"", 0)] + [(RESPONSE, a, 5 + k) for k, a in enumerate(p1)] +
             [(REQUEST, b"", 0)] + [(RESPONSE, a, 7 + k) for k, a in enumerate(p2)] + [(RESPONSE, b"", 9), (REQUEST, b"", 0)])
    # a composite odd q: gcd(v, q) = 3 (v = 2*3 - 9 = -3) gives r = r'^v; gcd(v, q) = 1 (v = 2*3 - 4 = 2) gives r = r'^(v^-1),
    # where Fermat's v^(q-2) is not the inverse.  The REQUEST that follows shows r; Fermat's exponent would give another r.
    gc = dict(kind="dsa", p=gk["p"], q=3 * 5 * 7 * 11 * 13 * 1000003 * (2 ** 61 - 1), g=gk["g"])
    qc = gc["q"]
    lam = [P.lagrange(x, [1, 2], qc) for x in (1, 2)]
    rp = pow(int.from_bytes(Rs[0], "big"), lam[0], gk["p"]) * pow(int.from_bytes(Rs[1], "big"), lam[1], gk["p"]) % gk["p"]
    for v2, want_e in ((9, lambda v: v), (4, lambda v: pow(v, -1, qc))):
        v = (3 * lam[0] + v2 * lam[1]) % qc
        assert v != 0 and pow(rp, want_e(v), gk["p"]) % qc != pow(rp, pow(v, qc - 2, qc), gk["p"]) % qc
        res = both(engine, "dsa", d, 1, [], p0 + [(RESPONSE, partial(gc, 1, Rs[0], 3), 5), (RESPONSE, partial(gc, 2, Rs[1], v2), 6),
                                                  (REQUEST, b"", 0)])
        assert res[3][0] == P.CONTINUE and res[4][2].endswith(O.chunk(O.bts(pow(rp, want_e(v), gk["p"]) % qc)))
    # ECDSA: v = 0, and a sum at infinity with v = 2 - 1 = 1, give r = 0; duplicate x doubles
    gp = group("p256")
    pt = lambda k: S.p256_marshal(S.p256_mul(k, S.P256_G))
    for p1 in ([partial(gp, 1, pt(5), 0), partial(gp, 2, pt(7), 0)], [partial(gp, 1, pt(5), 1), partial(gp, 2, pt(10), 1)],
               [partial(gp, 4, pt(5), 1), partial(gp, 4, pt(5), 2)]):
        both(engine, "p256", d, 1, [], p0 + [(RESPONSE, a, 5 + k) for k, a in enumerate(p1)] + [(REQUEST, b"", 0)] +
             [(RESPONSE, partial(gp, 1, O.bts(5), 0), 8), (RESPONSE, partial(gp, 2, O.bts(6), 0), 9)])
    # a phase-2 group that differs from phase 1's: a 160-bit r fits 2048/256's q; a 256-bit r overflows 1024/160's (Go panics)
    g2 = group("2048/256")
    for ga, gb in ((gk, g2), (g2, gk)):
        Ra = [O.bts(pow(ga["g"], a, ga["p"])) for a in (3, 5)]
        both(engine, "dsa", d, 1, [], p0 + [(RESPONSE, partial(ga, 1, Ra[0], 4), 5), (RESPONSE, partial(ga, 2, Ra[1], 9), 6),
                                            (REQUEST, b"", 0), (RESPONSE, partial(gb, 1, O.bts(5), 0), 7),
                                            (RESPONSE, partial(gb, 2, O.bts(8), 0), 8), (RESPONSE, b"", 9), (REQUEST, b"", 0)])


def test_failures(engine):
    from oracle import sss_oracle as S
    d = hashlib.sha256(b"f").digest()
    gk, gp = group("1024/160"), group("p256")
    p0 = [(RESPONSE, P.joint_share_response([(b"s", 1)]), 1), (RESPONSE, P.joint_share_response([(b"s", 1)]), 2)]
    good = [partial(gk, 1, b"\x05", 4), partial(gk, 2, b"\x07", 6)]
    # every truncation point of one answer of each phase: MALFORMED, the peer joins the node list
    for ph, ans in ((0, P.joint_share_response([(b"abc", 1), (b"de", 2)])), (1, good[0]), (2, partial(gk, 1, O.bts(5), 0))):
        pre = [] if ph == 0 else p0 + good[:0]
        if ph == 2:
            pre = p0 + [(RESPONSE, a, 5 + k) for k, a in enumerate(good)]
        cut = [(RESPONSE, ans[:c], 100 + c) for c in range(len(ans))]
        both(engine, "dsa", d, 1, [], pre + cut + [(REQUEST, b"", 0)])
    # Go's panics: an R_i Unmarshal rejects, a Lagrange denominator with no inverse, a short digest, formatDSA's overflow;
    # the process stays failed
    after = [(REQUEST, b"", 0), (RESPONSE, b"", 9)]
    bad_pt = b"\x04" + bytes(64)
    both(engine, "p256", d, 1, [], p0 + [(RESPONSE, partial(gp, 1, S.p256_marshal(S.P256_G), 1), 5), (RESPONSE, partial(gp, 2, bad_pt, 1), 6)] + after)
    gc = dict(kind="dsa", p=gk["p"], q=3 * (2 ** 61 - 1), g=gk["g"])
    both(engine, "dsa", d, 1, [], p0 + [(RESPONSE, partial(gc, 1, b"\x05", 1), 5), (RESPONSE, partial(gc, 4, b"\x07", 1), 6)] + after)
    both(engine, "dsa", d[:10], 1, [], p0 + [(RESPONSE, a, 5) for a in good] + after)
    g2 = group("2048/256")
    both(engine, "dsa", d, 1, [], p0 + [(RESPONSE, partial(g2, 1, b"\x05", 4), 5), (RESPONSE, partial(g2, 2, b"\x07", 6), 6),
                                        (REQUEST, b"", 0), (RESPONSE, partial(gk, 1, b"\x01", 0), 7), (RESPONSE, partial(gk, 2, b"\x02", 0), 8)] + after)
    # unsupported: a completing answer's group (p of 1536 bits), an x outside int32: the item changes nothing
    g1536 = dict(kind="dsa", p=(1 << 1535) + 1, q=gk["q"], g=2)
    for bad in (partial(g1536, 2, b"\x07", 6), partial(gk, 1 << 40, b"\x07", 6), partial(gk, -(1 << 33), b"\x07", 6)):
        h = engine.thdsa_proc_create(2, d, 1, [])
        proc = P.Proc("dsa", d, 1, [])
        items = p0 + [(RESPONSE, good[0], 5)]
        assert device_call(engine, h)(items) == [P.step(proc, op, x, p) for op, x, p in items]
        assert device_call(engine, h)([(RESPONSE, bad, 6)]) == [(P.FAILED, -4, b"")]
        rest = [(RESPONSE, good[1], 6), (REQUEST, b"", 0)]
        assert device_call(engine, h)(rest) == [P.step(proc, op, x, p) for op, x, p in rest]
        engine.thdsa_proc_destroy(h)
    # 2t > 255 at create
    with pytest.raises(_lib.BftqError) as ei:
        engine.thdsa_proc_create(2, d, 128, [])
    assert ei.value.code == -4
    # out_cap below out_need: INVALID_ARG before any work, out_need set, nothing changed
    import ctypes as C
    import numpy as np
    h = engine.thdsa_proc_create(2, d, 1, [11, 12])
    lib = _lib.load()
    tab = (C.c_void_p * 1)(h.value)
    z32, z64 = np.zeros(1, np.uint32), np.zeros(2, np.uint64)
    op = np.array([-1], np.int32)
    need = C.c_uint64(0)
    st, er, out = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(8, np.uint8)
    rc = lib.bftq_thdsa_process_batch(engine._h, tab, 1, z32.ctypes.data, op.ctypes.data, z64.ctypes.data, out.ctypes.data, z64.ctypes.data, 1,
                                      st.ctypes.data, er.ctypes.data, out.ctypes.data, 8, z64.ctypes.data, C.byref(need))
    assert rc == -3 and need.value > 8
    assert device_call(engine, h)([(REQUEST, b"", 0)]) == [(P.PENDING, 0, struct.pack(">IQQ", 2, 11, 12))]
    engine.thdsa_proc_destroy(h)


def test_threads_lifecycle_and_launches(engine):
    out = [None] * 8

    def work(i):
        name = ["1024/160", "p256"][i % 2]
        rd = Round(group(name), 4, 0xD5E0 + i)
        h = engine.thdsa_proc_create(ALGO[KIND(name)], rd.dgst, rd.t, rd.ids)
        out[i] = (rd.run(device_call(engine, h))[0], rd)
        engine.thdsa_proc_destroy(h)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    [x.start() for x in ts]
    [x.join() for x in ts]
    for i, (sig, rd) in enumerate(out):
        _verify(rd.g, rd.x, rd.dgst, sig)
    # a process destroyed mid-phase
    rd = Round(group("p256"), 4, 0xD5E9)
    h = engine.thdsa_proc_create(3, rd.dgst, rd.t, rd.ids)
    device_call(engine, h)([(RESPONSE, rd.phase0(j), rd.ids[j]) for j in range(3)])
    engine.thdsa_proc_destroy(h)
    # launches: a DSA CalculateR is 7 kernels, an ECDSA one 5, a calculateS 1.  Every one goes through launch() (no other
    # `<<<`: test_launch_accounting.py), and test_quirks' composite q tells thdsa_go_inverse_kernel's result from Fermat's
    for name, want in (("1024/160", 7), ("p256", 5)):
        rd = Round(group(name), 4, 0xD5EA)
        h = engine.thdsa_proc_create(ALGO[KIND(name)], rd.dgst, rd.t, rd.ids)
        call = device_call(engine, h)
        call([(RESPONSE, rd.phase0(j), rd.ids[j]) for j in range(4)])
        _, req1 = split_request(call([(REQUEST, b"", 0)])[0][2])
        answers = [(RESPONSE, rd.phase1(i, req1), rd.ids[i]) for i in range(4)]
        call(answers[:3])
        before = engine.stats()["launches"]
        assert call(answers[3:])[0][0] == P.CONTINUE
        assert engine.stats()["launches"] - before == want
        _, req2 = split_request(call([(REQUEST, b"", 0)])[0][2])
        call([(RESPONSE, rd.phase2(i, req2), rd.ids[i]) for i in range(3)])
        before = engine.stats()["launches"]
        assert call([(RESPONSE, rd.phase2(3, req2), rd.ids[3])])[0][0] == P.SIGNED
        assert engine.stats()["launches"] - before == 1
        engine.thdsa_proc_destroy(h)
