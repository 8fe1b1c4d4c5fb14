"""GPU suite: bftq_thrsa_sign_batch (K7) and bftq_thrsa_process_batch against the threshold-RSA oracle
(tests/threshold_rsa_oracle.py), end to end to the reference's TestCombine signature, checked by K1."""
import hashlib
import json
import os
import random
import struct
import threading

import numpy as np
import pytest

import threshold_rsa_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = json.load(open(os.path.join(ROOT, "tests", "golden", "thrsa_key.json")))
N, D = int(KEY["n"], 16), int(KEY["d"], 16)
ERR = {None: 0, "malformed": -8, "invalid_input": -13}
pytestmark = pytest.mark.gpu


def raw_share(frags, n_mod, pid, n):
    """frags: (idx, sign byte, magnitude bytes) exactly as stored"""
    out = struct.pack(">H", len(frags))
    for idx, sign, mag in frags:
        out += struct.pack(">IB", idx, sign) + O.chunk(mag)
    return out + O.chunk(O.int_bytes(n_mod)) + struct.pack(">IB", pid, n)


def check_sign(engine, shares, share_idx, reqs):
    handles = [engine.thrsa_share_create(s) for s in shares]
    try:
        err, outs = engine.thrsa_sign_batch(handles, share_idx, reqs)
    finally:
        for h in handles:
            engine.thrsa_share_destroy(h)
    for i, (s, r) in enumerate(zip(share_idx, reqs)):
        want, werr = O.sign(shares[s], r)
        assert err[i] == ERR[werr], (i, err[i], werr)
        assert outs[i] == (want or b""), i
    return outs


def test_sign_depths_signs_and_edges(engine, golden):
    rng = random.Random(11)
    n2 = int(golden["keys"]["a01"]["n"], 16)                                   # a second RSA-2048 modulus
    frags = []
    for idx, bits in enumerate([4100, 8200, 16400, 32800, 4096, 65536]):        # depths 1-4 and the 8 KB cap
        for sign in (0, 1):
            frags.append((100 * idx + sign, sign, O.int_bytes(rng.getrandbits(bits) | (1 << (bits - 1)))))
    frags += [(900, 0, b""), (901, 1, b""), (902, 0, b"\x00\x00\x05"), (903, 1, b"\x00" * 7 + b"\x09")]  # zero, -0, stored zeros
    share_a = raw_share(frags, N, 3, 10)
    share_b = raw_share(frags[::3], n2, 7, 10)
    h = O.hash_info_sha256(b"tbs")
    ids = [f[0] for f in frags]
    reqs, idx = [], []
    for s in (0, 1):
        for kid in ids:
            reqs.append(O.serialize_sign_request([kid], h)); idx.append(s)
    neg = [f[0] for f in frags if f[1] == 1]
    reqs += [O.serialize_sign_request(ids + [5, 77777], h),                  # every fragment + unknown ids
             O.serialize_sign_request([neg[0], 5, neg[0]], h),               # duplicated negative: the in-place Neg
             O.serialize_sign_request([neg[1], neg[1], neg[1]], h),
             O.serialize_sign_request([5, 6, 0xFFFFFFFF], h),                # none known: (nil, nil)
             O.serialize_sign_request([], h),
             O.serialize_sign_request([0], O.serialize_hash_info(b"\x01" * 200, b"\x02" * 53)),   # padlen 3
             O.serialize_sign_request([0], O.serialize_hash_info(b"\x01" * 200, b"\x02" * 54)),   # padlen 2
             O.serialize_sign_request([0], O.serialize_hash_info(b"", b"\x02" * 300))]
    full = O.serialize_sign_request([0, 1], h)
    reqs += [full[:c] for c in (0, 1, 2, 5, 9, 11, 20, len(full) - 1)]          # truncated requests
    reqs += [full[:10] + struct.pack(">Q", 1 << 40) + full[18:]]
    idx += [0] * (len(reqs) - len(idx))
    reqs += [O.serialize_sign_request(ids, h)]; idx += [1]
    outs = check_sign(engine, [share_a, share_b], idx, reqs)
    assert outs[-1] and any(o == b"" for o in outs)


def test_share_errors(engine):
    good = raw_share([(0, 0, b"\x05" * 10)], N, 1, 10)
    for cut in (0, 1, 5, 7, 20, len(good) - 1):
        with pytest.raises(Exception) as ei:
            engine.thrsa_share_create(good[:cut])
        assert ei.value.code == -8
    rng = random.Random(2)
    n3072 = rng.getrandbits(3072) | (1 << 3071) | 1
    for bad in (raw_share([(0, 0, b"\x05")], n3072, 1, 10), raw_share([(0, 0, b"\x05")], N - 1, 1, 10),
                raw_share([(0, 0, b"\x01" * 8193)], N, 1, 10)):
        with pytest.raises(Exception) as ei:
            engine.thrsa_share_create(bad)
        assert ei.value.code == -4


def gpu_round(engine, shares, active, hinfo, n=10, k=7, seed=0):
    """MakeRequest / Sign on the device / ProcessResponse on the device, until signed."""
    handles = [engine.thrsa_share_create(s) for s in shares]
    try:
        responses, req, rounds = [], O.serialize_sign_request([0], hinfo), 0
        while req is not None:
            rounds += 1
            order = list(active)
            random.Random(seed + rounds).shuffle(order)
            err, outs = engine.thrsa_sign_batch(handles, order, [req] * len(order))
            assert not err.any()
            responses += [o for o in outs if o]
            st, e, at, sig, missing = engine.thrsa_process_batch(n, k, [responses])[0]
            ost, oat, osig, omissing = O.process(n, k, responses)
            assert (at, sig, missing) == (oat, osig, omissing)
            if st == 1:
                return sig, rounds
            req = O.serialize_sign_request(missing, hinfo) if missing else None
        return None, rounds
    finally:
        for h in handles:
            engine.thrsa_share_destroy(h)


def test_end_to_end_combine_and_verify(engine, golden):
    kat = golden["ref_rsa_kat"]
    h = O.hash_info_sha256(b"tbs")
    sig1, r1 = gpu_round(engine, O.distribute(D, N, 10, 7, seed=21), range(10), h)
    sig2, r2 = gpu_round(engine, O.distribute(D, N, 10, 7, seed=22), [0, 2, 3, 4, 6, 8, 9], h, seed=5)
    assert r1 == 1 and r2 == 4
    assert sig1.hex() == kat["sig"] and sig2.hex() == kat["sig"]
    idx = engine.register_rsa_keys([N], [KEY["e"]])
    st = engine.rsa_verify_batch(np.array([idx, idx], np.uint32), np.frombuffer(sig1 + sig2, np.uint8).reshape(2, 256),
                                 np.frombuffer(hashlib.sha256(b"tbs").digest() * 2, np.uint8).reshape(2, 32))
    assert list(st) == [0, 0]


def test_process_orders_duplicates_errors_missing(engine):
    shares = O.distribute(D, N, 10, 7, seed=31)
    h = O.hash_info_sha256(b"abc")
    req = O.serialize_sign_request([0], h)
    resp = [O.sign(s, req)[0] for s in shares]
    rng = random.Random(9)
    procs = []
    for t in range(12):
        r = list(resp)
        rng.shuffle(r)
        procs.append(r)
    procs.append(resp[:5] + resp[:5] + resp[5:])                       # duplicates
    procs.append(resp[:4] + [resp[4][:-3]] + resp[4:])                 # malformed before completion: error
    procs.append(resp + [resp[0][:7], b""])                            # malformed after completion: never read
    procs.append(resp[:3] + [resp[3]] * 4)                             # incomplete: missing keys
    procs.append([resp[1], resp[3], resp[8]])
    procs.append([])
    got = engine.thrsa_process_batch(10, 7, procs)
    for p, (st, err, at, sig, missing) in zip(procs, got):
        ost, oat, osig, omissing = O.process(10, 7, p)
        assert {O.SIGNED: 1, O.FAILED: 2, O.INCOMPLETE: 0}[ost] == st and at == oat and sig == osig and missing == omissing
        assert err == (-8 if ost == O.FAILED else 0)


def test_threads_give_the_same_bytes(engine):
    shares = O.distribute(D, N, 10, 7, seed=41)
    handles = [engine.thrsa_share_create(s) for s in shares]
    reqs = [O.serialize_sign_request([0], O.hash_info_sha256(b"m%d" % i)) for i in range(64)]
    idx = [i % 10 for i in range(64)]
    want = engine.thrsa_sign_batch(handles, idx, reqs)[1]
    got, errs = [None] * 8, []

    def run(t):
        try:
            got[t] = engine.thrsa_sign_batch(handles, idx, reqs)[1]
        except Exception as ex:           # noqa: BLE001 - reported below
            errs.append(ex)
    ts = [threading.Thread(target=run, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for h in handles:
        engine.thrsa_share_destroy(h)
    assert not errs and all(g == want for g in got)
    assert want[0] == O.sign(shares[0], reqs[0])[0]


def test_destroy_frees_device_memory(engine):
    import torch
    share = raw_share([(i, i & 1, b"\x7f" * 8192) for i in range(4096)], N, 0, 10)      # 32 MB of fragments
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    h = engine.thrsa_share_create(share)
    free1 = torch.cuda.mem_get_info()[0]
    engine.thrsa_share_destroy(h)
    free2 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 >= 32 << 20 and free2 - free1 >= 32 << 20
