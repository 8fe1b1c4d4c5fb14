"""CPU suite: the threshold-RSA oracle (tests/threshold_rsa_oracle.py) pinned by the reference's own tests restated —
TestDistribution's checkSum at n = 10, k = 7 and TestCombine's signature of "tbs" under the fixture key — and K7's SASS."""
import hashlib
import json
import os
import subprocess

import threshold_rsa_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = json.load(open(os.path.join(ROOT, "tests", "golden", "thrsa_key.json")))
N, D = int(KEY["n"], 16), int(KEY["d"], 16)


def check_sum(kmap, idx, d, n):                           # rsa_test.go:114-129
    s = 0
    for i, m in enumerate(kmap):
        if idx in m:
            if not check_sum(kmap, (idx * n + i + 1) & O.M32, m[idx], n):
                return False
            s += m[idx]
    return s == 0 or s == d


def test_key_fixture_matches_kat(golden):
    assert int(golden["ref_rsa_kat"]["n"], 16) == N == int(KEY["p"], 16) * int(KEY["q"], 16)
    assert pow(pow(12345, KEY["e"], N), D, N) == 12345


def test_distribution_checksum():
    shares = O.distribute(D, N, 10, 7, seed=7)
    kmap = [O.parse_partial_param(s)[0] for s in shares]
    assert check_sum(kmap, 0, D, 10)
    # fragment lengths double per level: the fragments of key 0 about 4 100 bits, those of depth-3 keys about 32 800
    bits = {}
    for m in kmap:
        for i, v in m.items():
            bits[O.depth(i, 10)] = max(bits.get(O.depth(i, 10), 0), abs(v).bit_length())
    assert 4000 < bits[0] <= 4100 and 32000 < bits[3] <= 32800


def run_round(shares, n, k, active, hinfo, order_seed=0):
    import random
    responses = []
    req = O.serialize_sign_request([0], hinfo)
    rounds = 0
    while req is not None:
        rounds += 1
        order = list(active)
        random.Random(order_seed + rounds).shuffle(order)
        for j in order:
            out, err = O.sign(shares[j], req)
            assert err is None
            if out is not None:
                responses.append(out)
        st, at, sig, missing = O.process(n, k, responses)
        if st == O.SIGNED:
            return sig, rounds, responses[:at + 1]
        req = O.make_request(n, k, responses, hinfo)
    return None, rounds, responses


def test_combine_full_round(golden):
    shares = O.distribute(D, N, 10, 7, seed=3)
    sig, rounds, _ = run_round(shares, 10, 7, range(10), O.hash_info_sha256(b"tbs"))
    assert rounds == 1 and sig.hex() == golden["ref_rsa_kat"]["sig"]


def test_combine_three_silent_servers(golden):
    shares = O.distribute(D, N, 10, 7, seed=4)
    sig, rounds, responses = run_round(shares, 10, 7, [0, 1, 2, 4, 5, 7, 9], O.hash_info_sha256(b"tbs"))
    assert sig is not None and sig.hex() == golden["ref_rsa_kat"]["sig"]
    assert rounds == 4                                    # depth-2, -3 and -4 fragments come with later requests
    depths = {O.depth(i, 10) for r in responses for i, _ in O.parse_partial_signature(r)[0]}
    assert depths == {1, 2, 3, 4}


def test_sign_neg_quirk_and_unknown_ids():
    shares = O.distribute(D, N, 10, 7, seed=5)
    keys, _, pid, n = O.parse_partial_param(shares[2])
    neg = [i for i, v in keys.items() if v < 0]
    assert neg, "seed gives a negative fragment"
    kid = neg[0]
    h = O.hash_info_sha256(b"x")
    m = O.emsa_encode(O.SHA256_PREFIX, hashlib.sha256(b"x").digest(), N)
    once, _ = O.sign(shares[2], O.serialize_sign_request([kid], h))
    twice, _ = O.sign(shares[2], O.serialize_sign_request([kid, kid], h))
    v1 = O.parse_partial_signature(once)[0][0][1]
    v2 = O.parse_partial_signature(twice)[0][0][1]
    assert v1 * v2 % N == 1 and v2 == pow(m, -keys[kid], N)
    assert O.sign(shares[2], O.serialize_sign_request([0xFFFF0000], h)) == (None, None)


def test_k7_uses_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    bodies = [b for b in sass.split("Function :")[1:] if "thrsa_partial_sign_kernel" in b.split("\n", 1)[0]]
    assert bodies
    for b in bodies:
        assert "LDL" not in b and "STL" not in b, "thrsa_partial_sign_kernel spills to local memory"
    usage = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout.split("\n")
    hits = [i for i, line in enumerate(usage) if "thrsa_partial_sign_kernel" in line]
    assert hits
    for i in hits:
        assert "STACK:0 " in usage[i + 1] and "LOCAL:0 " in usage[i + 1], usage[i + 1]
