"""GPU parity suite for K1 (RSA PKCS#1 v1.5 batch verify) through the C ABI.
Bar: status bytes bit-identical to the oracle (oracle/c/bftq_oracle.c, pinned by
tests/test_oracle_golden.py) on the same seeded inputs."""
import hashlib
import os
import threading

import numpy as np
import pytest

from bftkv_b200 import Engine, workload
from bftkv_b200.engine import F_STRICT_RANGE
from oracle import c_oracle, pgp_oracle as pgp

pytestmark = pytest.mark.gpu
NCPU = os.cpu_count() or 1


@pytest.fixture(scope="module")
def batch64k():
    return workload.make_verify_batch(65536, n_keys=16)      # BASELINE config 2


def _engine_with(keys):
    e = Engine(0)
    e.register_rsa_keys([k["n"] for k in keys], [k["e"] for k in keys])
    return e


def test_config2_full_batch_bit_exact(batch64k, built):
    w = batch64k
    ns, es = [k["n"] for k in w["keys"]], [k["e"] for k in w["keys"]]
    ref = c_oracle.rsa_verify_batch(ns, es, w["key_idx"], w["sig"], w["digest"], threads=NCPU)
    assert np.array_equal(ref, w["expect"])
    e = _engine_with(w["keys"])
    got = e.rsa_verify_batch(w["key_idx"], w["sig"], w["digest"])
    assert np.array_equal(got, ref)
    assert (got == 0).sum() > 60000 and (got == 1).sum() > 300 and (got == 4).sum() > 20
    assert e.stats()["launches"] >= 1 and e.stats()["items"] == 65536
    e.close()


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 31, 33, 255, 1000])
def test_ragged_sizes(batch64k, engine_cfg2, n):
    w = batch64k
    got = engine_cfg2.rsa_verify_batch(w["key_idx"][:n].copy(), w["sig"][:n].copy(), w["digest"][:n].copy())
    assert np.array_equal(got, w["expect"][:n])


@pytest.fixture(scope="module")
def engine_cfg2(batch64k, built):
    e = _engine_with(batch64k["keys"])
    yield e
    e.close()


def test_empty_batch(engine_cfg2):
    out = engine_cfg2.rsa_verify_batch(np.zeros(0, np.uint32), np.zeros((0, 256), np.uint8), np.zeros((0, 32), np.uint8))
    assert out.shape == (0,)


def test_edge_values(batch64k, engine_cfg2):
    """s = 0, 1, n-1, n, n+s (Go 1.13 accepts s+n: big.Int.Exp reduces; strict mode rejects),
    all-ones, valid EM for a different digest."""
    w = batch64k
    keys = w["keys"]
    i = int(np.nonzero(w["expect"] == 0)[0][0])
    k = int(w["key_idx"][i])
    n = keys[k]["n"]
    s = int.from_bytes(w["sig"][i].tobytes(), "big")
    dig = w["digest"][i].tobytes()
    vals = [0, 1, n - 1, n, s, 2 ** 2048 - 1, (s * s) % n]
    if s + n < 2 ** 2048:
        vals.append(s + n)
    sig = np.frombuffer(b"".join(v.to_bytes(256, "big") for v in vals), np.uint8).reshape(-1, 256).copy()
    digs = np.frombuffer(dig * len(vals), np.uint8).reshape(-1, 32).copy()
    kidx = np.full(len(vals), k, np.uint32)
    ns, es = [x["n"] for x in keys], [x["e"] for x in keys]
    for strict in (False, True):
        ref = c_oracle.rsa_verify_batch(ns, es, kidx, sig, digs, strict_range=strict)
        got = engine_cfg2.rsa_verify_batch(kidx, sig, digs, flags=F_STRICT_RANGE if strict else 0)
        assert np.array_equal(got, ref), (strict, got, ref)
        assert got[4] == 0
        if s + n < 2 ** 2048:
            assert got[-1] == (1 if strict else 0)
    # python big-int cross-check of the non-strict answers
    for v, g in zip(vals, engine_cfg2.rsa_verify_batch(kidx, sig, digs)):
        assert (pow(v, 65537, n) == workload.em_for_digest(dig)) == (g == 0)


def test_other_exponents_and_key_sizes(built):
    """e = 3, 17, 257, 65537 and an even e mixed in one warp; 2047- and 2041-bit moduli (k is
    still 256).  Keys are built from the fixture primes; signatures with Python pow()."""
    import math
    from cryptography.hazmat.primitives.asymmetric import rsa
    fix = workload.load_keys(8)
    keys = []
    for e, f in zip((3, 17, 257, 65537, 5, 11), fix):
        phi = (f["p"] - 1) * (f["q"] - 1)
        while math.gcd(e, phi) != 1:
            e += 2
        keys.append({"n": f["n"], "e": e, "d": pow(e, -1, phi)})
    for bits in (2047, 2041):
        pn = rsa.generate_private_key(65537, bits).private_numbers()
        keys.append({"n": pn.public_numbers.n, "e": 65537, "d": pn.d})
    assert keys[-1]["n"].bit_length() == 2041
    ns, es = [k["n"] for k in keys], [k["e"] for k in keys]
    rng = np.random.default_rng(11)
    N = 300
    kidx = rng.integers(0, len(keys), N).astype(np.uint32)
    dig = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    sig = np.empty((N, 256), np.uint8)
    for i in range(N):
        k = keys[kidx[i]]
        s = pow(workload.em_for_digest(dig[i].tobytes()), k["d"], k["n"])
        sig[i] = np.frombuffer(s.to_bytes(256, "big"), np.uint8)
    flip = rng.random(N) < 0.3
    for i in np.nonzero(flip)[0]:
        sig[i, int(rng.integers(1, 256))] ^= 0x40
    ref = c_oracle.rsa_verify_batch(ns, es, kidx, sig, dig, threads=NCPU)
    assert set(ref[~flip]) == {0} and set(ref[flip]) == {1}
    e = _engine_with(keys)
    assert np.array_equal(e.rsa_verify_batch(kidx, sig, dig), ref)
    e.close()
    # an even public exponent cannot come from a valid key, but x/crypto parses it and
    # big.Int.Exp computes it: the decision must still equal s^e mod n == EM.
    keys2 = [{"n": fix[0]["n"], "e": 65536}, {"n": fix[1]["n"], "e": 2}, {"n": fix[2]["n"], "e": 1}]
    kidx2 = np.array([0, 1, 2, 2], np.uint32)
    em = workload.em_for_digest(dig[0].tobytes())
    sig2 = np.frombuffer(b"".join(v.to_bytes(256, "big") for v in (12345, 7, em, em + 1)), np.uint8).reshape(-1, 256).copy()
    dig2 = np.repeat(dig[:1], 4, axis=0).copy()
    ref2 = c_oracle.rsa_verify_batch([k["n"] for k in keys2], [k["e"] for k in keys2], kidx2, sig2, dig2)
    assert ref2.tolist() == [1, 1, 0, 1]
    e = _engine_with(keys2)
    assert np.array_equal(e.rsa_verify_batch(kidx2, sig2, dig2), ref2)
    e.close()


def test_gpg_golden_signatures(golden, built):
    """GnuPG-made detached signatures (SHA-256/SHA-512/SHA-1, binary and text mode) through K1:
    the packer side (packet parse + v4 digest) comes from the oracle here; the accept/reject
    decision from the GPU."""
    ring = []
    for name in ["a01", "a02", "a03", "a04", "u01"]:
        ring += pgp.read_entities(bytes.fromhex(golden["keys"][name]["pub"]))
    e = Engine(0)
    e.register_rsa_keys([x.primary_key.n for x in ring], [x.primary_key.e for x in ring])
    ids = [x.primary_key.key_id for x in ring]
    by_hash = {}
    for c in golden["cases"]:
        if c["signer"] == "x99":
            continue
        tbs = bytes.fromhex(c["tbs"])
        tag, body = pgp.read_packet(pgp.Reader(bytes.fromhex(c["sig"])))
        s = pgp.parse_signature(body)
        for tamper in (False, True):
            d = pgp.signature_digest(tbs + (b"!" if tamper else b""), s)
            by_hash.setdefault(s.hash_id, []).append((ids.index(s.issuer_key_id), s.rsa_sig_bytes.rjust(256, b"\0"), d, tamper))
    assert set(by_hash) == {2, 8, 10}
    for hid, items in by_hash.items():
        kidx = np.array([i[0] for i in items], np.uint32)
        sig = np.frombuffer(b"".join(i[1] for i in items), np.uint8).reshape(-1, 256).copy()
        dig = np.frombuffer(b"".join(i[2] for i in items), np.uint8).reshape(len(items), -1).copy()
        got = e.rsa_verify_batch(kidx, sig, dig, hash_alg=hid)
        assert got.tolist() == [1 if i[3] else 0 for i in items], hid
    k = golden["ref_rsa_kat"]                                   # reference-owned key, rsa_test.go:165-206
    first = e.register_rsa_keys([int(k["n"], 16)], [k["e"]])
    got = e.rsa_verify_batch(np.array([first], np.uint32), np.frombuffer(bytes.fromhex(k["sig"]), np.uint8).reshape(1, 256).copy(),
                             np.frombuffer(bytes.fromhex(k["digest"]), np.uint8).reshape(1, 32).copy())
    assert got.tolist() == [0]
    e.close()


def test_device_resident_api_and_concurrency(batch64k, engine_cfg2):
    import torch
    w = batch64k
    n = 8192
    dev = torch.device("cuda:0")
    d_idx = torch.from_numpy(w["key_idx"][:n].astype(np.int32)).to(dev)
    d_sig = torch.from_numpy(w["sig"][:n]).to(dev)
    d_dig = torch.from_numpy(w["digest"][:n]).to(dev)
    d_st = torch.full((n,), 255, dtype=torch.uint8, device=dev)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        engine_cfg2.rsa_verify_batch_dev(d_idx, d_sig, d_dig, n, d_st, stream=st.cuda_stream)
    st.synchronize()
    assert np.array_equal(d_st.cpu().numpy(), w["expect"][:n])
    # re-entrancy: four host threads share one engine (transport/transport.go:110-127 pattern)
    outs = [None] * 4

    def run(j):
        lo = j * 4096
        outs[j] = engine_cfg2.rsa_verify_batch(w["key_idx"][lo:lo + 4096].copy(), w["sig"][lo:lo + 4096].copy(), w["digest"][lo:lo + 4096].copy())
    ths = [threading.Thread(target=run, args=(j,)) for j in range(4)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    for j in range(4):
        assert np.array_equal(outs[j], w["expect"][j * 4096:(j + 1) * 4096])


def test_roundtrip_property_fresh_keys(built):
    """Size-independent property: sign -> verify accepts, any single bit flip in s rejects."""
    w = workload.make_verify_batch(4096, n_keys=31, seed=99, corrupt_rate=0.5, unknown_rate=0.0, corrupt_seed=7)
    e = _engine_with(w["keys"])
    got = e.rsa_verify_batch(w["key_idx"], w["sig"], w["digest"])
    assert np.array_equal(got, w["expect"]) and 1500 < int(got.sum()) < 2600
    e.close()


def test_r32_kernel_bit_exact(batch64k, built):
    """The radix-2^32 kernel (squarings through mont_sqr, rsa_square_r32.cuh, emulated limb for limb by tools/emu_sq.py)
    against the oracle on config 2, ragged sizes and the edge values of s."""
    w = batch64k
    ns, es = [k["n"] for k in w["keys"]], [k["e"] for k in w["keys"]]
    e = _engine_with(w["keys"])
    ref = c_oracle.rsa_verify_batch(ns, es, w["key_idx"], w["sig"], w["digest"], threads=NCPU)
    got = e.rsa_verify_batch(w["key_idx"], w["sig"], w["digest"])
    assert np.array_equal(got, ref)
    for n in (1, 7, 8, 9, 33, 1000):
        assert np.array_equal(e.rsa_verify_batch(w["key_idx"][:n].copy(), w["sig"][:n].copy(), w["digest"][:n].copy()), ref[:n])
    kidx = np.zeros(6, np.uint32)
    dig = w["digest"][:6].copy()
    sig = np.zeros((6, 256), np.uint8)
    for i, v in enumerate([0, 1, ns[0] - 1, ns[0], 2 ** 2048 - 1, 2 ** 2047]):
        sig[i] = np.frombuffer(int(v).to_bytes(256, "big"), np.uint8)
    got = e.rsa_verify_batch(kidx, sig, dig)
    exp = [0 if pgp.rsa_verify_pkcs1v15(ns[0], es[0], 8, dig[i].tobytes(), sig[i].tobytes()) else 1 for i in range(6)]
    assert got.tolist() == exp
    e.close()
