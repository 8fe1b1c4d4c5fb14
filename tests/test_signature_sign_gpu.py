"""PGPSignature.Sign on the device (bftq_signature_sign_batch: K4 digest, K12 rsa_crt_sign_kernel, K1 check): every packet
of tests/golden/signature_sign.json byte for byte, 10 000 random items in one call, every packet through the library's own
verification, getPrivateKey's choice of signer, the call-level errors and constant launch counts."""
import ctypes as C
import random
import sys
import os
import threading

import numpy as np
import pytest

import decrypt_edges as D
import read_answer_edges as RE
import signature_sign_oracle as O
from bftkv_b200 import workload as W

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_signature_sign as G  # noqa: E402

pytestmark = pytest.mark.gpu

CERT_NOT_FOUND, UNSUPPORTED, INVALID_ARG = -20, -11, -3


@pytest.fixture(scope="module")
def keys():
    """name -> (key, public block, primary key id) for the fixture's keys and a few more."""
    ks = dict(G.keys())
    more = W.load_keys(9)
    ks.update({"1": more[1], "2": more[2], "7": more[7], "8": more[8]})
    out = {}
    for name, k in ks.items():
        block, kid = O.key_block(k, b"signer-%s <%s@bftq.test>" % (name.encode(), name.encode()))
        out[name] = (k, block, kid)
    return out


def signer(engine, keys, names, private=None):
    """A keyring whose secring holds `names` in order, one registration each, with the private halves of `private`
    (default: all of them)."""
    from bftkv_b200.crypto_gpu import Keyring, Signature
    kr = Keyring(engine)
    for n in names:
        kr.register(keys[n][1], priv=True)
    priv = names if private is None else private
    if priv:
        assert kr.register_private(b"".join(D.secret_key_packet(keys[n][0]) for n in priv)) == len(priv)
    return kr, Signature(kr)


def verify_all(engine, keys, name, tbs, packets):
    """Every packet verifies through bftq_signature_verify_batch on a public keyring."""
    from bftkv_b200.crypto_gpu import Keyring, Signature
    kr = Keyring(engine)
    kr.register(keys[name][1])
    assert Signature(kr).verify_batch(tbs, packets) == [None] * len(tbs)
    kr.close()


@pytest.mark.parametrize("name", G.KEYS)
def test_fixture_packets(engine, keys, name):
    cases = [c for c in G_cases() if c["key"] == name]
    kr, sig = signer(engine, keys, [name])
    tbs = [G.tbs_bytes(c["tbs_len"], c["tbs_index"]) for c in cases]
    errs, packets = sig.sign_batch(tbs, [c["ctime"] for c in cases])
    assert errs == [None] * len(cases)
    for c, p in zip(cases, packets):
        assert p.hex() == c["packet"], (name, c["tbs_len"], c["ctime"], c["kind"])
    verify_all(engine, keys, name, tbs, packets)
    kr.close()


def G_cases():
    import json
    return json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "signature_sign.json")))["cases"]


def test_random_items_one_call(engine, keys):
    rng = random.Random(0xBF7C5161)
    k, _, kid = keys["H"]
    kr, sig = signer(engine, keys, ["H"])
    n = 10000
    lens = [rng.choice([0, 1, 55, 56, 64]) if rng.random() < 0.1 else rng.randrange(0, 1500) for _ in range(n)]
    tbs = [rng.randbytes(L) for L in lens]
    ct = [rng.getrandbits(32) for _ in range(n)]
    errs, packets = sig.sign_batch(tbs, ct)
    assert errs == [None] * n
    for t, c, p in zip(tbs, ct, packets):
        assert p == O.packet(k, kid, t, c, O.cryptography_s)
    short = sum(p[-256] == 0 for p in packets)
    assert short > 0                                   # leading-zero cases among them (about 1 in 128)
    verify_all(engine, keys, "H", tbs, packets)
    kr.close()


def test_secring_first_entity_signs(engine, keys):
    tbs = [b"<x, t, v>", b""]
    kr, sig = signer(engine, keys, ["1", "2", "7"])
    k, _, kid = keys["1"]
    errs, packets = sig.sign_batch(tbs, [7, 8])
    assert errs == [None, None] and packets == [O.packet(k, kid, t, c) for t, c in zip(tbs, [7, 8])]
    # replace(): re-adding the first entity keeps its place, and a later entity never moves ahead of it
    kr.register(keys["1"][1], priv=True)
    kr.register(keys["8"][1], priv=True)
    assert sig.sign_batch(tbs, [7, 8])[1] == packets
    kr.close()
    # a keyring whose first entity is another key signs with that key
    kr, sig = signer(engine, keys, ["2", "1"])
    k2, _, kid2 = keys["2"]
    assert sig.sign_batch(tbs, [7, 8])[1] == [O.packet(k2, kid2, t, c) for t, c in zip(tbs, [7, 8])]
    assert sig.sign(tbs[0], 9) == (O.packet(k2, kid2, tbs[0], 9), None)
    kr.close()


def test_primary_key_signs_not_subkey(engine, keys):
    from bftkv_b200.crypto_gpu import Keyring, Signature
    k, sub = keys["7"][0], keys["8"][0]
    block, sub_id = RE.subkey_block(k, sub, b"with-subkey <s@bftq.test>")
    kid = keys["7"][2]
    kr = Keyring(engine)
    kr.register(block, priv=True)
    assert kr.register_private(D.secret_key_packet(k) + D.secret_key_packet(sub, tag=7)) == 2
    errs, packets = Signature(kr).sign_batch([b"tbs"], [5])
    assert errs == [None] and packets[0] == O.packet(k, kid, b"tbs", 5) and sub_id != kid
    kr.close()
    # only the subkey's private half: the primary key cannot sign on the device, and the subkey is not used instead
    kr = Keyring(engine)
    kr.register(block, priv=True)
    assert kr.register_private(D.secret_key_packet(sub, tag=7)) == 1
    with pytest.raises(Exception) as ex:
        Signature(kr).sign_batch([b"tbs"], [5])
    assert ex.value.code == UNSUPPORTED
    kr.close()


def test_call_level_errors(engine, keys):
    from bftkv_b200.crypto_gpu import ErrCertificateNotFound, Keyring, Signature
    kr = Keyring(engine)
    kr.register(keys["1"][1])                          # a public keyring only: the secring is empty
    with pytest.raises(Exception) as ex:
        Signature(kr).sign_batch([b"a"], [1])
    assert ex.value.code == CERT_NOT_FOUND
    assert Signature(kr).sign(b"a") == (None, ErrCertificateNotFound)
    kr.close()
    kr, sig = signer(engine, keys, ["1"], private=[])   # no private half registered
    with pytest.raises(Exception) as ex:
        sig.sign_batch([b"a"], [1])
    assert ex.value.code == UNSUPPORTED
    kr.close()
    kr, sig = signer(engine, keys, ["1", "2"])
    kr.remove([keys["1"][2]])                          # drops the private half; Go's Remove leaves the secring alone
    with pytest.raises(Exception) as ex:
        sig.sign_batch([b"a"], [1])
    assert ex.value.code == UNSUPPORTED
    kr.close()


def test_invalid_args_leave_outputs_untouched(engine, keys):
    from bftkv_b200 import _lib
    lib = _lib.load()
    kr, _ = signer(engine, keys, ["1"])
    p = lambda a: C.c_void_p(a.ctypes.data)
    blob = np.frombuffer(b"abcdef", np.uint8).copy()
    good, bad = np.array([0, 3, 6], np.uint64), np.array([0, 4, 3], np.uint64)
    ct = np.array([1, 2], np.uint32)
    out = np.full(2 * O.PACKET_BYTES, 0xAB, np.uint8)
    err = np.full(2, 77, np.int32)
    calls = [(kr._h, p(blob), p(bad), p(ct), 2, p(out), p(err)),        # offsets that go backwards
             (kr._h, p(blob), None, p(ct), 2, p(out), p(err)),          # no offsets
             (kr._h, None, p(good), p(ct), 2, p(out), p(err)),          # no blob behind non-empty offsets
             (kr._h, p(blob), p(good), None, 2, p(out), p(err)),        # no creation times
             (kr._h, p(blob), p(good), p(ct), 2, None, p(err)),         # no output
             (kr._h, p(blob), p(good), p(ct), 2, p(out), None),         # no error array
             (None, p(blob), p(good), p(ct), 2, p(out), p(err))]        # no keyring
    for args in calls:
        assert lib.bftq_signature_sign_batch(*args) == INVALID_ARG
        assert (out == 0xAB).all() and (err == 77).all()
    assert lib.bftq_signature_sign_batch(kr._h, p(blob), p(good), p(ct), 2, p(out), p(err)) == 0
    assert (err == 0).all()
    empty = np.zeros(3, np.uint64)                     # every tbs empty: no blob is needed
    assert lib.bftq_signature_sign_batch(kr._h, None, p(empty), p(ct), 2, p(out), p(err)) == 0
    k, _, kid = keys["1"]
    assert (err == 0).all() and bytes(out[:O.PACKET_BYTES]) == O.packet(k, kid, b"", 1)
    kr.close()


def test_launch_count_is_constant(engine, keys):
    k, _, kid = keys["5"]
    kr, sig = signer(engine, keys, ["5"])
    rng = random.Random(3)
    for n in (1, 1000, 65536):
        tbs = [rng.randbytes(rng.randrange(0, 200)) for _ in range(n)]
        ct = [rng.getrandbits(32) for _ in range(n)]
        before = engine.stats()["launches"]
        errs, packets = sig.sign_batch(tbs, ct)
        assert engine.stats()["launches"] - before == 3, n
        assert errs == [None] * n
        for i in rng.sample(range(n), min(n, 200)):
            assert packets[i] == O.packet(k, kid, tbs[i], ct[i], O.cryptography_s)
    kr.close()


def test_concurrent_callers(engine, keys):
    k, _, kid = keys["L"]
    kr, sig = signer(engine, keys, ["L"])
    results, fails = {}, []

    def worker(t):
        rng = random.Random(100 + t)
        try:
            for call in range(4):
                n = rng.randrange(1, 400)
                tbs = [rng.randbytes(rng.randrange(0, 300)) for _ in range(n)]
                ct = [rng.getrandbits(32) for _ in range(n)]
                results[(t, call)] = (tbs, ct, sig.sign_batch(tbs, ct))
        except Exception as ex:          # noqa: BLE001 - reported below
            fails.append(ex)
    threads = [threading.Thread(target=worker, args=(t,)) for t in range(6)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not fails and len(results) == 24
    for tbs, ct, (errs, packets) in results.values():
        assert errs == [None] * len(tbs)
        assert packets == [O.packet(k, kid, t, c, O.cryptography_s) for t, c in zip(tbs, ct)]
    kr.close()
