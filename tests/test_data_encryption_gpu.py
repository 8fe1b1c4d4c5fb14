"""GPU suite: DataEncryption on the device (K11) against the oracle (tests/data_encryption_oracle.py): encrypt byte for byte
for the same random bytes at every length class and key length and over 10 000 random items in one call; decrypt of every
GnuPG-written and Go-shaped fixture message, of oracle-built messages with wrapped session keys of every AES size and
failed unwraps, and of round trips; wrong keys, a call mixing every status, the argument errors, the launch count and
concurrent calls."""
import base64
import ctypes as C
import hashlib
import json
import os
import random
import threading
import time

import numpy as np
import pytest

import data_encryption_oracle as O
from bftkv_b200 import _lib
from bftkv_b200.crypto_gpu import DataEncryption, ErrDecryptionFailed, ErrMDC
from bftkv_b200.workload import go_partial_write

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = json.load(open(os.path.join(ROOT, "tests", "golden", "data_encryption.json")))
INVALID_ARG = -3
LENGTHS = [0, 1, 2, 15, 16, 17, 511, 512, 513, 16383, 16384, 16385, 70000]


def _value(rng, n):
    return bytes(rng.getrandbits(8) for _ in range(n))


@pytest.mark.parametrize("key_len", [0, 1, 32, 100])
def test_encrypt_matches_the_oracle(engine, key_len):
    rng = random.Random(key_len)
    keys = [_value(rng, key_len) for _ in LENGTHS]
    plains = [_value(rng, n) for n in LENGTHS]
    rands = [_value(rng, 40) for _ in LENGTHS]
    err, outs = engine.data_encrypt_batch(keys, plains, rands)
    assert list(err) == [0] * len(LENGTHS)
    for k, p, r, o in zip(keys, plains, rands, outs):
        assert o == O.encrypt(k, p, r), len(p)


def test_encrypt_10000_random_items(engine):
    rng = random.Random(11)
    n = 10000
    lens = [rng.choice([0, 1, 17, 100, 255, 256, 600, 1024]) for _ in range(n)]
    keys = [_value(rng, rng.choice([0, 1, 16, 32, 33, 100])) for _ in range(n)]
    plains = [os.urandom(m) for m in lens]
    rands = [os.urandom(40) for _ in range(n)]
    err, outs = engine.data_encrypt_batch(keys, plains, rands)
    assert not err.any()
    for i in range(n):
        assert outs[i] == O.encrypt(keys[i], plains[i], rands[i]), i


@pytest.mark.parametrize("case", FIXTURE["cases"], ids=lambda c: c["name"])
def test_decrypt_fixture(engine, case):
    err, outs = engine.data_decrypt_batch([case["passphrase"].encode()], [base64.b64decode(case["message"])])
    assert err[0] == case["code"]
    if case["code"] == 0:
        assert hashlib.sha256(outs[0]).hexdigest() == case["gnupg_plain_sha256"]
    else:
        assert outs[0] == b""


def test_decrypt_whole_fixture_in_one_call(engine):
    cases = FIXTURE["cases"]
    err, outs = engine.data_decrypt_batch([c["passphrase"].encode() for c in cases], [base64.b64decode(c["message"]) for c in cases])
    assert list(err) == [c["code"] for c in cases]
    for c, o in zip(cases, outs):
        if c["code"] == 0:
            assert hashlib.sha256(o).hexdigest() == c["gnupg_plain_sha256"]


def _skesk(key, cipher, mode, salt, count_byte, esk_plain=None):
    """A v4 SKESK over SHA-256; esk_plain (cipher byte | key) is wrapped under the S2K output when given."""
    s2k = bytes([mode, 8]) + (salt if mode in (1, 3) else b"") + (bytes([count_byte]) if mode == 3 else b"")
    kek = O.s2k(mode, salt, O.count_of(count_byte) if mode == 3 else 0, key, O.KEY_SIZE[cipher])
    body = bytes([4, cipher]) + s2k + (O.cfb_encrypt(kek, esk_plain) if esk_plain else b"")
    return bytes([0xC3, len(body)]) + body, kek


def _seipd(session_key, plain, iv=bytes(range(16)), partial=True, tamper=None):
    lit = bytes([0xCB, len(plain) + 6]) + b"b\x00" + bytes(4) + plain if len(plain) + 6 < 192 else \
        bytes([0xCB]) + go_partial_write(b"b\x00" + bytes(4) + plain) + b"\x00"
    pre = iv + iv[14:16]
    pt = pre + lit + b"\xD3\x14"
    pt += hashlib.sha1(pt).digest()
    if tamper:
        pt = tamper(pt)
    body = b"\x01" + O.cfb_encrypt(session_key, pt)
    return b"\xD2" + (go_partial_write(body) + b"\x00" if partial else bytes([0xFF]) + len(body).to_bytes(4, "big") + body)


def test_decrypt_wrapped_session_keys(engine):
    rng = random.Random(5)
    keys, msgs, want = [], [], []
    for cipher in O.AES:
        for sess in O.AES:
            key = _value(rng, 32)
            sk = _value(rng, O.KEY_SIZE[sess])
            plain = _value(rng, rng.choice([0, 5, 300, 5000]))
            pk, _ = _skesk(key, cipher, 3, _value(rng, 8), 0x10, bytes([sess]) + sk)
            keys.append(key)
            msgs.append(pk + _seipd(sk, plain, partial=bool(rng.getrandbits(1))))
            want.append((0, plain))
    # failed unwraps first (unknown cipher byte, wrong key length, CAST5 of the right length), then a good SKESK
    key, sk, plain = b"multi", _value(rng, 32), b"after three skipped SKESKs"
    bad = [_skesk(key, 7, 1, b"saltsalt", 0, bytes([99]) + _value(rng, 16))[0],
           _skesk(key, 7, 1, b"saltsalt", 0, bytes([9]) + _value(rng, 16))[0],
           _skesk(key, 7, 1, b"saltsalt", 0, bytes([3]) + _value(rng, 16))[0]]
    good, _ = _skesk(key, 9, 0, b"", 0, bytes([9]) + sk)
    keys.append(key)
    msgs.append(b"".join(bad) + good + _seipd(sk, plain))
    want.append((0, plain))
    keys.append(key)                                               # only the failed unwraps: the prompt loop never ends
    msgs.append(b"".join(bad) + _seipd(sk, plain))
    want.append((O.DECRYPTION_FAILED, None))
    err, outs = engine.data_decrypt_batch(keys, msgs)
    for (code, plain), e, o, k, m in zip(want, err, outs, keys, msgs):
        assert O.decrypt(k, m) == (code, plain)
        assert e == code and (o == plain if code == 0 else o == b"")


def test_round_trips_and_wrong_keys(engine):
    rng = random.Random(7)
    de = DataEncryption(engine)
    keys = [_value(rng, rng.choice([0, 1, 32, 100])) for _ in range(64)]
    plains = [_value(rng, rng.choice(LENGTHS)) for _ in range(64)]
    enc = de.encrypt_batch(keys, plains)
    assert all(e is None for _, e in enc)
    dec = de.decrypt_batch(keys, [c for c, _ in enc])
    assert [p for p, _ in dec] == plains and all(e is None for _, e in dec)
    t0 = time.time()
    wrong = de.decrypt_batch([k + b"!" for k in keys], [c for c, _ in enc])
    assert time.time() - t0 < 30
    assert wrong == [(None, ErrDecryptionFailed)] * 64


def test_injected_randomness_is_go_byte_order(engine):
    stream = iter([bytes(range(40))])
    de = DataEncryption(engine, rand=lambda n: next(stream))
    msg, err = de.encrypt(b"key", b"value")
    assert err is None and msg == O.encrypt(b"key", b"value", bytes(range(40)))


def test_mixed_call_keeps_item_order(engine):
    rng = random.Random(9)
    good = O.encrypt(b"k", b"good value", bytes(40))
    mdc = bytearray(good)
    mdc[-2] ^= 1                                                   # the last MDC byte (before the closing 00)
    body_short_key, body_short_sk = b"short", bytes(16)
    pk, _ = _skesk(body_short_key, 7, 0, b"", 0, bytes([7]) + body_short_sk)
    # a literal that announces 100 bytes and carries 10: ReadAll's unexpected EOF
    lit = bytes([0xCB, 106]) + b"b\x00" + bytes(4) + bytes(10)
    pre = bytes(16) + bytes(2)
    pt = pre + lit + b"\xD3\x14"
    pt += hashlib.sha1(pt).digest()
    short_body = pk + b"\xD2" + bytes([len(pt) + 1]) + b"\x01" + O.cfb_encrypt(body_short_sk, pt)
    compressed = pk + _seipd(body_short_sk, b"", tamper=lambda p: p[:18] + bytes([0xC8, 2, 0, 0]) + p[18:])
    cases = [(b"k", good, 0, b"good value"), (b"x", good, O.DECRYPTION_FAILED, None), (b"k", bytes(mdc), O.MDC, None),
             (body_short_key, short_body, O.MESSAGE_BODY, None), (b"k", good[:40], O.MALFORMED, None),
             (b"k", good[32:], O.MALFORMED, None), (body_short_key, compressed, O.UNSUPPORTED, None), (b"k", b"", O.MALFORMED, None)]
    order = list(range(len(cases))) * 4
    rng.shuffle(order)
    err, outs = engine.data_decrypt_batch([cases[j][0] for j in order], [cases[j][1] for j in order])
    for j, e, o in zip(order, err, outs):
        k, m, code, plain = cases[j]
        assert O.decrypt(k, m)[0] == code, j
        assert e == code, j
        assert o == (plain if code == 0 else b""), j
    assert DataEncryption(engine).decrypt(b"k", bytes(mdc)) == (None, ErrMDC)


def _raw_call(engine, fn, args_before_out, cap, n):
    out = np.full(max(1, cap), 0xEE, np.uint8)
    off = np.full(n + 1, 7, np.uint64)
    err = np.full(max(1, n), 5, np.int32)
    need = C.c_uint64(123)
    rc = fn(engine._h, *args_before_out, C.c_void_p(out.ctypes.data), cap, C.c_void_p(off.ctypes.data), C.byref(need),
            C.c_void_p(err.ctypes.data))
    return rc, need.value, out, off, err


def test_out_cap_one_byte_short(engine):
    lib = _lib.load()
    keys, plains = [b"a", b"bb"], [b"x" * 100, b""]
    kb, ko = engine._secret_blob(keys)
    pb, po = engine._secret_blob(plains)
    rb = np.zeros(80, np.uint8)
    p = lambda a: C.c_void_p(a.ctypes.data)
    need = sum(O.encrypted_len(len(x)) for x in plains)
    rc, got_need, out, off, err = _raw_call(engine, lib.bftq_data_encrypt_batch, (p(kb), p(ko), p(pb), p(po), p(rb), 80, 2), need - 1, 2)
    assert rc == INVALID_ARG and got_need == need
    assert (out == 0xEE).all() and (off == 7).all() and (err == 5).all()
    rc, got_need, out, off, err = _raw_call(engine, lib.bftq_data_encrypt_batch, (p(kb), p(ko), p(pb), p(po), p(rb), 79, 2), need, 2)
    assert rc == INVALID_ARG and (out == 0xEE).all() and (off == 7).all() and (err == 5).all()   # rand of the wrong length
    msgs = [O.encrypt(b"a", b"x" * 100, bytes(40)), O.encrypt(b"bb", b"", bytes(40))]
    cb, co = engine._blob(msgs)
    rc, bound, *_ = _raw_call(engine, lib.bftq_data_decrypt_batch, (p(kb), p(ko), p(cb), p(co), 2), 0, 2)
    assert rc == INVALID_ARG and bound > 0
    rc, got, out, off, err = _raw_call(engine, lib.bftq_data_decrypt_batch, (p(kb), p(ko), p(cb), p(co), 2), bound - 1, 2)
    assert rc == INVALID_ARG and got == bound and (out == 0xEE).all() and (off == 7).all() and (err == 5).all()
    rc, got, out, off, err = _raw_call(engine, lib.bftq_data_decrypt_batch, (p(kb), p(ko), p(cb), p(co), 2), bound, 2)
    assert rc == 0 and list(err[:2]) == [0, 0] and bytes(out[int(off[0]):int(off[1])]) == b"x" * 100 and off[2] == off[1]


def test_launches_per_call_are_constant(engine):
    counts = []
    for n in (1, 7, 300):
        keys, plains, rands = [b"k"] * n, [b"v" * 50] * n, [bytes(40)] * n
        l0 = engine.stats()["launches"]
        _, msgs = engine.data_encrypt_batch(keys, plains, rands)
        l1 = engine.stats()["launches"]
        engine.data_decrypt_batch(keys, msgs)
        counts.append((l1 - l0, engine.stats()["launches"] - l1))
    assert counts == [(2, 3)] * 3


def test_concurrent_calls(engine):
    failures = []

    def work(t):
        rng = random.Random(100 + t)
        for _ in range(4):
            keys = [_value(rng, 8) for _ in range(50)]
            plains = [_value(rng, rng.choice([0, 100, 2000])) for _ in range(50)]
            rands = [_value(rng, 40) for _ in range(50)]
            err, msgs = engine.data_encrypt_batch(keys, plains, rands)
            if err.any() or any(m != O.encrypt(k, p, r) for k, p, r, m in zip(keys, plains, rands, msgs)):
                failures.append(("encrypt", t))
            err, outs = engine.data_decrypt_batch(keys, msgs)
            if err.any() or outs != plains:
                failures.append(("decrypt", t))

    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not failures
