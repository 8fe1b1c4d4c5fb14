"""bftq_message_decrypt_batch (K6a RSA-CRT + K6b AES-CFB / MDC) against the construction of each message and, for the
signature half, against bftq_message_verify_batch on the same inner stream."""
import random

import pytest

from bftkv_b200 import workload as W
import pgp_encrypt_ref as R


def test_cfb_by_hand_matches_cryptography():
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
    rng = random.Random(0xBF7C0600)
    for _ in range(200):
        key = bytes(rng.randrange(256) for _ in range(rng.choice([16, 24, 32])))
        data = bytes(rng.randrange(256) for _ in range(rng.randrange(1, 300)))
        e = Cipher(algorithms.AES(key), modes.CFB(bytes(16))).encryptor()
        ref = e.update(data) + e.finalize()
        assert R.cfb_encrypt(key, data) == ref
        assert R.cfb_decrypt(key, ref) == data


def _fixture():
    keys = W.load_keys(3)
    privs = [W._private_key(k) for k in keys]
    blocks = [W.pgp_public_key_block(k, pv, b"node%d" % i) for i, (k, pv) in enumerate(zip(keys, privs))]
    return keys, blocks


def _setup(engine):
    from bftkv_b200.crypto_gpu import Keyring
    keys, blocks = _fixture()
    kr = Keyring(engine)
    kr.register(blocks[0][0], priv=True)          # this node: secring
    kr.register(blocks[1][0])                     # a peer (signer)
    kr.register(blocks[2][0])                     # a public-only key
    assert kr.register_private(R.secret_key_packet(keys[0])) == 1
    return kr, keys, [b[1] for b in blocks]


def _oracle(raws):
    from oracle import pgp_oracle as O
    keys, blocks = _fixture()
    ids = [b[1] for b in blocks]
    ring = O.read_entities(blocks[0][0] + blocks[1][0] + blocks[2][0])     # secring ++ keyring
    return [R.message_decrypt(raw, {ids[0]: keys[0]}, {ids[0]}, {ids[1], ids[2]}, ring) for raw in raws]


def _branch_cases():
    """(raw message, expected BFTQ_ERR_* code) for every branch of the key loop and the SEIPD layer."""
    keys, blocks = _fixture()
    me, peer, other = keys
    ids = [b[1] for b in blocks]
    rng = random.Random(0xBF7C0601)

    def inner(signer=peer, sid=None):
        plain = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 400)))
        return W.make_transport_message(signer, sid if sid is not None else ids[1], plain, bytes(rng.randrange(256) for _ in range(32)))

    cases = []
    for cipher in (7, 8, 9):
        cases.append((R.encrypt(rng, me, ids[0], inner(), cipher=cipher), 0))
    cases.append((R.pkesk(ids[2], other, R.pkcs1_type2(rng, R.session_block(7, bytes(16)))) + R.encrypt(rng, me, ids[0], inner()), 0))  # first PKESK public-only
    cases.append((R.encrypt(rng, me, 0x1122334455667788, inner()), -8))                                      # unknown key id
    key = bytes(range(16))
    s = inner()
    blk = R.session_block(7, key)
    type1 = b"\x00\x01" + b"\xff" * (256 - 3 - len(blk)) + b"\x00" + blk                                   # block type 1, not 2
    cases.append((R.pkesk(ids[0], me, type1) + R.seipd(key, s, rng), -8))
    short_ps = b"\x00\x02" + bytes([1] * 5) + b"\x00" + bytes(256 - 8 - len(blk)) + blk                       # first zero at index 7
    cases.append((R.pkesk(ids[0], me, short_ps) + R.seipd(key, s, rng), -8))
    em = R.pkcs1_type2(rng, blk)
    cases.append((W._new_packet(1, bytes([3]) + ids[0].to_bytes(8, "big") + bytes([1]) + W._mpi(me["n"] + 1)) + R.seipd(key, s, rng), -8))  # c > n
    cases.append((R.pkesk(ids[0], me, R.pkcs1_type2(rng, bytes([7]) + key + b"\x00\x00")) + R.seipd(key, s, rng), 0))   # bad checksum: key kept
    cases.append((R.pkesk(ids[0], me, R.pkcs1_type2(rng, bytes([42]) + key + b"\x00\x00")) + R.seipd(key, s, rng), -8))  # unknown cipher
    cases.append((R.pkesk(ids[0], me, R.pkcs1_type2(rng, R.session_block(3, key))) + R.seipd(key, s, rng), -11))         # CAST5
    cases.append((R.pkesk(ids[0], me, em) + R.seipd(key, s, rng, bad_quick=True), -8))                      # quick check fails
    cases.append((R.pkesk(ids[0], me, em) + R.seipd(key, s, rng, flip_mdc=True), -12))                      # MDC mismatch
    cases.append((R.pkesk(ids[0], me, em) + bytes([0xC0 | 18, 30, 1]) + R.cfb_encrypt(key, bytes(29)), -8))  # truncated SEIPD
    cases.append((R.pkesk(ids[0], me, em) + W._new_packet(9, bytes(40)), -11))                             # tag 9
    cases.append((s, -9))                                                                                  # not encrypted
    cases.append((R.pkesk(ids[2], other, em) + s, -8))                                                     # key material, then no encrypted packet
    cases.append((R.pkesk(0x1122334455667788, me, em) + s, -9))                                            # ... matching no key: ReadMessage goes on
    cases.append((R.pkesk(ids[0], me, em) + R.seipd(key, W._new_packet(8, bytes([0]) + s), rng), -11))     # compressed inner stream
    cases.append((R.encrypt(rng, me, ids[0], inner(signer=other, sid=0x0102030405060708)), 0))             # unknown signer
    s_bad = bytearray(inner())
    s_bad[-5] ^= 1                                                                                         # a bad signature inside
    cases.append((R.encrypt(rng, me, ids[0], bytes(s_bad)), -6))
    cases.append((R.pkesk(ids[0], me, R.pkcs1_type2(rng, b"\x07\x01")) + R.seipd(key, s, rng), -8))        # < 3 bytes (the reference panics)
    return cases


def _seeded_batch(n=200):
    keys, blocks = _fixture()
    me, peer, other = keys
    ids = [b[1] for b in blocks]
    rng = random.Random(0xBF7C0603)
    out = []
    for _ in range(n):
        plain = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 600)))
        signer, sid = (peer, ids[1]) if rng.random() < 0.8 else (other, 0x0102030405060708)
        s = W.make_transport_message(signer, sid, plain, bytes(rng.randrange(256) for _ in range(32)))
        v = rng.randrange(6)
        raw = R.encrypt(rng, me, ids[0], s, cipher=rng.choice((7, 8, 9)), flip_mdc=v == 1, bad_quick=v == 2)
        if v == 3:
            raw = R.pkesk(ids[2], other, R.pkcs1_type2(rng, R.session_block(7, bytes(16)))) + raw
        out.append(raw)
    return out


def test_oracle_branches():
    """The reference decryption reaches every branch with the outcome the reference's code path gives."""
    cases = _branch_cases()
    got = _oracle([c[0] for c in cases])
    assert [g[0] for g in got] == [c[1] for c in cases]
    assert all(g[1] is not None for g, c in zip(got, cases) if c[1] in (0, -6))


@pytest.mark.gpu
def test_decrypt_matches_oracle(engine):
    from bftkv_b200.crypto_gpu import Message
    kr, keys, ids = _setup(engine)
    raws = [c[0] for c in _branch_cases()] + _seeded_batch()
    got = Message(kr).decrypt_batch(raws)
    ref = _oracle(raws)
    codes = set()
    for i, (g, (code, plain, nonce)) in enumerate(zip(got, ref)):
        codes.add(code)
        assert g["code"] == code, (i, g, code)
        if code in (0, -6):
            assert g["plain"] == plain and g["nonce"] == nonce, i
    assert {0, -6, -8, -9, -11, -12} <= codes
    kr.close()


@pytest.mark.gpu
def test_register_rejects_and_remove(engine):
    from bftkv_b200 import _lib
    from bftkv_b200.crypto_gpu import Message
    kr, keys, ids = _setup(engine)
    me, peer, other = keys
    bad = dict(me)
    bad["q"] = other["q"]                         # p q != n
    with pytest.raises(_lib.BftqError) as ei:
        kr.register_private(R.secret_key_packet(bad))
    assert ei.value.code == -4
    with pytest.raises(_lib.BftqError) as ei:
        kr.register_private(R.secret_key_packet(other, protected=True))
    assert ei.value.code == -4
    rng = random.Random(0xBF7C0602)
    s = W.make_transport_message(peer, ids[1], b"value", b"n" * 32)
    raw = R.encrypt(rng, me, ids[0], s)
    assert Message(kr).decrypt_batch([raw])[0]["code"] == 0
    kr.remove([ids[0]])                           # drops the entity's private half from the device
    assert Message(kr).decrypt_batch([raw])[0]["code"] == -11   # secring key without a private half: re-run on crypto/pgp
    kr.close()
