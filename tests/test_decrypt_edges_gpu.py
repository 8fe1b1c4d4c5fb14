"""The decryption edge cases (tests/decrypt_edges.py) on the device: bftq_message_decrypt_batch (K6a, K6b) family by family,
a grown and reshuffled private-key table, the encrypted read path's front stage (K6p, K6q), a K6a launch of more than
one grid wave, and keys whose secret-key packet carries a u in another convention."""
import random

import numpy as np
import pytest

import decrypt_edges as D
import pgp_encrypt_ref as R
from bftkv_b200 import workload as W
from test_read_encrypted_gpu import check_statuses, status_of_code

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def edges():
    return D.build()


def edge_keyring(engine, e):
    from bftkv_b200.crypto_gpu import Keyring
    kr = Keyring(engine)
    sec, pub = e.keyring_blocks()
    kr.register(sec, priv=True)
    kr.register(pub)
    assert kr.register_private(b"".join(D.secret_key_packet(e.keys[n]) for n in D.KEYS)) == len(D.KEYS)
    return kr


def check_decrypt(kr, rows, ref, seed):
    """One shuffled decrypt_batch call over rows; codes equal ref's, plain texts and nonces too where the code is 0 or -6."""
    from bftkv_b200.crypto_gpu import Message
    order = list(range(len(rows)))
    random.Random(seed).shuffle(order)
    got = Message(kr).decrypt_batch([rows[i]["raw"] for i in order])
    for g, i in zip(got, order):
        code, plain, nonce = ref[i]
        assert g["code"] == code, (rows[i]["name"], g["code"], code)
        if code in (0, -6):
            assert (g["plain"], g["nonce"]) == (plain, nonce), rows[i]["name"]


@pytest.mark.parametrize("family", ["A", "B", "C", "D"])
def test_family(engine, edges, family):
    kr = edge_keyring(engine, edges)
    rows = edges.family(family)
    ref = edges.oracle([r["raw"] for r in rows])
    for r, (code, plain, nonce) in zip(rows, ref):
        if r["want"] is not None:
            assert code == r["want"] and (code != 0 or (plain, nonce) == (r["plain"], r["nonce"])), r["name"]
    check_decrypt(kr, rows, ref, ord(family))
    kr.close()


def read_path(engine, kr, signer_id, rows, ref, ring):
    """bftq_read_encrypted_responses_batch over rows (one answer per read operation): each status is the one the row's
    decrypt code maps to, or for code 0 the signature half's verdict on the row's inner stream.  -> (answers the device
    decided, answers it handed to the host)."""
    from bftkv_b200.crypto_gpu import read_encrypted_responses_batch
    from oracle import pgp_oracle as O
    n = len(rows)
    nonces = np.frombuffer(b"".join(r["nonce"] or bytes(8) for r in rows), np.uint8).reshape(n, 8)
    s0 = engine.stats()
    got = read_encrypted_responses_batch(kr, [(1, 4, 2, 3, [signer_id, 1, 2, 3])], np.arange(n + 1, dtype=np.uint32),
                                         np.full(n, signer_id, np.uint64), [r["raw"] for r in rows], nonces)
    s1 = engine.stats()
    want = []
    for r, (code, plain, nonce) in zip(rows, ref):
        if code != 0:
            want.append((status_of_code(code), 0, b"", None, False))
        else:
            st, t, v = O.read_response_status(ring, r["inner"], r["nonce"], 0)
            want.append((st, t, v, plain, True))
    check_statuses(got, want)
    return s1["msg_gpu_items"] - s0["msg_gpu_items"], s1["msg_host_items"] - s0["msg_host_items"]


def test_key_table_and_read_path(engine, edges):
    """20 private keys in one keyring (the 17th grows the table past 16 slots), two removed and two new ones in their
    slots, one re-registered into a new slot, and an entity whose PKESKs name its encryption subkey.  Then one shuffled
    decrypt_batch call with 8 messages per live key and messages to the removed keys, and the same answers through the
    encrypted read path."""
    from bftkv_b200.crypto_gpu import Keyring
    from oracle import pgp_oracle as O
    from read_answer_edges import subkey_block
    e = edges
    fix = W.load_keys(26)
    # L first: the smallest modulus sits in slot 0, so K6p must read each answer's own slot to pass a c above it.  Fixture
    # key 1 signs the inner streams and stays out: one key id in two entities would send every answer to the host.
    keys = [e.keys["L"]] + [fix[i] for i in range(18) if i != D.SIGNER] + [e.keys["H"]] + [fix[18]]
    assert fix[5]["p"] > fix[5]["q"]
    blocks = [W.pgp_public_key_block(k, W._private_key(k), b"t%02d <t@bftq.test>" % i) for i, k in enumerate(keys + [fix[20], fix[21]])]
    kr = Keyring(engine)
    kr.register(b"".join(b for b, _ in blocks), priv=True)
    kr.register(e.signer_block)
    for i, k in enumerate(keys):                               # one at a time: slot i
        assert kr.register_private(D.secret_key_packet(k)) == 1, i
    removed = [blocks[3][1], blocks[11][1]]
    kr.remove(removed)                                         # slots 3 and 11 free; the entities stay in the secring
    assert kr.register_private(D.secret_key_packet(fix[20]) + D.secret_key_packet(fix[21])) == 2
    assert kr.register_private(D.secret_key_packet(keys[17])) == 1      # key in slot 17 moves to slot 20
    sub_block, sub_id = subkey_block(fix[22], fix[23], b"sub <sub@bftq.test>")
    kr.register(sub_block, priv=True)
    assert kr.register_private(D.secret_key_packet(fix[23], tag=7)) == 1
    live = {kid: k for (_, kid), k in zip(blocks, keys + [fix[20], fix[21]]) if kid not in removed}
    live[sub_id] = fix[23]
    assert len(live) == 21
    dead = {kid: k for (_, kid), k in zip(blocks, keys) if kid in removed}
    rng = random.Random(0xBF7C06E1)
    rows = []
    for kid, k in list(live.items()) + list(dead.items()):
        for j in range(8):
            inner = e.inners[rng.randrange(len(e.inners))]
            cipher = (7, 8, 9)[j % 3]
            key = rng.randbytes(D.KS[cipher])
            em = R.pkcs1_type2(rng, D.session_block(cipher, key))
            raw = D.pkesk_c(kid, D.enc(k, em)) + D.seipd_packet(D.seipd_body(key, inner[0], rng.randbytes(16)))
            rows.append(dict(name="%016x/%d" % (kid, j), raw=raw, c=D.enc(k, em), inner=inner[0], plain=inner[1], nonce=inner[2]))
    for kid in (blocks[18][1], blocks[19][1]):                  # c = n and c = n + 1 for keys in slots 18 and 19
        k = live[kid]
        for c in (k["n"], k["n"] + 1):
            inner = e.inners[0]
            rows.append(dict(name="c-edge", raw=D.pkesk_c(kid, c) + D.seipd_packet(D.seipd_body(bytes(16), inner[0], bytes(16))),
                             c=c, inner=inner[0], plain=None, nonce=None))
    assert sum(r["c"] > keys[0]["n"] for r in rows[8:8 * 21]) > 20, "too few c above slot 0's modulus"
    ring = O.read_entities(b"".join(b for b, _ in blocks) + sub_block + e.signer_block)
    ref = [R.message_decrypt(r["raw"], live, {kid for _, kid in blocks} | {sub_id}, {e.signer_id}, ring) for r in rows]
    assert {c for c, _, _ in ref} >= {0, -8, -11}
    check_decrypt(kr, rows, ref, 0xBF7C06E2)
    # the read path: every row has bftkv's shape; none reaches K6b's MDC mismatch, so the device decides all but the
    # answers to the removed keys, which the host key loop hands back
    host = sum(1 for c, _, _ in ref if c == -11)
    assert read_path(engine, kr, e.signer_id, rows, ref, ring) == (len(rows) - host, host)
    kr.close()


def test_read_path_on_family_rows(engine, edges):
    """Rows with bftkv's shape through the encrypted read path: statuses follow the decrypt codes, and only the answers
    whose MDC K6b finds wrong (a wrong session key that passes the quick check, a flipped MDC) or whose inner stream K0m
    cannot parse go to the host."""
    from oracle import pgp_oracle as O
    e = edges
    kr = edge_keyring(engine, e)
    rows = [r for r in e.rows if r["shape"]]
    ref = e.oracle([r["raw"] for r in rows])
    sec, pub = e.keyring_blocks()
    host = sum(r["host"] for r in rows)
    assert host == 7
    assert read_path(engine, kr, e.signer_id, rows, ref, O.read_entities(sec + pub)) == (len(rows) - host, host)
    kr.close()


def test_k6a_beyond_one_wave(engine, edges):
    """One decrypt_batch call of 16 * 16 * SMs + 37 PKESKs: rsa_crt_decrypt_kernel's grid holds 16 blocks of 16 items per
    SM, so the last 37 items take a second trip through the kernel's loop (and its scrubbed shared memory)."""
    import torch
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    try:
        from cryptography.hazmat.decrepit.ciphers.modes import CFB
    except ImportError:
        from cryptography.hazmat.primitives.ciphers.modes import CFB
    from bftkv_b200.crypto_gpu import Message
    import hashlib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert sms == engine.sm_count
    n = 16 * 16 * sms + 37
    e = edges
    kr = edge_keyring(engine, e)
    k, kid = e.keys["H"], e.ids["H"]
    rng = np.random.default_rng(0xBF7C06E3)
    raws, want = [], []
    for i in range(n):
        inner = e.inners[i % 3]
        key = rng.bytes(16)
        blk = D.session_block(7, key)
        ps = bytes(rng.integers(1, 256, 256 - 3 - len(blk), dtype=np.uint8))
        em = b"\x00\x02" + ps + b"\x00" + blk
        bad = i % 8 == 5
        if bad:
            em = b"\x00\x03" + em[2:]
        prefix = rng.bytes(16)
        body = prefix + prefix[14:16] + inner[0] + b"\xd3\x14"
        body += hashlib.sha1(body).digest()
        c = Cipher(algorithms.AES(key), CFB(bytes(16))).encryptor()
        raws.append(D.pkesk_c(kid, D.enc(k, em)) + D.seipd_packet(c.update(body) + c.finalize()))
        want.append((-8, None, None) if bad else (0, inner[1], inner[2]))
    got = Message(kr).decrypt_batch(raws)
    for i, (g, (code, plain, nonce)) in enumerate(zip(got, want)):
        assert g["code"] == code, (i, g["code"], code)
        if code == 0:
            assert (g["plain"], g["nonce"]) == (plain, nonce), i
    # the same count of invalid blocks: K6a runs and nothing after it (no candidate reaches K6b, no inner stream the
    # signature half), so the call's one launch is K6a over all n items
    bad_raw = raws[5]
    s0 = engine.stats()
    got = Message(kr).decrypt_batch([bad_raw] * n)
    s1 = engine.stats()
    assert all(g["code"] == -8 for g in got)
    assert s1["launches"] - s0["launches"] == 1
    kr.close()


@pytest.mark.parametrize("name", ["0", "H"])
def test_u_from_p_and_q(engine, edges, name):
    """The packet's u is not what Garner uses: u = q^-1 mod p (PKCS#1's qInv), u = 0 and u = p^-1 mod q + q all register
    and decrypt, as x/crypto, which never reads u, does."""
    from bftkv_b200.crypto_gpu import Keyring, Message
    e = edges
    k, kid = e.keys[name], e.ids[name]
    p, q = k["p"], k["q"]
    rng = random.Random(0xBF7C06E4)
    inner = e.inners[1]
    key = rng.randbytes(16)
    raw = D.pkesk_c(kid, D.enc(k, R.pkcs1_type2(rng, D.session_block(7, key)))) + D.seipd_packet(D.seipd_body(key, inner[0], rng.randbytes(16)))
    for u in (pow(q, -1, p), 0, pow(p, -1, q) + q):
        kr = Keyring(engine)
        kr.register(e.blocks[name], priv=True)
        kr.register(e.signer_block)
        assert kr.register_private(D.secret_key_packet(k, u=u)) == 1
        g = Message(kr).decrypt_batch([raw])[0]
        assert (g["code"], g["plain"], g["nonce"]) == (0, inner[1], inner[2])
        kr.close()
