"""bftq_read_encrypted_responses_batch: the raw wire answers (PKESK + SEIPD) in, Client.Read's decision out.  Statuses
follow the code bftq_message_decrypt_batch returns for the same bytes; the GPU tests check them against the oracle
composition (pgp_encrypt_ref.message_decrypt, the nonce check, packet.Parse, wotqs_oracle.read_decide) and against the
library's own host decryption path.  The CPU tests check the workload generator and the front-stage kernels' SASS."""
import os
import random
import subprocess
import sys
import threading

import numpy as np
import pytest

from bftkv_b200 import workload as W
import pgp_encrypt_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ST_DECRYPT_FAILED = 10


def status_of_code(code):
    """The status the encrypted read path gives an answer whose bftq_message_decrypt_batch code is `code` (not 0)."""
    return {-6: 1, -8: ST_DECRYPT_FAILED, -12: ST_DECRYPT_FAILED, -9: 3, -10: 3, -11: 5}[code]


# ---- CPU: the generator against the independent reference ----------------------------------------------------------
def _client():
    keys = W.load_keys(3)
    blocks = [W.pgp_public_key_block(k, W._private_key(k), b"node%d" % i) for i, k in enumerate(keys)]
    return keys, blocks


@pytest.mark.parametrize("cipher", [7, 8, 9])
def test_encrypt_answers_against_reference(cipher):
    from oracle import pgp_oracle as O
    keys, blocks = _client()
    ids = [b[1] for b in blocks]
    ring = O.read_entities(blocks[0][0] + blocks[1][0] + blocks[2][0])
    rng = random.Random(cipher)
    inners = [W.make_transport_message(keys[1], ids[1], bytes(rng.randrange(256) for _ in range(rng.randrange(0, 600))), bytes(8))
              for _ in range(24)]
    raws, fault = W.encrypt_answers(inners, keys[0], ids[0], seed=cipher, cipher=cipher, p_flip=0.25, p_bad_quick=0.25)
    assert set(fault.tolist()) == {0, W.ENC_FLIP, W.ENC_BAD_QUICK}
    for raw, inner, f in zip(raws, inners, fault):
        code, plain, nonce = R.message_decrypt(raw, {ids[0]: keys[0]}, {ids[0]}, {ids[1], ids[2]}, ring)
        want = {0: 0, W.ENC_FLIP: -12, W.ENC_BAD_QUICK: -8}[int(f)]
        assert code == want, (code, int(f))
        if f == 0:
            ref = O.message_verify(ring, inner)
            assert (plain, nonce) == (ref.plain, ref.nonce)
    assert W.encrypt_answers([b""], keys[0], ids[0])[0] == [b""]


def test_front_stage_sass(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    fns = {b.split("\n", 1)[0].strip(): b for b in sass.split("Function :")[1:]}
    # kernel -> threads per block at its launch
    launch = {"pkesk_seipd_parse_kernel": 128, "front_gate_kernel": 256, "seipd_decrypt_kernel": 128, "rsa_crt_decrypt_kernel": 64,
              "plain_gather_kernel": 256}
    for kernel in launch:
        bodies = [b for name, b in fns.items() if kernel in name]
        assert bodies, kernel
        assert all("LDL" not in b and "STL" not in b for b in bodies), kernel
    usage = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout.split("\n")
    seen = set()
    for i, line in enumerate(usage):
        for kernel, threads in launch.items():
            if kernel in line:
                f = dict(kv.split(":") for kv in usage[i + 1].split() if ":" in kv)
                assert f["STACK"] == "0" and f["LOCAL"] == "0", (kernel, usage[i + 1])
                assert int(f["REG"]) * threads <= 65536 and int(f["SHARED"]) <= 48 * 1024, (kernel, usage[i + 1])
                seen.add(kernel)
    assert seen == set(launch), seen


# ---- GPU ------------------------------------------------------------------------------------------------------------
N_REPLICAS = 10


def make_case(n_ops=300, seed=0xE11C):
    """Raw answers for n_ops reads from N_REPLICAS replicas, encrypted to the client (key R + 1), with every failure kind
    of the read path and of the encryption layer.  Returns a dict; `inner` holds what each answer decrypts to."""
    from oracle import packet_oracle
    keys = W.load_keys(N_REPLICAS + 3)
    blocks, kids = [], []
    for i, k in enumerate(keys):
        b, kid = W.pgp_public_key_block(k, W._private_key(k), b"a%02d (http://localhost:57%02d) <a%02d@x>" % (i, i, i))
        blocks.append(b); kids.append(kid)
    out_idx, cli, pub_only = N_REPLICAS, N_REPLICAS + 1, N_REPLICAS + 2      # outsider signer, client, public-only key
    rng = random.Random(seed)
    x = b"the variable"
    op_off, peers, raws, inners, nonces, pre, kind = [0], [], [], [], [], [], []
    for op in range(n_ops):
        order = list(range(N_REPLICAS))
        rng.shuffle(order)
        order = order[:rng.randint(0, N_REPLICAS)] if rng.random() < 0.1 else order
        cur_v = bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 32, 300])))
        for r_ in order:
            u = rng.random()
            nonce = bytes(rng.randrange(256) for _ in range(8))
            t, v, signer, bad_pre = 7, cur_v, r_, 0
            if u < 0.08:
                t, v = 6, b"older value"
            elif u < 0.12:
                v = cur_v + b"!"
            elif u < 0.15:
                signer = out_idx
            elif u < 0.18:
                bad_pre = 6
            plain = packet_oracle.serialize(x, v, t, None, None)
            m = bytearray(W.make_transport_message(keys[signer], kids[signer], plain, nonce))
            w = rng.random()
            if w < 0.04:
                m[rng.randrange(len(m))] ^= 1 << rng.randrange(8)          # bit flip in the inner stream
            elif w < 0.06:
                nonce = bytes(8)
            inner = bytes(m)
            e = rng.random()
            cipher = 8 if 0.80 <= e < 0.84 else (9 if 0.84 <= e < 0.88 else 7)
            if 0.97 <= e < 0.98:
                inner = W._new_packet(8, b"\x00" + inner)                  # compressed data (algorithm 0) around the stream
            [raw], [f] = W.encrypt_answers([inner], keys[cli], kids[cli], seed=rng.randrange(1 << 30), cipher=cipher,
                                           p_flip=1.0 if 0.88 <= e < 0.90 else 0.0, p_bad_quick=1.0 if 0.90 <= e < 0.92 else 0.0)
            k = 0
            if 0.92 <= e < 0.93:
                raw, k = raw[:rng.randrange(20, len(raw))], 1              # truncated
            elif 0.93 <= e < 0.95:
                raw = R.pkesk(kids[pub_only], keys[pub_only], R.pkcs1_type2(rng, R.session_block(7, bytes(16)))) + raw
            elif 0.95 <= e < 0.96:
                raw, k = W.encrypt_answers([inner], keys[cli], 0x1122334455667788, seed=op)[0][0], 2     # unknown PKESK id
            elif 0.96 <= e < 0.97:
                raw, k = inner, 3                                          # signed but not encrypted
            peers.append(kids[r_]); raws.append(raw); inners.append(inner); nonces.append(nonce); pre.append(bad_pre); kind.append(k)
        op_off.append(len(peers))
    qcs = [(3, 10, 4, 7, kids[:N_REPLICAS])]
    return {"keys": keys, "blocks": blocks, "kids": kids, "cli": cli, "pub_only": pub_only, "qcs": qcs, "op_off": np.array(op_off, np.uint32),
            "peers": np.array(peers, np.uint64), "raws": raws, "inners": inners, "nonces": np.frombuffer(b"".join(nonces), np.uint8).reshape(-1, 8),
            "pre": np.array(pre, np.uint8), "kind": np.array(kind, np.uint8)}


def make_keyring(engine, c, register_private=True):
    from bftkv_b200.crypto_gpu import Keyring
    kr = Keyring(engine)
    kr.register(c["blocks"][c["cli"]], priv=True)                   # the client: secring
    kr.register(b"".join(c["blocks"][:N_REPLICAS]) + c["blocks"][c["pub_only"]])
    if register_private:
        assert kr.register_private(W.secret_key_packet(c["keys"][c["cli"]])) == 1
    return kr


def run(kr, c, **kw):
    from bftkv_b200.crypto_gpu import read_encrypted_responses_batch
    return read_encrypted_responses_batch(kr, c["qcs"], c["op_off"], c["peers"], c["raws"], c["nonces"], pre_status=c["pre"], **kw)


def oracle_answers(c, codes):
    """(status, ts, value, plain, is_class) per answer from the bftq_message_decrypt_batch-style codes and the signature-half
    oracle; is_class: status is an oracle class (pgp_oracle.ST_*) rather than an exact status byte."""
    from oracle import pgp_oracle as O
    ents = O.read_entities(c["blocks"][c["cli"]] + b"".join(c["blocks"][:N_REPLICAS]) + c["blocks"][c["pub_only"]])
    out = []
    for p, code in enumerate(codes):
        if c["pre"][p]:
            out.append((int(c["pre"][p]), 0, b"", None, False))
        elif code != 0:
            out.append((status_of_code(code), 0, b"", None, False))
        else:
            st, t, v = O.read_response_status(ents, c["inners"][p], c["nonces"][p].tobytes(), 0)
            out.append((st, t, v, O.message_verify(ents, c["inners"][p]).plain, True))
    return out


def check_statuses(got, want):
    from oracle import pgp_oracle as O
    cls = {0: O.ST_OK, 8: O.ST_UNVERIFIED, 7: O.ST_NONCE, 1: O.ST_INVALID, 2: O.ST_INVALID}
    for p, (st, t, v, plain, is_class) in enumerate(want):
        g = int(got["status"][p])
        if is_class:                                                    # code 0: the signature half, nonce, packet.Parse
            assert cls.get(g, O.ST_OTHER) == st, (p, g, st)
            if st in (O.ST_OK, O.ST_UNVERIFIED):
                assert int(got["ts"][p]) == t and int(got["value_len"][p]) == len(v), p
                if "plain" in got:
                    assert got["plain"][p] == plain, p
                    vo = int(got["value_off"][p])
                    assert got["plain"][p][vo:vo + len(v)] == v, p
        elif st in (1, 2):
            assert g in (1, 2), (p, g)
        else:
            assert g == st, (p, g, st)


def check_decisions(c, got, want):
    from oracle import pgp_oracle as O, wotqs_oracle as wq
    quorum = wq.Quorum([wq.QC([wq.Node(i) for i in c["kids"][:N_REPLICAS]], 3, 10, 4, 7)])
    decs = set()
    for op in range(len(c["op_off"]) - 1):
        resp = []
        for p in range(c["op_off"][op], c["op_off"][op + 1]):
            st, t, v, _, is_class = want[p]
            good = is_class and st in (O.ST_OK, O.ST_UNVERIFIED)
            resp.append((wq.Node(int(c["peers"][p])), not good, t, v))
        kind, at, value, t = wq.read_decide(resp, quorum)
        assert (int(got["decision"][op]), int(got["decided_at"][op])) == (kind, at), op
        if kind == wq.READ_VALUE:
            wi = int(got["winner"][op])
            assert resp[wi][2] == t and resp[wi][3] == value
        decs.add(kind)
    return decs


@pytest.fixture(scope="module")
def case():
    return make_case()


@pytest.mark.gpu
def test_oracle_parity_and_self_consistency(engine, case):
    from bftkv_b200.crypto_gpu import Message
    c = case
    kr = make_keyring(engine, c)
    ids = c["kids"]
    priv = {ids[c["cli"]]: c["keys"][c["cli"]]}
    from oracle import pgp_oracle as O
    ring = O.read_entities(c["blocks"][c["cli"]] + b"".join(c["blocks"][:N_REPLICAS]) + c["blocks"][c["pub_only"]])
    codes = [R.message_decrypt(raw, priv, {ids[c["cli"]]}, set(ids[:N_REPLICAS]) | {ids[c["pub_only"]]}, ring)[0] for raw in c["raws"]]
    s0 = engine.stats()
    got = run(kr, c)
    s1 = engine.stats()
    on_gpu, on_host = s1["msg_gpu_items"] - s0["msg_gpu_items"], s1["msg_host_items"] - s0["msg_host_items"]
    n = len(c["raws"])
    assert on_gpu + on_host == n and on_gpu > 0.8 * n and on_host > 0, (on_gpu, on_host)
    want = oracle_answers(c, codes)
    check_statuses(got, want)
    assert set(codes) >= {0, -6, -8, -9, -11, -12}, set(codes)
    assert check_decisions(c, got, want) == {0, 1, 2}
    # the device path and the library's own host path agree
    lib_codes = [d["code"] for d in Message(kr).decrypt_batch(c["raws"])]
    check_statuses(got, oracle_answers(c, lib_codes))
    kr.close()


@pytest.mark.gpu
def test_unencrypted_answer_fails_only_here(engine, case):
    from bftkv_b200.crypto_gpu import read_encrypted_responses_batch, read_responses_batch
    c = case
    kr = make_keyring(engine, c)
    p = next(i for i in range(len(c["raws"])) if c["kind"][i] == 3 and not c["pre"][i] and c["peers"][i] in c["kids"][:N_REPLICAS]
             and read_responses_batch(kr, c["qcs"], np.array([0, 1], np.uint32), c["peers"][i:i + 1], [c["inners"][i]], c["nonces"][i:i + 1])["status"][0] == 0)
    args = (kr, c["qcs"], np.array([0, 1], np.uint32), c["peers"][p:p + 1], [c["raws"][p]], c["nonces"][p:p + 1])
    assert read_responses_batch(*args)["status"][0] == 0
    assert read_encrypted_responses_batch(*args)["status"][0] == 3
    kr.close()


def _dump(case_path, path):
    """Run in a subprocess with small BFTQ_READ_PIECE / BFTQ_READ_SUPER: the same call, outputs to `path`."""
    import pickle
    from bftkv_b200 import Engine
    with open(case_path, "rb") as f:
        c = pickle.load(f)
    eng = Engine(0)
    kr = make_keyring(eng, c)
    got = run(kr, c)
    np.savez(path, plain=np.frombuffer(b"".join(got.pop("plain")) or b"\0", np.uint8), **got)
    kr.close()
    eng.close()


@pytest.mark.gpu
def test_piece_and_super_chunk_boundaries(engine, case, tmp_path):
    kr = make_keyring(engine, case)
    got = run(kr, case)
    kr.close()
    import pickle
    path, case_path = str(tmp_path / "small.npz"), str(tmp_path / "case.pkl")
    with open(case_path, "wb") as f:
        pickle.dump(case, f)
    env = dict(os.environ, BFTQ_READ_PIECE="37", BFTQ_READ_SUPER="500")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_read_encrypted_gpu as T; T._dump(%r, %r)" % (ROOT, os.path.join(ROOT, "tests"), case_path, path)
    subprocess.run([sys.executable, "-c", code], env=env, check=True, cwd=ROOT)
    small = np.load(path)
    for k in ("status", "ts", "value_off", "value_len", "plain_len", "decision", "winner", "decided_at"):
        assert np.array_equal(small[k], got[k]), k
    assert small["plain"].tobytes() == (b"".join(got["plain"]) or b"\0")


@pytest.mark.gpu
def test_key_removed_or_never_registered(engine, case):
    """bftq_keyring_remove drops the client's private half but leaves its secring entity, so both a removed key and one
    registered priv = 1 without register_private make the host key loop hand the answer back (UNSUPPORTED).  Answers to
    an unknown key id and truncated PKESKs fail before any secring key is looked at (DECRYPT_FAILED); unencrypted ones
    are MALFORMED.  Every status follows the library's own decrypt code."""
    from bftkv_b200.crypto_gpu import Message
    c = case
    live = c["pre"] == 0
    for register_private in (True, False):
        kr = make_keyring(engine, c, register_private=register_private)
        if register_private:
            kr.remove([c["kids"][c["cli"]]])
        got = run(kr, c)
        codes = [d["code"] for d in Message(kr).decrypt_batch(c["raws"])]
        assert all(code != 0 for code, lv in zip(codes, live) if lv)
        want = np.array([int(c["pre"][p]) if c["pre"][p] else status_of_code(code) for p, code in enumerate(codes)], np.uint8)
        got_st = got["status"].copy()
        got_st[got_st == 2] = 1                                         # BAD_SIGNATURE / HASH_TAG
        assert np.array_equal(got_st, want)
        assert np.all(got["status"][live & (c["kind"] == 0)] == 5)
        check_decisions(c, got, [(int(s), 0, b"", None, False) for s in got["status"]])
        kr.close()


@pytest.mark.gpu
def test_concurrent_calls_agree(engine, case):
    kr = make_keyring(engine, case)
    outs = [None] * 4

    def work(i):
        outs[i] = run(kr, case)
    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for o in outs[1:]:
        for k in ("status", "ts", "value_off", "value_len", "plain_len", "decision", "winner", "decided_at"):
            assert np.array_equal(o[k], outs[0][k]), k
        assert o["plain"] == outs[0]["plain"]
    kr.close()


@pytest.mark.gpu
def test_argument_errors_match_read_responses(engine, case):
    from bftkv_b200 import _lib
    from bftkv_b200.crypto_gpu import Keyring, read_encrypted_responses_batch, read_responses_batch
    c = case
    kr = make_keyring(engine, c)
    n1 = np.array([0, 33], np.uint32)
    bad = [dict(op_off=n1, peers=np.zeros(33, np.uint64), msgs=[b"x"] * 33, nonces=np.zeros((33, 8), np.uint8)),
           dict(op_off=np.array([0, 1], np.uint32), peers=np.zeros(1, np.uint64), msgs=[b"x"], nonces=np.zeros((1, 25), np.uint8))]
    for b in bad:
        codes = []
        for fn in (read_responses_batch, read_encrypted_responses_batch):
            with pytest.raises(_lib.BftqError) as ei:
                fn(kr, c["qcs"], b["op_off"], b["peers"], b["msgs"], b["nonces"])
            codes.append(ei.value.code)
        assert codes[0] == codes[1] == -3, codes
    parse_only = Keyring(None)
    for fn in (read_responses_batch, read_encrypted_responses_batch):
        with pytest.raises(_lib.BftqError) as ei:
            fn(parse_only, c["qcs"], np.array([0, 1], np.uint32), np.zeros(1, np.uint64), [b"x"], np.zeros((1, 8), np.uint8))
        assert ei.value.code == -1
    got = read_encrypted_responses_batch(kr, c["qcs"], np.array([0], np.uint32), np.zeros(0, np.uint64), [], np.zeros((0, 8), np.uint8))
    assert len(got["status"]) == 0 and len(got["decision"]) == 0
    parse_only.close()
    kr.close()
