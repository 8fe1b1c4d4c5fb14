"""What the batched host entry points did and returned on seeded inputs: python tools/host_layer_counters.py [out.json]

Calls bftq_rsa_verify_batch (40 000 items), bftq_verify_read_batch, bftq_signature_verify_batch (with items the GPU parser
flags), bftq_collective_verify_batch, bftq_read_responses_batch, bftq_message_decrypt_batch,
bftq_read_encrypted_responses_batch and one small call of every flat entry point tests/test_launch_accounting_gpu.py pins,
and after each prints the bftq_stats counters that depend on the host layer's plumbing only (launches, items, bytes copied, chunks, GPU-/host-parsed messages) and a SHA-256 of every
output array.  A change to the host layer that is meant to keep behaviour is run against both builds (BFTQ_LIB_PATH selects
the library) and the two outputs are compared: they must be equal.  BFTQ_HOST_THREADS=1 makes the chunk counts deterministic."""
import hashlib
import json
import os
import random
import sys

os.environ["BFTQ_HOST_THREADS"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

from bftkv_b200 import Engine, workload  # noqa: E402
from bftkv_b200.crypto_gpu import CollectiveSignature, Keyring, Message, Quorum, Signature, read_encrypted_responses_batch, read_responses_batch  # noqa: E402
from test_launch_accounting_gpu import flat_calls  # noqa: E402

COUNTERS = ("launches", "items", "h2d_bytes", "d2h_bytes", "packer_chunks", "msg_gpu_items", "msg_host_items")


def digest(x):
    if isinstance(x, np.ndarray):
        return hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest()
    if isinstance(x, (tuple, list)):
        return hashlib.sha256("".join(digest(v) for v in x).encode()).hexdigest()
    return hashlib.sha256(repr(x).encode()).hexdigest()


def partial(pkt: bytes) -> bytes:
    """The signature packet under a new-format header with a partial body length: a form only the host packer walks."""
    body = pkt[3:]
    rest = body[256:]
    return bytes([0xC2, 224 + 8]) + body[:256] + bytes([len(rest)]) + rest


def main():
    report = {}
    eng = Engine(0)

    def step(name, fn, e=eng):
        s0 = e.stats()
        out = fn()
        s1 = e.stats()
        out = out if isinstance(out, dict) else {"out": out}
        report[name] = {"stats": {k: s1[k] - s0[k] for k in COUNTERS}, "outputs": {k: digest(v) for k, v in out.items()}}
        print(name, json.dumps(report[name]), flush=True)

    # ---- flat calls: one 40 000-item verify (chunked through the staging ring) and the fused verify + read decision
    pool = workload.make_verify_batch(40000, n_keys=16)
    eng.register_rsa_keys([k["n"] for k in pool["keys"]], [k["e"] for k in pool["keys"]])
    step("rsa_verify_batch", lambda: {"status": eng.rsa_verify_batch(pool["key_idx"], pool["sig"], pool["digest"])})
    clean = workload.make_verify_batch(8192, n_keys=16, corrupt_rate=0.0, unknown_rate=0.0)
    ops = workload.make_read_ops(clean, 4096, 16, mix=workload.HARD_MIX, shuffle_arrival=True)
    q = eng.quorum_create([(5, 16, 6, 11, list(range(16)))])
    step("verify_read_batch", lambda: dict(zip(("status", "decision", "winner", "decided_at"), eng.verify_read_batch(
        q, ops["op_off"], ops["key_idx"], ops["sig"], ops["digest"], ops["ts"], ops["value_id"], pre_status=ops["pre_status"]))))
    eng.quorum_destroy(q)

    # ---- packet-level calls
    w = workload.make_pgp_verify_batch(6000, n_keys=16)
    kr = Keyring(eng)
    kr.register(w["keyring"])
    keys = workload.load_keys(16)
    tbs, sigs = list(w["tbs"]), list(w["sigs"])
    for i in range(0, 6000, 397):                       # flagged by the GPU parser: partial body lengths, v3 packets
        ki = int(w["key_idx"][i])
        sigs[i] = partial(sigs[i]) if i % 2 else workload.sig_packet_v3(keys[ki], w["key_ids"][ki], 8, tbs[i], 0x5F000000 + i)
    step("signature_verify_batch", lambda: {"err": Signature(kr).verify_batch(tbs, sigs)})

    rng = random.Random(0xBF7C0011)
    doc = [workload.tbs_packet(b"variable-%d" % j, bytes([j]) * 32, 100 + j) for j in range(4)]
    one = {(j, i): workload.sig_packet_v4(keys[i], w["key_ids"][i], 8, doc[j], 0x5F000000 + i) for j in range(4) for i in range(16)}
    ctbs, css = [], []
    for t in range(3000):
        j = rng.randrange(4)
        parts = [one[(j, i)] for i in rng.sample(range(16), rng.choice([9, 10, 11, 11, 12, 16]))]
        if t % 211 == 0:
            parts[0] = partial(parts[0])
        if t % 97 == 0:
            parts.append(one[((j + 1) % 4, 3)])
        ctbs.append(doc[j]); css.append(b"".join(parts))
    cq = Quorum(eng, [(5, 16, 11, 11, w["key_ids"])])
    step("collective_verify_batch", lambda: {"err": CollectiveSignature(Signature(kr)).verify_batch(ctbs, css, cq)})
    kr.close()

    ra = workload.make_read_answers(2048, 16, ss_signers=11, mix=workload.HARD_MIX)
    kr2 = Keyring(eng)
    kr2.register(ra["keyring"])
    step("read_responses_batch", lambda: read_responses_batch(kr2, [(5, 16, 6, 11, ra["ids"])], ra["op_off"], ra["peer_ids"], ra["msgs"],
                                                             ra["nonces"], pre_status=ra["pre_status"]))
    # ---- the decryption layer: the same answers encrypted to a client key
    ck = workload.load_keys(17)[16]
    cblock, cid = workload.pgp_public_key_block(ck, workload._private_key(ck), b"client <client@bftq.test>")
    raws, _ = workload.encrypt_answers(ra["msgs"], ck, cid)
    kr2.register(cblock, priv=True)
    assert kr2.register_private(workload.secret_key_packet(ck)) == 1
    step("message_decrypt_batch", lambda: Message(kr2).decrypt_batch(raws[:512]))
    step("read_encrypted_responses_batch", lambda: read_encrypted_responses_batch(kr2, [(5, 16, 6, 11, ra["ids"])], ra["op_off"], ra["peer_ids"],
                                                                                 raws, ra["nonces"], pre_status=ra["pre_status"]))
    kr2.close()

    # ---- one small call of every flat entry point (the Ed25519 calls expect an engine whose table cache is empty)
    fresh = Engine(0)
    q = fresh.quorum_create([(1, 4, 2, 3, [0, 1, 2, 3])])
    for name, call in flat_calls(fresh, q):
        step(name, call, fresh)
    fresh.quorum_destroy(q)
    fresh.close()
    eng.close()
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(report, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
