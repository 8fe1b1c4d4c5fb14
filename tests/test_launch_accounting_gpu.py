"""What one call of each flat entry point adds to bftq_stats' launches and items.  Every launch is counted where it is
made (launch() in bftq.cu), so these are the kernels each call really runs.  The inputs are arbitrary bytes of the right
shapes: the counters depend on the shapes and the path a call takes, not on whether a signature verifies."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 96                                                   # items per call: well below one host chunk
P256_N = 0xFFFFFFFF00000000FFFFFFFFFFFFFFFFBCE6FAADA7179E84F3B9CAC2FC632551
DSA_Q = 0xE950511EAB424B9A19A2AEB4E159B7844C589C4F          # 160 bits: a whole number of bytes, so DSA verification runs kernels
# (launches, items) per call.  Ed25519 "first use" builds the base point's table (2 kernels) and the key's table
# (2), then verifies (accumulate + finish, 2).
EXPECTED = {
    "rsa_verify": (1, N),
    "verify_tally": (2, N),
    "read_decide": (1, 0),
    "ed25519_table_free": (1, 32),
    "ed25519_first_use": (6, 64),
    "ed25519_cached": (2, 64),
    "ecdsa_p256_verify": (1, N),
    "dsa_verify": (4, N),
    "modexp": (1, 0),
    "modprod": (1, 0),
    "lagrange_combine": (1, 0),
    "lagrange_exp_product": (3, 0),
    "dsa_calculate_r": (7, 0),
    "ecdsa_p256_calculate_r": (5, 0),
    "pgp_digest": (1, 0),
}


def _bytes(rng, *shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)


def flat_calls(eng, q):
    """(name, call) of every entry point above, in order; q: a quorum over keys 0..3."""
    from bftkv_b200 import workload
    rng = np.random.default_rng(0xBF7C0A11)
    r = random.Random(0xBF7C0A11)
    p = (1 << 1023) | r.getrandbits(1023) | 1                       # odd, exactly 1024 bits: the K5 class
    k = 4
    x = np.tile(np.arange(1, k + 1, dtype=np.int32), (N, 1))
    w = workload.make_verify_batch(N, n_keys=4)
    eng.register_rsa_keys([kk["n"] for kk in w["keys"]], [kk["e"] for kk in w["keys"]])
    op_off = (np.arange(N // 4 + 1) * 4).astype(np.uint32)
    ts, vid, status = np.full(N, 5, np.uint64), np.zeros(N, np.uint32), np.zeros(N, np.uint8)
    ed_pk, ed_sig, ed_msg = _bytes(rng, 2, 32), _bytes(rng, 64, 64), _bytes(rng, 64, 32)
    return [
        ("rsa_verify", lambda: eng.rsa_verify_batch(w["key_idx"], w["sig"], w["digest"])),
        ("verify_tally", lambda: eng.verify_tally_batch(q, op_off, w["key_idx"], w["sig"], w["digest"])),
        ("read_decide", lambda: eng.read_decide_batch(q, op_off, w["key_idx"], status, ts, vid)),
        # two new keys for 32 signatures is more than the tables pay for: the table-free kernel, and nothing is built
        ("ed25519_table_free", lambda: eng.ed25519_verify_batch(ed_pk, np.arange(32, dtype=np.uint32) % 2, _bytes(rng, 32, 64), _bytes(rng, 32, 32))),
        ("ed25519_first_use", lambda: eng.ed25519_verify_batch(ed_pk[:1], np.zeros(64, np.uint32), ed_sig, ed_msg)),
        ("ed25519_cached", lambda: eng.ed25519_verify_batch(ed_pk[:1], np.zeros(64, np.uint32), ed_sig, ed_msg)),
        ("ecdsa_p256_verify", lambda: eng.ecdsa_p256_verify_batch(_bytes(rng, 1, 64), np.zeros(N, np.uint32), _bytes(rng, N, 32),
                                                                  _bytes(rng, N, 32), _bytes(rng, N, 32))),
        ("dsa_verify", lambda: eng.dsa_verify_batch(p, DSA_Q, 2, 3, _bytes(rng, N, 32), _bytes(rng, N, 32), _bytes(rng, N, 20))),
        ("modexp", lambda: eng.modexp_batch(p, [r.getrandbits(1000) for _ in range(N)], [r.getrandbits(160) for _ in range(N)])),
        ("modprod", lambda: eng.modprod_batch(p, [[r.getrandbits(1000) for _ in range(k)] for _ in range(N)])),
        ("lagrange_combine", lambda: eng.lagrange_combine_batch(P256_N, x, _bytes(rng, N, k, 32))),
        ("lagrange_exp_product", lambda: eng.lagrange_exp_product_batch(p, DSA_Q, x, [[r.getrandbits(1000) for _ in range(k)] for _ in range(N)])),
        ("dsa_calculate_r", lambda: eng.dsa_calculate_r_batch(p, DSA_Q, x, [[r.getrandbits(1000) for _ in range(k)] for _ in range(N)],
                                                              [[r.getrandbits(150) for _ in range(k)] for _ in range(N)])),
        ("ecdsa_p256_calculate_r", lambda: eng.ecdsa_p256_calculate_r_batch(x, [[b"\x04" + r.randbytes(64) for _ in range(k)] for _ in range(N)],
                                                                            [[r.getrandbits(250) for _ in range(k)] for _ in range(N)])),
        ("pgp_digest", lambda: eng.pgp_digest_batch([b"tbs-%d" % i for i in range(8)], [r.randbytes(12) for _ in range(N)],
                                                    [i % 8 for i in range(N)])),
    ]


def measure(eng):
    """{entry point: (launches, items) one call added}, the calls in the order above on a fresh engine."""
    got = {}
    q = eng.quorum_create([(1, 4, 2, 3, [0, 1, 2, 3])])
    for name, call in flat_calls(eng, q):
        s0 = eng.stats()
        call()
        s1 = eng.stats()
        got[name] = (s1["launches"] - s0["launches"], s1["items"] - s0["items"])
    eng.quorum_destroy(q)
    return got


def test_each_entry_point_counts_its_kernels(built):
    from bftkv_b200 import Engine
    eng = Engine(0)                                    # fresh: the Ed25519 table cache starts empty
    try:
        assert measure(eng) == EXPECTED
    finally:
        eng.close()
