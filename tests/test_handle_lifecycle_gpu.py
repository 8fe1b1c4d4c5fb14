"""Handles that outlive their engine: a keyring with a private key, a threshold-RSA share, a threshold-DSA and a
threshold-ECDSA share and an auth server are registered on their own Engine(0) and used once; the engine is shut down
first and the handles destroyed afterwards.  Shutdown zeroes and frees every handle's device memory, and the later
destroys free host state only: no error, and the device's free memory is back where it was before the engine."""
import pytest

from bftkv_b200 import Engine
from bftkv_b200.crypto_gpu import ThresholdDSA
import threshold_dsa_oracle as D
import threshold_rsa_oracle as R
from test_auth_gpu import Pair, _params
from test_threshold_dsa_gpu import setup_round
from test_threshold_rsa_gpu import N, raw_share
import auth_oracle as A

pytestmark = pytest.mark.gpu

K7_BYTES = 32 << 20                                   # the share's fragments: a leak of them would show


def register_and_use(eng):
    """Registers one handle of each kind on eng, runs one checked batch through each, returns their destroys."""
    destroys = []
    # K6 private keys (in each node's keyring) and K8 shares of both algorithms, one phase-2 signature each
    for name in ("1024/160", "p256"):
        g, rng, t, net, x, coords, secs, joint, nonces, kmap = setup_round(eng, name, 4, 0x11FE)
        th = ThresholdDSA(eng, "p256" if name == "p256" else "dsa")
        got = th.sign(net.rings[0], secs[0], D.phase2_request(kmap), 0x51, net.ids[0], nonces[0])
        assert got == (D.phase2(g, [D.share_plain(joint[j][0]) for j in range(4)])[3], None), name
        destroys += [th.close] + [kr.close for kr in net.rings]
    # K7
    share = raw_share([(i, i & 1, b"\x7f" * 8192) for i in range(K7_BYTES // 8192)], N, 0, 10)
    h = eng.thrsa_share_create(share)
    req = R.serialize_sign_request([5], R.hash_info_sha256(b"tbs"))
    err, outs = eng.thrsa_sign_batch([h], [0], [req])
    assert int(err[0]) == 0 and outs[0] == R.sign(share, req)[0]
    destroys.append(lambda: eng.thrsa_share_destroy(h))
    # K9: phase 1 leaves ke and the MAC in the server's allocation
    rng = A.Rng(0x11FE)
    pair = Pair(eng, _params(rng), b"proof")
    xi, b = A.i2b(rng.randbelow(A.P)), rng.randbelow(A.P).to_bytes(256, "big")
    err, outs = eng.auth_server_respond_batch([pair.h], [0], [1], [xi], [b])
    assert (int(err[0]), outs[0]) == pair.oracle(1, xi, b)
    destroys.append(lambda: eng.auth_server_destroy(pair.h))
    return destroys


def test_handles_outlive_their_engine(engine):
    import torch
    torch.cuda.init()
    torch.cuda.synchronize()
    for _ in range(2):                                # the first pass loads every kernel the scenario launches; the second counts
        free0 = torch.cuda.mem_get_info()[0]
        eng = Engine(0)
        destroys = register_and_use(eng)
        held = free0 - torch.cuda.mem_get_info()[0]
        eng.close()
        for destroy in destroys:
            destroy()
        left = free0 - torch.cuda.mem_get_info()[0]
    assert held >= K7_BYTES
    assert left < 16 << 20, (held, left)
