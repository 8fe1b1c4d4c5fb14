"""K1b on one GPU: 262 144 Ed25519 verifies over 15 keys (BASELINE configs[3]), device-resident, CUDA events.
BFTQ_ED25519_TABLES=0 selects the classic double-and-add kernel (the switch is read when the engine is created)."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from bftkv_b200 import Engine, _lib
import ctypes as C

from cryptography.hazmat.primitives import serialization
from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey

N, K, BASE = 262144, 15, 32768
rng = np.random.default_rng(5)
sks = [Ed25519PrivateKey.from_private_bytes(rng.integers(0, 256, 32, dtype=np.uint8).tobytes()) for _ in range(K)]
pks = np.frombuffer(b"".join(k.public_key().public_bytes(serialization.Encoding.Raw, serialization.PublicFormat.Raw) for k in sks), np.uint8).reshape(K, 32).copy()
kidx = rng.integers(0, K, BASE).astype(np.uint32)
msg = rng.integers(0, 256, (BASE, 32), dtype=np.uint8)
sig = np.empty((BASE, 64), np.uint8)
for i in range(BASE):
    sig[i] = np.frombuffer(sks[kidx[i]].sign(msg[i].tobytes()), np.uint8)
bad = rng.random(BASE) < 0.01
sig[bad, 5] ^= 1
rep = N // BASE
kidx, msg, sig, bad = np.tile(kidx, rep), np.tile(msg, (rep, 1)), np.tile(sig, (rep, 1)), np.tile(bad, rep)
eng = Engine(0)
dev = torch.device("cuda", 0)
d = [torch.from_numpy(x).to(dev) for x in (pks, kidx.astype(np.int32), sig, msg)]
st = torch.empty(N, dtype=torch.uint8, device=dev)
stream = torch.cuda.Stream(device=dev)


def step():
    _lib.check(eng._lib.bftq_ed25519_verify_batch_dev(eng._h, pks.ctypes.data_as(C.c_void_p), K, C.c_void_p(d[1].data_ptr()), C.c_void_p(d[2].data_ptr()),
                                                      C.c_void_p(d[3].data_ptr()), N, C.c_void_p(st.data_ptr()), C.c_void_p(stream.cuda_stream)))


for _ in range(3):
    step()
stream.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(stream)
for _ in range(5):
    step()
e1.record(stream)
stream.synchronize()
ms = e0.elapsed_time(e1) / 5
assert np.array_equal(st.cpu().numpy() != 0, bad)
print({"tables": os.environ.get("BFTQ_ED25519_TABLES", "1"), "ms_per_step": ms, "verifies_per_sec": N / ms * 1e3})
