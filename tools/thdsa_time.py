#!/usr/bin/env python3
"""Times bftq_thdsa_sign_batch (K8, threshold DSA / ECDSA partial signing) on the device, and on the host the
exponentiation / scalar multiplication phase 2 needs (R_i = g^a_i mod p or a_i G) on every host thread: libcrypto's
BN_mod_exp_mont_consttime through ctypes in a thread pool (ctypes releases the GIL) for DSA, and `cryptography`'s
P-256 derive_private_key in a process pool (it holds the GIL) for ECDSA.  Prints one JSON line (also written to --out).

Workloads (n = 10 nodes, t = 5: every phase-2 item carries 2t = 10 encrypted joint shares, as a DistSign round):
  phase 2   --items requests through the whole call (10 decrypts each, K8 sums, R_i, v_i)
  phase 3   --items requests (one Z_q item each)
Rates are items per second of the whole call (host clock around a call that ends in a device synchronise) and, in a
separate profiled pass, of the K8 kernels alone (torch.profiler's CUDA activity: the summed device time of the kernels
named thdsa_*).  Every timed output is compared with the Python oracle.  Card name and power limit from nvidia-smi, read
in the same run."""
import argparse
import json
import os
import random
import subprocess
import sys
import time
import ctypes as C
import ctypes.util
from concurrent.futures import ProcessPoolExecutor, ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import threshold_dsa_oracle as O  # noqa: E402
from bftkv_b200 import Engine  # noqa: E402
from bftkv_b200.crypto_gpu import ThresholdDSA  # noqa: E402
from test_threshold_dsa_gpu import Net, group  # noqa: E402


def k8_seconds(fn):
    """Device time of the thdsa_* kernels during one call of fn (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    us = 0.0
    for ev in prof.key_averages():
        if "thdsa_" in ev.key:
            us += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    return us * 1e-6


def _p256_chunk(a_s):
    from cryptography.hazmat.primitives.asymmetric import ec
    for a in a_s:
        ec.derive_private_key(a, ec.SECP256R1()).public_key()
    return len(a_s)


class Libcrypto:
    def __init__(self):
        self.l = C.CDLL(ctypes.util.find_library("crypto") or "libcrypto.so.3")
        for f in ("BN_bin2bn", "BN_new", "BN_CTX_new"):
            getattr(self.l, f).restype = C.c_void_p
        self.l.BN_bin2bn.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
        self.l.BN_mod_exp_mont_consttime.argtypes = [C.c_void_p] * 6
        self.l.BN_free.argtypes = [C.c_void_p]
        self.l.BN_CTX_free.argtypes = [C.c_void_p]

    def exp(self, g, a, p):
        l = self.l
        bn = lambda x: l.BN_bin2bn(O.bts(x), len(O.bts(x)), None)   # noqa: E731
        bg, ba, bp, r, ctx = bn(g), bn(a), bn(p), l.BN_new(), l.BN_CTX_new()
        l.BN_mod_exp_mont_consttime(r, bg, ba, bp, ctx, None)
        for b in (bg, ba, bp, r):
            l.BN_free(b)
        l.BN_CTX_free(ctx)


def run(engine, name, items, reps):
    g = group(name)
    rng = random.Random(0xD5A9)
    n, t = 10, 5
    net = Net(engine, n)
    x, coords = O.deal(rng, g, n, t)
    sec = O.share_secret(g, *coords[0][:1], O.bts(coords[0][1]), t)
    nonce = bytes(16)
    reqs, want = [], []
    for k in range(min(items, 64)):                       # 64 distinct requests, repeated to fill the batch
        joint = [O.joint_shares(rng, g, n, t) for _ in range(n)]
        kmap = [(net.ids[0], [net.message(rng, j, 0, O.share_plain(joint[j][0]), nonce) for j in range(n)])]
        reqs.append(O.phase2_request(kmap))
        want.append(O.phase2(g, [O.share_plain(joint[j][0]) for j in range(n)]))
    th = ThresholdDSA(engine, "p256" if name == "p256" else "dsa")
    R2 = [reqs[i % len(reqs)] for i in range(items)]
    peers = list(range(items))
    res = {}
    th.sign_batch(net.rings[0], [sec] * items, R2, peers, net.ids[0], [nonce] * items)        # warm-up
    t0 = time.perf_counter()
    for _ in range(reps):
        out = th.sign_batch(net.rings[0], [sec] * items, R2, peers, net.ids[0], [nonce] * items)
    dt = (time.perf_counter() - t0) / reps
    assert all(o == (want[i % len(want)][3], None) for i, o in enumerate(out)), "phase 2 differs from the oracle"
    res["phase2_items_per_s"] = items / dt
    res["phase2_k8_kernel_s"] = k8_seconds(lambda: th.sign_batch(net.rings[0], [sec] * items, R2, peers, net.ids[0], [nonce] * items))
    q = O.order(g)
    mr = [(rng.randrange(q), rng.randrange(q)) for _ in range(items)]
    R3 = [O.phase3_request(m, r) for m, r in mr]
    t0 = time.perf_counter()
    for _ in range(reps):
        out = th.sign_batch(net.rings[0], [sec] * items, R3, peers, net.ids[0], [None] * items)
    dt = (time.perf_counter() - t0) / reps
    for i, o in enumerate(out):
        _, k, c, _ = want[i % len(want)]
        assert o == (O.phase3(g, coords[0][0], coords[0][1], mr[i][0], mr[i][1], k, c), None), "phase 3 differs from the oracle"
    res["phase3_items_per_s"] = items / dt
    res["phase3_k8_kernel_s"] = k8_seconds(lambda: th.sign_batch(net.rings[0], [sec] * items, R3, peers, net.ids[0], [None] * items))
    th.close()
    # the host comparison: R_i = a_i G / g^a_i mod p on every host thread
    a_s = [rng.randrange(1, q) for _ in range(items)]
    nt = os.cpu_count() or 1
    if name == "p256":
        import multiprocessing
        with ProcessPoolExecutor(nt, mp_context=multiprocessing.get_context("spawn")) as ex:
            list(ex.map(_p256_chunk, [a_s[:2]] * nt))                 # start the workers and import there: not timed
            t0 = time.perf_counter()
            list(ex.map(_p256_chunk, [a_s[i::nt] for i in range(nt)]))
            dt = time.perf_counter() - t0
    else:
        lc = Libcrypto()
        with ThreadPoolExecutor(nt) as ex:
            t0 = time.perf_counter()
            list(ex.map(lambda a: lc.exp(g["g"], a, g["p"]), a_s))
            dt = time.perf_counter() - t0
    res["host_R_per_s"] = items / dt
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    e = Engine(0)
    out = {"gpu": gpu, "items": a.items, "host_threads": os.cpu_count()}
    for name in ("p256", "2048/256"):
        out[name] = run(e, name, a.items, a.reps)
    e.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
