#!/usr/bin/env python3
"""Times bftq_auth_server_respond_batch (K9, the server half of crypto/auth's password authentication) on the device,
and on the host the exponentiation every answer needs: libcrypto's BN_mod_exp_mont_consttime through ctypes on 8 threads
(ctypes releases the GIL), a stand-in for Go's math/big.  Prints one JSON line (also written to --out).

Workloads, --items distinct servers per call:
  phase 0   Yi = X^y mod p                      (one 2048-bit exponentiation per item)
  phase 1   Bi = v^b, Ki = Xi^b, HKDF, HMAC     (two per item)
  phase 2   MAC check and AES-128-GCM seal of a 256-byte proof (--seal-items servers, whose MACs the oracle computes)
Rates are items per second of the whole call (host clock around a call that ends in a device synchronise) and, in a
separate profiled pass, of auth_pow_kernel alone (torch.profiler's CUDA activity: the kernel's device time).
Every timed Yi and Bi is compared with libcrypto's result, and a sample of every phase with the oracle.  Card name and
power limit from nvidia-smi, read in the same run."""
import argparse
import ctypes as C
import ctypes.util
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import auth_oracle as A  # noqa: E402
from bftkv_b200 import Engine  # noqa: E402


def pow_kernel_seconds(calls):
    """Device time of auth_pow_kernel in each of `calls`, in order, from one torch.profiler session (CUDA activity): a
    second session in the same process records no kernels here, so all calls share one."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls:
            fn()
    evs = sorted((ev for ev in prof.events() if "auth_pow_kernel" in ev.name), key=lambda ev: ev.time_range.start)
    assert len(evs) == len(calls), f"{len(evs)} auth_pow_kernel launches profiled for {len(calls)} calls"
    return [(ev.time_range.end - ev.time_range.start) * 1e-6 for ev in evs]


class Libcrypto:
    def __init__(self):
        self.l = C.CDLL(ctypes.util.find_library("crypto") or "libcrypto.so.3")
        for f in ("BN_bin2bn", "BN_new", "BN_CTX_new"):
            getattr(self.l, f).restype = C.c_void_p
        self.l.BN_bin2bn.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
        self.l.BN_bn2bin.argtypes = [C.c_void_p, C.c_char_p]
        self.l.BN_num_bits.argtypes = [C.c_void_p]
        self.l.BN_mod_exp_mont_consttime.argtypes = [C.c_void_p] * 6
        self.l.BN_free.argtypes = [C.c_void_p]
        self.l.BN_CTX_free.argtypes = [C.c_void_p]

    def exp(self, x: bytes, e: bytes, m: bytes) -> bytes:
        """x^e mod m, big.Int.Bytes() form; x < m."""
        l = self.l
        bx, be, bm, r, ctx = l.BN_bin2bn(x, len(x), None), l.BN_bin2bn(e, len(e), None), l.BN_bin2bn(m, len(m), None), l.BN_new(), l.BN_CTX_new()
        l.BN_mod_exp_mont_consttime(r, bx, be, bm, ctx, None)
        out = C.create_string_buffer(256)
        n = l.BN_bn2bin(r, out)
        for b in (bx, be, bm, r):
            l.BN_free(b)
        l.BN_CTX_free(ctx)
        return out.raw[:n]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-threads", type=int, default=8)
    ap.add_argument("--seal-items", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    rng = A.Rng(0xA71)
    n = a.items
    e = Engine(0)
    lc = Libcrypto()
    pb = A.i2b(A.P)
    ys = [rng.randbelow(A.Q) for _ in range(n)]
    vs = [rng.randbelow(A.P) for _ in range(n)]
    params = [A.serialize_params(i + 1, y, v, rng.randbytes(32)) for i, (y, v) in enumerate(zip(ys, vs))]
    proof = rng.randbytes(256)
    hs = [e.auth_server_create(p, proof) for p in params]
    idx = list(range(n))
    X = A.i2b(pow(A.PI(b"password"), rng.randbelow(A.Q), A.P))
    xis = [A.i2b(rng.randbelow(A.P)) for _ in range(n)]
    bs = [rng.randbelow(A.P).to_bytes(256, "big") for _ in range(n)]
    nonces = [rng.randbytes(12) for _ in range(n)]
    out = {"gpu": gpu, "items": n, "proof_bytes": len(proof), "host_threads": a.host_threads}

    def timed(phases, reqs, rands):
        e.auth_server_respond_batch(hs, idx, phases, reqs, rands)                 # warm-up
        t0 = time.perf_counter()
        for _ in range(a.reps):
            err, res = e.auth_server_respond_batch(hs, idx, phases, reqs, rands)
        return (time.perf_counter() - t0) / a.reps, err, res

    # phase 0
    dt, err, res = timed([0] * n, [X] * n, [b""] * n)
    with ThreadPoolExecutor(a.host_threads) as ex:
        t0 = time.perf_counter()
        want = list(ex.map(lambda y: lc.exp(X, A.i2b(y), pb), ys))
        host_dt = time.perf_counter() - t0
    assert all(int(x) == 0 for x in err)
    assert all(A.parse_yi(r)[1] == int.from_bytes(w, "big") for r, w in zip(res, want)), "Yi differs from libcrypto"
    for i in range(0, n, max(1, n // 16)):
        assert res[i] == A.Server(params[i], proof).make_yi(X), "Yi differs from the oracle"
    out["phase0_items_per_s"] = n / dt
    out["host_libcrypto_exp_per_s"] = n / host_dt
    # phase 1
    dt, err, res = timed([1] * n, xis, bs)
    with ThreadPoolExecutor(a.host_threads) as ex:
        want = list(ex.map(lambda i: lc.exp(A.i2b(vs[i]), bs[i], pb), range(n)))
    assert all(A.parse_bi(r) == int.from_bytes(w, "big") for r, w in zip(res, want)), "Bi differs from libcrypto"
    m = min(n, a.seal_items)                                            # phase 2 runs on the first m servers, every MAC known
    oracle = {i: A.Server(params[i], proof) for i in range(m)}
    for i, o in oracle.items():
        if i % max(1, m // 16) == 0:
            assert res[i] == o.make_bi(xis[i], int.from_bytes(bs[i], "big")), "Bi differs from the oracle"
        else:
            o.make_bi(xis[i], int.from_bytes(bs[i], "big"))
    out["phase1_items_per_s"] = n / dt
    t0k, t1k = pow_kernel_seconds([lambda: e.auth_server_respond_batch(hs, idx, [0] * n, [X] * n, [b""] * n),
                                   lambda: e.auth_server_respond_batch(hs, idx, [1] * n, xis, bs)])
    out["phase0_pow_kernel_s"], out["phase0_pow_kernel_items_per_s"] = t0k, n / t0k
    out["phase1_pow_kernel_s"], out["phase1_pow_kernel_items_per_s"] = t1k, n / t1k
    # phase 2: each timed call needs a fresh phase 1 before it (phase 2 wipes the state)
    macs = [oracle[i].mac for i in range(m)]
    seal_dt = 0.0
    for _ in range(a.reps):
        e.auth_server_respond_batch(hs[:m], idx[:m], [1] * m, xis[:m], bs[:m])
        t0 = time.perf_counter()
        err, res = e.auth_server_respond_batch(hs[:m], idx[:m], [2] * m, macs, nonces[:m])
        seal_dt += time.perf_counter() - t0
    for i, o in oracle.items():
        assert int(err[i]) == 0 and res[i] == o.make_zi(o.mac, nonces[i]), "the sealed proof differs from the oracle"
    out["phase2_seals_per_s"] = m * a.reps / seal_dt
    out["phase2_items"] = m
    for h in hs:
        e.auth_server_destroy(h)
    e.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
