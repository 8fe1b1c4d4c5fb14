#!/usr/bin/env python3
"""Times bftq_thrsa_sign_batch (K7, threshold-RSA partial signing) on the device and a libcrypto stand-in for Go's
big.Int.Exp on all host threads.  Prints one JSON line (also written to --out).

Workloads (shares of the golden fixture key split by the oracle's Distribute, n = 10, k = 7):
  depth1  65 536 items over 8 shares, each the fragment of key 0 (about 4 100 bits): every first DistSign request
  mixed   16 384 items over the fragments of keys at depths 0-3 (4 100 to 32 800-bit exponents)

Rates: partial signatures per second of the whole call (host clock around a call that ends in a device synchronise)
and of the kernels alone (torch.profiler, in a separate pass); word-MACs from shapes (Montgomery products x 8 256); the
share of bftq_measure_int_peak measured in the same run; card name and power limit from nvidia-smi.  Every timed
output is compared against libcrypto's BN_mod_exp_mont (+ BN_mod_inverse for negative fragments), and a sample
against the Python oracle."""
import argparse
import ctypes as C
import ctypes.util
import json
import os
import random
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import threshold_rsa_oracle as O  # noqa: E402
from bftkv_b200 import Engine  # noqa: E402

MACS_PER_PRODUCT = 2 * 64 * 64 + 64


def products(words):
    return 16 + 5 * 8 * words + 1          # table, 4 squarings + 1 product per 4-bit window, leaving Montgomery form


def workload(kind, rng, shares_raw):
    parsed = [O.parse_partial_param(s) for s in shares_raw]
    items = []
    if kind == "depth1":
        for i in range(65536):
            items.append((i % 8, 0))
    else:
        by_depth = {}
        for s, (keys, _, _, _) in enumerate(parsed):
            for kid in keys:
                by_depth.setdefault(O.depth(kid, 10), []).append((s, kid))
        for i in range(16384):
            items.append(rng.choice(by_depth[i % 4]))
    reqs = [O.serialize_sign_request([kid], O.hash_info_sha256(b"%s-%d" % (kind.encode(), i))) for i, (_, kid) in enumerate(items)]
    return [s for s, _ in items], reqs, parsed


class Libcrypto:
    def __init__(self):
        self.l = C.CDLL(ctypes.util.find_library("crypto") or "libcrypto.so.3")
        for f in ("BN_bin2bn", "BN_new", "BN_CTX_new"):
            getattr(self.l, f).restype = C.c_void_p
        self.l.BN_bin2bn.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
        self.l.BN_mod_exp_mont.argtypes = [C.c_void_p] * 5 + [C.c_void_p]
        self.l.BN_mod_inverse.restype = C.c_void_p
        self.l.BN_mod_inverse.argtypes = [C.c_void_p] * 4
        self.l.BN_bn2binpad.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        self.l.BN_free.argtypes = [C.c_void_p]
        self.l.BN_CTX_free.argtypes = [C.c_void_p]

    def sign_one(self, m, d, N):
        """m^d mod N, inverted when d < 0 (what Sign computes for one key id), via BN_mod_exp_mont."""
        l = self.l
        bn = lambda x: l.BN_bin2bn(O.int_bytes(x), len(O.int_bytes(x)), None)   # noqa: E731
        bm, bd, bN, r, ctx = bn(m), bn(abs(d)), bn(N), l.BN_new(), l.BN_CTX_new()
        l.BN_mod_exp_mont(r, bm, bd, bN, ctx, None)
        if d < 0:
            l.BN_mod_inverse(r, r, bN, ctx)
        buf = C.create_string_buffer(256)
        l.BN_bn2binpad(r, buf, 256)
        for b in (bm, bd, bN, r):
            l.BN_free(b)
        l.BN_CTX_free(ctx)
        return int.from_bytes(buf.raw, "big")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of each workload (a rehearsal uses a small one)")
    ap.add_argument("--cpu-items", type=int, default=4096, help="items the libcrypto stand-in times")
    ap.add_argument("--oracle-sample", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    key = json.load(open(os.path.join(ROOT, "tests", "golden", "thrsa_key.json")))
    N, D = int(key["n"], 16), int(key["d"], 16)
    shares_raw = O.distribute(D, N, 10, 7, seed=2024)
    rng = random.Random(1)
    threads = os.cpu_count() or 1
    lc = Libcrypto()
    eng = Engine(0)
    handles = [eng.thrsa_share_create(s) for s in shares_raw]
    res = {"tool": "tools/thrsa_time.py", "host_threads": threads}
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        res["gpu"] = smi.stdout.strip().split("\n")[0]
    except OSError:
        res["gpu"] = "unknown"
    res["int_peak_macs_per_s"] = eng.measure_int_peak()
    for kind in ("depth1", "mixed"):
        idx, reqs, parsed = workload(kind, rng, shares_raw)
        n = max(8, int(len(reqs) * a.scale))
        idx, reqs = idx[:n], reqs[:n]
        eng.thrsa_sign_batch(handles, idx[:256], reqs[:256])                # warm-up
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            err, outs = eng.thrsa_sign_batch(handles, idx, reqs)
            times.append(time.perf_counter() - t0)
        assert not err.any()
        # kernel time, separate pass under the profiler
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.thrsa_sign_batch(handles, idx, reqs)
            torch.cuda.synchronize()
        ktime = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA" and ("thrsa" in ev.name):
                ktime[ev.name.split("(")[0].split("<")[0]] = ktime.get(ev.name.split("(")[0].split("<")[0], 0.0) + ev.device_time_total * 1e-6
        k7 = sum(v for k, v in ktime.items() if "partial_sign" in k)
        # shapes
        macs = 0
        for s, r in zip(idx, reqs):
            kid = O.parse_sign_request(r)[0][0]
            words = (len(O.int_bytes(abs(parsed[s][0][kid]))) + 3) // 4
            macs += products(words) * MACS_PER_PRODUCT
        # correctness of every timed output against libcrypto, a sample against the oracle
        def check(i):
            keys, Nn, pid, nn = parsed[idx[i]]
            kids, (pre, dg) = O.parse_sign_request(reqs[i])
            m = O.emsa_encode(pre, dg, Nn)
            got = O.parse_partial_signature(outs[i])[0][0][1]
            return got == lc.sign_one(m, keys[kids[0]], Nn)
        with ThreadPoolExecutor(threads) as ex:
            ok = all(ex.map(check, range(n)))
        sample = random.Random(3).sample(range(n), min(a.oracle_sample, n))
        ok_oracle = all(outs[i] == O.sign(shares_raw[idx[i]], reqs[i])[0] for i in sample)
        # CPU stand-in: BN_mod_exp_mont on all host threads
        cn = min(a.cpu_items, n)
        jobs = []
        for i in range(cn):
            keys, Nn, _, _ = parsed[idx[i]]
            kids, (pre, dg) = O.parse_sign_request(reqs[i])
            jobs.append((O.emsa_encode(pre, dg, Nn), keys[kids[0]], Nn))
        t0 = time.perf_counter()
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(lambda j: lc.sign_one(*j), jobs))
        cpu_t = time.perf_counter() - t0
        best = min(times)
        res[kind] = {"items": n, "call_s": [round(t, 4) for t in times], "partials_per_s_call": n / best,
                     "kernel_s": ktime, "partials_per_s_kernel": n / k7 if k7 else None,
                     "word_macs": macs, "macs_per_s_kernel": macs / k7 if k7 else None,
                     "share_of_int_peak": (macs / k7) / res["int_peak_macs_per_s"] if k7 else None,
                     "outputs_match_libcrypto": ok, "outputs_match_oracle_sample": ok_oracle,
                     "cpu_libcrypto_items": cn, "cpu_libcrypto_partials_per_s": cn / cpu_t}
    for h in handles:
        eng.thrsa_share_destroy(h)
    eng.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
