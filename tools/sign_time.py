#!/usr/bin/env python3
"""Times PGPSignature.Sign on the device (bftq_signature_sign_batch: K4 digest, K12 rsa_crt_sign_kernel, K1 check) and prints
one JSON line (also written to --out).

Workload: RSA-2048 key 0 of tests/golden/rsa_keys_bf7c0001.json signs 65 536 items per call, tbs of 64 B and of 1 KiB.
Reported:
  - items per second through one call (host clock around a call, which ends in a device synchronise; best of --reps after
    a warm-up call of the same shape);
  - a separate torch.profiler pass (CUDA activity) of one call per tbs size: each kernel's device time, and K12's signatures
    per second from rsa_crt_sign_kernel's time alone;
  - K12's 32x32-bit multiply-accumulates per second from an operation count (macs_per_signature), next to
    bftq_measure_int_peak's rate;
  - a host stand-in for Go: `cryptography` (OpenSSL) RSA-2048 PKCS#1 v1.5 signing with SHA-256 of tbs || suffix, 8 threads.
A sample of every timed call is checked against the oracle (tests/signature_sign_oracle.py).  Card name and power limit
from nvidia-smi, read in the same run."""
import argparse
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
import decrypt_edges as D  # noqa: E402
import signature_sign_oracle as O  # noqa: E402
from bftkv_b200 import Engine, workload as W  # noqa: E402
from bftkv_b200.crypto_gpu import Keyring, Signature  # noqa: E402

SIZES = (64, 1024)
KERNELS = ("pgp_digest_kernel", "rsa_crt_sign_kernel", "rsa_verify_r32_kernel")


def macs_per_signature() -> int:
    """32x32-bit multiply-accumulates of one K12 signature.  A Montgomery product of W words costs 2 W^2 (product and
    reduction).  Per 1024-bit prime (W = 32): 1024 squarings and 256 window products over the 1024 exponent bits, 14 to
    fill the 16-entry window table, and 4 conversions in and out of Montgomery form.  Garner: one product of W = 32 and
    one of W = 64."""
    half = (1024 + 256 + 14 + 4) * 2 * 32 * 32
    return 2 * half + 2 * 32 * 32 + 2 * 64 * 64


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, pl, clk = [x.strip() for x in q.strip().split("\n")[0].split(",")]
    return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-items", type=int, default=4096)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = random.Random(0x5161)
    k = W.load_keys(1)[0]
    block, kid = O.key_block(k)
    e = Engine(0)
    kr = Keyring(e)
    kr.register(block, priv=True)
    assert kr.register_private(D.secret_key_packet(k)) == 1
    sig = Signature(kr)
    res = {"workload": "PGPSignature.Sign, RSA-2048, %d items per call" % a.items, **gpu_info(), "rates": []}
    n = a.items
    inputs = {}
    for size in SIZES:
        tbs = [rng.randbytes(size) for _ in range(n)]
        ct = [rng.getrandbits(32) for _ in range(n)]
        inputs[size] = (tbs, ct)
        sig.sign_batch(tbs, ct)                                              # warm-up of this shape
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            errs, packets = sig.sign_batch(tbs, ct)
            times.append(time.perf_counter() - t0)
        assert errs == [None] * n
        for i in rng.sample(range(n), 16):
            assert packets[i] == O.packet(k, kid, tbs[i], ct[i])
        res["rates"].append({"tbs_bytes": size, "items": n, "call_items_per_s": n / min(times), "call_s": min(times)})
    # host stand-in for Go: OpenSSL through `cryptography`, 8 threads
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding
    priv = W._private_key(k)
    res["host_8_threads_signatures_per_s"] = {}
    for size in SIZES:
        tbs, ct = inputs[size]
        work = [tbs[i] + O.suffix(ct[i], kid) for i in range(a.host_items)]
        with ThreadPoolExecutor(8) as ex:
            list(ex.map(lambda m: priv.sign(m, padding.PKCS1v15(), hashes.SHA256()), work[:64]))
            t0 = time.perf_counter()
            list(ex.map(lambda m: priv.sign(m, padding.PKCS1v15(), hashes.SHA256()), work))
            dt = time.perf_counter() - t0
        res["host_8_threads_signatures_per_s"][size] = a.host_items / dt
    # kernel times, a separate profiled pass
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for size in SIZES:
            sig.sign_batch(*inputs[size])
    evs = sorted((ev for ev in prof.events() if any(kn in ev.name for kn in KERNELS)), key=lambda ev: ev.time_range.start)
    assert len(evs) == 3 * len(SIZES), [ev.name for ev in evs]
    res["macs_per_signature"] = macs_per_signature()
    res["int_peak_macs_per_s"] = e.measure_int_peak()
    res["profile"] = []
    for j, size in enumerate(SIZES):
        t = {kn: (ev.time_range.end - ev.time_range.start) * 1e-6 for kn, ev in zip(KERNELS, evs[3 * j:3 * j + 3])}
        k12 = n / t["rsa_crt_sign_kernel"]
        res["profile"].append({"tbs_bytes": size, "items": n, "kernel_s": t, "k12_signatures_per_s": k12,
                               "k12_macs_per_s": k12 * res["macs_per_signature"],
                               "k12_share_of_int_peak": k12 * res["macs_per_signature"] / res["int_peak_macs_per_s"]})
    kr.close()
    e.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
