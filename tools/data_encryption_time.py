#!/usr/bin/env python3
"""Times DataEncryption on the device (K11: bftq_data_encrypt_batch / bftq_data_decrypt_batch) and prints one JSON line
(also written to --out).

Workload: values of 32 B, 1 KiB and 16 KiB under 32-byte binary keys (bftkv's login cipher key), 4 096 and 65 536 items
per call.  Reported:
  - encrypt and decrypt items per second through one call (host clock around a call that ends in a device synchronise,
    best of --reps after a warm-up call of the same shape);
  - a separate torch.profiler pass (CUDA activity) of one encrypt and one decrypt call per value size at 65 536 items:
    each K11 kernel's device time, s2k_kernel's SHA-256 compressions per second, and its integer instructions per second
    (compressions x SASS instructions per compression, counted from cuobjdump) next to bftq_measure_int_peak;
  - a host stand-in for Go: hashlib's SHA-256 S2K, `cryptography`'s AES-CFB and hashlib's SHA-1 per item, on 8 threads.
A sample of every timed call is checked against the oracle (tests/data_encryption_oracle.py).  Card name and power limit
from nvidia-smi, read in the same run."""
import argparse
import hashlib
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
import data_encryption_oracle as O  # noqa: E402
from bftkv_b200 import Engine, _lib  # noqa: E402

SIZES = (32, 1024, 16384)
KERNELS = ("s2k_kernel", "data_encrypt_kernel", "data_cand_kernel", "seipd_decrypt_kernel")


def s2k_compressions(key_len: int) -> int:
    return (max(65536, 8 + key_len) + 8) // 64 + 1


def host_encrypt(args):
    """The work Go's Encrypt does per item, in C libraries: the S2K, the session-key wrap, CFB over the packet, SHA-1."""
    from cryptography.hazmat.decrepit.ciphers.modes import CFB
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    key, plain, rand = args
    salt, sk, iv = rand[:8], rand[8:24], rand[24:40]
    kek = hashlib.sha256(((salt + key) * (65536 // (8 + len(key)) + 1))[:65536]).digest()[:16]
    wrap = Cipher(algorithms.AES(kek), CFB(bytes(16))).encryptor()
    wrap.update(b"\x07" + sk)
    body = iv + iv[14:16] + b"\xCB" + b"t\x00" + bytes(4) + plain + b"\x00\xD3\x14"
    mdc = hashlib.sha1(body).digest()
    c = Cipher(algorithms.AES(sk), CFB(bytes(16))).encryptor()
    return c.update(body + mdc) + c.finalize()


def sass_per_compression(so: str) -> int:
    """SASS instructions in one trip of s2k_kernel's table loop (one SHA-256 compression with its words read from the
    table): the kernel has two loops of more than 1000 instructions, one compression each, and the table loop is the
    shorter; the other assembles the words byte by byte."""
    import re
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    body = next(b for b in sass.split("Function :")[1:] if "s2k_kernel" in b.split("\n", 1)[0])
    spans = []
    for ln in body.split("\n"):
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*)", ln)
        b = re.search(r"BRA\s+(0x[0-9a-f]+)", m.group(2)) if m else None
        if b and int(b.group(1), 16) < int(m.group(1), 16):
            spans.append((int(m.group(1), 16) - int(b.group(1), 16)) // 16 + 1)
    return min(x for x in spans if x > 1000)       # a build without the table has only the byte loop


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, pl, clk = [x.strip() for x in q.strip().split("\n")[0].split(",")]
    return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4096,65536")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-items", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    batches = [int(x) for x in a.batches.split(",")]
    rng = random.Random(0xDA7A)
    e = Engine(0)
    res = {"workload": "DataEncryption, 32-byte keys", **gpu_info(), "rates": []}
    big = max(batches)
    keys = [os.urandom(32) for _ in range(big)]
    rands = [os.urandom(40) for _ in range(big)]
    msgs_by_size = {}
    for size in SIZES:
        plains_all = [os.urandom(size) for _ in range(big)]
        for n in batches:
            k, p, r = keys[:n], plains_all[:n], rands[:n]
            err, msgs = e.data_encrypt_batch(k, p, r)                       # warm-up of this shape
            t_enc = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                err, msgs = e.data_encrypt_batch(k, p, r)
                t_enc.append(time.perf_counter() - t0)
            assert not err.any()
            e.data_decrypt_batch(k, msgs)
            t_dec = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                derr, outs = e.data_decrypt_batch(k, msgs)
                t_dec.append(time.perf_counter() - t0)
            assert not derr.any()
            for i in rng.sample(range(n), 8):                               # a sample against the oracle
                assert msgs[i] == O.encrypt(k[i], p[i], r[i]) and outs[i] == p[i]
            res["rates"].append({"value_bytes": size, "items": n, "encrypt_items_per_s": n / min(t_enc),
                                 "decrypt_items_per_s": n / min(t_dec), "encrypt_s": min(t_enc), "decrypt_s": min(t_dec)})
            if n == big:
                msgs_by_size[size] = (p, msgs)
        # host stand-in for Go: 8 threads of hashlib + cryptography
        m = a.host_items
        work = list(zip(keys[:m], plains_all[:m], rands[:m]))
        with ThreadPoolExecutor(8) as ex:
            list(ex.map(host_encrypt, work[:64]))
            t0 = time.perf_counter()
            list(ex.map(host_encrypt, work))
            dt = time.perf_counter() - t0
        res.setdefault("host_8_threads_encrypt_items_per_s", {})[size] = m / dt
    # kernel times, a separate profiled pass at the largest batch
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:           # one session: a second records no kernels here
        for size in SIZES:
            p, msgs = msgs_by_size[size]
            e.data_encrypt_batch(keys[:len(p)], p, rands[:len(p)])
            e.data_decrypt_batch(keys[:len(p)], msgs)
    evs = sorted((ev for ev in prof.events() if any(k in ev.name for k in KERNELS)), key=lambda ev: ev.time_range.start)
    assert len(evs) == 5 * len(SIZES), [ev.name for ev in evs]
    prof_rows = []
    for j, size in enumerate(SIZES):
        n = len(msgs_by_size[size][0])
        names = ("encrypt s2k_kernel", "data_encrypt_kernel", "decrypt s2k_kernel", "data_cand_kernel", "seipd_decrypt_kernel")
        t = {nm: (ev.time_range.end - ev.time_range.start) * 1e-6 for nm, ev in zip(names, evs[5 * j:5 * j + 5])}
        prof_rows.append({"value_bytes": size, "items": n, "kernel_s": t,
                          "s2k_compressions_per_s": n * s2k_compressions(32) / t["encrypt s2k_kernel"]})
    res["profile"] = prof_rows
    per_comp = sass_per_compression(_lib.LIB_PATH)
    res["s2k_sass_instructions_per_compression"] = per_comp
    for row in prof_rows:
        row["s2k_instructions_per_s"] = row["s2k_compressions_per_s"] * per_comp
    res["int_peak_macs_per_s"] = e.measure_int_peak()
    e.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
