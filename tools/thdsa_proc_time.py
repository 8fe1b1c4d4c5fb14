#!/usr/bin/env python3
"""Times bftq_thdsa_process_batch (K8's client half) on the device, and libcrypto's CalculateR on the host threads.
Prints one JSON line (also written to --out).

Workloads (n = 10 nodes, t = 5: a completion combines 2t = 10 partial signatures), --procs processes per call:
  phase 1   every item is a process's 2t-th partial signature: CalculateR (DSA: 2t + 1 exponentiations mod p with a |q|-bit
            exponent; P-256: 2t + 1 scalar multiplications)
  phase 2   every item is a process's 2t-th s_i: calculateS and formatDSA
Rates are processes per second of the whole call (host clock around a call that ends in a device synchronise) and, in a
separate profiled pass, the summed device time of the call's kernels (torch.profiler's CUDA activity).  Every timed output is
compared with the client oracle (tests/threshold_dsa_proc_oracle.py).  The host comparison runs CalculateR's 2t + 1 big
operations per process on 8 host threads: DSA's exponentiations through libcrypto (BN_mod_exp_mont_consttime, ctypes,
threads), P-256's variable-base scalar multiplications as `cryptography` ECDH exchanges (processes: it holds the GIL).  The
kernel time is the mean over three profiled calls in one session.  Card name and power limit from nvidia-smi, read in the
same run."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor, ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import threshold_dsa_proc_oracle as P  # noqa: E402
from bftkv_b200 import Engine  # noqa: E402
from test_threshold_dsa_gpu import group  # noqa: E402
from test_threshold_dsa_proc import REQUEST, RESPONSE, Round, split_request  # noqa: E402
from thdsa_time import Libcrypto  # noqa: E402

N, T = 10, 5
HOST_THREADS = 8


def kernel_seconds(fns):
    """Mean device time of the kernels launched during one call, over the calls fns (torch.profiler, CUDA activity, one
    session; the device is synchronised inside it so that every kernel record is in).  Fails when no kernel was recorded."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in fns:
            fn()
        torch.cuda.synchronize()
    us, seen = 0.0, 0
    for ev in prof.key_averages():
        if "_kernel" in ev.key:
            us += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            seen += ev.count
    assert seen > 0, "the profiler recorded no kernel"
    return us * 1e-6 / len(fns)


def _ecdh_chunk(args):
    """CalculateR's 2t + 1 variable-base P-256 scalar multiplications for each process in the chunk (ECDH exchange)."""
    from cryptography.hazmat.primitives.asymmetric import ec
    n_procs, points = args
    pubs = [ec.EllipticCurvePublicNumbers(x, y, ec.SECP256R1()).public_key() for x, y in points]
    scalars = [ec.derive_private_key(0x1234567 + 7 * j, ec.SECP256R1()) for j in range(2 * T + 1)]
    for _ in range(n_procs):
        for j, d in enumerate(scalars):
            d.exchange(ec.ECDH(), pubs[j % len(pubs)])
    return n_procs


def run(engine, name, procs, reps):
    kind = "p256" if name == "p256" else "dsa"
    algo = 3 if kind == "p256" else 2
    rd = Round(group(name), N, 0xD5F0)
    oc = P.Proc(kind, rd.dgst, T, rd.ids)
    p0 = [rd.phase0(j) for j in range(2 * T)]
    for j in range(2 * T):
        P.step(oc, RESPONSE, p0[j], rd.ids[j])
    _, req1 = split_request(P.step(oc, REQUEST)[2])
    p1 = [rd.phase1(i, req1) for i in range(2 * T)]
    want1 = [P.step(oc, RESPONSE, p1[i], rd.ids[i]) for i in range(2 * T)][-1]
    _, req2 = split_request(P.step(oc, REQUEST)[2])
    p2 = [rd.phase2(i, req2) for i in range(2 * T)]
    want2 = [P.step(oc, RESPONSE, p2[i], rd.ids[i]) for i in range(2 * T)][-1]

    def call(hs, items):
        st, err, outs = engine.thdsa_process_batch(hs, [i for i, _, _, _ in items], [o for _, o, _, _ in items], [p for _, _, _, p in items],
                                                   [d for _, _, d, _ in items])
        return [(int(s), int(e), o) for s, e, o in zip(st, err, outs)]

    def fresh(upto_phase2):
        hs = [engine.thdsa_proc_create(algo, rd.dgst, T, rd.ids) for _ in range(procs)]
        items = [(k, RESPONSE, p0[j], rd.ids[j]) for k in range(procs) for j in range(2 * T)]
        items += [(k, RESPONSE, p1[i], rd.ids[i]) for k in range(procs) for i in range(2 * T - (0 if upto_phase2 else 1))]
        if upto_phase2:
            items += [(k, REQUEST, b"", 0) for k in range(procs)] + [(k, RESPONSE, p2[i], rd.ids[i]) for k in range(procs) for i in range(2 * T - 1)]
        got = call(hs, items)
        if upto_phase2:
            assert split_request(got[-(2 * T - 1) * procs - 1][2])[1] == req2, "phase-2 request differs from the oracle"
        return hs

    res = {}
    for ph, last, want in ((1, p1[-1], want1), (2, p2[-1], want2)):
        items = [(k, RESPONSE, last, rd.ids[2 * T - 1]) for k in range(procs)]
        call(fresh(ph == 2), items)                                        # warm-up
        dt = 0.0
        for _ in range(reps):
            hs = fresh(ph == 2)
            t0 = time.perf_counter()
            got = call(hs, items)
            dt += time.perf_counter() - t0
            assert got[::max(1, procs // 64)] == [want] * len(got[::max(1, procs // 64)]), f"phase {ph} differs from the oracle"
            for h in hs:
                engine.thdsa_proc_destroy(h)
        res[f"phase{ph}_procs_per_s"] = procs * reps / dt
        sets = [fresh(ph == 2) for _ in range(3)]
        res[f"phase{ph}_kernel_s"] = kernel_seconds([lambda hs=hs: call(hs, items) for hs in sets])
        for hs in sets:
            for h in hs:
                engine.thdsa_proc_destroy(h)
    if kind == "dsa":                                                      # 2t + 1 exponentiations per process on the host
        g, q = rd.g, rd.g["q"]
        lc = Libcrypto()
        with ThreadPoolExecutor(HOST_THREADS) as ex:
            t0 = time.perf_counter()
            list(ex.map(lambda a: lc.exp(g["g"], a, g["p"]), [(q - 3 - i) for i in range(procs * (2 * T + 1))]))
            dt = time.perf_counter() - t0
        res["host_calculate_r_per_s"] = procs / dt
    else:                                                                  # 2t + 1 scalar multiplications per process
        import multiprocessing
        from oracle import sss_oracle as S
        points = [S.p256_mul(k, S.P256_G) for k in (3, 5, 7)]
        with ProcessPoolExecutor(HOST_THREADS, mp_context=multiprocessing.get_context("spawn")) as ex:
            list(ex.map(_ecdh_chunk, [(1, points)] * HOST_THREADS))        # start the workers and import there: not timed
            t0 = time.perf_counter()
            list(ex.map(_ecdh_chunk, [(procs // HOST_THREADS + (i < procs % HOST_THREADS), points) for i in range(HOST_THREADS)]))
            dt = time.perf_counter() - t0
        res["host_calculate_r_per_s"] = procs / dt
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    e = Engine(0)
    out = {"gpu": gpu, "procs": a.procs, "n": N, "t": T, "host_threads": HOST_THREADS}
    for name in ("2048/256", "p256"):
        out[name] = run(e, name, a.procs, a.reps)
    e.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
