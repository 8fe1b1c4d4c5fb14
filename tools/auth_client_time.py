#!/usr/bin/env python3
"""Times bftq_auth_client_process_batch (K10, the client half of crypto/auth's password authentication) on the device,
and on the host the exponentiation a Go client makes 24 of per login: libcrypto's BN_mod_exp_mont_consttime through
ctypes on 8 threads (as tools/auth_time.py).  Prints one JSON line (also written to --out).

Workload: --sessions sessions per call at n = 10, k = 7, one whole login each: INITIATE, the 7 phase-0 answers (the 7th
completes the set), the 7 phase-1 answers, the 7 phase-2 answers, CIPHER_KEY.  The servers' answers come from K9 device
servers (one per session and peer) and are not timed.  Reported:
  - items per second through the call for each op (host clock around a call that ends in a device synchronise);
  - auth_pow_kernel's device time over a whole login round (torch.profiler's CUDA activity, a separate pass) and the
    2048-bit exponentiations per second it implies (17 per session run through it);
  - whole sessions per second through the five calls, against 8 host threads of libcrypto at 24 exponentiations per
    session (the host figure is derived from the measured exponentiation rate).
A sample of sessions is replayed on the oracle client (tests/auth_client_oracle.py) with the same a and a': every map and
cipher key must match byte for byte.  Card name and power limit from nvidia-smi, read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import auth_oracle as A  # noqa: E402
from auth_time import Libcrypto  # noqa: E402
from bftkv_b200 import Engine  # noqa: E402
from auth_client_oracle import OracleClient, wire_map  # noqa: E402

N, K = 10, 7
OPS = ("initiate", "phase0", "phase1", "phase2", "cipher_key")


def a_bytes(v: int) -> bytes:
    return v.to_bytes(256, "big")


class Round:
    """S fresh sessions logging in against their own K9 servers; each call() is one timed client call."""

    def __init__(self, e, S, params, pw, rng):
        self.e, self.S, self.rng = e, S, rng
        self.cl = [e.auth_client_create(pw, N, K) for _ in range(S)]
        self.srv = [[e.auth_server_create(params[i], b"proof %d" % i) for i in range(K)] for _ in range(S)]
        self.items = []                                           # per call: (idx, ops, peers, datas, rands)
        self.outs = []

    def call(self, idx, ops, peers, datas, rands):
        t0 = time.perf_counter()
        err, has, outs = self.e.auth_client_process_batch(self.cl, idx, ops, peers, datas, rands)
        dt = time.perf_counter() - t0
        assert not any(int(x) for x in err), "a client item failed"
        self.items.append((idx, ops, peers, datas, rands))
        self.outs.append((has, outs))
        return dt, has, outs

    def serve(self, phase, reqs, rands):
        """reqs[s][j]: session s's request to its server j; the answers, per session."""
        flat = [h for row in self.srv for h in row]
        err, outs = self.e.auth_server_respond_batch(flat, list(range(len(flat))), [phase] * len(flat),
                                                     [q for row in reqs for q in row], [r for row in rands for r in row])
        assert not any(int(x) for x in err)
        return [outs[s * K:(s + 1) * K] for s in range(self.S)]

    def run(self):
        S, rng, dts = self.S, self.rng, {}
        dts["initiate"], _, xs = self.call(list(range(S)), [-1] * S, [0] * S, [b""] * S, [a_bytes(rng.randrange(1, A.Q)) for _ in range(S)])
        yis = self.serve(0, [[x] * K for x in xs], [[b""] * K for _ in range(S)])
        idx = [s for s in range(S) for _ in range(K)]
        rands = [b"".join(a_bytes(rng.randrange(A.Q)) for _ in range(K)) if j == K - 1 else b"" for s in range(S) for j in range(K)]
        dts["phase0"], has, outs = self.call(idx, [0] * (S * K), list(range(K)) * S, [y for row in yis for y in row], rands)
        xis = [decode(outs[s * K + K - 1]) for s in range(S)]
        bis = self.serve(1, [[xis[s][j] for j in range(K)] for s in range(S)], [[a_bytes(rng.randrange(A.P)) for _ in range(K)] for _ in range(S)])
        dts["phase1"], has, outs = self.call(idx, [1] * (S * K), list(range(K)) * S, [b for row in bis for b in row], [b""] * (S * K))
        nis = [decode(outs[s * K + K - 1]) for s in range(S)]
        zis = self.serve(2, [[nis[s][j] for j in range(K)] for s in range(S)], [[rng.randbytes(12) for _ in range(K)] for _ in range(S)])
        dts["phase2"], has, outs = self.call(idx, [2] * (S * K), list(range(K)) * S, [z for row in zis for z in row], [b""] * (S * K))
        pis = [decode(outs[s * K + K - 1]) for s in range(S)]
        assert all(pis[s][j] == b"proof %d" % j for s in range(S) for j in range(K)), "a proof did not open"
        dts["cipher_key"], _, keys = self.call(list(range(S)), [-2] * S, [0] * S, [b""] * S, [b""] * S)
        return dts, keys

    def check(self, pw, sample):
        """Replays sessions `sample` on the oracle client: every output of every call must match."""
        for s in sample:
            o = OracleClient(pw, N, K)
            for (idx, ops, peers, datas, rands), (has, outs) in zip(self.items, self.outs):
                for i in (i for i, c in enumerate(idx) if c == s):
                    op, d, r = ops[i], datas[i], rands[i]
                    if op == -1:
                        want = o.initiate(int.from_bytes(r, "big"))
                    elif op == -2:
                        want = o.get_cipher_key()
                    else:
                        a2s = [int.from_bytes(r[256 * j:256 * j + 256], "big") for j in range(len(r) // 256)]
                        m = o.yi(d, peers[i], a2s) if op == 0 else o.bi(d, peers[i]) if op == 1 else o.zi(d, peers[i])
                        want = wire_map(m) if m is not None else b""
                    assert outs[i] == want, f"session {s} op {op} differs from the oracle"

    def close(self):
        for h in self.cl:
            self.e.auth_client_destroy(h)
        for row in self.srv:
            for h in row:
                self.e.auth_server_destroy(h)


def decode(b: bytes) -> list:
    """A map's values in order."""
    cnt, pos, out = int.from_bytes(b[:4], "big"), 4, []
    for _ in range(cnt):
        ln = int.from_bytes(b[pos + 8:pos + 16], "big")
        out.append(b[pos + 16:pos + 16 + ln])
        pos += 16 + ln
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-threads", type=int, default=8)
    ap.add_argument("--host-exps", type=int, default=2048)
    ap.add_argument("--sample", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    rng = random.Random(0xC11E)
    e = Engine(0)
    pw = b"password"
    params = A.generate_params(pw, N, K, A.Rng(0xC11E))
    S = a.sessions
    out = {"gpu": gpu, "sessions_per_call": S, "n": N, "k": K, "host_threads": a.host_threads}
    warm = Round(e, 8, params, pw, rng)
    warm.run()
    warm.close()
    tot = {op: 0.0 for op in OPS}
    for rep in range(a.reps):
        r = Round(e, S, params, pw, rng)
        dts, _ = r.run()
        if rep == 0:
            r.check(pw, range(0, S, max(1, S // max(1, a.sample))))
        r.close()
        for op in OPS:
            tot[op] += dts[op]
    items = {"initiate": S, "phase0": S * K, "phase1": S * K, "phase2": S * K, "cipher_key": S}
    for op in OPS:
        out[f"{op}_items_per_s"] = items[op] * a.reps / tot[op]
    login_s = sum(tot.values()) / a.reps
    out["login_seconds_per_call"] = login_s
    out["device_sessions_per_s"] = S / login_s
    # auth_pow_kernel's device time over one login round
    from torch.profiler import ProfilerActivity, profile
    r = Round(e, S, params, pw, rng)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r.run()
    pow_s = sum((ev.time_range.end - ev.time_range.start) * 1e-6 for ev in prof.events() if "auth_pow_kernel" in ev.name)
    r.close()
    out["pow_kernel_s_per_round"] = pow_s
    out["pow_kernel_exps_per_s"] = 17 * S / pow_s
    # host: libcrypto's constant-time exponentiation on 8 threads, 24 per session
    lc = Libcrypto()
    pb = A.i2b(A.P)
    xs = [A.i2b(rng.randrange(A.P)) for _ in range(a.host_exps)]
    es = [A.i2b(rng.randrange(A.Q)) for _ in range(a.host_exps)]
    with ThreadPoolExecutor(a.host_threads) as ex:
        t0 = time.perf_counter()
        got = list(ex.map(lambda i: lc.exp(xs[i], es[i], pb), range(a.host_exps)))
        host_dt = time.perf_counter() - t0
    for i in range(0, a.host_exps, max(1, a.host_exps // 8)):
        assert int.from_bytes(got[i], "big") == pow(int.from_bytes(xs[i], "big"), int.from_bytes(es[i], "big"), A.P)
    out["host_libcrypto_exp_per_s"] = a.host_exps / host_dt
    out["host_sessions_per_s_derived"] = a.host_exps / host_dt / 24
    e.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
