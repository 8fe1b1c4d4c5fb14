"""Times bftq_read_encrypted_responses_batch (raw wire answers in, Client.Read's decisions out) against
bftq_message_decrypt_batch alone on the same raw answers, alternating, and prints one JSON line.

    python tools/read_encrypted_time.py [--ops 8192] [--replicas 16] [--pairs 3] [--profile DIR]

The input is bench.py's configs[2] shape: ops x 16 replicas under HARD_MIX, about 3.9 kB answers, each encrypted to the
client as Message.Encrypt writes it (AES-128), from page-locked blobs.  The decrypt-alone call is a lower bound on the
two-step composition (decrypt, then bftq_read_responses_batch) a caller needs without the new entry point.  Statuses are
checked against the workload's expectation (good / bad), decisions against c_oracle.read_decide_batch.
--profile DIR: a separate torch.profiler run of one call, per-kernel device times into DIR and the JSON line, and K6a's
executed word-MACs against bftq_measure_int_peak."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bftkv_b200 import Engine, workload  # noqa: E402
from bftkv_b200.crypto_gpu import Keyring, _blob, read_encrypted_responses_batch  # noqa: E402
from oracle import c_oracle  # noqa: E402

# K6a per decryption: two 1024-bit CRT halves of 1298 Montgomery products each (2 to reduce c, 1 for one, 14 table
# entries, 256 windows x (4 squarings + 1 product), 1 to leave Montgomery form) at 2 * 32^2 word-MACs, plus Garner's
# 1024-bit and 2048-bit products (2 * 64^2)
K6A_MACS = 2 * 1298 * 2 * 32 * 32 + 2 * 32 * 32 + 2 * 64 * 64
KERNELS = {"K6p": "pkesk_seipd_parse_kernel", "K6a": "rsa_crt_decrypt_kernel", "K6q": "front_gate_kernel", "K6b": "seipd_decrypt_kernel",
           "K0m": "msg_parse_digest_kernel", "K1": "rsa_verify", "K2m": "read_responses_kernel", "gather": "plain_gather_kernel"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, pl, clk = [x.strip() for x in q.strip().split("\n")[0].split(",")]
    return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=8192)
    ap.add_argument("--replicas", type=int, default=16)
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    M, Rn = a.ops, a.replicas
    ra = workload.make_read_answers(M, Rn, mix=workload.HARD_MIX)
    ck = workload.load_keys(Rn + 1)[Rn]
    cblock, cid = workload.pgp_public_key_block(ck, workload._private_key(ck), b"client <client@bftq.test>")
    raws, _ = workload.encrypt_answers(ra["msgs"], ck, cid)
    eng = Engine(0)
    kr = Keyring(eng)
    kr.register(cblock, priv=True)
    kr.register(ra["keyring"])
    assert kr.register_private(workload.secret_key_packet(ck)) == 1
    blob, off = _blob(raws)
    pin = (eng.host_copy(blob), eng.host_copy(off))
    N = len(raws)
    qcs = [(5, 16, 6, 11, ra["ids"])]

    def read(want_plain=True):
        return read_encrypted_responses_batch(kr, qcs, ra["op_off"], ra["peer_ids"], None, ra["nonces"], pre_status=ra["pre_status"], blobs=pin,
                                              want_plain=want_plain)

    err, by, fl = np.zeros(N, np.int32), np.zeros(N, np.uint64), np.zeros(N, np.uint8)
    pl_, nl_ = np.zeros(N, np.uint32), np.zeros(N, np.uint32)
    pb, nb = eng.host_copy(np.zeros(len(blob), np.uint8)), eng.host_copy(np.zeros(len(blob), np.uint8))
    p = lambda x: C.c_void_p(x.ctypes.data)

    def decrypt_alone():
        from bftkv_b200 import _lib
        _lib.check(kr._lib.bftq_message_decrypt_batch(kr._h, p(pin[0]), p(pin[1]), N, p(err), p(by), p(fl), p(pb), p(pl_), p(nb), p(nl_)))

    got = read()
    decrypt_alone()
    st = got["status"]
    assert np.array_equal(st != 0, ra["expect_status"] != 0), "good / bad statuses differ from the workload's expectation"
    dec, win, at = c_oracle.read_decide_batch(qcs, ra["op_off"], ra["peer_ids"], st, got["ts"], ra["value_id"])
    assert np.array_equal(dec, got["decision"]) and np.array_equal(win, got["winner"]) and np.array_equal(at, got["decided_at"]), "decisions differ from the oracle"
    t_read, t_dec, t_noplain = [], [], []
    s0 = eng.stats()
    for _ in range(a.pairs):
        t0 = time.perf_counter(); read(); t_read.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); decrypt_alone(); t_dec.append(time.perf_counter() - t0)
    s1 = eng.stats()
    for _ in range(a.pairs):                       # without the plain-text output (no gather, no Python-side slicing)
        t0 = time.perf_counter(); read(want_plain=False); t_noplain.append(time.perf_counter() - t0)
    tr, td = statistics.median(t_read), statistics.median(t_dec)
    res = dict(card(), metric="read_encrypted_responses", answers=N, ops=M, bytes_per_answer=int(off[-1]) // max(N, 1),
               read_encrypted_ms=[round(x * 1e3, 2) for x in t_read], decrypt_alone_ms=[round(x * 1e3, 2) for x in t_dec],
               read_encrypted_no_plain_ms=[round(x * 1e3, 2) for x in t_noplain],
               answers_per_s=N / tr, ops_per_s=M / tr, speedup_vs_decrypt_alone=td / tr,
               h2d_gb_per_s=int(off[-1]) / tr / 1e9,
               gpu_decided=(s1["msg_gpu_items"] - s0["msg_gpu_items"]) // a.pairs, host_decided=(s1["msg_host_items"] - s0["msg_host_items"]) // a.pairs)
    if a.profile:
        import torch
        os.makedirs(a.profile, exist_ok=True)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            read()
            torch.cuda.synchronize()
        per = {k: 0.0 for k in KERNELS}
        total = 0.0
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            for k, sub in KERNELS.items():
                if sub in ev.name:
                    per[k] += us / 1e3
                    total += us / 1e3
        prof.export_chrome_trace(os.path.join(a.profile, "read_encrypted_trace.json"))
        peak = eng.measure_int_peak()
        k6a_s = per["K6a"] / 1e3
        res.update(kernel_ms={k: round(v, 3) for k, v in per.items()}, kernels_sum_ms=round(total, 3),
                   e2e_over_kernel_sum=tr * 1e3 / total if total else None,
                   e2e_no_plain_over_kernel_sum=statistics.median(t_noplain) * 1e3 / total if total else None,
                   k6a_decryptions_per_s=N / k6a_s if k6a_s else None,
                   k6a_word_macs_per_s=K6A_MACS * N / k6a_s if k6a_s else None, int_peak_macs_per_s=peak,
                   k6a_frac_of_int_peak=K6A_MACS * N / k6a_s / peak if k6a_s else None)
        with open(os.path.join(a.profile, "kernels.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    kr.close()
    eng.close()


if __name__ == "__main__":
    main()
