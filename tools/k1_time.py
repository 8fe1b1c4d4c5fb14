"""Times K1 alone (device-resident inputs, CUDA events on the launch streams):
python tools/k1_time.py [items] — prints verifies/s on one stream and on two.  BFTQ_LIB_PATH selects another build of
the library for an A/B run."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bftkv_b200 import Engine, workload  # noqa: E402

N = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
w = workload.make_verify_batch(N, 16)
dev = torch.device("cuda", 0)
eng = Engine(0)
eng.register_rsa_keys([k["n"] for k in w["keys"]], [k["e"] for k in w["keys"]])
copies = 8
d = [(torch.from_numpy(w["key_idx"].astype(np.int32)).to(dev), torch.from_numpy(w["sig"]).to(dev), torch.from_numpy(w["digest"]).to(dev),
      torch.empty(N, dtype=torch.uint8, device=dev)) for _ in range(copies)]
res = {}
for ns in (1, 2):
    streams = [torch.cuda.Stream(device=dev) for _ in range(ns)]
    for i in range(6):
        c = d[i % copies]
        eng.rsa_verify_batch_dev(c[0], c[1], c[2], N, c[3], stream=streams[i % ns].cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = 40
    e0.record(streams[0])
    for s in streams[1:]:
        s.wait_event(e0)
    for i in range(steps):
        c = d[i % copies]
        eng.rsa_verify_batch_dev(c[0], c[1], c[2], N, c[3], stream=streams[i % ns].cuda_stream)
    for s in streams[1:]:
        streams[0].wait_stream(s)
    e1.record(streams[0])
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res["streams%d" % ns] = {"ms": round(ms, 4), "Mverifies_s": round(N / ms / 1e3, 2)}
ok = bool(np.array_equal(d[0][3].cpu().numpy(), w["expect"]))
print(json.dumps({"ok": ok, **res}))
eng.close()
