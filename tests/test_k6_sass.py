"""CPU suite: the K6 kernels (msg_decrypt.cuh) hold private-key material and session keys; none of it may go through
local memory, which is never scrubbed.  No compute."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _functions(so):
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    return {b.split("\n", 1)[0].strip(): b for b in sass.split("Function :")[1:]}


def test_k6_kernels_use_no_local_memory(built):
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    fns = _functions(so)
    for kernel in ("rsa_crt_decrypt_kernel", "seipd_decrypt_kernel"):
        bodies = [b for name, b in fns.items() if kernel in name]
        assert bodies, kernel
        for b in bodies:
            assert "LDL" not in b and "STL" not in b, f"{kernel} spills to local memory"
    usage = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout.split("\n")
    for i, line in enumerate(usage):
        if "rsa_crt_decrypt_kernel" in line or "seipd_decrypt_kernel" in line:
            assert "STACK:0 " in usage[i + 1] and "LOCAL:0 " in usage[i + 1], usage[i + 1]
