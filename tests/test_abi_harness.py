"""include/bftq.h through a C compiler: tests/harness/abi_smoke.c (the call sequence of the Go shim, in plain C) is built
with gcc -std=c11 -Wall -Wextra -Werror against the header and libbftq.so and run on a fixture written here.
CPU suite: it builds, loads, and bftq_init fails loudly without a device (exit 77).  GPU suite: every call's result
matches the fixture's expectations (exit 0)."""
import os
import struct
import subprocess

import numpy as np
import pytest

from bftkv_b200 import workload
from oracle import packet_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "abi_smoke.c")


@pytest.fixture(scope="session")
def harness_exe(built, tmp_path_factory):
    """The harness, built once per session into a temporary directory: the tree may not be writable by the test user."""
    exe = str(tmp_path_factory.mktemp("harness") / "abi_smoke")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-O1", "-I" + os.path.join(ROOT, "include"), "-o", exe, SRC,
                           "-L" + os.path.join(ROOT, "bftkv_b200"), "-lbftq", "-Wl,-rpath," + os.path.join(ROOT, "bftkv_b200")])
    return exe


def u64(v):
    return struct.pack("<Q", int(v))


def blob(items):
    off = np.zeros(len(items) + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in items])
    return b"".join(items), off.tobytes()


def write_fixture(path):
    w = workload.make_pgp_verify_batch(96, n_keys=4, corrupt_rate=0.1, unknown_rate=0.05)
    out = [u64(len(w["keyring"])), w["keyring"], u64(4)]
    tb, to = blob(w["tbs"])
    sb, so = blob(w["sigs"])
    out += [u64(96), u64(len(tb)), u64(len(sb)), tb, to, sb, so, w["expect_ok"].astype(np.uint8).tobytes()]
    # collective signatures over a 4-clique (f = 1, min 4, AUTH threshold 3, suff 3)
    keys = workload.load_keys(4)
    kids = w["key_ids"]
    out += [u64(4), np.array(kids, np.uint64).tobytes(), u64(1), u64(4), u64(3), u64(3)]
    tbs = workload.tbs_packet(b"x" * 16, b"v" * 32, 9)
    sig = [workload.sig_packet_v4(keys[i], kids[i], 8, tbs, 0x5F000000 + i) for i in range(4)]
    bad = bytearray(sig[1]); bad[-7] ^= 2
    streams = [sig[0] + sig[1] + sig[2], sig[0] + bytes(bad) + sig[2], sig[0] + bytes(bad) + sig[2] + sig[3], sig[3] * 3, b"", b"\x01" + sig[0] + b"\x02" + sig[1] + sig[2]]
    expect = [1, 0, 1, 1, 0, 1]
    cb, co = blob([tbs] * len(streams))
    sb2, so2 = blob(streams)
    out += [u64(len(streams)), u64(len(cb)), u64(len(sb2)), cb, co, sb2, so2, bytes(expect)]
    # one read operation from raw answers: READ threshold of this descriptor is 3, so the third good answer decides
    plain = packet_oracle.serialize(b"x" * 16, b"v" * 32, 9)
    nonces = [bytes([i + 1]) * 8 for i in range(4)]
    msgs = [workload.make_transport_message(keys[i], kids[i], plain, nonces[i]) for i in range(4)]
    m1 = bytearray(msgs[1]); m1[-9] ^= 4
    msgs[1] = bytes(m1)
    mb, mo = blob(msgs)
    out += [u64(4), u64(len(mb)), u64(8), mb, mo, np.array(kids, np.uint64).tobytes(), b"".join(nonces), bytes([1, 0, 1, 1]), u64(0), u64(0), u64(4)]
    open(path, "wb").write(b"".join(out))


def test_header_compiles_as_c_and_fails_loudly_without_gpu(harness_exe, tmp_path):
    import torch
    fx = str(tmp_path / "fixture.bin")
    write_fixture(fx)
    r = subprocess.run([harness_exe, fx], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert r.returncode == 77, (r.returncode, r.stderr)        # BFTQ_ERR_NO_DEVICE: there is no CPU fallback
    else:
        assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_c_harness_drives_the_shim_sequence(harness_exe, tmp_path):
    fx = str(tmp_path / "fixture.bin")
    write_fixture(fx)
    r = subprocess.run([harness_exe, fx], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "abi_smoke ok" in r.stdout
