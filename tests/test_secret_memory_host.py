"""The key-material owners of bftkv_b200/csrc/device_secret.hpp on the CPU: tests/harness/secret_host.cpp builds the header
with g++ against a recording stand-in for the CUDA runtime (fake device blocks in host memory, every call logged, the n-th
call made to fail) and runs one scenario per entry point.  Also checks that the threshold and auth host files leave every
zeroing and freeing of secret device memory to those types."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
CUDA, NOMEM = "-2", "-5"                                           # BFTQ_ERR_CUDA, BFTQ_ERR_NOMEM


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libsecrethost.so")
    src = os.path.join(ROOT, "tests", "harness", "secret_host.cpp")
    deps = [src, os.path.join(ROOT, "bftkv_b200", "csrc", "device_secret.hpp")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        # -Bsymbolic: the harness's own operator delete serves its own frees only
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-I" + os.path.join(CUDA_HOME, "include"),
                               "-o", so, src])
    lib = ctypes.CDLL(so)
    for name in ("sh_release", "sh_upload", "sh_grow", "sh_scratch", "sh_wiped_vector", "sh_handles"):
        getattr(lib, name).restype = ctypes.c_char_p
    lib.sh_upload.argtypes = [ctypes.c_long]
    lib.sh_grow.argtypes = [ctypes.c_size_t, ctypes.c_size_t, ctypes.c_long]
    lib.sh_scratch.argtypes = [ctypes.c_long]
    return lib


def lines(raw):
    return [ln.split() for ln in raw.decode().splitlines()]


def section(log, start):
    """The log lines after the marker `-- start` up to the next marker."""
    i = next(k for k, ln in enumerate(log) if ln[:1] == ["--"] and " ".join(ln[1:]) == start)
    out = []
    for ln in log[i + 1:]:
        if ln[:1] == ["--"]:
            break
        out.append(ln)
    return out


def scrub(dev, ptr, size):
    """The release of one secret block: set its device, zero all of it, synchronise, free it (all zero by then)."""
    return [["setDevice", str(dev)], ["memset", ptr, "0", str(size)], ["sync"], ["free", ptr, "zero=1"]]


def frees(log):
    return [ln[1] for ln in log if ln[0] == "free"]


@pytest.mark.parametrize("how", ["reset", "destructor", "move_assign"])
def test_release_zeroes_then_frees_each_block_once(host, how):
    log = lines(host.sh_release({"reset": 0, "destructor": 1, "move_assign": 2}[how]))
    a, b = next(ln for ln in log if ln[0] == "A")[1::2]
    head = 20
    assert ["malloc", a, str(head + 24)] in log and ["malloc", b, str(head + 8)] in log
    released = section(log, "release")
    assert released[:4] == scrub(3, a, head + 24)
    after = released[4]
    if how == "move_assign":
        assert after == ["after", "a=" + b, "b=0"]
    else:
        assert after == ["after", "a=0", "b=" + b]
    assert section(log, "scope end") == scrub(5, b, head + 8)
    assert sorted(frees(log)) == sorted([a, b])                  # exactly once per block


def test_upload_keeps_nothing_when_a_step_fails(host):
    clean = lines(host.sh_upload(-1))
    calls = [ln for ln in clean[:clean.index(["--", "scope", "end"])] if ln[0] in ("setDevice", "malloc", "memcpy")]
    assert [c[0] for c in calls] == ["setDevice", "malloc", "memcpy", "memcpy"]
    assert ["rc", "0", "held=1", "bytes=44"] in clean and ["contents", "1"] in clean
    blk = calls[1][1]
    for n, op in enumerate(c[0] for c in calls):
        if op == "setDevice":
            continue
        log = lines(host.sh_upload(n))
        assert ["FAIL", op] in log
        rc = next(ln for ln in log if ln[0] == "rc")
        assert rc[2:] == ["held=0", "bytes=0"]
        assert rc[1] == (NOMEM if op == "malloc" else CUDA)
        if op == "memcpy":                                         # the block was made: zeroed and freed before returning
            after_fail = log[log.index(["FAIL", op]) + 1:]
            assert after_fail[:4] == scrub(2, blk, 44)
        assert section(log, "scope end") == []


def test_grow_keeps_contents_and_zeroes_the_old_block(host):
    log = lines(host.sh_grow(64, 128, -1))
    old = next(ln for ln in log if ln[0] == "old")[1]
    new = next(ln for ln in log if ln[0] == "malloc")[1]
    body = [ln for ln in log if ln[0] not in ("old",)]
    assert body[:4] == [["setDevice", "7"], ["malloc", new, "128"], ["memset", new, "0", "128"], ["memcpy", new, old, "64", "d2d"]]
    assert body[4:8] == scrub(7, old, 64)
    assert next(ln for ln in log if ln[0] == "rc") == ["rc", "0", "now", new, "128", "kept=1", "zero_tail=1"]
    assert section(log, "scope end") == scrub(7, new, 128)
    # from nothing: one zeroed block, no copy and no synchronisation
    log = lines(host.sh_grow(0, 1024, -1))
    new = next(ln for ln in log if ln[0] == "malloc")[1]
    assert [ln for ln in log if ln[0] not in ("old", "rc", "--")][:3] == [["setDevice", "7"], ["malloc", new, "1024"], ["memset", new, "0", "1024"]]
    assert [ln for ln in log if ln[0] in ("sync", "free")] == [["sync"], ["free", new, "zero=1"]]      # the final reset only


@pytest.mark.parametrize("step", [1, 2, 3])     # 1: the allocation, 2: zeroing the new block, 3: the copy
def test_grow_failure_leaves_the_old_block_intact(host, step):
    log = lines(host.sh_grow(64, 128, step))
    old = next(ln for ln in log if ln[0] == "old")[1]
    assert ["FAIL", ["malloc", "memset", "memcpy"][step - 1]] in log
    rc = next(ln for ln in log if ln[0] == "rc")
    assert rc[1] == (NOMEM if step == 1 else CUDA) and rc[2:] == ["now", old, "64", "kept=1", "zero_tail=1"]
    grown = log[:log.index(rc)]
    made = [ln[1] for ln in grown if ln[0] == "malloc"]
    if made:                                                       # the new block is zeroed and freed, the old one untouched
        assert grown[-4:] == scrub(7, made[0], 128)
    assert old not in frees(grown) and ["memset", old, "0", "64"] not in grown
    assert section(log, "scope end") == scrub(7, old, 64)


def test_grow_reports_a_failure_releasing_the_old_block(host):
    log = lines(host.sh_grow(64, 128, 5))                          # zeroing the old block fails after the copy
    old = next(ln for ln in log if ln[0] == "old")[1]
    new = next(ln for ln in log if ln[0] == "malloc")[1]
    assert log[log.index(["memcpy", new, old, "64", "d2d"]) + 1:][:4] == [["setDevice", "7"], ["FAIL", "memset"], ["sync"], ["free", old, "zero=0"]]
    rc = next(ln for ln in log if ln[0] == "rc")
    assert rc[1] == CUDA and rc[2:] == ["now", new, "128", "kept=1", "zero_tail=1"]
    assert section(log, "scope end") == scrub(7, new, 128)


def scratch_segments(log):
    segs = {ln[1]: (int(ln[2], 0), int(ln[3])) for ln in log if ln[0] == "seg"}
    base = int(next(ln for ln in log if ln[0] == "malloc")[1], 0)
    return base, segs


def test_scratch_layout_zeroing_uploads_downloads_and_scrub(host):
    log = lines(host.sh_scratch(-1))
    base, segs = scratch_segments(log)
    total = int(next(ln for ln in log if ln[0] == "malloc")[2])
    order = sorted(segs.values())
    for k, (ptr, size) in enumerate(order):
        assert (ptr - base) % 256 == 0
        nxt = order[k + 1][0] if k + 1 < len(order) else base + total
        assert ptr + size <= nxt                                   # disjoint, in declaration order
    assert total == sum((s + 255) // 256 * 256 for _, s in segs.values())
    assert ["zeroed", "1"] in log
    ops = [ln for ln in log if ln[0] in ("setDevice", "malloc", "memset", "memcpy", "sync", "free")]
    b = hex(base)
    assert ops[:3] == [["setDevice", "4"], ["malloc", b, str(total)], ["memset", b, "0", str(total)]]
    copies = [ln for ln in ops if ln[0] == "memcpy"]
    assert [(int(c[1], 0), c[3], c[4]) for c in copies[:3]] == [(segs["a"][0], "400", "h2d"), (segs["b"][0], "1", "h2d"), (segs["c"][0], "200", "h2d")]
    assert [(int(c[2], 0), c[3], c[4]) for c in copies[3:]] == [(segs["out"][0], "300", "d2h")]      # only what was asked
    assert ["downloaded", "300", "untouched_after=1"] in log
    assert section(log, "scope end") == scrub(4, b, total)
    assert ops.count(["sync"]) == 1


def test_scratch_is_scrubbed_when_a_copy_fails(host):
    clean = lines(host.sh_scratch(-1))
    copies = [k for k, ln in enumerate(ln for ln in clean if ln[0] in ("setDevice", "malloc", "memset", "memcpy", "sync", "free"))
              if ln[0] == "memcpy"]
    for n in copies:                                               # every upload, and the download
        log = lines(host.sh_scratch(n))
        assert ["FAIL", "memcpy"] in log and ["run", "1"] in log
        base = next(ln for ln in log if ln[0] == "malloc")
        assert section(log, "scope end") == scrub(4, base[1], int(base[2]))
    log = lines(host.sh_scratch(1))                                # the allocation fails: nothing to release
    assert ["FAIL", "malloc"] in log and ["prepare", "failed"] in log and not frees(log)
    log = lines(host.sh_scratch(2))                                # zeroing fails: the block is released at once
    base = next(ln for ln in log if ln[0] == "malloc")
    at = log.index(["FAIL", "memset"])
    assert log[at + 1:] == scrub(4, base[1], int(base[2])) + [["prepare", "failed"]]


def test_wiped_vector_blocks_are_zero_when_freed(host):
    log = lines(host.sh_wiped_vector())
    grown = [ln[2] for ln in log if ln[0] == "grow"]          # "grow from <block> <bytes>"
    assert len(grown) >= 4
    freed = [ln[1:] for ln in log if ln[0] == "hostfree"]
    destroyed = next(ln for ln in log if ln[0] == "destroy")[1]
    assert [f[0] for f in freed] == grown + [destroyed]
    assert all(f[1] == "zero=1" for f in freed)


def test_handle_list_shutdown_detaches_each_live_handle_once(host):
    log = lines(host.sh_handles())
    blk = {ln[1]: ln[2] for ln in log if ln[0] == "handle"}
    assert section(log, "destroy 0") == scrub(1, blk["0"], 24)
    assert section(log, "shutdown") == scrub(1, blk["1"], 28) + scrub(1, blk["2"], 32) + [["detached", "1", "1"]]
    assert section(log, "destroy 1 2") == []                       # after shutdown, destroy frees host state only


@pytest.mark.parametrize("name", ["thrsa_host.inc", "thdsa_host.inc", "auth_host.inc"])
def test_handle_files_leave_device_release_to_the_owners(name):
    src = open(os.path.join(ROOT, "bftkv_b200", "csrc", name)).read()
    assert not re.search(r"\bcudaFree\(", src)
    assert not re.search(r"\bcudaMemset\(", src)
