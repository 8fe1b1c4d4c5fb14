"""K1b on the device over tests/golden/ed25519_adversarial.json: every adversarial row through the window-table path
(ed25519_bases / multiples build the tables, accumulate + finish verify) and through the table-free kernel, each
rejected or edge row at every position of a finish-kernel inversion group and in every lane of an accumulate block, and
both encodings of one point as two cache slots.  The expected status is Go's crypto/ed25519.Verify (0 valid, 1 invalid)."""
import ctypes as C
import json
import os
import random
from contextlib import contextmanager

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
P = 2 ** 255 - 19
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vec():
    rows = json.load(open(os.path.join(HERE, "golden", "ed25519_adversarial.json")))["rows"]
    keys = sorted({r["a"] for r in rows})
    kix = {k: i for i, k in enumerate(keys)}
    return {
        "rows": rows,
        "pk": np.frombuffer(b"".join(bytes.fromhex(k) for k in keys), np.uint8).reshape(-1, 32).copy(),
        "kidx": np.array([kix[r["a"]] for r in rows], np.uint32),
        "sig": np.frombuffer(b"".join(bytes.fromhex(r["sig"]) for r in rows), np.uint8).reshape(-1, 64).copy(),
        "msg": np.frombuffer(b"".join(bytes.fromhex(r["msg"]) for r in rows), np.uint8).reshape(-1, 32).copy(),
        "expect": np.array([0 if r["expect"] else 1 for r in rows], np.uint8),
    }


@contextmanager
def _engine(tables):
    """A fresh engine (an empty table cache) with BFTQ_ED25519_TABLES set for its creation; the variable is restored."""
    from bftkv_b200 import Engine
    old = os.environ.get("BFTQ_ED25519_TABLES")
    os.environ["BFTQ_ED25519_TABLES"] = "1" if tables else "0"
    try:
        eng = Engine(0)
    finally:
        if old is None:
            os.environ.pop("BFTQ_ED25519_TABLES", None)
        else:
            os.environ["BFTQ_ED25519_TABLES"] = old
    try:
        yield eng
    finally:
        eng.close()


def _replicated(vec, sel=None, per_key=32, seed=1):
    """Row indices (of `sel`, default all) repeated so that every key has at least `per_key` signatures, shuffled: a batch
    that pays for a table per key."""
    sel = range(len(vec["rows"])) if sel is None else sel
    by_key = {}
    for i in sel:
        by_key.setdefault(int(vec["kidx"][i]), []).append(i)
    idx = []
    for k in sorted(by_key):
        g = by_key[k]
        idx += [g[t % len(g)] for t in range(max(per_key, len(g)))]
    random.Random(seed).shuffle(idx)
    return np.array(idx, np.int64)


def _run(eng, vec, idx):
    """Verifies rows `idx` with a key table of just the keys they use (every key passed counts as one the batch brings)."""
    used, kidx = np.unique(vec["kidx"][idx], return_inverse=True)
    launches = eng.stats()["launches"]
    got = eng.ed25519_verify_batch(vec["pk"][used].copy(), kidx.astype(np.uint32), vec["sig"][idx].copy(), vec["msg"][idx].copy())
    return got, eng.stats()["launches"] - launches


def _check(got, vec, idx):
    bad = np.nonzero(got != vec["expect"][idx])[0]
    assert bad.size == 0, [(int(p), vec["rows"][idx[p]]["tag"], vec["rows"][idx[p]]["note"], int(got[p])) for p in bad[:10]]


def test_table_path_every_row(vec):
    idx = _replicated(vec)
    with _engine(True) as eng:
        got, dl = _run(eng, vec, idx)
        _check(got, vec, idx)
        assert dl == 6                                   # base-point table 2, key tables 2, accumulate and finish 2
        got, dl = _run(eng, vec, idx)
        _check(got, vec, idx)
        assert dl == 2                                   # every key cached: accumulate + finish only
        # every row once, all keys cached: still the table path
        one = np.arange(len(vec["rows"]))
        got, dl = _run(eng, vec, one)
        _check(got, vec, one)
        assert dl == 2


def test_table_free_path_every_row(vec):
    with _engine(False) as eng:
        for idx in (np.arange(len(vec["rows"])), _replicated(vec, seed=2)):
            got, dl = _run(eng, vec, idx)
            _check(got, vec, idx)
            assert dl == 1                               # ed25519_verify_kernel only


def _specials(vec):
    return [i for i, r in enumerate(vec["rows"]) if not r["expect"] or r["tag"] in ("S_edge", "digit_edge")]


def test_placement_in_inversion_groups(vec):
    """Each rejected or edge row at position j = 0..7 of a finish-kernel inversion group (items t + j n_pad / 8 share one
    inversion), alone among accepted rows of its group, at ragged batch sizes; every call on the table path."""
    specials = _specials(vec)
    filler = [i for i, r in enumerate(vec["rows"]) if r["expect"]]
    with _engine(True) as eng:
        _run(eng, vec, _replicated(vec))                 # every key cached
        seen = {}
        for n in (1, 7, 513, 4097):
            n_pad = (n + 511) // 512 * 512
            thr = n_pad // 8
            base = np.array([filler[(7 * i + n) % len(filler)] for i in range(n)], np.int64)
            for j in range(8):
                groups = [t for t in range(thr) if t + j * thr < n]
                for c in range(0, len(specials), max(len(groups), 1)):
                    chunk = specials[c:c + len(groups)]
                    if not chunk:
                        break
                    idx = base.copy()
                    for t, s in zip(groups, chunk):
                        idx[t + j * thr] = s
                        seen.setdefault(s, set()).add(j)
                    got, dl = _run(eng, vec, idx)
                    _check(got, vec, idx)
                    assert dl == 2
        assert all(seen[s] == set(range(8)) for s in specials)


def test_placement_in_every_lane(vec):
    """Each rejected or edge row in every lane of a 128-thread accumulate block (batches of 4097 accepted rows otherwise)."""
    specials = _specials(vec)
    assert len(specials) <= 32 * 128
    filler = [i for i, r in enumerate(vec["rows"]) if r["expect"]]
    n = 4097
    base = np.array([filler[(5 * i) % len(filler)] for i in range(n)], np.int64)
    with _engine(True) as eng:
        _run(eng, vec, _replicated(vec))
        for rnd in range(128):
            idx = base.copy()
            for s_i, s in enumerate(specials):
                idx[(s_i % 32) * 128 + (s_i // 32 + rnd) % 128] = s
            got, dl = _run(eng, vec, idx)
            _check(got, vec, idx)
            assert dl == 2


def test_two_encodings_of_one_point_are_two_slots(vec):
    """The identity (01 00..00, y = p + 1, -0, both) and (0, -1) (canonical and -0) under the same batch: a key's table is
    found by its 32 bytes, so the other encodings are built as slots of their own, and each decides as Go does."""
    le = lambda v: v.to_bytes(32, "little").hex()
    canon = {le(1), le(P - 1)}
    other = {le(P + 1), le(1 | 1 << 255), le((P + 1) | 1 << 255), le((P - 1) | 1 << 255)}
    rows = vec["rows"]
    sel_c = [i for i, r in enumerate(rows) if r["a"] in canon]
    sel_o = [i for i, r in enumerate(rows) if r["a"] in other]
    assert len({rows[i]["a"] for i in sel_c}) == 2 and len({rows[i]["a"] for i in sel_o}) == 4
    assert any(rows[i]["expect"] for i in sel_o) and not all(rows[i]["expect"] for i in sel_o)
    with _engine(True) as eng:
        idx = _replicated(vec, sel_c)
        got, dl = _run(eng, vec, idx)
        _check(got, vec, idx)
        assert dl == 6                                   # base-point table 2, key tables 2, accumulate and finish 2
        idx = _replicated(vec, sel_c + sel_o, seed=3)
        got, dl = _run(eng, vec, idx)
        _check(got, vec, idx)
        assert dl == 4                                   # the four other encodings are new keys: a table build
        got, dl = _run(eng, vec, idx)
        _check(got, vec, idx)
        assert dl == 2


def test_device_resident_entry_point(vec):
    """bftq_ed25519_verify_batch_dev on device buffers and a caller's stream, as the benchmark calls it."""
    import torch
    from bftkv_b200 import _lib as L_
    idx = _replicated(vec, seed=4)
    dev = torch.device("cuda", 0)
    d_idx, d_sig, d_msg = (torch.from_numpy(np.ascontiguousarray(a)).to(dev)
                           for a in (vec["kidx"][idx].astype(np.int32), vec["sig"][idx], vec["msg"][idx]))
    d_st = torch.full((len(idx),), 0xEE, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    with _engine(True) as eng:
        for _ in range(2):                               # builds the tables, then reads them
            L_.check(eng._lib.bftq_ed25519_verify_batch_dev(eng._h, vec["pk"].ctypes.data_as(C.c_void_p), vec["pk"].shape[0],
                                                            C.c_void_p(d_idx.data_ptr()), C.c_void_p(d_sig.data_ptr()),
                                                            C.c_void_p(d_msg.data_ptr()), len(idx), C.c_void_p(d_st.data_ptr()),
                                                            C.c_void_p(stream.cuda_stream)))
            stream.synchronize()
            _check(d_st.cpu().numpy(), vec, idx)
            d_st.fill_(0xEE)
            torch.cuda.synchronize()
