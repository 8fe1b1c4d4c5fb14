"""The share-combine kernels on the device against tests/golden/threshold_edges.json (Python integers through
oracle/sss_oracle.py) and against the host build of the same K3 code (tests/harness/lagrange_host.cpp):
K3 lagrange_combine_kernel<8/16/32/64>, K5 modexp_kernel<W> / modprod_kernel<W>, auth.calculateSharedSecret
(lagrange_exp_product_batch) with q in every K3 limb class, and dsa.CalculateR on L1024/N160, L2048/N224 and
L2048/N256 including sums v_i lambda_i that are 0 mod q (status 3; Go's ModInverse returns nil there and its r is 1)."""
import ctypes
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

from oracle import sss_oracle as sss
import threshold_edges as te

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
mlen_of, limb_class = te.mlen_of, te.limb_class


@pytest.fixture(scope="module")
def vec():
    return te.load()


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    so_path = tmp_path_factory.mktemp("lagrange") / "liblagrange.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-o", str(so_path), os.path.join(HERE, "harness", "lagrange_host.cpp")], check=True)
    return ctypes.CDLL(str(so_path))


def group_arrays(vec, g):
    m, k, items = te.k3_items(g, vec["k3_moduli"])
    mlen = mlen_of(m)
    x = np.array([xs for xs, _ in items], np.int32).reshape(-1, k)
    y = np.frombuffer(b"".join(v.to_bytes(mlen, "big") for _, ys in items for v in ys), np.uint8).reshape(-1, k, mlen).copy()
    return m, k, mlen, x, y


def digest_of(st, out):
    """te.digest of device results: status bytes, out rows."""
    return te.digest(st.tolist(), [int.from_bytes(bytes(o), "big") for o in out], out.shape[1])


def test_k3_every_vector_every_limb_class(engine, vec, hostlib):
    """lagrange_combine_batch on every committed K3 vector: statuses and outputs equal the JSON (status list and output
    digest, which the CPU suite checks against sss_oracle) and the host build of lagrange_item byte for byte.  Every
    limb class runs, lagrange_combine_kernel<16> and <32> included."""
    ran = Counter()
    for g in vec["k3"]:
        m, k, mlen, x, y = group_arrays(vec, g)
        out, st = engine.lagrange_combine_batch(m, x, y)
        assert st.tolist() == g["status"], g["tag"]
        assert digest_of(st, out) == g["digest"], g["tag"]
        assert not out[st != 0].any(), g["tag"]
        hout = np.zeros_like(out)
        hst = np.zeros_like(st)
        hostlib.lagrange_combine_host(m.to_bytes(mlen, "big"), ctypes.c_uint32(mlen), ctypes.c_uint32(k), x.ctypes.data_as(ctypes.c_void_p),
                                      y.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(x.shape[0]), hout.ctypes.data_as(ctypes.c_void_p),
                                      hst.ctypes.data_as(ctypes.c_void_p), None)
        assert np.array_equal(hout, out) and np.array_equal(hst, st), g["tag"]
        for s in st.tolist():
            ran[(limb_class(mlen), s)] += 1
    for L in (8, 16, 32, 64):
        assert ran[(L, 0)] >= 30 and ran[(L, 3)] >= 15, ran


def test_k3_all_vectors_in_one_batch_per_modulus_and_dev_entry(engine, vec):
    """The k = 10 groups of each limb class concatenated per modulus into one batch (items at every lane of a block),
    and lagrange_combine_batch_dev (device pointers, caller's stream) on a subset."""
    import torch
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    checked = Counter()
    for g in vec["k3"]:
        if g["k"] != 10:
            continue
        m, k, mlen, x, y = group_arrays(vec, g)
        want_out, want_st = engine.lagrange_combine_batch(m, x, y)
        reps = 40                                               # 280 items: three blocks of 128 threads, the last partial
        X, Y = np.tile(x, (reps, 1)), np.tile(y, (reps, 1, 1))
        out, st = engine.lagrange_combine_batch(m, X, Y)
        assert digest_of(want_st, want_out) == g["digest"], g["tag"]
        assert np.array_equal(out, np.tile(want_out, (reps, 1))) and np.array_equal(st, np.tile(want_st, reps)), g["tag"]
        if checked[limb_class(mlen)] < 3:
            dx, dy = torch.from_numpy(X).to(dev), torch.from_numpy(Y).to(dev)
            dout = torch.full((X.shape[0], mlen), 0xAB, dtype=torch.uint8, device=dev)
            dst = torch.full((X.shape[0],), 0xAB, dtype=torch.uint8, device=dev)
            mb = np.frombuffer(m.to_bytes(mlen, "big"), np.uint8).copy()
            torch.cuda.synchronize()
            rc = engine._lib.bftq_lagrange_combine_batch_dev(engine._h, mb.ctypes.data_as(ctypes.c_void_p), mlen, k, ctypes.c_void_p(dx.data_ptr()),
                                                             ctypes.c_void_p(dy.data_ptr()), X.shape[0], ctypes.c_void_p(dout.data_ptr()),
                                                             ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(stream.cuda_stream))
            assert rc == 0
            stream.synchronize()
            assert np.array_equal(dout.cpu().numpy(), out) and np.array_equal(dst.cpu().numpy(), st), g["tag"]
        checked[limb_class(mlen)] += 1
    assert all(checked[L] >= 3 for L in (8, 16, 32, 64)), checked


def test_k5_modexp_edges(engine, vec):
    """modexp_batch at W = 8 and 16 on moduli 2^(128 W - 1) + c and 2^(128 W) - c, bases 0, 1, n - 1, n, 2^(128 W) - 1,
    exponents 0, 1, all-ones, one top bit, elen 1..256, warps of eight items mixing exponent lengths and zeros."""
    widths = Counter()
    for r in vec["modexp"]:
        n, bases, exps = te.modexp_operands(r)
        want = [pow(b, e, n) for b, e in zip(bases, exps)]
        assert te.digest([0] * len(want), want, mlen_of(n)) == r["digest"], r["tag"]
        got = engine.modexp_batch(n, bases, exps, elen=r["elen"])
        assert got == want, r["tag"]
        # shifted by 1..7 items, so that each item sits at other lanes next to other exponent lengths
        for s in (1, 3, 7):
            got = engine.modexp_batch(n, bases[s:] + bases[:s], exps[s:] + exps[:s], elen=r["elen"])
            assert got == want[s:] + want[:s], (r["tag"], s)
        widths[(n.bit_length(), r["elen"])] += 1
    assert {e for (_, e) in widths} == {1, 3, 21, 33, 129, 256} and {b for (b, _) in widths} == {1024, 2048}


def test_k5_modprod_inputs_at_and_above_n(engine, vec):
    """modprod_batch with k = 1 (the input itself, reduced) and k = 2 on inputs >= n."""
    for r in vec["modprod"]:
        n, rows = te.modprod_rows(r)
        assert any(v >= n for row in rows for v in row)
        want = [(row[0] * (row[1] if len(row) == 2 else 1)) % n for row in rows]
        assert te.digest([0] * len(want), want, mlen_of(n)) == r["digest"], r["tag"]
        got = engine.modprod_batch(n, rows)
        assert [int.from_bytes(g, "big") for g in got] == want, r["tag"]
    assert {r["k"] for r in vec["modprod"]} == {1, 2}


def test_exp_product_q_in_every_limb_class(engine, vec):
    """auth.calculateSharedSecret (prod y_i^lambda_i mod p) with q of 20..256 bytes: lambda_i from K3 at L = 8, 16, 32
    and 64, then K5.  Status 3 where a difference has no inverse mod q."""
    classes = set()
    for r in vec["exp_product"]:
        p, q, rows = te.exp_product_rows(r)
        outs, sts = [], []
        for xs, ys in rows:
            got, st = engine.lagrange_exp_product_batch(p, q, np.array([xs], np.int32).reshape(1, len(xs)), [ys])
            outs.append(got[0]); sts.append(int(st[0]))
        assert sts == r["status"], r["tag"]
        assert te.digest(sts, outs, mlen_of(p)) == r["digest"], r["tag"]
        classes.add(limb_class(mlen_of(q)))
    assert classes == {8, 16, 32, 64}


def test_dsa_calculate_r_three_domains(engine, vec):
    """dsa.CalculateR on L1024/N160, L2048/N224 and L2048/N256: r as sss_oracle computes it, status 3 where
    sum v_i lambda_i is 0 mod q (a share solved for it) or a difference has no inverse."""
    zero_rows = 0
    for d in vec["dsa"]:
        p, q, items = te.dsa_items(d)
        outs, sts = [0] * len(items), [0] * len(items)
        by_k = {}
        for i, (xs, _, _) in enumerate(items):
            by_k.setdefault(len(xs), []).append(i)
        for k, idx in by_k.items():
            got, st = engine.dsa_calculate_r_batch(p, q, np.array([items[i][0] for i in idx], np.int32).reshape(-1, k),
                                                   [items[i][1] for i in idx], [items[i][2] for i in idx])
            for i, r, s in zip(idx, got, st.tolist()):
                outs[i], sts[i] = r, s
                if s == 0:
                    assert r == sss.dsa_calculate_r(list(zip(*items[i])), p, q), (d["domain"], i)
        assert sts == d["status"] and te.digest(sts, outs, mlen_of(q)) == d["digest"], d["domain"]
        zero_rows += sum(z and s == 3 for z, s in zip(d["zero_v"], sts))
    assert {d["domain"] for d in vec["dsa"]} == {"L1024N160", "L2048N224", "L2048N256"}
    assert zero_rows >= 6
