"""Limb-level emulation of one whole K1 verification (rsa_verify_r32_kernel, unified program, squarings through
mont_sqr): the square-and-multiply chain of e on the plain signature s (emu_sq.py, emu_r32.py), the check product of
one or two owner steps with the key's c * 2^k, mont_finish on every product, and the final comparison
(Y - Q) mod n == hc through cond_sub / group_sub.  K1 accepts iff this returns True.

`nbmax` > e's bit length emulates a lane whose warp (or block) runs a longer exponent: the squarings above the lane's
own top bit are computed and not applied, as in the kernel."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from emu_r32 import (B, T, W, cond_sub_emu, group_sub_emu, lanes, mont_finish_emu, montmul_acc,  # noqa: E402
                     value)
from emu_sq import montsqr_acc  # noqa: E402

R = 1 << 2048


def key_consts(n, e):
    """The per-key constants of RsaKey32 (bignum_host.hpp), from their definition."""
    c = pow(R, -(e - 1), n)
    return {"c16": c * (1 << 512) % n, "hc16": ((1 << 2033) - (1 << 512)) * c % n,
            "c32": c * (1 << 1024) % n, "hc32": ((1 << 2033) - (1 << 1024)) * c % n}


def em_int(prefix, digest):
    """EMSA-PKCS1-v1_5 for k = 256 as a number"""
    t = prefix + digest
    return int.from_bytes(b"\x00\x01" + b"\xff" * (256 - len(t) - 3) + b"\x00" + t, "big")


def verify_emu(n, e, s, em, tlen, consts=None, nbmax=None):
    consts = consts or key_consts(n, e)
    n0inv = (-pow(n, -1, B)) % B
    mul_ = lambda a, b, owners=T: value(mont_finish_emu(*montmul_acc(a, b, n, n0inv, owners), n))  # noqa: E731
    sqr_ = lambda a: value(mont_finish_emu(*montsqr_acc(a, n, n0inv)[:4], n))  # noqa: E731
    nb = e.bit_length()
    nbmax = nbmax or nb
    wide = tlen > 63
    y = s
    bit = nbmax - 2
    op = 1 if bit >= 0 else 3
    while True:
        if op == 1:
            t = sqr_(y)
            if bit <= nb - 2:
                y = t
            if bit <= nb - 2 and (e >> bit) & 1:
                op = 2
            else:
                bit -= 1
                op = 1 if bit >= 0 else 3
        elif op == 2:
            y = mul_(y, s)
            bit -= 1
            op = 1 if bit >= 0 else 3
        else:
            q = mul_(consts["c32" if wide else "c16"], em, 2 if wide else 1)
            break
    assert y < R and q < R and q < 2 * n
    nl = lanes(n)
    d, b = group_sub_emu(cond_sub_emu(lanes(y), nl), cond_sub_emu(lanes(q), nl))
    f, _ = group_sub_emu(lanes(consts["hc32" if wide else "hc16"]), d)
    return value(f) == (n if b else 0)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bftkv_b200 import workload
    k = workload.load_keys(1)[0]
    em = workload.em_for_digest(bytes(range(32)))
    s = pow(em, k["d"], k["n"])
    assert verify_emu(k["n"], k["e"], s, em, 51) and not verify_emu(k["n"], k["e"], s ^ 1, em, 51)
    print("emulation ok")
