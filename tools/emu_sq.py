"""Python emulation of the triangular lane-distributed Montgomery SQUARING of
bftkv_b200/csrc/rsa_square_r32.cuh (same E/O/Z/cin bookkeeping as tools/emu_r32.py), against big-int arithmetic.

Tiling of a^2 over the lock-step rounds.  Row J = 16*Y + j (owner lane Y broadcasts limb a_J); lane X multiplies a_J by
    X <  Y :  2 * (A_X with limbs <  j zeroed)            pairs (i in X, J) with i_loc >= j_loc
    X >  Y :  2 * (A_X with limbs <= j zeroed)            pairs (i in X, J) with i_loc >  j_loc
    X == Y :  a_j  +  2 * (A_X with limbs <= j zeroed)    the diagonal term once, the rest of the row twice
Every unordered limb pair is met exactly once (the pair {i in L, j in M}, L != M, sits either in row j of lane L or
in row i of lane M, never both), every lane multiplies 16 - j (+/- 1) limbs in round j, so the lock-step rounds
shrink together: 136 limb products per lane and step instead of 256.
The doubled operand is the lane-local a2 = 2 * A_X (17 limbs, a2[16] = carry bit); a row uses a2[k] for k >= j + 2,
two patched limbs at k = j, j + 1, and the bit a2[16] as an addend of the chain's first carry limb.
The chains into the E pairs up to (16, 17) put their carry on position 18, which is O[17] (`end` asserts that it never
overflows), and the limbs handed down by the lane above carry into position 16 after the shift, which is O[15].
No pending limb is kept at position 0: a step ends by folding the next step's position 0 into one limb, and the carry out
of it (cy1) waits at position 1 and enters with the n x q1 chain.
"""
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from emu_r32 import mont_finish_emu, value  # noqa: E402

B = 1 << 32; T = 4; W = 16; M32 = B - 1


def chain(arr, pairs, xs, m, c=0):
    """pairs: (acc index of the low word, operand index).  Returns the carry out."""
    for lo, xi in pairs:
        v = arr[lo] + (arr[lo + 1] << 32) + xs[xi] * m + c
        arr[lo] = v & M32; arr[lo + 1] = (v >> 32) & M32; c = v >> 64
    return c


def end(arr, idx, c, n2, add=0):
    """carry limbs: arr[idx] += add + c, ripple over n2 words"""
    c += add
    for k in range(n2):
        v = arr[idx + k] + c; arr[idx + k] = v & M32; c = v >> 32
    assert c == 0


def row_operand(a2, X, Y, j):
    """17 limbs lane X multiplies the broadcast limb a_{16Y+j} with (index = window slot at offset 0)."""
    a_j = ((a2[j] >> 1) | (a2[j + 1] << 31)) & M32
    m = [0] * 17
    for k in range(j + 2, 17):
        m[k] = a2[k]
    if X < Y:
        m[j] = a2[j] & ~1 & M32
        m[j + 1] = a2[j + 1]
    elif X > Y:
        m[j] = 0
        m[j + 1] = a2[j + 1] & ~1 & M32
    else:
        m[j] = a_j
        m[j + 1] = a2[j + 1] & ~1 & M32
    if j + 1 == 16:                 # slot 16 is the carry bit: 2*a_15's overflow only counts when limb 15 itself is doubled
        m[16] = a2[16] if X < Y else 0
    return m, a_j


def montsqr_acc(a, n, n0inv):
    """the accumulators (E, O, Z, cin) after the four owner steps, and the a x a limb products per lane"""
    al = [[(a >> (32 * (r * W + j))) & M32 for j in range(W)] for r in range(T)]
    nl = [[(n >> (32 * (r * W + j))) & M32 for j in range(W)] for r in range(T)]
    a2 = []
    for r in range(T):
        v = sum(al[r][k] << (32 * k) for k in range(W)) * 2
        a2.append([(v >> (32 * k)) & M32 for k in range(17)])
    E = [[0] * 20 for _ in range(T)]; O = [[0] * 18 for _ in range(T)]; cy1 = [0] * T
    nprod = 0
    for Y in range(T):
        for jj in range(0, W, 2):
            ops0 = [row_operand(a2[r], r, Y, jj) for r in range(T)]
            ops1 = [row_operand(a2[r], r, Y, jj + 1) for r in range(T)]
            b0 = ops0[Y][1]; b1 = ops1[Y][1]
            assert b0 == al[Y][jj] and b1 == al[Y][jj + 1]
            ev0 = [k for k in range(jj, W, 2)]            # even limbs >= jj       (offset 0 -> E pairs (k, k+1))
            od0 = [k for k in range(jj + 1, W, 2)]        # odd limbs  >= jj       (offset 0 -> O pairs (k-1, k))
            ev1 = [k for k in range(jj + 2, W, 2)]        # even limbs >= jj + 1   (offset 1 -> O pairs (k, k+1))
            od1 = [k for k in range(jj + 1, W, 2)]        # odd limbs  >= jj + 1   (offset 1 -> E pairs (k+1, k+2))
            nprod += len(ev0) + len(od0) + len(ev1) + len(od1)
            for r in range(T):
                m0, _ = ops0[r]
                c = chain(E[r], [(k, k) for k in ev0], m0, b0); end(E[r], 16, c, 2, add=m0[16] * b0)
            q0 = ((E[0][0] & M32) * n0inv) & M32
            for r in range(T):
                m0, _ = ops0[r]; m1, _ = ops1[r]
                c = chain(O[r], [(k - 1, k) for k in od0], m0, b0); end(O[r], 16, c, 2)
                c = chain(O[r], [(k, k) for k in ev1], m1, b1); end(O[r], 16, c, 2, add=m1[16] * b1)
                c = chain(E[r], [(k + 1, k) for k in od1], m1, b1); end(O[r], 17, c, 1)     # position 18 = O[17]
                c = chain(E[r], [(k, k) for k in range(0, W, 2)], nl[r], q0); end(E[r], 16, c, 2)
                c = chain(O[r], [(k - 1, k) for k in range(1, W, 2)], nl[r], q0); end(O[r], 16, c, 2)
            p0 = [E[r][0] for r in range(T)]
            q1 = (((E[0][1] + O[0][0] + cy1[0]) & M32) * n0inv) & M32
            p1 = [0] * T; e0 = [0] * T
            for r in range(T):
                c = chain(O[r], [(k, k) for k in range(0, W, 2)], nl[r], q1, cy1[r]); end(O[r], 16, c, 2)   # cy1 enters at position 1
                c = chain(E[r], [(k + 1, k) for k in range(1, W, 2)], nl[r], q1); end(O[r], 17, c, 1)
                s = E[r][1] + O[r][0]; p1[r] = s & M32
                s = E[r][2] + O[r][1] + (s >> 32); e0[r] = s & M32; cy1[r] = s >> 32     # the next step's position 0, one limb
            assert p0[0] == 0 and p1[0] == 0
            for r in range(T):
                r0 = p0[r + 1] if r < T - 1 else 0; r1 = p1[r + 1] if r < T - 1 else 0
                assert E[r][18] == 0 and E[r][19] == 0            # the kernel keeps no limbs above E[17]
                # E and O keep 16 limbs each plus two carry limbs that start every step at zero; position 16 is O[15]
                E[r] = [e0[r]] + E[r][3:18] + [0, 0, 0, 0]; O[r] = O[r][2:] + [0, 0]
                v = E[r][14] + (E[r][15] << 32) + (O[r][15] << 64) + r0 + (r1 << 32)
                E[r][14] = v & M32; E[r][15] = (v >> 32) & M32; O[r][15] = (v >> 64) & M32
                assert v >> 96 == 0
    for r in range(T):                                    # mont_sqr's tail: cy1 rippled into O (position 1 on)
        v = sum(O[r][k] << (32 * k) for k in range(W)) + cy1[r]
        assert v >> (32 * W) == 0
        O[r][:W] = [(v >> (32 * k)) & M32 for k in range(W)]
    return E, O, [0] * T, [0] * T, nprod


def montsqr_emu(a, n, n0inv):
    E, O, Z, cin, nprod = montsqr_acc(a, n, n0inv)
    tot = 0
    for r in range(T):
        loc = cin[r] + Z[r] + sum(E[r][k] << (32 * k) for k in range(20)) + sum(O[r][k] << (32 * (k + 1)) for k in range(18))
        # what the kernel's merge reads: E[0..16], O[0..15] (hi = E[16] + O[15] + carry); everything above must be zero
        assert E[r][17] == 0 and E[r][18] == 0 and E[r][19] == 0 and O[r][16] == 0 and O[r][17] == 0 and E[r][16] + O[r][15] <= 8, (E[r][16:], O[r][15:])
        tot += loc << (32 * W * r)
    return tot, nprod


def mont_sqr_emu(a, n, trace=None):
    """mont_sqr with its mont_finish (emu_r32.mont_finish_emu, `trace` as there): a^2 R^-1 mod n, < R"""
    E, O, Z, cin, _ = montsqr_acc(a, n, (-pow(n, -1, B)) % B)
    return value(mont_finish_emu(E, O, Z, cin, n, W, trace))


def check_random(iters=300, seed=2):
    """random and adversarial squarings (operands R - 1, alternating limbs, single bits; modulus R - 1) against
    big-int arithmetic; returns the a x a limb products per lane and squaring"""
    random.seed(seed)
    R = 1 << 2048
    for it in range(iters):
        n = random.getrandbits(2048) | (1 << 2047) | 1
        a = random.getrandbits(2048)
        if it % 7 == 0: a = R - 1
        if it % 11 == 0: n = R - 1
        if it % 13 == 0: a = sum(0x80000000 << (32 * k) for k in range(64))
        if it % 17 == 0: a = sum(0xffffffff << (32 * k) for k in range(0, 64, 2))
        if it % 19 == 0: a = 1 << (32 * (it % 64) + 31)
        n0inv = (-pow(n, -1, B)) % B
        t, nprod = montsqr_emu(a, n, n0inv)
        assert t == (a * a + ((a * a * (-pow(n, -1, R))) % R) * n) // R, it
        assert t < R + n
    return nprod


if __name__ == "__main__":
    nprod = check_random()
    print("emulation ok; a x a limb products per lane and squaring:", nprod, "(general product: 1024)")
