"""K1b Ed25519 (BASELINE config 4).  The reference cannot verify Ed25519 at all (x/crypto/openpgp
has no EdDSA, SURVEY F5), so parity is pinned on RFC 8032 test vectors, OpenSSL (`cryptography`) and
libsodium (`pynacl`) instead.  CPU tests run the kernel's own __host__ __device__ arithmetic compiled
for the host (tests/harness/ed25519_host.cpp); the gpu test runs the kernel through the C ABI."""
import ctypes
import hashlib
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2 ** 255 - 19
L = 2 ** 252 + 27742317777372353535851937790883648493

# RFC 8032 §7.1 test vectors 1-3 (secret key, public key, message, signature)
RFC8032 = [
    ("d75a980182b10ab7d54bfed3c964073a0ee172f3daa62325af021a68f707511a", "",
     "e5564300c360ac729086e2cc806e828a84877f1eb8e5d974d873e065224901555fb8821590a33bacc61e39701cf9b46bd25bf5f0595bbe24655141438e7a100b"),
    ("3d4017c3e843895a92b70aa74d1b7ebc9c982ccf2ec4968cc0cd55f12af4660c", "72",
     "92a009a9f0d4cab8720e820b5f642540a2b27b5416503f8fb3762223ebdb69da085ac1e43e15996e458f3613d0f11d8c387b2eaeb4302aeeb00d291612bb0c00"),
    ("fc51cd8e6218a1a38da47ed00230f0580816ed13ba3303ac5deb911548908025", "af82",
     "6291d657deec24024827e69c3abe01a30ce548a284743a445e3680d7db5ac3ac18ff9b538d16f290ae67f760984dc6594a7c15e9716ed28dc027beceea1ec40a"),
]


@pytest.fixture(scope="module")
def host():
    so = os.path.join(ROOT, "tests", "harness", "libedhost.so")
    src = os.path.join(ROOT, "tests", "harness", "ed25519_host.cpp")
    hdrs = [os.path.join(ROOT, "bftkv_b200", "csrc", h) for h in ("ed25519.cuh", "ed25519_fast.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def make_sigs(n, n_keys, seed):
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    rng = random.Random(seed)
    sks = [Ed25519PrivateKey.from_private_bytes(bytes(rng.randrange(256) for _ in range(32))) for _ in range(n_keys)]
    pks = [k.public_key().public_bytes(serialization.Encoding.Raw, serialization.PublicFormat.Raw) for k in sks]
    kidx = np.array([rng.randrange(n_keys) for _ in range(n)], np.uint32)
    msg = np.frombuffer(bytes(rng.randrange(256) for _ in range(32 * n)), np.uint8).reshape(n, 32).copy()
    sig = np.empty((n, 64), np.uint8)
    for i in range(n):
        sig[i] = np.frombuffer(sks[kidx[i]].sign(msg[i].tobytes()), np.uint8)
    return sks, pks, kidx, msg, sig, rng


def openssl_ok(sk, sig, msg):
    try:
        sk.public_key().verify(sig, msg)
        return True
    except Exception:
        return False


def test_field_and_scalar_arithmetic(host):
    rng = random.Random(1)
    out = ctypes.create_string_buffer(32)
    b = lambda x: int(x).to_bytes(32, "little")
    for i in range(1500):
        x, y = rng.randrange(P), rng.randrange(P)
        if i % 50 == 0:
            x = P - 1
        if i % 77 == 0:
            y = P - 1 - (i % 3)
        host.ed_fe_mul_host(b(x), b(y), out)
        assert int.from_bytes(out.raw, "little") == x * y % P
        host.ed_fe_addsubmul_host(b(x), b(y), out)
        assert int.from_bytes(out.raw, "little") == (x + y) * (x - y) % P
    for _ in range(40):
        x = rng.randrange(1, P)
        host.ed_fe_invert_host(b(x), out)
        assert int.from_bytes(out.raw, "little") == pow(x, -1, P)
    for v in [bytes(64), b"\xff" * 64, L.to_bytes(32, "little") + bytes(32), (L - 1).to_bytes(32, "little") + bytes(32)] + [os.urandom(64) for _ in range(100)]:
        host.ed_sc_reduce_host(v, out)
        assert int.from_bytes(out.raw, "little") == int.from_bytes(v, "little") % L


def test_rfc8032_vectors_and_openssl(host):
    import nacl.exceptions
    import nacl.signing
    for pk, msg, sig in RFC8032:
        pk, msg, sig = bytes.fromhex(pk), bytes.fromhex(msg), bytes.fromhex(sig)
        # the kernel signs/verifies 32-byte digests; the core takes k = H(R||A||M) for any M
        k = hashlib.sha512(sig[:32] + pk + msg).digest()
        assert host.ed_verify_core_host(sig, pk, k) == 1
        bad = bytearray(sig); bad[5] ^= 2
        assert host.ed_verify_core_host(bytes(bad), pk, hashlib.sha512(bytes(bad[:32]) + pk + msg).digest()) == 0
    sks, pks, kidx, msg, sig, rng = make_sigs(120, 5, 3)
    for i in range(120):
        pk, m = pks[kidx[i]], msg[i].tobytes()
        s = bytearray(sig[i].tobytes())
        if i % 2:
            s[rng.randrange(64)] ^= 1 << rng.randrange(8)
        s = bytes(s)
        got = host.ed_verify_core_host(s, pk, hashlib.sha512(s[:32] + pk + m).digest()) == 1
        assert got == openssl_ok(sks[kidx[i]], s, m)
        try:
            nacl.signing.VerifyKey(pk).verify(m, s)
            sodium = True
        except nacl.exceptions.BadSignatureError:
            sodium = False
        assert got == sodium
    # non-canonical S (S + L); keys the signature is not for: y = p + 1 (the identity), y = 2 (no point), ff..ff (y = p + 18)
    s0 = sig[0].tobytes()
    S = int.from_bytes(s0[32:], "little") + L
    pk0, m0 = pks[kidx[0]], msg[0].tobytes()
    if S < 2 ** 256:
        s1 = s0[:32] + S.to_bytes(32, "little")
        assert host.ed_verify_core_host(s1, pk0, hashlib.sha512(s1[:32] + pk0 + m0).digest()) == 0
    for badpk in [(P + 1).to_bytes(32, "little"), (2).to_bytes(32, "little"), b"\xff" * 32]:
        assert host.ed_verify_core_host(s0, badpk, hashlib.sha512(s0[:32] + badpk + m0).digest()) == 0


D = -121665 * pow(121666, -1, P) % P


def _edwards_add(p, q):
    (x1, y1), (x2, y2) = p, q
    t = D * x1 * x2 * y1 * y2 % P
    return ((x1 * y2 + x2 * y1) * pow(1 + t, -1, P) % P, (y1 * y2 + x1 * x2) * pow(1 - t, -1, P) % P)


def _edwards_mul(k, p):
    r = (0, 1)
    while k:
        if k & 1:
            r = _edwards_add(r, p)
        p = _edwards_add(p, p)
        k >>= 1
    return r


def _decode_point(b):
    y = int.from_bytes(b, "little") & ((1 << 255) - 1)
    sign = b[31] >> 7
    x2 = (y * y - 1) * pow(D * y * y + 1, -1, P) % P
    x = pow(x2, (P + 3) // 8, P)
    if (x * x - x2) % P:
        x = x * pow(2, (P - 1) // 4, P) % P
    assert (x * x - x2) % P == 0
    if x & 1 != sign:
        x = P - x
    return (x, y)


def test_fast_field_scalar_and_tables(host):
    """ed25519_fast.cuh on the host: inlined product / squaring (carried and uncarried operands at the documented bounds),
    the addition-chain powers, canonical words, the Barrett reduction mod L, the signed radix-2^10 / 2^12 recodings, and window-table
    entries against big-integer Edwards arithmetic (affine y+x, y-x, 2dxy; limbs carried)."""
    rng = random.Random(2)
    out = ctypes.create_string_buffer(64)
    b = lambda x: int(x).to_bytes(32, "little")
    for i in range(2000):
        x, y = rng.randrange(P), rng.randrange(P)
        if i % 50 == 0:
            x = P - 1
        if i % 77 == 0:
            y = P - 1 - (i % 3)
        if i % 91 == 0:
            x = 2 ** 255 - 20                              # non-canonical input representative
        host.ed_fex_mul_host(b(x), b(y), out)
        assert int.from_bytes(out.raw[:32], "little") == x * y % P
        host.ed_fex_sq_host(b(x), out)
        assert int.from_bytes(out.raw[:32], "little") == x * x % P
        host.ed_fex_uncarried_host(b(x), b(y), out)
        assert int.from_bytes(out.raw[:32], "little") == (x + y) ** 2 % P and int.from_bytes(out.raw[32:], "little") == (x + y) * (x - y) % P
        host.ed_fex_towords_host(b(x), b(y), out)
        assert int.from_bytes(out.raw[:32], "little") == x * y % P
    for _ in range(40):
        x = rng.randrange(1, P)
        host.ed_fex_pow_host(b(x), 1, out)
        assert int.from_bytes(out.raw[:32], "little") == pow(x, P - 2, P)
        host.ed_fex_pow_host(b(x), 0, out)
        assert int.from_bytes(out.raw[:32], "little") == pow(x, (P - 5) // 8, P)
    edge = [bytes(64), b"\xff" * 64, L.to_bytes(32, "little") + bytes(32), (L - 1).to_bytes(32, "little") + bytes(32), (L * 2 ** 259).to_bytes(64, "little"),
            (L * 2 ** 259 - 1).to_bytes(64, "little"), (2 ** 252).to_bytes(64, "little"), (L << 200).to_bytes(64, "little"), (2 ** 511).to_bytes(64, "little")]
    near = [(rng.randrange(2 ** 259) * L + rng.choice([0, 1, L - 1, L - 2])).to_bytes(64, "little") for _ in range(500)]
    for v in edge + near + [os.urandom(64) for _ in range(2000)]:
        host.ed_sc_reduce512_host(v, out)
        assert int.from_bytes(out.raw[:32], "little") == int.from_bytes(v, "little") % L, v.hex()
    dg = (ctypes.c_int32 * 32)()
    for _ in range(500):                                   # sum d_i 2^(W i) == s, d_i in [-2^(W-1), 2^(W-1) - 1], for both window widths
        sc = rng.choice([rng.randrange(L), L - 1, 0, 1, 2 ** 252, int("80" * 31, 16), int("7f" * 31, 16), int("ff" * 31, 16), 2 ** 252 + 2 ** 251,
                         int("1f" + "ff" * 31, 16), int("0f" + "ff" * 31, 16), (1 << 250) - 1, 511 * sum(1 << (10 * i) for i in range(25)),
                         512 * sum(1 << (10 * i) for i in range(25)), 2048 * sum(1 << (12 * i) for i in range(21))])
        for wbits, nw in ((10, 26), (12, 22)):
            host.ed_digits_host(sc.to_bytes(32, "little"), wbits, dg)
            d = list(dg)[:nw]
            assert all(-(1 << (wbits - 1)) <= v < (1 << (wbits - 1)) for v in d) and sum(v << (wbits * i) for i, v in enumerate(d)) == sc, (hex(sc), wbits)
    # 3 P through gex_dbl / gex_add / the inversion chain
    sks, pks, *_ = make_sigs(1, 3, 21)
    for pk in pks:
        assert host.ed_gex_roundtrip_host(pk, out) == 1
        x3, y3 = _edwards_mul(3, _decode_point(pk))
        assert int.from_bytes(out.raw[:32], "little") == y3 | ((x3 & 1) << 255)
    # table entries: j * 2^(10 w) * A for a key (26 windows x 512 multiples), j * 2^(12 w) * B for the base point (22 x 2048)
    A = _decode_point(pks[0])
    Bpt = _decode_point((4 * pow(5, -1, P) % P).to_bytes(32, "little"))
    e1, e2, e3 = (ctypes.create_string_buffer(32) for _ in range(3))
    cases = [(0, 0, 1), (0, 0, 2), (0, 0, 8), (0, 0, 9), (0, 0, 512), (0, 1, 1), (0, 1, 77), (0, 5, 505), (0, 17, 64), (0, 25, 1), (0, 25, 8), (0, 25, 512),
             (1, 0, 1), (1, 0, 2048), (1, 3, 2041), (1, 21, 1), (1, 21, 2), (1, 10, 1025)] + \
            [(0, rng.randrange(26), rng.randrange(1, 513)) for _ in range(15)] + [(1, rng.randrange(22), rng.randrange(1, 2049)) for _ in range(15)]
    for base, w, j in cases:
        assert host.ed_fx_table_entry_host(pks[0], base, w, j, e1, e2, e3) == 1, "entry not carried"
        x, y = _edwards_mul(j << ((12 if base else 10) * w), Bpt if base else A)
        assert int.from_bytes(e1.raw, "little") == (y + x) % P and int.from_bytes(e2.raw, "little") == (y - x) % P
        assert int.from_bytes(e3.raw, "little") == 2 * D * x * y % P


def test_fast_core_equals_classic_core(host):
    """The cached-window-table verification (what the batch kernels run when signatures share keys: accumulate + finish)
    against the classic double-and-add core, OpenSSL and the RFC 8032 vectors: valid, bit-flipped, S >= L, undecodable A,
    small-order A and R; and the accumulator's limbs stay inside the lazy-carry bounds."""
    for pk, msg, sig in RFC8032:
        pk, msg, sig = bytes.fromhex(pk), bytes.fromhex(msg), bytes.fromhex(sig)
        assert host.ed_verify_fast_host(sig, pk, hashlib.sha512(sig[:32] + pk + msg).digest()) == 1
        assert host.ed_verify_core_fast_host(sig, pk, hashlib.sha512(sig[:32] + pk + msg).digest()) == 1
        bad = bytearray(sig); bad[5] ^= 2
        assert host.ed_verify_fast_host(bytes(bad), pk, hashlib.sha512(bytes(bad[:32]) + pk + msg).digest()) == 0
        assert host.ed_verify_core_fast_host(bytes(bad), pk, hashlib.sha512(bytes(bad[:32]) + pk + msg).digest()) == 0
    sks, pks, kidx, msg, sig, rng = make_sigs(400, 6, 7)
    order = sorted(range(400), key=lambda i: kidx[i])       # the harness caches the last key's table
    n_ok = 0
    for i in order:
        pk, m = pks[kidx[i]], msg[i].tobytes()
        s = bytearray(sig[i].tobytes())
        if i % 3 == 1:
            s[rng.randrange(64)] ^= 1 << rng.randrange(8)
        if i % 7 == 3:                                     # S + L: same residue, non-canonical
            S = int.from_bytes(s[32:], "little") + L
            if S < 2 ** 256:
                s[32:] = S.to_bytes(32, "little")
        s = bytes(s)
        k = hashlib.sha512(s[:32] + pk + m).digest()
        a, b, c = host.ed_verify_core_host(s, pk, k), host.ed_verify_fast_host(s, pk, k), host.ed_verify_core_fast_host(s, pk, k)
        assert a == b == c == int(openssl_ok(sks[kidx[i]], s, m)), i
        n_ok += a
    assert 150 < n_ok < 400
    s0, m0 = sig[0].tobytes(), msg[0].tobytes()
    weird = [(P + 1).to_bytes(32, "little"), (2).to_bytes(32, "little"), b"\xff" * 32,
             (1).to_bytes(32, "little"),                    # the identity (order 1)
             (P - 1).to_bytes(32, "little"),                # (0, -1): order 2
             bytes(32)]                                      # y = 0: order 4
    for badpk in weird:
        for sg in (s0, bytes(32) + bytes(32), (1).to_bytes(32, "little") + bytes(32)):
            k = hashlib.sha512(sg[:32] + badpk + m0).digest()
            assert host.ed_verify_core_host(sg, badpk, k) == host.ed_verify_fast_host(sg, badpk, k) == host.ed_verify_core_fast_host(sg, badpk, k), (badpk.hex(), sg.hex())
    for i in range(6):
        pk = pks[kidx[i]]
        s = sig[i].tobytes()
        m = host.ed_fast_limb_bound_host(s, pk, hashlib.sha512(s[:32] + pk + msg[i].tobytes()).digest())
        assert 0 < m <= int(1.01 * 2 ** 25)


@pytest.mark.gpu
def test_ed25519_gpu_batch(engine):
    n = 4096
    sks, pks, kidx, msg, sig, rng = make_sigs(n, 15, 0xBF7C0005)          # config 4: K = 15 keys
    expect = np.zeros(n, np.uint8)
    for i in range(n):
        if rng.random() < 0.3:
            sig[i, rng.randrange(64)] ^= np.uint8(1 << rng.randrange(8))
            expect[i] = 0 if openssl_ok(sks[kidx[i]], sig[i].tobytes(), msg[i].tobytes()) else 1
    unk = [5, 77, 901]
    kidx[unk] = 99
    expect[unk] = 4
    # a 16th key that does not decode to a curve point: everything under it is invalid (both kernels)
    bad_key = [11, 500, 3000]
    kidx[bad_key] = 15
    expect[bad_key] = 1
    pk_arr = np.frombuffer(b"".join(pks) + (2).to_bytes(32, "little"), np.uint8).reshape(16, 32).copy()
    got = engine.ed25519_verify_batch(pk_arr, kidx, sig, msg)          # 4096 signatures, 16 keys: the window-table kernel
    assert np.array_equal(got, expect)
    assert (got == 0).sum() > 2500 and (got == 1).sum() > 1000
    for size in (1, 2, 31, 129):                                        # tiny batches under keys that are cached by now
        assert np.array_equal(engine.ed25519_verify_batch(pk_arr, kidx[:size].copy(), sig[:size].copy(), msg[:size].copy()), expect[:size])
    # every signature under its own new key (no sharing): the table-free double-and-add kernel
    sks2, pks2, kidx2, msg2, sig2, _ = make_sigs(300, 300, 5)
    kidx2 = np.arange(300, dtype=np.uint32)
    for i in range(300):
        sig2[i] = np.frombuffer(sks2[i].sign(msg2[i].tobytes()), np.uint8)
    sig2[7, 3] ^= 4
    got2 = engine.ed25519_verify_batch(np.frombuffer(b"".join(pks2), np.uint8).reshape(300, 32).copy(), kidx2, sig2, msg2)
    assert got2[7] == 1 and got2.sum() == 1
    pk2 = np.frombuffer(b"".join(pks2), np.uint8).reshape(300, 32).copy()
    got2b = engine.ed25519_verify_batch(pk2[5:12], np.arange(7, dtype=np.uint32), sig2[5:12].copy(), msg2[5:12].copy())   # 7 signatures, 7 new keys
    assert got2b.tolist() == [0, 0, 1, 0, 0, 0, 0]
    # the table cache: the same keys again (no build), the keys in another order with a duplicate and a NEW key (one build),
    # a size that is not a multiple of the finish kernel's 512-item tiles, S >= L, and every signature invalid
    builds0 = engine.stats()["launches"]
    assert np.array_equal(engine.ed25519_verify_batch(pk_arr, kidx, sig, msg), expect)
    assert engine.stats()["launches"] - builds0 == 2                   # accumulate + finish only
    sks3, pks3, _, _, _, _ = make_sigs(1, 1, 99)
    perm = [3, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15]   # key 3 twice (positions 0 and 4)
    pk_perm = np.concatenate([pk_arr[perm], np.frombuffer(pks3[0], np.uint8).reshape(1, 32)])
    n2 = 5000
    rep = np.resize(np.arange(n), n2)
    k2 = kidx[rep].copy(); s2 = sig[rep].copy(); m2 = msg[rep].copy(); e2 = expect[rep].copy()
    new_pos = {old: pos for pos, old in enumerate(perm) if pos != 0}    # old index -> a position of the same key
    k2m = np.array([new_pos.get(int(k), 99) if k < 16 else 99 for k in k2], np.uint32)
    k2m[::2] = np.where(k2[::2] == 3, 0, k2m[::2])                     # half of key 3's items through its other position
    for i in range(40):                                                 # items under the new key: valid and corrupted
        j = 100 + i
        m2[j] = np.frombuffer(bytes(rng.randrange(256) for _ in range(32)), np.uint8)
        s2[j] = np.frombuffer(sks3[0].sign(m2[j].tobytes()), np.uint8)
        k2m[j] = 17
        e2[j] = 0
        if i % 4 == 0:
            s2[j, 40] ^= 1
            e2[j] = 1
    Sbig = (int.from_bytes(s2[101, 32:].tobytes(), "little") + L).to_bytes(32, "little")
    s2[101, 32:] = np.frombuffer(Sbig, np.uint8)                      # S + L: non-canonical
    e2[101] = 1
    got3 = engine.ed25519_verify_batch(pk_perm, k2m, s2, m2)
    assert np.array_equal(got3, e2)
    allbad = sig[:2304].copy(); allbad[:, 1] ^= 0x10                   # R damaged everywhere (two earlier flips are undone by it)
    kb = np.minimum(kidx[:2304], 14)
    expb = np.array([0 if openssl_ok(sks[kb[i]], allbad[i].tobytes(), msg[i].tobytes()) else 1 for i in range(2304)], np.uint8)
    gotb = engine.ed25519_verify_batch(pk_arr, kb, allbad, msg[:2304])
    assert np.array_equal(gotb, expb) and (gotb == 1).sum() > 2290


@pytest.mark.gpu
def test_ed25519_table_cache_full_gpu():
    """A table cache of four slots: a second key set that pays for its tables (>= 128 signatures per new key) empties the
    full cache and is verified against fresh tables; a small batch under yet other keys takes the table-free kernel; the
    first key set comes back afterwards.  Every status against OpenSSL."""
    from bftkv_b200 import Engine
    old = os.environ.get("BFTQ_ED25519_CACHE_SLOTS")
    os.environ["BFTQ_ED25519_CACHE_SLOTS"] = "4"
    eng = Engine(0)
    try:
        def batch(n, n_keys, seed):
            sks, pks, kidx, msg, sig, rng = make_sigs(n, n_keys, seed)
            expect = np.zeros(n, np.uint8)
            for i in range(0, n, 7):
                sig[i, rng.randrange(64)] ^= np.uint8(1 << rng.randrange(8))
                expect[i] = 0 if openssl_ok(sks[kidx[i]], sig[i].tobytes(), msg[i].tobytes()) else 1
            return np.frombuffer(b"".join(pks), np.uint8).reshape(n_keys, 32).copy(), kidx, sig, msg, expect
        a = batch(600, 3, 301)
        b = batch(600, 3, 302)
        c = batch(100, 3, 303)
        for pk, kidx, sig, msg, expect in (a, b, c, a, b):
            assert np.array_equal(eng.ed25519_verify_batch(pk, kidx, sig, msg), expect)
    finally:
        eng.close()
        if old is None:
            os.environ.pop("BFTQ_ED25519_CACHE_SLOTS", None)
        else:
            os.environ["BFTQ_ED25519_CACHE_SLOTS"] = old
