"""Writes tests/golden/decrypt_edges.json: the fixed inputs of the decryption edge tests (tests/decrypt_edges.py).

- Two RSA-2048 keys (e = 65537) with 1024-bit primes at extreme ratios: "L" with p / q ~ 1/2 and "H" with p / q ~ 2.  n has
  exactly 2048 bits.  For H, m mod p >= q holds for about half of all m, and Garner's m1 reaches almost 2q.
- Per AES size, a quick-check collision: a session key and a 16-byte random prefix, and a wrong key of the same size under
  which the first 18 ciphertext bytes still pass OpenPGP's quick check (bytes 14, 15 of the decrypted prefix equal bytes
  16, 17).  About 2^16 trial keys each.

Deterministic: seeded candidates and seeded Miller-Rabin.  `python tests/golden/make_decrypt_edges.py [out.json]`."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
from read_answer_edges import _is_prime  # noqa: E402
from pgp_encrypt_ref import _aes_ecb, cfb_encrypt  # noqa: E402

SEED = 0xBF7C0DE6
E = 65537


def _prime(rng, lo, width_bits):
    """A prime in [lo, lo + 2^width_bits) with gcd(p - 1, e) = 1."""
    while True:
        c = lo + rng.getrandbits(width_bits) | 1
        if (c - 1) % E and _is_prime(c, rng):
            return c


def ratio_key(rng, p_small):
    """p ~ 2^1023 (1 + 2^-7), q ~ 2^1024 (1 - 2^-9): p / q ~ 0.504, and p q > 2^2047.  Swapped when not p_small."""
    a = _prime(rng, (1 << 1023) + (1 << 1016), 1016)
    b = _prime(rng, (1 << 1024) - (1 << 1015), 1014)
    p, q = (a, b) if p_small else (b, a)
    n = p * q
    assert n.bit_length() == 2048 and p.bit_length() == q.bit_length() == 1024
    return {"p": p, "q": q, "n": n, "e": E, "d": pow(E, -1, (p - 1) * (q - 1))}


def quick_check_passes(key: bytes, ct18: bytes) -> bool:
    pre = bytes(a ^ b for a, b in zip(ct18[:16], _aes_ecb(key, bytes(16)))) + \
        bytes(a ^ b for a, b in zip(ct18[16:18], _aes_ecb(key, ct18[:16])))
    return pre[14:16] == pre[16:18]


def collision(rng, ks):
    key = rng.randbytes(ks)
    prefix = rng.randbytes(16)
    ct18 = cfb_encrypt(key, prefix + prefix[14:16])
    while True:
        wrong = rng.randbytes(ks)
        if wrong != key and quick_check_passes(wrong, ct18):
            return {"cipher": {16: 7, 24: 8, 32: 9}[ks], "key": key.hex(), "prefix": prefix.hex(), "wrong": wrong.hex()}


def generate():
    rng = random.Random(SEED)
    keys = {"L": ratio_key(rng, True), "H": ratio_key(rng, False)}
    out = {"seed": SEED,
           "keys": {name: {f: "%x" % k[f] for f in ("p", "q")} for name, k in keys.items()},
           "e": E,
           "collisions": [collision(rng, ks) for ks in (16, 24, 32)]}
    return json.dumps(out, indent=1, sort_keys=True) + "\n"


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "decrypt_edges.json")
    with open(path, "w") as f:
        f.write(generate())
