"""Writes tests/golden/signature_sign.json: detached signatures as PGPSignature.Sign writes them (tests/signature_sign_oracle.py),
each checked two ways when it is written: `cryptography`'s RSA PKCS#1 v1.5 signature of the digest must equal the packet's
256 bytes of s, and GnuPG (`gpg --verify`) is asked about every packet, its verdict recorded as gnupg_ok.

Keys: fixture keys 0 (p < q) and 5 (p > q) of rsa_keys_bf7c0001.json, and L (p / q ~ 1/2) and H (p / q ~ 2) of
decrypt_edges.json, each registered as pgp_public_key_block makes it.
tbs lengths: 0, 1; 27 / 28 and 91 / 92, which with the 28 suffix bytes end the hashed stream at 55 / 56 and 119 / 120 bytes,
on both sides of the point where SHA-256's padding needs another block; 33 / 34 and 97 / 98; 4096 and 70 000.  Every length
is signed at every creation time of CTIMES.  Then, per key, creation times are ground from GRIND upward until s < 2^2047
(the top bit clear) and until s < 2^2040 (a leading zero byte, which the 08 00 MPI header keeps).

GnuPG 2.4.4 accepts every packet made at a creation time after the key's (0x5E000000), the 08 00 headers over a short s
included.  It refuses the ones made at ctime 0 and 1 with "Time conflict": the signature predates the key.  Go does not
check that, and neither does this library's verification, so those packets stay as Go writes them.

tbs bytes come from tbs_bytes(length, index).  `python tests/golden/make_signature_sign.py [out.json]` (needs gpg)."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import signature_sign_oracle as O  # noqa: E402
from decrypt_edges import load_fixture  # noqa: E402
from bftkv_b200 import workload as W  # noqa: E402

KEYS = ("0", "5", "L", "H")
LENGTHS = (0, 1, 27, 28, 33, 34, 91, 92, 97, 98, 4096, 70000)
CTIMES = (0, 1, 1 << 31, (1 << 32) - 1)
GRIND = 0x5F000000


def keys():
    fix = W.load_keys(6)
    extra, _ = load_fixture()
    return {"0": fix[0], "5": fix[5], "L": extra["L"], "H": extra["H"]}


def tbs_bytes(length: int, index: int) -> bytes:
    out, c = b"", 0
    while len(out) < length:
        out += hashlib.sha256(b"bftq-sign-tbs %d %d %d" % (length, index, c)).digest()
        c += 1
    return out[:length]


def cases():
    """-> [(key name, tbs length, tbs index, ctime, kind)] in fixture order."""
    ks = keys()
    out = []
    for name in KEYS:
        for i, length in enumerate(LENGTHS):
            for ct in CTIMES:
                out.append((name, length, i, ct, "grid"))
        k, kid = ks[name], O.key_block(ks[name])[1]
        for kind, bound in (("s<2^2047", 1 << 2047), ("s<2^2040", 1 << 2040)):
            ct = GRIND
            while O.sign_s(k, O.digest(tbs_bytes(64, 0), ct, kid)) >= bound:
                ct += 1
            out.append((name, 64, 0, ct, kind))
    return out


def gpg(home, *args):
    return subprocess.run(["gpg", "--homedir", home, "--batch", "--quiet"] + list(args), capture_output=True)


def generate():
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding
    from cryptography.hazmat.primitives.asymmetric.utils import Prehashed
    ks = keys()
    home = tempfile.mkdtemp(prefix="bftq-gpg-")
    blocks = {name: O.key_block(k) for name, k in ks.items()}
    for name in KEYS:
        r = subprocess.run(["gpg", "--homedir", home, "--batch", "--quiet", "--import"], input=blocks[name][0], capture_output=True)
        assert r.returncode == 0, r.stderr
    rows = []
    for name, length, idx, ct, kind in cases():
        k, kid = ks[name], blocks[name][1]
        tbs = tbs_bytes(length, idx)
        pkt = O.packet(k, kid, tbs, ct)
        dg = O.digest(tbs, ct, kid)
        ref = W._private_key(k).sign(dg, padding.PKCS1v15(), Prehashed(hashes.SHA256()))
        assert ref.rjust(256, b"\0") == pkt[-256:], (name, length, ct)
        s = int.from_bytes(pkt[-256:], "big")
        assert kind != "s<2^2047" or s < 1 << 2047
        assert kind != "s<2^2040" or (s < 1 << 2040 and pkt[-256] == 0)
        tp, sp = os.path.join(home, "tbs.bin"), os.path.join(home, "sig.bin")
        open(tp, "wb").write(tbs)
        open(sp, "wb").write(pkt)
        v = gpg(home, "--verify", sp, tp)
        rows.append({"key": name, "key_id": "%016x" % kid, "tbs_len": length, "tbs_index": idx, "ctime": ct, "kind": kind,
                     "s_bits": s.bit_length(), "packet": pkt.hex(), "gnupg_ok": v.returncode == 0})
    ver = subprocess.run(["gpg", "--version"], capture_output=True, text=True).stdout.splitlines()[0]
    return json.dumps({"gnupg": ver, "cases": rows}, indent=1) + "\n"


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "signature_sign.json")
    with open(path, "w") as f:
        f.write(generate())
