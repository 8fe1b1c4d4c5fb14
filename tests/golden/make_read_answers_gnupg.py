#!/usr/bin/env python3
"""Makes tests/golden/read_answers_gnupg.json: read answers written by GnuPG — one-pass signature, literal data whose
FileName is base64(nonce), signature — around bftkv packets, each signed from a file (old-format definite length) and
from stdin (GnuPG's partial-length chunks), with small and > 8 KiB values, plus tampered copies, and GnuPG's own
--verify verdict on each.  GnuPG makes fresh keys and timestamps on every run, so the output is not reproducible byte
for byte; it is committed.

  python tests/golden/make_read_answers_gnupg.py        # needs gpg (2.4 here); writes the JSON next to this file
"""
import base64
import hashlib
import json
import os
import random
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
from oracle import packet_oracle  # noqa: E402  (makes the packet bytes only)


def gpg(home, *args, stdin=None):
    return subprocess.run(["gpg", "--homedir", home, "--batch", "--yes", "--quiet", "--pinentry-mode", "loopback", "--passphrase", ""] + list(args),
                          input=stdin, capture_output=True)


def framing(msg: bytes) -> str:
    """How the literal data packet behind the one-pass signature packet is framed."""
    p = 2 + msg[1]                                            # the one-pass packet: header, one length octet, body
    h = msg[p]
    if not h & 0x40:
        return "old-definite" if h & 3 != 3 else "old-indeterminate"
    return "partial" if 224 <= msg[p + 1] < 255 else "new-definite"


def main():
    rng = random.Random(0xBF7C6A0)
    home = tempfile.mkdtemp(prefix="bftq-gpg-")
    os.chmod(home, 0o700)
    r = gpg(home, "--quick-gen-key", "r01 (http://localhost:5701) <r01@bftq.test>", "rsa2048", "sign,cert", "never")
    assert r.returncode == 0, r.stderr
    keyring = gpg(home, "--export", "r01").stdout
    cases = []
    for vlen in (5, 300, 9000):
        value = bytes(rng.randrange(256) for _ in range(vlen))
        t = rng.randrange(1, 1 << 40)
        body = packet_oracle.serialize(b"the variable", value, t, None, None)
        for via_stdin in (False, True):
            for tamper in ("", "body", "signature"):
                nonce = b"/"
                while b"/" in base64.b64encode(nonce):             # GnuPG keeps only what follows the last '/' of --set-filename
                    nonce = bytes(rng.randrange(256) for _ in range(8))
                out, src = os.path.join(home, "out.gpg"), os.path.join(home, "in.bin")
                open(src, "wb").write(body)
                a = ["--sign", "-u", "r01", "-o", out, "--set-filename", base64.b64encode(nonce).decode(), "--digest-algo", "SHA256", "--compress-algo", "none"]
                r = gpg(home, *a, stdin=body) if via_stdin else gpg(home, *(a + [src]))
                assert r.returncode == 0, r.stderr
                msg = bytearray(open(out, "rb").read())
                if tamper == "body":
                    i = bytes(msg).find(body[8:40])
                    assert i > 0
                    msg[i + 9] ^= 0x04
                elif tamper == "signature":
                    msg[-7] ^= 0x01
                open(out, "wb").write(bytes(msg))
                v = gpg(home, "--verify", out)
                cases.append({"name": "v%d-%s%s" % (vlen, "stdin" if via_stdin else "file", "-tampered-" + tamper if tamper else ""),
                              "msg": bytes(msg).hex(), "nonce": nonce.hex(), "framing": framing(bytes(msg)), "gpg_good": v.returncode == 0,
                              "value_sha256": hashlib.sha256(value).hexdigest(), "t": t})
    ver = subprocess.run(["gpg", "--version"], capture_output=True, text=True).stdout.splitlines()[0]
    json.dump({"made_by": ver, "keyring": keyring.hex(), "cases": cases}, open(os.path.join(HERE, "read_answers_gnupg.json"), "w"), indent=1)
    print("wrote", len(cases), "cases;", ver)


if __name__ == "__main__":
    main()
