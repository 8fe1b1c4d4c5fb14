#!/usr/bin/env python3
"""Makes tests/golden/data_encryption.json: passphrase-encrypted OpenPGP messages and GnuPG's verdict on each, the
external pin for DataEncryption's oracle (tests/data_encryption_oracle.py) and for K11.

  gnupg   messages GnuPG wrote (gpg --symmetric --rfc4880 --compress-algo none): S2K modes 0 / 1 / 3 at counts 1024,
          65536 and 2^20 over SHA-256, AES-128 / 192 / 256, bodies of 0 .. 70000 bytes, one with a flipped MDC byte, one
          truncated, one compressed and one under 3DES.
  go      messages in Go's shape (SymmetricallyEncrypt's writer cascade) written by the oracle from fixed randomness,
          with GnuPG's decryption of each.
Each case: the passphrase, the message (base64), GnuPG's verdict, the length and SHA-256 of the plain text GnuPG returned,
the seed of the value that was encrypted (tests/data_encryption_oracle.py's fixture_value) and the error code the device
answers.  GnuPG passphrases are text, so binary keys are covered by the oracle only.  Plain texts carry
no CR byte: GnuPG rewrites CR LF in text-mode literal data.

  python tests/golden/make_data_encryption.py        # needs gpg (2.4 here); writes the JSON next to this file
"""
import base64
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import data_encryption_oracle as O  # noqa: E402

OK, MALFORMED, UNSUPPORTED, MDC = 0, -8, -11, -12


def gpg(home, passphrase, *args, stdin=None):
    return subprocess.run(["gpg", "--homedir", home, "--batch", "--yes", "--quiet", "--pinentry-mode", "loopback", "--passphrase", passphrase]
                          + list(args), input=stdin, capture_output=True)


def main():
    home = tempfile.mkdtemp(prefix="bftq-gpg-")
    os.chmod(home, 0o700)
    cases = []

    def verdict(pw, msg):
        r = gpg(home, pw, "--decrypt", stdin=msg)
        return r.returncode == 0, r.stdout

    def add(name, pw, msg, plain, code, source):
        ok, got = verdict(pw, msg)
        if code == OK:
            assert ok and got == plain, name
        cases.append({"name": name, "source": source, "passphrase": pw, "message": base64.b64encode(msg).decode(), "seed": seed,
                      "plain_len": len(plain) if plain is not None else None, "gnupg_ok": ok,
                      "gnupg_plain_sha256": hashlib.sha256(got).hexdigest() if ok else None, "code": code})

    def sym(pw, plain, *extra):
        r = gpg(home, pw, "--symmetric", "--rfc4880", "--s2k-digest-algo", "SHA256", *extra, stdin=plain)
        assert r.returncode == 0, r.stderr
        return r.stdout

    base = ("--compress-algo", "none")
    seed = 0
    for mode, counts in ((0, (None,)), (1, (None,)), (3, (1024, 65536, 1 << 20))):
        for cnt in counts:
            for algo in ("AES", "AES192", "AES256"):
                seed += 1
                plain = O.fixture_value(513, seed)
                args = base + ("--cipher-algo", algo, "--s2k-mode", str(mode)) + (("--s2k-count", str(cnt)) if cnt else ())
                add("mode%d-count%s-%s" % (mode, cnt, algo), "pw-%d" % seed, sym("pw-%d" % seed, plain, *args), plain, OK, "gnupg")
    for n in (0, 1, 511, 512, 513, 16383, 16384, 16385, 70000):
        seed += 1
        plain = O.fixture_value(n, seed)
        add("body-%d" % n, "secret", sym("secret", plain, *base, "--cipher-algo", "AES"), plain, OK, "gnupg")
    seed += 1
    plain = O.fixture_value(300, seed)
    msg = bytearray(sym("secret", plain, *base, "--cipher-algo", "AES"))
    msg[-1] ^= 0x01                                                # the last byte of the MDC
    add("flipped-mdc", "secret", bytes(msg), None, MDC, "gnupg")
    msg = sym("secret", plain, *base, "--cipher-algo", "AES")
    add("truncated", "secret", msg[:-30], None, MALFORMED, "gnupg")
    add("compressed", "secret", sym("secret", plain, "--cipher-algo", "AES"), None, UNSUPPORTED, "gnupg")
    add("3des", "secret", sym("secret", plain, *base, "--cipher-algo", "3DES"), None, UNSUPPORTED, "gnupg")
    # Go's writer, from fixed randomness
    for n in (0, 1, 2, 15, 16, 17, 511, 512, 513, 16385):
        seed += 1
        plain = O.fixture_value(n, seed)
        rand = hashlib.sha512(b"rand/%d" % seed).digest()[:40]
        pw = "go-%d" % seed
        add("go-%d" % n, pw, O.encrypt(pw.encode(), plain, rand), plain, OK, "go")
        cases[-1]["rand"] = rand.hex()
    json.dump({"gnupg": subprocess.run(["gpg", "--version"], capture_output=True, text=True).stdout.split("\n")[0], "cases": cases},
              open(os.path.join(HERE, "data_encryption.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
