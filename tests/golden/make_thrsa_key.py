#!/usr/bin/env python3
"""Generates tests/golden/thrsa_key.json — run once with BFTKV_SRC naming a yahoo/bftkv checkout.  The output is committed.

crypto/threshold/rsa/test.pkcs8 is the reference-owned key whose public half and PKCS#1 v1.5 signature over "tbs" are
golden.json's ref_rsa_kat (read the same way as make_golden.py).  The threshold tests split its private exponent d with
splitKey, so they need d (and p, q to check it) as numbers."""
import json, os, sys
from cryptography.hazmat.primitives import serialization

SRC = os.environ.get("BFTKV_SRC", "")
raw = open(os.path.join(SRC, "crypto/threshold/rsa/test.pkcs8"), "rb").read()
try:
    key = serialization.load_der_private_key(raw, None)
except ValueError:
    key = serialization.load_pem_private_key(raw, None)
pr = key.private_numbers()
assert pr.p * pr.q == pr.public_numbers.n
out = os.path.join(os.path.dirname(__file__), "thrsa_key.json")
json.dump({"generator": "tests/golden/make_thrsa_key.py", "source": "crypto/threshold/rsa/test.pkcs8",
           "n": "%x" % pr.public_numbers.n, "e": pr.public_numbers.e, "d": "%x" % pr.d, "p": "%x" % pr.p, "q": "%x" % pr.q},
          open(out, "w"), indent=0)
print("wrote", out, file=sys.stderr)
