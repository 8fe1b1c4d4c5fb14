#!/usr/bin/env python3
"""Generates tests/golden/thdsa_key.json — run once with BFTKV_SRC naming a yahoo/bftkv checkout.  The output is committed.

crypto/threshold/dsa/test.pkcs8 is the reference-owned DSA key its threshold tests load (dsa_test.go:26-28): a
1024-bit p with a 160-bit q.  The threshold tests here deal its private x with the oracle's Distribute."""
import json, os, sys
from cryptography.hazmat.primitives import serialization

SRC = os.environ.get("BFTKV_SRC", "")
raw = open(os.path.join(SRC, "crypto/threshold/dsa/test.pkcs8"), "rb").read()
try:
    key = serialization.load_der_private_key(raw, None)
except ValueError:
    key = serialization.load_pem_private_key(raw, None)
pr = key.private_numbers()
pn = pr.public_numbers.parameter_numbers
assert pow(pn.g, pr.x, pn.p) == pr.public_numbers.y
out = os.path.join(os.path.dirname(__file__), "thdsa_key.json")
json.dump({"generator": "tests/golden/make_thdsa_key.py", "source": "crypto/threshold/dsa/test.pkcs8",
           "p": "%x" % pn.p, "q": "%x" % pn.q, "g": "%x" % pn.g, "y": "%x" % pr.public_numbers.y, "x": "%x" % pr.x},
          open(out, "w"), indent=0)
print("wrote", out, file=sys.stderr)
