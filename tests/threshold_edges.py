"""Operands of tests/golden/threshold_edges.json (written by tests/golden/make_threshold_edges.py).

Big operands are stored as one-character tokens relative to a modulus n and a width of w bytes, and random ones as
SHAKE-256 of their position in the file, so the file stays small:
  "0".."9" the integer;  "-" n - 1;  "=" n - 2;  "n" n;  "+" n + 1 (at most T);  "D" 2 n;  "T" 2^(8 w) - 1;
  "B" 2^(8 w - 1);  "r" random below n;  "G" random in [n, T] (T when n = T);  "s" random below min(n, 2^48);
  "f" random w-byte value;  "h" random w-byte value shifted right by a random amount;  "M" a random multiple of n;
  "L" n shifted left to the top of w bytes, minus 1;  "x<hex>" the value itself (in token lists).
Each record freezes its outputs as `digest`: SHA-256 over (status byte, then the output bytes when the status is 0)."""
import hashlib
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def load():
    return json.load(open(os.path.join(HERE, "golden", "threshold_edges.json")))


def rnd(key, nbytes):
    return int.from_bytes(hashlib.shake_256(key.encode()).digest(nbytes), "big")


def value(tok, n, w, key):
    top = (1 << (8 * w)) - 1
    if tok[0] == "x":
        return int(tok[1:], 16)
    if tok.isdigit():
        return int(tok)
    r = rnd(key, w + 8)
    v = {"-": lambda: n - 1, "=": lambda: n - 2, "n": lambda: n, "+": lambda: min(n + 1, top), "D": lambda: 2 * n,
         "T": lambda: top, "B": lambda: 1 << (8 * w - 1), "r": lambda: r % n,
         "G": lambda: n + r % (top - n + 1) if n < top else top, "s": lambda: r % min(n, 1 << 48), "f": lambda: r & top,
         "h": lambda: (r & top) >> (rnd(key + ">", 2) % (8 * w)), "M": lambda: n * (r % max(1, top // n)),
         "L": lambda: (n << max(0, 8 * w - n.bit_length() - 1)) - 1}[tok]()
    assert 0 <= v <= top, (tok, key)
    return v


def values(toks, n, w, key):
    """toks: a string of one-character tokens or a list of tokens."""
    return [value(t, n, w, "%s/%d" % (key, j)) for j, t in enumerate(toks)]


def digest(statuses, outs, width):
    """outs[i]: int (ignored where statuses[i] != 0)."""
    h = hashlib.sha256()
    for s, o in zip(statuses, outs):
        h.update(bytes([s]) + (int(o).to_bytes(width, "big") if s == 0 else b""))
    return h.hexdigest()[:32]


def mlen_of(m):
    return (m.bit_length() + 7) // 8


def limb_class(mlen):
    return 8 if mlen <= 32 else 16 if mlen <= 64 else 32 if mlen <= 128 else 64


def k3_items(g, moduli):
    """(m, k, [(xs, ys)]) of one K3 group; moduli: the file's "k3_moduli"."""
    m = int(moduli[g["m"]], 16)
    return m, g["k"], [(it["x"], values(it["y"], m, mlen_of(m), "%s/%d" % (g["tag"], i))) for i, it in enumerate(g["items"])]


def modexp_operands(r):
    n = int(r["n"], 16)
    return n, values(r["base"], n, mlen_of(n), r["tag"] + "/b"), values(r["exp"], n, r["elen"], r["tag"] + "/e")


def modprod_rows(r):
    n = int(r["n"], 16)
    return n, [values(row, n, mlen_of(n), "%s/%d" % (r["tag"], i)) for i, row in enumerate(r["vals"])]


def exp_product_rows(r):
    p, q = int(r["p"], 16), int(r["q"], 16)
    return p, q, [(row["x"], values(row["y"], p, mlen_of(p), "%s/%d" % (r["tag"], i))) for i, row in enumerate(r["rows"])]


def dsa_items(d):
    """(p, q, [(xs, Rs, vs)]); R token "g" is g^(random below q) mod p."""
    p, q, g = (int(d[c], 16) for c in "pqg")
    out = []
    for i, it in enumerate(d["items"]):
        key = "%s/%d" % (d["domain"], i)
        Rs = [pow(g, rnd("%s/R/%d" % (key, j), 40) % q, p) if t == "g" else value(t, p, mlen_of(p), "%s/R/%d" % (key, j))
              for j, t in enumerate(it["R"])]
        out.append((it["x"], Rs, values(it["v"], q, mlen_of(q), key + "/v")))
    return p, q, out
