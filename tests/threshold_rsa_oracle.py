"""CPU restatement of crypto/threshold/rsa/rsa.go in Python ints: the test oracle for bftq_thrsa_sign_batch and
bftq_thrsa_process_batch.

splitKey / makeKeyTree / collectKeys / Distribute (a seeded random.Random stands in for crypto/rand), every serializer
and parser, rsaContext.Sign (with the in-place Neg of a negative fragment), and rsaProc.ProcessResponse / missingKeys.
Where Go iterates a map (fragments of a share, entries of a partial signature) the order here is the library's:
fragments by key index, partial-signature entries in the order the request first lists them, responses' entries
registered in the order they are listed."""
import hashlib
import random
import struct

M32 = 0xFFFFFFFF
SHA256_PREFIX = bytes([0x30, 0x31, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01, 0x65, 0x03, 0x04, 0x02, 0x01, 0x05, 0x00, 0x04, 0x20])


class ParseError(Exception):
    pass


class InvalidInput(Exception):
    """crypto.ErrInvalidInput"""


# ---- key distribution (rsa.go:48-135) ----------------------------------------------------------------------------
def depth(idx, n):
    d = 0
    while idx != 0:
        idx = (idx - 1) // n
        d += 1
    return d


def in_path(i, path, n):
    while path != 0:
        if i == ((path - 1) & M32) % n:
            return True
        path = (path - 1) // n
    return False


def split_key(d, n, rng):
    mx = 1 << (d.bit_length() * 2)
    di, s = [], 0
    for _ in range(n - 1):
        x = rng.randrange(mx)
        sign = x & 1
        x >>= 1
        if sign:
            x = -x
        di.append(x)
        s += x
    di.append(d - s)
    return di


def make_key_tree(key, idx, n, k, rng):
    """(idx, di, children: {i: subtree} or None)"""
    if depth(idx, n) > n - k:
        return (idx, key, None)
    di = split_key(key, n - depth(idx, n), rng)
    children, j = {}, 0
    for i in range(n):
        if not in_path(i, idx, n):
            children[i] = make_key_tree(di[j], (idx * n + i + 1) & M32, n, k, rng)
            j += 1
    return (idx, key, children)


def collect_keys(tr, i, keys):
    idx, _, children = tr
    for j, c in (children or {}).items():
        if j == i:
            keys[idx] = c[1]
        else:
            collect_keys(c, i, keys)


def distribute(d, N, n, k, seed=1):
    """Distribute: the n serialized shares."""
    rng = random.Random(seed)
    kt = make_key_tree(d, 0, n, k, rng)
    shares = []
    for i in range(n):
        keys = {}
        collect_keys(kt, i, keys)
        shares.append(serialize_partial_param(keys, N, i, n))
    return shares


# ---- marshaling (rsa.go:399-605) ---------------------------------------------------------------------------------
def int_bytes(x):
    return x.to_bytes((x.bit_length() + 7) // 8, "big") if x else b""


def chunk(b):
    return struct.pack(">Q", len(b)) + b


class Reader:
    def __init__(self, b):
        self.b, self.p = b, 0

    def take(self, n):
        if len(self.b) - self.p < n:
            raise ParseError("EOF")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def u8(self):
        return self.take(1)[0]

    def u16(self):
        return struct.unpack(">H", self.take(2))[0]

    def u32(self):
        return struct.unpack(">I", self.take(4))[0]

    def chunk(self):
        return self.take(struct.unpack(">Q", self.take(8))[0])


def serialize_partial_param(keys, N, pid, n):
    out = struct.pack(">H", len(keys))
    for idx in sorted(keys):
        k = keys[idx]
        out += struct.pack(">IB", idx, 1 if k < 0 else 0) + chunk(int_bytes(abs(k)))
    return out + chunk(int_bytes(N)) + struct.pack(">IB", pid, n)


def parse_partial_param(b):
    r = Reader(b)
    keys = {}
    for _ in range(r.u16()):
        idx = r.u32()
        sign = r.u8()
        v = int.from_bytes(r.chunk(), "big")
        keys[idx] = -v if sign else v
    N = int.from_bytes(r.chunk(), "big")
    pid = r.u32()
    n = r.u8()
    return keys, N, pid, n


def serialize_hash_info(prefix, dgst):
    return chunk(prefix) + chunk(dgst)


def hash_info_sha256(tbs):
    return serialize_hash_info(SHA256_PREFIX, hashlib.sha256(tbs).digest())


def serialize_sign_request(keys, hinfo):
    return struct.pack(">H", len(keys)) + b"".join(struct.pack(">I", k) for k in keys) + chunk(hinfo)


def parse_sign_request(b):
    r = Reader(b)
    keys = [r.u32() for _ in range(r.u16())]
    hr = Reader(r.chunk())
    return keys, (hr.chunk(), hr.chunk())


def serialize_partial_signature(sigs, N):
    """sigs: list of (idx, value) in output order"""
    return struct.pack(">H", len(sigs)) + b"".join(struct.pack(">I", i) + chunk(int_bytes(s)) for i, s in sigs) + chunk(int_bytes(N))


def parse_partial_signature(b):
    """(list of (idx, value) in first-appearance order with the last value, N)"""
    r = Reader(b)
    sigs, pos = [], {}
    for _ in range(r.u16()):
        idx = r.u32()
        v = int.from_bytes(r.chunk(), "big")
        if idx in pos:
            sigs[pos[idx]] = (idx, v)
        else:
            pos[idx] = len(sigs)
            sigs.append((idx, v))
    N = int.from_bytes(r.chunk(), "big")
    return sigs, N


def emsa_encode(prefix, dgst, N):
    emlen = (N.bit_length() + 7) // 8
    padlen = emlen - (len(prefix) + len(dgst))
    if padlen < 3:
        raise InvalidInput()
    em = b"\x00\x01" + b"\xff" * (padlen - 3) + b"\x00" + prefix + dgst
    return int.from_bytes(em, "big")


def i2os(x, sz):
    c = int_bytes(x)
    return c if len(c) >= sz else b"\x00" * (sz - len(c)) + c


# ---- server: rsaContext.Sign (rsa.go:140-178) --------------------------------------------------------------------
def sign(sec, req):
    """(bytes or None, None) or (None, 'malformed' | 'invalid_input')."""
    try:
        keys, (prefix, dgst) = parse_sign_request(req)
    except ParseError:
        return None, "malformed"
    try:
        frags, N, pid, n = parse_partial_param(sec)
    except ParseError:
        return None, "malformed"
    try:
        m = emsa_encode(prefix, dgst, N)
    except InvalidInput:
        return None, "invalid_input"
    frags = dict(frags)                      # parsed per call: the Neg below does not outlive it
    sigs, order = {}, []
    for kid in keys:
        if kid in frags:
            di = frags[kid]
            if di < 0:
                di = -di
                frags[kid] = di              # di.Neg(di) negates the map's entry in place
                ci = pow(pow(m, di, N), -1, N)
            else:
                ci = pow(m, di, N)
            o = (kid * n + pid + 1) & M32
            if o not in sigs:
                order.append(o)
            sigs[o] = ci
    if not sigs:
        return None, None
    return serialize_partial_signature([(o, sigs[o]) for o in order], N), None


# ---- client: rsaProc.ProcessResponse (rsa.go:235-338) ------------------------------------------------------------
class Node:
    def __init__(self, idx, psig=None, completed=False):
        self.idx, self.psig, self.completed, self.children = idx, psig, completed, {}


def register(st, idx, psig, d, n):
    self_ = idx
    for _ in range(d - 1):
        self_ = (self_ - 1) // n
    i = ((self_ - 1) & M32) % n
    c = st.children.get(i)
    if c is None:
        c = Node(self_, psig, True) if d <= 1 else Node(self_)
        st.children[i] = c
    if d > 1:
        register(c, idx, psig, d - 1, n)
    if len(st.children) >= n - depth(st.idx, n):
        st.completed = all(ch.completed for ch in st.children.values())


def missing_keys(st, keys, n, k):
    if st is None or st.completed:
        return keys
    if not st.children:
        keys.append(st.idx)
    else:
        if depth(st.idx, n) >= n - k:
            return keys
        for i in range(n):
            if in_path(i, st.idx, n):
                continue
            c = st.children.get(i)
            if c is None:
                keys.append((st.idx * n + i + 1) & M32)
            elif not c.completed:
                keys = missing_keys(c, keys, n, k)
    return keys


def calculate(st, s, N):
    if not st.completed:
        return s
    if st.psig is not None:
        return s * st.psig % N
    for c in st.children.values():
        s = calculate(c, s, N)
    return s


SIGNED, FAILED, INCOMPLETE = "signed", "failed", "incomplete"


def process(n, k, responses):
    """ProcessResponse over responses in arrival order, stopping at the first signature or error:
    (state, index of the deciding response or len(responses), signature or None, missing keys)."""
    root = Node(0)
    for j, data in enumerate(responses):
        try:
            sigs, N = parse_partial_signature(data)
        except ParseError:
            return FAILED, j, None, []
        for idx, s in sigs:
            register(root, idx, s, depth(idx, n), n)
        if root.completed:
            return SIGNED, j, i2os(calculate(root, 1, N), (N.bit_length() + 7) // 8), []
    return INCOMPLETE, len(responses), None, missing_keys(root, [], n, k)


def make_request(n, k, responses, hinfo):
    """MakeRequest after the given responses: the next request, or None when missingKeys is empty."""
    st, _, _, keys = process(n, k, responses)
    if st != INCOMPLETE or not keys:
        return None
    return serialize_sign_request(keys, hinfo)
