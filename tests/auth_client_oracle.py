"""The client half of crypto/auth (auth.go AuthClient) as the device runs it, on top of auth_oracle.Client: the caller
chooses a and every a', maps carry every secret's entry (empty for a peer with no Ni or Pi), a failed open leaves the
peer with no Pi, and the wire form of a returned map.  Shared by tests/test_auth_client_gpu.py and tools/auth_client_time.py."""
import struct

import auth_oracle as A


class NoAuthData(Exception):
    pass


class Insufficient(Exception):
    pass


class OracleClient(A.Client):
    """auth_oracle.Client driven by the caller's a and a' values (a' in the order the secrets first arrived), with the
    map entries of peers that never answered (empty Ni / Pi), and the device's fail-closed phase 2: with
    reference_zero_key_quirk False, a peer with no phase-1 keys, or a nonce that is not 12 bytes, is ErrDecryptionFailed
    (auth.go opens under an all-zero key, and panics on the nonce)."""

    def __init__(self, password, n, k, reference_zero_key_quirk=False):
        super().__init__(password, n, k, None)
        self.quirk = reference_zero_key_quirk
        self.a = None

    def initiate(self, a: int) -> bytes:
        self.a = a
        return A.i2b(pow(A.PI(self.password), a, A.P))

    def yi(self, res, pid, a2s):
        x, yi, salt = A.parse_yi(res)
        self.secrets[pid] = {"x": x, "Y": yi, "salt": salt}
        if len(self.secrets) < self.k:
            return None
        self.gs = self.calculate_shared_secret()
        out = {}
        for (i, s), a2 in zip(self.secrets.items(), a2s):
            s["a2"] = a2
            si = int.from_bytes(A.h(self.password, s["salt"]), "big")
            s["Xi"] = A.i2b(pow(self.gs, a2 * si % A.Q, A.P))
            out[i] = s["Xi"]
        self.nresponses = 0
        return out

    def bi(self, res, pid):
        bi = A.parse_bi(res)
        if pid not in self.secrets:
            raise NoAuthData()
        s = self.secrets[pid]
        ki = pow(bi, self.a * s["a2"] % A.Q, A.P)
        s["km"], s["ke"] = A.key_sched(A.i2b(ki), s["salt"])
        s["Ni"] = A.calculate_mac(s["km"], s["Xi"], A.i2b(bi))
        self.nresponses += 1
        if self.nresponses >= len(self.secrets):
            self.nresponses = 0
            return {i: t.get("Ni", b"") for i, t in self.secrets.items()}
        return None

    def zi(self, res, pid):
        zi, nonce = A.parse_zi(res)
        if pid not in self.secrets:
            raise NoAuthData()
        s = self.secrets[pid]
        s["Pi"] = b""                                   # secret.Pi, err = decrypt(...): a failed open leaves nil
        if not self.quirk and ("ke" not in s or len(nonce) != 12):
            raise A.DecryptionFailed()
        s["Pi"] = A.gcm_open(s.get("ke", bytes(16)), nonce, zi, s.get("Ni", b""))
        self.nresponses += 1
        if self.nresponses >= len(self.secrets):
            return {i: t.get("Pi", b"") for i, t in self.secrets.items()}
        return None

    def cipher_key(self):
        if self.gs is None:
            raise Insufficient()
        return self.get_cipher_key()


def wire_map(m):
    return struct.pack(">I", len(m)) + b"".join(struct.pack(">QQ", i, len(v)) + v for i, v in m.items())
