"""CPU suite: the crypto/auth oracle (tests/auth_oracle.py) restates TestAuth, its symmetric layer agrees with
`cryptography` and RFC 5869, its serializers round-trip, and it reproduces the reference's zero-key quirk (a phase 2
before any phase 1 is answered, and the proof is readable under an all-zero key)."""
import pytest

import auth_oracle as A


def test_group_is_a_safe_prime():
    assert A.P.bit_length() == 2048 and A.P == 2 * A.Q + 1
    for base in (2, 3, 5, 7):
        assert pow(base, A.P - 1, A.P) == 1 and pow(base, A.Q - 1, A.Q) == 1


@pytest.mark.parametrize("n,k,rounds", [(10, 7, 10), (4, 3, 3)])
def test_test_auth_restated(n, k, rounds):
    rng = A.Rng(0xA17 + n)
    for _ in range(rounds):
        password, proof = rng.randbytes(8), rng.randbytes(16)
        c, pis = A.run_round(password, proof, n, k, rng)
        assert pis is not None and len(pis) >= k
        assert all(p == proof for p in pis.values())
        assert len(c.get_cipher_key()) == 32


def test_servers_and_client_share_keys():
    rng = A.Rng(0xA18)
    params = A.generate_params(b"password", 4, 3, rng)
    servers = [A.Server(p, b"proof") for p in params]
    c = A.Client(b"password", 4, 3, rng)
    X = c.generate_x()
    xis = None
    for i in range(4):
        xis = c.process_yi(servers[i].make_yi(X), i)
        if xis:
            break
    for i, xi in xis.items():
        c.process_bi(servers[i].make_bi(xi, rng.randbelow(A.P)), i)
        assert c.secrets[i]["km"] == servers[i].km and c.secrets[i]["ke"] == servers[i].ke
        assert c.secrets[i]["Ni"] == servers[i].mac


def test_hkdf_rfc5869_a1():
    ikm = bytes([0x0b] * 22)
    salt = bytes(range(13))
    info = bytes(range(0xf0, 0xfa))
    okm = A.hkdf_sha256(ikm, salt, info, 42)
    assert okm.hex() == ("3cb25f25faacd57a90434f64d0362f2a2d2d0a90cf1a5a4c5db02d56ecc4c5bf34007208d5b887185865")


@pytest.mark.parametrize("salt_len", [0, 1, 32, 64, 65, 200])
@pytest.mark.parametrize("ikm_len", [0, 1, 255, 256])
def test_hkdf_and_hmac_match_cryptography(salt_len, ikm_len):
    from cryptography.hazmat.primitives import hashes, hmac
    from cryptography.hazmat.primitives.kdf.hkdf import HKDF
    rng = A.Rng(salt_len * 1000 + ikm_len)
    salt, ikm = rng.randbytes(salt_len), rng.randbytes(ikm_len)
    want = HKDF(hashes.SHA256(), 32, salt or None, None).derive(ikm)
    assert A.hkdf_sha256(ikm, salt) == want
    km, ke = A.key_sched(ikm, salt)
    assert km + ke == want
    m = hmac.HMAC(km, hashes.SHA256())
    m.update(ikm + salt)
    assert A.calculate_mac(km, ikm, salt) == m.finalize()


@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 4096])
def test_gcm_matches_cryptography(n):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    rng = A.Rng(n)
    key, nonce, pt, aad = rng.randbytes(16), rng.randbytes(12), rng.randbytes(n), rng.randbytes(32)
    ct = A.gcm_seal(key, nonce, pt, aad)
    assert ct == AESGCM(key).encrypt(nonce, pt, aad)
    assert A.gcm_open(key, nonce, ct, aad) == pt


def test_serializers_round_trip():
    rng = A.Rng(5)
    for x, y, v, salt in [(1, 0, 0, b""), (-7, A.Q - 1, A.P - 1, rng.randbytes(100)), (2 ** 31 - 1, 5, 1, b"\0\1")]:
        assert A.parse_params(A.serialize_params(x, y, v, salt)) == (x, y, v, salt)
        assert A.parse_yi(A.serialize_yi(x, v, salt)) == (x, v, salt)
    assert A.parse_bi(A.serialize_bi(0)) == 0 and A.serialize_bi(0) == bytes(8)
    assert A.parse_bi(A.serialize_bi(A.P - 1)) == A.P - 1
    assert A.parse_zi(A.serialize_zi(b"ab", b"n" * 12)) == (b"ab", b"n" * 12)
    with pytest.raises(ValueError):
        A.parse_params(A.serialize_params(1, 2, 3, b"salt")[:-1])


def test_reference_zero_key_quirk_leaks_the_proof():
    """auth.go: a fresh server (mac == nil) answers a phase 2 with an empty Ni; AES-GCM under the all-zero key opens it."""
    rng = A.Rng(9)
    params = A.generate_params(b"pw", 4, 3, rng)
    proof = b"a collective signature over the variable"
    s = A.Server(params[0], proof, reference_zero_key_quirk=True)
    res, done, err = s.make_response(2, b"", rng.randbytes(12))
    assert err is None and done
    zi, nonce = A.parse_zi(res)
    assert A.gcm_open(bytes(16), nonce, zi, b"") == proof
    s2 = A.Server(params[0], proof, reference_zero_key_quirk=False)
    assert s2.make_response(2, b"", rng.randbytes(12)) == (None, True, "authentication failure")


def test_wrong_ni_fails():
    rng = A.Rng(10)
    params = A.generate_params(b"pw", 4, 3, rng)
    s = A.Server(params[0], b"proof")
    s.make_bi(A.i2b(rng.randbelow(A.P)), rng.randbelow(A.P))
    bad = bytes([s.mac[0] ^ 1]) + s.mac[1:]
    assert s.make_response(2, bad, rng.randbytes(12))[2] == "authentication failure"
    zi, nonce = A.parse_zi(s.make_response(2, s.mac, rng.randbytes(12))[0])
    assert A.gcm_open(s.ke, nonce, zi, s.mac) == b"proof"
