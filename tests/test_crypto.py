"""CPU tier: the plain entry-cipher references (tests/crypto_ref.py) against the published known answers (FIPS 197, RFC 2202,
RFC 6070), against the oracle at every short length and password length, and against `cryptography` and zipfile where
they exist; and the entry-cipher kernels run the GPU tier's small cases (tests/test_gpu_crypto_edges.py, "emu") on the
CUDA emulator, in the default schedule and with the threads and blocks resumed in reverse order."""
import hashlib
import hmac
import os
import subprocess
import sys

import numpy as np
import pytest

import crypto_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PT = bytes.fromhex("00112233445566778899aabbccddeeff")


def _enc1(key, block):
    return R.aes_encrypt(key, np.frombuffer(block, np.uint8)).tobytes()


def test_aes_known_answers():
    """FIPS 197: the S-box entries of 5.1.1, Appendix A's last round-key words, Appendix B and C.1 / C.3"""
    assert (int(R.SBOX[0x00]), int(R.SBOX[0x53]), int(R.SBOX[0xFF])) == (0x63, 0xED, 0x16)
    assert sorted(R.SBOX.tolist()) == list(range(256))
    k128 = bytes.fromhex("2b7e151628aed2a6abf7158809cf4f3c")
    k256 = bytes.fromhex("603deb1015ca71be2b73aef0857d77811f352c073b6108d72d9810a30914dff4")
    assert R.expand_key(k128)[-1, 12:].tobytes().hex() == "b6630ca6"  # A.1, w[43]
    assert R.expand_key(k256)[-1, 12:].tobytes().hex() == "706c631e"  # A.3, w[59]
    assert _enc1(k128, bytes.fromhex("3243f6a8885a308d313198a2e0370734")).hex() == "3925841d02dc09fbdc118597196a0b32"  # B
    assert _enc1(bytes(range(16)), PT).hex() == "69c4e0d86a7b0430d8cdb78070b4c55a"  # C.1
    assert _enc1(bytes(range(32)), PT).hex() == "8ea2b7ca516745bfeafc49904b496089"  # C.3


def test_hmac_and_pbkdf2_known_answers():
    """RFC 2202 section 3 (HMAC-SHA1, all seven cases) and RFC 6070 (PBKDF2-HMAC-SHA1)"""
    rfc2202 = [
        (b"\x0b" * 20, b"Hi There", "b617318655057264e28bc0b6fb378c8ef146be00"),
        (b"Jefe", b"what do ya want for nothing?", "effcdf6ae5eb2fa2d27416d5f184df9c259a7c79"),
        (b"\xaa" * 20, b"\xdd" * 50, "125d7342b9ac11cd91a39af48aa17b4f63f175d3"),
        (bytes(range(1, 26)), b"\xcd" * 50, "4c9007f4026250c6bc8414f9bf50c86c2d7235da"),
        (b"\x0c" * 20, b"Test With Truncation", "4c1a03424b55e07fe7f27be1d58bb9324a9a5a04"),
        (b"\xaa" * 80, b"Test Using Larger Than Block-Size Key - Hash Key First", "aa4ae5e15272d00e95705637ce8a3b55ed402112"),
        (b"\xaa" * 80, b"Test Using Larger Than Block-Size Key and Larger Than One Block-Size Data",
         "e8e99d0f45237d786d6bbaa7965c7808bbff1a91"),
    ]
    for key, data, want in rfc2202:
        mac = R.new_mac(key)
        R.mac_update(mac, data[:7])
        R.mac_update(mac, data[7:])
        assert mac.hexdigest() == want, key
    rfc6070 = [
        (b"password", b"salt", 1, 20, "0c60c80f961f0e71f3a9b524af6012062fe037a6"),
        (b"password", b"salt", 2, 20, "ea6c014dc72d6f8ccd1ed92ace1d41f0d8de8957"),
        (b"password", b"salt", 4096, 20, "4b007901b765489abead49d926f721d065a429c1"),
        (b"passwordPASSWORDpassword", b"saltSALTsaltSALTsaltSALTsaltSALTsalt", 4096, 25,
         "3d2eec4fe41c849b80c8d83662c0e44a8b291a964cf2f07038"),
        (b"pass\0word", b"sa\0lt", 4096, 16, "56fa6aa75548099dcc37d7f03425e0c3"),
    ]
    for pw, salt, c, n, want in rfc6070:
        assert hashlib.pbkdf2_hmac("sha1", pw, salt, c, n).hex() == want, (pw, c)


def test_keystream_layout():
    """block k is AES(k + 1, little-endian); a keystream from any start is the matching slice of the one from 0"""
    key = bytes(range(100, 132))
    assert R.counter_blocks([0, 255, 2 ** 32])[:, :6].tolist() == [[1, 0, 0, 0, 0, 0], [0, 1, 0, 0, 0, 0], [1, 0, 0, 0, 1, 0]]
    whole = R.zip_aes_keystream(key, 0, 300)
    assert whole[:16].tobytes() == _enc1(key, (1).to_bytes(16, "little"))
    for start in (0, 1, 15, 16, 17, 100):
        for n in (0, 1, 16, 33, 300 - start):
            assert (R.zip_aes_keystream(key, start, n) == whole[start:start + n]).all(), (start, n)


@pytest.mark.parametrize("key_bytes", [16, 32])
def test_zip_aes_matches_the_oracle_at_every_short_length(oracle, key_bytes):
    """every entry length 0-300, both directions: output, verifier and all 20 bytes of the auth code"""
    rng = np.random.default_rng(key_bytes)
    pw, salt = "pässwörd", rng.bytes(key_bytes // 2)
    data = rng.bytes(300)
    for n in range(301):
        ct, pv, mac = R.zip_aes(pw, salt, key_bytes, True, data[:n])
        assert (ct, pv, mac) == oracle.zip_aes(pw.encode(), salt, key_bytes, True, data[:n]), n
        assert (data[:n], pv, mac) == R.zip_aes(pw, salt, key_bytes, False, ct) == \
            oracle.zip_aes(pw.encode(), salt, key_bytes, False, ct), n


def password_set():
    """every password length 0-200 plus 255 and 1000 (ASCII, binary and UTF-8 mixed), and a few UTF-8 words"""
    out = []
    for n in list(range(201)) + [255, 1000]:
        if n % 3 == 0:
            out.append(bytes((33 + (7 * i + n) % 94) for i in range(n)))
        elif n % 3 == 1:
            out.append(bytes((i * 131 + n * 17) & 0xFF for i in range(n)))
        else:
            out.append(("é" * n).encode()[:n])
    return out + ["pässwörd".encode(), "密码".encode(), "🔑".encode() * 17]


def test_password_lengths_match_the_oracle(oracle):
    """PBKDF2 for every password length 0-200, 255 and 1000: the hashed-key branch past 64 bytes and its two-block padding
    (lengths 120-127 and 184-191)"""
    for kb in (16, 32):
        for i, pw in enumerate(password_set()):
            salt = bytes((i + j) & 0xFF for j in range(kb // 2))
            want = oracle.pbkdf2_sha1(pw, salt, 1000, 2 * kb + 2)
            assert b"".join(R.derive(pw, salt, kb)) == want, (kb, len(pw))


def test_pkzip_matches_the_oracle():
    """generate_keys for seeds of length 1-300, transform at lengths 0-300 in both directions with the keys after"""
    import oracle_lib as O
    rng = np.random.default_rng(9)
    seed = rng.bytes(300)
    for n in range(1, 301):
        assert R.generate_keys(seed[:n]) == O.pkzip_generate_keys(seed[:n]), n
    keys = R.generate_keys(b"secret")
    data = rng.bytes(300)
    for n in range(301):
        enc = R.transform(keys, True, data[:n])
        assert enc == O.pkzip_transform(keys, True, data[:n]), n
        dec = R.transform(keys, False, enc[0])
        assert dec == O.pkzip_transform(keys, False, enc[0]) and dec == (data[:n], enc[1]), n


def test_references_against_cryptography():
    hz = pytest.importorskip("cryptography.hazmat.primitives")  # noqa: F841
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
    rng = np.random.default_rng(11)
    for kb in (16, 32):
        key = rng.bytes(kb)
        blocks = rng.integers(0, 256, (4099, 16), dtype=np.uint8)
        enc = Cipher(algorithms.AES(key), modes.ECB()).encryptor()
        assert R.aes_encrypt(key, blocks).tobytes() == enc.update(blocks.tobytes()) + enc.finalize()
        # the keystream from its definition, with the little-endian counters made here from Python integers
        starts = [0, 255, 2 ** 32 - 2, 2 ** 40 + 7]
        for s in starts:
            enc = Cipher(algorithms.AES(key), modes.ECB()).encryptor()
            want = b"".join(enc.update((k + 1).to_bytes(16, "little")) for k in range(s, s + 300))
            assert R.zip_aes_keystream(key, 16 * s + 5, 300 * 16 - 5).tobytes() == want[5:], s


def test_pkzip_against_zipfile():
    import zipfile
    Dec = getattr(zipfile, "_ZipDecrypter", None)
    if Dec is None:
        pytest.skip("this Python's zipfile has no _ZipDecrypter")
    data = np.random.default_rng(12).bytes(1000)
    for pw in (b"a", b"secret", bytes(range(256))):
        ct, _ = R.transform(R.generate_keys(pw), True, data)
        assert bytes(Dec(pw)(ct)) == data, pw


def test_mac_from_chunks(monkeypatch):
    """mac_update over bounded chunks and sub-ranges gives the one-shot HMAC"""
    import checksum_ref
    monkeypatch.setattr(checksum_ref, "CHUNK", 1000)
    d = np.random.default_rng(13).integers(0, 256, 10007, dtype=np.uint8)
    key = b"k" * 32
    assert R.mac_update(R.new_mac(key), d).digest() == hmac.new(key, d.tobytes(), hashlib.sha1).digest()
    m = R.mac_update(R.new_mac(key), d, 0, 999)
    assert R.mac_update(m, d, 999, 10007).digest() == hmac.new(key, d.tobytes(), hashlib.sha1).digest()


@pytest.mark.parametrize("order", ["fwd", "rev"])
def test_crypto_kernels_on_the_emulator(order):
    env = dict(os.environ)
    if order == "rev":
        env["B200Z_EMU_ORDER"] = "rev"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"),
                        os.path.join(ROOT, "tests", "test_gpu_crypto_edges.py"), "-k", "emu"],
                       capture_output=True, text=True, timeout=1500, env=env)
    assert r.returncode == 0 and " passed" in r.stdout and "deselected" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
