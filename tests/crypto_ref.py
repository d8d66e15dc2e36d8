"""Plain references for the entry ciphers, to hold the kernels of b200z_crypto.cu against.

AES-128 / AES-256 encryption is restated from FIPS 197 and vectorised over blocks with numpy: the S-box is derived from
its definition (the multiplicative inverse in GF(2^8), then the affine map of section 5.1.1), the key is expanded per
section 5.2 and MixColumns multiplies with xtime.  There are no T-tables and no word-packed state, so nothing here can
share a mistake with the kernel's table rounds or its byte order.  About 1 M AES-256 blocks (16 MiB of keystream) take a
few seconds on one CPU core.

WinZip AES (the format ZipAESTransform writes): PBKDF2-HMAC-SHA1 with 1000 rounds gives key1 | key2 | a 2-byte password
verifier; the keystream for 16-byte block k is AES(key1, k + 1 as a 16-byte little-endian integer), all 16 bytes for
either key size; the authentication code is HMAC-SHA1(key2) of the ciphertext.  PBKDF2 and HMAC are Python's (hashlib,
hmac), which are held to RFC 6070 / RFC 2202 by the CPU tier.

PKZIP classic (APPNOTE 6.1): three 32-bit keys updated per plaintext byte with a CRC-32 step, a linear congruential
step (x 134775813 + 1) and a second CRC step; the keystream byte is the high byte of temp * (temp ^ 1), temp = key2 | 2."""
import hashlib
import hmac

import numpy as np

from checksum_ref import CRC_POLY, _chunks


# ---- GF(2^8) and the S-box (FIPS 197 4.2, 5.1.1) -------------------------------------------------------------------------
def gf_mul(a, b):
    """product in GF(2^8) modulo x^8 + x^4 + x^3 + x + 1"""
    p = 0
    while b:
        if b & 1:
            p ^= a
        a = (a << 1) ^ (0x11B if a & 0x80 else 0)
        b >>= 1
    return p


def _sbox():
    box = np.zeros(256, np.uint8)
    for x in range(256):
        inv = next((y for y in range(1, 256) if gf_mul(x, y) == 1), 0)  # 0 maps to 0
        s = 0
        for i in range(8):  # b'_i = b_i ^ b_{i+4} ^ b_{i+5} ^ b_{i+6} ^ b_{i+7} ^ c_i, c = 0x63
            bit = ((inv >> i) ^ (inv >> ((i + 4) % 8)) ^ (inv >> ((i + 5) % 8)) ^ (inv >> ((i + 6) % 8)) ^ (inv >> ((i + 7) % 8))
                   ^ (0x63 >> i)) & 1
            s |= bit << i
        box[x] = s
    return box


SBOX = _sbox()
# ShiftRows on the state as 16 bytes in input order (byte 4c + r is row r, column c): row r moves left by r columns
_SHIFT = np.array([4 * ((c + r) % 4) + r for c in range(4) for r in range(4)])


def expand_key(key):
    """FIPS 197 5.2: the round keys as an (Nr + 1) x 16 byte array"""
    key = bytes(key)
    nk = len(key) // 4
    assert len(key) in (16, 32), len(key)
    nr = nk + 6
    w = [list(key[4 * i:4 * i + 4]) for i in range(nk)]
    rcon = 1
    for i in range(nk, 4 * (nr + 1)):
        t = list(w[i - 1])
        if i % nk == 0:
            t = [int(SBOX[b]) for b in t[1:] + t[:1]]  # SubWord(RotWord(t))
            t[0] ^= rcon
            rcon = gf_mul(rcon, 2)
        elif nk > 6 and i % nk == 4:
            t = [int(SBOX[b]) for b in t]
        w.append([a ^ b for a, b in zip(w[i - nk], t)])
    return np.array(w, np.uint8).reshape(nr + 1, 16)


def _xtime(a):
    return (a << 1) ^ ((a >> 7) * np.uint8(0x1B))


def aes_encrypt(key, blocks):
    """FIPS 197 Cipher() on an (n, 16) uint8 array of blocks"""
    rk = expand_key(key)
    s = np.asarray(blocks, np.uint8).reshape(-1, 16) ^ rk[0]
    for r in range(1, len(rk)):
        s = SBOX[s][:, _SHIFT]
        if r < len(rk) - 1:  # MixColumns, one column of four bytes at a time
            c = s.reshape(-1, 4, 4)
            a0, a1, a2, a3 = c[:, :, 0], c[:, :, 1], c[:, :, 2], c[:, :, 3]
            t = a0 ^ a1 ^ a2 ^ a3
            s = np.stack([a0 ^ t ^ _xtime(a0 ^ a1), a1 ^ t ^ _xtime(a1 ^ a2), a2 ^ t ^ _xtime(a2 ^ a3), a3 ^ t ^ _xtime(a3 ^ a0)],
                         axis=2).reshape(-1, 16)
        s = s ^ rk[r]
    return s


# ---- WinZip AES ------------------------------------------------------------------------------------------------------------
def counter_blocks(block_numbers):
    """the CTR input of 16-byte keystream block k: k + 1 as a 16-byte little-endian integer"""
    k = (np.asarray(block_numbers, np.uint64).reshape(-1) + np.uint64(1)).astype("<u8")
    return np.concatenate([k.view(np.uint8).reshape(-1, 8), np.zeros((k.size, 8), np.uint8)], axis=1)


def keystream_blocks(key1, block_numbers):
    """(len(block_numbers), 16) keystream bytes of the given 16-byte blocks"""
    return aes_encrypt(key1, counter_blocks(block_numbers))


def zip_aes_keystream(key1, start, n):
    """keystream bytes for stream positions start .. start + n"""
    if n <= 0:
        return np.zeros(0, np.uint8)
    b0, b1 = start // 16, (start + n + 15) // 16
    ks = keystream_blocks(key1, np.arange(b0, b1, dtype=np.uint64)).reshape(-1)
    return ks[start - 16 * b0:start - 16 * b0 + n]


def derive(password, salt, key_bytes):
    """ZipAESTransform's constructor: (key1, key2, 2-byte verifier) from PBKDF2-HMAC-SHA1, 1000 rounds"""
    pw = password.encode("utf-8") if isinstance(password, str) else bytes(password)
    d = hashlib.pbkdf2_hmac("sha1", pw, bytes(salt), 1000, 2 * key_bytes + 2)
    return d[:key_bytes], d[key_bytes:2 * key_bytes], d[2 * key_bytes:]


def split_keys(keys_row, key_bytes):
    """one row of key1 | key2 | verifier (what b200z_aes_derive_keys returns) -> (key1, key2, verifier)"""
    k = bytes(np.asarray(keys_row, np.uint8).tobytes())
    return k[:key_bytes], k[key_bytes:2 * key_bytes], k[2 * key_bytes:2 * key_bytes + 2]


def new_mac(key2):
    """the incremental HMAC-SHA1 of the ciphertext: .update() with each piece in order, .digest() for the 20-byte code"""
    return hmac.new(bytes(key2), digestmod=hashlib.sha1)


def mac_update(mac, data, lo=0, hi=None):
    """feed data[lo:hi] to `mac` in bounded chunks (a torch tensor on the device is copied back one chunk at a time)"""
    for c in _chunks(data, lo, hi):
        mac.update(c)
    return mac


def zip_aes_with_keys(key1, key2, write_mode, data, start=0):
    """TransformBlock over `data` at stream position `start`: (output, the ciphertext of this piece)"""
    d = np.frombuffer(bytes(data), np.uint8)
    out = (d ^ zip_aes_keystream(key1, start, d.size)).tobytes()
    return out, (out if write_mode else d.tobytes())


def zip_aes(password, salt, key_bytes, write_mode, data):
    """new ZipAESTransform(password, salt, key_bytes, write_mode).TransformBlock(data): (output, verifier, 20-byte auth code)"""
    key1, key2, verifier = derive(password, salt, key_bytes)
    out, ct = zip_aes_with_keys(key1, key2, write_mode, data)
    return out, verifier, hmac.new(key2, ct, hashlib.sha1).digest()


# ---- PKZIP classic ---------------------------------------------------------------------------------------------------------
def _crc_byte_table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ CRC_POLY if c & 1 else c >> 1
        t.append(c)
    return t


_CRC = _crc_byte_table()


def _update_keys(k0, k1, k2, b):
    k0 = _CRC[(k0 ^ b) & 0xFF] ^ (k0 >> 8)
    k1 = ((k1 + (k0 & 0xFF)) * 134775813 + 1) & 0xFFFFFFFF
    k2 = _CRC[(k2 ^ (k1 >> 24)) & 0xFF] ^ (k2 >> 8)
    return k0, k1, k2


def _pack(k0, k1, k2):
    return b"".join(k.to_bytes(4, "little") for k in (k0, k1, k2))


def _unpack(keys12):
    k = bytes(keys12)
    return tuple(int.from_bytes(k[4 * i:4 * i + 4], "little") for i in range(3))


def generate_keys(seed):
    """the three keys after the password bytes, as 12 little-endian bytes"""
    k = (0x12345678, 0x23456789, 0x34567890)
    for b in bytes(seed):
        k = _update_keys(*k, b)
    return _pack(*k)


def transform(keys12, encrypt, data):
    """encrypt or decrypt `data` from the keys `keys12`: (output, keys after)"""
    k0, k1, k2 = _unpack(keys12)
    out = bytearray(len(data))
    for i, c in enumerate(bytes(data)):
        temp = (k2 | 2) & 0xFFFF
        o = c ^ (((temp * (temp ^ 1)) >> 8) & 0xFF)
        out[i] = o
        k0, k1, k2 = _update_keys(k0, k1, k2, c if encrypt else o)
    return bytes(out), _pack(k0, k1, k2)
