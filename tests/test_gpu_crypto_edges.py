"""GPU tier: the entry-cipher kernels (b200z_crypto.cu: k_aes_ctr, k_hmac_sha1, k_pbkdf2, k_pkzip) against the plain
references of tests/crypto_ref.py (FIPS 197 AES in numpy, hashlib / hmac, the APPNOTE key update), with the oracle as a
second witness, at the edges where they can go wrong: every password length around SHA-1's block and its padding, every
entry length around the 16-byte AES block, the 64-byte SHA-1 block and the 16 KiB tile of k_aes_ctr, TransformBlock split at
every point, device calls at every offset mod 16, in place, with state carried over three calls, more than 65535 entries
in one call, entries long enough for the grid-stride loop, a deflate plan's output blob, and one entry past 4 GiB.

Tests whose name holds "emu" are small enough for the CUDA emulator; the CPU tier runs them there.  The case past 4 GiB
checks free device and host memory first and skips, saying why, when it is short."""
import time

import numpy as np
import pytest

import crypto_ref as R
from test_crypto import password_set
from test_gpu_checksums import BIG, MiB, _need, _release

pytestmark = pytest.mark.gpu

TILE_BLOCKS = 1024  # kAesTile / 16: keystream blocks per CTA and grid-stride step of k_aes_ctr
WRAP_BLOCKS = 1024 * TILE_BLOCKS  # kAesMaxTiles tiles: one step of the grid-stride loop (16 MiB)
EDGE_LENS = list(range(301)) + sorted({16384 * k + d for k in (1, 2) for d in (-17, -16, -1, 0, 1, 15, 16, 17)})
KEY_SIZES = pytest.mark.parametrize("key_bytes", [16, 32], ids=["aes128", "aes256"])
MODES = pytest.mark.parametrize("write_mode", [True, False], ids=["write", "read"])


def _dev(a):
    """numpy -> device tensor (a copy, also on the emulator where device tensors are host tensors)"""
    import torch
    return torch.from_numpy(np.array(a, copy=True)).cuda()


def _host(t):
    return np.array(t.cpu().numpy(), copy=True)


def _random_keys(rng, n, key_bytes):
    """n rows of key1 | key2 | verifier: the device calls take derived keys as they are"""
    return rng.integers(0, 256, (n, 2 * key_bytes + 2), dtype=np.uint8)


def _aes_device(z, d_in, d_out, offs, lens, key_bytes, d_keys, write_mode, d_state, finish, d_auth, max_len=None):
    import torch
    offs, lens = np.asarray(offs, np.int64), np.asarray(lens, np.int64)
    d_off, d_len = _dev(offs), _dev(lens)
    max_len = int(lens.max()) if max_len is None else max_len
    rc = z.lib().b200z_aes_device(d_in.data_ptr(), d_out.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), max_len, len(lens), key_bytes,
                                  d_keys.data_ptr(), 1 if write_mode else 0, d_state.data_ptr(), 1 if finish else 0, d_auth.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream)
    assert rc == 0, z.lib().b200z_last_error()
    torch.cuda.synchronize()


def _pkzip_device(z, d_in, d_out, offs, lens, d_keys, encrypt):
    import torch
    d_off, d_len = _dev(np.asarray(offs, np.int64)), _dev(np.asarray(lens, np.int64))
    rc = z.lib().b200z_pkzip_device(d_in.data_ptr(), d_out.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), len(lens), d_keys.data_ptr(),
                                    1 if encrypt else 0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, z.lib().b200z_last_error()
    torch.cuda.synchronize()


def _mac(key2, ct):
    return R.mac_update(R.new_mac(key2), np.frombuffer(bytes(ct), np.uint8)).digest()


# ---- 1. PBKDF2 --------------------------------------------------------------------------------------------------------------
@KEY_SIZES
def test_emu_pbkdf2_every_password_length(z, key_bytes):
    """aes_derive_keys on every password length 0-200, 255 and 1000 (UTF-8 ones too) in one call, against hashlib; a
    transform made with the empty password"""
    from sharpziplib_b200 import encryption as E
    pws = password_set()
    salts = [bytes((7 * i + j) & 0xFF for j in range(key_bytes // 2)) for i in range(len(pws))]
    keys = E.aes_derive_keys(pws, salts, key_bytes)
    bad = [len(p) for p, s, k in zip(pws, salts, keys) if k.tobytes() != b"".join(R.derive(p, s, key_bytes))]
    assert not bad, bad
    salt = bytes(range(key_bytes // 2))
    data = bytes(range(100))
    want_ct, want_pv, want_mac = R.zip_aes("", salt, key_bytes, True, data)
    t = E.ZipAESTransform("", salt, key_bytes, True)
    out = bytearray(100)
    t.TransformBlock(data, 0, 100, out, 0)
    assert (bytes(out), t.PwdVerifier, t.GetAuthCode()) == (want_ct, want_pv, want_mac)
    t.Dispose()


# ---- 2. aes_batch at every length edge ------------------------------------------------------------------------------------
@KEY_SIZES
def test_emu_aes_batch_every_length_edge(z, key_bytes):
    """lengths 0-300 and 16384 k + {-17, -16, -1, 0, 1, 15, 16, 17}, k = 1, 2, in one batch, both directions: the output
    and all 20 bytes of every auth code"""
    from sharpziplib_b200 import encryption as E
    rng = np.random.default_rng(20 + key_bytes)
    bufs = [rng.bytes(n) for n in EDGE_LENS]
    keys = _random_keys(rng, len(bufs), key_bytes)
    want_ct, want_mac = [], []
    for b, k in zip(bufs, keys):
        k1, k2, _ = R.split_keys(k, key_bytes)
        ct, _ = R.zip_aes_with_keys(k1, k2, True, b)
        want_ct.append(ct)
        want_mac.append(_mac(k2, ct))
    outs, auth = E.aes_batch(bufs, keys, key_bytes, True)
    bad = [len(b) for i, b in enumerate(bufs) if outs[i] != want_ct[i] or auth[i].tobytes() != want_mac[i]]
    assert not bad, bad
    back, auth2 = E.aes_batch(want_ct, keys, key_bytes, False)
    bad = [len(b) for i, b in enumerate(bufs) if back[i] != b or auth2[i].tobytes() != want_mac[i]]
    assert not bad, bad


# ---- 3. the transform handle in pieces --------------------------------------------------------------------------------------
@KEY_SIZES
@MODES
def test_emu_aes_transform_in_pieces(z, key_bytes, write_mode):
    """one 200-byte input split at every point into two TransformBlock calls, and into three around the 16- and 64-byte
    edges; GetAuthCode() before any data is the HMAC of the empty message, and asking twice gives the same code"""
    from sharpziplib_b200.encryption import ZipAESTransform
    rng = np.random.default_rng(30 + key_bytes)
    pw, salt = "pieces", rng.bytes(key_bytes // 2)
    plain = rng.bytes(200)
    ct, pv, mac = R.zip_aes(pw, salt, key_bytes, True, plain)
    src, want = (plain, ct) if write_mode else (ct, plain)
    t = ZipAESTransform(pw, salt, key_bytes, write_mode)
    empty_mac = _mac(R.derive(pw, salt, key_bytes)[1], b"")
    assert t.GetAuthCode() == empty_mac and t.GetAuthCode() == empty_mac and t.PwdVerifier == pv
    t.Dispose()
    splits = [(c,) for c in range(201)]
    splits += [(a, b) for a in (1, 15, 16, 17, 63, 64, 65) for b in (a + 1, 31, 32, 33, 127, 128, 129, 191, 192, 193) if b > a]
    for cuts in splits:
        t = ZipAESTransform(pw, salt, key_bytes, write_mode)
        out = bytearray(200)
        for lo, hi in zip((0,) + cuts, cuts + (200,)):
            assert t.TransformBlock(src, lo, hi - lo, out, lo) == hi - lo
        assert bytes(out) == want, cuts
        assert t.GetAuthCode() == mac and t.GetAuthCode() == mac, cuts
        t.Dispose()


# ---- 4./5. device calls with carried state ----------------------------------------------------------------------------------
N_STREAMS = 41
PIECE_LENS = (0, 1, 3, 15, 16, 17, 31, 47, 63, 64, 65, 100, 127, 128, 129, 200, 300)


def _pieces(rng):
    """lens[call][stream] for three calls: stream 0 is empty throughout, stream 1 only in the last call, stream 2 only in
    the first; the others ragged, zeros included"""
    lens = rng.choice(PIECE_LENS, (3, N_STREAMS))
    lens[:, 0] = 0
    lens[:2, 1] = 0
    lens[1:, 2] = 0
    return lens


def _layout(lens, shift):
    """offsets of one call's pieces in one blob: stream i starts at residue (i + shift) mod 16, with gaps between"""
    offs, pos = [], 64
    for i, L in enumerate(lens):
        pos = (pos + 15) // 16 * 16 + (i + shift) % 16
        offs.append(pos)
        pos += int(L) + 24
    assert {o % 16 for o in offs} == set(range(16))
    return offs, pos + 64


def _device_calls(rng, lens, streams_in, in_place, run):
    """three calls over one blob each; run(call, d_in, d_out, offs, lens) launches.  streams_in[i] is stream i's whole input.
    Returns per stream its whole output, and checks that no byte outside the pieces changed (in place) or was written (out of
    place)"""
    import torch
    got = [bytearray() for _ in lens[0]]
    done = [0] * len(lens[0])
    for c in range(3):
        offs, size = _layout(lens[c], 5 * c)
        host = rng.integers(0, 256, size, dtype=np.uint8)
        for i, (o, L) in enumerate(zip(offs, lens[c])):
            host[o:o + L] = np.frombuffer(streams_in[i][done[i]:done[i] + L], np.uint8)
        d_in = _dev(host)
        d_out = d_in if in_place else torch.full((size,), 0xA5, dtype=torch.uint8).cuda()
        before = host if in_place else np.full(size, 0xA5, np.uint8)
        run(c, d_in, d_out, offs, lens[c])
        res = _host(d_out)
        mask = np.ones(size, bool)
        for i, (o, L) in enumerate(zip(offs, lens[c])):
            got[i] += res[o:o + L].tobytes()
            done[i] += int(L)
            mask[o:o + L] = False
        assert (res[mask] == before[mask]).all(), ("bytes outside the pieces changed", c)
        if not in_place:
            assert (_host(d_in) == host).all(), ("the input changed", c)
    return [bytes(g) for g in got]


@KEY_SIZES
@MODES
@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
def test_emu_aes_device_carried_state(z, key_bytes, write_mode, in_place):
    """b200z_aes_device: 41 streams at offsets of every residue mod 16, three calls with ragged per-stream lengths (zeros
    too), finish on the last call only; the auth codes are written by that call and by no other"""
    import torch
    rng = np.random.default_rng(40 + key_bytes + 2 * write_mode + 4 * in_place)
    lens = _pieces(rng)
    keys = _random_keys(rng, N_STREAMS, key_bytes)
    plain = [rng.bytes(int(n)) for n in lens.sum(axis=0)]
    ref = [R.zip_aes_with_keys(*R.split_keys(k, key_bytes)[:2], True, p)[0] for k, p in zip(keys, plain)]
    d_keys, d_state = _dev(keys), torch.zeros(128 * N_STREAMS, dtype=torch.uint8).cuda()
    d_auth = torch.full((20 * N_STREAMS,), 0x5A, dtype=torch.uint8).cuda()

    def call(c, d_in, d_out, offs, L):
        _aes_device(z, d_in, d_out, offs, L, key_bytes, d_keys, write_mode, d_state, c == 2, d_auth, max_len=int(L.max()))
        if c < 2:
            assert (_host(d_auth) == 0x5A).all(), c
    got = _device_calls(rng, lens, plain if write_mode else ref, in_place, call)
    want = ref if write_mode else plain
    bad = [i for i in range(N_STREAMS) if got[i] != want[i]]
    assert not bad, [(i, lens[:, i].tolist()) for i in bad]
    auth = _host(d_auth).reshape(N_STREAMS, 20)
    bad = [i for i in range(N_STREAMS) if auth[i].tobytes() != _mac(R.split_keys(keys[i], key_bytes)[1], ref[i])]
    assert not bad, [(i, lens[:, i].tolist()) for i in bad]
    st = _host(d_state).reshape(N_STREAMS, 128)[:, :8].copy().view("<u8").reshape(-1)
    assert st.tolist() == lens.sum(axis=0).tolist()  # the stream position carried in the state


@pytest.mark.parametrize("encrypt", [True, False], ids=["encrypt", "decrypt"])
@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
def test_emu_pkzip_device_carried_state(z, encrypt, in_place):
    """b200z_pkzip_device the same way: the keys come back advanced after every call and the next call goes on from them"""
    rng = np.random.default_rng(50 + 2 * encrypt + in_place)
    lens = _pieces(rng)
    keys = [R.generate_keys(b"seed %d" % i + bytes(i)) for i in range(N_STREAMS)]
    plain = [rng.bytes(int(n)) for n in lens.sum(axis=0)]
    ct = [R.transform(k, True, p)[0] for k, p in zip(keys, plain)]
    src = plain if encrypt else ct
    d_keys = _dev(np.frombuffer(b"".join(keys), np.uint8).view(np.int32))
    done = [0] * N_STREAMS

    def call(c, d_in, d_out, offs, L):
        _pkzip_device(z, d_in, d_out, offs, L, d_keys, encrypt)
        after = _host(d_keys).view(np.uint8).reshape(N_STREAMS, 12)
        for i in range(N_STREAMS):
            done[i] += int(L[i])
            want = R.transform(keys[i], encrypt, src[i][:done[i]])[1]
            assert after[i].tobytes() == want, (c, i, lens[:, i].tolist())
    got = _device_calls(rng, lens, src, in_place, call)
    want = ct if encrypt else plain
    bad = [i for i in range(N_STREAMS) if got[i] != want[i]]
    assert not bad, [(i, lens[:, i].tolist()) for i in bad]


@pytest.mark.parametrize("encrypt", [True, False], ids=["encrypt", "decrypt"])
def test_emu_pkzip_batch_every_length(z, encrypt):
    """pkzip_batch at lengths 0-300, one key set per entry: the output and the keys after"""
    from sharpziplib_b200 import encryption as E
    rng = np.random.default_rng(60 + encrypt)
    bufs = [rng.bytes(n) for n in range(301)]
    keys = [R.generate_keys(rng.bytes(1 + i % 40)) for i in range(301)]
    outs, after = E.pkzip_batch(bufs, np.frombuffer(b"".join(keys), np.uint8).reshape(301, 12), encrypt)
    for i, b in enumerate(bufs):
        assert (outs[i], after[i].tobytes()) == R.transform(keys[i], encrypt, b), i


# ---- 6. more than 65535 entries ---------------------------------------------------------------------------------------------
N_MANY = 65536 + 1000


def _many(rng, key_bytes):
    """N_MANY entries of 0-48 bytes; 64 key sets from aes_derive_keys tiled over them, with their first three keystream blocks"""
    from sharpziplib_b200 import encryption as E
    bufs = [rng.bytes(int(n)) for n in rng.integers(0, 49, N_MANY)]
    pws, salts = [b"many %d" % i for i in range(64)], [rng.bytes(key_bytes // 2) for _ in range(64)]
    sets = E.aes_derive_keys(pws, salts, key_bytes)
    assert all(sets[i].tobytes() == b"".join(R.derive(pws[i], salts[i], key_bytes)) for i in range(64))
    ks = [R.zip_aes_keystream(R.split_keys(k, key_bytes)[0], 0, 48) for k in sets]
    macs = [R.new_mac(R.split_keys(k, key_bytes)[1]) for k in sets]
    ct = [(np.frombuffer(b, np.uint8) ^ ks[i % 64][:len(b)]).tobytes() for i, b in enumerate(bufs)]
    mac = [_mac_from(macs[i % 64], c) for i, c in enumerate(ct)]
    return bufs, np.tile(sets, (N_MANY // 64 + 1, 1))[:N_MANY], ct, mac


def _mac_from(base, data):
    m = base.copy()
    m.update(data)
    return m.digest()


@KEY_SIZES
def test_more_than_65535_entries(z, key_bytes):
    """aes_batch and b200z_aes_device (both modes, packed at ragged offsets) and pkzip_batch on 66536 entries of 0-48 bytes"""
    import torch
    from sharpziplib_b200 import encryption as E
    rng = np.random.default_rng(70 + key_bytes)
    t0 = time.time()
    bufs, keys, ct, mac = _many(rng, key_bytes)
    outs, auth = E.aes_batch(bufs, keys, key_bytes, True)
    bad = [i for i in range(N_MANY) if outs[i] != ct[i] or auth[i].tobytes() != mac[i]]
    assert not bad, (len(bad), bad[:10])
    back, auth = E.aes_batch(ct, keys, key_bytes, False)
    bad = [i for i in range(N_MANY) if back[i] != bufs[i] or auth[i].tobytes() != mac[i]]
    assert not bad, (len(bad), bad[:10])
    # the device entry point: every entry packed back to back (offsets at every residue), write in place, then read back
    lens = np.array([len(b) for b in bufs], np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    blob = _dev(np.frombuffer(b"".join(bufs), np.uint8))
    d_keys = _dev(keys)
    for write_mode in (True, False):
        d_state = torch.zeros(128 * N_MANY, dtype=torch.uint8).cuda()
        d_auth = torch.zeros(20 * N_MANY, dtype=torch.uint8).cuda()
        d_out = blob if write_mode else torch.zeros_like(blob)
        _aes_device(z, blob, d_out, offs, lens, key_bytes, d_keys, write_mode, d_state, True, d_auth)
        res, a = _host(d_out).tobytes(), _host(d_auth).reshape(N_MANY, 20)
        want = ct if write_mode else bufs
        bad = [i for i in range(N_MANY) if res[offs[i]:offs[i] + lens[i]] != want[i] or a[i].tobytes() != mac[i]]
        assert not bad, (write_mode, len(bad), bad[:10])
    # PKZIP classic: 64 key sets tiled
    sets = [R.generate_keys(b"classic %d" % i) for i in range(64)]
    k12 = np.frombuffer(b"".join(sets[i % 64] for i in range(N_MANY)), np.uint8).reshape(N_MANY, 12)
    outs, after = E.pkzip_batch(bufs, k12, True)
    bad = [i for i in range(N_MANY) if (outs[i], after[i].tobytes()) != R.transform(sets[i % 64], True, bufs[i])]
    assert not bad, (len(bad), bad[:10])
    print("more than 65535 entries (%d-bit keys): %.1f s" % (8 * key_bytes, time.time() - t0))


# ---- 7. long entries: the grid-stride loop of k_aes_ctr ----------------------------------------------------------------------
def _edge_blocks(first_blk, last_blk):
    """keystream blocks within 2 of every tile edge and every grid-stride wrap of a call whose blocks are first_blk ..
    last_blk - 1 (tiles are counted from the call's first block)"""
    e = np.arange(first_blk, last_blk + TILE_BLOCKS, TILE_BLOCKS, dtype=np.int64)
    b = (e[:, None] + np.arange(-2, 3)[None, :]).reshape(-1)
    return np.unique(b[(b >= first_blk) & (b < last_blk)])


def _check_keystream(key1, start, src, out, blocks):
    """out ^ src at the given 16-byte keystream blocks (of a piece at stream position `start`) is the reference keystream"""
    s, o = np.frombuffer(src, np.uint8), np.frombuffer(out, np.uint8)
    ks = R.keystream_blocks(key1, blocks.astype(np.uint64))
    for j, b in enumerate(blocks):
        lo, hi = max(16 * int(b), start), min(16 * int(b) + 16, start + len(s))
        got = s[lo - start:hi - start] ^ o[lo - start:hi - start]
        assert (got == ks[j, lo - 16 * int(b):hi - 16 * int(b)]).all(), ("keystream block", int(b))


def test_long_entries_through_the_grid_stride_loop(z, oracle):
    """entries of 16 MiB + {-16, -1, 0, 1, 17} and one of 80 MiB beside 200 short ones in one batch: the keystream around
    every tile edge and every 16 MiB wrap, the whole ciphertext against the oracle, the auth codes against hmac"""
    from sharpziplib_b200 import encryption as E
    rng = np.random.default_rng(80)
    kb = 32
    lens = [16 * MiB + d for d in (-16, -1, 0, 1, 17)] + [80 * MiB] + [int(n) for n in rng.integers(0, 5000, 200)]
    bufs = [rng.bytes(n) for n in lens]
    pws, salts = [b"long %d" % i for i in range(len(lens))], [rng.bytes(kb // 2) for _ in lens]
    keys = E.aes_derive_keys(pws, salts, kb)
    t0 = time.time()
    outs, auth = E.aes_batch(bufs, keys, kb, True)
    secs = time.time() - t0
    for i, (b, o) in enumerate(zip(bufs, outs)):
        k1, k2, _ = R.split_keys(keys[i], kb)
        if len(b) > TILE_BLOCKS * 16:
            _check_keystream(k1, 0, b, o, _edge_blocks(0, (len(b) + 15) // 16))
        assert auth[i].tobytes() == _mac(k2, o), i
        assert (o, auth[i].tobytes()) == oracle.zip_aes(pws[i], salts[i], kb, True, b)[::2], i
    back, auth2 = E.aes_batch(outs, keys, kb, False)
    assert back == bufs and (auth2 == auth).all()
    print("aes_batch over %d bytes in %d entries (longest 80 MiB): %.2f s" % (sum(lens), len(lens), secs))


@MODES
def test_long_transform_block_at_an_odd_position(z, oracle, write_mode):
    """one handle: 12345 bytes, then one TransformBlock of 40 MiB that starts at an odd stream position, then 77 bytes"""
    from sharpziplib_b200.encryption import ZipAESTransform
    rng = np.random.default_rng(90)
    kb, pw, salt = 16, "odd start", rng.bytes(8)
    plain = rng.bytes(12345 + 40 * MiB + 77)
    ct, pv, mac = oracle.zip_aes(pw.encode(), salt, kb, True, plain)
    src, want = (plain, ct) if write_mode else (ct, plain)
    t = ZipAESTransform(pw, salt, kb, write_mode)
    out = bytearray(len(src))
    cuts = (0, 12345, 12345 + 40 * MiB, len(src))
    t0 = time.time()
    for lo, hi in zip(cuts, cuts[1:]):
        t.TransformBlock(src, lo, hi - lo, out, lo)
    secs = time.time() - t0
    assert (t.PwdVerifier, t.GetAuthCode()) == (pv, mac)
    t.Dispose()
    out = bytes(out)
    assert out == want
    lo, hi = cuts[1], cuts[2]
    _check_keystream(R.derive(pw, salt, kb)[0], lo, src[lo:hi], out[lo:hi], _edge_blocks(lo // 16, (hi + 15) // 16))
    assert mac == _mac(R.derive(pw, salt, kb)[1], ct)
    print("transform of 40 MiB at position 12345: %.2f s" % secs)


# ---- 8. the documented integration path: ciphers on a deflate plan's output blob ----------------------------------------------
def test_ciphers_on_a_deflate_plan_output(z, oracle):
    """DeflatePlan on the device, then b200z_aes_device in place on its output blob (plan.out_offsets, the plan's d_out_len),
    and b200z_pkzip_device in place on a second copy; against the oracle's deflate put through the references"""
    import torch
    from sharpziplib_b200 import datagen, encryption as E
    bufs = [datagen.silesia_mix(i, n, config=8).tobytes() for i, n in enumerate((0, 1, 100, 5000, 65536, 70001, 300000, 1 << 20))]
    plan = z.DeflatePlan([len(b) for b in bufs], level=6)
    host = np.zeros(plan.in_bytes, np.uint8)
    for o, b in zip(plan.in_offsets, bufs):
        host[o:o + len(b)] = np.frombuffer(b, np.uint8)
    d_in = torch.from_numpy(host).cuda()
    d_out = torch.zeros(plan.out_bytes, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(plan.n, dtype=torch.int64, device="cuda")
    d_st = torch.zeros(plan.n, dtype=torch.int32, device="cuda")
    plan.run(d_in, d_out, d_len, d_st)
    torch.cuda.synchronize()
    assert d_st.cpu().tolist() == [0] * plan.n
    comp = [oracle.deflate(b, level=6) for b in bufs]
    lens = d_len.cpu().numpy()
    assert lens.tolist() == [len(c) for c in comp]
    d_copy = d_out.clone()
    kb, n = 32, plan.n
    pws, salts = [b"plan %d" % i for i in range(n)], [bytes([i]) * (kb // 2) for i in range(n)]
    keys = E.aes_derive_keys(pws, salts, kb)
    d_off = _dev(plan.out_offsets)
    d_keys, d_state = _dev(keys), torch.zeros(128 * n, dtype=torch.uint8, device="cuda")
    d_auth = torch.zeros(20 * n, dtype=torch.uint8, device="cuda")
    rc = z.lib().b200z_aes_device(d_out.data_ptr(), d_out.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), int(lens.max()), n, kb,
                                  d_keys.data_ptr(), 1, d_state.data_ptr(), 1, d_auth.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, z.lib().b200z_last_error()
    sets = [R.generate_keys(b"plan classic %d" % i) for i in range(n)]
    d_k12 = _dev(np.frombuffer(b"".join(sets), np.uint8).view(np.int32))
    rc = z.lib().b200z_pkzip_device(d_copy.data_ptr(), d_copy.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), n, d_k12.data_ptr(), 1,
                                    torch.cuda.current_stream().cuda_stream)
    assert rc == 0, z.lib().b200z_last_error()
    torch.cuda.synchronize()
    enc, classic, auth = _host(d_out), _host(d_copy), _host(d_auth).reshape(n, 20)
    k12 = _host(d_k12).view(np.uint8).reshape(n, 12)
    for i, c in enumerate(comp):
        o = int(plan.out_offsets[i])
        want, pv, mac = R.zip_aes(pws[i], salts[i], kb, True, c)
        assert enc[o:o + len(c)].tobytes() == want and auth[i].tobytes() == mac, i
        assert (classic[o:o + len(c)].tobytes(), k12[i].tobytes()) == R.transform(sets[i], True, c), i
    plan.close()


# ---- 9. one entry past 4 GiB --------------------------------------------------------------------------------------------------
def test_aes_device_entry_past_4gib(z):
    """write mode in place through b200z_aes_device on one entry of 2^32 + 64 KiB bytes: the auth code against hmac over
    chunked copies, the keystream around byte 2^32, at a sample of tile edges and wraps and at random blocks, and the stream
    position carried in the state"""
    import torch
    from sharpziplib_b200 import encryption as E
    n = BIG + 64 * 1024
    _need(n + 256 * MiB, 512 * MiB)
    kb = 32
    keys = E.aes_derive_keys([b"past 4 GiB"], [bytes(range(16))], kb)
    key1, key2, _ = R.split_keys(keys[0], kb)
    nblk = n // 16
    rng = np.random.default_rng(99)
    edges = _edge_blocks(0, nblk)
    sample = np.unique(np.concatenate([
        np.arange(BIG // 16 - 3, BIG // 16 + 3), np.arange(nblk - 3, nblk), np.arange(0, 3),
        edges[::997], edges[(edges % WRAP_BLOCKS <= 2) | (edges % WRAP_BLOCKS >= WRAP_BLOCKS - 2)],
        rng.integers(0, nblk, 4096)]))
    g = torch.Generator(device="cuda")
    g.manual_seed(0xAE5)
    blob = torch.empty(n, dtype=torch.uint8, device="cuda").random_(0, 256, generator=g)
    idx = torch.from_numpy(sample.astype(np.int64)).cuda()
    before = blob.view(-1, 16)[idx].cpu().numpy()
    d_keys = _dev(keys)
    d_state = torch.zeros(128, dtype=torch.uint8, device="cuda")
    d_auth = torch.zeros(20, dtype=torch.uint8, device="cuda")
    t0 = time.time()
    _aes_device(z, blob, blob, [0], [n], kb, d_keys, True, d_state, True, d_auth)
    secs = time.time() - t0
    print("b200z_aes_device: one entry of %d bytes, write mode, in place: %.1f s" % (n, secs))
    after = blob.view(-1, 16)[idx].cpu().numpy()
    mac = R.mac_update(R.new_mac(key2), blob).digest()
    state = _host(d_state)
    del blob, idx
    _release(z)
    assert int(state[:8].view("<u8")[0]) == n
    ks = R.keystream_blocks(key1, sample.astype(np.uint64))
    bad = sample[((before ^ after) != ks).any(axis=1)]
    assert not bad.size, bad[:10]
    assert _host(d_auth).tobytes() == mac
