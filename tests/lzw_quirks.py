"""TEST INFRASTRUCTURE: hand-built .Z streams for every quirk of LzwInputStream (Lzw/LzwInputStream.cs), shared by the CPU
tests of the reference model and the GPU tests.  pack() lays codes out as the decoder reads them: LSB-first, the width
growing before a code whose freeEnt passed maxCode, and the position padded to a whole group of codes at every width
change and CLEAR."""


def pack(codes, max_bits=16, block=True, flags=None, cut_bits=None):
    """the stream of `codes` (256 is CLEAR in block mode); cut_bits: keep only that many code bits"""
    out = bytearray([0x1F, 0x9D, flags if flags is not None else (max_bits | (0x80 if block else 0))])
    bit = group = 0
    n, maxcode, free_ent, first = 9, 511, (257 if block else 256), True
    maxmax = 1 << max_bits
    acc = 0

    def pad():
        nonlocal bit, group
        g = 8 * n
        bit = group + (bit - group + g - 1) // g * g
        group = bit

    for c in codes:
        if free_ent > maxcode:
            pad()
            n += 1
            maxcode = maxmax if n == max_bits else (1 << n) - 1
        acc |= (c & ((1 << n) - 1)) << bit
        bit += n
        if first:
            first = False
            continue
        if c == 256 and block:
            pad()
            n, maxcode, free_ent = 9, 511, 256
            continue
        if free_ent < maxmax:
            free_ent += 1
    total = bit if cut_bits is None else cut_bits
    acc &= (1 << total) - 1
    out += acc.to_bytes((total + 7) // 8, "little")
    return bytes(out)


def _kwk_every_width():
    # literals grow freeEnt cheaply; at every width one KwK (code == freeEnt) and one code a step past it is not taken
    codes, free_ent = [97], 257
    for width in range(9, 17):
        top = (1 << width) - 1 if width < 16 else 65535
        while free_ent < top - 2:
            codes.append(98)
            free_ent += 1
        codes.append(free_ent)  # KwK
        free_ent += 1
    return codes


def zeros_stream(n):
    """a block-mode, 16-bit stream of n zero bytes (n >= 1), as compress(1) writes it without a CLEAR"""
    codes, total, k = [0], 1, 1
    while k < 65280 and total + k + 1 <= n:
        codes.append(256 + k)  # every code is a KwK: its string is one byte longer than the last
        total += k + 1
        k += 1
    longest = k  # entries 257 .. 256 + k - 1 hold 2 .. k bytes
    while n - total >= longest:
        codes.append(256 + longest - 1 if longest > 1 else 0)
        total += longest
    r = n - total
    if r >= 2:
        codes.append(255 + r)
    elif r == 1:
        codes.append(0)
    return pack(codes, 16, True)


QUIRKS = [
    # (name, stream)
    ("empty", b""),
    ("one_byte", b"\x1f"),
    ("magic_only", b"\x1f\x9d"),  # maxBits 0: the header's table initialisation indexes past a table of 1
    ("bad_magic", b"\x1f\x9e\x90abc"),
    ("max_bits_17", b"\x1f\x9d\x91abc"),
    ("reserved_bits", b"\x1f\x9d\xb0abc"),
    ("max_bits_7", pack([65, 66], 7, True)),
    ("max_bits_8_literals", pack([65, 66, 67, 256, 68], 8, True)),
    ("max_bits_8_kwk", pack([65, 257, 66], 8, True)),
    ("max_bits_8_kwk_on_kwk", pack([65, 257, 257], 8, True)),
    ("max_bits_8_nonblock_kwk_on_kwk", pack([65, 256, 256], 8, False)),
    ("max_bits_9_to_10", pack([97] + [98] * 300 + [511, 512, 600], 9, True)),  # 10-bit codes; 512 is a KwK
    ("first_code_clear", pack([256, 65], 16, True)),
    ("clear_every_code", pack([65, 256, 66, 256, 67, 256, 68, 69, 258, 256, 70], 16, True)),
    ("clear_then_kwk_code", pack([65, 66, 256, 67, 257], 16, True)),  # 67 defines the dead entry 256; 257 is a KwK
    ("kwk_every_width", pack(_kwk_every_width(), 16, True)),
    ("kwk_nonblock_256", pack([65, 256, 257, 66], 16, False)),
    ("code_gt_free_ent", pack([65, 66, 67, 300], 16, True)),
    ("truncated_in_code", pack([65, 66, 257, 67, 259], 16, True)[:-1]),
    ("truncated_after_pad", pack([65, 66, 256], 16, True, cut_bits=72)),  # the data ends on the CLEAR's padding point
    ("truncated_before_pad", pack([65, 66, 256], 16, True, cut_bits=32)),  # padding lands past the end: ResetBuf fails
    ("trailing_bits", pack([65, 66, 67], 16, True, cut_bits=32)),
]
