"""A test-only PNG decoder built from zlib and numpy unfiltering, plus the checks of a file's structure: chunk CRCs, IHDR fields,
the zlib stream's Adler-32 and the deflate block headers (BFINAL only on the last block).  Also the CRC-32 and Adler-32 combine
formulas the encoder uses, restated to document them."""
from __future__ import annotations

import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 6: 4}


def chunks(data: bytes):
    """[(type, payload, crc_ok)] of a PNG file."""
    assert data[:8] == SIG, "not a PNG signature"
    out, p = [], 8
    while p < len(data):
        (n,) = struct.unpack(">I", data[p:p + 4])
        typ = data[p + 4:p + 8]
        payload = data[p + 8:p + 8 + n]
        (crc,) = struct.unpack(">I", data[p + 8 + n:p + 12 + n])
        out.append((typ, payload, zlib.crc32(typ + payload) == crc))
        p += 12 + n
    assert p == len(data), "trailing bytes"
    return out


def ihdr(data: bytes):
    typ, payload, _ = chunks(data)[0]
    assert typ == b"IHDR" and len(payload) == 13
    W, H, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", payload)
    return dict(W=W, H=H, depth=depth, ctype=ctype, comp=comp, filter=filt, interlace=inter)


def unfilter(raw: bytes, H: int, W: int, C: int) -> np.ndarray:
    L = W * C
    buf = np.frombuffer(raw, dtype=np.uint8)
    assert buf.size == H * (L + 1), (buf.size, H, L)
    rows = buf.reshape(H, L + 1)
    out = np.zeros((H, L), dtype=np.uint8)
    prev = np.zeros(L, dtype=np.int32)
    for y in range(H):
        f, r = int(rows[y, 0]), rows[y, 1:].astype(np.int32)
        if f == 0:
            cur = r
        elif f == 2:
            cur = (r + prev) & 255
        elif f in (1, 3, 4):
            cur = np.zeros(L, dtype=np.int32)
            for j in range(L):  # left neighbours make these sequential; vectorised over the C channels of one pixel
                a = int(cur[j - C]) if j >= C else 0
                b = int(prev[j])
                c = int(prev[j - C]) if j >= C else 0
                if f == 1:
                    pred = a
                elif f == 3:
                    pred = (a + b) >> 1
                else:
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
                cur[j] = (int(r[j]) + pred) & 255
        else:
            raise ValueError("bad filter type %d" % f)
        out[y] = cur
        prev = cur
    return out.reshape(H, W, C) if C > 1 else out.reshape(H, W)


def decode(data: bytes) -> np.ndarray:
    """Pixels of an 8-bit, non-interlaced grey / RGB / RGBA PNG: [H,W] or [H,W,C] uint8."""
    h = ihdr(data)
    assert h["depth"] == 8 and h["interlace"] == 0 and h["ctype"] in CHANNELS, h
    z = b"".join(p for t, p, _ in chunks(data) if t == b"IDAT")
    return unfilter(zlib.decompress(z), h["H"], h["W"], CHANNELS[h["ctype"]])


def block_finals(data: bytes):
    """BFINAL of every deflate block of the file's zlib stream, walking the stream with a minimal inflater (stored, fixed and
    dynamic blocks)."""
    z = b"".join(p for t, p, _ in chunks(data) if t == b"IDAT")
    bits = np.unpackbits(np.frombuffer(z[2:-4], dtype=np.uint8), bitorder="little")
    pos = 0

    def get(n):
        nonlocal pos
        v = 0
        for k in range(n):
            v |= int(bits[pos + k]) << k
        pos += n
        return v

    def table(lengths):
        code, codes, bl = 0, {}, [0] * 16
        for x in lengths:
            if x:
                bl[x] += 1
        nxt, c = [0] * 16, 0
        for b in range(1, 16):
            c = (c + bl[b - 1]) << 1
            nxt[b] = c
        for s, x in enumerate(lengths):
            if x:
                codes[(x, nxt[x])] = s
                nxt[x] += 1
        return codes

    def sym(t):
        c, n = 0, 0
        while True:
            c = (c << 1) | get(1)
            n += 1
            if (n, c) in t:
                return t[(n, c)]

    LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    DEXT = [0, 0, 0, 0] + [k // 2 - 1 for k in range(4, 30)]
    fixed_l = table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
    fixed_d = table([5] * 30)
    finals = []
    while True:
        final, btype = get(1), get(2)
        finals.append(final)
        if btype == 0:
            pos = (pos + 7) // 8 * 8
            n = get(16)
            get(16)
            pos += 8 * n
        else:
            if btype == 1:
                lt, dt = fixed_l, fixed_d
            else:
                hlit, hdist, hclen = get(5) + 257, get(5) + 1, get(4) + 4
                order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
                cl = [0] * 19
                for k in range(hclen):
                    cl[order[k]] = get(3)
                ct = table(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = sym(ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + get(2))
                    elif s == 17:
                        lens += [0] * (3 + get(3))
                    else:
                        lens += [0] * (11 + get(7))
                lt, dt = table(lens[:hlit]), table(lens[hlit:])
            while True:
                s = sym(lt)
                if s == 256:
                    break
                if s > 256:
                    get(LEXT[s - 257])
                    get(DEXT[sym(dt)])
        if final:
            break
    return finals


# ---------------------------------------------------------------------------------------------------- the combine formulas
POLY = 0xEDB88320


def multmodp(a: int, b: int) -> int:
    """a(x) b(x) mod the CRC-32 polynomial, bit-reflected (x^0 is bit 31)."""
    m, p = 1 << 31, 0
    while True:
        if a & m:
            p ^= b
            if (a & (m - 1)) == 0:
                break
        m >>= 1
        b = (b >> 1) ^ POLY if b & 1 else b >> 1
    return p


def x8nmodp(n: int) -> int:
    x2n = [1 << 30]
    for _ in range(63):
        x2n.append(multmodp(x2n[-1], x2n[-1]))
    p, k = 1 << 31, 3
    while n:
        if n & 1:
            p = multmodp(x2n[k], p)
        n >>= 1
        k += 1
    return p


def crc32_combine(c1: int, c2: int, len2: int) -> int:
    """crc32(A + B) from crc32(A), crc32(B) and len(B)."""
    return multmodp(x8nmodp(len2), c1) ^ c2


def adler_sums(data: bytes):
    """(s1, s2, n) of a segment: sum d_i and sum (n - i) d_i, mod 65521."""
    d = np.frombuffer(data, dtype=np.uint8).astype(np.int64)
    n = len(d)
    return int(d.sum() % 65521), int(((n - np.arange(n)) * d).sum() % 65521), n


def adler_of_segments(segs) -> int:
    """Adler-32 of the concatenation from each segment's sums, as the encoder combines its chunks."""
    N = sum(n for _, _, n in segs)
    s1 = s2 = 0
    after = N
    for a, b, n in segs:
        after -= n
        s1 += a
        s2 += b + (after % 65521) * a
    A = (1 + s1) % 65521
    B = (N + s2) % 65521
    return (B << 16) | A
