"""Host-side checks of the PNG encoder: the test decoder against PIL and cv2 and against numpy-built streams of every filter type,
the CRC-32 / Adler-32 combine formulas, and the host-only C-ABI pieces (gsr_png_bound, workspace sizing)."""
from __future__ import annotations

import ctypes as C
import io
import struct
import zlib

import numpy as np
import pytest

from tests import png_ref as PR


def _img(H, W, Cn, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = ((x * 3 + y * 5) % 256).astype(np.uint8)
    a = np.stack([base + 40 * c for c in range(Cn)], -1).astype(np.uint8)
    a[rng.random((H, W)) < 0.1] = rng.integers(0, 256, (Cn,), dtype=np.uint8)
    return a if Cn > 1 else a[:, :, 0]


@pytest.mark.parametrize("Cn", [1, 3, 4])
def test_decoder_agrees_with_pil(Cn):
    from PIL import Image
    a = _img(23, 37, Cn, Cn)
    b = io.BytesIO()
    Image.fromarray(a).save(b, format="PNG")
    assert np.array_equal(PR.decode(b.getvalue()), a)
    assert all(ok for _, _, ok in PR.chunks(b.getvalue()))


@pytest.mark.parametrize("Cn", [1, 3, 4])
def test_decoder_agrees_with_cv2(Cn):
    cv2 = pytest.importorskip("cv2")
    a = _img(19, 41, Cn, 10 + Cn)
    ok, enc = cv2.imencode(".png", a)
    assert ok
    got = PR.decode(enc.tobytes())
    want = a if Cn == 1 else (a[:, :, ::-1] if Cn == 3 else a[:, :, [2, 1, 0, 3]])  # cv2 stores RGB(A) from BGR(A)
    assert np.array_equal(got, want)


def _filter_row(cur, prev, f, bpp):
    L = cur.size
    out = np.zeros(L, dtype=np.int32)
    for j in range(L):
        a = int(cur[j - bpp]) if j >= bpp else 0
        b = int(prev[j])
        c = int(prev[j - bpp]) if j >= bpp else 0
        pred = [0, a, b, (a + b) >> 1, None][f]
        if f == 4:
            p = a + b - c
            pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
            pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
        out[j] = (int(cur[j]) - pred) & 255
    return out.astype(np.uint8)


@pytest.mark.parametrize("f", range(5))
def test_decoder_unfilters_each_filter_type(f):
    a = _img(9, 13, 4, 30 + f)
    H, W = a.shape[:2]
    rows = a.reshape(H, -1)
    raw = b""
    prev = np.zeros(rows.shape[1], dtype=np.uint8)
    for y in range(H):
        ft = (f + y) % 5 if y else f  # every row type, starting with f
        raw += bytes([ft]) + _filter_row(rows[y], prev, ft, 4).tobytes()
        prev = rows[y]
    assert np.array_equal(PR.unfilter(raw, H, W, 4), a)


def test_crc32_combine_matches_zlib():
    rng = np.random.default_rng(1)
    for n1, n2 in [(0, 5), (5, 0), (1, 1), (100, 3000), (70000, 12345)]:
        a, b = rng.bytes(n1), rng.bytes(n2)
        assert PR.crc32_combine(zlib.crc32(a), zlib.crc32(b), n2) == zlib.crc32(a + b)


def test_adler32_combine_matches_zlib():
    rng = np.random.default_rng(2)
    data = rng.bytes(200000)
    segs = [data[i:i + 32768] for i in range(0, len(data), 32768)]
    assert PR.adler_of_segments([PR.adler_sums(s) for s in segs]) == zlib.adler32(data)
    assert PR.adler_of_segments([PR.adler_sums(b"\xff" * 70000)]) == zlib.adler32(b"\xff" * 70000)


def _lib():
    from autovfx_b200 import _lib as L
    return L


@pytest.mark.parametrize("H,W,Cn", [(1, 1, 1), (1080, 1920, 4), (1081, 1921, 3), (2160, 3840, 4), (7, 5, 1)])
def test_png_bound(H, W, Cn):
    L = _lib()
    raw = H * (1 + W * Cn)
    chunks = (raw + 32767) // 32768
    # signature 8, IHDR 25, IDAT framing 12, zlib header 2 + Adler 4, IEND 12; a stored block costs 5 bytes per 32 KiB
    assert L.lib.gsr_png_bound(H, W, Cn) == 8 + 25 + 12 + 6 + 12 + raw + 5 * chunks


@pytest.mark.parametrize("H,W,Cn", [(0, 5, 3), (5, 0, 3), (5, 5, 2), (5, 5, 5), (60000, 60000, 4)])
def test_png_bound_rejects(H, W, Cn):
    assert _lib().lib.gsr_png_bound(H, W, Cn) == 0


def test_workspace_bytes():
    L = _lib()
    shapes = [(1080, 1920, 4, False), (1080, 1920, 1, True), (3, 3, 3, False)]
    arr = (L.gsr_png_image * 3)()
    for k, (H, W, Cn, lut) in enumerate(shapes):
        arr[k].H, arr[k].W, arr[k].C, arr[k].lut = H, W, Cn, (1 if lut else None)
    raws = [H * (1 + W * (3 if lut else Cn)) for H, W, Cn, lut in shapes]
    al = sum((r + 255) // 256 * 256 for r in raws)
    chunks = sum((r + 32767) // 32768 for r in raws)
    want = 5 * al + chunks * (32768 + 256) + (chunks * 16 + 255) // 256 * 256
    assert L.lib.gsr_png_workspace_bytes(3, arr) == want
    assert L.lib.gsr_png_workspace_bytes(-1, arr) == 0


def test_encode_rejects_before_launching():
    L = _lib()
    im = L.gsr_png_image()
    im.data, im.H, im.W, im.C, im.stride_h, im.stride_w, im.stride_c = 4096, 4, 4, 2, 8, 2, 1
    outs = (C.c_void_p * 1)(4096)
    rc = L.lib.gsr_png_encode(C.byref(im), 1, outs, 4096, 4096, 1 << 20, None)
    assert rc == -1 and b"channels" in L.lib.gsr_last_error()
    im.C, im.lut = 3, 4096
    assert L.lib.gsr_png_encode(C.byref(im), 1, outs, 4096, 4096, 1 << 20, None) == -1
    assert b"lookup table" in L.lib.gsr_last_error()
    im.lut, im.H = None, 0
    assert L.lib.gsr_png_encode(C.byref(im), 1, outs, 4096, 4096, 1 << 20, None) == -1
    im.H = 4
    assert L.lib.gsr_png_encode(C.byref(im), 1, outs, 4096, 4096, 16, None) == -2


def test_header_bytes_restated():
    """The 43 bytes before the deflate data, as k_png_assemble writes them: signature, IHDR with its CRC, IDAT length and type, and
    the zlib header 78 01 (deflate, 32 KiB window, a valid check)."""
    W, H = 1920, 1080
    ih = b"IHDR" + struct.pack(">IIBBBBB", W, H, 8, 6, 0, 0, 0)
    hdr = PR.SIG + struct.pack(">I", 13) + ih + struct.pack(">I", zlib.crc32(ih))
    assert len(hdr) + 8 + 2 == 43
    assert (0x78 * 256 + 0x01) % 31 == 0
    iend = struct.pack(">I", 0) + b"IEND" + struct.pack(">I", zlib.crc32(b"IEND"))
    assert iend == bytes([0, 0, 0, 0, 0x49, 0x45, 0x4E, 0x44, 0xAE, 0x42, 0x60, 0x82])
