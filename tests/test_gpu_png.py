"""PNG encoding on the GPU (autovfx_b200.png): exact round trips through PIL, cv2 and the test decoder (tests/png_ref.py), the same
pixels as the reference loop's files, file structure, determinism, size against the bound and PIL, no host synchronisation in the
asynchronous writer, and the argument errors."""
from __future__ import annotations

import io
import os
import tempfile
import zlib

import numpy as np
import pytest
import torch

from tests import png_ref as PR

pytestmark = pytest.mark.gpu

# Files are at most this many times PIL's for the same pixels.  Rendered 1080p frames measured 1.11-1.12 on an H100; the synthetic
# 1080p RGBA gradient measured 1.55: PIL stores it in 11 KB, where the 250 dynamic-block headers and sync flushes of 32 KiB chunks
# (about 60 bytes each) dominate, so gradients get the looser bound.
SIZE_RATIO_K = 1.3
SIZE_RATIO_K_GRADIENT = 1.6


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _bytes(img, lut=None, swap_rb=False):
    from autovfx_b200 import png
    buf, size = png.encode_png(img, lut=lut, swap_rb=swap_rb)
    return buf[: int(size)].cpu().numpy().tobytes()


def _pil(data):
    from PIL import Image
    return np.array(Image.open(io.BytesIO(data)))


def _cv2(data):
    import cv2
    a = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)
    if a.ndim == 3:
        a = a[:, :, ::-1] if a.shape[2] == 3 else a[:, :, [2, 1, 0, 3]]
    return a


def _check_file(data, want, small=None):
    """Every decoder gives `want`; the chunk CRCs, IHDR, Adler-32 and BFINAL flags are right; no file exceeds the bound."""
    from autovfx_b200 import png
    H, W = want.shape[:2]
    Cn = want.shape[2] if want.ndim == 3 else 1
    assert len(data) <= png.png_bound(H, W, Cn)
    assert all(ok for _, _, ok in PR.chunks(data)), "chunk CRC"
    h = PR.ihdr(data)
    assert (h["W"], h["H"], h["depth"], h["ctype"], h["interlace"]) == (W, H, 8, {1: 0, 3: 2, 4: 6}[Cn], 0)
    z = b"".join(p for t, p, _ in PR.chunks(data) if t == b"IDAT")
    zlib.decompress(z)  # checks the Adler-32
    assert np.array_equal(_pil(data), want)
    assert np.array_equal(_cv2(data), want)
    if small if small is not None else H * W <= 4096:
        assert np.array_equal(PR.decode(data), want)
        f = PR.block_finals(data)
        assert f[-1] == 1 and not any(f[:-1])


def _gradient(H, W, Cn):
    y, x = np.mgrid[0:H, 0:W]
    a = np.stack([(x * 255 // max(W - 1, 1) + 37 * c) % 256 if c % 2 == 0 else (y * 255 // max(H - 1, 1) + 11 * c) % 256 for c in range(Cn)], -1)
    return a.astype(np.uint8) if Cn > 1 else a[:, :, 0].astype(np.uint8)


@pytest.mark.parametrize("W", [1, 2, 3, 5, 17, 1921])
@pytest.mark.parametrize("H", [1, 2, 1081])
@pytest.mark.parametrize("Cn", [1, 3, 4])
def test_round_trip_gradients(dev, H, W, Cn):
    a = _gradient(H, W, Cn)
    _check_file(_bytes(torch.from_numpy(a).to(dev)), a)


@pytest.mark.parametrize("Cn", [1, 3, 4])
def test_constant_images(dev, Cn):
    for v in (0, 200):
        a = np.full((1081, 1921, Cn), v, np.uint8) if Cn > 1 else np.full((1081, 1921), v, np.uint8)
        data = _bytes(torch.from_numpy(a).to(dev))
        _check_file(data, a)
        assert len(data) < a.size // 100


@pytest.mark.parametrize("Cn", [1, 4])
def test_noise_falls_back_to_stored(dev, Cn):
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, (517, 601, Cn) if Cn > 1 else (517, 601), dtype=np.uint8)
    data = _bytes(torch.from_numpy(a).to(dev))
    _check_file(data, a)
    from autovfx_b200 import png
    assert len(data) <= png.png_bound(517, 601, Cn)


def test_4k_rgba(dev):
    rng = np.random.default_rng(6)
    a = np.concatenate([_gradient(2160, 3840, 3), np.full((2160, 3840, 1), 255, np.uint8)], -1)
    a[rng.random((2160, 3840)) < 0.02] = 7
    _check_file(_bytes(torch.from_numpy(a).to(dev)), a)


def test_strided_and_channel_reversed(dev):
    a = _gradient(301, 403, 4)
    t = torch.from_numpy(a).to(dev)
    _check_file(_bytes(t[::2, 1::3]), a[::2, 1::3])
    _check_file(_bytes(t[:, :, :3], swap_rb=True), a[:, :, 2::-1].copy())
    _check_file(_bytes(t, swap_rb=True), a[:, :, [2, 1, 0, 3]])
    chw = t.permute(2, 0, 1).contiguous()
    _check_file(_bytes(chw.permute(1, 2, 0)), a)  # a CHW tensor read in place


@pytest.mark.parametrize("delta", [-1, 0, 1])
@pytest.mark.parametrize("n", [1, 2])
def test_stream_length_on_chunk_boundaries(dev, delta, n):
    # one grey row: the filtered stream is 1 + W = n 32768 + delta bytes
    W = n * 32768 + delta - 1
    a = _gradient(1, W, 1)
    a[:, ::3] = 9
    _check_file(_bytes(torch.from_numpy(a).to(dev)), a, small=True)


def test_lut_index_image(dev):
    from autovfx_b200 import png
    from autovfx_b200.renderer import TURBO_LUT_BGR
    a = _gradient(257, 333, 1)
    lut = png.turbo_lut_rgb(dev)
    data = _bytes(torch.from_numpy(a).to(dev), lut=lut)
    _check_file(data, TURBO_LUT_BGR.numpy()[a][:, :, ::-1].copy())


def _render_frames(dev, n, W, H, P, product=True):
    from autovfx_b200 import render_loop as RL, scene
    g = scene.synthetic_gaussians(P, seed=4)
    cams = [scene.lookat_camera((0.3 * i, -3.0, 0.4), (0, 0, 0), W, H, 60.0) for i in range(n)]
    loop = RL.FrameLoop({k: v.to(dev) for k, v in g.items()}, 3, W, H, device=dev, to_host=False, pack8=True, product=product)
    return loop, RL.pack_cameras(cams)


@pytest.mark.parametrize("W,H,P", [(320, 192, 20000), (1920, 1080, 3_000_000)])
def test_rendered_frames_round_trip_and_size(dev, W, H, P):
    from PIL import Image
    from autovfx_b200 import png
    loop, cams = _render_frames(dev, 1, W, H, P)
    got = []

    def consume(i, fr, stats):
        lut = png.turbo_lut_rgb(dev)
        for img, kw, want in ((fr["rgba8"], {}, fr["rgba8"].cpu().numpy()), (fr["normal8"], {}, fr["normal8"].cpu().numpy()),
                              (fr["depth8"], {"lut": lut}, lut.cpu().numpy()[fr["depth8"].cpu().numpy()])):
            data = _bytes(img, **kw)
            _check_file(data, want, small=False)
            b = io.BytesIO()
            Image.fromarray(want).save(b, format="PNG")
            got.append(len(data) / len(b.getvalue()))
    loop.render(cams, consume)
    print("size vs PIL (rgba, normal, depth):", ["%.3f" % r for r in got])
    assert max(got) <= SIZE_RATIO_K, got


def test_gradient_size_vs_pil(dev):
    from PIL import Image
    a = _gradient(1080, 1920, 4)
    data = _bytes(torch.from_numpy(a).to(dev))
    b = io.BytesIO()
    Image.fromarray(a).save(b, format="PNG")
    print("gradient size vs PIL: %.3f" % (len(data) / len(b.getvalue())))
    assert len(data) <= SIZE_RATIO_K_GRADIENT * len(b.getvalue())


def test_deterministic_bytes(dev):
    from autovfx_b200 import png
    a = torch.from_numpy(_gradient(1081, 1921, 4)).to(dev)
    a[::7, ::5] = 3
    g = torch.from_numpy(_gradient(513, 700, 1)).to(dev)
    ref = _bytes(a)
    assert _bytes(a) == ref
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        buf, size = png.encode_png(a)
    side.synchronize()
    assert buf[: int(size)].cpu().numpy().tobytes() == ref
    buf, spans, sizes = png.encode_pngs([g, a, (g, png.turbo_lut_rgb(dev))])
    torch.cuda.synchronize()
    o, _ = spans[1]
    assert buf[o: o + int(sizes[1])].cpu().numpy().tobytes() == ref
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        assert _bytes(a) == ref
    finally:
        torch.use_deterministic_algorithms(prev)


def test_save_image_matches_torchvision(dev):
    import torchvision
    from autovfx_b200 import png
    torch.manual_seed(0)
    for Cn in (1, 3, 4):
        x = torch.rand(Cn, 97, 131, device=dev) * 1.2 - 0.1
        with tempfile.TemporaryDirectory() as tmp:
            p1, p2 = os.path.join(tmp, "a.png"), os.path.join(tmp, "b.png")
            torchvision.utils.save_image(x, p1)
            png.save_image(x, p2)
            from PIL import Image
            assert np.array_equal(np.array(Image.open(p1)), np.array(Image.open(p2)))
    with pytest.raises(ValueError):
        png.save_image(x, "unused.png", nrow=2)


def test_imwrite_matches_cv2(dev):
    import cv2
    from autovfx_b200 import png
    rng = np.random.default_rng(3)
    for shape in ((61, 83), (61, 83, 3), (61, 83, 4)):
        a = (rng.integers(0, 4, shape) * 60).astype(np.uint8)
        with tempfile.TemporaryDirectory() as tmp:
            p1, p2 = os.path.join(tmp, "a.png"), os.path.join(tmp, "b.png")
            cv2.imwrite(p1, a)
            assert png.imwrite(p2, a) is True
            assert png.imwrite(p2, torch.from_numpy(a).to(dev)) is True
            f = cv2.IMREAD_UNCHANGED
            assert np.array_equal(cv2.imread(p1, f), cv2.imread(p2, f))


def test_frame_files_match_the_reference_loop_lines(dev):
    """FrameFiles' files against the reference loop's lines (scene_representation.py:424-438) on the same frame: save_image of the
    RGBA render, np.save of the depth, depth2img + cv2.imwrite and the normal map's (n+1)/2*255 + cvtColor + imwrite; no host
    synchronisation in consume."""
    import cv2
    from PIL import Image
    from autovfx_b200 import png
    from autovfx_b200.renderer import TURBO_LUT_BGR
    loop, cams = _render_frames(dev, 3, 320, 192, 20000)
    ref = {}
    with tempfile.TemporaryDirectory() as tmp:
        ff = png.FrameFiles(tmp, names=["f%d" % i for i in range(3)])

        def consume(i, fr, stats):
            torch.cuda.set_sync_debug_mode("error")
            try:
                ff(i, fr, stats)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            ref[i] = {k: v.cpu().numpy() for k, v in fr.items()}
        loop.render(cams, consume)
        ff.close()
        for i in range(3):
            r = ref[i]
            b = io.BytesIO()
            np.save(b, r["depth"].astype(np.float32))
            assert open(os.path.join(tmp, "depth", "f%d.npy" % i), "rb").read() == b.getvalue()
            # depth2img(depth, 3.0) with cv2.applyColorMap == TURBO_LUT_BGR[depth8] (renderer.pack_frame), written by cv2
            with tempfile.TemporaryDirectory() as t2:
                cv2.imwrite(os.path.join(t2, "d.png"), TURBO_LUT_BGR.numpy()[r["depth8"]])
                cv2.imwrite(os.path.join(t2, "n.png"), cv2.cvtColor(r["normal8"], cv2.COLOR_RGB2BGR))
                f = cv2.IMREAD_UNCHANGED
                assert np.array_equal(cv2.imread(os.path.join(tmp, "depth", "f%d.png" % i), f), cv2.imread(os.path.join(t2, "d.png"), f))
                assert np.array_equal(cv2.imread(os.path.join(tmp, "normal", "f%d.png" % i), f), cv2.imread(os.path.join(t2, "n.png"), f))
            assert np.array_equal(np.array(Image.open(os.path.join(tmp, "images", "f%d.png" % i))), r["rgba8"])


def test_writer_no_host_sync_and_errors(dev):
    from autovfx_b200 import png
    a = torch.from_numpy(_gradient(200, 300, 4)).to(dev)
    with tempfile.TemporaryDirectory() as tmp:
        w = png.PngWriter(ring=2)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for k in range(5):
                w.submit(os.path.join(tmp, "%d.png" % k), a, swap_rb=bool(k % 2))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        w.flush()
        for k in range(5):
            want = a.cpu().numpy()
            if k % 2:
                want = want[:, :, [2, 1, 0, 3]]
            assert np.array_equal(_pil(open(os.path.join(tmp, "%d.png" % k), "rb").read()), want)
        w.submit(os.path.join(tmp, "missing_dir", "x.png"), a)
        with pytest.raises(RuntimeError):
            w.flush()
        w.close()


def test_argument_errors(dev):
    from autovfx_b200 import png
    with pytest.raises(RuntimeError):
        png.encode_png(torch.zeros(4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):
        png.encode_png(torch.zeros(4, 4, 3, device=dev))
    with pytest.raises(ValueError):
        png.encode_png(torch.zeros(4, 4, 2, dtype=torch.uint8, device=dev))
    with pytest.raises(ValueError):
        png.encode_png(torch.zeros(4, 4, 3, dtype=torch.uint8, device=dev), lut=png.turbo_lut_rgb(dev))
    with pytest.raises(ValueError):
        png.encode_png(torch.zeros(0, 4, 3, dtype=torch.uint8, device=dev))
    with pytest.raises(ValueError):
        png.imwrite("x.jpg", np.zeros((2, 2, 3), np.uint8))


def test_blend_frames_with_png_writer(dev):
    """blend_frames(png_writer=...) writes frames with the same pixels as the default PIL path, and the same video frames."""
    from PIL import Image
    from autovfx_b200 import png
    from tests import test_gpu_composite as TC
    from tests import composite_ref as CR
    m = TC._loaders_module()
    got = TC._install(m)
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, cases = CR.write_dir(tmp, 3, 500, 31, 45)
        m.blend_frames(results, cfg)
        pil = [np.array(Image.open(os.path.join(results, "frames", "%04d.png" % i))) for i in range(3)]
        frames0 = got.pop("frames")
        with png.PngWriter() as w:
            m.blend_frames(results, cfg, png_writer=w)
        ours = [np.array(Image.open(os.path.join(results, "frames", "%04d.png" % i))) for i in range(3)]
    assert np.array_equal(frames0, got["frames"])
    for a, b in zip(pil, ours):
        assert np.array_equal(a, b)
