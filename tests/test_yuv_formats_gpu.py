"""GPU tests of the 4:2:2 / 4:4:4 / 4:4:0 / 10-bit video front (bilinear.cu, yuv_rgba_kernel<F> and its tiled twin):
b200timg_yuv_scale for every new format against the float64 restatement (tests/yuv_cases.py) within 1 LSB, limited
and full range, through both kernels; the table cache under alternating formats; the batch entry points (host and
device-resident) against the staged pipeline; the rejected arguments.  The restatement's own distance to libswscale
is pinned on the CPU in test_yuv_formats_oracle.py."""
import base64
import ctypes as C
import os
import sys

import numpy as np
import pytest

import timg_b200
from timg_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import yuv_cases as Y  # noqa: E402
from test_graphics_oracle import iterm2_payload, kitty_payload, png_pixels  # noqa: E402

pytestmark = pytest.mark.gpu

# test_yuv_gpu.py's geometries: width 130 is not a multiple of 8 and runs the per-pixel kernel, the others the tiled
# one unless B200TIMG_YUV_SIMPLE is set; plus odd sizes where the format allows them
GEOMS = [(640, 480, 450, 337, "photo"), (1920, 1080, 320, 90, "photo"), (256, 128, 300, 200, "noise"),
         (3840, 216, 2700, 152, "photo"), (64, 48, 64, 48, "noise"), (130, 98, 67, 50, "alpha")]
ODD = {Y.I422: (130, 97), Y.I444: (131, 97), Y.I440: (131, 98), Y.I422_10: (130, 97), Y.I444_10: (131, 97)}


def _frame(fmt, iw, ih, kind, seed=3):
    return Y.rgba_to_yuv_np(synth.frame_np(seed + iw, iw, ih, kind), fmt)


def _check(ctx, buf, fmt, iw, ih, ow, oh):
    planes = Y.planes_np(buf, fmt, iw, ih)
    for fr in (0, timg_b200.FMT_FULL_RANGE):
        got = ctx.yuv_scale(buf, iw, ih, ow, oh, fmt | fr)
        want = Y.yuv_to_rgba_np(planes, fmt, ow, oh, full_range=bool(fr))
        e = np.abs(got.astype(int) - want)
        assert e.max() <= 1, (Y.NAMES[fmt], fr, int(e.max()), float(e.mean()))


@pytest.mark.parametrize("simple", [False, True], ids=["tiled", "simple"])
@pytest.mark.parametrize("fmt", Y.NEW_FORMATS, ids=lambda f: Y.NAMES[f])
@pytest.mark.parametrize("iw,ih,ow,oh,kind", GEOMS)
def test_new_format_matches_restatement(ctx, monkeypatch, iw, ih, ow, oh, kind, fmt, simple):
    if simple:
        monkeypatch.setenv("B200TIMG_YUV_SIMPLE", "1")
    _check(ctx, _frame(fmt, iw, ih, kind), fmt, iw, ih, ow, oh)


@pytest.mark.parametrize("fmt", sorted(ODD), ids=lambda f: Y.NAMES[f])
def test_odd_sizes_where_the_format_allows_them(ctx, fmt):
    iw, ih = ODD[fmt]
    for ow, oh in ((70, 41), (iw, ih), (200, 151)):
        _check(ctx, _frame(fmt, iw, ih, "photo"), fmt, iw, ih, ow, oh)


@pytest.mark.parametrize("fmt", (Y.I420_10, Y.I422_10, Y.I444_10, Y.P010), ids=lambda f: Y.NAMES[f])
@pytest.mark.parametrize("iw,ih,ow,oh", [(640, 480, 450, 337), (130, 98, 67, 50)])
def test_10bit_reads_only_the_value_bits(ctx, fmt, iw, ih, ow, oh):
    buf = _frame(fmt, iw, ih, "photo")
    stray = np.random.default_rng(iw + fmt).integers(0, 64, buf.size).astype(np.uint16)
    noisy = buf | (stray if fmt == Y.P010 else stray << 10)
    assert (ctx.yuv_scale(noisy, iw, ih, ow, oh, fmt) == ctx.yuv_scale(buf, iw, ih, ow, oh, fmt)).all()


def test_table_cache_keys_on_the_chroma_layout(ctx):
    """One context alternating formats at one geometry gives what a fresh context gives for each call."""
    for iw, ih, ow, oh in ((640, 480, 450, 337), (64, 48, 64, 48)):
        bufs = {f: _frame(f, iw, ih, "photo", seed=17) for f in (Y.I420, Y.I444, Y.I422_10)}
        fresh = {}
        for f, buf in bufs.items():
            c = timg_b200.Context(0)
            fresh[f] = c.yuv_scale(buf, iw, ih, ow, oh, f)
            c.close()
        for f in (Y.I420, Y.I444, Y.I422_10, Y.I444, Y.I420, Y.I422_10, Y.I420):
            assert (ctx.yuv_scale(bufs[f], iw, ih, ow, oh, f) == fresh[f]).all(), (iw, Y.NAMES[f])


def _batch(n, iw, ih, fmt, ow, oh, flags=0, animation=0):
    return timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=fmt, out_w=ow, out_h=oh, has_bg=1,
                           bg=timg_b200.rgba_u32(0, 0, 0), pattern=0, pattern_w=0, pattern_h=0, flags=flags,
                           x_indent_cells=0, animation=animation)


@pytest.mark.parametrize("fmt", (Y.I422, Y.I444, Y.I440, Y.I422_10, Y.P010), ids=lambda f: Y.NAMES[f])
def test_batches_equal_staged_pipeline(ctx, fmt):
    """Frames of a new format through the batch entry points == b200timg_yuv_scale followed by the RGBA stages."""
    n, iw, ih = 3, 320, 240
    _, ow, oh = timg_b200.calc_fit(iw, ih, 80, 50, 1, 2)
    frames = np.stack([_frame(fmt, iw, ih, "photo", seed=70 + i) for i in range(n)])
    b = _batch(n, iw, ih, fmt, ow, oh)
    blocks = ctx.blocks_batch(frames, b)
    for f in range(n):
        assert blocks[f] == ctx.blocks_encode(ctx.yuv_scale(frames[f], iw, ih, ow, oh, fmt)), f
    b2 = _batch(n, iw, ih, fmt | timg_b200.FMT_FULL_RANGE, 200, 150)
    sixels = ctx.sixel_batch(frames, b2)
    for f in range(n):
        assert sixels[f] == ctx.sixel_encode(ctx.yuv_scale(frames[f], iw, ih, 200, 150, fmt | timg_b200.FMT_FULL_RANGE)), f
    b3 = _batch(n, iw, ih, fmt, 161, 97)
    for proto in (timg_b200.KITTY, timg_b200.ITERM2):
        outs = ctx.graphics_batch(frames, b3, proto, False, [5, 6, 7])
        for f in range(n):
            payload = kitty_payload(outs[f]) if proto == timg_b200.KITTY else iterm2_payload(outs[f], 161, 97)
            assert (png_pixels(base64.b64decode(payload))[0] == ctx.yuv_scale(frames[f], iw, ih, 161, 97, fmt)).all(), (proto, f)


def _dev_batch(ctx, fn, frames, b, cap):
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("device-resident variants need torch with CUDA")
    d = torch.from_numpy(np.ascontiguousarray(frames).reshape(frames.shape[0], -1).view(np.uint8)).cuda()
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(b.n_frames + 1, dtype=torch.int64, device="cuda")
    ctx._chk(fn(ctx.h, C.byref(b), d.data_ptr(), out.data_ptr(), cap, offs.data_ptr()))
    torch.cuda.synchronize()
    o, ob = offs.cpu().numpy(), out.cpu().numpy()
    return [ob[int(o[i]):int(o[i + 1])].tobytes() for i in range(b.n_frames)]


@pytest.mark.parametrize("fmt", (Y.I444, Y.I420_10, Y.P010), ids=lambda f: Y.NAMES[f])
def test_host_and_device_batches_agree(ctx, monkeypatch, fmt):
    """Host variants, cut into several chunks by the pipeline, give the device-resident variants' bytes."""
    L = timg_b200.lib()
    n, iw, ih = 7, 256, 144
    frames = np.stack([_frame(fmt, iw, ih, "noise" if i % 2 else "photo", seed=90 + i) for i in range(n)])
    quarter = _batch(n, iw, ih, fmt, 128, 72, flags=timg_b200.QUARTER, animation=1)
    sixel = _batch(n, iw, ih, fmt, 200, 113)
    dev_blocks = _dev_batch(ctx, L.b200timg_blocks_batch_dev, frames, quarter, int(L.b200timg_blocks_bound(128, 72)) * n + 64)
    dev_sixel = _dev_batch(ctx, L.b200timg_sixel_batch_dev, frames, sixel, n * int(L.b200timg_sixel_bound(200, 114)))
    iterm2 = _batch(n, iw, ih, fmt, 96, 54)
    dev_iterm2 = _dev_batch(ctx, lambda h, b, s, o, cap, offs: L.b200timg_graphics_batch_dev(
        h, b, C.byref(timg_b200.graphics(timg_b200.ITERM2)[0]), s, o, cap, offs), frames, iterm2,
        n * int(timg_b200.graphics_size(timg_b200.ITERM2, 96, 54)))
    for chunk in (None, "3", "1"):
        if chunk:
            monkeypatch.setenv("B200TIMG_CHUNK_FRAMES", chunk)
        assert ctx.blocks_batch(frames, quarter) == dev_blocks, chunk
        assert ctx.sixel_batch(frames, sixel) == dev_sixel, chunk
        assert ctx.graphics_batch(frames, iterm2, timg_b200.ITERM2) == dev_iterm2, chunk


def test_rejected_arguments(ctx):
    img = synth.frame_np(1, 64, 48, "photo")
    out = np.empty((10, 10, 4), np.uint8)
    L = timg_b200.lib()
    # odd sizes where the format subsamples
    for fmt, (iw, ih) in ((Y.I420, (63, 48)), (Y.I422, (63, 48)), (Y.I440, (64, 47)), (Y.I420_10, (64, 47)),
                          (Y.I422_10, (63, 48)), (Y.P010, (63, 48)), (Y.NV12, (64, 47))):
        buf = np.zeros(4 * 64 * 48, np.uint8)
        rc = L.b200timg_yuv_scale(ctx.h, buf.ctypes.data_as(timg_b200.u8p), iw, ih, fmt, out.ctypes.data_as(timg_b200.u8p), 10, 10)
        assert rc == timg_b200.EINVAL, Y.NAMES[fmt]
        assert Y.NAMES[fmt] in L.b200timg_last_error(ctx.h).decode()
        b = _batch(1, iw, ih, fmt, 10, 10)
        with pytest.raises(timg_b200.B200Error) as ex:
            ctx.blocks_batch(buf[None, : timg_b200.yuv_frame_bytes(fmt, iw, ih)], b)
        assert ex.value.code == timg_b200.EINVAL
    # unknown codes (the buffer holds an RGBA frame of the size: a batch takes any unknown code for RGBA-sized frames)
    buf = np.zeros(64 * 48 * 4, np.uint8)
    for fmt in (11, 12, 15, 11 | timg_b200.FMT_FULL_RANGE):
        rc = L.b200timg_yuv_scale(ctx.h, buf.ctypes.data_as(timg_b200.u8p), 64, 48, fmt, out.ctypes.data_as(timg_b200.u8p), 10, 10)
        assert rc == timg_b200.EINVAL, fmt
        with pytest.raises(timg_b200.B200Error) as ex:
            ctx.blocks_batch(buf[None], _batch(1, 64, 48, fmt, 10, 10))
        assert ex.value.code == timg_b200.EINVAL
    # a buffer that is not one frame of the format
    for fmt in Y.NEW_FORMATS:
        good = Y.rgba_to_yuv_np(img, fmt)
        for bad in (good[:-1], np.concatenate([good, good[:1]]), Y.rgba_to_yuv_np(img, Y.I420)):
            if bad.nbytes == good.nbytes:
                continue
            with pytest.raises(timg_b200.B200Error) as ex:
                ctx.yuv_scale(bad, 64, 48, 10, 10, fmt)
            assert ex.value.code == timg_b200.EINVAL
        with pytest.raises(TypeError):
            ctx.yuv_scale(good.astype(np.float32), 64, 48, 10, 10, fmt)
