"""GIF decode on the device (b200timg_gif_frames / _dev) against the reference's own decode: every canvas the STB
source's loop collects and the count, byte for byte, for the corpus (tests/gif_cases.py, stored in
tests/golden/gif.npz with SHA-256 pins of the reference's canvases), Pillow-written files, and three large animations;
a fixed number of launches whatever the frame count; the canvases feeding the existing batches on the device."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import gif_cases
import oracle
import timg_b200
from oracle import gif as G

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "gif.npz"))
NAMES = [str(n) for n in GOLD["names"]]
KEYS = [f"c/{n}" for n in NAMES] + [f"pil/{k}" for k in range(int(GOLD["pil_count"]))]
BG = oracle.rgba_u32(0, 0, 0)
needs_ref = pytest.mark.skipif(not G.have_ref(), reason="oracle/_ref/libtimg_gif_ref.so not built")


def _dev():
    import torch
    return "cuda" if torch.cuda.is_available() else "cpu"     # cpu: only under the CPU kernel simulator


def _sha(frames):
    return hashlib.sha256(b"".join(np.ascontiguousarray(f).tobytes() for f in frames)).hexdigest()


def _decodable(key):
    data = GOLD[f"{key}/file"].tobytes()
    try:
        timg_b200.gif_parse(data)
    except timg_b200.B200Error:
        return None
    return data


@pytest.mark.parametrize("key", KEYS)
def test_canvases_equal_the_reference_pins(ctx, key):
    data = _decodable(key)
    want_n = int(GOLD[f"{key}/n_valid"])
    if data is None:
        assert want_n == 0                                   # the reference's source fails too
        return
    frames, n_valid = ctx.gif_frames(data)
    assert n_valid == want_n
    assert _sha(frames[:n_valid]) == str(GOLD[f"{key}/sha"])


@needs_ref
@pytest.mark.parametrize("key", KEYS)
def test_canvases_equal_the_live_reference(ctx, key):
    data = _decodable(key)
    if data is None:
        return
    ref = G.ref_stb_gif(data)
    want = ref[0] if ref is not None else []
    frames, n_valid = ctx.gif_frames(data)
    assert n_valid == len(want)
    for k in range(n_valid):
        assert (frames[k] == want[k]).all(), k


@pytest.mark.parametrize("key", ["c/no-clear-frame1", "c/too-many-codes-frame1", "c/anim-64x48x12", "pil/0"])
def test_dev_form_equals_host_form(ctx, key):
    import torch
    data = GOLD[f"{key}/file"].tobytes()
    w, h, delays = timg_b200.gif_parse(data)
    n = len(delays)
    host, n_valid = ctx.gif_frames(data)
    d = torch.full((n * h * w * 4,), 7, dtype=torch.uint8, device=_dev())
    timg_b200.device_sync(torch)
    d_valid = ctx.gif_frames_dev(data, d, n)
    timg_b200.device_sync(torch)
    assert int(d_valid.cpu()[0]) == n_valid
    got = d.cpu().numpy().reshape(n, h, w, 4)
    assert (got[:n_valid] == host[:n_valid]).all()
    # fewer frames than the file has: the first ones, the same count rule
    if n > 1:
        part, nv = ctx.gif_frames(data, n - 1)
        assert nv == min(n_valid, n - 1) and (part[:nv] == host[:nv]).all()


@pytest.mark.parametrize("name", gif_cases.SIZED)
def test_sized_animations_equal_the_reference_pins(ctx, name):
    data = gif_cases.sized(name)
    frames, n_valid = ctx.gif_frames(data)
    assert n_valid == int(GOLD[f"sized/{name}/n_valid"]) == frames.shape[0]
    assert _sha(frames) == str(GOLD[f"sized/{name}/sha"])


def test_launch_count_does_not_depend_on_frames(ctx):
    one = gif_cases.sized("4096x2160x1")
    many = gif_cases.sized("480x270x120")
    l0 = ctx.launches
    ctx.gif_frames(one)
    l1 = ctx.launches
    ctx.gif_frames(many)
    l2 = ctx.launches
    assert l1 - l0 == l2 - l1 == 3


def _batch(n, w, h, ow, oh, **kw):
    d = dict(n_frames=n, src_w=w, src_h=h, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=BG, pattern=0, pattern_w=0,
             pattern_h=0, flags=0, x_indent_cells=0, animation=0)
    d.update(kw)
    return timg_b200.Batch(**d)


def _decode_dev(ctx, data):
    import torch
    w, h, delays = timg_b200.gif_parse(data)
    n = len(delays)
    d = torch.empty(n * h * w * 4, dtype=torch.uint8, device=_dev())
    d_valid = ctx.gif_frames_dev(data, d, n)
    timg_b200.device_sync(torch)                   # d_valid is read on torch's stream, the call ran on the context's
    return d, int(d_valid.cpu()[0]), w, h


def _run_dev(ctx, fn, b, d_src, cap, *extra):
    import torch
    d_out = torch.zeros(cap, dtype=torch.uint8, device=_dev())
    d_offs = torch.zeros(b.n_frames + 1, dtype=torch.int64, device=_dev())
    timg_b200.device_sync(torch)
    ctx._chk(fn(ctx.h, C.byref(b), *extra, d_src.data_ptr(), d_out.data_ptr(), cap, d_offs.data_ptr()))
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    return [data[o[f]:o[f + 1]].tobytes() for f in range(b.n_frames)]


@needs_ref
def test_quarter_animation_from_decoded_canvases_equals_reference_canvas(ctx):
    """-p quarter: the reference's STB source scales and composes every frame and its UnicodeBlockCanvas emits the
    animation with dy = -height; the device decodes, then one blocks batch (animation = 1) scales, composes and
    emits the same bytes."""
    data = gif_cases.sized("480x270x120")
    ref = G.ref_stb_gif(data, width=160, height=100, cell=(2, 2), has_bg=True, bg=BG)
    frames, meta = ref
    ow, oh = int(meta[0, 0]), int(meta[0, 1])
    canvas = oracle.RefBlockCanvas(quarter=True)
    want = [canvas.send(frames[k], int(meta[k, 2]), int(meta[k, 3])) for k in range(len(frames))]
    assert all(int(meta[k, 3]) == (-oh if k else 0) for k in range(len(frames)))
    d, n_valid, w, h = _decode_dev(ctx, data)
    assert n_valid == len(frames)
    b = _batch(n_valid, w, h, ow, oh, flags=timg_b200.QUARTER, animation=1)
    outs = _run_dev(ctx, timg_b200.lib().b200timg_blocks_batch_dev, b, d,
                    timg_b200.lib().b200timg_blocks_bound(ow, oh) * n_valid)
    up = b"\033[%dA" % ((oh + 1) // 2)                      # the adapter's cursor-up; the ABI returns image bytes
    for k in range(n_valid):
        assert (up if k else b"") + outs[k] == want[k], k


def test_sixel_and_kitty_batches_on_decoded_canvases(ctx):
    """Decoded canvases feed the existing batches on the device: the same bytes as those batches on the reference's
    canvases (the host decode, pinned to the reference's SHA-256 above)."""
    key = "c/anim-64x48x12"
    data = GOLD[f"{key}/file"].tobytes()
    ref, n_valid = ctx.gif_frames(data)
    assert _sha(ref[:n_valid]) == str(GOLD[f"{key}/sha"])
    d, nv, w, h = _decode_dev(ctx, data)
    assert nv == n_valid
    ow, oh = 40, 30
    b = _batch(n_valid, w, h, ow, oh)
    hp = (oh + 5) // 6 * 6
    six = _run_dev(ctx, timg_b200.lib().b200timg_sixel_batch_dev, b, d, timg_b200.lib().b200timg_sixel_bound(ow, hp) * n_valid)
    assert six == ctx.sixel_batch(ref[:n_valid], _batch(n_valid, w, h, ow, oh))
    for protocol in (timg_b200.KITTY, timg_b200.ITERM2):
        g, keep = timg_b200.graphics(protocol, ids=list(range(1, n_valid + 1)))
        cap = sum(timg_b200.lib().b200timg_graphics_size(C.byref(g), ow, oh, k + 1) for k in range(n_valid))
        gfx = _run_dev(ctx, timg_b200.lib().b200timg_graphics_batch_dev, b, d, cap, C.byref(g))
        want = ctx.graphics_batch(ref[:n_valid], _batch(n_valid, w, h, ow, oh), protocol, ids=list(range(1, n_valid + 1)))
        assert gfx == want, protocol


def test_rejections(ctx):
    import torch
    data = GOLD["c/anim-64x48x12/file"].tobytes()
    w, h, delays = timg_b200.gif_parse(data)
    n = len(delays)
    d = torch.empty(n * h * w * 4, dtype=torch.uint8, device=_dev())
    v = torch.empty(1, dtype=torch.int32, device=_dev())
    L = timg_b200.lib()
    png = b"\x89PNG\r\n\x1a\n" + bytes(64)
    assert L.b200timg_gif_frames_dev(ctx.h, png, len(png), 1, d.data_ptr(), v.data_ptr()) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(ctx.h, data, len(data), n + 1, d.data_ptr(), v.data_ptr()) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(ctx.h, data, len(data), 0, d.data_ptr(), v.data_ptr()) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(ctx.h, None, len(data), 1, d.data_ptr(), v.data_ptr()) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(ctx.h, data, len(data), 1, None, v.data_ptr()) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(ctx.h, data, len(data), 1, d.data_ptr(), None) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(None, data, len(data), 1, d.data_ptr(), v.data_ptr()) == timg_b200.EINVAL
    # misaligned outputs (canvases are stored as whole pixels, the count as int32) are rejected before any launch
    launches = ctx.launches
    assert L.b200timg_gif_frames_dev(ctx.h, data, len(data), 1, d.data_ptr() + 1, v.data_ptr()) == timg_b200.EINVAL
    assert L.b200timg_gif_frames_dev(ctx.h, data, len(data), 1, d.data_ptr(), v.data_ptr() + 2) == timg_b200.EINVAL
    assert ctx.launches == launches
    out = np.empty(n * h * w * 4, np.uint8)
    nv = C.c_int()
    assert L.b200timg_gif_frames(ctx.h, data, len(data), n + 1, out.ctypes.data, C.byref(nv)) == timg_b200.EINVAL
    assert L.b200timg_gif_frames(ctx.h, data, len(data), n, None, C.byref(nv)) == timg_b200.EINVAL
    assert L.b200timg_gif_frames(ctx.h, data, len(data), n, out.ctypes.data, None) == timg_b200.EINVAL
    with pytest.raises(timg_b200.B200Error):
        ctx.gif_frames(png)
    frames, nv = ctx.gif_frames(data)                     # the context still works
    assert nv == n
