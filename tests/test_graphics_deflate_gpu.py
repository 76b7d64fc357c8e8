"""B200TIMG_DEFLATE on the GPU: every frame's PNG is valid (chunk CRCs, zlib's Adler-32) and decodes to the frame,
the reference's own PNG writer and canvases write exactly our bytes around our deflate stream (replay oracle), the
compressed size is bounded by the stored size and close to zlib level 1, a frame's bytes depend on that frame only,
and the capacity contract and argument checks hold."""
import base64
import ctypes as C
import os
import re
import sys
import zlib

import numpy as np
import pytest

import timg_b200
from timg_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_cases as gcases  # noqa: E402
from test_graphics_deflate_oracle import ReplayCanvas, scanlines  # noqa: E402
from test_graphics_oracle import iterm2_payload, kitty_payload, png_pixels  # noqa: E402
from test_graphics_tmux_oracle import kitty_tmux_payload  # noqa: E402

pytestmark = pytest.mark.gpu

D = timg_b200.DEFLATE
PROTOS = {"kitty": timg_b200.KITTY, "iterm2": timg_b200.ITERM2, "tmux": timg_b200.KITTY_TMUX}
CELL = (9, 18)


def _batch(n, iw, ih, ow, oh, **kw):
    d = dict(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=0, bg=0, pattern=0, pattern_w=0,
             pattern_h=0, flags=0, x_indent_cells=0, animation=0)
    d.update(kw)
    return timg_b200.Batch(**d)


def _png(text, proto, w, h):
    if proto == timg_b200.KITTY:
        b64 = kitty_payload(text)
    elif proto == timg_b200.ITERM2:
        b64 = iterm2_payload(text, w, h)
    else:
        b64 = kitty_tmux_payload(text)[0]
    return base64.b64decode(b64, validate=True)


def _idat(png):
    n = int.from_bytes(png[33:37], "big")
    assert png[37:41] == b"IDAT"
    return png[41:41 + n]


def _kw(proto):
    return dict(cell=CELL) if proto == timg_b200.KITTY_TMUX else {}


@pytest.mark.parametrize("pname", list(PROTOS))
def test_frames_decode_and_equal_the_replayed_reference(ctx, pname):
    """Every frame case, both colour types: PNG valid and equal to the frame; the reference's canvas, given our zlib
    stream, writes exactly our bytes (kitty ids: ours are rerun with the id the reference picked)."""
    proto = PROTOS[pname]
    for name, fb, rgb24 in gcases.graphics_frame_cases():
        h, w = fb.shape[:2]
        b = _batch(1, w, h, w, h)
        text = ctx.graphics_batch(fb[None], b, proto | D, rgb24, [1], **_kw(proto))[0]
        png = _png(text, proto, w, h)
        px, ctype = png_pixels(png)
        assert (px == (fb[..., :3] if rgb24 else fb)).all(), name
        assert len(png) <= timg_b200.lib().b200timg_png_size(w, h, rgb24), name
        want = ReplayCanvas(proto, rgb24, CELL).send(_idat(png), fb)
        if proto != timg_b200.ITERM2:
            id_ = int(re.search(rb"i=(\d+),", want).group(1))
            text = ctx.graphics_batch(fb[None], b, proto | D, rgb24, [id_], **_kw(proto))[0]
        assert text == want, name


def test_scale_and_compose_in_the_batch(ctx):
    n, iw, ih, ow, oh = 3, 640, 480, 251, 187
    frames = np.stack([synth.frame_np(900 + f, iw, ih, "alpha") for f in range(n)])
    bg = timg_b200.rgba_u32(20, 30, 40)
    b = _batch(n, iw, ih, ow, oh, has_bg=1, bg=bg)
    for proto in PROTOS.values():
        outs = ctx.graphics_batch(frames, b, proto | D, False, [5, 6, 7], **_kw(proto))
        for f in range(n):
            want = ctx.compose_bg(ctx.scale(frames[f], ow, oh), bg)
            assert (png_pixels(_png(outs[f], proto, ow, oh))[0] == want).all(), (proto, f)


def _ui(seed, w, h):
    """A screenshot-like frame: flat panels, borders and rows of glyph-like marks."""
    rng = np.random.default_rng(seed)
    fb = np.zeros((h, w, 4), np.uint8)
    fb[..., 3] = 255
    fb[..., :3] = (236, 236, 240)
    for _ in range(12):
        x0, y0 = int(rng.integers(0, w - 8)), int(rng.integers(0, h - 8))
        x1, y1 = min(w, x0 + int(rng.integers(8, w // 2))), min(h, y0 + int(rng.integers(8, h // 2)))
        fb[y0:y1, x0:x1, :3] = rng.integers(0, 256, 3)
        fb[y0, x0:x1, :3] = 40
        fb[y1 - 1, x0:x1, :3] = 40
    glyphs = rng.integers(0, 2, (16, 8, 12)).astype(bool)
    for y in range(4, h - 12, 16):
        for x in range(4, w - 8, 9):
            if rng.random() < 0.6:
                fb[y:y + 12, x:x + 8][glyphs[int(rng.integers(0, 16))].T] = (20, 20, 20, 255)
    return fb


def _corpus(w, h):
    photo = synth.frame_np(31 + w, w, h, "photo")
    poster = photo.copy()
    poster[..., :3] &= 0xC0
    return {"photo": photo, "posterised": poster, "ui": _ui(w, w, h), "noise": synth.frame_np(37 + w, w, h, "noisea")}


@pytest.mark.parametrize("w,h", [(337, 190), (1280, 720)])
def test_size_is_bounded_by_stored_and_close_to_zlib_level_1(ctx, w, h):
    for kind, fb in _corpus(w, h).items():
        for rgb24 in (0, 1):
            text = ctx.graphics_batch(fb[None], _batch(1, w, h, w, h), timg_b200.ITERM2 | D, rgb24)[0]
            png = _png(text, timg_b200.ITERM2, w, h)
            assert (png_pixels(png)[0] == (fb[..., :3] if rgb24 else fb)).all(), kind
            assert len(png) <= timg_b200.lib().b200timg_png_size(w, h, rgb24), kind
            z1 = len(zlib.compress(scanlines(fb, rgb24), 1))
            if kind != "noise":
                assert len(_idat(png)) <= 1.10 * z1 + 64, (kind, rgb24, len(_idat(png)), z1)


@pytest.mark.parametrize("proto", list(PROTOS.values()))
def test_bytes_depend_on_the_frame_only(ctx, proto, monkeypatch):
    """Batch position, batch size, chunking, host / device variant and repeated calls change nothing."""
    import torch
    n, iw, ih, ow, oh = 5, 400, 300, 210, 157
    frames = np.stack([synth.frame_np(700 + f, iw, ih, "photo" if f % 2 else "alpha") for f in range(n)])
    ids = [9, 123456789, 4294967295, 10, 77]
    b = _batch(n, iw, ih, ow, oh, has_bg=1, bg=timg_b200.rgba_u32(20, 30, 40))
    kw = _kw(proto)
    outs, offs = ctx.graphics_batch(frames, b, proto | D, False, ids, with_offsets=True, **kw)
    assert ctx.graphics_batch(frames, b, proto | D, False, ids, **kw) == outs
    rev = ctx.graphics_batch(frames[::-1].copy(), b, proto | D, False, ids[::-1], **kw)
    assert rev[::-1] == outs
    for f in (0, 3):
        assert ctx.graphics_batch(frames[f:f + 1], _batch(1, iw, ih, ow, oh, has_bg=1, bg=b.bg), proto | D, False,
                                  ids[f:f + 1], **kw) == [outs[f]]
    d_out, d_offs = ctx.graphics_batch_dev(torch.tensor(frames).cuda(), b, proto | D, False, ids, **kw)
    torch.cuda.synchronize()
    assert (d_offs.cpu().numpy().astype(np.uint64) == offs).all()
    ob = d_out.cpu().numpy().tobytes()
    assert [ob[int(offs[f]):int(offs[f + 1])] for f in range(n)] == outs
    monkeypatch.setenv("B200TIMG_CHUNK_FRAMES", "2")
    assert ctx.graphics_batch(frames, b, proto | D, False, ids, **kw) == outs


def test_capacity_contract(ctx):
    """_dev: exact offsets from the device, frames past out_cap not written, nothing at or past out_cap.  Host: ENOSPC
    with offsets complete (offsets[n] = the bytes needed) and nothing written at or past out_cap."""
    import torch
    n, w, h = 4, 300, 200
    frames = np.stack([synth.frame_np(810 + f, w, h, "photo") for f in range(n)])
    ids = [1, 22, 333, 4444]
    b = _batch(n, w, h, w, h)
    want, offs = ctx.graphics_batch(frames, b, timg_b200.KITTY | D, False, ids, with_offsets=True)
    k = 2
    cap = int(offs[k]) + (int(offs[k + 1]) - int(offs[k])) // 2
    guard = 4096
    d_out = torch.full((cap + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    _, d_offs = ctx.graphics_batch_dev(torch.tensor(frames).cuda(), b, timg_b200.KITTY | D, False, ids, d_out=d_out, out_cap=cap)
    torch.cuda.synchronize()
    ob = d_out.cpu().numpy()
    assert (d_offs.cpu().numpy().astype(np.uint64) == offs).all()
    for f in range(k):
        assert ob[int(offs[f]):int(offs[f + 1])].tobytes() == want[f], f
    assert (ob[int(offs[k]):] == 0xA5).all()
    g, keep = timg_b200.graphics(timg_b200.KITTY | D, False, ids)
    for chunk in (None, "1"):
        if chunk:
            os.environ["B200TIMG_CHUNK_FRAMES"] = chunk
        try:
            out = np.full(cap + guard, 0xA5, np.uint8)
            hoffs = np.zeros(n + 1, np.uint64)
            rc = timg_b200.lib().b200timg_graphics_batch(ctx.h, C.byref(b), C.byref(g), frames.ctypes.data, out.ctypes.data,
                                                         cap, hoffs.ctypes.data)
        finally:
            os.environ.pop("B200TIMG_CHUNK_FRAMES", None)
        assert rc == timg_b200.ENOSPC
        assert (hoffs == offs).all()
        assert (out[cap:] == 0xA5).all()


def test_graphics_size_is_the_stored_bound_and_the_stored_path_is_unchanged(ctx):
    for proto in PROTOS.values():
        kw = _kw(proto)
        assert timg_b200.graphics_size(proto | D, 97, 61, True, 5, **kw) == timg_b200.graphics_size(proto, 97, 61, True, 5, **kw)
        fb = synth.frame_np(3, 97, 61, "photo")
        stored = ctx.graphics_batch(fb[None], _batch(1, 97, 61, 97, 61), proto, True, [5], **kw)[0]
        assert len(stored) == timg_b200.graphics_size(proto, 97, 61, True, 5, **kw)
        assert len(ctx.graphics_batch(fb[None], _batch(1, 97, 61, 97, 61), proto | D, True, [5], **kw)[0]) < len(stored)
    assert timg_b200.graphics_size(3 | D, 10, 10) == 0
    assert timg_b200.graphics_size(16 | timg_b200.KITTY, 10, 10) == 0


def test_rejected_arguments(ctx):
    import torch
    L = timg_b200.lib()
    src = torch.zeros(64 * 64 * 4, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(2, dtype=torch.int64, device="cuda")
    ids = np.array([5], np.uint32)
    idp = ids.ctypes.data_as(C.POINTER(C.c_uint32))
    b = _batch(1, 64, 64, 64, 64)
    for protocol in (3 | D, 16 | timg_b200.KITTY, 32 | timg_b200.ITERM2 | D, D):
        g = timg_b200.Graphics(protocol, 0, idp)
        rc = L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g), src.data_ptr(), out.data_ptr(), out.numel(), offs.data_ptr())
        assert rc == timg_b200.EINVAL and "protocol" in L.b200timg_last_error(ctx.h).decode(), protocol
    g = timg_b200.Graphics(timg_b200.KITTY | D, 0, None)
    assert L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g), src.data_ptr(), out.data_ptr(), out.numel(),
                                         offs.data_ptr()) == timg_b200.EINVAL
    g = timg_b200.Graphics(timg_b200.KITTY | D, 0, idp)
    assert L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g), src.data_ptr(), out.data_ptr(), out.numel(),
                                         offs.data_ptr()) == timg_b200.OK
    torch.cuda.synchronize()
