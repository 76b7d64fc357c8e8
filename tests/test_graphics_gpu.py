"""Kitty / iTerm2 batches (b200timg_graphics_batch[_dev]) on the GPU: byte identity with what the reference's own
canvases write around a stored-block PNG (tests/golden/graphics.npz), scale + compose inside the batch, the host and
device-resident variants, the output capacity contract and the rejected arguments."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import timg_b200
from timg_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_cases as gcases  # noqa: E402
from test_graphics_oracle import GOLD, PROTOCOLS, iterm2_payload, kitty_payload, png_pixels  # noqa: E402

pytestmark = pytest.mark.gpu


def _batch(n, iw, ih, ow, oh, **kw):
    d = dict(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=0, bg=0, pattern=0, pattern_w=0,
             pattern_h=0, flags=0, x_indent_cells=0, animation=0)
    d.update(kw)
    return timg_b200.Batch(**d)


def _golden(key):
    """(bytes or None, sha or None, id)"""
    full = GOLD[key].tobytes() if key in GOLD else None
    sha = GOLD[key + "/sha"].tobytes() if key + "/sha" in GOLD else None
    return full, sha, int(GOLD[key + "/id"][0])


def _same(got, full, sha):
    return got == full if full is not None else gcases.sha(got) == sha


def _decode(text, proto, w, h):
    import base64
    return png_pixels(base64.b64decode(kitty_payload(text) if proto == gcases.KITTY else iterm2_payload(text, w, h)))[0]


@pytest.mark.parametrize("pname", ["kitty", "iterm2"])
def test_single_frames_equal_the_reference_canvas_bytes(ctx, pname):
    """Unscaled (the scaler copies), not composed: every frame case, both colour types."""
    proto = PROTOCOLS[pname]
    for name, fb, rgb24 in gcases.graphics_frame_cases():
        full, sha, id_ = _golden(f"{pname}/{name}")
        h, w = fb.shape[:2]
        got = ctx.graphics_batch(fb[None], _batch(1, w, h, w, h), proto, rgb24, [id_])[0]
        assert _same(got, full, sha), name


@pytest.mark.parametrize("new_id", [0, 7, 12345, 4294967295])
def test_kitty_ids_of_any_digit_count(ctx, new_id):
    """i= is the only part of a frame that depends on the id: a batch of the same frame under several ids equals the
    golden with its i= replaced (1 to 10 digits, 0xffffffff included)."""
    for name in ("2x3_rgb1", "chunk1eq_rgb1", "chunk1p1_rgb1", "blocks_rgb0"):
        fb = dict((n, f) for n, f, _ in gcases.graphics_frame_cases())[name]
        rgb24 = int(name[-1])
        full, _, id_ = _golden(f"kitty/{name}")
        h, w = fb.shape[:2]
        outs, offs = ctx.graphics_batch(np.stack([fb, fb, fb]), _batch(3, w, h, w, h), gcases.KITTY, rgb24,
                                        [new_id, id_, new_id], with_offsets=True)
        want = full.replace(b"i=%d," % id_, b"i=%d," % new_id, 1)
        assert outs == [want, full, want], name
        assert int(offs[3]) == 2 * len(want) + len(full)


def test_checkerboard_scale_and_compose_in_the_batch(ctx):
    src, ow, oh, kw = gcases.graphics_checker_case()
    ih, iw = src.shape[:2]
    b = _batch(2, iw, ih, ow, oh, has_bg=1, bg=kw["bg"], pattern=kw["pattern"], pattern_w=kw["pw"], pattern_h=kw["ph"])
    for pname, rgb24 in (("kitty", 1), ("iterm2", 0)):
        full, _, id_ = _golden(f"{pname}/checker_rgb{rgb24}")
        outs = ctx.graphics_batch(np.stack([src, src]), b, PROTOCOLS[pname], rgb24, [id_, id_])
        assert outs == [full, full], pname


def test_c4_geometry_batch_equals_reference_scale_compose_canvas(ctx):
    """C4: 4K frames -> 337x190, composed onto black, kitty with rgb24 (digests of the reference's bytes)."""
    n = gcases.C4_GRAPHICS_FRAMES
    frames = gcases.c4_frames(n)
    ids = [_golden(f"kitty/c4_rgb1/{f}")[2] for f in range(n)]
    outs = ctx.graphics_batch(frames, _batch(n, 3840, 2160, 337, 190, has_bg=1, bg=timg_b200.rgba_u32(0, 0, 0)),
                              gcases.KITTY, True, ids)
    for f in range(n):
        _, sha, _ = _golden(f"kitty/c4_rgb1/{f}")
        assert len(outs[f]) == int(GOLD[f"kitty/c4_rgb1/{f}/len"][0]) and gcases.sha(outs[f]) == sha, f


def test_i420_source_decodes_to_the_yuv_scaler_output(ctx):
    import oracle
    n, iw, ih, ow, oh = 3, 320, 240, 161, 97
    yuv = np.stack([oracle.rgba_to_i420_np(synth.frame_np(610 + f, iw, ih, "photo")) for f in range(n)])
    for proto in (gcases.KITTY, gcases.ITERM2):
        outs = ctx.graphics_batch(yuv, _batch(n, iw, ih, ow, oh, src_fmt=timg_b200.FMT_I420), proto, False, [1, 2, 3])
        for f in range(n):
            want = ctx.yuv_scale(yuv[f], iw, ih, ow, oh)
            assert (_decode(outs[f], proto, ow, oh) == want).all(), f


def test_fast_scale_within_one_lsb_of_the_exact_scaler(ctx):
    n, iw, ih, ow, oh = 3, 640, 480, 251, 187
    frames = np.stack([synth.frame_np(620 + f, iw, ih, "photo") for f in range(n)])
    outs = ctx.graphics_batch(frames, _batch(n, iw, ih, ow, oh, flags=timg_b200.FAST_SCALE), gcases.ITERM2, True)
    for f in range(n):
        got = _decode(outs[f], gcases.ITERM2, ow, oh).astype(int)
        want = ctx.scale(frames[f], ow, oh)[..., :3].astype(int)
        assert np.abs(got - want).max() <= 1, f


@pytest.mark.parametrize("chunk", [None, "1"])
@pytest.mark.parametrize("proto", [gcases.KITTY, gcases.ITERM2])
def test_host_and_device_variants_give_identical_bytes_and_offsets(ctx, chunk, proto, monkeypatch):
    import torch
    if chunk:
        monkeypatch.setenv("B200TIMG_CHUNK_FRAMES", chunk)
    n, iw, ih, ow, oh = 5, 400, 300, 210, 157
    frames = np.stack([synth.frame_np(700 + f, iw, ih, "alpha") for f in range(n)])
    ids = [9, 123456789, 4294967295, 10, 77]
    b = _batch(n, iw, ih, ow, oh, has_bg=1, bg=timg_b200.rgba_u32(20, 30, 40))
    outs, offs = ctx.graphics_batch(frames, b, proto, False, ids, with_offsets=True)
    d_out, d_offs = ctx.graphics_batch_dev(torch.tensor(frames).cuda(), b, proto, False, ids)
    torch.cuda.synchronize()
    assert (d_offs.cpu().numpy().astype(np.uint64) == offs).all()
    ob = d_out.cpu().numpy().tobytes()
    assert [ob[int(offs[f]):int(offs[f + 1])] for f in range(n)] == outs
    for f in range(n):
        fb = ctx.compose_bg(ctx.scale(frames[f], ow, oh), b.bg)
        assert (_decode(outs[f], proto, ow, oh) == fb).all(), f


def test_capacity_contract(ctx):
    """out_cap ending inside frame k: earlier frames intact, nothing written at or past out_cap, offsets complete;
    the host variant reports ENOSPC before running anything and leaves offsets[n] = the bytes needed."""
    import torch
    n, w, h = 4, 90, 40
    frames = np.stack([synth.frame_np(800 + f, w, h, "noisea") for f in range(n)])
    ids = [1, 22, 333, 4444]
    b = _batch(n, w, h, w, h)
    want, offs = ctx.graphics_batch(frames, b, gcases.KITTY, False, ids, with_offsets=True)
    k = 2
    cap = int(offs[k]) + (int(offs[k + 1]) - int(offs[k])) // 2
    guard = 4096
    d_out = torch.full((cap + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    d_out2, d_offs = ctx.graphics_batch_dev(torch.tensor(frames).cuda(), b, gcases.KITTY, False, ids, d_out=d_out, out_cap=cap)
    torch.cuda.synchronize()
    ob = d_out.cpu().numpy()
    assert (d_offs.cpu().numpy().astype(np.uint64) == offs).all()
    for f in range(k):
        assert ob[int(offs[f]):int(offs[f + 1])].tobytes() == want[f], f
    assert (ob[cap:] == 0xA5).all()
    assert (ob[int(offs[k]):cap] == 0xA5).all()                       # frame k is not written at all
    g, keep = timg_b200.graphics(gcases.KITTY, False, ids)
    out = np.full(cap + guard, 0xA5, np.uint8)
    hoffs = np.zeros(n + 1, np.uint64)
    rc = timg_b200.lib().b200timg_graphics_batch(ctx.h, C.byref(b), C.byref(g), frames.ctypes.data, out.ctypes.data, cap,
                                                 hoffs.ctypes.data)
    assert rc == timg_b200.ENOSPC
    assert hoffs[n] == offs[n] and (hoffs == offs).all()
    assert (out == 0xA5).all()


def test_rejected_arguments(ctx):
    import torch
    L = timg_b200.lib()
    src = torch.zeros(64 * 64 * 4, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(2, dtype=torch.int64, device="cuda")
    ids = np.array([5], np.uint32)

    def call(b, g):
        return L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g) if g is not None else None, src.data_ptr(),
                                             out.data_ptr(), out.numel(), offs.data_ptr())
    ok = timg_b200.Graphics(gcases.KITTY, 0, ids.ctypes.data_as(C.POINTER(C.c_uint32)))
    cases_ = [("animation", _batch(1, 64, 64, 64, 64, animation=1), ok, "animation"),
              ("protocol", _batch(1, 64, 64, 64, 64), timg_b200.Graphics(3, 0, None), "protocol"),
              ("ids", _batch(1, 64, 64, 64, 64), timg_b200.Graphics(gcases.KITTY, 0, None), "ids"),
              ("idat", _batch(1, 64, 64, 30000, 30000), ok, "IDAT"),
              ("null", _batch(1, 64, 64, 64, 64), None, "null")]
    for what, b, g, word in cases_:
        rc = call(b, g)
        msg = L.b200timg_last_error(ctx.h).decode()
        assert rc == timg_b200.EINVAL and word in msg, (what, rc, msg)
    assert call(_batch(1, 64, 64, 64, 64), ok) == timg_b200.OK
    torch.cuda.synchronize()
