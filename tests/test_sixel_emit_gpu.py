"""emit5 (the default emitter up to 4095 px) writes the bytes of oracle.sixel_stream, the CPU statement of the device's
sixel stream, for every input: the shapes of the other emitter tests, bands whose bytes overflow the staging area, the
smallest frames, a solid band, all 256 colours, the widest frames it serves and batches through every caller of the
front."""
import ctypes

import numpy as np
import pytest

import oracle
import timg_b200
from timg_b200 import synth

pytestmark = pytest.mark.gpu


def _stream_of_last_encode(ctx, fb):
    """oracle.sixel_stream of the palette and index plane the device computed for fb (ctx.sixel_debug)."""
    h, w = fb.shape[:2]
    pal, _, idx = ctx.sixel_debug(w, h)
    return oracle.sixel_stream(pal, idx)


def _cpu_stream(fb):
    """oracle.sixel_stream of the CPU encoder's palette and index plane (the device computes the same: test_sixel_shapes_gpu)."""
    _, det = oracle.sixel_encode(fb, True, mode=1)
    return oracle.sixel_stream(det["palette"], det["index"])


def _opaque(seed, w, h, kind):
    fb = synth.frame_np(seed, w, h, kind)
    fb[..., 3] = 255
    return fb


def _batch(n, iw, ih, ow, oh):
    return timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1,
                           bg=timg_b200.rgba_u32(0, 0, 0), pattern=0, pattern_w=0, pattern_h=0, flags=0, x_indent_cells=0,
                           animation=0)


@pytest.mark.parametrize("kind,w,h", [("photo", 675, 384), ("noise", 337, 192), ("photo", 2700, 36), ("alpha", 160, 120),
                                      ("photo", 3500, 12),     # > 3072 px: column entries are recomputed, not stashed
                                      ("noise", 2700, 24),     # C2's width, every band far past the staging area
                                      ("photo", 1, 6), ("noise", 2, 12), ("noise", 64, 6),
                                      ("photo", 4095, 12), ("noise", 4095, 12), ("photo", 3073, 18), ("noise", 3073, 6)])
def test_emit5_equals_stream(ctx, monkeypatch, kind, w, h):
    fb = _opaque(900 + w, w, h, kind)
    monkeypatch.setenv("B200TIMG_EMIT", "5")
    assert ctx.sixel_encode(fb) == _stream_of_last_encode(ctx, fb)


@pytest.mark.parametrize("w", [64, 4095])
def test_emit5_is_the_default_and_writes_the_stream(ctx, monkeypatch, w):
    """Without B200TIMG_EMIT the sixel path launches emit5 (its own profile name) and writes the stream's bytes."""
    fb = _opaque(3, w, 6, "noise")
    monkeypatch.delenv("B200TIMG_EMIT", raising=False)
    ctx.profile(True)
    try:
        out = ctx.sixel_encode(fb)
        kernels = ctx.profile_report()
    finally:
        ctx.profile(False)
    assert "sixel_emit5_kernel" in kernels and "sixel_emit2_kernel" not in kernels
    assert out == _stream_of_last_encode(ctx, fb)


def test_emit5_solid_band_writes_the_stream(ctx):
    """One colour over a 2700-px band: one run of the whole width, '!2700~'."""
    fb = np.zeros((6, 2700, 4), np.uint8)
    fb[...] = (40, 90, 200, 255)
    out = ctx.sixel_encode(fb)
    assert b"!2700~" in out
    assert out == _stream_of_last_encode(ctx, fb)


def test_emit5_all_256_colours_write_the_stream(ctx):
    """256 distinct colours (no dithering, palette index = colour): colour numbers up to '#255', every run length."""
    w, h = 1536, 24
    x = np.arange(w)[None, :].repeat(h, 0)
    y = np.arange(h)[:, None].repeat(w, 1)
    c = ((x // 3 + y * 7) % 256).astype(np.uint8)
    rgb = np.stack([(c & 7) * 32 + 16, ((c >> 3) & 7) * 32 + 16, (c >> 6) * 64 + 32], -1).astype(np.uint8)
    fb = np.concatenate([rgb, np.full((h, w, 1), 255, np.uint8)], -1)
    out = ctx.sixel_encode(fb)
    assert b"#255" in out
    assert out == _stream_of_last_encode(ctx, fb)


@pytest.mark.parametrize("parts", [None, "4"])
def test_emit5_batches_equal_stream(ctx, monkeypatch, parts):
    """C2's geometry (4K -> 2700x1519, padded to 1524) through the device-resident batch; with B200TIMG_PARTS=4 the
    front runs as four slices on their own streams (the C5 form), each emitting at its frame offset.  Every frame's
    bytes are the stream of the framebuffer the batch encoded, computed on the CPU."""
    torch = pytest.importorskip("torch")
    if parts:
        monkeypatch.setenv("B200TIMG_PARTS", parts)
    monkeypatch.delenv("B200TIMG_EMIT", raising=False)
    n, iw, ih = 4, 3840, 2160
    _, ow, oh = timg_b200.calc_fit(iw, ih, 2700, 1800, 9, 18, 1.0)
    frames = np.stack([synth.frame_np(11 + i, iw, ih, "photo") for i in range(n)])
    d = torch.from_numpy(frames.reshape(n, -1)).cuda()
    cap = n * int(timg_b200.lib().b200timg_sixel_bound(ow, oh + 5))
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    ctx._chk(timg_b200.lib().b200timg_sixel_batch_dev(ctx.h, ctypes.byref(_batch(n, iw, ih, ow, oh)), d.data_ptr(),
                                                      out.data_ptr(), cap, offs.data_ptr()))
    torch.cuda.synchronize()
    o, ob = offs.cpu().numpy(), out.cpu().numpy()
    got = [ob[int(o[i]):int(o[i + 1])].tobytes() for i in range(n)]
    for f in range(n):
        assert got[f] == _cpu_stream(_padded_frame(frames[f], ow, oh)), f


def _padded_frame(src, ow, oh):
    """What the sixel batch encodes for one source frame (CPU): scale, compose on the background, pad to a multiple of 6
    rows, compose the pad strip only."""
    bg = oracle.rgba_u32(0, 0, 0)
    padded = np.zeros(((oh + 5) // 6 * 6, ow, 4), np.uint8)
    padded[:oh] = oracle.compose_bg(oracle.stb_resize(src, ow, oh), bg)
    return oracle.compose_bg(padded, bg, start_row=oh)


def test_emit5_host_pipeline_chunks_write_the_stream(ctx, monkeypatch):
    """The host-buffer batch in chunks of two frames: every frame's bytes are the stream of the framebuffer it encoded."""
    monkeypatch.setenv("B200TIMG_CHUNK_FRAMES", "2")
    monkeypatch.delenv("B200TIMG_EMIT", raising=False)
    n, iw, ih = 5, 640, 360
    frames = np.stack([synth.frame_np(60 + i, iw, ih, "photo") for i in range(n)])
    _, ow, oh = timg_b200.calc_fit(iw, ih, 2700, 1800, 9, 18, 1.0)
    outs = ctx.sixel_batch(frames, _batch(n, iw, ih, ow, oh))
    for f in range(n):
        assert outs[f] == _cpu_stream(_padded_frame(frames[f], ow, oh)), f
