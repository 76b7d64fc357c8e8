"""The alternative code paths of round 2 against each other and the oracle: TMA-staged vs LDG-staged scaler windows, the
sixel emitters (emit5, emit2), the 16-byte identity copy with the compose fused, the staged first pass of the
two-pass scaler.  The knobs are the library's own environment switches (read at call time)."""
import numpy as np
import pytest

import oracle
import timg_b200
from timg_b200 import synth

pytestmark = pytest.mark.gpu


def _batch(n, iw, ih, ow, oh, **kw):
    d = dict(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=timg_b200.rgba_u32(0, 0, 0),
             pattern=0, pattern_w=0, pattern_h=0, flags=0, x_indent_cells=0, animation=0)
    d.update(kw)
    return timg_b200.Batch(**d)


@pytest.mark.parametrize("kind,iw,ih,ow,oh", [("photo", 3840, 2160, 2700, 1519), ("alpha", 1280, 720, 900, 506),
                                               ("photo", 1000, 600, 1300, 780), ("noise", 644, 480, 450, 335)])
def test_tma_staged_window_equals_ldg_staged(ctx, monkeypatch, kind, iw, ih, ow, oh):
    """The v3 scaler's window comes in through cp.async.bulk.tensor (default) or plain 16-byte loads (B200TIMG_TMA=0):
    same pixels, within the FAST mode's 1 LSB of the oracle."""
    src = synth.frame_np(31 + iw, iw, ih, kind)
    fast_tma = ctx.scale(src, ow, oh, fast=True)
    monkeypatch.setenv("B200TIMG_TMA", "0")
    fast_ldg = ctx.scale(src, ow, oh, fast=True)
    assert (fast_tma == fast_ldg).all()
    d = np.abs(fast_tma.astype(int) - oracle.stb_resize(src, ow, oh).astype(int))
    assert d.max() <= 1                                        # the FAST mode's stated tolerance


@pytest.mark.parametrize("kind,w,h", [("photo", 675, 384), ("noise", 337, 192), ("photo", 2700, 36), ("alpha", 160, 120),
                                      ("photo", 3500, 12)])      # > 3072 px: column entries are recomputed, not stashed
def test_sixel_emitters_agree(ctx, monkeypatch, kind, w, h):
    """emit5 writes oracle.sixel_stream's bytes for the palette and index plane the device computed; the single-pass
    emit2 (other '$' placement) the same picture."""
    fb = synth.frame_np(900 + w, w, h, kind)
    fb[..., 3] = 255
    out = {}
    for mode in ("5", "2"):
        monkeypatch.setenv("B200TIMG_EMIT", mode)
        out[mode] = ctx.sixel_encode(fb)
    pal, _, idx = ctx.sixel_debug(w, h)
    assert out["5"] == oracle.sixel_stream(pal, idx)
    ref, _ = oracle.sixel_decode(out["5"])
    got, _ = oracle.sixel_decode(out["2"])
    assert (ref == got).all()


def test_sixel_emit5_slot_overflow_falls_back(ctx, monkeypatch):
    """A noise band gives a thread more bytes than its shared-memory slot holds: the byte-wise write walk takes over,
    same bytes as oracle.sixel_stream."""
    fb = synth.frame_np(5, 1300, 36, "noise")
    monkeypatch.setenv("B200TIMG_EMIT", "5")
    out = ctx.sixel_encode(fb)
    pal, _, idx = ctx.sixel_debug(1300, 36)
    assert out == oracle.sixel_stream(pal, idx)


def test_unscaled_frames_copy_with_compose(ctx):
    """Frames shown at their own size (the C5 shape) take the 16-byte copy with AlphaComposeBackground fused."""
    n, w, h = 3, 128, 64
    frames = np.stack([synth.frame_np(40 + i, w, h, "alpha") for i in range(n)])
    bg = timg_b200.rgba_u32(30, 60, 90)
    outs = ctx.blocks_batch(frames, _batch(n, w, h, w, h, bg=bg))
    for f in range(n):
        assert (ctx.scale(frames[f], w, h) == frames[f]).all()
        assert outs[f] == oracle.BlockCanvas(False).send(oracle.compose_bg(frames[f], bg))


@pytest.mark.parametrize("kind,iw,ih,ow,oh", [("alpha", 3840, 2160, 337, 190), ("noisea", 1000, 300, 37, 190),
                                               ("photo", 1920, 360, 170, 100), ("alpha", 640, 480, 67, 50),
                                               ("noisea", 517, 211, 33, 41)])
def test_two_pass_first_pass_variants_agree(ctx, monkeypatch, kind, iw, ih, ow, oh):
    """The horizontal first pass of the two-pass scaler has three thread mappings (staged through shared memory for mostly
    full 32-column tiles, flat (row, column) pairs for few output columns, the plain tiled one): same bits, the oracle's."""
    src = synth.frame_np(77, iw, ih, kind)
    if kind == "noisea":
        src[::3, ::5, 3] = 0                                   # holes: the un-weighted (plain) passes run too
    default = ctx.scale(src, ow, oh)
    monkeypatch.setenv("B200TIMG_NO_H1S", "1")
    no_staged = ctx.scale(src, ow, oh)
    monkeypatch.setenv("B200TIMG_NO_H1F", "1")
    plain = ctx.scale(src, ow, oh)
    assert (default == plain).all() and (no_staged == plain).all()
    assert (plain == oracle.stb_resize(src, ow, oh)).all()
