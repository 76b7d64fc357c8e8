"""PNG decode, b200timg_png_frames(_dev), on the GPU: canvases and statuses against the pins of tests/golden/png.npz
and, where oracle/gif.mk's door onto the unmodified STBImageSource is built, against the reference byte for byte;
sized files, launch count, rejections and the hand-off into the mixed batches."""
import hashlib

import numpy as np
import pytest

import png_cases as pc
import timg_b200
from oracle import gif as G

pytestmark = pytest.mark.gpu

LAUNCHES = 38


@pytest.fixture(scope="module")
def ctx():
    c = timg_b200.Context(0)
    yield c
    c.close()


def _ref(data):
    if not G.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    r = G.ref_stb_gif(data)
    return None if r is None else r[0][0]


def _check(name, data, canvas, status):
    want = _ref(data)
    if status == -1:
        assert want is not None, f"{name}: undefined canvas reported but the reference fails"
        return
    if want is None:
        assert status == 0, f"{name}: the reference fails, status {status}"
        return
    assert status == 1, f"{name}: status {status} but the reference decodes it"
    assert canvas.shape == want.shape
    bad = np.argwhere((canvas != want).any(-1))
    assert bad.size == 0, f"{name}: {len(bad)} pixels differ, first at {bad[0].tolist()}: {canvas[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


def test_golden_corpus_one_call(ctx):
    cases = [g for g in pc.golden() if g[4]]
    canv, status = ctx.png_frames([g[1] for g in cases])
    for (name, data, sha, want, _), c, s in zip(cases, canv, status):
        assert int(s) == want, f"{name}: status {int(s)}, pinned {want}"
        if want == 1:
            assert hashlib.sha256(c.tobytes()).hexdigest() == sha, f"{name}: canvas differs from the pin"
        if G.have_ref():
            _check(name, data, c, int(s))


SIZED = ["4k_rgb_photo", "4k_rgba_photo", "4k_screenshot_l9", "4k_interlaced", "solid_8192", "1x1", "1x16384",
         "16384x1"]


@pytest.mark.parametrize("k", range(len(SIZED)), ids=SIZED)
def test_sized(ctx, k):
    name, data = pc.sized_cases()[k]
    assert name == SIZED[k]
    canv, status = ctx.png_frames([data])
    if G.have_ref():
        _check(name, data, canv[0], int(status[0]))
    else:
        from PIL import Image
        import io
        want = np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"))
        assert int(status[0]) == 1 and (canv[0] == want).all(), name


def test_stream_far_past_the_image(ctx):
    """300 MB of output past a 64x64 image: decoded in bounded scratch, the final block reached, status 1."""
    data = pc.bomb_case()
    canv, status = ctx.png_frames([data])
    assert int(status[0]) == 1
    want = pc.photo(64, 64, 17)
    assert (canv[0][..., :3] == want).all() and (canv[0][..., 3] == 255).all()


def test_dev_matches_host_and_order(ctx):
    import torch
    cases = [g for g in pc.golden() if g[4]][:40]
    files = [g[1] for g in cases]
    canv, status = ctx.png_frames(files)
    total = sum(c.size for c in canv)
    d_frames = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    d_status = ctx.png_frames_dev(files, d_frames)
    torch.cuda.synchronize()
    ok = np.concatenate([np.full(c.size, s == 1) for c, s in zip(canv, status)])
    assert (d_frames.cpu().numpy()[ok] == np.concatenate([c.ravel() for c in canv])[ok]).all()
    assert (d_status.cpu().numpy() == status).all()
    rev, rstatus = ctx.png_frames(files[::-1])
    for a, b, s in zip(canv, rev[::-1], status):
        if s == 1:
            assert (a == b).all()
    assert (rstatus[::-1] == status).all()


def test_launch_count_does_not_grow(ctx):
    data = pc.pillow(pc.photo(200, 120), "RGB")
    l0 = ctx.launches
    ctx.png_frames([data])
    l1 = ctx.launches
    canv, status = ctx.png_frames([data] * 64)
    l2 = ctx.launches
    assert l1 - l0 == l2 - l1 == LAUNCHES
    assert (status == 1).all() and all((c == canv[0]).all() for c in canv)


def test_rejections_launch_nothing(ctx):
    import torch
    good = pc.pillow(pc.photo(16, 16), "RGB")
    i = good.index(b"IDAT") - 4
    huge_chunk = good[:i] + (0x80000000).to_bytes(4, "big") + b"tEXt" + good[i:]
    assert not timg_b200.png_parse(huge_chunk)["supported"]
    d = torch.empty(16 * 16 * 4 + 16, dtype=torch.uint8, device="cuda:0")
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error, match="file 1"):
        ctx.png_frames([good, huge_chunk])
    with pytest.raises(timg_b200.B200Error, match="file 0"):
        ctx.png_frames_dev([good[:40]], d)
    with pytest.raises(timg_b200.B200Error):
        ctx.png_frames([b"GIF89a"])
    with pytest.raises(timg_b200.B200Error):
        ctx.png_frames([])
    with pytest.raises(timg_b200.B200Error, match="aligned"):
        ctx.png_frames_dev([good], d[1:])
    assert ctx.launches == l0


def test_own_kitty_pngs_decode_to_their_frame(ctx):
    """The PNGs the kitty / iTerm2 canvases send (stored blocks, RGBA and RGB) decode to the frame they encoded."""
    fb = pc.photo(45, 31, 21, 4)
    for rgb24 in (False, True):
        data, _ = ctx.png_encode(fb, rgb24=rgb24, want_base64=False)
        canv, status = ctx.png_frames([data])
        assert int(status[0]) == 1
        want = fb.copy()
        if rgb24:
            want[..., 3] = 255
        assert (canv[0] == want).all()


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
@pytest.mark.parametrize("rgb24", [False, True], ids=["rgba", "rgb24"])
def test_own_kitty_batch_pngs_decode_to_their_frame(ctx, deflate, rgb24):
    """The PNGs inside a kitty mixed batch, stored blocks or deflate.cu's Huffman blocks (B200TIMG_DEFLATE), decode to
    the scaled frame they carry."""
    import base64
    from test_graphics_oracle import kitty_payload, png_pixels
    imgs = [pc.photo(90, 60, 31, 4), pc.photo(33, 17, 32, 4), pc.screenshot(200, 96, 33)]
    imgs[2] = np.concatenate([imgs[2], np.full(imgs[2].shape[:2] + (1,), 255, np.uint8)], -1)
    outs = [(45, 30), (33, 17), (200, 96)]
    texts = ctx.graphics_mixed(imgs, outs, timg_b200.KITTY, rgb24=rgb24, ids=[1, 2, 3], deflate=deflate)
    pngs = [base64.b64decode(kitty_payload(t)) for t in texts]
    canv, status = ctx.png_frames(pngs)
    assert (status == 1).all()
    for png, c in zip(pngs, canv):
        want = png_pixels(png)[0]
        assert c.shape[:2] == want.shape[:2]
        assert (c[..., :want.shape[2]] == want).all()
        if want.shape[2] == 3:
            assert (c[..., 3] == 255).all()


@pytest.mark.parametrize("enc", ["blocks", "sixel", "kitty", "iterm2", "kitty_tmux", "kitty_deflate"])
def test_handoff_into_mixed_batches(ctx, enc):
    """A page decoded on the device goes into the mixed encoders in place; the bytes equal the same call on the
    reference's canvases."""
    import torch
    if not G.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    page = [g for g in pc.golden() if g[3] == 1 and g[4]][:12]
    files = [g[1] for g in page]
    refs = [_ref(d) for d in files]
    shapes = [r.shape for r in refs]
    total = sum(r.size for r in refs)
    d_dec = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    st = ctx.png_frames_dev(files, d_dec)
    timg_b200.device_sync(torch)                   # the status is read on torch's stream, the call ran on the context's
    flat, offs = timg_b200.pack_mixed(refs)
    assert (st.cpu().numpy() == 1).all()
    d_ref = timg_b200._device_tensor(torch, flat)
    outs = [(max(1, s[1] // 2), max(1, s[0] // 3)) for s in shapes]
    b, keep = timg_b200.mixed_batch(shapes, outs, offs, [0] * len(page), timg_b200.UPPER if enc == "blocks" else 0)

    def run(d_src):
        if enc == "blocks":
            d_out, d_offs = ctx.blocks_mixed_dev(d_src, b)
        elif enc == "sixel":
            d_out, d_offs = ctx.sixel_mixed_dev(d_src, b)
        else:
            proto = {"kitty": timg_b200.KITTY, "iterm2": timg_b200.ITERM2, "kitty_tmux": timg_b200.KITTY_TMUX,
                     "kitty_deflate": timg_b200.KITTY | timg_b200.DEFLATE}[enc]
            g, ids = timg_b200.graphics(proto, ids=list(range(1, len(page) + 1)), cell=(9, 18))
            d_out, d_offs = ctx.graphics_mixed_dev(d_src, b, g)
        timg_b200.device_sync(torch)
        o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
        return [data[o[f]:o[f + 1]].tobytes() for f in range(len(page))]

    assert run(d_dec) == run(d_ref)
