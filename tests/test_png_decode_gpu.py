"""PNG decode, b200timg_png_frames(_dev), on the GPU, what is particular to PNG: sized files, a stream far past its
image, the rejections of files the device does not take, and the project's own kitty PNGs.  test_decode_gpu.py holds
what PNG shares with JPEG."""
import numpy as np
import pytest

import png_cases as pc
import timg_b200
from oracle import gif as G
from test_decode_gpu import check, device

pytestmark = pytest.mark.gpu


SIZED = ["4k_rgb_photo", "4k_rgba_photo", "4k_screenshot_l9", "4k_interlaced", "solid_8192", "1x1", "1x16384",
         "16384x1"]


@pytest.mark.parametrize("k", range(len(SIZED)), ids=SIZED)
def test_sized(ctx, k):
    name, data = pc.sized_cases()[k]
    assert name == SIZED[k]
    canv, status = ctx.png_frames([data])
    if G.have_ref():
        check(name, data, canv[0], int(status[0]))
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


def test_rejections_launch_nothing(ctx):
    import torch
    good = pc.pillow(pc.photo(16, 16), "RGB")
    i = good.index(b"IDAT") - 4
    huge_chunk = good[:i] + (0x80000000).to_bytes(4, "big") + b"tEXt" + good[i:]
    assert not timg_b200.png_parse(huge_chunk)["supported"]
    d = torch.empty(16 * 16 * 4 + 16, dtype=torch.uint8, device=device())
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error, match="file 1"):
        ctx.png_frames([good, huge_chunk])
    with pytest.raises(timg_b200.B200Error, match="file 0"):
        ctx.png_frames_dev([good[:40]], d)
    with pytest.raises(timg_b200.B200Error):
        ctx.png_frames([b"GIF89a"])
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
