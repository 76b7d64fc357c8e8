"""What the JPEG and PNG decodes, b200timg_jpeg_frames(_dev) and b200timg_png_frames(_dev), share on the GPU: canvases
and statuses against the pins of tests/golden/{jpeg,png}.npz and, where oracle/gif.mk's door onto the unmodified
STBImageSource is built, against the reference byte for byte; the dev form against the host form and file order; the
launch count; the common rejections; the hand-off into the mixed batches.  test_jpeg_gpu.py and test_png_decode_gpu.py
hold what is particular to each format."""
import hashlib

import numpy as np
import pytest

import jpeg_cases as jc
import png_cases as pc
import timg_b200
from oracle import gif as G

pytestmark = pytest.mark.gpu


def _jpeg_taken():
    def supported(d):
        try:
            return timg_b200.jpeg_parse(d)["supported"]
        except timg_b200.B200Error:
            return False
    return [d for _, d in jc.small_cases() if supported(d)]


# per format: its pinned corpus, kernels per call, a 16x16 and a 200x120 file, and the files of the dev / host test
FORMATS = {
    "jpeg": dict(golden=jc.golden, launches=7, small=lambda: jc.jpeg(jc.photo(16, 16), quality=85),
                 medium=lambda: jc.jpeg(jc.photo(200, 120), quality=85, subsampling=2), dev_files=_jpeg_taken),
    "png": dict(golden=pc.golden, launches=38, small=lambda: pc.pillow(pc.photo(16, 16), "RGB"),
                medium=lambda: pc.pillow(pc.photo(200, 120), "RGB"),
                dev_files=lambda: [g[1] for g in pc.golden() if g[4]][:40]),
}
fmts = pytest.mark.parametrize("fmt", list(FORMATS))


def device():
    import torch
    return "cuda" if torch.cuda.is_available() else "cpu"     # cpu: only under the CPU kernel simulator


def ref_canvas(data):
    """The reference's canvas of a file (None where its STB source fails); skips where the door is not built."""
    if not G.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    r = G.ref_stb_gif(data)
    return None if r is None else r[0][0]


def check(name, data, canvas, status):
    """A decoded canvas and its status against the reference: -1 only where the reference decodes (its canvas is
    undefined), 0 exactly where it fails, else status 1 and every pixel equal."""
    want = ref_canvas(data)
    if status == -1:
        assert want is not None, f"{name}: status -1 reported but the reference fails"
        return
    if want is None:
        assert status == 0, f"{name}: the reference fails, status {status}"
        return
    assert status == 1, f"{name}: status {status} but the reference decodes it"
    assert canvas.shape == want.shape
    bad = np.argwhere((canvas != want).any(-1))
    assert bad.size == 0, f"{name}: {len(bad)} pixels differ, first at {bad[0].tolist()}: {canvas[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


def _frames(ctx, fmt, files):
    return getattr(ctx, f"{fmt}_frames")(files)


def _frames_dev(ctx, fmt, files, d_frames):
    return getattr(ctx, f"{fmt}_frames_dev")(files, d_frames)


@fmts
def test_golden_corpus_one_call(ctx, fmt):
    cases = [g for g in FORMATS[fmt]["golden"]() if g[4]]
    canv, status = _frames(ctx, fmt, [g[1] for g in cases])
    for (name, data, sha, want, _), c, s in zip(cases, canv, status):
        assert int(s) == want, f"{name}: status {int(s)}, pinned {want}"
        if want == 1:
            assert hashlib.sha256(c.tobytes()).hexdigest() == sha, f"{name}: canvas differs from the pin"
        if G.have_ref():
            check(name, data, c, int(s))


@fmts
def test_dev_matches_host_and_order(ctx, fmt):
    import torch
    files = FORMATS[fmt]["dev_files"]()
    canv, status = _frames(ctx, fmt, files)
    assert (status == 1).all()
    total = sum(c.size for c in canv)
    d_frames = torch.empty(total, dtype=torch.uint8, device=device())
    d_status = _frames_dev(ctx, fmt, files, d_frames)
    timg_b200.device_sync(torch)                   # the tensors are read on torch's stream, the call ran on the context's
    assert (d_frames.cpu().numpy() == np.concatenate([c.ravel() for c in canv])).all()
    assert (d_status.cpu().numpy() == status).all()
    rev, rstatus = _frames(ctx, fmt, files[::-1])
    for a, b in zip(canv, rev[::-1]):
        assert (a == b).all()
    assert (rstatus[::-1] == status).all()
    one, _ = _frames(ctx, fmt, [files[5]])
    assert (one[0] == canv[5]).all()


@fmts
def test_launch_count_does_not_grow(ctx, fmt):
    data = FORMATS[fmt]["medium"]()
    l0 = ctx.launches
    _frames(ctx, fmt, [data])
    l1 = ctx.launches
    canv, status = _frames(ctx, fmt, [data] * 64)
    l2 = ctx.launches
    assert l1 - l0 == l2 - l1 == FORMATS[fmt]["launches"]
    assert (status == 1).all() and all((c == canv[0]).all() for c in canv)


@fmts
def test_common_rejections_launch_nothing(ctx, fmt):
    import torch
    good = FORMATS[fmt]["small"]()
    d = torch.empty(16 * 16 * 4 + 16, dtype=torch.uint8, device=device())
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error):
        _frames(ctx, fmt, [])
    with pytest.raises(timg_b200.B200Error, match="aligned"):
        _frames_dev(ctx, fmt, [good], d[1:])
    assert ctx.launches == l0


@pytest.mark.parametrize("enc", ["blocks", "sixel", "kitty", "iterm2", "kitty_tmux", "kitty_deflate"])
@fmts
def test_handoff_into_mixed_batches(ctx, fmt, enc):
    """A page decoded on the device goes into the mixed encoders in place; the bytes equal the same call on the
    reference's canvases."""
    import torch
    if not G.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    page = [g for g in FORMATS[fmt]["golden"]() if g[3] == 1 and g[4]][:12]
    files = [g[1] for g in page]
    refs = [ref_canvas(d) for d in files]
    shapes = [r.shape for r in refs]
    total = sum(r.size for r in refs)
    d_dec = torch.empty(total, dtype=torch.uint8, device=device())
    st = _frames_dev(ctx, fmt, files, d_dec)
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
