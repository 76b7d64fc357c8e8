"""The BMP / TGA / PNM decode on the GPU, b200timg_raster_frames(_dev): canvases and statuses against the pins of
tests/golden/raster.npz and, where oracle/gif.mk's door onto the unmodified STBImageSource is built, against the
reference byte for byte; the RLE tile cases alone and behind front files; interleaved pages; the dev form against the
host form and file order; the launch count; rejections; sized files; the status -1 cases; the hand-off into the mixed
batches."""
import hashlib

import numpy as np
import pytest

import png_cases as pc
import raster_cases as rc
import timg_b200
from oracle import raster as R

pytestmark = pytest.mark.gpu


def device():
    import torch
    return "cuda" if torch.cuda.is_available() else "cpu"     # cpu: only under the CPU kernel simulator


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def decoded():
    return [g for g in rc.golden() if g[2] == 1]


def check(cases, canv, status, label=""):
    for (name, data, _, want_sha, want_st, _, _), c, s in zip(cases, canv, status):
        assert int(s) == want_st, f"{name}{label}: status {int(s)}, pinned {want_st}"
        if want_st == 1:
            assert sha(c) == want_sha, f"{name}{label}: canvas differs from the pin"


def test_golden_corpus_one_call(ctx):
    cases = decoded()
    canv, status = ctx.raster_frames([g[1] for g in cases])
    check(cases, canv, status)
    if R.have_ref():
        for (name, data, *_), c, s in zip(cases, canv, status):
            if int(s) == 1:
                assert (c == R.ref_stb(data)).all(), f"{name}: canvas differs from the reference"


@pytest.mark.parametrize("fronts", [0, 1, 2, 5])
def test_tile_cases_behind_fronts(ctx, fronts):
    """Every RLE tile case and every status -1 case, each behind `fronts` files of the three formats, so their tiles,
    chunks and super-chunks sit at call-global positions that differ with the files in front."""
    names = {n for n, _, _ in rc.tile_cases()} | {"bmp8_index_past_psize", "bmp1_psize_1", "tga10_cut_stream"}
    cases = [g for g in decoded() if g[0] in names]
    front = rc.front_files(fronts)
    files = []
    for g in cases:
        files += front + [g[1]]
    canv, status = ctx.raster_frames(files)
    alone = ctx.raster_frames(front)[0] if fronts else []
    for i, g in enumerate(cases):
        k = i * (fronts + 1) + fronts
        check([g], [canv[k]], [status[k]], f" behind {fronts} files")
        for j in range(fronts):
            assert int(status[k - fronts + j]) == 1 and (canv[k - fronts + j] == alone[j]).all()


def test_interleaved_pages(ctx):
    cases = decoded()
    bmp = [g for g in cases if g[0].startswith("bmp")]
    tga = [g for g in cases if g[0].startswith(("tga", "rle"))]
    pnm = [g for g in cases if g[0].startswith("p")]
    page = [x for trio in zip(tga, pnm * 5, bmp) for x in trio]
    canv, status = ctx.raster_frames([g[1] for g in page])
    check(page, canv, status, " (interleaved)")


def test_dev_matches_host_and_order(ctx):
    import torch
    files = [g[1] for g in decoded()]
    canv, status = ctx.raster_frames(files)
    total = sum(c.size for c in canv)
    d_frames = torch.empty(total, dtype=torch.uint8, device=device())
    d_status = ctx.raster_frames_dev(files, d_frames)
    timg_b200.device_sync(torch)
    assert (d_status.cpu().numpy() == status).all()
    got = d_frames.cpu().numpy()
    o = 0
    for c, s in zip(canv, status):
        if s == 1:
            assert (got[o:o + c.size] == c.ravel()).all()
        o += c.size
    rev, rstatus = ctx.raster_frames(files[::-1])
    for a, b, s in zip(canv, rev[::-1], status):
        if s == 1:
            assert (a == b).all()
    assert (rstatus[::-1] == status).all()


def test_launch_count_does_not_grow(ctx):
    files = [d for n, d in rc.corpus()]
    for call in ([files[0]], files, [d for _, d, _ in rc.tile_cases()][:3], [rc.front_files(3)[2]] * 64):
        l0 = ctx.launches
        ctx.raster_frames(call)
        assert ctx.launches - l0 == rc.LAUNCHES


def test_rejections_launch_nothing(ctx):
    import torch
    good = R.pnm(np.zeros((4, 4), np.uint8))
    d = torch.empty(16 * 4 + 16, dtype=torch.uint8, device=device())
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error):
        ctx.raster_frames([])
    with pytest.raises(timg_b200.B200Error, match="aligned"):
        ctx.raster_frames_dev([good], d[1:])
    for name, data, want in rc.rejections():
        if want != "ok":
            with pytest.raises(timg_b200.B200Error, match="file 1"):
                ctx.raster_frames_dev([good, data], d)
    assert ctx.launches == l0


def sized():
    """(name, file, image): the writers round-trip their input, so the image is the canvas."""
    img = pc.photo(3840, 2160, 1)
    a = rc.rgba(img)
    yield "bmp24_4k", R.bmp(img, 24), a
    yield "tga2_24_4k", rc.tga_file(img, rle=False), a
    yield "tga10_24_4k", rc.tga_file(img, rle=True), a
    yield "pnm_p6_4k", R.pnm(img), a
    flat = np.repeat(np.repeat(pc.photo(64, 64, 2), 128, 0), 128, 1)
    yield "tga10_24_8192", rc.tga_file(flat, rle=True), rc.rgba(flat)
    row = pc.photo(16384, 1, 3)
    yield "bmp24_row_16384x1", R.bmp(row, 24), rc.rgba(row)
    yield "tga10_24_col_1x16384", rc.tga_file(pc.photo(1, 16384, 4), rle=True), rc.rgba(pc.photo(1, 16384, 4))
    yield "pnm_col_1x16384", R.pnm(pc.photo(1, 16384, 5)), rc.rgba(pc.photo(1, 16384, 5))


@pytest.mark.parametrize("name", [n for n, _, _ in sized()])
def test_sized(ctx, name):
    data, img = next((d, i) for n, d, i in sized() if n == name)
    canv, status = ctx.raster_frames([data])
    assert int(status[0]) == 1
    assert canv[0].shape == img.shape
    bad = np.argwhere((canv[0] != img).any(-1))
    assert bad.size == 0, f"{name}: {len(bad)} pixels differ from the written image, first at {bad[0].tolist()}"
    if R.have_ref():
        assert (canv[0] == R.ref_stb(data)).all()


def test_status_minus_one_cases(ctx):
    cases = [g for g in rc.golden() if g[4] == -1]
    assert len(cases) >= 4
    _, status = ctx.raster_frames([g[1] for g in cases])
    assert (status == -1).all()


def test_scaled_frames(ctx):
    o = rc.FRAME_OPTS
    cases = [g for g in rc.golden() if g[5]]
    canv, status = ctx.raster_frames([g[1] for g in cases])
    for (name, _, _, _, _, frame_sha, out), c in zip(cases, canv):
        (got,) = ctx.scale_mixed([c], [out], has_bg=True, bg=o["bg"], pattern=o["pattern"],
                                 pattern_w=o["pattern_size"] * o["cell"][0], pattern_h=o["pattern_size"] * o["cell"][1] // 2)
        assert sha(got) == frame_sha, f"{name}: frame differs from the reference's"


@pytest.mark.parametrize("enc", ["blocks", "sixel", "kitty", "iterm2", "kitty_tmux", "kitty_deflate"])
def test_handoff_into_mixed_batches(ctx, enc):
    """A page decoded on the device goes into the mixed encoders in place; the bytes equal the same call on the
    reference's canvases."""
    import torch
    if not R.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    names = ("bmp24_h40", "bmp32_alpha", "bmp8_w33", "bmp16_565_bitfields", "tga10_24", "tga1_8_pal24", "tga2_32",
             "tga3_16_grey_alpha", "p6_8", "p5_16", "p6_comments", "bmp4_h124_gap")
    page = [g for g in decoded() if g[0] in names]
    files = [g[1] for g in page]
    refs = [R.ref_stb(d) for d in files]
    shapes = [r.shape for r in refs]
    d_dec = torch.empty(sum(r.size for r in refs), dtype=torch.uint8, device=device())
    st = ctx.raster_frames_dev(files, d_dec)
    timg_b200.device_sync(torch)
    assert (st.cpu().numpy() == 1).all()
    flat, offs = timg_b200.pack_mixed(refs)
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
