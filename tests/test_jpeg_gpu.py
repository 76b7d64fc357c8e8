"""b200timg_jpeg_frames(_dev) on the GPU: canvases and statuses against the pins of tests/golden/jpeg.npz and, where
oracle/gif.mk's door onto the unmodified STBImageSource is built, against the reference byte for byte; launch count,
rejections and the hand-off into the mixed batches."""
import hashlib

import numpy as np
import pytest

import jpeg_cases as jc
import timg_b200
from oracle import gif as G

pytestmark = pytest.mark.gpu


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
        assert want is not None, f"{name}: bail reported but the reference fails"
        return
    if want is None:
        assert status == 0, f"{name}: the reference fails, status {status}"
        return
    assert status == 1, f"{name}: status {status} but the reference decodes it"
    assert canvas.shape == want.shape
    bad = np.argwhere((canvas != want).any(-1))
    assert bad.size == 0, f"{name}: {len(bad)} pixels differ, first at {bad[0].tolist()}: {canvas[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


def _taken(cases):
    return [(n, d) for n, d in cases if _supported(d)]


def _supported(d):
    try:
        return timg_b200.jpeg_parse(d)["supported"]
    except timg_b200.B200Error:
        return False


def test_golden_corpus_one_call(ctx):
    cases = [g for g in jc.golden() if g[4]]
    canv, status = ctx.jpeg_frames([g[1] for g in cases])
    for (name, data, sha, want, _), c, s in zip(cases, canv, status):
        assert int(s) == want, f"{name}: status {int(s)}, pinned {want}"
        if want == 1:
            assert hashlib.sha256(c.tobytes()).hexdigest() == sha, f"{name}: canvas differs from the pin"
        if G.have_ref():
            _check(name, data, c, int(s))


def test_review_case_and_sweep_each_alone(ctx):
    """Segments of 1, 2 and 3 mod 64 bytes: the last subsequence starts after the marker was reached."""
    for name, data, sha, want, _ in jc.golden():
        if name.startswith(("seg_", "sweep")):
            canv, status = ctx.jpeg_frames([data])
            assert int(status[0]) == want == 1
            assert hashlib.sha256(canv[0].tobytes()).hexdigest() == sha, name


@pytest.mark.parametrize("k", range(5))
def test_sized(ctx, k):
    name, data = jc.sized_cases()[k]
    canv, status = ctx.jpeg_frames([data])
    _check(name, data, canv[0], int(status[0]))


def test_dev_matches_host_and_order(ctx):
    import torch
    cases = _taken(jc.small_cases())
    files = [d for _, d in cases]
    canv, status = ctx.jpeg_frames(files)
    total = sum(c.size for c in canv)
    d_frames = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    d_status = ctx.jpeg_frames_dev(files, d_frames)
    torch.cuda.synchronize()
    assert (d_frames.cpu().numpy() == np.concatenate([c.ravel() for c in canv])).all()
    assert (d_status.cpu().numpy() == status).all()
    rev, rstatus = ctx.jpeg_frames(files[::-1])
    for a, b in zip(canv, rev[::-1]):
        assert (a == b).all()
    assert (rstatus[::-1] == status).all()
    one, _ = ctx.jpeg_frames([files[5]])
    assert (one[0] == canv[5]).all()


def test_launch_count_does_not_grow(ctx):
    data = jc.jpeg(jc.photo(200, 120), quality=85, subsampling=2)
    l0 = ctx.launches
    ctx.jpeg_frames([data])
    l1 = ctx.launches
    canv, status = ctx.jpeg_frames([data] * 64)
    l2 = ctx.launches
    assert l1 - l0 == l2 - l1 == 7
    assert (status == 1).all() and all((c == canv[0]).all() for c in canv)


def test_rejections_launch_nothing(ctx):
    import torch
    good = jc.jpeg(jc.photo(16, 16), quality=85)
    prog = jc.jpeg(jc.photo(16, 16), quality=85, progressive=True)
    d = torch.empty(16 * 16 * 4 + 16, dtype=torch.uint8, device="cuda:0")
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error, match="file 1"):
        ctx.jpeg_frames([good, prog])
    with pytest.raises(timg_b200.B200Error):
        ctx.jpeg_frames([b"\xff\xd8\xff\xd9"])
    with pytest.raises(timg_b200.B200Error):
        ctx.jpeg_frames([])
    with pytest.raises(timg_b200.B200Error, match="aligned"):
        ctx.jpeg_frames_dev([good], d[1:])
    assert ctx.launches == l0


@pytest.mark.parametrize("enc", ["blocks", "sixel", "kitty", "iterm2", "kitty_tmux", "kitty_deflate"])
def test_handoff_into_mixed_batches(ctx, enc):
    """A page decoded on the device goes into the mixed encoders in place; the bytes equal the same call on the
    reference's canvases."""
    import torch
    if not G.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    page = [g for g in jc.golden() if g[3] == 1][:12]
    files = [g[1] for g in page]
    refs = [_ref(d) for d in files]
    shapes = [r.shape for r in refs]
    total = sum(r.size for r in refs)
    d_dec = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    st = ctx.jpeg_frames_dev(files, d_dec)
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
