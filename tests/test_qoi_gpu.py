"""The QOI decode on the GPU, b200timg_qoi_frames(_dev): canvases and statuses against the pins of tests/golden/qoi.npz
and, where oracle/qoi.mk's door onto the unmodified QOIImageSource is built, against the reference byte for byte; the
split-point cases of qoi_cases.split_cases() alone and behind front files; the dev form against the host form and file
order; the launch count; rejections; sized files; the hand-off into the mixed batches."""
import hashlib

import numpy as np
import pytest

import png_cases as pc
import qoi_cases as qc
import timg_b200
from oracle import qoi as Q

pytestmark = pytest.mark.gpu


def device():
    import torch
    return "cuda" if torch.cuda.is_available() else "cpu"     # cpu: only under the CPU kernel simulator


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def decoded():
    return [g for g in qc.golden() if g[2] == 1]


def test_golden_corpus_one_call(ctx):
    cases = decoded()
    canv, status = ctx.qoi_frames([g[1] for g in cases])
    for (name, data, _, want_sha, want_st, _, _), c, s in zip(cases, canv, status):
        assert int(s) == want_st, f"{name}: status {int(s)}, pinned {want_st}"
        assert sha(c) == want_sha, f"{name}: canvas differs from the pin"
        if Q.have_ref():
            assert (c == Q.ref_qoi(data)).all(), f"{name}: canvas differs from the reference"


def _split_pins():
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "qoi.npz"))
    return {str(n): (str(s), int(st)) for n, s, st in zip(z["split_name"], z["split_sha"], z["split_status"])}


@pytest.mark.parametrize("fronts", [0, 1, 2, 5])
def test_split_cases(ctx, fronts):
    """Every split-point case in one call, each behind `fronts` ordinary files, so its tiles, chunks and segments
    sit at call-global positions that differ with the files in front."""
    pins = _split_pins()
    cases = qc.split_cases()
    front = qc.front_files(fronts)
    files = []
    for _, data, _ in cases:
        files += front + [data]
    canv, status = ctx.qoi_frames(files)
    for i, (name, data, _) in enumerate(cases):
        k = i * (fronts + 1) + fronts
        assert int(status[k]) == pins[name][1], name
        assert sha(canv[k]) == pins[name][0], f"{name} behind {fronts} files: canvas differs from the pin"
        for j in range(fronts):
            assert (canv[k - fronts + j] == ctx.qoi_frames([front[j]])[0][0]).all()


def test_live_reference_split_cases(ctx):
    if not Q.have_ref():
        pytest.skip("the reference's QOI source is not built (oracle/qoi.mk)")
    cases = qc.split_cases()
    canv, _ = ctx.qoi_frames([d for _, d, _ in cases])
    for (name, data, _), c in zip(cases, canv):
        assert (c == Q.ref_qoi(data)).all(), name


def test_dev_matches_host_and_order(ctx):
    import torch
    files = [g[1] for g in decoded()]
    canv, status = ctx.qoi_frames(files)
    total = sum(c.size for c in canv)
    d_frames = torch.empty(total, dtype=torch.uint8, device=device())
    d_status = ctx.qoi_frames_dev(files, d_frames)
    timg_b200.device_sync(torch)
    assert (d_frames.cpu().numpy() == np.concatenate([c.ravel() for c in canv])).all()
    assert (d_status.cpu().numpy() == status).all()
    rev, rstatus = ctx.qoi_frames(files[::-1])
    for a, b in zip(canv, rev[::-1]):
        assert (a == b).all()
    assert (rstatus[::-1] == status).all()
    one, _ = ctx.qoi_frames([files[5]])
    assert (one[0] == canv[5]).all()


def test_launch_count_does_not_grow(ctx):
    data = Q.encode(qc.rgba(pc.photo(200, 120, 3)), 3)
    l0 = ctx.launches
    ctx.qoi_frames([data])
    l1 = ctx.launches
    canv, status = ctx.qoi_frames([data] * 64)
    l2 = ctx.launches
    assert l1 - l0 == l2 - l1 == qc.LAUNCHES
    assert (status == 1).all() and all((c == canv[0]).all() for c in canv)


def test_rejections_launch_nothing(ctx):
    import torch
    good = Q.stream(4, 4, Q.Ops().rgb(1, 2, 3))
    d = torch.empty(16 * 4 + 16, dtype=torch.uint8, device=device())
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error):
        ctx.qoi_frames([])
    with pytest.raises(timg_b200.B200Error, match="aligned"):
        ctx.qoi_frames_dev([good], d[1:])
    for name, data, ok in qc.rejections():
        if not ok:
            with pytest.raises(timg_b200.B200Error, match="file 1"):
                ctx.qoi_frames_dev([good, data], d)
    assert ctx.launches == l0


def sized():
    """(name, image, header channels): our encoder round-trips its input exactly, so the image is the canvas."""
    yield "photo_4k", qc.rgba(pc.photo(3840, 2160, 1)), 3
    yield "photo_smooth_4k", qc.photo_smooth(3840, 2160, 1), 3
    yield "screenshot_4k", qc.rgba(pc.screenshot(3840, 2160, 2)), 3
    yield "solid_8192", np.full((8192, 8192, 4), (40, 50, 60, 255), np.uint8), 4
    yield "gradient_4k", qc.gradient(3840, 2160), 3


@pytest.mark.parametrize("name", [n for n, _, _ in sized()])
def test_sized(ctx, name):
    img, ch = next((i, c) for n, i, c in sized() if n == name)
    data = Q.encode(img, ch)
    canv, status = ctx.qoi_frames([data])
    assert int(status[0]) == 1
    assert canv[0].shape == img.shape
    bad = np.argwhere((canv[0] != img).any(-1))
    assert bad.size == 0, f"{name}: {len(bad)} pixels differ from the encoded image, first at {bad[0].tolist()}"
    if Q.have_ref():
        assert (canv[0] == Q.ref_qoi(data)).all()


def test_scaled_frames_compose_and_no_compose(ctx):
    """The frame timg sends at real options: status 1 composes with the background and pattern, status 2 (3-channel
    header, alpha below 255) does not -- a mixed call with has_bg = 0 reproduces it."""
    o = qc.FRAME_OPTS
    cases = [g for g in qc.golden() if g[5]]
    canv, status = ctx.qoi_frames([g[1] for g in cases])
    for (name, data, _, _, st, frame_sha, out), c, s in zip(cases, canv, status):
        (got,) = ctx.scale_mixed([c], [out], has_bg=int(s) == 1, bg=o["bg"], pattern=o["pattern"],
                                 pattern_w=o["pattern_size"] * o["cell"][0], pattern_h=o["pattern_size"] * o["cell"][1] // 2)
        assert sha(got) == frame_sha, f"{name} (status {int(s)}): frame differs from the reference's"


@pytest.mark.parametrize("enc", ["blocks", "sixel", "kitty", "iterm2", "kitty_tmux", "kitty_deflate"])
def test_handoff_into_mixed_batches(ctx, enc):
    """A page decoded on the device goes into the mixed encoders in place; the bytes equal the same call on the
    reference's canvases."""
    import torch
    if not Q.have_ref():
        pytest.skip("the reference's QOI source is not built (oracle/qoi.mk)")
    page = [g for g in decoded() if g[4] == 1 and not g[0].startswith(("row_", "col_"))][:12]   # sixel: w <= 4095
    files = [g[1] for g in page]
    refs = [Q.ref_qoi(d) for d in files]
    shapes = [r.shape for r in refs]
    d_dec = torch.empty(sum(r.size for r in refs), dtype=torch.uint8, device=device())
    st = ctx.qoi_frames_dev(files, d_dec)
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


@pytest.mark.parametrize("enc", ["blocks", "kitty", "iterm2"])
def test_status2_handoff_without_compose(ctx, enc):
    """Status-2 files (3-channel header, alpha below 255) at real options: decoded on the device and sent through a
    mixed call with has_bg = 0, the scaled frames are the reference's frames, and the encoders' bytes equal the same
    call on the reference's canvases."""
    import torch
    o = qc.FRAME_OPTS
    page = [g for g in qc.golden() if g[4] == 2 and g[5]]
    assert any(g[6] != (qoi_wh(g[1])) for g in page), "no status-2 file is scaled at FRAME_OPTS"
    files = [g[1] for g in page]
    geo = [timg_b200.qoi_parse(d) for d in files]
    shapes = [(g["h"], g["w"], 4) for g in geo]
    d_dec = torch.empty(sum(h * w * 4 for h, w, _ in shapes), dtype=torch.uint8, device=device())
    st = ctx.qoi_frames_dev(files, d_dec)
    timg_b200.device_sync(torch)
    assert (st.cpu().numpy() == 2).all()
    outs = [g[6] for g in page]
    dec = np.split(d_dec.cpu().numpy(), np.cumsum([h * w * 4 for h, w, _ in shapes])[:-1])
    frames = ctx.scale_mixed([c.reshape(sh) for c, sh in zip(dec, shapes)], outs, has_bg=False)
    for g, f in zip(page, frames):
        assert sha(f) == g[5], f"{g[0]}: the uncomposed frame differs from the reference's"
    if not Q.have_ref():
        pytest.skip("the reference's QOI source is not built (oracle/qoi.mk)")
    refs = [Q.ref_qoi(d) for d in files]
    flat, offs = timg_b200.pack_mixed(refs)
    d_ref = timg_b200._device_tensor(torch, flat)
    b, keep = timg_b200.mixed_batch(shapes, outs, offs, [0] * len(page), timg_b200.UPPER if enc == "blocks" else 0,
                                    has_bg=False, bg=o["bg"], pattern=o["pattern"])

    def run(d_src):
        if enc == "blocks":
            d_out, d_offs = ctx.blocks_mixed_dev(d_src, b)
        else:
            proto = {"kitty": timg_b200.KITTY, "iterm2": timg_b200.ITERM2}[enc]
            g, ids = timg_b200.graphics(proto, ids=list(range(1, len(page) + 1)), cell=o["cell"])
            d_out, d_offs = ctx.graphics_mixed_dev(d_src, b, g)
        timg_b200.device_sync(torch)
        off, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
        return [data[off[f]:off[f + 1]].tobytes() for f in range(len(page))]

    assert run(d_dec) == run(d_ref)


def qoi_wh(data):
    i = timg_b200.qoi_parse(data)
    return i["w"], i["h"]
