"""kitty's tmux form (B200TIMG_KITTY_TMUX) on the GPU: byte identity with what the reference's own KittyGraphicsCanvas
writes with tmux_passthrough_needed = true (tests/golden/graphics_tmux.npz) -- passthrough framing, chunking and the
Unicode placeholder grid -- over every golden case and id seed, scale + compose inside the batch, the host and
device-resident variants, the output capacity contract and the rejected arguments; and the plain kitty / iTerm2
forms ignoring the three fields only the tmux form reads."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import timg_b200
from timg_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_cases as gcases  # noqa: E402
import graphics_tmux_cases as tcases  # noqa: E402
from test_graphics_gpu import _batch  # noqa: E402
from test_graphics_oracle import GOLD as PLAIN_GOLD, PROTOCOLS  # noqa: E402
from test_graphics_tmux_oracle import GOLD, all_cases, check_grid, diacritic_values, golden_keys, kitty_tmux_payload  # noqa: E402

pytestmark = pytest.mark.gpu
T = timg_b200.KITTY_TMUX


def _geo(key):
    w, h, rgb24, cx, cy, indent = (int(v) for v in GOLD[key + "/geo"])
    return w, h, rgb24, (cx, cy), indent


def _matches(got, key):
    if key in GOLD.files:
        return got == GOLD[key].tobytes()
    return len(got) == int(GOLD[key + "/len"][0]) and gcases.sha(got) == GOLD[key + "/sha"].tobytes()


def _single(ctx, key, fb):
    w, h, rgb24, cell, indent = _geo(key)
    id_ = int(GOLD[key + "/id"][0])
    return ctx.graphics_batch(fb[None], _batch(1, w, h, w, h), T, rgb24, [id_], cell=cell, indent=indent)[0]


@pytest.mark.parametrize("seed", list(tcases.SEEDS))
def test_single_frames_equal_the_reference_tmux_canvas_bytes(ctx, seed):
    """t0: graphics_cases' frames at 9x18 cells with indent 2 (both colour types, 3072*k-byte PNGs and one byte either
    side, several stored blocks, alpha), 1-px cells on 300x4 and 4x300 frames (diacritics 283..296 and none past 296),
    no column, heights of exactly two cells and one pixel more, indents 0, 1 and 12; every seed: small frames whose ids
    have no, a 2-byte, a 3-byte and the largest id diacritic."""
    cases = all_cases()
    keys = [k for k in golden_keys() if k.startswith(seed + "/") and k.split("/", 1)[1] in cases and k != "t0/c2_rgb1"]
    assert len(keys) == (len(tcases.frame_cases() + tcases.geometry_cases()) if seed == "t0" else 0) + len(tcases.seed_cases())
    for key in keys:
        fb = cases[key.split("/", 1)[1]][0]
        assert _matches(_single(ctx, key, fb), key), key


def test_c2_geometry_frame_equals_the_reference(ctx):
    """One 2700x1519 frame at 9x18 cells: 300 columns (two grid items per row, the last diacritics and none past
    them), 85 rows, 4005 chunk separators."""
    assert _matches(_single(ctx, "t0/c2_rgb1", tcases.c2_frame()), "t0/c2_rgb1")


def test_c4_batch_with_scale_and_compose_equals_the_reference(ctx):
    n = tcases.C4_FRAMES
    keys = [f"t0/c4_rgb1/{f}" for f in range(n)]
    ids = [int(GOLD[k + "/id"][0]) for k in keys]
    _, _, _, cell, indent = _geo(keys[0])
    outs = ctx.graphics_batch(tcases.c4_graphics_frames(), _batch(n, 3840, 2160, 337, 190, has_bg=1, bg=timg_b200.rgba_u32(0, 0, 0)),
                              T, True, ids, cell=cell, indent=indent)
    for f in range(n):
        assert _matches(outs[f], keys[f]), f


def test_4k_row_at_one_pixel_cells(ctx):
    """A 3840x3 frame at 1-px cells: rows of 3840 placeholders (about 34 KB each) go out in 15 items of 256."""
    fb = synth.frame_np(91, 3840, 3, "noisea")
    id_ = 0xFF9ABC81
    out = ctx.graphics_batch(fb[None], _batch(1, 3840, 3, 3840, 3), T, False, [id_], cell=(1, 1), indent=5)[0]
    assert len(out) == timg_b200.graphics_size(T, 3840, 3, False, id_, cell=(1, 1), indent=5)
    _, got_id, cols, rows, grid = kitty_tmux_payload(out)
    assert (got_id, cols, rows) == (id_, 3840, 3)
    check_grid(grid, id_, cols, rows, 5, diacritic_values())


@pytest.mark.parametrize("chunk", [None, "1"])
def test_host_and_device_variants_give_identical_bytes_and_offsets(ctx, chunk, monkeypatch):
    import torch
    if chunk:
        monkeypatch.setenv("B200TIMG_CHUNK_FRAMES", chunk)
    n, iw, ih, ow, oh = 5, 400, 300, 310, 157
    frames = np.stack([synth.frame_np(710 + f, iw, ih, "alpha") for f in range(n)])
    ids = [9, 0xC8009181, 4294967295, 0x03000280, 77]
    b = _batch(n, iw, ih, ow, oh, has_bg=1, bg=timg_b200.rgba_u32(20, 30, 40))
    for cell, indent in (((9, 18), 2), ((1, 1), 0)):
        outs, offs = ctx.graphics_batch(frames, b, T, False, ids, with_offsets=True, cell=cell, indent=indent)
        d_out, d_offs = ctx.graphics_batch_dev(torch.tensor(frames).cuda(), b, T, False, ids, cell=cell, indent=indent)
        torch.cuda.synchronize()
        assert (d_offs.cpu().numpy().astype(np.uint64) == offs).all()
        ob = d_out.cpu().numpy().tobytes()
        assert [ob[int(offs[f]):int(offs[f + 1])] for f in range(n)] == outs
        values = diacritic_values()
        for f in range(n):
            _, id_, cols, rows, grid = kitty_tmux_payload(outs[f])
            assert (id_, cols, rows) == (ids[f], ow // cell[0], -(-oh // cell[1]))
            check_grid(grid, id_, cols, rows, indent, values)


def test_capacity_contract(ctx):
    """out_cap ending inside frame k (in its placeholder grid): earlier frames intact, nothing written at or past
    out_cap, offsets complete; the host variant reports ENOSPC before running anything."""
    import torch
    n, w, h = 4, 90, 40
    frames = np.stack([synth.frame_np(810 + f, w, h, "noisea") for f in range(n)])
    ids = [1, 0x03000002, 0xC8000003, 0xFF000004]
    b = _batch(n, w, h, w, h)
    cell, indent = (3, 2), 4
    want, offs = ctx.graphics_batch(frames, b, T, False, ids, with_offsets=True, cell=cell, indent=indent)
    k = 2
    cap = int(offs[k + 1]) - 50
    guard = 4096
    d_out = torch.full((cap + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    _, d_offs = ctx.graphics_batch_dev(torch.tensor(frames).cuda(), b, T, False, ids, d_out=d_out, out_cap=cap, cell=cell,
                                       indent=indent)
    torch.cuda.synchronize()
    ob = d_out.cpu().numpy()
    assert (d_offs.cpu().numpy().astype(np.uint64) == offs).all()
    for f in range(k):
        assert ob[int(offs[f]):int(offs[f + 1])].tobytes() == want[f], f
    assert (ob[int(offs[k]):] == 0xA5).all()                         # frame k is not written at all, nor anything after
    g, keep = timg_b200.graphics(T, False, ids, cell, indent)
    out = np.full(cap + guard, 0xA5, np.uint8)
    hoffs = np.zeros(n + 1, np.uint64)
    rc = timg_b200.lib().b200timg_graphics_batch(ctx.h, C.byref(b), C.byref(g), frames.ctypes.data, out.ctypes.data, cap,
                                                 hoffs.ctypes.data)
    assert rc == timg_b200.ENOSPC
    assert (hoffs == offs).all()
    assert (out == 0xA5).all()


def test_rejected_arguments(ctx):
    import torch
    L = timg_b200.lib()
    src = torch.zeros(64 * 64 * 4, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 17, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(2, dtype=torch.int64, device="cuda")
    ids = np.array([5], np.uint32)
    idp = ids.ctypes.data_as(C.POINTER(C.c_uint32))
    b = _batch(1, 64, 64, 64, 64)

    def call(g):
        return L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g), src.data_ptr(), out.data_ptr(), out.numel(),
                                             offs.data_ptr())
    for what, g, word in (("cell_x", timg_b200.Graphics(T, 0, idp, 0, 18, 0), "cell"),
                          ("cell_y", timg_b200.Graphics(T, 0, idp, 9, -1, 0), "cell"),
                          ("indent", timg_b200.Graphics(T, 0, idp, 9, 18, -1), "indent"),
                          ("ids", timg_b200.Graphics(T, 0, None, 9, 18, 0), "ids"),
                          ("protocol 3", timg_b200.Graphics(3, 0, idp, 9, 18, 0), "protocol")):
        rc = call(g)
        msg = L.b200timg_last_error(ctx.h).decode()
        assert rc == timg_b200.EINVAL and word in msg, (what, rc, msg)
    assert call(timg_b200.Graphics(T, 0, idp, 9, 18, 0)) == timg_b200.OK
    torch.cuda.synchronize()


@pytest.mark.parametrize("pname", ["kitty", "iterm2"])
def test_plain_forms_do_not_read_the_tmux_fields(ctx, pname):
    """Garbage in cell_x_px / cell_y_px / indent_cells changes nothing for B200TIMG_KITTY and B200TIMG_ITERM2: the
    output still equals the reference's (graphics.npz), through both variants."""
    import torch
    proto = PROTOCOLS[pname]
    L = timg_b200.lib()
    for name in ("2x3_rgb1", "chunk1p1_rgb1", "blocks_rgb0"):
        fb = dict((n, f) for n, f, _ in gcases.graphics_frame_cases())[name]
        rgb24 = int(name[-1])
        key = f"{pname}/{name}"
        want, id_ = PLAIN_GOLD[key].tobytes(), int(PLAIN_GOLD[key + "/id"][0])
        h, w = fb.shape[:2]
        b = _batch(1, w, h, w, h)
        ids = np.array([id_], np.uint32)
        for junk in ((0, 0, 0), (-7, 0x7FFFFFFF, -123456), (1, 1, 99)):
            g = timg_b200.Graphics(proto, rgb24, ids.ctypes.data_as(C.POINTER(C.c_uint32)), *junk)
            assert L.b200timg_graphics_size(C.byref(g), w, h, id_) == len(want)
            out = np.zeros(len(want), np.uint8)
            offs = np.zeros(2, np.uint64)
            assert L.b200timg_graphics_batch(ctx.h, C.byref(b), C.byref(g), fb.ctypes.data, out.ctypes.data, len(want),
                                             offs.ctypes.data) == timg_b200.OK
            assert out.tobytes() == want, (name, junk)
            d_out = torch.zeros(len(want), dtype=torch.uint8, device="cuda")
            d_offs = torch.zeros(2, dtype=torch.int64, device="cuda")
            d_fb = torch.tensor(fb).cuda()
            assert L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g), d_fb.data_ptr(), d_out.data_ptr(), len(want),
                                                 d_offs.data_ptr()) == timg_b200.OK
            torch.cuda.synchronize()
            assert d_out.cpu().numpy().tobytes() == want, (name, junk)
