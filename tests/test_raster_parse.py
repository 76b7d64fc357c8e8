"""b200timg_raster_parse against the pins of tests/golden/raster.npz and the damaged-header outcomes, EINVAL against the
reference's STB source where its door is built, the plan model of raster_cases.py against raster.cu's constexprs, and
each RLE tile case landing where its name says (no GPU)."""
import ctypes as C
import os
import re

import pytest

import raster_cases as rc
import timg_b200
from oracle import raster as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def outcome(data, size=None):
    if size is None:
        try:
            info = timg_b200.raster_parse(data)
        except timg_b200.B200Error:
            return "einval"
        return "ok" if info["supported"] else "unsupported"
    info = timg_b200.RasterInfo()
    rc_ = timg_b200.lib().b200timg_raster_parse(data, size, C.byref(info))
    if rc_ != timg_b200.OK:
        return "einval"
    return "ok" if info.supported else "unsupported"


def test_parse_matches_pins():
    for name, data, parse, _, _, _, _ in rc.golden():
        got = outcome(data)
        assert (got == "einval") == (parse < 0), name
        if parse == 1:
            assert got == "ok", name


def test_rejection_outcomes():
    for name, data, want in rc.rejections():
        assert outcome(data) == want, name


def test_big_files_by_size():
    for name, head, size, want in rc.unsupported_big():
        assert outcome(head, size) == want, name


def test_einval_iff_reference_fails():
    if not R.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    for name, data, want in rc.rejections():
        info = None if want == "einval" else timg_b200.raster_parse(data)
        if info is not None and info["w"] * info["h"] > rc.DECODED_MAX_PX:
            continue
        assert (R.ref_stb(data) is None) == (want == "einval"), name


def test_corpus_fields():
    info = {n: timg_b200.raster_parse(d) for n, d in rc.corpus()}
    assert all(i["supported"] for i in info.values())
    assert info["bmp24_top_down"]["top_down"] and not info["bmp24_h40"]["top_down"]
    assert info["bmp24_ma_ff000000"]["channels"] == 3 and info["bmp32_alpha"]["channels"] == 4
    assert info["bmp8_small_palette"]["palette"] == 12 and info["bmp8_psize_negative"]["palette"] < 0
    assert info["tga3_15_as_rgb16"]["channels"] == 3 and info["tga3_16_grey_alpha"]["channels"] == 2
    assert info["tga10_24"]["rle"] and not info["tga2_24_bottom_up"]["rle"]
    assert info["tga1_16_pal16"]["palette"] == 300
    assert info["p5_16"]["bpp"] == 16 and info["p6_16"]["bpp"] == 48 and info["p5_maxval_overflow"]["bpp"] == 8
    assert {i["format"] for i in info.values()} == {"bmp", "tga", "pnm"}


def test_model_constants_match_kernels():
    src = open(os.path.join(ROOT, "timg_b200", "csrc", "raster.cu")).read()
    for name in ("TILE", "P", "CHUNK"):
        m = re.search(rf"constexpr int {name} = (\d+);", src)
        assert m and int(m.group(1)) == getattr(rc, name), name
    assert f"A call launches {rc.LAUNCHES} kernels" in src
    assert rc.P == 1 + 128 * 4 and rc.P <= rc.TILE     # an entry byte lies inside its tile


def test_tile_cases_land_where_named():
    names, tags = set(), set()
    for name, data, where in rc.tile_cases():
        assert name not in names
        names.add(name)
        info = timg_b200.raster_parse(data)
        assert info["rle"] and info["supported"], name
        starts = rc.packet_starts(data, where["B"])
        for h in where["header_at"]:
            assert h in starts, name
            tags.add((h % rc.TILE, h // rc.TILE % rc.CHUNK == 0))
        if "densest" in name:
            assert all(data[rc.TGA_HEADER + s] & 128 for s in starts), name
        if "sparsest" in name:
            lens = [b - a for a, b in zip(starts, starts[1:])]
            assert set(lens) == {1 + 128 * where["B"]}, name
            assert len(starts) * (1 + 128 * where["B"]) > 2 * rc.CHUNK * rc.TILE
        if where.get("spans_super"):
            assert starts[-1] > rc.CHUNK * rc.CHUNK * rc.TILE, name
    assert {(0, False), (rc.TILE - 1, False), (0, True), (rc.TILE - 1, False)} <= tags
