"""Host-only checks of the sixel launch shapes: b200timg_sixel_shape_of against the thresholds DESIGN.md section 4 and
include/b200timg.h document, and the case table of tests/test_sixel_shapes_gpu.py against the list of classes it is there to
cover -- for several SM counts, so the matrix stays honest when a threshold moves or the suite runs on another part."""
import pytest

import sixel_shape_cases as sc
import timg_b200


@pytest.fixture(autouse=True)
def no_knobs(monkeypatch):
    for k in sc.KNOBS:
        monkeypatch.delenv(k, raising=False)


def shape(w, h, n=1, n_total=None, sm=132):
    return timg_b200.sixel_shape(w, h, n, n_total, sm)


def test_palette_thresholds():
    """Sampling step npix / 18383 (6 below 18383 pixels); entries = samples, at most 32768; tables in shared memory up to
    25600 entries."""
    for npix6, step, cap, glob in ((3063, 6, 3063, 0), (3064, 1, 18384, 0), (4266, 1, 25596, 0), (4267, 1, 25602, 1), (5461, 1, 32766, 1),
                                   (5462, 1, 32768, 1), (6127, 1, 32768, 1), (6128, 2, 18384, 0), (8533, 2, 25599, 0), (8534, 2, 25602, 1),
                                   (9191, 2, 27573, 1), (9192, 3, 18384, 0), (12800, 4, 19200, 0), (99999, 32, 18750, 0)):
        s = shape(npix6, 6)
        assert (s["step_px"], s["ent_cap"], s["palette_global"]) == (step, cap, glob), (npix6 * 6, s)
    # the boundary itself, on pixel counts a frame cannot have (h is a multiple of 6) but the rule is stated for
    for npix in range(18370, 18400):
        if npix % 6 == 0:
            assert shape(npix // 6, 6)["step_px"] == (6 if npix < 18383 else 1)
    assert max(shape(w, 6)["ent_cap"] for w in range(1, 20000, 7)) == 32768


@pytest.mark.parametrize("sm", sc.SM_COUNTS)
def test_dither_thresholds(sm):
    """CTAs per frame: 1 for a batch of at least sm_count frames, else min(sm_count / n_total, (nb32 + 7) / 8) -- never more
    CTAs in a launch than SMs; at most 24 warps per CTA, in full rounds; at most 2048 bands."""
    for h in (6, 36, 198, 258, 384, 804, 1524, 6144, 65532):
        nb32 = (h + 31) // 32
        for n in (1, 2, 3, 7, sm // 8, sm // 2, sm // 2 + 1, sm - 1, sm, sm + 5):
            s = shape(64, h, n, sm=sm)
            assert s["nb32"] == nb32
            want = 1 if n >= sm else max(1, min(sm // n, (nb32 + 7) // 8))
            bands = -(-nb32 // want)
            assert (s["bands_per_cta"], s["dither_ctas"]) == (bands, -(-nb32 // bands)), (h, n, s)
            assert s["dither_ctas"] * n <= sm or s["dither_ctas"] == 1
            assert s["dither_rounds"] == -(-bands // 24) and s["dither_warps"] == -(-bands // s["dither_rounds"]) <= 24
            assert s["dither_warps"] * s["dither_rounds"] >= bands
    assert shape(4, 65532, sm=sm)["nb32"] == 2048
    # a slice of a larger batch splits by the batch's size, not its own
    assert shape(120, 288, 2, 8, sm)["dither_ctas"] == shape(120, 288, 8, 8, sm)["dither_ctas"] == min(sm // 8, 2)


def test_dither_knobs_are_clamped(monkeypatch):
    """B200TIMG_DITHER_SPLIT never takes a launch beyond one CTA per SM, nor a frame beyond one CTA per band."""
    monkeypatch.setenv("B200TIMG_DITHER_SPLIT", "6")
    assert shape(100, 330)["dither_ctas"] == 6
    assert shape(100, 96)["dither_ctas"] == 3                       # three bands
    assert shape(100, 330, 40)["dither_ctas"] == 3                  # 132 / 40
    assert shape(100, 330, 100)["dither_ctas"] == 1
    assert shape(100, 330, 132)["dither_ctas"] == 1                 # a full batch is never split
    monkeypatch.setenv("B200TIMG_DITHER_SPLIT", "5")
    assert shape(100, 198)["dither_ctas"] == 4                      # 7 bands in CTAs of 2
    monkeypatch.delenv("B200TIMG_DITHER_SPLIT")
    monkeypatch.setenv("B200TIMG_DITHER_WARPS", "99")
    assert shape(100, 1524, 132)["dither_warps"] == 24
    monkeypatch.setenv("B200TIMG_DITHER_WARPS", "0")
    assert shape(100, 198)["dither_rounds"] == 7


def test_emit_thresholds(monkeypatch):
    """emit5 up to 4095 px, the column-tiled single-pass emitter beyond, in (w + 4095) / 4096 tiles of whole 32-column steps."""
    for w in (1, 337, 2700, 4095, 4096, 4097, 8192, 8193, 12289, 99999):
        s = shape(w, 6)
        assert s["emit_mode"] == (5 if w <= 4095 else 2), w
        assert s["emit_tiles"] == (w + 4095) // 4096
        assert s["tile_w"] % 32 == 0 and s["tile_w"] <= 4096 and s["tile_w"] * s["emit_tiles"] >= w > s["tile_w"] * (s["emit_tiles"] - 1)
    monkeypatch.setenv("B200TIMG_EMIT", "2")
    assert shape(337, 6)["emit_mode"] == 2
    monkeypatch.setenv("B200TIMG_EMIT", "5")
    assert shape(4096, 6)["emit_mode"] == 2                          # emit5's entry word holds x in 12 bits


def test_limits_are_einval():
    for args in ((100000, 6), (4, 65538), (10, 7), (0, 6), (10, 0), (10, 6, 0), (10, 6, 65536), (10, 6, 3, 2)):
        with pytest.raises(timg_b200.B200Error) as e:
            shape(*args)
        assert e.value.code == timg_b200.EINVAL
    with pytest.raises(timg_b200.B200Error):
        shape(10, 6, sm=0)
    assert shape(99999, 6) and shape(4, 65532) and shape(10, 6, 65535)


@pytest.mark.parametrize("sm", sc.SM_COUNTS)
def test_case_table_covers_every_class(sm, monkeypatch):
    """Every case is in the class it is named after, and together they hit every class the matrix promises."""
    seen = []
    all_cases = sc.cases(sm)
    assert [c.name for c in all_cases] == [c.name for c in sc.cases(sc.SM_COUNTS[0])]      # ids do not depend on the device
    assert len({(c.group, c.name) for c in all_cases}) == len(all_cases)
    for c in all_cases:
        sc.apply_env(monkeypatch, c)
        seen.append((c, sc.check_class(c, sm)))

    def hit(group, **want):
        return [c for c, d in seen if c.group == group and all(d[k] == v for k, v in want.items())]

    for cls in sc.PALETTE_CLASSES:
        kinds = {c.kind for c in hit("palette", palette=cls)}
        assert {"noise", "photo"} <= kinds, f"palette class {cls}: kinds {kinds}"
    npix = sorted(c.w * c.h for c in hit("palette"))
    for edge in sc.PALETTE_EDGES:
        assert any(edge - 8 <= p < edge for p in npix) and any(edge <= p < edge + 8 for p in npix), f"palette edge {edge}"
    assert [c for c in hit("palette", palette_global=1) if c.diffuse is False], "few-colour frame in the global-table range"
    assert [c for c in hit("palette", ent_cap=32768) if c.kind == "allcells"]
    for ctas in range(1, 7):
        assert hit("dither", dither_ctas=ctas), f"dither: {ctas} CTAs per frame"
    rounds = {d["dither_rounds"] for c, d in seen if c.group == "dither"}
    assert {1, 2} <= rounds and max(rounds) > 2
    for flag in ("short_last_cta", "single_band_cta", "remote_and_local"):
        assert hit("dither", **{flag: True}), flag
    assert [c for c, d in seen if c.group == "dither" and d["dither_ctas"] > 1 and d["dither_rounds"] > 1], "split x rounds"
    assert [c for c in hit("dither") if c.env.get("B200TIMG_DITHER_SPIN") == 0 and c.env.get("B200TIMG_DITHER_SPLIT")]
    assert {c.h - 32 * ((c.h - 1) // 32) for c in hit("dither") if c.name.startswith("lastband")} == {6, 12, 18, 24, 30, 32}
    assert {c.w for c in hit("dither") if c.name.startswith("width")} == set(sc.WIDTHS)
    assert all(c.h >= 66 for c in hit("dither") if c.name.startswith("width"))
    # batches: natural split over a full grid, more frames than SMs, natural rounds, slices
    assert [c for c in hit("batch", dither_ctas=2) if not c.env and 2 * c.n > sm - 2]
    assert [c for c in hit("batch") if c.n > sm] and [c for c in hit("batch") if c.n == sm - 1]
    assert [c for c in hit("batch", dither_rounds=2) if not c.env]
    assert {c.env.get("B200TIMG_PARTS") for c in hit("batch") if c.n_total > c.n} == {2, 4}
    assert all(not (set(c.env) - {"B200TIMG_PARTS"}) for c in hit("batch"))
    assert hit("wide", emit_mode=5) and {d["emit_tiles"] for c, d in seen if c.group == "wide" and d["emit_mode"] == 2} >= {1, 2, 3, 4}
    assert hit("wide", nb32=192) and hit("wide", nb32=2048) and [c for c in hit("wide") if c.w == 99999]
    assert hit("capacity", emit_mode=5) and hit("capacity", emit_mode=2, emit_tiles=2)
