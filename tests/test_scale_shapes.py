"""Host-only checks of the scaler's launch shapes: b200timg_scale_shape_of against the thresholds DESIGN.md section 4 and
include/b200timg.h document, and the case table of tests/test_scale_shapes_gpu.py against the classes default dispatch
can reach (found here by walking a grid of geometries, so a class that becomes reachable or unreachable fails the test)."""
import pytest

import scale_shape_cases as sc
import timg_b200

S = timg_b200.scale_shape


@pytest.fixture(autouse=True)
def no_knobs(monkeypatch):
    sc.apply_env(monkeypatch)


def pair(a, b, **kw):
    return S(*a, **kw), S(*b, **kw)


def test_planar_thresholds():
    """planar_smem <= 75 KB and 32 * 33 <= 3 * the window's words; beyond either, the fixed kernel."""
    a, b = pair((200, 200, 114, 114), (200, 200, 113, 114))
    assert a["route"] == "planar" and a["planar_smem"] <= 75 * 1024 < b["planar_smem"] and b["route"] == "fixed"
    assert a["planar_reuse"] == b["planar_reuse"] == 1 and (a["hc"], a["vc"]) == (b["hc"], b["vc"]) == (8, 8)
    a, b = pair((100, 100, 198, 198), (100, 100, 199, 199))
    assert (a["planar_reuse"], b["planar_reuse"]) == (1, 0) and b["route"] == "fixed"


def test_v3_thresholds():
    """FAST takes v3 where planar fits and 32 * 65 <= the v3 window's words; v3's 100 KB never decides, because no
    geometry planar takes needs more than 80 KB of v3 shared memory."""
    a, b = pair((128, 100, 132, 104), (128, 100, 133, 104), fast=True)
    assert (a["route"], b["route"]) == ("v3", "planar") and (a["v3_reuse"], b["v3_reuse"]) == (1, 0)
    assert S(128, 100, 132, 104)["route"] == "planar"                       # bit-exact scaling never takes v3
    worst = max(S(iw, int(oh * r), int(iw / r), oh, fast=True)["v3_smem"]
                for iw in range(64, 600, 12) for r in (1.5, 1.6, 1.7, 1.75, 1.8) for oh in (60, 114)
                if S(iw, int(oh * r), int(iw / r), oh, fast=True)["route"] in ("v3", "planar"))
    assert 0 < worst <= 100 * 1024, worst
    s = S(640, 360, 450, 253, fast=True)
    assert s["route"] == "v3" and s["v3_tma"] == int(s["win_w"] <= 256 and s["win_h"] <= 256)


def test_fixed_threshold_and_the_two_pass_fall_through():
    """fixed_smem <= 100 KB; 8 taps on both axes beyond it run the two-pass kernels."""
    a, b = pair((113, 115, 60, 61), (114, 115, 60, 61))
    assert a["route"] == "fixed" and a["fixed_smem"] <= 100 * 1024 < b["fixed_smem"]
    assert b["route"] == "tp_v" and (b["h_widest"], b["v_widest"]) == (8, 8) and (b["hc"], b["vc"]) == (8, 8)
    s = S(379, 127, 196, 82)
    assert s["route"] == "tp_h1s" and s["fixed_smem"] > 100 * 1024 and max(s["h_widest"], s["v_widest"]) <= 8


def test_two_pass_first_pass_thresholds():
    """h1s: h1s_smem <= 72 KB and ceil(ow / 32) * 32 <= 1.15 * ow; h1f for the rest up to ow = 4096 -- which never decides,
    since every ow >= 207 fills its 32-column tiles to 115 %."""
    a, b = pair((3776, 100, 256, 50), (3780, 100, 256, 50))
    assert (a["route"], b["route"]) == ("tp_h1s", "tp_h1") and a["h1s_smem"] <= 72 * 1024 < b["h1s_smem"]
    a, b = pair((400, 100, 28, 50), (400, 100, 27, 50))
    assert (a["route"], a["tiles_full"], b["route"], b["tiles_full"]) == ("tp_h1s", 1, "tp_h1f", 0)
    assert 4 <= b["h1f_rows"] <= 64 and a["h1f_rows"] == 0
    assert S(2000, 100, 27, 50)["route"] == "tp_h1f" and S(2000, 100, 28, 50)["route"] == "tp_h1"
    assert all((ow + 31) // 32 * 32 * 100 <= ow * 115 for ow in range(207, 5000))
    assert S(65536, 4, 4096, 1)["route"] == S(65540, 4, 4097, 1)["route"] == "tp_h1"


def test_alignment_and_width_rules():
    """planar and v3 need iw % 4 == 0 and a 16-byte aligned source; the 16-byte copy needs ow % 4 == 0 and both pointers
    aligned."""
    assert S(640, 360, 450, 253)["route"] == "planar"
    assert S(641, 360, 450, 253)["route"] == S(642, 360, 450, 253)["route"] == "fixed"
    assert S(640, 360, 450, 253, src_aligned16=False)["route"] == "fixed"
    assert S(640, 360, 450, 253, fast=True, src_aligned16=False)["route"] == "fixed"
    assert S(128, 30, 128, 30)["route"] == "copy4" and S(130, 30, 130, 30)["route"] == "copy"
    assert S(128, 30, 128, 30, src_aligned16=False)["route"] == S(128, 30, 128, 30, dst_aligned16=False)["route"] == "copy"
    assert S(128, 30, 128, 30, n_frames=70000)["route"] == "copy"


def test_knobs_reach_the_shape(monkeypatch):
    monkeypatch.setenv("B200TIMG_NO_PLANAR", "1")
    assert S(640, 360, 450, 253)["route"] == "fixed"
    monkeypatch.setenv("B200TIMG_NO_H1S", "1")
    assert S(3840, 200, 337, 18)["route"] == "tp_h1"
    monkeypatch.setenv("B200TIMG_NO_H1F", "1")
    assert S(400, 100, 27, 50)["route"] == "tp_h1"


def test_invalid_arguments():
    for args in ((0, 4, 4, 4), (4, 4, 0, 4), (4, 4, 4, 4, 0), (5, 5, 7, 7, 65536)):
        with pytest.raises(timg_b200.B200Error):
            S(*args)


INS = (1, 2, 3, 4, 5, 7, 8, 12, 20, 33, 44, 64, 100, 256, 640, 1000)
RATIOS = (0.35, 0.45, 0.55, 0.62, 0.7, 0.8, 0.9, 1.5, 2.0, 2.7)
# routes the grid has no geometry for: 8 x 8 taps past the fixed kernel's shared memory, the plain tiled first pass, the copies
LARGE = ((114, 115, 60, 61), (379, 127, 196, 82), (132, 4578, 66, 2813), (2000, 100, 28, 50), (128, 64, 128, 64),
         (130, 64, 130, 64))


def reached():
    """Every class key default dispatch takes over a grid of 1-D geometries (each source size against shrinks and
    enlargements), both arithmetic modes."""
    axis = sorted({(i, o) for i in INS for o in {i - 1, i + 1, *(max(1, round(i * r)) for r in RATIOS)} if o >= 1 and o != i})
    s = timg_b200.ScaleShape()
    seen = set()
    for iw, ow in axis:
        for ih, oh in axis:
            for fast in (0, 1):
                seen.add(sc.shape_raw(iw, ih, ow, oh, fast, s))
    for g in LARGE:
        seen.add(sc.shape_raw(*g, 0, s))
    return seen


def test_reachable_classes_are_the_documented_ones():
    seen = reached()
    assert seen == sc.REACHABLE, (f"newly reachable: {sorted(seen - sc.REACHABLE)}; no longer reached: "
                                  f"{sorted(sc.REACHABLE - seen)} -- update scale_shape_cases.py")
    assert not set(sc.UNREACHABLE) & seen
    # every tap-class instantiation of v3, planar and both fixed orders is either reached or listed with a reason
    for route, vfs in (("v3", (1,)), ("planar", (1,)), ("fixed", (0, 1))):
        for hc in (2, 4, 6, 8):
            for vc in (2, 4, 6, 8):
                for vf in vfs:
                    for hw in ((3, 4) if hc == 4 else (0,)):
                        k = (route, hc, vc, hw, vf)
                        assert k in seen or k in sc.UNREACHABLE, f"{k}: neither reached nor listed as unreachable"


def test_case_table_covers_every_class(monkeypatch):
    cases = sc.cases()
    assert len({(c.group, c.name) for c in cases}) == len(cases)
    shapes = [(c, sc.check_class(c)) for c in cases]
    keys = {sc.class_key(s) for _, s in shapes}
    assert sc.REACHABLE <= keys, sorted(sc.REACHABLE - keys)
    for route in ("copy4", "copy", "v3", "planar", "fixed", "tp_v", "tp_h1s", "tp_h1f", "tp_h1"):
        fmts = {c.fmt for c, s in shapes if s["route"] == route}
        assert fmts == {0, 1}, f"{route}: byte orders {fmts}"
    for kind in sc.KINDS:
        assert {s["route"] for c, s in shapes if c.kind == kind} >= {"v3", "planar", "tp_h1s"}, kind
    assert any(s["v_gather"] == 0 for _, s in shapes) and any(s["h_filter"] == 0 and s["v_filter"] for _, s in shapes)
    assert any(s["v_filter"] == 0 and s["h_filter"] for _, s in shapes)
    assert any(timg_b200.resample_plan(c.iw, c.ih, c.ow, c.oh, 0)["lead"].max() > 0 for c, s in shapes if c.group == "filter")
    ows, ohs = {c.ow for c in cases}, {c.oh for c in cases}
    assert {1, 31, 32, 33, 63, 64, 65} <= ows and {1, 15, 16, 17, 31, 32, 33} <= ohs
    assert {1, 2, 3, 4} <= {c.iw for c in cases} and {1, 2, 3, 4} <= {c.ih for c in cases}
