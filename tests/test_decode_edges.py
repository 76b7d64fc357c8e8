"""The decoder edge cases (tests/decode_edge_cases.py) without a GPU: the plan model's constants are the kernels' own,
every planned class has cases, each case lands where its name says, and every failure case differs from its clean
twin by its event alone."""
import collections

import numpy as np
import pytest

import decode_edge_cases as E

PLANNED = ["png_window_len286", "png_window_len287", "png_window_dist30", "png_window_dist31", "png_window_dist_far",
           "png_window_unused_code", "png_window_threshold", "png_block_end", "png_stored", "png_end", "png_copy",
           "png_unfilter_height", "png_unfilter_edge_rows", "png_unfilter_adam7", "png_unfilter_late_event",
           "jpeg_flip", "jpeg_cut", "jpeg_huffman_error", "jpeg_restart_order", "jpeg_dc_order", "gif_string_length", "gif_kwkwk", "gif_full_dictionary", "gif_area_end",
           "gif_interlaced", "gif_many_frames"]


@pytest.fixture(scope="module")
def cases():
    return E.all_cases()


@pytest.mark.parametrize("src", sorted(E.MODEL_CONSTANTS))
def test_model_constants_are_the_kernels(src):
    """If a kernel is retuned, this names the constant; the cases aimed by it then need re-aiming."""
    got = E.kernel_constants(src)
    for name, v in E.MODEL_CONSTANTS[src].items():
        assert got.get(name) == v, f"{src}: {name} is {got.get(name)}, the plan model assumes {v}"


def test_every_planned_class_has_cases(cases):
    n = collections.Counter(c.cls for c in cases)
    assert not [k for k in PLANNED if not n[k]], [k for k in PLANNED if not n[k]]
    assert set(n) <= set(PLANNED) | {"png_twin", "jpeg_twin"}


def test_names_unique_and_pinned(cases):
    names = [c.name for c in cases]
    assert len(set(names)) == len(names)
    assert set(names) == set(E.golden()), "tests/golden/decode_edges.npz is stale: rerun make_decode_edges_golden.py"


def test_png_cases_land_where_named(cases):
    for c in cases:
        w = c.where
        if c.cls.startswith("png_window_") and c.cls != "png_window_threshold":
            assert E.png_locate(w["plan"]["windows"], w["bit"]) == (w["window"], w["sub"], w["delta"]), c.name
            assert f"w{w['window']}t" in c.name and c.name.endswith(f"d{w['delta']}")
            assert w["sub"] in (0, 1, 3, 4, 255, 510, 511) or w["window"] == 1
            if w["window"] == 1:
                assert w["sub"] in (0, w["nact"] - 1), c.name
        elif c.cls == "png_window_threshold":
            assert w["nact"] == w["room"] // E.SUB_BITS and w["windowed"] == (w["nact"] >= 4), c.name
        elif c.cls == "png_block_end" and "eob" in c.name:
            assert E.png_locate(w["plan"]["windows"], w["bit"]) == (0, w["sub"], w["delta"]), c.name
        elif c.cls == "png_block_end":
            assert w["plan"]["windows"], c.name
        elif c.cls == "png_stored":
            assert w["plan"]["windows"], c.name       # the stored block follows a window
            if "end_mod8" in w:
                assert (w["plan"]["blocks"][1][0] + w["plan"]["off"]) % 8 == w["end_mod8"], c.name
        elif c.cls == "png_end":
            assert w["windows"] and w["cut_bits"] <= 48, c.name
        elif c.cls == "png_copy" and "distances" in w:
            assert w["distances"] == [1, 2, 3, 258, 32767, 32768]
            assert w["chain_windows"] == [0, 1, 2], w["chain_windows"]
            assert w["last_copy"] is not None, "the copy across the image's end is decoded by a window"


def test_png_window_events_cover_every_subsequence_and_offset(cases):
    got = {(c.cls, c.where["window"], c.where["sub"] if c.where["window"] == 0 else ("first", "last")[c.where["sub"] > 0],
            c.where["delta"]) for c in cases if c.cls.startswith("png_window_") and "bit" in c.where}
    for ev in E.PNG_EVENTS:
        for t in (0, 1, 3, 4, 255, 510, 511):
            for d in (0, 1, 8, 255):
                if t or d != 1:
                    assert (f"png_window_{ev}", 0, t, d) in got, (ev, t, d)
        for t in ("first", "last"):
            for d in (0, 1, 8, 255):
                if t == "last" or d != 1:
                    assert (f"png_window_{ev}", 1, t, d) in got, (ev, t, d)


def test_png_unfilter_cases_cross_row_groups(cases):
    widths = {c.where["fb"] for c in cases if c.cls == "png_unfilter_height"}
    assert widths == {1, 2, 3, 4, 6, 8}
    for c in cases:
        w = c.where
        if c.cls == "png_unfilter_height":
            assert w["rows"] == E.unfilter_rows(w["fb"])
        elif c.cls == "png_unfilter_adam7":
            assert max(w["pass_rows"]) > w["rows"], c.name
        elif c.cls == "png_unfilter_late_event":
            assert w["row"] // w["rows"] == w["group"] == 1, c.name


def test_jpeg_cases_land_where_named(cases):
    """Each flip, run of ones and cut sits at 64k - 1, 64k or 64k + 1 of the call-global subsequence k it names when
    the file follows the named number of front files; k is at a sync CTA's edge (CTA c owns 127c - 1 .. 127c + 126)
    or a fix-up batch's (512 per batch)."""
    fronts = [[len(s) for s in E.destuffed_map(f)] for f in E.front_files()]
    assert all(sum(E.jpeg_subsequences(f)) % 2 for f in fronts)
    bases = {**{n: E.destuffed_map(d) for n, d in E.golden_bases().items()}}
    aimed = collections.Counter()
    for c in cases:
        w = c.where
        if c.cls not in ("jpeg_flip", "jpeg_huffman_error", "jpeg_cut"):
            continue
        lengths = [len(s) for s in bases[c.name.split("_")[1]]]
        p = E.jpeg_place(fronts[:w["front"]], lengths, w["seg"], w["off"])
        assert p["sub"] == w["k"] - (w["d"] < 0), c.name
        assert p["sub_off"] == (w["d"] % E.SUB_BYTES), c.name
        if w["k"] in E.CTA_KS:
            assert any((E.SYNC_T - 1) * cta - 2 <= p["sub"] <= (E.SYNC_T - 1) * cta + 1 for cta in (1, 2)), c.name
            assert len(p["cta"]) == 2 or p["sub"] in (126, 253) or p["sub"] % (E.SYNC_T - 1) in (0, 1, 125), c.name
        else:
            assert w["front"] == 0 and p["local_sub"] in (E.FIX_T - 2, E.FIX_T - 1, E.FIX_T, E.FIX_T + 1), c.name
        aimed[(c.cls, w["k"], w["front"])] += 1
    for cls in ("jpeg_flip", "jpeg_huffman_error"):
        for k in E.CTA_KS:
            for n in E.FRONT_AIMS:
                assert aimed[(cls, k, n)], (cls, k, n)
        for k in E.FIX_KS:
            assert aimed[(cls, k, 0)], (cls, k)
    pins = E.golden()
    assert {pins[c.name][0] for c in cases if c.cls == "jpeg_huffman_error"} == {0}
    order = {c.name: (c.where["events"], pins[c.name][0]) for c in cases if c.cls in ("jpeg_restart_order", "jpeg_dc_order")}
    assert order["j_dri_bail0_then_error_seg2"][1] == -1 and order["j_dri_error_seg0_then_bail1"][1] == 0
    dc = [c for c in cases if c.cls == "jpeg_dc_order" and len(c.where["events"]) == 2]
    assert {tuple(c.where["events"]) for c in dc} == {("dc", "error"), ("error", "dc")}
    for c in dc:
        first, second = (c.where[e]["cta"] for e in c.where["events"])
        assert max(first) < max(second), c.name        # the two events in different sync CTAs, in the named order


def test_gif_cases_land_where_named(cases):
    for c in cases:
        w = c.where
        plan = w.get("plan")
        if c.cls == "gif_string_length":
            lens = [p[2] for p in plan]
            assert max(lens) == w["longest"] and plan[-1][4] == "eoi"
        elif c.cls == "gif_kwkwk":
            assert any(p[4] == "kwkwk" and p[3] == w["period"] for p in plan)
        elif c.cls == "gif_area_end":
            assert sum(p[2] for p in plan) > w["area"] and max(p[2] for p in plan) > E.GIF_SHORT
        elif c.name == "gif_cs12_dict8191":
            assert plan[-1][4] == "eoi" and max(p[2] for p in plan) > E.GIF_SHORT
        elif c.name == "gif_cs12_dict_overflow":
            assert plan[-1][4] == "illegal"


def _bits_differ_only_by_event(d):
    a, b = (np.asarray(x, np.uint8) for x in d["bits"])
    at = d["at"]
    assert (a[:at] == b[:at]).all(), "the streams differ before the event"
    if d.get("prefix"):
        assert len(a) < len(b) and (a == b[:len(a)]).all()
    elif d.get("same_size"):
        assert (a[d["end"]:] == b[d["twin_end"]:]).all() and len(a) - d["end"] == len(b) - d["twin_end"]


def test_failure_cases_differ_from_their_twin_by_the_event_alone(cases):
    by = {c.name: c for c in cases}
    pins = E.golden()
    n = 0
    for c in cases:
        if c.twin is None:
            continue
        tw = by[c.twin]
        assert tw.twin is None
        st = pins[tw.name][0]
        assert st == 1 or (tw.fmt == "gif" and st == tw.where["frames"]), f"{tw.name}: the twin's pin is {st}"
        d = c.diff
        if "bits" in d:
            _bits_differ_only_by_event(d)
        elif "bytes" in d:
            a, b = d["bytes"]
            assert a != b
            if d.get("prefix"):
                assert b.startswith(a) and len(a) == d["at"]
            else:
                i = next(i for i in range(min(len(a), len(b))) if a[i] != b[i])
                j = next(j for j in range(1, min(len(a), len(b))) if a[-j] != b[-j])
                if d.get("same_size"):
                    assert len(a) == len(b) and i == d["at"] == len(a) - j, c.name
                else:
                    assert i < len(a) - j + 1 and len(b) - j - i < 4096, c.name
        elif "destuffed" in d:                       # a run of ones replacing as many scan bytes
            a, b = d["bytes"]
            seg, off, n = d["destuffed"]
            sa, sb = E.destuffed_map(a)[seg], E.destuffed_map(b)[seg]
            assert len(sa) == len(sb), c.name
            da, db = bytes(a[i] for i in sa), bytes(b[i] for i in sb)
            assert da[:off] == db[:off] and da[off + n:] == db[off + n:] and da[off:off + n] == b"\xff" * n, c.name
        elif "rst" in d:                              # one restart marker dropped or written twice
            a, b = d["rst"]
            assert abs(len(a) - len(b)) == 2, c.name
            da, db = (b"".join(bytes(x[i] for i in seg) for seg in E.destuffed_map(x)) for x in (a, b))
            assert da == db and a[:E.jc.scan_start(a)] == b[:E.jc.scan_start(b)], c.name
        elif "codes" in d:
            a, b = d["codes"]
            assert a[:-1] == b[:len(a) - 1] and a[-1] != b[len(a) - 1], c.name
        elif "samples" in d:
            a, b = d["samples"]
            ys, xs = np.nonzero((a != b).reshape(a.shape[0], a.shape[1], -1).any(-1))
            assert len(ys) and len(set(ys // 8)) == 1 and len(set(xs // 8)) == 1, c.name   # one sample or one block
        elif "filters" in d:
            a, b = d["filters"]
            assert sum(x != y for x, y in zip(a, b)) == 1, c.name
        else:
            raise AssertionError(f"{c.name}: no twin comparison")
        n += 1
    assert n > 300
