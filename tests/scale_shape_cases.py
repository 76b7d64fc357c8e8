"""Case table of the scaler's launch-shape matrix (tests/test_scale_shapes_gpu.py runs it on the device, tests/test_scale_shapes.py
checks on the host that it covers every class).  A case names the shape it is there for in `expect`: fields of
b200timg_scale_shape (route by name).  The shape is always asked of the library (timg_b200.scale_shape, launch_scale's own
arithmetic), so a moved threshold fails the case instead of quietly turning it into a test of something else."""
import ctypes as C
import zlib
from collections import namedtuple

import numpy as np

import timg_b200
from timg_b200 import synth

# fmt: 0 RGBA, 1 RGB32; fast: the FAST arithmetic; src_off: byte offset of the source inside its device buffer (16-byte
# aligned or not); kind: content (see frame())
Case = namedtuple("Case", "group name iw ih ow oh kind fmt fast expect src_off")

KNOBS = ("B200TIMG_NO_PLANAR", "B200TIMG_NO_H1S", "B200TIMG_NO_H1F", "B200TIMG_TMA")
KINDS = ("photo", "noise", "noisea", "holes", "edgepx", "clear", "faint")

# (route, hc, vc, h_widest if hc == 4 else 0, vertical_first) that default dispatch reaches; the host test finds exactly
# these in its grid of geometries (plus the 8 x 8 two-pass fall-through, which needs larger frames than the grid has)
REACHABLE = {
    ("v3", 2, 2, 0, 1), ("v3", 2, 4, 0, 1), ("v3", 2, 6, 0, 1), ("v3", 2, 8, 0, 1), ("v3", 4, 4, 4, 1), ("v3", 4, 6, 4, 1),
    ("v3", 4, 8, 4, 1), ("v3", 6, 4, 0, 1), ("v3", 6, 6, 0, 1), ("v3", 6, 8, 0, 1), ("v3", 8, 6, 0, 1), ("v3", 8, 8, 0, 1),
    ("planar", 2, 2, 0, 1), ("planar", 2, 4, 0, 1), ("planar", 2, 6, 0, 1), ("planar", 2, 8, 0, 1), ("planar", 4, 4, 4, 1),
    ("planar", 4, 6, 4, 1), ("planar", 4, 8, 4, 1), ("planar", 6, 4, 0, 1), ("planar", 6, 6, 0, 1), ("planar", 6, 8, 0, 1),
    ("planar", 8, 6, 0, 1), ("planar", 8, 8, 0, 1),
    ("fixed", 2, 2, 0, 1), ("fixed", 2, 4, 0, 1), ("fixed", 2, 6, 0, 1), ("fixed", 2, 8, 0, 1), ("fixed", 4, 2, 3, 1),
    ("fixed", 4, 4, 3, 1), ("fixed", 4, 4, 4, 1), ("fixed", 4, 6, 3, 1), ("fixed", 4, 6, 4, 1), ("fixed", 4, 8, 3, 1),
    ("fixed", 4, 8, 4, 1), ("fixed", 6, 4, 0, 1), ("fixed", 6, 6, 0, 1), ("fixed", 6, 8, 0, 1), ("fixed", 8, 4, 0, 1),
    ("fixed", 8, 6, 0, 1), ("fixed", 8, 8, 0, 1),
    ("fixed", 2, 2, 0, 0), ("fixed", 2, 4, 0, 0), ("fixed", 2, 6, 0, 0), ("fixed", 4, 2, 3, 0), ("fixed", 4, 2, 4, 0),
    ("fixed", 4, 4, 3, 0), ("fixed", 4, 4, 4, 0), ("fixed", 4, 6, 3, 0), ("fixed", 4, 6, 4, 0), ("fixed", 4, 8, 3, 0),
    ("fixed", 4, 8, 4, 0), ("fixed", 6, 2, 0, 0), ("fixed", 6, 4, 0, 0), ("fixed", 6, 6, 0, 0), ("fixed", 6, 8, 0, 0),
    ("fixed", 8, 2, 0, 0), ("fixed", 8, 4, 0, 0), ("fixed", 8, 6, 0, 0), ("fixed", 8, 8, 0, 0),
    ("tp_v", 0, 0, 0, 1), ("tp_v", 8, 8, 0, 1), ("tp_h1s", 0, 0, 0, 0), ("tp_h1s", 8, 8, 0, 0), ("tp_h1f", 0, 0, 0, 0),
    ("tp_h1f", 8, 8, 0, 0), ("tp_h1", 0, 0, 0, 0), ("copy", 0, 0, 0, 1), ("copy4", 0, 0, 0, 1),
}
# tap-class instantiations default dispatch cannot reach, with the reason
_W3 = "widest 3 occurs for 3-pixel source rows only (3 -> 1, 3 -> 2), and v3 / planar need iw % 4 == 0"
_VUP = "a vertical enlargement (vc = 2) under a horizontal shrink of 4 or more taps runs the horizontal pass first"
_V4H8 = "vc = 4 is a shrink by at most 4 / 3 (or a 4-row source); with 7-8 horizontal taps the cost model runs horizontal first"
UNREACHABLE = {
    **{(r, 4, vc, 3, 1): _W3 for r in ("v3", "planar") for vc in (2, 4, 6, 8)},
    **{(r, hc, 2, 4 if hc == 4 else 0, 1): _VUP for r in ("v3", "planar") for hc in (4, 6, 8)},
    ("fixed", 4, 2, 4, 1): _VUP, ("fixed", 6, 2, 0, 1): _VUP, ("fixed", 8, 2, 0, 1): _VUP,
    ("v3", 8, 4, 0, 1): _V4H8, ("planar", 8, 4, 0, 1): _V4H8,
    ("fixed", 2, 8, 0, 0): "a vertical shrink of 7-8 taps under a horizontal enlargement runs the vertical pass first",
}

# one geometry per reachable class: (iw, ih, ow, oh, fast); v3 needs fast, planar and fixed take either
CLASS_GEOMS = {
    ("v3", 2, 2, 0, 1): (64, 64, 65, 65), ("v3", 2, 4, 0, 1): (64, 33, 65, 32), ("v3", 2, 6, 0, 1): (44, 44, 45, 31),
    ("v3", 2, 8, 0, 1): (44, 44, 45, 24), ("v3", 4, 4, 4, 1): (64, 33, 63, 32), ("v3", 4, 6, 4, 1): (44, 44, 43, 31),
    ("v3", 4, 8, 4, 1): (44, 44, 43, 24), ("v3", 6, 4, 0, 1): (64, 33, 58, 32), ("v3", 6, 6, 0, 1): (44, 44, 31, 31),
    ("v3", 6, 8, 0, 1): (44, 44, 31, 24), ("v3", 8, 6, 0, 1): (44, 44, 27, 31), ("v3", 8, 8, 0, 1): (44, 44, 24, 24),
    ("planar", 2, 2, 0, 1): (8, 33, 9, 34), ("planar", 2, 4, 0, 1): (8, 33, 9, 32), ("planar", 2, 6, 0, 1): (4, 44, 5, 31),
    ("planar", 2, 8, 0, 1): (4, 44, 5, 24), ("planar", 4, 4, 4, 1): (8, 33, 7, 32), ("planar", 4, 6, 4, 1): (4, 44, 3, 31),
    ("planar", 4, 8, 4, 1): (4, 44, 3, 24), ("planar", 6, 4, 0, 1): (12, 33, 10, 32), ("planar", 6, 6, 0, 1): (8, 33, 5, 23),
    ("planar", 6, 8, 0, 1): (8, 33, 5, 18), ("planar", 8, 6, 0, 1): (8, 33, 4, 23), ("planar", 8, 8, 0, 1): (8, 33, 3, 18),
    ("fixed", 2, 2, 0, 1): (1, 1, 2, 2), ("fixed", 2, 4, 0, 1): (1, 3, 2, 1), ("fixed", 2, 6, 0, 1): (1, 5, 2, 2),
    ("fixed", 2, 8, 0, 1): (1, 7, 2, 2), ("fixed", 4, 2, 3, 1): (3, 2, 1, 1), ("fixed", 4, 4, 3, 1): (3, 3, 1, 1),
    ("fixed", 4, 4, 4, 1): (4, 3, 1, 1), ("fixed", 4, 6, 3, 1): (3, 5, 1, 2), ("fixed", 4, 6, 4, 1): (4, 5, 2, 2),
    ("fixed", 4, 8, 3, 1): (3, 7, 1, 2), ("fixed", 4, 8, 4, 1): (4, 7, 1, 2), ("fixed", 6, 4, 0, 1): (5, 4, 2, 2),
    ("fixed", 6, 6, 0, 1): (5, 5, 2, 2), ("fixed", 6, 8, 0, 1): (5, 7, 2, 2), ("fixed", 8, 4, 0, 1): (8, 5, 4, 4),
    ("fixed", 8, 6, 0, 1): (7, 5, 2, 2), ("fixed", 8, 8, 0, 1): (7, 7, 2, 2),
    ("fixed", 2, 2, 0, 0): (1, 1, 3, 2), ("fixed", 2, 4, 0, 0): (2, 7, 1, 6), ("fixed", 2, 6, 0, 0): (2, 20, 1, 18),
    ("fixed", 4, 2, 3, 0): (3, 1, 1, 2), ("fixed", 4, 2, 4, 0): (4, 1, 1, 2), ("fixed", 4, 4, 3, 0): (3, 3, 1, 2),
    ("fixed", 4, 4, 4, 0): (4, 3, 1, 2), ("fixed", 4, 6, 3, 0): (3, 5, 1, 3), ("fixed", 4, 6, 4, 0): (4, 5, 1, 2),
    ("fixed", 4, 8, 3, 0): (3, 12, 1, 7), ("fixed", 4, 8, 4, 0): (4, 7, 1, 3), ("fixed", 6, 2, 0, 0): (5, 1, 2, 2),
    ("fixed", 6, 4, 0, 0): (5, 3, 2, 1), ("fixed", 6, 6, 0, 0): (5, 7, 2, 5), ("fixed", 6, 8, 0, 0): (5, 7, 3, 2),
    ("fixed", 8, 2, 0, 0): (7, 1, 2, 2), ("fixed", 8, 4, 0, 0): (7, 3, 2, 1), ("fixed", 8, 6, 0, 0): (7, 5, 2, 3),
    ("fixed", 8, 8, 0, 0): (7, 8, 2, 4),
    ("tp_v", 0, 0, 0, 1): (1, 12, 2, 4), ("tp_v", 8, 8, 0, 1): (114, 115, 60, 61), ("tp_h1s", 0, 0, 0, 0): (44, 12, 31, 4),
    ("tp_h1s", 8, 8, 0, 0): (379, 127, 196, 82), ("tp_h1f", 0, 0, 0, 0): (4, 12, 1, 5), ("tp_h1f", 8, 8, 0, 0): (132, 4578, 66, 2813),
    ("tp_h1", 0, 0, 0, 0): (2000, 100, 28, 50), ("copy", 0, 0, 0, 1): (130, 64, 130, 64), ("copy4", 0, 0, 0, 1): (128, 64, 128, 64),
}


def class_key(s):
    return (s["route"], s["hc"], s["vc"], s["h_widest"] if s["hc"] == 4 else 0, s["vertical_first"])


def shape(case):
    return timg_b200.scale_shape(case.iw, case.ih, case.ow, case.oh, 1, case.fast, case.src_off % 16 == 0, True)


def apply_env(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def check_class(case):
    """The case's shape; fails unless it is in the class it is named after."""
    s = shape(case)
    for k, v in case.expect.items():
        got = class_key(s) if k == "class" else s[k]
        assert got == v, f"{case.group}/{case.name}: {k} = {got}, the case is there for {v} ({s})"
    return s


def frame(case, i=0):
    """Frame i of the case: RGBA [ih, iw, 4] (RGB32 cases read the same bytes as BGRA)."""
    w, h, seed = case.iw, case.ih, 7000 + 7919 * i + zlib.crc32(case.name.encode()) % 1000
    k = case.kind
    if k in ("photo", "noise", "noisea", "alpha"):
        return synth.frame_np(seed, w, h, k)
    fb = synth.frame_np(seed, w, h, "photo" if k != "faint" else "noisea")
    rng = np.random.default_rng(seed)
    if k == "holes":                                  # patches of alpha 0 and alpha 1 in an opaque photo
        for a in (0, 1, 0, 1):
            x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
            fb[y0:y0 + max(1, h // 3), x0:x0 + max(1, w // 3), 3] = a
    elif k == "edgepx":                               # one transparent pixel on the first column / row of tile 1's window
        x, y = min(w - 1, 4 * ((w * 32 // max(1, case.ow)) // 4)), min(h - 1, h * 32 // max(1, case.oh))
        fb[y, x, 3] = 0
        fb[0, w - 1, 3] = 0
    elif k == "taporder":                             # opaque rows whose 3-tap sums round differently in the other order
        fb[..., 3] = 255
        rows = tap_order_rows(case)
        fb[..., :3] = rows[np.arange(h * 3) % len(rows)].reshape(h, 3, 3).transpose(0, 2, 1)
    elif k == "clear":                                # fully transparent, colour left in place
        fb[..., 3] = 0
    elif k == "faint":                                # alpha below 255 everywhere
        fb[..., 3] = 1 + fb[..., 3] % 254
    else:
        raise ValueError(k)
    return fb


def tap_order_rows(case):
    """Byte triples (p0, p1, p2) of a 3-pixel row for which output column 0's opaque colour encodes to another byte when its
    three horizontal taps are summed ((t0 + t2) + t1, two accumulators) instead of in order ((t0 + t1) + t2, h_sequential):
    float32 products and sums as the kernels do them, p0 in 1..8."""
    p = timg_b200.resample_plan(case.iw, case.ih, case.ow, case.oh, 0)
    assert p["first"][0] == 0 and p["count"][0] == 3
    f32 = np.float32
    cf = p["coeff"][0].astype(f32)
    a = f32(255) * f32(1 / 255.0)
    k0, k1, k2 = np.meshgrid(np.arange(1, 9), np.arange(256), np.arange(256), indexing="ij")
    x = [(k.astype(f32) * f32(1 / 255.0)) * a * cf[i] for i, k in enumerate((k0, k1, k2))]

    def enc(v, A):
        return np.trunc(np.clip((v * (f32(1) / A)) * f32(255) + f32(0.5), 0, 255))

    differ = enc((x[0] + x[1]) + x[2], (a * cf[0] + a * cf[1]) + a * cf[2]) != enc((x[0] + x[2]) + x[1], (a * cf[0] + a * cf[2]) + a * cf[1])
    rows = np.stack([k0[differ], k1[differ], k2[differ]], -1).astype(np.uint8)
    assert len(rows) >= 16, len(rows)
    return rows


def cases():
    out = []

    def add(group, name, g, expect, kind="photo", fmt=None, fast=None, src_off=0):
        iw, ih, ow, oh = g[:4]
        if fast is None:
            fast = expect.get("route") == "v3" or expect.get("class", ("",))[0] == "v3"
        out.append(Case(group, name, iw, ih, ow, oh, kind, len(out) % 2 if fmt is None else fmt, bool(fast), expect, src_off))

    # ---- every reachable tap-class instantiation; content rotates through the kinds
    for j, (key, g) in enumerate(sorted(CLASS_GEOMS.items(), key=str)):
        route, hc, vc, hw, vf = key
        add("class", f"{route}-{hc}x{vc}" + (f"-w{hw}" if hw else "") + ("-vfirst" if route == "fixed" and vf else "")
            + f"-{g[0]}x{g[1]}-{g[2]}x{g[3]}", g, {"class": key}, kind=KINDS[j % len(KINDS)])
    # ---- both sides of every threshold
    T = [
        ("planar-smem-in", (200, 200, 114, 114), {"route": "planar", "planar_reuse": 1}),
        ("planar-smem-out", (200, 200, 113, 114), {"route": "fixed", "planar_reuse": 1}),
        ("planar-reuse-in", (100, 100, 198, 198), {"route": "fixed", "planar_reuse": 1}),
        ("planar-reuse-out", (100, 100, 199, 199), {"route": "fixed", "planar_reuse": 0}),
        ("planar-reuse-in-vf", (128, 100, 132, 104), {"route": "planar", "planar_reuse": 1}),
        ("v3-reuse-in", (128, 100, 132, 104), {"route": "v3", "v3_reuse": 1}),
        ("v3-reuse-out", (128, 100, 133, 104), {"route": "planar", "v3_reuse": 0}),
        ("v3-smem-largest", (116, 114, 61, 60), {"route": "v3"}),
        ("fixed-smem-in", (113, 115, 60, 61), {"route": "fixed"}),
        ("fixed-smem-out-8x8", (114, 115, 60, 61), {"route": "tp_v", "h_widest": 8, "v_widest": 8}),
        ("h1s-smem-in", (3776, 100, 256, 50), {"route": "tp_h1s"}),
        ("h1s-smem-out", (3780, 100, 256, 50), {"route": "tp_h1"}),
        ("h1s-tiles-full-out", (2000, 100, 27, 50), {"route": "tp_h1f", "tiles_full": 0}),
        ("h1s-tiles-full-in", (2000, 100, 28, 50), {"route": "tp_h1", "tiles_full": 1}),
        ("h1s-tiles-full-in-small", (400, 100, 28, 50), {"route": "tp_h1s", "tiles_full": 1}),
        ("h1s-tiles-full-out-small", (400, 100, 27, 50), {"route": "tp_h1f", "tiles_full": 0}),
        ("h1-ow4096", (65536, 4, 4096, 1), {"route": "tp_h1", "tiles_full": 1}),
        ("h1-ow4097", (65540, 4, 4097, 1), {"route": "tp_h1", "tiles_full": 1}),
        ("iw-mod4-0", (640, 360, 450, 253), {"route": "planar"}),
        ("iw-mod4-1", (641, 360, 450, 253), {"route": "fixed"}),
        ("iw-mod4-2", (642, 360, 450, 253), {"route": "fixed"}),
        ("copy4-ow-mod4-0", (128, 30, 128, 30), {"route": "copy4"}),
        ("copy-ow-mod4-2", (130, 30, 130, 30), {"route": "copy"}),
        ("copy-ow-mod4-1", (33, 7, 33, 7), {"route": "copy"}),
    ]
    for j, (name, g, expect) in enumerate(T):
        add("threshold", name, g, expect, kind=("photo", "noisea", "holes")[j % 3], fast=expect.get("route") == "v3")
    # ---- filter modes
    F = [
        ("point-h-mitchell-v", (100, 80, 100, 60), {"h_filter": 0, "v_filter": 2}),
        ("point-v-box-h", (50, 40, 75, 40), {"h_filter": 1, "v_filter": 0}),
        ("box-integer-2x", (50, 40, 100, 80), {"h_filter": 1, "v_filter": 1}),
        ("box-noninteger", (50, 40, 75, 61), {"h_filter": 1, "v_filter": 1}),
        ("mitchell-ratio-1.99", (199, 199, 100, 100), {"h_filter": 2, "v_filter": 2}),
        ("mitchell-ratio-2.01", (201, 201, 100, 100), {"h_filter": 2, "v_filter": 2}),
        ("scatter-v", (100, 900, 50, 100), {"v_gather": 0, "route": "tp_v"}),
        ("scatter-v-h-first", (640, 900, 67, 100), {"v_gather": 0}),
        ("lead-nonzero", (100, 80, 37, 80), {"h_widest": 11}),
        ("lead-small", (10, 10, 7, 7), {"route": "fixed"}),
    ]
    for j, (name, g, expect) in enumerate(F):
        add("filter", name, g, expect, kind=("noisea", "photo", "holes", "edgepx", "faint")[j % 5], fast=False)
    # ---- tile edges: output widths / heights around the 32 / 64 and 16 / 32 tile sizes, sources of 1 to 4 pixels
    for ow in (1, 31, 32, 33, 63, 64, 65):
        add("edge", f"ow{ow}", (int(ow * 1.3) + 4, 52, ow, 40), {}, kind="noisea")
    for oh in (1, 15, 16, 17, 31, 32, 33):
        add("edge", f"oh{oh}", (52, int(oh * 1.3) + 4, 40, oh), {}, kind="holes")
    for n in (1, 2, 3, 4):
        add("edge", f"iw{n}", (n, 40, 37, 29), {}, kind="noisea")
        add("edge", f"ih{n}", (40, n, 29, 37), {}, kind="noisea")
    add("edge", "partial-both-planar", (160, 140, 97, 81), {"route": "planar"}, kind="edgepx")
    add("edge", "partial-both-v3", (160, 140, 97, 81), {"route": "v3"}, kind="edgepx", fast=True)
    add("edge", "partial-both-fixed", (161, 140, 97, 81), {"route": "fixed"}, kind="edgepx")
    # ---- h_sequential (one horizontal accumulator, widest 3: 3-pixel rows only) on many output rows, both pass orders
    # (the order of three taps changes a byte only near a rounding edge, which noise meets by chance: the taporder rows
    # are chosen to sit on such edges)
    add("filter", "hseq-w3-taporder-3x512", (3, 512, 2, 512), {"class": ("fixed", 4, 2, 3, 0), "h_sequential": 1}, kind="taporder")
    add("filter", "hseq-w3-vfirst-3x2000", (3, 2000, 2, 1500), {"class": ("fixed", 4, 6, 3, 1), "h_sequential": 1}, kind="noise")
    add("filter", "hseq-w3-hfirst-3x2000", (3, 2000, 2, 3000), {"class": ("fixed", 4, 2, 3, 0), "h_sequential": 1}, kind="noisea")
    # ---- content on the routes the v3 / planar split depends on
    for kind in KINDS:
        add("content", f"v3-{kind}", (640, 360, 450, 253), {"route": "v3"}, kind=kind, fast=True)
        add("content", f"planar-{kind}", (640, 360, 450, 253), {"route": "planar"}, kind=kind)
        add("content", f"tp_h1s-{kind}", (3840, 200, 337, 18), {"route": "tp_h1s"}, kind=kind)
    return out


def by_name(group):
    return {c.name: c for c in cases() if c.group == group}


def names(group):
    return [c.name for c in cases() if c.group == group]


def shape_raw(iw, ih, ow, oh, fast, s=None):
    """The class key of one geometry through the ABI directly (the host test walks tens of thousands of them)."""
    s = s or timg_b200.ScaleShape()
    rc = timg_b200.lib().b200timg_scale_shape_of(iw, ih, ow, oh, 1, fast, 1, 1, C.byref(s))
    assert rc == timg_b200.OK
    return (timg_b200.SCALE_ROUTES[s.route], s.hc, s.vc, s.h_widest if s.hc == 4 else 0, s.vertical_first)


def ref_f64(img, ow, oh, fmt=0):
    """Plain float64 statement of the scaler from the tables timg_b200.resample_plan exports: decode byte / 255, premultiply
    by alpha, the two 1-D sums (tap i of output x reads input first[x] + i with coeff[x][i]), un-weight by the filtered
    alpha unless it is below 2^-120 (then the filtered un-weighted colour), encode trunc(clamp(v * 255 + 0.5)).  Summation
    order does not matter at this precision, so it checks the kernels independently of the STB restatement's float32 order."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    ih, iw = img.shape[:2]
    px = img.astype(np.float64) / 255.0
    if fmt == timg_b200.FMT_RGB32:
        px = px[..., [2, 1, 0, 3]]
    a = px[..., 3:4]
    planes = np.concatenate([px[..., :3] * a, a, px[..., :3]], -1)         # R*A G*A B*A A R G B

    def axis_sum(axis, x, along):
        """The 1-D filter of one axis over dimension `along` of x, as a gather of every tap (padded taps weigh 0)."""
        p = timg_b200.resample_plan(iw, ih, ow, oh, axis)
        n_in = x.shape[along]
        acc = 0.0
        for i in range(p["coeff"].shape[1]):
            w = p["coeff"][:, i].astype(np.float64) * (i < p["count"])
            idx = np.minimum(p["first"] + i, n_in - 1)
            tap = np.take(x, idx, axis=along)
            acc = acc + tap * (w[:, None, None] if along == 0 else w[None, :, None])
        return acc

    r = axis_sum(0, axis_sum(1, planes, 0), 1)
    A = r[..., 3:4]
    hole = A < 2.0 ** -120
    rgb = np.where(hole, r[..., 4:7], r[..., :3] / np.where(hole, 1.0, A))
    out = np.concatenate([rgb, A], -1)
    return np.trunc(np.clip(out * 255.0 + 0.5, 0, 255)).astype(np.uint8)
