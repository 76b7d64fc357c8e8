"""Case table of the sixel launch-shape matrix (tests/test_sixel_shapes_gpu.py runs it on the device, tests/test_sixel_shapes.py
checks on the host that it covers every class).  A case names the launch shape it is there for in `expect`: fields of
b200timg_sixel_shape plus the classes derived() adds.  The shape is always asked of the library (timg_b200.sixel_shape, the
launchers' own arithmetic), with the SM count of the device at hand, so a moved threshold fails the case instead of quietly
turning it into a test of something else."""
from collections import namedtuple

import numpy as np

import timg_b200
from timg_b200 import synth

# n frames launched out of a batch of n_total; env: the knobs the launch runs under; diffuse: True = more than 256 sampled
# cells (median cut + Floyd-Steinberg), False = at most 256 (table lookup per pixel), None = not asserted
Case = namedtuple("Case", "group name kind w h seed n n_total env expect diffuse")

KNOBS = ("B200TIMG_DITHER_SPLIT", "B200TIMG_DITHER_WARPS", "B200TIMG_DITHER_SPIN", "B200TIMG_DITHER_V1", "B200TIMG_PARTS",
         "B200TIMG_EMIT", "B200TIMG_EMIT_V2", "B200TIMG_EMIT_MATCH")
SM_COUNTS = (132, 114, 108)          # H100 SXM, H100 PCIe and a smaller part: the host-side coverage check walks the table for each

PALETTE_CLASSES = ("step6", "step1_shared", "step1_global", "step1_global_saturated", "step2_shared", "step2_global", "step3plus")
# first pixel count of the class to the right of each edge: sampling step 6 -> 1, tables shared -> global (25600 entries),
# entries saturate at 32768, step 1 -> 2, shared -> global again (2 * 25600 pixels), step 2 -> 3
PALETTE_EDGES = (18383, 25601, 32769, 36766, 51201, 55149)
WIDTHS = (1, 2, 3, 15, 16, 17, 31, 32, 33, 61, 62, 63, 64, 65, 79, 80, 81, 82, 95, 96, 97)
LAST_BAND_ROWS = {102: 6, 108: 12, 114: 18, 120: 24, 126: 30, 96: 32}      # frame height -> live rows of its last band


def palette_class(s):
    if s["step_px"] == 6:
        return "step6"
    if s["step_px"] >= 3:
        return "step3plus"
    tables = "global" if s["palette_global"] else "shared"
    return "step%d_%s%s" % (s["step_px"], tables, "_saturated" if s["ent_cap"] == 32768 else "")


def derived(s):
    """The shape plus the classes that follow from it: bands of each dither CTA of a frame and how they are handed over."""
    d = dict(s)
    sizes = [min(s["bands_per_cta"], s["nb32"] - g * s["bands_per_cta"]) for g in range(s["dither_ctas"])]
    d["palette"] = palette_class(s)
    d["short_last_cta"] = sizes[-1] < sizes[0]
    d["single_band_cta"] = len(sizes) > 1 and 1 in sizes
    d["remote_and_local"] = any(n >= 2 for n in sizes[1:])     # a CTA whose first band waits on another CTA, its second on a warp
    return d


def apply_env(monkeypatch, case):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env.items():
        monkeypatch.setenv(k, str(v))


def check_class(case, sm_count):
    """The case's shape on a device of sm_count SMs (call under apply_env); fails unless it is in the class it is named after."""
    d = derived(timg_b200.sixel_shape(case.w, case.h, case.n, case.n_total, sm_count))
    for k, v in case.expect.items():
        assert d[k] == v, f"{case.group}/{case.name} on {sm_count} SMs: {k} = {d[k]}, the case is there for {v} ({d})"
    if case.n_total < sm_count:
        assert d["dither_ctas"] * case.n <= sm_count, f"{case.group}/{case.name}: split CTAs of a launch must be co-resident"
    return d


def frame(case, i=0):
    """Frame i of the case: RGBA [h, w, 4], alpha 255."""
    w, h, seed = case.w, case.h, case.seed + 7919 * i
    if case.kind in ("noise", "photo"):
        return synth.frame_np(seed, w, h, case.kind)
    y, x = np.mgrid[0:h, 0:w]
    fb = np.empty((h, w, 4), np.uint8)
    fb[..., 3] = 255
    if case.kind.startswith("cells"):                # cellsN: N colours in distinct 15-bit cells, in noise order
        n = int(case.kind[5:])
        c = synth.frame_np(seed, w, h, "noise")[..., 0].astype(np.int64) % n
        fb[..., 0], fb[..., 1], fb[..., 2] = (c % 32) * 8 + 3, (c // 32) * 8 + 5, 64 + (c % 3) * 8
    elif case.kind == "allcells":                    # every 15-bit cell at least once: the histogram is full
        c = ((y * w + x) * 12347 + seed) % 32768
        low = synth.frame_np(seed, w, h, "noise")[..., :3] & 7
        fb[..., 0], fb[..., 1], fb[..., 2] = (c >> 10) * 8 + low[..., 0], ((c >> 5) & 31) * 8 + low[..., 1], (c & 31) * 8 + low[..., 2]
    elif case.kind == "runs":                        # runs of 1000 columns, shifted from row to row: they cross every tile edge
        c = ((x + 37 * y + seed) // 1000) % 5
        fb[..., 0], fb[..., 1], fb[..., 2] = 40 + 48 * c, 200 - 40 * c, 16 * c
    elif case.kind == "solid":
        fb[..., :3] = (40, 80, 120)
    else:
        raise ValueError(case.kind)
    return fb


def _up6(v):
    return (v + 5) // 6 * 6


def cases(sm):
    """Every case for a device of sm SMs.  Names do not depend on sm; batch sizes and the natural splits of tall frames do."""
    out = []

    def add(group, name, kind, w, h, expect, env=None, n=1, n_total=None, diffuse=None, seed=None):
        out.append(Case(group, name, kind, w, h, 1000 + len(out) if seed is None else seed, n, n if n_total is None else n_total,
                        env or {}, expect, diffuse))

    # ---- palette: sampling step x where the median-cut tables live, and both sides of every edge
    for cls, w, h in (("step6", 200, 60), ("step1_shared", 160, 132), ("step1_global", 200, 150), ("step1_global_saturated", 180, 186),
                      ("step2_shared", 220, 192), ("step2_global", 230, 228), ("step3plus", 337, 192)):
        for kind in ("noise", "photo"):
            add("palette", f"{cls}-{kind}-{w}x{h}", kind, w, h, {"palette": cls}, diffuse=True)
    add("palette", "step3plus-noise-400x240", "noise", 400, 240, {"palette": "step3plus", "step_px": 5}, diffuse=True)
    for cls, w, h in (("step6", 1021, 18), ("step1_shared", 383, 48), ("step1_shared", 474, 54), ("step1_global", 251, 102),
                      ("step1_global", 127, 258), ("step1_global_saturated", 2731, 12), ("step1_global_saturated", 557, 66),
                      ("step2_shared", 383, 96), ("step2_shared", 371, 138), ("step2_global", 251, 204), ("step2_global", 707, 78),
                      ("step3plus", 383, 144)):
        add("palette", f"edge-{cls}-{w}x{h}", "noise", w, h, {"palette": cls}, diffuse=True)
    add("palette", "fewcolours-4-global-200x150", "cells4", 200, 150, {"palette": "step1_global"}, diffuse=False)
    add("palette", "fewcolours-200-saturated-180x186", "cells200", 180, 186, {"palette": "step1_global_saturated"}, diffuse=False)
    add("palette", "fullhistogram-2731x12", "allcells", 2731, 12, {"palette": "step1_global_saturated", "ent_cap": 32768}, diffuse=True)

    # ---- dither, one frame: rounds, splits, hand-overs, last-band rows, widths around the kernel's constants
    for warps, rounds, kind in ((5, 2, "noise"), (2, 4, "photo"), (1, 7, "noise")):
        add("dither", f"rounds{rounds}-warps{warps}", kind, 100, 198, {"nb32": 7, "dither_ctas": 1, "dither_rounds": rounds},
            {"B200TIMG_DITHER_WARPS": warps}, diffuse=True)
    for split, h, expect in ((2, 198, {"dither_ctas": 2, "bands_per_cta": 4, "short_last_cta": True, "remote_and_local": True}),
                             (2, 192, {"dither_ctas": 2, "bands_per_cta": 3, "short_last_cta": False}),
                             (3, 198, {"dither_ctas": 3, "bands_per_cta": 3, "single_band_cta": True}),
                             (4, 198, {"dither_ctas": 4, "bands_per_cta": 2, "single_band_cta": True, "remote_and_local": True}),
                             (5, 288, {"dither_ctas": 5, "bands_per_cta": 2, "short_last_cta": True}),
                             (6, 330, {"dither_ctas": 6, "bands_per_cta": 2, "short_last_cta": True}),
                             (7, 198, {"dither_ctas": 7, "bands_per_cta": 1, "remote_and_local": False})):
        for kind, w in (("noise", 100), ("photo", 203)):
            add("dither", f"split{split}-{kind}-{w}x{h}", kind, w, h, dict(expect, dither_rounds=1), {"B200TIMG_DITHER_SPLIT": split},
                diffuse=True)
    add("dither", "split2-rounds2", "noise", 100, 198, {"dither_ctas": 2, "dither_rounds": 2, "dither_warps": 2},
        {"B200TIMG_DITHER_SPLIT": 2, "B200TIMG_DITHER_WARPS": 2}, diffuse=True)
    add("dither", "split3-rounds3-warps1", "photo", 203, 198, {"dither_ctas": 3, "dither_rounds": 3, "dither_warps": 1},
        {"B200TIMG_DITHER_SPLIT": 3, "B200TIMG_DITHER_WARPS": 1}, diffuse=True)
    add("dither", "split3-spin0", "noise", 100, 198, {"dither_ctas": 3}, {"B200TIMG_DITHER_SPLIT": 3, "B200TIMG_DITHER_SPIN": 0},
        diffuse=True)
    for h, rows in LAST_BAND_ROWS.items():
        add("dither", f"lastband{rows}-50x{h}", "noise", 50, h, {"nb32": (h + 31) // 32, "dither_ctas": 1}, diffuse=True)
    for w in WIDTHS:                                 # enough pixels for more than 256 sampled cells, at least 66 rows
        h = max(66, _up6(-(-2400 // w)))
        add("dither", f"width{w}-{w}x{h}", "noise", w, h, {}, diffuse=True)

    # ---- batches without knobs (frames of a batch differ: seed + 7919 * i)
    add("batch", "half-sm-split2", "noise", 96, 384, {"dither_ctas": 2, "bands_per_cta": 6, "dither_rounds": 1}, n=sm // 2, diffuse=True)
    add("batch", "sm-minus-1", "noise", 64, 36, {"dither_ctas": 1}, n=sm - 1, diffuse=True)
    add("batch", "sm-plus-5", "noise", 64, 36, {"dither_ctas": 1}, n=sm + 5, diffuse=True)
    add("batch", "natural-rounds2", "noise", 40, 804, {"dither_ctas": 1, "nb32": 26, "dither_rounds": 2, "dither_warps": 13,
                                                         "palette": "step1_global"}, n=sm, diffuse=True)
    for parts in (2, 4):
        add("batch", f"parts{parts}", "photo", 120, 288, {"dither_ctas": 2, "bands_per_cta": 5, "short_last_cta": True, "remote_and_local": True},
            {"B200TIMG_PARTS": parts}, n=8 // parts, n_total=8, diffuse=True)

    # ---- wide and tall frames, default emitter
    for w, tiles in ((4095, 1), (4096, 1), (4097, 2), (8192, 2), (8193, 3), (12289, 4)):
        expect = {"emit_mode": 5 if w <= 4095 else 2, "emit_tiles": tiles}
        add("wide", f"noise-{w}x6", "noise", w, 6, expect, diffuse=True)
        add("wide", f"noise-{w}x12", "noise", w, 12, expect, diffuse=True)
        add("wide", f"runs-{w}x12", "runs", w, 12, expect, diffuse=False)
        add("wide", f"solid-{w}x6", "solid", w, 6, expect, diffuse=False)
    add("wide", "tall-16x6144", "noise", 16, 6144, {"nb32": 192, "dither_ctas": min(sm, 24), "emit_mode": 5}, diffuse=True)
    per = min(sm, 256)
    bands = -(-2048 // per)
    add("wide", "tallest-4x65532", "noise", 4, 65532, {"nb32": 2048, "bands_per_cta": bands, "dither_ctas": -(-2048 // bands)}, diffuse=True)
    add("wide", "widest-99999x6", "runs", 99999, 6, {"emit_mode": 2, "emit_tiles": 25, "nb32": 1}, diffuse=False)

    # ---- output capacity contract of the uniform entry points
    add("capacity", "emit5-337x192", "photo", 337, 192, {"emit_mode": 5}, n=4)
    add("capacity", "emit2-4200x12", "noise", 4200, 12, {"emit_mode": 2, "emit_tiles": 2}, n=4)
    return out


def by_name(sm, group):
    return {c.name: c for c in cases(sm) if c.group == group}


def names(group):
    return [c.name for c in cases(SM_COUNTS[0]) if c.group == group]
