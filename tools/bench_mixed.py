#!/usr/bin/env python
"""Mixed batches on the GPU: a `timg --grid` page of differently sized images, block-, sixel- or kitty-encoded in one call
(b200timg_blocks_mixed_dev, b200timg_sixel_mixed_dev, b200timg_graphics_mixed_dev) against the ways to send it without
one.  One JSON line per page.

  python tools/bench_mixed.py [--steps K] [--warmup W] [--only NAME]

  grid8x8-quarter  --grid=8x8 -g300x100 -p quarter: 64 images, each fitted to the grid's 75 x 25 px box
  grid4x4-half     --grid=4x4 -g300x100 -p half: 16 images fitted to 75 x 50 px (larger outputs per image)
  grid4x4-sixel    --grid=4x4 -g300x100 -p sixel at 9 x 18 px cells: 16 images fitted to 675 x 450 px
  grid8x8-sixel    --grid=8x8 -g300x100 -p sixel at 9 x 18 px cells: 64 images fitted to 337 x 225 px
  grid8x8-kitty[-deflate]  --grid=8x8 -g300x100 -p kitty at 9 x 18 px cells (tmux off, rgb24): 64 images fitted to
                   337 x 225 px, stored-block PNGs (timg's --compress 0) or B200TIMG_DEFLATE (its default, level 1)
  grid4x4-kitty[-deflate]  the same at --grid=4x4: 16 images fitted to 675 x 450 px
Source sizes cycle through 3840x2160, 2160x3840, 4032x3024, 3000x2000, 1920x1080, 1280x720, 1080x1080 and 640x480
(every image's pixels distinct); indents are the renderer's column offsets (src/renderer.cc:124-142).

Timed, alternating within each step, every call ending in a device-wide synchronise:
  (a) mixed     one b200timg_blocks_mixed_dev (sixel pages: b200timg_sixel_mixed_dev, kitty pages:
                b200timg_graphics_mixed_dev) call for the page
  (b) per_image one b200timg_blocks_batch_dev (b200timg_sixel_batch_dev, b200timg_graphics_batch_dev) call per image
                (n_frames = 1): the status quo
  (c) per_geom  one uniform batch call per distinct geometry (sources regrouped by geometry)
  (d) the cost of generality: C3 geometry (1920x1080 -> 320x90, -p quarter, 64 frames) through the mixed call against
      b200timg_blocks_batch_dev, and C4's (3840x2160 -> 337x190, -p sixel, 64 frames) through the sixel mixed call
      against b200timg_sixel_batch_dev with flags = 0, and C4's through the kitty mixed call (stored and deflate) against
      b200timg_graphics_batch_dev with flags = 0
(a), (b) and (c) must produce the same bytes for every image (asserted); so must both sides of (d).  Per-kernel ms of one
(a) and one (b) page come from b200timg_profile in a separate run.  The GPU's name, power limit and max SM clock are read
in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import timg_b200  # noqa: E402
from timg_b200 import synth  # noqa: E402

SIZES = [(3840, 2160), (2160, 3840), (4032, 3024), (3000, 2000), (1920, 1080), (1280, 720), (1080, 1080), (640, 480)]
PAGES = {
    "grid8x8-quarter": dict(cols=8, rows=8, term=(300, 100), quarter=True),
    "grid4x4-half": dict(cols=4, rows=4, term=(300, 100), quarter=False),
    "grid4x4-sixel": dict(cols=4, rows=4, term=(300, 100), quarter=False, sixel=True),
    "grid8x8-sixel": dict(cols=8, rows=8, term=(300, 100), quarter=False, sixel=True),
    "grid8x8-kitty": dict(cols=8, rows=8, term=(300, 100), quarter=False, kitty=True, deflate=False),
    "grid8x8-kitty-deflate": dict(cols=8, rows=8, term=(300, 100), quarter=False, kitty=True, deflate=True),
    "grid4x4-kitty": dict(cols=4, rows=4, term=(300, 100), quarter=False, kitty=True, deflate=False),
    "grid4x4-kitty-deflate": dict(cols=4, rows=4, term=(300, 100), quarter=False, kitty=True, deflate=True),
}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                      # the numbers still stand, without their card
        return f"unavailable ({e})"


def page_layout(cfg):
    """(images' source sizes, fitted outputs, indents) of one page, as timg.cc:938-939 and renderer.cc lay it out."""
    pixels = cfg.get("sixel") or cfg.get("kitty")
    cx, cy = (9, 18) if pixels else (2, 2) if cfg["quarter"] else (1, 2)
    box_w = cfg["term"][0] * cx // cfg["cols"]
    box_h = cfg["term"][1] * cy // cfg["rows"]
    n = cfg["cols"] * cfg["rows"]
    srcs, outs, indents = [], [], []
    for i in range(n):
        iw, ih = SIZES[i % len(SIZES)]
        _, ow, oh = timg_b200.calc_fit(iw, ih, box_w, box_h, cx, cy)
        srcs.append((iw, ih))
        outs.append((ow, oh))
        indents.append(0 if pixels else (i % cfg["cols"]) * box_w // cx)   # UnicodeBlockCanvas::Send's x / cell_x_px
    return srcs, outs, indents


def device_images(torch, srcs):
    """One generated base image per size; image i is its base with a per-image byte rotation of the colours."""
    base = {s: synth.frame_torch(700 + k, s[0], s[1], "photo") for k, s in enumerate(SIZES)}
    imgs = []
    for i, s in enumerate(srcs):
        im = base[s].clone()
        im[..., :3] += (29 * (i // len(SIZES)) + 1) & 255
        imgs.append(im)
    return imgs


def pack(torch, imgs):
    sizes = [im.numel() for im in imgs]
    offs = np.cumsum([0] + sizes)
    flat = torch.empty(int(offs[-1]), dtype=torch.uint8, device="cuda")
    for im, o in zip(imgs, offs):
        flat[int(o):int(o) + im.numel()] = im.reshape(-1)
    return flat, [int(o) for o in offs[:-1]]


def timed(torch, fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def encoder(L, cfg, n):
    """(mixed call, uniform batch call, per-frame staging bound) of the block, sixel or kitty encoder.  Both calls take
    (ctx, batch, src, out, cap, offsets); the uniform one also the frames it encodes (kitty: their ids)."""
    if cfg.get("sixel"):
        return (L.b200timg_sixel_mixed_dev, lambda *a: L.b200timg_sixel_batch_dev(*a[:6]),
                lambda ow, oh: L.b200timg_sixel_bound(ow, (oh + 5) // 6 * 6))
    if cfg.get("kitty"):                       # -pk, tmux off, rgb24 (timg's default local_alpha_handling), 9 x 18 px cells
        proto = timg_b200.KITTY | (timg_b200.DEFLATE if cfg["deflate"] else 0)
        ids = (C.c_uint32 * n)(*range(1, n + 1))
        page = timg_b200.Graphics(proto, 1, C.cast(ids, C.POINTER(C.c_uint32)), 9, 18, 0)
        per_call = {}                          # the frames of a uniform call -> its description (built outside the timing)

        def uniform(h, b, src, out, cap, offs, members):
            key = tuple(members)
            if key not in per_call:
                arr = (C.c_uint32 * len(key))(*[ids[i] for i in key])
                per_call[key] = (timg_b200.Graphics(proto, 1, C.cast(arr, C.POINTER(C.c_uint32)), 9, 18, 0), arr)
            return L.b200timg_graphics_batch_dev(h, b, C.byref(per_call[key][0]), src, out, cap, offs)
        bound_g = timg_b200.Graphics(proto, 1, None, 9, 18, 0)
        return ((lambda h, b, *a, _keep=(ids, page): L.b200timg_graphics_mixed_dev(h, b, C.byref(page), *a)), uniform,
                lambda ow, oh: L.b200timg_graphics_size(C.byref(bound_g), ow, oh, 0xFFFFFFFF))
    return L.b200timg_blocks_mixed_dev, lambda *a: L.b200timg_blocks_batch_dev(*a[:6]), L.b200timg_blocks_bound


def run_page(name, cfg, steps, warmup, torch):
    L = timg_b200.lib()
    ctx = timg_b200.Context(0)
    flags = timg_b200.QUARTER if cfg["quarter"] else 0
    bg = timg_b200.rgba_u32(0, 0, 0)
    srcs, outs, indents = page_layout(cfg)
    n = len(srcs)
    mixed_fn, batch_fn, bound_fn = encoder(L, cfg, n)
    imgs = device_images(torch, srcs)
    flat, offs = pack(torch, imgs)
    torch.cuda.synchronize()                   # sources are written on torch's stream, read on the context's
    mb, keep = timg_b200.mixed_batch([(h, w) for w, h in srcs], outs, offs, indents, flags, has_bg=True, bg=bg)
    bounds = [bound_fn(ow, oh) for ow, oh in outs]
    cap = sum(bounds)
    d_out_a = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_offs_a = torch.empty(n + 1, dtype=torch.int64, device="cuda")

    def batch(iw, ih, ow, oh, nf, indent):
        return timg_b200.Batch(n_frames=nf, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=bg, pattern=0,
                               pattern_w=0, pattern_h=0, flags=flags, x_indent_cells=indent, animation=0)

    def run_a():
        ctx._chk(mixed_fn(ctx.h, C.byref(mb), flat.data_ptr(), d_out_a.data_ptr(), cap, d_offs_a.data_ptr()))

    # (b): one call per image, image i's bytes in its own slot
    slot = np.cumsum([0] + bounds)
    d_out_b = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_offs_b = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    b_batches = [batch(srcs[i][0], srcs[i][1], outs[i][0], outs[i][1], 1, indents[i]) for i in range(n)]

    def run_b():
        for i in range(n):
            ctx._chk(batch_fn(ctx.h, C.byref(b_batches[i]), flat.data_ptr() + offs[i],
                              d_out_b.data_ptr() + int(slot[i]), bounds[i], d_offs_b[i].data_ptr(), [i]))

    # (c): images regrouped by geometry; one uniform call per geometry (the indent is per call, so frames of a group
    # that sit in different columns would need one call each: the bytes are compared with indents folded in below)
    geoms = {}
    for i in range(n):
        geoms.setdefault((srcs[i], outs[i], indents[i]), []).append(i)
    order = [i for g in geoms.values() for i in g]
    flat_c, offs_c = pack(torch, [imgs[i] for i in order])
    torch.cuda.synchronize()
    d_out_c = torch.empty(cap, dtype=torch.uint8, device="cuda")
    c_calls, pos = [], 0
    for (src, out, indent), members in geoms.items():
        k = len(members)
        gcap = k * bound_fn(*out)
        c_calls.append((batch(src[0], src[1], out[0], out[1], k, indent), offs_c[pos], gcap,
                        torch.empty(k + 1, dtype=torch.int64, device="cuda"), members))
        pos += k
    c_base = np.cumsum([0] + [c[2] for c in c_calls])

    def run_c():
        for j, (b, o, gcap, d_o, members) in enumerate(c_calls):
            ctx._chk(batch_fn(ctx.h, C.byref(b), flat_c.data_ptr() + o, d_out_c.data_ptr() + int(c_base[j]), gcap, d_o.data_ptr(),
                              members))

    for _ in range(warmup):
        run_a(); run_b(); run_c()
    torch.cuda.synchronize()
    t = {"a": 0.0, "b": 0.0, "c": 0.0}
    for _ in range(steps):                     # alternating, one page each
        t["a"] += timed(torch, run_a, 1)
        t["b"] += timed(torch, run_b, 1)
        t["c"] += timed(torch, run_c, 1)
    t = {k: v / steps for k, v in t.items()}

    # same bytes, image by image
    oa, da = d_offs_a.cpu().numpy(), d_out_a.cpu().numpy()
    ob, db = d_offs_b.cpu().numpy(), d_out_b.cpu().numpy()
    dc = d_out_c.cpu().numpy()
    got_a = [da[oa[i]:oa[i + 1]].tobytes() for i in range(n)]
    got_b = [db[int(slot[i]) + ob[i][0]:int(slot[i]) + ob[i][1]].tobytes() for i in range(n)]
    got_c = [None] * n
    for j, (_, _, _, d_o, members) in enumerate(c_calls):
        oc = d_o.cpu().numpy()
        for k, i in enumerate(members):
            got_c[i] = dc[int(c_base[j]) + oc[k]:int(c_base[j]) + oc[k + 1]].tobytes()
    assert got_a == got_b, "mixed call differs from per-image calls"
    assert got_a == got_c, "mixed call differs from per-geometry calls"

    kernels = {}
    for key, fn in (("a", run_a), ("b", run_b)):
        ctx.profile(True)
        fn()
        kernels[key] = {k: [v[0], round(v[1], 4)] for k, v in ctx.profile_report().items()}
        ctx.profile(False)
    src_px = sum(w * h for w, h in srcs)
    res = dict(page=name, images=n, distinct_geometries=len({(s, o) for s, o in zip(srcs, outs)}), uniform_calls_c=len(c_calls),
               outs=sorted({f"{o[0]}x{o[1]}" for o in outs}), src_mpx=round(src_px / 1e6, 1), encoded_bytes=int(oa[-1]),
               steps=steps, same_bytes=True)
    for k, label in (("a", "mixed"), ("b", "per_image"), ("c", "per_geom")):
        res[f"{label}_ms"] = round(t[k], 3)
        res[f"{label}_mpx_s"] = round(src_px / t[k] / 1e3, 1)
    res["per_image_over_mixed"] = round(t["b"] / t["a"], 2)
    res["per_geom_over_mixed"] = round(t["c"] / t["a"], 2)
    res["kernels_ms_mixed"] = kernels["a"]
    res["kernels_ms_per_image"] = kernels["b"]
    ctx.close()
    return res


GENERALITY = {
    "C3-generality": dict(iw=1920, ih=1080, ow=320, oh=90, flags=timg_b200.QUARTER, sixel=False),
    "C4-generality": dict(iw=3840, ih=2160, ow=337, oh=190, flags=0, sixel=True),
    "C4-kitty-generality": dict(iw=3840, ih=2160, ow=337, oh=190, flags=0, kitty=True, deflate=False),
    "C4-kitty-deflate-generality": dict(iw=3840, ih=2160, ow=337, oh=190, flags=0, kitty=True, deflate=True),
}


def run_generality(name, g, steps, warmup, torch):
    """(d): one geometry through the mixed call and through the uniform batch."""
    L = timg_b200.lib()
    ctx = timg_b200.Context(0)
    mixed_fn, batch_fn, bound_fn = encoder(L, g, 64)
    n, iw, ih, ow, oh, indent, flags = 64, g["iw"], g["ih"], g["ow"], g["oh"], 0, g["flags"]
    bg = timg_b200.rgba_u32(0, 0, 0)
    base = synth.frame_torch(800, iw, ih, "photo")
    d_src = torch.empty((n, ih, iw, 4), dtype=torch.uint8, device="cuda")
    for f in range(n):
        d_src[f] = base
        d_src[f, ..., :3] += (37 * f + 1) & 255
    fbytes = iw * ih * 4
    mb, keep = timg_b200.mixed_batch([(ih, iw)] * n, [(ow, oh)] * n, [f * fbytes for f in range(n)], [indent] * n,
                                     flags, has_bg=True, bg=bg)
    ub = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=bg, pattern=0, pattern_w=0,
                         pattern_h=0, flags=flags, x_indent_cells=indent, animation=0)
    cap = n * bound_fn(ow, oh)
    outs = [torch.empty(cap, dtype=torch.uint8, device="cuda") for _ in range(2)]
    offs = [torch.empty(n + 1, dtype=torch.int64, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()

    def mixed():
        ctx._chk(mixed_fn(ctx.h, C.byref(mb), d_src.data_ptr(), outs[0].data_ptr(), cap, offs[0].data_ptr()))

    def uniform():
        ctx._chk(batch_fn(ctx.h, C.byref(ub), d_src.data_ptr(), outs[1].data_ptr(), cap, offs[1].data_ptr(), list(range(n))))
    for _ in range(warmup):
        mixed(); uniform()
    tm = tu = 0.0
    for _ in range(steps):
        tm += timed(torch, mixed, 1)
        tu += timed(torch, uniform, 1)
    tm, tu = tm / steps, tu / steps
    same = bool((offs[0] == offs[1]).all()) and bool((outs[0][:int(offs[0][-1])] == outs[1][:int(offs[1][-1])]).all())
    assert same, f"mixed call differs from the uniform batch ({name})"
    kernels = {}
    for key, fn in (("mixed", mixed), ("uniform", uniform)):
        ctx.profile(True)
        fn()
        kernels[key] = {k: [v[0], round(v[1], 4)] for k, v in ctx.profile_report().items()}
        ctx.profile(False)
    ctx.close()
    return dict(page=name, frames=n, src=f"{iw}x{ih}", out=f"{ow}x{oh}", steps=steps, same_bytes=same,
                mixed_ms=round(tm, 3), uniform_ms=round(tu, 3), mixed_over_uniform=round(tm / tu, 2),
                mixed_mpx_s=round(n * iw * ih / tm / 1e3, 1), uniform_mpx_s=round(n * iw * ih / tu / 1e3, 1),
                kernels_ms_mixed=kernels["mixed"], kernels_ms_uniform=kernels["uniform"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    import torch
    info = gpu_info()
    for name, cfg in PAGES.items():
        if a.only and a.only != name:
            continue
        r = run_page(name, cfg, a.steps, a.warmup, torch)
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    for name, g in GENERALITY.items():
        if a.only and a.only != name:
            continue
        r = run_generality(name, g, a.steps, a.warmup, torch)
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
