#!/usr/bin/env python
"""Kitty / iTerm2 batches on the GPU (b200timg_graphics_batch[_dev]): one JSON line per configuration.

  python tools/bench_graphics.py [--steps K] [--warmup W] [--only NAME]

  C2-kitty       3840x2160 RGBA -> 2700x1519 (C2 geometry), 132 frames, kitty, rgb24 (PNG colour type 2)
  C2-kitty-tmux  the same in kitty's tmux form at 9x18-px cells: passthrough framing and a 300 x 85 placeholder grid
  C2-iterm2      the same through iTerm2
  C4-kitty       3840x2160 RGBA -> 337x190 (C4 geometry), 128 frames, kitty, rgb24, composed onto black
  *-deflate      the same with B200TIMG_DEFLATE (compressed PNGs), run right after its stored configuration;
                 encoded bytes against the stored bytes, and the IDAT bytes of 8 sampled frames against zlib level 1
                 (Python's zlib on the host, same scaled frames)

Per configuration: device-resident Mpx/s of input pixels and encoded GB/s; B_alg = (source bytes + encoded bytes)
over the chain time, as a share of the H100 SXM's 3350 GB/s (DESIGN.md section 4); the per-kernel ms of one batch
(b200timg_profile); the host-buffer end-to-end rate (b200timg_graphics_batch: source upload, kernels, download of
the framed text); and beside it the route that existed before: scale + compose + b200timg_png_batch_dev (unframed
PNG + base64 on the device), download of both, framing on the host (numpy).  That route starts from frames already
on the device, so its end-to-end time has no source upload in it.  The tmux form never had such a route (its
placeholder grid was not built anywhere), so its png_batch_route is null.  The GPU's name, power limit and max SM clock are read in the same run.
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

HBM_GBS = 3350.0
PROTOCOL_NAMES = {timg_b200.KITTY: "kitty", timg_b200.ITERM2: "iterm2", timg_b200.KITTY_TMUX: "kitty-tmux"}
CONFIGS = {
    "C2-kitty": dict(iw=3840, ih=2160, ow=2700, oh=1519, n=132, proto=timg_b200.KITTY, has_bg=0),
    "C2-kitty-tmux": dict(iw=3840, ih=2160, ow=2700, oh=1519, n=132, proto=timg_b200.KITTY_TMUX, has_bg=0, cell=(9, 18)),
    "C2-iterm2": dict(iw=3840, ih=2160, ow=2700, oh=1519, n=132, proto=timg_b200.ITERM2, has_bg=0),
    "C2-kitty-deflate": dict(iw=3840, ih=2160, ow=2700, oh=1519, n=132, proto=timg_b200.KITTY, has_bg=0, deflate=True),
    "C2-iterm2-deflate": dict(iw=3840, ih=2160, ow=2700, oh=1519, n=132, proto=timg_b200.ITERM2, has_bg=0, deflate=True),
    "C4-kitty": dict(iw=3840, ih=2160, ow=337, oh=190, n=128, proto=timg_b200.KITTY, has_bg=1),
    "C4-kitty-deflate": dict(iw=3840, ih=2160, ow=337, oh=190, n=128, proto=timg_b200.KITTY, has_bg=1, deflate=True),
}
ORDER = ["C2-kitty", "C2-kitty-deflate", "C2-kitty-tmux", "C2-iterm2", "C2-iterm2-deflate", "C4-kitty", "C4-kitty-deflate"]


def scanlines(fb):
    """The Sub-filtered rgb24 scanline stream of a frame (the PNG's raw IDAT content, src/timg-png.cc:119-134)."""
    px = np.ascontiguousarray(fb[..., :3])
    d = px.copy()
    d[:, 1:] = px[:, 1:] - px[:, :-1]
    return np.concatenate([np.ones((px.shape[0], 1), np.uint8), d.reshape(px.shape[0], -1)], axis=1).tobytes()


def idat_bytes(text):
    """IDAT length of the PNG in one framed kitty or iTerm2 frame: its base64 payload, decoded."""
    import base64
    import re
    if text.startswith(b"\033]1337;"):
        b64 = text[text.index(b":") + 1:text.rindex(b"\a")]
    else:
        b64 = b"".join(re.findall(rb"\033_G[^;]*;([A-Za-z0-9+/=]*)\033\\", text))
    return int.from_bytes(base64.b64decode(b64)[33:37], "big")


def zlib1_ratio(torch, L, ctx, d_src, b, cfg, out, offs, n):
    """IDAT bytes of 8 sampled frames over zlib level 1's stream of the same scanlines."""
    import zlib
    ow, oh = cfg["ow"], cfg["oh"]
    d_fb = torch.empty((n, oh, ow, 4), dtype=torch.uint8, device="cuda")
    ctx._chk(L.b200timg_scale_dev(ctx.h, d_src.data_ptr(), cfg["iw"], cfg["ih"], 0, d_fb.data_ptr(), ow, oh, n))
    ctx._chk(L.b200timg_compose_dev(ctx.h, d_fb.data_ptr(), ow, oh, n, cfg["has_bg"], b.bg, 0, 0, 0, 0))
    torch.cuda.synchronize()
    ours = ref = 0
    for f in range(0, n, max(1, n // 8))[:8]:
        ours += idat_bytes(out[int(offs[f]):int(offs[f + 1])].tobytes())
        ref += len(zlib.compress(scanlines(d_fb[f].cpu().numpy()), 1))
    return round(ours / ref, 4)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                      # the numbers still stand, without their card
        return f"unavailable ({e})"


def frames_on_device(torch, iw, ih, n):
    """n distinct frames from four generated 4K ones (a per-frame byte rotation of the colour channels)."""
    base = torch.tensor(np.stack([synth.frame_np(900 + i, iw, ih, "photo") for i in range(4)])).cuda()
    d = torch.empty((n, ih, iw, 4), dtype=torch.uint8, device="cuda")
    for f in range(n):
        d[f] = base[f % 4]
        d[f, ..., :3] += (37 * (f // 4)) & 255
    return d


def frame_text(b64, proto, png_len, w, h, id_):
    """The framing the kitty / iTerm2 adapters did on the host before, vectorised (numpy) for one frame."""
    if proto == timg_b200.ITERM2:
        head = b"\033]1337;File=size=%d;width=%dpx;height=%dpx;inline=1:" % (png_len, w, h)
        return b"".join((head, b64.tobytes(), b"\a\n"))
    nfull = (len(b64) - 1) // 4096
    body = b64[:nfull * 4096].reshape(nfull, 4096)
    sep = np.frombuffer(b"\033\\\033_Gq=2,m=1;", np.uint8)
    parts = np.concatenate([body, np.broadcast_to(sep, (nfull, len(sep)))], 1).reshape(-1)
    if nfull:                                   # the last separator announces the last chunk
        last_more = png_len - nfull * 3072 > 3072
        parts[-2] = ord("1" if last_more else "0")
    head = b"\033_Ga=T,i=%d,q=2,f=100,m=%d;" % (id_, png_len > 3072)
    return b"".join((head, parts.tobytes(), b64[nfull * 4096:].tobytes(), b"\033\\\n"))


def run(name, cfg, steps, warmup, torch):
    iw, ih, ow, oh, n, proto = cfg["iw"], cfg["ih"], cfg["ow"], cfg["oh"], cfg["n"], cfg["proto"]
    ctx = timg_b200.Context(0)
    L = timg_b200.lib()
    b = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=cfg["has_bg"],
                        bg=timg_b200.rgba_u32(0, 0, 0), pattern=0, pattern_w=0, pattern_h=0, flags=0, x_indent_cells=0,
                        animation=0)
    ids = np.arange(1, n + 1, dtype=np.uint32) + np.uint32(1_700_000_000)
    deflate = cfg.get("deflate", False)
    g, keep = timg_b200.graphics(proto | (timg_b200.DEFLATE if deflate else 0), True, ids, cfg.get("cell"))
    d_src = frames_on_device(torch, iw, ih, n)
    total = sum(L.b200timg_graphics_size(C.byref(g), ow, oh, int(i)) for i in ids)
    d_out = torch.empty(total, dtype=torch.uint8, device="cuda")
    d_offs = torch.empty(n + 1, dtype=torch.int64, device="cuda")

    def step():
        ctx._chk(L.b200timg_graphics_batch_dev(ctx.h, C.byref(b), C.byref(g), d_src.data_ptr(), d_out.data_ptr(), total,
                                               d_offs.data_ptr()))
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()                   # a device-wide synchronise: it also waits for the context's own stream
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    encoded = int(d_offs[-1])
    assert encoded == total or deflate and encoded <= total
    src_bytes = n * iw * ih * 4
    ctx.profile(True)
    step()
    kernels = {k: round(v[1], 3) for k, v in ctx.profile_report().items()}
    ctx.profile(False)

    # host buffers end to end
    h_src = d_src.cpu().numpy()
    out = np.empty(total, np.uint8)
    offs = np.zeros(n + 1, np.uint64)
    ctx._chk(L.b200timg_graphics_batch(ctx.h, C.byref(b), C.byref(g), h_src.ctypes.data, out.ctypes.data, total, offs.ctypes.data))
    t0 = time.perf_counter()
    for _ in range(steps):
        ctx._chk(L.b200timg_graphics_batch(ctx.h, C.byref(b), C.byref(g), h_src.ctypes.data, out.ctypes.data, total,
                                           offs.ctypes.data))
    host_s = (time.perf_counter() - t0) / steps
    same = out[:encoded].tobytes() == d_out[:encoded].cpu().numpy().tobytes() and bool((offs == d_offs.cpu().numpy().astype(np.uint64)).all())
    result = dict(config=name, frames=n, src=f"{iw}x{ih}", out=f"{ow}x{oh}", protocol=PROTOCOL_NAMES[proto],
                  rgb24=True, has_bg=bool(cfg["has_bg"]), deflate=deflate, encoded_bytes=encoded, stored_bytes=total,
                  encoded_over_stored=round(encoded / total, 4), steps=steps,
                  dev_ms=round(ms, 3), dev_mpx_s=round(n * iw * ih / ms / 1e3, 1), dev_encoded_gbs=round(encoded / ms / 1e6, 2),
                  b_alg_gbs=round((src_bytes + encoded) / ms / 1e6, 1), b_alg_share=round((src_bytes + encoded) / ms / 1e6 / HBM_GBS, 4),
                  kernels_ms=kernels, host_e2e_ms=round(host_s * 1e3, 2), host_e2e_mpx_s=round(n * iw * ih / host_s / 1e6, 1),
                  host_equals_dev=same, png_batch_route=None)
    if deflate:
        result["idat_over_zlib1"] = zlib1_ratio(torch, L, ctx, d_src, b, cfg, out, offs, n)
    if proto == timg_b200.KITTY_TMUX or deflate:
        ctx.close()
        return result

    # the earlier route: scale + compose, png_batch_dev (PNG + base64), both downloaded, framed on the host
    png_len = L.b200timg_png_size(ow, oh, 1)
    b64_len = L.b200timg_base64_size(png_len)
    d_fb = torch.empty((n, oh, ow, 4), dtype=torch.uint8, device="cuda")
    d_png = torch.empty(n * png_len, dtype=torch.uint8, device="cuda")
    d_b64 = torch.empty(n * b64_len, dtype=torch.uint8, device="cuda")
    h_png = torch.empty(n * png_len, dtype=torch.uint8).pin_memory()
    h_b64 = torch.empty(n * b64_len, dtype=torch.uint8).pin_memory()

    def route_dev():
        ctx._chk(L.b200timg_scale_dev(ctx.h, d_src.data_ptr(), iw, ih, 0, d_fb.data_ptr(), ow, oh, n))
        ctx._chk(L.b200timg_compose_dev(ctx.h, d_fb.data_ptr(), ow, oh, n, cfg["has_bg"], b.bg, 0, 0, 0, 0))
        ctx._chk(L.b200timg_png_batch_dev(ctx.h, d_fb.data_ptr(), ow, oh, n, 1, d_png.data_ptr(), d_b64.data_ptr()))
    route_dev()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        route_dev()
    torch.cuda.synchronize()
    route_ms = (time.perf_counter() - t0) * 1e3 / steps
    t0 = time.perf_counter()
    for _ in range(steps):
        route_dev()
        torch.cuda.synchronize()
        h_png.copy_(d_png)
        h_b64.copy_(d_b64)
        hb = h_b64.numpy()
        texts = [frame_text(hb[f * b64_len:(f + 1) * b64_len], proto, png_len, ow, oh, int(ids[f])) for f in range(n)]
    route_e2e_s = (time.perf_counter() - t0) / steps
    route_same = b"".join(texts) == out.tobytes()
    ctx.close()
    result["png_batch_route"] = dict(dev_ms=round(route_ms, 3), d2h_bytes=n * (png_len + b64_len),
                                     e2e_ms=round(route_e2e_s * 1e3, 2), e2e_mpx_s=round(n * iw * ih / route_e2e_s / 1e6, 1),
                                     same_bytes=route_same)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    import torch
    info = gpu_info()
    for name in ORDER:
        if a.only and name != a.only:
            continue
        r = run(name, CONFIGS[name], a.steps, a.warmup, torch)
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
