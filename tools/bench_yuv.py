#!/usr/bin/env python
"""bench_yuv.py -- the video front per decoder format, device-resident.

For each format, bench.py's C2 geometry (3840x2160 -> 2700x1519 sixel, 132 frames) and C3 geometry (1920x1080 ->
320x90 quarter blocks, delta frames, 300 frames) run through b200timg_{sixel,blocks}_batch_dev from YUV frames of
that format that already sit on the device (the same synthetic frames bench.py uses, converted BT.601 limited range
with box-filtered chroma).  Per row: input Mpx/s of the whole batch call, source bytes per frame, and the scale
kernel's time from b200timg_profile (a separate pass, profiling on).  Formats run interleaved, round after round, so
every format (I420 included) is measured under the same conditions; the card name and power limit are read in the
same run.

    python tools/bench_yuv.py [--formats I420,I444,...] [--configs C2,C3] [--rounds 2] [--steps 5] [--warmup 2]

Prints one JSON line per (round, config, format) and a first line describing the card.  Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (CONFIGS, frames_torch: the flagship's geometries and frames)

FORMATS = ["I420", "NV12", "I422", "I444", "I440", "I420_10", "I422_10", "I444_10", "P010"]
# name -> (chroma shift x, chroma shift y, bytes per sample, interleaved chroma)
LAYOUT = {"I420": (1, 1, 1, False), "NV12": (1, 1, 1, True), "I422": (1, 0, 1, False), "I444": (0, 0, 1, False),
          "I440": (0, 1, 1, False), "I420_10": (1, 1, 2, False), "I422_10": (1, 0, 2, False), "I444_10": (0, 0, 2, False),
          "P010": (1, 1, 2, True)}


def card(index):
    q = "name,power.limit,power.max_limit,clocks.max.sm,driver_version"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in r.split(",")]))
    except Exception as ex:
        return {"error": str(ex)[:80]}


def to_yuv(fr, name):
    """One RGBA frame [h, w, 4] (device) -> one tightly packed frame of the format, as bytes (device)."""
    import torch
    sx, sy, bps, semi = LAYOUT[name]
    ih, iw = fr.shape[:2]
    c = fr[..., :3].to(torch.float32)
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    y = 16 + 0.256788 * r + 0.504129 * g + 0.097906 * b
    u = 128 - 0.148223 * r - 0.290993 * g + 0.439216 * b
    v = 128 + 0.439216 * r - 0.367788 * g - 0.071427 * b
    box = lambda p: p.reshape(ih >> sy, 1 << sy, iw >> sx, 1 << sx).mean((1, 3))
    scale, top = (1.0, 255) if bps == 1 else (4.0, 1023)
    q = lambda p: (p * scale).round().clamp(0, top).to(torch.int32)
    Y, U, V = q(y), q(box(u)), q(box(v))
    chroma = torch.stack([U, V], -1).reshape(-1) if semi else torch.cat([U.reshape(-1), V.reshape(-1)])
    s = torch.cat([Y.reshape(-1), chroma])
    if bps == 1:
        return s.to(torch.uint8)
    if name == "P010":
        s = s << 6
    return torch.stack([s & 255, s >> 8], -1).reshape(-1).to(torch.uint8)      # little-endian 16-bit samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--formats", default=",".join(FORMATS))
    ap.add_argument("--configs", default="C2,C3")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import torch
    import timg_b200
    from timg_b200 import synth

    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ctx = timg_b200.Context(args.device, stream.cuda_stream)
    L = timg_b200.lib()
    formats = args.formats.split(",")
    print(json.dumps({"card": card(args.device), "library": os.path.relpath(timg_b200.LIB_PATH, ROOT),
                      "torch": torch.__version__}), flush=True)

    runs = []
    for cname in args.configs.split(","):
        cfg = bench.CONFIGS[cname]
        iw, ih, n = cfg["iw"], cfg["ih"], cfg["frames"]
        fw, fh, cx, cy, st = cfg["fit"]
        _, ow, oh = timg_b200.calc_fit(iw, ih, fw, fh, cx, cy, st)
        sixel = cfg["canvas"] == "sixel"
        hp = (oh + 5) // 6 * 6 if sixel else oh
        rgba = bench.frames_torch(synth, cfg, n, bench.SEED, dev)
        srcs = {}
        for name in formats:
            fb = timg_b200.yuv_frame_bytes(getattr(timg_b200, "FMT_" + name), iw, ih)
            srcs[name] = torch.empty((n, fb), dtype=torch.uint8, device=dev)
            for i in range(n):
                srcs[name][i] = to_yuv(rgba[i], name)
        del rgba
        cap = n * max(1 << 16, 2 * ow * hp) if sixel else int(L.b200timg_blocks_bound(ow, oh)) * n + 64
        out = torch.empty(cap, dtype=torch.uint8, device=dev)
        offs = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        call = L.b200timg_sixel_batch_dev if sixel else L.b200timg_blocks_batch_dev
        flags = cfg["flags"] | (bench.FAST_SCALE if sixel else 0)
        runs.append((cname, cfg, iw, ih, n, ow, oh, srcs, out, offs, call, flags, cap))

    def step(call, b, src, out, offs, cap):
        rc = call(ctx.h, C.byref(b), src.data_ptr(), out.data_ptr(), cap, offs.data_ptr())
        if rc != 0:
            raise RuntimeError(L.b200timg_last_error(ctx.h).decode())

    for rnd in range(args.rounds):
        for cname, cfg, iw, ih, n, ow, oh, srcs, out, offs, call, flags, cap in runs:
            for name in formats:                       # interleaved: every format sees the same conditions
                src = srcs[name]
                b = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=getattr(timg_b200, "FMT_" + name), out_w=ow,
                                    out_h=oh, has_bg=1, bg=timg_b200.rgba_u32(*bench.BG), pattern=0, pattern_w=0,
                                    pattern_h=0, flags=flags, x_indent_cells=0, animation=cfg["animation"])
                for _ in range(args.warmup):
                    step(call, b, src, out, offs, cap)
                torch.cuda.synchronize(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.steps):
                    step(call, b, src, out, offs, cap)
                e1.record(stream)
                torch.cuda.synchronize(dev)
                ms = e0.elapsed_time(e1) / args.steps
                ctx.profile(True)
                step(call, b, src, out, offs, cap)
                rep = ctx.profile_report()
                ctx.profile(False)
                scale = {k: v[1] for k, v in rep.items() if k.startswith("yuv")}
                print(json.dumps({"round": rnd, "config": cname, "format": name, "frames": n, "src": [iw, ih],
                                  "out": [ow, oh], "mpx_s": n * iw * ih / 1e6 / (ms / 1e3), "ms_per_batch": ms,
                                  "src_bytes_per_frame": int(src.shape[1]), "scale_kernel": scale,
                                  "scale_ms": sum(scale.values()), "encoded_bytes": int(offs[-1].item())}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
