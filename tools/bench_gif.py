#!/usr/bin/env python
"""bench_gif.py -- animated GIF decode on the device against the reference's STB source on the host.

For each of the animations of tests/gif_cases.sized() (480x270 x 120 frames with small transparent sub-rectangles,
1920x1080 x 64 frames, one 4096x2160 frame), one JSON line with:
- dev_decode_ms: b200timg_gif_frames_dev between two CUDA events on the context's stream (also torch's current
  stream), each call after a device synchronise, median over --steps warm calls.  The stream is idle when the first
  event is recorded, so the time runs from the call's start: the host walk (host_walk_ms on its own), the upload
  through pinned staging and the three kernels.
  kernels_ms: the per-kernel split from b200timg_profile (a separate call, profiling on);
- ref_decode_ms: one run of the reference's STBImageSource (LoadAndScale + SendFrames of the raw canvases into a
  sink that drops them, one thread, as timg's loader runs it) through oracle/_ref/libtimg_gif_ref.so, median over
  --ref-steps runs;
- h2d_file_bytes against h2d_canvas_bytes: what crosses PCIe when the device decodes, and when the host does;
- e2e_dev_ms: file -> -p quarter animation bytes (gif_frames_dev, then one blocks batch with animation = 1) against
  e2e_host_ms: one reference decode on the host with its canvases copied into pinned memory, their upload and the
  same blocks batch; both with a host clock from the start to a device synchronise.
The first line describes the card (name, power limit, max SM clock), read in the same run.

    python tools/bench_gif.py [--steps 5] [--warmup 2] [--ref-steps 3] [--only 480x270x120,...]

Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import gif_cases  # noqa: E402
import timg_b200  # noqa: E402
from oracle import gif as G  # noqa: E402

BOX = (160, 100)                 # -p quarter box in pixels (80x50 cells of 2x2 pixels)


def card(index=0):
    q = "name,power.limit,power.max_limit,clocks.max.sm,driver_version"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in r.split(",")]))
    except Exception as ex:
        return {"error": str(ex)[:80]}


def timed(fn, steps, warmup, sync):
    for _ in range(warmup):
        fn()
    sync()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-steps", type=int, default=3)
    ap.add_argument("--only", default=",".join(gif_cases.SIZED))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_gif.py measures on a GPU; none is available")
    print(json.dumps({"card": card(0)}), flush=True)
    stream = torch.cuda.Stream()                               # a real stream (not the legacy default one) ...
    ctx = timg_b200.Context(0, stream=stream.cuda_stream)     # ... that the context launches on: the events see its work
    torch.cuda.set_stream(stream)
    L = timg_b200.lib()
    sync = torch.cuda.synchronize
    tmp = tempfile.TemporaryDirectory()
    for name in a.only.split(","):
        data = gif_cases.sized(name)
        w, h, delays = timg_b200.gif_parse(data)
        n = len(delays)
        d_frames = torch.empty(n * h * w * 4, dtype=torch.uint8, device="cuda")
        for _ in range(a.warmup):
            ctx.gif_frames_dev(data, d_frames, n)
        sync()
        ev = []
        for _ in range(a.steps):
            sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ctx.gif_frames_dev(data, d_frames, n)
            e1.record(stream)
            e1.synchronize()
            ev.append(e0.elapsed_time(e1))
        dev_ms = statistics.median(ev)
        walk_ms, _ = timed(lambda: timg_b200.gif_parse(data), a.steps, 1, lambda: None)
        ctx.profile(True)
        ctx.gif_frames_dev(data, d_frames, n)
        sync()
        kernels = ctx.profile_report()
        ctx.profile(False)
        row = {"gif": name, "frames": n, "w": w, "h": h, "file_bytes": len(data), "dev_decode_ms": round(dev_ms, 3),
               "dev_decode_all_ms": [round(t, 3) for t in ev], "host_walk_ms": round(walk_ms, 3), "kernels_ms": kernels,
               "h2d_file_bytes": len(data), "h2d_canvas_bytes": n * w * h * 4,
               "canvas_over_file": round(n * w * h * 4 / len(data), 1)}
        if G.have_ref():
            path = os.path.join(tmp.name, name + ".gif")
            with open(path, "wb") as f:
                f.write(data)
            # one decode per step: the sink drops the frames (as timg's loader keeps them, nothing is copied out)
            ref_ms, ref_all = timed(lambda: G.ref_stb_gif_path(path, capture=False), a.ref_steps, 0, lambda: None)
            row.update({"ref_decode_ms": round(ref_ms, 3), "ref_decode_all_ms": [round(t, 3) for t in ref_all],
                        "decode_speedup": round(ref_ms / dev_ms, 2)})
            # end to end: file -> -p quarter animation bytes
            _, ow, oh = timg_b200.calc_fit(w, h, BOX[0], BOX[1], 2, 2)
            b = timg_b200.Batch(n_frames=n, src_w=w, src_h=h, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=0xFF000000,
                                pattern=0, pattern_w=0, pattern_h=0, flags=timg_b200.QUARTER, x_indent_cells=0,
                                animation=1)
            cap = L.b200timg_blocks_bound(ow, oh) * n
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            d_offs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
            pinned = torch.empty(n * h * w * 4, dtype=torch.uint8).pin_memory()
            d_up = torch.empty(n * h * w * 4, dtype=torch.uint8, device="cuda")

            def blocks(src):
                ctx._chk(L.b200timg_blocks_batch_dev(ctx.h, C.byref(b), src.data_ptr(), d_out.data_ptr(), cap,
                                                     d_offs.data_ptr()))

            def e2e_dev():
                ctx.gif_frames_dev(data, d_frames, n)
                blocks(d_frames)

            def e2e_host():
                G.ref_stb_gif_path(path, out=pinned.numpy())          # one decode, frames copied into pinned memory
                d_up.copy_(pinned, non_blocking=True)
                blocks(d_up)

            e2e_dev_ms, _ = timed(e2e_dev, a.steps, a.warmup, sync)
            e2e_host_ms, _ = timed(e2e_host, a.ref_steps, 1, sync)
            row.update({"quarter_out": [ow, oh], "e2e_dev_ms": round(e2e_dev_ms, 3), "e2e_host_ms": round(e2e_host_ms, 3),
                        "e2e_speedup": round(e2e_host_ms / e2e_dev_ms, 2)})
            del pinned, d_up
        else:
            row["ref_decode_ms"] = "not measured (oracle/_ref/libtimg_gif_ref.so absent)"
        print(json.dumps(row), flush=True)
        del d_frames
        torch.cuda.empty_cache()
    ctx.close()
    tmp.cleanup()


if __name__ == "__main__":
    main()
