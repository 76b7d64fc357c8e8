"""Device JPEG, PNG, QOI, BMP, TGA or PNM decode (b200timg_{jpeg,png,qoi,raster}_frames_dev) against the reference's STB
source (JPEG, PNG, BMP, TGA, PNM) or QOI source on one host core.

Device time: two CUDA events on the context's stream (also torch's current stream) around the call, recorded after a
device synchronise, so the upload of the files from pinned staging and every kernel are inside it; the per-kernel split
comes from ctx.profile in a separate call (png_jump_kernel and qoi_sync_kernel summed over their rounds).  Reference
time: the door onto the unmodified STBImageSource (oracle/gif.mk) or QOIImageSource (oracle/qoi.mk) at capture=0, one
decode per file, on the calling thread.  Prints one JSON
line per case with the card's name and power limit read in the same run.

    python tools/bench_decode.py --format {jpeg,png,qoi,bmp,tga,pnm} [--steps 5] [--warmup 2] [--ref-steps 1]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import jpeg_cases as jc  # noqa: E402
import png_cases as pc  # noqa: E402
import qoi_cases as qc  # noqa: E402
import raster_cases as rc  # noqa: E402
import timg_b200  # noqa: E402
from oracle import gif as G  # noqa: E402
from oracle import qoi as Q  # noqa: E402
from oracle import raster as R  # noqa: E402


def jpeg_cases():
    yield "4k_420", [jc.jpeg(jc.photo(3840, 2160, 1), quality=85, subsampling=2)]
    yield "4k_420_rst_per_row", [jc.jpeg(jc.photo(3840, 2160, 1), quality=85, subsampling=2, restart_marker_rows=1)]
    yield "grid64_1080p", [jc.jpeg(jc.photo(1920 - 8 * (k % 5), 1080 - 4 * (k % 7), k), quality=85, subsampling=2)
                           for k in range(64)]
    yield "thumbs1024_480x270", [jc.jpeg(jc.photo(480, 270, k % 16), quality=85, subsampling=2) for k in range(1024)]


def png_cases():
    yield "4k_photo_rgb", [pc.pillow(pc.photo(3840, 2160, 1), "RGB")]
    yield "4k_screenshot_l9", [pc.pillow(pc.screenshot(3840, 2160, 2), "RGB", compress_level=9)]
    yield "grid64_1080p", [pc.pillow(pc.photo(1920 - 8 * (k % 5), 1080 - 4 * (k % 7), k), "RGB") for k in range(64)]
    yield "thumbs1024_480x270", [pc.pillow(pc.photo(480, 270, k % 16), "RGB") for k in range(1024)]


def qoi_cases():
    yield "4k_photo_rgb", [Q.encode(qc.rgba(pc.photo(3840, 2160, 1)), 3)]
    yield "4k_photo_smooth_rgb", [Q.encode(qc.photo_smooth(3840, 2160, 1), 3)]
    yield "4k_screenshot_rgb", [Q.encode(qc.rgba(pc.screenshot(3840, 2160, 2)), 3)]
    yield "4k_gradient_diff_only", [Q.encode(qc.gradient(3840, 2160), 3)]
    yield "grid64_1080p", [Q.encode(qc.rgba(pc.photo(1920 - 8 * (k % 5), 1080 - 4 * (k % 7), k)), 3) for k in range(64)]
    yield "thumbs1024_480x270", [Q.encode(qc.rgba(pc.photo(480, 270, k % 16)), 3) for k in range(1024)]


def _grid_photos():
    return [pc.photo(1920 - 8 * (k % 5), 1080 - 4 * (k % 7), k) for k in range(64)]


def bmp_cases():
    yield "4k_photo_24", [R.bmp(pc.photo(3840, 2160, 1), 24)]
    yield "grid64_1080p", [R.bmp(p, 24) for p in _grid_photos()]
    yield "thumbs1024_480x270", [R.bmp(pc.photo(480, 270, k % 16), 24) for k in range(1024)]


def tga_cases():
    for rle in (False, True):
        tag = "rle" if rle else "raw"
        yield f"4k_photo_{tag}", [rc.tga_file(pc.photo(3840, 2160, 1), rle)]
        yield f"4k_screenshot_{tag}", [rc.tga_file(pc.screenshot(3840, 2160, 2), rle)]
        yield f"grid64_1080p_{tag}", [rc.tga_file(p, rle) for p in _grid_photos()]
        yield f"thumbs1024_480x270_{tag}", [rc.tga_file(pc.photo(480, 270, k % 16), rle) for k in range(1024)]


def pnm_cases():
    yield "4k_photo_p6", [R.pnm(pc.photo(3840, 2160, 1))]
    yield "grid64_1080p", [R.pnm(p) for p in _grid_photos()]
    yield "thumbs1024_480x270", [R.pnm(pc.photo(480, 270, k % 16)) for k in range(1024)]


FORMATS = {"jpeg": (jpeg_cases, timg_b200.jpeg_parse, "jpg"), "png": (png_cases, timg_b200.png_parse, "png"),
           "qoi": (qoi_cases, timg_b200.qoi_parse, "qoi"), "bmp": (bmp_cases, timg_b200.raster_parse, "bmp"),
           "tga": (tga_cases, timg_b200.raster_parse, "tga"), "pnm": (pnm_cases, timg_b200.raster_parse, "ppm")}
RASTER = ("bmp", "tga", "pnm")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--format", choices=sorted(FORMATS), required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-steps", type=int, default=1)
    a = ap.parse_args()
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    stream = torch.cuda.Stream()                               # a real stream that the context launches on
    ctx = timg_b200.Context(0, stream=stream.cuda_stream)
    torch.cuda.set_stream(stream)
    cases, parse, ext = FORMATS[a.format]
    frames_dev = getattr(ctx, "raster_frames_dev" if a.format in RASTER else f"{a.format}_frames_dev")
    prefixes = ("tga_", "raster_") if a.format in RASTER else (a.format + "_", "decode_")
    for name, files in cases():
        geo = [parse(f) for f in files]
        rgba = sum(g["w"] * g["h"] * 4 for g in geo)
        d = torch.empty(rgba, dtype=torch.uint8, device="cuda:0")
        for _ in range(a.warmup):
            frames_dev(files, d)
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.steps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            st = frames_dev(files, d)
            e1.record(stream)
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 1e3)
        status = st.cpu().numpy()
        ctx.profile(True)
        frames_dev(files, d)
        torch.cuda.synchronize()
        prof = {k: round(v[1], 3) for k, v in ctx.profile_report().items() if k.startswith(prefixes)}
        ctx.profile(False)
        ref_ms = None
        have_ref, ref_run = (Q.have_ref(), Q.ref_qoi_path) if a.format == "qoi" else (G.have_ref(), G.ref_stb_gif_path)
        if have_ref:
            with tempfile.TemporaryDirectory() as td:
                paths = []
                for i, f in enumerate(files):
                    p = os.path.join(td, f"{i}.{ext}")
                    open(p, "wb").write(f)
                    paths.append(p)
                rt = []
                for _ in range(a.ref_steps):
                    t0 = time.perf_counter()
                    for p in paths:
                        ref_run(p, capture=False)
                    rt.append(time.perf_counter() - t0)
                ref_ms = 1e3 * float(np.median(rt))
        dev_ms = 1e3 * float(np.median(ts))
        print(json.dumps(dict(case=name, files=len(files), upload_bytes=sum(len(f) for f in files), rgba_bytes=rgba,
                              device_ms=round(dev_ms, 3), kernels_ms=prof, ref_one_core_ms=None if ref_ms is None else round(ref_ms, 1),
                              speedup=None if ref_ms is None else round(ref_ms / dev_ms, 2),
                              status_ok=int((status == 1).sum()), card=card)), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
