#!/usr/bin/env python
"""bench_sixel_emit.py -- the sixel emitters (B200TIMG_EMIT modes) on the flagship's geometries, device-resident.

bench.py's C2 geometry (3840x2160 -> 2700x1519, padded to 1524, 132 frames) and C5 geometry (1280x720 unscaled, 1250
frames: four-stream slices) run through b200timg_sixel_batch_dev from bench.py's frames.  Per (round, config, mode):
milliseconds per batch call (CUDA events), and the emit-side kernels' times from b200timg_profile in a separate profiled
call -- the emit kernel, sixel_layout_kernel, sixel_sizes_to_offsets_kernel, sixel_compact_kernel.  Modes run
interleaved, round after round, so every mode is measured under the same conditions; the card name and power limit
are read in the same run.

--clocks also compiles sixel.cu with -DB200TIMG_EMIT_CLOCKS into a temporary directory, links it with the tree's other
objects (left there by the regular build) and reports, for mode 5 (emit5, the instrumented kernel), the share of each
phase in the SM cycles its CTAs spent (the instrumented build adds CTA barriers at the phase boundaries, so its kernel
times are not the product's).

    python tools/bench_sixel_emit.py [--configs C2,C5] [--modes 5,2] [--rounds 2] [--steps 5] [--warmup 2] [--clocks]

Prints one JSON line per (round, config, mode), a first line describing the card, and with --clocks one line per
(config, mode) of phase shares.  Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (CONFIGS, frames_torch: the flagship's geometries and frames)

SRC = os.path.join(ROOT, "timg_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# the phases emit5 stamps, in order (sixel.cu EMIT_CLK)
PHASES = ["zero+count", "offsets", "scatter", "walk", "scan", "copy-out"]
EMIT_KEYS = ("emit", "layout", "offsets", "compact")


def card(index):
    q = "name,power.limit,power.max_limit,clocks.max.sm,driver_version"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in r.split(",")]))
    except Exception as ex:
        return {"error": str(ex)[:80]}


def build_instrumented(tmp):
    """sixel.cu with the phase clocks + the tree's other objects -> tmp/libb200timg_clocks.so"""
    obj = os.path.join(tmp, "sixel_clocks.o")
    subprocess.run([NVCC, *ARCH, "-O3", "-std=c++17", "-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off",
                    "-I" + os.path.join(ROOT, "include"), "-DB200TIMG_EMIT_CLOCKS", "-c", os.path.join(SRC, "sixel.cu"),
                    "-o", obj], check=True)
    # the regular build's objects of every other source, and only if none is older than a source or header it depends on
    srcs = [f for f in sorted(os.listdir(SRC)) if f.endswith(".cu") and f != "sixel.cu"]
    objs = [os.path.join(SRC, f[:-3] + ".o") for f in srcs]
    deps = [os.path.join(SRC, f) for f in os.listdir(SRC) if f.endswith((".cuh", ".h"))] + [
        os.path.join(ROOT, "include", "b200timg.h")]
    newest_dep = max(os.path.getmtime(p) for p in deps)
    for src, o in zip(srcs, objs):
        if not os.path.exists(o) or os.path.getmtime(o) < max(newest_dep, os.path.getmtime(os.path.join(SRC, src))):
            sys.exit(f"bench_sixel_emit: {os.path.relpath(o, ROOT)} is missing or older than its sources: run the regular "
                     "build first (--clocks links against its objects)")
    lib = os.path.join(tmp, "libb200timg_clocks.so")
    subprocess.run([NVCC, *ARCH, "-shared", "-o", lib, *objs, obj, "-cudart", "static"], check=True)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C5")
    ap.add_argument("--modes", default="5,2")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--clocks", action="store_true", help="also report the phase shares of an instrumented build")
    ap.add_argument("--clocks-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    modes = [int(m) for m in args.modes.split(",")]

    if not args.clocks_child:
        print(json.dumps({"card": card(args.device)}), flush=True)
        run(args, modes, clocks=False)
        if args.clocks:
            tmp = tempfile.mkdtemp(prefix="b200timg_clocks_")
            try:
                env = dict(os.environ, B200TIMG_LIBFILE=build_instrumented(tmp))
                argv = [a for a in sys.argv[1:] if a != "--clocks"]
                subprocess.run([sys.executable, os.path.abspath(__file__), *argv, "--clocks-child"], env=env, check=True)
            finally:
                shutil.rmtree(tmp, ignore_errors=True)
        return
    run(args, [m for m in modes if m == 5], clocks=True)


def run(args, modes, clocks):
    import torch
    import timg_b200
    from timg_b200 import synth

    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ctx = timg_b200.Context(args.device, stream.cuda_stream)
    L = timg_b200.lib()
    if clocks:
        get_clocks = L.b200timg_emit_clocks
        get_clocks.restype, get_clocks.argtypes = C.c_int, [C.c_void_p]

    runs = []
    for cname in args.configs.split(","):
        cfg = bench.CONFIGS[cname]
        iw, ih, n = cfg["iw"], cfg["ih"], cfg["frames"]
        fw, fh, cx, cy, st = cfg["fit"]
        _, ow, oh = timg_b200.calc_fit(iw, ih, fw, fh, cx, cy, st)
        hp = (oh + 5) // 6 * 6
        src = bench.frames_torch(synth, cfg, n, bench.SEED, dev)
        cap = n * max(1 << 16, 2 * ow * hp)
        out = torch.empty(cap, dtype=torch.uint8, device=dev)
        offs = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        b = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1,
                            bg=timg_b200.rgba_u32(*bench.BG), pattern=0, pattern_w=0, pattern_h=0,
                            flags=cfg["flags"] | bench.FAST_SCALE, x_indent_cells=0, animation=cfg["animation"])
        runs.append((cname, n, ow, hp, src, out, offs, b, cap))

    def step(b, src, out, offs, cap):
        rc = L.b200timg_sixel_batch_dev(ctx.h, C.byref(b), src.data_ptr(), out.data_ptr(), cap, offs.data_ptr())
        if rc != 0:
            raise RuntimeError(L.b200timg_last_error(ctx.h).decode())

    for rnd in range(1 if clocks else args.rounds):
        for cname, n, ow, hp, src, out, offs, b, cap in runs:
            for mode in modes:                          # interleaved: every mode sees the same conditions
                os.environ["B200TIMG_EMIT"] = str(mode)
                for _ in range(args.warmup):
                    step(b, src, out, offs, cap)
                torch.cuda.synchronize(dev)
                if clocks:
                    raw = (C.c_ulonglong * 8)()
                    get_clocks(raw)
                    for _ in range(args.steps):
                        step(b, src, out, offs, cap)
                    if get_clocks(raw) != 0:
                        raise RuntimeError("b200timg_emit_clocks failed")
                    row = [raw[k] for k in range(len(PHASES))]
                    tot = sum(row) or 1
                    print(json.dumps({"clocks": True, "config": cname, "mode": mode, "bands": n * hp // 6,
                                      "sm_cycles_per_band": tot / (args.steps * n * hp // 6),
                                      "share": {p: round(v / tot, 4) for p, v in zip(PHASES, row)}}), flush=True)
                    continue
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.steps):
                    step(b, src, out, offs, cap)
                e1.record(stream)
                torch.cuda.synchronize(dev)
                ms = e0.elapsed_time(e1) / args.steps
                ctx.profile(True)
                step(b, src, out, offs, cap)
                rep = ctx.profile_report()
                ctx.profile(False)
                kern = {k: round(v[1], 4) for k, v in rep.items() if any(s in k for s in EMIT_KEYS)}
                print(json.dumps({"round": rnd, "config": cname, "mode": mode, "frames": n, "out": [ow, hp],
                                  "ms_per_batch": round(ms, 4), "emit_side_ms": round(sum(kern.values()), 4),
                                  "kernels_ms": kern, "encoded_bytes": int(offs[-1].item())}), flush=True)
    os.environ.pop("B200TIMG_EMIT", None)
    ctx.close()


if __name__ == "__main__":
    main()
