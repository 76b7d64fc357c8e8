"""timg_b200 -- Python door onto libb200timg.so (the C ABI in include/b200timg.h).

This module is harness plumbing for tests and bench.py: it loads the in-tree shared
library with ctypes, declares every symbol of the ABI, and offers small numpy/torch
conveniences.  The product is the CUDA library; there is no Python or CPU fallback:
loading fails loudly if the library is missing, and Context() raises if no CUDA
device is visible.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200TIMG_LIBFILE") or os.path.join(_HERE, "libb200timg.so")   # tuning runs load a variant build

OK, EINVAL, ENOMEM, ECUDA, ENOSPC, ENODEV = 0, -1, -2, -3, -4, -5
QUARTER, UPPER, COLOR8, FAST_SCALE, BILINEAR_SCALE = 1, 2, 4, 8, 16
FMT_RGBA, FMT_RGB32, FMT_I420, FMT_NV12, FMT_FULL_RANGE = 0, 1, 2, 3, 0x10
FMT_I422, FMT_I444, FMT_I440, FMT_I420_10, FMT_I422_10, FMT_I444_10, FMT_P010 = 4, 5, 6, 7, 8, 9, 10
YUV_FORMATS = (FMT_I420, FMT_NV12, FMT_I422, FMT_I444, FMT_I440, FMT_I420_10, FMT_I422_10, FMT_I444_10, FMT_P010)
# low nibble -> (chroma shift x, chroma shift y, bytes per sample): the tightly packed layouts of include/b200timg.h
_YUV_LAYOUT = {FMT_I420: (1, 1, 1), FMT_NV12: (1, 1, 1), FMT_I422: (1, 0, 1), FMT_I444: (0, 0, 1), FMT_I440: (0, 1, 1),
               FMT_I420_10: (1, 1, 2), FMT_I422_10: (1, 0, 2), FMT_I444_10: (0, 0, 2), FMT_P010: (1, 1, 2)}


def yuv_frame_bytes(fmt, w, h):
    """Bytes of one tightly packed frame of a YUV format (FULL_RANGE bit ignored), as the library computes them."""
    sx, sy, bps = _YUV_LAYOUT[fmt & 0xF]
    return bps * (w * h + 2 * (w >> sx) * (h >> sy))


KITTY, ITERM2, KITTY_TMUX = 1, 2, 4
DEFLATE = 8      # OR'ed into a protocol: compressed PNGs (timg's --compress 1-9); sizes are then upper bounds

u8p = C.POINTER(C.c_uint8)
u64p = C.POINTER(C.c_uint64)


class FitOpts(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("cell_x_px", C.c_int), ("cell_y_px", C.c_int),
                ("width_stretch", C.c_float), ("upscale", C.c_int), ("upscale_integer", C.c_int),
                ("fill_width", C.c_int), ("fill_height", C.c_int)]


class Batch(C.Structure):
    _fields_ = [("n_frames", C.c_int), ("src_w", C.c_int), ("src_h", C.c_int), ("src_fmt", C.c_int),
                ("out_w", C.c_int), ("out_h", C.c_int), ("has_bg", C.c_int), ("bg", C.c_uint32),
                ("pattern", C.c_uint32), ("pattern_w", C.c_int), ("pattern_h", C.c_int),
                ("flags", C.c_int), ("x_indent_cells", C.c_int), ("animation", C.c_int)]


class Graphics(C.Structure):
    _fields_ = [("protocol", C.c_int), ("rgb24", C.c_int), ("ids", C.POINTER(C.c_uint32)),
                ("cell_x_px", C.c_int), ("cell_y_px", C.c_int), ("indent_cells", C.c_int)]


class Frame(C.Structure):
    _fields_ = [("src_offset", C.c_uint64), ("src_w", C.c_int), ("src_h", C.c_int), ("out_w", C.c_int), ("out_h", C.c_int),
                ("x_indent_cells", C.c_int)]


class SixelShape(C.Structure):
    _fields_ = [(k, C.c_int) for k in ("step_px", "ent_cap", "palette_global", "nb32", "dither_ctas", "bands_per_cta",
                                       "dither_warps", "dither_rounds", "emit_mode", "emit_tiles", "tile_w")]


SCALE_ROUTES = {1: "copy4", 2: "copy", 3: "v3", 4: "planar", 5: "fixed", 6: "tp_v", 7: "tp_h1s", 8: "tp_h1f", 9: "tp_h1"}


class ScaleShape(C.Structure):
    _fields_ = [(k, C.c_int) for k in ("route", "hc", "vc", "h_widest", "v_widest", "vertical_first", "h_sequential", "h_filter",
                                       "v_filter", "h_gather", "v_gather", "h1f_rows", "v3_tma", "planar_reuse", "v3_reuse",
                                       "tiles_full", "planar_smem", "v3_smem", "fixed_smem", "h1s_smem", "tiles_x", "tiles_y",
                                       "win_w", "win_h")]


class MixedBatch(C.Structure):
    _fields_ = [("n_frames", C.c_int), ("src_fmt", C.c_int), ("flags", C.c_int), ("has_bg", C.c_int), ("bg", C.c_uint32),
                ("pattern", C.c_uint32), ("pattern_w", C.c_int), ("pattern_h", C.c_int), ("frames", C.POINTER(Frame))]


# name -> (restype, argtypes); this table IS the list of exported symbols tests check.
ABI = {
    "b200timg_version": (C.c_int, []),
    "b200timg_ctx_create": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "b200timg_ctx_destroy": (None, [C.c_void_p]),
    "b200timg_last_error": (C.c_char_p, [C.c_void_p]),
    "b200timg_kernel_launches": (C.c_uint64, [C.c_void_p]),
    "b200timg_calc_fit": (C.c_int, [C.POINTER(FitOpts), C.c_int, C.c_int, C.c_int,
                                    C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "b200timg_as256": (C.c_int, [C.c_uint32]),
    "b200timg_scale_rgba": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, u8p, C.c_int, C.c_int]),
    "b200timg_scale_rgba_mode": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, u8p, C.c_int, C.c_int, C.c_int]),
    "b200timg_yuv_scale": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, u8p, C.c_int, C.c_int]),
    "b200timg_compose_bg": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                      C.c_int, C.c_int, C.c_int]),
    "b200timg_compose_bg_resident": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                               C.c_int, C.c_int, C.c_int]),
    "b200timg_has_transparency": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "b200timg_blocks_bound": (C.c_size_t, [C.c_int, C.c_int]),
    "b200timg_blocks_encode": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, u8p, C.c_int, C.c_int,
                                         C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200timg_sixel_bound": (C.c_size_t, [C.c_int, C.c_int]),
    "b200timg_sixel_encode": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_char_p, C.c_size_t,
                                        C.POINTER(C.c_size_t)]),
    "b200timg_blocks_batch_dev": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_size_t,
                                            C.c_void_p]),
    "b200timg_sixel_batch_dev": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_size_t,
                                           C.c_void_p]),
    "b200timg_blocks_batch": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.c_void_p]),
    "b200timg_sixel_batch": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_size_t,
                                       C.c_void_p]),
    "b200timg_scale_mixed_dev": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.c_void_p, C.c_void_p]),
    "b200timg_blocks_mixed_dev": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_blocks_mixed": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_sixel_mixed_dev": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_sixel_mixed": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_scale_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                     C.c_int, C.c_int]),
    "b200timg_compose_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32,
                                       C.c_uint32, C.c_int, C.c_int, C.c_int]),
    "b200timg_sixel_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
    "b200timg_exif_op": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, C.c_int, u8p]),
    "b200timg_exif_op_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200timg_trim_bbox": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "b200timg_windows": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_longlong, C.c_int,
                                   C.c_int, C.c_longlong, C.c_int, u8p]),
    "b200timg_windows_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                                       C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_void_p]),
    "b200timg_png_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "b200timg_base64_size": (C.c_size_t, [C.c_size_t]),
    "b200timg_png_encode": (C.c_int, [C.c_void_p, u8p, C.c_int, C.c_int, C.c_int, u8p, C.c_size_t, C.c_char_p, C.c_size_t]),
    "b200timg_png_batch_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200timg_graphics_size": (C.c_size_t, [C.POINTER(Graphics), C.c_int, C.c_int, C.c_uint32]),
    "b200timg_graphics_batch_dev": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.POINTER(Graphics), C.c_void_p, C.c_void_p,
                                              C.c_size_t, C.c_void_p]),
    "b200timg_graphics_batch": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.POINTER(Graphics), C.c_void_p, C.c_void_p,
                                          C.c_size_t, C.c_void_p]),
    "b200timg_graphics_mixed_dev": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.POINTER(Graphics), C.c_void_p, C.c_void_p,
                                              C.c_size_t, C.c_void_p]),
    "b200timg_graphics_mixed": (C.c_int, [C.c_void_p, C.POINTER(MixedBatch), C.POINTER(Graphics), C.c_void_p, C.c_void_p,
                                          C.c_size_t, C.c_void_p]),
    "b200timg_gather_unique_id": (C.c_int, [C.c_char_p]),
    "b200timg_gather_init": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int]),
    "b200timg_gather_attach": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "b200timg_gather_shutdown": (None, [C.c_void_p]),
    "b200timg_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int]),
    "b200timg_gather_wait": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "b200timg_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "b200timg_profile_report": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "b200timg_sixel_debug": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "b200timg_resample_plan": (C.c_int, [C.c_int] * 5 + [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p,
                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "b200timg_sixel_shape_of": (C.c_int, [C.c_int] * 5 + [C.POINTER(SixelShape)]),
    "b200timg_scale_shape_of": (C.c_int, [C.c_int] * 8 + [C.POINTER(ScaleShape)]),
    "b200timg_gif_parse": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                     C.c_void_p, C.c_int]),
    "b200timg_gif_frames_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]),
    "b200timg_gif_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.POINTER(C.c_int)]),
    "b200timg_jpeg_parse": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_jpeg_frames_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_jpeg_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_png_parse": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_png_frames_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_png_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_qoi_parse": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_qoi_frames_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_qoi_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_raster_parse": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200timg_raster_frames_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200timg_raster_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None


def build(verbose=False):
    """Compile every CUDA source for sm_90a into timg_b200/libb200timg.so (in-tree)."""
    subprocess.run(["make", "-C", os.path.join(_HERE, "csrc"), "-j8"], check=True,
                   stdout=None if verbose else subprocess.DEVNULL)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(timg_b200 has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in ABI.items():
            f = getattr(L, name)          # AttributeError if a declared symbol is not exported
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200timg error {code}: {msg}")
        self.code = code


def rgba_u32(r, g, b, a=255):
    return (r & 255) | ((g & 255) << 8) | ((b & 255) << 16) | ((a & 255) << 24)


def calc_fit(iw, ih, width, height, cell_x=1, cell_y=2, stretch=1.0, upscale=False,
             upscale_integer=False, fill_width=False, fill_height=False, rotated=False):
    o = FitOpts(width, height, cell_x, cell_y, stretch, int(upscale), int(upscale_integer),
                int(fill_width), int(fill_height))
    tw, th = C.c_int(), C.c_int()
    r = lib().b200timg_calc_fit(C.byref(o), iw, ih, int(rotated), C.byref(tw), C.byref(th))
    if r < 0:
        raise B200Error(r, "calc_fit")
    return bool(r), tw.value, th.value


def resample_plan(iw, ih, ow, oh, axis):
    """Host-side resampling plan of one axis as numpy arrays (see include/b200timg.h)."""
    n = ow if axis == 0 else oh
    widest, flags = C.c_int(), C.c_int()
    rc = lib().b200timg_resample_plan(iw, ih, ow, oh, axis, C.byref(widest), C.byref(flags), None, None, None,
                                      None, 1 << 62)
    if rc != OK:
        raise B200Error(rc, "resample_plan")
    first, count, lead = (np.zeros(n, np.int32) for _ in range(3))
    coeff = np.zeros(n * widest.value, np.float32)
    rc = lib().b200timg_resample_plan(iw, ih, ow, oh, axis, None, None, first.ctypes.data, count.ctypes.data,
                                      lead.ctypes.data, coeff.ctypes.data, coeff.size)
    if rc != OK:
        raise B200Error(rc, "resample_plan")
    return dict(widest=widest.value, flags=flags.value, first=first, count=count, lead=lead,
                coeff=coeff.reshape(n, widest.value))


def sixel_shape(w, h, n_frames=1, n_total=None, sm_count=132):
    """Host-side launch shape of the sixel kernels for n_frames frames of w x h out of a batch of n_total (default: the
    whole batch) on a device with sm_count SMs, as a dict of b200timg_sixel_shape's fields (see include/b200timg.h)."""
    s = SixelShape()
    rc = lib().b200timg_sixel_shape_of(w, h, n_frames, n_frames if n_total is None else n_total, sm_count, C.byref(s))
    if rc != OK:
        raise B200Error(rc, f"sixel_shape: {w} x {h}, {n_frames} frames: not a geometry the sixel path takes")
    return {k: getattr(s, k) for k, _ in SixelShape._fields_}


def scale_shape(iw, ih, ow, oh, n_frames=1, fast=False, src_aligned16=True, dst_aligned16=True):
    """Host-side launch shape of the scaler for n_frames frames of iw x ih -> ow x oh, as a dict of b200timg_scale_shape's
    fields (see include/b200timg.h) with the route's name under "route"."""
    s = ScaleShape()
    rc = lib().b200timg_scale_shape_of(iw, ih, ow, oh, n_frames, int(bool(fast)), int(src_aligned16), int(dst_aligned16), C.byref(s))
    if rc != OK:
        raise B200Error(rc, f"scale_shape: {iw} x {ih} -> {ow} x {oh}, {n_frames} frames: not a geometry the scaler takes")
    d = {k: getattr(s, k) for k, _ in ScaleShape._fields_}
    d["route"] = SCALE_ROUTES[d["route"]]
    return d


def graphics(protocol, rgb24=False, ids=None, cell=None, indent=0):
    """(b200timg_graphics, the uint32 id array it points to): keep both alive for the call.
    cell=(cell_x_px, cell_y_px) and indent (cells) place the KITTY_TMUX form's placeholder grid."""
    arr = None if ids is None else np.ascontiguousarray(ids, dtype=np.uint32)
    cx, cy = cell if cell is not None else (0, 0)
    g = Graphics(protocol, int(rgb24), arr.ctypes.data_as(C.POINTER(C.c_uint32)) if arr is not None else None,
                 cx, cy, indent)
    return g, arr


def graphics_size(protocol, w, h, rgb24=False, id=0, cell=None, indent=0):
    """Exact bytes of one framed kitty / iTerm2 frame (host only); 0 for invalid arguments."""
    g, _ = graphics(protocol, rgb24, cell=cell, indent=indent)
    return lib().b200timg_graphics_size(C.byref(g), w, h, id)


def gif_parse(data):
    """b200timg_gif_parse (host only): (w, h, delays_ms) of a GIF, one delay per frame the STB source collects unless
    an LZW error (found only by decoding) ends the animation earlier.  Raises B200Error(EINVAL) for what is not a
    GIF87a / GIF89a, has no frame or a zero-sized screen."""
    data = bytes(data)
    w, h, n = C.c_int(), C.c_int(), C.c_int()
    rc = lib().b200timg_gif_parse(data, len(data), C.byref(w), C.byref(h), C.byref(n), None, 0)
    if rc != OK:
        raise B200Error(rc, "gif_parse: not a GIF, no frame or a zero-sized screen")
    delays = np.zeros(max(1, n.value), np.int32)
    lib().b200timg_gif_parse(data, len(data), C.byref(w), C.byref(h), C.byref(n), delays.ctypes.data, n.value)
    return w.value, h.value, [int(d) for d in delays[:n.value]]


class JpegInfo(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("n_comp", C.c_int), ("h_samp", C.c_int * 4), ("v_samp", C.c_int * 4),
                ("restart_interval", C.c_int), ("progressive", C.c_int), ("supported", C.c_int),
                ("reason", C.c_char * 96)]


def jpeg_parse(data):
    """b200timg_jpeg_parse (host only): a dict of w, h, n_comp, h_samp, v_samp, restart_interval, progressive,
    supported and reason.  Raises B200Error(EINVAL) where stb's marker walk fails (so the reference's source fails)."""
    data = bytes(data)
    info = JpegInfo()
    rc = lib().b200timg_jpeg_parse(data, len(data), C.byref(info))
    if rc != OK:
        raise B200Error(rc, "jpeg_parse: stb's JPEG header walk fails")
    n = info.n_comp
    return dict(w=info.w, h=info.h, n_comp=n, h_samp=list(info.h_samp[:n]), v_samp=list(info.v_samp[:n]),
                restart_interval=info.restart_interval, progressive=bool(info.progressive),
                supported=bool(info.supported), reason=info.reason.decode())


class PngInfo(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("bit_depth", C.c_int), ("color_type", C.c_int), ("interlace", C.c_int),
                ("palette_len", C.c_int), ("trns", C.c_int), ("cgbi", C.c_int), ("apng", C.c_int),
                ("idat_bytes", C.c_ulonglong), ("supported", C.c_int), ("reason", C.c_char * 96)]


def png_parse(data):
    """b200timg_png_parse (host only): a dict of w, h, bit_depth, color_type, interlace, palette_len, trns (0 none,
    1 palette alpha, 2 colour key), cgbi, apng, idat_bytes, supported and reason.  Raises B200Error(EINVAL) where stb's
    chunk walk fails (so the reference's source fails), a non-PNG file included."""
    data = bytes(data)
    info = PngInfo()
    rc = lib().b200timg_png_parse(data, len(data), C.byref(info))
    if rc != OK:
        raise B200Error(rc, "png_parse: stb's PNG chunk walk fails")
    return dict(w=info.w, h=info.h, bit_depth=info.bit_depth, color_type=info.color_type, interlace=info.interlace,
                palette_len=info.palette_len, trns=info.trns, cgbi=bool(info.cgbi), apng=bool(info.apng),
                idat_bytes=info.idat_bytes, supported=bool(info.supported), reason=info.reason.decode())


class QoiInfo(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("channels", C.c_int), ("colorspace", C.c_int), ("supported", C.c_int),
                ("reason", C.c_char * 96)]


def qoi_parse(data):
    """b200timg_qoi_parse (host only): a dict of w, h, channels, colorspace, supported and reason.  Raises
    B200Error(EINVAL) where qoi_decode returns NULL (so the reference's QOI source fails and timg tries STB)."""
    data = bytes(data)
    info = QoiInfo()
    rc = lib().b200timg_qoi_parse(data, len(data), C.byref(info))
    if rc != OK:
        raise B200Error(rc, "qoi_parse: qoi_decode rejects the header")
    return dict(w=info.w, h=info.h, channels=info.channels, colorspace=info.colorspace,
                supported=bool(info.supported), reason=info.reason.decode())


class RasterInfo(C.Structure):
    _fields_ = [("format", C.c_int), ("w", C.c_int), ("h", C.c_int), ("channels", C.c_int), ("bpp", C.c_int),
                ("palette", C.c_int), ("top_down", C.c_int), ("rle", C.c_int), ("supported", C.c_int),
                ("reason", C.c_char * 96)]


RASTER_FORMATS = ("bmp", "tga", "pnm")


def raster_parse(data):
    """b200timg_raster_parse (host only) of a BMP, TGA or binary PNM file: a dict of format ('bmp', 'tga' or 'pnm'),
    w, h, channels, bpp, palette, top_down, rle, supported and reason.  Raises B200Error(EINVAL) where stb's test
    rejects the file or its load fails before the pixels (so the reference's STB source fails)."""
    data = bytes(data)
    info = RasterInfo()
    rc = lib().b200timg_raster_parse(data, len(data), C.byref(info))
    if rc != OK:
        raise B200Error(rc, "raster_parse: stb's header walk fails")
    return dict(format=RASTER_FORMATS[info.format], w=info.w, h=info.h, channels=info.channels, bpp=info.bpp,
                palette=info.palette, top_down=bool(info.top_down), rle=bool(info.rle),
                supported=bool(info.supported), reason=info.reason.decode())


def _file_args(files):
    files = [bytes(f) for f in files]
    bufs = (C.c_char_p * len(files))(*files)
    sizes = (C.c_size_t * len(files))(*[len(f) for f in files])
    return files, bufs, sizes


def _np_ptr(a):
    return a.ctypes.data_as(u8p)


def _source_frames(frames):
    """Batch sources as contiguous bytes, frame-major: RGBA [n,h,w,4] uint8, or one flat YUV frame per row in uint8
    or uint16 samples (the 10-bit formats), reinterpreted bytewise, never converted."""
    frames = np.ascontiguousarray(frames)
    if frames.dtype == np.uint16:
        return frames.reshape(frames.shape[0], -1).view(np.uint8)
    return np.ascontiguousarray(frames, dtype=np.uint8)


def pack_mixed(images):
    """Source frames of differing shapes ([h, w, 4] uint8 each) back to back in one uint8 array, and each frame's byte
    offset (whole RGBA frames keep every offset a multiple of 4)."""
    images = [np.ascontiguousarray(im, dtype=np.uint8) for im in images]
    offsets = np.cumsum([0] + [im.nbytes for im in images])
    flat = np.empty(max(1, int(offsets[-1])), np.uint8)
    for im, o in zip(images, offsets):
        flat[int(o):int(o) + im.nbytes] = im.reshape(-1)
    return flat, [int(o) for o in offsets[:-1]]


def mixed_batch(shapes, outs, src_offsets, indents=None, flags=0, src_fmt=FMT_RGBA, has_bg=True, bg=0xFF000000, pattern=0,
                pattern_w=0, pattern_h=0):
    """(b200timg_mixed_batch, its frame array): keep both alive for the call.  shapes: each source's (h, w[, 4]); outs:
    each frame's (out_w, out_h); indents: each frame's x_indent_cells (default 0)."""
    n = len(outs)
    frames = (Frame * max(1, n))()
    for f in range(n):
        h, w = shapes[f][:2]
        frames[f] = Frame(src_offsets[f], w, h, outs[f][0], outs[f][1], indents[f] if indents is not None else 0)
    return MixedBatch(n, src_fmt, flags, int(has_bg), bg, pattern, pattern_w, pattern_h, frames), frames


def _device_tensor(torch, a):
    """Device copy of a numpy array for the _dev entry points.  torch without CUDA only reaches here under the CPU kernel
    simulator (tools/cusim), whose device memory is host memory: a Context cannot exist otherwise."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.cuda() if torch.cuda.is_available() else t.clone()


def device_sync(torch):
    """Wait for every stream of the device, the context's own included (torch's copies run on torch's stream, which
    does not wait for the context's).  Nothing to wait for under the CPU kernel simulator."""
    if torch.cuda.is_available():
        torch.cuda.synchronize()


class Context:
    """One b200timg_ctx.  Raises B200Error(ENODEV) when no CUDA device is usable."""

    def __init__(self, device=0, stream=None):
        h = C.c_void_p()
        rc = lib().b200timg_ctx_create(device, stream, C.byref(h))
        if rc != OK:
            raise B200Error(rc, "ctx_create failed (no usable CUDA device? this library has no CPU path)")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.b200timg_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _chk(self, rc):
        if rc != OK:
            raise B200Error(rc, lib().b200timg_last_error(self.h).decode())

    @property
    def launches(self):
        return lib().b200timg_kernel_launches(self.h)

    # ---- single-frame host entry points (numpy in / numpy or bytes out)
    def scale(self, img, ow, oh, fmt=FMT_RGBA, fast=False):
        """fast: False/0 bit-exact STB semantics, True/1 <= 1 LSB mode, 2 libswscale-style bilinear."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        ih, iw = img.shape[:2]
        out = np.empty((oh, ow, 4), np.uint8)
        self._chk(lib().b200timg_scale_rgba_mode(self.h, _np_ptr(img), iw, ih, fmt, _np_ptr(out), ow, oh, int(fast)))
        return out

    def yuv_scale(self, yuv, iw, ih, ow, oh, fmt=FMT_I420):
        """yuv: one frame of a YUV format as a flat uint8 or uint16 array (uint16 for the 10-bit formats' samples)
        whose byte size is the format's layout (I420 / NV12: iw*ih*3/2 bytes) -> RGBA [oh, ow, 4]."""
        yuv = np.ascontiguousarray(yuv).reshape(-1)
        if yuv.dtype not in (np.uint8, np.uint16):
            raise TypeError(f"yuv_scale: uint8 or uint16 samples, not {yuv.dtype}")
        yuv = yuv.view(np.uint8)
        if (fmt & 0xF) in _YUV_LAYOUT and yuv.size != yuv_frame_bytes(fmt, iw, ih):
            raise B200Error(EINVAL, f"yuv_scale: {yuv.size} bytes, format {fmt} at {iw}x{ih} has {yuv_frame_bytes(fmt, iw, ih)}")
        out = np.empty((oh, ow, 4), np.uint8)
        self._chk(lib().b200timg_yuv_scale(self.h, _np_ptr(yuv), iw, ih, fmt, _np_ptr(out), ow, oh))
        return out

    def exif_op(self, fb, mirror=False, angle=0):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        out = np.empty((w, h, 4) if angle in (90, -90) else (h, w, 4), np.uint8)
        self._chk(lib().b200timg_exif_op(self.h, _np_ptr(fb), w, h, int(mirror), angle, _np_ptr(out)))
        return out

    def trim_bbox(self, fb):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        r = (C.c_int * 4)()
        self._chk(lib().b200timg_trim_bbox(self.h, _np_ptr(fb), w, h, r))
        return tuple(r)

    def windows(self, img, dw, dh, x0=0, y0=0, dx=0, dy=0, first_pos=0, n_pos=1):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        h, w = img.shape[:2]
        out = np.empty((n_pos, dh, dw, 4), np.uint8)
        self._chk(lib().b200timg_windows(self.h, _np_ptr(img), w, h, dw, dh, x0, y0, dx, dy, first_pos, n_pos, _np_ptr(out)))
        return out

    def png_encode(self, fb, rgb24=False, want_base64=True):
        """(PNG bytes, base64 text or None) of an RGBA frame, as the kitty / iTerm2 canvases would send it."""
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        n = lib().b200timg_png_size(w, h, int(rgb24))
        out = np.empty(n, np.uint8)
        nb = lib().b200timg_base64_size(n)
        b64 = C.create_string_buffer(nb) if want_base64 else None
        self._chk(lib().b200timg_png_encode(self.h, _np_ptr(fb), w, h, int(rgb24), _np_ptr(out), n, b64, nb if want_base64 else 0))
        return out.tobytes(), (b64.raw if want_base64 else None)

    def compose_bg(self, fb, bg, pattern=0, pw=0, ph=0, start_row=0, has_bg=True):
        out = np.ascontiguousarray(fb, dtype=np.uint8).copy()
        h, w = out.shape[:2]
        self._chk(lib().b200timg_compose_bg(self.h, _np_ptr(out), w, h, int(has_bg), bg, pattern, pw, ph,
                                            start_row))
        return out

    def has_transparency(self, fb, start_row=0):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        r = C.c_int()
        self._chk(lib().b200timg_has_transparency(self.h, _np_ptr(fb), w, h, start_row, C.byref(r)))
        return bool(r.value)

    def blocks_encode(self, fb, prev=None, flags=0, x_indent_cells=0):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        cap = lib().b200timg_blocks_bound(w, h) + 64
        buf = C.create_string_buffer(cap)
        n = C.c_size_t()
        pp = None
        if prev is not None:
            prev = np.ascontiguousarray(prev, dtype=np.uint8)
            assert prev.shape == fb.shape
            pp = _np_ptr(prev)
        self._chk(lib().b200timg_blocks_encode(self.h, _np_ptr(fb), w, h, pp, flags, x_indent_cells, buf, cap,
                                               C.byref(n)))
        return buf.raw[:n.value]

    def sixel_encode(self, fb):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        cap = 4096 + 6 * w * h
        buf = C.create_string_buffer(cap)
        n = C.c_size_t()
        rc = lib().b200timg_sixel_encode(self.h, _np_ptr(fb), w, h, buf, cap, C.byref(n))
        if rc == ENOSPC:                       # sized exactly by the library before anything is written
            cap = n.value
            buf = C.create_string_buffer(cap)
            rc = lib().b200timg_sixel_encode(self.h, _np_ptr(fb), w, h, buf, cap, C.byref(n))
        self._chk(rc)
        return buf.raw[:n.value]

    def profile(self, enable=True):
        self._chk(lib().b200timg_profile(self.h, int(enable)))

    def profile_report(self):
        """{kernel name: (launches, total_ms)} since profile(True)."""
        buf = C.create_string_buffer(1 << 16)
        self._chk(lib().b200timg_profile_report(self.h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms = line.split()
            out[name] = (int(n), float(ms))
        return out

    def sixel_debug(self, w, h):
        """(palette[n,3] uint8, origcolors, index[h,w]) of the last sixel_encode call."""
        pal = np.zeros(256, np.uint32)
        cnt = np.zeros(2, np.uint32)
        idx = np.zeros((h, w), np.uint8)
        self._chk(lib().b200timg_sixel_debug(self.h, pal.ctypes.data, cnt.ctypes.data, idx.ctypes.data, idx.size))
        rgb = np.stack([pal & 255, (pal >> 8) & 255, (pal >> 16) & 255], -1).astype(np.uint8)
        return rgb[: int(cnt[0])], int(cnt[1]), idx

    # ---- batches, host buffers (numpy [n,h,w,4]) -> list of bytes
    def _batch_host(self, fn, frames, b, sixel=False):
        frames = _source_frames(frames)
        n = frames.shape[0]
        if sixel:
            cap = n * (4096 + 6 * b.out_w * (b.out_h + 5))      # far above typical (~1 B/px); ENOSPC reports the need
        else:
            cap = lib().b200timg_blocks_bound(b.out_w, b.out_h) * n + 64
        out = np.empty(cap, np.uint8)
        offs = np.zeros(n + 1, np.uint64)
        self._chk(fn(self.h, C.byref(b), frames.ctypes.data, out.ctypes.data, cap, offs.ctypes.data))
        return [out[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]

    def blocks_batch(self, frames, b):
        return self._batch_host(lib().b200timg_blocks_batch, frames, b)

    def sixel_batch(self, frames, b):
        return self._batch_host(lib().b200timg_sixel_batch, frames, b, sixel=True)

    def graphics_batch(self, frames, b, protocol, rgb24=False, ids=None, with_offsets=False, cell=None, indent=0):
        """Framed kitty / iTerm2 text of every frame (list of bytes); ids: one kitty image id per frame; cell and
        indent: see graphics().  frames: numpy source frames (RGBA [n,h,w,4], or one flat YUV frame per row, uint8 or
        uint16 samples)."""
        frames = _source_frames(frames)
        n = b.n_frames
        g, keep = graphics(protocol, rgb24, ids, cell, indent)
        sizes = [lib().b200timg_graphics_size(C.byref(g), b.out_w, b.out_h, int(keep[f]) if keep is not None else 0)
                 for f in range(n)]
        cap = max(1, sum(sizes))
        out = np.empty(cap, np.uint8)
        offs = np.zeros(n + 1, np.uint64)
        self._chk(lib().b200timg_graphics_batch(self.h, C.byref(b), C.byref(g), frames.ctypes.data, out.ctypes.data, cap,
                                                offs.ctypes.data))
        res = [out[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]
        return (res, offs) if with_offsets else res

    # ---- mixed batches: images of differing geometry (numpy [h, w, 4] each)
    def scale_mixed(self, images, outs, src_fmt=FMT_RGBA, has_bg=True, bg=0xFF000000, pattern=0, pattern_w=0, pattern_h=0):
        """b200timg_scale_mixed_dev on the packed images: the scaled, composed frames as a list of [oh, ow, 4] arrays."""
        import torch
        flat, offs = pack_mixed(images)
        b, keep = mixed_batch([im.shape for im in images], outs, offs, None, 0, src_fmt, has_bg, bg, pattern, pattern_w,
                              pattern_h)
        d_src = _device_tensor(torch, flat)
        sizes = [ow * oh * 4 for ow, oh in outs]
        d_out = torch.empty(max(1, sum(sizes)), dtype=torch.uint8, device=d_src.device)
        self._chk(lib().b200timg_scale_mixed_dev(self.h, C.byref(b), d_src.data_ptr(), d_out.data_ptr()))
        device_sync(torch)
        host = d_out.cpu().numpy()
        res, o = [], 0
        for (ow, oh), n in zip(outs, sizes):
            res.append(host[o:o + n].reshape(oh, ow, 4).copy())
            o += n
        return res

    def blocks_mixed(self, images, outs, indents=None, flags=0, src_fmt=FMT_RGBA, has_bg=True, bg=0xFF000000, pattern=0,
                     pattern_w=0, pattern_h=0):
        """b200timg_blocks_mixed (host buffers): each frame's block bytes, as a list of bytes."""
        flat, offs = pack_mixed(images)
        b, keep = mixed_batch([im.shape for im in images], outs, offs, indents, flags, src_fmt, has_bg, bg, pattern,
                              pattern_w, pattern_h)
        n = len(outs)
        cap = sum(lib().b200timg_blocks_bound(ow, oh) for ow, oh in outs) + 64
        out = np.empty(cap, np.uint8)
        o = np.zeros(n + 1, np.uint64)
        self._chk(lib().b200timg_blocks_mixed(self.h, C.byref(b), flat.ctypes.data, out.ctypes.data, cap, o.ctypes.data))
        return [out[int(o[i]):int(o[i + 1])].tobytes() for i in range(n)]

    def blocks_mixed_dev(self, d_src, b, d_out=None, out_cap=None, d_offsets=None):
        """b200timg_blocks_mixed_dev on a packed source tensor (see pack_mixed / mixed_batch): returns (d_out, d_offsets)
        after the (asynchronous) call -- device_sync() before reading them; d_out defaults to the sum of the frames' block
        bounds."""
        import torch
        n = b.n_frames
        if d_out is None:
            cap = sum(lib().b200timg_blocks_bound(b.frames[f].out_w, b.frames[f].out_h) for f in range(n))
            d_out = torch.empty(cap, dtype=torch.uint8, device=d_src.device)
        if out_cap is None:
            out_cap = d_out.numel()
        if d_offsets is None:
            d_offsets = torch.empty(n + 1, dtype=torch.int64, device=d_src.device)
        self._chk(lib().b200timg_blocks_mixed_dev(self.h, C.byref(b), d_src.data_ptr(), d_out.data_ptr(), out_cap,
                                                  d_offsets.data_ptr()))
        return d_out, d_offsets

    @staticmethod
    def sixel_mixed_bound(outs):
        """Staging bytes of a sixel mixed batch: the sum of b200timg_sixel_bound(out_w, round_to_sixel(out_h))."""
        return sum(lib().b200timg_sixel_bound(ow, (oh + 5) // 6 * 6) for ow, oh in outs)

    def sixel_mixed(self, images, outs, src_fmt=FMT_RGBA, has_bg=True, bg=0xFF000000, pattern=0, pattern_w=0, pattern_h=0):
        """b200timg_sixel_mixed (host buffers): each frame's sixel stream, as a list of bytes."""
        flat, offs = pack_mixed(images)
        b, keep = mixed_batch([im.shape for im in images], outs, offs, None, 0, src_fmt, has_bg, bg, pattern, pattern_w,
                              pattern_h)
        n = len(outs)
        cap = self.sixel_mixed_bound(outs)
        out = np.empty(cap, np.uint8)
        o = np.zeros(n + 1, np.uint64)
        self._chk(lib().b200timg_sixel_mixed(self.h, C.byref(b), flat.ctypes.data, out.ctypes.data, cap, o.ctypes.data))
        return [out[int(o[i]):int(o[i + 1])].tobytes() for i in range(n)]

    def sixel_mixed_dev(self, d_src, b, d_out=None, out_cap=None, d_offsets=None):
        """b200timg_sixel_mixed_dev on a packed source tensor (see pack_mixed / mixed_batch): returns (d_out, d_offsets)
        after the (asynchronous) call -- device_sync() before reading them; d_out defaults to the sum of the frames' sixel
        bounds."""
        import torch
        n = b.n_frames
        if d_out is None:
            cap = self.sixel_mixed_bound([(b.frames[f].out_w, b.frames[f].out_h) for f in range(n)])
            d_out = torch.empty(cap, dtype=torch.uint8, device=d_src.device)
        if out_cap is None:
            out_cap = d_out.numel()
        if d_offsets is None:
            d_offsets = torch.empty(n + 1, dtype=torch.int64, device=d_src.device)
        self._chk(lib().b200timg_sixel_mixed_dev(self.h, C.byref(b), d_src.data_ptr(), d_out.data_ptr(), out_cap,
                                                 d_offsets.data_ptr()))
        return d_out, d_offsets

    def graphics_batch_dev(self, d_src, b, protocol, rgb24=False, ids=None, d_out=None, out_cap=None, d_offsets=None,
                           cell=None, indent=0):
        """Device-resident variant on torch CUDA tensors: returns (d_out, d_offsets) after the (asynchronous) call;
        allocates them when not given (out_cap defaults to the exact size of the batch)."""
        import torch
        g, keep = graphics(protocol, rgb24, ids, cell, indent)
        n = b.n_frames
        if d_out is None:
            need = sum(lib().b200timg_graphics_size(C.byref(g), b.out_w, b.out_h, int(keep[f]) if keep is not None else 0)
                       for f in range(n))
            d_out = torch.empty(max(1, need), dtype=torch.uint8, device=d_src.device)
        if out_cap is None:
            out_cap = d_out.numel()
        if d_offsets is None:
            d_offsets = torch.empty(n + 1, dtype=torch.int64, device=d_src.device)
        self._chk(lib().b200timg_graphics_batch_dev(self.h, C.byref(b), C.byref(g), d_src.data_ptr(), d_out.data_ptr(),
                                                    out_cap, d_offsets.data_ptr()))
        return d_out, d_offsets

    def gif_frames(self, data, n=None):
        """b200timg_gif_frames: (canvases [n, h, w, 4] uint8, n_valid) of a GIF's first n frames (default: every frame
        gif_parse reports); canvases from n_valid on are unspecified."""
        data = bytes(data)
        w, h, delays = gif_parse(data)
        n = len(delays) if n is None else n
        out = np.empty((max(1, n), h, w, 4), np.uint8)
        valid = C.c_int()
        self._chk(lib().b200timg_gif_frames(self.h, data, len(data), n, out.ctypes.data, C.byref(valid)))
        return out[:n], valid.value

    def gif_frames_dev(self, data, d_frames, n):
        """b200timg_gif_frames_dev into a device tensor of at least n * h * w * 4 bytes (the source of a uniform batch):
        returns d_valid, a one-element int32 device tensor, after the (asynchronous) call."""
        import torch
        data = bytes(data)
        w, h, _ = gif_parse(data)
        if d_frames.numel() * d_frames.element_size() < n * w * h * 4:
            raise B200Error(EINVAL, f"gif_frames_dev: d_frames holds fewer than {n} canvases of {w}x{h}")
        d_valid = torch.empty(1, dtype=torch.int32, device=d_frames.device)
        self._chk(lib().b200timg_gif_frames_dev(self.h, data, len(data), n, d_frames.data_ptr(), d_valid.data_ptr()))
        return d_valid

    def _files_frames(self, fn, parse, files):
        """The host form of a multi-file decode (jpeg_frames, png_frames, qoi_frames); parse gives each file's w and h."""
        files, bufs, sizes = _file_args(files)
        geo = [parse(f) for f in files]
        total = sum(g["w"] * g["h"] * 4 for g in geo)
        out = np.empty(max(1, total), np.uint8)
        status = np.zeros(max(1, len(files)), np.int32)
        self._chk(fn(self.h, len(files), bufs, sizes, out.ctypes.data, status.ctypes.data))
        canv, o = [], 0
        for g in geo:
            canv.append(out[o:o + g["w"] * g["h"] * 4].reshape(g["h"], g["w"], 4))
            o += g["w"] * g["h"] * 4
        return canv, status[:len(files)]

    def _files_frames_dev(self, fn, files, d_frames, d_status):
        """The dev form of a multi-file decode (jpeg_frames_dev, png_frames_dev, qoi_frames_dev)."""
        import torch
        files, bufs, sizes = _file_args(files)
        if d_status is None:
            d_status = torch.empty(max(1, len(files)), dtype=torch.int32, device=d_frames.device)
        self._chk(fn(self.h, len(files), bufs, sizes, d_frames.data_ptr(), d_status.data_ptr()))
        return d_status

    def jpeg_frames(self, files):
        """b200timg_jpeg_frames: (list of [h, w, 4] uint8 canvases, int32 status per file) for a list of JPEG files."""
        return self._files_frames(lib().b200timg_jpeg_frames, jpeg_parse, files)

    def jpeg_frames_dev(self, files, d_frames, d_status=None):
        """b200timg_jpeg_frames_dev into a device tensor holding every canvas back to back (the src_offset layout of a
        mixed batch): returns d_status, an int32 device tensor with one entry per file, after the (asynchronous) call."""
        return self._files_frames_dev(lib().b200timg_jpeg_frames_dev, files, d_frames, d_status)

    def png_frames(self, files):
        """b200timg_png_frames: (list of [h, w, 4] uint8 canvases, int32 status per file) for a list of PNG files."""
        return self._files_frames(lib().b200timg_png_frames, png_parse, files)

    def png_frames_dev(self, files, d_frames, d_status=None):
        """b200timg_png_frames_dev into a device tensor holding every canvas back to back (the src_offset layout of a
        mixed batch): returns d_status, an int32 device tensor with one entry per file, after the (asynchronous) call."""
        return self._files_frames_dev(lib().b200timg_png_frames_dev, files, d_frames, d_status)

    def qoi_frames(self, files):
        """b200timg_qoi_frames: (list of [h, w, 4] uint8 canvases, int32 status per file) for a list of QOI files;
        status 2 marks a 3-channel file with alpha below 255, which timg shows uncomposed."""
        return self._files_frames(lib().b200timg_qoi_frames, qoi_parse, files)

    def qoi_frames_dev(self, files, d_frames, d_status=None):
        """b200timg_qoi_frames_dev into a device tensor holding every canvas back to back (the src_offset layout of a
        mixed batch): returns d_status, an int32 device tensor with one entry per file, after the (asynchronous) call."""
        return self._files_frames_dev(lib().b200timg_qoi_frames_dev, files, d_frames, d_status)

    def raster_frames(self, files):
        """b200timg_raster_frames: (list of [h, w, 4] uint8 canvases, int32 status per file) for a list of BMP, TGA and
        PNM files in any mix; status -1 marks a BMP whose canvas reads stb's uninitialised palette."""
        return self._files_frames(lib().b200timg_raster_frames, raster_parse, files)

    def raster_frames_dev(self, files, d_frames, d_status=None):
        """b200timg_raster_frames_dev into a device tensor holding every canvas back to back (the src_offset layout of
        a mixed batch): returns d_status, an int32 device tensor with one entry per file, after the (asynchronous) call."""
        return self._files_frames_dev(lib().b200timg_raster_frames_dev, files, d_frames, d_status)

    @staticmethod
    def graphics_mixed_bound(b, g):
        """Bytes of a kitty / iTerm2 mixed batch with stored blocks (the exact size; an upper bound with DEFLATE): the sum
        of b200timg_graphics_size over the frames, each with its own indent and id."""
        kitty = (g.protocol & ~DEFLATE) != ITERM2
        total = 0
        for f in range(b.n_frames):
            F = b.frames[f]
            gf = Graphics(g.protocol, g.rgb24, None, g.cell_x_px, g.cell_y_px, F.x_indent_cells)
            total += lib().b200timg_graphics_size(C.byref(gf), F.out_w, F.out_h, int(g.ids[f]) if kitty else 0)
        return total

    def graphics_mixed(self, images, outs, protocol, rgb24=False, ids=None, indents=None, cell=None, deflate=False,
                       with_offsets=False, **compose):
        """b200timg_graphics_mixed (host buffers): each frame's framed kitty / iTerm2 text, as a list of bytes (and the
        offsets with with_offsets).  ids: one kitty image id per frame; indents: each frame's tmux placeholder indent
        (x_indent_cells); cell: (cell_x_px, cell_y_px) of the tmux form; compose: has_bg, bg, pattern, ... as mixed_batch."""
        flat, offs = pack_mixed(images)
        b, keep = mixed_batch([im.shape for im in images], outs, offs, indents, compose.pop("flags", 0), **compose)
        g, keep_ids = graphics(protocol | (DEFLATE if deflate else 0), rgb24, ids, cell)
        n = len(outs)
        cap = max(1, self.graphics_mixed_bound(b, g))
        out = np.empty(cap, np.uint8)
        o = np.zeros(n + 1, np.uint64)
        self._chk(lib().b200timg_graphics_mixed(self.h, C.byref(b), C.byref(g), flat.ctypes.data, out.ctypes.data, cap,
                                                o.ctypes.data))
        res = [out[int(o[i]):int(o[i + 1])].tobytes() for i in range(n)]
        return (res, o) if with_offsets else res

    def graphics_mixed_dev(self, d_src, b, g, d_out=None, out_cap=None, d_offsets=None):
        """b200timg_graphics_mixed_dev on a packed source tensor (see pack_mixed / mixed_batch) with a protocol description
        from graphics() (keep its id array alive): returns (d_out, d_offsets) after the (asynchronous) call --
        device_sync() before reading them; d_out defaults to graphics_mixed_bound."""
        import torch
        n = b.n_frames
        if d_out is None:
            d_out = torch.empty(max(1, self.graphics_mixed_bound(b, g)), dtype=torch.uint8, device=d_src.device)
        if out_cap is None:
            out_cap = d_out.numel()
        if d_offsets is None:
            d_offsets = torch.empty(n + 1, dtype=torch.int64, device=d_src.device)
        self._chk(lib().b200timg_graphics_mixed_dev(self.h, C.byref(b), C.byref(g), d_src.data_ptr(), d_out.data_ptr(), out_cap,
                                                    d_offsets.data_ptr()))
        return d_out, d_offsets
