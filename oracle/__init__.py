"""TEST INFRASTRUCTURE ONLY.

ctypes doors onto (a) oracle/liboracle.so -- our CPU restatement of the reference's
hot-path arithmetic (oracle/*.c) and (b) oracle/_ref/libtimg_ref.so -- the reference's
own translation units compiled in place by oracle/Makefile (present only where it was
built: this container, or shipped prebuilt to the GPU box).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this package.  The product (timg_b200) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORC = None
_REF = None


def build(quiet=True):
    """Compile liboracle.so and (if /root/reference is present) _ref/libtimg_ref.so."""
    subprocess.run(["make", "-C", _HERE, "all"], check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def _sig(lib, name, res, args):
    f = getattr(lib, name)
    f.restype = res
    f.argtypes = args
    return f


u8p = C.POINTER(C.c_uint8)


def _ptr(a):
    return a.ctypes.data_as(u8p)


def lib():
    global _ORC
    if _ORC is None:
        p = os.path.join(_HERE, "liboracle.so")
        srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith(".c")]
        if (not os.path.exists(p)) or any(os.path.getmtime(s) > os.path.getmtime(p) for s in srcs):
            build()
        L = C.CDLL(p)
        _sig(L, "orc_as256", C.c_int, [C.c_uint32])
        _sig(L, "orc_compose_bg", None, [u8p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                         C.c_int, C.c_int, C.c_int])
        _sig(L, "orc_calc_fit", C.c_int, [C.c_int] * 6 + [C.c_float] + [C.c_int] * 5 +
             [C.POINTER(C.c_int)] * 2)
        _sig(L, "orc_blocks_new", C.c_void_p, [C.c_int] * 3)
        _sig(L, "orc_blocks_free", None, [C.c_void_p])
        _sig(L, "orc_blocks_bound", C.c_long, [C.c_int, C.c_int])
        _sig(L, "orc_blocks_send", C.c_long, [C.c_void_p, C.c_int, C.c_int, u8p, C.c_int, C.c_int,
                                              C.c_char_p, C.c_int, C.c_char_p])
        _sig(L, "orc_stb_resize", C.c_int, [u8p, C.c_int, C.c_int, C.c_int, u8p, C.c_int, C.c_int,
                                            C.POINTER(C.c_int)])
        _sig(L, "orc_stb_plan", C.c_int, [C.c_int] * 5 + [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p])
        _sig(L, "orc_sixel_encode", C.c_long, [u8p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_long, u8p,
                                              C.POINTER(C.c_int), C.POINTER(C.c_int), u8p])
        _sig(L, "orc_sixel_palette", C.c_int, [u8p, C.c_int, C.c_int, C.c_int, u8p, C.POINTER(C.c_int)])
        _sig(L, "orc_sixel_stream", C.c_long, [u8p, C.c_int, C.c_int, u8p, C.c_int, C.c_char_p, C.c_long])
        _sig(L, "orc_sixel_decode", C.c_int, [C.c_char_p, C.c_long, u8p, C.c_long, C.POINTER(C.c_int),
                                              C.POINTER(C.c_int), C.POINTER(C.c_int)])
        _ORC = L
    return _ORC


def have_ref():
    return os.path.exists(os.path.join(_HERE, "_ref", "libtimg_ref.so"))


def ref():
    """The reference itself (UNMODIFIED timg TUs). Raises if it was not built."""
    global _REF
    if _REF is None:
        p = os.path.join(_HERE, "_ref", "libtimg_ref.so")
        if not os.path.exists(p):
            if os.path.exists("/root/reference/src/framebuffer.cc"):
                build()
            else:
                raise RuntimeError("oracle/_ref/libtimg_ref.so not built and /root/reference absent")
        L = C.CDLL(p)
        _sig(L, "ref_calc_fit", C.c_int, [C.c_int] * 6 + [C.c_float] + [C.c_int] * 5 +
             [C.POINTER(C.c_int)] * 2)
        _sig(L, "ref_scale", C.c_int, [u8p, C.c_int, C.c_int, C.c_int, u8p, C.c_int, C.c_int])
        _sig(L, "ref_compose", None, [u8p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                      C.c_int, C.c_int, C.c_int])
        _sig(L, "ref_as256", C.c_int, [C.c_uint32])
        _sig(L, "ref_parse_color", C.c_uint32, [C.c_char_p])
        _sig(L, "ref_blocks_new", C.c_void_p, [C.c_int] * 4)
        _sig(L, "ref_blocks_prefix", None, [C.c_void_p, C.c_char_p, C.c_int])
        _sig(L, "ref_blocks_send", C.c_long, [C.c_void_p, C.c_int, C.c_int, u8p, C.c_int, C.c_int,
                                              C.c_int, C.c_char_p, C.c_long])
        _sig(L, "ref_blocks_free", None, [C.c_void_p])
        _sig(L, "ref_fb_new", C.c_void_p, [C.c_int, C.c_int])
        _sig(L, "ref_fb_free", None, [C.c_void_p])
        _sig(L, "ref_fb_data", u8p, [C.c_void_p])
        _sig(L, "ref_scale_fb", C.c_int, [C.c_void_p, C.c_void_p])
        _sig(L, "ref_compose_fb", None, [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32,
                                         C.c_int, C.c_int, C.c_int])
        _sig(L, "ref_blocks_send_fb", None, [C.c_void_p, C.c_int, C.c_int, C.c_void_p])
        _sig(L, "ref_blocks_flush", None, [C.c_void_p])
        _REF = L
    return _REF


def rgba_u32(r, g, b, a=255):
    return (r & 255) | ((g & 255) << 8) | ((b & 255) << 16) | ((a & 255) << 24)


# ----------------------------------------------------------------- restatement (ours)
def as256(rgba):
    return lib().orc_as256(rgba)


def compose_bg(fb, bg, pattern=0, pw=0, ph=0, start_row=0, has_bg=True):
    out = np.ascontiguousarray(fb, dtype=np.uint8).copy()
    h, w = out.shape[:2]
    lib().orc_compose_bg(_ptr(out), w, h, int(has_bg), bg, pattern, pw, ph, start_row)
    return out


def calc_fit(iw, ih, width, height, cell_x=1, cell_y=2, stretch=1.0, upscale=False,
             upscale_integer=False, fill_width=False, fill_height=False, rotated=False,
             impl=None):
    tw, th = C.c_int(), C.c_int()
    f = (impl or lib().orc_calc_fit)
    r = f(iw, ih, width, height, cell_x, cell_y, stretch, int(upscale), int(upscale_integer),
          int(fill_width), int(fill_height), int(rotated), C.byref(tw), C.byref(th))
    return bool(r), tw.value, th.value


def stb_resize(img, ow, oh, fmt=0, want_info=False):
    """Restatement of ImageScaler::Scale (STB build). info = [vertical_first, h_widest, v_widest, channels]."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    ih, iw = img.shape[:2]
    out = np.empty((oh, ow, 4), np.uint8)
    info = (C.c_int * 4)()
    rc = lib().orc_stb_resize(_ptr(img), iw, ih, fmt, _ptr(out), ow, oh, info)
    assert rc == 0, rc
    return (out, list(info)) if want_info else out


def stb_plan(iw, ih, ow, oh, axis):
    n = ow if axis == 0 else oh
    widest, flags = C.c_int(), C.c_int()
    assert lib().orc_stb_plan(iw, ih, ow, oh, axis, C.byref(widest), C.byref(flags), None, None, None, None) == 0
    first, count, lead = (np.zeros(n, np.int32) for _ in range(3))
    coeff = np.zeros(n * widest.value, np.float32)
    assert lib().orc_stb_plan(iw, ih, ow, oh, axis, None, None, first.ctypes.data, count.ctypes.data,
                              lead.ctypes.data, coeff.ctypes.data) == 0
    return dict(widest=widest.value, flags=flags.value, first=first, count=count, lead=lead,
                coeff=coeff.reshape(n, widest.value))


def sixel_encode(fb, want_details=False, mode=0):
    """Restatement of libsixel's encode for the reference's call sequence (PARITY UNPINNED).
    mode 0 = libsixel-faithful; mode 1 = order-free "device semantics" (see oracle/sixel_oracle.c)."""
    fb = np.ascontiguousarray(fb, dtype=np.uint8)
    h, w = fb.shape[:2]
    cap = 1024 + w * h * 5 + 256 * 24        # the reference's own bound, src/sixel-canvas.cc:123
    buf = C.create_string_buffer(cap)
    pal = np.zeros((256, 3), np.uint8)
    idx = np.zeros((h, w), np.uint8)
    nc, oc = C.c_int(), C.c_int()
    n = lib().orc_sixel_encode(_ptr(fb), w, h, mode, buf, cap, _ptr(pal), C.byref(nc), C.byref(oc), _ptr(idx))
    assert n > 0, n
    if want_details:
        return buf.raw[:n], dict(palette=pal[:nc.value], ncolors=nc.value, origcolors=oc.value, index=idx)
    return buf.raw[:n]


def sixel_palette(fb, mode=0):
    fb = np.ascontiguousarray(fb, dtype=np.uint8)
    h, w = fb.shape[:2]
    pal = np.zeros((256, 3), np.uint8)
    oc = C.c_int()
    n = lib().orc_sixel_palette(_ptr(fb), w, h, mode, _ptr(pal), C.byref(oc))
    return pal[:n], oc.value


def sixel_stream(palette, index):
    """The device emitters' bytes for a palette ([n,3] uint8) and an index plane ([h,w] uint8): the same framing as
    sixel_encode, bands written colour by colour (see orc_sixel_stream in oracle/sixel_oracle.c)."""
    pal = np.ascontiguousarray(palette, dtype=np.uint8).reshape(-1, 3)
    idx = np.ascontiguousarray(index, dtype=np.uint8)
    h, w = idx.shape
    cap = 4096 + 256 * 24 + ((h + 5) // 6) * (6 * w * 14 + 256 * 6)    # <= 6 runs a column, <= 14 bytes with its gap
    buf = C.create_string_buffer(cap)
    n = lib().orc_sixel_stream(_ptr(idx), w, h, _ptr(pal), len(pal), buf, cap)
    assert n > 0, n
    return buf.raw[:n]


def sixel_decode(data, max_px=1 << 26):
    """Decode a DCS sixel stream -> (HxWx3 uint8, colours used)."""
    w, h, used = C.c_int(), C.c_int(), C.c_int()
    out = np.zeros(max_px * 3, np.uint8)
    rc = lib().orc_sixel_decode(data, len(data), _ptr(out), max_px, C.byref(w), C.byref(h), C.byref(used))
    if rc != 0:
        raise ValueError(f"malformed sixel stream ({rc})")
    return out[: w.value * h.value * 3].reshape(h.value, w.value, 3).copy(), used.value


def rgb_to_lab(rgb):
    """sRGB (D65) -> CIE L*a*b*, float64, for CIE76 delta-E."""
    c = rgb.astype(np.float64) / 255.0
    c = np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)
    m = np.array([[0.4124564, 0.3575761, 0.1804375], [0.2126729, 0.7151522, 0.0721750],
                  [0.0193339, 0.1191920, 0.9503041]])
    xyz = c @ m.T / np.array([0.95047, 1.0, 1.08883])
    f = np.where(xyz > 216 / 24389, np.cbrt(xyz), (24389 / 27 * xyz + 16) / 116)
    return np.stack([116 * f[..., 1] - 16, 500 * (f[..., 0] - f[..., 1]), 200 * (f[..., 1] - f[..., 2])], -1)


def mean_delta_e(a_rgb, b_rgb, blur=0):
    """Mean CIE76 delta-E between two RGB images; blur>0 box-filters both first (dither noise
    averages out over a (2*blur+1)^2 neighbourhood, which is how a dithered image is perceived)."""
    a, b = a_rgb.astype(np.float64), b_rgb.astype(np.float64)
    if blur:
        k = 2 * blur + 1

        def box(x):
            p = np.pad(x, ((blur, blur), (blur, blur), (0, 0)), mode="edge")
            cs = np.cumsum(np.cumsum(np.pad(p, ((1, 0), (1, 0), (0, 0))), 0), 1)
            return (cs[k:, k:] - cs[:-k, k:] - cs[k:, :-k] + cs[:-k, :-k]) / (k * k)
        a, b = box(a), box(b)
    d = rgb_to_lab(a) - rgb_to_lab(b)
    return float(np.sqrt((d ** 2).sum(-1)).mean())


class BlockCanvas:
    """Restatement of UnicodeBlockCanvas (stateful: backing store, last height/indent)."""

    def __init__(self, quarter=False, upper=False, color8=False):
        self._h = lib().orc_blocks_new(int(quarter), int(upper), int(color8))

    def send(self, fb, x=0, dy=0, prefix=b""):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        if dy < 0:
            # Send(): MoveCursorDY(cell_height_for_pixels(dy)) (src/unicode-block-canvas.cc:329,
            # .h:42-45: (pixels - 1) / 2 with C truncation) -> "ESC[nA" (src/terminal-canvas.cc:66-73)
            rows = int((dy - 1) / 2)
            if rows != 0:
                prefix = prefix + (b"\033[%dA" % -rows if rows < 0 else b"\033[%dB" % rows)
        buf = C.create_string_buffer(lib().orc_blocks_bound(w, h) + len(prefix))
        n = lib().orc_blocks_send(self._h, x, dy, _ptr(fb), w, h, prefix, len(prefix), buf)
        return buf.raw[:n]

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_blocks_free(self._h)
            self._h = None


# ----------------------------------------------------------------- the reference itself
class RefBlockCanvas:
    """The reference's UnicodeBlockCanvas behind its own BufferedWriteSequencer."""

    def __init__(self, quarter=False, upper=False, color8=False):
        self._h = ref().ref_blocks_new(int(quarter), int(upper), int(color8), 1)

    def prefix(self, data):
        ref().ref_blocks_prefix(self._h, data, len(data))

    def send(self, fb, x=0, dy=0):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        cap = 1 << 16
        cap += ((h + 1) // 2) * (16 + w * 39 + 5)
        buf = C.create_string_buffer(cap)
        n = ref().ref_blocks_send(self._h, x, dy, _ptr(fb), w, h, 1, buf, cap)
        assert n >= 0, n
        return buf.raw[:n]

    def __del__(self):
        if getattr(self, "_h", None):
            ref().ref_blocks_free(self._h)
            self._h = None


def ref_scale(img, ow, oh, fmt=0):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    ih, iw = img.shape[:2]
    out = np.empty((oh, ow, 4), np.uint8)
    rc = ref().ref_scale(_ptr(img), iw, ih, fmt, _ptr(out), ow, oh)
    assert rc == 0
    return out


def ref_compose_bg(fb, bg, pattern=0, pw=0, ph=0, start_row=0, has_bg=True):
    out = np.ascontiguousarray(fb, dtype=np.uint8).copy()
    h, w = out.shape[:2]
    ref().ref_compose(_ptr(out), w, h, int(has_bg), bg, pattern, pw, ph, start_row)
    return out


# ---- native multi-threaded CPU baseline (oracle/cpu_pipeline.c): no Python inside the timed region
def _stage_ptrs():
    """(scale, compose, kind): the reference's own TUs when oracle/_ref is built, else the restatements."""
    cast = lambda f: C.cast(f, C.c_void_p)
    if have_ref():
        R = ref()
        return cast(R.ref_scale), cast(R.ref_compose), "reference STB TU + reference AlphaComposeBackground (oracle/_ref)"
    L = lib()
    return cast(L.orc_stb_resize7), cast(L.orc_compose_bg), "STB + compose restatements (oracle/*.c)"


def cpu_sixel_jobs(frames, n_jobs, ow, oh, bg, threads, mode=0, has_bg=True):
    """Scale -> compose -> pad -> libsixel restatement for n_jobs frames (job j = frames[j % len]) on
    `threads` native threads.  Returns (wall seconds, encoded sizes, description of the stages)."""
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    n, ih, iw = frames.shape[:3]
    L = lib()
    f = _sig(L, "orc_cpu_sixel_jobs", C.c_double, [u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                   C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p])
    sf, cf, what = _stage_ptrs()
    sizes = np.zeros(n_jobs, np.int64)
    dt = f(_ptr(frames), n, iw, ih, n_jobs, ow, oh, int(has_bg), bg, mode, threads, sf, cf, sizes.ctypes.data)
    return dt, sizes, what + "; sixel = libsixel restatement (libsixel is not vendored in the reference)"


def cpu_blocks_jobs(frames, n_jobs, ow, oh, bg, threads, flags=0, animation=False, has_bg=True):
    """Scale -> compose -> UnicodeBlockCanvas::Send through the reference's own TUs (needs oracle/_ref)."""
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    n, ih, iw = frames.shape[:3]
    L, R = lib(), ref()
    f = _sig(L, "orc_cpu_blocks_jobs", C.c_double, [u8p] + [C.c_int] * 7 + [C.c_uint32, C.c_int, C.c_int, C.c_int] +
             [C.c_void_p] * 5)
    cast = lambda fn: C.cast(fn, C.c_void_p)
    dt = f(_ptr(frames), n, iw, ih, n_jobs, ow, oh, int(has_bg), bg, flags, int(animation), threads,
           cast(R.ref_scale), cast(R.ref_compose), cast(R.ref_blocks_new), cast(R.ref_blocks_send), cast(R.ref_blocks_free))
    return dt, "reference TUs (oracle/_ref): ImageScaler(STB) + AlphaComposeBackground + UnicodeBlockCanvas::Send to /dev/null"


# ---- libswscale-style bilinear scaling and YUV 4:2:0 -> RGBA (PARITY UNPINNED: libswscale is not in the reference tree)
def _tri_axis(src, dst):
    """Float64 statement of the triangle filter the device tables use: centre-aligned sampling, half-width
    max(1, src/dst), edge clamp by folding weights onto the border sample.  Returns a dense [dst, src] matrix."""
    r = src / dst
    half = max(r, 1.0)
    M = np.zeros((dst, src))
    for i in range(dst):
        c = (i + 0.5) * r - 0.5
        lo, hi = int(np.ceil(c - half)), int(np.floor(c + half))
        if lo == hi and half == 1.0:
            hi = lo + 1
        w = np.maximum(0.0, 1.0 - np.abs(np.arange(lo, hi + 1) - c) / half)
        w = w / w.sum()
        for j, v in zip(range(lo, hi + 1), w):
            M[i, min(max(j, 0), src - 1)] += v
    return M


def bilinear_rgba_np(img, ow, oh, fmt=0):
    img = np.asarray(img, dtype=np.float64)
    ih, iw = img.shape[:2]
    out = np.einsum("oy,yxc->oxc", _tri_axis(ih, oh), np.einsum("px,yxc->ypc", _tri_axis(iw, ow), img))
    if fmt == 1:
        out = out[..., [2, 1, 0, 3]]
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def yuv420_to_rgba_np(yuv, iw, ih, ow, oh, nv12=False, full_range=False):
    """Float64 statement of timg_b200/csrc/bilinear.cu's yuv420_rgba_kernel (BT.601)."""
    yuv = np.asarray(yuv, dtype=np.uint8).reshape(-1)
    cw, ch = iw // 2, ih // 2
    Y = yuv[: iw * ih].reshape(ih, iw).astype(np.float64)
    if nv12:
        uv = yuv[iw * ih:].reshape(ch, cw, 2).astype(np.float64)
        U, V = uv[..., 0], uv[..., 1]
    else:
        U = yuv[iw * ih: iw * ih + cw * ch].reshape(ch, cw).astype(np.float64)
        V = yuv[iw * ih + cw * ch:].reshape(ch, cw).astype(np.float64)
    # chroma is carried at half the output width (libswscale's packed-RGB writers without SWS_FULL_CHR_H_INT):
    # the two pixels of an output pair share one chroma sample
    cow = (ow + 1) // 2
    y = _tri_axis(ih, oh) @ Y @ _tri_axis(iw, ow).T
    Mv = _tri_axis(ch, oh)
    if (ow, oh) == (iw, ih):        # unscaled: chroma rows are replicated (2x2 blocks share a sample), as libswscale's unscaled path does
        Mv = np.zeros((oh, ch))
        Mv[np.arange(oh), np.arange(oh) // 2] = 1.0
    chroma = lambda P: np.repeat(Mv @ P @ _tri_axis(cw, cow).T, 2, 1)[:, :ow] - 128.0
    u, v = chroma(U), chroma(V)
    if full_range:
        r, g, b = y + 1.402 * v, y - 0.344136 * u - 0.714136 * v, y + 1.772 * u
    else:
        yl = 1.164383 * (y - 16.0)
        r, g, b = yl + 1.596027 * v, yl - 0.391762 * u - 0.812968 * v, yl + 2.017232 * u
    out = np.stack([r, g, b, np.full_like(r, 255.0)], -1)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def rgba_to_i420_np(img):
    """BT.601 limited-range RGB -> I420 bytes (2x2 box chroma), for building YUV test inputs from RGBA frames."""
    img = np.asarray(img, dtype=np.float64)
    r, g, b = img[..., 0], img[..., 1], img[..., 2]
    y = 16 + 0.256788 * r + 0.504129 * g + 0.097906 * b
    u = 128 - 0.148223 * r - 0.290993 * g + 0.439216 * b
    v = 128 + 0.439216 * r - 0.367788 * g - 0.071427 * b
    h, w = y.shape
    box = lambda p: p.reshape(h // 2, 2, w // 2, 2).mean((1, 3))
    q = lambda p: np.clip(np.rint(p), 0, 255).astype(np.uint8)
    return np.concatenate([q(y).reshape(-1), q(box(u)).reshape(-1), q(box(v)).reshape(-1)])


_SWS = None


def swscale():
    """The libswscale that happens to be bundled with the image's OpenCV wheel (9.1.100), or None.  NOT the
    reference's pinned dependency (none is pinned, CMakeLists.txt:72-74): informational distance checks only."""
    global _SWS
    if _SWS is None:
        import glob
        import sysconfig
        _SWS = False
        for d in glob.glob(os.path.join(sysconfig.get_paths()["purelib"], "opencv_python*.libs")):
            pending = sorted(glob.glob(os.path.join(d, "*.so*")))
            for _ in range(6):                       # the wheel's private libraries depend on each other
                nxt = []
                for p in pending:
                    try:
                        C.CDLL(p, mode=C.RTLD_GLOBAL)
                    except OSError:
                        nxt.append(p)
                pending = nxt
            cand = glob.glob(os.path.join(d, "libswscale-*.so*"))
            if cand and not pending:
                L = C.CDLL(cand[0])
                L.sws_getContext.restype = C.c_void_p
                L.sws_getContext.argtypes = [C.c_int] * 7 + [C.c_void_p] * 3
                L.sws_scale.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int, C.c_int,
                                        C.POINTER(C.c_void_p), C.POINTER(C.c_int)]
                L.sws_freeContext.argtypes = [C.c_void_p]
                _SWS = L
                break
    return _SWS or None


def sws_scale_np(planes, strides, iw, ih, src_fmt, ow, oh):
    """sws_getContext(src_fmt -> AV_PIX_FMT_RGBA, SWS_BILINEAR) + sws_scale, as the reference calls it
    (src/image-scaler.cc:50-66, src/video-source.cc:74-77,352-354).  src_fmt: 0 = YUV420P, 23 = NV12, 26 = RGBA."""
    L = swscale()
    ctx = L.sws_getContext(iw, ih, src_fmt, ow, oh, 26, 2, None, None, None)
    assert ctx
    out = np.zeros((oh + 1, ow, 4), np.uint8)          # Framebuffer allocates one spare row for sws overruns (src/framebuffer.cc:62)
    planes = [np.ascontiguousarray(p) for p in planes]
    src = (C.c_void_p * 4)(*([p.ctypes.data for p in planes] + [None] * (4 - len(planes))))
    sst = (C.c_int * 4)(*(list(strides) + [0] * (4 - len(strides))))
    dst = (C.c_void_p * 4)(out.ctypes.data, None, None, None)
    dstr = (C.c_int * 4)(ow * 4, 0, 0, 0)
    L.sws_scale(ctx, src, sst, 0, ih, dst, dstr)
    L.sws_freeContext(ctx)
    return out[:oh].copy()
