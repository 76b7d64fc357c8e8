"""Float64 restatement of the fused YUV -> RGBA scaler (timg_b200/csrc/bilinear.cu, yuv_rgba_kernel) for every
decoder format of include/b200timg.h, the matching input builder, and libav pixel-format ids looked up by name.

PARITY UNPINNED, as for 4:2:0 (oracle.yuv420_to_rgba_np): libswscale is not part of the reference tree.  The rules
restated here are what the libswscale 9.1 bundled with the image's OpenCV wheel does with SWS_BILINEAR:
  * 4:4:4 sources (8- and 10-bit): chroma is interpolated at the full output width (libswscale switches on full
    chroma interpolation for sources without chroma subsampling);
  * every other format: chroma at half the output width, two output pixels per chroma sample, the chroma plane's own
    width and height feeding the triangle tables;
  * unscaled (ow, oh) == (iw, ih): only 8-bit 4:2:0 (I420 / NV12) replicates chroma rows, as libswscale's unscaled
    yuv2rgb converters do; the other formats go through the triangle filter at scale 1 as well;
  * 10-bit samples are divided by 4 into the 8-bit domain, then the 8-bit BT.601 coefficients apply.
"""
import ctypes as C
import glob
import os

import numpy as np

import oracle
from oracle import _tri_axis

I420, NV12, I422, I444, I440, I420_10, I422_10, I444_10, P010 = 2, 3, 4, 5, 6, 7, 8, 9, 10
FULL_RANGE = 0x10
# format -> (libav name, chroma shift x, chroma shift y, bytes per sample, interleaved chroma)
LAYOUT = {I420: ("yuv420p", 1, 1, 1, False), NV12: ("nv12", 1, 1, 1, True), I422: ("yuv422p", 1, 0, 1, False),
          I444: ("yuv444p", 0, 0, 1, False), I440: ("yuv440p", 0, 1, 1, False),
          I420_10: ("yuv420p10le", 1, 1, 2, False), I422_10: ("yuv422p10le", 1, 0, 2, False),
          I444_10: ("yuv444p10le", 0, 0, 2, False), P010: ("p010le", 1, 1, 2, True)}
NEW_FORMATS = (I422, I444, I440, I420_10, I422_10, I444_10, P010)
NAMES = {I420: "I420", NV12: "NV12", I422: "I422", I444: "I444", I440: "I440", I420_10: "I420_10", I422_10: "I422_10",
         I444_10: "I444_10", P010: "P010"}


def frame_samples(fmt, iw, ih):
    """Samples (not bytes) of one frame."""
    _, sx, sy, _, _ = LAYOUT[fmt & 0xF]
    return iw * ih + 2 * (iw >> sx) * (ih >> sy)


def planes_np(buf, fmt, iw, ih):
    """(Y, U, V) sample-value planes of one tightly packed frame; 10-bit formats give their 10 value bits."""
    _, sx, sy, bps, semi = LAYOUT[fmt & 0xF]
    buf = np.ascontiguousarray(buf).reshape(-1)
    s = buf.view(np.uint16) if bps == 2 and buf.dtype != np.uint16 else buf
    if bps == 2:
        s = (s >> 6) if fmt & 0xF == P010 else (s & 0x3FF)
    cw, ch = iw >> sx, ih >> sy
    Y = s[: iw * ih].reshape(ih, iw)
    if semi:
        uv = s[iw * ih: iw * ih + 2 * cw * ch].reshape(ch, cw, 2)
        return Y, uv[..., 0], uv[..., 1]
    return Y, s[iw * ih: iw * ih + cw * ch].reshape(ch, cw), s[iw * ih + cw * ch: iw * ih + 2 * cw * ch].reshape(ch, cw)


def yuv_to_rgba_np(planes, fmt, ow, oh, full_range=False):
    """Float64 statement of yuv_rgba_kernel<fmt>: planes = (Y, U, V) sample values (planes_np), -> RGBA [oh, ow, 4]."""
    f = fmt & 0xF
    _, sx, sy, bps, _ = LAYOUT[f]
    Y, U, V = (np.asarray(p, dtype=np.float64) for p in planes)
    if bps == 2:                        # 10-bit -> 8-bit domain
        Y, U, V = Y / 4.0, U / 4.0, V / 4.0
    ih, iw = Y.shape
    ch, cw = U.shape
    full = sx == 0 and sy == 0
    cow = ow if full else (ow + 1) // 2
    y = _tri_axis(ih, oh) @ Y @ _tri_axis(iw, ow).T
    Mv = _tri_axis(ch, oh)
    if f in (I420, NV12) and (ow, oh) == (iw, ih):
        Mv = np.zeros((oh, ch))
        Mv[np.arange(oh), np.arange(oh) // 2] = 1.0
    Mh = _tri_axis(cw, cow)
    if full:
        chroma = lambda P: Mv @ P @ Mh.T - 128.0
    else:
        chroma = lambda P: np.repeat(Mv @ P @ Mh.T, 2, 1)[:, :ow] - 128.0
    u, v = chroma(U), chroma(V)
    if full_range:
        r, g, b = y + 1.402 * v, y - 0.344136 * u - 0.714136 * v, y + 1.772 * u
    else:
        yl = 1.164383 * (y - 16.0)
        r, g, b = yl + 1.596027 * v, yl - 0.391762 * u - 0.812968 * v, yl + 2.017232 * u
    out = np.stack([r, g, b, np.full_like(r, 255.0)], -1)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def rgba_to_yuv_np(img, fmt):
    """BT.601 limited-range RGB -> one tightly packed frame of fmt (box-filtered chroma), for building test inputs:
    uint8 for the 8-bit formats, uint16 samples for the 10-bit ones (P010: value in the high 10 bits).  I420 equals
    oracle.rgba_to_i420_np."""
    f = fmt & 0xF
    _, sx, sy, bps, semi = LAYOUT[f]
    img = np.asarray(img, dtype=np.float64)
    r, g, b = img[..., 0], img[..., 1], img[..., 2]
    y = 16 + 0.256788 * r + 0.504129 * g + 0.097906 * b
    u = 128 - 0.148223 * r - 0.290993 * g + 0.439216 * b
    v = 128 + 0.439216 * r - 0.367788 * g - 0.071427 * b
    h, w = y.shape
    bx, by = 1 << sx, 1 << sy
    box = lambda p: p.reshape(h // by, by, w // bx, bx).mean((1, 3))
    if bps == 1:
        q = lambda p: np.clip(np.rint(p), 0, 255).astype(np.uint8)
    else:
        q = lambda p: np.clip(np.rint(p * 4.0), 0, 1023).astype(np.uint16)
    Y, U, V = q(y), q(box(u)), q(box(v))
    if semi:
        out = np.concatenate([Y.reshape(-1), np.stack([U, V], -1).reshape(-1)])
    else:
        out = np.concatenate([Y.reshape(-1), U.reshape(-1), V.reshape(-1)])
    return out << 6 if f == P010 else out


_AVUTIL = None


def av_pix_fmt(name):
    """AVPixelFormat id of a libav pixel-format name through the wheel's av_get_pix_fmt, or None when the wheel's
    libraries are not there (ids differ between libav versions, so they are never hard-coded)."""
    global _AVUTIL
    if _AVUTIL is None:
        _AVUTIL = False
        if oracle.swscale():                     # loads the wheel's libraries, libavutil among them
            import sysconfig
            for d in glob.glob(os.path.join(sysconfig.get_paths()["purelib"], "opencv_python*.libs")):
                cand = glob.glob(os.path.join(d, "libavutil-*.so*"))
                if cand:
                    L = C.CDLL(cand[0])
                    L.av_get_pix_fmt.restype = C.c_int
                    L.av_get_pix_fmt.argtypes = [C.c_char_p]
                    _AVUTIL = L
                    break
    if not _AVUTIL:
        return None
    v = _AVUTIL.av_get_pix_fmt(name.encode())
    return None if v < 0 else v


def sws_yuv_to_rgba(buf, fmt, iw, ih, ow, oh):
    """libswscale (sws_getContext(fmt -> RGBA, SWS_BILINEAR) + sws_scale, as the reference calls it) on one tightly
    packed frame of fmt.  The FULL_RANGE bit selects the yuvj twin for the formats that have one."""
    f = fmt & 0xF
    name, sx, sy, bps, semi = LAYOUT[f]
    if fmt & FULL_RANGE:
        name = {"yuv420p": "yuvj420p", "yuv422p": "yuvj422p", "yuv444p": "yuvj444p", "yuv440p": "yuvj440p"}[name]
    raw = np.ascontiguousarray(buf).reshape(-1).view(np.uint8)
    cw, ch = iw >> sx, ih >> sy
    ny = iw * ih * bps
    if semi:
        planes, strides = [raw[:ny], raw[ny:]], [iw * bps, 2 * cw * bps]
    else:
        nc = cw * ch * bps
        planes, strides = [raw[:ny], raw[ny:ny + nc], raw[ny + nc:ny + 2 * nc]], [iw * bps, cw * bps, cw * bps]
    return oracle.sws_scale_np(planes, strides, iw, ih, av_pix_fmt(name), ow, oh)
