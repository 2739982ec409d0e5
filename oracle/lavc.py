"""FFmpeg's H.264 decoder through ctypes: each access unit -> its Y, Cb and Cr planes -- TEST INFRASTRUCTURE ONLY.

cv2.VideoCapture returns only the luma plane of raw decoder output; this module reads all three, so the encoder's
chroma is held to an independent decoder too.  It uses the libavcodec / libavutil that the opencv-python wheel
bundles next to the cv2 package (opencv_python*.libs) and reads these fields of FFmpeg's public structs:

  AVPacket.data at byte 24
  AVFrame.data[8] at 0, linesize[8] at 64, width at 104, height at 108, format at 116

Those are the offsets of FFmpeg 8 (libavcodec 62, libavutil 60).  Every picture is checked for format YUV420P, the
display size the SPS gives and one picture per access unit, so a changed struct layout fails loudly instead of
comparing garbage.
"""
import ctypes
import glob
import os

import numpy as np

AV_CODEC_ID_H264 = 27
AV_PIX_FMT_YUV420P = 0
_EAGAIN = -11
_PKT_DATA = 24
_FRAME_LINESIZE, _FRAME_WIDTH, _FRAME_HEIGHT, _FRAME_FORMAT = 64, 104, 108, 116

_LIBS = None


class Unavailable(RuntimeError):
    """no libavcodec is bundled with cv2 here"""


def _find(libdirs, stem):
    for d in libdirs:
        hits = sorted(glob.glob(os.path.join(d, f"{stem}-*.so*")) + glob.glob(os.path.join(d, f"{stem}.so*")))
        if hits:
            return hits[0]
    return None


def libs():
    """(libavcodec, libavutil) as ctypes libraries; raises Unavailable when the cv2 wheel bundles none."""
    global _LIBS
    if _LIBS is None:
        try:
            import cv2
        except ImportError as e:
            raise Unavailable(f"cv2 is not importable: {e}")
        site = os.path.dirname(os.path.dirname(os.path.abspath(cv2.__file__)))
        dirs = sorted(glob.glob(os.path.join(site, "opencv_python*.libs")))
        avutil, avcodec = _find(dirs, "libavutil"), _find(dirs, "libavcodec")
        if not avutil or not avcodec:
            raise Unavailable(f"no libavcodec / libavutil bundled with cv2 (looked in {dirs or site})")
        u = ctypes.CDLL(avutil, mode=ctypes.RTLD_GLOBAL)
        c = ctypes.CDLL(avcodec)
        vp = ctypes.c_void_p
        for name, res, args in (("avcodec_find_decoder", vp, [ctypes.c_int]),
                                ("avcodec_alloc_context3", vp, [vp]),
                                ("avcodec_open2", ctypes.c_int, [vp, vp, vp]),
                                ("avcodec_free_context", None, [vp]),
                                ("av_packet_alloc", vp, []),
                                ("av_packet_free", None, [vp]),
                                ("av_packet_unref", None, [vp]),
                                ("av_new_packet", ctypes.c_int, [vp, ctypes.c_int]),
                                ("avcodec_send_packet", ctypes.c_int, [vp, vp]),
                                ("avcodec_receive_frame", ctypes.c_int, [vp, vp])):
            f = getattr(c, name)
            f.restype, f.argtypes = res, args
        for name, res, args in (("av_frame_alloc", vp, []), ("av_frame_free", None, [vp]),
                                ("av_frame_unref", None, [vp])):
            f = getattr(u, name)
            f.restype, f.argtypes = res, args
        _LIBS = (c, u)
    return _LIBS


def _field(ptr, off, ctype):
    return ctype.from_address(ptr + off).value


def _planes(frame):
    w, h = _field(frame, _FRAME_WIDTH, ctypes.c_int), _field(frame, _FRAME_HEIGHT, ctypes.c_int)
    fmt = _field(frame, _FRAME_FORMAT, ctypes.c_int)
    if fmt != AV_PIX_FMT_YUV420P:
        raise RuntimeError(f"FFmpeg returned pixel format {fmt}, not YUV420P ({AV_PIX_FMT_YUV420P})")
    out = []
    for p, (pw, ph) in enumerate(((w, h), ((w + 1) // 2, (h + 1) // 2), ((w + 1) // 2, (h + 1) // 2))):
        data = _field(frame, 8 * p, ctypes.c_void_p)
        ls = _field(frame, _FRAME_LINESIZE + 4 * p, ctypes.c_int)
        if not data or ls < pw:
            raise RuntimeError(f"FFmpeg plane {p}: data {data}, linesize {ls} for width {pw}")
        buf = (ctypes.c_uint8 * (ls * (ph - 1) + pw)).from_address(data)
        a = np.frombuffer(buf, np.uint8)
        out.append(np.lib.stride_tricks.as_strided(a, (ph, pw), (ls, 1)).copy())
    return (w, h), tuple(out)


def decode(access_units, size=None):
    """Annex-B access units of one stream, one packet each -> [(Y, Cb, Cr) uint8 planes] in output order.
    size: the (width, height) every picture must have (the SPS's cropped display size)."""
    c, u = libs()
    codec = c.avcodec_find_decoder(AV_CODEC_ID_H264)
    if not codec:
        raise Unavailable("the bundled libavcodec has no H.264 decoder")
    ctx = ctypes.c_void_p(c.avcodec_alloc_context3(codec))
    pkt = ctypes.c_void_p(c.av_packet_alloc())
    frame = ctypes.c_void_p(u.av_frame_alloc())
    out = []
    try:
        if not ctx or not pkt or not frame or c.avcodec_open2(ctx, codec, None) < 0:
            raise RuntimeError("could not open FFmpeg's H.264 decoder")
        for i, au in enumerate(access_units):
            if c.av_new_packet(pkt, len(au)) < 0:
                raise MemoryError(len(au))
            ctypes.memmove(_field(pkt.value, _PKT_DATA, ctypes.c_void_p), bytes(au), len(au))
            rc = c.avcodec_send_packet(ctx, pkt)
            c.av_packet_unref(pkt)
            if rc < 0:
                raise RuntimeError(f"avcodec_send_packet failed on access unit {i}: {rc}")
            got = 0
            while (rc := c.avcodec_receive_frame(ctx, frame)) == 0:
                wh, planes = _planes(frame.value)
                size_ok = size is None or wh == tuple(size)
                u.av_frame_unref(frame)
                if not size_ok:
                    raise RuntimeError(f"access unit {i} decoded to {wh[0]}x{wh[1]}, not {size[0]}x{size[1]}")
                out.append(planes)
                got += 1
            if rc != _EAGAIN:
                raise RuntimeError(f"avcodec_receive_frame failed after access unit {i}: {rc}")
            if got != 1:
                raise RuntimeError(f"access unit {i} gave {got} pictures, not 1")
        if c.avcodec_send_packet(ctx, None) < 0:  # flush: nothing may be left behind
            raise RuntimeError("avcodec_send_packet(NULL) failed")
        if c.avcodec_receive_frame(ctx, frame) == 0:
            u.av_frame_unref(frame)
            raise RuntimeError("the decoder held back a picture")
    finally:
        u.av_frame_free(ctypes.byref(frame))
        c.av_packet_free(ctypes.byref(pkt))
        c.avcodec_free_context(ctypes.byref(ctx))
    return out
