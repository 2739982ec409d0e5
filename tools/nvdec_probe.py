#!/usr/bin/env python
"""Probe a GPU for NVDEC: is libnvcuvid there, and what does cuvidGetDecoderCaps say for
H.264 4:2:0 8-bit?  (SURVEY.md Appendix B: 'call it first on the GPU'.)  Prints one JSON line."""
import ctypes
import glob
import json
import sys


class CUVIDDECODECAPS(ctypes.Structure):
    _fields_ = [("eCodecType", ctypes.c_int), ("eChromaFormat", ctypes.c_int),
                ("nBitDepthMinus8", ctypes.c_uint), ("reserved1", ctypes.c_uint * 3),
                ("bIsSupported", ctypes.c_ubyte), ("nNumNVDECs", ctypes.c_ubyte),
                ("nOutputFormatMask", ctypes.c_ushort), ("nMaxWidth", ctypes.c_uint),
                ("nMaxHeight", ctypes.c_uint), ("nMaxMBCount", ctypes.c_uint),
                ("nMinWidth", ctypes.c_ushort), ("nMinHeight", ctypes.c_ushort),
                ("bIsHistogramSupported", ctypes.c_ubyte), ("nCounterBitDepth", ctypes.c_ubyte),
                ("nMaxHistogramBins", ctypes.c_ushort), ("reserved3", ctypes.c_uint * 10)]


def main():
    out = {"libnvcuvid": None, "candidates": sorted(glob.glob("/usr/lib/x86_64-linux-gnu/libnvcuvid*") +
                                                    glob.glob("/usr/lib64/libnvcuvid*") +
                                                    glob.glob("/usr/local/nvidia/lib64/libnvcuvid*")),
           "nvenc": sorted(glob.glob("/usr/lib/x86_64-linux-gnu/libnvidia-encode*"))}
    try:
        cuda = ctypes.CDLL("libcuda.so.1")
    except OSError as e:
        out["error"] = f"libcuda: {e}"
        print(json.dumps(out))
        return 0
    lib = None
    for name in ["libnvcuvid.so.1", "libnvcuvid.so"] + out["candidates"]:
        try:
            lib = ctypes.CDLL(name)
            out["libnvcuvid"] = name
            break
        except OSError as e:
            out.setdefault("dlopen_errors", []).append(str(e))
    if lib is None:
        print(json.dumps(out))
        return 0
    assert cuda.cuInit(0) == 0
    dev = ctypes.c_int()
    assert cuda.cuDeviceGet(ctypes.byref(dev), 0) == 0
    ctx = ctypes.c_void_p()
    assert cuda.cuDevicePrimaryCtxRetain(ctypes.byref(ctx), dev) == 0
    assert cuda.cuCtxPushCurrent_v2(ctx) == 0
    caps_out = {}
    for codec_name, codec in [("h264", 4), ("hevc", 8), ("jpeg", 5), ("av1", 11), ("vp9", 10)]:
        caps = CUVIDDECODECAPS()
        caps.eCodecType = codec
        caps.eChromaFormat = 1
        caps.nBitDepthMinus8 = 0
        rc = lib.cuvidGetDecoderCaps(ctypes.byref(caps))
        caps_out[codec_name] = {"rc": rc, "supported": int(caps.bIsSupported), "n_nvdec": int(caps.nNumNVDECs),
                                "max_w": caps.nMaxWidth, "max_h": caps.nMaxHeight, "max_mb": caps.nMaxMBCount,
                                "min_w": caps.nMinWidth, "min_h": caps.nMinHeight,
                                "fmt_mask": caps.nOutputFormatMask}
    out["caps"] = caps_out
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
