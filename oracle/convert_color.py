"""cv::cvtColor on 8-bit frames restated in integer numpy -- the ConvertColor op's oracle (test infrastructure).

scannertools' ConvertColor is cv::cvtColor with the named code.  For CV_8U input OpenCV's conversions of the
codes below are integer fixed point, so they can be written down exactly; tests/test_convert_color_cpu.py holds
every formula to live cv2.cvtColor and to recorded hashes of its output on all 2^24 RGB triples.
Channels are named for RGB input; a BGR code reads the first channel as blue.
"""
import numpy as np

# name -> (input channels, output channels); the order is the code numbering of include/scn_kernels.h
CODES = {
    "COLOR_RGB2GRAY": (3, 1), "COLOR_BGR2GRAY": (3, 1),
    "COLOR_RGB2YCrCb": (3, 3), "COLOR_BGR2YCrCb": (3, 3),
    "COLOR_RGB2HSV": (3, 3), "COLOR_BGR2HSV": (3, 3),
    "COLOR_RGB2HSV_FULL": (3, 3), "COLOR_BGR2HSV_FULL": (3, 3),
    "COLOR_RGB2BGR": (3, 3), "COLOR_BGR2RGB": (3, 3),
    "COLOR_GRAY2RGB": (1, 3), "COLOR_GRAY2BGR": (1, 3),
}

HSV_SHIFT = 12


def _d(x, n):
    """D(x, n) = (x + 2^(n-1)) >> n, OpenCV's CV_DESCALE (arithmetic shift)."""
    return (x + (1 << (n - 1))) >> n


def hsv_tables(hrange):
    """RGB2HSV_b's division tables: sdiv[i] = round((255 << 12) / i), hdiv[i] = round((hrange << 12) / (6 i)),
    both 0 at i = 0.  (No quotient here is a tie, so the rounding mode does not matter.)"""
    i = np.arange(1, 256, dtype=np.float64)
    sdiv = np.zeros(256, np.int64)
    hdiv = np.zeros(256, np.int64)
    sdiv[1:] = np.rint((255 << HSV_SHIFT) / i)
    hdiv[1:] = np.rint((hrange << HSV_SHIFT) / (6.0 * i))
    return sdiv, hdiv


def _rgb(frame, bgr):
    f = frame.astype(np.int64)
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    return (b, g, r) if bgr else (r, g, b)


def gray(r, g, b):
    return _d(9798 * r + 19235 * g + 3735 * b, 15)


def ycrcb(r, g, b):
    y = _d(4899 * r + 9617 * g + 1868 * b, 14)
    cr = np.clip(_d((r - y) * 11682 + (128 << 14), 14), 0, 255)
    cb = np.clip(_d((b - y) * 9241 + (128 << 14), 14), 0, 255)
    return y, cr, cb


def hsv(r, g, b, hrange):
    sdiv, hdiv = hsv_tables(hrange)
    v = np.maximum(np.maximum(r, g), b)
    diff = v - np.minimum(np.minimum(r, g), b)
    s = _d(diff * sdiv[v], HSV_SHIFT)
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = _d(h * hdiv[diff], HSV_SHIFT)
    h = np.where(h < 0, h + hrange, h) & 0xFF
    return h, s, v


def convert_color(frame, code):
    """frame: (..., C) uint8 with C the code's input channel count -> (..., C_out) uint8."""
    if code not in CODES:
        raise ValueError(f"unsupported conversion {code!r}")
    cin, _ = CODES[code]
    frame = np.asarray(frame, np.uint8)
    assert frame.shape[-1] == cin, (frame.shape, code)
    if cin == 1:
        return np.repeat(frame, 3, axis=-1)
    bgr = code.startswith("COLOR_BGR")
    if code in ("COLOR_RGB2BGR", "COLOR_BGR2RGB"):
        return np.ascontiguousarray(frame[..., ::-1])
    rgb = _rgb(frame, bgr)
    if code.endswith("GRAY"):
        out = [gray(*rgb)]
    elif code.endswith("YCrCb"):
        out = ycrcb(*rgb)
    else:
        out = hsv(*rgb, 256 if code.endswith("_FULL") else 180)
    return np.stack(out, -1).astype(np.uint8)


def all_triples():
    """Every RGB triple once: a 4096 x 4096 x 3 image, pixel (y, x) = (y >> 4, ((y & 15) << 4) | (x >> 8), x & 255)."""
    k = np.arange(1 << 24, dtype=np.uint32)
    img = np.empty((1 << 24, 3), np.uint8)
    img[:, 0] = k >> 16
    img[:, 1] = (k >> 8) & 255
    img[:, 2] = k & 255
    return img.reshape(4096, 4096, 3)
