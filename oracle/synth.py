"""Seeded synthetic inputs shared by oracle/make_golden.py and tests/ (test infrastructure)."""
import numpy as np


def rand_frame(seed, h, w, c=3):
    return np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)


def smooth_frame(seed, h, w):
    """Config-1 style content (SURVEY 8d): gradient + inverted 16x16 block + gaussian noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)),
                     ((xx + yy) * 255 // max(w + h - 2, 1))], -1).astype(np.float32)
    bx, by = (seed * 7) % max(w - 16, 1), (seed * 3) % max(h - 16, 1)
    base[by:by + 16, bx:bx + 16] = 255 - base[by:by + 16, bx:bx + 16]
    base += rng.normal(0, 8, base.shape)
    return np.clip(base, 0, 255).astype(np.uint8)


def frame(seed, h, w, kind):
    return rand_frame(seed, h, w) if kind == 0 else smooth_frame(seed, h, w)


# Sides at which a Resize table changes behaviour: 1 px (both taps clamp), small integer factors, powers of two and
# their neighbours, the 224 model input, video heights and widths.
RESIZE_SIDES = (1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 31, 33, 63, 64, 65, 100, 223, 224, 225, 479, 480, 1079, 1080, 1920)


def resize_geometries(seed, n, sides=RESIZE_SIDES):
    """n seeded (src_w, src_h, dst_w, dst_h), every side drawn from `sides`.  Every 10th geometry is an exact 2x
    downscale on both axes (the INTER_AREA re-route) and every 10th + 5 on the width only (which stays linear)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        sw, sh, dw, dh = (int(x) for x in rng.choice(sides, 4))
        if i % 10 == 0:
            dw, dh = (int(x) for x in rng.choice([s for s in sides if 2 * s <= max(sides)], 2))
            sw, sh = 2 * dw, 2 * dh
        elif i % 10 == 5:
            dw = int(rng.choice([s for s in sides if 2 * s <= max(sides)]))
            sw = 2 * dw
            if sh == 2 * dh:
                dh = sh
        out.append((sw, sh, dw, dh))
    return out


def nv12_surface(seed, h, w, pitch=None):
    pitch = pitch or w
    rng = np.random.default_rng(seed)
    luma = rng.integers(0, 256, (h, pitch), dtype=np.uint8)
    chroma = rng.integers(0, 256, (h // 2, pitch), dtype=np.uint8)
    return luma, chroma


def flow_pair(seed, h, w, kind="shift"):
    """Two RGB frames with a known relation: "shift" = smooth texture translated by a sub-pixel
    amount (well-conditioned flow), "noise" = unrelated noise (ill-conditioned: tests robustness).
    No cv2 here: the texture is a sum of sinusoids, the shift is analytic."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rand_frame(seed, h, w), rand_frame(seed + 1, h, w)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    dx, dy = 1.5, -0.75

    def tex(x, y):
        out = np.zeros((h, w, 3))
        for c in range(3):
            acc = np.zeros((h, w))
            r2 = np.random.default_rng(seed * 10 + c)
            for _ in range(6):
                fx, fy, ph = r2.uniform(0.02, 0.25), r2.uniform(0.02, 0.25), r2.uniform(0, 6.28)
                acc += np.sin(fx * x + fy * y + ph)
            out[..., c] = 127.5 + 20 * acc
        return np.clip(out, 0, 255).astype(np.uint8)

    return tex(xx, yy), tex(xx - dx, yy - dy)


# ---- exhaustive NV12 -> RGB input (oracle/_ref pin) -------------------------------------------
EXH_FRAMES, EXH_W, EXH_H = 64, 512, 2048


def nv12_exhaustive(f):
    """Frame f (0..63) of a 64 x (512 x 2048) set that presents every (Y, Cb, Cr) triple on an EVEN
    luma row (co-sited chroma, image.cu:153-170): chroma row j of frame f carries the constant pair
    (Cb, Cr) = divmod(f * 1024 + j, 256) and the even luma row above it every Y twice.  Odd rows
    exercise the rounded chroma average (:133-151) with a scrambled Y, and each frame's last odd row
    the no-average case (:138)."""
    j = np.arange(EXH_H // 2, dtype=np.int64) + f * (EXH_H // 2)
    chroma = np.empty((EXH_H // 2, EXH_W), np.uint8)
    chroma[:, 0::2] = (j >> 8)[:, None]
    chroma[:, 1::2] = (j & 255)[:, None]
    x = np.arange(EXH_W, dtype=np.int64)
    luma = np.empty((EXH_H, EXH_W), np.uint8)
    luma[0::2] = (x & 255)[None, :]
    luma[1::2] = ((x[None, :] * 5 + j[:, None] * 3) & 255)
    return luma, chroma
