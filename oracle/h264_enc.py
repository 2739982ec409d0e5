"""Integer numpy model of the H.264 encoder behind scn_h264_encode_u8 (scanner_b200/csrc/h264_enc.cu).

The kernel is held to this module byte for byte; this module is held to FFmpeg (tests/test_h264_encode_cpu.py):
the decoder must output exactly the reconstruction computed here.  Clause numbers refer to H.264 (04/2017).

  colour      integer BT.601 studio range, `>>` a floor:
                Y  = ((66 R + 129 G + 25 B + 128) >> 8) + 16
                Cb = ((-38 SR - 74 SG + 112 SB + 512) >> 10) + 128   (SR, SG, SB: sums over each 2x2 block)
                Cr = ((112 SR - 94 SG - 18 SB + 512) >> 10) + 128
              the Y, Cb and Cr planes are padded to the macroblock grid by repeating their last column and row;
              SPS cropping gives the display size
  stream      Baseline (constraint_set0 and 1), level 4.1 or 5.1, POC type 2, VUI with BT.601 colour and
              max_num_reorder_frames 0; CAVLC, one slice per picture, deblocking off; an IDR (with SPS + PPS)
              starts each item and every keyframe_distance pictures, the pictures between are non-IDR I pictures
  macroblock  Intra16x16 only.  Luma mode (V 0, H 1, DC 2, Plane 3) and chroma mode (DC 0, H 1, V 2, Plane 3)
              each minimise the SAD of the residual (Cb + Cr for chroma) among the modes whose neighbours are
              available, ties to the lower mode number
  residual    4x4 core transform; luma DC 4x4 Hadamard (H W H) >> 1, chroma DC 2x2 Hadamard; quantisation
              sign(x) ((|x| MF + f) >> qbits) with qbits = 15 + QP / 6, f = (1 << qbits) / 3, the DC paths with
              qbits + 1 and 2 f; chroma QP from Table 8-15.  Every level is clamped to +-2063, the largest
              magnitude a level_prefix of at most 15 (the Baseline limit) codes at any suffixLength.  Luma AC is
              coded for all 16 blocks or none; chroma cbp is 2 if any chroma AC level is nonzero, else 1 if any
              chroma DC level is, else 0.  Levels that are not coded are zero in the reconstruction.
"""
import re

import numpy as np

from scanner_b200.synth_h264 import _Codes

_EPB = re.compile(b"\x00\x00(?=[\x00-\x03])")
LEVEL_MAX = 2063
MAX_SIDE = 4096
MAX_MBS = 36864

# ---- tables ---------------------------------------------------------------------------------------------------
_MF = np.array([[13107, 5243, 8066], [11916, 4660, 7490], [10082, 4194, 6554], [9362, 3647, 5825],
                [8192, 3355, 5243], [7282, 2893, 4559]], np.int64)
_V = np.array([[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]], np.int64)
_POS = np.array([[0 if (i % 2 == 0 and j % 2 == 0) else 1 if (i % 2 and j % 2) else 2 for j in range(4)]
                 for i in range(4)])
MF = _MF[:, _POS]   # (6, 4, 4)
V = _V[:, _POS]
_QPC = [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
ZIGZAG = np.array([0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15])   # scan index -> raster (row * 4 + col)
_CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
_H4 = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
_H2 = np.array([[1, 1], [1, -1]], np.int64)
# luma4x4BlkIdx -> (column, row) of the 4x4 block in its macroblock (6.4.3)
BLK_XY = [(((b >> 2) & 1) * 2 + (b & 1), ((b >> 3) & 1) * 2 + ((b >> 1) & 1)) for b in range(16)]

# Table 9-5, [nC class][TotalCoeff * 4 + TrailingOnes]: nC 0-1, 2-3, 4-7, 8+ (FLC); then nC = -1
COEFF_TOKEN_LEN = [
    [1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9,
     13, 13, 13, 10, 14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15,
     16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16],
    [2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6,
     11, 11, 11, 7, 12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13,
     13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14],
    [4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4,
     8, 7, 7, 5, 8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10,
     10, 10, 10, 10, 10, 10, 10, 10],
    [6] * 68,
    [2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7],
]
COEFF_TOKEN_BITS = [
    [1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4,
     8, 10, 13, 4, 15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12,
     11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8],
    [3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4,
     11, 14, 13, 4, 15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12,
     7, 11, 6, 8, 9, 8, 10, 1, 7, 6, 5, 4],
    [15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9,
     8, 10, 9, 8, 15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8,
     13, 7, 9, 12, 9, 12, 11, 10, 5, 8, 7, 6, 1, 4, 3, 2],
    [3, 0, 0, 0] + [((tc - 1) << 2) | t1 if t1 <= tc else 0 for tc in range(1, 17) for t1 in range(4)],
    [1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0],
]
# Tables 9-7 / 9-8, [TotalCoeff - 1][total_zeros]
TOTAL_ZEROS_LEN = [
    [1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9], [3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6],
    [4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6], [5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5],
    [4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5], [6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6], [6, 5, 3, 3, 3, 2, 3, 4, 3, 6],
    [6, 4, 5, 3, 2, 2, 3, 3, 6], [6, 6, 4, 2, 2, 3, 2, 5], [5, 5, 3, 2, 2, 2, 4], [4, 4, 3, 3, 1, 3],
    [4, 4, 2, 1, 3], [3, 3, 1, 2], [2, 2, 1], [1, 1]]
TOTAL_ZEROS_BITS = [
    [1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1], [7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0],
    [5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0], [3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0],
    [5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 5, 4, 3, 3, 2, 1, 1, 0],
    [1, 1, 1, 3, 3, 2, 2, 1, 0], [1, 0, 1, 3, 2, 1, 1, 1], [1, 0, 1, 3, 2, 1, 1], [0, 1, 1, 2, 1, 3],
    [0, 1, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1], [0, 1]]
# Table 9-9a (chroma DC 2x2), [TotalCoeff - 1][total_zeros]
CDC_TOTAL_ZEROS_LEN = [[1, 2, 3, 3], [1, 2, 2], [1, 1]]
CDC_TOTAL_ZEROS_BITS = [[1, 1, 1, 0], [1, 1, 0], [1, 0]]
# Table 9-10, [min(zerosLeft, 7) - 1][run_before]
RUN_LEN = [[1, 1], [1, 2, 2], [2, 2, 2, 2], [2, 2, 2, 3, 3], [2, 2, 3, 3, 3, 3], [2, 3, 3, 3, 3, 3, 3],
           [3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
RUN_BITS = [[1, 0], [1, 1, 0], [3, 2, 1, 0], [3, 2, 1, 1, 0], [3, 2, 3, 2, 1, 0], [3, 0, 1, 3, 2, 5, 4],
            [7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1]]


def chroma_qp(qp):
    return qp if qp < 30 else _QPC[qp - 30]


def level_idc(width, height):
    mbs = ((width + 15) // 16) * ((height + 15) // 16)
    return 41 if mbs <= 8192 else 51


# ---- colour ---------------------------------------------------------------------------------------------------
def rgb_to_planes(rgb):
    """(H, W, 3) uint8, H and W even -> padded Y (16 hmb, 16 wmb), Cb, Cr (8 hmb, 8 wmb) as int64."""
    h, w, _ = rgb.shape
    x = rgb.astype(np.int64)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16
    s = x.reshape(h // 2, 2, w // 2, 2, 3).sum((1, 3))
    sr, sg, sb = s[..., 0], s[..., 1], s[..., 2]
    cb = ((-38 * sr - 74 * sg + 112 * sb + 512) >> 10) + 128
    cr = ((112 * sr - 94 * sg - 18 * sb + 512) >> 10) + 128
    wmb, hmb = (w + 15) // 16, (h + 15) // 16
    pad = lambda p, k: np.pad(p, ((0, hmb * k - p.shape[0]), (0, wmb * k - p.shape[1])), mode="edge")
    return pad(y, 16), pad(cb, 8), pad(cr, 8)


# ---- transforms -----------------------------------------------------------------------------------------------
def _fwd4(x):
    return _CF @ x @ _CF.T


def _inv_rows(d, axis):
    d0, d1, d2, d3 = (np.take(d, i, axis=axis) for i in range(4))
    e0, e1, e2, e3 = d0 + d2, d0 - d2, (d1 >> 1) - d3, d1 + (d3 >> 1)
    return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], axis=axis)


def _inv4(d):
    """8.5.12.2: rows (horizontal) first, then columns; (x + 32) >> 6"""
    return (_inv_rows(_inv_rows(d, -1), -2) + 32) >> 6


def _quant(w, mf, qbits, dc=False):
    f = (1 << qbits) // 3
    if dc:
        q = (np.abs(w) * mf + 2 * f) >> (qbits + 1)
    else:
        q = (np.abs(w) * mf + f) >> qbits
    return np.clip(np.sign(w) * q, -LEVEL_MAX, LEVEL_MAX)


# ---- prediction (8.3.3, 8.3.4), vectorised over the k macroblocks of one anti-diagonal --------------------------
def _luma_preds(top, left, corner, has_t, has_l):
    """top, left (k, 16), corner (k,) -> preds (k, 4, 16, 16), valid (k, 4)"""
    k = top.shape[0]
    x = np.arange(16)
    pv = np.broadcast_to(top[:, None, :], (k, 16, 16))
    ph = np.broadcast_to(left[:, :, None], (k, 16, 16))
    st, sl = top.sum(1), left.sum(1)
    dc = np.where(has_t & has_l, (st + sl + 16) >> 5,
                  np.where(has_t, (st + 8) >> 4, np.where(has_l, (sl + 8) >> 4, 128)))
    pd = np.broadcast_to(dc[:, None, None], (k, 16, 16))
    te = np.concatenate([corner[:, None], top], 1)    # te[i + 1] = p[i, -1]
    le = np.concatenate([corner[:, None], left], 1)
    xp = np.arange(8)
    hh = ((xp + 1) * (te[:, 9 + xp] - te[:, 7 - xp])).sum(1)
    vv = ((xp + 1) * (le[:, 9 + xp] - le[:, 7 - xp])).sum(1)
    a = 16 * (left[:, 15] + top[:, 15])
    b, c = (5 * hh + 32) >> 6, (5 * vv + 32) >> 6
    pp = np.clip((a[:, None, None] + b[:, None, None] * (x[None, None, :] - 7) + c[:, None, None] * (x[None, :, None] - 7)
                  + 16) >> 5, 0, 255)
    preds = np.stack([pv, ph, pd, pp], 1)
    valid = np.stack([has_t, has_l, np.ones_like(has_t), has_t & has_l], 1)
    return preds, valid


def _chroma_dc(top, left, has_t, has_l):
    """per 4x4 chroma block (8.3.4.1-3): top, left (k, 8) -> (k, 8, 8)"""
    k = top.shape[0]
    out = np.empty((k, 8, 8), np.int64)
    for yo in (0, 4):
        for xo in (0, 4):
            st, sl = top[:, xo:xo + 4].sum(1), left[:, yo:yo + 4].sum(1)
            both = (st + sl + 4) >> 3
            t_only, l_only = (st + 2) >> 2, (sl + 2) >> 2
            if (xo, yo) == (4, 0):
                v = np.where(has_t, t_only, np.where(has_l, l_only, 128))
            elif (xo, yo) == (0, 4):
                v = np.where(has_l, l_only, np.where(has_t, t_only, 128))
            else:
                v = np.where(has_t & has_l, both, np.where(has_l, l_only, np.where(has_t, t_only, 128)))
            out[:, yo:yo + 4, xo:xo + 4] = v[:, None, None]
    return out


def _chroma_preds(top, left, corner, has_t, has_l):
    """top, left (k, 8), corner (k,) of one component -> (k, 4, 8, 8) in mode order DC, H, V, Plane"""
    k = top.shape[0]
    x = np.arange(8)
    te = np.concatenate([corner[:, None], top], 1)
    le = np.concatenate([corner[:, None], left], 1)
    xp = np.arange(4)
    hh = ((xp + 1) * (te[:, 5 + xp] - te[:, 3 - xp])).sum(1)
    vv = ((xp + 1) * (le[:, 5 + xp] - le[:, 3 - xp])).sum(1)
    a = 16 * (left[:, 7] + top[:, 7])
    b, c = (34 * hh + 32) >> 6, (34 * vv + 32) >> 6
    pp = np.clip((a[:, None, None] + b[:, None, None] * (x[None, None, :] - 3) + c[:, None, None] * (x[None, :, None] - 3)
                  + 16) >> 5, 0, 255)
    return np.stack([_chroma_dc(top, left, has_t, has_l), np.broadcast_to(left[:, :, None], (k, 8, 8)),
                     np.broadcast_to(top[:, None, :], (k, 8, 8)), pp], 1)


def _blocks(p, n):
    """(k, 4n, 4n) -> (k, n, n, 4, 4) [block row, block column, row, column]"""
    k = p.shape[0]
    return p.reshape(k, n, 4, n, 4).transpose(0, 1, 3, 2, 4)


def _unblocks(b):
    k, n = b.shape[0], b.shape[1]
    return b.transpose(0, 1, 3, 2, 4).reshape(k, 4 * n, 4 * n)


# ---- one picture: the reconstruction wavefront ------------------------------------------------------------------
def _reconstruct(planes, qp, st):
    """-> reconstructed padded planes and per-macroblock coding decisions (arrays indexed [my, mx, ...])."""
    y_src, cb_src, cr_src = planes
    hmb, wmb = y_src.shape[0] // 16, y_src.shape[1] // 16
    rec = [np.zeros_like(y_src), np.zeros_like(cb_src), np.zeros_like(cr_src)]
    qpc = chroma_qp(qp)
    m = dict(lmode=np.zeros((hmb, wmb), np.int64), cmode=np.zeros((hmb, wmb), np.int64),
             cbpl=np.zeros((hmb, wmb), np.int64), cbpc=np.zeros((hmb, wmb), np.int64),
             ldc=np.zeros((hmb, wmb, 4, 4), np.int64), lac=np.zeros((hmb, wmb, 4, 4, 4, 4), np.int64),
             cdc=np.zeros((hmb, wmb, 2, 2, 2), np.int64), cac=np.zeros((hmb, wmb, 2, 2, 2, 4, 4), np.int64))
    for d in range(wmb + hmb - 1):
        my = np.arange(max(0, d - wmb + 1), min(hmb, d + 1))
        mx = d - my
        k = len(my)
        has_t, has_l = my > 0, mx > 0
        # luma neighbours from the reconstruction (zeros where unavailable; those modes are excluded)
        ys, xs = 16 * my, 16 * mx
        rows = np.arange(16)
        top = np.where(has_t[:, None], rec[0][np.maximum(ys - 1, 0)[:, None], xs[:, None] + rows], 0)
        left = np.where(has_l[:, None], rec[0][ys[:, None] + rows, np.maximum(xs - 1, 0)[:, None]], 0)
        corner = np.where(has_t & has_l, rec[0][np.maximum(ys - 1, 0), np.maximum(xs - 1, 0)], 0)
        src = y_src[ys[:, None, None] + rows[None, :, None], xs[:, None, None] + rows[None, None, :]]
        preds, valid = _luma_preds(top, left, corner, has_t, has_l)
        sad = np.abs(src[:, None] - preds).sum((2, 3))
        sad = np.where(valid, sad, np.iinfo(np.int64).max)
        lmode = sad.argmin(1)
        pred = preds[np.arange(k), lmode]
        w = _fwd4(_blocks(src - pred, 4))                           # (k, 4, 4, 4, 4)
        qb = 15 + qp // 6
        ac = _quant(w, MF[qp % 6], qb)
        ac[..., 0, 0] = 0
        wdc = w[..., 0, 0]                                          # (k, 4, 4) [block row, block column]
        ydc = (_H4 @ wdc @ _H4) >> 1
        ldc = _quant(ydc, MF[qp % 6, 0, 0], qb, dc=True)
        cbpl = np.where((ac != 0).any((1, 2, 3, 4)), 15, 0)
        ac = ac * (cbpl > 0)[:, None, None, None, None]
        f = _H4 @ ldc @ _H4
        ls = 16 * V[qp % 6, 0, 0]
        if qp >= 36:
            dcy = (f * ls) << (qp // 6 - 6)
        else:
            dcy = (f * ls + (1 << (5 - qp // 6))) >> (6 - qp // 6)
        dq = (ac * V[qp % 6]) << (qp // 6)
        dq[..., 0, 0] = dcy
        rec_y = np.clip(pred + _unblocks(_inv4(dq)), 0, 255)
        rec[0][ys[:, None, None] + rows[None, :, None], xs[:, None, None] + rows[None, None, :]] = rec_y
        # chroma
        ys, xs = 8 * my, 8 * mx
        r8 = np.arange(8)
        cpreds, csrc = [], []
        for c in (1, 2):
            top = np.where(has_t[:, None], rec[c][np.maximum(ys - 1, 0)[:, None], xs[:, None] + r8], 0)
            left = np.where(has_l[:, None], rec[c][ys[:, None] + r8, np.maximum(xs - 1, 0)[:, None]], 0)
            corner = np.where(has_t & has_l, rec[c][np.maximum(ys - 1, 0), np.maximum(xs - 1, 0)], 0)
            cpreds.append(_chroma_preds(top, left, corner, has_t, has_l))
            csrc.append(planes[c][ys[:, None, None] + r8[None, :, None], xs[:, None, None] + r8[None, None, :]])
        cpreds, csrc = np.stack(cpreds, 1), np.stack(csrc, 1)       # (k, 2, 4, 8, 8), (k, 2, 8, 8)
        cvalid = np.stack([np.ones_like(has_t), has_l, has_t, has_t & has_l], 1)
        csad = np.abs(csrc[:, :, None] - cpreds).sum((1, 3, 4))
        csad = np.where(cvalid, csad, np.iinfo(np.int64).max)
        cmode = csad.argmin(1)
        cpred = cpreds[np.arange(k), :, cmode]                      # (k, 2, 8, 8)
        qbc = 15 + qpc // 6
        w = _fwd4(_blocks((csrc - cpred).reshape(k * 2, 8, 8), 2)).reshape(k, 2, 2, 2, 4, 4)
        cac = _quant(w, MF[qpc % 6], qbc)
        cac[..., 0, 0] = 0
        cdc = _quant(_H2 @ w[..., 0, 0] @ _H2, MF[qpc % 6, 0, 0], qbc, dc=True)   # (k, 2, 2, 2)
        cbpc = np.where((cac != 0).any((1, 2, 3, 4, 5)), 2, np.where((cdc != 0).any((1, 2, 3)), 1, 0))
        cac = cac * (cbpc == 2)[:, None, None, None, None, None]
        cdc = cdc * (cbpc > 0)[:, None, None, None]
        dcc = ((_H2 @ cdc @ _H2) * 16 * V[qpc % 6, 0, 0] << (qpc // 6)) >> 5
        dq = (cac * V[qpc % 6]) << (qpc // 6)
        dq[..., 0, 0] = dcc
        res = _unblocks(_inv4(dq).reshape(k * 2, 2, 2, 4, 4)).reshape(k, 2, 8, 8)
        rec_c = np.clip(cpred + res, 0, 255)
        for c in (1, 2):
            rec[c][ys[:, None, None] + r8[None, :, None], xs[:, None, None] + r8[None, None, :]] = rec_c[:, c - 1]
        for key, v in (("lmode", lmode), ("cmode", cmode), ("cbpl", cbpl), ("cbpc", cbpc), ("ldc", ldc),
                       ("lac", ac), ("cdc", cdc), ("cac", cac)):
            m[key][my, mx] = v
    for i in range(4):
        st["luma_mode"][i] += int((m["lmode"] == i).sum())
        st["chroma_mode"][i] += int((m["cmode"] == i).sum())
    return rec, m


# ---- CAVLC (9.2) ----------------------------------------------------------------------------------------------
def _nc_class(nc):
    return 4 if nc < 0 else 0 if nc < 2 else 1 if nc < 4 else 2 if nc < 8 else 3


def _cavlc(b, coef, nc, max_num, st):
    """residual_block_cavlc of `coef` (scan order, length max_num) -> TotalCoeff"""
    nz = [i for i, v in enumerate(coef) if v]
    tc = len(nz)
    t1 = 0
    for i in reversed(nz):
        if abs(coef[i]) == 1 and t1 < 3:
            t1 += 1
        else:
            break
    cls = _nc_class(nc)
    st["nc_class"][cls] += 1
    b.u(COEFF_TOKEN_LEN[cls][tc * 4 + t1], COEFF_TOKEN_BITS[cls][tc * 4 + t1])
    if tc == 0:
        return 0
    if tc == 16:
        st["total_coeff_16"] += 1
    sl = 1 if tc > 10 and t1 < 3 else 0
    for i, i_nz in enumerate(reversed(nz)):
        lv = int(coef[i_nz])
        if i < t1:
            b.u(1, 1 if lv < 0 else 0)
            continue
        code = 2 * lv - 2 if lv > 0 else -2 * lv - 1
        if i == t1 and t1 < 3:
            code -= 2
        if sl == 0 and code < 14:
            b.u(code + 1, 1)
        elif sl == 0 and code < 30:
            b.u(15, 1)
            b.u(4, code - 14)
            st["level_prefix_14"] += 1
        elif sl > 0 and (code >> sl) < 15:
            b.u((code >> sl) + 1, 1)
            b.u(sl, code & ((1 << sl) - 1))
        else:
            esc = code - (30 if sl == 0 else 15 << sl)
            assert 0 <= esc < 4096, (lv, sl)
            b.u(16, 1)
            b.u(12, esc)
            st["level_prefix_15"] += 1
        if sl == 0:
            sl = 1
        if abs(lv) > (3 << (sl - 1)) and sl < 6:
            sl += 1
    if tc < max_num:
        tz = nz[-1] + 1 - tc
        if max_num == 4:
            b.u(CDC_TOTAL_ZEROS_LEN[tc - 1][tz], CDC_TOTAL_ZEROS_BITS[tc - 1][tz])
        else:
            b.u(TOTAL_ZEROS_LEN[tc - 1][tz], TOTAL_ZEROS_BITS[tc - 1][tz])
        zl = tz
        for j in range(tc - 1, 0, -1):
            if zl == 0:
                break
            run = nz[j] - nz[j - 1] - 1
            r = min(zl, 7) - 1
            b.u(RUN_LEN[r][run], RUN_BITS[r][run])
            zl -= run
    return tc


def _nc(tot, gy, gx):
    a = tot[gy, gx - 1] if gx > 0 else None
    t = tot[gy - 1, gx] if gy > 0 else None
    if a is not None and t is not None:
        return (int(a) + int(t) + 1) >> 1
    return int(a) if a is not None else int(t) if t is not None else 0


def _slice_data(b, m, st):
    hmb, wmb = m["lmode"].shape
    ltot = np.zeros((4 * hmb, 4 * wmb), np.int64)
    ctot = np.zeros((2, 2 * hmb, 2 * wmb), np.int64)
    zz = ZIGZAG
    for my in range(hmb):
        for mx in range(wmb):
            cbpl, cbpc = int(m["cbpl"][my, mx]), int(m["cbpc"][my, mx])
            b.ue(1 + int(m["lmode"][my, mx]) + 4 * cbpc + (12 if cbpl else 0))   # mb_type I_16x16_*
            b.ue(int(m["cmode"][my, mx]))                                       # intra_chroma_pred_mode
            b.se(0)                                                             # mb_qp_delta
            _cavlc(b, m["ldc"][my, mx].ravel()[zz], _nc(ltot, 4 * my, 4 * mx), 16, st)
            if cbpl:
                for blk in range(16):
                    bx, by = BLK_XY[blk]
                    gy, gx = 4 * my + by, 4 * mx + bx
                    ltot[gy, gx] = _cavlc(b, m["lac"][my, mx, by, bx].ravel()[zz][1:], _nc(ltot, gy, gx), 15, st)
            if cbpc:
                for c in range(2):
                    _cavlc(b, m["cdc"][my, mx, c].ravel(), -1, 4, st)
            if cbpc == 2:
                for c in range(2):
                    for blk in range(4):
                        bx, by = blk & 1, blk >> 1
                        gy, gx = 2 * my + by, 2 * mx + bx
                        ctot[c, gy, gx] = _cavlc(b, m["cac"][my, mx, c, by, bx].ravel()[zz][1:],
                                                 _nc(ctot[c], gy, gx), 15, st)


# ---- parameter sets and slice header --------------------------------------------------------------------------
def _nal(ref_idc, nal_type, rbsp, st=None):
    n = len(_EPB.findall(rbsp))
    if st is not None:
        st["emulation_prevention"] += n
    return b"\x00\x00\x00\x01" + bytes([(ref_idc << 5) | nal_type]) + _EPB.sub(b"\x00\x00\x03", rbsp)


def sps(width, height):
    wmb, hmb = (width + 15) // 16, (height + 15) // 16
    b = _Codes()
    b.u(8, 66)                       # profile_idc Baseline
    b.u(8, 0xC0)                     # constraint_set0_flag, constraint_set1_flag
    b.u(8, level_idc(width, height))
    b.ue(0)                          # seq_parameter_set_id
    b.ue(0)                          # log2_max_frame_num_minus4: frame_num is 4 bits
    b.ue(2)                          # pic_order_cnt_type
    b.ue(1)                          # max_num_ref_frames
    b.u(1, 0)                        # gaps_in_frame_num_value_allowed_flag
    b.ue(wmb - 1)
    b.ue(hmb - 1)
    b.u(1, 1)                        # frame_mbs_only_flag
    b.u(1, 1)                        # direct_8x8_inference_flag
    crop = wmb * 16 != width or hmb * 16 != height
    b.u(1, int(crop))
    if crop:
        b.ue(0)
        b.ue((wmb * 16 - width) // 2)
        b.ue(0)
        b.ue((hmb * 16 - height) // 2)
    b.u(1, 1)                        # vui_parameters_present_flag
    b.u(1, 0)                        # aspect_ratio_info_present_flag
    b.u(1, 0)                        # overscan_info_present_flag
    b.u(1, 1)                        # video_signal_type_present_flag
    b.u(3, 5)                        # video_format: unspecified
    b.u(1, 0)                        # video_full_range_flag: studio range
    b.u(1, 1)                        # colour_description_present_flag
    b.u(8, 6)                        # colour_primaries: BT.601 (SMPTE 170M)
    b.u(8, 6)                        # transfer_characteristics
    b.u(8, 6)                        # matrix_coefficients
    b.u(1, 0)                        # chroma_loc_info_present_flag
    b.u(1, 0)                        # timing_info_present_flag
    b.u(1, 0)                        # nal_hrd_parameters_present_flag
    b.u(1, 0)                        # vcl_hrd_parameters_present_flag
    b.u(1, 0)                        # pic_struct_present_flag
    b.u(1, 1)                        # bitstream_restriction_flag
    b.u(1, 1)                        # motion_vectors_over_pic_boundaries_flag
    b.ue(0)                          # max_bytes_per_pic_denom
    b.ue(0)                          # max_bits_per_mb_denom
    b.ue(16)                         # log2_max_mv_length_horizontal
    b.ue(16)                         # log2_max_mv_length_vertical
    b.ue(0)                          # max_num_reorder_frames
    b.ue(1)                          # max_dec_frame_buffering
    return b.tobytes()


def pps(qp):
    b = _Codes()
    b.ue(0)                          # pic_parameter_set_id
    b.ue(0)                          # seq_parameter_set_id
    b.u(1, 0)                        # entropy_coding_mode_flag: CAVLC
    b.u(1, 0)                        # bottom_field_pic_order_in_frame_present_flag
    b.ue(0)                          # num_slice_groups_minus1
    b.ue(0)                          # num_ref_idx_l0_default_active_minus1
    b.ue(0)                          # num_ref_idx_l1_default_active_minus1
    b.u(1, 0)                        # weighted_pred_flag
    b.u(2, 0)                        # weighted_bipred_idc
    b.se(qp - 26)                    # pic_init_qp_minus26
    b.se(0)                          # pic_init_qs_minus26
    b.se(0)                          # chroma_qp_index_offset
    b.u(1, 1)                        # deblocking_filter_control_present_flag
    b.u(1, 0)                        # constrained_intra_pred_flag
    b.u(1, 0)                        # redundant_pic_cnt_present_flag
    return b.tobytes()


def picture_kind(pos, keyframe_distance):
    """position within the item -> (idr, frame_num, idr_pic_id)"""
    k = pos % keyframe_distance
    return k == 0, k % 16, (pos // keyframe_distance) & 1


def slice_header(b, idr, frame_num, idr_pic_id):
    b.ue(0)                          # first_mb_in_slice
    b.ue(7)                          # slice_type I (every slice of the picture)
    b.ue(0)                          # pic_parameter_set_id
    b.u(4, frame_num)
    if idr:
        b.ue(idr_pic_id)
        b.u(1, 0)                    # no_output_of_prior_pics_flag
        b.u(1, 0)                    # long_term_reference_flag
    else:
        b.u(1, 0)                    # adaptive_ref_pic_marking_mode_flag
    b.se(0)                          # slice_qp_delta
    b.ue(1)                          # disable_deblocking_filter_idc


def new_stats():
    return {"luma_mode": [0] * 4, "chroma_mode": [0] * 4, "nc_class": [0] * 5, "level_prefix_14": 0,
            "level_prefix_15": 0, "total_coeff_16": 0, "emulation_prevention": 0}


def check_args(width, height, qp):
    if width <= 0 or height <= 0 or width % 2 or height % 2:
        raise ValueError(f"H.264 frames need an even width and height, got {width}x{height}")
    if width > MAX_SIDE or height > MAX_SIDE or ((width + 15) // 16) * ((height + 15) // 16) > MAX_MBS:
        raise ValueError(f"{width}x{height} is beyond level 5.1 (a side over {MAX_SIDE} or over {MAX_MBS} macroblocks)")
    if not 0 <= qp <= 51:
        raise ValueError(f"QP {qp} is outside 0-51")


def encode_frame(rgb, qp=23, pos=0, keyframe_distance=120, stats=None):
    """One (H, W, 3) uint8 RGB frame at position `pos` of its item -> (access unit bytes, (Y, Cb, Cr) uint8
    reconstruction at display size)."""
    h, w, _ = rgb.shape
    check_args(w, h, qp)
    st = stats if stats is not None else new_stats()
    planes = rgb_to_planes(rgb)
    rec, m = _reconstruct(planes, qp, st)
    idr, frame_num, idr_id = picture_kind(pos, keyframe_distance)
    b = _Codes()
    slice_header(b, idr, frame_num, idr_id)
    _slice_data(b, m, st)
    au = b""
    if idr:
        au = _nal(3, 7, sps(w, h)) + _nal(3, 8, pps(qp))
    au += _nal(3 if idr else 2, 5 if idr else 1, b.tobytes(), st)
    planes_out = (rec[0][:h, :w].astype(np.uint8), rec[1][:h // 2, :w // 2].astype(np.uint8),
                  rec[2][:h // 2, :w // 2].astype(np.uint8))
    return au, planes_out


def encode(frames, qp=23, keyframe_distance=120, positions=None, stats=None):
    """(N, H, W, 3) uint8 RGB frames of one item -> (list of N access units, list of N (Y, Cb, Cr) reconstructions).
    positions: each frame's position within its item (default 0..N-1)."""
    aus, recs = [], []
    for i, f in enumerate(frames):
        au, rec = encode_frame(f, qp, i if positions is None else positions[i], keyframe_distance, stats)
        aus.append(au)
        recs.append(rec)
    return aus, recs


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def to_nv12(rec):
    """(Y, Cb, Cr) -> (luma (H, W), interleaved chroma (H / 2, W)) as oracle.nv12_to_rgb takes them"""
    y, cb, cr = rec
    c = np.empty((cb.shape[0], 2 * cb.shape[1]), np.uint8)
    c[:, 0::2], c[:, 1::2] = cb, cr
    return y, c


# ---- the test sweep ---------------------------------------------------------------------------------------------
SWEEP_QPS = (0, 1, 12, 23, 35, 51)
# even sizes over every residue mod 16 of both sides, with the 2 x 2, 2 x N and N x 2 extremes
SWEEP_SIZES = [(2, 2), (2, 34), (34, 2)] + [(16 + r, 32 + (r + 6) % 16) for r in range(0, 16, 2)]


def content(kind, h, w, seed):
    """(H, W, 3) uint8 test frames: noise, gradient, flat, saturated, checkerboard, stripes."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "gradient":
        a, b = rng.integers(1, 6, 2)
        return np.stack([(xx * a + seed) % 256, (yy * b) % 256, ((xx + yy) * 2) % 256], -1).astype(np.uint8)
    if kind == "flat":
        return np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()
    if kind == "saturated":
        return np.where(rng.random((h // 8 + 1, w // 8 + 1, 3))[yy // 8, xx // 8] < 0.5, 0, 255).astype(np.uint8)
    if kind == "checkerboard":
        return np.where(((yy // 2 + xx // 2) % 2)[..., None] == 0, 255, 0).repeat(3, -1).astype(np.uint8)
    if kind == "stripes":  # vertical stripes over horizontal ones: the V and H modes win somewhere
        v = ((xx * 37) % 251).astype(np.int64)
        hz = ((yy * 53) % 241).astype(np.int64)
        pick = (xx // 16 + yy // 16) % 2 == 0
        return np.stack([np.where(pick, v, hz)] * 3, -1).astype(np.uint8)
    raise ValueError(kind)


SWEEP_CONTENT = ("noise", "gradient", "flat", "saturated", "checkerboard", "stripes")


def natural(h, w, seed):
    """smooth fields plus mild noise: content where the quantiser, not the source, decides the quality"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    planes = []
    for c in range(3):
        f = sum(np.sin(rng.uniform(0.01, 0.08) * xx + rng.uniform(0.01, 0.08) * yy + rng.uniform(0, 6)) for _ in range(4))
        planes.append(128 + 28 * f + rng.normal(0, 4, (h, w)))
    return np.clip(np.stack(planes, -1), 0, 255).astype(np.uint8)


# ---- the float reference the integer colour stage approximates -------------------------------------------------
def bt601_float(rgb):
    """BT.601 studio range in float64, from Kr = 0.299 and Kb = 0.114 (not from the integer coefficients above):
    (..., 3) RGB -> Y, Cb, Cr.  Pass 2x2 block means to get 4:2:0 chroma."""
    kr, kb = 0.299, 0.114
    x = np.asarray(rgb, np.float64)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    y = kr * r + (1 - kr - kb) * g + kb * b
    return (16 + 219 / 255 * y, 128 + 224 / 255 * (b - y) / (2 - 2 * kb), 128 + 224 / 255 * (r - y) / (2 - 2 * kr))


def bt601_planes(frame):
    """(H, W, 3) uint8 frame, H and W even -> float64 Y (H, W) and Cb, Cr (H / 2, W / 2), each chroma sample from
    the mean of its 2x2 block: what an exact encoder's planes would hold before rounding"""
    h, w, _ = frame.shape
    y = bt601_float(frame)[0]
    _, cb, cr = bt601_float(frame.astype(np.float64).reshape(h // 2, 2, w // 2, 2, 3).mean((1, 3)))
    return y, cb, cr


def sweep():
    """(name, frames (3, H, W, 3), qp) over SWEEP_SIZES x SWEEP_CONTENT x SWEEP_QPS; encode them as one item with
    keyframe_distance 2 (IDR, non-IDR I, IDR)."""
    for w, h in SWEEP_SIZES:
        for ci, kind in enumerate(SWEEP_CONTENT):
            frames = np.stack([content(kind, h, w, 1000 * w + 10 * h + 3 * ci + i) for i in range(3)])
            for qp in SWEEP_QPS:
                yield f"{kind}-{w}x{h}-qp{qp}", frames, qp
