"""cv2.imencode('.jpg') with IMWRITE_JPEG_SAMPLING_FACTOR, IMWRITE_JPEG_LUMA_QUALITY and IMWRITE_JPEG_CHROMA_QUALITY,
restated in integer numpy on top of oracle/jpeg.py (the default encoder's oracle, whose colour conversion, FDCT,
quantisation and entropy coder are used as they are).  What the options change:

  sampling   luma factors (h, v), chroma at (1, 1): "444" (1, 1), "422" (2, 1), "420" (2, 2, the default),
             "440" (1, 2), "411" (4, 1).  MCUs are 8h x 8v pixels: Y0 .. Y(hv-1) in row-major order, then Cb, Cr.
             Chroma is downsampled as libjpeg's jcsample.c does it: the last pixel column replicated out to the MCU
             width, the last pixel row out to a multiple of v (jcprepct.c), the h x v pixels under each chroma
             sample summed, then
               1 x 1  fullsize_downsample: the sum
               2 x 1  h2v1_downsample: (sum + bias) >> 1, bias 0, 1, 0, 1, ... along the row
               2 x 2  h2v2_downsample: (sum + bias) >> 2, bias 1, 2, 1, 2, ...
               other  int_downsample: (sum + hv / 2) / hv
             and the last downsampled row replicated down to the block height.  Y blocks outside the
             ceil(W/8) x ceil(H/8) grid are dummies (jccoefct.c): AC zero and the DC of the block coded before them,
             which is libjpeg's rule for right-edge dummies (the block to the left) and bottom-edge dummies (the
             last block of the row above) alike.
  qualities  cv2 4.13 (grfmt_jpeg.cpp), probed: a luma quality alone scales both tables (in place of `quality`);
             a chroma quality alone is ignored; both together scale each table by its own (jpeg_default_qtables
             with q_scale_factor); two different ones code 4:4:4 whatever the sampling option says; the order the
             parameters are given in does not matter.
  gray       one table and no chroma: the sampling option is ignored and the luma quality (or quality) applies.
  optimize   IMWRITE_JPEG_OPTIMIZE, libjpeg's two passes (jchuff.c): the symbols of the whole frame are counted per
             table (dummy blocks included; Cb and Cr share table 1), each table is built by jpeg_gen_optimal_table
             (gen_optimal_table below) and listed in the frame's own DHT segments, which name only the symbols that
             occur.
"""
import numpy as np

from oracle import jpeg as J

SAMPLING = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2), "411": (4, 1)}
# IMWRITE_JPEG_SAMPLING_FACTOR values
CV2_SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def settings(channels, quality=95, sampling=None, luma_quality=0, chroma_quality=0):
    """cv2's rules -> ((luma quality, chroma quality), (h, v)); ValueError for what the encoder refuses."""
    sampling = "420" if sampling is None else sampling
    if sampling not in SAMPLING:
        raise ValueError(f"unknown sampling {sampling!r}")
    for q in (luma_quality, chroma_quality):
        if not 0 <= q <= 100:
            raise ValueError(f"quality {q} outside 1-100")
    if not 1 <= quality <= 100:
        raise ValueError(f"quality {quality} outside 1-100")
    lq = luma_quality or quality
    cq = chroma_quality if luma_quality and chroma_quality else lq
    if channels != 3 or lq != cq:
        return (lq, cq), (1, 1)
    return (lq, cq), SAMPLING[sampling]


def downsample(plane, h_s, v_s, rows, cols):
    """jcsample.c's downsampling of a full-resolution component to (rows, cols) for luma factors (h_s, v_s)."""
    h, w = plane.shape
    ch_rows = -(-h // v_s)
    p = np.pad(plane, ((0, ch_rows * v_s - h), (0, h_s * cols - w)), mode="edge")
    s = sum(p[dy::v_s, dx::h_s] for dy in range(v_s) for dx in range(h_s))
    odd = np.arange(cols) % 2
    if (h_s, v_s) == (1, 1):
        out = s
    elif (h_s, v_s) == (2, 1):
        out = (s + odd) >> 1
    elif (h_s, v_s) == (2, 2):
        out = (s + 1 + odd) >> 2
    else:
        out = (s + h_s * v_s // 2) // (h_s * v_s)
    return np.pad(out, ((0, rows - out.shape[0]), (0, 0)), mode="edge")


def gen_optimal_table(freq):
    """jpeg_gen_optimal_table: 256 symbol frequencies -> (BITS[1..16], HUFFVAL).  Symbol 256 is reserved with
    frequency 1 so that no code is all 1-bits.  The two smallest nonzero frequencies are merged until one is left,
    the scan taking the last of equal frequencies (libjpeg's "<="), the second pick excluding the first; code lengths
    over 16 are folded back by the K.3 adjust loop; HUFFVAL lists the symbols by unadjusted length, then value."""
    freq = [int(x) for x in freq] + [1]
    codesize, others = [0] * 257, [-1] * 257
    while True:
        c1, v = -1, None
        for i in range(257):
            if freq[i] and (v is None or freq[i] <= v):
                c1, v = i, freq[i]
        c2, v = -1, None
        for i in range(257):
            if freq[i] and (v is None or freq[i] <= v) and i != c1:
                c2, v = i, freq[i]
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = [0] * 33
    for c in codesize:
        if c:
            bits[c] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while i > 0 and bits[i] == 0:
        i -= 1
    if i > 0:
        bits[i] -= 1
    vals = [j for length in range(1, 33) for j in range(256) if codesize[j] == length]
    return bits[1:17], vals


def header(width, height, channels, qualities, factors, tables=None):
    """SOI, APP0 JFIF, DQT per table (each at its own quality), SOF0 with the luma factors, DHT, SOS.  tables:
    ((dc, ac) of table 0, (dc, ac) of table 1) as (BITS, HUFFVAL), the Annex K ones when None."""
    lq, cq = qualities
    out = b"\xFF\xD8" + J._marker(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    ntab = 2 if channels == 3 else 1
    for t, (base, q) in enumerate(((J.LUMA_Q, lq), (J.CHROMA_Q, cq))[:ntab]):
        out += J._marker(0xDB, [t] + J.quant_table(base, q)[J.ZIGZAG].tolist())
    hv = factors[0] << 4 | factors[1]
    comps = [(1, hv, 0), (2, 0x11, 1), (3, 0x11, 1)] if channels == 3 else [(1, 0x11, 0)]
    sof = [8, height >> 8, height & 255, width >> 8, width & 255, len(comps)]
    for c in comps:
        sof += list(c)
    out += J._marker(0xC0, sof)
    tables = tables or ((J.DC_LUMA, J.AC_LUMA), (J.DC_CHROMA, J.AC_CHROMA))
    for t, (dc, ac) in enumerate(tables[:ntab]):
        out += J._marker(0xC4, [t] + dc[0] + dc[1])
        out += J._marker(0xC4, [0x10 | t] + ac[0] + ac[1])
    sos = [len(comps)]
    for cid, _, t in comps:
        sos += [cid, (t << 4) | t]
    return out + J._marker(0xDA, sos + [0, 63, 0])


def _blocks_in_order(frame, quality, sampling, luma_quality, chroma_quality):
    """-> (width, height, channels, qualities, factors, coefficients in coding order, component of each block)"""
    frame = np.asarray(frame, np.uint8)
    if frame.ndim == 3 and frame.shape[2] == 1:
        frame = frame[..., 0]
    h, w = frame.shape[:2]
    channels = 1 if frame.ndim == 2 else frame.shape[2]
    if channels not in (1, 3) or not (0 < w <= J.MAX_DIMENSION and 0 < h <= J.MAX_DIMENSION):
        raise ValueError(f"unsupported frame {frame.shape}")
    (lq, cq), (hs, vs) = settings(channels, quality, sampling, luma_quality, chroma_quality)
    bh, bw = -(-h // 8), -(-w // 8)
    if channels == 1:
        y = np.pad(frame.astype(np.int64), ((0, 8 * bh - h), (0, 8 * bw - w)), mode="edge")
        coefs = J.fdct_quant(J.blocks(y), J.quant_table(J.LUMA_Q, lq)).reshape(-1, 64)
        return w, h, channels, (lq, cq), (hs, vs), coefs, np.zeros(len(coefs), np.int64)
    y, cb, cr = J.rgb_ycc(frame)
    mh, mw = -(-h // (8 * vs)), -(-w // (8 * hs))
    ycoef = J.fdct_quant(J.blocks(np.pad(y, ((0, 8 * bh - h), (0, 8 * bw - w)), mode="edge")),
                         J.quant_table(J.LUMA_Q, lq))
    grid = np.zeros((vs * mh, hs * mw, 64), np.int64)
    grid[:bh, :bw] = ycoef
    real = np.zeros((vs * mh, hs * mw), bool)
    real[:bh, :bw] = True
    ny = hs * vs
    mcu = grid.reshape(mh, vs, mw, hs, 64).transpose(0, 2, 1, 3, 4).reshape(mh, mw, ny, 64)
    mreal = real.reshape(mh, vs, mw, hs).transpose(0, 2, 1, 3).reshape(mh, mw, ny)
    for b in range(1, ny):
        mcu[..., b, 0] = np.where(mreal[..., b], mcu[..., b, 0], mcu[..., b - 1, 0])
    cqt = J.quant_table(J.CHROMA_Q, cq)
    cbq = J.fdct_quant(J.blocks(downsample(cb, hs, vs, 8 * mh, 8 * mw)), cqt)
    crq = J.fdct_quant(J.blocks(downsample(cr, hs, vs, 8 * mh, 8 * mw)), cqt)
    coefs = np.concatenate([mcu, cbq[:, :, None], crq[:, :, None]], axis=2).reshape(-1, 64)
    comps = np.tile(np.array([0] * ny + [1, 2]), mh * mw)
    return w, h, channels, (lq, cq), (hs, vs), coefs, comps


def _luts(tables):
    (dc0, ac0), (dc1, ac1) = tables
    return (J._lut(dc0), J._lut(dc1)), (J._lut(ac0), J._lut(ac1))


ANNEX_K = ((J.DC_LUMA, J.AC_LUMA), (J.DC_CHROMA, J.AC_CHROMA))


def optimal_tables(coefs, comps):
    """The frame's symbol counts per table (the symbols do not depend on the tables) -> its optimised tables"""
    syms = J._coded(coefs, comps, *_luts(ANNEX_K))[1]
    out = []
    for t in (0, 1):
        if not (syms[:, 1] == t).any():  # gray frames have no table 1
            out.append(ANNEX_K[t])
            continue
        tab = []
        for cls in (0, 1):
            s = syms[(syms[:, 0] == cls) & (syms[:, 1] == t), 2]
            tab.append(gen_optimal_table(np.bincount(s, minlength=256)))
        out.append(tuple(tab))
    return tuple(out)


def _encode(frame, quality, sampling, luma_quality, chroma_quality, optimize):
    """-> (header, scan before stuffing)"""
    w, h, c, qs, fs, coefs, comps = _blocks_in_order(frame, quality, sampling, luma_quality, chroma_quality)
    tables = optimal_tables(coefs, comps) if optimize else ANNEX_K
    return header(w, h, c, qs, fs, tables), J._coded(coefs, comps, *_luts(tables))[0].tobytes()


def encode(frame, quality=95, *, sampling=None, luma_quality=0, chroma_quality=0, optimize=False):
    """-> the bytes of cv2_encode(frame, quality, sampling=..., ...)."""
    head, data = _encode(frame, quality, sampling, luma_quality, chroma_quality, optimize)
    return head + J.stuff(data) + b"\xFF\xD9"


def scan(frame, quality=95, *, sampling=None, luma_quality=0, chroma_quality=0, optimize=False):
    """The entropy-coded segment of encode() before stuffing."""
    return _encode(frame, quality, sampling, luma_quality, chroma_quality, optimize)[1]


def dht_segments(data):
    """The payloads of the DHT segments of a JPEG file, in order."""
    out, at = [], 2
    while at + 4 <= len(data) and data[at + 1] != 0xDA:
        n = data[at + 2] << 8 | data[at + 3]
        if data[at + 1] == 0xC4:
            out.append(bytes(data[at + 4:at + 2 + n]))
        at += 2 + n
    return out


def cv2_encode(frame, quality=95, *, sampling=None, luma_quality=0, chroma_quality=0, optimize=False):
    """cv2.imencode of an RGB or gray frame with the options given (0 / None: the parameter is not passed)."""
    import cv2
    f = frame[..., ::-1] if frame.ndim == 3 and frame.shape[2] == 3 else frame
    params = [cv2.IMWRITE_JPEG_QUALITY, int(quality)]
    if sampling is not None:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, CV2_SAMPLING[sampling]]
    if luma_quality:
        params += [cv2.IMWRITE_JPEG_LUMA_QUALITY, int(luma_quality)]
    if chroma_quality:
        params += [cv2.IMWRITE_JPEG_CHROMA_QUALITY, int(chroma_quality)]
    if optimize:
        params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(f), params)
    assert ok
    return buf.tobytes()


# ---- the sweep the tests hold the encoder to ----------------------------------------------------------------------
QUALITIES = (1, 50, 75, 95, 100)
# (luma_quality, chroma_quality): alone, ignored alone, equal, different (forced 4:4:4), extremes
QUALITY_PAIRS = ((60, 0), (0, 30), (40, 40), (40, 70), (90, 20), (1, 100), (100, 1))


def sweep():
    """[(name, frame, quality, options)]: for every sampling mode, every residue of W mod the MCU width (widths 1 to
    twice it, up to 64 for 4:1:1) and of H mod the MCU height, RGB, content kinds and qualities cycling; gray frames
    with each mode (which they ignore); the luma / chroma pairs on two odd sizes in 4:2:2 and 4:2:0; every other one
    of those again with optimised tables, and every mode x kind x quality x channels with them."""
    cases = []
    for mode, (hs, vs) in SAMPLING.items():
        mw, mh = 8 * hs, 8 * vs
        sizes = [(1 + (3 * w) % (2 * mh), w) for w in range(1, 2 * mw + 1)]
        sizes += [(h, 1 + (5 * h) % (2 * mw)) for h in range(1, 2 * mh + 1)]
        sizes = list(dict.fromkeys(sizes + [(1, 1), (37, 53)]))
        for i, (h, w) in enumerate(sizes):
            kind, q = J.KINDS[i % len(J.KINDS)], QUALITIES[i % len(QUALITIES)]
            cases.append((f"{mode}_{kind}_{h}x{w}x3_q{q}", J.content(kind, h, w, 3, i), q, {"sampling": mode}))
        cases.append((f"{mode}_noise_19x27x1_q75", J.content("noise", 19, 27, 1, 7), 75, {"sampling": mode}))
    for mode in ("422", "420"):
        for lq, cq in QUALITY_PAIRS:
            for h, w in ((23, 41), (40, 72)):
                opts = {"sampling": mode, "luma_quality": lq, "chroma_quality": cq}
                cases.append((f"{mode}_l{lq}_c{cq}_noise_{h}x{w}x3", J.content("noise", h, w, 3, h + lq), 95, opts))
    for lq, cq in QUALITY_PAIRS:
        cases.append((f"default_l{lq}_c{cq}_gradient_33x19x1", J.content("gradient", 33, 19, 1, 3), 80,
                      {"luma_quality": lq, "chroma_quality": cq}))
    # optimised tables: every other case again with optimize, plus each mode x kind x quality on an odd size
    cases += [(name + "_opt", f, q, {**o, "optimize": True}) for name, f, q, o in cases[::2]]
    for mode in SAMPLING:
        for i, kind in enumerate(J.KINDS):
            for q in QUALITIES:
                for c in (3, 1):
                    cases.append((f"{mode}_{kind}_29x45x{c}_q{q}_opt", J.content(kind, 29, 45, c, q + i), q,
                                  {"sampling": mode, "optimize": True}))
    return cases
