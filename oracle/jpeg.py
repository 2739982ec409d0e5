"""cv2.imencode('.jpg') restated in integer numpy -- the JPEG ImageEncoder's oracle (test infrastructure).

cv2 writes JPEG through libjpeg-turbo with its defaults: baseline sequential, the islow integer FDCT, Annex K
quantisation tables scaled by `quality`, Annex K Huffman tables, no restart markers, a JFIF APP0 header, 4:2:0
for three channels.  Every step below is libjpeg's integer arithmetic, so the file bytes can be written down
exactly; tests/test_jpeg_cpu.py holds encode() to live cv2.imencode and to recorded hashes of its output.
Frames are RGB (the pipeline's order); cv2 is given the same frame as BGR.
"""
import numpy as np

# Annex K tables K.1 / K.2, natural (row-major) order
LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
CHROMA_Q = np.full(64, 99, np.int64)
CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]


def _zigzag():
    """ZIGZAG[k] = natural index of the k-th coefficient in zig-zag order."""
    order = sorted(((r + c, r if (r + c) % 2 else c, r * 8 + c) for r in range(8) for c in range(8)))
    return np.array([i for _, _, i in order], np.int64)


ZIGZAG = _zigzag()

# Annex K tables K.3-K.6: (BITS[1..16], HUFFVAL)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))


def _ac_vals(head):
    """HUFFVAL of an Annex K AC table: `head` (the short codes), then every remaining (run, size) with size 1-10
    in increasing order, as both tables list them."""
    rest = [(r << 4) | s for r in range(16) for s in range(1, 11) if (r << 4) | s not in head]
    return head + rest


AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125], _ac_vals([
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7,
    0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5,
    0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2,
    0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA]))
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119], _ac_vals([
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0,
    0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26,
    0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5,
    0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
    0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA,
    0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA]))

MAX_DIMENSION = 65500  # libjpeg's JPEG_MAX_DIMENSION


def quant_table(base, quality):
    """jpeg_set_quality: the Annex K table scaled by quality (1-100), clamped to [1, 255] (baseline)."""
    s = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * s + 50) // 100, 1, 255)


def huff_codes(table):
    """(BITS, HUFFVAL) -> {symbol: (code, length)}, the canonical codes of Annex C."""
    bits, vals = table
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


def _lut(table):
    """symbol -> (code, length) as two 256-entry arrays."""
    code = np.zeros(256, np.int64)
    size = np.zeros(256, np.int64)
    for s, (c, n) in huff_codes(table).items():
        code[s], size[s] = c, n
    return code, size


def _fix(x):
    return int(x * 65536 + 0.5)


def rgb_ycc(frame):
    """libjpeg's rgb_ycc_convert (jccolor.c), 16-bit fixed point."""
    f = frame.astype(np.int64)
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    half, cbias = 1 << 15, (128 << 16) + (1 << 15) - 1
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + cbias) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + cbias) >> 16
    return y, cb, cr


def downsample(plane, rows, cols):
    """h2v2_downsample (jcsample.c) of a full-resolution component: the last pixel column replicated out to 2 cols,
    the last row duplicated when the height is odd, then the last downsampled row replicated down to `rows`."""
    h, w = plane.shape
    p = np.pad(plane, ((0, h & 1), (0, 2 * cols - w)), mode="edge")
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = np.where(np.arange(cols) % 2 == 0, 1, 2)
    s = (s + bias) >> 2
    return np.pad(s, ((0, rows - s.shape[0]), (0, 0)), mode="edge")


def blocks(plane):
    """(8 by, 8 bx) plane -> (by, bx, 8, 8) blocks."""
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).transpose(0, 2, 1, 3)


CONST_BITS, PASS1_BITS = 13, 2
F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
         f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, pass1):
    """One pass of jpeg_fdct_islow (jfdctint.c) along the last axis of d (..., 8)."""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = np.empty_like(d)
    sh = CONST_BITS - PASS1_BITS if pass1 else CONST_BITS + PASS1_BITS
    if pass1:
        out[..., 0] = (t10 + t11) << PASS1_BITS
        out[..., 4] = (t10 - t11) << PASS1_BITS
    else:
        out[..., 0] = _descale(t10 + t11, PASS1_BITS)
        out[..., 4] = _descale(t10 - t11, PASS1_BITS)
    z1 = (t12 + t13) * F["f0541"]
    out[..., 2] = _descale(z1 + t13 * F["f0765"], sh)
    out[..., 6] = _descale(z1 - t12 * F["f1847"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F["f1175"]
    t4, t5, t6, t7 = t4 * F["f0298"], t5 * F["f2053"], t6 * F["f3072"], t7 * F["f1501"]
    z1, z2 = z1 * -F["f0899"], z2 * -F["f2562"]
    z3, z4 = z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
    out[..., 7] = _descale(t4 + z1 + z3, sh)
    out[..., 5] = _descale(t5 + z2 + z4, sh)
    out[..., 3] = _descale(t6 + z2 + z3, sh)
    out[..., 1] = _descale(t7 + z1 + z4, sh)
    return out


def fdct(blk):
    """(..., 8, 8) samples -> (..., 8, 8) jpeg_fdct_islow of samples - 128 (8 times the orthonormal DCT)."""
    d = _fdct_1d(blk.astype(np.int64) - 128, True)
    return _fdct_1d(d.swapaxes(-1, -2), False).swapaxes(-1, -2)


def fdct_quant(blk, qtab):
    """(..., 8, 8) samples -> (..., 64) quantised coefficients in zig-zag order."""
    d = fdct(blk)
    c = d.reshape(d.shape[:-2] + (64,))[..., ZIGZAG]
    q = 8 * qtab[ZIGZAG]
    return np.sign(c) * ((np.abs(c) + (q >> 1)) // q)


def _nbits(v):
    """bit length of |v| (0 for 0)."""
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while (a >> n).any():
        n += (a >> n) > 0
    return n


def _coded(coefs, comps, dc_luts, ac_luts):
    """coefs (nblocks, 64) in coding order; comps[i] = component of block i (DC predictor and table:
    0 -> luma tables, else chroma) -> (the scan's bytes before stuffing, 1-padded; the symbols coded as an
    (nsymbols, 3) array of (class 0 DC / 1 AC, table 0 luma / 1 chroma, symbol))."""
    nb = coefs.shape[0]
    dc = coefs[:, 0]
    prev = np.zeros(nb, np.int64)
    for c in np.unique(comps):
        idx = np.nonzero(comps == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    tab = (comps != 0).astype(np.int64)
    keys, vals, lens, syms = [], [], [], []

    def sym(key, lut_code, lut_size, s, v, nbits, cls, t):
        # a Huffman symbol followed by nbits extra bits: negative values send v - 1 in nbits bits
        extra = np.where(v < 0, v - 1, v) & ((1 << nbits) - 1)
        keys.append(key)
        vals.append((lut_code[s] << nbits) | extra)
        lens.append(lut_size[s] + nbits)
        syms.append(np.stack(np.broadcast_arrays(cls, t, s), -1).reshape(-1, 3))

    diff = dc - prev
    n = _nbits(diff)
    bidx = np.arange(nb, dtype=np.int64)
    for t in (0, 1):
        m = tab == t
        sym(bidx[m] * 1024, *dc_luts[t], n[m], diff[m], n[m], 0, t)
    blk, k = np.nonzero(coefs[:, 1:])
    k = k + 1
    v = coefs[blk, k]
    first = np.ones(len(blk), bool)
    first[1:] = blk[1:] != blk[:-1]
    prevk = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prevk - 1
    nz = _nbits(v)
    for t in (0, 1):
        m = tab[blk] == t
        code, size = ac_luts[t]
        for j in range(3):  # ZRL (0xF0) for every full 16 zeros of the run
            z = m & (run >> 4 > j)
            zero = np.zeros(z.sum(), np.int64)
            sym(blk[z] * 1024 + k[z] * 8 + j, code, size, np.full(z.sum(), 0xF0), zero, zero, 1, t)
        sym(blk[m] * 1024 + k[m] * 8 + 4, code, size, ((run[m] & 15) << 4) | nz[m], v[m], nz[m], 1, t)
    last = np.zeros(nb, np.int64)
    last[blk] = k  # the last nonzero index of each block (k increases within a block)
    for t in (0, 1):
        e = (last < 63) & (tab == t)
        zero = np.zeros(e.sum(), np.int64)
        sym(bidx[e] * 1024 + 1000, *ac_luts[t], zero, zero, zero, 1, t)
    keys, vals, lens = (np.concatenate(a) for a in (keys, vals, lens))
    o = np.argsort(keys, kind="stable")
    vals, lens = vals[o], lens[o]
    ends = np.cumsum(lens)
    total = int(ends[-1]) if len(ends) else 0
    nbytes = (total + 7) // 8
    bits = np.ones(nbytes * 8, np.uint8)  # the tail stays 1: libjpeg pads the last byte with 1-bits
    starts = ends - lens
    for j in range(int(lens.max()) if len(lens) else 0):
        m = lens > j
        bits[starts[m] + j] = (vals[m] >> (lens[m] - 1 - j)) & 1
    return np.packbits(bits), np.concatenate(syms)


def stuff(data):
    """a 0x00 after every 0xFF of the scan"""
    data = np.frombuffer(bytes(data), np.uint8)
    return np.insert(data, np.nonzero(data == 0xFF)[0] + 1, 0).tobytes()


def entropy_code(coefs, comps, dc_luts, ac_luts):
    """coefs (nblocks, 64) in coding order; comps[i] = component of block i (DC predictor and table:
    0 -> luma tables, else chroma) -> the scan's bytes, 1-padded and 0x00-stuffed."""
    return stuff(_coded(coefs, comps, dc_luts, ac_luts)[0])


def _marker(m, payload):
    return bytes([0xFF, m]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def header(width, height, channels, quality):
    """SOI, APP0 JFIF, DQT per table, SOF0, DHT per table, SOS -- what libjpeg writes before the scan."""
    out = b"\xFF\xD8"
    out += _marker(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    ntab = 2 if channels == 3 else 1
    for t, base in enumerate((LUMA_Q, CHROMA_Q)[:ntab]):
        out += _marker(0xDB, [t] + quant_table(base, quality)[ZIGZAG].tolist())
    comps = [(1, 0x22, 0), (2, 0x11, 1), (3, 0x11, 1)] if channels == 3 else [(1, 0x11, 0)]
    sof = [8, height >> 8, height & 255, width >> 8, width & 255, len(comps)]
    for c in comps:
        sof += list(c)
    out += _marker(0xC0, sof)
    for t, (dc, ac) in enumerate(((DC_LUMA, AC_LUMA), (DC_CHROMA, AC_CHROMA))[:ntab]):
        out += _marker(0xC4, [t] + dc[0] + dc[1])
        out += _marker(0xC4, [0x10 | t] + ac[0] + ac[1])
    sos = [len(comps)]
    for cid, _, t in comps:
        sos += [cid, (t << 4) | t]
    out += _marker(0xDA, sos + [0, 63, 0])
    return out


def _blocks_in_order(frame, quality):
    """-> (width, height, channels, coefficients in coding order, component of each block, Huffman lookups)"""
    frame = np.asarray(frame, np.uint8)
    if frame.ndim == 3 and frame.shape[2] == 1:
        frame = frame[..., 0]
    h, w = frame.shape[:2]
    channels = 1 if frame.ndim == 2 else frame.shape[2]
    if channels not in (1, 3) or not (1 <= quality <= 100) or not (0 < w <= MAX_DIMENSION and 0 < h <= MAX_DIMENSION):
        raise ValueError(f"unsupported frame {frame.shape} or quality {quality}")
    lq, cq = quant_table(LUMA_Q, quality), quant_table(CHROMA_Q, quality)
    bh, bw = -(-h // 8), -(-w // 8)
    luts = (_lut(DC_LUMA), _lut(DC_CHROMA)), (_lut(AC_LUMA), _lut(AC_CHROMA))
    if channels == 1:
        y = np.pad(frame.astype(np.int64), ((0, 8 * bh - h), (0, 8 * bw - w)), mode="edge")
        coefs = fdct_quant(blocks(y), lq).reshape(-1, 64)
        comps = np.zeros(len(coefs), np.int64)
    else:
        y, cb, cr = rgb_ycc(frame)
        mh, mw = -(-h // 16), -(-w // 16)
        ycoef = fdct_quant(blocks(np.pad(y, ((0, 8 * bh - h), (0, 8 * bw - w)), mode="edge")), lq)
        # every MCU's four Y blocks; those outside the real bh x bw grid are dummies: AC zero, the DC of the block
        # coded before them in the MCU
        grid = np.zeros((2 * mh, 2 * mw, 64), np.int64)
        grid[:bh, :bw] = ycoef
        real = np.zeros((2 * mh, 2 * mw), bool)
        real[:bh, :bw] = True
        mcu = grid.reshape(mh, 2, mw, 2, 64).transpose(0, 2, 1, 3, 4).reshape(mh, mw, 4, 64)
        mreal = real.reshape(mh, 2, mw, 2).transpose(0, 2, 1, 3).reshape(mh, mw, 4)
        for b in range(1, 4):
            mcu[..., b, 0] = np.where(mreal[..., b], mcu[..., b, 0], mcu[..., b - 1, 0])
        cbq = fdct_quant(blocks(downsample(cb, 8 * mh, 8 * mw)), cq)
        crq = fdct_quant(blocks(downsample(cr, 8 * mh, 8 * mw)), cq)
        coefs = np.concatenate([mcu, cbq[:, :, None], crq[:, :, None]], axis=2).reshape(-1, 64)
        comps = np.tile(np.array([0, 0, 0, 0, 1, 2]), mh * mw)
    return w, h, channels, coefs, comps, luts


def encode(frame, quality=95):
    """frame: (H, W, 3) RGB or (H, W) / (H, W, 1) gray uint8 -> the bytes of
    cv2.imencode('.jpg', frame[..., ::-1] (or the gray frame), [cv2.IMWRITE_JPEG_QUALITY, quality])."""
    w, h, channels, coefs, comps, luts = _blocks_in_order(frame, quality)
    return header(w, h, channels, quality) + entropy_code(coefs, comps, *luts) + b"\xFF\xD9"


def scan(frame, quality=95):
    """The entropy-coded segment of encode(frame, quality) before stuffing: the 1-padded bit stream, whose bytes
    the encoder's 0xFF passes split into chunks."""
    _, _, _, coefs, comps, luts = _blocks_in_order(frame, quality)
    return _coded(coefs, comps, *luts)[0].tobytes()


def symbols(frame, quality=95):
    """{(class, table, symbol): count} of the Huffman symbols encode(frame, quality) codes: class 0 DC (symbol the
    category 0-11) or 1 AC (symbol run << 4 | size, 0x00 EOB, 0xF0 ZRL); table 0 luma or 1 chroma."""
    _, _, _, coefs, comps, luts = _blocks_in_order(frame, quality)
    keys, counts = np.unique(_coded(coefs, comps, *luts)[1], axis=0, return_counts=True)
    return {tuple(int(x) for x in k): int(c) for k, c in zip(keys, counts)}


# ---- the sweep the tests hold encoders to -------------------------------------------------------------------------
KINDS = ("noise", "gradient", "saturated", "checker")
QUALITIES = (1, 2, 25, 50, 75, 95, 100)


def content(kind, h, w, channels, seed):
    """A deterministic (h, w, channels) uint8 frame of one kind."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        f = rng.integers(0, 256, (h, w, channels))
    elif kind == "gradient":
        yy, xx = np.mgrid[0:h, 0:w]
        f = np.stack([(xx * 255 // max(w - 1, 1) + 60 * c + yy * 7) % 256 for c in range(channels)], -1)
    elif kind == "saturated":  # blocks of 0 and 255 per channel: the largest coefficients and DC steps
        f = rng.integers(0, 2, (-(-h // 5), -(-w // 5), channels)).repeat(5, 0).repeat(5, 1)[:h, :w] * 255
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        f = np.repeat((((xx + yy) & 1) * 255)[..., None], channels, -1)
    return np.ascontiguousarray(f, np.uint8)


def sweep():
    """[(name, frame, quality)]: every residue of W and H mod 16 (1 x 1, 1 x N and N x 1 among them), RGB and gray,
    each content kind and quality, plus every kind x quality on two odd sizes."""
    sizes = [(h, w) for h in range(1, 18) for w in (1, 8, 13, 16, 23)]
    sizes += [(h, w) for w in range(1, 34) for h in (1, 7, 16, 30)]
    sizes = list(dict.fromkeys(sizes + [(34, 45), (1080 // 40, 1920 // 40)]))
    cases = []
    for i, (h, w) in enumerate(sizes):
        for channels in (3, 1):
            kind, q = KINDS[i % len(KINDS)], QUALITIES[(i + channels) % len(QUALITIES)]
            cases.append((f"{kind}_{h}x{w}x{channels}_q{q}", content(kind, h, w, channels, i), q))
    for kind in KINDS:
        for q in QUALITIES:
            for h, w, channels in ((17, 31, 3), (33, 19, 1)):
                cases.append((f"{kind}_{h}x{w}x{channels}_q{q}", content(kind, h, w, channels, q), q))
    return cases


# every Huffman symbol a table can code: DC categories 0-11; AC (run, size) for runs 0-15 and sizes 1-10, EOB, ZRL
DC_SYMBOLS = tuple(range(12))
AC_SYMBOLS = tuple(sorted({(r << 4) | s for r in range(16) for s in range(1, 11)} | {0x00, 0xF0}))


def symbol_corpus_frames(corpus):
    """The frames of tests/golden/jpeg_symbols.npz (oracle/make_golden_jpeg_symbols.py) -> [(name, frame, quality)].
    Key "luma_q<Q>" holds 8 x 8 blocks laid side by side in a gray 8 x 8n frame, coded in that order.  Key
    "chroma_q<Q>" holds 8 x 8 blocks X, each doubled to a 16 x 16 MCU of pixels (255 - X, 255 - X, X), whose
    Cb is X exactly; the MCUs lie side by side in a 16 x 16n RGB frame."""
    out = []
    for key in sorted(corpus.keys(), key=lambda k: (k.split("_")[0], -int(k.split("_q")[1]))):
        table, q = key.split("_q")
        b = np.asarray(corpus[key], np.uint8)
        if table == "luma":
            frame = np.ascontiguousarray(b.transpose(1, 0, 2).reshape(8, -1))
        else:
            x = b.repeat(2, 1).repeat(2, 2).transpose(1, 0, 2).reshape(16, -1)
            frame = np.ascontiguousarray(np.stack([255 - x, 255 - x, x], -1))
        out.append((key, frame, int(q)))
    return out


def cv2_encode(frame, quality):
    """cv2.imencode of an RGB or gray frame, as encode() restates it."""
    import cv2
    f = frame[..., ::-1] if frame.ndim == 3 and frame.shape[2] == 3 else frame
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(f), [cv2.IMWRITE_JPEG_QUALITY, int(quality)])
    assert ok
    return buf.tobytes()
