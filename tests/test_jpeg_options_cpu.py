"""cv2's JPEG options (sampling factor, optimised Huffman tables, luma and chroma quality), host side: the options
oracle (tests/helpers/jpeg_options.py) against live cv2.imencode and against recorded hashes of cv2 4.13's bytes;
its DHT segments against those parsed out of cv2's files; its jpeg_gen_optimal_table against a second, literal
restatement of JPEG Annex K.2 / K.3 on synthetic frequencies (ties, one symbol, lengths over 16); cv2's rules for
the two qualities; the C ABI's refusals and bound; the client's encoding of the new ImageEncoder fields.
The GPU kernels are held to the same oracle in tests/test_jpeg_options_gpu.py."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from helpers import jpeg_options as O
from oracle import jpeg as J
from scanner_b200 import cabi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_options_cv2.json")
SWEEP = O.sweep()


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)["sha256"]


def _sof_factors(data):
    i = data.index(b"\xff\xc0")
    return data[i + 11]  # component 1's h << 4 | v


def test_oracle_equals_live_cv2_on_the_sweep():
    pytest.importorskip("cv2")
    bad = [name for name, f, q, o in SWEEP if O.encode(f, q, **o) != O.cv2_encode(f, q, **o)]
    assert not bad, bad[:10]


def test_oracle_equals_recorded_cv2_hashes():
    golden = _golden()
    big = [(f"{m}_noise_1080x1920x3_q95", J.content("noise", 1080, 1920, 3, 1080), 95, {"sampling": m})
           for m in O.SAMPLING]
    big += [(f"{m}_noise_1080x1920x3_q95_opt", J.content("noise", 1080, 1920, 3, 1080), 95,
             {"sampling": m, "optimize": True}) for m in ("444", "420")]
    cases = SWEEP + big
    assert set(golden) == {name for name, _, _, _ in cases}
    bad = [name for name, f, q, o in cases if hashlib.sha256(O.encode(f, q, **o)).hexdigest() != golden[name]]
    assert not bad, bad[:10]


def test_sweep_covers_every_residue_of_every_mcu():
    for mode, (hs, vs) in O.SAMPLING.items():
        shapes = [f.shape for name, f, _, o in SWEEP if o.get("sampling") == mode and f.shape[-1] == 3
                  and "_l" not in name and not o.get("optimize")]
        assert {w % (8 * hs) for _, w, _ in shapes} == set(range(8 * hs)), mode
        assert {h % (8 * vs) for h, _, _ in shapes} == set(range(8 * vs)), mode
        qs = {q for name, _, q, o in SWEEP if o.get("sampling") == mode}
        assert set(O.QUALITIES) <= qs, mode
    assert max(f.shape[1] for _, f, _, o in SWEEP if o.get("sampling") == "411") == 64
    assert {name.split("_")[1] for name, _, _, o in SWEEP if "_l" not in name and "default" not in name} \
        == set(J.KINDS)
    opt = [(f, q, o) for _, f, q, o in SWEEP if o.get("optimize")]
    assert {o.get("sampling") for _, _, o in opt} >= set(O.SAMPLING) and {q for _, q, _ in opt} >= set(O.QUALITIES)
    assert {f.ndim == 3 and f.shape[2] == 3 for f, _, _ in opt} == {True, False}


# ---- optimised tables -------------------------------------------------------------------------------------------
def k2_k3(freq):
    """A second restatement of the table builder, written from JPEG Annex K.2 (Figure K.1, Code_size), K.3 (Figure
    K.3, Adjust_BITS) and K.4 (Figure K.4, Sort_input) with libjpeg's choices made explicit: FREQ(256) = 1 is the
    reserved point, V1 is the least FREQ with the largest index among equals and V2 the next least other than V1."""
    FREQ = list(freq) + [1]
    CODESIZE, OTHERS = [0] * 257, [-1] * 257
    nonzero = lambda: [i for i in range(257) if FREQ[i] > 0]  # noqa: E731
    while len(nonzero()) > 1:
        cand = nonzero()
        V1 = max(cand, key=lambda i: (-FREQ[i], i))
        V2 = max((i for i in cand if i != V1), key=lambda i: (-FREQ[i], i))
        FREQ[V1] += FREQ[V2]
        FREQ[V2] = 0
        for start, tail_link in ((V1, True), (V2, False)):
            i = start
            CODESIZE[i] += 1
            while OTHERS[i] != -1:
                i = OTHERS[i]
                CODESIZE[i] += 1
            if tail_link:
                OTHERS[i] = V2
    BITS = [0] * 33
    for c in CODESIZE:
        if c:
            BITS[c] += 1
    I = 32
    while I > 16:
        if BITS[I] > 0:
            J_ = I - 1
            while True:
                J_ -= 1
                if BITS[J_] > 0:
                    break
            BITS[I] -= 2
            BITS[I - 1] += 1
            BITS[J_ + 1] += 2
            BITS[J_] -= 1
        else:
            I -= 1
    while I > 0 and BITS[I] == 0:
        I -= 1
    if I > 0:
        BITS[I] -= 1
    HUFFVAL = [j for size in range(1, 33) for j in range(256) if CODESIZE[j] == size]
    return BITS[1:17], HUFFVAL


def synthetic_frequencies():
    """{name: 256 frequencies}: equal counts (every pick a tie), one symbol, Fibonacci counts and powers of two
    (lengths up to 30 before K.3; libjpeg refuses a table with a length over 32), and random counts"""
    rng = np.random.default_rng(5)
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    out = {"equal_162": [7 if i < 162 else 0 for i in range(256)], "equal_all": [3] * 256,
           "equal_12": [5 if i < 12 else 0 for i in range(256)], "one_symbol": [0] * 255 + [40],
           "one_symbol_0": [9] + [0] * 255, "two_symbols": [0, 4] + [0] * 253 + [4],
           "fibonacci": [fib[i] if i < 30 else 0 for i in range(256)],
           "fibonacci_spread": [fib[i // 8] if i % 8 == 0 and i // 8 < 30 else 0 for i in range(256)],
           "powers_of_two": [1 << i if i < 30 else 0 for i in range(256)],
           "random": rng.integers(0, 1000, 256).tolist(), "random_sparse": (rng.integers(0, 3, 256) *
                                                                          rng.integers(0, 10 ** 6, 256)).tolist()}
    return out


@pytest.mark.parametrize("name", sorted(synthetic_frequencies()))
def test_gen_optimal_table_equals_annex_k(name):
    freq = synthetic_frequencies()[name]
    bits, vals = O.gen_optimal_table(freq)
    assert (bits, vals) == k2_k3(freq)
    assert max(i for i in range(16) if bits[i] or i == 0) < 16 and sum(bits) == len(vals)
    assert sorted(vals) == [i for i in range(256) if freq[i]]
    if name.startswith("fibonacci"):
        assert bits[15] > 0  # lengths over 16 were folded back to 16


def test_dht_segments_equal_cv2s():
    pytest.importorskip("cv2")
    n = 0
    for name, f, q, o in SWEEP:
        if o.get("optimize"):
            ours, theirs = O.dht_segments(O.encode(f, q, **o)), O.dht_segments(O.cv2_encode(f, q, **o))
            assert ours == theirs, name
            n += 1
    assert n > 100
    # per-frame headers: the optimised header's length follows the frame
    a = O.encode(J.content("noise", 53, 37, 3, 1), 95, optimize=True)
    b = O.encode(J.content("gradient", 53, 37, 3, 1), 95, optimize=True)
    assert a.index(b"\xff\xda") != b.index(b"\xff\xda")


def test_default_options_are_the_default_encoder():
    for name, frame, q in J.sweep()[::7]:
        assert O.encode(frame, q) == O.encode(frame, q, sampling="420") == J.encode(frame, q), name


def test_luma_and_chroma_quality_rules():
    cv2 = pytest.importorskip("cv2")  # noqa: F841
    f = J.content("noise", 37, 53, 3, 9)
    g = np.ascontiguousarray(f[..., 0])
    # a luma quality alone sets both tables, in place of `quality`
    assert O.encode(f, 80, luma_quality=50) == O.encode(f, 50) == O.cv2_encode(f, 80, luma_quality=50)
    # a chroma quality alone is ignored
    assert O.encode(f, 60, chroma_quality=30) == O.encode(f, 60) == O.cv2_encode(f, 60, chroma_quality=30)
    # equal: as one quality, the sampling option kept
    for mode in O.SAMPLING:
        got = O.encode(f, 95, sampling=mode, luma_quality=40, chroma_quality=40)
        assert got == O.encode(f, 40, sampling=mode) == O.cv2_encode(f, 95, sampling=mode, luma_quality=40,
                                                                        chroma_quality=40)
        assert _sof_factors(got) == {"444": 0x11, "422": 0x21, "420": 0x22, "440": 0x12, "411": 0x41}[mode]
    # different: each table at its own quality, and 4:4:4 whatever the sampling option says
    for mode in O.SAMPLING:
        got = O.encode(f, 95, sampling=mode, luma_quality=40, chroma_quality=70)
        assert got == O.cv2_encode(f, 95, sampling=mode, luma_quality=40, chroma_quality=70)
        assert _sof_factors(got) == 0x11
        assert got != O.encode(f, 40, sampling="444") and got != O.encode(f, 70, sampling="444")
    # gray frames: one table at the luma quality, the sampling ignored
    for mode in O.SAMPLING:
        assert O.encode(g, 95, sampling=mode, luma_quality=40, chroma_quality=70) == J.encode(g, 40) \
            == O.cv2_encode(g, 95, sampling=mode, luma_quality=40, chroma_quality=70)
    assert O.settings(3, 95, None, 40, 70) == ((40, 70), (1, 1))
    assert O.settings(3, 95, "411", 0, 70) == ((95, 95), (4, 1))
    assert O.settings(1, 95, "422", 40, 70) == ((40, 70), (1, 1))


def test_oracle_refuses_what_the_encoder_refuses():
    f = np.zeros((4, 4, 3), np.uint8)
    for kw in ({"sampling": "423"}, {"sampling": ""}, {"luma_quality": 101}, {"chroma_quality": -1}):
        with pytest.raises(ValueError):
            O.encode(f, 95, **kw)


def _call(opts, n=1, w=8, h=8, c=3, q=95):
    L = cabi.lib()
    sizes = (ctypes.c_size_t * 1)()
    alloc = cabi.ALLOC_FN(lambda ctx, nbytes: None)
    return L.scn_jpeg_encode_u8_opts(None, n, w, h, c, q, ctypes.byref(opts) if opts is not None else None, alloc,
                                     None, sizes, None)


def test_c_abi_refuses_bad_options_before_launching():
    bad = [cabi.JpegOptions(s, 0, 0) for s in (0x13, 0x22 | 0x100, -1, 0x31, 0x14)]
    bad += [cabi.JpegOptions(0, q, 0) for q in (-1, 101)] + [cabi.JpegOptions(0, 0, q) for q in (-1, 101)]
    bad += [cabi.JpegOptions(0, 0, 0, k) for k in (-1, 2)]
    L = cabi.lib()
    for o in bad:
        assert _call(o) == -1, (o.sampling, o.luma_quality, o.chroma_quality)  # SCN_E_BADARG
        assert _call(o, c=1) == -1  # refused for gray frames too
        assert L.scn_jpeg_encode_bound_opts(8, 8, 3, ctypes.byref(o)) == 0
    assert _call(cabi.JpegOptions(0x11, 0, 0), q=0) == -1
    assert _call(cabi.JpegOptions(0x11, 50, 0), c=2) == -2  # SCN_E_UNSUPPORTED, as without options
    assert _call(cabi.JpegOptions(0x41, 50, 60)) == -1  # no frame pointers
    assert _call(cabi.JpegOptions(0x41, 50, 60), n=0) == 0
    assert _call(None, n=0) == 0


def test_bound_follows_the_sampling():
    L = cabi.lib()

    def bound(w, h, c, **kw):
        from scanner_b200 import kernels
        return kernels.jpeg_encode_bound(w, h, c, **kw)

    for w, h in ((16, 16), (53, 37), (65500, 8), (8, 65500)):
        assert bound(w, h, 3) == bound(w, h, 3, sampling="420") == L.scn_jpeg_encode_bound(w, h, 3)
        for mode, (hs, vs) in O.SAMPLING.items():
            mcus = -(-w // (8 * hs)) * -(-h // (8 * vs))
            want = len(O.header(w, h, 3, (95, 95), (hs, vs))) + 2 * ((mcus * (hs * vs + 2) * 1660 + 7) // 8) + 2
            assert bound(w, h, 3, sampling=mode) == want, (w, h, mode)
            assert bound(w, h, 1, sampling=mode) == L.scn_jpeg_encode_bound(w, h, 1)
        # different qualities code 4:4:4
        assert bound(w, h, 3, sampling="411", luma_quality=40, chroma_quality=70) == bound(w, h, 3, sampling="444")
    assert bound(16, 16, 3, sampling="444") > bound(16, 16, 3)
    assert bound(8, 8, 3, sampling="4:2:0") == 0
    # optimised DC codes can be 16 bits long: 5 more bits per block, the same header
    for mode, (hs, vs) in O.SAMPLING.items():
        w, h = 53, 37
        blocks = -(-w // (8 * hs)) * -(-h // (8 * vs)) * (hs * vs + 2)
        want = len(O.header(w, h, 3, (95, 95), (hs, vs))) + 2 * ((blocks * 1665 + 7) // 8) + 2
        assert bound(w, h, 3, sampling=mode, optimize=True) == want
    for name, f, q, o in SWEEP[::5]:
        h, w, c = f.shape
        assert len(O.encode(f, q, **o)) <= bound(w, h, c, **o), name


def test_client_encodes_the_options_into_image_encoder_args():
    import scanner_b200 as sp
    from scanner_b200 import protolite
    sc = sp.Client(gpus=[], cpu_instances=1)
    try:
        frames = sc.io.Input([sp.NamedVideoStream(sc, "a", frames=np.zeros((2, 4, 4, 3), np.uint8))])
        msg = sc._op_protos["ImageEncoder"]["init"]
        node = sc.ops.ImageEncoder(frame=frames, format="jpg", quality=80, sampling="444", optimize=True,
                                   luma_quality=70, chroma_quality=60)._op
        assert node.args == protolite.encode(msg, {"format": "jpg", "quality": 80, "sampling": "444",
                                                   "optimize": True, "luma_quality": 70, "chroma_quality": 60})
        assert node.args == b"\x0a\x03jpg\x10\x50\x1a\x03444\x20\x01\x28\x46\x30\x3c"
        # without the options the message is what it was before the fields existed
        assert sc.ops.ImageEncoder(frame=frames, format="jpg", quality=80)._op.args == b"\x0a\x03jpg\x10\x50"
    finally:
        sc.stop()
