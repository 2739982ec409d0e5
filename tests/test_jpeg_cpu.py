"""JPEG output of ImageEncoder, host side: the numpy restatement of libjpeg's encoder (oracle/jpeg.py) against
live cv2.imencode and against recorded hashes of cv2 4.13's bytes; the C ABI's argument checks and bound; the
client's encoding of `quality=`.  The GPU kernels are held to the same oracle in tests/test_jpeg_gpu.py."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import jpeg as J
from scanner_b200 import cabi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_cv2.json")
SWEEP = J.sweep()


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)["sha256"]


def test_oracle_equals_live_cv2_on_the_sweep():
    pytest.importorskip("cv2")
    bad = [name for name, frame, q in SWEEP if J.encode(frame, q) != J.cv2_encode(frame, q)]
    assert not bad, bad[:10]


def test_oracle_equals_recorded_cv2_hashes():
    golden = _golden()
    cases = SWEEP + [("noise_1080x1920x3_q95", J.content("noise", 1080, 1920, 3, 1080), 95)]
    assert set(golden) == {name for name, _, _ in cases}
    bad = [name for name, frame, q in cases if hashlib.sha256(J.encode(frame, q)).hexdigest() != golden[name]]
    assert not bad, bad[:10]


def test_sweep_covers_every_residue_and_the_degenerate_shapes():
    shapes = {frame.shape for _, frame, _ in SWEEP}
    assert {h % 16 for h, _, _ in shapes} == set(range(16)) and {w % 16 for _, w, _ in shapes} == set(range(16))
    assert {(1, 1, 3), (1, 1, 1), (1, 23, 3), (17, 1, 3)} <= shapes
    assert {q for _, _, q in SWEEP} == set(J.QUALITIES)
    assert {name.split("_")[0] for name, _, _ in SWEEP} == set(J.KINDS)


def test_oracle_refuses_what_the_encoder_refuses():
    for bad in (np.zeros((4, 4, 2), np.uint8), np.zeros((4, 4, 4), np.uint8)):
        with pytest.raises(ValueError):
            J.encode(bad)
    for q in (0, 101):
        with pytest.raises(ValueError):
            J.encode(np.zeros((4, 4, 3), np.uint8), q)


def test_c_abi_refuses_bad_arguments_before_launching():
    L = cabi.lib()
    sizes = (ctypes.c_size_t * 1)()
    alloc = cabi.ALLOC_FN(lambda ctx, n: None)
    args = dict(n=1, w=8, h=8, c=3, q=95)

    def call(**kw):
        a = {**args, **kw}
        return L.scn_jpeg_encode_u8(None, a["n"], a["w"], a["h"], a["c"], a["q"], alloc, None, sizes, None)

    assert call(c=2) == -2 and call(c=4) == -2  # SCN_E_UNSUPPORTED
    assert call(w=65501) == -2 and call(h=65501) == -2
    assert call(q=0) == -1 and call(q=101) == -1 and call(w=0) == -1 and call(n=-1) == -1  # SCN_E_BADARG
    assert call() == -1  # no frame pointers
    assert call(n=0) == 0
    assert L.scn_jpeg_encode_bound(8, 8, 2) == 0 and L.scn_jpeg_encode_bound(65501, 8, 3) == 0


def test_bound_covers_the_longest_files_of_the_sweep():
    L = cabi.lib()
    for name, frame, q in SWEEP:
        h, w, c = frame.shape
        assert len(J.encode(frame, q)) <= L.scn_jpeg_encode_bound(w, h, c), name
    # header + 2 bytes per worst-case bit-stream byte + EOI: 1660 bits per block, 6 blocks per 16 x 16 MCU
    assert L.scn_jpeg_encode_bound(16, 16, 3) == len(J.header(16, 16, 3, 95)) + 2 * (6 * 1660 // 8) + 2


def test_client_encodes_quality_into_image_encoder_args():
    import scanner_b200 as sp
    from scanner_b200 import protolite
    sc = sp.Client(gpus=[], cpu_instances=1)
    try:
        frames = sc.io.Input([sp.NamedVideoStream(sc, "a", frames=np.zeros((2, 4, 4, 3), np.uint8))])
        node = sc.ops.ImageEncoder(frame=frames, format="jpg", quality=80)._op
        msg = sc._op_protos["ImageEncoder"]["init"]
        assert node.args == protolite.encode(msg, {"format": "jpg", "quality": 80})
        assert node.args == b"\x0a\x03jpg\x10\x50"  # field 1 length-delimited, field 2 varint
        # without quality the message is what it was before the field existed
        assert sc.ops.ImageEncoder(frame=frames, format="png")._op.args == b"\x0a\x03png"
    finally:
        sc.stop()
