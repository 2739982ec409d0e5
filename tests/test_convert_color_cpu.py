"""ConvertColor without a GPU: the numpy restatement of cv::cvtColor that the GPU tests compare with
(oracle/convert_color.py) against live cv2 and against recorded hashes of cv2's output, on all 2^24 RGB
triples; the code table of the C ABI; the client's encoding of `conversion=[...]`."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import convert_color as C
from scanner_b200 import cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "convert_color_cv2.json")))


@pytest.fixture(scope="module")
def triples():
    return C.all_triples()


def _source(img, code):
    return img if C.CODES[code][0] == 3 else np.ascontiguousarray(img[..., :1])


def test_all_triples_holds_every_rgb_value_once(triples):
    k = (triples[..., 0].astype(np.int64) << 16) | (triples[..., 1].astype(np.int64) << 8) | triples[..., 2]
    assert (np.sort(k.ravel()) == np.arange(1 << 24)).all()


@pytest.mark.parametrize("code", list(C.CODES))
def test_oracle_equals_live_cv2(code, triples):
    cv2 = pytest.importorskip("cv2")
    src = _source(triples, code)
    want = cv2.cvtColor(src, getattr(cv2, code))
    got = C.convert_color(src, code)
    assert got.shape == (4096, 4096, C.CODES[code][1])
    assert (got.reshape(want.shape) == want).all()


@pytest.mark.parametrize("code", list(C.CODES))
def test_oracle_equals_recorded_cv2_hashes(code, triples):
    got = C.convert_color(_source(triples, code), code)
    assert hashlib.sha256(got.tobytes()).hexdigest() == GOLDEN["sha256"][code]


def test_hsv_tables_are_opencvs():
    """RGB2HSV_b builds them with saturate_cast<int>(double): round to nearest."""
    sdiv, hdiv = C.hsv_tables(180)
    assert sdiv[0] == hdiv[0] == 0
    assert sdiv[1] == 255 << 12 and sdiv[255] == 4096 and sdiv[3] == 348160
    assert hdiv[1] == 122880 and hdiv[7] == 17554  # 122880 / 7 = 17554.29
    assert C.hsv_tables(256)[1][255] == 685      # 1048576 / 1530 = 685.34


def test_code_table_of_the_c_abi_matches_the_oracle():
    L = cabi.lib()
    names = []
    while L.scn_convert_color_name(len(names)):
        names.append(L.scn_convert_color_name(len(names)).decode())
    assert names == list(C.CODES)
    for code, name in enumerate(names):
        assert L.scn_convert_color_code(name.encode()) == code
        cin, cout = ctypes.c_int(), ctypes.c_int()
        assert L.scn_convert_color_channels(code, ctypes.byref(cin), ctypes.byref(cout)) == 0
        assert (cin.value, cout.value) == C.CODES[name]
    for bad in (b"COLOR_RGB2Lab", b"COLOR_BGR2YUV", b"COLOR_RGBA2GRAY", b"rgb2gray", b""):
        assert L.scn_convert_color_code(bad) == -2  # SCN_E_UNSUPPORTED
    assert L.scn_convert_color_name(-1) is None
    # argument errors are caught before anything is launched
    assert L.scn_convert_color_u8(None, 1, 4, 4, 12, None, None) == -1
    assert L.scn_convert_color_u8(None, 0, 4, 4, 0, None, None) == 0
    assert L.scn_convert_color_nv12(None, None, 8, 1, 8, 8, 10, None, None) == -1  # GRAY2RGB of a decoded picture
    assert L.scn_convert_color_nv12(None, None, 8, 1, 7, 8, 0, None, None) == -1  # odd width


def test_unknown_code_is_named_by_the_binding():
    from scanner_b200 import kernels
    with pytest.raises(cabi.ScnError, match=r"'COLOR_RGB2Lab'.*COLOR_RGB2GRAY, COLOR_BGR2GRAY"):
        kernels.convert_color_code("COLOR_RGB2Lab")
    assert kernels.convert_color_code("COLOR_GRAY2BGR") == (11, 1, 3)


def test_client_encodes_conversion_as_per_stream_convert_color_args():
    import scanner_b200 as sp
    from scanner_b200 import protolite
    sc = sp.Client(gpus=[], cpu_instances=1)
    try:
        frames = sc.io.Input([sp.NamedVideoStream(sc, "a", frames=np.zeros((2, 4, 4, 3), np.uint8)),
                              sp.NamedVideoStream(sc, "b", frames=np.zeros((2, 4, 4, 3), np.uint8))])
        gray = sc.ops.ConvertColor(frame=frames, conversion=["COLOR_RGB2GRAY", "COLOR_BGR2HSV_FULL"])
        node = gray._op
        assert node.name == "ConvertColor" and node.args == b""
        msg = sc._op_protos["ConvertColor"]["stream"]
        assert node.per_stream == [protolite.encode(msg, {"conversion": "COLOR_RGB2GRAY"}),
                                   protolite.encode(msg, {"conversion": "COLOR_BGR2HSV_FULL"})]
        # field 1, length-delimited
        assert node.per_stream[0] == b"\x0a\x0eCOLOR_RGB2GRAY"
        with pytest.raises(sp.ScannerException, match="does not take argument"):
            sc.ops.ConvertColor(frame=frames, conversion="COLOR_RGB2GRAY")  # per-stream: a list
    finally:
        sc.stop()
