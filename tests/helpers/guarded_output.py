"""One call of an encoder entry point (scn_jpeg_encode_u8, scn_h264_encode_u8) into an output pre-filled with a byte
and followed by guard bytes of it, so that a byte the encoder never writes and a byte written past the end both
fail.  Shared by the JPEG and H.264 GPU tests."""
import ctypes

import torch

from scanner_b200 import cabi

GUARD = 4096
SENTINEL = 0xDEADBEEFDEADBEEF


def encode_raw(name, n, fill, call):
    """call(alloc_fn, sizes, stream) runs entry point `name` on n frames.  Checks that it asks for its output once,
    reports every frame's size, that the sizes sum to what it asked for and that the guard is untouched -> the n
    outputs as bytes."""
    out = {}

    def alloc(_ctx, nbytes):
        assert "n" not in out, "the output was asked for twice"
        out["n"] = int(nbytes)
        out["buf"] = torch.full((int(nbytes) + GUARD,), fill, dtype=torch.uint8, device="cuda")
        return out["buf"].data_ptr()

    sizes = (ctypes.c_size_t * n)(*[SENTINEL] * n)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    cabi.check(call(cabi.ALLOC_FN(alloc), sizes, stream), name)
    data = out["buf"].cpu().numpy()
    assert SENTINEL not in list(sizes)
    assert out["n"] == sum(sizes)
    assert (data[out["n"]:] == fill).all(), "bytes written past the end of the output"
    got, at = [], 0
    for s in sizes:
        got.append(data[at:at + s].tobytes())
        at += s
    return got
