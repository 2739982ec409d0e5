"""ctypes loader for oracle/_ref/libref_image.so -- the reference's own scanner/util/image.cu,
compiled unmodified by oracle/Makefile (`make -C oracle ref`).  TEST INFRASTRUCTURE ONLY: used by
oracle/make_golden_ref.py to record what the reference's kernel computes, the golden data that pins the
oracle and the CUDA kernels.  Needs a GPU; nothing under scanner_b200/ imports it.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libref_image.so")
# scanner::convertNV12toRGBA(const u8*, size_t, u8*, size_t, int, int, cudaStream_t)  (image.cu:229-239)
_SYM = "_ZN7scanner17convertNV12toRGBAEPKhmPhmiiP11CUstream_st"
_LIB = None


def available():
    return os.path.exists(SO)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(SO)
        fn = getattr(_LIB, _SYM)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int,
                       ctypes.c_void_p]
    return _LIB


def nv12_to_rgb(surface, width, height):
    """surface: CUDA uint8 tensor (height*3/2, pitch), luma rows then CbCr rows (the layout
    nvidia_video_decoder.cpp:284-296 hands to convertNV12toRGBA) -> (height, width, 3) uint8 CUDA tensor."""
    import torch
    assert surface.is_cuda and surface.dtype == torch.uint8 and surface.dim() == 2
    assert surface.shape[0] == height * 3 // 2 and surface.is_contiguous()
    out = torch.empty((height, width, 3), dtype=torch.uint8, device=surface.device)
    rc = getattr(lib(), _SYM)(surface.data_ptr(), surface.shape[1], out.data_ptr(), width * 3, width, height,
                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc != 0:
        raise RuntimeError(f"convertNV12toRGBA -> cudaError {rc}")
    return out
