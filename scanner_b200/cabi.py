"""ctypes binding of include/scn_kernels.h (libscn_kernels.so).

The library is built in-tree by `__graft_entry__.build()` / `make -C scanner_b200/csrc`.
If it is missing this module raises on first use -- there is no fallback implementation.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SCN_KERNELS_LIB: developer switch to load another build of the library (to time two builds side by side)
LIB_PATH = os.environ.get("SCN_KERNELS_LIB") or os.path.join(_HERE, "lib", "libscn_kernels.so")

_c = ctypes
_VP = _c.c_void_p
_PP = _c.POINTER(_c.c_void_p)
# scn_alloc_fn: (ctx, bytes) -> device pointer
ALLOC_FN = _c.CFUNCTYPE(_c.c_void_p, _c.c_void_p, _c.c_size_t)

# name -> (restype, argtypes); must list every symbol declared in include/scn_kernels.h
SIGNATURES = {
    "scn_abi_version": (_c.c_int, []),
    "scn_launch_count": (_c.c_uint64, []),
    "scn_prof_enable": (None, [_c.c_int]),
    "scn_prof_report": (_c.c_int, [_c.c_char_p, _c.c_size_t]),
    "scn_hist16_u8c3": (_c.c_int, [_PP, _c.c_int, _c.c_int, _c.c_int, _VP, _VP]),
    "scn_hist16_u8c3_strided": (_c.c_int, [_VP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _VP, _VP]),
    "scn_resize_target": (None, [_c.c_int] * 6 + [_c.POINTER(_c.c_int)] * 2),
    "scn_resize_plan_bytes": (_c.c_size_t, [_c.c_int, _c.c_int]),
    "scn_resize_plan_fill": (_c.c_int, [_c.c_int] * 4 + [_VP]),
    "scn_resize_bilinear_u8c3": (_c.c_int, [_PP, _c.c_int, _c.c_int, _c.c_int, _PP, _c.c_int, _c.c_int, _VP, _VP]),
    "scn_resize_bilinear_u8c3_strided": (_c.c_int, [_VP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _VP,
                                                    _c.c_size_t, _c.c_int, _c.c_int, _VP, _VP]),
    "scn_box_blur_u8c3": (_c.c_int, [_PP, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _PP, _VP]),
    "scn_box_blur_u8c3_strided": (_c.c_int, [_VP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _VP, _VP]),
    "scn_nv12_to_rgb24": (_c.c_int, [_PP, _PP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _PP, _c.c_size_t, _VP]),
    "scn_nv12_pack": (_c.c_int, [_PP, _PP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _PP, _VP]),
    "scn_farneback_workspace_bytes": (_c.c_size_t, [_c.c_int, _c.c_int]),
    "scn_farneback_u8c3": (_c.c_int, [_PP, _PP, _c.c_int, _c.c_int, _c.c_int, _PP, _c.c_int, _c.c_double, _c.c_int,
                                      _c.c_int, _c.c_int, _c.c_double, _VP, _c.c_size_t, _VP]),
    "scn_farneback_u8c3_chain": (_c.c_int, [_PP, _PP, _c.c_int, _c.c_int, _c.c_int, _PP, _c.c_int, _c.c_double,
                                            _c.c_int, _c.c_int, _c.c_int, _c.c_double, _VP, _c.c_size_t, _c.c_int,
                                            _c.POINTER(_c.c_int), _VP]),
    "scn_nv12_hist_resize": (_c.c_int, [_PP, _PP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _VP, _PP,
                                        _c.c_int, _c.c_int, _VP, _VP]),
    "scn_frame_digest": (_c.c_int, [_PP, _c.c_int, _c.c_size_t, _VP, _VP]),
    "scn_convert_color_code": (_c.c_int, [_c.c_char_p]),
    "scn_convert_color_name": (_c.c_char_p, [_c.c_int]),
    "scn_convert_color_channels": (_c.c_int, [_c.c_int, _c.POINTER(_c.c_int), _c.POINTER(_c.c_int)]),
    "scn_convert_color_u8": (_c.c_int, [_PP, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _PP, _VP]),
    "scn_convert_color_nv12": (_c.c_int, [_PP, _PP, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _PP,
                                          _VP]),
    "scn_jpeg_encode_bound": (_c.c_size_t, [_c.c_int, _c.c_int, _c.c_int]),
    "scn_jpeg_encode_u8": (_c.c_int, [_PP, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int, ALLOC_FN, _VP,
                                      _c.POINTER(_c.c_size_t), _VP]),
    "scn_h264_encode_bound": (_c.c_size_t, [_c.c_int, _c.c_int]),
    "scn_h264_encode_u8": (_c.c_int, [_PP, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.POINTER(_c.c_int), _c.c_int,
                                      ALLOC_FN, _VP, _c.POINTER(_c.c_size_t), _VP]),
    "scn_tvl1_workspace_bytes": (_c.c_size_t, [_c.c_int, _c.c_int, _c.c_int]),
    "scn_tvl1_u8": (_c.c_int, [_PP, _PP, _c.c_int, _c.c_int, _c.c_int, _PP, _c.c_float, _c.c_float, _c.c_float,
                               _c.c_int, _c.c_int, _c.c_float, _c.c_int, _c.c_float, _c.c_int, _c.POINTER(_c.c_int),
                               _VP, _c.c_size_t, _VP]),
}

_lib = None


class ScnError(RuntimeError):
    pass


def lib():
    """Load libscn_kernels.so; raise loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ScnError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a). scanner_b200 has no CPU fallback.")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)  # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        kind = "CUDA error" if rc > 0 else "argument error"
        raise ScnError(f"{what} failed: {kind} {rc}")


def ptr_array(ptrs):
    arr = (_c.c_void_p * len(ptrs))(*[int(p) for p in ptrs])
    return _c.cast(arr, _PP), arr  # keep `arr` alive while the call runs


def prof_report():
    """Per-kernel {name: {"launches": n, "ms": total}} recorded since scn_prof_enable(1)."""
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    n = lib().scn_prof_report(buf, len(buf))
    if n < 0:
        raise ScnError(f"scn_prof_report failed: {n}")
    return json.loads(buf.value.decode()) if n else {}
