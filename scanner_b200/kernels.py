"""Torch-tensor convenience wrappers over the C ABI (tests / bench / the Python op surface).

torch is used only for device memory and streams; every function below enqueues hand-written
sm_90a kernels from libscn_kernels.so on the current torch CUDA stream.
"""
import ctypes

import numpy as np
import torch

from . import cabi


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise cabi.ScnError("scanner_b200 kernels need CUDA tensors (no CPU fallback)")


def histogram(frames):
    """frames: (N,H,W,3) uint8 CUDA tensor (or list of (H,W,3) tensors) -> (N,3,16) int32."""
    lst = list(frames) if not isinstance(frames, torch.Tensor) else None
    if lst is None:
        _need_cuda(frames)
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        frames = frames.contiguous()
        n, h, w, _ = frames.shape
        out = torch.empty((n, 3, 16), dtype=torch.int32, device=frames.device)
        rc = cabi.lib().scn_hist16_u8c3_strided(frames.data_ptr(), h * w * 3, n, w, h, out.data_ptr(), _stream())
        cabi.check(rc, "scn_hist16_u8c3_strided")
        return out
    _need_cuda(*lst)
    n = len(lst)
    h, w, _ = lst[0].shape
    out = torch.empty((n, 3, 16), dtype=torch.int32, device=lst[0].device)
    pp, keep = cabi.ptr_array([t.data_ptr() for t in lst])
    rc = cabi.lib().scn_hist16_u8c3(pp, n, w, h, out.data_ptr(), _stream())
    cabi.check(rc, "scn_hist16_u8c3")
    return out


class ResizePlan:
    """Device copy of the coefficient table for one (src size, dst size) pair."""

    def __init__(self, src_w, src_h, dst_w, dst_h, device="cuda"):
        L = cabi.lib()
        nbytes = L.scn_resize_plan_bytes(dst_w, dst_h)
        host = np.zeros(nbytes, np.uint8)
        cabi.check(L.scn_resize_plan_fill(src_w, src_h, dst_w, dst_h, host.ctypes.data), "scn_resize_plan_fill")
        self.host = host
        self.dev = torch.from_numpy(host).to(device)
        self.key = (src_w, src_h, dst_w, dst_h)

    @property
    def ptr(self):
        return self.dev.data_ptr()


def resize_target(src_w, src_h, width=0, height=0, min=False, preserve_aspect=False):
    ow, oh = ctypes.c_int(), ctypes.c_int()
    cabi.lib().scn_resize_target(src_w, src_h, width, height, int(min), int(preserve_aspect),
                                 ctypes.byref(ow), ctypes.byref(oh))
    return ow.value, oh.value


def resize(frames, dst_w, dst_h, plan=None):
    """frames (N,H,W,3) uint8 CUDA -> (N,dst_h,dst_w,3) uint8, OpenCV INTER_LINEAR semantics."""
    _need_cuda(frames)
    frames = frames.contiguous()
    n, h, w, _ = frames.shape
    plan = plan or ResizePlan(w, h, dst_w, dst_h, frames.device)
    assert plan.key == (w, h, dst_w, dst_h)
    out = torch.empty((n, dst_h, dst_w, 3), dtype=torch.uint8, device=frames.device)
    rc = cabi.lib().scn_resize_bilinear_u8c3_strided(frames.data_ptr(), h * w * 3, n, w, h, out.data_ptr(),
                                                     dst_h * dst_w * 3, dst_w, dst_h, plan.ptr, _stream())
    cabi.check(rc, "scn_resize_bilinear_u8c3_strided")
    return out


def blur(frames, kernel_size):
    _need_cuda(frames)
    frames = frames.contiguous()
    n, h, w, _ = frames.shape
    out = torch.empty_like(frames)
    rc = cabi.lib().scn_box_blur_u8c3_strided(frames.data_ptr(), h * w * 3, n, w, h, int(kernel_size),
                                              out.data_ptr(), _stream())
    cabi.check(rc, "scn_box_blur_u8c3_strided")
    return out


def _surface_ptrs(surfaces, height):
    """surfaces: (N, H*3/2, pitch) uint8 CUDA tensor, NVDEC layout (luma rows then CbCr rows)."""
    n, rows, pitch = surfaces.shape
    assert rows == height * 3 // 2
    base = surfaces.data_ptr()
    stride = rows * pitch
    lum = [base + i * stride for i in range(n)]
    chr_ = [base + i * stride + height * pitch for i in range(n)]
    return lum, chr_, pitch


def nv12_to_rgb(surfaces, width, height):
    _need_cuda(surfaces)
    surfaces = surfaces.contiguous()
    n = surfaces.shape[0]
    lum, chr_, pitch = _surface_ptrs(surfaces, height)
    out = torch.empty((n, height, width, 3), dtype=torch.uint8, device=surfaces.device)
    lp, k1 = cabi.ptr_array(lum)
    cp, k2 = cabi.ptr_array(chr_)
    op, k3 = cabi.ptr_array([out.data_ptr() + i * height * width * 3 for i in range(n)])
    rc = cabi.lib().scn_nv12_to_rgb24(lp, cp, pitch, n, width, height, op, width * 3, _stream())
    cabi.check(rc, "scn_nv12_to_rgb24")
    return out


def nv12_pack(surfaces, width, height):
    """Pitched NVDEC-layout surfaces (N, H*3/2, pitch) -> packed NV12 frame elements (N, H*3/2, width)."""
    _need_cuda(surfaces)
    surfaces = surfaces.contiguous()
    n = surfaces.shape[0]
    lum, chr_, pitch = _surface_ptrs(surfaces, height)
    out = torch.empty((n, height * 3 // 2, width), dtype=torch.uint8, device=surfaces.device)
    lp, k1 = cabi.ptr_array(lum)
    cp, k2 = cabi.ptr_array(chr_)
    op, k3 = cabi.ptr_array([out.data_ptr() + i * (height * 3 // 2) * width for i in range(n)])
    cabi.check(cabi.lib().scn_nv12_pack(lp, cp, pitch, n, width, height, op, _stream()), "scn_nv12_pack")
    return out


def nv12_hist_resize(surfaces, width, height, dst_w, dst_h, plan=None, want_resize=True, want_hist=True):
    """Fused configs[1] DAG on NVDEC-layout surfaces -> (hist (N,3,16) i32, resized (N,dh,dw,3) u8)."""
    _need_cuda(surfaces)
    surfaces = surfaces.contiguous()
    n = surfaces.shape[0]
    lum, chr_, pitch = _surface_ptrs(surfaces, height)
    hist = torch.empty((n, 3, 16), dtype=torch.int32, device=surfaces.device) if want_hist else None
    lp, k1 = cabi.ptr_array(lum)
    cp, k2 = cabi.ptr_array(chr_)
    res = None
    op = None
    pptr = None
    if want_resize:
        plan = plan or ResizePlan(width, height, dst_w, dst_h, surfaces.device)
        res = torch.empty((n, dst_h, dst_w, 3), dtype=torch.uint8, device=surfaces.device)
        op, k3 = cabi.ptr_array([res.data_ptr() + i * dst_h * dst_w * 3 for i in range(n)])
        pptr = plan.ptr
    rc = cabi.lib().scn_nv12_hist_resize(lp, cp, pitch, n, width, height, hist.data_ptr() if want_hist else None,
                                         op, dst_w, dst_h, pptr, _stream())
    cabi.check(rc, "scn_nv12_hist_resize")
    return hist, res


def optical_flow_sequence(frames, workspace=None, pairs_per_call=None):
    """Flow of every consecutive pair of a clip: (N,H,W,3) uint8 -> (N-1,H,W,2) float32.  Every frame is expanded
    once (scn_farneback_u8c3_chain); pairs_per_call splits the clip over several calls on one workspace, the way
    the OpticalFlow op walks it."""
    _need_cuda(frames)
    frames = frames.contiguous()
    n, h, w, _ = frames.shape
    out = torch.empty((max(n - 1, 0), h, w, 2), dtype=torch.float32, device=frames.device)
    need = cabi.lib().scn_farneback_workspace_bytes(w, h)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=frames.device)
    fb = h * w * 3
    chain = ctypes.c_int(0)
    step = pairs_per_call or max(n - 1, 1)
    for p0 in range(0, n - 1, step):
        m = min(step, n - 1 - p0)
        pp, k1 = cabi.ptr_array([frames.data_ptr() + (p0 + i) * fb for i in range(m)])
        np_, k2 = cabi.ptr_array([frames.data_ptr() + (p0 + i + 1) * fb for i in range(m)])
        op, k3 = cabi.ptr_array([out.data_ptr() + (p0 + i) * h * w * 8 for i in range(m)])
        rc = cabi.lib().scn_farneback_u8c3_chain(pp, np_, m, w, h, op, 3, 0.5, 15, 3, 5, 1.2, workspace.data_ptr(),
                                                 workspace.numel(), 1, ctypes.byref(chain), _stream())
        cabi.check(rc, "scn_farneback_u8c3_chain")
    return out


def optical_flow(prev_frames, next_frames, num_levels=3, pyr_scale=0.5, win_size=15, num_iters=3, poly_n=5,
                 poly_sigma=1.2, workspace=None):
    """Farneback flow of n frame pairs: (N,H,W,3) uint8 x2 -> (N,H,W,2) float32 (reference OpticalFlow op)."""
    _need_cuda(prev_frames, next_frames)
    prev_frames, next_frames = prev_frames.contiguous(), next_frames.contiguous()
    n, h, w, _ = prev_frames.shape
    out = torch.empty((n, h, w, 2), dtype=torch.float32, device=prev_frames.device)
    need = cabi.lib().scn_farneback_workspace_bytes(w, h)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=prev_frames.device)
    fb = h * w * 3
    pp, k1 = cabi.ptr_array([prev_frames.data_ptr() + i * fb for i in range(n)])
    np_, k2 = cabi.ptr_array([next_frames.data_ptr() + i * fb for i in range(n)])
    op, k3 = cabi.ptr_array([out.data_ptr() + i * h * w * 8 for i in range(n)])
    rc = cabi.lib().scn_farneback_u8c3(pp, np_, n, w, h, op, num_levels, pyr_scale, win_size, num_iters, poly_n,
                                       poly_sigma, workspace.data_ptr(), workspace.numel(), _stream())
    cabi.check(rc, "scn_farneback_u8c3")
    return out


def frame_digest(frames):
    """frames: (N, ...) contiguous CUDA tensor -> (N, 2) uint64-as-int64 fingerprints (scn_frame_digest)."""
    _need_cuda(frames)
    frames = frames.contiguous()
    n = frames.shape[0]
    nbytes = frames[0].numel() * frames.element_size()
    out = torch.empty((n, 2), dtype=torch.int64, device=frames.device)
    pp, keep = cabi.ptr_array([frames.data_ptr() + i * nbytes for i in range(n)])
    cabi.check(cabi.lib().scn_frame_digest(pp, n, nbytes, out.data_ptr(), _stream()), "scn_frame_digest")
    return out
