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


def convert_color_code(name):
    """OpenCV conversion name ('COLOR_RGB2GRAY', ...) -> (code, input channels, output channels)."""
    L = cabi.lib()
    code = L.scn_convert_color_code(name.encode())
    if code < 0:
        supported = []
        while L.scn_convert_color_name(len(supported)):
            supported.append(L.scn_convert_color_name(len(supported)).decode())
        raise cabi.ScnError(f"unsupported conversion {name!r}; supported: {', '.join(supported)}")
    cin, cout = ctypes.c_int(), ctypes.c_int()
    cabi.check(L.scn_convert_color_channels(code, ctypes.byref(cin), ctypes.byref(cout)), "scn_convert_color_channels")
    return code, cin.value, cout.value


def convert_color(frames, code, width=None, height=None):
    """cv2.cvtColor(frame, cv2.<code>) on the GPU, bit-exact.  `code` is the OpenCV name, e.g. 'COLOR_RGB2GRAY'.

    frames: (N,H,W,C) uint8 CUDA tensor -> (N,H,W,C_out); a list of (H,W,C) tensors, shapes may differ -> list
    (one launch per run of equal shape); or, with width and height, (N, H*3/2, pitch) NV12 surfaces (as
    nv12_to_rgb takes them) -> (N,H,W,C_out), converted from the RGB24 frame nv12_to_rgb would give."""
    cc, cin, cout = convert_color_code(code)
    L = cabi.lib()
    if width is not None:
        _need_cuda(frames)
        surfaces = frames.contiguous()
        n = surfaces.shape[0]
        lum, chr_, pitch = _surface_ptrs(surfaces, height)
        out = torch.empty((n, height, width, cout), dtype=torch.uint8, device=surfaces.device)
        lp, k1 = cabi.ptr_array(lum)
        cp, k2 = cabi.ptr_array(chr_)
        op, k3 = cabi.ptr_array([out.data_ptr() + i * height * width * cout for i in range(n)])
        cabi.check(L.scn_convert_color_nv12(lp, cp, pitch, n, width, height, cc, op, _stream()),
                   "scn_convert_color_nv12")
        return out
    def run(src_ptrs, h, w, c, device):
        """frames of one shape -> one (n,h,w,C_out) tensor; the frames need not be 16-byte aligned"""
        if c != cin:
            raise cabi.ScnError(f"{code} takes {cin}-channel frames, got {c} channels")
        out = torch.empty((len(src_ptrs), h, w, cout), dtype=torch.uint8, device=device)
        sp, k1 = cabi.ptr_array(src_ptrs)
        dp, k2 = cabi.ptr_array([out.data_ptr() + i * h * w * cout for i in range(len(src_ptrs))])
        cabi.check(L.scn_convert_color_u8(sp, len(src_ptrs), w, h, cc, dp, _stream()), "scn_convert_color_u8")
        return out

    if isinstance(frames, torch.Tensor):
        _need_cuda(frames)
        assert frames.dtype == torch.uint8 and frames.dim() == 4
        frames = frames.contiguous()
        n, h, w, c = frames.shape
        return run([frames.data_ptr() + i * h * w * c for i in range(n)], h, w, c, frames.device)
    lst = [t.contiguous() for t in frames]
    _need_cuda(*lst)
    for t in lst:
        assert t.dtype == torch.uint8 and t.dim() == 3
    outs = []
    i = 0
    while i < len(lst):
        j = i + 1
        while j < len(lst) and lst[j].shape == lst[i].shape:
            j += 1
        outs += list(run([t.data_ptr() for t in lst[i:j]], *lst[i].shape, lst[i].device))
        i = j
    return outs


def jpeg_encode_bound(width, height, channels=3):
    """Bytes no JPEG file of that geometry exceeds at any quality (scn_jpeg_encode_bound)."""
    return cabi.lib().scn_jpeg_encode_bound(width, height, channels)


def jpeg_encode(frames, quality=95):
    """Baseline JPEG files of uint8 frames, byte for byte cv2.imencode('.jpg', bgr, [cv2.IMWRITE_JPEG_QUALITY,
    quality]) with bgr the frame's channels reversed (frames are RGB) or the gray frame itself.

    frames: (N,H,W,C) uint8 CUDA tensor or a list of (H,W,C) tensors, shapes may differ (one call per run of
    equal shape); C is 3 or 1, and a frame need not be aligned.  -> list of N bytes objects.  Synchronises
    the current stream."""
    L = cabi.lib()

    def run(src_ptrs, h, w, c, device):
        keep = []

        def alloc(_ctx, nbytes):
            keep.append(torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device))
            return keep[-1].data_ptr()

        cb = cabi.ALLOC_FN(alloc)
        sizes = (ctypes.c_size_t * len(src_ptrs))()
        sp, k1 = cabi.ptr_array(src_ptrs)
        rc = L.scn_jpeg_encode_u8(sp, len(src_ptrs), w, h, c, int(quality), cb, None, sizes, _stream())
        cabi.check(rc, "scn_jpeg_encode_u8")
        data = keep[0].cpu().numpy().tobytes()  # on the current stream, after the files are written
        out, at = [], 0
        for s in sizes:
            out.append(data[at:at + s])
            at += s
        return out

    if isinstance(frames, torch.Tensor):
        _need_cuda(frames)
        assert frames.dtype == torch.uint8 and frames.dim() == 4
        frames = frames.contiguous()
        n, h, w, c = frames.shape
        if n == 0:
            return []
        return run([frames.data_ptr() + i * h * w * c for i in range(n)], h, w, c, frames.device)
    lst = [t.contiguous() for t in frames]
    _need_cuda(*lst)
    for t in lst:
        assert t.dtype == torch.uint8 and t.dim() == 3
    outs = []
    i = 0
    while i < len(lst):
        j = i + 1
        while j < len(lst) and lst[j].shape == lst[i].shape:
            j += 1
        outs += run([t.data_ptr() for t in lst[i:j]], *lst[i].shape, lst[i].device)
        i = j
    return outs


def h264_encode_bound(width, height):
    """Bytes no access unit of that geometry exceeds at any QP (scn_h264_encode_bound); 0 if it is refused."""
    return cabi.lib().scn_h264_encode_bound(width, height)


def h264_encode(frames, qp=23, keyframe_distance=120, positions=None):
    """Intra-only Baseline H.264 (CAVLC, constant QP) of RGB frames: one Annex-B access unit per frame, the bytes
    oracle/h264_enc.py writes.  Frame i is at position positions[i] of its item (default 0, 1, ...): an IDR picture
    with SPS and PPS when the position is a multiple of keyframe_distance, a non-IDR I picture otherwise, so the
    concatenated access units of one item are a stream any H.264 decoder plays.

    frames: (N,H,W,3) uint8 CUDA tensor or a list of (H,W,3) tensors of one shape; a frame need not be aligned.
    Width and height even, each side at most 4096 and at most 36,864 macroblocks; QP 0-51.  -> list of N bytes
    objects.  Synchronises the current stream."""
    if isinstance(frames, torch.Tensor):
        _need_cuda(frames)
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
            raise cabi.ScnError(f"h264_encode takes (N,H,W,3) uint8 frames, got {tuple(frames.shape)} {frames.dtype}")
        frames = frames.contiguous()
        n, h, w, _ = frames.shape
        ptrs = [frames.data_ptr() + i * h * w * 3 for i in range(n)]
        device = frames.device
    else:
        lst = [t.contiguous() for t in frames]
        _need_cuda(*lst)
        if any(t.dtype != torch.uint8 or t.dim() != 3 or t.shape != lst[0].shape or t.shape[2] != 3 for t in lst):
            raise cabi.ScnError("h264_encode takes (H,W,3) uint8 frames of one shape")
        n = len(lst)
        h, w = (lst[0].shape[0], lst[0].shape[1]) if n else (0, 0)
        ptrs = [t.data_ptr() for t in lst]
        device = lst[0].device if n else None
    if n == 0:
        return []
    if not 0 <= int(qp) <= 51:
        raise cabi.ScnError(f"h264_encode: QP {qp} is outside 0-51")
    if int(keyframe_distance) < 1:
        raise cabi.ScnError(f"h264_encode: keyframe_distance {keyframe_distance} is below 1")
    if w % 2 or h % 2:
        raise cabi.ScnError(f"h264_encode: {w}x{h} frames have an odd side (4:2:0 needs even sizes)")
    if h264_encode_bound(w, h) == 0:
        raise cabi.ScnError(f"h264_encode: {w}x{h} is beyond level 5.1 (a side over 4096 or over 36,864 macroblocks)")
    if positions is not None and len(positions) != n:
        raise cabi.ScnError(f"h264_encode: {len(positions)} positions for {n} frames")
    keep = []

    def alloc(_ctx, nbytes):
        keep.append(torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device))
        return keep[-1].data_ptr()

    cb = cabi.ALLOC_FN(alloc)
    sizes = (ctypes.c_size_t * n)()
    pos = None if positions is None else (ctypes.c_int * n)(*[int(p) for p in positions])
    sp, k1 = cabi.ptr_array(ptrs)
    rc = cabi.lib().scn_h264_encode_u8(sp, n, w, h, int(qp), pos, int(keyframe_distance), cb, None, sizes,
                                       _stream())
    cabi.check(rc, "scn_h264_encode_u8")
    data = keep[0].cpu().numpy().tobytes()  # on the current stream, after the access units are written
    out, at = [], 0
    for s in sizes:
        out.append(data[at:at + s])
        at += s
    return out


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


def tvl1_workspace_bytes(width, height, n):
    """Device scratch one scn_tvl1_u8 call of n pairs needs (reusable across calls on one stream)."""
    return cabi.lib().scn_tvl1_workspace_bytes(width, height, n)


def tvl1_flow(prev, next, tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300,
              scale_step=0.8, median_filtering=5, return_iterations=False, workspace=None):
    """TV-L1 dense flow of n pairs (scn_tvl1_u8; DESIGN.md "TV-L1"): (N,H,W) gray or (N,H,W,3) RGB uint8 CUDA
    tensors x2 -> (N,H,W,2) float32 (dx, dy).  RGB goes through convert_color(COLOR_RGB2GRAY) first.  epsilon <= 0
    runs every warp for all `iterations`.  With return_iterations, also an int32 numpy array [N][nscales][warps]
    of the iterations each (pair, level, warp) ran (level 0 = finest); the call then waits for the GPU."""
    _need_cuda(prev, next)
    grays = []
    for t in (prev, next):
        assert t.dtype == torch.uint8, t.dtype
        if t.dim() == 4 and t.shape[3] == 3:
            t = convert_color(t, "COLOR_RGB2GRAY")[..., 0]
        elif t.dim() == 4 and t.shape[3] == 1:
            t = t[..., 0]
        if t.dim() != 3:
            raise cabi.ScnError(f"tvl1_flow takes (N,H,W) gray or (N,H,W,3) RGB frames, got {tuple(t.shape)}")
        grays.append(t.contiguous())
    g0, g1 = grays
    if g0.shape != g1.shape:
        raise cabi.ScnError(f"tvl1_flow: prev {tuple(g0.shape)} and next {tuple(g1.shape)} differ")
    n, h, w = g0.shape
    out = torch.empty((n, h, w, 2), dtype=torch.float32, device=g0.device)
    need = tvl1_workspace_bytes(w, h, n)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(max(need, 1), dtype=torch.uint8, device=g0.device)
    pp, k1 = cabi.ptr_array([g0.data_ptr() + i * h * w for i in range(n)])
    np_, k2 = cabi.ptr_array([g1.data_ptr() + i * h * w for i in range(n)])
    op, k3 = cabi.ptr_array([out.data_ptr() + i * h * w * 8 for i in range(n)])
    iters = np.zeros((n, int(nscales), int(warps)), np.int32) if return_iterations else None
    ip = iters.ctypes.data_as(ctypes.POINTER(ctypes.c_int)) if return_iterations else None
    rc = cabi.lib().scn_tvl1_u8(pp, np_, n, w, h, op, tau, lambda_, theta, int(nscales), int(warps), epsilon,
                                int(iterations), scale_step, int(median_filtering), ip, workspace.data_ptr(),
                                workspace.numel(), _stream())
    cabi.check(rc, "scn_tvl1_u8")
    return (out, iters) if return_iterations else out
