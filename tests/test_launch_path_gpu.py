"""The host side every batched entry point shares (scn_common.cuh): batches go out in launches of at most 64 frames,
each launch picks its kernel from its own frames, a call validates its pointers before it enqueues anything, every
launch is profiled under the name of the kernel it launches, and raised shared-memory limits hold on every device."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from oracle import synth
from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu

SCN_E_BADARG = -1


def _ran(fn):
    """fn() and the {kernel: launches} it caused."""
    L = cabi.lib()
    L.scn_prof_enable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
        rep = cabi.prof_report()
    finally:
        L.scn_prof_enable(0)
    return out, {k: v["launches"] for k, v in rep.items()}


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_histogram_picks_the_kernel_per_launch():
    """130 frames as a pointer list, only frame 129 off 16-byte alignment: the first two launches of 64 frames keep
    the bit-sliced kernel, only the last one takes the generic kernel."""
    n, h, w = 130, 128, 128
    nbytes = h * w * 3                       # 8 warp blocks: the smallest frame hist16_csa_kernel takes
    g = torch.Generator(device="cuda").manual_seed(21)
    buf = torch.randint(0, 256, (n * nbytes + 16,), dtype=torch.uint8, device="cuda", generator=g)
    offs = [i * nbytes for i in range(n - 1)] + [(n - 1) * nbytes + 1]
    frames = [buf[o:o + nbytes].view(h, w, 3) for o in offs]
    got, ran = _ran(lambda: kernels.histogram(frames))
    assert ran == {"hist16_csa_kernel": 2, "hist16_generic_kernel": 1}, ran
    off = torch.arange(0, 48, 16, device="cuda")
    for i, f in enumerate(frames):
        want = torch.bincount(((f.reshape(-1, 3) >> 4).long() + off).flatten(), minlength=48).view(3, 16)
        assert (got[i].long() == want).all(), i


def test_frame_digest_rejects_a_misaligned_pointer_before_enqueueing():
    """A misaligned pointer at index 70 (the second launch's frames) fails the call before the first launch and
    before the output is cleared."""
    n, nbytes = 100, 64
    buf = torch.zeros((n + 1) * nbytes, dtype=torch.uint8, device="cuda")
    ptrs = [buf.data_ptr() + i * nbytes + (1 if i == 70 else 0) for i in range(n)]
    out = torch.full((n, 2), -1, dtype=torch.int64, device="cuda")
    pp, keep = cabi.ptr_array(ptrs)
    L = cabi.lib()
    torch.cuda.synchronize()
    before = L.scn_launch_count()
    assert L.scn_frame_digest(pp, n, nbytes, out.data_ptr(), _stream()) == SCN_E_BADARG
    torch.cuda.synchronize()
    assert L.scn_launch_count() == before
    assert (out == -1).all()


@pytest.mark.parametrize("h,w,pitch,kernel", [(32, 64, 64, "nv12_to_rgb16_kernel"), (30, 50, 52, "nv12_to_rgb_kernel")])
def test_nv12_to_rgb_is_profiled_under_its_kernel(h, w, pitch, kernel):
    n = 3
    surf = np.zeros((n, h * 3 // 2, pitch), np.uint8)
    for i in range(n):
        surf[i, :h], surf[i, h:] = synth.nv12_surface(50 + i, h, w, pitch)
    got, ran = _ran(lambda: kernels.nv12_to_rgb(torch.from_numpy(surf).cuda(), w, h))
    assert ran == {kernel: 1}, ran
    got = got.cpu().numpy()
    for i in range(n):
        assert (got[i] == oracle.nv12_to_rgb(surf[i, :h], surf[i, h:], w)).all(), i


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_raised_shared_memory_limits_hold_on_a_second_device():
    """nv12_stream_kernel (96 KiB of dynamic shared memory) and the fused Farneback kernels (up to 160 KiB) on cuda:1
    after cuda:0 in one process: function attributes belong to each device's context, so each device needs its own
    raised limit.  Same bits on both devices."""
    n, h, w, pitch = 4, 1080, 1920, 2048
    g = torch.Generator().manual_seed(31)
    surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, generator=g)
    a, b = synth.flow_pair(941, h, w, "shift")
    a, b = torch.from_numpy(a[None]), torch.from_numpy(b[None])
    outs = []
    for d in (0, 1):
        with torch.cuda.device(d):
            (hist, res), ran = _ran(lambda: kernels.nv12_hist_resize(surf.cuda(d), w, h, 224, 224))
            assert ran.get("nv12_stream_kernel") == 1, (d, ran)
            flow, ran = _ran(lambda: kernels.optical_flow(a.cuda(d), b.cuda(d)))
            assert "flow_gauss_fused_kernel" in ran and "flow_box_solve_f32_kernel" in ran, (d, ran)
            outs.append((hist.cpu(), res.cpu(), flow.cpu()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)
