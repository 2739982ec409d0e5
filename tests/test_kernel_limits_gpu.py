"""The histogram kernels at the limits of their bit-sliced counters, and every batched entry point over 64 frames.

Both large-frame histogram kernels count with carry-save counters of 10 bit planes (at most 1023) and flush them
before they can wrap: hist16_csa_kernel every 63 warp blocks (63 x 16 = 1008), nv12_stream_kernel every 127 steps
(127 x 8 = 1016).  Bin 15 is never counted directly but recovered from the total.  Uniform random frames bring a
counter to about 1/16 of its ceiling; a frame whose pixels all fall in one bin (black frames, letterbox bars, title
cards) brings it to the ceiling.  So the tests below run constant, saturating and letterboxed frames through launches
in which every warp's range is longer than the flush limit (each test first asserts that, from the launch formulas),
at the streaming kernel's edge geometries, and batches that the launchers split into launches of 64 pointers.

Every comparison is exact: histograms against torch.bincount of v >> 4 (of kernels.nv12_to_rgb for NV12 surfaces,
pinned to the reference's own kernel by test_ref_pin_gpu.py) or the closed form of a constant frame, Resize against
kernels.resize of that RGB (pinned to the cv2 goldens) and the oracle on a sample."""
import numpy as np
import pytest
import torch

import oracle
from oracle import synth
from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu

MAX_PTRS = 64                          # SCN_MAX_PTRS: frames per launch
CSA_BLOCK, CSA_WARPS, CSA_MAX_BLOCKS = 6144, 8, 63   # hist_csa.cuh: kWarpBlock, kWarps, kMaxBlocks
NVS_WARPS, NVS_MAX_STEPS = 12, 127                   # nv12_stream.cuh: kWarps, kMaxSteps
BLACK, WHITE, PAD = (16, 128, 128), (255, 128, 128), (0, 0, 0)   # PAD: what the padding lanes of a last step hold


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count   # what the library's sm_count() reads


def _warp_ranges(total, per_frame, nwarps):
    """(range length, longest run inside one frame) of every warp: both kernels give warp g the global range
    [total * g / nwarps, total * (g + 1) / nwarps) and flush at least at every frame boundary."""
    out = []
    for g in range(nwarps):
        b, e = total * g // nwarps, total * (g + 1) // nwarps
        n, longest = e - b, 0
        while b < e:
            stop = min(e, (b // per_frame + 1) * per_frame)
            longest, b = max(longest, stop - b), stop
        out.append((n, longest))
    return out


def _assert_spans_exceed(what, n, per_frame, per_cta, warps, limit):
    """Premise of a flush-limit test: in every launch every warp's range is longer than `limit`, and some warp runs
    longer than `limit` inside one frame, so the kernel must split it into several flushes."""
    sm = _sm_count()
    for i0 in range(0, n, MAX_PTRS):
        total = min(MAX_PTRS, n - i0) * per_frame
        ctas = max(1, min(-(-total // per_cta), sm))
        r = _warp_ranges(total, per_frame, ctas * warps)
        shortest, longest = min(x for x, _ in r), max(y for _, y in r)
        assert shortest > limit and longest > limit, (
            f"{what}: on {sm} SMs the per-warp ranges are {shortest}.. (longest run in a frame {longest}), "
            f"no longer above the flush limit {limit}: the launch heuristics changed and this test lost its coverage")


def _csa_premise(n, nbytes):
    # csa::launch in hist_csa.cuh: blocks_per_frame = nbytes / kWarpBlock, ctas = ceil(total / (kWarps * 4)) capped
    # at sm_count(); hist16_csa_kernel splits total_blocks evenly over the warps
    assert nbytes >= 8 * CSA_BLOCK
    _assert_spans_exceed("hist16_csa_kernel", n, nbytes // CSA_BLOCK, CSA_WARPS * 4, CSA_WARPS, CSA_MAX_BLOCKS)


def _nvs_premise(n, h, w, pitch):
    # nvs::eligible and nvs::launch in nv12_stream.cuh: steps_per_frame = ceil(width / 16 * height / 2 / 32),
    # ctas = ceil(total / (kWarps * 8)) capped at sm_count()
    assert w % 16 == 0 and pitch % 16 == 0 and h % 2 == 0 and w * h >= 64 * 1024
    spf = -(-(w // 16 * (h // 2)) // 32)
    _assert_spans_exceed("nv12_stream_kernel", n, spf, NVS_WARPS * 8, NVS_WARPS, NVS_MAX_STEPS)


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


# ----------------------------------------------------------------------------- references
def _rgb_hist(frames):
    """(N,H,W,3) u8 CUDA -> (N,3,16) int64: bincount of v >> 4 per channel, one frame at a time."""
    off = torch.arange(0, 48, 16, device=frames.device)
    return torch.stack([torch.bincount(((f.reshape(-1, 3) >> 4).long() + off).flatten(), minlength=48).view(3, 16)
                        for f in frames])


def _nv12_refs(surf, w, h, dw=0, dh=0, chunk=4):
    """Histogram (and Resize) of NV12 surfaces through the RGB frame, a few surfaces at a time."""
    hs, rs = [], []
    for i in range(0, surf.shape[0], chunk):
        rgb = kernels.nv12_to_rgb(surf[i:i + chunk], w, h)
        hs.append(_rgb_hist(rgb))
        if dw:
            rs.append(kernels.resize(rgb, dw, dh))
        del rgb
    return torch.cat(hs), (torch.cat(rs) if dw else None)


def _bins_of(triples):
    """(R, G, B) >> 4 of every (Y, Cb, Cr) triple: the oracle on a 2 x 2 surface per triple."""
    t = np.asarray(triples, np.uint8).reshape(-1, 3)
    luma = np.repeat(np.repeat(t[:, 0], 2)[None], 2, axis=0)
    chroma = t[:, 1:].reshape(1, -1)
    rgb = oracle.nv12_to_rgb(luma, chroma)
    assert (rgb[0] == rgb[1]).all() and (rgb[:, 0::2] == rgb[:, 1::2]).all()
    return rgb[0, 0::2] >> 4


def _covering_triples(seed):
    """Black, white, the padding colour, then seeded random triples picked greedily until every bin of every
    channel is hit by one of them."""
    pool = np.random.default_rng(seed).integers(0, 256, (4096, 3))
    hit = np.zeros((len(pool), 48), bool)
    hit[np.arange(len(pool))[:, None], _bins_of(pool) + np.arange(0, 48, 16)] = True
    chosen = [BLACK, WHITE, PAD]
    covered = np.zeros(48, bool)
    covered[(_bins_of(chosen) + np.arange(0, 48, 16)).ravel()] = True
    while not covered.all():
        gain = (hit & ~covered).sum(1)
        i = int(gain.argmax())
        assert gain[i] > 0
        chosen.append(tuple(int(x) for x in pool[i]))
        covered |= hit[i]
    assert (_bins_of([WHITE]) == 15).all()   # white puts all three channels in bin 15
    return chosen


def _fill_constant(surf, triples, h, w):
    """Surfaces i of a (N, H*3/2, pitch) batch become the constant triples[i] over the width (bytes past it kept)."""
    t = torch.tensor(triples, dtype=torch.uint8, device=surf.device)[:, :, None, None]
    surf[:, :h, :w] = t[:, 0]
    c = surf[:, h:, :w].unflatten(2, (w // 2, 2))
    c[..., 0] = t[:, 1]
    c[..., 1] = t[:, 2]


def _letterbox(surf, h, w):
    """Black bars over the top and bottom 13 % (even rows, so whole chroma rows), the content between kept."""
    bar = h * 13 // 100 & ~1
    surf[:, :bar, :w] = 16
    surf[:, h - bar:h, :w] = 16
    surf[:, h:h + bar // 2, :w] = 128
    surf[:, h + (h - bar) // 2:, :w] = 128


def _batch(n, h, w, pitch, seed):
    """Constant surfaces covering every bin (only black, white, the padding colour when n is small), two
    letterboxed ones, the rest uniform random; bytes past the width random too."""
    triples = _covering_triples(seed) if n >= 32 else [BLACK, WHITE, PAD]
    assert len(triples) + 2 <= n
    g = torch.Generator(device="cuda").manual_seed(seed)
    surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
    _fill_constant(surf[:len(triples)], triples, h, w)
    _letterbox(surf[len(triples):len(triples) + 2], h, w)
    return surf, triples


def _hist_resize(surf, w, h, dw=0, dh=0, fill=0, want_hist=True):
    """scn_nv12_hist_resize on (N, H*3/2, pitch) surfaces, the Resize output filled with `fill` beforehand."""
    n, _, pitch = surf.shape
    lum, chr_, _ = kernels._surface_ptrs(surf, h)
    lp, k1 = cabi.ptr_array(lum)
    cp, k2 = cabi.ptr_array(chr_)
    hist = torch.full((n, 3, 16), -1, dtype=torch.int32, device="cuda") if want_hist else None
    res = op = plan = None
    if dw:
        plan = kernels.ResizePlan(w, h, dw, dh)
        res = torch.full((n, dh, dw, 3), fill, dtype=torch.uint8, device="cuda")
        op, k3 = cabi.ptr_array([res.data_ptr() + i * dh * dw * 3 for i in range(n)])
    rc = cabi.lib().scn_nv12_hist_resize(lp, cp, pitch, n, w, h, hist.data_ptr() if want_hist else None, op, dw, dh,
                                         plan.ptr if plan else None, kernels._stream())
    cabi.check(rc, "scn_nv12_hist_resize")
    torch.cuda.synchronize()
    return hist, res


def _check_nv12(surf, w, h, dw, dh, triples=(), oracle_frames=(0,)):
    """Histogram + Resize, Histogram alone and Resize alone (each Resize twice, over outputs filled with 0 and
    with 255, so a byte the call does not write cannot match) against the references."""
    want_h, want_r = _nv12_refs(surf, w, h, dw, dh)
    for i, t in enumerate(triples):   # constant surfaces: all W*H pixels in the bins of the triple
        closed = np.zeros((3, 16), np.int64)
        closed[np.arange(3), _bins_of([t])[0]] = w * h
        assert (want_h[i].cpu().numpy() == closed).all(), t
    for fill in (0, 255):
        got_h, got_r = _hist_resize(surf, w, h, dw, dh, fill)
        bad = (got_h.long() != want_h).flatten(1).any(1).nonzero().flatten().tolist()
        assert not bad, ("histogram", fill, bad[:8])
        bad = (got_r != want_r).flatten(1).any(1).nonzero().flatten().tolist()
        assert not bad, ("resize", fill, bad[:8])
        _, got_r = _hist_resize(surf, w, h, dw, dh, fill, want_hist=False)
        assert (got_r == want_r).all(), ("resize alone", fill)
    got_h, _ = _hist_resize(surf, w, h)
    assert (got_h.long() == want_h).all(), "histogram alone"
    for i in oracle_frames:
        rgb = kernels.nv12_to_rgb(surf[i:i + 1], w, h)[0].cpu().numpy()
        assert (want_r[i].cpu().numpy() == oracle.resize(rgb, dw, dh)).all(), ("oracle resize", i)


# --------------------------------------------------------------------- B. hist16_csa_kernel at its flush limit
_CSA_VALUES = [16 * b + o for b in range(16) for o in (0, 7, 15)]   # every bin; 0x7F / 0x80 (A / B word), 0xF0, 0xFF


def test_hist_csa_saturating_frames_across_the_flush_limit():
    """64 x 3000 x 2000 RGB (177 blocks per warp on 132 SMs, a 4224-byte tail per frame): frames 0-47 constant per
    channel (each channel through every value of _CSA_VALUES), an all-0xFF frame (every A counter saturates), a frame
    whose bytes depend only on offset mod 512 (every lane reads the same 16 bytes every round: all lanes saturate
    at once, on different bins), a letterboxed frame and random ones; pointer list (permuted) and strided."""
    n, h, w = 64, 2000, 3000
    nbytes = h * w * 3
    assert nbytes % CSA_BLOCK == 4224
    _csa_premise(n, nbytes)
    g = torch.Generator(device="cuda").manual_seed(11)
    frames = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    vals = torch.tensor([[_CSA_VALUES[(i + 5 * c) % 48] for c in range(3)] for i in range(48)], dtype=torch.uint8)
    frames[:48] = vals.cuda()[:, None, None, :]
    frames[48] = 255
    lut = torch.tensor([(97 * k + 13) % 256 for k in range(512)], dtype=torch.uint8, device="cuda")
    frames[49].view(-1)[:] = lut[torch.arange(nbytes, device="cuda") % 512]
    bar = h * 13 // 100
    frames[50, :bar] = 0
    frames[50, h - bar:] = 0
    want = _rgb_hist(frames)
    for i in range(48):
        closed = torch.zeros((3, 16), dtype=torch.int64)
        closed[torch.arange(3), vals[i].long() >> 4] = w * h
        assert (want[i].cpu() == closed).all()
    assert (want[48, :, 15] == w * h).all()
    got, ran = _ran(lambda: kernels.histogram(frames))
    assert ran == {"hist16_csa_kernel": 1}
    bad = (got.long() != want).flatten(1).any(1).nonzero().flatten().tolist()
    assert not bad, ("strided", bad)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(3)).tolist()
    got = kernels.histogram([frames[i] for i in perm])
    bad = (got.long() != want[perm]).flatten(1).any(1).nonzero().flatten().tolist()
    assert not bad, ("pointer list", bad)


@pytest.mark.parametrize("h,w,kernel", [(128, 128, "hist16_csa_kernel"), (127, 129, "hist16_generic_kernel")])
def test_hist_constant_frames_at_the_csa_eligibility_edge(h, w, kernel):
    """49152 bytes (8 warp blocks) is the smallest frame the bit-sliced kernel takes; 49149 goes to the generic one."""
    frames = np.empty((18, h, w, 3), np.uint8)
    for i in range(16):
        frames[i] = [_CSA_VALUES[(3 * i + 16 * c) % 48] for c in range(3)]
    frames[16] = 255
    frames[17] = np.resize(np.arange(512, dtype=np.uint8) * 97 + 13, h * w * 3).reshape(h, w, 3)
    for got, ran in (_ran(lambda: kernels.histogram(torch.from_numpy(frames).cuda())),
                     _ran(lambda: kernels.histogram(list(torch.from_numpy(frames).cuda())))):
        assert ran == {kernel: 1}
        got = got.cpu().numpy()
        for i in range(len(frames)):
            assert (got[i] == oracle.hist16(frames[i])).all(), i


# --------------------------------------------------------------- C. nv12_stream_kernel at its limits and edges
LIMIT_CASES = {               # (n, h, w, pitch, dw, dh)
    "4k": (64, 2160, 3840, 4096, 224, 224),       # ~327 steps per warp, flushes that cross frames
    "padded": (64, 2160, 3824, 3840, 224, 224),   # 24 padding lanes in every frame's last step
    "narrow": (64, 8190, 496, 512, 224, 224),     # 31 units per row: the row-wrap loop, 31 padding lanes
}
RESIZE_CASES = dict(LIMIT_CASES, **{
    "upscale": (8, 128, 1024, 1024, 1500, 700),   # dh > h: many destination rows share tap row 0
    "ragged": (8, 1080, 1920, 2048, 301, 157),
})


@pytest.mark.parametrize("name", list(RESIZE_CASES))
def test_nv12_stream_saturating_surfaces(name):
    n, h, w, pitch, dw, dh = RESIZE_CASES[name]
    if name in LIMIT_CASES:
        _nvs_premise(n, h, w, pitch)
    surf, triples = _batch(n, h, w, pitch, seed=sum(map(ord, name)))
    _check_nv12(surf, w, h, dw, dh, triples, oracle_frames=(1, n - 1))


@pytest.mark.parametrize("h,w,pitch,n,kernel", [(4096, 16, 16, 64, "nv12_stream_kernel"),
                                                (4096, 16, 48, 8, "nv12_stream_kernel"),
                                                (2048, 48, 64, 48, "nv12_stream_kernel"),
                                                (4094, 16, 16, 8, "nv12_hist_kernel")])
def test_nv12_stream_narrowest_surfaces(h, w, pitch, n, kernel):
    """1 and 3 units per row (a step wraps 32 or 10 row pairs); 16 x 4096 is exactly the 64 K-pixel eligibility edge,
    16 x 4094 goes to nv12_hist_kernel."""
    surf, triples = _batch(n, h, w, pitch, seed=h + w + pitch)
    got, ran = _ran(lambda: _hist_resize(surf, w, h)[0])
    assert kernel in ran and ran[kernel] == 1, ran
    _check_nv12(surf, w, h, 12, 300, triples)


# ------------------------------------------------------------------------------- D. batches over 64 frames
def _distinct_surfaces(n, h, w, pitch, seed):
    """Random surfaces, every 37th letterboxed: every surface's histogram differs from every other's."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
    _letterbox(surf[::37], h, w)
    return surf


def test_nv12_hist_resize_bench_shape_over_64_surfaces():
    """130 x 1080p, pitch 2048, Histogram + Resize 224 x 224: three streaming launches and three Resize launches."""
    n, h, w, pitch = 130, 1080, 1920, 2048
    surf = _distinct_surfaces(n, h, w, pitch, 5)
    _, ran = _ran(lambda: _hist_resize(surf, w, h, 224, 224))
    assert ran.get("nv12_stream_kernel") == 3, ran
    _check_nv12(surf, w, h, 224, 224, oracle_frames=(63, 64, 129))


@pytest.mark.parametrize("n,h,w,pitch", [(70, 34, 46, 51), (70, 480, 640, 640)])
def test_nv12_hist_and_area_resize_over_64_surfaces(n, h, w, pitch):
    """The exact-2x Resize (INTER_AREA) over 64 surfaces: ragged ones (generic nv12_hist_kernel) and streamed ones."""
    surf = _distinct_surfaces(n, h, w, pitch, 6)
    host = surf.cpu().numpy()
    for fill in (0, 255):
        got_h, got_r = _hist_resize(surf, w, h, w // 2, h // 2, fill)
        got_h, got_r = got_h.cpu().numpy(), got_r.cpu().numpy()
        for i in range(n):
            rgb = oracle.nv12_to_rgb(host[i, :h], host[i, h:], w)
            assert (got_h[i] == oracle.hist16(rgb)).all(), (fill, i)
            assert (got_r[i] == oracle.resize(rgb, w // 2, h // 2)).all(), (fill, i)


def test_histogram_pointer_list_and_strided_over_64_frames():
    n, h, w = 130, 480, 640
    g = torch.Generator(device="cuda").manual_seed(8)
    frames = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    frames[::37, : h // 3] = 0
    want = _rgb_hist(frames)
    got = kernels.histogram(frames)
    assert (got.long() == want).all(), (got.long() != want).flatten(1).any(1).nonzero().flatten().tolist()
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(4)).tolist()
    got, ran = _ran(lambda: kernels.histogram([frames[i] for i in perm]))
    assert ran == {"hist16_csa_kernel": 3}
    assert (got.long() == want[perm]).all(), (got.long() != want[perm]).flatten(1).any(1).nonzero().flatten().tolist()


def test_small_frame_ops_over_64_frames():
    """Resize, Blur, NV12 -> RGB and the NV12 pack, 70 frames each (two launches)."""
    n = 70
    frames = np.stack([synth.rand_frame(300 + i, 37, 53) for i in range(n)])
    aligned = np.stack([synth.rand_frame(400 + i, 40, 64) for i in range(n)])
    res = kernels.resize(torch.from_numpy(frames).cuda(), 30, 20).cpu().numpy()
    bl = kernels.blur(torch.from_numpy(frames).cuda(), 3).cpu().numpy()
    bl2 = kernels.blur(torch.from_numpy(aligned).cuda(), 5).cpu().numpy()
    for i in range(n):
        assert (res[i] == oracle.resize(frames[i], 30, 20)).all(), i
        assert (bl[i] == oracle.blur(frames[i], 3)).all(), i
        assert (bl2[i] == oracle.blur(aligned[i], 5)).all(), i
    h, w, pitch = 30, 50, 64
    surf = _distinct_surfaces(n, h, w, pitch, 7)
    host = surf.cpu().numpy()
    rgb = kernels.nv12_to_rgb(surf, w, h).cpu().numpy()
    packed = kernels.nv12_pack(surf, w, h).cpu().numpy()
    assert (packed == host[:, :, :w]).all()
    for i in range(n):
        assert (rgb[i] == oracle.nv12_to_rgb(host[i, :h], host[i, h:], w)).all(), i

