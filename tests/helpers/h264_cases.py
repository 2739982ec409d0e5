"""H.264 inputs shared by the GPU tests of h264_enc.cu (test_h264_ffmpeg_gpu.py, test_h264_encode_gpu.py).  Plain
data: importing it loads no GPU library."""
import numpy as np

# 512 x 256 noise at QP 0 from these seeds, found by searching seeds 0-399 with the oracle: seed 25 puts a zero
# pair across a lane boundary (at 58735) and across a chunk boundary (at 204799), seed 88 starts one exactly at a
# chunk (at 28672).  The payload offsets are where the kernel's passes see them: its slice RBSP starts 16-aligned.
EPB_SEEDS = (25, 88)


def epb_seam_frames():
    """(2, 256, 512, 3) uint8: the frames of EPB_SEEDS, to be coded at QP 0"""
    return np.stack([np.random.default_rng(s).integers(0, 256, (256, 512, 3), dtype=np.uint8) for s in EPB_SEEDS])
