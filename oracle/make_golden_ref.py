#!/usr/bin/env python3
"""Golden vectors from the REFERENCE'S OWN kernel (oracle/_ref/libref_image.so = scanner/util/image.cu
compiled unmodified for sm_90a by `make -C oracle ref`).  Runs on a GPU where that library was built:

    python oracle/make_golden_ref.py tests/golden/nv12_ref.npz

Contents, all from scanner::convertNV12toRGBA:
  * c<i>_meta / c<i>_out (or c<i>_sha256 where the RGB24 output is large): the seeded surfaces of CASES
    (oracle/synth.py nv12_surface);
  * rand<seed>_sha256: the SHA-256 of its output on the surfaces of RAND_CASES (tests/test_ref_pin_gpu.py);
  * exhaustive_sha256: the SHA-256 of its output over the exhaustive input set synth.nv12_exhaustive (every
    (Y,Cb,Cr) triple on an even row + averaged-chroma odd rows).
The CPU suite (tests/test_oracle_golden.py) holds the oracle to them, the GPU suite (tests/test_ref_pin_gpu.py) the
product's kernels.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(300, 16, 32, 32), (301, 270, 480, 512), (302, 1080, 1920, 2048), (303, 34, 70, 128), (304, 2, 2, 64),
         (305, 18, 30, 32), (306, 64, 62, 64)]
RAND_CASES = [(1, 1080, 1920, 2048), (2, 270, 480, 512), (3, 34, 70, 128), (4, 2, 2, 64), (5, 18, 30, 32),
              (6, 1088, 1920, 1920)]
MAX_STORED_BYTES = 64 * 1024   # larger outputs are stored as their SHA-256


def main(dst):
    import torch

    from oracle import ref, synth

    def run(seed, h, w, pitch):
        luma, chroma = synth.nv12_surface(seed, h, w, pitch)
        surf = torch.from_numpy(np.concatenate([luma, chroma], 0)).cuda()
        return ref.nv12_to_rgb(surf, w, h).cpu().numpy()

    out = {}
    for i, case in enumerate(CASES):
        rgb = run(*case)
        out[f"c{i}_meta"] = np.array(case, np.int64)
        if rgb.nbytes <= MAX_STORED_BYTES:
            out[f"c{i}_out"] = rgb
        else:
            out[f"c{i}_sha256"] = np.frombuffer(hashlib.sha256(rgb.tobytes()).digest(), np.uint8)
    for case in RAND_CASES:
        out[f"rand{case[0]}_sha256"] = np.frombuffer(hashlib.sha256(run(*case).tobytes()).digest(), np.uint8)
    sha = hashlib.sha256()
    for f in range(synth.EXH_FRAMES):
        luma, chroma = synth.nv12_exhaustive(f)
        surf = torch.from_numpy(np.concatenate([luma, chroma], 0)).cuda()
        sha.update(ref.nv12_to_rgb(surf, synth.EXH_W, synth.EXH_H).cpu().numpy().tobytes())
    out["exhaustive_sha256"] = np.frombuffer(sha.digest(), np.uint8)
    out["provenance"] = np.array(
        f"scanner::convertNV12toRGBA from the reference's scanner/util/image.cu, nvcc default flags, sm_90a, "
        f"run on {torch.cuda.get_device_name(0)}")
    os.makedirs(os.path.dirname(os.path.abspath(dst)), exist_ok=True)
    np.savez_compressed(dst, **out)
    print("wrote", dst, sha.hexdigest())


if __name__ == "__main__":
    main(sys.argv[1])
