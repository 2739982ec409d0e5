"""This repo's H.264 indexer (scanner_b200/csrc/engine/h264.cpp) against the reference's OWN index creator.

oracle/_ref/libref_h264_index.so is the reference's scanner/video/h264_byte_stream_index_creator.cpp compiled
UNMODIFIED (with the reference's scanner/util/h264.h SPS / PPS / slice-header parsers and is_new_access_unit) behind a
C shim.  The reference is fed what its demuxer would give it -- one packet per access unit, here the samples this
repo's indexer cut out of the stream -- and must count exactly one new frame per packet (a sample that held two access
units, or half of one, would not), name the same key pictures and the same sample sizes.  On a key picture the reference
additionally writes a copy of every SPS / PPS it has seen in front of the packet, each with the 3 bytes before and
after the NAL (:135-139, :193-214): sizes differ there by exactly that amount.
The reference's answers are replayed from tests/golden/ref_h264_index.json; where oracle/_ref is built,
`python tests/test_reference_h264_index_cpu.py` runs the library itself and records them again."""
import ctypes
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.recorded import Answers  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402
from scanner_b200 import synth_h264  # noqa: E402

REF_SO = os.path.join(ROOT, "oracle", "_ref", "libref_h264_index.so")
REF = Answers("ref_h264_index")


def nal_units(buf):
    """[(type, payload_len)] of an Annex-B buffer (start codes 00 00 01 / 00 00 00 01)."""
    out, i, n = [], 0, len(buf)
    starts = []
    while i + 3 <= n:
        if buf[i] == 0 and buf[i + 1] == 0 and buf[i + 2] == 1:
            starts.append(i + 3)
            i += 3
        else:
            i += 1
    for k, s in enumerate(starts):
        e = starts[k + 1] - 3 if k + 1 < len(starts) else n
        while e > s and buf[e - 1] == 0 and k + 1 < len(starts):
            e -= 1
        out.append((buf[s] & 0x1F, e - s))
    return out


def my_index(tmp_path, name, stream):
    import importlib.util                 # the descriptor classes built on the real protobuf runtime
    spec = importlib.util.spec_from_file_location("scn_test_storage", os.path.join(ROOT, "tests", "test_storage_cpu.py"))
    ts = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ts)
    db = E.Database(str(tmp_path / f"db_{name}"))
    db.ingest_h264(name, stream)
    vd = ts.parse_ref("VideoDescriptor", str(tmp_path / f"db_{name}" / "tables/0/1_0_video_metadata.bin"))
    data = open(str(tmp_path / f"db_{name}" / "tables/0/1_0.bin"), "rb").read()
    db.close()
    return data, list(vd.sample_offsets), list(vd.sample_sizes), list(vd.keyframe_indices)


def live_reference_index(data, offs, sizes):
    lib = ctypes.CDLL(REF_SO)
    n = len(offs)
    UL = ctypes.c_ulong
    so, ss, kf = (UL * (n + 8))(), (UL * (n + 8))(), (UL * (n + 8))()
    nf, nk, slen = ctypes.c_int(0), ctypes.c_int(0), UL(0)
    cap = 2 * len(data) + (1 << 20)
    out = (ctypes.c_ubyte * cap)()
    err = ctypes.create_string_buffer(256)
    buf = (ctypes.c_ubyte * len(data)).from_buffer_copy(data)
    rc = lib.ref_h264_index(buf, (UL * n)(*offs), (UL * n)(*sizes), n, so, ss, kf, n + 8, ctypes.byref(nf), ctypes.byref(nk),
                            out, UL(cap), ctypes.byref(slen), err, 256)
    assert rc == 0, err.value
    nfv, stream = nf.value, bytes(out[:slen.value])
    so, ss = list(so[:nfv]), list(ss[:nfv])
    # recorded: the demuxed stream's SHA-256 and the bytes the reference wrote in front of each sample
    inserted = [stream[so[i]:so[i] + max(0, ss[i] - sizes[i])] for i in range(nfv)]
    return [nfv, so, ss, list(kf[:nk.value]), hashlib.sha256(stream).hexdigest(), inserted]


def streams():
    rng = np.random.default_rng(5)
    h, w, n = 48, 64, 23
    for mode, gop in (("pcm", 4), ("skip", 5), ("bidir", 6)):
        k = n if mode != "skip" else (n + gop - 1) // gop
        yuv = rng.integers(0, 256, (k, h * w * 3 // 2), dtype=np.uint8)
        yield mode, E.h264_synth(yuv, w, h, gop=gop, non_key=mode, frames=n), n
    yield "cavlc", synth_h264.write(160, 96, 31, gop=7, seed=3)[0], 31


@pytest.mark.parametrize("case", list(streams()), ids=lambda c: c[0])
def test_indexer_agrees_with_the_reference_index_creator(tmp_path, case):
    name, stream, n = case
    data, offs, sizes, keys = my_index(tmp_path, name, stream)
    assert len(offs) == n
    frames, r_offs, r_sizes, r_keys, r_sha, inserted = REF(data, offs, sizes)
    # the reference's demuxed stream: what it wrote in front of each sample, then the sample (held by its SHA-256)
    r_stream = b"".join(inserted[i] + data[offs[i]:offs[i] + sizes[i]] for i in range(min(frames, n)))
    assert hashlib.sha256(r_stream).hexdigest() == r_sha
    assert frames == n                       # every sample is exactly one access unit for the reference's parser
    assert r_keys == keys                    # the same key pictures (IDR access units)
    # parameter sets the reference has seen so far, as it copies them: NAL + 3 bytes on each side
    extra_by_frame, seen = {}, {}
    for i in range(n):
        au = data[offs[i]:offs[i] + sizes[i]]
        for t, plen in nal_units(au):
            if t in (7, 8):
                seen[t] = plen + 6          # one SPS id and one PPS id in these streams: the latest copy replaces it
        if i in keys:
            extra_by_frame[i] = sum(seen.values())
    for i in range(n):
        assert r_sizes[i] == sizes[i] + extra_by_frame.get(i, 0), (name, i, r_sizes[i], sizes[i])
    assert r_offs[0] == 0 and all(r_offs[i + 1] == r_offs[i] + r_sizes[i] for i in range(n - 1))
    assert len(r_stream) == sum(r_sizes)
    # with the inserted copies taken out again the reference's demuxed stream is the stream this repo stores
    rebuilt = b"".join(r_stream[r_offs[i] + extra_by_frame.get(i, 0):r_offs[i] + r_sizes[i]] for i in range(n))
    assert rebuilt == data


if __name__ == "__main__":
    import pathlib
    import tempfile
    REF = Answers("ref_h264_index", live_reference_index)
    for c in streams():
        with tempfile.TemporaryDirectory() as d:
            test_indexer_agrees_with_the_reference_index_creator(pathlib.Path(d), c)
    REF.save()
    print("wrote", REF.path, len(REF.table), "answers")
