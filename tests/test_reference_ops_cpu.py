"""The reference's OWN op library inside this engine.

oracle/_ref/libref_test_ops.so is the reference's tests/test_ops.cpp compiled UNMODIFIED against this repo's plugin
headers (oracle/Makefile; the cv:: calls of its Histogram / Resize / OpticalFlow kernels are stubs that abort -- there
is no OpenCV C++ here).  Two things follow from loading it with scn_load_op_library:
  * the drop-in boundary is real: the reference's REGISTER_OP / REGISTER_KERNEL source registers and runs here;
  * the kernels whose arithmetic is written out in that file are the reference itself: its Blur pins oracle.blur (and
    with it every GPU blur kernel, which the -m gpu tests hold to the oracle), its TestIncrement* ops give the values
    this repo's test ops must reproduce under the engine's bounded-state warm-up and unbounded-state semantics.
What the reference's ops computed is replayed from tests/golden/ref_test_ops.json; where oracle/_ref is built,
`python tests/test_reference_ops_cpu.py` checks that the library registers through the plugin headers, runs its ops
again and records what they computed.  The library registers the names Histogram / Resize / Blur / ... too, so every
engine run happens in its own process."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle  # noqa: E402
from oracle import synth  # noqa: E402
from oracle.recorded import Answers  # noqa: E402

REF_SO = os.path.join(ROOT, "oracle", "_ref", "libref_test_ops.so")
TEST_OPS_SO = os.path.join(ROOT, "build", "tests", "libtest_plugin_ops.so")
# (k, h, w, frames): every kernel size on a frame a few pixels larger than the window, and frames whose interior is
# empty (a side shorter than the window, one row, one column) or a single pixel (both sides equal to the window)
BLUR_CASES = ([(3, 37, 53, 3), (4, 40, 31, 2), (5, 64, 48, 2), (8, 33, 47, 1), (15, 40, 56, 1)] +
              [(k, k + 5, 2 * k + 3, 1) for k in range(1, 32)] +
              [(k, k, k, 1) for k in (1, 2, 3, 4, 16, 30, 31)] +
              [(k, k - 1, 40, 1) for k in (2, 3, 17, 31)] + [(k, 40, k - 1, 1) for k in (2, 4, 31)] +
              [(k, 1, 37, 1) for k in (2, 3, 31)] + [(k, 37, 1, 1) for k in (2, 5, 31)])

PRELUDE = r'''
import hashlib, json, os, struct, sys
import numpy as np
sys.path.insert(0, os.environ["SCN_ROOT"])
import oracle
from oracle import synth
from scanner_b200 import engine as E, protolite
E.load_op_library(os.environ["SCN_OPS_LIB"])
REF_ARGS = protolite.parse_proto("message BlurArgs { int32 kernel_size = 1; float sigma = 2; }")
'''

# reference tests/test_ops.cpp:239-310 (BlurKernel, CPU) run by this engine, on the region the reference writes (it
# leaves the border of its new frame uninitialised): {"k,h,w,n": [SHA-256 of the interior bytes of frame i, ...]}
BLUR_BODY = r'''
out = {}
for (k, h, w, n) in %r:
    frames = np.stack([synth.rand_frame(900 + 7 * k + i, h, w) for i in range(n)])
    eng = E.Engine(gpus=[], cpu_instances=2)
    g = E.Graph(); src = g.add_source(True)
    bl = g.add_op("Blur", [(src, "frame")], device=0,
                  args=protolite.encode(REF_ARGS["BlurArgs"], {"kernel_size": k, "sigma": 0.5}))
    sink = g.add_sink((bl, "frame"))
    j = E.Job(); j.bind_source(src, eng.add_raw_frames(frames))
    eng.run(g, [j], 2, 4)
    ys, xs = oracle.blur_interior(h, w, k)
    rows = []
    for i in range(n):
        got = j.output_row(sink, i)
        assert got.shape == (h, w, 3)
        rows.append(hashlib.sha256(np.ascontiguousarray(got[ys, xs]).tobytes()).hexdigest())
    out["%%d,%%d,%%d,%%d" %% (k, h, w, n)] = rows
    eng.close()
print("REF_JSON" + json.dumps(out))
''' % (BLUR_CASES,)

# py_test.py:407-423 (bounded state, warm-up 3, Gather [0,10,25,26,27]) and :426-435 (unbounded state under
# Slice(all(50)) / Unslice) with whichever TestIncrement* ops SCN_OPS_LIB registers
INCREMENT_BODY = r'''
n = 120
rows = [struct.pack("<q", i) for i in range(n)]
eng = E.Engine(gpus=[], cpu_instances=2)
g = E.Graph(); src = g.add_source(False)
inc = g.add_op("TestIncrementBounded", [(src, "column")], warmup=3)
s = g.add_sample((inc, "integer")); sink = g.add_sink((s, "integer"))
j = E.Job(); j.bind_source(src, eng.add_bytes(rows))
j.set_sampler(s, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": [0, 10, 25, 26, 27]}))
eng.run(g, [j], 10, 100)
bounded = [struct.unpack("<q", j.output_row(sink, i))[0] for i in range(j.output_rows(sink))]
g = E.Graph(); src = g.add_source(False)
sl = g.add_slice((src, "column"))
inc = g.add_op("TestIncrementUnbounded", [(sl, "column")])
un = g.add_unslice((inc, "integer")); sink = g.add_sink((un, "integer"))
j = E.Job(); j.bind_source(src, eng.add_bytes(rows))
j.set_partitioner(sl, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedPartitionerArgs"], {"stride": 1, "group_size": 50}))
eng.run(g, [j], 5, 25)
unbounded = [struct.unpack("<q", j.output_row(sink, i))[0] for i in range(j.output_rows(sink))]
eng.close()
print("REF_JSON" + json.dumps({"bounded": bounded, "unbounded": unbounded}))
'''


def run(body, lib):
    out = subprocess.run([sys.executable, "-c", PRELUDE + body], env=dict(os.environ, SCN_ROOT=ROOT, SCN_OPS_LIB=lib),
                         cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "REF_JSON" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
    return json.loads(out.stdout.split("REF_JSON", 1)[1])


def live(kind):
    return run(BLUR_BODY if kind == "blur" else INCREMENT_BODY, REF_SO)


REF = Answers("ref_test_ops")


def check_reference_op_source_registers():
    """The reference's REGISTER_OP / REGISTER_KERNEL source, compiled against this repo's plugin headers, registers
    its ops with the names, argument messages and flags it declares (needs oracle/_ref, so part of recording)."""
    body = r'''
ops = E.list_ops()
for name in ("Histogram", "OpticalFlow", "Resize", "Blur", "TestIncrementUnbounded", "TestIncrementUnboundedFrame",
             "TestIncrementBounded", "TestIncrementBoundedFrame", "Sleep", "SleepFrame"):
    assert name in ops, name
assert ops["Blur"]["protobuf_name"] == "BlurArgs" and ops["Resize"]["stream_protobuf_name"] == "ResizeArgs"
assert ops["OpticalFlow"]["can_stencil"] and ops["TestIncrementBounded"]["bounded"] and ops["TestIncrementUnbounded"]["unbounded"]
print("REF_JSON{}")
'''
    run(body, REF_SO)


def test_reference_blur_kernel_pins_the_oracle():
    """The reference's Blur, run by this engine, == oracle.blur on the region the reference writes, odd and even
    kernel sizes."""
    got = REF("blur")
    for (k, h, w, n) in BLUR_CASES:
        ys, xs = oracle.blur_interior(h, w, k)
        for i in range(n):
            want = np.ascontiguousarray(oracle.blur(synth.rand_frame(900 + 7 * k + i, h, w), k)[ys, xs])
            assert hashlib.sha256(want.tobytes()).hexdigest() == got[f"{k},{h},{w},{n}"][i], (k, i)


def test_reference_increment_ops_give_the_values_the_reference_tests_expect():
    """The values the reference's own TestIncrementKernel (:173-236) gives under this engine -- bounded state with
    warm-up 3 under Gather [0,10,25,26,27] -> [0,3,3,4,5] (py_test.py:407-423), unbounded state under Slice(all(50)) /
    Unslice: as many rows as the input, a count that restarts with every slice group (:426-435) -- and this repo's
    test ops of the same names must give the same."""
    want = REF("increment")
    assert want["bounded"] == [0, 3, 3, 4, 5]
    assert want["unbounded"] == [i % 50 for i in range(120)]
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp")], stdout=subprocess.DEVNULL)
    assert run(INCREMENT_BODY, TEST_OPS_SO) == want


if __name__ == "__main__":
    REF = Answers("ref_test_ops", live)
    check_reference_op_source_registers()
    test_reference_blur_kernel_pins_the_oracle()
    test_reference_increment_ops_give_the_values_the_reference_tests_expect()
    REF.save()
    print("wrote", REF.path, len(REF.table), "answers")
