"""The engine's Sample / Space / Slice row algebra against the reference's OWN samplers and partitioners.

oracle/_ref/libref_sampler.so is the reference's scanner/engine/sampler.cpp compiled UNMODIFIED (oracle/Makefile) behind
a C shim (oracle/ref_sampler_shim.cpp).  For random arguments the rows a pipeline `source -> Sample/Space -> sink`
produces in this engine (values = the source row each output row carries, None = null row) must be what the
reference's get_num_downstream_rows / get_downstream_rows say for the full input, and the Slice groups must be the
reference partitioner's groups.  The argument bytes are the same proto3 wire bytes on both sides.
The reference's answers are replayed from tests/golden/ref_samplers.json; where oracle/_ref is built,
`python tests/test_reference_samplers_cpu.py` runs these tests against the library itself and records them again."""
import ctypes
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.recorded import Answers  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402
from scanner_b200 import protolite  # noqa: E402

REF_SO = os.path.join(ROOT, "oracle", "_ref", "libref_sampler.so")
SA = protolite.SAMPLER_ARGS
_L = ctypes.c_long


def live_reference(lib):
    """The reference library called through its shim: (kind, fn, args, x) -> the answer the tests record."""
    lib.ref_sampler_downstream.restype = _L
    lib.ref_sampler_upstream.restype = _L
    lib.ref_partitioner_groups.restype = _L

    def call(kind, fn, args, x):
        err = ctypes.create_string_buffer(512)
        if kind == "downstream":
            n = x
            cap = 64 * n + 64
            rows, mp, nd = (_L * cap)(), (_L * cap)(), _L(0)
            k = lib.ref_sampler_downstream(fn.encode(), args, len(args), _L(n), rows, mp, ctypes.c_size_t(cap),
                                           ctypes.byref(nd), err, ctypes.c_size_t(512))
            assert k >= 0, (fn, err.value)
            return [nd.value, list(rows[:k]), list(mp[:k])]
        if kind == "upstream":
            out, down = (_L * 64)(), (_L * len(x))(*x)
            k = lib.ref_sampler_upstream(fn.encode(), args, len(args), down, ctypes.c_size_t(len(x)), out,
                                         ctypes.c_size_t(64), None, ctypes.c_size_t(0))
            return list(out[:k])
        n = x
        rows, offs = (_L * (8 * n + 64))(), (_L * 256)()
        ng = lib.ref_partitioner_groups(fn.encode(), args, len(args), _L(n), rows, ctypes.c_size_t(8 * n + 64), offs,
                                        ctypes.c_size_t(256), err, ctypes.c_size_t(512))
        assert ng >= 0, (fn, err.value)
        return [list(rows[offs[g]:offs[g + 1]]) for g in range(ng)]
    return call


@pytest.fixture(scope="module")
def ref():
    return Answers("ref_samplers")


def load_plugin():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "liborc.so"], stdout=subprocess.DEVNULL)
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp")], stdout=subprocess.DEVNULL)
    if "TestWindow" not in E.list_ops():
        E.load_op_library(os.path.join(ROOT, "build", "tests", "libtest_plugin_ops.so"))


@pytest.fixture(scope="module", autouse=True)
def plugin():
    load_plugin()


def ref_downstream(ref, fn, args, n):
    nd, rows, mp = ref("downstream", fn, args, n)
    k = len(rows)
    assert list(rows[:k]) == list(range(k)) or fn in ("Gather", "Strided", "StridedRanges", "All")
    return nd, rows, mp


def engine_rows(eng, n, fn, args, space):
    g = E.Graph()
    src = g.add_source(False)
    s = g.add_space((src, "column")) if space else g.add_sample((src, "column"))
    sink = g.add_sink((s, "column"))
    j = E.Job()
    j.bind_source(src, eng.add_bytes([struct.pack("<q", i) for i in range(n)]))
    j.set_sampler(s, fn, args)
    eng.run(g, [j], 3, 9)
    out = []
    for i in range(j.output_rows(sink)):
        r = j.output_row(sink, i)
        out.append(None if r is None else struct.unpack("<q", r)[0])
    return out


def test_samplers_agree_with_the_reference_on_random_arguments(ref):
    rng = np.random.default_rng(2024)
    eng = E.Engine(gpus=[], cpu_instances=2)
    cases = [("All", b"", False, 17)]
    for _ in range(12):
        n = int(rng.integers(1, 90))
        cases.append(("Strided", protolite.encode(SA["StridedSamplerArgs"], {"stride": int(rng.integers(1, 12))}), False, n))
        k = int(rng.integers(1, 4))
        cuts = sorted(int(x) for x in rng.integers(0, n + 1, 2 * k))       # non-overlapping ascending ranges
        starts, ends = cuts[0::2], cuts[1::2]
        cases.append(("StridedRanges", protolite.encode(SA["StridedRangeSamplerArgs"],
                      {"stride": int(rng.integers(1, 6)), "starts": starts, "ends": ends}), False, n))
        rows = sorted(set(int(x) for x in rng.integers(0, n, int(rng.integers(1, 10)))))
        cases.append(("Gather", protolite.encode(SA["GatherSamplerArgs"], {"rows": rows}), False, n))
        sp = int(rng.integers(1, 6))
        cases.append(("SpaceNull", protolite.encode(SA["SpaceNullSamplerArgs"], {"spacing": sp}), True, int(rng.integers(1, 25))))
        cases.append(("SpaceRepeat", protolite.encode(SA["SpaceRepeatSamplerArgs"], {"spacing": sp}), True, int(rng.integers(1, 25))))
    for fn, args, space, n in cases:
        nd, rows, mp = ref_downstream(ref, fn, args, n)
        want = [None if m < 0 else m for m in mp]
        assert nd == len(rows), (fn, nd, len(rows))
        got = engine_rows(eng, n, fn, args, space)
        assert got == want, (fn, n, args.hex(), got, want)
    eng.close()


def test_samplers_required_upstream_rows_agree(ref):
    """get_upstream_rows (what the stencil / requirement analysis asks): a Gather of a Strided stream decodes exactly
    the source rows the two reference samplers name, observed through a counting source (frames_used of a raw stream
    is not exposed, so the check composes the two reference samplers and compares the produced VALUES)."""
    rng = np.random.default_rng(7)
    eng = E.Engine(gpus=[], cpu_instances=1)
    for _ in range(10):
        n, stride = int(rng.integers(20, 120)), int(rng.integers(1, 7))
        a1 = protolite.encode(SA["StridedSamplerArgs"], {"stride": stride})
        n1, _, m1 = ref_downstream(ref, "Strided", a1, n)
        pick = sorted(set(int(x) for x in rng.integers(0, n1, 5)))
        a2 = protolite.encode(SA["GatherSamplerArgs"], {"rows": pick})
        _, _, m2 = ref_downstream(ref, "Gather", a2, n1)
        want = [m1[i] for i in m2]
        # the reference's own answer to "which rows of the Strided stream do these Gather rows need"
        assert ref("upstream", "Gather", a2, list(range(len(pick)))) == pick
        g = E.Graph()
        src = g.add_source(False)
        s1 = g.add_sample((src, "column"))
        s2 = g.add_sample((s1, "column"))
        sink = g.add_sink((s2, "column"))
        j = E.Job()
        j.bind_source(src, eng.add_bytes([struct.pack("<q", i) for i in range(n)]))
        j.set_sampler(s1, "Strided", a1)
        j.set_sampler(s2, "Gather", a2)
        eng.run(g, [j], 2, 4)
        got = [struct.unpack("<q", j.output_row(sink, i))[0] for i in range(j.output_rows(sink))]
        assert got == want, (n, stride, pick)
    eng.close()


def test_partitioners_agree_with_the_reference(ref):
    """Slice groups: an unbounded-state counter restarts at every group, so `TestIncrementUnbounded` under
    Slice / Unslice spells the groups out: output row k of the concatenation is the position of its row inside its
    group -- compared with the reference partitioner's groups (sizes and order)."""
    rng = np.random.default_rng(99)
    eng = E.Engine(gpus=[], cpu_instances=2)
    cases = []
    for _ in range(6):
        n = int(rng.integers(10, 80))
        cases.append(("Strided", protolite.encode(SA["StridedPartitionerArgs"],
                      {"stride": int(rng.integers(1, 4)), "group_size": int(rng.integers(1, 20))}), n, None))
        k = int(rng.integers(1, 4))
        cuts = sorted(int(x) for x in rng.integers(0, n + 1, 2 * k))
        starts, ends = cuts[0::2], cuts[1::2]
        if all(a < b for a, b in zip(starts, ends)):
            cases.append(("StridedRange", protolite.encode(SA["StridedRangePartitionerArgs"],
                          {"stride": int(rng.integers(1, 4)), "starts": starts, "ends": ends}), n, None))
        group_rows = [sorted(set(int(x) for x in rng.integers(0, n, int(rng.integers(1, 8)))))
                      for _g in range(int(rng.integers(1, 4)))]
        groups = [protolite.encode(SA["GatherList"], {"rows": rows_}) for rows_ in group_rows]
        cases.append(("Gather", protolite.encode(SA["GatherPartitionerArgs"], {"groups": groups}), n, group_rows))
    for fn, args, n, want_groups in cases:
        ref_groups = ref("groups", fn, args, n)
        g = E.Graph()
        src = g.add_source(False)
        sl = g.add_slice((src, "column"))
        inc = g.add_op("TestIncrementUnbounded", [(sl, "column")])
        val = g.add_unslice((sl, "column"))
        cnt = g.add_unslice((inc, "integer"))
        s_val, s_cnt = g.add_sink((val, "column")), g.add_sink((cnt, "integer"))
        j = E.Job()
        j.bind_source(src, eng.add_bytes([struct.pack("<q", i) for i in range(n)]))
        j.set_partitioner(sl, fn, args)
        eng.run(g, [j], 3, 6)
        vals = [struct.unpack("<q", j.output_row(s_val, i))[0] for i in range(j.output_rows(s_val))]
        cnts = [struct.unpack("<q", j.output_row(s_cnt, i))[0] for i in range(j.output_rows(s_cnt))]
        if fn == "Gather":
            # reference defect: GatherPartitioner::group_at(group_idx) reads args_.groups(curr_group_idx_) -- the
            # iteration cursor, not its argument (sampler.cpp:707-712) -- so every group comes back as group 0.  The
            # group SIZES (total_rows_per_group, from the arguments) and group 0 are comparable; the engine follows the
            # arguments for the other groups, which is what the sizes the reference itself reports describe.
            assert len(ref_groups) == len(want_groups)
            assert ref_groups[0] == want_groups[0] and all(grp == ref_groups[0] for grp in ref_groups)
            ref_groups = want_groups
        assert vals == [r for grp in ref_groups for r in grp], (fn, vals, ref_groups)       # rows, group after group
        assert cnts == [i for grp in ref_groups for i in range(len(grp))], (fn, cnts)          # state restarts per group
    eng.close()


if __name__ == "__main__":
    live = Answers("ref_samplers", live_reference(ctypes.CDLL(REF_SO)))
    load_plugin()
    test_samplers_agree_with_the_reference_on_random_arguments(live)
    test_samplers_required_upstream_rows_agree(live)
    test_partitioners_agree_with_the_reference(live)
    live.save()
    print("wrote", live.path, len(live.table), "answers")
