"""scannerpy-shaped graph surface over the in-process engine.

Keeps the names and call shapes of the reference's Python API for the hot path so pipelines read
the same (python/scannerpy/client.py:1282-1590 `Client.run`, op.py:121-314 `sc.ops.<Name>(...)`,
streams.py `sc.streams.Stride/Range/Gather/...`, storage.py:250-372 `NamedVideoStream`,
`NamedStream`, common.py:78-234 `PerfParams`).  The transport underneath is not gRPC: the graph is
handed to libscn_engine.so through its C ABI.  With `Client(db_path=...)` named streams live in a
database directory in the reference's on-disk layout (engine.Database): videos are ingested from
.mp4 / .h264 files once and re-bound from their stored index afterwards, outputs are committed as
tables and can be loaded by a later session.  Python kernels (`@register_python_op`, pyops.py) run
inside the engine's evaluate threads.  Not reproduced: the multi-node master.

    sc = Client(gpus=[0])
    video = NamedVideoStream(sc, 'clip', path='clip.h264')         # Annex-B elementary stream
    frames = sc.io.Input([video])
    hists = sc.ops.Histogram(frame=sc.streams.Stride(frames, [2]), device=DeviceType.GPU)
    out = NamedStream(sc, 'clip_hist')
    sc.run(sc.io.Output(hists, [out]), PerfParams.manual(32, 64))
    for h in out.load(): ...            # 3 arrays of 16 int32, like scannerpy.types.Histogram
"""
import enum
import os
import pickle

import numpy as np

from . import engine as E
from . import protolite
from . import pyops
from . import types as sctypes


class DeviceType(enum.IntEnum):
    CPU = 0
    GPU = 1


class ColumnType(enum.Enum):
    """What a column holds (reference common.py:57-69)."""
    Blob = 0
    Video = 1


class DeviceHandle:
    """(device type, device id), as KernelConfig.devices lists them (reference common.py:51-54)."""

    def __init__(self, device, device_id):
        self.device, self.device_id = device, device_id

    def __iter__(self):  # unpacks like the (type, id) pair it replaces
        return iter((self.device, self.device_id))

    def __getitem__(self, i):
        return (self.device, self.device_id)[i]

    def __repr__(self):
        return f"DeviceHandle({self.device!r}, {self.device_id})"


class CacheMode(enum.Enum):
    Error = 1
    Ignore = 2
    Overwrite = 3


class NullElement:
    """A null row of a loaded stream (reference storage.py:8-16): what RepeatNull spacing or a kernel
    returning None leaves behind.  Falsy and equal to None, so `if row:` and `row == None` both work."""

    def __repr__(self):
        return "NullElement()"

    def __bool__(self):
        return False

    def __eq__(self, other):
        return other is None or isinstance(other, NullElement)

    def __hash__(self):
        return hash(None)


def _is_null(row):
    return row is None or isinstance(row, NullElement)


class ScannerException(Exception):
    pass


class PerfParams:
    def __init__(self, work_packet_size, io_packet_size, pipeline_instances_per_node=None, **_ignored):
        self.work_packet_size = work_packet_size
        self.io_packet_size = io_packet_size
        self.pipeline_instances_per_node = pipeline_instances_per_node

    @classmethod
    def manual(cls, work_packet_size, io_packet_size, **kwargs):
        return cls(work_packet_size, io_packet_size, **kwargs)

    @classmethod
    def estimate(cls, max_memory_util=0.7, total_memory=None, work_io_ratio=0.2, **kwargs):
        # the reference sizes packets from host RAM (common.py:149-234); on a 180 GB GPU a packet of
        # 64 1080p frames (398 MB) per instance is comfortably small: fixed, GOP-friendly defaults
        return cls(32, 64 if work_io_ratio <= 0.5 else 32, **kwargs)


# ------------------------------------------------------------------------------------------------
class OpColumn:
    """An edge of the graph: output column `column` of node `op` (reference scannerpy/op.py:26-119)."""

    def __init__(self, op, column, is_frame, encode_options=None):
        self._op, self._col, self._is_frame = op, column, is_frame
        self._encode_options = encode_options

    # How a frame column is stored when it reaches an Output (op.py:57-98).  `compress_video()` on a client with
    # GPUs and a database stores each task's frames as intra-only H.264 (scn_h264_encode_u8, on the pipeline
    # instance's GPU); `lossless()`, `compress("default")` and unannotated columns are stored uncompressed, and so
    # is everything on CPU-only clients and in clients without a database (their outputs stay in memory).
    def _stored_as(self, options):
        if not self._is_frame:
            raise ScannerException(f'Compression only supported for sequences of type "video". Sequence '
                                   f'{self._col} type is Bytes.')
        return OpColumn(self._op, self._col, self._is_frame, options)

    def compress(self, codec="video", **kwargs):
        codecs = {"video": self.compress_video, "default": self.compress_default, "raw": self.lossless}
        if codec not in codecs:
            raise ScannerException(f"Compression codec {codec} not currently supported. Available codecs are: "
                                   f"{' '.join(codecs)}.")
        return codecs[codec](**kwargs)

    def compress_video(self, quality=-1, bitrate=-1, keyframe_distance=-1):
        """Store the frames as H.264 (3-channel uint8 frames of one even size per task, no null rows; anything
        else fails the run).  quality: the constant QP, 0-51 (-1: 23, x264's default CRF); keyframe_distance:
        pictures between IDRs (-1: 120, the reference encoder's gop_size).  bitrate is accepted and not honoured:
        the encoder is constant-QP, without rate control."""
        return self._stored_as({"codec": "h264", "quality": quality, "bitrate": bitrate,
                                "keyframe_distance": keyframe_distance})

    def lossless(self):
        return self._stored_as({"codec": "raw"})

    def compress_default(self):
        return self._stored_as({"codec": "default"})


def _h264_encoding(col):
    """compress_video() options of an output's column -> (QP, keyframe_distance); None when it is stored raw."""
    opts = col._encode_options
    if not opts or opts.get("codec") != "h264":
        return None
    q, kd = opts.get("quality", -1), opts.get("keyframe_distance", -1)
    if q == -1:
        q = 23
    elif isinstance(q, bool) or not isinstance(q, int) or not 0 <= q <= 51:
        raise ScannerException(f"compress_video(quality={q!r}): quality is the H.264 QP, 0-51 (or -1 for 23)")
    if kd == -1:
        kd = 120
    elif isinstance(kd, bool) or not isinstance(kd, int) or kd < 1:
        raise ScannerException(f"compress_video(keyframe_distance={kd!r}): at least 1 (or -1 for 120)")
    return q, kd


class SliceList(list):
    """Per-slice-group arguments (reference scannerpy.common.SliceList): inside a Slice, one entry
    per group where an un-sliced stream takes one value."""


class _Node:
    def __init__(self, kind, name=None, inputs=(), device=DeviceType.CPU, args=b"", batch=-1, stencil=(),
                 warmup=-1, per_stream=None, streams=None, sampler=None):
        self.kind, self.name, self.inputs = kind, name, list(inputs)
        self.device, self.args, self.batch, self.stencil, self.warmup = device, args, batch, list(stencil), warmup
        self.per_stream = per_stream      # list (one per job) of serialized stream args / sampler args
        self.streams = streams            # Input: list of stored streams; Output: list of NamedStream
        self.sampler = sampler            # Sample/Space: sampler function name


class OpGenerator:
    """sc.ops.<Name>(col=..., device=..., batch=..., stencil=..., bounded_state=..., **args)"""

    def __init__(self, sc):
        self._sc = sc

    def __getattr__(self, name):
        ops = E.list_ops()
        if name not in ops:
            raise ScannerException(f"Op {name} is not registered (load_op first?)")

        def make(*varargs, device=None, batch=-1, stencil=(), bounded_state=None, **kwargs):
            if device is None:
                # the reference defaults to DeviceType.CPU (op.py:184); the stdlib pixel ops here have
                # GPU kernels only, so an op without a CPU kernel defaults to the GPU instead of failing
                has_cpu = E.lib().scn_kernel_registered(name.encode(), int(DeviceType.CPU)) == 1
                has_gpu = E.lib().scn_kernel_registered(name.encode(), int(DeviceType.GPU)) == 1
                device = DeviceType.GPU if (has_gpu and not has_cpu) else DeviceType.CPU
            cols = [(k, v) for k, v in kwargs.items() if isinstance(v, OpColumn)]
            rest = {k: v for k, v in kwargs.items() if not isinstance(v, OpColumn)}
            if varargs:  # variadic inputs are positional (op.py:196-205)
                if cols or not all(isinstance(v, OpColumn) for v in varargs):
                    raise ScannerException(f"Op {name}: positional arguments are variadic input columns and "
                                           f"cannot be mixed with named inputs")
                cols = [(f"arg{i}", v) for i, v in enumerate(varargs)]
            pyop = pyops.PYTHON_OP_REGISTRY.get(name)
            if pyop is not None:
                return self._make_python(pyop, cols, rest, device, batch, stencil, bounded_state)
            protos = self._sc._op_protos.get(name, {})
            init_fields, stream_fields = protos.get("init"), protos.get("stream")
            init_vals, stream_vals = {}, {}
            for k, v in rest.items():
                # list-valued kwargs matching the stream message are per-stream args (op.py:278-314)
                if stream_fields and any(f[0] == k for f in stream_fields) and isinstance(v, (list, tuple)):
                    stream_vals[k] = list(v)
                elif init_fields and any(f[0] == k for f in init_fields):
                    init_vals[k] = v
                else:
                    raise ScannerException(f"Op {name} does not take argument {k!r}")
            args = protolite.encode(init_fields, init_vals) if init_fields and init_vals else b""
            per_stream = None
            if stream_vals:
                n = len(next(iter(stream_vals.values())))
                per_stream = []
                for i in range(n):
                    vals = {k: v[i] for k, v in stream_vals.items()}
                    sliced = [v for v in vals.values() if isinstance(v, SliceList)]
                    if sliced:  # inside a Slice: one new_stream argument per slice group
                        groups = max(len(v) for v in sliced)
                        per_stream.append(SliceList(
                            protolite.encode(stream_fields,
                                             {k: (v[g if len(v) > 1 else 0] if isinstance(v, SliceList) else v)
                                              for k, v in vals.items()}) for g in range(groups)))
                    else:
                        per_stream.append(protolite.encode(stream_fields, vals))
            node = _Node("op", name, [c for _, c in cols], DeviceType(device), args, batch, stencil,
                         -1 if bounded_state is None else bounded_state, per_stream)
            node.input_names = [k for k, _ in cols]
            outs = self._sc._op_outputs(name)
            res = [OpColumn(node, c, t) for c, t in outs]
            return res[0] if len(res) == 1 else tuple(res)

        return make


    def _make_python(self, pyop, cols, rest, device, batch, stencil, bounded_state):
        """A Python op: init arguments and per-stream arguments travel pickled (op.py:296-298,
        kernel.py:12 `pickle.loads(config.args())`), list-valued kwargs named like a parameter of
        `new_stream` are per-stream arguments."""
        if not pyop.variadic:
            given = dict(cols)
            for c in pyop.inputs:
                if c.name not in given:
                    raise ScannerException(f"Op {pyop.name} required sequence {c.name} as input")
            extra = sorted(set(given) - {c.name for c in pyop.inputs})
            if extra:
                raise ScannerException(f"Op {pyop.name} has no input named {extra[0]!r}")
            cols = [(c.name, given[c.name]) for c in pyop.inputs]  # the engine binds inputs by position
        # every other keyword is an init argument (function kernels read them from config.args,
        # class kernels receive them in __init__), except the parameters of new_stream (op.py:189-222)
        rest = dict(rest)
        explicit = rest.pop("args", None)
        rest.pop("extra", None)
        init_vals, stream_vals = {}, {}
        for k, v in rest.items():
            if k in pyop.stream_params:
                if not isinstance(v, (list, tuple)):
                    raise ScannerException(f"The argument `{k}` to op `{pyop.name}` is a stream config argument "
                                           f"and must be a list.")
                stream_vals[k] = list(v)
            else:
                init_vals[k] = v
        if explicit is not None:
            init_vals = explicit
        if pyop.stream_params and not stream_vals:
            raise ScannerException(f"No arguments provided to op `{pyop.name}` for stream parameters.")
        per_stream = None
        if stream_vals:
            n = len(next(iter(stream_vals.values())))
            if any(len(v) != n for v in stream_vals.values()):
                raise ScannerException(f"Op {pyop.name}: stream arguments must all list one value per stream")
            per_stream = []
            for i in range(n):
                vals = {k: v[i] for k, v in stream_vals.items()}
                sliced = [v for v in vals.values() if isinstance(v, SliceList)]
                if sliced:
                    groups = max(len(v) for v in sliced)
                    per_stream.append(SliceList(
                        pickle.dumps({k: (v[g if len(v) > 1 else 0] if isinstance(v, SliceList) else v)
                                      for k, v in vals.items()}) for g in range(groups)))
                else:
                    per_stream.append(pickle.dumps(vals))
        node = _Node("op", pyop.name, [c for _, c in cols], DeviceType(device), pickle.dumps(init_vals), batch,
                     stencil, -1 if bounded_state is None else bounded_state, per_stream)
        node.input_names = [k for k, _ in cols]
        node.type_names = {c.name: ("" if c.is_frame else c.info.cpp_name) for c in pyop.outputs}
        res = [OpColumn(node, c.name, c.is_frame) for c in pyop.outputs]
        return res[0] if len(res) == 1 else tuple(res)


class StreamsGenerator:
    """Row sampling ops; arguments are one entry per input stream (reference streams.py)."""

    def __init__(self, sc):
        self._sc = sc

    def _sample(self, col, fn, msg, per_stream_dicts, kind="sample"):
        def enc(d):
            if isinstance(d, SliceList):  # one sampler argument per slice group
                return SliceList(enc(e) for e in d)
            return protolite.encode(protolite.SAMPLER_ARGS[msg], d) if msg else b""
        node = _Node(kind, fn, [col], per_stream=[enc(d) for d in per_stream_dicts], sampler=fn)
        return OpColumn(node, col._col, col._is_frame)

    @staticmethod
    def _map(v, fn):
        """fn over a per-stream value, or over every entry of a SliceList"""
        return SliceList(fn(e) for e in v) if isinstance(v, SliceList) else fn(v)

    @staticmethod
    def _pair(r):
        return (r["start"], r["end"]) if isinstance(r, dict) else (r[0], r[1])

    @staticmethod
    def _fields(e, names):
        """One per-stream sampler argument as the reference accepts it (op.py extra/arg_builder:
        a dict is keyword arguments, a tuple positional ones, anything else the single argument)."""
        if isinstance(e, dict):
            missing = [n for n in names if n not in e]
            if missing:
                raise ScannerException(f"sampler argument {e!r} lacks {missing[0]!r}")
            return tuple(e[n] for n in names)
        if isinstance(e, tuple) or (isinstance(e, list) and len(names) > 1):
            if len(e) != len(names):
                raise ScannerException(f"sampler argument {e!r} must have {len(names)} entries {names}")
            return tuple(e)
        return (e,)

    def Slice(self, input, partitions):
        """partitions: one partitioner per stream (sc.partitioner.all / strided / ranges / ...)."""
        node = _Node("slice", "Slice", [input], per_stream=list(partitions))
        return OpColumn(node, input._col, input._is_frame)

    def Unslice(self, input):
        node = _Node("unslice", "Unslice", [input])
        return OpColumn(node, input._col, input._is_frame)

    def All(self, input):
        return self._sample(input, "All", None, [{}])

    def Stride(self, input, strides):
        return self._sample(input, "Strided", "StridedSamplerArgs",
                            [self._map(s, lambda e: {"stride": self._fields(e, ["stride"])[0]}) for s in strides])

    def Range(self, input, ranges):
        ds = [self._map(r, lambda e: {"stride": 1, "starts": [self._pair(e)[0]], "ends": [self._pair(e)[1]]})
              for r in ranges]
        return self._sample(input, "StridedRanges", "StridedRangeSamplerArgs", ds)

    def Ranges(self, input, intervals):
        return self.StridedRanges(input, intervals, [1] * len(intervals))

    def StridedRange(self, input, ranges):
        triples = [self._fields(r, ["start", "end", "stride"]) for r in ranges]
        return self.StridedRanges(input, [[(s, e)] for s, e, _ in triples], [st for _, _, st in triples])

    def StridedRanges(self, input, intervals, strides=None, stride=None):
        if strides is None:
            strides = 1 if stride is None else stride  # the reference's single `stride` for every stream
        strides = strides if isinstance(strides, (list, tuple)) else [strides] * len(intervals)
        return self._sample(input, "StridedRanges", "StridedRangeSamplerArgs",
                            [{"stride": st, "starts": [self._pair(p)[0] for p in iv],
                              "ends": [self._pair(p)[1] for p in iv]} for iv, st in zip(intervals, strides)])

    def Gather(self, input, indices):
        return self._sample(input, "Gather", "GatherSamplerArgs",
                            [self._map(r, lambda e: {"rows": list(e["rows"] if isinstance(e, dict) else e)})
                             for r in indices])

    def RepeatNull(self, input, spacings):
        return self._sample(input, "SpaceNull", "SpaceNullSamplerArgs",
                            [{"spacing": self._fields(s, ["spacing"])[0]} for s in spacings], "space")

    def Repeat(self, input, spacings):
        return self._sample(input, "SpaceRepeat", "SpaceRepeatSamplerArgs",
                            [{"spacing": self._fields(s, ["spacing"])[0]} for s in spacings], "space")


class Partitioner:
    """Slice partitioners (reference scannerpy/partitioner.py): how a Slice cuts its input into groups."""

    @staticmethod
    def _enc(msg, d):
        return protolite.encode(protolite.SAMPLER_ARGS[msg], d)

    def all(self, group_size=250):
        return self.strided(1, group_size)

    def strided(self, stride, group_size=250):
        return ("Strided", self._enc("StridedPartitionerArgs", {"stride": stride, "group_size": group_size}))

    def range(self, start, end):
        return self.ranges([(start, end)])

    def ranges(self, intervals):
        return self.strided_ranges(intervals, 1)

    def strided_range(self, start, end, stride):
        return self.strided_ranges([(start, end)], stride)

    def strided_ranges(self, intervals, stride):
        return ("StridedRange", self._enc("StridedRangePartitionerArgs", {
            "stride": stride, "starts": [a for a, _ in intervals], "ends": [b for _, b in intervals]}))

    def gather(self, groups_of_rows):
        groups = [self._enc("GatherList", {"rows": list(g)}) for g in groups_of_rows]
        return ("Gather", self._enc("GatherPartitionerArgs", {"groups": groups}))


class IOGenerator:
    def __init__(self, sc):
        self._sc = sc

    def _attach(self, streams):
        for st in streams:
            if hasattr(st, "_attach"):
                st._attach(self._sc)

    def Input(self, streams):
        self._attach(streams)
        is_video = isinstance(streams[0], NamedVideoStream) or getattr(streams[0], "_is_frame", False)
        node = _Node("input", "Input", streams=list(streams))
        return OpColumn(node, "frame" if is_video else "column", is_video)

    def Output(self, op, streams):
        self._attach(streams)
        return _Node("output", "Output", [op], streams=list(streams))


# ------------------------------------------------------------------------------------------------
class NamedVideoStream:
    """A stored video.  path: an .mp4/.mov or an H.264 Annex-B file; data: the bytes of either;
    frames: (n,h,w,3) uint8 RAW frames (kept in memory only).  With a database the video becomes
    (or already is) the table `name` and is bound from its stored index."""

    def __init__(self, sc, name, path=None, data=None, frames=None, inplace=False):
        self._sc, self._name = sc, name
        self._job, self._sink, self._type, self._sid = None, None, None, None  # output role (see NamedStream)
        db = sc._db
        if name in sc._streams and path is None and data is None and frames is None:
            self._sid = sc._streams[name]
            return
        if frames is not None:
            self._sid = sc._engine.add_raw_frames(frames)
        elif db is not None:
            if not db.has_table(name):
                if path is None and data is None:
                    return  # not stored yet: usable as the target of an Output (frames are stored RAW)
                try:
                    if path is not None:
                        db.ingest_video(name, path, inplace=inplace)
                    else:
                        stream = E.mp4_demux(data)[0] if _is_mp4(data) else data
                        db.ingest_h264(name, stream)
                except E.EngineError as e:
                    raise ScannerException(str(e)) from e
            self._sid = db.add_video_stream(sc._engine, name)
        else:
            if data is None:
                if path is None:
                    return  # target of an Output
                with open(path, "rb") as f:
                    data = f.read()
            try:
                if _is_mp4(data):
                    data = E.mp4_demux(data)[0]
                self._sid = sc._engine.add_h264(data)
            except E.EngineError as e:
                raise ScannerException(str(e)) from e
        sc._streams[name] = self._sid

    def name(self):
        return self._name

    def _stored(self):
        db = self._sc._db
        return db is not None and db.has_table(self._name)

    def _bind(self):
        """stream id for use as an input; a video written by an earlier job binds lazily"""
        if self._sid is None:
            db = self._sc._db
            if self._job is None and db is not None and db.has_table(self._name) and \
                    db.table_info(self._name)["keyframes"] > 0:
                self._sid = db.add_video_stream(self._sc._engine, self._name)  # ingested H.264
            elif self._job is not None or self._stored():
                # frames written by an earlier job (stored uncompressed): the next job's input
                frames = list(NamedStream.load(self))
                if not frames or any(_is_null(f) for f in frames):
                    raise ScannerException(f"video stream {self._name} has null or no frames: it cannot be an input")
                self._sid = self._sc._engine.add_raw_frames(np.stack(frames))
            else:
                raise ScannerException(f"video stream {self._name} does not exist (no table, no path, not written yet)")
            self._sc._streams[self._name] = self._sid
        return self._sid

    def len(self):
        if self._sid is None and (self._job is not None or self._stored()):
            return NamedStream.len(self)
        return self._sc._engine.stream_rows(self._bind())

    def info(self):
        return self._sc._engine.stream_info(self._bind())

    def exists(self):
        return self._sid is not None or self._job is not None or self._stored()

    committed = exists

    def load_bytes(self, rows=None):
        return NamedStream.load_bytes(self, rows)

    def load(self, ty=None, fn=None, rows=None):
        """Generator over frames (ndarrays).  Frames a job stored uncompressed are read back as they are; an
        ingested H.264 video, or a job output stored with compress_video(), is decoded for the asked rows (the
        reference runs a Gather + ImageEncoder job for this, column.py:227-240; here the decode stage is called
        directly, which needs a GPU).  A compressed job output of several items (one per task) reads as one
        stream."""
        if self._job is None and self._sid is None and self._stored() and \
                self._sc._db.table_info(self._name)["keyframes"] > 0:
            self._bind()
        if self._job is None and self._sid is not None and self._is_compressed():
            return self._decode(rows)
        return NamedStream.load(self, ty, fn, rows)

    def _is_compressed(self):
        try:
            return self._sc._engine.stream_info(self._sid)["keyframes"] > 0
        except E.EngineError:
            return False

    def _decode(self, rows, chunk=32):
        if not self._sc._gpus:
            raise ScannerException(f"loading frames of the compressed video {self._name} needs a GPU (NVDEC)")
        n = self._sc._engine.stream_rows(self._sid)
        rows = list(range(n)) if rows is None else [int(r) for r in rows]
        order = sorted(set(rows))
        if order and (order[0] < 0 or order[-1] >= n):
            raise ScannerException(f"rows must be inside [0, {n})")
        def chunks():
            for i in range(0, len(order), chunk):
                part = order[i:i + chunk]
                try:
                    frames = self._sc._engine.decode_to_device(self._sid, part, gpu=self._sc._gpus[0]).cpu().numpy()
                except E.EngineError as e:
                    raise ScannerException(str(e)) from e
                yield part, frames

        if rows == order:  # ascending: stream chunk by chunk
            for _, frames in chunks():
                yield from frames
            return
        decoded = {}
        for part, frames in chunks():
            decoded.update(zip(part, frames))
        for r in rows:
            yield decoded[r]

    def delete(self, sc=None):
        NamedStream.delete(self, sc)

    def save_mp4(self, output_name, fps=None):
        """Write the video as `<output_name>.mp4` (reference storage.py NamedVideoStream.save_mp4).
        An ingested H.264 table, or a job output stored with compress_video(), is re-wrapped sample for
        sample without re-encoding.  Frames a job stored uncompressed are converted to BT.601 4:2:0 and
        written as intra-PCM H.264 -- every player opens it, the file is as large as the raw video."""
        path = output_name if output_name.endswith(".mp4") else output_name + ".mp4"
        db = self._sc._db
        if db is not None and db.has_table(self._name) and self._job is None:
            info = db.table_info(self._name)
            if info.get("keyframes", 0) > 0:  # compressed column: container work only
                try:
                    db.export_mp4(self._name, path, int(fps) if fps else 0, 1 if fps else 0)
                except E.EngineError as e:
                    raise ScannerException(str(e)) from e
                return path
        if not self.exists():
            raise ScannerException(f"stream {self._name} does not exist")
        planes, size = [], None
        for f in self.load():
            if _is_null(f):
                continue
            if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] not in (1, 3):
                raise ScannerException("save_mp4 writes uint8 frames with 1 or 3 channels")
            if size is None:
                size = f.shape[:2]
            elif f.shape[:2] != size:
                raise ScannerException("save_mp4 needs frames of one size")
            planes.append(_rgb_to_i420(f))
        if not planes:
            raise ScannerException(f"stream {self._name} has no frames")
        h, w = size[0] + (size[0] & 1), size[1] + (size[1] & 1)
        stream = E.h264_synth(np.stack(planes), w, h, gop=1)
        with open(path, "wb") as out:
            out.write(E.mp4_mux(stream, int(fps) if fps else 25, 1))
        return path


def _rgb_to_i420(frame):
    """uint8 (H, W, 3|1) -> flat I420 planes (BT.601 studio range, 2x2 box chroma), odd sizes padded
    by edge replication."""
    h, w = frame.shape[:2]
    if (h & 1) or (w & 1):
        frame = np.pad(frame, ((0, h & 1), (0, w & 1), (0, 0)), mode="edge")
        h, w = frame.shape[:2]
    f = frame.astype(np.float32)
    if f.shape[2] == 1:
        f = np.repeat(f, 3, axis=2)
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    y = 16.0 + 0.257 * r + 0.504 * g + 0.098 * b
    cb = 128.0 - 0.148 * r - 0.291 * g + 0.439 * b
    cr = 128.0 + 0.439 * r - 0.368 * g - 0.071 * b
    sub = lambda p: p.reshape(h // 2, 2, w // 2, 2).mean(axis=(1, 3))  # noqa: E731
    q = lambda p: np.clip(np.rint(p), 0, 255).astype(np.uint8).reshape(-1)  # noqa: E731
    return np.concatenate([q(y), q(sub(cb)), q(sub(cr))])


def _is_mp4(data):
    return len(data) >= 12 and bytes(data[4:8]) in (b"ftyp", b"moov", b"mdat", b"free", b"skip", b"wide", b"styp")


def _column_type_name(col):
    """Type name stored with an output column: what the producing op declared (the reference keeps
    it in ColumnDescriptor.type_name), through row-sampling nodes."""
    node = col._op
    while node is not None and node.kind in ("sample", "space", "slice", "unslice") and node.inputs:
        col = node.inputs[0]
        node = col._op
    names = getattr(node, "type_names", None)
    if names and col._col in names:
        return names[col._col]
    return "Histogram" if col._col == "histogram" else ""


def _typed(row, ty):
    """Deserialise a stored byte row by its column type name (scannerpy.types registry)."""
    if row is None:
        return NullElement()
    if isinstance(row, np.ndarray) or not ty:
        return row
    if isinstance(ty, str):
        if ty in ("Bytes", "bytes"):
            return row
        try:
            info = sctypes.get_type_info_cpp(ty)
        except sctypes.ScannerTypeError:
            return row  # a type this process has not registered: the raw bytes
    else:
        info = sctypes.get_type_info(ty)
    return info.deserialize(bytes(row))


class NamedStream:
    """An output column (or a byte-row input when created with rows=[...]).  With a database it is
    the table `name` with one data column, readable by later sessions."""

    def __init__(self, sc, name, rows=None):
        self._sc, self._name, self._job, self._sink, self._type = sc, name, None, None, None
        self._sid = None
        if rows is not None:
            self._sid = sc._engine.add_bytes(rows)
            sc._streams[name] = self._sid

    def name(self):
        return self._name

    def _stored(self):
        db = self._sc._db
        return db is not None and db.has_table(self._name)

    def _bind(self):
        """stream id for use as an input: the rows an earlier job wrote (in memory or in the
        database) become a byte stream of the engine"""
        if self._sid is None:
            if self._job is None and not self._stored():
                raise ScannerException(f"stream {self._name} does not exist (not written yet)")
            rows = list(self.load_bytes())
            if any(isinstance(r, np.ndarray) for r in rows):
                raise ScannerException(f"stream {self._name} holds frames: bind it as a NamedVideoStream")
            self._sid = self._sc._engine.add_bytes([b"" if _is_null(r) else bytes(r) for r in rows])
            self._sc._streams[self._name] = self._sid
        return self._sid

    def exists(self):
        return self._job is not None or self._sid is not None or self._stored()

    committed = exists

    def len(self):
        if self._job is not None:
            return self._job.output_rows(self._sink)
        if self._sid is not None:
            return self._sc._engine.stream_rows(self._sid)
        if self._stored():
            return self._sc._db.table_info(self._name)["rows"]
        raise ScannerException(f"stream {self._name} does not exist")

    def load_bytes(self, rows=None):
        """Rows as stored: bytes (frame columns: ndarrays), no deserialisation (storage.py:88-100)."""
        return self.load(ty="Bytes", rows=rows)

    def load(self, ty=None, fn=None, rows=None):
        """Generator over rows, deserialised like scannerpy.types (types.py:91-132): frame columns
        as ndarrays, byte columns through the serializer registered for the column's type name
        (`Histogram`: a list of three int32 arrays; unknown or empty type name: bytes).  `ty` may
        be a type name or a registered Python type; `fn` is a custom bytes -> value function that
        takes precedence (storage.py:135-173)."""
        if self._job is not None:
            ty = ty or self._type
            idx = range(self.len()) if rows is None else rows
            fetched = (self._job.output_row(self._sink, i) for i in idx)
        elif self._stored():
            info = self._sc._db.table_info(self._name)
            col = info["columns"][1]
            ty = ty or col["type_name"] or None
            fetched = iter(self._sc._db.read_rows(self._name, col["name"], rows))
        else:
            raise ScannerException(f"stream {self._name} has not been written by a job")
        for r in fetched:
            if fn is not None and r is not None and not isinstance(r, np.ndarray):
                yield fn(bytes(r))
            else:
                yield _typed(r, ty)

    def delete(self, sc=None):
        self._job = None
        if self._stored():
            self._sc._db.delete_table(self._name)


class FilesStream(NamedStream):
    """One row per file (scannertools.storage.files.FilesStream, used by the reference's tutorial
    05_sources_sinks.py): as an Input the rows are the files' bytes, as an Output every row is
    written to its path when the job finishes (null rows leave no file)."""

    _counter = 0

    def __init__(self, sc_or_paths, paths=None):
        # the scannertools class takes only `paths`; the client is picked up when the stream is used
        sc, paths = (None, sc_or_paths) if paths is None else (sc_or_paths, paths)
        FilesStream._counter += 1
        self._paths = [str(p) for p in paths]
        self._sc, self._name = sc, f"__files_{FilesStream._counter}"
        self._job, self._sink, self._type, self._sid = None, None, None, None

    def _attach(self, sc):
        if self._sc is None:
            self._sc = sc

    def len(self):
        return len(self._paths)

    def exists(self):
        return all(os.path.exists(p) for p in self._paths)

    committed = exists

    def _bind(self):
        if self._sid is None:
            rows = []
            for p in self._paths:
                with open(p, "rb") as f:
                    rows.append(f.read())
            self._sid = self._sc._engine.add_bytes(rows)
        return self._sid

    def _after_run(self):
        rows = list(NamedStream.load(self, ty="Bytes"))
        if len(rows) != len(self._paths):
            raise ScannerException(f"FilesStream lists {len(self._paths)} paths but the job wrote {len(rows)} rows")
        for p, r in zip(self._paths, rows):
            if _is_null(r):
                continue
            if isinstance(r, np.ndarray):
                raise ScannerException("FilesStream stores byte rows; encode frames first (ImageEncoder)")
            with open(p, "wb") as f:
                f.write(bytes(r))
        if self._stored():  # the rows went through a scratch table
            self._sc._db.delete_table(self._name)
        self._job = None

    def load(self, ty=None, fn=None, rows=None):
        idx = range(len(self._paths)) if rows is None else rows
        for i in idx:
            with open(self._paths[i], "rb") as f:
                blob = f.read()
            yield fn(blob) if fn is not None else _typed(blob, ty)

    def delete(self, sc=None):
        for p in self._paths:
            if os.path.exists(p):
                os.remove(p)


class Column:
    """A stored column (reference scannerpy/column.py): `load()` yields its rows."""

    def __init__(self, table, desc):
        self._table, self._desc = table, desc

    def name(self):
        return self._desc["name"]

    def type(self):
        return self._desc["type"]

    def load(self, ty=None, fn=None, rows=None):
        """Rows of the column (reference column.py:200-260): byte columns through their type's
        deserializer, stored frames as ndarrays, a compressed (ingested) video column decoded."""
        if self._desc["type"] == "Video" and self._table._info.get("keyframes", 0) > 0:
            if self._table._sc is None:
                raise ScannerException("loading a compressed video column needs the table from Client.table()")
            yield from NamedVideoStream(self._table._sc, self._table._name).load(rows=rows)
            return
        ty = ty or self._desc["type_name"] or None
        for r in self._table._db.read_rows(self._table._name, self._desc["name"], rows):
            if fn is not None and r is not None and not isinstance(r, np.ndarray):
                yield fn(bytes(r))
            else:
                yield _typed(r, ty)


class Table:
    """A stored table (reference scannerpy/table.py): id, name, rows, columns."""

    def __init__(self, db, name, sc=None):
        self._db, self._name, self._sc = db, name, sc
        self._info = db.table_info(name)

    def id(self):
        return self._info["id"]

    def name(self):
        return self._name

    def num_rows(self):
        return self._info["rows"]

    def column_names(self):
        return [c["name"] for c in self._info["columns"]]

    def column(self, name):
        for c in self._info["columns"]:
            if c["name"] == name:
                return Column(self, c)
        raise ScannerException(f"table {self._name} has no column {name}")

    def committed(self):
        return True


class Profile:
    def __init__(self, sc):
        self._sc = sc

    def statistics(self):
        return self._sc._engine.stats()

    def write_trace(self, path):
        if not self._sc._profiling:
            raise ScannerException("this Client was created with profiling=False: no trace was recorded")
        self._sc._engine.write_trace(path)


# ------------------------------------------------------------------------------------------------
class Client:
    """In-process stand-in for scannerpy.Client: same graph-building surface, runs on local GPUs."""

    def __init__(self, gpus=None, instances_per_gpu=0, cpu_instances=1, load_stdlib=True, db_path=None,
                 **_ignored):
        import torch
        if gpus is None:
            gpus = list(range(torch.cuda.device_count())) if torch.cuda.is_available() else []
        self._engine = E.Engine(gpus, instances_per_gpu, cpu_instances)
        self._gpus = list(gpus)
        # the reference always records a profile (get_profile after any job); interval records are a
        # few dozen bytes per task and kernel call, so it is on unless profiling=False is passed
        self._profiling = bool(_ignored.get("profiling", True))
        if self._profiling:
            self._engine.set_trace(True)
        self._db = E.Database(db_path) if db_path else None
        self._bulk_jobs = 0
        self._streams = {}
        self._op_protos = {}
        self.ops, self.streams, self.io = OpGenerator(self), StreamsGenerator(self), IOGenerator(self)
        self.partitioner = Partitioner()
        if load_stdlib:
            E.load_stdlib()
            std = protolite.parse_proto(open(os.path.join(os.path.dirname(E.ENGINE_PATH), "..", "csrc", "ops",
                                                          "stdlib_args.proto")).read())
            self._op_protos["Blur"] = {"init": std["BlurArgs"]}
            self._op_protos["Resize"] = {"stream": std["ResizeArgs"]}
            self._op_protos["ConvertColor"] = {"stream": std["ConvertColorArgs"]}
            self._op_protos["GaussianBlur"] = {"init": std["GaussianBlurArgs"]}
            self._op_protos["ImageEncoder"] = {"init": std["ImageEncoderArgs"]}
            self._op_protos["OpticalFlowTVL1"] = {"init": std["OpticalFlowTVL1Args"]}

    # ---- table catalogue (reference client.py: ingest_videos :1009-1078, has_table, delete_table)
    def _need_db(self):
        if self._db is None:
            raise ScannerException("this Client was created without db_path: there is no table catalogue")
        return self._db

    def ingest_videos(self, videos, inplace=False, force=False):
        """videos: [(table name, path)] -> (ingested NamedVideoStreams, [(path, error message)])."""
        db, done, failed = self._need_db(), [], []
        for name, path in videos:
            try:
                if db.has_table(name):
                    if not force:
                        raise ScannerException(f"table {name} already exists")
                    db.delete_table(name)
                    self._streams.pop(name, None)
                db.ingest_video(name, path, inplace=inplace)
                done.append(NamedVideoStream(self, name))
            except (E.EngineError, ScannerException) as e:
                failed.append((path, str(e)))
        return done, failed

    def new_table(self, name, columns, rows, fns=None, force=False):
        """A table of byte columns from Python rows (reference Client.new_table, client.py:1068-1121):
        `rows` is a list of rows, each a list with one serialized element per column."""
        db = self._need_db()
        if db.has_table(name):
            if not force:
                raise ScannerException(f"Attempted to create table with existing name {name}")
            db.delete_table(name)
        if fns is not None:
            rows = [[fn(col, None) for fn, col in zip(fns, row)] for row in rows]
        try:
            db.new_table_from_rows(name, list(columns), [list(r) for r in rows])
        except E.EngineError as e:
            raise ScannerException(str(e)) from e
        return self.table(name)

    def has_table(self, name):
        return self._need_db().has_table(name)

    def table(self, name):
        if not self._need_db().has_table(name):
            raise ScannerException(f"table {name} does not exist")
        return Table(self._db, name, self)

    def summarize(self):
        """Text table of the catalogue (reference client.py summarize): name, id, rows, columns."""
        lines = [f"{'name':<28} {'id':>4} {'rows':>9}  columns"]
        for n in sorted(self._need_db().tables()):
            t = Table(self._db, n)
            lines.append(f"{n:<28} {t.id():>4} {t.num_rows():>9}  {', '.join(t.column_names())}")
        return "\n".join(lines)

    def table_names(self):
        return self._need_db().tables()

    def delete_table(self, name):
        self._need_db().delete_table(name)
        self._streams.pop(name, None)

    def delete_tables(self, names):
        """Reference Client.delete_tables (client.py:1044-1056)."""
        for name in names:
            self.delete_table(name)

    def sequence(self, name):
        """The data column of a table (reference client.py:1158-1164): `frame` of a video table,
        else the single column a job wrote."""
        t = self.table(name)
        cols = [c for c in t.column_names() if c != "index"]
        return t.column("frame" if "frame" in cols else cols[0])

    def get_active_jobs(self):
        """run() returns when the job is done: there is never a job in flight to report."""
        return []

    def wait_on_job(self, bulk_job_id=None, show_progress=True):
        """Jobs run synchronously inside run(); kept so scripts that wait explicitly still work."""
        return None

    def load_op(self, so_path, proto_path=None, protos=None):
        """Load an op library (reference Client.load_op, client.py:514-537).  `protos` maps op name to
        {"init": MessageName, "stream": MessageName} inside `proto_path`."""
        E.load_op_library(so_path)
        if proto_path:
            msgs = protolite.parse_proto(open(proto_path).read())
            # the message names an op registered with (.protobuf_name / .stream_protobuf_name) are looked
            # up in the proto file, as the reference does with the compiled module (op.py:299-307)
            for op, info in E.list_ops().items():
                if op in self._op_protos:
                    continue
                found = {}
                if info["protobuf_name"] in msgs:
                    found["init"] = msgs[info["protobuf_name"]]
                if info["stream_protobuf_name"] in msgs:
                    found["stream"] = msgs[info["stream_protobuf_name"]]
                if found:
                    self._op_protos[op] = found
            for op, d in (protos or {}).items():
                self._op_protos[op] = {k: msgs[v] for k, v in d.items()}

    def _op_outputs(self, name):
        g = E.Graph()
        n_in = E.list_ops()[name]["inputs"]
        src = g.add_source(True)
        # a scratch graph only to ask the registry for the op's output columns
        idx = E.lib().scn_graph_add_op(g._h, name.encode(), 0, (E._c.c_int * max(1, n_in))(*([src] * n_in)),
                                       (E._c.c_char_p * max(1, n_in))(*([b"frame"] * n_in)), n_in, None, 0, -1,
                                       (E._c.c_int * 1)(), 0, -1)
        E.check(idx, f"op {name}")
        cols = g.op_outputs(idx)
        types = self._op_output_types.get(name) if hasattr(self, "_op_output_types") else None
        return [(c, (types or {}).get(c, c in ("frame", "flow"))) for c in cols]

    def run(self, outputs, perf_params, cache_mode=CacheMode.Error, show_progress=False, out_dir=None, **_ignored):
        outputs = outputs if isinstance(outputs, (list, tuple)) else [outputs]
        order, seen = [], set()

        def visit(node):
            if id(node) in seen:
                return
            seen.add(id(node))
            for c in node.inputs:
                visit(c._op)
            order.append(node)

        for o in outputs:
            visit(o)
        # ---- output tables that already exist (reference CacheMode, client.py:1325-1370)
        out_nodes = [n for n in order if n.kind == "output"]
        encodings = {id(n): _h264_encoding(n.inputs[0]) for n in out_nodes}
        skip = set()
        if self._db is not None and out_nodes:
            for j in range(len(out_nodes[0].streams)):
                present = [n.streams[j].name() for n in out_nodes if self._db.has_table(n.streams[j].name())]
                if not present:
                    continue
                if cache_mode == CacheMode.Error:
                    raise ScannerException(f"output stream {present[0]} already exists (CacheMode.Error)")
                if cache_mode == CacheMode.Overwrite:
                    for name in present:
                        self._db.delete_table(name)
                elif len(present) == len(out_nodes):
                    skip.add(j)  # CacheMode.Ignore: every output of this job is already stored
                else:
                    for name in present:
                        self._db.delete_table(name)
        g = E.Graph()
        index, n_jobs = {}, None
        for node in order:
            if node.kind == "input":
                index[id(node)] = g.add_source(isinstance(node.streams[0], NamedVideoStream))
                n_jobs = len(node.streams) if n_jobs is None else n_jobs
                if len(node.streams) != n_jobs:
                    raise ScannerException("all Inputs must list the same number of streams")
            elif node.kind == "op":
                ins = [(index[id(c._op)], c._col) for c in node.inputs]
                index[id(node)] = g.add_op(node.name, ins, int(node.device), node.args, node.batch, node.stencil,
                                           node.warmup)
            elif node.kind in ("sample", "space", "slice", "unslice"):
                c = node.inputs[0]
                fn = {"sample": g.add_sample, "space": g.add_space, "slice": g.add_slice, "unslice": g.add_unslice}[
                    node.kind]
                index[id(node)] = fn((index[id(c._op)], c._col))
            elif node.kind == "output":
                c = node.inputs[0]
                index[id(node)] = g.add_sink((index[id(c._op)], c._col), node.streams[0].name())
        jobs, job_of = [], {}
        for j in range(n_jobs):
            if j in skip:
                continue
            job_of[j] = len(jobs)
            job = E.Job()
            for node in order:
                if node.kind == "input":
                    st = node.streams[j]
                    job.bind_source(index[id(node)], st._bind())
                elif node.kind in ("sample", "space"):
                    args = node.per_stream[j if len(node.per_stream) > 1 else 0]
                    if isinstance(args, SliceList):
                        for grp, a in enumerate(args):
                            job.set_group_sampler(index[id(node)], grp, node.sampler, a)
                    else:
                        job.set_sampler(index[id(node)], node.sampler, args)
                elif node.kind == "slice":
                    name, args = node.per_stream[j if len(node.per_stream) > 1 else 0]
                    job.set_partitioner(index[id(node)], name, args)
                elif node.kind == "op" and node.per_stream:
                    args = node.per_stream[j if len(node.per_stream) > 1 else 0]
                    if isinstance(args, SliceList):
                        for grp, a in enumerate(args):
                            job.set_group_stream_args(index[id(node)], grp, a)
                    else:
                        job.set_stream_args(index[id(node)], args)
            jobs.append(job)
        bulk_job_id = self._bulk_jobs
        self._bulk_jobs += 1
        # with a database the save stage writes every finished task as an item of the output
        # stream's table and drops the rows from memory (reference SaveWorker / ColumnSink)
        reserved = []  # (table id, table name, job)
        if self._db is not None:
            try:
                for node in out_nodes:
                    src_col = node.inputs[0]
                    type_name = _column_type_name(src_col)
                    for j, s in enumerate(node.streams):
                        if j in skip:
                            continue
                        tid = self._db.new_table(s.name(), src_col._col, src_col._is_frame, type_name, bulk_job_id)
                        reserved.append((tid, s.name(), jobs[job_of[j]]))
                        jobs[job_of[j]].set_sink_table(index[id(node)], tid, keep_rows=False)
                        if encodings[id(node)] and self._gpus:
                            jobs[job_of[j]].set_sink_encoding(index[id(node)], *encodings[id(node)])
            except E.EngineError as e:
                for _, name, _ in reserved:
                    self._db.delete_table(name)
                raise ScannerException(str(e)) from e
            out_dir = self._db.path
        try:
            if jobs:
                self._engine.run(g, jobs, perf_params.work_packet_size, perf_params.io_packet_size, out_dir)
            for tid, _, job in reserved:
                self._db.commit_job_table(tid, job)
        except E.EngineError as e:
            for _, name, _ in reserved:
                try:
                    self._db.delete_table(name)
                except E.EngineError:
                    pass
            raise ScannerException(str(e)) from e
        for node in out_nodes:
            src_col = node.inputs[0]
            type_name = _column_type_name(src_col)
            for j, s in enumerate(node.streams):
                if j not in skip:  # freshly written: an input binding made from older rows is stale
                    s._sid = None
                    self._streams.pop(s.name(), None)
                if j in skip or self._db is not None:
                    s._job = None  # served from the stored table
                    continue
                s._job, s._sink = jobs[job_of[j]], index[id(node)]
                s._type = type_name or None
        for node in out_nodes:
            for j, s in enumerate(node.streams):
                if j not in skip and hasattr(s, "_after_run"):
                    s._after_run()
        self._last_graph = g
        return len(jobs)

    def stats(self):
        return self._engine.stats()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.stop()
        return False

    def has_gpu(self):
        """True if this client's engine drives at least one GPU (reference Client.has_gpu)."""
        return bool(self._gpus)

    def get_profile(self, job_id=None):
        """Like scannerpy's `sc.get_profile(job_id)` for the last run: `.statistics()` and, if the
        client was created with profiling=True, `.write_trace(path)` (Chrome trace events)."""
        return Profile(self)

    def stop(self):
        self._engine.close()
        if self._db is not None:
            self._db.close()
