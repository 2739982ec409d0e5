"""ctypes binding of include/scn_engine.h (libscn_engine.so) -- the C++ host pipeline."""
import ctypes
import json
import os
import sys

import numpy as np

from . import cabi

_HERE = os.path.dirname(os.path.abspath(__file__))
ENGINE_PATH = os.path.join(_HERE, "lib", "libscn_engine.so")
STDLIB_PATH = os.path.join(_HERE, "lib", "libscn_stdlib.so")

_c = ctypes
_VP, _I, _I64, _SZ, _CP = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_size_t, _c.c_char_p
_IP = _c.POINTER(_c.c_int)

SIGNATURES = {
    "scn_last_error": (_CP, []),
    "scn_load_op_library": (_I, [_CP]),
    "scn_op_registered": (_I, [_CP]),
    "scn_kernel_registered": (_I, [_CP, _I]),
    "scn_list_ops": (_I, [_CP, _SZ]),
    "scn_engine_create": (_VP, [_IP, _I, _I, _I]),
    "scn_engine_destroy": (None, [_VP]),
    "scn_stream_add_h264": (_I64, [_VP, _VP, _SZ]),
    "scn_stream_add_raw_frames": (_I64, [_VP, _VP, _I64, _I, _I, _I, _I]),
    "scn_stream_add_bytes": (_I64, [_VP, _VP, _VP, _I64]),
    "scn_stream_rows": (_I64, [_VP, _I64]),
    "scn_stream_may_reorder": (_I, [_VP, _I64]),
    "scn_db_ingest_video_inplace": (_I, [_VP, _CP, _CP]),
    "scn_db_new_table_from_rows": (_I, [_VP, _CP, _I, _VP, _I64, _VP, _VP]),
    # host-language kernels: pyops.py binds the struct / callback types over these
    "scn_register_callback_op": (_I, [_VP, _VP, _VP]),
    "scn_cb_emit_bytes": (_I, [_VP, _I, _VP, _SZ]),
    "scn_cb_emit_frame": (_I, [_VP, _I, _VP, _I, _I, _I, _I]),
    "scn_stream_info": (_I, [_VP, _I64, _c.POINTER(_I64)]),
    "scn_stream_remove": (_I, [_VP, _I64]),
    "scn_engine_decode_to_device": (_I, [_VP, _I64, _c.POINTER(_I64), _I64, _I, _VP]),
    "scn_graph_create": (_VP, []),
    "scn_graph_destroy": (None, [_VP]),
    "scn_graph_add_source": (_I, [_VP, _I]),
    "scn_graph_add_op": (_I, [_VP, _CP, _I, _IP, _c.POINTER(_CP), _I, _VP, _SZ, _I, _IP, _I, _I]),
    "scn_graph_add_sample": (_I, [_VP, _I, _CP]),
    "scn_graph_add_space": (_I, [_VP, _I, _CP]),
    "scn_graph_add_sink": (_I, [_VP, _I, _CP, _CP]),
    "scn_graph_op_outputs": (_I, [_VP, _I, _CP, _SZ]),
    "scn_job_create": (_VP, []),
    "scn_job_destroy": (None, [_VP]),
    "scn_job_bind_source": (_I, [_VP, _I, _I64]),
    "scn_job_set_sampler": (_I, [_VP, _I, _CP, _VP, _SZ]),
    "scn_job_set_stream_args": (_I, [_VP, _I, _VP, _SZ]),
    "scn_engine_run": (_I, [_VP, _VP, _c.POINTER(_VP), _I, _I, _I, _CP]),
    "scn_job_output_rows": (_I64, [_VP, _I]),
    "scn_job_output_row": (_I, [_VP, _I, _I64, _c.POINTER(_VP), _c.POINTER(_c.c_uint64), _IP]),
    "scn_job_output_copy": (_I, [_VP, _I, _I64, _I64, _VP, _SZ]),
    "scn_engine_stats_json": (_I, [_VP, _CP, _SZ]),
    "scn_h264_synth": (_I64, [_VP, _I, _I, _I64, _I, _I, _VP, _SZ]),
    "scn_engine_share_task_queue": (_I, [_VP, _CP]),
    "scn_engine_reset_task_queue": (_I, [_VP]),
    "scn_nvdec_caps": (_I, [_I, _IP]),
    "scn_swdec_caps": (_I, [_IP]),
    "scn_graph_add_slice": (_I, [_VP, _I, _CP]),
    "scn_graph_add_unslice": (_I, [_VP, _I, _CP]),
    "scn_job_set_partitioner": (_I, [_VP, _I, _CP, _VP, _SZ]),
    "scn_job_set_group_sampler": (_I, [_VP, _I, _I, _CP, _VP, _SZ]),
    "scn_job_set_group_stream_args": (_I, [_VP, _I, _I, _VP, _SZ]),
    "scn_engine_comm_unique_id": (_I, [_VP]),
    "scn_engine_comm_init": (_I, [_VP, _I, _I, _I, _VP]),
    "scn_engine_set_halo_callback": (_I, [_VP, _I, _I, _VP, _VP]),
    "scn_job_set_shard": (_I, [_VP, _I, _I, _c.POINTER(_I64), _IP]),
    "scn_engine_set_trace": (_I, [_VP, _I]),
    "scn_engine_write_trace": (_I, [_VP, _CP]),
    "scn_db_open": (_VP, [_CP]),
    "scn_db_close": (None, [_VP]),
    "scn_db_ingest_video": (_I, [_VP, _CP, _CP]),
    "scn_db_ingest_h264": (_I, [_VP, _CP, _VP, _SZ, _I, _I]),
    "scn_db_has_table": (_I, [_VP, _CP]),
    "scn_db_delete_table": (_I, [_VP, _CP]),
    "scn_db_list_tables": (_I, [_VP, _CP, _SZ]),
    "scn_db_table_info": (_I, [_VP, _CP, _c.POINTER(_I64), _CP, _SZ]),
    "scn_db_add_video_stream": (_I64, [_VP, _VP, _CP]),
    "scn_db_save_job": (_I, [_VP, _VP, _CP, _IP, _c.POINTER(_CP), _c.POINTER(_CP), _I, _I]),
    "scn_db_new_table": (_I, [_VP, _CP, _CP, _I, _CP, _I]),
    "scn_job_set_sink_table": (_I, [_VP, _I, _I, _I]),
    "scn_job_set_sink_encoding": (_I, [_VP, _I, _I, _I]),
    "scn_db_new_tables": (_I, [_VP, _I, _c.POINTER(_CP), _c.POINTER(_CP), _IP, _c.POINTER(_CP), _IP, _IP]),
    "scn_db_commit_job_tables": (_I, [_VP, _I, _IP, _c.POINTER(_VP)]),
    "scn_db_delete_tables": (_I, [_VP, _I, _c.POINTER(_CP)]),
    "scn_db_commit_job_table": (_I, [_VP, _I, _VP]),
    "scn_db_read_rows": (_VP, [_VP, _CP, _CP, _c.POINTER(_I64), _I64]),
    "scn_rows_count": (_I64, [_VP]),
    "scn_rows_get": (_I, [_VP, _I64, _c.POINTER(_VP), _c.POINTER(_c.c_uint64), _IP]),
    "scn_rows_free": (None, [_VP]),
    "scn_db_export_mp4": (_I, [_VP, _CP, _CP, _I, _I]),
    "scn_mp4_mux": (_I64, [_VP, _SZ, _I, _I, _VP, _SZ]),
    "scn_mp4_demux": (_I64, [_VP, _SZ, _VP, _SZ, _c.POINTER(_I64)]),
}

_lib = None


class EngineError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ENGINE_PATH):
            raise EngineError(f"{ENGINE_PATH} not found: run __graft_entry__.build()")
        cabi.lib()  # the engine links libscn_kernels.so
        if "SCN_FFMPEG_DIR" not in os.environ:  # where CPU instances find libavcodec (swdec.h); unused by GPU instances
            d = _default_ffmpeg_dir()
            if d:
                os.environ["SCN_FFMPEG_DIR"] = d
        l = ctypes.CDLL(ENGINE_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def last_error():
    return lib().scn_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc is None or rc < 0:
        raise EngineError(f"{what}: {last_error()}")
    return rc


def load_op_library(path):
    check(lib().scn_load_op_library(os.path.abspath(path).encode()), f"load_op({path})")


_stdlib_loaded = False


def load_stdlib():
    global _stdlib_loaded
    if not _stdlib_loaded:
        load_op_library(STDLIB_PATH)
        _stdlib_loaded = True


def list_ops():
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib().scn_list_ops(buf, len(buf)), "scn_list_ops")
    out = {}
    for line in buf.value.decode().splitlines():
        n, ni, no, st, b, ub, w, *names = line.split(":")
        out[n] = dict(inputs=int(ni), outputs=int(no), can_stencil=bool(int(st)), bounded=bool(int(b)),
                      unbounded=bool(int(ub)), warmup=int(w), protobuf_name=names[0] if names else "",
                      stream_protobuf_name=names[1] if len(names) > 1 else "")
    return out


def _default_ffmpeg_dir():
    """The FFmpeg build this image ships: inside the opencv-python-headless wheel (no system libavcodec here).
    Only a path is computed -- cv2 is not imported."""
    import importlib.util
    spec = importlib.util.find_spec("cv2")
    if not spec or not spec.origin:
        return None
    site = os.path.dirname(os.path.dirname(spec.origin))
    for name in ("opencv_python_headless.libs", "opencv_python.libs", "opencv_contrib_python_headless.libs"):
        d = os.path.join(site, name)
        if os.path.isdir(d) and any(f.startswith("libavcodec") for f in os.listdir(d)):
            return d
    return None


def swdec_caps():
    """Software (CPU instance) H.264 decoder: FFmpeg libraries found and their majors.  SCN_FFMPEG_DIR selects the
    directory; when it is unset and the image's OpenCV wheel bundles FFmpeg, that copy is used."""
    info = (ctypes.c_int * 4)()
    lib().scn_swdec_caps(info)
    d = dict(zip(["available", "avcodec", "avutil", "swscale"], list(info)))
    d["where" if d["available"] else "error"] = last_error()
    return d


def nvdec_caps(gpu=0):
    info = (ctypes.c_int * 6)()
    lib().scn_nvdec_caps(gpu, info)
    keys = ["available", "h264", "engines", "max_w", "max_h", "min_w"]
    d = dict(zip(keys, list(info)))
    if not d["available"]:
        d["error"] = last_error()
    return d


def h264_synth(yuv_frames, width, height, gop=30, non_key="pcm", frames=None):
    """yuv_frames: uint8 I420 pictures, flat (k, w*h*3/2) (Y plane, then U, then V).
    non_key="pcm": k = number of frames, every picture is coded (P slices of I_PCM macroblocks
    between IDRs).  non_key="skip": k = number of GOPs, `frames` total pictures are emitted, the
    non-key ones as P_Skip repeats.  non_key="bidir": k = number of frames; odd GOP positions with a
    later anchor in the GOP become B pictures coded after that anchor (decode order != display
    order), decoding to the rounded mean of the two anchors -- see bidir_expected().
    Returns the Annex-B stream as bytes."""
    arr = np.ascontiguousarray(yuv_frames, dtype=np.uint8).reshape(len(yuv_frames), -1)
    assert arr.shape[1] == width * height * 3 // 2
    mode = {"pcm": 0, "skip": 1, "bidir": 2}[non_key]
    if mode == 1:
        n = frames if frames is not None else arr.shape[0] * gop
        assert arr.shape[0] >= (n + gop - 1) // gop
    else:
        n = arr.shape[0]
    need = lib().scn_h264_synth(arr.ctypes.data, width, height, n, gop, mode, None, 0)
    check(need, "scn_h264_synth")
    out = np.empty(need, np.uint8)
    got = lib().scn_h264_synth(arr.ctypes.data, width, height, n, gop, mode, out.ctypes.data, out.size)
    assert got == need
    return out.tobytes()


def bidir_expected(yuv_frames, gop):
    """What a decoder shows, in display order, for h264_synth(yuv_frames, ..., non_key="bidir")."""
    src = np.asarray(yuv_frames, dtype=np.uint8)
    out = src.copy()
    n = len(src)
    for g0 in range(0, n, gop):
        ln = min(gop, n - g0)
        for k in range(1, ln - 1, 2):
            out[g0 + k] = ((src[g0 + k - 1].astype(np.uint16) + src[g0 + k + 1] + 1) >> 1).astype(np.uint8)
    return out


def mp4_mux(annexb, fps_num=25, fps_den=1):
    """H.264 Annex-B bytes -> the bytes of a non-fragmented .mp4 holding that one track."""
    buf = np.frombuffer(bytes(annexb), np.uint8)
    need = check(lib().scn_mp4_mux(buf.ctypes.data, buf.size, fps_num, fps_den, None, 0), "scn_mp4_mux")
    out = np.empty(need, np.uint8)
    check(lib().scn_mp4_mux(buf.ctypes.data, buf.size, fps_num, fps_den, out.ctypes.data, out.size), "scn_mp4_mux")
    return out.tobytes()


def mp4_demux(data):
    """.mp4/.mov bytes -> (Annex-B stream of the first H.264 track, info dict)."""
    buf = np.frombuffer(bytes(data), np.uint8)
    info = (ctypes.c_int64 * 6)()
    need = check(lib().scn_mp4_demux(buf.ctypes.data, buf.size, None, 0, info), "scn_mp4_demux")
    out = np.empty(need, np.uint8)
    check(lib().scn_mp4_demux(buf.ctypes.data, buf.size, out.ctypes.data, out.size, info), "scn_mp4_demux")
    keys = ["width", "height", "timescale", "duration", "samples", "sync_samples"]
    return out.tobytes(), dict(zip(keys, list(info)))


class Database:
    """A Scanner database directory (reference layout: db_metadata.bin, tables/<id>/...)."""

    def __init__(self, path):
        self._h = lib().scn_db_open(os.path.abspath(path).encode())
        if not self._h:
            raise EngineError(f"scn_db_open({path}): {last_error()}")
        self.path = os.path.abspath(path)

    def close(self):
        if self._h:
            lib().scn_db_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def ingest_video(self, table, video_path, inplace=False):
        """inplace: keep the bitstream where it is (the table records the path) instead of copying it"""
        fn = lib().scn_db_ingest_video_inplace if inplace else lib().scn_db_ingest_video
        check(fn(self._h, table.encode(), os.path.abspath(video_path).encode()), f"ingest_video({video_path})")

    def ingest_h264(self, table, data, fps_num=25, fps_den=1):
        buf = np.frombuffer(bytes(data), np.uint8)
        check(lib().scn_db_ingest_h264(self._h, table.encode(), buf.ctypes.data, buf.size, fps_num, fps_den),
              f"ingest_h264({table})")

    def export_mp4(self, table, out_path, fps_num=0, fps_den=0):
        check(lib().scn_db_export_mp4(self._h, table.encode(), os.path.abspath(out_path).encode(), fps_num, fps_den),
              f"export_mp4({table})")

    def has_table(self, table):
        return bool(lib().scn_db_has_table(self._h, table.encode()))

    def delete_table(self, table):
        check(lib().scn_db_delete_table(self._h, table.encode()), f"delete_table({table})")

    def tables(self):
        buf = ctypes.create_string_buffer(1 << 20)
        check(lib().scn_db_list_tables(self._h, buf, len(buf)), "scn_db_list_tables")
        return [t for t in buf.value.decode().split("\n") if t]

    def table_info(self, table):
        info = (ctypes.c_int64 * 8)()
        cols = ctypes.create_string_buffer(1 << 16)
        check(lib().scn_db_table_info(self._h, table.encode(), info, cols, len(cols)), f"table_info({table})")
        d = dict(zip(["id", "rows", "num_columns", "items", "job_id", "width", "height", "keyframes"], list(info)))
        d["columns"] = []
        for line in cols.value.decode().splitlines():
            n, t, tn = line.split(":", 2)
            d["columns"].append({"name": n, "type": "Video" if int(t) == 1 else "Bytes", "type_name": tn})
        return d

    def add_video_stream(self, engine, table):
        return check(lib().scn_db_add_video_stream(self._h, engine._h, table.encode()), f"add_video_stream({table})")

    def new_table_from_rows(self, table, columns, rows):
        """rows: list of rows, each a list of bytes (or None) per column -> table id"""
        n_cols, n_rows = len(columns), len(rows)
        names = (ctypes.c_char_p * n_cols)(*[c.encode() for c in columns])
        cells = [None if v is None else bytes(v) for row in rows for v in row]
        if len(cells) != n_cols * n_rows:
            raise EngineError(f"new_table_from_rows({table}): every row must have {n_cols} elements")
        keep = [ctypes.create_string_buffer(v, len(v)) if v else None for v in cells]
        ptrs = (ctypes.c_void_p * max(1, len(cells)))(*[ctypes.addressof(b) if b is not None else None for b in keep])
        sizes = (ctypes.c_uint64 * max(1, len(cells)))(*[len(v) if v else 0 for v in cells])
        return check(lib().scn_db_new_table_from_rows(self._h, table.encode(), n_cols, names, n_rows, ptrs, sizes),
                     f"new_table_from_rows({table})")

    def new_table(self, table, column, is_video=False, type_name="", job_id=-1):
        """Reserve a one-column table a job will save into while it runs -> table id."""
        return check(lib().scn_db_new_table(self._h, table.encode(), column.encode(), 1 if is_video else 0,
                                            (type_name or "").encode(), job_id), f"new_table({table})")

    def new_tables(self, specs):
        """specs: [(table, column, is_video, type_name, job_id)] -> table ids, under one catalogue lock."""
        n = len(specs)
        names = (ctypes.c_char_p * n)(*[s[0].encode() for s in specs])
        cols = (ctypes.c_char_p * n)(*[s[1].encode() for s in specs])
        vid = (ctypes.c_int * n)(*[1 if s[2] else 0 for s in specs])
        tys = (ctypes.c_char_p * n)(*[(s[3] or "").encode() for s in specs])
        jids = (ctypes.c_int * n)(*[int(s[4]) for s in specs])
        out = (ctypes.c_int * n)()
        check(lib().scn_db_new_tables(self._h, n, names, cols, vid, tys, jids, out), "new_tables")
        return list(out)

    def commit_job_tables(self, pairs):
        """pairs: [(table id, job)], under one catalogue lock."""
        n = len(pairs)
        ids = (ctypes.c_int * n)(*[p[0] for p in pairs])
        jobs = (ctypes.c_void_p * n)(*[p[1]._h for p in pairs])
        check(lib().scn_db_commit_job_tables(self._h, n, ids, jobs), "commit_job_tables")

    def delete_tables(self, tables):
        n = len(tables)
        names = (ctypes.c_char_p * n)(*[t.encode() for t in tables])
        check(lib().scn_db_delete_tables(self._h, n, names), "delete_tables")

    def commit_job_table(self, table_id, job):
        check(lib().scn_db_commit_job_table(self._h, table_id, job._h), "commit_job_table")

    def save_job(self, job, table, columns, job_id=-1):
        """columns: [(sink op index, column name, type name)] -> table id"""
        n = len(columns)
        sinks = (ctypes.c_int * n)(*[c[0] for c in columns])
        names = (ctypes.c_char_p * n)(*[c[1].encode() for c in columns])
        types = (ctypes.c_char_p * n)(*[(c[2] or "").encode() for c in columns])
        return check(lib().scn_db_save_job(self._h, job._h, table.encode(), sinks, names, types, n, job_id),
                     f"save_job({table})")

    def read_rows(self, table, column, rows=None):
        """-> list of rows: bytes for byte columns, ndarrays for frame columns, None for null rows."""
        if rows is None:
            rows = range(self.table_info(table)["rows"])
        rows = list(rows)
        arr = (ctypes.c_int64 * max(1, len(rows)))(*rows)
        h = lib().scn_db_read_rows(self._h, table.encode(), column.encode(), arr, len(rows))
        if not h:
            raise EngineError(f"read_rows({table}.{column}): {last_error()}")
        try:
            out = []
            for i in range(lib().scn_rows_count(h)):
                data, size, shape = ctypes.c_void_p(), ctypes.c_uint64(), (ctypes.c_int * 4)()
                check(lib().scn_rows_get(h, i, ctypes.byref(data), ctypes.byref(size), shape), "scn_rows_get")
                out.append(_row_to_python(data.value, size.value, list(shape)))
            return out
        finally:
            lib().scn_rows_free(h)


_FRAME_DTYPES = {0: np.uint8, 1: np.float32, 2: np.float64, 3: np.uint16}


def _row_to_python(addr, size, shape):
    if size == 0:
        return None
    raw = ctypes.string_at(addr, size)
    if shape[3] >= 0:
        return np.frombuffer(raw, _FRAME_DTYPES[shape[3]]).reshape(shape[0], shape[1], shape[2]).copy()
    return raw


class Engine:
    def __init__(self, gpus=(), instances_per_gpu=0, cpu_instances=1):
        gpus = list(gpus)
        arr = (ctypes.c_int * max(1, len(gpus)))(*gpus)
        self._h = lib().scn_engine_create(arr, len(gpus), instances_per_gpu, cpu_instances)
        self.gpus = gpus

    def close(self):
        if self._h:
            lib().scn_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def share_task_queue(self, path):
        """Take tasks from a queue shared with the engines of other processes that run the same job list
        (scn_engine_share_task_queue); None returns to the private queue."""
        check(lib().scn_engine_share_task_queue(self._h, path.encode() if path else None), "share_task_queue")

    def reset_task_queue(self):
        check(lib().scn_engine_reset_task_queue(self._h), "reset_task_queue")

    def add_h264(self, data):
        buf = np.frombuffer(data, np.uint8)
        return check(lib().scn_stream_add_h264(self._h, buf.ctypes.data, buf.size), "add_h264")

    def add_raw_frames(self, frames):
        frames = np.ascontiguousarray(frames)
        tcode = {np.dtype(np.uint8): 0, np.dtype(np.float32): 1, np.dtype(np.float64): 2, np.dtype(np.uint16): 3}[
            frames.dtype]
        n, h, w, c = frames.shape
        return check(lib().scn_stream_add_raw_frames(self._h, frames.ctypes.data, n, h, w, c, tcode), "add_raw_frames")

    def add_bytes(self, rows):
        sizes = np.array([len(r) for r in rows], np.uint64)
        data = np.frombuffer(b"".join(bytes(r) for r in rows) or b"\0", np.uint8)
        return check(lib().scn_stream_add_bytes(self._h, data.ctypes.data, sizes.ctypes.data, len(rows)), "add_bytes")

    # ---- one clip across several ranks: stencil halo exchange (include/scn_engine.h) ----
    def init_comm(self, gpu, group=None):
        """NCCL transport between the ranks' GPUs for the halo exchange of sharded jobs.  Collective over
        the torch.distributed group: rank 0's ncclUniqueId travels through broadcast_object_list."""
        import torch.distributed as dist
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        ident = (ctypes.c_uint8 * 128)()
        if rank == 0:
            check(lib().scn_engine_comm_unique_id(ident), "comm_unique_id")
        box = [bytes(ident)]
        dist.broadcast_object_list(box, src=0, group=group)
        ident = (ctypes.c_uint8 * 128).from_buffer_copy(box[0])
        check(lib().scn_engine_comm_init(self._h, gpu, rank, world, ident), "comm_init")

    def init_host_halo(self, group=None):
        """Host transport for the halo exchange (CPU instances over raw-frame streams): the buffers are
        moved with torch.distributed point-to-point operations of `group` (gloo)."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(group), dist.get_world_size(group)

        def exchange(_user, n, peers, buffers, nbytes, is_send):
            try:
                ops = []
                for i in range(n):
                    arr = np.ctypeslib.as_array(ctypes.cast(buffers[i], ctypes.POINTER(ctypes.c_uint8)), shape=(nbytes[i],))
                    t = torch.from_numpy(arr)
                    ops.append(dist.P2POp(dist.isend if is_send[i] else dist.irecv, t, peers[i], group))
                for req in dist.batch_isend_irecv(ops):
                    req.wait()
                return 0
            except Exception as e:  # noqa: BLE001 -- reported through the C return code
                sys.stderr.write(f"halo exchange failed: {e}\n")
                return 1

        proto = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                 ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int))
        self._halo_cb = proto(exchange)  # keep the trampoline alive as long as the engine
        check(lib().scn_engine_set_halo_callback(self._h, rank, world, ctypes.cast(self._halo_cb, ctypes.c_void_p), None),
              "set_halo_callback")

    def set_trace(self, on=True):
        """Keep every profiler interval of the following runs (see write_trace)."""
        check(lib().scn_engine_set_trace(self._h, 1 if on else 0), "set_trace")

    def write_trace(self, path):
        """The last run as a Chrome trace-event JSON file (pid = GPU, tid = pipeline instance)."""
        check(lib().scn_engine_write_trace(self._h, os.path.abspath(path).encode()), "write_trace")

    def stream_rows(self, sid):
        return check(lib().scn_stream_rows(self._h, sid), "stream_rows")

    def stream_info(self, sid):
        info = (ctypes.c_int64 * 6)()
        check(lib().scn_stream_info(self._h, sid, info), "stream_info")
        return dict(zip(["is_video", "width", "height", "channels", "keyframes", "bytes"], list(info)))

    def stream_may_reorder(self, sid):
        return bool(check(lib().scn_stream_may_reorder(self._h, sid), "stream_may_reorder"))

    def decode_to_device(self, sid, rows, gpu=0):
        """Decode `rows` (ascending) of an H.264 stream into a (n,h,w,3) uint8 CUDA tensor."""
        import torch
        info = self.stream_info(sid)
        rows = list(rows)
        out = torch.empty((len(rows), info["height"], info["width"], 3), dtype=torch.uint8, device=f"cuda:{gpu}")
        arr = (ctypes.c_int64 * max(1, len(rows)))(*rows)
        torch.cuda.synchronize(gpu)
        check(lib().scn_engine_decode_to_device(self._h, sid, arr, len(rows), gpu, out.data_ptr()), "decode_to_device")
        return out

    def remove_stream(self, sid):
        check(lib().scn_stream_remove(self._h, sid), "remove_stream")

    def run(self, graph, jobs, work_packet_size, io_packet_size, out_dir=None):
        arr = (ctypes.c_void_p * len(jobs))(*[j._h for j in jobs])
        rc = lib().scn_engine_run(self._h, graph._h, arr, len(jobs), work_packet_size, io_packet_size,
                                  out_dir.encode() if out_dir else None)
        check(rc, "scn_engine_run")

    def stats(self):
        buf = ctypes.create_string_buffer(1 << 18)
        check(lib().scn_engine_stats_json(self._h, buf, len(buf)), "stats")
        return json.loads(buf.value.decode())


class Graph:
    def __init__(self):
        self._h = lib().scn_graph_create()

    def __del__(self):
        if getattr(self, "_h", None):
            lib().scn_graph_destroy(self._h)
            self._h = None

    def add_source(self, is_video=True):
        return check(lib().scn_graph_add_source(self._h, int(is_video)), "add_source")

    def add_op(self, name, inputs, device=0, args=b"", batch=-1, stencil=(), warmup=-1):
        n = len(inputs)
        ops = (ctypes.c_int * max(1, n))(*[i[0] for i in inputs])
        cols = (ctypes.c_char_p * max(1, n))(*[i[1].encode() for i in inputs])
        st = (ctypes.c_int * max(1, len(stencil)))(*stencil)
        abuf = ctypes.create_string_buffer(args, len(args)) if args else None
        return check(lib().scn_graph_add_op(self._h, name.encode(), int(device), ops, cols, n,
                                            ctypes.cast(abuf, ctypes.c_void_p) if abuf else None, len(args), batch,
                                            st, len(stencil), warmup), f"add_op({name})")

    def add_sample(self, inp):
        return check(lib().scn_graph_add_sample(self._h, inp[0], inp[1].encode()), "add_sample")

    def add_space(self, inp):
        return check(lib().scn_graph_add_space(self._h, inp[0], inp[1].encode()), "add_space")

    def add_slice(self, inp):
        return check(lib().scn_graph_add_slice(self._h, inp[0], inp[1].encode()), "add_slice")

    def add_unslice(self, inp):
        return check(lib().scn_graph_add_unslice(self._h, inp[0], inp[1].encode()), "add_unslice")

    def add_sink(self, inp, name=None):
        return check(lib().scn_graph_add_sink(self._h, inp[0], inp[1].encode(), (name or inp[1]).encode()), "add_sink")

    def op_outputs(self, idx):
        buf = ctypes.create_string_buffer(4096)
        check(lib().scn_graph_op_outputs(self._h, idx, buf, len(buf)), "op_outputs")
        return [c for c in buf.value.decode().split("\n") if c]


class Job:
    def __init__(self):
        self._h = lib().scn_job_create()

    def __del__(self):
        if getattr(self, "_h", None):
            lib().scn_job_destroy(self._h)
            self._h = None

    def bind_source(self, op, stream_id):
        check(lib().scn_job_bind_source(self._h, op, stream_id), "bind_source")

    def set_sampler(self, op, function, args=b""):
        buf = ctypes.create_string_buffer(args, len(args)) if args else None
        check(lib().scn_job_set_sampler(self._h, op, function.encode(), ctypes.cast(buf, ctypes.c_void_p) if buf else None,
                                        len(args)), f"set_sampler({function})")

    def set_shard(self, index, bounds, ranks):
        """This job computes output rows [bounds[index], bounds[index+1]) of its clip; interval q belongs to
        rank ranks[q] (rows a stencil needs from a neighbouring interval come from that rank)."""
        n = len(ranks)
        assert len(bounds) == n + 1
        b = (ctypes.c_int64 * (n + 1))(*[int(x) for x in bounds])
        r = (ctypes.c_int * n)(*[int(x) for x in ranks])
        check(lib().scn_job_set_shard(self._h, int(index), n, b, r), "set_shard")

    def set_partitioner(self, slice_op, name, args):
        buf = ctypes.create_string_buffer(args, len(args)) if args else None
        check(lib().scn_job_set_partitioner(self._h, slice_op, name.encode(),
                                            ctypes.cast(buf, ctypes.c_void_p) if buf else None, len(args)),
              f"set_partitioner({name})")

    def set_group_sampler(self, op, group, function, args=b""):
        buf = ctypes.create_string_buffer(args, len(args)) if args else None
        check(lib().scn_job_set_group_sampler(self._h, op, group, function.encode(),
                                              ctypes.cast(buf, ctypes.c_void_p) if buf else None, len(args)),
              f"set_group_sampler({function})")

    def set_group_stream_args(self, op, group, args):
        buf = ctypes.create_string_buffer(args, len(args)) if args else None
        check(lib().scn_job_set_group_stream_args(self._h, op, group,
                                                  ctypes.cast(buf, ctypes.c_void_p) if buf else None, len(args)),
              "set_group_stream_args")

    def set_sink_table(self, sink, table_id, keep_rows=False):
        check(lib().scn_job_set_sink_table(self._h, sink, table_id, 1 if keep_rows else 0), "set_sink_table")

    def set_sink_encoding(self, sink, qp=23, keyframe_distance=120):
        """Store the sink's frames as intra-only H.264 at constant QP (scn_job_set_sink_encoding)."""
        check(lib().scn_job_set_sink_encoding(self._h, sink, int(qp), int(keyframe_distance)), "set_sink_encoding")

    def set_stream_args(self, op, args):
        buf = ctypes.create_string_buffer(args, len(args)) if args else None
        check(lib().scn_job_set_stream_args(self._h, op, ctypes.cast(buf, ctypes.c_void_p) if buf else None, len(args)),
              "set_stream_args")

    def output_rows(self, sink):
        return check(lib().scn_job_output_rows(self._h, sink), "output_rows")

    def output_row(self, sink, row):
        """-> bytes for a byte row, ndarray for a frame row, None for a null row."""
        data, size, shape = ctypes.c_void_p(), ctypes.c_uint64(), (ctypes.c_int * 4)()
        check(lib().scn_job_output_row(self._h, sink, row, ctypes.byref(data), ctypes.byref(size), shape),
              "output_row")
        if size.value == 0:
            return None
        raw = ctypes.string_at(data.value, size.value)
        if shape[3] >= 0:
            dt = {0: np.uint8, 1: np.float32, 2: np.float64, 3: np.uint16}[shape[3]]
            return np.frombuffer(raw, dt).reshape(shape[0], shape[1], shape[2])
        return raw

    def output_array(self, sink, row_bytes, dtype=np.uint8, row0=0):
        """All rows of equal size as one (n, row_bytes/itemsize) array.  row0: first row id the job computed
        (a sharded job addresses its rows by their position in the whole clip)."""
        n = self.output_rows(sink)
        out = np.empty((n, row_bytes), np.uint8)
        check(lib().scn_job_output_copy(self._h, sink, row0, n, out.ctypes.data, row_bytes), "output_copy")
        return out.view(dtype)
