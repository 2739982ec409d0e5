/*
 * scn_engine.h -- C ABI of the scanner-b200 host pipeline (libscn_engine.so).
 *
 * What a foreign binding (the scannerpy-shaped Python layer in scanner_b200/, or a cgo/JNI stub)
 * drives: register op plugins, describe an op graph, bind per-job streams and run the
 * load -> decode -> evaluate -> save pipeline of the reference's worker
 * (scanner/engine/worker.cpp:868-2148 process_job; load_worker.cpp, evaluate_worker.cpp,
 * save_worker.cpp) on the GPUs of one box.  Plain pointers and sizes only.
 *
 * All functions return 0 / a non-negative id on success and a negative value on error;
 * scn_last_error() gives the message of the last failure on the calling thread.
 * Device type codes: 0 = CPU, 1 = GPU (scanner/metadata.proto DeviceType).
 */
#ifndef SCN_ENGINE_H_
#define SCN_ENGINE_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define SCN_ENGINE_API __attribute__((visibility("default")))
#else
#define SCN_ENGINE_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct scn_engine scn_engine;
typedef struct scn_graph scn_graph;
typedef struct scn_job scn_job;

SCN_ENGINE_API const char* scn_last_error(void);

/* ---- op plugins (reference Client.load_op -> dlopen, worker.cpp:732-744) ------------------ */
SCN_ENGINE_API int scn_load_op_library(const char* so_path);
SCN_ENGINE_API int scn_op_registered(const char* op_name);                    /* 1 / 0 */
SCN_ENGINE_API int scn_kernel_registered(const char* op_name, int device_type); /* 1 / 0 */
/* Writes "name:n_inputs:n_outputs:can_stencil:bounded:unbounded:warmup:protobuf_name:stream_protobuf_name\n"
 * per registered op (the last two: the op's argument message names, empty if it declared none). */
SCN_ENGINE_API int scn_list_ops(char* host_buf, size_t cap);

/* ---- engine ------------------------------------------------------------------------------- */
/* gpu_ids/n_gpus: GPUs this process drives (n_gpus = 0: CPU only).
 * instances_per_gpu: pipeline instances (thread + CUDA stream + NVDEC session) per GPU
 *   (reference pipeline_instances_per_node, worker.cpp:1297-1337); 0 = auto.
 * cpu_instances: instances without a GPU (CPU kernels only); used when n_gpus = 0; 0 = 1. */
SCN_ENGINE_API scn_engine* scn_engine_create(const int* gpu_ids, int n_gpus, int instances_per_gpu,
                                             int cpu_instances);
SCN_ENGINE_API void scn_engine_destroy(scn_engine* e);

/* ---- input streams (the "tables" a job reads) ---------------------------------------------- */
/* Ingest an H.264 Annex-B elementary stream: builds the sample/keyframe index
 * (reference h264_byte_stream_index_creator.cpp).  The bytes are copied.  Returns a stream id. */
SCN_ENGINE_API int64_t scn_stream_add_h264(scn_engine* e, const uint8_t* bytes, size_t size);
/* n dense HWC frames of `type` (FrameType: 0 U8, 1 F32, 2 F64, 3 U16), copied; the reference's
 * RAW (uncompressed) video column. */
SCN_ENGINE_API int64_t scn_stream_add_raw_frames(scn_engine* e, const uint8_t* frames, int64_t n, int height,
                                                 int width, int channels, int type);
/* n byte-string rows: data is the concatenation, sizes[i] their lengths (size 0 = null row). */
SCN_ENGINE_API int64_t scn_stream_add_bytes(scn_engine* e, const uint8_t* data, const uint64_t* sizes,
                                            int64_t n);
SCN_ENGINE_API int64_t scn_stream_rows(scn_engine* e, int64_t stream);
/* info[0..5] = is_video, width, height, channels, keyframes, encoded_bytes */
SCN_ENGINE_API int scn_stream_info(scn_engine* e, int64_t stream, int64_t info[6]);
/* 1 if the H.264 stream's SPS allows display order to differ from coding order (B pictures): the
 * decode stage then feeds a GOP past the last wanted picture until that picture is displayed.
 * 0 for POC type 2 streams, for a VUI with max_num_reorder_frames == 0, and for non-H.264. */
SCN_ENGINE_API int scn_stream_may_reorder(scn_engine* e, int64_t stream);
SCN_ENGINE_API int scn_stream_remove(scn_engine* e, int64_t stream);

/* The decode stage on its own: `n` ascending frame indices of an H.264 stream -> dense RGB24 frames
 * (n * w * h * 3 bytes) in caller-owned DEVICE memory on gpu_id; returns when the frames are
 * complete.  Used by multi-GPU stencil jobs that exchange boundary frames between ranks
 * (scanner_b200/halo.py) and by tests. */
SCN_ENGINE_API int scn_engine_decode_to_device(scn_engine* e, int64_t stream, const int64_t* rows, int64_t n,
                                               int gpu_id, uint8_t* dst_device);

/* ---- op graph ------------------------------------------------------------------------------ */
SCN_ENGINE_API scn_graph* scn_graph_create(void);
SCN_ENGINE_API void scn_graph_destroy(scn_graph* g);
/* Every add_* returns the new op's index (inputs must refer to earlier indices). */
SCN_ENGINE_API int scn_graph_add_source(scn_graph* g, int is_video);
SCN_ENGINE_API int scn_graph_add_op(scn_graph* g, const char* op_name, int device_type, const int* input_ops,
                                    const char* const* input_columns, int n_inputs, const uint8_t* args,
                                    size_t args_size, int batch /* -1 = kernel default */,
                                    const int* stencil, int n_stencil /* 0 = op default */,
                                    int warmup /* -1 = op default */);
SCN_ENGINE_API int scn_graph_add_sample(scn_graph* g, int input_op, const char* input_column);
SCN_ENGINE_API int scn_graph_add_space(scn_graph* g, int input_op, const char* input_column);
SCN_ENGINE_API int scn_graph_add_sink(scn_graph* g, int input_op, const char* input_column,
                                      const char* stored_name);
/* Output column names of op `index`, '\n'-separated. */
SCN_ENGINE_API int scn_graph_op_outputs(scn_graph* g, int index, char* host_buf, size_t cap);

/* ---- jobs (one per output stream; reference proto::Job) ------------------------------------ */
SCN_ENGINE_API scn_job* scn_job_create(void);
SCN_ENGINE_API void scn_job_destroy(scn_job* j);
SCN_ENGINE_API int scn_job_bind_source(scn_job* j, int source_op, int64_t stream);
/* sampler function: All | Strided | StridedRanges | Gather | SpaceNull | SpaceRepeat; args are the
 * proto3 bytes of the matching message of scanner/sampler_args.proto. */
SCN_ENGINE_API int scn_job_set_sampler(scn_job* j, int op, const char* function, const uint8_t* args,
                                       size_t args_size);
/* Slice / Unslice (reference sc.streams.Slice / Unslice; dag_analysis.cpp:70-271, sampler.cpp:500-770):
 * a Slice op cuts its input into groups with a partitioner ("Strided" {stride, group_size},
 * "StridedRange" {stride, starts, ends}, "Gather" {groups{rows}}: the reference's
 * sampler_args.proto messages); ops between Slice and Unslice see every group as an independent
 * stream (state reset, stencils clamped at the group's edges, one task never spans two groups);
 * Unslice concatenates the groups and may only feed sinks.  Inside the slice a Sample/Space op or a
 * kernel op may be given one argument per group (the reference's SliceList). */
SCN_ENGINE_API int scn_graph_add_slice(scn_graph* g, int input_op, const char* input_column);
SCN_ENGINE_API int scn_graph_add_unslice(scn_graph* g, int input_op, const char* input_column);
SCN_ENGINE_API int scn_job_set_partitioner(scn_job* j, int slice_op, const char* name, const uint8_t* args,
                                           size_t size);
SCN_ENGINE_API int scn_job_set_group_sampler(scn_job* j, int op, int group, const char* function,
                                             const uint8_t* args, size_t size);
SCN_ENGINE_API int scn_job_set_group_stream_args(scn_job* j, int op, int group, const uint8_t* args, size_t size);

SCN_ENGINE_API int scn_job_set_stream_args(scn_job* j, int op, const uint8_t* args, size_t args_size);

/* ---- one clip across several ranks (BASELINE configs[3]; SURVEY 8e "stencil halo") -------------
 * The reference hands every task the stencil rows beyond its interval by loading and decoding them
 * again (derive_stencil_requirements, scanner/engine/dag_analysis.cpp:1634-1657; gathered at
 * evaluate_worker.cpp:1068-1089).  Here a job may compute ONE contiguous interval of its output rows
 * (scn_job_set_shard: bounds[0] = 0 <= ... <= bounds[n] = rows, interval q belongs to rank ranks[q],
 * this job computes interval `index`); rows its stencil needs from a neighbouring interval arrive as
 * decoded elements from the rank that owns them, exchanged inside scn_engine_run before the pipeline
 * instances start -- ncclSend/ncclRecv between the ranks' GPUs (scn_engine_comm_init; every rank
 * passes the 128 bytes rank 0 got from scn_engine_comm_unique_id, the call is collective), or a host
 * callback moving n buffers (scn_engine_set_halo_callback; CPU runs, tests).  Every rank must list
 * the same jobs in the same order.  Counters halo_bytes_sent / halo_bytes_received /
 * halo_exchange_us appear in scn_engine_stats_json. */
#define SCN_COMM_ID_BYTES 128
typedef int (*scn_halo_exchange_fn)(void* user, int n, const int* peers, void* const* buffers,
                                    const uint64_t* bytes, const int* is_send);
SCN_ENGINE_API int scn_engine_comm_unique_id(uint8_t out[SCN_COMM_ID_BYTES]);
SCN_ENGINE_API int scn_engine_comm_init(scn_engine* e, int gpu_id, int rank, int world,
                                        const uint8_t id[SCN_COMM_ID_BYTES]);
SCN_ENGINE_API int scn_engine_set_halo_callback(scn_engine* e, int rank, int world, scn_halo_exchange_fn fn,
                                                void* user);
SCN_ENGINE_API int scn_job_set_shard(scn_job* j, int index, int n, const int64_t* bounds, const int* ranks);

/* ---- one task queue for the engines of several processes (one rank per GPU) ------------------
 * The reference's workers PULL tasks from the master (master.cpp NextWork), so a slow worker simply does fewer.
 * Here: every rank builds the SAME job list (same clips, same order, same packet sizes) and maps the same small file
 * (a directory all ranks see, e.g. the database's); scn_engine_run then takes each next task with an atomic
 * fetch-add on a counter in that file, so every task of the run is executed by exactly one rank.  A rank's jobs
 * hold outputs only for the tasks it ran; sink tables (scn_job_set_sink_table with ids every rank agrees on) collect
 * the items of all ranks.  Between runs ONE rank calls scn_engine_reset_task_queue while no rank is inside
 * scn_engine_run (i.e. between two barriers).  path == NULL returns the engine to its private queue. */
SCN_ENGINE_API int scn_engine_share_task_queue(scn_engine* e, const char* path);
SCN_ENGINE_API int scn_engine_reset_task_queue(scn_engine* e);

/* ---- run ----------------------------------------------------------------------------------- */
/* work_packet_size / io_packet_size: rows per evaluate packet / per task (reference
 * BulkJobParameters, rpc.proto:238-274; io must be a multiple of work).  out_dir: if non-NULL the
 * sink columns are also written in the reference's column file layout
 * (<out_dir>/tables/<job>/<col>_<task>.bin + _metadata.bin, column_sink.cpp:159-195).
 * Tasks of all jobs are sharded over the engine's pipeline instances (one shared work queue). */
SCN_ENGINE_API int scn_engine_run(scn_engine* e, scn_graph* g, scn_job* const* jobs, int n_jobs,
                                  int work_packet_size, int io_packet_size, const char* out_dir);

/* ---- results ------------------------------------------------------------------------------- */
SCN_ENGINE_API int64_t scn_job_output_rows(scn_job* j, int sink_op);
/* Row `row` of sink `sink_op`: *data and *size point into engine-owned host memory valid until the job
 * is destroyed; shape[0..3] = {h, w, c, frame_type} for frame rows, {0,0,0,-1} for byte rows.
 * A null row has size 0. */
SCN_ENGINE_API int scn_job_output_row(scn_job* j, int sink_op, int64_t row, const uint8_t** data,
                                      uint64_t* size, int shape[4]);
/* Copies rows [row0, row0+n) of equal-sized elements into dst (n * row_bytes). */
SCN_ENGINE_API int scn_job_output_copy(scn_job* j, int sink_op, int64_t row0, int64_t n, uint8_t* dst,
                                       size_t row_bytes);

/* JSON: profiler interval totals / counters of the last run (frames_decoded, frames_used, ...). */
/* Tracing (reference util/profiler.{h,cpp} interval records + scannerpy Profile.write_trace,
 * profiler.py): with tracing on, every profiler interval of a run (task, get_frames, op:<Name>,
 * evaluate:<Name>, op_marshal, ...) is kept with the pipeline instance that recorded it;
 * scn_engine_write_trace writes the last run as a Chrome trace-event JSON file (chrome://tracing,
 * Perfetto): pid = GPU id (-1 for CPU instances), tid = pipeline instance, times in microseconds. */
SCN_ENGINE_API int scn_engine_set_trace(scn_engine* e, int on);
SCN_ENGINE_API int scn_engine_write_trace(scn_engine* e, const char* path);
SCN_ENGINE_API int scn_engine_stats_json(scn_engine* e, char* host_buf, size_t cap);

/* ---- kernels written in the host language ---------------------------------------------------
 * The reference's `@scannerpy.register_python_op` (python/scannerpy/op.py:317-620, kernel.py:17-81,
 * scanner/engine/python_kernel.cpp:49-361): an op whose kernel is a callable of the embedding
 * process.  One callback per op receives every kernel event; `instance` identifies the kernel object
 * (one per pipeline instance and graph node, constructed and called by that instance's evaluate
 * thread only -- different instances call concurrently).  EXECUTE passes the input elements as
 * elems[(col * n_rows + row) * n_stencil + s] (host memory, valid during the call; frames dense HWC)
 * and expects exactly n_rows elements per output column through scn_cb_emit_*, which copy.
 * The callback returns 0, or non-zero after writing a message to err: the run then fails with that
 * message (CONSTRUCT / FETCH_RESOURCES / SETUP_WITH_RESOURCES failures are validation errors). */
enum { SCN_CB_CONSTRUCT = 0, SCN_CB_DESTROY = 1, SCN_CB_NEW_STREAM = 2, SCN_CB_RESET = 3, SCN_CB_EXECUTE = 4,
       SCN_CB_FETCH_RESOURCES = 5, SCN_CB_SETUP_WITH_RESOURCES = 6 };
typedef struct scn_cb_elem {
  const uint8_t* data; /* NULL: null row */
  uint64_t size;
  int32_t shape[3];    /* frames: height, width, channels */
  int32_t frame_type;  /* frames: 0 U8, 1 F32, 2 F64, 3 U16; -1 for byte elements */
  int64_t index;       /* row id in the op's input domain */
} scn_cb_elem;
typedef struct scn_cb_call {
  int32_t event;
  int32_t node_id;
  int64_t instance;
  int32_t device_type, device_id;
  const uint8_t* args; /* CONSTRUCT: the op's kernel args; NEW_STREAM: the job's stream args */
  uint64_t args_size;
  int32_t n_cols, n_rows, n_stencil; /* EXECUTE */
  int32_t reserved;
  const scn_cb_elem* elems;
  void* out;           /* EXECUTE: handle for scn_cb_emit_* */
} scn_cb_call;
typedef int (*scn_kernel_callback)(void* user, const scn_cb_call* call, char* err, size_t err_cap);
typedef struct scn_cb_op_desc {
  const char* name;
  int32_t n_inputs;                 /* ignored when variadic_inputs */
  const char* const* input_names;
  const int32_t* input_is_frame;
  int32_t variadic_inputs;
  int32_t n_outputs;
  const char* const* output_names;
  const int32_t* output_is_frame;
  const char* const* output_type_names; /* may be NULL; stored as the column's type name */
  const int32_t* stencil;           /* n_stencil == 0: the op cannot stencil */
  int32_t n_stencil;
  int32_t bounded_state;            /* warmup rows, -1: none */
  int32_t unbounded_state;
  int32_t batch;                    /* >= 1; > 1: the kernel batches */
  int32_t also_gpu;                 /* also register for DeviceType GPU (columns stay in host memory) */
} scn_cb_op_desc;
SCN_ENGINE_API int scn_register_callback_op(const scn_cb_op_desc* desc, scn_kernel_callback cb, void* user);
SCN_ENGINE_API int scn_cb_emit_bytes(void* out, int col, const uint8_t* data, size_t size); /* size 0: null row */
SCN_ENGINE_API int scn_cb_emit_frame(void* out, int col, const uint8_t* data, int height, int width, int channels,
                                     int frame_type);

/* ---- synthetic H.264 (tests / bench input generation; no encoder exists offline) ----------- */
/* Encodes `frames` I420 pictures (planes at yuv + f*(w*h*3/2): Y, U, V) as an Annex-B stream of
 * I_PCM macroblocks, IDR every `gop` frames; non_key_mode 0 = P slices of I_PCM macroblocks
 * (yuv holds `frames` pictures), 1 = P_Skip pictures that repeat the last key picture (yuv holds
 * only the ceil(frames/gop) key pictures, consecutively), 2 = Main profile with B pictures: the odd
 * positions of a GOP that have a later anchor in it are non-reference B_Skip pictures, coded after
 * that anchor and decoding to (anchor_before + anchor_after + 1) >> 1; yuv holds `frames` pictures
 * of which only the anchors are read.  Returns the stream size, or the required size if cap is too
 * small (nothing written then). */
SCN_ENGINE_API int64_t scn_h264_synth(const uint8_t* yuv, int width, int height, int64_t frames, int gop,
                                      int non_key_mode, uint8_t* out, size_t cap);
/* NVDEC probe: info[0..5] = available, h264_supported, engines, max_w, max_h, min_w. */
SCN_ENGINE_API int scn_nvdec_caps(int gpu_id, int info[6]);
/* Software decoder probe (CPU pipeline instances; reference SoftwareVideoDecoder = FFmpeg, software_video_decoder.cpp):
 * info[0..3] = available, libavcodec major, libavutil major, libswscale major.  The libraries are resolved with
 * dlopen from $SCN_FFMPEG_DIR or the system search path; when unavailable scn_last_error() says why. */
SCN_ENGINE_API int scn_swdec_caps(int info[4]);

/* ---------------------------------------------------------------------------------------------
 * Tables on disk: a Scanner database directory in the reference's layout (db_metadata.bin,
 * tables/<id>/descriptor.bin, <col>_<item>.bin + _metadata.bin / _video_metadata.bin; reference
 * scanner/engine/metadata.h:37-86, metadata.proto:6-23,55-126).  POSIX file systems only.
 *   scn_db_ingest_video   what Client.ingest_videos does per file (ingest.cpp:175-380): demux an
 *                         .mp4/.mov (or take a raw Annex-B .h264), index it, write the video table
 *   scn_db_add_video_stream  bind a stored video table to an engine as an H.264 input stream using
 *                         the stored sample/keyframe index (no rescan) -- load_worker's view of it
 *   scn_db_save_job       write the rows a job left in memory as a new table (one item per task,
 *                         column 0 = index column; frame-valued sinks are stored uncompressed with
 *                         a RAW VideoDescriptor, column_sink.cpp:159-176).  Returns the table id.
 *   scn_db_read_rows      rows of a stored column back to host memory (Column.load)
 */
typedef struct scn_db scn_db;
typedef struct scn_rows scn_rows;
SCN_ENGINE_API scn_db* scn_db_open(const char* path);
SCN_ENGINE_API void scn_db_close(scn_db* db);
SCN_ENGINE_API int scn_db_ingest_video(scn_db* db, const char* table, const char* video_path);
/* As above without copying the bitstream into the database (reference ingest `inplace`): the table
 * records the absolute path; binding or exporting it reads (and, for .mp4, demuxes) that file again
 * and fails if it no longer yields the ingested stream. */
SCN_ENGINE_API int scn_db_ingest_video_inplace(scn_db* db, const char* table, const char* video_path);
SCN_ENGINE_API int scn_db_ingest_h264(scn_db* db, const char* table, const uint8_t* bytes, size_t size, int fps_num,
                                      int fps_den);
SCN_ENGINE_API int scn_db_has_table(scn_db* db, const char* table);
SCN_ENGINE_API int scn_db_delete_table(scn_db* db, const char* table);
SCN_ENGINE_API int scn_db_list_tables(scn_db* db, char* buf, size_t cap); /* names, one per line */
/* info: {table id, rows, columns (incl. index), items, job id, width, height, keyframes (-1: RAW)};
 * columns (optional): "name:type:type_name" per line */
SCN_ENGINE_API int scn_db_table_info(scn_db* db, const char* table, int64_t info[8], char* columns, size_t cap);
SCN_ENGINE_API int64_t scn_db_add_video_stream(scn_db* db, scn_engine* e, const char* table);
SCN_ENGINE_API int scn_db_save_job(scn_db* db, scn_job* j, const char* table, const int* sinks,
                                   const char* const* column_names, const char* const* type_names, int n_columns,
                                   int job_id);
/* Saving during the run (reference SaveWorker, one item per task as tasks finish): reserve a one-column
 * table, point a sink of the job at it, run with out_dir = the database path, commit.  With
 * keep_rows = 0 the rows of such sinks leave host memory as soon as their item is on disk (they are
 * then read with scn_db_read_rows, not scn_job_output_row). */
SCN_ENGINE_API int scn_db_new_table(scn_db* db, const char* table, const char* column_name, int is_video,
                                    const char* type_name, int job_id); /* -> table id */
SCN_ENGINE_API int scn_job_set_sink_table(scn_job* j, int sink, int table_id, int keep_rows);
/* Store a sink's frames as H.264 (reference compress_video()): when the sink also has a table and runs on a GPU
 * pipeline instance, each task's item becomes one intra-only H.264 stream at constant `qp` (0-51) with an IDR
 * every `keyframe_distance` pictures from the task's first row (scn_h264_encode_u8), encoded on the instance's GPU
 * before anything crosses to the host.  Frames must be 3-channel uint8 of one even size per task and no row may
 * be null; anything else fails the run.  On CPU instances, and for sinks without a table, rows stay raw. */
SCN_ENGINE_API int scn_job_set_sink_encoding(scn_job* j, int sink, int qp, int keyframe_distance);
/* The same for many tables with ONE catalogue lock / rewrite per call (a job list with hundreds of output streams;
 * several ranks sharing the directory): n one-column tables -> out_ids[n]; commit of n (table, job) pairs; delete. */
SCN_ENGINE_API int scn_db_new_tables(scn_db* db, int n, const char* const* tables, const char* const* column_names,
                                     const int* is_video, const char* const* type_names, const int* job_ids,
                                     int* out_ids);
SCN_ENGINE_API int scn_db_commit_job_tables(scn_db* db, int n, const int* table_ids, scn_job* const* jobs);
SCN_ENGINE_API int scn_db_delete_tables(scn_db* db, int n, const char* const* tables);
/* A table of byte columns written from host rows in one call (reference Client.new_table ->
 * master.cpp NewTable: one item holding every row): element (row r, column c) is the
 * sizes[r * n_cols + c] bytes at data[r * n_cols + c] (size 0: null).  -> table id */
SCN_ENGINE_API int scn_db_new_table_from_rows(scn_db* db, const char* table, int n_cols,
                                              const char* const* column_names, int64_t n_rows,
                                              const uint8_t* const* data, const uint64_t* sizes);
SCN_ENGINE_API int scn_db_commit_job_table(scn_db* db, int table_id, scn_job* j);
SCN_ENGINE_API scn_rows* scn_db_read_rows(scn_db* db, const char* table, const char* column, const int64_t* rows,
                                          int64_t n);
SCN_ENGINE_API int64_t scn_rows_count(const scn_rows* r);
SCN_ENGINE_API int scn_rows_get(const scn_rows* r, int64_t i, const uint8_t** data, uint64_t* size, int shape[4]);
SCN_ENGINE_API void scn_rows_free(scn_rows* r);

/* ISO base media container (the part of libavformat ingest needs, ingest.cpp:54-168,228-300):
 * scn_mp4_demux extracts the first H.264 track as an Annex-B stream (info: width, height, timescale,
 * duration, samples, sync samples); scn_mp4_mux wraps an Annex-B stream into a non-fragmented .mp4.
 * Both return the byte count needed; the output is written only if cap is large enough. */
/* NamedVideoStream.save_mp4 (reference storage.py): a stored H.264 video table back into an .mp4 file
 * (fps <= 0: the table's stored time base). */
SCN_ENGINE_API int scn_db_export_mp4(scn_db* db, const char* table, const char* out_path, int fps_num, int fps_den);
SCN_ENGINE_API int64_t scn_mp4_mux(const uint8_t* annexb, size_t size, int fps_num, int fps_den, uint8_t* out,
                                   size_t cap);
SCN_ENGINE_API int64_t scn_mp4_demux(const uint8_t* file, size_t size, uint8_t* out, size_t cap, int64_t info[6]);

#ifdef __cplusplus
}
#endif
#endif /* SCN_ENGINE_H_ */
