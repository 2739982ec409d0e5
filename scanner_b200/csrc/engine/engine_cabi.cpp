// engine_cabi.cpp -- extern "C" surface of include/scn_engine.h over the C++ pipeline.
#include <algorithm>
#include <cstring>
#include <sstream>

#include <sys/mman.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include "nvdec.h"
#include "swdec.h"
#include "pipeline.h"
#include "mp4.h"
#include "scn_engine.h"
#include "storage.h"

using namespace scanner;
using namespace scanner::internal;

struct scn_engine {
  std::unique_ptr<Engine> impl;
  void* shared_map = nullptr;  // the mapped task-queue file (scn_engine_share_task_queue)
  ~scn_engine() {
    if (shared_map) {
      if (impl) impl->set_shared_task_counter(nullptr);
      munmap(shared_map, 64);
    }
  }
};
struct scn_graph {
  Graph g;
  bool analyzed = false;
};
struct scn_job {
  Job j;
};
struct scn_db {
  std::unique_ptr<Database> impl;
};
struct scn_rows {
  std::vector<u8> data;
  std::vector<u64> sizes, offsets;
  std::vector<i32> shapes;
};

namespace {
thread_local std::string t_error;
int fail(const std::string& msg, int code = -1) {
  t_error = msg;
  return code;
}
int from_result(const Result& r) { return r.success() ? 0 : fail(r.msg()); }
int copy_out(const std::string& s, char* buf, size_t cap) {
  if (!buf || cap < s.size() + 1) return fail("buffer too small", -2);
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int)s.size();
}
}  // namespace

namespace scanner {
namespace internal {
Result register_callback_op(const scn_cb_op_desc& d, scn_kernel_callback cb, void* user);  // callback_op.cpp
}
}  // namespace scanner

extern "C" {

const char* scn_last_error(void) { return t_error.c_str(); }

int scn_load_op_library(const char* so_path) {
  if (!so_path) return fail("null path");
  return from_result(load_op_library(so_path));
}
int scn_register_callback_op(const scn_cb_op_desc* desc, scn_kernel_callback cb, void* user) {
  if (!desc) return fail("null op description");
  Result r = scanner::internal::register_callback_op(*desc, cb, user);
  return r.success() ? 0 : fail(r.msg());
}

int scn_op_registered(const char* name) { return name && get_op_registry()->has_op(name) ? 1 : 0; }
int scn_kernel_registered(const char* name, int device_type) {
  return name && get_kernel_registry()->has_kernel(name, device_type == 1 ? proto::GPU : proto::CPU) ? 1 : 0;
}
int scn_list_ops(char* buf, size_t cap) {
  std::ostringstream ss;
  for (const std::string& n : get_op_registry()->names()) {
    const OpInfo* i = get_op_registry()->get_op_info(n);
    ss << n << ":" << i->input_columns.size() << ":" << i->output_columns.size() << ":" << i->can_stencil << ":"
       << i->has_bounded_state << ":" << i->has_unbounded_state << ":" << i->warmup << ":" << i->protobuf_name << ":"
       << i->stream_protobuf_name << "\n";
  }
  return copy_out(ss.str(), buf, cap);
}

scn_engine* scn_engine_create(const int* gpu_ids, int n_gpus, int instances_per_gpu, int cpu_instances) {
  std::vector<i32> ids;
  for (int i = 0; i < n_gpus; ++i) ids.push_back(gpu_ids[i]);
  scn_engine* e = new scn_engine();
  e->impl.reset(new Engine(ids, instances_per_gpu, cpu_instances));
  return e;
}
void scn_engine_destroy(scn_engine* e) { delete e; }

int64_t scn_stream_add_h264(scn_engine* e, const uint8_t* bytes, size_t size) {
  if (!e || !bytes || !size) return fail("bad arguments");
  std::unique_ptr<InputStream> s(new InputStream());
  s->kind = InputStream::H264;
  s->encoded.assign(bytes, bytes + size);
  Result r = index_bytestream(s->encoded.data(), s->encoded.size(), s->index);
  if (!r.success()) return fail(r.msg());
  return e->impl->add_stream(std::move(s));
}

int64_t scn_stream_add_raw_frames(scn_engine* e, const uint8_t* frames, int64_t n, int height, int width,
                                  int channels, int type) {
  if (!e || n < 0 || height <= 0 || width <= 0 || channels <= 0 || (n > 0 && !frames)) return fail("bad arguments");
  std::unique_ptr<InputStream> s(new InputStream());
  s->kind = InputStream::RawFrames;
  s->info = FrameInfo(height, width, channels, FrameType((proto::FrameType)type));
  const size_t fb = s->info.size();
  s->data.assign(frames, frames + (size_t)n * fb);
  for (int64_t i = 0; i < n; ++i) {
    s->offsets.push_back((u64)i * fb);
    s->sizes.push_back(fb);
  }
  return e->impl->add_stream(std::move(s));
}

int64_t scn_stream_add_bytes(scn_engine* e, const uint8_t* data, const uint64_t* sizes, int64_t n) {
  if (!e || n < 0 || (n > 0 && !sizes)) return fail("bad arguments");
  std::unique_ptr<InputStream> s(new InputStream());
  s->kind = InputStream::Bytes;
  u64 total = 0;
  for (int64_t i = 0; i < n; ++i) {
    s->offsets.push_back(total);
    s->sizes.push_back(sizes[i]);
    total += sizes[i];
  }
  if (total) s->data.assign(data, data + total);
  else s->data.assign(1, 0);  // keep a non-empty backing store so rows are addressable
  return e->impl->add_stream(std::move(s));
}

int64_t scn_stream_rows(scn_engine* e, int64_t id) {
  InputStream* s = e ? e->impl->stream(id) : nullptr;
  return s ? s->rows() : fail("unknown stream");
}

int scn_stream_info(scn_engine* e, int64_t id, int64_t info[6]) {
  InputStream* s = e ? e->impl->stream(id) : nullptr;
  if (!s || !info) return fail("unknown stream");
  memset(info, 0, 6 * sizeof(int64_t));
  if (s->kind == InputStream::H264) {
    info[0] = 1;
    info[1] = s->index.width;
    info[2] = s->index.height;
    info[3] = 3;
    info[4] = (int64_t)s->index.keyframe_indices.size();
    info[5] = (int64_t)s->encoded.size();
  } else if (s->kind == InputStream::RawFrames) {
    info[0] = 1;
    info[1] = s->info.width();
    info[2] = s->info.height();
    info[3] = s->info.channels();
    info[5] = (int64_t)s->data.size();
  } else {
    info[5] = (int64_t)s->data.size();
  }
  return 0;
}
int scn_stream_may_reorder(scn_engine* e, int64_t id) {
  InputStream* s = e ? e->impl->stream(id) : nullptr;
  if (!s) return fail("unknown stream");
  return s->kind == InputStream::H264 && s->index.may_reorder ? 1 : 0;
}
int scn_stream_remove(scn_engine* e, int64_t id) { return e && e->impl->remove_stream(id) ? 0 : fail("unknown stream"); }

int scn_engine_decode_to_device(scn_engine* e, int64_t stream, const int64_t* rows, int64_t n, int gpu_id,
                                uint8_t* dst) {
  if (!e || n < 0 || (n > 0 && !rows)) return fail("bad arguments");
  std::vector<i64> r(rows, rows + n);
  return from_result(e->impl->decode_rows_to_device(stream, r, gpu_id, dst));
}

scn_graph* scn_graph_create(void) { return new scn_graph(); }
void scn_graph_destroy(scn_graph* g) { delete g; }

int scn_graph_add_source(scn_graph* g, int is_video) {
  if (!g) return fail("null graph");
  GraphOp op;
  op.kind = OpKind::Source;
  op.name = "Input";
  op.column_type = is_video ? proto::Video : proto::Bytes;
  op.output_columns = {is_video ? "frame" : "column"};
  g->g.ops.push_back(op);
  return (int)g->g.ops.size() - 1;
}

int scn_graph_add_op(scn_graph* g, const char* name, int device_type, const int* input_ops,
                     const char* const* input_columns, int n_inputs, const uint8_t* args, size_t args_size,
                     int batch, const int* stencil, int n_stencil, int warmup) {
  if (!g || !name || n_inputs < 0) return fail("bad arguments");
  const OpInfo* info = get_op_registry()->get_op_info(name);
  if (!info) return fail(std::string("Op ") + name + " is not registered.");
  GraphOp op;
  op.kind = OpKind::Kernel;
  op.name = name;
  op.device_type = device_type == 1 ? proto::GPU : proto::CPU;
  for (int i = 0; i < n_inputs; ++i) op.inputs.push_back({input_ops[i], input_columns[i] ? input_columns[i] : ""});
  if (args && args_size) op.args.assign(args, args + args_size);
  op.batch = batch;
  for (int i = 0; i < n_stencil; ++i) op.stencil.push_back(stencil[i]);
  op.warmup = warmup;
  for (auto& c : info->output_columns) op.output_columns.push_back(c.name);
  g->g.ops.push_back(op);
  return (int)g->g.ops.size() - 1;
}

static int add_builtin(scn_graph* g, OpKind kind, const char* name, int input_op, const char* col, const char* stored) {
  if (!g || !col) return fail("bad arguments");
  if (input_op < 0 || input_op >= (int)g->g.ops.size()) return fail("input op out of range");
  GraphOp op;
  op.kind = kind;
  op.name = name;
  op.inputs.push_back({input_op, col});
  if (kind != OpKind::Sink) op.output_columns = {col};
  if (stored) op.sink_column_name = stored;
  g->g.ops.push_back(op);
  return (int)g->g.ops.size() - 1;
}
int scn_graph_add_sample(scn_graph* g, int input_op, const char* col) {
  return add_builtin(g, OpKind::Sample, "Sample", input_op, col, nullptr);
}
int scn_graph_add_space(scn_graph* g, int input_op, const char* col) {
  return add_builtin(g, OpKind::Space, "Space", input_op, col, nullptr);
}
int scn_graph_add_sink(scn_graph* g, int input_op, const char* col, const char* stored) {
  return add_builtin(g, OpKind::Sink, "Output", input_op, col, stored ? stored : col);
}
int scn_graph_op_outputs(scn_graph* g, int index, char* buf, size_t cap) {
  if (!g || index < 0 || index >= (int)g->g.ops.size()) return fail("op out of range");
  std::string s;
  for (auto& c : g->g.ops[index].output_columns) s += c + "\n";
  return copy_out(s, buf, cap);
}

scn_job* scn_job_create(void) { return new scn_job(); }
void scn_job_destroy(scn_job* j) { delete j; }
int scn_job_bind_source(scn_job* j, int op, int64_t stream) {
  if (!j) return fail("null job");
  j->j.source_streams[op] = stream;
  return 0;
}
int scn_job_set_sampler(scn_job* j, int op, const char* fn, const uint8_t* args, size_t n) {
  if (!j || !fn) return fail("bad arguments");
  std::unique_ptr<DomainSampler> s;
  std::vector<u8> a(args ? args : (const uint8_t*)"", args ? args + n : (const uint8_t*)"");
  Result r = make_domain_sampler(fn, a, s);
  if (!r.success()) return fail(r.msg());
  j->j.params.samplers[op] = {fn, a};
  return 0;
}
int scn_job_set_stream_args(scn_job* j, int op, const uint8_t* args, size_t n) {
  if (!j) return fail("null job");
  j->j.params.stream_args[op] = std::vector<u8>(args ? args : (const uint8_t*)"", args ? args + n : (const uint8_t*)"");
  return 0;
}

int scn_engine_run(scn_engine* e, scn_graph* g, scn_job* const* jobs, int n_jobs, int wps, int ios,
                   const char* out_dir) {
  if (!e || !g || n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail("bad arguments");
  std::vector<Job*> js;
  for (int i = 0; i < n_jobs; ++i) js.push_back(&jobs[i]->j);
  return from_result(e->impl->run(g->g, js, wps, ios, out_dir ? out_dir : ""));
}

int scn_graph_add_slice(scn_graph* g, int input_op, const char* column) {
  if (!g || !column) return fail("bad arguments");
  GraphOp op;
  op.kind = OpKind::Sample;
  op.slice_role = SliceRole::Slice;
  op.name = "Slice";
  op.inputs.push_back({input_op, column});
  g->g.ops.push_back(op);
  g->analyzed = false;
  return (int)g->g.ops.size() - 1;
}
int scn_graph_add_unslice(scn_graph* g, int input_op, const char* column) {
  if (!g || !column) return fail("bad arguments");
  GraphOp op;
  op.kind = OpKind::Sample;
  op.slice_role = SliceRole::Unslice;
  op.name = "Unslice";
  op.inputs.push_back({input_op, column});
  g->g.ops.push_back(op);
  g->analyzed = false;
  return (int)g->g.ops.size() - 1;
}
int scn_job_set_partitioner(scn_job* j, int slice_op, const char* name, const uint8_t* args, size_t size) {
  if (!j || !name) return fail("bad arguments");
  j->j.params.partitioners[slice_op] = {name, std::vector<u8>(args, args + (args ? size : 0))};
  return 0;
}
int scn_job_set_group_sampler(scn_job* j, int op, int group, const char* name, const uint8_t* args, size_t size) {
  if (!j || !name || group < 0) return fail("bad arguments");
  auto& v = j->j.params.group_samplers[op];
  if (v.size() <= (size_t)group) v.resize((size_t)group + 1);
  v[(size_t)group] = {name, std::vector<u8>(args, args + (args ? size : 0))};
  return 0;
}
int scn_job_set_group_stream_args(scn_job* j, int op, int group, const uint8_t* args, size_t size) {
  if (!j || group < 0) return fail("bad arguments");
  auto& v = j->j.params.group_stream_args[op];
  if (v.size() <= (size_t)group) v.resize((size_t)group + 1);
  v[(size_t)group] = std::vector<u8>(args, args + (args ? size : 0));
  return 0;
}

int64_t scn_job_output_rows(scn_job* j, int sink) {
  if (!j) return fail("null job");
  auto it = j->j.outputs.find(sink);
  if (it == j->j.outputs.end()) return fail("op is not a sink of this job");
  int64_t n = 0;
  for (const TaskOutput& t : it->second) n += (int64_t)t.sizes.size();
  return n;
}

static const TaskOutput* locate(scn_job* j, int sink, int64_t row, size_t& idx) {
  auto it = j->j.outputs.find(sink);
  const std::vector<i64>& starts = j->j.task_starts;
  if (it == j->j.outputs.end() || starts.size() < 2 || row < 0 || row >= starts.back()) return nullptr;
  const size_t task = (size_t)(std::upper_bound(starts.begin(), starts.end(), row) - starts.begin()) - 1;
  if (task >= it->second.size() || it->second[task].dropped) return nullptr;
  idx = (size_t)(row - starts[task]);
  const TaskOutput& t = it->second[task];
  return idx < t.sizes.size() ? &t : nullptr;
}

int scn_job_output_row(scn_job* j, int sink, int64_t row, const uint8_t** data, uint64_t* size, int shape[4]) {
  if (!j) return fail("null job");
  size_t idx;
  const TaskOutput* t = locate(j, sink, row, idx);
  if (!t) return fail("row out of range");
  if (data) *data = t->row(idx);
  if (size) *size = t->sizes[idx];
  if (shape)
    for (int k = 0; k < 4; ++k) shape[k] = t->shapes[idx * 4 + k];
  return 0;
}

int scn_job_output_copy(scn_job* j, int sink, int64_t row0, int64_t n, uint8_t* dst, size_t row_bytes) {
  if (!j || !dst) return fail("bad arguments");
  for (int64_t i = 0; i < n; ++i) {
    size_t idx;
    const TaskOutput* t = locate(j, sink, row0 + i, idx);
    if (!t) return fail("row out of range");
    if (t->sizes[idx] != row_bytes) return fail("row " + std::to_string(row0 + i) + " has " +
                                                std::to_string(t->sizes[idx]) + " bytes, expected " +
                                                std::to_string(row_bytes));
    memcpy(dst + (size_t)i * row_bytes, t->row(idx), row_bytes);
  }
  return 0;
}

int scn_engine_set_trace(scn_engine* e, int on) {
  if (!e) return fail("null engine");
  e->impl->set_trace(on != 0);
  return 0;
}
int scn_engine_write_trace(scn_engine* e, const char* path) {
  if (!e || !path) return fail("bad arguments");
  return from_result(e->impl->write_trace(path));
}

int scn_engine_stats_json(scn_engine* e, char* buf, size_t cap) {
  if (!e) return fail("null engine");
  const RunStats& s = e->impl->stats();
  std::ostringstream ss;
  ss << "{\"wall_seconds\": " << s.wall_seconds << ", \"counters\": {";
  bool first = true;
  for (auto& kv : s.counters) {
    ss << (first ? "" : ", ") << "\"" << kv.first << "\": " << kv.second;
    first = false;
  }
  ss << "}, \"intervals_ms\": {";
  first = true;
  for (auto& kv : s.interval_ns) {
    ss << (first ? "" : ", ") << "\"" << kv.first << "\": " << (double)kv.second * 1e-6;
    first = false;
  }
  ss << "}, \"interval_counts\": {";
  first = true;
  for (auto& kv : s.interval_counts) {
    ss << (first ? "" : ", ") << "\"" << kv.first << "\": " << kv.second;
    first = false;
  }
  ss << "}}";
  return copy_out(ss.str(), buf, cap);
}

int64_t scn_h264_synth(const uint8_t* yuv, int width, int height, int64_t frames, int gop, int non_key_mode,
                       uint8_t* out, size_t cap) {
  if (!yuv || width <= 0 || height <= 0 || (width & 1) || (height & 1) || frames <= 0) return fail("bad arguments");
  const size_t ysz = (size_t)width * height, csz = ysz / 4, fsz = ysz + 2 * csz;
  std::vector<u8> stream;
  stream.reserve((size_t)frames * (fsz + fsz / 64 + 4096));
  if (non_key_mode < 0 || non_key_mode > 2) return fail("non_key_mode must be 0 (pcm), 1 (skip) or 2 (bidir)");
  write_ipcm_stream(width, height, frames, gop, (SynthNonKey)non_key_mode,
                    [&](i64 f, u8* y, u8* u, u8* v) {
                      // skip mode: only key pictures carry content, yuv holds one per GOP
                      const u8* src = yuv + (size_t)(non_key_mode == 1 ? f / (gop < 1 ? 1 : gop) : f) * fsz;
                      memcpy(y, src, ysz);
                      memcpy(u, src + ysz, csz);
                      memcpy(v, src + ysz + csz, csz);
                    },
                    stream);
  if (out && cap >= stream.size()) memcpy(out, stream.data(), stream.size());
  return (int64_t)stream.size();
}

int scn_nvdec_caps(int gpu_id, int info[6]) {
  if (!info) return fail("null info");
  const NvdecCaps& c = nvdec_caps(gpu_id);
  info[0] = c.available;
  info[1] = c.h264_supported;
  info[2] = c.num_engines;
  info[3] = c.max_width;
  info[4] = c.max_height;
  info[5] = c.min_width;
  if (!c.available) t_error = c.error;
  return 0;
}

int scn_swdec_caps(int info[4]) {
  if (!info) return fail("null info");
  const SwdecCaps& c = swdec_caps();
  info[0] = c.available;
  info[1] = c.avcodec_major;
  info[2] = c.avutil_major;
  info[3] = c.swscale_major;
  t_error = c.available ? c.where : c.error;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// database directory (include/scn_engine.h "tables on disk")
scn_db* scn_db_open(const char* path) {
  if (!path) {
    fail("null path");
    return nullptr;
  }
  std::unique_ptr<Database> db;
  Result r = Database::open(path, db);
  if (!r.success()) {
    fail(r.msg());
    return nullptr;
  }
  scn_db* h = new scn_db();
  h->impl = std::move(db);
  return h;
}
void scn_db_close(scn_db* db) { delete db; }

int scn_db_ingest_video(scn_db* db, const char* table, const char* video_path) {
  if (!db || !table || !video_path) return fail("bad arguments");
  return from_result(db->impl->ingest_video(table, video_path));
}
int scn_db_ingest_video_inplace(scn_db* db, const char* table, const char* video_path) {
  if (!db || !table || !video_path) return fail("bad arguments");
  return from_result(db->impl->ingest_video(table, video_path, true));
}
int scn_db_ingest_h264(scn_db* db, const char* table, const uint8_t* bytes, size_t size, int fps_num, int fps_den) {
  if (!db || !table || !bytes || !size) return fail("bad arguments");
  return from_result(db->impl->ingest_h264(table, bytes, size, fps_den > 0 ? fps_den : 1, fps_num > 0 ? fps_num : 25));
}
int scn_db_has_table(scn_db* db, const char* table) { return db && table && db->impl->has_table(table) ? 1 : 0; }
int scn_db_delete_table(scn_db* db, const char* table) {
  if (!db || !table) return fail("bad arguments");
  return from_result(db->impl->delete_table(table));
}
int scn_db_list_tables(scn_db* db, char* buf, size_t cap) {
  if (!db) return fail("null database");
  std::string s;
  for (const std::string& n : db->impl->table_names()) s += n + "\n";
  return copy_out(s, buf, cap);
}

int scn_db_table_info(scn_db* db, const char* table, int64_t info[8], char* columns, size_t cap) {
  if (!db || !table || !info) return fail("bad arguments");
  tables::TableDescriptor td;
  Result r = db->impl->read_table(table, td);
  if (!r.success()) return fail(r.msg());
  for (int i = 0; i < 8; ++i) info[i] = 0;
  info[0] = td.id();
  info[1] = td.end_rows_size() ? td.end_rows(td.end_rows_size() - 1) : 0;
  info[2] = td.columns_size();
  info[3] = td.end_rows_size();
  info[4] = td.job_id();
  std::string cols;
  bool video = false;
  for (const auto& c : td.columns()) {
    cols += c.name() + ":" + std::to_string(c.type()) + ":" + c.type_name() + "\n";
    if (c.type() == (int)proto::Video) video = true;
  }
  if (video) {
    tables::VideoDescriptor vd;
    std::string file;
    if (db->impl->read_video(table, vd, file).success()) {
      info[5] = vd.width();
      info[6] = vd.height();
      info[7] = vd.codec_type() == 0 ? vd.keyframe_indices_size() : -1;  // -1: stored uncompressed
    }
  }
  if (columns) return copy_out(cols, columns, cap);
  return 0;
}

int64_t scn_db_add_video_stream(scn_db* db, scn_engine* e, const char* table) {
  if (!db || !e || !table) return fail("bad arguments");
  tables::VideoDescriptor vd;
  std::unique_ptr<InputStream> s(new InputStream());
  s->kind = InputStream::H264;
  Result r = db->impl->load_video(table, vd, s->encoded);
  if (!r.success()) return fail(r.msg());
  r = index_from_descriptor(vd, s->index);
  if (!r.success()) return fail(r.msg());
  r = check_index(s->index, s->encoded.size());
  if (!r.success())
    return fail("video descriptor of table " + std::string(table) + " does not match its data: " + r.msg());
  return e->impl->add_stream(std::move(s));
}

int scn_engine_comm_unique_id(uint8_t out[SCN_COMM_ID_BYTES]) {
  if (!out) return fail("null buffer");
  Result r = halo_nccl_unique_id(out);
  return r.success() ? 0 : fail(r.msg());
}

int scn_engine_comm_init(scn_engine* e, int gpu_id, int rank, int world, const uint8_t id[SCN_COMM_ID_BYTES]) {
  if (!e || !id || world < 1 || rank < 0 || rank >= world || gpu_id < 0) return fail("bad arguments");
  std::unique_ptr<HaloTransport> t;
  Result r = make_nccl_transport(gpu_id, rank, world, id, t);
  if (!r.success()) return fail(r.msg());
  e->impl->set_halo_transport(std::move(t));
  return 0;
}

int scn_engine_set_halo_callback(scn_engine* e, int rank, int world, scn_halo_exchange_fn fn, void* user) {
  if (!e || !fn || world < 1 || rank < 0 || rank >= world) return fail("bad arguments");
  e->impl->set_halo_transport(make_callback_transport(rank, world, fn, user));
  return 0;
}

int scn_engine_share_task_queue(scn_engine* e, const char* path) {
  if (!e) return fail("null engine");
  e->impl->set_shared_task_counter(nullptr);
  if (e->shared_map) {
    munmap(e->shared_map, 64);
    e->shared_map = nullptr;
  }
  if (!path) return 0;
  const int fd = open(path, O_RDWR | O_CREAT, 0600);
  if (fd < 0) return fail(std::string("cannot open ") + path + ": " + strerror(errno));
  // a fresh file reads as zeros; ranks that arrive later must not shrink what another rank already counts in
  struct stat sb;
  if (fstat(fd, &sb) != 0 || (sb.st_size < 64 && ftruncate(fd, 64) != 0)) {
    close(fd);
    return fail(std::string("cannot size ") + path + ": " + strerror(errno));
  }
  void* m = mmap(nullptr, 64, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (m == MAP_FAILED) return fail(std::string("cannot map ") + path + ": " + strerror(errno));
  e->shared_map = m;
  e->impl->set_shared_task_counter(static_cast<volatile unsigned long long*>(m));
  return 0;
}

int scn_engine_reset_task_queue(scn_engine* e) {
  if (!e) return fail("null engine");
  volatile unsigned long long* c = e->impl->shared_task_counter();
  if (!c) return fail("the engine has no shared task queue");
  __atomic_store_n(c, 0ull, __ATOMIC_SEQ_CST);
  return 0;
}

int scn_job_set_shard(scn_job* j, int index, int n, const int64_t* bounds, const int* ranks) {
  if (!j || n < 1 || index < 0 || index >= n || !bounds || !ranks) return fail("bad arguments");
  j->j.shard_index = index;
  j->j.shard_bounds.assign(bounds, bounds + n + 1);
  j->j.shard_ranks.assign(ranks, ranks + n);
  return 0;
}

int scn_job_set_sink_table(scn_job* j, int sink, int table_id, int keep_rows) {
  if (!j || table_id < 0) return fail("bad arguments");
  j->j.sink_tables[sink] = table_id;
  j->j.keep_rows = keep_rows != 0;
  return 0;
}

int scn_job_set_sink_encoding(scn_job* j, int sink, int qp, int keyframe_distance) {
  if (!j || qp < 0 || qp > 51 || keyframe_distance < 1)
    return fail("bad arguments: H.264 QP must be 0-51 and keyframe_distance at least 1");
  j->j.sink_encoding[sink] = Job::SinkEncoding{qp, keyframe_distance};
  return 0;
}

int scn_db_new_table(scn_db* db, const char* table, const char* column_name, int is_video, const char* type_name,
                     int job_id) {
  if (!db || !table || !column_name) return fail("bad arguments");
  ColumnSpec cs;
  cs.name = column_name;
  cs.type = is_video ? proto::Video : proto::Bytes;
  cs.type_name = type_name ? type_name : "";
  i32 id = -1;
  Result r = db->impl->new_table(table, {cs}, job_id, id);
  return r.success() ? id : fail(r.msg());
}

int scn_db_new_table_from_rows(scn_db* db, const char* table, int n_cols, const char* const* column_names,
                               int64_t n_rows, const uint8_t* const* data, const uint64_t* sizes) {
  if (!db || !table || n_cols <= 0 || !column_names || n_rows < 0 || (n_rows > 0 && (!data || !sizes)))
    return fail("bad arguments");
  std::vector<ColumnSpec> specs((size_t)n_cols);
  for (int c = 0; c < n_cols; ++c) {
    if (!column_names[c] || !column_names[c][0]) return fail("empty column name");
    specs[(size_t)c].name = column_names[c];
    specs[(size_t)c].type = proto::Bytes;
  }
  i32 id = -1;
  Result r = db->impl->new_table(table, specs, -1, id);
  if (!r.success()) return fail(r.msg());
  r = db->impl->write_index_item(id, 0, 0, n_rows);
  for (int c = 0; c < n_cols && r.success(); ++c) {
    std::vector<u8> bytes;
    std::vector<u64> row_sizes((size_t)n_rows);
    for (int64_t row = 0; row < n_rows; ++row) {
      const size_t k = (size_t)row * (size_t)n_cols + (size_t)c;
      row_sizes[(size_t)row] = data[k] ? sizes[k] : 0;
      if (row_sizes[(size_t)row]) bytes.insert(bytes.end(), data[k], data[k] + sizes[k]);
    }
    ItemColumn ic;
    ic.data = bytes.data();
    ic.bytes = bytes.size();
    ic.sizes = &row_sizes;
    r = db->impl->write_item(id, c + 1, 0, ic, false);  // column 0 is the index column
  }
  if (r.success()) r = db->impl->commit_table(id, {n_rows});
  if (!r.success()) {
    db->impl->delete_table(table);
    return fail(r.msg());
  }
  return id;
}

int scn_db_new_tables(scn_db* db, int n, const char* const* tables, const char* const* column_names, const int* is_video,
                      const char* const* type_names, const int* job_ids, int* out_ids) {
  if (!db || n < 0 || (n > 0 && (!tables || !column_names || !is_video || !out_ids))) return fail("bad arguments");
  std::vector<Database::NewTable> specs((size_t)n);
  for (int i = 0; i < n; ++i) {
    if (!tables[i] || !column_names[i]) return fail("bad arguments");
    ColumnSpec cs;
    cs.name = column_names[i];
    cs.type = is_video[i] ? proto::Video : proto::Bytes;
    cs.type_name = type_names && type_names[i] ? type_names[i] : "";
    specs[(size_t)i] = Database::NewTable{tables[i], {cs}, job_ids ? job_ids[i] : -1};
  }
  std::vector<i32> ids;
  Result r = db->impl->new_tables(specs, ids);
  if (!r.success()) return fail(r.msg());
  for (int i = 0; i < n; ++i) out_ids[i] = ids[(size_t)i];
  return 0;
}

int scn_db_commit_job_tables(scn_db* db, int n, const int* table_ids, scn_job* const* jobs) {
  if (!db || n < 0 || (n > 0 && (!table_ids || !jobs))) return fail("bad arguments");
  std::vector<std::pair<i32, std::vector<i64>>> v;
  for (int i = 0; i < n; ++i) {
    if (!jobs[i] || jobs[i]->j.task_starts.size() < 1) return fail("bad arguments");
    v.emplace_back(table_ids[i], std::vector<i64>(jobs[i]->j.task_starts.begin() + 1, jobs[i]->j.task_starts.end()));
  }
  return from_result(db->impl->commit_tables(v));
}

int scn_db_delete_tables(scn_db* db, int n, const char* const* tables) {
  if (!db || n < 0 || (n > 0 && !tables)) return fail("bad arguments");
  std::vector<std::string> names;
  for (int i = 0; i < n; ++i) {
    if (!tables[i]) return fail("bad arguments");
    names.push_back(tables[i]);
  }
  return from_result(db->impl->delete_tables(names));
}

int scn_db_commit_job_table(scn_db* db, int table_id, scn_job* j) {
  if (!db || !j || j->j.task_starts.size() < 1) return fail("bad arguments");
  std::vector<i64> end_rows(j->j.task_starts.begin() + 1, j->j.task_starts.end());
  return from_result(db->impl->commit_table(table_id, end_rows));
}

int scn_db_save_job(scn_db* db, scn_job* j, const char* table, const int* sinks, const char* const* column_names,
                    const char* const* type_names, int n_columns, int job_id) {
  if (!db || !j || !table || !sinks || !column_names || n_columns <= 0) return fail("bad arguments");
  std::vector<ColumnSpec> cols;
  std::vector<const std::vector<TaskOutput>*> outs;
  size_t n_tasks = 0;
  for (int c = 0; c < n_columns; ++c) {
    auto it = j->j.outputs.find(sinks[c]);
    if (it == j->j.outputs.end()) return fail("op " + std::to_string(sinks[c]) + " is not a sink of this job");
    outs.push_back(&it->second);
    if (c == 0) n_tasks = it->second.size();
    else if (it->second.size() != n_tasks) return fail("sinks of one job must have the same number of tasks");
    // declared type of the sink's column, recorded by the run (not inferred from the rows: a column
    // of null rows is still a frame column)
    auto sf = j->j.sink_is_frame.find(sinks[c]);
    const bool is_frame = sf != j->j.sink_is_frame.end() && sf->second;
    ColumnSpec cs;
    cs.name = column_names[c];
    cs.type = is_frame ? proto::Video : proto::Bytes;
    cs.type_name = type_names && type_names[c] ? type_names[c] : "";
    cols.push_back(cs);
  }
  i32 id = -1;
  Result r = db->impl->new_table(table, cols, job_id, id);
  if (!r.success()) return fail(r.msg());
  std::vector<i64> end_rows;
  i64 row = 0;
  for (size_t t = 0; t < n_tasks && r.success(); ++t) {
    const i64 n = (i64)(*outs[0])[t].sizes.size();
    r = db->impl->write_index_item(id, (i32)t, row, row + n);
    for (int c = 0; c < n_columns && r.success(); ++c) {
      const TaskOutput& to = (*outs[c])[t];
      if ((i64)to.sizes.size() != n) {
        r.set_success(false);
        r.set_msg("columns of one task disagree on the number of rows");
        break;
      }
      ItemColumn ic;
      std::vector<u8> flat;  // rows kept in page-locked blocks are gathered for the writer
      if (to.held.empty()) {
        ic.data = to.data.data();
        ic.bytes = to.data.size();
      } else {
        flat.reserve(to.total_bytes());
        for (size_t i = 0; i < to.sizes.size(); ++i) flat.insert(flat.end(), to.row(i), to.row(i) + to.sizes[i]);
        ic.data = flat.data();
        ic.bytes = flat.size();
      }
      ic.sizes = &to.sizes;
      ic.shapes = &to.shapes;
      r = db->impl->write_item(id, c + 1, (i32)t, ic, cols[c].type == proto::Video);
    }
    row += n;
    end_rows.push_back(row);
  }
  if (r.success()) r = db->impl->commit_table(id, end_rows);
  if (!r.success()) {
    db->impl->delete_table(table);
    return fail(r.msg());
  }
  return id;
}

scn_rows* scn_db_read_rows(scn_db* db, const char* table, const char* column, const int64_t* rows, int64_t n) {
  if (!db || !table || !column || (n > 0 && !rows)) {
    fail("bad arguments");
    return nullptr;
  }
  std::unique_ptr<scn_rows> out(new scn_rows());
  std::vector<i64> want(rows, rows + (n > 0 ? n : 0));
  Result r = db->impl->read_rows(table, column, want, out->data, out->sizes, out->shapes);
  if (!r.success()) {
    fail(r.msg());
    return nullptr;
  }
  u64 off = 0;
  for (u64 s : out->sizes) {
    out->offsets.push_back(off);
    off += s;
  }
  return out.release();
}
int64_t scn_rows_count(const scn_rows* r) { return r ? (int64_t)r->sizes.size() : 0; }
int scn_rows_get(const scn_rows* r, int64_t i, const uint8_t** data, uint64_t* size, int shape[4]) {
  if (!r || i < 0 || (size_t)i >= r->sizes.size()) return fail("row out of range");
  if (data) *data = r->data.data() + r->offsets[(size_t)i];
  if (size) *size = r->sizes[(size_t)i];
  if (shape)
    for (int k = 0; k < 4; ++k) shape[k] = r->shapes[(size_t)i * 4 + k];
  return 0;
}
void scn_rows_free(scn_rows* r) { delete r; }

int scn_db_export_mp4(scn_db* db, const char* table, const char* out_path, int fps_num, int fps_den) {
  if (!db || !table || !out_path) return fail("bad arguments");
  tables::VideoDescriptor vd;
  std::vector<u8> stream;
  Result r = db->impl->load_video(table, vd, stream);
  if (!r.success()) return fail(r.msg());
  H264Index idx;
  r = index_from_descriptor(vd, idx);
  if (!r.success()) return fail(r.msg());
  if (fps_num <= 0 || fps_den <= 0) {  // default: the stored time base (ticks per second / ticks per frame 1)
    fps_num = vd.time_base_denom() > 0 ? vd.time_base_denom() : 25;
    fps_den = vd.time_base_num() > 0 ? vd.time_base_num() : 1;
  }
  std::vector<u8> mp4;
  r = mux_mp4(stream.data(), stream.size(), idx, fps_num, fps_den, mp4);
  if (!r.success()) return fail(r.msg());
  FILE* o = fopen(out_path, "wb");
  if (!o) return fail(std::string("cannot write ") + out_path);
  const size_t put = fwrite(mp4.data(), 1, mp4.size(), o);
  fclose(o);
  return put == mp4.size() ? 0 : fail(std::string("short write to ") + out_path);
}

// ---- mp4 container helpers (ingest reads .mp4; tests and benchmarks write it)
int64_t scn_mp4_mux(const uint8_t* annexb, size_t size, int fps_num, int fps_den, uint8_t* out, size_t cap) {
  if (!annexb || !size) return fail("bad arguments");
  H264Index idx;
  Result r = index_bytestream(annexb, size, idx);
  if (!r.success()) return fail(r.msg());
  std::vector<u8> file;
  r = mux_mp4(annexb, size, idx, fps_num, fps_den, file);
  if (!r.success()) return fail(r.msg());
  if (out && cap >= file.size()) memcpy(out, file.data(), file.size());
  return (int64_t)file.size();
}
int64_t scn_mp4_demux(const uint8_t* file, size_t size, uint8_t* out, size_t cap, int64_t info[6]) {
  if (!file || !size) return fail("bad arguments");
  Mp4Track t;
  Result r = demux_mp4(file, size, t);
  if (!r.success()) return fail(r.msg());
  if (info) {
    info[0] = t.width;
    info[1] = t.height;
    info[2] = t.timescale;
    info[3] = (int64_t)t.duration;
    info[4] = t.samples;
    info[5] = t.sync_samples;
  }
  if (out && cap >= t.annexb.size()) memcpy(out, t.annexb.data(), t.annexb.size());
  return (int64_t)t.annexb.size();
}

}  // extern "C"
