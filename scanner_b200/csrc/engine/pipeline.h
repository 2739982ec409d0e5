// pipeline.h -- the worker: input streams, jobs, tasks and the pipeline instances that run
// load -> decode -> evaluate -> post -> save for them.
// Restates reference scanner/engine/worker.cpp:868-2148 (process_job: instances, task pull loop),
// load_worker.cpp:80-189 + column_source.cpp:124-301 (rows -> keyframe intervals -> encoded bytes),
// evaluate_worker.cpp:316-406 (PreEvaluateWorker::yield: one frame block per work packet),
// :1373-1557 (PostEvaluateWorker: move sink columns to the host) and save_worker.cpp /
// column_sink.cpp:71-265 (column files).  The master/worker gRPC control plane is replaced by one
// in-process task queue shared by every pipeline instance of every GPU (SURVEY 8e).
#pragma once
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <cstdlib>
#include <new>
#include <vector>

#include "evaluate.h"
#include "graph.h"
#include "halo.h"
#include "h264.h"
#include "scanner/api/frame.h"

namespace scanner {
namespace internal {

// Payload storage that owns whole pages: the engine page-locks it in place (cudaHostRegister
// works on page granularity -- a buffer sharing its first/last page with other heap objects would
// leave those half-registered, and a later cudaMemcpy touching them fails with "invalid argument").
template <typename T>
struct PageAllocator {
  using value_type = T;
  static constexpr size_t kPage = 4096;
  PageAllocator() = default;
  template <typename U>
  PageAllocator(const PageAllocator<U>&) {}
  static size_t padded(size_t bytes) { return (bytes + kPage - 1) / kPage * kPage; }
  T* allocate(size_t n) {
    void* p = nullptr;
    if (posix_memalign(&p, kPage, padded(n ? n * sizeof(T) : 1)) != 0) throw std::bad_alloc();
    return static_cast<T*>(p);
  }
  void deallocate(T* p, size_t) { free(p); }
  template <typename U>
  bool operator==(const PageAllocator<U>&) const { return true; }
  template <typename U>
  bool operator!=(const PageAllocator<U>&) const { return false; }
};
using PageBuffer = std::vector<u8, PageAllocator<u8>>;

struct InputStream {
  enum Kind { H264, RawFrames, Bytes } kind = Bytes;
  // H264
  std::vector<u8> encoded;
  H264Index index;
  // RawFrames: n dense frames of `info`
  FrameInfo info;
  // RawFrames / Bytes payload + per-row extents
  PageBuffer data;
  std::vector<u64> offsets, sizes;
  bool registered = false;  // payload is cudaHostRegister'ed
  i64 rows() const { return kind == H264 ? index.frames() : (i64)sizes.size(); }
};

// Rows a sink stored for one task, host memory.  Small rows are appended to `data`; rows of
// kLargeRow bytes or more (frames, flow fields) stay in the page-locked block the post-evaluate
// stage copied them into -- the element is kept instead of being copied again into a growing vector
// whose fresh pages fault in at ~1 GB/s (a 1080p flow field is 16.6 MB per row).
struct TaskOutput {
  static constexpr size_t kLargeRow = 64 * 1024;
  bool done = false;
  std::vector<u8> data;
  std::vector<u64> offsets, sizes;
  std::vector<i32> shapes;       // 4 per row: h, w, c, frame type (-1 for byte rows)
  std::vector<const u8*> ext;    // per row: non-null = the row lives in a held host block
  Elements held;                 // host elements that keep those blocks alive
  bool dropped = false;          // payload written to a table and released (sizes/shapes remain)
  bool h264 = false;             // rows are the H.264 access units of the task's frames (one item per task)

  TaskOutput() = default;
  TaskOutput(const TaskOutput&) = delete;
  TaskOutput& operator=(const TaskOutput&) = delete;
  TaskOutput(TaskOutput&& o) noexcept { *this = std::move(o); }
  TaskOutput& operator=(TaskOutput&& o) noexcept {
    if (this != &o) {
      release();
      done = o.done;
      data = std::move(o.data);
      offsets = std::move(o.offsets);
      sizes = std::move(o.sizes);
      shapes = std::move(o.shapes);
      ext = std::move(o.ext);
      held = std::move(o.held);
      dropped = o.dropped;
      h264 = o.h264;
      o.held.clear();
    }
    return *this;
  }
  ~TaskOutput() { release(); }
  void release();  // frees the held blocks (pipeline.cpp)
  const u8* row(size_t i) const { return i < ext.size() && ext[i] ? ext[i] : data.data() + offsets[i]; }
  size_t total_bytes() const {
    size_t n = 0;
    for (u64 s : sizes) n += s;
    return n;
  }
};

struct Job {
  std::map<i32, i64> source_streams;  // source op -> stream id
  JobParams params;
  // filled by the run
  std::vector<i64> rows_per_op;
  SliceInfo slices;              // groups == 0 unless the graph slices
  i64 total_rows = 0;
  i32 io_packet = 0;
  std::vector<i64> task_starts;  // first output row of every task, then total_rows (tasks never
                                 // span slice groups, so they are not all io_packet long)
  std::map<i32, std::vector<TaskOutput>> outputs;  // sink op -> per task
  std::map<i32, bool> sink_is_frame;               // sink op -> its column is declared a frame (Video) column
  // save stage to disk (reference SaveWorker / ColumnSink, one item per task): sink op -> id of a
  // table reserved with Database::new_table in the database rooted at the run's out_dir.  With
  // keep_rows == false the rows of such sinks are dropped from memory once their item is written.
  std::map<i32, i32> sink_tables;
  bool keep_rows = true;
  // sink op -> H.264 encoding of its frames (scn_job_set_sink_encoding).  Applies to a sink in sink_tables on a
  // GPU pipeline instance: each task's item is then one intra-only H.264 stream (scn_h264_encode_u8) instead of
  // raw frames.
  struct SinkEncoding {
    i32 qp = 23;
    i32 keyframe_distance = 120;
  };
  std::map<i32, SinkEncoding> sink_encoding;
  // One clip split into contiguous output-row intervals across ranks (configs[3]): this job computes
  // rows [shard_bounds[shard_index], shard_bounds[shard_index + 1]) only; shard q is computed by rank
  // shard_ranks[q].  Source rows a stencil reaches into a neighbouring interval are not decoded here:
  // the owning rank sends them as decoded elements before the run's instances start (halo.h).
  std::vector<i64> shard_bounds;
  std::vector<i32> shard_ranks;
  i32 shard_index = -1;
};

struct TraceEvent {
  std::string key;
  i64 start_ns, end_ns;
  i32 worker, node;
};

struct RunStats {
  std::vector<TraceEvent> trace;  // filled when tracing is on (Engine::set_trace)
  std::map<std::string, i64> counters;
  std::map<std::string, i64> interval_ns;
  std::map<std::string, i64> interval_counts;
  double wall_seconds = 0;
};

class Engine {
 public:
  Engine(std::vector<i32> gpu_ids, i32 instances_per_gpu, i32 cpu_instances);
  ~Engine();

  i64 add_stream(std::unique_ptr<InputStream> s);
  InputStream* stream(i64 id);
  bool remove_stream(i64 id);

  Result run(Graph& graph, const std::vector<Job*>& jobs, i32 work_packet_size, i32 io_packet_size,
             const std::string& out_dir);

  // Decode stage on its own: rows (ascending frame indices) of an H.264 stream -> dense RGB24
  // frames in caller-owned device memory on `gpu_id` (n * w * h * 3 bytes); returns when done.
  Result decode_rows_to_device(i64 stream_id, const std::vector<i64>& rows, i32 gpu_id, u8* dst);

  const RunStats& stats() const { return stats_; }
  // Keep every profiler interval of the next runs with the instance that recorded it (reference
  // Profiler records, util/profiler.h; off by default: a long job records millions of intervals).
  void set_trace(bool on) { trace_ = on; }
  // The last run's intervals as a Chrome trace-event file (what scannerpy's Profile.write_trace
  // produces from the reference's profiler files, profiler.py): one "X" event per interval,
  // pid = GPU id (-1: CPU instance), tid = pipeline instance.
  Result write_trace(const std::string& path) const;
  const std::vector<i32>& gpu_ids() const { return gpu_ids_; }
  // Transport for the stencil halo exchange of sharded jobs (NCCL between the ranks' GPUs, or a host
  // callback); the engine owns it.
  void set_halo_transport(std::unique_ptr<HaloTransport> t) { halo_ = std::move(t); }
  // One task queue for several engines (one per process / GPU) that run the SAME job list: `counter` lives in
  // memory they all map (scn_engine_share_task_queue); a pipeline instance takes the next task of the run with an
  // atomic fetch-add on it instead of the engine's own counter, so every task is executed by exactly one engine
  // and a slow engine simply takes fewer (the reference's workers pull tasks from the master: master.cpp NextWork).
  void set_shared_task_counter(volatile unsigned long long* counter) { shared_next_ = counter; }
  volatile unsigned long long* shared_task_counter() const { return shared_next_; }
  const HaloTransport* halo_transport() const { return halo_.get(); }

 private:
  struct Instance;
  struct Slot;
  void instance_main(Instance* inst);
  std::vector<std::unique_ptr<Slot>> slots_;  // persistent per-instance state (stream, decoders)

  std::vector<i32> gpu_ids_;
  i32 instances_per_gpu_, cpu_instances_;
  std::mutex streams_mu_;
  std::map<i64, std::unique_ptr<InputStream>> streams_;
  i64 next_stream_id_ = 1;
  RunStats stats_;
  bool trace_ = false;

  std::unique_ptr<HaloTransport> halo_;
  volatile unsigned long long* shared_next_ = nullptr;
  Result exchange_halos(Graph& graph, const std::vector<Job*>& jobs);
  // `reuse`: a persistent decode session + stream (the halo exchange of every run decodes a few boundary rows;
  // creating a decoder costs ~0.25 s); nullptr: a session for this call only
  struct DecodeContext;
  Result decode_rows(InputStream& st, const std::vector<i64>& rows, i32 gpu_id, bool nv12, u8* dst,
                     DecodeContext* reuse = nullptr);
  std::map<i32, std::unique_ptr<DecodeContext>> halo_decoders_;  // per GPU

  // state of the run in flight
  struct RunState;
  std::unique_ptr<RunState> run_;
};

}  // namespace internal
}  // namespace scanner
