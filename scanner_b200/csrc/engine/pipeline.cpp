// pipeline.cpp -- see pipeline.h.
#include "pipeline.h"

#include <cuda_runtime.h>
#include <sys/stat.h>

#include <algorithm>
#include <chrono>
#include <functional>
#include <deque>
#include <condition_variable>
#include <cstring>
#include <fstream>
#include <thread>

#include <sched.h>

#include "engine_internal.h"
#include "nvdec.h"
#include "swdec.h"
#include "storage.h"
#include "scn_kernels.h"

namespace scanner {
namespace internal {

namespace {

Result ok() {
  Result r;
  r.set_success(true);
  return r;
}

void mkdirs(const std::string& path) {
  std::string cur;
  for (size_t i = 0; i <= path.size(); ++i) {
    if (i == path.size() || path[i] == '/') {
      if (!cur.empty()) mkdir(cur.c_str(), 0755);
    }
    if (i < path.size()) cur.push_back(path[i]);
  }
}

// One keyframe interval of a task's rows (reference column_source.cpp:124-184
// slice_into_video_intervals): frames [kf_start, kf_end) must be fed, `wanted` are the positions
// (relative to kf_start) of the rows this task needs, out_base their index in the task's rows.
struct VideoInterval {
  i64 kf_start, kf_end;
  std::vector<i64> wanted;
  i64 out_base;
};

// `skip` (optional, one flag per row): rows delivered by other means (halo elements received from a
// neighbouring rank); they form a prefix and/or suffix of `rows`, so the decoded rows in between keep
// consecutive indices.
std::vector<VideoInterval> slice_into_intervals(const H264Index& idx, const std::vector<i64>& rows,
                                                const std::vector<u8*>* skip = nullptr) {
  std::vector<VideoInterval> out;
  const std::vector<i64>& kf = idx.keyframe_indices;
  for (size_t i = 0; i < rows.size(); ++i) {
    if (skip && (*skip)[i]) continue;
    const i64 r = rows[i];
    // keyframe interval containing r
    const size_t k = (size_t)(std::upper_bound(kf.begin(), kf.end(), r) - kf.begin()) - 1;
    const i64 start = kf[k];
    const i64 end = k + 1 < kf.size() ? kf[k + 1] : idx.frames();
    if (out.empty() || out.back().kf_start != start) out.push_back({start, end, {}, (i64)i});
    out.back().wanted.push_back(r - start);
  }
  return out;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// Save workers (reference SaveWorker threads, worker.cpp:1718-1800: `save_workers_per_node`, default 4): finished
// tasks are written to their table items by these threads while the pipeline instance that produced them goes on
// decoding.  A bounded queue: a producer that finds it full writes its item itself.
class SavePool {
 public:
  explicit SavePool(int threads) {
    for (int i = 0; i < threads; ++i) workers_.emplace_back([this] { loop(); });
  }
  ~SavePool() {
    {
      std::lock_guard<std::mutex> g(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    for (auto& t : workers_) t.join();
  }
  // false: the queue is full (the caller runs the job itself)
  bool submit(std::function<void()> job) {
    {
      std::lock_guard<std::mutex> g(mu_);
      if (queue_.size() >= kMaxPending) return false;
      queue_.push_back(std::move(job));
      ++pending_;
    }
    cv_.notify_one();
    return true;
  }
  void wait_idle() {
    std::unique_lock<std::mutex> g(mu_);
    idle_.wait(g, [this] { return pending_ == 0; });
  }

 private:
  static constexpr size_t kMaxPending = 32;
  void loop() {
    for (;;) {
      std::function<void()> job;
      {
        std::unique_lock<std::mutex> g(mu_);
        cv_.wait(g, [this] { return stop_ || !queue_.empty(); });
        if (queue_.empty()) return;
        job = std::move(queue_.front());
        queue_.pop_front();
      }
      job();
      {
        std::lock_guard<std::mutex> g(mu_);
        if (--pending_ == 0) idle_.notify_all();
      }
    }
  }
  std::mutex mu_;
  std::condition_variable cv_, idle_;
  std::deque<std::function<void()>> queue_;
  std::vector<std::thread> workers_;
  size_t pending_ = 0;
  bool stop_ = false;
};

struct Engine::RunState {
  Graph* graph = nullptr;
  GraphAnalysis an;
  std::vector<Job*> jobs;
  i32 wps = 0, ios = 0;
  std::string out_dir;
  struct Task {
    i32 job, task;
    i64 row0, row1;
    i32 group;  // slice group the rows belong to, -1 if the job is not sliced
  };
  std::vector<Task> tasks;
  std::atomic<size_t> next{0};
  std::atomic<bool> failed{false};
  std::mutex err_mu;
  std::string error;
  Profiler profiler;
  ResourceGate resource_gate;  // fetch_resources once per op and run
  std::unique_ptr<Database> db;  // open when a job saves sinks into tables of out_dir
  std::unique_ptr<SavePool> savers;  // with db: the threads that write finished tasks
  std::atomic<i64> frames_decoded{0}, frames_used{0}, frames_native{0};
  // decoded elements received from neighbouring ranks: (input stream, source row) -> buffer on halo_dev
  std::map<std::pair<const InputStream*, i64>, u8*> halo_rows;
  DeviceHandle halo_dev = CPU_DEVICE;
  i64 halo_bytes_sent = 0, halo_bytes_received = 0, halo_ns = 0;

  void fail(const std::string& msg) {
    std::lock_guard<std::mutex> g(err_mu);
    if (!failed.exchange(true)) error = msg;
  }
};

struct Engine::Instance {
  Engine* eng;
  i32 gpu_id;
  i32 node_id;
  i32 index = 0;  // position in this run's instance list (trace tid)
  std::thread th;
  // what this instance did in the run (per-session decode rate = frames_decoded / decode_busy_ns)
  i64 frames_decoded = 0, decode_busy_ns = 0, wall_ns = 0, tasks_done = 0;
};

// What survives between runs for pipeline-instance slot `node_id`: its CUDA stream and its NVDEC
// sessions (creating a decoder costs ~0.25 s; the reference re-creates parser and decoder on
// every configure(), nvidia_video_decoder.cpp:100-112).
struct Engine::Slot {
  i32 gpu_id = -1;
  cudaStream_t stream = nullptr;
  std::map<i32, std::unique_ptr<NvdecSession>> sessions;     // per video source op index
  std::map<i32, std::unique_ptr<SwdecSession>> sw_sessions;  // the same for a CPU instance (swdec.h)
};

Engine::Engine(std::vector<i32> gpu_ids, i32 instances_per_gpu, i32 cpu_instances)
  : gpu_ids_(std::move(gpu_ids)), instances_per_gpu_(instances_per_gpu), cpu_instances_(cpu_instances) {
  if (!gpu_ids_.empty() && !cuda_available()) {
    LOG(ERROR) << "engine created with GPUs but CUDA is not available; GPU work will fail";
  }
  init_memory_allocators(MemoryPoolConfig(), gpu_ids_);
}

Engine::~Engine() {
  halo_decoders_.clear();
  halo_.reset();
  for (auto& sl : slots_) {
    if (sl->gpu_id >= 0 && cuda_available()) {
      cudaSetDevice(sl->gpu_id);
      sl->sessions.clear();
      if (sl->stream) cudaStreamDestroy(sl->stream);
    }
  }
  slots_.clear();
  std::lock_guard<std::mutex> g(streams_mu_);
  for (auto& kv : streams_)
    if (!kv.second->data.empty()) {
      disown_block(CPU_DEVICE, kv.second->data.data());
      // the payload was page-locked in add_stream: release the registration before the memory
      if (kv.second->registered && cudaHostUnregister(kv.second->data.data()) != cudaSuccess) cudaGetLastError();
    }
}

i64 Engine::add_stream(std::unique_ptr<InputStream> s) {
  if (!s->data.empty()) {
    adopt_block(CPU_DEVICE, s->data.data(), s->data.size());
    // page-lock the payload so GPU instances can DMA straight from it
    if (cuda_available() && !gpu_ids_.empty()) {
      if (cudaHostRegister(s->data.data(), PageAllocator<u8>::padded(s->data.size()), cudaHostRegisterPortable) ==
          cudaSuccess)
        s->registered = true;
      else
        cudaGetLastError();
    }
  }
  std::lock_guard<std::mutex> g(streams_mu_);
  const i64 id = next_stream_id_++;
  streams_[id] = std::move(s);
  return id;
}

InputStream* Engine::stream(i64 id) {
  std::lock_guard<std::mutex> g(streams_mu_);
  auto it = streams_.find(id);
  return it == streams_.end() ? nullptr : it->second.get();
}

bool Engine::remove_stream(i64 id) {
  std::lock_guard<std::mutex> g(streams_mu_);
  auto it = streams_.find(id);
  if (it == streams_.end()) return false;
  if (!it->second->data.empty()) {
    disown_block(CPU_DEVICE, it->second->data.data());
    if (it->second->registered && cudaHostUnregister(it->second->data.data()) != cudaSuccess) cudaGetLastError();
  }
  streams_.erase(it);
  return true;
}

// ---------------------------------------------------------------------------------------------
namespace {

// Per-source cursor over the rows one task needs.
struct SourceCursor {
  i32 op = 0;
  InputStream* stream = nullptr;
  std::vector<i64> rows;
  // video state
  std::vector<VideoInterval> intervals;
  size_t cur_interval = 0;
  bool interval_open = false;
  std::unique_ptr<NvdecSession> session;
  std::vector<u8*> halo;      // per row: non-null = the element was received from another rank (not decoded here)
  std::map<i64, u8*> blocks;  // packet index -> frame block on the GPU (RGB24, or NV12 surfaces)
  size_t frame_bytes = 0;
  bool nv12 = false;          // deliver decoder-native surfaces (every consumer accepts them)
  i64 wps = 1;
  DeviceHandle gpu_dev;

  // destination of decoded picture `out_index` (index into `rows`); packet blocks are allocated
  // on first touch because a decoder may deliver pictures of the next packet early
  u8* slot(i64 out_index) {
    const i64 pk = out_index / wps;
    auto it = blocks.find(pk);
    if (it == blocks.end()) {
      const size_t n = std::min(rows.size(), (size_t)(pk + 1) * (size_t)wps) - (size_t)pk * (size_t)wps;
      it = blocks.emplace(pk, new_block_buffer_size(gpu_dev, frame_bytes, (i32)n)).first;
    }
    return it->second + (size_t)(out_index - pk * wps) * frame_bytes;
  }
};

}  // namespace

void TaskOutput::release() {
  if (!held.empty()) delete_elements(CPU_DEVICE, held);
  held.clear();
  ext.clear();
}

// Run the calling thread on the CPUs that are local to `gpu` (its PCIe root's NUMA node,
// /sys/bus/pci/devices/<bdf>/local_cpulist) intersected with what the process may use.  A decode
// thread spends its life in cuvidMapVideoFrame waiting for doorbells from that GPU; on a two-socket
// host a thread on the far socket adds a cross-socket hop to every wake-up.
// SCN_PIN_NUMA=0 disables.  Returns the number of CPUs in the mask (0: left alone).
static int pin_thread_to_gpu_numa(i32 gpu) {
  const char* e = getenv("SCN_PIN_NUMA");
  if (e && e[0] == '0') return 0;
  char bdf[32] = {0};
  if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), gpu) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  for (char* c = bdf; *c; ++c) *c = (char)tolower(*c);
  std::ifstream f(std::string("/sys/bus/pci/devices/") + bdf + "/local_cpulist");
  std::string list;
  if (!f || !std::getline(f, list) || list.empty()) return 0;
  cpu_set_t allowed, want;
  CPU_ZERO(&want);
  if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return 0;
  size_t pos = 0;
  while (pos < list.size()) {  // "0-31,64-95"
    size_t end = list.find(',', pos);
    if (end == std::string::npos) end = list.size();
    const std::string part = list.substr(pos, end - pos);
    const size_t dash = part.find('-');
    const int a = atoi(part.c_str()), b = dash == std::string::npos ? a : atoi(part.c_str() + dash + 1);
    for (int c = a; c <= b && c < CPU_SETSIZE; ++c)
      if (c >= 0 && CPU_ISSET(c, &allowed)) CPU_SET(c, &want);
    pos = end + 1;
  }
  const int n = CPU_COUNT(&want);
  if (n == 0 || n == CPU_COUNT(&allowed)) return 0;
  return sched_setaffinity(0, sizeof(want), &want) == 0 ? n : 0;
}

void Engine::instance_main(Instance* inst) {
  RunState& rs = *run_;
  const i32 gpu = inst->gpu_id;
  if (gpu >= 0 && cuda_available()) {
    const int pinned = pin_thread_to_gpu_numa(gpu);
    if (pinned && inst->index == 0) rs.profiler.increment("numa_pinned_cpus", pinned);
  }
  Slot& slot = *slots_[(size_t)inst->node_id];
  if (gpu >= 0) {
    if (cudaSetDevice(gpu) != cudaSuccess) {
      rs.fail("cannot initialise GPU " + std::to_string(gpu));
      return;
    }
    if (slot.gpu_id != gpu || !slot.stream) {
      slot.sessions.clear();
      if (slot.stream) cudaStreamDestroy(slot.stream);
      slot.stream = nullptr;
      if (cudaStreamCreateWithFlags(&slot.stream, cudaStreamNonBlocking) != cudaSuccess) {
        rs.fail("cannot create a stream on GPU " + std::to_string(gpu));
        return;
      }
      slot.gpu_id = gpu;
    }
    set_thread_stream(gpu, slot.stream);
  }
  cudaStream_t stream = slot.stream;
  Profiler::thread_worker() = inst->index;
  const DeviceHandle gpu_dev(DeviceType::GPU, gpu);
  const DeviceHandle dec_dev = gpu >= 0 ? gpu_dev : CPU_DEVICE;  // where decoded pictures live
  {
    EvaluateWorker ew(*rs.graph, rs.an, gpu, inst->node_id, &rs.profiler, &rs.resource_gate);
    Result r = ew.init();
    if (!r.success()) {
      rs.fail(r.msg());
      return;
    }
    std::map<i32, std::unique_ptr<NvdecSession>>& sessions = slot.sessions;
    i64 decoded0 = 0, used0 = 0, busy0 = 0;
    for (auto& kv : sessions) {
      decoded0 += kv.second->frames_decoded();
      used0 += kv.second->frames_used();
      busy0 += kv.second->busy_ns();
    }
    for (auto& kv : slot.sw_sessions) {
      decoded0 += kv.second->frames_decoded();
      used0 += kv.second->frames_used();
    }
    const auto inst_t0 = std::chrono::steady_clock::now();

    while (!rs.failed.load()) {
      const size_t ti = shared_next_ ? (size_t)__atomic_fetch_add(shared_next_, 1ull, __ATOMIC_RELAXED)
                                    : rs.next.fetch_add(1);
      if (ti >= rs.tasks.size()) break;
      const RunState::Task& t = rs.tasks[ti];
      Job& job = *rs.jobs[t.job];
      const timepoint_t task_start = now();

      std::vector<i64> out_rows;
      for (i64 row = t.row0; row < t.row1; ++row) out_rows.push_back(row);
      std::vector<TaskStream> streams;
      if (t.group >= 0) {
        // a task of a sliced job sees its group's domain: Slice = gather of the group's rows,
        // Unslice = offset into the concatenated output, per-group samplers / stream args
        JobParams view;
        std::vector<i64> view_rows;
        rs.graph->slice_view(job.params, job.slices, t.group, view, view_rows);
        r = rs.graph->derive_task_streams(rs.an, view, view_rows, out_rows, streams);
        if (r.success()) r = ew.new_task(view, view_rows, streams);
      } else {
        r = rs.graph->derive_task_streams(rs.an, job.params, job.rows_per_op, out_rows, streams);
        if (r.success()) r = ew.new_task(job.params, job.rows_per_op, streams);
      }
      if (!r.success()) {
        rs.fail(r.msg());
        break;
      }

      // ---- load stage: cursors over every source's rows (reference LoadWorker::yield)
      std::vector<SourceCursor> cursors;
      size_t max_rows = 0;
      for (size_t k = 0; k < rs.graph->ops.size() && r.success(); ++k) {
        if (rs.graph->ops[k].kind != OpKind::Source) continue;
        SourceCursor c;
        c.op = (i32)k;
        {
          auto bit = job.source_streams.find((i32)k);
          c.stream = bit == job.source_streams.end() ? nullptr : this->stream(bit->second);
        }
        c.wps = rs.wps;
        c.gpu_dev = dec_dev;
        c.rows = streams[k].valid_output_rows;
        if (!c.stream) {
          RESULT_ERROR(&r, "job %d does not bind source op %zu to a stream", t.job, k);
          break;
        }
        max_rows = std::max(max_rows, c.rows.size());
        if (!rs.halo_rows.empty()) {
          c.halo.assign(c.rows.size(), nullptr);
          bool any = false;
          for (size_t i = 0; i < c.rows.size(); ++i) {
            auto hit = rs.halo_rows.find({c.stream, c.rows[i]});
            if (hit != rs.halo_rows.end()) {
              c.halo[i] = hit->second;
              any = true;
            }
          }
          if (!any) c.halo.clear();
        }
        if (c.stream->kind == InputStream::H264) {
          if (gpu < 0) {
            // CPU instance: libavcodec + libswscale -> RGB24 in host memory (swdec.h; reference
            // SoftwareVideoDecoder).  Fails here, with the reason, when no FFmpeg can be loaded.
            auto& s = slot.sw_sessions[(i32)k];
            if (!s) {
              // libavcodec threads per session (reference: num_cpus / instances, worker.cpp:1631).  One by default:
              // on the 640x480 configs[0] clip 8 frame threads gave 1,045 frames/s against 986 with one -- the
              // instance's own swscale + op work is the serial part; SCN_SWDEC_THREADS raises it
              int threads = 1;
              if (const char* e = getenv("SCN_SWDEC_THREADS")) threads = atoi(e);
              threads = threads < 1 ? 1 : (threads > 64 ? 64 : threads);
              s.reset(new SwdecSession(threads));
              Result ir = s->init();
              if (!ir.success()) {
                slot.sw_sessions.erase((i32)k);
                r = ir;
                break;
              }
            }
          } else {
            auto& s = sessions[(i32)k];
            if (!s) {
              s.reset(new NvdecSession(gpu, stream));
              Result ir = s->init();
              if (!ir.success()) {
                r = ir;
                break;
              }
            }
          }
          c.intervals = slice_into_intervals(c.stream->index, c.rows, c.halo.empty() ? nullptr : &c.halo);
          // decoder-native delivery when every consumer kernel takes NV12 (frame.h FrameLayout);
          // SCN_DECODE_RGB=1 forces the reference's RGB24 elements
          const char* force_rgb = getenv("SCN_DECODE_RGB");
          c.nv12 = gpu >= 0 && !(force_rgb && force_rgb[0] == '1') &&
                   rs.graph->consumers_accept_layout((i32)k, FrameLayout::NV12);
          const size_t px = (size_t)c.stream->index.width * c.stream->index.height;
          c.frame_bytes = c.nv12 ? px + px / 2 : px * 3;
        }
        cursors.push_back(std::move(c));
      }
      if (!r.success()) {
        rs.fail(r.msg());
        break;
      }

      const size_t n_packets = (max_rows + (size_t)rs.wps - 1) / (size_t)rs.wps;
      std::map<i32, TaskOutput*> outs;
      for (auto& kv : job.outputs) outs[kv.first] = &kv.second[t.task];

      for (size_t p = 0; p < n_packets && r.success(); ++p) {
        std::map<i32, ColumnBatch> src_cols;
        for (SourceCursor& c : cursors) {
          const size_t i0 = std::min(c.rows.size(), p * (size_t)rs.wps);
          const size_t i1 = std::min(c.rows.size(), (p + 1) * (size_t)rs.wps);
          ColumnBatch cb;
          InputStream& st = *c.stream;
          if (st.kind == InputStream::H264) {
            // ---- decode stage (reference PreEvaluateWorker::yield + DecoderAutomata::get_frames)
            const timepoint_t d0 = now();
            cb.device = dec_dev;
            NvdecSession* hw = gpu >= 0 ? sessions[c.op].get() : nullptr;
            SwdecSession* sw = gpu >= 0 ? nullptr : slot.sw_sessions[c.op].get();
            auto sess_delivered = [&] { return hw ? hw->delivered() : sw->delivered(); };
            const FrameInfo finfo = c.nv12 ? FrameInfo::nv12(st.index.width, st.index.height)
                                           : FrameInfo(st.index.height, st.index.width, 3, FrameType::U8);
            size_t delivered_global = c.cur_interval < c.intervals.size()
                                          ? (size_t)c.intervals[c.cur_interval].out_base +
                                                (c.interval_open ? sess_delivered() : 0)
                                          : c.rows.size();
            while (delivered_global < i1 && r.success()) {
              VideoInterval& iv = c.intervals[c.cur_interval];
              if (!c.interval_open) {
                std::vector<u64> offs(st.index.sample_offsets.begin() + iv.kf_start,
                                      st.index.sample_offsets.begin() + iv.kf_end);
                std::vector<u64> szs(st.index.sample_sizes.begin() + iv.kf_start,
                                     st.index.sample_sizes.begin() + iv.kf_end);
                const size_t w = (size_t)st.index.width, h = (size_t)st.index.height;
                if (sw)
                  r = sw->begin_interval(st.encoded.data(), offs, szs, st.index.metadata_packets, st.index.may_reorder,
                                         iv.wanted, iv.out_base, (int)w, (int)h,
                                         [cur = &c](i64 out_index) { return cur->slot(out_index); });
                else
                r = hw->begin_interval(
                    st.encoded.data(), offs, szs, st.index.metadata_packets, st.index.may_reorder, iv.wanted, iv.out_base,
                    (int)w, (int)h, [cur = &c, rsp = &rs, stream, w, h](i64 out_index, const Nv12Surface& s) {
                      const u8* lp = s.luma;
                      const u8* cp = s.chroma;
                      u8* dst = cur->slot(out_index);
                      // the element slots are sized from the index; a stream whose own SPS says
                      // otherwise (resolution change mid-stream, foreign descriptor) must not be copied
                      if ((size_t)s.width != w || (size_t)s.height != h) {
                        rsp->fail("decoded picture is " + std::to_string(s.width) + "x" + std::to_string(s.height) +
                                  " but the stream index says " + std::to_string(w) + "x" + std::to_string(h));
                        return;
                      }
                      if (cur->nv12) {
                        const int rc = scn_nv12_pack(&lp, &cp, s.pitch, 1, (int)w, (int)h, &dst, stream);
                        if (rc != 0) rsp->fail("scn_nv12_pack failed: " + std::to_string(rc));
                        return;
                      }
                      const int rc = scn_nv12_to_rgb24(&lp, &cp, s.pitch, 1, (int)w, (int)h, &dst, w * 3, stream);
                      if (rc != 0) rsp->fail("scn_nv12_to_rgb24 failed: " + std::to_string(rc));
                    });
                if (!r.success()) break;
                c.interval_open = true;
              }
              const size_t want_in_iv = std::min(iv.wanted.size(), i1 - (size_t)iv.out_base);
              r = hw ? hw->advance(want_in_iv) : sw->advance(want_in_iv);
              if (!r.success()) break;
              if (sess_delivered() >= iv.wanted.size()) {
                r = hw ? hw->end_interval() : sw->end_interval();
                c.interval_open = false;
                ++c.cur_interval;
                delivered_global = c.cur_interval < c.intervals.size() ? (size_t)c.intervals[c.cur_interval].out_base
                                                                       : c.rows.size();
              } else {
                delivered_global = (size_t)iv.out_base + sess_delivered();
              }
            }
            if (!r.success()) break;
            for (size_t i = i0; i < i1; ++i) {
              if (!c.halo.empty() && c.halo[i]) {  // received from the rank that owns the row
                add_buffer_ref(dec_dev, c.halo[i]);
                cb.elements.push_back(Element(new Frame(finfo, c.halo[i])));
                // the packet's block counts one reference per row: give back this row's unused slot
                if (c.blocks.count((i64)i / c.wps)) delete_buffer(dec_dev, c.slot((i64)i));
              } else {
                cb.elements.push_back(Element(new Frame(finfo, c.slot((i64)i))));
              }
              cb.row_ids.push_back(c.rows[i]);
            }
            if (c.nv12) rs.frames_native += (i64)(i1 - i0);
            c.blocks.erase((i64)p);  // ownership of the packet's block now rides on its elements
            rs.profiler.add_interval("get_frames", d0, now());
          } else {
            cb.device = CPU_DEVICE;
            for (size_t i = i0; i < i1; ++i) {
              const i64 row = c.rows[i];
              if (row < 0 || row >= st.rows()) {
                RESULT_ERROR(&r, "source row %ld out of range (%ld rows)", (long)row, (long)st.rows());
                break;
              }
              u8* ptr = st.data.data() + st.offsets[row];
              if (!c.halo.empty() && c.halo[i] && st.kind == InputStream::RawFrames) {
                add_buffer_ref(CPU_DEVICE, c.halo[i]);
                cb.elements.push_back(Element(new Frame(st.info, c.halo[i])));
              } else if (st.kind == InputStream::RawFrames) {
                add_buffer_ref(CPU_DEVICE, ptr);
                cb.elements.push_back(Element(new Frame(st.info, ptr)));
              } else if (st.sizes[row] == 0) {
                cb.elements.emplace_back();  // null row
              } else {
                add_buffer_ref(CPU_DEVICE, ptr);
                cb.elements.push_back(Element(ptr, st.sizes[row]));
              }
              cb.row_ids.push_back(row);
            }
            rs.profiler.increment("io_read", (i64)(i1 - i0));
          }
          src_cols[c.op] = std::move(cb);
        }
        if (!r.success()) break;

        // ---- evaluate stage
        std::map<i32, ColumnBatch> sink_cols;
        r = ew.feed(src_cols, sink_cols);
        if (!r.success()) break;

        // ---- post-evaluate + save: bring sink rows to the host and append them to the task
        for (auto& kv : sink_cols) {
          ColumnBatch& cb = kv.second;
          Elements host = cb.device.is_gpu() ? copy_or_ref_elements(cb.device, CPU_DEVICE, cb.elements) : cb.elements;
          TaskOutput& to = *outs[kv.first];
          for (Element& e : host) {
            const u8* src = nullptr;
            size_t n = 0;
            i32 shape[4] = {0, 0, 0, -1};
            if (!e.is_null()) {
              if (e.is_frame) {
                const Frame* f = e.as_const_frame();
                src = f->data;
                n = f->size();
                shape[0] = f->shape[0];
                shape[1] = f->shape[1];
                shape[2] = f->shape[2];
                shape[3] = (i32)(proto::FrameType)f->type;
              } else {
                src = e.buffer;
                n = e.size;
              }
            }
            to.offsets.push_back(to.data.size());
            to.sizes.push_back(n);
            to.shapes.insert(to.shapes.end(), shape, shape + 4);
            // rows that pass an input stream through unchanged still point into the stream's adopted
            // storage, which goes away with the stream (remove_stream / ~Engine), possibly before the
            // job's outputs do: those are copied, only engine-allocated blocks are held by reference
            if (n >= TaskOutput::kLargeRow && !block_is_external(CPU_DEVICE, src)) {
              to.ext.resize(to.sizes.size(), nullptr);
              to.ext.back() = src;
              to.held.push_back(e);  // the reference this element holds on its block moves to the task
              e = Element();
            } else if (n) {
              to.data.insert(to.data.end(), src, src + n);
            }
          }
          delete_elements(CPU_DEVICE, host);  // rows kept above were replaced by null elements
          if (cb.device.is_gpu()) delete_elements(cb.device, cb.elements);
        }
      }
      // close decoder intervals left open by a task that did not need their tail
      for (SourceCursor& c : cursors) {
        if (c.interval_open) {
          Result e = sessions[c.op]->end_interval();
          if (r.success() && !e.success()) r = e;
        }
        for (auto& kv : c.blocks) delete_buffer(gpu_dev, kv.second);
      }
      if (r.success()) r = ew.end_task();
      if (!r.success()) {
        rs.fail(r.msg());
        break;
      }
      for (auto& kv : outs) {
        if ((i64)kv.second->sizes.size() != t.row1 - t.row0) {
          rs.fail("sink " + std::to_string(kv.first) + " stored " + std::to_string(kv.second->sizes.size()) +
                  " rows for a task of " + std::to_string(t.row1 - t.row0));
          break;
        }
        kv.second->done = true;
      }
      if (rs.failed.load()) break;

      // ---- save stage into database tables (reference SaveWorker::feed + ColumnSink::write,
      // save_worker.cpp:73-151, column_sink.cpp:71-201): one item per task, then the memory goes
      if (!job.sink_tables.empty()) {
        for (auto& kv : outs) {
          auto st = job.sink_tables.find(kv.first);
          if (st == job.sink_tables.end()) continue;
          TaskOutput* to = kv.second;
          // Video or Bytes item: from the declared type of the column (a task whose rows are all null
          // has no frame to look at and must still be a video item of a Video table)
          const bool video = job.sink_is_frame.count(kv.first) && job.sink_is_frame.at(kv.first);
          const i32 table = st->second, task_id = t.task;
          const i64 row0 = t.row0, row1 = t.row1;
          const bool keep = job.keep_rows;
          RunState* rsp = &rs;
          auto write = [rsp, to, video, table, task_id, row0, row1, keep] {
            std::vector<u8> flat;
            ItemColumn ic;
            if (to->held.empty()) {
              ic.data = to->data.data();
              ic.bytes = to->data.size();
            } else {
              flat.reserve(to->total_bytes());
              for (size_t i = 0; i < to->sizes.size(); ++i) flat.insert(flat.end(), to->row(i), to->row(i) + to->sizes[i]);
              ic.data = flat.data();
              ic.bytes = flat.size();
            }
            ic.sizes = &to->sizes;
            ic.shapes = &to->shapes;
            Result wr = rsp->db->write_index_item(table, task_id, row0, row1);
            if (wr.success()) wr = rsp->db->write_item(table, 1, task_id, ic, video);
            if (!wr.success()) {
              rsp->fail(wr.msg());
              return;
            }
            rsp->profiler.increment("io_write", (i64)ic.bytes);
            if (!keep) {
              to->release();
              std::vector<u8>().swap(to->data);
              to->dropped = true;
            }
          };
          // the rows of a finished task are complete and nobody else touches them until the run ends
          if (!rs.savers || !rs.savers->submit(write)) write();
        }
        if (rs.failed.load()) break;
      } else if (!rs.out_dir.empty()) {
        // ---- plain column files (reference ColumnSink::write, column_sink.cpp:159-195)
        const std::string dir = rs.out_dir + "/tables/" + std::to_string(t.job);
        mkdirs(dir);
        auto write_col = [&](i32 col, const std::vector<u64>& sizes, const u8* data, size_t nbytes) {
          const std::string base = dir + "/" + std::to_string(col) + "_" + std::to_string(t.task);
          std::ofstream meta(base + "_metadata.bin", std::ios::binary);
          const u64 n = sizes.size();
          meta.write((const char*)&n, 8);
          meta.write((const char*)sizes.data(), (std::streamsize)(8 * sizes.size()));
          std::ofstream dat(base + ".bin", std::ios::binary);
          dat.write((const char*)data, (std::streamsize)nbytes);
          rs.profiler.increment("io_write", (i64)nbytes);
        };
        // column 0: the index column, row i = little-endian int64 i (reference ingest.cpp:337-345)
        std::vector<u64> isz((size_t)(t.row1 - t.row0), 8);
        std::vector<i64> idx;
        for (i64 row = t.row0; row < t.row1; ++row) idx.push_back(row);
        write_col(0, isz, (const u8*)idx.data(), idx.size() * 8);
        i32 col = 1;
        for (auto& kv : outs) {
          const TaskOutput& to = *kv.second;
          if (to.held.empty()) {
            write_col(col++, to.sizes, to.data.data(), to.data.size());
          } else {  // rows kept in page-locked blocks: gather them for the writer
            std::vector<u8> flat;
            flat.reserve(to.total_bytes());
            for (size_t i = 0; i < to.sizes.size(); ++i) flat.insert(flat.end(), to.row(i), to.row(i) + to.sizes[i]);
            write_col(col++, to.sizes, flat.data(), flat.size());
          }
        }
      }
      rs.profiler.add_interval("task", task_start, now());
      ++inst->tasks_done;
    }
    i64 busy1 = 0, decoded1 = 0;
    for (auto& kv : sessions) {
      kv.second->drain();
      rs.frames_decoded += kv.second->frames_decoded();
      rs.frames_used += kv.second->frames_used();
      decoded1 += kv.second->frames_decoded();
      busy1 += kv.second->busy_ns();
    }
    for (auto& kv : slot.sw_sessions) {
      rs.frames_decoded += kv.second->frames_decoded();
      rs.frames_used += kv.second->frames_used();
      decoded1 += kv.second->frames_decoded();
    }
    rs.frames_decoded -= decoded0;
    rs.frames_used -= used0;
    inst->frames_decoded = decoded1 - decoded0;
    inst->decode_busy_ns = busy1 - busy0;
    inst->wall_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - inst_t0).count();
    if (gpu >= 0) cudaStreamSynchronize(stream);
  }  // kernels destroyed here, while the stream is alive
  if (gpu >= 0) {
    cudaStreamSynchronize(stream);
    set_thread_stream(gpu, nullptr);
  }
}

Result Engine::write_trace(const std::string& path) const {
  Result r;
  std::ofstream f(path, std::ios::trunc);
  if (!f) {
    RESULT_ERROR(&r, "cannot write %s", path.c_str());
    return r;
  }
  auto esc = [](const std::string& s) {
    std::string o;
    for (char c : s) {
      if (c == '"' || c == '\\') o.push_back('\\');
      o.push_back(c);
    }
    return o;
  };
  f << "{\"displayTimeUnit\": \"ms\", \"traceEvents\": [\n";
  bool first = true;
  for (const TraceEvent& e : stats_.trace) {
    char buf[96];
    snprintf(buf, sizeof(buf), "\"ts\": %.3f, \"dur\": %.3f", (double)e.start_ns * 1e-3,
             (double)(e.end_ns - e.start_ns) * 1e-3);
    f << (first ? "" : ",\n") << "{\"name\": \"" << esc(e.key) << "\", \"ph\": \"X\", " << buf
      << ", \"pid\": " << e.node << ", \"tid\": " << e.worker << "}";
    first = false;
  }
  f << "\n]}\n";
  r.set_success((bool)f);
  if (!f) r.set_msg("short write to " + path);
  return r;
}

Result Engine::decode_rows_to_device(i64 stream_id, const std::vector<i64>& rows, i32 gpu_id, u8* dst) {
  Result r;
  InputStream* st = stream(stream_id);
  if (!st || st->kind != InputStream::H264) {
    RESULT_ERROR(&r, "stream %ld is not an H.264 stream", (long)stream_id);
    return r;
  }
  return decode_rows(*st, rows, gpu_id, false, dst);
}

// rows (ascending) of an H.264 stream -> dense elements in device memory: packed NV12 surfaces
// (w*h*3/2 bytes each) or RGB24 frames
struct Engine::DecodeContext {
  i32 gpu = -1;
  cudaStream_t stream = nullptr;
  std::unique_ptr<NvdecSession> session;
  ~DecodeContext() {
    if (gpu >= 0 && cuda_available()) {
      ScopedDevice sd(gpu);
      session.reset();
      if (stream) cudaStreamDestroy(stream);
    }
  }
};

Result Engine::decode_rows(InputStream& stref, const std::vector<i64>& rows, i32 gpu_id, bool nv12, u8* dst,
                           DecodeContext* reuse) {
  Result r;
  InputStream* st = &stref;
  for (size_t i = 0; i < rows.size(); ++i)
    if (rows[i] < 0 || rows[i] >= st->rows() || (i && rows[i] <= rows[i - 1])) {
      RESULT_ERROR(&r, "rows must be ascending and inside [0, %ld)", (long)st->rows());
      return r;
    }
  if (rows.empty()) return ok();
  if (!cuda_available() || gpu_id < 0 || !dst) {
    RESULT_ERROR(&r, "decoding rows into device memory (scn_engine_decode_to_device, halo rows of a sharded clip) "
                     "needs a GPU: it goes through NVDEC; CPU pipeline instances decode inside scn_engine_run");
    return r;
  }
  ScopedDevice sd(gpu_id);
  DecodeContext local;
  DecodeContext& ctx = reuse ? *reuse : local;
  if (!ctx.stream) {
    ctx.gpu = gpu_id;
    if (cudaStreamCreateWithFlags(&ctx.stream, cudaStreamNonBlocking) != cudaSuccess) {
      RESULT_ERROR(&r, "cannot create a stream on GPU %d", gpu_id);
      return r;
    }
  }
  cudaStream_t cs = ctx.stream;
  if (!ctx.session) {
    ctx.session.reset(new NvdecSession(gpu_id, cs));
    r = ctx.session->init();
    if (!r.success()) {
      ctx.session.reset();
      return r;
    }
  } else {
    r.set_success(true);
  }
  {
    NvdecSession& sess = *ctx.session;
    const size_t w = (size_t)st->index.width, h = (size_t)st->index.height, fb = nv12 ? w * h * 3 / 2 : w * h * 3;
    std::string kerr;
    for (const VideoInterval& iv : slice_into_intervals(st->index, rows)) {
      if (!r.success()) break;
      std::vector<u64> offs(st->index.sample_offsets.begin() + iv.kf_start, st->index.sample_offsets.begin() + iv.kf_end);
      std::vector<u64> szs(st->index.sample_sizes.begin() + iv.kf_start, st->index.sample_sizes.begin() + iv.kf_end);
      r = sess.begin_interval(st->encoded.data(), offs, szs, st->index.metadata_packets, st->index.may_reorder, iv.wanted,
                              iv.out_base, (int)w, (int)h,
                              [&, w, h, fb](i64 out_index, const Nv12Surface& s) {
                                const u8* lp = s.luma;
                                const u8* cp = s.chroma;
                                u8* d = dst + (size_t)out_index * fb;
                                if ((size_t)s.width != w || (size_t)s.height != h) {
                                  kerr = "decoded picture is " + std::to_string(s.width) + "x" + std::to_string(s.height) +
                                         " but the stream index says " + std::to_string(w) + "x" + std::to_string(h);
                                  return;
                                }
                                const int rc = nv12 ? scn_nv12_pack(&lp, &cp, s.pitch, 1, (int)w, (int)h, &d, cs)
                                                    : scn_nv12_to_rgb24(&lp, &cp, s.pitch, 1, (int)w, (int)h, &d, w * 3, cs);
                                if (rc != 0) kerr = "decode-stage kernel failed: " + std::to_string(rc);
                              });
      if (r.success()) r = sess.end_interval();
    }
    sess.drain();
    cudaStreamSynchronize(cs);
    if (r.success() && !kerr.empty()) RESULT_ERROR(&r, "%s", kerr.c_str());
  }
  return r;  // a call-local context (session, stream) is destroyed here
}

// ---- stencil halo exchange of sharded jobs (halo.h) ------------------------------------------------
// For every job that computes one interval of a clip: which source rows do the OTHER intervals' tasks
// need from mine (derive_task_streams over their output rows -- the same back-propagation the reference
// uses to over-fetch, dag_analysis.cpp:1470-1718), which do mine need from theirs.  Mine are decoded
// once here and sent; theirs are received into element buffers the decode stage then hands out instead
// of decoding.  Every rank builds its transfer list in (job, source op, row) order, so the lists of a
// pair of ranks match; all transfers of the run go out in one group.
Result Engine::exchange_halos(Graph& graph, const std::vector<Job*>& jobs) {
  Result r = ok();
  RunState& rs = *run_;
  bool any = false;
  for (Job* jb : jobs) any = any || jb->shard_index >= 0;
  if (!any) return r;
  const auto t0 = std::chrono::steady_clock::now();
  const i32 my_rank = halo_ ? halo_->rank() : 0;
  struct Plan {
    Job* job;
    InputStream* st;
    i32 peer;
    std::vector<i64> rows;
    bool send;
    bool nv12;
    size_t frame_bytes;
    u8* staging = nullptr;  // sends: rows.size() dense elements
  };
  std::vector<Plan> plans;
  for (Job* jb : jobs) {
    if (jb->shard_index < 0) continue;
    Job& job = *jb;
    const size_t nsh = job.shard_ranks.size();
    auto window_rows = [&](size_t q) {
      std::vector<i64> rows;
      for (i64 row = job.shard_bounds[q]; row < job.shard_bounds[q + 1]; ++row) rows.push_back(row);
      return rows;
    };
    const i64 w0 = job.shard_bounds[(size_t)job.shard_index], w1 = job.shard_bounds[(size_t)job.shard_index + 1];
    for (size_t k = 0; k < graph.ops.size(); ++k) {
      if (graph.ops[k].kind != OpKind::Source) continue;
      auto bit = job.source_streams.find((i32)k);
      InputStream* st = bit == job.source_streams.end() ? nullptr : stream(bit->second);
      if (!st || st->kind == InputStream::Bytes) continue;  // byte rows are read from the stream, never decoded
      if (job.rows_per_op[k] != job.total_rows) {
        RESULT_ERROR(&r, "a sharded job needs sources with one row per output row (source %zu has %ld rows, the job %ld)",
                     k, (long)job.rows_per_op[k], (long)job.total_rows);
        return r;
      }
      const bool nv12 = st->kind == InputStream::H264 && !(getenv("SCN_DECODE_RGB") && getenv("SCN_DECODE_RGB")[0] == '1') &&
                        graph.consumers_accept_layout((i32)k, FrameLayout::NV12);
      size_t fb;
      if (st->kind == InputStream::H264) {
        const size_t px = (size_t)st->index.width * st->index.height;
        fb = nv12 ? px + px / 2 : px * 3;
      } else {
        fb = st->info.size();
      }
      for (size_t q = 0; q < nsh; ++q) {
        if ((i32)q == job.shard_index || job.shard_ranks[q] == my_rank) continue;
        // what shard q needs from my interval -> send; what I need from shard q's interval -> receive
        std::vector<TaskStream> ts;
        Result d = graph.derive_task_streams(rs.an, job.params, job.rows_per_op, window_rows(q), ts);
        if (!d.success()) return d;
        Plan snd{jb, st, job.shard_ranks[q], {}, true, nv12, fb};
        for (i64 row : ts[k].valid_output_rows)
          if (row >= w0 && row < w1) snd.rows.push_back(row);
        d = graph.derive_task_streams(rs.an, job.params, job.rows_per_op, window_rows((size_t)job.shard_index), ts);
        if (!d.success()) return d;
        Plan rcv{jb, st, job.shard_ranks[q], {}, false, nv12, fb};
        for (i64 row : ts[k].valid_output_rows)
          if (row >= job.shard_bounds[q] && row < job.shard_bounds[q + 1]) rcv.rows.push_back(row);
        if (!snd.rows.empty()) plans.push_back(std::move(snd));
        if (!rcv.rows.empty()) plans.push_back(std::move(rcv));
      }
    }
  }
  if (plans.empty()) return r;
  if (!halo_) {
    RESULT_ERROR(&r, "a sharded job needs rows from another rank but the engine has no halo transport "
                     "(scn_engine_comm_init / scn_engine_set_halo_callback)");
    return r;
  }
  const bool on_device = halo_->device_buffers();
  const DeviceHandle dev = on_device ? DeviceHandle(DeviceType::GPU, halo_->gpu_id()) : CPU_DEVICE;
  rs.halo_dev = dev;
  std::vector<HaloXfer> xfers;
  for (Plan& p : plans) {
    if ((p.st->kind == InputStream::H264) != on_device) {
      RESULT_ERROR(&r, "halo exchange: H.264 sources travel over the NCCL transport, raw-frame sources over the host "
                       "transport (stream kind %d, transport on %s)", (int)p.st->kind, on_device ? "device" : "host");
      break;
    }
    if (p.send) {
      if (on_device) {
        p.staging = new_buffer(dev, p.rows.size() * p.frame_bytes);
        std::unique_ptr<DecodeContext>& hd = halo_decoders_[dev.id];
        if (!hd) hd.reset(new DecodeContext());
        r = decode_rows(*p.st, p.rows, dev.id, p.nv12, p.staging, hd.get());
        if (!r.success()) break;
        for (size_t i = 0; i < p.rows.size(); ++i) xfers.push_back({p.peer, p.staging + i * p.frame_bytes, p.frame_bytes, true});
      } else {
        for (i64 row : p.rows) xfers.push_back({p.peer, p.st->data.data() + p.st->offsets[(size_t)row], p.frame_bytes, true});
      }
      rs.halo_bytes_sent += (i64)(p.rows.size() * p.frame_bytes);
    } else {
      for (i64 row : p.rows) {
        u8* buf = new_buffer(dev, p.frame_bytes);
        rs.halo_rows[{p.st, row}] = buf;
        xfers.push_back({p.peer, buf, p.frame_bytes, false});
      }
      rs.halo_bytes_received += (i64)(p.rows.size() * p.frame_bytes);
    }
  }
  if (r.success()) r = halo_->exchange(xfers);
  for (Plan& p : plans)
    if (p.staging) delete_buffer(dev, p.staging);
  rs.halo_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
  return r;
}

Result Engine::run(Graph& graph, const std::vector<Job*>& jobs, i32 wps, i32 ios, const std::string& out_dir) {
  Result r;
  if (wps <= 0 || ios <= 0 || ios % wps != 0) {
    // reference master.cpp:1421
    RESULT_ERROR(&r, "IO packet size (%d) must be a multiple of work packet size (%d).", ios, wps);
    return r;
  }
  run_.reset(new RunState());
  RunState& rs = *run_;
  rs.graph = &graph;
  rs.jobs = jobs;
  rs.wps = wps;
  rs.ios = ios;
  rs.out_dir = out_dir;
  for (Job* jb : jobs)
    if (!jb->sink_tables.empty() && !rs.db) {
      if (out_dir.empty()) {
        RESULT_ERROR(&r, "a job saves into tables but the run has no database directory (out_dir)");
        return r;
      }
      Result dr = Database::open(out_dir, rs.db);
      if (!dr.success()) return dr;
    }
  r = graph.analyze(rs.an);
  if (!r.success()) return r;

  // per job: bind source sizes, domain sizes, partition output rows into tasks
  // (reference master.cpp:1543-1606)
  for (size_t j = 0; j < jobs.size(); ++j) {
    Job& job = *jobs[j];
    job.params.source_rows.clear();
    for (auto& kv : job.source_streams) {
      InputStream* s = stream(kv.second);
      if (!s) {
        RESULT_ERROR(&r, "job %zu binds source %d to unknown stream %ld", j, kv.first, (long)kv.second);
        return r;
      }
      const GraphOp& op = graph.ops.at(kv.first);
      if (op.kind != OpKind::Source) {
        RESULT_ERROR(&r, "job %zu binds op %d which is not a Source", j, kv.first);
        return r;
      }
      if ((op.column_type == proto::Video) != (s->kind != InputStream::Bytes)) {
        RESULT_ERROR(&r, "job %zu: source %d column type does not match stream %ld", j, kv.first, (long)kv.second);
        return r;
      }
      job.params.source_rows[kv.first] = s->rows();
    }
    r = graph.domain_sizes(job.params, job.rows_per_op, &job.slices);
    if (!r.success()) return r;
    job.total_rows = 0;
    job.outputs.clear();
    for (size_t k = 0; k < graph.ops.size(); ++k)
      if (graph.ops[k].kind == OpKind::Sink) job.total_rows = job.rows_per_op[k];
    job.io_packet = ios;
    // tasks: io_packet-sized intervals of the output rows, never across a slice group boundary
    // (reference master.cpp:1567-1606 enumerates (slice group, row interval) the same way)
    job.task_starts.clear();
    std::vector<i32> groups_of_task;
    if (job.slices.groups > 0 && !job.slices.out_base.empty()) {
      for (i32 gi = 0; gi < job.slices.groups; ++gi)
        for (i64 row = job.slices.out_base[(size_t)gi]; row < job.slices.out_base[(size_t)gi + 1]; row += ios) {
          job.task_starts.push_back(row);
          groups_of_task.push_back(gi);
        }
    } else {
      for (i64 row = 0; row < job.total_rows; row += ios) {
        job.task_starts.push_back(row);
        groups_of_task.push_back(-1);
      }
    }
    i64 window_end = job.total_rows;
    if (job.shard_index >= 0 && shared_next_) {
      // a shared task queue indexes ONE task list that every rank builds identically; an interval-sharded job
      // (scn_job_set_shard) gives every rank different tasks
      RESULT_ERROR(&r, "job %zu: scn_job_set_shard cannot be combined with a shared task queue "
                       "(scn_engine_share_task_queue): the ranks' task lists would differ", j);
      return r;
    }
    if (job.shard_index >= 0) {
      // one interval of the clip: tasks cover [bounds[index], bounds[index + 1]) only
      const size_t nsh = job.shard_ranks.size();
      bool good = job.slices.groups == 0 && nsh >= 1 && job.shard_bounds.size() == nsh + 1 && (size_t)job.shard_index < nsh &&
                  job.shard_bounds.front() == 0 && job.shard_bounds.back() == job.total_rows;
      for (size_t q = 0; good && q < nsh; ++q) good = job.shard_bounds[q] <= job.shard_bounds[q + 1];
      if (!good) {
        RESULT_ERROR(&r, "job %zu: shard bounds must ascend from 0 to the job's %ld rows, one rank per interval, and the "
                         "graph must not slice", j, (long)job.total_rows);
        return r;
      }
      job.task_starts.clear();
      groups_of_task.clear();
      window_end = job.shard_bounds[(size_t)job.shard_index + 1];
      for (i64 row = job.shard_bounds[(size_t)job.shard_index]; row < window_end; row += ios) {
        job.task_starts.push_back(row);
        groups_of_task.push_back(-1);
      }
    }
    const i64 n_tasks = (i64)job.task_starts.size();
    job.task_starts.push_back(window_end);
    job.sink_is_frame.clear();
    for (size_t k = 0; k < graph.ops.size(); ++k)
      if (graph.ops[k].kind == OpKind::Sink) {
        job.outputs[(i32)k].resize((size_t)n_tasks);
        const OpInput& in = graph.ops[k].inputs.at(0);
        job.sink_is_frame[(i32)k] = graph.column_type_of(in.op_index, in.column) == proto::Video;
      }
    for (i64 t = 0; t < n_tasks; ++t) {
      i64 end = job.task_starts[(size_t)t + 1];
      if (groups_of_task[(size_t)t] >= 0) end = std::min(end, job.slices.out_base[(size_t)groups_of_task[(size_t)t] + 1]);
      end = std::min(end, job.task_starts[(size_t)t] + ios);
      rs.tasks.push_back({(i32)j, (i32)t, job.task_starts[(size_t)t], end, groups_of_task[(size_t)t]});
    }
  }

  // pipeline instances (reference worker.cpp:1297-1337)
  std::vector<std::unique_ptr<Instance>> instances;
  i32 node = 0;
  if (!gpu_ids_.empty()) {
    for (i32 g : gpu_ids_) {
      // default: one pipeline instance (= one decode session) per NVDEC engine of the GPU -- more
      // sessions than engines share an engine and the slowest pair sets the wall time
      i32 per = instances_per_gpu_;
      if (per <= 0) {
        const NvdecCaps& caps = nvdec_caps(g);
        per = caps.available && caps.num_engines > 0 ? caps.num_engines : 4;
      }
      for (i32 i = 0; i < per; ++i) instances.emplace_back(new Instance{this, g, node++, {}});
    }
  } else {
    const i32 n = cpu_instances_ > 0 ? cpu_instances_ : 1;
    for (i32 i = 0; i < n; ++i) instances.emplace_back(new Instance{this, -1, node++, {}});
  }
  while (slots_.size() < instances.size()) slots_.emplace_back(new Slot());
  // never more instances than tasks
  while (instances.size() > std::max<size_t>(1, rs.tasks.size())) instances.pop_back();

  rs.profiler.keep_records(trace_);
  for (size_t i = 0; i < instances.size(); ++i) instances[i]->index = (i32)i;

  // Decode sessions that do not exist yet are created here, one after the other and before any
  // instance decodes, by pushing the first IDR of the job's first video through them: the driver
  // places a session on an NVDEC engine when its decoder is created, and sessions created by the
  // instance threads while others already decode sometimes end up two to an engine (one engine
  // idle, end-to-end 6.7 K instead of 8.6 K frames/s).  SCN_NVDEC_PRIME=0 disables it.
  {
    const char* pe = getenv("SCN_NVDEC_PRIME");
    const bool prime = !(pe && pe[0] == '0');
    for (size_t i = 0; prime && i < instances.size() && !jobs.empty(); ++i) {
      Instance& in = *instances[i];
      if (in.gpu_id < 0 || !cuda_available()) continue;
      Slot& slot = *slots_[(size_t)in.node_id];
      ScopedDevice sd(in.gpu_id);
      if (slot.gpu_id != in.gpu_id || !slot.stream) {
        slot.sessions.clear();
        if (slot.stream) cudaStreamDestroy(slot.stream);
        slot.stream = nullptr;
        if (cudaStreamCreateWithFlags(&slot.stream, cudaStreamNonBlocking) != cudaSuccess) break;
        slot.gpu_id = in.gpu_id;
      }
      for (auto& kv : jobs[0]->source_streams) {
        InputStream* st = stream(kv.second);
        if (!st || st->kind != InputStream::H264 || st->index.frames() == 0 || slot.sessions.count(kv.first)) continue;
        std::unique_ptr<NvdecSession> sess(new NvdecSession(in.gpu_id, slot.stream));
        if (!sess->init().success()) continue;
        const std::vector<u64> offs(st->index.sample_offsets.begin(), st->index.sample_offsets.begin() + 1);
        const std::vector<u64> szs(st->index.sample_sizes.begin(), st->index.sample_sizes.begin() + 1);
        Result pr = sess->begin_interval(st->encoded.data(), offs, szs, st->index.metadata_packets, false, {0}, 0,
                                         st->index.width, st->index.height, [](i64, const Nv12Surface&) {});
        if (pr.success()) pr = sess->advance(1);
        if (pr.success()) pr = sess->end_interval();
        sess->drain();
        if (pr.success()) slot.sessions[kv.first] = std::move(sess);
      }
    }
  }
  if (rs.db) {
    const char* sw = getenv("SCN_SAVE_WORKERS");
    const int n = sw ? atoi(sw) : 4;  // reference default save_workers_per_node (scanner/api/database.cpp:68-84)
    if (n > 0) rs.savers.reset(new SavePool(n));
  }
  const auto t0 = std::chrono::steady_clock::now();
  {
    Result hr = exchange_halos(graph, jobs);
    if (!hr.success()) rs.fail(hr.msg());
  }
  if (!rs.failed.load()) {
    for (auto& inst : instances) inst->th = std::thread([this, p = inst.get()] { instance_main(p); });
    for (auto& inst : instances) inst->th.join();
  }
  if (rs.savers) {
    rs.savers->wait_idle();  // every item is on disk before the run returns (the caller commits the tables next)
    rs.savers.reset();
  }
  for (auto& kv : rs.halo_rows) delete_buffer(rs.halo_dev, kv.second);
  rs.halo_rows.clear();
  stats_ = RunStats();
  stats_.wall_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  stats_.counters = rs.profiler.counters();
  stats_.counters["frames_decoded"] = rs.frames_decoded.load();
  stats_.counters["frames_delivered_nv12"] = rs.frames_native.load();
  stats_.counters["frames_used"] = rs.frames_used.load();
  {
    long long ns[6];
    nvdec_host_ns(ns);
    static const char* names[6] = {"nvdec_parse_us", "nvdec_decode_call_us", "nvdec_map_us", "nvdec_consume_us",
                                   "nvdec_release_wait_us", "nvdec_create_us"};
    for (int i = 0; i < 6; ++i) stats_.counters[names[i]] = ns[i] / 1000;
  }
  // live allocator bytes after the run: everything a run allocates is released when it ends
  // (input streams are adopted, not allocated), so anything left here is a leak
  stats_.counters["cpu_bytes_live"] = (i64)current_memory_allocated(CPU_DEVICE);
  stats_.counters["cpu_bytes_peak"] = (i64)max_memory_allocated(CPU_DEVICE);
  for (i32 g : gpu_ids_) {
    stats_.counters["gpu" + std::to_string(g) + "_bytes_live"] = (i64)current_memory_allocated(DeviceHandle(DeviceType::GPU, g));
    stats_.counters["gpu" + std::to_string(g) + "_bytes_peak"] = (i64)max_memory_allocated(DeviceHandle(DeviceType::GPU, g));
  }
  stats_.counters["tasks"] = (i64)rs.tasks.size();
  stats_.counters["instances"] = (i64)instances.size();
  stats_.counters["halo_bytes_sent"] = rs.halo_bytes_sent;
  stats_.counters["halo_bytes_received"] = rs.halo_bytes_received;
  stats_.counters["halo_exchange_us"] = rs.halo_ns / 1000;
  // per pipeline instance (= per decode session): what it decoded and how long it waited on its NVDEC
  // engine -- frames / busy is the session's picture rate, the evidence for where an end-to-end
  // number below the expected one went
  for (size_t i = 0; i < instances.size(); ++i) {
    const Instance& in = *instances[i];
    const std::string k = "inst" + std::to_string(i) + "_";
    stats_.counters[k + "gpu"] = in.gpu_id;
    stats_.counters[k + "tasks"] = in.tasks_done;
    stats_.counters[k + "frames_decoded"] = in.frames_decoded;
    stats_.counters[k + "decode_busy_us"] = in.decode_busy_ns / 1000;
    stats_.counters[k + "wall_us"] = in.wall_ns / 1000;
  }
  // GPU decode sessions that run FFmpeg on the host because the GPU exposes no NVDEC engine (nvdec.h)
  i64 software_sessions = 0;
  for (const auto& sl : slots_)
    for (const auto& kv : sl->sessions) software_sessions += kv.second->software() ? 1 : 0;
  stats_.counters["gpu_software_decode_sessions"] = software_sessions;
  stats_.interval_ns = rs.profiler.interval_totals_ns();
  stats_.interval_counts = rs.profiler.interval_counts();
  for (const Profiler::TaskRecord& rec : rs.profiler.records()) {
    const i32 w = rec.worker;
    // trace "process" = the device the instance drives (-1: CPU instance)
    const i32 node = (w >= 0 && (size_t)w < instances.size()) ? instances[(size_t)w]->gpu_id : -1;
    stats_.trace.push_back({rec.key, rec.start_ns, rec.end_ns, w, node});
  }
  if (rs.failed.load()) {
    RESULT_ERROR(&r, "%s", rs.error.c_str());
    return r;
  }
  return ok();
}

}  // namespace internal
}  // namespace scanner
