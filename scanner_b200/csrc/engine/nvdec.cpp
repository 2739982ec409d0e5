// nvdec.cpp -- see nvdec.h.  The NVCUVID structs below are minimal re-declarations of the public
// driver ABI (Video Codec SDK nvcuvid.h / cuviddec.h: field order and sizes, reserved tails kept
// as opaque padding); only the fields this file touches are named.
#include "nvdec.h"
#include "swdec.h"

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <atomic>
#include <chrono>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>

#include "engine_internal.h"
#include "scanner/util/memory.h"

namespace scanner {
namespace internal {

namespace {

// ---- driver ABI -----------------------------------------------------------------------------
constexpr int kCodecH264 = 4;        // cudaVideoCodec_H264
constexpr int kChroma420 = 1;        // cudaVideoChromaFormat_420
constexpr int kSurfaceNV12 = 0;      // cudaVideoSurfaceFormat_NV12
constexpr int kDeinterlaceWeave = 0;
constexpr unsigned long kCreatePreferCUVID = 0x04;
constexpr unsigned long kPktEndOfStream = 0x01, kPktDiscontinuity = 0x04, kPktEndOfPicture = 0x08;

struct CuvidDecodeCaps {  // CUVIDDECODECAPS
  int codec, chroma;
  unsigned bit_depth_minus8, reserved1[3];
  unsigned char supported, num_nvdecs;
  unsigned short output_format_mask;
  unsigned max_width, max_height, max_mb_count;
  unsigned short min_width, min_height;
  unsigned char hist_supported, counter_bit_depth;
  unsigned short max_hist_bins;
  unsigned reserved3[10];
};
struct CuvidVideoFormat {  // CUVIDEOFORMAT (64 bytes)
  int codec;
  unsigned fr_num, fr_den;
  unsigned char progressive, bit_depth_luma_minus8, bit_depth_chroma_minus8, min_num_decode_surfaces;
  unsigned coded_width, coded_height;
  int left, top, right, bottom;
  int chroma_format;
  unsigned bitrate;
  int dar_x, dar_y;
  unsigned char vsd[4];
  unsigned seqhdr_data_length;
};
struct CuvidParserParams {  // CUVIDPARSERPARAMS (136 bytes)
  int codec;
  unsigned max_num_decode_surfaces, clock_rate, error_threshold, max_display_delay;
  unsigned reserved1[5];
  void* user;
  int (*on_sequence)(void*, CuvidVideoFormat*);
  int (*on_decode)(void*, void*);
  int (*on_display)(void*, void*);
  void* reserved2[7];
  void* ext_video_info;
};
struct CuvidPacket {  // CUVIDSOURCEDATAPACKET
  unsigned long flags, payload_size;
  const unsigned char* payload;
  long long timestamp;
};
struct CuvidCreateInfo {  // CUVIDDECODECREATEINFO (176 bytes)
  unsigned long width, height, num_decode_surfaces;
  int codec, chroma;
  unsigned long creation_flags, bit_depth_minus8, intra_decode_only, max_width, max_height, reserved1;
  short da_left, da_top, da_right, da_bottom;
  int output_format, deinterlace;
  unsigned long target_width, target_height, num_output_surfaces;
  void* vid_lock;
  short tr_left, tr_top, tr_right, tr_bottom;
  unsigned long reserved2[5];
};
struct CuvidDispInfo {  // CUVIDPARSERDISPINFO
  int picture_index, progressive_frame, top_field_first, repeat_first_field;
  long long timestamp;
};
struct CuvidProcParams {  // CUVIDPROCPARAMS (264 bytes)
  int progressive_frame, second_field, top_field_first, unpaired_field;
  unsigned reserved_flags, reserved_zero;
  unsigned long long raw_input_dptr;
  unsigned raw_input_pitch, raw_input_format;
  unsigned long long raw_output_dptr;
  unsigned raw_output_pitch, reserved1;
  void* output_stream;
  unsigned reserved[46];
  void* reserved2[2];
};
static_assert(sizeof(CuvidVideoFormat) == 64, "CUVIDEOFORMAT layout");
static_assert(sizeof(CuvidParserParams) == 136, "CUVIDPARSERPARAMS layout");
static_assert(sizeof(CuvidPacket) == 32, "CUVIDSOURCEDATAPACKET layout");
static_assert(sizeof(CuvidCreateInfo) == 176, "CUVIDDECODECREATEINFO layout");
static_assert(sizeof(CuvidProcParams) == 264, "CUVIDPROCPARAMS layout");

struct Driver {
  void* lib = nullptr;
  int (*GetDecoderCaps)(CuvidDecodeCaps*) = nullptr;
  int (*CreateVideoParser)(void**, CuvidParserParams*) = nullptr;
  int (*ParseVideoData)(void*, CuvidPacket*) = nullptr;
  int (*DestroyVideoParser)(void*) = nullptr;
  int (*CreateDecoder)(void**, CuvidCreateInfo*) = nullptr;
  int (*DestroyDecoder)(void*) = nullptr;
  int (*DecodePicture)(void*, void*) = nullptr;
  int (*MapVideoFrame64)(void*, int, unsigned long long*, unsigned*, CuvidProcParams*) = nullptr;
  int (*UnmapVideoFrame64)(void*, unsigned long long) = nullptr;
  std::string error;
};

Driver& driver() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnvcuvid.so.1", "libnvcuvid.so", "/usr/local/nvidia/lib64/libnvcuvid.so.1",
                           "/usr/lib/x86_64-linux-gnu/libnvcuvid.so.1", "/usr/lib64/libnvcuvid.so.1"};
    for (const char* n : names) {
      d.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (d.lib) break;
    }
    if (!d.lib) {
      const char* msg = dlerror();
      d.error = std::string("libnvcuvid not found: ") + (msg ? msg : "");
      return;
    }
    auto sym = [&](const char* name, auto& fn) {
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(d.lib, name));
      if (!fn && d.error.empty()) d.error = std::string("libnvcuvid lacks ") + name;
    };
    sym("cuvidGetDecoderCaps", d.GetDecoderCaps);
    sym("cuvidCreateVideoParser", d.CreateVideoParser);
    sym("cuvidParseVideoData", d.ParseVideoData);
    sym("cuvidDestroyVideoParser", d.DestroyVideoParser);
    sym("cuvidCreateDecoder", d.CreateDecoder);
    sym("cuvidDestroyDecoder", d.DestroyDecoder);
    sym("cuvidDecodePicture", d.DecodePicture);
    sym("cuvidMapVideoFrame64", d.MapVideoFrame64);
    sym("cuvidUnmapVideoFrame64", d.UnmapVideoFrame64);
  });
  return d;
}

void make_context_current(int gpu) {
  cudaSetDevice(gpu);
  // once per (thread, gpu): force primary-context creation so the driver-API calls inside
  // libnvcuvid find a current context
  thread_local int initialised_mask = 0;
  if (gpu < 31 && !(initialised_mask & (1 << gpu))) {
    cudaFree(nullptr);
    initialised_mask |= 1 << gpu;
  }
}

// cumulative host time inside the driver calls, all sessions (exposed through the run stats)
std::atomic<long long> g_ns[6];  // parse(total), decode_picture, map, consume, release_wait, create
struct ScopedNs {
  int k;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  explicit ScopedNs(int kk) : k(kk) {}
  ~ScopedNs() {
    g_ns[k] += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
  }
};

constexpr int kMaxMapped = 6;
constexpr int kOutputSurfaces = 8;

}  // namespace

const NvdecCaps& nvdec_caps(int gpu_id) {
  static std::mutex mu;
  static std::map<int, NvdecCaps> cache;
  std::lock_guard<std::mutex> g(mu);
  auto it = cache.find(gpu_id);
  if (it != cache.end()) return it->second;
  NvdecCaps c;
  Driver& d = driver();
  if (!d.error.empty() || !d.lib) {
    c.error = d.error.empty() ? "libnvcuvid unavailable" : d.error;
  } else if (!cuda_available()) {
    c.error = "no CUDA device";
  } else {
    ScopedDevice sd(gpu_id);
    make_context_current(gpu_id);
    CuvidDecodeCaps caps;
    memset(&caps, 0, sizeof(caps));
    caps.codec = kCodecH264;
    caps.chroma = kChroma420;
    const int rc = d.GetDecoderCaps(&caps);
    if (rc != 0) {
      c.error = "cuvidGetDecoderCaps failed: " + std::to_string(rc);
    } else {
      c.available = true;
      c.h264_supported = caps.supported != 0;
      c.num_engines = caps.num_nvdecs;
      c.max_width = (int)caps.max_width;
      c.max_height = (int)caps.max_height;
      c.min_width = caps.min_width;
      c.min_height = caps.min_height;
    }
  }
  return cache.emplace(gpu_id, c).first->second;
}

// ---------------------------------------------------------------------------------------------
struct NvdecSession::Impl {
  int gpu;
  cudaStream_t stream;
  void* parser = nullptr;
  void* decoder = nullptr;
  CuvidVideoFormat fmt{};
  bool have_fmt = false;
  std::string error;

  // per-interval state
  std::vector<i64> wanted_store;
  bool may_reorder = false;
  const std::vector<i64>* wanted = nullptr;
  size_t wanted_pos = 0;
  i64 display_pos = 0;
  i64 out_base = 0;
  Consumer consumer_store;
  const Consumer* consumer = nullptr;
  const u8* data = nullptr;
  std::vector<u64> offsets, sizes;
  size_t next_sample = 0;
  bool first_packet = true, flushed = false, active = false;
  i64* decoded_counter = nullptr;
  i64* used_counter = nullptr;

  // software decode (no NVDEC engine on the GPU): pictures decoded by FFmpeg wait in host memory until advance()
  // uploads each into `sw_surface` on the session stream and hands it to the consumer (stream order keeps the next
  // upload behind the consumer's work)
  std::unique_ptr<SwdecSession> sw;
  std::deque<std::pair<i64, std::vector<u8>>> sw_pending;
  u8* sw_surface = nullptr;
  size_t sw_surface_bytes = 0;
  int sw_width = 0, sw_height = 0;

  Result sw_deliver() {
    Result r;
    const size_t bytes = (size_t)sw_width * sw_height * 3 / 2;
    while (!sw_pending.empty()) {
      auto& p = sw_pending.front();
      if (bytes > sw_surface_bytes) {
        if (sw_surface) {
          cudaStreamSynchronize(stream);
          cudaFree(sw_surface);
        }
        sw_surface = nullptr;
        sw_surface_bytes = 0;
        if (cudaMalloc((void**)&sw_surface, bytes) != cudaSuccess) {
          RESULT_ERROR(&r, "software decode: cudaMalloc of %zu bytes failed", bytes);
          return r;
        }
        sw_surface_bytes = bytes;
      }
      // from pageable memory: the call returns once the source has been staged, so the buffer may go
      if (cudaMemcpyAsync(sw_surface, p.second.data(), bytes, cudaMemcpyHostToDevice, stream) != cudaSuccess) {
        RESULT_ERROR(&r, "software decode: upload of a picture failed");
        return r;
      }
      Nv12Surface s;
      s.luma = sw_surface;
      s.chroma = sw_surface + (size_t)sw_width * sw_height;
      s.pitch = (size_t)sw_width;
      s.width = sw_width;
      s.height = sw_height;
      {
        ScopedNs t(3);
        (*consumer)(p.first, s);
      }
      sw_pending.pop_front();
    }
    r.set_success(true);
    return r;
  }

  struct Mapped {
    unsigned long long dptr;
    cudaEvent_t done;
    int pic_index;
  };
  std::deque<Mapped> mapped;
  std::vector<cudaEvent_t> event_pool;

  cudaEvent_t get_event() {
    if (!event_pool.empty()) {
      cudaEvent_t e = event_pool.back();
      event_pool.pop_back();
      return e;
    }
    cudaEvent_t e;
    cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    return e;
  }
  void release_oldest() {
    Mapped m = mapped.front();
    mapped.pop_front();
    ScopedNs t(4);
    cudaEventSynchronize(m.done);
    driver().UnmapVideoFrame64(decoder, m.dptr);
    event_pool.push_back(m.done);
  }
  void release_all() {
    while (!mapped.empty()) release_oldest();
  }

  static int on_sequence(void* user, CuvidVideoFormat* f) { return ((Impl*)user)->sequence(f); }
  static int on_decode(void* user, void* pic) { return ((Impl*)user)->decode(pic); }
  static int on_display(void* user, void* disp) { return ((Impl*)user)->display((CuvidDispInfo*)disp); }

  int sequence(CuvidVideoFormat* f) {
    const int surfaces = std::max<int>(f->min_num_decode_surfaces ? f->min_num_decode_surfaces : 8, 8) + 8;
    if (decoder && have_fmt && f->coded_width == fmt.coded_width && f->coded_height == fmt.coded_height &&
        f->chroma_format == fmt.chroma_format && f->bit_depth_luma_minus8 == fmt.bit_depth_luma_minus8) {
      fmt = *f;
      return surfaces;  // same geometry: keep the decoder (the reference recreates it every time)
    }
    release_all();
    if (decoder) {
      driver().DestroyDecoder(decoder);
      decoder = nullptr;
    }
    if (f->codec != kCodecH264 || f->chroma_format != kChroma420 || f->bit_depth_luma_minus8 != 0) {
      error = "unsupported stream format (need H.264 4:2:0 8-bit)";
      return 0;
    }
    fmt = *f;
    have_fmt = true;
    CuvidCreateInfo ci;
    memset(&ci, 0, sizeof(ci));
    ci.width = f->coded_width;
    ci.height = f->coded_height;
    ci.num_decode_surfaces = (unsigned long)surfaces;
    ci.codec = kCodecH264;
    ci.chroma = kChroma420;
    ci.creation_flags = kCreatePreferCUVID;
    ci.max_width = f->coded_width;
    ci.max_height = f->coded_height;
    ci.da_left = (short)f->left;
    ci.da_top = (short)f->top;
    ci.da_right = (short)f->right;
    ci.da_bottom = (short)f->bottom;
    ci.output_format = kSurfaceNV12;
    ci.deinterlace = kDeinterlaceWeave;
    ci.target_width = (unsigned long)(f->right - f->left);
    ci.target_height = (unsigned long)(f->bottom - f->top);
    ci.num_output_surfaces = kOutputSurfaces;
    ScopedNs t(5);
    const int rc = driver().CreateDecoder(&decoder, &ci);
    if (rc != 0) {
      error = "cuvidCreateDecoder failed: " + std::to_string(rc);
      decoder = nullptr;
      return 0;
    }
    return surfaces;
  }

  int decode(void* pic) {
    if (!decoder) return 0;
    const int cur = ((int*)pic)[2];  // CUVIDPICPARAMS.CurrPicIdx
    // never let the engine overwrite a decode surface a pending map still reads from
    for (size_t i = 0; i < mapped.size(); ++i)
      if (mapped[i].pic_index == cur) {
        while (mapped.size() > 0) {
          const bool hit = mapped.front().pic_index == cur;
          release_oldest();
          if (hit) break;
        }
        break;
      }
    ScopedNs t(1);
    const int rc = driver().DecodePicture(decoder, pic);
    if (rc != 0) {
      error = "cuvidDecodePicture failed: " + std::to_string(rc);
      return 0;
    }
    return 1;
  }

  int display(CuvidDispInfo* d) {
    if (!d) return 1;  // end-of-stream marker
    const i64 pos = display_pos++;
    if (decoded_counter) ++*decoded_counter;
    if (!wanted || wanted_pos >= wanted->size() || (*wanted)[wanted_pos] != pos) return 1;  // skipped, never mapped
    if ((int)mapped.size() >= kMaxMapped) release_oldest();
    CuvidProcParams pp;
    memset(&pp, 0, sizeof(pp));
    pp.progressive_frame = d->progressive_frame;
    pp.top_field_first = d->top_field_first;
    pp.output_stream = stream;
    unsigned long long dptr = 0;
    unsigned pitch = 0;
    int rc;
    {
      ScopedNs t(2);
      rc = driver().MapVideoFrame64(decoder, d->picture_index, &dptr, &pitch, &pp);
    }
    if (rc != 0) {
      error = "cuvidMapVideoFrame failed: " + std::to_string(rc);
      return 0;
    }
    Nv12Surface s;
    s.luma = (const u8*)dptr;
    s.width = fmt.right - fmt.left;
    s.height = fmt.bottom - fmt.top;
    s.pitch = pitch;
    s.chroma = s.luma + (size_t)pitch * (size_t)((s.height + 1) & ~1);
    {
      ScopedNs t(3);
      (*consumer)(out_base + (i64)wanted_pos, s);
    }
    Mapped m{dptr, get_event(), d->picture_index};
    cudaEventRecord(m.done, stream);
    mapped.push_back(m);
    ++wanted_pos;
    if (used_counter) ++*used_counter;
    return 1;
  }
};

NvdecSession::NvdecSession(int gpu_id, void* stream) : impl_(new Impl()) {
  impl_->gpu = gpu_id;
  impl_->stream = (cudaStream_t)stream;
}

NvdecSession::~NvdecSession() {
  if (!impl_) return;
  if (cuda_available()) {
    ScopedDevice sd(impl_->gpu);
    make_context_current(impl_->gpu);
    if (impl_->sw_surface) {
      cudaStreamSynchronize(impl_->stream);
      cudaFree(impl_->sw_surface);
    }
    impl_->release_all();
    if (impl_->decoder) driver().DestroyDecoder(impl_->decoder);
    if (impl_->parser) driver().DestroyVideoParser(impl_->parser);
    for (cudaEvent_t e : impl_->event_pool) cudaEventDestroy(e);
  }
}

bool NvdecSession::software() const { return impl_->sw != nullptr; }

Result NvdecSession::init() {
  Result r;
  const NvdecCaps& caps = nvdec_caps(impl_->gpu);
  if (!caps.available || !caps.h264_supported) {
    impl_->sw.reset(new SwdecSession(1, true));
    Result sr = impl_->sw->init();
    if (!sr.success()) {
      impl_->sw.reset();
      RESULT_ERROR(&r, "NVDEC unavailable on GPU %d (%s) and no software decoder: %s", impl_->gpu,
                   caps.error.empty() ? "H.264 not supported" : caps.error.c_str(), sr.msg().c_str());
      return r;
    }
    r.set_success(true);
    return r;
  }
  ScopedDevice sd(impl_->gpu);
  make_context_current(impl_->gpu);
  CuvidParserParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.codec = kCodecH264;
  pp.max_num_decode_surfaces = 1;  // the sequence callback returns the real count
  // Pictures are displayed `delay` decodes late, so cuvidMapVideoFrame finds its picture already
  // decoded instead of blocking (while holding the driver's per-context lock) until the engine
  // finishes it: with delay 0 a session keeps one picture in flight and N sessions serialise on
  // that lock (measured: 820 fps at 1 session, 780 fps at 8, r01 e2e probe).
  static const int kDelay = [] {
    const char* e = getenv("SCN_NVDEC_DISPLAY_DELAY");
    const int v = e ? atoi(e) : 4;
    return v < 0 ? 0 : (v > 16 ? 16 : v);
  }();
  pp.max_display_delay = (unsigned)kDelay;
  pp.user = impl_.get();
  pp.on_sequence = &Impl::on_sequence;
  pp.on_decode = &Impl::on_decode;
  pp.on_display = &Impl::on_display;
  const int rc = driver().CreateVideoParser(&impl_->parser, &pp);
  if (rc != 0) {
    RESULT_ERROR(&r, "cuvidCreateVideoParser failed: %d", rc);
    return r;
  }
  r.set_success(true);
  return r;
}

namespace {
int send_packet(void* parser, const u8* p, size_t n, unsigned long flags) {
  CuvidPacket pkt;
  memset(&pkt, 0, sizeof(pkt));
  pkt.flags = flags;
  pkt.payload = p;
  pkt.payload_size = n;
  ScopedNs t(0);
  return driver().ParseVideoData(parser, &pkt);
}
}  // namespace

void nvdec_host_ns(long long out[6]) {
  for (int i = 0; i < 6; ++i) out[i] = g_ns[i].load();
}

Result NvdecSession::begin_interval(const u8* data, const std::vector<u64>& offsets,
                                    const std::vector<u64>& sizes, const std::vector<u8>& prefix,
                                    bool may_reorder, const std::vector<i64>& wanted, i64 out_base,
                                    int width, int height, Consumer consumer) {
  Result r;
  Impl& s = *impl_;
  if (s.active) {
    Result e = end_interval();
    if (!e.success()) return e;
  }
  ScopedDevice sd(s.gpu);
  make_context_current(s.gpu);
  if (s.sw) {
    s.wanted_store = wanted;
    s.consumer_store = std::move(consumer);
    s.consumer = &s.consumer_store;
    s.sw_pending.clear();
    s.sw_width = width;
    s.sw_height = height;
    const size_t bytes = (size_t)width * height * 3 / 2;
    Impl* ip = &s;
    r = s.sw->begin_interval(data, offsets, sizes, prefix, may_reorder, wanted, out_base, width, height,
                             [ip, bytes](i64 out_index) {
                               ip->sw_pending.emplace_back(out_index, std::vector<u8>(bytes));
                               return ip->sw_pending.back().second.data();
                             });
    s.active = r.success();
    return r;
  }
  s.wanted_store = wanted;
  s.wanted = &s.wanted_store;
  s.wanted_pos = 0;
  s.display_pos = 0;
  s.out_base = out_base;
  s.consumer_store = std::move(consumer);
  s.consumer = &s.consumer_store;
  s.decoded_counter = &frames_decoded_;
  s.used_counter = &frames_used_;
  s.error.clear();
  s.data = data;
  s.offsets = offsets;
  s.sizes = sizes;
  s.next_sample = 0;
  s.may_reorder = may_reorder;
  s.first_packet = true;
  s.flushed = false;
  s.active = true;
  if (!prefix.empty()) {
    const int rc = send_packet(s.parser, prefix.data(), prefix.size(), kPktDiscontinuity);
    s.first_packet = false;
    if (rc != 0 || !s.error.empty()) {
      RESULT_ERROR(&r, "NVDEC rejected the SPS/PPS prefix (rc %d): %s", rc, s.error.c_str());
      return r;
    }
  }
  r.set_success(true);
  return r;
}

size_t NvdecSession::delivered() const { return impl_->sw ? impl_->sw->delivered() : impl_->wanted_pos; }

Result NvdecSession::advance(size_t count) {
  Result r;
  Impl& s = *impl_;
  if (!s.active) {
    RESULT_ERROR(&r, "advance() without an open interval");
    return r;
  }
  ScopedDevice sd(s.gpu);
  if (count > s.wanted_store.size()) count = s.wanted_store.size();
  // Without reordering, display position k is sample k: samples after the last wanted picture are
  // never fed and the end-of-stream flush below releases whatever the display delay still holds
  // back.  With B pictures a later sample can display earlier, so feeding continues until the
  // wanted pictures have come out or the interval (= up to the next IDR) is exhausted.
  const size_t last_needed = s.wanted_store.empty() ? 0
                             : s.may_reorder        ? s.offsets.size()
                                                    : (size_t)s.wanted_store.back() + 1;
  struct Busy {
    i64& acc;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    ~Busy() { acc += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(); }
  } busy{busy_ns_};
  if (s.sw) {
    r = s.sw->advance(count);
    frames_decoded_ = s.sw->frames_decoded();
    frames_used_ = s.sw->frames_used();
    if (!r.success()) return r;
    return s.sw_deliver();
  }
  while (s.wanted_pos < count) {
    if (s.next_sample < s.offsets.size() && s.next_sample < last_needed) {
      const size_t i = s.next_sample++;
      const int rc = send_packet(s.parser, s.data + s.offsets[i], s.sizes[i],
                                 kPktEndOfPicture | (s.first_packet ? kPktDiscontinuity : 0));
      s.first_packet = false;
      if (rc != 0 || !s.error.empty()) {
        RESULT_ERROR(&r, "NVDEC failed on sample %zu (rc %d): %s", i, rc, s.error.c_str());
        return r;
      }
    } else if (!s.flushed) {
      s.flushed = true;
      const int rc = send_packet(s.parser, nullptr, 0, kPktEndOfStream);
      if (rc != 0 || !s.error.empty()) {
        RESULT_ERROR(&r, "NVDEC end-of-stream flush failed (rc %d): %s", rc, s.error.c_str());
        return r;
      }
    } else {
      RESULT_ERROR(&r, "NVDEC delivered %zu of %zu wanted pictures (%ld displayed)", s.wanted_pos,
                   s.wanted_store.size(), (long)s.display_pos);
      return r;
    }
  }
  r.set_success(true);
  return r;
}

Result NvdecSession::end_interval() {
  Result r;
  Impl& s = *impl_;
  if (!s.active) {
    r.set_success(true);
    return r;
  }
  ScopedDevice sd(s.gpu);
  make_context_current(s.gpu);
  if (s.sw) {
    Result a = s.sw->end_interval();
    frames_decoded_ = s.sw->frames_decoded();
    frames_used_ = s.sw->frames_used();
    if (a.success()) a = s.sw_deliver();
    s.sw_pending.clear();
    s.active = false;
    s.consumer = nullptr;
    return a;
  }
  Result a = advance(s.wanted_store.size());
  // always leave the parser flushed so the next interval starts clean
  if (!s.flushed) {
    s.wanted = nullptr;  // nothing further is wanted: pending pictures are dropped unmapped
    send_packet(s.parser, nullptr, 0, kPktEndOfStream);
    s.flushed = true;
  }
  s.active = false;
  s.wanted = nullptr;
  s.consumer = nullptr;
  if (!a.success()) return a;
  r.set_success(true);
  return r;
}

void NvdecSession::drain() {
  ScopedDevice sd(impl_->gpu);
  make_context_current(impl_->gpu);
  impl_->release_all();
}

}  // namespace internal
}  // namespace scanner
