// swdec.cpp -- see swdec.h.  FFmpeg's public ABI as used here (stable over libavcodec 58..62 = FFmpeg 4.x..8.x):
//   AVPacket  begins { AVBufferRef* buf; int64_t pts, dts; uint8_t* data; int size; ... }
//   AVFrame   begins { uint8_t* data[8]; int linesize[8]; uint8_t** extended_data; int width, height;
//                      int nb_samples; int format; ... }
//   AV_CODEC_ID_H264 = 27, AV_PIX_FMT_RGB24 = 2, SWS_BICUBIC = 4, AVERROR(EAGAIN) = -11, AVERROR_EOF = -'EOF '
// Nothing else of any FFmpeg struct is touched: options go through av_opt_set_int by name.
#include "swdec.h"

#include <dirent.h>
#include <dlfcn.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

namespace scanner {
namespace internal {
namespace {

struct AvPacketHead {
  void* buf;
  int64_t pts, dts;
  uint8_t* data;
  int size;
};
struct AvFrameHead {
  uint8_t* data[8];
  int linesize[8];
  uint8_t** extended_data;
  int width, height;
  int nb_samples;
  int format;
};
constexpr int kCodecH264 = 27, kPixRgb24 = 2, kSwsBicubic = 4, kLogPanic = 0;
constexpr int kPixYuv420p = 0, kPixYuvj420p = 12;  // AV_PIX_FMT_YUV420P, AV_PIX_FMT_YUVJ420P
constexpr int kErrAgain = -11;
constexpr int kErrEof = -(int)((unsigned)'E' | ((unsigned)'O' << 8) | ((unsigned)'F' << 16) | ((unsigned)' ' << 24));

struct Ffmpeg {
  SwdecCaps caps;
  const void* (*find_decoder)(int) = nullptr;
  void* (*alloc_context3)(const void*) = nullptr;
  int (*open2)(void*, const void*, void**) = nullptr;
  void (*free_context)(void**) = nullptr;
  int (*send_packet)(void*, const void*) = nullptr;
  int (*receive_frame)(void*, void*) = nullptr;
  void (*flush_buffers)(void*) = nullptr;
  void* (*packet_alloc)() = nullptr;
  void (*packet_free)(void**) = nullptr;
  int (*new_packet)(void*, int) = nullptr;
  void (*packet_unref)(void*) = nullptr;
  unsigned (*avcodec_version)() = nullptr;
  void* (*frame_alloc)() = nullptr;
  void (*frame_free)(void**) = nullptr;
  void (*frame_unref)(void*) = nullptr;
  int (*opt_set_int)(void*, const char*, int64_t, int) = nullptr;
  void (*log_set_level)(int) = nullptr;
  unsigned (*avutil_version)() = nullptr;
  int (*strerror)(int, char*, size_t) = nullptr;
  void* (*sws_get_context)(int, int, int, int, int, int, int, void*, void*, const double*) = nullptr;
  int (*sws_scale)(void*, const uint8_t* const*, const int*, int, int, uint8_t* const*, const int*) = nullptr;
  void (*sws_free_context)(void*) = nullptr;
  unsigned (*swscale_version)() = nullptr;
};

// dlopen `path`; a dependency the loader cannot find ("libX.so.N: cannot open shared object file") is looked up in
// the same directory and opened first (wheels bundle their libraries side by side without a RUNPATH)
void* open_with_deps(const std::string& dir, const std::string& path, std::string& err, int depth = 0) {
  for (int attempt = 0; attempt < 24; ++attempt) {
    void* h = dlopen(path.c_str(), RTLD_NOW | RTLD_GLOBAL);
    if (h) return h;
    const char* e = dlerror();
    err = e ? e : "dlopen failed";
    const size_t colon = err.find(": cannot open shared object file");
    if (dir.empty() || colon == std::string::npos || depth > 6) return nullptr;
    const std::string missing = err.substr(0, colon);
    if (missing.find('/') != std::string::npos || missing == path) return nullptr;
    std::string sub;
    if (!open_with_deps(dir, dir + "/" + missing, sub, depth + 1)) return nullptr;
  }
  return nullptr;
}

std::string find_in_dir(const std::string& dir, const char* stem) {
  std::string best;
  if (DIR* d = opendir(dir.c_str())) {
    while (dirent* e = readdir(d)) {
      const std::string n = e->d_name;
      if (n.compare(0, strlen(stem), stem) == 0 && n.find(".so") != std::string::npos && n > best) best = n;
    }
    closedir(d);
  }
  return best.empty() ? best : dir + "/" + best;
}

Ffmpeg* load_ffmpeg() {
  Ffmpeg* f = new Ffmpeg();
  std::string err;
  void *hu = nullptr, *hc = nullptr, *hs = nullptr;
  const char* env = getenv("SCN_FFMPEG_DIR");
  if (env && env[0]) {
    const std::string dir = env;
    const std::string pu = find_in_dir(dir, "libavutil"), pc = find_in_dir(dir, "libavcodec"),
                      ps = find_in_dir(dir, "libswscale");
    if (pu.empty() || pc.empty() || ps.empty()) {
      f->caps.error = "SCN_FFMPEG_DIR=" + dir + " does not hold libavutil, libavcodec and libswscale";
      return f;
    }
    hu = open_with_deps(dir, pu, err);
    if (hu) hc = open_with_deps(dir, pc, err);
    if (hc) hs = open_with_deps(dir, ps, err);
    f->caps.where = pc;
  } else {
    // the system's FFmpeg: matching majors of one release line are tried together
    static const int sets[][3] = {{62, 60, 9}, {61, 59, 8}, {60, 58, 7}, {59, 57, 6}, {58, 56, 5}};
    for (const auto& s : sets) {
      const std::string pu = "libavutil.so." + std::to_string(s[1]), pc = "libavcodec.so." + std::to_string(s[0]),
                        ps = "libswscale.so." + std::to_string(s[2]);
      hu = dlopen(pu.c_str(), RTLD_NOW | RTLD_GLOBAL);
      if (!hu) continue;
      hc = dlopen(pc.c_str(), RTLD_NOW | RTLD_GLOBAL);
      hs = hc ? dlopen(ps.c_str(), RTLD_NOW | RTLD_GLOBAL) : nullptr;
      if (hc && hs) {
        f->caps.where = pc;
        break;
      }
      const char* e = dlerror();
      err = e ? e : "";
      hu = hc = hs = nullptr;
    }
    if (!hu && err.empty()) err = "no libavcodec.so.{58..62} on the library path and SCN_FFMPEG_DIR is not set";
  }
  if (!hu || !hc || !hs) {
    f->caps.error = "FFmpeg libraries not loadable: " + err;
    return f;
  }
  bool ok = true;
  auto sym = [&](void* h, const char* name, auto& fn) {
    fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
    if (!fn) {
      ok = false;
      f->caps.error = std::string("FFmpeg symbol missing: ") + name;
    }
  };
  sym(hc, "avcodec_find_decoder", f->find_decoder);
  sym(hc, "avcodec_alloc_context3", f->alloc_context3);
  sym(hc, "avcodec_open2", f->open2);
  sym(hc, "avcodec_free_context", f->free_context);
  sym(hc, "avcodec_send_packet", f->send_packet);
  sym(hc, "avcodec_receive_frame", f->receive_frame);
  sym(hc, "avcodec_flush_buffers", f->flush_buffers);
  sym(hc, "av_packet_alloc", f->packet_alloc);
  sym(hc, "av_packet_free", f->packet_free);
  sym(hc, "av_new_packet", f->new_packet);
  sym(hc, "av_packet_unref", f->packet_unref);
  sym(hc, "avcodec_version", f->avcodec_version);
  sym(hu, "av_frame_alloc", f->frame_alloc);
  sym(hu, "av_frame_free", f->frame_free);
  sym(hu, "av_frame_unref", f->frame_unref);
  sym(hu, "av_opt_set_int", f->opt_set_int);
  sym(hu, "av_log_set_level", f->log_set_level);
  sym(hu, "avutil_version", f->avutil_version);
  sym(hu, "av_strerror", f->strerror);
  sym(hs, "sws_getContext", f->sws_get_context);
  sym(hs, "sws_scale", f->sws_scale);
  sym(hs, "sws_freeContext", f->sws_free_context);
  sym(hs, "swscale_version", f->swscale_version);
  if (!ok) return f;
  f->caps.avcodec_major = (int)(f->avcodec_version() >> 16);
  f->caps.avutil_major = (int)(f->avutil_version() >> 16);
  f->caps.swscale_major = (int)(f->swscale_version() >> 16);
  if (f->caps.avcodec_major < 58 || f->caps.avcodec_major > 62) {
    f->caps.error = "libavcodec major " + std::to_string(f->caps.avcodec_major) +
                    " is outside 58..62, the range whose AVPacket / AVFrame layout this file declares";
    return f;
  }
  f->log_set_level(kLogPanic);  // reference software_video_decoder.cpp:47
  f->caps.available = true;
  return f;
}

Ffmpeg& ffmpeg() {
  static Ffmpeg* f = load_ffmpeg();
  return *f;
}

std::string av_error(int rc) {
  char buf[160] = {0};
  if (ffmpeg().strerror && ffmpeg().strerror(rc, buf, sizeof(buf)) == 0) return std::string(buf) + " (" + std::to_string(rc) + ")";
  return std::to_string(rc);
}

}  // namespace

const SwdecCaps& swdec_caps() { return ffmpeg().caps; }

struct SwdecSession::Impl {
  int threads = 1;
  bool nv12 = false;       // deliver the decoded 4:2:0 planes as NV12 instead of RGB24
  void* ctx = nullptr;     // AVCodecContext
  void* packet = nullptr;  // AVPacket
  void* frame = nullptr;   // AVFrame
  void* sws = nullptr;
  int sws_w = 0, sws_h = 0, sws_fmt = -1;
  bool used = false;       // the codec has seen data since the last flush
  // the open interval
  bool active = false, flushed = false, first = true;
  const u8* data = nullptr;
  std::vector<u64> offsets, sizes;
  std::vector<u8> prefix;
  std::vector<i64> wanted;
  size_t next_sample = 0, wanted_pos = 0;
  i64 display_pos = 0, out_base = 0;
  bool may_reorder = false;
  int width = 0, height = 0;
  Dest dest;
  std::string error;

  ~Impl() {
    Ffmpeg& f = ffmpeg();
    if (sws) f.sws_free_context(sws);
    if (frame) f.frame_free(&frame);
    if (packet) f.packet_free(&packet);
    if (ctx) f.free_context(&ctx);
  }

  // every picture the decoder has ready: count it, convert the wanted ones
  int receive_all(i64& decoded, i64& used_count) {
    Ffmpeg& f = ffmpeg();
    for (;;) {
      const int rc = f.receive_frame(ctx, frame);
      if (rc == kErrAgain || rc == kErrEof) return rc;
      if (rc < 0) {
        error = "avcodec_receive_frame: " + av_error(rc);
        return rc;
      }
      const AvFrameHead* fh = static_cast<const AvFrameHead*>(frame);
      ++decoded;
      const i64 pos = display_pos++;
      if (wanted_pos < wanted.size() && wanted[wanted_pos] == pos) {
        if (fh->width != width || fh->height != height) {
          error = "decoded picture is " + std::to_string(fh->width) + "x" + std::to_string(fh->height) +
                  " but the stream index says " + std::to_string(width) + "x" + std::to_string(height);
          f.frame_unref(frame);
          return -1;
        }
        if (nv12) {
          // 8-bit 4:2:0 planes as decoded: luma rows, then Cb / Cr interleaved (what an NVDEC surface holds)
          u8* dst = dest(out_base + (i64)wanted_pos);
          if (!dst || (fh->format != kPixYuv420p && fh->format != kPixYuvj420p)) {
            error = "software decode to NV12: unsupported pixel format " + std::to_string(fh->format);
            f.frame_unref(frame);
            return -1;
          }
          for (int y = 0; y < height; ++y) memcpy(dst + (size_t)y * width, fh->data[0] + (size_t)y * fh->linesize[0], width);
          u8* c = dst + (size_t)width * height;
          for (int y = 0; y < height / 2; ++y) {
            const u8* cb = fh->data[1] + (size_t)y * fh->linesize[1];
            const u8* cr = fh->data[2] + (size_t)y * fh->linesize[2];
            u8* row = c + (size_t)y * width;
            for (int x = 0; x < width / 2; ++x) {
              row[2 * x] = cb[x];
              row[2 * x + 1] = cr[x];
            }
          }
          ++wanted_pos;
          ++used_count;
          f.frame_unref(frame);
          continue;
        }
        if (!sws || sws_w != width || sws_h != height || sws_fmt != fh->format) {
          if (sws) f.sws_free_context(sws);
          // reference software_video_decoder.cpp:188-192: same size, -> RGB24, SWS_BICUBIC
          sws = f.sws_get_context(width, height, fh->format, width, height, kPixRgb24, kSwsBicubic, nullptr, nullptr,
                                  nullptr);
          sws_w = width;
          sws_h = height;
          sws_fmt = fh->format;
          if (!sws) {
            error = "sws_getContext failed for pixel format " + std::to_string(fh->format);
            f.frame_unref(frame);
            return -1;
          }
        }
        uint8_t* dst[4] = {dest(out_base + (i64)wanted_pos), nullptr, nullptr, nullptr};
        const int dst_stride[4] = {width * 3, 0, 0, 0};
        if (!dst[0] || f.sws_scale(sws, fh->data, fh->linesize, 0, fh->height, dst, dst_stride) < 0) {
          error = "sws_scale failed";
          f.frame_unref(frame);
          return -1;
        }
        ++wanted_pos;
        ++used_count;
      }
      f.frame_unref(frame);
    }
  }
};

SwdecSession::SwdecSession(int threads, bool nv12) : impl_(new Impl()) {
  impl_->threads = threads < 1 ? 1 : threads;
  impl_->nv12 = nv12;
}
SwdecSession::~SwdecSession() {}

Result SwdecSession::init() {
  Result r;
  Ffmpeg& f = ffmpeg();
  if (!f.caps.available) {
    RESULT_ERROR(&r, "software H.264 decoder unavailable: %s", f.caps.error.c_str());
    return r;
  }
  Impl& s = *impl_;
  const void* codec = f.find_decoder(kCodecH264);
  if (!codec) {
    RESULT_ERROR(&r, "this libavcodec has no H.264 decoder");
    return r;
  }
  s.ctx = f.alloc_context3(codec);
  if (!s.ctx) {
    RESULT_ERROR(&r, "avcodec_alloc_context3 failed");
    return r;
  }
  f.opt_set_int(s.ctx, "threads", s.threads, 0);  // reference :57 cc_->thread_count
  const int rc = f.open2(s.ctx, codec, nullptr);
  if (rc < 0) {
    RESULT_ERROR(&r, "avcodec_open2 failed: %s", av_error(rc).c_str());
    return r;
  }
  s.packet = f.packet_alloc();
  s.frame = f.frame_alloc();
  if (!s.packet || !s.frame) {
    RESULT_ERROR(&r, "cannot allocate an AVPacket / AVFrame");
    return r;
  }
  r.set_success(true);
  return r;
}

Result SwdecSession::begin_interval(const u8* data, const std::vector<u64>& offsets, const std::vector<u64>& sizes,
                                    const std::vector<u8>& prefix, bool may_reorder, const std::vector<i64>& wanted,
                                    i64 out_base, int width, int height, Dest dest) {
  Result r;
  Impl& s = *impl_;
  if (!s.ctx) {
    RESULT_ERROR(&r, "SwdecSession used before init()");
    return r;
  }
  if (s.active) {
    Result e = end_interval();
    if (!e.success()) return e;
  }
  if (s.used) {  // discontinuity (reference feed(..., discontinuity = true), :124-141)
    ffmpeg().flush_buffers(s.ctx);
    s.used = false;
  }
  s.data = data;
  s.offsets = offsets;
  s.sizes = sizes;
  s.prefix = prefix;
  s.wanted = wanted;
  s.next_sample = 0;
  s.wanted_pos = 0;
  s.display_pos = 0;
  s.out_base = out_base;
  s.may_reorder = may_reorder;
  s.width = width;
  s.height = height;
  s.dest = std::move(dest);
  s.flushed = false;
  s.first = true;
  s.active = true;
  s.error.clear();
  r.set_success(true);
  return r;
}

size_t SwdecSession::delivered() const { return impl_->wanted_pos; }

Result SwdecSession::advance(size_t count) {
  Result r;
  Impl& s = *impl_;
  Ffmpeg& f = ffmpeg();
  if (!s.active) {
    RESULT_ERROR(&r, "advance() without an open interval");
    return r;
  }
  if (count > s.wanted.size()) count = s.wanted.size();
  // libavcodec may hold pictures back (reordering, frame threads); samples after the last wanted picture are only
  // fed when the stream can reorder, then the decoder is drained
  const size_t last_needed = s.wanted.empty() ? 0 : s.may_reorder ? s.offsets.size() : (size_t)s.wanted.back() + 1;
  while (s.wanted_pos < count) {
    int rc = 0;
    if (s.next_sample < s.offsets.size() && s.next_sample < last_needed) {
      const size_t i = s.next_sample++;
      const size_t pre = s.first ? s.prefix.size() : 0;
      if (f.new_packet(s.packet, (int)(pre + s.sizes[i])) < 0) {
        RESULT_ERROR(&r, "av_new_packet(%zu) failed", pre + (size_t)s.sizes[i]);
        return r;
      }
      AvPacketHead* ph = static_cast<AvPacketHead*>(s.packet);
      if (pre) memcpy(ph->data, s.prefix.data(), pre);
      memcpy(ph->data + pre, s.data + s.offsets[i], s.sizes[i]);
      s.first = false;
      s.used = true;
      rc = f.send_packet(s.ctx, s.packet);
      f.packet_unref(s.packet);
      if (rc < 0 && rc != kErrEof) {
        RESULT_ERROR(&r, "avcodec_send_packet failed on sample %zu: %s", i, av_error(rc).c_str());
        return r;
      }
      rc = s.receive_all(frames_decoded_, frames_used_);
    } else if (!s.flushed) {
      s.flushed = true;
      s.used = true;
      f.send_packet(s.ctx, nullptr);  // drain
      rc = s.receive_all(frames_decoded_, frames_used_);
    } else {
      RESULT_ERROR(&r, "the software decoder delivered %zu of %zu wanted pictures (%ld displayed)", s.wanted_pos,
                   s.wanted.size(), (long)s.display_pos);
      return r;
    }
    if (rc != kErrAgain && rc != kErrEof) {
      RESULT_ERROR(&r, "software decode failed: %s", s.error.c_str());
      return r;
    }
  }
  r.set_success(true);
  return r;
}

Result SwdecSession::end_interval() {
  Result r;
  Impl& s = *impl_;
  if (!s.active) {
    r.set_success(true);
    return r;
  }
  Result a = advance(s.wanted.size());
  s.active = false;
  s.dest = nullptr;
  if (!a.success()) return a;
  r.set_success(true);
  return r;
}

}  // namespace internal
}  // namespace scanner
