// image_ops.cpp -- ImageEncoder / ImageDecoder of the stdlib op library (libscn_stdlib.so).
//   ImageEncoder  frame -> PNG bytes.  The reference's in-tree op (scanner/util/image_encoder.cpp:
//                 8-131): CPU kernel, png only, U8/U16 frames with 1-4 channels, output column "img"
//                 of type "Image", ImageEncoderArgs{format}.  The reference compresses with lodepng;
//                 here the stream is written with zlib (deflate) and the standard minimum-sum filter
//                 heuristic -- the file bytes differ, the decoded pixels are identical (lossless).
//                 The GPU kernel of the op also writes JPEG (format "jpg"): scannertools encoded with
//                 cv::imencode, and scn_jpeg_encode_u8 gives cv2.imencode's bytes exactly (HWC u8 frames with
//                 1 or 3 channels, ImageEncoderArgs.quality, 95 when 0; cv2's sampling, optimize and luma /
//                 chroma quality options through scn_jpeg_encode_u8_opts).  "png" on the GPU kernel copies the
//                 frames to the host and writes the same PNG as the CPU kernel.
//   ImageDecoder  PNG bytes -> frame (the op pipelines pair with it: examples/tutorials/
//                 05_sources_sinks.py:41-47; upstream it lives in scannertools and calls
//                 cv::imdecode).  Non-interlaced PNG of colour types 0, 2, 4, 6 with 8 or 16 bits.
//                 The GPU kernel of the op also takes JPEG: decoded by nvJPEG (a CUDA toolkit
//                 library, as SURVEY 8f rank 3 names it) straight into a device frame, RGB order;
//                 PNG elements reaching the GPU kernel are inflated on the host and copied up.
// The CPU kernels are like the reference's: the pipeline moves frame elements between devices.
#include <cuda_runtime.h>
#include <nvjpeg.h>
#include <zlib.h>

#include <cstring>
#include <string>
#include <vector>

#include "scanner/api/kernel.h"
#include "scanner/api/op.h"
#include "scanner/util/memory.h"
#include "scn_kernels.h"
#include "stdlib_args.pb.h"

namespace scanner {
namespace {

void put_be32(std::vector<u8>& o, u32 v) {
  o.push_back((u8)(v >> 24));
  o.push_back((u8)(v >> 16));
  o.push_back((u8)(v >> 8));
  o.push_back((u8)v);
}
u32 get_be32(const u8* p) { return ((u32)p[0] << 24) | ((u32)p[1] << 16) | ((u32)p[2] << 8) | p[3]; }

void put_chunk(std::vector<u8>& o, const char type[4], const u8* data, size_t n) {
  put_be32(o, (u32)n);
  const size_t at = o.size();
  o.insert(o.end(), type, type + 4);
  if (n) o.insert(o.end(), data, data + n);
  put_be32(o, (u32)crc32(0L, o.data() + at, (uInt)(n + 4)));
}

int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

const u8 kPngSig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};

// -> empty string on success
std::string encode_png(const Frame* f, std::vector<u8>& out) {
  const int ch = f->channels();
  static const int color_of[5] = {-1, 0, 4, 2, 6};  // grey, grey+alpha, rgb, rgba
  if (ch < 1 || ch > 4) return "Invalid frame type for ImageEncoder.";
  int depth;
  if ((proto::FrameType)f->type == proto::U8) depth = 8;
  else if ((proto::FrameType)f->type == proto::U16) depth = 16;
  else return "Invalid frame bitdepth for ImageEncoder.";
  const int w = f->width(), h = f->height(), bps = depth / 8, bpp = ch * bps;
  const size_t row = (size_t)w * bpp;
  // scanlines: big-endian samples, one filter byte in front
  std::vector<u8> raw((row + 1) * h), cur(row), prev(row, 0), cand(row);
  for (int y = 0; y < h; ++y) {
    const u8* src = f->data + (size_t)y * row;
    if (bps == 1) {
      memcpy(cur.data(), src, row);
    } else {
      for (size_t i = 0; i < row; i += 2) {
        cur[i] = src[i + 1];
        cur[i + 1] = src[i];
      }
    }
    // minimum sum of absolute differences over the five filters (what libpng / lodepng default to)
    long best = -1;
    u8* dst = raw.data() + (size_t)y * (row + 1);
    for (int t = 0; t < 5; ++t) {
      long sum = 0;
      for (size_t i = 0; i < row; ++i) {
        const int a = i >= (size_t)bpp ? cur[i - bpp] : 0, b = prev[i], c = i >= (size_t)bpp ? prev[i - bpp] : 0;
        int pred = 0;
        switch (t) {
          case 1: pred = a; break;
          case 2: pred = b; break;
          case 3: pred = (a + b) >> 1; break;
          case 4: pred = paeth(a, b, c); break;
        }
        const u8 v = (u8)(cur[i] - pred);
        cand[i] = v;
        sum += v < 128 ? v : 256 - v;
      }
      if (best < 0 || sum < best) {
        best = sum;
        dst[0] = (u8)t;
        memcpy(dst + 1, cand.data(), row);
      }
    }
    prev.swap(cur);
  }
  uLongf zn = compressBound((uLong)raw.size());
  std::vector<u8> z(zn);
  if (compress2(z.data(), &zn, raw.data(), (uLong)raw.size(), 6) != Z_OK)
    return "Failed to encode image to PNG in ImageEncoder.";
  out.clear();
  out.insert(out.end(), kPngSig, kPngSig + 8);
  std::vector<u8> ihdr;
  put_be32(ihdr, (u32)w);
  put_be32(ihdr, (u32)h);
  ihdr.push_back((u8)depth);
  ihdr.push_back((u8)color_of[ch]);
  ihdr.push_back(0);
  ihdr.push_back(0);
  ihdr.push_back(0);
  put_chunk(out, "IHDR", ihdr.data(), ihdr.size());
  put_chunk(out, "IDAT", z.data(), (size_t)zn);
  put_chunk(out, "IEND", nullptr, 0);
  return "";
}

// -> empty string on success; allocates the frame on the CPU
std::string decode_png(const u8* p, size_t n, Frame*& out) {
  if (n < 8 + 25 || memcmp(p, kPngSig, 8) != 0) return "ImageDecoder: not a PNG stream";
  size_t off = 8;
  int w = 0, h = 0, depth = 0, color = -1;
  std::vector<u8> z;
  bool end = false;
  while (!end && off + 12 <= n) {
    const u32 len = get_be32(p + off);
    if (len > n - off - 12) return "ImageDecoder: truncated PNG chunk";
    const u8* type = p + off + 4;
    const u8* data = p + off + 8;
    if (get_be32(data + len) != (u32)crc32(0L, type, (uInt)(len + 4))) return "ImageDecoder: PNG chunk CRC mismatch";
    if (!memcmp(type, "IHDR", 4)) {
      if (len != 13) return "ImageDecoder: bad IHDR";
      w = (int)get_be32(data);
      h = (int)get_be32(data + 4);
      depth = data[8];
      color = data[9];
      if (data[10] != 0 || data[11] != 0) return "ImageDecoder: unknown PNG compression / filter method";
      if (data[12] != 0) return "ImageDecoder: interlaced PNG is not supported";
    } else if (!memcmp(type, "IDAT", 4)) {
      z.insert(z.end(), data, data + len);
    } else if (!memcmp(type, "IEND", 4)) {
      end = true;
    } else if (!(type[0] & 0x20)) {
      return std::string("ImageDecoder: unsupported critical PNG chunk ") + std::string((const char*)type, 4);
    }
    off += (size_t)len + 12;
  }
  if (!end || w <= 0 || h <= 0) return "ImageDecoder: incomplete PNG stream";
  int ch;
  switch (color) {
    case 0: ch = 1; break;
    case 2: ch = 3; break;
    case 4: ch = 2; break;
    case 6: ch = 4; break;
    default: return "ImageDecoder: palette PNG is not supported";
  }
  if (depth != 8 && depth != 16) return "ImageDecoder: PNG bit depth must be 8 or 16";
  const int bps = depth / 8, bpp = ch * bps;
  const size_t row = (size_t)w * bpp;
  std::vector<u8> raw((row + 1) * h);
  uLongf got = (uLongf)raw.size();
  if (uncompress(raw.data(), &got, z.data(), (uLong)z.size()) != Z_OK || got != raw.size())
    return "ImageDecoder: PNG image data does not inflate to the declared size";
  out = new_frame(CPU_DEVICE, FrameInfo(h, w, ch, bps == 1 ? FrameType::U8 : FrameType::U16));
  std::vector<u8> prev(row, 0), cur(row);
  for (int y = 0; y < h; ++y) {
    const u8* line = raw.data() + (size_t)y * (row + 1);
    const int t = line[0];
    if (t > 4) return "ImageDecoder: bad PNG filter type";
    for (size_t i = 0; i < row; ++i) {
      const int a = i >= (size_t)bpp ? cur[i - bpp] : 0, b = prev[i], c = i >= (size_t)bpp ? prev[i - bpp] : 0;
      int pred = 0;
      switch (t) {
        case 1: pred = a; break;
        case 2: pred = b; break;
        case 3: pred = (a + b) >> 1; break;
        case 4: pred = paeth(a, b, c); break;
      }
      cur[i] = (u8)(line[1 + i] + pred);
    }
    u8* dst = out->data + (size_t)y * row;
    if (bps == 1) {
      memcpy(dst, cur.data(), row);
    } else {
      for (size_t i = 0; i < row; i += 2) {
        dst[i] = cur[i + 1];
        dst[i + 1] = cur[i];
      }
    }
    prev.swap(cur);
  }
  return "";
}

// ---------------------------------------------------------------------------------------------
class ImageEncoderKernel : public BatchedKernel {
 public:
  ImageEncoderKernel(const KernelConfig& config) : BatchedKernel(config) {
    ImageEncoderArgs args;
    if (!args.ParseFromArray(config.args.data(), (int)config.args.size())) {
      RESULT_ERROR(&valid_, "Could not parse ImageEncoderArgs");
      return;
    }
    const std::string fmt = args.format().empty() ? "png" : args.format();
    if (!(fmt == "png" || fmt == "PNG")) {
      RESULT_ERROR(&valid_, "Invalid format type specified to ImageEncoder: %s. Valid types are: png.", fmt.c_str());
      return;
    }
    if (!args.sampling().empty() || args.optimize() || args.luma_quality() || args.chroma_quality()) {
      RESULT_ERROR(&valid_, "ImageEncoder sampling, optimize, luma_quality and chroma_quality are JPEG options; "
                   "format is %s",
                   fmt.c_str());
      return;
    }
    valid_.set_success(true);
  }
  void validate(Result* result) override { result->CopyFrom(valid_); }

  void execute(const BatchedElements& in, BatchedElements& out) override {
    for (const Element& e : in[0]) {
      std::vector<u8> png;
      const std::string err = e.is_null() ? std::string("null frame") : encode_png(e.as_const_frame(), png);
      if (!err.empty()) {
        report_kernel_error("ImageEncoder, row " + std::to_string(e.index) + ": " + err);
        out[0].push_back(Element());
        continue;
      }
      u8* buf = new_buffer(CPU_DEVICE, png.size());
      memcpy(buf, png.data(), png.size());
      insert_element(out[0], buf, png.size());
    }
  }

 private:
  Result valid_;
};

REGISTER_OP(ImageEncoder).frame_input("frame").output("img", ColumnType::Bytes, "Image").protobuf_name("ImageEncoderArgs");
REGISTER_KERNEL(ImageEncoder, ImageEncoderKernel).device(DeviceType::CPU).batch(8).num_devices(1);

// ---- GPU kernel: JPEG from sm_90a kernels (scn_jpeg_encode_u8), the encoded bytes delivered on the host -----
class ImageEncoderKernelGPU : public BatchedKernel {
 public:
  ImageEncoderKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {
    ImageEncoderArgs args;
    if (!args.ParseFromArray(config.args.data(), (int)config.args.size())) {
      RESULT_ERROR(&valid_, "Could not parse ImageEncoderArgs");
      return;
    }
    const std::string fmt = args.format().empty() ? "png" : args.format();
    if (fmt == "png" || fmt == "PNG") {
      jpeg_ = false;
    } else if (fmt == "jpg" || fmt == "jpeg" || fmt == "JPEG") {
      jpeg_ = true;
    } else {
      RESULT_ERROR(&valid_, "Invalid format type specified to ImageEncoder: %s. Valid types are: png, jpg.",
                   fmt.c_str());
      return;
    }
    quality_ = args.quality() == 0 ? 95 : args.quality();
    if (quality_ < 1 || quality_ > 100) {
      RESULT_ERROR(&valid_, "ImageEncoder quality %d is outside [1, 100]", quality_);
      return;
    }
    const std::string& sampling = args.sampling();
    const bool options = !sampling.empty() || args.optimize() || args.luma_quality() || args.chroma_quality();
    if (options && !jpeg_) {
      RESULT_ERROR(&valid_, "ImageEncoder sampling, optimize, luma_quality and chroma_quality are JPEG options; "
                   "format is %s",
                   fmt.c_str());
      return;
    }
    if (!sampling.empty()) {
      static const struct { const char* name; int hv; } kModes[] = {
          {"444", SCN_JPEG_444}, {"422", SCN_JPEG_422}, {"420", SCN_JPEG_420}, {"440", SCN_JPEG_440},
          {"411", SCN_JPEG_411}};
      for (const auto& m : kModes)
        if (sampling == m.name) opts_.sampling = m.hv;
      if (!opts_.sampling) {
        RESULT_ERROR(&valid_, "ImageEncoder sampling %s is not one of 444, 422, 420, 440, 411", sampling.c_str());
        return;
      }
    }
    for (int q : {args.luma_quality(), args.chroma_quality()})
      if (q < 0 || q > 100) {
        RESULT_ERROR(&valid_, "ImageEncoder luma / chroma quality %d is outside [1, 100]", q);
        return;
      }
    opts_.luma_quality = args.luma_quality();
    opts_.chroma_quality = args.chroma_quality();
    opts_.optimize = args.optimize() ? 1 : 0;
    valid_.set_success(true);
  }
  void validate(Result* result) override { result->CopyFrom(valid_); }

  void execute(const BatchedElements& in, BatchedElements& out) override {
    const Elements& frames = in[0];
    if (frames.empty()) return;
    if (cudaSetDevice(device_.id) != cudaSuccess) LOG(FATAL) << "ImageEncoder: cannot select GPU " << device_.id;
    if (!jpeg_) {
      for (const Element& e : frames) encode_png_row(e, out[0]);
      return;
    }
    // runs of equal geometry, one scn_jpeg_encode_u8 call each
    size_t i = 0;
    while (i < frames.size()) {
      size_t j = i + 1;
      if (!frames[i].is_null())
        while (j < frames.size() && !frames[j].is_null() &&
               frames[j].as_const_frame()->as_frame_info() == frames[i].as_const_frame()->as_frame_info())
          ++j;
      encode_jpeg_run(frames, i, j, out[0]);
      i = j;
    }
  }

 private:
  static std::string unsupported(const Frame* f) {
    if (f->layout != FrameLayout::HWC) return "JPEG needs HWC frames, got an NV12 element";
    if ((proto::FrameType)f->type != proto::U8)
      return "JPEG needs uint8 frames, got type " + std::to_string((int)(proto::FrameType)f->type);
    if (f->channels() != 1 && f->channels() != 3)
      return "JPEG needs 1- or 3-channel frames, got " + std::to_string(f->channels()) + " channels";
    if (f->width() > 65500 || f->height() > 65500)
      return "JPEG frames are at most 65500 x 65500, got " + std::to_string(f->width()) + " x " +
             std::to_string(f->height());
    return "";
  }

  void encode_png_row(const Element& e, Elements& col) {
    std::string err = e.is_null() ? std::string("null frame") : "";
    std::vector<u8> png;
    if (err.empty()) {
      const Frame* f = e.as_const_frame();
      Frame* host = new_frame(CPU_DEVICE, f->as_frame_info());
      memcpy_buffer(host->data, CPU_DEVICE, f->data, device_, f->size());
      err = encode_png(host, png);
      delete_buffer(CPU_DEVICE, host->data);
      delete host;
    }
    if (!err.empty()) {
      report_kernel_error("ImageEncoder, row " + std::to_string(e.index) + ": " + err);
      col.push_back(Element());
      return;
    }
    u8* buf = new_buffer(CPU_DEVICE, png.size());
    memcpy(buf, png.data(), png.size());
    insert_element(col, buf, png.size());
  }

  static void* alloc_on(void* ctx, size_t bytes) {
    auto* self = static_cast<ImageEncoderKernelGPU*>(ctx);
    self->staging_ = new_buffer(self->device_, bytes ? bytes : 1);
    return self->staging_;
  }

  void encode_jpeg_run(const Elements& frames, size_t i0, size_t i1, Elements& col) {
    const size_t n = i1 - i0;
    const Frame* f0 = frames[i0].is_null() ? nullptr : frames[i0].as_const_frame();
    const std::string why = f0 ? unsupported(f0) : std::string("null frame");
    if (!why.empty()) {
      report_kernel_error("ImageEncoder, row " + std::to_string(frames[i0].index) + ": " + why);
      for (size_t k = 0; k < n; ++k) col.push_back(Element());
      return;
    }
    std::vector<const u8*> src;
    for (size_t k = i0; k < i1; ++k) src.push_back(frames[k].as_const_frame()->data);
    std::vector<size_t> sizes(n);
    staging_ = nullptr;
    cudaStream_t stream = (cudaStream_t)device_stream(device_);
    const int rc = scn_jpeg_encode_u8_opts(src.data(), (int)n, f0->width(), f0->height(), f0->channels(), quality_,
                                           &opts_, &ImageEncoderKernelGPU::alloc_on, this, sizes.data(), stream);
    if (rc != 0) LOG(FATAL) << "scn_jpeg_encode_u8_opts failed with code " << rc;
    // one copy of the packed files to the host, in the synchronisation the encoder needs anyway
    u8* block = new_block_buffer_sizes(CPU_DEVICE, sizes);
    size_t total = 0;
    for (size_t s : sizes) total += s;
    if (cudaMemcpyAsync(block, staging_, total, cudaMemcpyDeviceToHost, stream) != cudaSuccess ||
        cudaStreamSynchronize(stream) != cudaSuccess)
      LOG(FATAL) << "ImageEncoder: copying encoded JPEG files from GPU " << device_.id << " failed";
    delete_buffer(device_, staging_);
    staging_ = nullptr;
    size_t at = 0;
    for (size_t k = 0; k < n; ++k) {
      insert_element(col, block + at, sizes[k]);
      at += sizes[k];
    }
  }

  DeviceHandle device_;
  bool jpeg_ = false;
  int quality_ = 95;
  scn_jpeg_options opts_ = {0, 0, 0, 0};  // sampling, luma and chroma quality, optimize: 0 when absent
  u8* staging_ = nullptr;  // the device buffer scn_jpeg_encode_u8 writes the files of one run into
  Result valid_;
};

REGISTER_KERNEL(ImageEncoder, ImageEncoderKernelGPU)
    .device(DeviceType::GPU)
    .batch(64)
    .num_devices(1)
    .output_device("img", DeviceType::CPU);

class ImageDecoderKernel : public BatchedKernel {
 public:
  ImageDecoderKernel(const KernelConfig& config) : BatchedKernel(config) {}
  void execute(const BatchedElements& in, BatchedElements& out) override {
    for (const Element& e : in[0]) {
      Frame* f = nullptr;
      const std::string err = e.is_null() ? std::string("ImageDecoder: null element") : decode_png(e.buffer, e.size, f);
      if (!err.empty()) {
        report_kernel_error(err + " (row " + std::to_string(e.index) + ")");
        out[0].push_back(Element());
        continue;
      }
      insert_frame(out[0], f);
    }
  }
};

REGISTER_OP(ImageDecoder).input("img").frame_output("frame");
REGISTER_KERNEL(ImageDecoder, ImageDecoderKernel).device(DeviceType::CPU).batch(8).num_devices(1);

// ---- GPU kernel: JPEG through nvJPEG, output frames in device memory ---------------------------
class ImageDecoderKernelGPU : public BatchedKernel {
 public:
  ImageDecoderKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {
    if (cudaSetDevice(device_.id) != cudaSuccess) {
      RESULT_ERROR(&valid_, "ImageDecoder: cannot select GPU %d", device_.id);
      return;
    }
    nvjpegStatus_t st = nvjpegCreateSimple(&handle_);
    if (st == NVJPEG_STATUS_SUCCESS) st = nvjpegJpegStateCreate(handle_, &state_);
    if (st != NVJPEG_STATUS_SUCCESS) {
      RESULT_ERROR(&valid_, "ImageDecoder: nvJPEG initialisation failed (status %d)", (int)st);
      return;
    }
    valid_.set_success(true);
  }
  ~ImageDecoderKernelGPU() override {
    if (state_) nvjpegJpegStateDestroy(state_);
    if (handle_) nvjpegDestroy(handle_);
  }
  void validate(Result* result) override { result->CopyFrom(valid_); }

  void execute(const BatchedElements& in, BatchedElements& out) override {
    if (cudaSetDevice(device_.id) != cudaSuccess) LOG(FATAL) << "ImageDecoder: cannot select GPU " << device_.id;
    cudaStream_t stream = (cudaStream_t)device_stream(device_);
    auto bad = [&](const Element& e, const std::string& why) {
      report_kernel_error("ImageDecoder, row " + std::to_string(e.index) + ": " + why);
      out[0].push_back(Element());
    };
    for (const Element& e : in[0]) {
      if (e.is_null()) {
        bad(e, "null element");
        continue;
      }
      if (e.size >= 8 && memcmp(e.buffer, kPngSig, 8) == 0) {
        Frame* host = nullptr;
        const std::string err = decode_png(e.buffer, e.size, host);
        if (!err.empty()) {
          bad(e, err);
          continue;
        }
        Frame* dev = new_frame(device_, host->as_frame_info());
        if (cudaMemcpyAsync(dev->data, host->data, host->size(), cudaMemcpyHostToDevice, stream) != cudaSuccess ||
            cudaStreamSynchronize(stream) != cudaSuccess)
          LOG(FATAL) << "ImageDecoder: copying a decoded PNG to GPU " << device_.id << " failed";
        delete_buffer(CPU_DEVICE, host->data);
        delete host;
        insert_frame(out[0], dev);
        continue;
      }
      int components = 0, widths[NVJPEG_MAX_COMPONENT] = {0}, heights[NVJPEG_MAX_COMPONENT] = {0};
      nvjpegChromaSubsampling_t subsampling;
      nvjpegStatus_t st = nvjpegGetImageInfo(handle_, e.buffer, e.size, &components, &subsampling, widths, heights);
      if (st != NVJPEG_STATUS_SUCCESS || widths[0] <= 0 || heights[0] <= 0) {
        bad(e, "neither PNG nor a JPEG that nvJPEG can parse (status " + std::to_string((int)st) + ")");
        continue;
      }
      Frame* f = new_frame(device_, FrameInfo(heights[0], widths[0], 3, FrameType::U8));
      nvjpegImage_t img;
      memset(&img, 0, sizeof(img));
      img.channel[0] = f->data;
      img.pitch[0] = (size_t)widths[0] * 3;
      st = nvjpegDecode(handle_, state_, e.buffer, e.size, NVJPEG_OUTPUT_RGBI, &img, stream);
      if (st != NVJPEG_STATUS_SUCCESS) {
        Element dead(f);
        delete_element(device_, dead);
        bad(e, "nvjpegDecode failed (status " + std::to_string((int)st) + ")");
        continue;
      }
      insert_frame(out[0], f);
    }
    // the encoded bytes are borrowed from the engine: nothing of this batch may still be reading them
    if (cudaStreamSynchronize(stream) != cudaSuccess) LOG(FATAL) << "ImageDecoder: stream synchronisation failed";
  }

 private:
  DeviceHandle device_;
  nvjpegHandle_t handle_ = nullptr;
  nvjpegJpegState_t state_ = nullptr;
  Result valid_;
};

REGISTER_KERNEL(ImageDecoder, ImageDecoderKernelGPU)
    .device(DeviceType::GPU)
    .batch(8)
    .num_devices(1)
    .input_device("img", DeviceType::CPU);

// ---------------------------------------------------------------------------------------------
// Histogram on a CPU pipeline instance (BASELINE configs[0]: "Histogram op on one 640x480 H.264 clip, CPU
// pipeline_instances=1 (plumbing, no GPU)").  The reference registers its Histogram kernel for DeviceType::CPU
// (tests/test_ops.cpp:13-59: cv::calcHist, 16 bins over [0, 256) per channel, int32 counts); this is that kernel
// without OpenCV: bin = value >> 4.  It is chosen only by a graph that places the op on the CPU -- a GPU
// placement runs HistogramKernelGPU (stdlib_ops.cu) and fails without CUDA; nothing falls back to this.
class HistogramKernelCPU : public BatchedKernel {
 public:
  HistogramKernelCPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {}

  void execute(const BatchedElements& input_columns, BatchedElements& output_columns) override {
    const Elements& frames = input_columns[0];
    const i32 n = (i32)num_rows(frames);
    if (n == 0) return;
    constexpr size_t kHistBytes = 3 * 16 * sizeof(i32);
    u8* block = new_block_buffer_size(device_, kHistBytes, n);
    for (i32 i = 0; i < n; ++i) {
      const Frame* f = frames[i].as_const_frame();
      if (f->layout != FrameLayout::HWC || f->channels() != 3 || (proto::FrameType)f->type != proto::U8) {
        report_kernel_error("Histogram, row " + std::to_string(frames[i].index) + ": expects HxWx3 uint8 frames, got " +
                            std::to_string(f->height()) + "x" + std::to_string(f->width()) + "x" +
                            std::to_string(f->channels()) + " type " + std::to_string((int)(proto::FrameType)f->type) +
                            (f->layout == FrameLayout::HWC ? "" : " (an NV12 frame element)"));
        output_columns[0].push_back(Element());
        delete_buffer(device_, block);  // the refused row's reference
        continue;
      }
      i32* out = reinterpret_cast<i32*>(block + (size_t)i * kHistBytes);
      // four sub-histograms per channel break the store-to-load chain on runs of equal values
      i32 part[4][3][16];
      memset(part, 0, sizeof(part));
      const u8* p = f->data;
      const size_t px = (size_t)f->width() * f->height();
      size_t k = 0;
      for (; k + 4 <= px; k += 4, p += 12)
        for (int u = 0; u < 4; ++u) {
          ++part[u][0][p[3 * u] >> 4];
          ++part[u][1][p[3 * u + 1] >> 4];
          ++part[u][2][p[3 * u + 2] >> 4];
        }
      for (; k < px; ++k, p += 3) {
        ++part[0][0][p[0] >> 4];
        ++part[0][1][p[1] >> 4];
        ++part[0][2][p[2] >> 4];
      }
      for (int c = 0; c < 3; ++c)
        for (int b = 0; b < 16; ++b) out[c * 16 + b] = part[0][c][b] + part[1][c][b] + part[2][c][b] + part[3][c][b];
      insert_element(output_columns[0], reinterpret_cast<u8*>(out), kHistBytes);
    }
  }

 private:
  DeviceHandle device_;
};

REGISTER_KERNEL(Histogram, HistogramKernelCPU).device(DeviceType::CPU).batch(8).num_devices(1);

}  // namespace
}  // namespace scanner
