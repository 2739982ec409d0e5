// stdlib_ops.cu -- the per-frame ops of the hot path as a Scanner op plugin (libscn_stdlib.so).
// Same op names, columns and argument messages as the reference's in-tree ops
// (tests/test_ops.cpp:13-59 Histogram, :114-170 Resize, :239-310 Blur) -- but the kernels are
// registered for DeviceType::GPU and run the sm_90a kernels of libscn_kernels.so on the
// pipeline instance's stream.  Loaded with dlopen like any user op library (Client.load_op).
#include <climits>
#include <map>
#include <string>

#include "scanner/api/kernel.h"
#include "scanner/api/op.h"
#include "scanner/util/cuda.h"
#include "scanner/util/memory.h"
#include "scn_kernels.h"
#include "stdlib_args.pb.h"

namespace scanner {
namespace {

#define SCN_CHECK(call__)                                                              \
  do {                                                                                 \
    const int rc__ = (call__);                                                         \
    if (rc__ != 0) LOG(FATAL) << #call__ << " failed with code " << rc__;              \
  } while (0)

// batches may mix frame sizes (different videos): process runs of equal geometry
template <typename F>
void for_each_run(const Elements& col, F&& fn) {
  size_t i = 0;
  while (i < col.size()) {
    const Frame* f0 = col[i].as_const_frame();
    size_t j = i + 1;
    while (j < col.size() && col[j].as_const_frame()->as_frame_info() == f0->as_frame_info()) ++j;
    fn(i, j, f0);
    i = j;
  }
}

bool is_nv12(const Frame* f) { return f->layout == FrameLayout::NV12; }

// geometry of the picture a frame element holds (an NV12 element is (H*3/2, W, 1))
int pic_width(const Frame* f) { return f->width(); }
int pic_height(const Frame* f) { return is_nv12(f) ? f->height() / 3 * 2 : f->height(); }

// why a frame element is neither an HxWx3 uint8 frame nor a well-formed NV12 element; empty when it is one
std::string rgb8_problem(const Frame* f) {
  if (is_nv12(f)) {
    if (f->channels() != 1 || (proto::FrameType)f->type != proto::U8 || f->height() % 3 != 0 || (f->width() & 1))
      return "malformed NV12 frame element " + std::to_string(f->height()) + "x" + std::to_string(f->width());
    return "";
  }
  if (f->channels() != 3 || (proto::FrameType)f->type != proto::U8)
    return "expects HxWx3 uint8 frames, got " + std::to_string(f->height()) + "x" + std::to_string(f->width()) + "x" +
           std::to_string(f->channels()) + " type " + std::to_string((int)(proto::FrameType)f->type);
  return "";
}

void require_rgb8(const Frame* f, const char* op) {
  const std::string why = rgb8_problem(f);
  if (!why.empty()) LOG(FATAL) << op << ": " << why;
}

// ---------------------------------------------------------------------------------------------
class HistogramKernelGPU : public BatchedKernel {
 public:
  HistogramKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {}

  void execute(const BatchedElements& input_columns, BatchedElements& output_columns) override {
    const Elements& frames = input_columns[0];
    const i32 n = (i32)num_rows(frames);
    if (n == 0) return;
    CU_CHECK(cudaSetDevice(device_.id));
    constexpr size_t kHistBytes = 3 * 16 * sizeof(i32);
    u8* block = new_block_buffer_size(device_, kHistBytes, n);  // one block for the batch
    for_each_run(frames, [&](size_t i0, size_t i1, const Frame* f0) {
      require_rgb8(f0, "Histogram");
      std::vector<const u8*> ptrs;
      for (size_t i = i0; i < i1; ++i) ptrs.push_back(frames[i].as_const_frame()->data);
      if (is_nv12(f0)) {
        // decoder-native surface: colour conversion happens in registers, RGB24 never exists
        const int w = pic_width(f0), h = pic_height(f0);
        std::vector<const u8*> chroma;
        for (const u8* p : ptrs) chroma.push_back(p + (size_t)w * h);
        SCN_CHECK(scn_nv12_hist_resize(ptrs.data(), chroma.data(), (size_t)w, (int)ptrs.size(), w, h,
                                       (int32_t*)(block + i0 * kHistBytes), nullptr, 0, 0, nullptr,
                                       device_stream(device_)));
        return;
      }
      SCN_CHECK(scn_hist16_u8c3(ptrs.data(), (int)ptrs.size(), f0->width(), f0->height(),
                                (int32_t*)(block + i0 * kHistBytes), device_stream(device_)));
    });
    for (i32 i = 0; i < n; ++i) insert_element(output_columns[0], block + (size_t)i * kHistBytes, kHistBytes);
  }

 private:
  DeviceHandle device_;
};

REGISTER_OP(Histogram).frame_input("frame").output("histogram", ColumnType::Bytes, "Histogram");

REGISTER_KERNEL(Histogram, HistogramKernelGPU)
    .device(DeviceType::GPU)
    .batch(64)
    .num_devices(1)
    .input_layout("frame", FrameLayout::NV12);

// ---------------------------------------------------------------------------------------------
class ResizeKernelGPU : public BatchedKernel {
 public:
  ResizeKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {}
  ~ResizeKernelGPU() {
    for (auto& kv : plans_) delete_buffer(device_, kv.second);
  }

  // a parse failure is reported by execute(), where the failing row is known
  void new_stream(const std::vector<u8>& args) override {
    args_ = ResizeArgs();
    args_ok_ = args_.ParseFromArray(args.data(), (int)args.size());
  }

  void execute(const BatchedElements& input_columns, BatchedElements& output_columns) override {
    const Elements& frames = input_columns[0];
    if (frames.empty()) return;
    CU_CHECK(cudaSetDevice(device_.id));
    for_each_run(frames, [&](size_t i0, size_t i1, const Frame* f0) {
      const i32 n = (i32)(i1 - i0);
      const int sw = pic_width(f0), sh = pic_height(f0);
      int tw = 0, th = 0;
      std::string why = args_ok_ ? rgb8_problem(f0) : "could not parse ResizeArgs";
      if (why.empty()) {
        scn_resize_target(sw, sh, args_.width(), args_.height(), args_.min(), args_.preserve_aspect(), &tw, &th);
        if (tw <= 0 || th <= 0 || (int64_t)tw * th > INT_MAX)
          why = "invalid target size " + std::to_string(tw) + "x" + std::to_string(th) + " for a " +
                std::to_string(sw) + "x" + std::to_string(sh) + " frame";
      }
      if (!why.empty()) {
        report_kernel_error("Resize, row " + std::to_string(frames[i0].index) + ": " + why);
        for (i32 i = 0; i < n; ++i) output_columns[0].push_back(Element());
        return;
      }
      FrameInfo info(th, tw, 3, FrameType::U8);
      std::vector<Frame*> outs = new_frames(device_, info, n);
      std::vector<const u8*> src;
      std::vector<u8*> dst;
      for (i32 i = 0; i < n; ++i) {
        src.push_back(frames[i0 + i].as_const_frame()->data);
        dst.push_back(outs[i]->data);
      }
      if (is_nv12(f0)) {
        std::vector<const u8*> chroma;
        for (const u8* p : src) chroma.push_back(p + (size_t)sw * sh);
        SCN_CHECK(scn_nv12_hist_resize(src.data(), chroma.data(), (size_t)sw, n, sw, sh, nullptr, dst.data(), tw, th,
                                       plan_for(sw, sh, tw, th), device_stream(device_)));
      } else {
        SCN_CHECK(scn_resize_bilinear_u8c3(src.data(), n, sw, sh, dst.data(), tw, th, plan_for(sw, sh, tw, th),
                                           device_stream(device_)));
      }
      for (i32 i = 0; i < n; ++i) insert_frame(output_columns[0], outs[i]);
    });
  }

 private:
  // coefficient tables are built on the host once per geometry and kept on the device
  const void* plan_for(int sw, int sh, int dw, int dh) {
    const std::array<int, 4> key = {sw, sh, dw, dh};
    auto it = plans_.find(key);
    if (it != plans_.end()) return it->second;
    const size_t bytes = scn_resize_plan_bytes(dw, dh);
    std::vector<u8> host(bytes);
    SCN_CHECK(scn_resize_plan_fill(sw, sh, dw, dh, host.data()));
    u8* dev = new_buffer(device_, bytes);
    memcpy_buffer(dev, device_, host.data(), CPU_DEVICE, bytes);
    plans_[key] = dev;
    return dev;
  }

  DeviceHandle device_;
  ResizeArgs args_;
  bool args_ok_ = true;
  std::map<std::array<int, 4>, u8*> plans_;
};

REGISTER_OP(Resize).frame_input("frame").frame_output("frame").stream_protobuf_name("ResizeArgs");

REGISTER_KERNEL(Resize, ResizeKernelGPU)
    .device(DeviceType::GPU)
    .batch(64)
    .num_devices(1)
    .input_layout("frame", FrameLayout::NV12);

// ---------------------------------------------------------------------------------------------
// ConvertColor: scannertools' op (cv::cvtColor with ConvertColorArgs.conversion, a per-stream OpenCV code name),
// bit-exact for the codes scn_convert_color_code knows.  Gray output is (H, W, 1).  A decoded NV12 element is
// converted from the RGB24 frame the decoder would have delivered, without writing that frame.
class ConvertColorKernelGPU : public BatchedKernel {
 public:
  ConvertColorKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {}

  void new_stream(const std::vector<u8>& args) override {
    ConvertColorArgs a;
    code_ = -1;
    if (!a.ParseFromArray(args.data(), (int)args.size())) {
      report_kernel_error("Could not parse ConvertColorArgs");
      return;
    }
    code_ = scn_convert_color_code(a.conversion().c_str());
    if (code_ < 0) {
      std::string supported;
      for (int c = 0; scn_convert_color_name(c); ++c) supported += std::string(c ? ", " : "") + scn_convert_color_name(c);
      report_kernel_error("ConvertColor: unsupported conversion '" + a.conversion() + "'; supported: " + supported);
      return;
    }
    SCN_CHECK(scn_convert_color_channels(code_, &in_channels_, &out_channels_));
  }

  void execute(const BatchedElements& input_columns, BatchedElements& output_columns) override {
    const Elements& frames = input_columns[0];
    if (frames.empty()) return;
    CU_CHECK(cudaSetDevice(device_.id));
    for_each_run(frames, [&](size_t i0, size_t i1, const Frame* f0) {
      const i32 n = (i32)(i1 - i0);
      // an NV12 element is a 1-channel frame too: its picture has three channels
      const bool nv12 = is_nv12(f0);
      const int channels = nv12 ? 3 : f0->channels();
      std::string why;
      if ((proto::FrameType)f0->type != proto::U8)
        why = "expects uint8 frames, got type " + std::to_string((int)(proto::FrameType)f0->type);
      else if (nv12 && (f0->channels() != 1 || f0->height() % 3 != 0 || (f0->width() & 1)))
        why = "malformed NV12 frame element " + std::to_string(f0->height()) + "x" + std::to_string(f0->width());
      else if (channels != in_channels_)
        why = std::string(scn_convert_color_name(code_)) + " takes " + std::to_string(in_channels_) +
              "-channel frames, got " + std::to_string(channels) + " channels";
      if (!why.empty()) {
        report_kernel_error("ConvertColor, row " + std::to_string(frames[i0].index) + ": " + why);
        for (i32 i = 0; i < n; ++i) output_columns[0].push_back(Element());
        return;
      }
      const int w = pic_width(f0), h = pic_height(f0);
      std::vector<Frame*> outs = new_frames(device_, FrameInfo(h, w, out_channels_, FrameType::U8), n);
      std::vector<const u8*> src;
      std::vector<u8*> dst;
      for (i32 i = 0; i < n; ++i) {
        src.push_back(frames[i0 + i].as_const_frame()->data);
        dst.push_back(outs[i]->data);
      }
      if (nv12) {
        std::vector<const u8*> chroma;
        for (const u8* p : src) chroma.push_back(p + (size_t)w * h);
        SCN_CHECK(scn_convert_color_nv12(src.data(), chroma.data(), (size_t)w, n, w, h, code_, dst.data(),
                                         device_stream(device_)));
      } else {
        SCN_CHECK(scn_convert_color_u8(src.data(), n, w, h, code_, dst.data(), device_stream(device_)));
      }
      for (i32 i = 0; i < n; ++i) insert_frame(output_columns[0], outs[i]);
    });
  }

 private:
  DeviceHandle device_;
  int code_ = -1;
  int in_channels_ = 0, out_channels_ = 0;
};

REGISTER_OP(ConvertColor).frame_input("frame").frame_output("frame").stream_protobuf_name("ConvertColorArgs");

REGISTER_KERNEL(ConvertColor, ConvertColorKernelGPU)
    .device(DeviceType::GPU)
    .batch(64)
    .num_devices(1)
    .input_layout("frame", FrameLayout::NV12);

// ---------------------------------------------------------------------------------------------
class BlurKernelGPU : public BatchedKernel {
 public:
  BlurKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {
    BlurArgs args;
    const bool parsed = args.ParseFromArray(config.args.data(), (int)config.args.size());
    if (!parsed || config.args.empty()) {
      RESULT_ERROR(&valid_, "Could not parse BlurArgs");
      return;
    }
    kernel_size_ = args.kernel_size();
    if (kernel_size_ < 1 || kernel_size_ > 31) {
      RESULT_ERROR(&valid_, "Blur kernel_size %d is outside [1, 31]", kernel_size_);
      return;
    }
    valid_.set_success(true);
  }

  void validate(Result* result) override { result->CopyFrom(valid_); }

  void execute(const BatchedElements& input_columns, BatchedElements& output_columns) override {
    const Elements& frames = input_columns[0];
    if (frames.empty()) return;
    CU_CHECK(cudaSetDevice(device_.id));
    for_each_run(frames, [&](size_t i0, size_t i1, const Frame* f0) {
      require_rgb8(f0, "Blur");
      const i32 n = (i32)(i1 - i0);
      std::vector<Frame*> outs = new_frames(device_, f0->as_frame_info(), n);
      std::vector<const u8*> src;
      std::vector<u8*> dst;
      for (i32 i = 0; i < n; ++i) {
        src.push_back(frames[i0 + i].as_const_frame()->data);
        dst.push_back(outs[i]->data);
      }
      SCN_CHECK(scn_box_blur_u8c3(src.data(), n, f0->width(), f0->height(), kernel_size_, dst.data(),
                                  device_stream(device_)));
      for (i32 i = 0; i < n; ++i) insert_frame(output_columns[0], outs[i]);
    });
  }

 private:
  DeviceHandle device_;
  i32 kernel_size_ = 0;
  Result valid_;
};

REGISTER_OP(Blur).frame_input("frame").frame_output("frame").protobuf_name("BlurArgs");

REGISTER_KERNEL(Blur, BlurKernelGPU).device(DeviceType::GPU).batch(16).num_devices(1);

// ---------------------------------------------------------------------------------------------
// OpticalFlow: stencil {0,1}, Farneback with the reference's constructor arguments
// (tests/test_ops.cpp:68-69), output Frame(H, W, 2, F32) on the GPU (:85-87).
class OpticalFlowKernelGPU : public StenciledKernel, public VideoKernel {
 public:
  OpticalFlowKernelGPU(const KernelConfig& config) : StenciledKernel(config), device_(config.devices[0]) {}
  ~OpticalFlowKernelGPU() {
    if (workspace_) delete_buffer(device_, workspace_);
    for (u8*& b : rgb_)
      if (b) delete_buffer(device_, b);
  }

  void new_frame_info() override {
    if (workspace_) delete_buffer(device_, workspace_);
    const int w = pic_width_, h = pic_height_;
    workspace_bytes_ = scn_farneback_workspace_bytes(w, h);
    workspace_ = new_buffer(device_, workspace_bytes_);
    for (u8*& b : rgb_) {
      if (b) delete_buffer(device_, b);
      b = nullptr;
    }
    rgb_of_[0] = rgb_of_[1] = -1;
    chain_ = 0;
    last_next_row_ = -1;
  }

  void reset() override {  // row ids identify a frame within one task only
    rgb_of_[0] = rgb_of_[1] = -1;
    chain_ = 0;
    last_next_row_ = -1;
  }

  void execute(const StenciledElements& input_columns, Elements& output_columns) override {
    const Elements& window = input_columns[0];
    CU_CHECK(cudaSetDevice(device_.id));
    const Frame* f0 = window[0].as_const_frame();
    const Frame* f1 = window[1].as_const_frame();
    require_rgb8(f0, "OpticalFlow");
    pic_width_ = pic_width(f0);
    pic_height_ = pic_height(f0);
    check_frame(device_, window[0]);
    if (!(f0->as_frame_info() == f1->as_frame_info())) LOG(FATAL) << "OpticalFlow: frames of one window differ in size";
    const int w = pic_width_, h = pic_height_;
    FrameInfo out_info(h, w, 2, FrameType::F32);
    Frame* out = new_frame(device_, out_info);
    // decoder-native (packed NV12) elements are converted here with the reference's NV12 -> RGB
    // arithmetic; the frame that was `next` of the previous row is `prev` of this one and is reused
    const u8* prev = is_nv12(f0) ? rgb_of(f0, window[0].index, w, h) : f0->data;
    const u8* next = is_nv12(f1) ? rgb_of(f1, window[1].index, w, h) : f1->data;
    float* flow = reinterpret_cast<float*>(out->data);
    // rows are walked in order: the `next` frame of the last window is this window's `prev` (same input row), and
    // its pyramid of polynomial expansions is still in the workspace
    const int reuse = window[0].index >= 0 && window[0].index == last_next_row_;
    SCN_CHECK(scn_farneback_u8c3_chain(&prev, &next, 1, w, h, &flow, 3, 0.5, 15, 3, 5, 1.2, workspace_,
                                       workspace_bytes_, reuse, &chain_, device_stream(device_)));
    last_next_row_ = window[1].index;
    insert_frame(output_columns[0], out);
  }

 private:
  const u8* rgb_of(const Frame* f, i64 row, int w, int h) {
    for (int k = 0; k < 2; ++k)
      if (rgb_of_[k] == row && row >= 0 && rgb_[k]) {
        last_used_ = k;
        return rgb_[k];
      }
    const int k = 1 - last_used_;  // overwrite the copy not used by the other frame of this window
    if (!rgb_[k]) rgb_[k] = new_buffer(device_, (size_t)w * h * 3);
    const u8* lp = f->data;
    const u8* cp = f->data + (size_t)w * h;
    u8* dst = rgb_[k];
    SCN_CHECK(scn_nv12_to_rgb24(&lp, &cp, (size_t)w, 1, w, h, &dst, (size_t)w * 3, device_stream(device_)));
    rgb_of_[k] = row;
    last_used_ = k;
    return rgb_[k];
  }

  DeviceHandle device_;
  u8* workspace_ = nullptr;
  size_t workspace_bytes_ = 0;
  int pic_width_ = 0, pic_height_ = 0;
  u8* rgb_[2] = {nullptr, nullptr};          // RGB24 copies of the window's NV12 elements
  i64 rgb_of_[2] = {-1, -1};                 // input row (Element::index) each holds
  int last_used_ = 1;
  int chain_ = 0;                            // scn_farneback_u8c3_chain state of workspace_
  i64 last_next_row_ = -1;                   // input row whose expansion the workspace holds
};

REGISTER_OP(OpticalFlow).frame_input("frame").frame_output("flow").stencil({0, 1});

REGISTER_KERNEL(OpticalFlow, OpticalFlowKernelGPU)
    .device(DeviceType::GPU)
    .num_devices(1)
    .input_layout("frame", FrameLayout::NV12);

// ---------------------------------------------------------------------------------------------
// OpticalFlowTVL1: stencil {0,1}, TV-L1 dense flow (scn_tvl1_u8, DESIGN.md "TV-L1"), output Frame(H, W, 2, F32).
// Not a reference op.  A batch of up to 8 windows is one scn_tvl1_u8 call; each distinct input frame of the batch
// is converted to gray once (COLOR_RGB2GRAY from RGB24 or NV12 elements; 1-channel u8 frames are used as they are).
class OpticalFlowTVL1KernelGPU : public StenciledBatchedKernel {
 public:
  OpticalFlowTVL1KernelGPU(const KernelConfig& config) : StenciledBatchedKernel(config), device_(config.devices[0]) {
    OpticalFlowTVL1Args a;
    if (!a.ParseFromArray(config.args.data(), (int)config.args.size())) {
      args_problem_ = "could not parse OpticalFlowTVL1Args";
      return;
    }
    // 0 (absent) means the default; a negative epsilon disables the early stop
    tau_ = a.tau() != 0.f ? a.tau() : 0.25f;
    lambda_ = a.lambda_() != 0.f ? a.lambda_() : 0.15f;
    theta_ = a.theta() != 0.f ? a.theta() : 0.3f;
    nscales_ = a.nscales() != 0 ? a.nscales() : 5;
    warps_ = a.warps() != 0 ? a.warps() : 5;
    epsilon_ = a.epsilon() != 0.f ? (a.epsilon() < 0.f ? -1.f : a.epsilon()) : 0.01f;
    iterations_ = a.iterations() != 0 ? a.iterations() : 300;
    scale_step_ = a.scale_step() != 0.f ? a.scale_step() : 0.8f;
    median_ = a.median_filtering() != 0 ? a.median_filtering() : 5;
    if (call(nullptr, nullptr, 0, 16, 16, nullptr) != 0)
      args_problem_ = "invalid arguments (tau " + std::to_string(tau_) + ", lambda " + std::to_string(lambda_) +
                      ", theta " + std::to_string(theta_) + ", nscales " + std::to_string(nscales_) + ", warps " +
                      std::to_string(warps_) + ", epsilon " + std::to_string(epsilon_) + ", iterations " +
                      std::to_string(iterations_) + ", scale_step " + std::to_string(scale_step_) +
                      ", median_filtering " + std::to_string(median_) + ")";
  }
  ~OpticalFlowTVL1KernelGPU() {
    if (workspace_) delete_buffer(device_, workspace_);
    if (gray_) delete_buffer(device_, gray_);
  }

  void execute(const StenciledBatchedElements& input_columns, BatchedElements& output_columns) override {
    const std::vector<Elements>& windows = input_columns[0];
    const size_t nb = windows.size();
    if (nb == 0) return;
    CU_CHECK(cudaSetDevice(device_.id));
    // runs of windows of one geometry
    auto first = [&](size_t q) { return windows[q][0].is_null() ? nullptr : windows[q][0].as_const_frame(); };
    size_t i = 0;
    while (i < nb) {
      const Frame* f0 = first(i);
      size_t j = i + 1;
      while (f0 && j < nb && first(j) && first(j)->as_frame_info() == f0->as_frame_info()) ++j;
      run(windows, i, j, output_columns[0]);
      i = j;
    }
  }

 private:
  int call(const u8* const* prev, const u8* const* next, int n, int w, int h, float* const* flow) {
    return scn_tvl1_u8(prev, next, n, w, h, flow, tau_, lambda_, theta_, nscales_, warps_, epsilon_, iterations_,
                       scale_step_, median_, nullptr, workspace_, workspace_bytes_, device_stream(device_));
  }

  static std::string frame_problem(const Frame* f) {
    if ((proto::FrameType)f->type != proto::U8)
      return "expects uint8 frames, got type " + std::to_string((int)(proto::FrameType)f->type);
    if (is_nv12(f)) {
      if (f->channels() != 1 || f->height() % 3 != 0 || (f->width() & 1))
        return "malformed NV12 frame element " + std::to_string(f->height()) + "x" + std::to_string(f->width());
    } else if (f->channels() != 1 && f->channels() != 3) {
      return "expects gray (HxWx1), RGB24 (HxWx3) or NV12 frames, got " + std::to_string(f->height()) + "x" +
             std::to_string(f->width()) + "x" + std::to_string(f->channels());
    }
    if (pic_width(f) < 2 || pic_height(f) < 2)
      return "frames must be at least 2x2, got " + std::to_string(pic_width(f)) + "x" + std::to_string(pic_height(f));
    return "";
  }

  void run(const std::vector<Elements>& windows, size_t i0, size_t i1, Elements& out) {
    const i32 n = (i32)(i1 - i0);
    const Frame* f0 = windows[i0][0].is_null() ? nullptr : windows[i0][0].as_const_frame();
    std::string why = args_problem_;
    for (size_t q = i0; q < i1 && why.empty(); ++q)
      for (const Element& e : windows[q]) {
        if (e.is_null()) {
          why = "null input frame";
          break;
        }
        why = frame_problem(e.as_const_frame());
        if (why.empty() && (!f0 || !(e.as_const_frame()->as_frame_info() == f0->as_frame_info())))
          why = "frames of one window differ in size";
        if (!why.empty()) break;
      }
    if (!why.empty()) {
      report_kernel_error("OpticalFlowTVL1, row " + std::to_string(windows[i0][0].index) + ": " + why);
      for (i32 k = 0; k < n; ++k) out.push_back(Element());
      return;
    }
    const int w = pic_width(f0), h = pic_height(f0);
    const size_t px = (size_t)w * h;
    // each distinct frame of the run once (the `next` of one window is the `prev` of the following one)
    std::map<const u8*, int> slot;
    std::vector<const u8*> distinct;
    for (size_t q = i0; q < i1; ++q)
      for (const Element& e : windows[q]) {
        const u8* d = e.as_const_frame()->data;
        if (slot.emplace(d, (int)distinct.size()).second) distinct.push_back(d);
      }
    const bool direct = !is_nv12(f0) && f0->channels() == 1;
    std::vector<const u8*> gray(distinct.size());
    if (direct) {
      gray = distinct;
    } else {
      if (gray_bytes_ < px * distinct.size()) {
        if (gray_) delete_buffer(device_, gray_);
        gray_bytes_ = px * distinct.size();
        gray_ = new_buffer(device_, gray_bytes_);
      }
      std::vector<u8*> dst(distinct.size());
      for (size_t k = 0; k < distinct.size(); ++k) dst[k] = gray_ + k * px;
      const int code = scn_convert_color_code("COLOR_RGB2GRAY");
      if (is_nv12(f0)) {
        std::vector<const u8*> chroma;
        for (const u8* p : distinct) chroma.push_back(p + px);
        SCN_CHECK(scn_convert_color_nv12(distinct.data(), chroma.data(), (size_t)w, (int)distinct.size(), w, h, code,
                                         dst.data(), device_stream(device_)));
      } else {
        SCN_CHECK(scn_convert_color_u8(distinct.data(), (int)distinct.size(), w, h, code, dst.data(),
                                       device_stream(device_)));
      }
      for (size_t k = 0; k < distinct.size(); ++k) gray[k] = dst[k];
    }
    const size_t need = scn_tvl1_workspace_bytes(w, h, n);
    if (workspace_bytes_ < need) {
      if (workspace_) delete_buffer(device_, workspace_);
      workspace_bytes_ = need;
      workspace_ = new_buffer(device_, need);
    }
    std::vector<Frame*> outs = new_frames(device_, FrameInfo(h, w, 2, FrameType::F32), n);
    std::vector<const u8*> prev, next;
    std::vector<float*> flow;
    for (size_t q = i0; q < i1; ++q) {
      prev.push_back(gray[slot[windows[q][0].as_const_frame()->data]]);
      next.push_back(gray[slot[windows[q][1].as_const_frame()->data]]);
      flow.push_back(reinterpret_cast<float*>(outs[q - i0]->data));
    }
    SCN_CHECK(call(prev.data(), next.data(), n, w, h, flow.data()));
    for (i32 k = 0; k < n; ++k) insert_frame(out, outs[k]);
  }

  DeviceHandle device_;
  std::string args_problem_;
  float tau_ = 0.25f, lambda_ = 0.15f, theta_ = 0.3f, epsilon_ = 0.01f, scale_step_ = 0.8f;
  int nscales_ = 5, warps_ = 5, iterations_ = 300, median_ = 5;
  u8* workspace_ = nullptr;
  size_t workspace_bytes_ = 0;
  u8* gray_ = nullptr;  // gray copies of the batch's distinct RGB24 / NV12 frames
  size_t gray_bytes_ = 0;
};

REGISTER_OP(OpticalFlowTVL1).frame_input("frame").frame_output("flow").stencil({0, 1}).protobuf_name(
    "OpticalFlowTVL1Args");

REGISTER_KERNEL(OpticalFlowTVL1, OpticalFlowTVL1KernelGPU)
    .device(DeviceType::GPU)
    .batch(8)
    .num_devices(1)
    .input_layout("frame", FrameLayout::NV12);

// ---------------------------------------------------------------------------------------------
// FrameDigest: frame -> 16 bytes (scn_frame_digest).  Lets frame-valued columns that are too large to
// bring back (flow fields) be compared exactly between runs; not a reference op.
class FrameDigestKernelGPU : public BatchedKernel {
 public:
  FrameDigestKernelGPU(const KernelConfig& config) : BatchedKernel(config), device_(config.devices[0]) {}

  void execute(const BatchedElements& input_columns, BatchedElements& output_columns) override {
    const Elements& frames = input_columns[0];
    const i32 n = (i32)num_rows(frames);
    if (n == 0) return;
    CU_CHECK(cudaSetDevice(device_.id));
    u8* block = new_block_buffer_size(device_, 16, n);
    for_each_run(frames, [&](size_t i0, size_t i1, const Frame* f0) {
      std::vector<const u8*> ptrs;
      for (size_t i = i0; i < i1; ++i) ptrs.push_back(frames[i].as_const_frame()->data);
      SCN_CHECK(scn_frame_digest(ptrs.data(), (int)ptrs.size(), f0->size(), (uint64_t*)(block + i0 * 16), device_stream(device_)));
    });
    for (i32 i = 0; i < n; ++i) insert_element(output_columns[0], block + (size_t)i * 16, 16);
  }

 private:
  DeviceHandle device_;
};

REGISTER_OP(FrameDigest).frame_input("frame").output("digest");

REGISTER_KERNEL(FrameDigest, FrameDigestKernelGPU).device(DeviceType::GPU).batch(8).num_devices(1);

}  // namespace
}  // namespace scanner
