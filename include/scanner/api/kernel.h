// scanner/api/kernel.h -- the Kernel side of Scanner's plugin boundary (reference
// scanner/api/kernel.h:28-475, kernel.cpp:23-145), re-declared so that op sources written for the
// reference compile against scanner-b200:
//   Element / Elements / BatchedElements / StenciledBatchedElements, insert_element/frame,
//   add_element_ref / delete_element, KernelConfig, BaseKernel and the four calling conventions
//   (Kernel, BatchedKernel, StenciledKernel, StenciledBatchedKernel), VideoKernel::check_frame,
//   REGISTER_KERNEL(...).device().num_devices().batch().input_device().output_device().
// Calling contract (SURVEY 8b): one evaluate thread owns a kernel instance; inputs are borrowed;
// outputs are allocated by the kernel on its declared output device, exactly one per input row.
// Addition to the reference's API: GPU kernels enqueue on device_stream(device) and need not synchronise.
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "scanner/api/frame.h"
#include "scanner/util/common.h"
#include "scanner/util/memory.h"
#include "scanner/util/profiler.h"

namespace scanner {

struct Element {
  Element() = default;
  Element(u8* buffer_, size_t size_) : buffer(buffer_), size(size_), is_frame(false) {}
  Element(Frame* frame) : buffer((u8*)frame), size(sizeof(Frame)), is_frame(true) {}

  Frame* as_frame() { return reinterpret_cast<Frame*>(buffer); }
  const Frame* as_const_frame() const { return reinterpret_cast<Frame*>(buffer); }
  FrameInfo* as_frame_info() { return reinterpret_cast<FrameInfo*>(buffer); }
  const FrameInfo* as_const_frame_info() const { return reinterpret_cast<FrameInfo*>(buffer); }
  bool is_null() const { return buffer == nullptr; }

  u8* buffer = nullptr;
  size_t size = 0;
  bool is_frame = false;
  i64 index = 0;  // row id of the element in the op's input domain
};

using Elements = std::vector<Element>;
using BatchedElements = std::vector<Elements>;
using StenciledElements = std::vector<Elements>;
using StenciledBatchedElements = std::vector<std::vector<Elements>>;  // column -> batch -> stencil

inline size_t num_rows(const Elements& column) { return column.size(); }

inline void insert_element(Elements& column, u8* buffer, size_t size) {
  column.push_back(Element{buffer, size});
}
inline void insert_frame(Elements& column, Frame* frame) { column.push_back(Element{frame}); }
inline void insert_element(Element& element, u8* buffer, size_t size) {
  element = Element{buffer, size};
}
inline void insert_frame(Element& element, Frame* frame) { element = Element{frame}; }

// A second handle on the same payload: bumps the block refcount; frame elements get their own
// Frame header (headers are not refcounted).
// A second owner of the same payload (the block's reference count goes up; frame elements get
// their own Frame header), and giving an element up.  Null elements pass through.  (api.cpp)
Element add_element_ref(DeviceHandle device, Element& element);
void delete_element(DeviceHandle device, Element& element);

struct KernelConfig {
  std::vector<DeviceHandle> devices;  // non-empty; devices[0] is where the kernel runs
  std::vector<std::string> input_columns;
  std::vector<proto::ColumnType> input_column_types;
  std::vector<std::string> output_columns;
  std::vector<proto::ColumnType> output_column_types;
  std::vector<u8> args;  // serialized <Op>Args (proto3 wire bytes), may be empty
  i32 node_id = 0;

  static KernelConfig dummy() {
    KernelConfig config;
    config.devices.push_back(CPU_DEVICE);
    return config;
  }
};

class BaseKernel {
 public:
  static const i32 UnlimitedDevices = 0;
  BaseKernel(const KernelConfig&) {}
  virtual ~BaseKernel() {}

  virtual void validate(proto::Result* result) { result->set_success(true); }
  virtual void fetch_resources(proto::Result* result) { result->set_success(true); }
  virtual void setup_with_resources(proto::Result* result) { result->set_success(true); }
  virtual void new_stream(const std::vector<u8>& /*args*/) {}
  virtual void reset() {}

  // engine entry point; the typed subclasses below adapt it to their execute() shape
  virtual void execute_kernel(const StenciledBatchedElements& input_columns,
                              BatchedElements& output_columns) = 0;
  virtual void set_profiler(Profiler* profiler) { profiler_ = profiler; }

  Profiler* profiler_ = nullptr;
};

class StenciledBatchedKernel : public BaseKernel {
 public:
  StenciledBatchedKernel(const KernelConfig& config) : BaseKernel(config) {}
  void execute_kernel(const StenciledBatchedElements& input_columns,
                      BatchedElements& output_columns) override;

 protected:
  virtual void execute(const StenciledBatchedElements& input_columns,
                       BatchedElements& output_columns) = 0;
};

class BatchedKernel : public BaseKernel {
 public:
  BatchedKernel(const KernelConfig& config) : BaseKernel(config) {}
  void execute_kernel(const StenciledBatchedElements& input_columns,
                      BatchedElements& output_columns) override;

 protected:
  virtual void execute(const BatchedElements& input_columns,
                       BatchedElements& output_columns) = 0;
};

class StenciledKernel : public BaseKernel {
 public:
  StenciledKernel(const KernelConfig& config) : BaseKernel(config) {}
  void execute_kernel(const StenciledBatchedElements& input_columns,
                      BatchedElements& output_columns) override;

 protected:
  virtual void execute(const StenciledElements& input_columns, Elements& output_columns) = 0;
};

class Kernel : public BaseKernel {
 public:
  Kernel(const KernelConfig& config) : BaseKernel(config) {}
  void execute_kernel(const StenciledBatchedElements& input_columns,
                      BatchedElements& output_columns) override;

 protected:
  virtual void execute(const Elements& input_columns, Elements& output_columns) = 0;
};

// Mix-in for kernels that consume frame columns: check_frame() fires new_frame_info() when the
// shape/type differs from the cached one (reference kernel.cpp:97-109).
// Fails the running job with `message` without taking the process down.  The reference's only
// runtime error path is LOG(FATAL) (a worker failure the master recovers from); here the engine
// lives inside the user's process, so kernels facing bad DATA (an undecodable image, a raising
// host-language kernel) report it and return normally -- still producing one element per row, null
// where they have nothing -- and the evaluate loop ends the run with the message.  Call it from the
// thread that runs execute() / new_stream() / reset().
void report_kernel_error(const std::string& message);

class VideoKernel {
 protected:
  void check_frame(const DeviceHandle& device, const Element& element);
  void check_frame_info(const DeviceHandle& device, const Element& element);
  virtual void new_frame_info() {}
  virtual ~VideoKernel() {}

  FrameInfo frame_info_{};
};

// What REGISTER_KERNEL(...) accumulates: one implementation of an op for one device type.
using KernelConstructor = std::function<BaseKernel*(const KernelConfig& config)>;
struct KernelDeclaration {
  std::string op_name;
  KernelConstructor make;
  DeviceType device = DeviceType::CPU;
  i32 max_devices = 1;
  bool batches = false;           // .batch() was called
  i32 batch_size = 1;             // preferred rows per execute() when the graph does not say
  // columns that live on another device type than the kernel (e.g. encoded bytes for a GPU decoder)
  std::map<std::string, DeviceType> input_devices, output_devices;
  // frame columns the kernel also accepts in a non-HWC layout (an addition to the reference's API: decoder-native NV12)
  std::map<std::string, FrameLayout> input_layouts;
};

namespace internal {

using ::scanner::KernelConstructor;

class KernelBuilder {
 public:
  KernelBuilder(const std::string& op_name, KernelConstructor make) {
    decl_.op_name = op_name;
    decl_.make = std::move(make);
  }
  KernelBuilder& device(DeviceType type) {
    decl_.device = type;
    return *this;
  }
  KernelBuilder& num_devices(i32 n) {
    decl_.max_devices = n;
    return *this;
  }
  KernelBuilder& batch(i32 preferred_batch_size = 1) {
    decl_.batches = true;
    decl_.batch_size = preferred_batch_size;
    return *this;
  }
  KernelBuilder& input_device(const std::string& column, DeviceType type) {
    decl_.input_devices[column] = type;
    return *this;
  }
  KernelBuilder& output_device(const std::string& column, DeviceType type) {
    decl_.output_devices[column] = type;
    return *this;
  }
  KernelBuilder& input_layout(const std::string& column, FrameLayout layout) {
    decl_.input_layouts[column] = layout;
    return *this;
  }
  const KernelDeclaration& declaration() const { return decl_; }

 private:
  KernelDeclaration decl_;
};

// Constructing one files the kernel with the registry under (op name, device type) (registry.cpp).
struct KernelRegistration {
  KernelRegistration(const KernelBuilder& builder);
};

}  // namespace internal

#define SCN_KERNEL_PASTE2(a__, b__) a__##b__
#define SCN_KERNEL_PASTE(a__, b__) SCN_KERNEL_PASTE2(a__, b__)
// REGISTER_KERNEL(Op, Class).device(...).batch(...): Class must be constructible from a KernelConfig.
#define REGISTER_KERNEL(op__, class__)                                                                        \
  static const ::scanner::internal::KernelRegistration SCN_KERNEL_PASTE(scn_registered_kernel_, __COUNTER__) \
      __attribute__((unused)) = ::scanner::internal::KernelBuilder(                                           \
          #op__, [](const ::scanner::KernelConfig& config) -> ::scanner::BaseKernel* { return new class__(config); })

}  // namespace scanner
