// nvdec.h -- the hardware H.264 decode stage: one NVCUVID parser + decoder session that turns the
// encoded samples of a keyframe interval into NV12 surfaces on the session's CUDA stream.
// Replaces reference scanner/video/nvidia/nvidia_video_decoder.cpp:92-374 (which upstream
// hard-disables, evaluate_worker.cpp:90-93) and the feeder/retriever threads of
// scanner/video/decoder_automata.cpp:104-351.
//
// Design (H100: 7 NVDEC engines per GPU, cuvidGetDecoderCaps at run time):
//  * libnvcuvid / libcuda are resolved with dlopen at first use -- no SDK headers or link-time
//    stubs; the handful of driver structs used are declared in nvdec.cpp from the public ABI.
//  * No threads, no polling: cuvidParseVideoData runs its callbacks synchronously, so feeding a
//    sample and consuming the pictures it completes is one call.  Pictures whose frame index is
//    not wanted are never mapped (the reference maps, converts and discards them).
//  * A wanted picture is mapped with CUVIDPROCPARAMS.output_stream = the session stream, handed
//    to the consumer callback (which enqueues NV12->RGB or the fused histogram/resize kernels on
//    that stream), and unmapped only after a CUDA event recorded behind the consumer completes --
//    up to kMaxMapped surfaces in flight, no cudaDeviceSynchronize per frame (reference :297).
//  * Many sessions per GPU (one per pipeline instance) keep all NVDEC engines busy.
//  * A GPU that exposes no NVDEC engine to the process (a container started without the driver's video
//    capability: cuvidGetDecoderCaps fails) still decodes: the session runs FFmpeg's H.264 decoder on the host
//    (swdec.h, as the reference's pipelines do), uploads each wanted picture's NV12 planes on the session stream
//    and hands the consumer the same surface layout.  H.264 decoding is bit-exact, so the pictures are the ones
//    NVDEC would deliver.  software() says which decoder a session uses; the engine reports it per instance.
#pragma once
#include <functional>
#include <memory>
#include <vector>

#include "scanner/util/common.h"

namespace scanner {
namespace internal {

struct NvdecCaps {
  bool available = false;
  bool h264_supported = false;
  int num_engines = 0;
  int max_width = 0, max_height = 0, min_width = 0, min_height = 0;
  std::string error;
};

// Probes driver libraries + cuvidGetDecoderCaps on `gpu_id` (cached per GPU).
const NvdecCaps& nvdec_caps(int gpu_id);

// One mapped decoder surface: luma rows then interleaved CbCr rows, `pitch` bytes apart.
struct Nv12Surface {
  const u8* luma;
  const u8* chroma;
  size_t pitch;
  i32 width, height;  // display size
};

// cumulative host nanoseconds inside driver calls since process start:
// parse (whole cuvidParseVideoData), decode_picture, map, consumer, release wait, create decoder
void nvdec_host_ns(long long out[6]);

class NvdecSession {
 public:
  // consumer(frame_index_in_request_order, surface): enqueue work reading the surface on
  // `stream`; must not synchronise.
  using Consumer = std::function<void(i64, const Nv12Surface&)>;

  NvdecSession(int gpu_id, void* stream);
  ~NvdecSession();
  Result init();

  // Start a keyframe interval.
  //   data/offsets/sizes: the encoded samples of the interval, the first one an IDR (copied
  //   by reference: must stay valid until end_interval);
  //   prefix: SPS/PPS bytes sent before the first sample (may be empty);
  //   may_reorder: the stream may display pictures in another order than it codes them (B
  //   pictures; H264Index::may_reorder).  Display position k can then depend on samples after the
  //   k-th, so samples are fed until the wanted pictures have come out (at most to the end of the
  //   interval) instead of stopping at the last wanted position;
  //   wanted: ascending 0-based positions (display order, relative to the first sample) of the
  //   pictures to deliver; delivered picture k is passed to `consumer` as index out_base + k;
  //   width / height: the picture size the stream index announces.
  Result begin_interval(const u8* data, const std::vector<u64>& offsets, const std::vector<u64>& sizes,
                        const std::vector<u8>& prefix, bool may_reorder, const std::vector<i64>& wanted,
                        i64 out_base, int width, int height, Consumer consumer);
  // Feed samples until at least `count` of the wanted pictures have been delivered (the decoder
  // may deliver more); flushes at the end of the interval.
  Result advance(size_t count);
  size_t delivered() const;
  // Flush, verify every wanted picture was delivered, forget the interval.
  Result end_interval();

  // Wait until every surface handed to a consumer has been released.
  void drain();

  i64 frames_decoded() const { return frames_decoded_; }
  i64 frames_used() const { return frames_used_; }
  // true: no NVDEC engine on this GPU, the session decodes with FFmpeg on the host
  bool software() const;
  // host nanoseconds this session has spent feeding samples (cuvidParseVideoData with its decode /
  // map callbacks: waiting for the NVDEC engine); frames_decoded / busy = the session's picture rate
  i64 busy_ns() const { return busy_ns_; }

  struct Impl;

 private:
  std::unique_ptr<Impl> impl_;
  i64 frames_decoded_ = 0, frames_used_ = 0, busy_ns_ = 0;
};

}  // namespace internal
}  // namespace scanner
