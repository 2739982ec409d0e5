// swdec.h -- the software H.264 decode stage of CPU pipeline instances (BASELINE configs[0]: "Histogram op on one
// 640x480 H.264 clip, CPU pipeline_instances=1").  Replaces reference
// scanner/video/software/software_video_decoder.cpp:38-330: libavcodec's H.264 decoder, pictures converted to packed
// RGB24 with libswscale (sws_getContext(..., AV_PIX_FMT_RGB24, SWS_BICUBIC), :188-192).
//
// Like the reference this IS FFmpeg -- but resolved at run time: libavcodec / libavutil / libswscale are opened with
// dlopen (no headers, no link-time dependency; the few public structs used are declared in swdec.cpp from their
// stable ABI prefixes and everything else goes through av_opt_set_int), from
//   SCN_FFMPEG_DIR   a directory holding the three libraries and their dependencies under any file names
//                    (scanner_b200/engine.py points it at the FFmpeg build that ships inside the image's
//                    opencv-python-headless wheel when the variable is unset), else
//   the system's libavcodec.so.{62..58} / libavutil / libswscale through the normal search path.
// Without them a CPU instance that is handed an H.264 source fails with an error that says so.  GPU instances decode
// with NVDEC (nvdec.h); on a GPU that exposes no NVDEC engine to the process their NvdecSession decodes here, to NV12.
//
// No frame pool / queue threads (reference :45-46): avcodec_send_packet / avcodec_receive_frame are called from the
// pipeline instance's own thread and every wanted picture is scaled straight into its element's memory.
#pragma once
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "scanner/util/common.h"

namespace scanner {
namespace internal {

struct SwdecCaps {
  bool available = false;
  int avcodec_major = 0, avutil_major = 0, swscale_major = 0;
  std::string where;  // the libavcodec file that was opened
  std::string error;
};
// Loads the libraries on first use (cached).
const SwdecCaps& swdec_caps();

class SwdecSession {
 public:
  // dest(out_index) -> where the packed RGB24 picture (width * height * 3 bytes, rows `width * 3` apart) goes; with
  // nv12 the packed NV12 picture (width * height luma bytes, then height / 2 rows of interleaved Cb Cr, rows `width`
  // apart: the decoded planes unconverted)
  using Dest = std::function<u8*(i64)>;

  explicit SwdecSession(int threads = 1, bool nv12 = false);
  ~SwdecSession();
  Result init();

  // Same contract as NvdecSession::begin_interval (nvdec.h): samples of one keyframe interval (Annex-B access
  // units, the first an IDR), SPS/PPS prefix, ascending wanted display positions; wanted picture k is written to
  // dest(out_base + k).  width / height: the picture size the stream index announces (a stream that decodes to
  // another size is an error, as in the NVDEC path).
  Result begin_interval(const u8* data, const std::vector<u64>& offsets, const std::vector<u64>& sizes,
                        const std::vector<u8>& prefix, bool may_reorder, const std::vector<i64>& wanted, i64 out_base,
                        int width, int height, Dest dest);
  Result advance(size_t count);
  size_t delivered() const;
  Result end_interval();

  i64 frames_decoded() const { return frames_decoded_; }
  i64 frames_used() const { return frames_used_; }

  struct Impl;

 private:
  std::unique_ptr<Impl> impl_;
  i64 frames_decoded_ = 0, frames_used_ = 0;
};

}  // namespace internal
}  // namespace scanner
