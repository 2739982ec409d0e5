// C entry point over the reference's OWN H.264 byte-stream index creator -- test infrastructure.
// oracle/Makefile compiles this with the reference's scanner/video/h264_byte_stream_index_creator.cpp (unmodified; it
// parses with the reference's scanner/util/h264.h) into oracle/_ref/libref_h264_index.so.
// tests/test_reference_h264_index_cpu.py feeds it the access units of the synthetic streams and compares frame count,
// key pictures and sample sizes with this repo's indexer (scanner_b200/csrc/engine/h264.cpp).
#include <cstring>

#include "scanner/video/h264_byte_stream_index_creator.h"

// packets: n access units, unit i = data[offsets[i] .. offsets[i] + sizes[i]).  Outputs (caller-sized, cap entries):
// sample_offsets / sample_sizes per frame, keyframe indices; *n_frames, *n_key; the demuxed byte stream the reference
// would store goes to stream_out (cap stream_cap), its length to *stream_len.  Returns 0, -1 on a parse error (err).
extern "C" int ref_h264_index(const unsigned char* data, const unsigned long* offsets, const unsigned long* sizes, int n,
                              unsigned long* sample_offsets, unsigned long* sample_sizes, unsigned long* keyframes,
                              int cap, int* n_frames, int* n_key, unsigned char* stream_out, unsigned long stream_cap,
                              unsigned long* stream_len, char* err, int err_cap) {
  storehouse::WriteFile file;
  scanner::internal::H264ByteStreamIndexCreator ic(&file);
  for (int i = 0; i < n; ++i) {
    std::vector<scanner::u8> pkt(data + offsets[i], data + offsets[i] + sizes[i]);
    pkt.resize(pkt.size() + 8, 0);  // the parser looks a few bytes past a NAL's end (nal_start + nal_size + 3)
    if (!ic.feed_packet(pkt.data(), sizes[i])) {
      if (err && err_cap > 0) {
        strncpy(err, ic.error_message().c_str(), (size_t)err_cap - 1);
        err[err_cap - 1] = 0;
      }
      return -1;
    }
  }
  *n_frames = ic.frames();
  *n_key = (int)ic.keyframe_indices().size();
  if (ic.frames() > cap || *n_key > cap || file.bytes.size() > stream_cap) return -2;
  for (int i = 0; i < ic.frames(); ++i) {
    sample_offsets[i] = ic.sample_offsets()[(size_t)i];
    sample_sizes[i] = ic.sample_sizes()[(size_t)i];
  }
  for (int i = 0; i < *n_key; ++i) keyframes[i] = ic.keyframe_indices()[(size_t)i];
  memcpy(stream_out, file.bytes.data(), file.bytes.size());
  *stream_len = file.bytes.size();
  return 0;
}
