/*
 * scn_kernels.h -- C-ABI kernel layer of scanner-b200 (libscn_kernels.so).
 *
 * The thin layer the C++ host pipeline (and any foreign binding: ctypes, cgo, JNI ...) calls
 * to run the per-frame pixel ops of Scanner's decode->evaluate->save hot path on an H100.
 * Plain pointers and sizes only -- no torch, no C++ types.  Each entry point names the
 * reference interface it replaces (paths relative to scanner-research/scanner @ 04a0c4b).
 *
 * Conventions
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Every call
 *     only ENQUEUES work on that stream and returns; nothing synchronises, nothing allocates
 *     (except scn_jpeg_encode_u8, whose output size depends on the data: see there).
 *   - Pointers are DEVICE pointers on the current CUDA device unless the parameter name
 *     starts with `host_`.  `host_*_ptrs` arrays are read synchronously during the call
 *     (they are copied into the kernel's launch parameters) and may be freed on return.
 *   - Frames are dense HWC, no row padding, exactly Scanner's `Frame` layout
 *     (scanner/api/frame.h:34-82: shape = {H, W, C}, u8* data).
 *   - Return value: 0 on success, a positive cudaError_t from the launch, or a negative
 *     SCN_E_* for bad arguments.  Never throws, never aborts.
 *   - There is NO CPU fallback: on a box without a usable CUDA device every launch returns
 *     the CUDA error.
 */
#ifndef SCN_KERNELS_H_
#define SCN_KERNELS_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define SCN_API __attribute__((visibility("default")))
#else
#define SCN_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define SCN_E_BADARG (-1)
#define SCN_E_UNSUPPORTED (-2)
#define SCN_E_PLAN (-3)

/* Library/ABI version (bumped on any signature change). */
SCN_API int scn_abi_version(void);

/* Number of kernels this library has launched since load (all streams, this process).
 * bench.py reports it as `gpu_launches`. */
SCN_API uint64_t scn_launch_count(void);

/* Per-kernel device timing (CUDA events recorded on the launch stream around every kernel this
 * library launches).  Off by default; bench.py turns it on for the roofline leg only.
 *   scn_prof_enable(1|0)  start / stop recording (resets the records when turned on)
 *   scn_prof_report(buf, cap)  synchronises the recorded events and writes a JSON object
 *       {"<kernel>": {"launches": n, "ms": total_ms}, ...}; returns the length written
 *       (0 if nothing was recorded, negative on error). */
SCN_API void scn_prof_enable(int on);
SCN_API int scn_prof_report(char* host_buf, size_t cap);

/* ---------------------------------------------------------------------------------------
 * Histogram  (replaces HistogramKernelCPU::execute, tests/test_ops.cpp:19-49:
 *             cv::calcHist 16 bins x 3 channels, CV_32S, channel-major)
 * For each of `n` u8 HWC 3-channel frames writes int32[3][16] (192 bytes) to out + i*48.
 * `out` is fully overwritten (no pre-zeroing needed).  n may be 0.  Bit-exact.
 */
SCN_API int scn_hist16_u8c3(const uint8_t* const* host_frame_ptrs, int n, int width, int height,
                    int32_t* out, void* stream);
/* Same, frames at base + i*stride_bytes (a block from new_block_buffer_size,
 * scanner/util/memory.h:59-62). */
SCN_API int scn_hist16_u8c3_strided(const uint8_t* base, size_t stride_bytes, int n, int width,
                            int height, int32_t* out, void* stream);

/* ---------------------------------------------------------------------------------------
 * Resize  (replaces ResizeKernel::execute, tests/test_ops.cpp:124-162: cv::resize(img, out,
 *          Size(w,h)) == INTER_LINEAR on CV_8UC3, OpenCV's 11-bit fixed-point path,
 *          including its exact-2x INTER_AREA re-route).  Bit-exact vs cv2.resize.
 *
 * scn_resize_target: the output size rule of test_ops.cpp:126-147 (ResizeArgs width, height,
 * min, preserve_aspect; `interpolation` is ignored by the reference).
 *
 * A "plan" is the per-(src size, dst size) coefficient table (x/y tap offsets and 11-bit
 * weights).  The caller owns its storage: ask for the size, fill it on the host, copy it to the
 * device once, pass the device copy to every launch with those sizes.  A destination of more
 * than INT_MAX pixels returns SCN_E_BADARG (here and in scn_nv12_hist_resize) before any launch.
 */
SCN_API void scn_resize_target(int src_w, int src_h, int arg_w, int arg_h, int arg_min,
                       int arg_preserve_aspect, int* out_w, int* out_h);
SCN_API size_t scn_resize_plan_bytes(int dst_w, int dst_h);
SCN_API int scn_resize_plan_fill(int src_w, int src_h, int dst_w, int dst_h, void* host_plan);
SCN_API int scn_resize_bilinear_u8c3(const uint8_t* const* host_src_ptrs, int n, int src_w, int src_h,
                             uint8_t* const* host_dst_ptrs, int dst_w, int dst_h,
                             const void* plan, void* stream);
SCN_API int scn_resize_bilinear_u8c3_strided(const uint8_t* src, size_t src_stride, int n, int src_w,
                                     int src_h, uint8_t* dst, size_t dst_stride, int dst_w,
                                     int dst_h, const void* plan, void* stream);

/* ---------------------------------------------------------------------------------------
 * Blur  (replaces BlurKernel::execute, tests/test_ops.cpp:265-294: integer box filter of
 *        BlurArgs.kernel_size, interior pixels only; sigma is unused by the reference).
 * Border pixels (which the reference leaves uninitialised) are written as 0.
 * kernel_size in [1, 31].  Bit-exact on the interior.
 */
SCN_API int scn_box_blur_u8c3(const uint8_t* const* host_src_ptrs, int n, int width, int height,
                      int kernel_size, uint8_t* const* host_dst_ptrs, void* stream);
SCN_API int scn_box_blur_u8c3_strided(const uint8_t* src, size_t stride_bytes, int n, int width,
                              int height, int kernel_size, uint8_t* dst, void* stream);

/* ---------------------------------------------------------------------------------------
 * NV12 -> RGB24  (replaces convertNV12toRGBA, scanner/util/image.cu:229-239 and its kernel
 *                 :109-200; called from NVIDIAVideoDecoder::get_frame,
 *                 scanner/video/nvidia/nvidia_video_decoder.cpp:288-296)
 * One decoder surface per frame: luma plane `pitch` x height, interleaved CbCr plane
 * `pitch` x height/2.  width and height must be even.  Output dense RGB24 (rgb_pitch >= 3*w).
 * Bit-exact vs the reference arithmetic (float matrix, clamp, truncate, >>2).
 */
SCN_API int scn_nv12_to_rgb24(const uint8_t* const* host_luma_ptrs,
                      const uint8_t* const* host_chroma_ptrs, size_t pitch, int n, int width,
                      int height, uint8_t* const* host_rgb_ptrs, size_t rgb_pitch,
                      void* stream);

/* Pitched decoder surface -> packed NV12 frame element: `width` x `height` luma rows followed by
 * `width` x height/2 interleaved CbCr rows, no padding (the FrameLayout::NV12 element of
 * include/scanner/api/frame.h; what the decode stage hands to kernels that registered for it
 * instead of the RGB24 frame of nvidia_video_decoder.cpp:288-296).  Byte copy. */
SCN_API int scn_nv12_pack(const uint8_t* const* host_luma_ptrs, const uint8_t* const* host_chroma_ptrs,
                          size_t pitch, int n, int width, int height, uint8_t* const* host_dst_ptrs,
                          void* stream);

/* ---------------------------------------------------------------------------------------
 * Fused decode-side DAG of BASELINE.json configs[1]:
 *      NV12 surface -> RGB24 -> { Histogram , Resize(dst_w, dst_h) }
 * without materialising the RGB24 frame (what the reference does in three passes:
 * image.cu NV12_to_RGB, then test_ops.cpp Histogram and Resize kernels over the RGB frame).
 * hist_out: int32[n][3][16] (fully overwritten; NULL skips the histogram); resized: n dense RGB24
 * dst_h x dst_w frames at host_dst_ptrs[i] (NULL skips the resize) -- so the same entry point is
 * also "Histogram on an NV12 frame" and "Resize on an NV12 frame".  Results are bit-identical to
 * running scn_nv12_to_rgb24 + scn_hist16_u8c3 + scn_resize_bilinear_u8c3.
 */
SCN_API int scn_nv12_hist_resize(const uint8_t* const* host_luma_ptrs,
                         const uint8_t* const* host_chroma_ptrs, size_t pitch, int n,
                         int width, int height, int32_t* hist_out,
                         uint8_t* const* host_dst_ptrs, int dst_w, int dst_h, const void* plan,
                         void* stream);

/* ---------------------------------------------------------------------------------------
 * ConvertColor  (replaces scannertools' ConvertColor kernel: cv::cvtColor(frame, out, code) on
 *                CV_8U frames).  Bit-exact vs cv2.cvtColor.  Codes, numbered in this order:
 *   0 COLOR_RGB2GRAY      1 COLOR_BGR2GRAY        HxWx3 -> HxWx1
 *   2 COLOR_RGB2YCrCb     3 COLOR_BGR2YCrCb       HxWx3 -> HxWx3
 *   4 COLOR_RGB2HSV       5 COLOR_BGR2HSV         HxWx3 -> HxWx3 (hue 0..179)
 *   6 COLOR_RGB2HSV_FULL  7 COLOR_BGR2HSV_FULL    HxWx3 -> HxWx3 (hue 0..255)
 *   8 COLOR_RGB2BGR       9 COLOR_BGR2RGB         HxWx3 -> HxWx3
 *  10 COLOR_GRAY2RGB     11 COLOR_GRAY2BGR        HxWx1 -> HxWx3
 * scn_convert_color_code: the code of an OpenCV name, SCN_E_UNSUPPORTED for any other name.
 * scn_convert_color_name: the name of a code, NULL past the last one.
 * scn_convert_color_channels: a code's input and output channel counts.
 * scn_convert_color_u8: n dense frames of the code's input channels -> n dense frames of its output
 *   channels, any alignment.  Pointer list; batches over 64 frames are split into launches.
 * scn_convert_color_nv12: n NV12 surfaces (as scn_nv12_to_rgb24 takes them) converted to RGB24 with the
 *   reference's arithmetic and then by `code`, without writing the RGB24 frame; identical to
 *   scn_nv12_to_rgb24 followed by scn_convert_color_u8.  GRAY2* codes are SCN_E_BADARG here.
 */
SCN_API int scn_convert_color_code(const char* name);
SCN_API const char* scn_convert_color_name(int code);
SCN_API int scn_convert_color_channels(int code, int* in_channels, int* out_channels);
SCN_API int scn_convert_color_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int code,
                                 uint8_t* const* host_dst_ptrs, void* stream);
SCN_API int scn_convert_color_nv12(const uint8_t* const* host_luma_ptrs, const uint8_t* const* host_chroma_ptrs,
                                   size_t pitch, int n, int width, int height, int code,
                                   uint8_t* const* host_dst_ptrs, void* stream);

/* ---------------------------------------------------------------------------------------
 * JPEG  (the GPU kernel of the ImageEncoder op with format "jpg": upstream, scannertools encoded
 *        with cv::imencode(".jpg")).  Byte for byte what cv2.imencode('.jpg', frame, [IMWRITE_JPEG_QUALITY,
 *        quality]) writes with cv2's libjpeg defaults: baseline JFIF, 4:2:0 for three channels, Annex K
 *        Huffman tables, no restart markers.
 * scn_jpeg_encode_u8: n dense u8 frames of one geometry, `channels` 3 (RGB, as the pipeline stores them;
 *   cv2 would be given the BGR frame) or 1 (gray), any base alignment -> n complete JFIF files.  Quality
 *   1-100.  Pointer list; batches over 64 frames are split into launches.
 *   Unlike the rest of this header the call synchronises `stream` twice (it reads back each frame's bit count
 *   to size its scratch, then each frame's 0xFF count to size the output) and allocates its device scratch
 *   from a stream-ordered pool the library keeps per device.  When the sizes are known it calls
 *   alloc_out(alloc_ctx, total) once for a device buffer of `total` bytes, writes host_sizes[0..n), and
 *   enqueues the files into that buffer back to back (file i at the sum of the sizes before it); they are
 *   ready in stream order when the call returns.  A null alloc_out result returns SCN_E_ALLOC.
 *   channels other than 1 and 3, or a side over 65,500 (libjpeg's JPEG_MAX_DIMENSION): SCN_E_UNSUPPORTED.
 * scn_jpeg_encode_bound: bytes no file of that geometry exceeds at any quality (0 for an unsupported
 *   geometry): the header, every block at its longest code (26 bits per AC coefficient, 22 for the DC),
 *   every byte stuffed, and the EOI.
 */
#define SCN_E_ALLOC (-4)
typedef void* (*scn_alloc_fn)(void* ctx, size_t bytes);
SCN_API size_t scn_jpeg_encode_bound(int width, int height, int channels);
SCN_API int scn_jpeg_encode_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int channels,
                               int quality, scn_alloc_fn alloc_out, void* alloc_ctx, size_t* host_sizes,
                               void* stream);

/* ---------------------------------------------------------------------------------------
 * H.264  (the save stage's video encoder: upstream, compress_video() outputs went through libavcodec).
 *        Intra-only Baseline H.264 with CAVLC, every macroblock Intra16x16, constant QP, one slice per
 *        picture, deblocking off.  oracle/h264_enc.py is the same encoder in integer numpy and documents every
 *        decision (colour conversion, mode choice, quantisation); the output is byte for byte the oracle's.
 * scn_h264_encode_u8: n dense RGB24 frames of one geometry, any base alignment -> n Annex-B access units.
 *   positions[i] is frame i's position within its item (null: 0, 1, ..., n - 1): position p is an IDR
 *   picture, with SPS and PPS in its access unit, when p % keyframe_distance == 0, and a non-IDR I picture
 *   with frame_num (p % keyframe_distance) % 16 otherwise.  QP 0-51, keyframe_distance >= 1, positions >= 0,
 *   else SCN_E_BADARG.  An odd width or height, a side over 4096 or more than 36,864 macroblocks (level
 *   5.1's MaxFS): SCN_E_UNSUPPORTED.  Pointer list; batches over 64 frames are split into launches.
 *   Scratch, the output callback, host_sizes and the two stream synchronisations are as in
 *   scn_jpeg_encode_u8: access unit i is at the sum of the sizes before it in the buffer alloc_out returned.
 * scn_h264_encode_bound: bytes no access unit of that geometry exceeds at any QP (0 for a geometry
 *   scn_h264_encode_u8 refuses).
 */
SCN_API size_t scn_h264_encode_bound(int width, int height);
SCN_API int scn_h264_encode_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int qp,
                               const int* host_positions, int keyframe_distance, scn_alloc_fn alloc_out,
                               void* alloc_ctx, size_t* host_sizes, void* stream);

/* ---------------------------------------------------------------------------------------
 * OpticalFlow  (replaces OpticalFlowKernelCPU::execute, tests/test_ops.cpp:79-98:
 *   cvtColor(COLOR_BGR2GRAY) on each RGB frame of the {0,1} stencil window, then
 *   cv::FarnebackOpticalFlow(numLevels, pyrScale, fastPyramids=false, winSize, numIters, polyN,
 *   polySigma, flags=0)->calc; the reference constructs it with (3, 0.5, 15, 3, 5, 1.2), :68-69)
 * For each of n frame pairs writes a dense flow field float32[H][W][2] (dx, dy) to
 * host_flow_ptrs[i].  Floating point: matches cv2.calcOpticalFlowFarneback within a tolerance
 * (max |d| <= 2e-3 px, mean <= 1e-4 px on well-conditioned input), not bit-exact.  That holds over the
 * supported range, not only at the reference's arguments: tests/test_flow_params_gpu.py checks it for
 * num_levels 0-8, pyr_scale 0.3-0.8, win_size 2-21, num_iters 1-6, poly_n 1-7 and frames from 1 x 1 up.
 * Two kinds of pixel can lie further off: windows too small to condition the 2x2 solve (win_size 2), and
 * a pixel whose warped position lands within float rounding of the frame edge, where UpdateMatrices
 * switches branch (one window footprint in that test's 1080p case).
 * Supported: win_size >= 2, 1 <= poly_n <= 7, poly_sigma > 0, 0 <= num_levels <= 15,
 * 0 < pyr_scale < 1, num_iters >= 1.  Anything else returns SCN_E_BADARG.  win_size 1 is refused
 * because OpenCV's window-sum code does not compute a 1 x 1 box there, so no result could match cv2.
 * A pyramid level whose Gaussian needs more than 65 taps returns SCN_E_UNSUPPORTED before any launch
 * (ksize = max(3, lrint(5 sigma) | 1) with sigma = (1 / pyr_scale^k - 1) / 2: num_levels <= 4 at
 * pyr_scale 0.5; levels that the 32-pixel minimum cuts off do not count).
 * `workspace` is caller-owned device scratch of scn_farneback_workspace_bytes(w, h) bytes,
 * reusable across calls on the same stream.
 */
SCN_API size_t scn_farneback_workspace_bytes(int width, int height);
SCN_API int scn_farneback_u8c3(const uint8_t* const* host_prev_ptrs, const uint8_t* const* host_next_ptrs,
                               int n, int width, int height, float* const* host_flow_ptrs, int num_levels,
                               double pyr_scale, int win_size, int num_iters, int poly_n, double poly_sigma,
                               void* workspace, size_t workspace_bytes, void* stream);
/* The same for a caller that walks a clip pair by pair and keeps the workspace between calls (the OpticalFlow op,
 * stencil [0, 1]: one pair per call).  Within a call, a pair whose `prev` pointer equals the previous pair's `next`
 * reuses that frame's pyramid of polynomial expansions (gray conversion, the full-resolution Gaussians, resizes and
 * expansions are per frame, about 40 % of a pair's work).  `chain` (host int owned by the caller with the workspace,
 * 0 initially and after anything else used the workspace) carries this over calls: with reuse_prev != 0 and
 * *chain != 0 the caller asserts that pair 0's `prev` frame has the content of the last call's last `next` frame (the
 * same table row), and it is not expanded again.  Results are identical to scn_farneback_u8c3's. */
SCN_API int scn_farneback_u8c3_chain(const uint8_t* const* host_prev_ptrs, const uint8_t* const* host_next_ptrs,
                                     int n, int width, int height, float* const* host_flow_ptrs, int num_levels,
                                     double pyr_scale, int win_size, int num_iters, int poly_n, double poly_sigma,
                                     void* workspace, size_t workspace_bytes, int reuse_prev, int* chain,
                                     void* stream);

/* ---------------------------------------------------------------------------------------
 * FrameDigest: a 16-byte fingerprint of each of n equally sized buffers (`bytes` a multiple of 4):
 *     out[2i]   = sum of the buffer's little-endian 32-bit words            (mod 2^64)
 *     out[2i+1] = sum of word[k] * (k mod 65521 + 1)                         (mod 2^64)
 * Exact integer arithmetic on the raw bytes: two runs agree iff (up to collisions) their buffers are
 * byte-identical.  No counterpart in the reference; it exists so that frame-valued results too large to
 * bring back (a 1080p flow field is 16.6 MB per row) can be compared between a run on one GPU and a run
 * sharded over several (bench.py --config 3, SURVEY 8d configs[3] "must be identical").  `out` is fully
 * overwritten. */
SCN_API int scn_frame_digest(const uint8_t* const* host_ptrs, int n, size_t bytes, uint64_t* out, void* stream);

/* ---------------------------------------------------------------------------------------
 * TV-L1 dense optical flow (no counterpart in the reference; DESIGN.md "TV-L1" is the specification): the
 * Zach-Pock-Bischof duality scheme of Sanchez Perez et al. (IPOL 2013) with OpenCV DualTVL1OpticalFlow's
 * parameter names and defaults (tau 0.25, lambda 0.15, theta 0.3, nscales 5, warps 5, epsilon 0.01,
 * iterations 300, scale_step 0.8, median_filtering 5), gamma = 0.
 * n pairs of dense u8 gray frames (prev_i, next_i), all width x height -> n float32 [height][width][2] flows
 * (dx, dy) with prev(x, y) ~ next(x + dx, y + dy).  Pointer lists; any n (batches over 64 pairs run in 64-pair
 * chunks).  Every (level, warp) step is one launch per kernel for all pairs of a chunk; the iterations of a
 * step run inside one cooperative kernel that decides each pair's stop on the device.  Nothing synchronises
 * with the host unless host_iterations is non-NULL: then it receives int [n][nscales][warps], level 0
 * (finest) first, the iterations each (pair, level, warp) ran (0 for levels the pyramid stops before), and
 * the call waits for the stream.  A pair's flow does not depend on the other pairs of the call (bit for bit).
 * Refused with SCN_E_BADARG before any launch: a non-finite float, tau, lambda or theta <= 0,
 * nscales outside 1-10, warps outside 1-20, iterations outside 1-10000, scale_step outside (0, 1),
 * median_filtering other than 1, 3, 5, a side under 2, n < 0, a null pointer list or workspace, or
 * workspace_bytes < scn_tvl1_workspace_bytes(width, height, n).  epsilon <= 0 disables the early stop.
 */
SCN_API size_t scn_tvl1_workspace_bytes(int width, int height, int n);
SCN_API int scn_tvl1_u8(const uint8_t* const* host_prev_ptrs, const uint8_t* const* host_next_ptrs, int n,
                        int width, int height, float* const* host_flow_ptrs, float tau, float lambda, float theta,
                        int nscales, int warps, float epsilon, int iterations, float scale_step,
                        int median_filtering, int* host_iterations, void* workspace, size_t workspace_bytes,
                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SCN_KERNELS_H_ */
