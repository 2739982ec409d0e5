// resize_plan.cuh -- layout of a Resize plan, filled on the host (resize.cu, resize_interp.cu) and read by the Resize
// kernels of resize.cu, fused.cu and resize_interp.cu.  Every plan starts with a PlanHeader; `kind` says what follows:
//   kPlanLinearTaps  dst_w column Taps, then dst_h row Taps (scn_resize_plan_fill: INTER_LINEAR, and INTER_AREA when a
//                    scale is below 1, which is INTER_LINEAR's arithmetic with other taps)
//   kPlanNearest     int32 source column of each destination column [dst_w], then source row of each row [dst_h]
//   kPlanArea        int32 xofs[dst_w + 1], int32 yofs[dst_h + 1], padding to 8 bytes, AreaTap xtab[xofs[dst_w]],
//                    AreaTap ytab[yofs[dst_h]]: destination column d sums xtab[xofs[d] .. xofs[d + 1]), in order
//                    (INTER_AREA when both scales are >= 1)
#pragma once
#include <stdint.h>

namespace scn {

struct PlanHeader {
  int32_t magic, src_w, src_h, dst_w, dst_h, area2x, kind, pad1;
};
enum PlanKind { kPlanLinearTaps = 0, kPlanNearest = 1, kPlanArea = 2 };
// One tap entry per destination column / row: {src index 0, src index 1, weight 0, weight 1}
struct Tap {
  int32_t i0, i1, w0, w1;
};
// One INTER_AREA table entry: a source column (or row) and its float weight
struct AreaTap {
  int32_t s;
  float w;
};
static_assert(sizeof(PlanHeader) == 32, "the taps behind the header stay 16-byte aligned");
static_assert(sizeof(Tap) == 16, "the kernels read a tap as one int4");

// Fills a kPlanLinearTaps plan (scn_resize_plan_bytes(dst_w, dst_h) bytes) with INTER_LINEAR's taps or, with `area`,
// INTER_AREA's taps for a scale below 1.  resize.cu.
void fill_linear_plan(int src_w, int src_h, int dst_w, int dst_h, bool area, void* host_plan);

}  // namespace scn
