// resize_plan.cuh -- layout of a Resize plan (scn_resize_plan_fill): a PlanHeader, then dst_w column taps, then
// dst_h row taps.  resize.cu fills it on the host; the Resize kernels of resize.cu and fused.cu read the taps.
#pragma once
#include <stdint.h>

namespace scn {

struct PlanHeader {
  int32_t magic, src_w, src_h, dst_w, dst_h, area2x, pad0, pad1;
};
// One tap entry per destination column / row: {src index 0, src index 1, weight 0, weight 1}
struct Tap {
  int32_t i0, i1, w0, w1;
};
static_assert(sizeof(PlanHeader) == 32, "the taps behind the header stay 16-byte aligned");
static_assert(sizeof(Tap) == 16, "the kernels read a tap as one int4");

}  // namespace scn
