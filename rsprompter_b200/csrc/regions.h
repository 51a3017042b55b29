#pragma once
#include "host_util.h"

namespace rsp {

// SAM's remove_small_regions on bit-packed masks (rsp_mask_small_regions_bits in include/rsp_b200.h).
// mode 0 = holes, 1 = islands; ws: n * (32 + 4 * ceil(H / 2) * ceil(W / 2)) bytes, 8-byte aligned.
int mask_small_regions_bits(const unsigned char* in, unsigned char* out, int n, int H, int W, int ld,
                            long long min_area, int mode, void* ws, unsigned char* changed, int* boxes,
                            cudaStream_t stream);

}  // namespace rsp
