// Test-only: the host build of snap_b200/csrc/sg_spacing.h behind C entry points (tests/test_infer_spacing.py).
#include <math.h>
#include "../../snap_b200/csrc/sg_spacing.h"

extern "C" void host_spacing_range(const int64_t *sorted, int64_t w, int32_t *minSpacing, int32_t *maxSpacing)
{
    sg_spacing_range(sorted, w, minSpacing, maxSpacing);
}

extern "C" void host_spacing_samples(int64_t n, const snapgpu_paired_result *r, const uint8_t *useful, int32_t filterFlags, int32_t forceSpacing,
                                     int64_t *out)
{
    for (int64_t i = 0; i < n; i++) {
        const bool u[2] = {useful[2 * i] != 0, useful[2 * i + 1] != 0};
        out[i] = sg_spacing_sample(r[i], u, filterFlags, forceSpacing != 0, SNAPGPU_INVALID_LOCATION_32);
    }
}
