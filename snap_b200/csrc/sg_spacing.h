// sg_spacing.h -- insert-size inference of `snap paired -ins`: which pairs add a sample to the window, and the range a full
// window gives.  Host and device.  Reference: PairedAligner.cpp:822-925 (the per-pair tail) and :424-458 (computeSpacingDist).
//
// Stock keeps a window of W = 262144 samples per worker thread.  A pair that is not useless adds a sample when its primary
// record survives the filters (`firstIsPrimary`) and its ends point at each other (FORWARD/RC or RC/FORWARD); the sample is the
// absolute difference of the two locations, NotFound ends (InvalidGenomeLocation) included.  The pair that fills the window
// sets the intersecting aligner's range for the pairs after it.
#pragma once
#include "sg_common.h"             // sqrt: <math.h> on the host (included first by its users), the CUDA math library on the device

#define SG_SPACING_WINDOW 262144     // DEFAULT_BATCH_SIZE_IS_ESTIMATION, PairedAligner.h:32

// AlignerOptions::FilterFlags (AlignerOptions.h:174-181)
enum { SG_FILTER_UNALIGNED = 0x1, SG_FILTER_SINGLE_HIT = 0x2, SG_FILTER_MULTIPLE_HITS = 0x4, SG_FILTER_BOTH_MATES = 0x8,
       SG_FILTER_TOO_SHORT = 0x10 };

// AlignerOptions::passFilter (AlignerOptions.cpp:1061-1090) for a primary record (secondaryAlignment = false).
SG_HD bool sg_pass_filter(int32_t filterFlags, int32_t status, bool tooShort)
{
    if (filterFlags == 0) return true;
    if (tooShort) return (filterFlags & SG_FILTER_TOO_SHORT) != 0;
    switch (status) {
    case SNAPGPU_NOT_FOUND: return (filterFlags & SG_FILTER_UNALIGNED) != 0;
    case SNAPGPU_SINGLE_HIT: return (filterFlags & SG_FILTER_SINGLE_HIT) != 0;
    case SNAPGPU_MULTIPLE_HITS: return (filterFlags & SG_FILTER_MULTIPLE_HITS) != 0;
    default: return false;
    }
}

// The sample a pair adds, or -1 for none.  useful[w]: read w is long enough and has few enough Ns (a pair with neither useful
// never gets here in stock and adds none).  forceSpacing: -fs, whose fix-up (PairedAligner.cpp:822-830) turns an end that is not
// a single hit beside one that is into a NotFound pair; it keeps the directions.  invalidLocation: InvalidGenomeLocation.
SG_HD int64_t sg_spacing_sample(const snapgpu_paired_result &r, const bool useful[2], int32_t filterFlags, bool forceSpacing,
                                int64_t invalidLocation)
{
    if (!useful[0] && !useful[1]) return -1;
    int32_t status[2] = {r.status[0], r.status[1]};
    int64_t loc[2] = {r.location[0], r.location[1]};
    if (forceSpacing && (status[0] == SNAPGPU_SINGLE_HIT) != (status[1] == SNAPGPU_SINGLE_HIT)) {
        status[0] = status[1] = SNAPGPU_NOT_FOUND;
        loc[0] = loc[1] = invalidLocation;
    }
    const bool pass0 = sg_pass_filter(filterFlags, status[0], !useful[0]);
    const bool pass1 = sg_pass_filter(filterFlags, status[1], !useful[1]);
    const bool firstIsPrimary = (filterFlags & SG_FILTER_BOTH_MATES) ? (pass0 && pass1) : (pass0 || pass1);
    if (!firstIsPrimary || r.direction[0] == r.direction[1]) return -1;
    return loc[0] > loc[1] ? loc[0] - loc[1] : loc[1] - loc[0];     // DistanceBetweenGenomeLocations
}

// C's (int) of a double as x86-64 computes it (cvttsd2si): truncation, and 0x80000000 for NaN and for values out of range.
SG_HD int32_t sg_double_to_int(double v)
{
    if (!(v > -2147483649.0 && v < 2147483648.0)) return (int32_t)0x80000000u;
    return (int32_t)v;
}

// computeSpacingDist over a window of w samples sorted ascending: the new (minSpacing, maxSpacing).  The quartiles are at w/4 and
// 3w/4 as int(.25 * w) and int(.75 * w) give for the reference's w.  Sums are sequential doubles in sorted order, as stock's.
// The int conversions are stock's: int64 -> int keeps the low 32 bits, double -> int as sg_double_to_int.
SG_HD void sg_spacing_range(const int64_t *s, int64_t w, int32_t *minSpacing, int32_t *maxSpacing)
{
    const int64_t s25 = s[(int64_t)(0.25 * (double)w)], s75 = s[(int64_t)(0.75 * (double)w)];
    const int64_t iqr = s75 - s25;
    int32_t mn = (int32_t)(uint32_t)(uint64_t)(s25 - 2 * iqr > 1 ? s25 - 2 * iqr : 1);       // OUTLIER_BOUND
    int32_t mx = (int32_t)(uint32_t)(uint64_t)(s75 + 2 * iqr);
    double sum = 0;
    int count = 0;
    for (int64_t i = 0; i < w; i++) {
        if (s[i] >= mn && s[i] <= mx) { sum += (double)s[i]; count++; }
    }
    const double avg = sum / count;
    sum = 0;
    for (int64_t i = 0; i < w; i++) {
        if (s[i] >= mn && s[i] <= mx) { const double d = (double)s[i] - avg; sum += d * d; }
    }
    const double stddev = sqrt(sum / count);
    mn = (int32_t)(uint32_t)(uint64_t)(s25 - 3 * iqr);      // MAPPING_BOUND
    mx = (int32_t)(uint32_t)(uint64_t)(s75 + 3 * iqr);
    const double lo = avg - 4 * stddev, hi = avg + 4 * stddev;   // MAX_STDDEV
    mn = sg_double_to_int(lo < mn ? lo : (double)mn);       // __min(double, int) is a double
    mx = sg_double_to_int(hi > mx ? hi : (double)mx);
    *minSpacing = mn > 1 ? mn : 1;
    *maxSpacing = mx;
}
