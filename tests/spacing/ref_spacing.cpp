// Test-only: the reference's PairedAlignerContext::computeSpacingDist (a protected member) behind a C entry point.  Compiled
// against the reference headers under oracle/_ref/include and linked with oracle/_ref/libsnapref.so by tests/test_infer_spacing.py.
#include "stdafx.h"
#define protected public
#include "PairedAligner.h"
#undef protected
#include <stdlib.h>

extern "C" void ref_compute_spacing_dist(const long long *sorted, int *minSpacing, int *maxSpacing)
{
    // the method reads nothing of the object: raw storage of the right size stands in for a constructed context
    static PairedAlignerContext *ctx = (PairedAlignerContext *)calloc(1, sizeof(PairedAlignerContext));
    GenomeDistance *s = (GenomeDistance *)malloc(sizeof(GenomeDistance) * DEFAULT_BATCH_SIZE_IS_ESTIMATION);
    for (int i = 0; i < DEFAULT_BATCH_SIZE_IS_ESTIMATION; i++) s[i] = sorted[i];
    double avg, stddev;
    ctx->computeSpacingDist(s, minSpacing, maxSpacing, &avg, &stddev);
    free(s);
}
