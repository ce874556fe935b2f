// buildsim.cpp -- TEST-ONLY host build of what the device index build and save rest on when they run in passes
// (snap_b200/csrc/sg_bucket.h, sg_host.h): the bucket mix and its inverse, sequential bucket insertion, the slot decode, re-laying
// buckets into the reference's tables, and the pass planner.  Built into tests/_build/ by tests/buildsim_lib.py; never loaded by the
// snap_b200 package.
#include <string>
#include <vector>
#include <string.h>
#include <stdlib.h>
#include "../../snap_b200/csrc/sg_align.h"
#include "../../snap_b200/csrc/sg_host.h"

struct BsIndex {
    SgHostIndex host;
    SgIndexView view;
};

static std::string g_err;

extern "C" {

const char *bs_last_error(void) { return g_err.c_str(); }

void *bs_index_open(const char *dir)
{
    BsIndex *ix = new BsIndex;
    if (!sg_load_index_directory(dir, ix->host, g_err)) { delete ix; return NULL; }
    ix->view = ix->host.view();
    return ix;
}

void bs_index_close(void *v) { delete (BsIndex *)v; }

// switches the index to the sector-bucket layout (sg_host_relayout)
int bs_index_relayout(void *v, double load)
{
    BsIndex *ix = (BsIndex *)v;
    if (!sg_host_relayout(ix->host, load > 0 ? load : sg_bucket_default_load(), g_err)) return 1;
    ix->view = ix->host.view();
    return 0;
}

// switches a bucket-layout index back to the reference's tables (its own table geometry), re-laid from the buckets
int bs_index_buckets_to_tables(void *v)
{
    BsIndex *ix = (BsIndex *)v;
    if (!sg_host_buckets_to_tables(ix->host, g_err)) return 1;
    ix->view = ix->host.view();
    return 0;
}

// per-table used counts (as loaded from the directory, or as recomputed by bs_index_buckets_to_tables); returns nTables
int64_t bs_index_table_used(void *v, uint64_t *used, int64_t cap)
{
    BsIndex *ix = (BsIndex *)v;
    for (int64_t t = 0; t < (int64_t)ix->host.tableUsed.size() && t < cap; t++) used[t] = ix->host.tableUsed[t];
    return (int64_t)ix->host.tableUsed.size();
}

// sg_lookup_seed32 of nSeeds seeds of seedLen bases each: hit counts [2 per seed] and up to maxHitsPerSeed hits per direction
void bs_lookup_seeds(void *v, const char *seeds, int64_t nSeeds, uint32_t maxHitsPerSeed, int64_t *nHits, uint32_t *hits)
{
    BsIndex *ix = (BsIndex *)v;
    const uint32_t sl = ix->host.seedLen;
    for (int64_t i = 0; i < nSeeds; i++) {
        uint64_t b, rc;
        nHits[2 * i] = nHits[2 * i + 1] = 0;
        uint32_t examined = 0, ow = 0;
        if (!sg_seed_pack((const uint8_t *)seeds + i * sl, sl, &b, &rc)) continue;
        SgHits h;
        sg_lookup_seed32(ix->view, b, rc, &h, &examined, &ow);
        for (int d = 0; d < 2; d++) {
            nHits[2 * i + d] = h.nHits[d];
            for (uint32_t k = 0; k < h.nHits[d] && k < maxHitsPerSeed; k++) hits[(2 * i + d) * (int64_t)maxHitsPerSeed + k] = h.hits[d][k];
        }
    }
}

uint64_t bs_bucket_count_for(uint64_t nEntries, uint32_t seedLen, double load) { return sg_bucket_count_for(nEntries, seedLen, load); }
uint64_t bs_bucket_min_count(uint32_t bits) { return sg_bucket_min_count(bits); }
uint64_t bs_bucket_mix(uint64_t c, uint32_t bits) { return sg_bucket_mix(c, bits); }
uint64_t bs_bucket_unmix(uint64_t h, uint32_t bits) { return sg_bucket_unmix(h, bits); }

int bs_bucket_insert_seq(uint64_t *buckets, uint64_t nBuckets, uint32_t bits, uint64_t canonical, uint32_t orient, uint32_t value)
{
    return sg_bucket_insert_seq(buckets, nBuckets, bits, canonical, orient, value) ? 1 : 0;
}

// sg_bucket_slot_decode of the slots slotIdx[0..n) of a bucket image: seeds[i], orients[i] (255: not decodable)
void bs_bucket_decode(const uint64_t *buckets, uint64_t nBuckets, uint32_t seedLen, const uint64_t *slotIdx, int64_t n, uint64_t *seeds, uint8_t *orients)
{
    for (int64_t i = 0; i < n; i++) {
        const uint64_t s = slotIdx[i];
        uint32_t o = 0;
        seeds[i] = 0;
        orients[i] = sg_bucket_slot_decode(buckets[s], s / SG_BUCKET_SLOTS, nBuckets, seedLen, &seeds[i], &o) ? (uint8_t)o : 255;
    }
}

// sg_plan_passes: returns the number of passes (bounds gets P + 1 edges, room for nBins + 1), or -1 with *badBin
int64_t bs_plan_passes(const uint64_t *binBytes, uint32_t nBins, uint64_t budget, uint32_t minPasses, uint32_t *bounds, uint32_t *badBin)
{
    std::vector<uint32_t> b;
    if (!sg_plan_passes(binBytes, nBins, budget, minPasses, b, badBin)) return -1;
    for (size_t i = 0; i < b.size(); i++) bounds[i] = b[i];
    return (int64_t)b.size() - 1;
}

}
