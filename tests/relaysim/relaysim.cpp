// relaysim.cpp -- TEST-ONLY host build of what snapgpu_index_save_ex writes (snap_b200/csrc/sg_bucket.h, sg_host.h): buckets re-laid
// into the reference's tables of any key size, default or -large, and the Genome, GenomeIndexHash and GenomeIndex writers.  Built into
// tests/_build/ by tests/relaysim_lib.py; never loaded by the snap_b200 package.
#include <string>
#include <vector>
#include <stdio.h>
#include <string.h>
#include "../../snap_b200/csrc/sg_align.h"
#include "../../snap_b200/csrc/sg_host.h"

static std::string g_err;

extern "C" {

const char *rs_last_error(void) { return g_err.c_str(); }

// a reference-format directory loaded on the host (sg_load_index_directory); relayout != 0: switched to sector buckets
void *rs_index_open(const char *dir, int relayout)
{
    SgHostIndex *ix = new SgHostIndex;
    if (!sg_load_index_directory(dir, *ix, g_err) || (relayout && !sg_host_relayout(*ix, sg_bucket_default_load(), g_err))) { delete ix; return NULL; }
    return ix;
}

void rs_index_close(void *v) { delete (SgHostIndex *)v; }

// Writes the Genome file from the index's contig lines and bases (sg_genome_file_header + the bases)
int rs_write_genome(void *v, const char *path)
{
    const SgHostIndex &h = *(SgHostIndex *)v;
    FILE *f = fopen(path, "wb");
    if (!f) { g_err = "cannot write " + std::string(path); return 1; }
    const std::string head = sg_genome_file_header(h.nBases, h.contigLines);
    fwrite(head.data(), 1, head.size(), f);
    fwrite(h.basesPadded.data() + SG_N_PADDING, 1, (size_t)h.nBases, f);
    fclose(f);
    return 0;
}

// Writes a bucket-layout index as a reference-format directory in the given table geometry, as snapgpu_index_save_ex does on the
// device: tables sized from their exact entry counts (sg_host_relay_count, sg_table_slots), re-laid (sg_host_relay_tables), the
// overflow table as it is.
int rs_relay_save(void *v, const char *dir, uint32_t keyBytes, uint32_t large, double slack)
{
    const SgHostIndex &h = *(SgHostIndex *)v;
    std::vector<uint64_t> used, size;
    std::vector<uint8_t> packed;
    if (!sg_host_relay_count(h, keyBytes, large, used, g_err)) return 1;
    for (size_t t = 0; t < used.size(); t++) size.push_back(sg_table_slots(used[t], slack));
    if (!sg_host_relay_tables(h, keyBytes, large, size, packed, g_err)) return 1;
    const std::string d(dir);
    if (rs_write_genome(v, (d + "/Genome").c_str())) return 1;
    FILE *f = fopen((d + "/OverflowTable").c_str(), "wb");
    if (!f) { g_err = "cannot write OverflowTable"; return 1; }
    fwrite(h.overflow.data(), 4, (size_t)h.overflowSize, f);
    fclose(f);
    f = fopen((d + "/GenomeIndexHash").c_str(), "wb");
    if (!f) { g_err = "cannot write GenomeIndexHash"; return 1; }
    uint64_t hashBytes = 0, off = 0;
    const uint32_t fb = sg_relay_file_bytes(keyBytes, large);
    for (size_t t = 0; t < used.size(); t++) {
        uint8_t head[36];
        sg_table_header(head, size[t], used[t], keyBytes, large, h.invalidValue);
        fwrite(head, 1, 36, f);
        fwrite(packed.data() + off, 1, (size_t)size[t] * fb, f);
        off += (size_t)size[t] * fb;
        hashBytes += 36 + (uint64_t)size[t] * fb;
    }
    fclose(f);
    f = fopen((d + "/GenomeIndex").c_str(), "w");
    if (!f) { g_err = "cannot write GenomeIndex"; return 1; }
    fputs(sg_genome_index_text((uint32_t)used.size(), h.overflowSize, h.seedLen, h.chromosomePadding, keyBytes, hashBytes, large).c_str(), f);
    fclose(f);
    return 0;
}

}
