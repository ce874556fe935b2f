// sg_host.h -- host-side C++: reading a SNAP index directory (format v7.1), probability tables, parameter
// derivation.  Header-only; used by the CUDA library and by the test-only host simulation build.
#pragma once
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <limits.h>
#include <algorithm>
#include <string>
#include <vector>
#include "sg_common.h"
#include "sg_seed.h"

// One contig line of the Genome file (Genome::saveToFile, Genome.cpp:216-228), field for field: beginningLocation, the ALT flag,
// originalContigNumber, the projection start and its reverse-complement flag, the name, the projection CIGAR ("*" for none).
struct SgContigLine {
    int64_t start = 0, projStart = 0;
    uint32_t flags = 0, projFlags = 0;
    int32_t original = 0;
    std::string name, projCigar = "*";
};

struct SgHostIndex {
    std::vector<uint8_t>  tables;        // repacked: entries of all tables back to back (+8 bytes slack)
    std::vector<uint64_t> tableStart, tableSize, tableUsed, tableMagic;
    std::vector<uint32_t> overflow;      // +1 word slack
    std::vector<uint8_t>  basesPadded;   // SG_N_PADDING 'n' + bases + SG_N_PADDING 'n'
    std::vector<int64_t>  contigStart;
    std::vector<uint8_t>  contigIsAlt;
    std::vector<int32_t>  contigOriginal;   // Genome::Contig::originalContigNumber (order in the FASTA; what sorted output is ordered by)
    std::vector<std::string> contigName;
    std::vector<SgContigLine> contigLines;   // the Genome file's contig lines as read (sg_set_contigs)
    // ALT liftover data of each contig line (SgIndexView::projStart / projRC / projOps); empty when no contig is ALT
    std::vector<int64_t>  projStart;
    std::vector<uint8_t>  projRC;
    std::vector<uint32_t> projOps;
    int64_t  nBases = 0, altFirstLocation = LLONG_MAX;
    uint32_t seedLen = 0, keyBytes = 0, nTables = 0, large = 0, entryBytes = 0, chromosomePadding = 0, locationSize = 4;
    uint32_t invalidValue = 0xffffffffu;
    uint64_t overflowSize = 0, totalSlots = 0;
    // sector-bucket layout (sg_bucket.h), filled by sg_host_relayout(); layout says which one view() hands out
    uint32_t layout = SG_LAYOUT_SNAP;
    std::vector<uint64_t> buckets;
    uint64_t nBuckets = 0;

    SgIndexView view() const {           // host-memory view (test build); the CUDA library builds a device one
        SgIndexView v;
        v.tables = tables.data(); v.tableStart = tableStart.data(); v.tableSize = tableSize.data(); v.tableMagic = tableMagic.data();
        v.overflow = overflow.data(); v.bases = basesPadded.data() + SG_N_PADDING; v.contigStart = contigStart.data();
        v.nBases = nBases; v.altFirstLocation = altFirstLocation; v.overflowSize = overflowSize;
        v.nContigs = (uint32_t)contigStart.size(); v.seedLen = seedLen; v.keyBytes = keyBytes; v.nTables = nTables;
        v.large = large; v.entryBytes = entryBytes; v.chromosomePadding = chromosomePadding; v.invalidValue = invalidValue;
        v.layout = layout; v.pad0 = 0; v.buckets = buckets.empty() ? (const uint64_t *)0 : buckets.data(); v.nBuckets = nBuckets;
        v.projStart = projStart.empty() ? (const int64_t *)0 : projStart.data();
        v.projRC = projRC.empty() ? (const uint8_t *)0 : projRC.data();
        v.projOps = projOps.empty() ? (const uint32_t *)0 : projOps.data();
        return v;
    }
};

// The contig metadata of an index from its Genome file lines, as Genome::loadFromFile keeps it (Genome.cpp:348-403): starts, names,
// ALT flags, original numbers, and the liftover arrays when some contig is ALT.  False on a malformed projection CIGAR, or an ALT
// contig followed by a non-ALT one (the index keeps the ALTs last, FASTA.cpp, so genomeLocationOfFirstALTContig bounds them).
static inline bool sg_set_contigs(SgHostIndex &ix, const std::vector<SgContigLine> &lines, std::string &err)
{
    ix.contigLines = lines;
    ix.contigStart.clear(); ix.contigIsAlt.clear(); ix.contigName.clear(); ix.contigOriginal.clear();
    ix.projStart.clear(); ix.projRC.clear(); ix.projOps.clear();
    std::vector<uint32_t> projOpBegin, ops;
    for (size_t i = 0; i < lines.size(); i++) {
        const SgContigLine &L = lines[i];
        if (i > 0 && ix.contigIsAlt.back() && !(L.flags & 1)) { err = "Genome contigs: a non-ALT contig follows an ALT contig (ALT contigs must come last)"; return false; }
        ix.contigStart.push_back(L.start);
        ix.contigIsAlt.push_back((L.flags & 1) ? 1 : 0);
        ix.contigOriginal.push_back(L.original);
        ix.contigName.push_back(L.name);
        ix.projStart.push_back(L.projStart);
        ix.projRC.push_back(0);
        projOpBegin.push_back((uint32_t)ops.size());
        // a CIGAR of length 1 is the "*" of a contig without a liftover line (Genome.cpp:380-401)
        if (L.projCigar.size() > 1) {
            const char *c = L.projCigar.data(), *ce = c + L.projCigar.size();
            while (c < ce) {
                long long count = 0; const char *d = c;
                while (c < ce && *c >= '0' && *c <= '9') { count = count * 10 + (*c - '0'); c++; if (count > 0x7fffffLL) break; }
                if (c == d || c >= ce || count > 0x7fffffLL || !*c || !strchr("MIDNSHP=X", *c)) { err = "Genome contig line: malformed projection CIGAR"; return false; }
                ops.push_back(((uint32_t)count << 8) | (uint8_t)*c);
                c++;
            }
            ix.projRC.back() = (L.projFlags & 1) ? 1 : 0;       // GENOME_FLAG_ALT_PROJ_CONTIG_IS_RC
        }
    }
    projOpBegin.push_back((uint32_t)ops.size());
    if (std::find(ix.contigIsAlt.begin(), ix.contigIsAlt.end(), (uint8_t)1) == ix.contigIsAlt.end()) {
        ix.projStart.clear(); ix.projRC.clear();        // nothing can be lifted over
    } else {
        for (size_t c = 0; c < projOpBegin.size(); c++) ix.projOps.push_back((uint32_t)projOpBegin.size() + projOpBegin[c]);
        ix.projOps.insert(ix.projOps.end(), ops.begin(), ops.end());
    }
    // genomeLocationOfFirstALTContig, Genome.cpp:460-476
    ix.altFirstLocation = LLONG_MAX;
    for (size_t i = 0; i < ix.contigStart.size(); i++)
        if (ix.contigIsAlt[i] && ix.contigStart[i] < ix.altFirstLocation) ix.altFirstLocation = ix.contigStart[i];
    return true;
}

// The text of a Genome file before its bases (Genome::saveToFile): the header line, then one line per contig, a name's spaces
// written as '_' as the reference does (the line is space-separated).
static inline std::string sg_genome_file_header(int64_t nBases, const std::vector<SgContigLine> &lines)
{
    std::string out;
    char buf[160];
    snprintf(buf, sizeof(buf), "%lld %d %d\n", (long long)nBases, (int)lines.size(), 1);       // GENOME_FLAG_ALT_CONTIGS_MARKED
    out += buf;
    for (size_t c = 0; c < lines.size(); c++) {
        const SgContigLine &L = lines[c];
        std::string name = L.name;
        for (size_t k = 0; k < name.size(); k++) if (name[k] == ' ') name[k] = '_';
        snprintf(buf, sizeof(buf), "%lld %x %d %lld %x %d %d ", (long long)L.start, L.flags, (int)L.original, (long long)L.projStart, L.projFlags,
                 (int)name.size(), (int)L.projCigar.size());
        out += buf; out += name; out += ' '; out += L.projCigar; out += '\n';
    }
    return out;
}

// The GenomeIndex file (GenomeIndex.cpp:1007-1008): major minor nHashTables overflowTableSize seedLen chromosomePadding keySize
// hashTablesFileSize smallHashTable locationSize
static inline std::string sg_genome_index_text(uint32_t nTables, uint64_t overflowSize, uint32_t seedLen, uint32_t chromosomePadding, uint32_t keyBytes,
                                               uint64_t hashBytes, uint32_t large)
{
    char buf[200];
    snprintf(buf, sizeof(buf), "%d %d %d %lld %d %d %d %lld %d %d", 7, 1, (int)nTables, (long long)overflowSize, (int)seedLen, (int)chromosomePadding,
             (int)keyBytes, (long long)hashBytes, large ? 0 : 1, 4);
    return buf;
}

// A table's header in GenomeIndexHash (SNAPHashTable::saveToFile, HashTable.cpp:199-240): 36 bytes
static inline void sg_table_header(uint8_t out[36], uint64_t size, uint64_t used, uint32_t keyBytes, uint32_t large, uint32_t invalidValue)
{
    const uint32_t magic = 0xb111b010u, vs = 4, vc = large ? 2 : 1;
    memcpy(out, &magic, 4); memcpy(out + 4, &size, 8); memcpy(out + 12, &used, 8); memcpy(out + 20, &keyBytes, 4);
    memcpy(out + 24, &vs, 4); memcpy(out + 28, &vc, 4); memcpy(out + 32, &invalidValue, 4);
}

// Slots of a table holding `used` entries: (1 + slack) x its content (GenomeIndex.cpp:1084-1100 with exact counts), at least 100
static inline uint64_t sg_table_slots(uint64_t used, double slack)
{
    const uint64_t sz = (uint64_t)((double)used * (1.0 + slack)) + 1;
    return sz < 100 ? 100 : sz;
}

static inline bool sg_read_file(const std::string &path, std::vector<uint8_t> &out, std::string &err)
{
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) { err = "unable to open '" + path + "'"; return false; }
    fseeko(f, 0, SEEK_END);
    off_t n = ftello(f);
    fseeko(f, 0, SEEK_SET);
    out.resize((size_t)n);
    size_t got = n ? fread(out.data(), 1, (size_t)n, f) : 0;
    fclose(f);
    if (got != (size_t)n) { err = "short read on '" + path + "'"; return false; }
    return true;
}

// Replaces GenomeIndex::loadFromDirectory + Genome::loadFromFile + SNAPHashTable::loadCommon
// (reference GenomeIndex.cpp:1838-2093, Genome.cpp:276-440, HashTable.cpp:98-175).
static inline bool sg_load_index_directory(const std::string &dir, SgHostIndex &ix, std::string &err)
{
    std::vector<uint8_t> buf;
    // --- GenomeIndex: "major minor nHashTables overflowTableSize seedLen chromosomePadding keySize hashFileSize small locationSize"
    if (!sg_read_file(dir + "/GenomeIndex", buf, err)) return false;
    buf.push_back(0);
    unsigned major, minor, nHashTables, seedLen, chromosomePadding, keySize, smallHashTable, locationSize;
    long long overflowTableSize, hashTablesFileSize;
    if (10 != sscanf((const char *)buf.data(), "%u %u %u %lld %u %u %u %lld %u %u", &major, &minor, &nHashTables, &overflowTableSize,
                     &seedLen, &chromosomePadding, &keySize, &hashTablesFileSize, &smallHashTable, &locationSize)) {
        err = "GenomeIndex header unparsable (index older than 1.0.4?)"; return false;
    }
    if (major != 7) { err = "index format major version is not 7"; return false; }      // GenomeIndex.h:170
    if (locationSize != 4) { err = "only 4-byte genome locations (lookupSeed32 path) are supported"; return false; }
    if (seedLen == 0 || seedLen > 32) { err = "bad seed length"; return false; }
    ix.seedLen = seedLen; ix.chromosomePadding = chromosomePadding; ix.keyBytes = keySize; ix.nTables = nHashTables;
    ix.large = smallHashTable ? 0 : 1; ix.locationSize = locationSize; ix.overflowSize = (uint64_t)overflowTableSize;

    // --- Genome: "%lld %d %d\n", per contig "%lld %x %d %lld %x %d %d %s %s\n", then raw bases
    if (!sg_read_file(dir + "/Genome", buf, err)) return false;
    {
        const char *p = (const char *)buf.data();
        const char *endp = p + buf.size();
        long long nBases; int nContigs, flags;
        const char *nl = (const char *)memchr(p, '\n', buf.size());
        if (!nl || 3 != sscanf(p, "%lld %d %d", &nBases, &nContigs, &flags)) { err = "Genome header unparsable"; return false; }
        p = nl + 1;
        ix.nBases = nBases;
        std::vector<SgContigLine> lines;
        for (int i = 0; i < nContigs; i++) {
            nl = (const char *)memchr(p, '\n', endp - p);
            if (!nl) { err = "Genome contig line truncated"; return false; }
            long long start, projStart; unsigned cflags, projRC; int origNum, nameLen, cigarLen;
            if (7 != sscanf(p, "%lld %x %d %lld %x %d %d", &start, &cflags, &origNum, &projStart, &projRC, &nameLen, &cigarLen)) {
                err = "Genome contig line unparsable"; return false;
            }
            // name starts after the 7th space
            const char *q = p; int spaces = 0;
            while (q < nl && spaces < 7) { if (*q == ' ') spaces++; q++; }
            if (nameLen < 0 || (long long)nameLen > (long long)(nl - q)) { err = "Genome contig line: name length runs past the line"; return false; }
            SgContigLine L;
            L.start = start; L.flags = cflags; L.original = origNum; L.projStart = projStart; L.projFlags = projRC;
            L.name.assign(q, (size_t)nameLen);
            // the projection CIGAR follows the name ("*" without a liftover line)
            const char *c = q + nameLen + 1;
            if (cigarLen < 0 || c > nl || (long long)cigarLen > (long long)(nl - c)) { err = "Genome contig line: projection CIGAR runs past the line"; return false; }
            L.projCigar.assign(c, (size_t)cigarLen);
            lines.push_back(L);
            p = nl + 1;
        }
        if (!sg_set_contigs(ix, lines, err)) return false;
        if ((long long)(endp - p) != nBases) { err = "Genome: base count does not match file size"; return false; }
        ix.basesPadded.assign((size_t)nBases + 2 * SG_N_PADDING, (uint8_t)'n');
        memcpy(ix.basesPadded.data() + SG_N_PADDING, p, (size_t)nBases);
    }

    // --- OverflowTable: raw u32[]
    if (!sg_read_file(dir + "/OverflowTable", buf, err)) return false;
    if (buf.size() != ix.overflowSize * 4) { err = "OverflowTable size mismatch"; return false; }
    ix.overflow.assign((size_t)ix.overflowSize + 8, 0);
    if (!buf.empty()) memcpy(ix.overflow.data(), buf.data(), buf.size());

    // --- GenomeIndexHash: per table {u32 magic, u64 tableSize, u64 used, u32 keySize, u32 valueSize, u32 valueCount, valueSize bytes invalid} + data
    if (!sg_read_file(dir + "/GenomeIndexHash", buf, err)) return false;
    if ((long long)buf.size() != hashTablesFileSize) { err = "GenomeIndexHash has unexpected size"; return false; }
    const uint32_t valueCount = ix.large ? 2 : 1;
    ix.entryBytes = 4 * valueCount + ix.keyBytes;
    ix.tableStart.assign(nHashTables, 0); ix.tableSize.assign(nHashTables, 0); ix.tableUsed.assign(nHashTables, 0);
    // first pass: sizes
    {
        size_t off = 0; uint64_t slots = 0;
        for (unsigned t = 0; t < nHashTables; t++) {
            if (off + 36 > buf.size()) { err = "GenomeIndexHash truncated"; return false; }
            uint32_t magic, ks, vs, vc, inval; uint64_t tsz, used;
            memcpy(&magic, &buf[off], 4); memcpy(&tsz, &buf[off + 4], 8); memcpy(&used, &buf[off + 12], 8);
            memcpy(&ks, &buf[off + 20], 4); memcpy(&vs, &buf[off + 24], 4); memcpy(&vc, &buf[off + 28], 4);
            if (magic != 0xb111b010u) { err = "hash table magic mismatch"; return false; }      // HashTable.cpp:343
            if (vs != 4 || vc != valueCount || ks != ix.keyBytes) { err = "hash table key/value geometry unsupported"; return false; }
            if (tsz == 0 || tsz > (buf.size() - off) / ix.entryBytes) { err = "hash table size field is zero or runs past the file"; return false; }
            memcpy(&inval, &buf[off + 32], 4);
            ix.invalidValue = inval;
            ix.tableStart[t] = slots; ix.tableSize[t] = tsz; ix.tableUsed[t] = used;
            slots += tsz;
            off += 36 + (size_t)tsz * ix.entryBytes;
        }
        if (off != buf.size()) { err = "GenomeIndexHash has trailing bytes"; return false; }
        ix.totalSlots = slots;
        ix.tableMagic.assign(nHashTables, 0);
        for (unsigned t = 0; t < nHashTables; t++) ix.tableMagic[t] = ~0ULL / ix.tableSize[t];
    }
    // The image keeps every entry 4-byte aligned: the lookup reads an entry's values -- and hands out a pointer to a singleton hit -- as 32-bit words
    // (sg_fill_hits), which a GPU cannot do at an odd address.  Seed lengths whose key is not a multiple of 4 bytes (-s 21..32: 5-7 key bytes, entries of
    // 9-11 bytes in the file; 13-15 with -large) are therefore re-strided to the next multiple of 4, the key's bytes followed by zero padding the
    // lookup never reads (it loads keyBytes bytes).  Seed length 20 (8-byte entries; 12 with -large) is copied as it is.
    const uint32_t fileEntryBytes = ix.entryBytes;
    ix.entryBytes = (fileEntryBytes + 3u) & ~3u;
    ix.tables.assign((size_t)ix.totalSlots * ix.entryBytes + 16, 0);
    {
        size_t off = 0;
        for (unsigned t = 0; t < nHashTables; t++) {
            off += 36;
            size_t bytes = (size_t)ix.tableSize[t] * fileEntryBytes;
            uint8_t *dst = ix.tables.data() + (size_t)ix.tableStart[t] * ix.entryBytes;
            if (fileEntryBytes == ix.entryBytes) {
                memcpy(dst, &buf[off], bytes);
            } else {
                const uint8_t *src = &buf[off];
                for (uint64_t e = 0; e < ix.tableSize[t]; e++) memcpy(dst + (size_t)e * ix.entryBytes, src + (size_t)e * fileEntryBytes, fileEntryBytes);
            }
            off += bytes;
        }
    }
    return true;
}

// Number of 32-byte buckets for nEntries (seed, orientation) entries at the given load (entries per slot).
static inline uint64_t sg_bucket_count_for(uint64_t nEntries, uint32_t seedLen, double load)
{
    if (load < 0.05) load = 0.05;
    if (load > 0.9) load = 0.9;
    uint64_t n = (uint64_t)((double)nEntries / (SG_BUCKET_SLOTS * load)) + 1;
    const uint64_t mn = sg_bucket_min_count(2 * seedLen);
    return n < mn ? mn : n;
}

static inline double sg_bucket_default_load()
{
    double load = 0.5;           // sectors per lookup ~1.2 (0.6: 1.45, 0.4: 1.1) for 48 GB of buckets at 3 Gbp
    if (const char *e = getenv("SNAPGPU_BUCKET_LOAD")) { double v = atof(e); if (v > 0.0) load = v; }
    return load;
}

// Re-lays a loaded reference-format index (default or -large tables) into sector buckets on the host: every used value of every
// table entry becomes one (canonical seed, orientation) -> value slot.  Sequential; the CUDA library does the same on the device
// (sg_build.cuh), this form serves the host-side tests.
static inline bool sg_host_relayout(SgHostIndex &ix, double load, std::string &err)
{
    if (ix.keyBytes != 4 || ix.seedLen < 16 || ix.seedLen > 24) { err = "bucket layout needs 4-byte keys (seed length 16..24)"; return false; }
    const uint32_t nv = ix.large ? 2u : 1u, keyBits = ix.keyBytes * 8, bits = 2 * ix.seedLen;
    uint64_t nEntries = 0;
    for (uint64_t s = 0; s < ix.totalSlots; s++) {
        const uint8_t *p = ix.tables.data() + (size_t)s * ix.entryBytes;
        for (uint32_t j = 0; j < nv; j++) {
            uint32_t v; memcpy(&v, p + 4 * j, 4);
            if (v != ix.invalidValue && v != 0xfffffffeu) nEntries++;
        }
    }
    for (int attempt = 0; attempt < 4; attempt++, load *= 0.7) {
        ix.nBuckets = sg_bucket_count_for(nEntries, ix.seedLen, load);
        ix.buckets.assign((size_t)ix.nBuckets * SG_BUCKET_SLOTS, SG_BUCKET_EMPTY);
        bool ok = true;
        for (uint32_t t = 0; t < ix.nTables && ok; t++) {
            for (uint64_t k = 0; k < ix.tableSize[t] && ok; k++) {
                const uint8_t *p = ix.tables.data() + (size_t)(ix.tableStart[t] + k) * ix.entryBytes;
                uint32_t v[2] = {0xfffffffeu, 0xfffffffeu}; uint32_t key;
                memcpy(&v[0], p, 4); if (nv == 2) memcpy(&v[1], p + 4, 4);
                memcpy(&key, p + 4 * nv, 4);
                if (v[0] == ix.invalidValue) continue;
                const uint64_t seed = ((uint64_t)t << keyBits) | key;
                if (ix.large) {
                    for (uint32_t o = 0; o < 2 && ok; o++)
                        if (v[o] != 0xfffffffeu) ok = sg_bucket_insert_seq(ix.buckets.data(), ix.nBuckets, bits, seed, o, v[o]);
                } else {
                    const uint64_t rc = sg_seed_revcomp(seed, ix.seedLen);
                    const uint64_t c = seed < rc ? seed : rc;
                    ok = sg_bucket_insert_seq(ix.buckets.data(), ix.nBuckets, bits, c, seed == c ? 0u : 1u, v[0]);
                }
            }
        }
        if (ok) { ix.layout = SG_LAYOUT_BUCKET; return true; }
    }
    err = "bucket layout: a key landed too far from home even at low load";
    return false;
}

// Entries per table of the bucket-layout index re-laid into the reference's tables of the given geometry (sg_bucket.h): the
// sequential form of sg_relay_count_kernel.
static inline bool sg_host_relay_count(const SgHostIndex &ix, uint32_t keyBytes, uint32_t large, std::vector<uint64_t> &used, std::string &err)
{
    if (ix.layout != SG_LAYOUT_BUCKET || !sg_relay_geometry_ok(ix.seedLen, keyBytes)) { err = "re-lay needs a bucket-layout index and a key size the seed fills"; return false; }
    used.assign((size_t)1 << (2 * ix.seedLen - 8 * keyBytes), 0);
    for (uint64_t s = 0; s < ix.nBuckets * SG_BUCKET_SLOTS; s++) {
        uint32_t t; bool ok;
        if (sg_relay_counts(ix.buckets.data(), ix.nBuckets, s, ix.seedLen, keyBytes, large, &t, &ok)) used[t]++;
        if (!ok) { err = "a bucket slot is out of reach of its home"; return false; }
    }
    return true;
}

// Re-lays the buckets into the reference's tables of the given geometry, table t with tableSize[t] slots: `packed` gets the tables
// back to back at the file's entry stride.  The sequential form of what snapgpu_index_save_ex does on the device, through the same
// staging form and probe sequence.
static inline bool sg_host_relay_tables(const SgHostIndex &ix, uint32_t keyBytes, uint32_t large, const std::vector<uint64_t> &tableSize,
                                        std::vector<uint8_t> &packed, std::string &err)
{
    const uint32_t sb = sg_relay_stage_bytes(keyBytes, large), fb = sg_relay_file_bytes(keyBytes, large);
    std::vector<uint64_t> start(tableSize.size() + 1, 0);
    for (size_t t = 0; t < tableSize.size(); t++) start[t + 1] = start[t] + tableSize[t];
    std::vector<uint8_t> stage((size_t)start.back() * sb);
    for (uint64_t i = 0; i < start.back(); i++) sg_relay_stage_clear(stage.data() + i * sb, sb);
    for (uint64_t s = 0; s < ix.nBuckets * SG_BUCKET_SLOTS; s++) {
        const uint64_t slot = ix.buckets[s];
        if ((uint32_t)slot == 0xffffffffu) continue;
        uint32_t t, which; uint64_t key;
        if (!sg_relay_entry(slot, s / SG_BUCKET_SLOTS, ix.nBuckets, ix.seedLen, keyBytes, large, &t, &key, &which)) { err = "a bucket slot is out of reach of its home"; return false; }
        if (t >= tableSize.size()) { err = "re-lay: table out of range"; return false; }
        if (!sg_relay_insert_seq(stage.data() + (size_t)start[t] * sb, sb, tableSize[t], key, which, (uint32_t)slot)) { err = "hash table overflow"; return false; }
    }
    packed.assign((size_t)start.back() * fb, 0);
    for (uint64_t i = 0; i < start.back(); i++) sg_relay_pack(stage.data(), sb, i, packed.data(), keyBytes, large);
    return true;
}

// Writes the reference's tables (tableStart / tableSize as they stand, the index's own key size and table kind) from the sector
// buckets, recounting tableUsed; afterwards view() hands out the tables.  The host-side tests use it.
static inline bool sg_host_buckets_to_tables(SgHostIndex &ix, std::string &err)
{
    if (ix.layout != SG_LAYOUT_BUCKET || ix.keyBytes != 4) { err = "buckets -> tables needs a bucket-layout index with 4-byte keys"; return false; }
    std::vector<uint8_t> packed;
    if (!sg_host_relay_count(ix, ix.keyBytes, ix.large, ix.tableUsed, err) || !sg_host_relay_tables(ix, ix.keyBytes, ix.large, ix.tableSize, packed, err)) return false;
    packed.resize(packed.size() + 16, 0);
    ix.tables.swap(packed);
    ix.layout = SG_LAYOUT_SNAP;
    ix.buckets.clear(); ix.nBuckets = 0;
    return true;
}

// Splits bins [0, nBins) into contiguous ranges (passes) whose bytes each fit `budget`: at least minPasses of them, or one per
// non-empty bin if there are fewer, and as few as that allows otherwise (one when everything fits).  bounds gets the P + 1 range
// edges.  False, with *badBin, when one bin alone exceeds the budget.
static inline bool sg_plan_passes(const uint64_t *binBytes, uint32_t nBins, uint64_t budget, uint32_t minPasses, std::vector<uint32_t> &bounds, uint32_t *badBin)
{
    uint64_t total = 0, nonEmptyLeft = 0;
    for (uint32_t b = 0; b < nBins; b++) {
        if (binBytes[b] > budget) { *badBin = b; return false; }
        total += binBytes[b];
        nonEmptyLeft += binBytes[b] > 0;
    }
    if (minPasses < 1) minPasses = 1;
    uint64_t cap = total / minPasses;                          // forcing P passes: spread the bytes evenly
    if (cap < 1) cap = 1;
    if (cap > budget) cap = budget;
    bounds.assign(1, 0);
    uint64_t cur = 0, curNonEmpty = 0;
    for (uint32_t b = 0; b < nBins; b++) {
        const uint64_t w = binBytes[b];
        if (w == 0) continue;
        const uint64_t passesAfterThis = minPasses > bounds.size() ? minPasses - bounds.size() : 0;
        if (curNonEmpty > 0 && (cur + w > cap || nonEmptyLeft <= passesAfterThis)) {
            bounds.push_back(b);
            cur = 0; curNonEmpty = 0;
        }
        cur += w; curNonEmpty++; nonEmptyLeft--;
    }
    bounds.push_back(nBins);
    return true;
}

// ---- probability tables (reference LandauVishkin.cpp:715-763), MAPQ thresholds (mapq.h:54), wrap table ----

// SeedSequencer::SeedSequencer (reference SeedSequencer.cpp:36-103): breadth-first midpoint order; the table is
// indexed by position and stores the fill order, and is *read* as offsets[wrapCount] (SeedSequencer.h:40-43).
static inline void sg_seed_sequencer(unsigned seedSize, uint32_t *offsets)
{
    for (unsigned i = 0; i < seedSize; i++) offsets[i] = 0;
    if (seedSize == 1) return;
    struct Item { unsigned lo, hi; };
    std::vector<Item> queue;
    size_t head = 0;
    unsigned nFilled = 1;
    Item first; first.lo = 1; first.hi = seedSize - 1;
    queue.push_back(first);
    while (head < queue.size()) {
        Item it = queue[head++];
        unsigned sel = (it.lo + it.hi) / 2;
        offsets[sel] = nFilled++;
        if (it.hi > sel) { Item up; up.lo = sel + 1; up.hi = it.hi; queue.push_back(up); }
        if (it.lo < sel) { Item lowItem; lowItem.lo = it.lo; lowItem.hi = sel - 1; queue.push_back(lowItem); }
    }
}

static inline int sg_mapq_of_x(double x) { return (int)(-10 * log10(x)); }

static inline void sg_init_tables(SgTables &T, unsigned seedLen)
{
    const double SNP_PROB = 0.001, GAP_OPEN_PROB = 0.001, GAP_EXTEND_PROB = 0.5;      // BaseAligner.h:368-370
    T.indel[0] = 1.0;
    T.indel[1] = GAP_OPEN_PROB;
    for (int i = 2; i < SG_MAX_INDEL_TABLE; i++) T.indel[i] = T.indel[i - 1] * GAP_EXTEND_PROB;
    const double mutationRate = SNP_PROB;
    for (int i = 0; i < 33; i++) T.phred[i] = mutationRate;
    for (int i = 33; i <= 93 + 33; i++) T.phred[i] = 1.0 - (1.0 - pow(10.0, -1.0 * (i - 33.0) / 10.0)) * (1.0 - mutationRate);
    for (int i = 93 + 33 + 1; i < 256; i++) T.phred[i] = mutationRate;
    T.perfect[0] = 1.0;
    for (int i = 1; i < SG_MAX_PERFECT_TABLE; i++) T.perfect[i] = T.perfect[i - 1] * (1 - SNP_PROB);
    // BaseAligner.cpp:1314 `pow(1 - SNP_PROB, seedLen)` with an int exponent: the reference is built as C++98, where that
    // resolves to std::pow(double,int) = __builtin_powi, i.e. libgcc's square-and-multiply __powidf2 (NOT libm pow).
    {
        double x = 1 - SNP_PROB; unsigned n = seedLen;
        double y = (n % 2) ? x : 1;
        while (n >>= 1) { x = x * x; if (n % 2) y *= x; }
        T.snpPowSeedLen = y;
    }
    // mapqThreshold[m]: the largest double x in (0,1] with (int)(-10*log10(x)) >= m, by bisection on the bit pattern
    // (positive doubles order like their bit patterns; glibc log10 is monotone).
    T.mapqThreshold[0] = 1.0;
    for (int m = 1; m <= 71; m++) {
        uint64_t lo, hi; double dlo = 4.9406564584124654e-324, dhi = 1.0;
        memcpy(&lo, &dlo, 8); memcpy(&hi, &dhi, 8);
        // invariant: f(lo) >= m, f(hi) < m  (f(1.0) = 0 < m)
        while (hi - lo > 1) {
            uint64_t mid = lo + (hi - lo) / 2; double dm; memcpy(&dm, &mid, 8);
            if (sg_mapq_of_x(dm) >= m) lo = mid; else hi = mid;
        }
        memcpy(&T.mapqThreshold[m], &lo, 8);
    }
    uint32_t offs[33];
    memset(offs, 0, sizeof(offs));
    sg_seed_sequencer(seedLen, offs);
    for (unsigned i = 0; i < 33; i++) T.wrapSeed[i] = (i < seedLen) ? offs[i] : 0;
}

static inline uint32_t sg_next_pow2(uint32_t x) { uint32_t p = 1; while (p < x) p <<= 1; return p; }

// snapgpu_params -> SgParams, with the constructor-time derivations of BaseAligner::BaseAligner (BaseAligner.cpp:173-183).
static inline bool sg_derive_params(const snapgpu_params &in, unsigned seedLen, uint32_t maxReadLen, SgParams &p, std::string &err)
{
    if (in.struct_size != sizeof(snapgpu_params)) { err = "snapgpu_params.struct_size mismatch (ABI)"; return false; }
    if (in.maxSecondaryAlignmentAdditionalEditDistance < -1) { err = "maxSecondaryAlignmentAdditionalEditDistance (-om) must be -1 (off) or >= 0"; return false; }
    if (in.maxSecondaryAlignmentAdditionalEditDistance > (int)in.extraSearchDepth) {
        err = "the max edit distance for secondary alignments (-om) cannot be bigger than the max search depth (-D)"; return false;      // AlignerContext.cpp:784-788
    }
    if (!in.ignoreAlignmentAdjustmentsForOm) { err = "alignment adjustment (-ae) is not supported"; return false; }
    if ((unsigned)in.subPenalty > (unsigned)(in.gapOpenPenalty + in.gapExtendPenalty)) {
        err = "subPenalty must be < gapOpen + gapExtend"; return false;                    // BaseAligner.cpp:141-144
    }
    if (in.maxDist > SG_MAX_K - 1) { err = "maxDist must be < MAX_K"; return false; }
    if (maxReadLen > SNAPGPU_MAX_READ_LENGTH) { err = "maxReadLen exceeds MAX_READ_LENGTH"; return false; }
    memset(&p, 0, sizeof(p));
    p.maxHits = in.maxHits; p.maxK = in.maxDist; p.numSeedsFromCommandLine = in.numSeedsFromCommandLine;
    p.seedCoverage = in.seedCoverage;
    p.minWeightToCheck = in.minWeightToCheck > 1 ? in.minWeightToCheck : 1;                 // max(1u, ...)
    p.extraSearchDepth = in.extraSearchDepth; p.minReadLength = in.minReadLength;
    p.useAffineGap = in.useAffineGap; p.matchReward = in.matchReward; p.subPenalty = in.subPenalty;
    p.gapOpenPenalty = in.gapOpenPenalty; p.gapExtendPenalty = in.gapExtendPenalty;
    p.fivePrimeEndBonus = in.fivePrimeEndBonus; p.threePrimeEndBonus = in.threePrimeEndBonus;
    p.noUkkonen = in.noUkkonen; p.noOrderedEvaluation = in.noOrderedEvaluation; p.noTruncation = in.noTruncation;
    p.noEditDistance = in.noEditDistance; p.noBandedAffineGap = in.noBandedAffineGap;
    p.altAwareness = in.altAwareness; p.maxScoreGapToPreferNonAltAlignment = in.maxScoreGapToPreferNonAltAlignment;
    p.explorePopularSeeds = in.explorePopularSeeds; p.stopOnFirstHit = in.stopOnFirstHit;
    unsigned maxSeedsToUse;
    if (0 != in.numSeedsFromCommandLine) maxSeedsToUse = in.numSeedsFromCommandLine;
    else maxSeedsToUse = (unsigned)(int)(in.seedCoverage * SNAPGPU_MAX_READ_LENGTH / (int)seedLen);
    if (maxSeedsToUse == 0) { err = "no seeds to use"; return false; }
    p.numWeightLists = maxSeedsToUse + 1;
    uint64_t pool = (uint64_t)in.maxHits * maxSeedsToUse * 2;
    if (pool > (1u << 24)) { err = "maxHits*maxSeeds too large"; return false; }
    p.poolSize = (uint32_t)pool;
    p.tableSlots = sg_next_pow2(p.poolSize * 2 + 16);
    p.maxReadLen = maxReadLen;
    return true;
}

#ifdef SG_WITH_PAIRED
// snapgpu_params + snapgpu_paired_params -> the parameter blocks of the paired path: `pr` for the intersecting aligner
// (IntersectingPairedEndAligner ctor, IntersectingPairedEndAligner.cpp:36-100), `prSingle` for the Chimeric aligner's
// BaseAligner (maxK/2 and -N seeds, ChimericPairedEndAligner.cpp:80-87), `pp` for both.
static inline bool sg_derive_paired_params(const snapgpu_params &in, const snapgpu_paired_params &pin, unsigned seedLen, uint32_t maxReadLen,
                                           SgParams &pr, SgParams &prSingle, SgPairedParams &pp, std::string &err)
{
    if (pin.struct_size != sizeof(snapgpu_paired_params)) { err = "snapgpu_paired_params.struct_size mismatch (ABI)"; return false; }
    if (in.maxSecondaryAlignmentAdditionalEditDistance != -1) { err = "paired path: secondary alignments (-om) are not supported"; return false; }
    if (!in.useAffineGap && pin.useSoftClipping && pin.enableHammingScoringBaseAligner) {
        // The reference asserts against this combination (`_ASSERT(useAffineGap)` before the single-end aligner's alignAffineGap in the soft-clipping
        // branch, ChimericPairedEndAligner.cpp:359); its release build runs on regardless, and on reads with junk tails a few pairs per thousand then
        // come out differently from this engine.  `-G-` / `-ne` for pairs therefore needs `-hc` (no soft clipping) or `-eh-`, where results are identical.
        err = "paired path: affine gap off (-G- / -ne) together with soft clipping and the Hamming base aligner is a combination the reference asserts "
              "against (ChimericPairedEndAligner.cpp:359): add -hc or -eh-";
        return false;
    }
    if (!sg_derive_params(in, seedLen, maxReadLen, pr, err)) return false;
    snapgpu_params s = in;
    s.maxDist = in.maxDist / 2;
    s.numSeedsFromCommandLine = pin.maxSeedsSingleEnd;
    if (!sg_derive_params(s, seedLen, maxReadLen, prSingle, err)) return false;
    if (in.stopOnFirstHit) { err = "paired path: stopOnFirstHit is not supported"; return false; }
    memset(&pp, 0, sizeof(pp));
    pp.minSpacing = pin.minSpacing; pp.maxSpacing = pin.maxSpacing; pp.maxBigHits = pin.intersectingAlignerMaxHits;
    pp.maxSeedsSingleEnd = pin.maxSeedsSingleEnd; pp.maxKForIndels = pin.maxDistForIndels; pp.forceSpacing = pin.forceSpacing;
    pp.minScoreRealignment = pin.minScoreRealignment; pp.minScoreGapRealignmentALT = pin.minScoreGapRealignmentALT;
    pp.minAGScoreImprovement = pin.minAGScoreImprovement; pp.enableHammingScoringBaseAligner = pin.enableHammingScoringBaseAligner;
    pp.useSoftClip = pin.useSoftClipping; pp.flattenMAPQAtOrBelow = pin.flattenMAPQAtOrBelow;
    pp.numSeedsFromCommandLine = in.numSeedsFromCommandLine < SG_MAX_MAX_SEEDS ? in.numSeedsFromCommandLine : SG_MAX_MAX_SEEDS;
    if (0 != pp.numSeedsFromCommandLine) pp.maxSeedsToUse = pp.numSeedsFromCommandLine;
    else pp.maxSeedsToUse = (unsigned)(SNAPGPU_MAX_READ_LENGTH * in.seedCoverage / seedLen);
    if (pp.maxSeedsToUse == 0) { err = "no seeds to use"; return false; }
    uint64_t pool = (uint64_t)pin.intersectingAlignerMaxHits * pp.maxSeedsToUse * 2;
    if (pool > pin.maxCandidatePoolSize) pool = pin.maxCandidatePoolSize;
    if (pool < 2 || pool > (1u << 22)) { err = "paired candidate pool size out of range"; return false; }
    pp.poolSize = (uint32_t)pool;
    pp.poolCap = pp.poolSize; pp.agCandCap = SG_MAX_AG_CANDIDATES;
    return true;
}
#endif
