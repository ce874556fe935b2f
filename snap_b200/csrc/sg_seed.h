// sg_seed.h -- seed packing, index hash probe, lookupSeed32, genome substring.  Scalar form, host+device.
#pragma once
#include "sg_common.h"
#include "sg_bucket.h"

// BASE_VALUE, reference Tables.cpp:52-58: A=0 G=1 C=2 T=3, everything else 4.
SG_HD uint32_t sg_base_value(uint8_t c)
{
    // bits 2:1 of the ASCII code separate A(0) C(1) T(2) G(3); two packed constants give the expected character (to reject
    // everything else) and SNAP's value (A=0 G=1 C=2 T=3)
    const uint32_t i = (c >> 1) & 3u;
    const uint32_t expected = (0x47544341u >> (8u * i)) & 0xffu;
    const uint32_t value = (0x1320u >> (4u * i)) & 0xfu;
    return expected == c ? value : 4u;
}

// rcTranslationTable, reference BaseAligner.cpp:199-210: anything but ACGT becomes 'N'.
SG_HD uint8_t sg_complement(uint8_t c)
{
    return c == 'A' ? 'T' : c == 'G' ? 'C' : c == 'C' ? 'G' : c == 'T' ? 'A' : 'N';
}

// Seed::Seed + Seed::DoesTextRepresentASeed (reference Seed.h:40-53, Seed.cpp:28-42).
// bases: first base in the most significant position; reverseComplement: (v^3) with the first base least significant.
SG_HD bool sg_seed_pack(const uint8_t *text, uint32_t seedLen, uint64_t *bases, uint64_t *rc)
{
    uint64_t b = 0, r = 0;
    bool ok = true;
    for (uint32_t i = 0; i < seedLen; i++) {
        uint32_t v = sg_base_value(text[i]);
        ok = ok && (v < 4);
        b |= (uint64_t)(v & 3) << ((seedLen - i - 1) * 2);
        r |= (uint64_t)((v & 3) ^ 3) << (i * 2);
    }
    *bases = b;
    *rc = r;
    return ok;
}

// The packed reverse complement of a packed seed (both in the `bases` convention of sg_seed_pack: first base most significant):
// reverse the order of the 2-bit digits and complement each (v ^ 3, Seed.h:40-53).
SG_HD uint64_t sg_seed_revcomp(uint64_t bases, uint32_t seedLen)
{
    uint64_t x = ~bases;                                       // complement every digit
    x = ((x >> 2) & 0x3333333333333333ULL) | ((x & 0x3333333333333333ULL) << 2);
    x = ((x >> 4) & 0x0f0f0f0f0f0f0f0fULL) | ((x & 0x0f0f0f0f0f0f0f0fULL) << 4);
    x = ((x >> 8) & 0x00ff00ff00ff00ffULL) | ((x & 0x00ff00ff00ff00ffULL) << 8);
    x = ((x >> 16) & 0x0000ffff0000ffffULL) | ((x & 0x0000ffff0000ffffULL) << 16);
    x = (x >> 32) | (x << 32);                                 // all 32 digits reversed
    return x >> (64 - 2 * seedLen);
}

// SNAPHashTable::hash: MurmurHash3 fmix64 (reference HashTable.h:72-85).
SG_HD uint64_t sg_fmix64(uint64_t key)
{
    key ^= key >> 33;
    key *= 0xff51afd7ed558ccdULL;
    key ^= key >> 33;
    key *= 0xc4ceb9fe1a85ec53ULL;
    key ^= key >> 33;
    return key;
}

// SNAPHashTable's probe sequence (HashTable.h:87-118): quadratic for nProbes 1..4, then linear -- the sequence sg_probe walks.
// Every insertion into the reference's table layout (sg_build.cuh, sg_host_buckets_to_tables) takes its steps from here.
SG_HD uint64_t sg_table_probe_next(uint64_t idx, uint64_t nProbes, uint64_t size)
{
    return nProbes < 5 ? (idx + nProbes * nProbes) % size : (idx + 1) % size;
}

// Little-endian load of n (<=8) bytes from a possibly unaligned address.
SG_HD uint64_t sg_load_le(const uint8_t *p, uint32_t n)
{
    uint64_t v = 0;
    for (uint32_t i = 0; i < n; i++) v |= (uint64_t)p[i] << (8 * i);
    return v;
}

// Entry accessors (reference HashTable.h:149-198): valueCount 4-byte values, then keyBytes of key.
SG_HD void sg_entry_load(const SgIndexView &ix, uint64_t globalSlot, uint32_t *value0, uint64_t *key)
{
    if (ix.entryBytes == 8) {
        // default index: 4-byte location + 4-byte key, 8-byte aligned in our HBM image => one 64-bit load
        uint64_t e = ((const uint64_t *)ix.tables)[globalSlot];
        *value0 = (uint32_t)e;
        *key = e >> 32;
    } else {
        const uint8_t *p = ix.tables + globalSlot * ix.entryBytes;
        uint32_t nv = ix.large ? 2u : 1u;
        *value0 = (uint32_t)sg_load_le(p, 4);
        *key = sg_load_le(p + 4 * nv, ix.keyBytes);
    }
}

// SNAPHashTable::GetFirstValueForKey (reference HashTable.h:87-118): quadratic probing for nProbes 1..4
// (QUADRATIC_CHAINING_DEPTH 5), then linear.  Returns the global slot of the matching entry or ~0 if absent;
// *examined += entries looked at.
SG_HD uint64_t sg_probe(const SgIndexView &ix, uint32_t table, uint64_t key, uint32_t *examined)
{
    const uint64_t size = ix.tableSize[table];
    const uint64_t base = ix.tableStart[table];
    uint64_t idx = sg_fmix64(key) % size;
    uint32_t v; uint64_t k;
    sg_entry_load(ix, base + idx, &v, &k);
    (*examined)++;
    if (k == key && v != ix.invalidValue) {
        return base + idx;
    }
    uint64_t nProbes = 0;
    do {
        nProbes++;
        if (nProbes > size + 5) {
            return ~0ULL;
        }
        if (nProbes < 5) {
            idx = (idx + nProbes * nProbes) % size;
        } else {
            idx = (idx + 1) % size;
        }
        sg_entry_load(ix, base + idx, &v, &k);
        (*examined)++;
    } while (k != key && v != ix.invalidValue);
    if (v == ix.invalidValue) {
        return ~0ULL;
    }
    return base + idx;
}

struct SgHits {
    uint32_t nHits[2];
    const uint32_t *hits[2];         // into HBM: either &entry.value (singleton) or &overflow[off+1]; descending order
};

// GenomeIndex::fillInLookedUpResults32 (reference GenomeIndex.cpp:2159-2202).
SG_HD void sg_fill_hits(const SgIndexView &ix, const uint32_t *subEntry, uint32_t *nHits, const uint32_t **hits, uint32_t *overflowWords)
{
    uint32_t v = *subEntry;
    if ((int64_t)v < ix.nBases) {
        *nHits = 1;                  // singleton: the value is the location
        *hits = subEntry;
    } else if (v == 0xfffffffeu) {
        *nHits = 0;                  // unused half of a -large entry
        *hits = subEntry;
    } else {
        uint32_t off = v - (uint32_t)ix.nBases;
        uint32_t count = ix.overflow[off];
        *nHits = count;
        *hits = &ix.overflow[off + 1];
        (*overflowWords)++;
    }
}

// GenomeIndex::lookupSeed32 (reference GenomeIndex.cpp:2095-2157).  `bases`/`rc` from sg_seed_pack.
SG_HD void sg_lookup_seed32(const SgIndexView &ix, uint64_t bases, uint64_t rc, SgHits *out, uint32_t *examined, uint32_t *overflowWords)
{
    if (ix.layout == SG_LAYOUT_BUCKET) {
        sg_bucket_lookup_seed32(ix, bases, rc, out->nHits, out->hits, examined, overflowWords);
        return;
    }
    const uint32_t keyBits = ix.keyBytes * 8;
    out->nHits[0] = out->nHits[1] = 0;
    out->hits[0] = out->hits[1] = ix.overflow;
    if (ix.large) {
        bool lookedUpComplement = bases > rc;                 // Seed::isBiggerThanItsReverseComplement
        uint64_t s = lookedUpComplement ? rc : bases;
        uint64_t sOther = lookedUpComplement ? bases : rc;
        uint64_t low = (ix.keyBytes == 8) ? s : (s & ((1ULL << keyBits) - 1));
        uint32_t high = (ix.keyBytes == 8) ? 0u : (uint32_t)(s >> keyBits);
        uint64_t slot = sg_probe(ix, high, low, examined);
        if (slot == ~0ULL) {
            return;
        }
        const uint32_t *entry = (const uint32_t *)(ix.tables + slot * ix.entryBytes);
        sg_fill_hits(ix, lookedUpComplement ? entry + 1 : entry, &out->nHits[0], &out->hits[0], overflowWords);
        if (s == sOther) {                                     // isOwnReverseComplement
            out->nHits[1] = out->nHits[0];
            out->hits[1] = out->hits[0];
        } else {
            sg_fill_hits(ix, lookedUpComplement ? entry : entry + 1, &out->nHits[1], &out->hits[1], overflowWords);
        }
    } else {
        uint64_t s = bases;
        for (int dir = 0; dir < 2; dir++) {
            uint64_t low = (ix.keyBytes == 8) ? s : (s & ((1ULL << keyBits) - 1));
            uint32_t high = (ix.keyBytes == 8) ? 0u : (uint32_t)(s >> keyBits);
            uint64_t slot = sg_probe(ix, high, low, examined);
            if (slot != ~0ULL) {
                const uint32_t *entry = (const uint32_t *)(ix.tables + slot * ix.entryBytes);
                sg_fill_hits(ix, entry, &out->nHits[dir], &out->hits[dir], overflowWords);
            }
            s = rc;                                            // seed = ~seed
        }
    }
}

// Genome::getSubstring (reference Genome.h:339-367) + getContigAtLocation (Genome.cpp:573-594).
// Returns NULL when the window is unusable (past the genome end, or crossing into the next contig).
SG_HD const uint8_t *sg_get_substring(const SgIndexView &ix, int64_t location, int64_t lengthNeeded)
{
    if (location > ix.nBases || location + lengthNeeded > ix.nBases + SG_N_PADDING) {
        return (const uint8_t *)0;
    }
    if (location < 0) {
        return (const uint8_t *)0;   // the reference reads 'n' padding here and then finds no contig
    }
    if (lengthNeeded <= (int64_t)ix.chromosomePadding && ix.bases[location] != 'n') {
        return ix.bases + location;
    }
    if (lengthNeeded == 0) {
        return ix.bases + location;
    }
    int low = 0, high = (int)ix.nContigs - 1, found = -1;
    while (low <= high) {
        int mid = (low + high) / 2;
        int64_t b = ix.contigStart[mid];
        if (b <= location && (mid == (int)ix.nContigs - 1 || ix.contigStart[mid + 1] > location)) {
            found = mid;
            break;
        } else if (b <= location) {
            low = mid + 1;
        } else {
            high = mid - 1;
        }
    }
    if (found < 0) {
        return (const uint8_t *)0;
    }
    int64_t end = (found == (int)ix.nContigs - 1) ? ix.nBases : ix.contigStart[found + 1];   // beginning + length
    if (end <= location + lengthNeeded) {
        return (const uint8_t *)0;
    }
    return ix.bases + location;
}

// computeMAPQ (reference mapq.h:32-68) with log10 replaced by a host-libm-derived threshold table.
SG_HD int sg_compute_mapq(const SgTables &T, double probabilityOfAllCandidates, double probabilityOfBestCandidate, int popularSeedsSkipped)
{
    if (probabilityOfAllCandidates < probabilityOfBestCandidate) probabilityOfAllCandidates = probabilityOfBestCandidate;  // __max
    double correctnessProbability = probabilityOfBestCandidate / probabilityOfAllCandidates;
    int baseMAPQ;
    if (correctnessProbability >= 1) {
        baseMAPQ = 70;
    } else {
        double x = 1 - correctnessProbability;
        // (int)(-10*log10(x)) >= m  <=>  x <= mapqThreshold[m]; find the largest such m (capped at 70)
        int lo = 0, hi = 70;     // invariant: x <= thr[lo] (thr[0] = +inf conceptually), answer in [lo, hi]
        while (lo < hi) {
            int mid = (lo + hi + 1) / 2;
            if (x <= T.mapqThreshold[mid]) lo = mid; else hi = mid - 1;
        }
        baseMAPQ = lo;
    }
    int pen = popularSeedsSkipped - 10;
    if (pen < 0) pen = 0;
    baseMAPQ = baseMAPQ - pen / 2;
    if (baseMAPQ < 0) baseMAPQ = 0;
    return baseMAPQ;
}
