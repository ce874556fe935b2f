// sg_bucket.h -- the GPU-native index layout: one 32-byte DRAM sector resolves a lookup.  Host+device.
//
// The reference's tables (HashTable.h:87-198) store one (value, key) entry per slot and chain by quadratic-then-linear probing:
// a `lookupSeed32` on the default index walks two chains (seed and reverse complement, GenomeIndex.cpp:2138-2155), 10.6 entries
// on average at 3 Gbp, each in its own sector -- >= 10 random DRAM sectors per lookup.  Random sectors are what HBM is slowest at
// (the device serves a fixed number of random sector accesses per second, whatever the access width from 8 to 32 bytes),
// so the layout here is organised around the sector, not the entry:
//
//   * keyed by the CANONICAL seed c = min(seed, reverse complement), like the reference's own `-large` layout (GenomeIndex.cpp:2131,
//     Seed.h:99): both strands of a lookup come from one place;
//   * bucket = 4 slots x 8 bytes = 32 bytes = one sector, 32-byte aligned.  A slot is
//         [63] "continue" flag (slot 0 of a bucket only)   [62] orientation (0: locations of c, 1: locations of rc(c))
//         [61:32] tag = low 30 bits of h                   [31:0] value
//     with h = a bijective mix of c on 2*seedLen bits and the home bucket = floor(h * nBuckets / 2^(2*seedLen)).  The value is the
//     reference's: a location (< countOfBases: singleton, fillInLookedUpResults32 GenomeIndex.cpp:2159-2202) or countOfBases +
//     offset into the overflow table (count, then the locations descending, :879-889).  An empty slot has value 0xffffffff;
//   * a key that finds its home bucket full goes to the next bucket with room and sets the "continue" flag of every bucket it
//     passed; a lookup scans its home bucket and goes on only while the bucket just scanned carries the flag (and it has not yet
//     seen both orientations).  At load 0.6 that is ~1.1 sectors per lookup, present or absent;
//   * the high 2*seedLen - 30 bits of h are not stored: they follow from the bucket, because a key is never more than
//     SG_BUCKET_MAX_DISP buckets from home and nBuckets is kept >= 2^(2*seedLen - 30) * 2 * (SG_BUCKET_MAX_DISP + 1), so two keys with
//     equal tags whose homes are that close cannot exist (their h differ by a multiple of 2^30).
//
// What is kept from the reference is the RESULT of a lookup: the same hit set, in the same (descending) order, with `hits` pointing
// at 32-bit locations in HBM (SURVEY 8c: "parity is defined on results, so the GPU may re-layout the table").
#pragma once
#include "sg_common.h"

#define SG_BUCKET_SLOTS 4
#define SG_BUCKET_MAX_DISP 127
#define SG_BUCKET_EMPTY 0x3fffffffffffffffULL          // tag all ones, orientation 0, no flag, value invalid
#define SG_BUCKET_FLAG (1ULL << 63)
#define SG_BUCKET_ORIENT (1ULL << 62)

// Bijective mix of a `bits`-wide value (32 <= bits <= 48): odd multiplications and right xor-shifts are permutations of [0, 2^bits).
SG_HD uint64_t sg_bucket_mix(uint64_t c, uint32_t bits)
{
    const uint64_t mask = (bits >= 64) ? ~0ULL : ((1ULL << bits) - 1);
    const uint32_t s = bits / 2;
    uint64_t x = c & mask;
    x = (x * 0xff51afd7ed558ccdULL) & mask;
    x ^= x >> s;
    x = (x * 0xc4ceb9fe1a85ec53ULL) & mask;
    x ^= x >> s;
    x = (x * 0x9e3779b97f4a7c15ULL) & mask;
    x ^= x >> s;
    return x;
}

// Inverse of an odd multiplier mod 2^64 (Newton: each step doubles the correct low bits, 3 -> 96).
SG_HD uint64_t sg_odd_inverse(uint64_t m)
{
    uint64_t x = m;                                            // m * m == 1 mod 8
    for (int i = 0; i < 5; i++) x *= 2 - m * x;
    return x;
}

// Inverse of sg_bucket_mix: the xor-shifts by bits/2 undo themselves on a bits-wide value, the multiplications by the inverses.
SG_HD uint64_t sg_bucket_unmix(uint64_t h, uint32_t bits)
{
    const uint64_t mask = (bits >= 64) ? ~0ULL : ((1ULL << bits) - 1);
    const uint32_t s = bits / 2;
    uint64_t x = h & mask;
    x ^= x >> s;
    x = (x * sg_odd_inverse(0x9e3779b97f4a7c15ULL)) & mask;
    x ^= x >> s;
    x = (x * sg_odd_inverse(0xc4ceb9fe1a85ec53ULL)) & mask;
    x ^= x >> s;
    x = (x * sg_odd_inverse(0xff51afd7ed558ccdULL)) & mask;
    return x;
}

SG_HD uint64_t sg_mulhi64(uint64_t a, uint64_t b)
{
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// floor(h * nBuckets / 2^bits)
SG_HD uint64_t sg_bucket_home(uint64_t h, uint32_t bits, uint64_t nBuckets)
{
    return sg_mulhi64(h << (64 - bits), nBuckets);
}

// Smallest bucket count for which tags identify keys (see the header comment).
SG_HD uint64_t sg_bucket_min_count(uint32_t bits)
{
    const uint32_t hidden = bits > 30 ? bits - 30 : 0;
    return (1ULL << hidden) * 2ULL * (SG_BUCKET_MAX_DISP + 1);
}

SG_HD uint64_t sg_bucket_slot_make(uint64_t h, uint32_t orient, uint32_t value)
{
    return ((uint64_t)orient << 62) | ((h & 0x3fffffffULL) << 32) | value;
}

SG_HD uint64_t sg_seed_revcomp(uint64_t bases, uint32_t seedLen);      // sg_seed.h

// The seed whose locations a used slot of bucket b holds (the canonical seed, or its reverse complement for orientation 1).  The
// hidden high bits of h: the key's home is b or up to SG_BUCKET_MAX_DISP buckets before it (wrapping at bucket 0), and homes of
// h values that differ in their high bits lie >= 2 * (SG_BUCKET_MAX_DISP + 1) buckets apart, so of the largest high part whose
// homes start at or before b and the one below it, exactly one places the key within reach.  False if neither does.
SG_HD bool sg_bucket_slot_decode(uint64_t slot, uint64_t b, uint64_t nBuckets, uint32_t seedLen, uint64_t *seed, uint32_t *orient)
{
    const uint32_t bits = 2 * seedLen, hidden = bits - 30;
    const uint64_t tag = (slot >> 32) & 0x3fffffffULL, nHigh = 1ULL << hidden;
    // largest hi with floor(hi * nBuckets / 2^hidden) <= b, i.e. hi * nBuckets < (b + 1) * 2^hidden
    const uint64_t top = (((b + 1) << hidden) + nBuckets - 1) / nBuckets - 1;
    for (int k = 0; k < 2; k++) {
        const uint64_t hi = (top + nHigh - (uint64_t)k) & (nHigh - 1);
        const uint64_t h = (hi << 30) | tag;
        const uint64_t home = sg_bucket_home(h, bits, nBuckets);
        const uint64_t disp = b >= home ? b - home : b + nBuckets - home;
        if (disp <= SG_BUCKET_MAX_DISP) {
            const uint64_t c = sg_bucket_unmix(h, bits);
            *orient = (uint32_t)((slot >> 62) & 1);
            *seed = *orient ? sg_seed_revcomp(c, seedLen) : c;
            return true;
        }
    }
    return false;
}

// ---- re-laying buckets into the reference's tables of any geometry (snapgpu_index_save_ex on the device, sg_host.h on the host) ----
// A table entry is keyBytes bytes of key after 1 value (default tables) or 2 (-large) of 4 bytes.  The table of a key is its seed's
// bits above the low 8 * keyBytes; default tables key the seed as it lies in the genome, -large tables the smaller of the seed and
// its reverse complement, with value 0 for the locations of that canonical seed and value 1 for those of its reverse complement
// (GenomeIndex.cpp:1528-1570).  A seed that is its own reverse complement fills value 0 only, as it has only orientation 0 here.
//
// Entries are 6..14 bytes in the file, so they are first inserted into an aligned staging form, slot for slot:
//   8 bytes  (default tables, keyBytes <= 4): key << 32 | value, empty = value 0xffffffff and key 0, as in the reference;
//   16 bytes (-large, or keyBytes > 4):       u64 key + 1 (0: empty), then the two values, 0xfffffffe where unused,
// and then packed to the file stride (sg_relay_pack).
SG_HD uint64_t sg_fmix64(uint64_t key);                                             // sg_seed.h
SG_HD uint64_t sg_table_probe_next(uint64_t idx, uint64_t nProbes, uint64_t size); // sg_seed.h

#define SG_RELAY_EMPTY8 0x00000000ffffffffULL

SG_HD uint32_t sg_relay_stage_bytes(uint32_t keyBytes, uint32_t large) { return (!large && keyBytes <= 4) ? 8u : 16u; }
SG_HD uint32_t sg_relay_file_bytes(uint32_t keyBytes, uint32_t large) { return (large ? 8u : 4u) + keyBytes; }

// Geometries the reference's `snap index` accepts for a seed length (GenomeIndex.cpp runIndexer): the seed fills the key, and at most
// 4^8 tables.
SG_HD bool sg_relay_geometry_ok(uint32_t seedLen, uint32_t keyBytes)
{
    return keyBytes >= 2 && keyBytes <= 8 && 2 * seedLen >= 8 * keyBytes && 2 * seedLen - 8 * keyBytes <= 16;
}

// The entry a used slot of bucket b becomes: its table, key and which value it fills.  False if the slot does not decode.
SG_HD bool sg_relay_entry(uint64_t slot, uint64_t b, uint64_t nBuckets, uint32_t seedLen, uint32_t keyBytes, uint32_t large,
                          uint32_t *table, uint64_t *key, uint32_t *which)
{
    uint64_t seed; uint32_t orient;
    if (!sg_bucket_slot_decode(slot, b, nBuckets, seedLen, &seed, &orient)) return false;
    const uint64_t k = (large && orient) ? sg_seed_revcomp(seed, seedLen) : seed;     // -large: back to the canonical seed
    const uint32_t keyBits = 8 * keyBytes;
    *table = (uint32_t)(k >> keyBits);
    *key = keyBits >= 64 ? k : (k & ((1ULL << keyBits) - 1));
    *which = large ? orient : 0u;
    return true;
}

// Whether the buckets hold (canonical, orient): a -large entry is counted once, by its orientation-0 slot when there is one.
SG_HD bool sg_bucket_holds(const uint64_t *buckets, uint64_t nBuckets, uint32_t bits, uint64_t canonical, uint32_t orient)
{
    const uint64_t h = sg_bucket_mix(canonical, bits);
    uint64_t b = sg_bucket_home(h, bits, nBuckets);
    const uint64_t want = ((uint64_t)orient << 62) | ((h & 0x3fffffffULL) << 32);
    for (int disp = 0; disp <= SG_BUCKET_MAX_DISP; disp++) {
        for (int k = 0; k < SG_BUCKET_SLOTS; k++) {
            const uint64_t s = buckets[b * SG_BUCKET_SLOTS + k];
            if ((s & 0x7fffffff00000000ULL) == want && (uint32_t)s != 0xffffffffu) return true;
        }
        if (!(buckets[b * SG_BUCKET_SLOTS] & SG_BUCKET_FLAG)) return false;
        b = (b + 1 == nBuckets) ? 0 : b + 1;
    }
    return false;
}

// Whether a used slot of bucket b counts as an entry of its table (which it gets) in the given geometry.
SG_HD bool sg_relay_counts(const uint64_t *buckets, uint64_t nBuckets, uint64_t s, uint32_t seedLen, uint32_t keyBytes, uint32_t large, uint32_t *table, bool *ok)
{
    const uint64_t slot = buckets[s];
    *ok = true;
    if ((uint32_t)slot == 0xffffffffu) return false;
    uint64_t key; uint32_t which;
    if (!sg_relay_entry(slot, s / SG_BUCKET_SLOTS, nBuckets, seedLen, keyBytes, large, table, &key, &which)) { *ok = false; return false; }
    // SNAPHashTable::Insert counts an entry when it changes the slot's key (HashTable.cpp:329-332), and an empty slot's key is 0: the
    // reference's used count leaves out key 0, and so does the count written here
    if (key == 0) return false;
    if (which == 1) {
        const uint64_t canonical = ((uint64_t)*table << (8 * keyBytes)) | key;
        if (sg_bucket_holds(buckets, nBuckets, 2 * seedLen, canonical, 0)) return false;
    }
    return true;
}

// Sequential insertion into one table's staging slots (stage: the table's first slot), along SNAPHashTable's probe sequence;
// the device does the same with compare-and-swap (sg_build.cuh).  False if the table is full.
SG_HD bool sg_relay_insert_seq(uint8_t *stage, uint32_t stageBytes, uint64_t size, uint64_t key, uint32_t which, uint32_t value)
{
    uint64_t idx = sg_fmix64(key) % size;
    for (uint64_t nProbes = 0;;) {
        uint64_t *p = (uint64_t *)(stage + idx * stageBytes);
        if (stageBytes == 8) {
            if (p[0] == SG_RELAY_EMPTY8) { p[0] = (key << 32) | value; return true; }
        } else if (p[0] == 0 || p[0] == key + 1) {
            p[0] = key + 1;
            ((uint32_t *)(p + 1))[which] = value;
            return true;
        }
        if (++nProbes > size + 5) return false;
        idx = sg_table_probe_next(idx, nProbes, size);
    }
}

// The staging slots' initial content
SG_HD void sg_relay_stage_clear(uint8_t *slot, uint32_t stageBytes)
{
    uint64_t *p = (uint64_t *)slot;
    if (stageBytes == 8) { p[0] = SG_RELAY_EMPTY8; return; }
    p[0] = 0;
    p[1] = 0xfffffffefffffffeULL;
}

// Staging slot i -> file entry i (values, then the key's keyBytes bytes, little-endian); an empty slot becomes the reference's
// empty entry (value 0 invalid, key 0).
SG_HD void sg_relay_pack(const uint8_t *stage, uint32_t stageBytes, uint64_t i, uint8_t *out, uint32_t keyBytes, uint32_t large)
{
    const uint64_t *p = (const uint64_t *)(stage + i * stageBytes);
    uint32_t v[2] = {0xffffffffu, 0u};
    uint64_t key = 0;
    if (stageBytes == 8) {
        v[0] = (uint32_t)p[0]; key = p[0] >> 32;
    } else if (p[0] != 0) {
        key = p[0] - 1; v[0] = (uint32_t)p[1]; v[1] = (uint32_t)(p[1] >> 32);
    }
    uint8_t *e = out + i * sg_relay_file_bytes(keyBytes, large);
    const uint32_t nv = large ? 2u : 1u;
    for (uint32_t j = 0; j < nv; j++)
        for (uint32_t k = 0; k < 4; k++) e[4 * j + k] = (uint8_t)(v[j] >> (8 * k));
    for (uint32_t k = 0; k < keyBytes; k++) e[4 * nv + k] = (uint8_t)(key >> (8 * k));
}

// The four slots of bucket b, one sector.
struct SgBucket { uint64_t s[SG_BUCKET_SLOTS]; };

SG_HD SgBucket sg_bucket_load(const uint64_t *buckets, uint64_t b)
{
    SgBucket r;
#if defined(__CUDA_ARCH__)
    const ulonglong2 *p = (const ulonglong2 *)(buckets + b * SG_BUCKET_SLOTS);
    const ulonglong2 lo = __ldg(p), hi = __ldg(p + 1);
    r.s[0] = lo.x; r.s[1] = lo.y; r.s[2] = hi.x; r.s[3] = hi.y;
#else
    for (int k = 0; k < SG_BUCKET_SLOTS; k++) r.s[k] = buckets[b * SG_BUCKET_SLOTS + k];
#endif
    return r;
}

// Host-side (sequential) insertion; the device builder does the same with atomics (sg_build.cuh).  Returns false if the key would
// land more than SG_BUCKET_MAX_DISP buckets from home (table too full: rebuild with more buckets).
SG_HD bool sg_bucket_insert_seq(uint64_t *buckets, uint64_t nBuckets, uint32_t bits, uint64_t canonical, uint32_t orient, uint32_t value)
{
    const uint64_t h = sg_bucket_mix(canonical, bits);
    uint64_t b = sg_bucket_home(h, bits, nBuckets);
    const uint64_t slot = sg_bucket_slot_make(h, orient, value);
    for (int disp = 0; disp <= SG_BUCKET_MAX_DISP; disp++) {
        uint64_t *p = buckets + b * SG_BUCKET_SLOTS;
        for (int k = 0; k < SG_BUCKET_SLOTS; k++) {
            if ((uint32_t)p[k] == 0xffffffffu) {
                p[k] = slot | (k == 0 ? (p[0] & SG_BUCKET_FLAG) : 0ULL);
                return true;
            }
        }
        p[0] |= SG_BUCKET_FLAG;
        b = (b + 1 == nBuckets) ? 0 : b + 1;
    }
    return false;
}

// GenomeIndex::lookupSeed32 on the bucket layout: the semantics of sg_lookup_seed32 (sg_seed.h), i.e. of the reference's
// lookupSeed32 + fillInLookedUpResults32 (GenomeIndex.cpp:2095-2202).  `bases` / `rc` from sg_seed_pack.  *examined counts slots
// examined (4 per bucket), *overflowWords overflow-table count words read.
struct SgHits;
SG_HD void sg_fill_hits(const SgIndexView &ix, const uint32_t *subEntry, uint32_t *nHits, const uint32_t **hits, uint32_t *overflowWords);

SG_HD void sg_bucket_lookup_seed32(const SgIndexView &ix, uint64_t bases, uint64_t rc, uint32_t *nHits /*[2]*/, const uint32_t **hits /*[2]*/,
                                   uint32_t *examined, uint32_t *overflowWords)
{
    nHits[0] = nHits[1] = 0;
    hits[0] = hits[1] = ix.overflow;
    const uint32_t bits = 2 * ix.seedLen;
    const bool lookedUpComplement = bases > rc;               // Seed::isBiggerThanItsReverseComplement (Seed.h:99)
    const uint64_t c = lookedUpComplement ? rc : bases;
    const uint64_t h = sg_bucket_mix(c, bits);
    uint64_t b = sg_bucket_home(h, bits, ix.nBuckets);
    const uint64_t want = (h & 0x3fffffffULL) << 32;
    const uint32_t *found[2] = {(const uint32_t *)0, (const uint32_t *)0};
    #pragma unroll 1
    for (int disp = 0; disp <= SG_BUCKET_MAX_DISP; disp++) {
        const SgBucket B = sg_bucket_load(ix.buckets, b);
        *examined += SG_BUCKET_SLOTS;
        #pragma unroll
        for (int k = 0; k < SG_BUCKET_SLOTS; k++) {
            const uint64_t s = B.s[k];
            if ((s & 0x3fffffff00000000ULL) == want && (uint32_t)s != 0xffffffffu) {
                found[(s >> 62) & 1] = (const uint32_t *)(ix.buckets + b * SG_BUCKET_SLOTS + k);      // little-endian: the value is the slot's first word
            }
        }
        if (!(B.s[0] & SG_BUCKET_FLAG)) break;
        if (found[0] && (found[1] || bases == rc)) break;
        b = (b + 1 == ix.nBuckets) ? 0 : b + 1;
    }
    // found[o]: orientation o of the canonical seed.  Direction 0 of the lookup is the seed as given, direction 1 its reverse complement.
    const uint32_t *e0 = lookedUpComplement ? found[1] : found[0];
    const uint32_t *e1 = lookedUpComplement ? found[0] : found[1];
    if (bases == rc) e1 = e0;                                  // isOwnReverseComplement: both directions share the entry (GenomeIndex.cpp:2131)
    if (e0) sg_fill_hits(ix, e0, &nHits[0], &hits[0], overflowWords);
    if (e1) {
        if (e1 == e0) { nHits[1] = nHits[0]; hits[1] = hits[0]; }
        else sg_fill_hits(ix, e1, &nHits[1], &hits[1], overflowWords);
    }
}
