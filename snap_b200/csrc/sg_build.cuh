// sg_build.cuh -- building the lookup structure on the device (SURVEY 8f N3; replaces, in *results*,
// GenomeIndex::BuildIndexToDirectory, reference SNAPLib/GenomeIndex.cpp:527-1110 and its worker :1447-1530).
//
// Contract kept from the reference: every position whose seedLen bases are all ACGT is indexed under its forward
// seed (small-table layout: key = low keyBytes of the seed, table = the remaining high bases); a seed that occurs
// once stores its location in the entry, a repeated seed stores countOfBases + offset into the overflow table,
// where the list is `count` followed by the locations in DESCENDING order (:879-889).  Slot placement inside a
// table is not part of the contract (the reference's own depends on thread interleaving, :1523-1530).
//
// Method: emit (seed, location) for locations in descending order, stable LSD radix sort on the seed (so equal
// seeds keep descending locations), then one pass sizes the tables and one pass inserts run heads with atomicCAS
// along the very probe sequence lookups use.  When the sort scratch (24 bytes per position) does not fit the device at once, the
// builder runs the same sort / count / insert in passes over ranges of the seed's top 16 bits, each pass selecting its own
// positions in the same descending order (snapgpu.cu build_index_on_device).
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>


__global__ void sg_build_emit_kernel(const uint8_t *bases /* location 0 */, long long nPositions, uint32_t seedLen,
                                     unsigned long long *keys, uint32_t *locs)
{
    const unsigned long long SG_BUILD_INVALID_KEY = 1ULL << (2 * seedLen);
    long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; j < nPositions; j += stride) {
        long long loc = nPositions - 1 - j;      // descending locations
        unsigned long long b = 0;
        bool ok = true;
        for (uint32_t i = 0; i < seedLen; i++) {
            uint32_t v = sg_base_value(bases[loc + i]);
            ok = ok && v < 4;
            b = (b << 2) | (v & 3);
        }
        keys[j] = ok ? b : (SG_BUILD_INVALID_KEY | b);
        locs[j] = (uint32_t)loc;
    }
}

// pass 1: per run head, count unique seeds per table and overflow words.  The keys are sorted, so a thread sees the same table
// for long stretches: counts are kept in registers, flushed to a per-block shared histogram when the table changes, and each
// block adds its totals to the global counters once (one atomic per seed on three hot words cost 2 s at 3 Gbp).
__global__ void sg_build_count_kernel(const unsigned long long *keys, long long n, uint32_t keyBits, uint32_t seedLen, uint32_t nTables, int hist,
                                      unsigned long long *tableUsed, unsigned long long *overflowWords, unsigned long long *nValid)
{
    // shared per-block histogram when the tables fit (seed length <= 22); for more tables the per-thread run counts go straight to
    // the global histogram (still one atomic per run of equal tables, not per seed)
    extern __shared__ unsigned long long sUsed[];       // [nTables or 0] + nValid + overflowWords
    const bool sharedHist = hist == 1;
    const uint32_t nShared = sharedHist ? nTables : 0;
    for (uint32_t t = threadIdx.x; t < nShared + 2; t += blockDim.x) sUsed[t] = 0;
    __syncthreads();
    const unsigned long long SG_BUILD_INVALID_KEY = 1ULL << (2 * seedLen);
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    uint32_t curTable = 0xffffffffu;
    unsigned long long curUsed = 0, valid = 0, over = 0;
    for (; i < n; i += stride) {
        unsigned long long k = keys[i];
        if (k & SG_BUILD_INVALID_KEY) continue;
        if (i > 0 && keys[i - 1] == k) continue;
        long long e = i + 1;
        while (e < n && keys[e] == k) e++;
        unsigned long long count = (unsigned long long)(e - i);
        const uint32_t table = (uint32_t)(k >> keyBits);
        if (table != curTable) {
            if (curUsed) atomicAdd(sharedHist ? &sUsed[curTable] : &tableUsed[curTable], curUsed);
            curTable = table; curUsed = 0;
        }
        curUsed++;
        valid += count;
        if (count > 1) over += count + 1;
    }
    if (curUsed) atomicAdd(sharedHist ? &sUsed[curTable] : &tableUsed[curTable], curUsed);
    if (valid) atomicAdd(&sUsed[nShared], valid);
    if (over) atomicAdd(&sUsed[nShared + 1], over);
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < nShared; t += blockDim.x) if (sUsed[t]) atomicAdd(&tableUsed[t], sUsed[t]);
    if (threadIdx.x == 0) {
        if (sUsed[nShared]) atomicAdd(nValid, sUsed[nShared]);
        if (sUsed[nShared + 1]) atomicAdd(overflowWords, sUsed[nShared + 1]);
    }
}

// Sector-bucket insertion (sg_bucket.h) with atomics: claims the first empty slot of the home bucket, or of the next bucket with room,
// setting the "continue" flag (bit 63 of slot 0) of every full bucket it passes.  Slot 0 can change under us in two ways -- another
// key claims it, or a passer-by sets its flag -- hence the compare-and-swap retry.
__device__ __forceinline__ bool sg_bucket_insert_atomic(unsigned long long *buckets, unsigned long long nBuckets, uint32_t bits, unsigned long long canonical,
                                                        uint32_t orient, uint32_t value)
{
    const unsigned long long h = sg_bucket_mix(canonical, bits);
    unsigned long long b = sg_bucket_home(h, bits, nBuckets);
    const unsigned long long slot = sg_bucket_slot_make(h, orient, value);
    for (int disp = 0; disp <= SG_BUCKET_MAX_DISP; disp++) {
        unsigned long long *p = buckets + b * SG_BUCKET_SLOTS;
        #pragma unroll 1
        for (int k = 0; k < SG_BUCKET_SLOTS; k++) {
            unsigned long long old = ((volatile unsigned long long *)p)[k];
            while ((uint32_t)old == 0xffffffffu) {
                const unsigned long long desired = slot | (k == 0 ? (old & SG_BUCKET_FLAG) : 0ULL);
                const unsigned long long prev = atomicCAS(&p[k], old, desired);
                if (prev == old) return true;
                old = prev;
            }
        }
        atomicOr(&p[0], SG_BUCKET_FLAG);
        b = (b + 1 == nBuckets) ? 0 : b + 1;
    }
    return false;
}

// Re-lays the reference's tables (as uploaded from an index directory: 8-byte default or 12-byte -large entries) into sector buckets.
__global__ void sg_build_relayout_kernel(const uint8_t *tables, const uint64_t *tableStart, const uint64_t *tableSize, uint32_t nTables, uint32_t entryBytes,
                                         uint32_t large, uint32_t keyBits, uint32_t seedLen, uint32_t invalidValue, unsigned long long *buckets,
                                         unsigned long long nBuckets, int *failed)
{
    const uint32_t nv = large ? 2u : 1u, bits = 2 * seedLen;
    for (uint32_t t = blockIdx.y; t < nTables; t += gridDim.y) {
        const uint64_t size = tableSize[t], base = tableStart[t];
        for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < size; k += (uint64_t)gridDim.x * blockDim.x) {
            const uint8_t *p = tables + (base + k) * entryBytes;
            const uint32_t v0 = *(const uint32_t *)p, v1 = nv == 2 ? *(const uint32_t *)(p + 4) : 0xfffffffeu, key = *(const uint32_t *)(p + 4 * nv);
            if (v0 == invalidValue) continue;
            const unsigned long long seed = ((unsigned long long)t << keyBits) | key;
            bool ok = true;
            if (large) {
                if (v0 != 0xfffffffeu) ok = sg_bucket_insert_atomic(buckets, nBuckets, bits, seed, 0, v0);
                if (ok && v1 != 0xfffffffeu) ok = sg_bucket_insert_atomic(buckets, nBuckets, bits, seed, 1, v1);
            } else {
                const unsigned long long rc = sg_seed_revcomp(seed, seedLen);
                const unsigned long long c = seed < rc ? seed : rc;
                ok = sg_bucket_insert_atomic(buckets, nBuckets, bits, c, seed == c ? 0u : 1u, v0);
            }
            if (!ok) *failed = 1;
        }
    }
}

// counts the used values of the reference's tables (= bucket slots needed)
__global__ void sg_build_count_values_kernel(const uint8_t *tables, unsigned long long totalSlots, uint32_t entryBytes, uint32_t large, uint32_t invalidValue,
                                             unsigned long long *count)
{
    unsigned long long local = 0;
    const uint32_t nv = large ? 2u : 1u;
    for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < totalSlots; k += (unsigned long long)gridDim.x * blockDim.x) {
        const uint8_t *p = tables + k * entryBytes;
        for (uint32_t j = 0; j < nv; j++) {
            const uint32_t v = *(const uint32_t *)(p + 4 * j);
            if (v != invalidValue && v != 0xfffffffeu) local++;
        }
    }
    local = __reduce_add_sync(0xffffffffu, (unsigned)local) ;
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

// Places (key, value) in one of the reference's tables along SNAPHashTable's probe sequence; false if the table is full.
__device__ __forceinline__ bool sg_table_insert_atomic(unsigned long long *table, uint64_t size, unsigned long long low, uint32_t value)
{
    const unsigned long long EMPTY = 0x00000000ffffffffULL;   // key 0, value invalid (HashTable.cpp:66-72)
    const unsigned long long entry = (low << 32) | value;
    uint64_t idx = sg_fmix64(low) % size;
    for (unsigned long long nProbes = 0;;) {
        if (atomicCAS(&table[idx], EMPTY, entry) == EMPTY) return true;
        if (++nProbes > size + 5) return false;
        idx = sg_table_probe_next(idx, nProbes, size);
    }
}

// pass 2: insert run heads.  buckets != NULL: into sector buckets (sg_bucket.h); else into the reference's table layout.
__global__ void sg_build_insert_kernel(const unsigned long long *keys, const uint32_t *locs, long long n, uint32_t keyBits, uint32_t seedLen,
                                       const uint64_t *tableStart, const uint64_t *tableSize, unsigned long long *tables,
                                       uint32_t *overflow, unsigned long long *overflowCursor, long long nBases, int *failed,
                                       unsigned long long *buckets, unsigned long long nBuckets)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const unsigned long long SG_BUILD_INVALID_KEY = 1ULL << (2 * seedLen);
    for (; i < n; i += stride) {
        unsigned long long k = keys[i];
        if (k & SG_BUILD_INVALID_KEY) continue;
        if (i > 0 && keys[i - 1] == k) continue;
        long long e = i + 1;
        while (e < n && keys[e] == k) e++;
        unsigned long long count = (unsigned long long)(e - i);
        uint32_t value;
        if (count == 1) {
            value = locs[i];
        } else {
            unsigned long long off = atomicAdd(overflowCursor, count + 1);
            overflow[off] = (uint32_t)count;
            for (unsigned long long c = 0; c < count; c++) overflow[off + 1 + c] = locs[i + c];   // already descending
            value = (uint32_t)((unsigned long long)nBases + off);
        }
        if (buckets) {
            const unsigned long long rc = sg_seed_revcomp(k, seedLen);
            const unsigned long long c = k < rc ? k : rc;
            if (!sg_bucket_insert_atomic(buckets, nBuckets, 2 * seedLen, c, k == c ? 0u : 1u, value)) *failed = 1;
            continue;
        }
        const uint32_t table = (uint32_t)(k >> keyBits);
        if (!sg_table_insert_atomic(tables + tableStart[table], tableSize[table], k & ((1ULL << keyBits) - 1), value)) *failed = 1;
    }
}

// ---- key-range passes (a build whose sort scratch does not fit at once; snapgpu.cu build_index_on_device) ----
// A pass takes the valid seeds whose top 16 bits (the bin) lie in [binLo, binHi): all locations of a seed fall in one pass.

#define SG_BUILD_BINS 65536u

// the forward seed at loc, false if its bases are not all ACGT
__device__ __forceinline__ bool sg_build_seed_at(const uint8_t *bases, long long loc, uint32_t seedLen, unsigned long long *seed)
{
    unsigned long long b = 0;
    bool ok = true;
    for (uint32_t i = 0; i < seedLen; i++) {
        const uint32_t v = sg_base_value(bases[loc + i]);
        ok = ok && v < 4;
        b = (b << 2) | (v & 3);
    }
    *seed = b;
    return ok;
}

// valid seeds per bin, over all positions
__global__ void sg_build_histogram_kernel(const uint8_t *bases, long long nPositions, uint32_t seedLen, unsigned long long *bins)
{
    const uint32_t shift = 2 * seedLen - 16;
    long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; j < nPositions; j += stride) {
        unsigned long long s;
        if (sg_build_seed_at(bases, j, seedLen, &s)) atomicAdd(&bins[s >> shift], 1ULL);
    }
}

// Selection predicate over j = nPositions - 1 - location (descending locations, as sg_build_emit_kernel orders them).
struct SgBuildPassSelect {
    const uint8_t *bases;
    long long nPositions;
    uint32_t seedLen, binLo, binHi;
    __device__ __forceinline__ bool operator()(uint32_t j) const
    {
        unsigned long long s;
        if (!sg_build_seed_at(bases, nPositions - 1 - (long long)j, seedLen, &s)) return false;
        const uint32_t bin = (uint32_t)(s >> (2 * seedLen - 16));
        return bin >= binLo && bin < binHi;
    }
};

// the selected j (in order) -> (seed, location) pairs for the sort
__global__ void sg_build_pass_keys_kernel(const uint8_t *bases, long long nPositions, uint32_t seedLen, long long n, uint32_t *locs, unsigned long long *keys)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const long long loc = nPositions - 1 - (long long)locs[i];
        unsigned long long s;
        sg_build_seed_at(bases, loc, seedLen, &s);
        keys[i] = s;
        locs[i] = (uint32_t)loc;
    }
}

// ---- saving a bucket index in the reference's layout, any key size, default or -large tables (snapgpu_index_save_ex) ----
// Every used bucket slot becomes (a value of) an entry of its table, its value unchanged (a location, or countOfBases + an offset
// into the index's own overflow table); sg_bucket.h has the mapping, the staging form and the packing.

// Entries per table in the target geometry.  Few tables: a per-block shared histogram, added to the global one once per block.
#define SG_RELAY_SHARED_TABLES 8192u
__global__ void sg_relay_count_kernel(const unsigned long long *buckets, unsigned long long nBuckets, uint32_t seedLen, uint32_t keyBytes, uint32_t large,
                                      uint32_t nTables, unsigned long long *used, int *failed)
{
    __shared__ uint32_t sUsed[SG_RELAY_SHARED_TABLES];
    const bool shared = nTables <= SG_RELAY_SHARED_TABLES;
    if (shared) for (uint32_t t = threadIdx.x; t < nTables; t += blockDim.x) sUsed[t] = 0;
    __syncthreads();
    const unsigned long long nSlots = nBuckets * SG_BUCKET_SLOTS;
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < nSlots; s += (unsigned long long)gridDim.x * blockDim.x) {
        uint32_t t; bool ok;
        if (sg_relay_counts((const uint64_t *)buckets, nBuckets, s, seedLen, keyBytes, large, &t, &ok)) {
            if (shared) atomicAdd(&sUsed[t], 1u); else atomicAdd(&used[t], 1ULL);
        }
        if (!ok) *failed = 1;
    }
    __syncthreads();
    if (shared) for (uint32_t t = threadIdx.x; t < nTables; t += blockDim.x) if (sUsed[t]) atomicAdd(&used[t], (unsigned long long)sUsed[t]);
}

// sg_relay_insert_seq with compare-and-swap: an 8-byte slot is claimed whole; a 16-byte slot is claimed (or found) by its key word,
// and the value this slot fills is then its own word (the two orientations of a -large entry come from two bucket slots).
__device__ __forceinline__ bool sg_relay_insert_atomic(uint8_t *stage, uint32_t stageBytes, uint64_t size, unsigned long long key, uint32_t which, uint32_t value)
{
    uint64_t idx = sg_fmix64(key) % size;
    for (unsigned long long nProbes = 0;;) {
        unsigned long long *p = (unsigned long long *)(stage + idx * stageBytes);
        if (stageBytes == 8) {
            if (atomicCAS(p, SG_RELAY_EMPTY8, (key << 32) | value) == SG_RELAY_EMPTY8) return true;
        } else {
            const unsigned long long prev = atomicCAS(p, 0ULL, key + 1);
            if (prev == 0 || prev == key + 1) { ((uint32_t *)(p + 1))[which] = value; return true; }
        }
        if (++nProbes > size + 5) return false;
        idx = sg_table_probe_next(idx, nProbes, size);
    }
}

// The entries of tables [tableLo, tableHi) into their staging slots: table t at slot tableStart[t] - rangeBase of `stage`.
__global__ void sg_relay_insert_kernel(const unsigned long long *buckets, unsigned long long nBuckets, uint32_t seedLen, uint32_t keyBytes, uint32_t large,
                                       uint32_t tableLo, uint32_t tableHi, const uint64_t *tableStart, const uint64_t *tableSize, uint64_t rangeBase,
                                       uint8_t *stage, uint32_t stageBytes, int *failed)
{
    const unsigned long long nSlots = nBuckets * SG_BUCKET_SLOTS;
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < nSlots; s += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long slot = buckets[s];
        if ((uint32_t)slot == 0xffffffffu) continue;
        uint32_t t, which; uint64_t key;
        if (!sg_relay_entry(slot, s / SG_BUCKET_SLOTS, nBuckets, seedLen, keyBytes, large, &t, &key, &which)) { *failed = 1; continue; }
        if (t < tableLo || t >= tableHi) continue;
        if (!sg_relay_insert_atomic(stage + (size_t)(tableStart[t] - rangeBase) * stageBytes, stageBytes, tableSize[t], key, which, (uint32_t)slot)) *failed = 1;
    }
}

__global__ void sg_relay_stage_clear_kernel(uint8_t *stage, uint32_t stageBytes, unsigned long long n)
{
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        sg_relay_stage_clear(stage + i * stageBytes, stageBytes);
}

// staging slots [0, n) -> file entries at their stride (6..14 bytes), back to back
__global__ void sg_relay_pack_kernel(const uint8_t *stage, uint32_t stageBytes, unsigned long long n, uint8_t *out, uint32_t keyBytes, uint32_t large)
{
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        sg_relay_pack(stage, stageBytes, i, out, keyBytes, large);
}

__global__ void sg_build_fill_kernel(unsigned long long *p, long long n, unsigned long long v)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) p[i] = v;
}
