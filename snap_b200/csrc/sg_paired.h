// sg_paired.h -- the per-pair state machine.  Scalar form, host+device.
// Restates IntersectingPairedEndAligner::align (reference SNAPLib/IntersectingPairedEndAligner.cpp:169-252):
// alignLandauVishkin (:254-1435: phase 1 seed lookups into four hit sets, phase 2 fuzzy set intersection walking the
// hits in descending genome order, phase 2a big-indel hints, phase 3 scoring by best-possible-score bucket with merge
// anchors), alignAffineGap (:2489-2969, phase 4), scoreLocation (:3283-3399), scoreLocationWithAffineGap (:3119-3282),
// HashTableHitSet (:3500-3817), MergeAnchor::checkMerge (:3820-3871), ScoreSet (:3873-3973), computeScoreLimit
// (:3975-3988); and ChimericPairedEndAligner::align (ChimericPairedEndAligner.cpp:126-448), which falls back to /
// cross-checks with the single-end aligner of sg_align.h.
// alignHamming (:1441-2487) is the same three phases with gapless (Hamming + end clipping) scoring
// (scoreLocationWithHammingDistance :3401-3497); it is restated here as the `hamming` mode of the same function.
// Configuration covered: no secondary results (-om unset).  ALT awareness is covered in full: the two score sets, firstALTResult
// (the best pair when it lies on ALT contigs and a non-ALT one is emitted; kept per pair, not written out: -ea is not supported) and
// the liftover of ALT pairs onto their primary contig (alignAffineGap :2865-2966).
#pragma once
#include <limits.h>
#include "sg_align.h"
#include "sg_cigar.h"

#define SG_MAX_MAX_SEEDS 30          // IntersectingPairedEndAligner.h:216
#define SG_PAIRED_MERGE_DIST 31      // maxMergeDistance, IntersectingPairedEndAligner.cpp:3990
#define SG_LOCATION_NOT_YET_SCORED (-2)
#define SG_MAX_AG_CANDIDATES 4096    // PairedAligner.cpp:570-573
// bit of sg_paired_align_stage1's return value: the last of the nLVCand phase-4 candidates it hands over is the pair's firstALTResult
#define SG_STAGE_ALT_RESULT 4

// Genome::getProjContigNumAtLocation, getContigProjSpan, getProjLocation, isProjContigRC (Genome.cpp:634-715) over SgIndexView::projStart /
// projRC / projOps.  Only called on an index with ALT contigs (projStart != NULL).
SG_HD int sg_proj_contig_num_at(const SgIndexView &ix, int64_t location)
{
    const int p = sg_contig_at(ix, ix.projStart[sg_contig_at(ix, location)]);
    return p < 0 ? -2 : p;           // no contig there (a contig without a liftover line): the reference's number then matches no contig either
}

SG_HD int64_t sg_contig_proj_span(const SgIndexView &ix, int contig)
{
    int64_t offset = 0;
    const uint32_t b = ix.projOps[contig], e = ix.projOps[contig + 1];
    for (uint32_t i = b; i < e; i++) {
        const char action = (char)(ix.projOps[i] & 0xff);
        const int64_t count = (int64_t)(ix.projOps[i] >> 8);
        if (i == b ? (action != 'S' && action != 'H') : (action == 'M' || action == 'I')) offset += count;
    }
    return offset;
}

// the bwa-postalt walk; `invalid` (InvalidGenomeLocation) inside a soft / hard clip of the ALT contig
SG_HD int64_t sg_proj_location(const SgIndexView &ix, int64_t location, int alnSpan, int64_t invalid)
{
    const int contig = sg_contig_at(ix, location);
    const int64_t begin = ix.contigStart[contig];
    const int64_t offset = !ix.projRC[contig] ? location - begin : sg_contig_proj_span(ix, contig) - (location - begin + alnSpan);
    int64_t projOffset = 0, x = 0, y = 0;        // x: primary (REF), y: ALT
    uint32_t i = ix.projOps[contig];
    const uint32_t e = ix.projOps[contig + 1];
    if (i < e && ((ix.projOps[i] & 0xff) == 'S' || (ix.projOps[i] & 0xff) == 'H')) i++;
    for (; i < e; i++) {
        const char action = (char)(ix.projOps[i] & 0xff);
        const int64_t count = (int64_t)(ix.projOps[i] >> 8);
        if (action == 'M') {
            if (y <= offset && offset < y + count) { projOffset = x + (offset - y); break; }
            x += count; y += count;
        } else if (action == 'D') {
            x += count;
        } else if (action == 'I') {
            if (y <= offset && offset < y + count) { projOffset = x; break; }
            y += count;
        } else if (action == 'S' || action == 'H') {
            if (y <= offset && offset < y + count) { projOffset = -1; break; }
            y += count;
        }
    }
    if (projOffset == -1) return invalid;
    return ix.projStart[contig] + projOffset;
}

SG_HD int sg_proj_contig_rc(const SgIndexView &ix, int64_t location) { return ix.projRC[sg_contig_at(ix, location)] ? SNAPGPU_RC : SNAPGPU_FORWARD; }

struct SgPairedParams {
    int32_t  minSpacing; uint32_t maxSpacing; uint32_t maxBigHits; uint32_t poolSize; uint32_t maxSeedsSingleEnd; uint32_t maxKForIndels;
    int32_t  forceSpacing, minScoreRealignment, minScoreGapRealignmentALT, minAGScoreImprovement, enableHammingScoringBaseAligner,
             useSoftClip, flattenMAPQAtOrBelow;
    uint32_t numSeedsFromCommandLine;   // min(MAX_MAX_SEEDS, -n)
    uint32_t maxSeedsToUse;             // ctor-time value sizing the hit sets
    // capacities of THIS worker's arena (<= the reference's poolSize / 4096): a pair that needs more is retried by a worker
    // with full-size pools (error code 4) -- results do not depend on the caps
    uint32_t poolCap, agCandCap;
    int32_t  stage2Packed;              // device tuning knob (no effect on results): SgAgParams.usePacked of stage 2 (1 loop-compact, 2 unrolled)
};

struct SgHitLookup {                 // HashTableLookup<unsigned>, IntersectingPairedEndAligner.h
    const uint32_t *hits;
    int64_t  nHits;
    int64_t  currentHitForIntersection;
    uint32_t seedOffset;
    uint32_t whichDisjointHitSet;
};

struct SgHitSet {                    // HashTableHitSet
    SgHitLookup *lookups;            // [maxSeeds]
    uint32_t *exhausted;             // [maxSeeds] DisjointHitSet::countOfExhaustedHits
    uint32_t *missCount;             // [maxSeeds]
    uint32_t nLookupsUsed;
    int      currentDisjointHitSet;
    int64_t  mostRecentLocationReturned;

    SG_HD void init() { nLookupsUsed = 0; currentDisjointHitSet = -1; }

    SG_HD void recordLookup(uint32_t seedOffset, int64_t nHits, const uint32_t *hits, bool beginsDisjointHitSet) {   // :3536-3576
        if (beginsDisjointHitSet) {
            currentDisjointHitSet++;
            exhausted[currentDisjointHitSet] = 0;
        }
        if (0 == nHits) {
            exhausted[currentDisjointHitSet]++;
        } else {
            SgHitLookup &lk = lookups[nLookupsUsed];
            lk.currentHitForIntersection = 0;
            lk.hits = hits;
            lk.nHits = nHits;
            lk.seedOffset = seedOffset;
            lk.whichDisjointHitSet = (uint32_t)currentDisjointHitSet;
            #pragma unroll 1
            while (lk.nHits > 0 && lk.hits[lk.nHits - 1] < lk.seedOffset) lk.nHits--;
            nLookupsUsed++;
        }
    }

    SG_HD static bool within(int64_t a, int64_t b, int64_t d) { int64_t x = a - b; if (x < 0) x = -x; return x <= d; }

    SG_HD uint32_t computeBestPossibleScoreForCurrentHit() {       // :3585-3625
        for (int i = 0; i <= currentDisjointHitSet; i++) missCount[i] = exhausted[i];
        for (uint32_t i = 0; i < nLookupsUsed; i++) {
            const SgHitLookup &lk = lookups[i];
            bool near = (lk.currentHitForIntersection != lk.nHits &&
                         within((int64_t)lk.hits[lk.currentHitForIntersection], mostRecentLocationReturned + lk.seedOffset, SG_PAIRED_MERGE_DIST)) ||
                        (lk.currentHitForIntersection != 0 &&
                         within((int64_t)lk.hits[lk.currentHitForIntersection - 1], mostRecentLocationReturned + lk.seedOffset, SG_PAIRED_MERGE_DIST));
            if (!near) missCount[lk.whichDisjointHitSet]++;
        }
        uint32_t best = 0;
        for (int i = 0; i <= currentDisjointHitSet; i++) if (missCount[i] > best) best = missCount[i];
        return best;
    }

    SG_HD bool getNextHitLessThanOrEqualTo(int64_t maxGenomeLocationToFind, int64_t *actualGenomeLocationFound, uint32_t *seedOffsetFound) {   // :3627-3716
        bool anyFound = false;
        int64_t bestLocationFound = 0;
        for (uint32_t i = 0; i < nLookupsUsed; i++) {
            SgHitLookup &lk = lookups[i];
            int64_t lo = lk.currentHitForIntersection, hi = lk.nHits - 1;
            const int64_t maxThisSeed = maxGenomeLocationToFind + lk.seedOffset;
            while (lo <= hi) {
                int64_t probe = (lo + hi) / 2;
                int64_t probeHit = lk.hits[probe];
                bool clause1 = probeHit <= maxThisSeed;
                bool clause2 = probe == 0;
                if (clause1 && (clause2 || (int64_t)lk.hits[probe - 1] > maxThisSeed)) {
                    if (probeHit - lk.seedOffset > bestLocationFound) {
                        anyFound = true;
                        mostRecentLocationReturned = *actualGenomeLocationFound = bestLocationFound = probeHit - lk.seedOffset;
                        *seedOffsetFound = lk.seedOffset;
                    }
                    lk.currentHitForIntersection = probe;
                    break;
                }
                if (probeHit > maxThisSeed) lo = probe + 1; else hi = probe - 1;
            }
            if (lo > hi) lk.currentHitForIntersection = lk.nHits;
        }
        return anyFound;
    }

    SG_HD bool getFirstHit(int64_t *genomeLocation, uint32_t *seedOffsetFound) {      // :3719-3747 (true = nothing found)
        bool anyFound = false;
        *genomeLocation = 0;
        for (uint32_t i = 0; i < nLookupsUsed; i++) {
            const SgHitLookup &lk = lookups[i];
            if (lk.nHits > 0 && (int64_t)(uint32_t)(lk.hits[0] - lk.seedOffset) > *genomeLocation) {
                mostRecentLocationReturned = *genomeLocation = (int64_t)(uint32_t)(lk.hits[0] - lk.seedOffset);
                *seedOffsetFound = lk.seedOffset;
                anyFound = true;
            }
        }
        return !anyFound;
    }

    SG_HD bool getNextLowerHit(int64_t *genomeLocation, uint32_t *seedOffsetFound) {   // :3749-3817
        int64_t foundLocation = 0;
        bool anyFound = false;
        for (uint32_t i = 0; i < nLookupsUsed; i++) {
            SgHitLookup &lk = lookups[i];
            int64_t hitLocation = 0;
            if (lk.nHits != lk.currentHitForIntersection) hitLocation = lk.hits[lk.currentHitForIntersection];
            if (lk.currentHitForIntersection != lk.nHits && hitLocation - lk.seedOffset == mostRecentLocationReturned) {
                lk.currentHitForIntersection++;
                if (lk.currentHitForIntersection == lk.nHits) continue;
                hitLocation = lk.hits[lk.currentHitForIntersection];
            }
            if (lk.currentHitForIntersection != lk.nHits) {
                if (foundLocation < hitLocation - lk.seedOffset && hitLocation >= (int64_t)lk.seedOffset) {
                    *genomeLocation = foundLocation = hitLocation - lk.seedOffset;
                    *seedOffsetFound = lk.seedOffset;
                    anyFound = true;
                }
            }
        }
        if (anyFound) mostRecentLocationReturned = foundLocation;
        return anyFound;
    }
};

struct SgMergeAnchor {               // MergeAnchor
    double  matchProbability;
    int64_t locationForReadWithMoreHits, locationForReadWithFewerHits;
    int     pairScore, pairAGScore;
};

struct SgMateCandidate {             // ScoringMateCandidate
    double   matchProbability;
    int64_t  readWithMoreHitsGenomeLocation;
    int64_t  largestBigIndelDetected;
    int      bestPossibleScore, score, scoreLimit;
    uint32_t seedOffset;
    int      genomeOffset, basesClippedBefore, basesClippedAfter, agScore, lvIndels, refSpan;
    uint8_t  usedAffineGapScoring, usedGaplessClipping;
};

struct SgScoringCandidate {          // ScoringCandidate
    double   matchProbability;
    int64_t  readWithFewerHitsGenomeLocation;
    int32_t  scoreListNext;          // pool index or -1
    int32_t  mergeAnchor;            // pool index or -1
    uint32_t scoringMateCandidateIndex, whichSetPair, seedOffset, bestPossibleScore;
    int      largestBigIndelDetected, basesClippedBefore, basesClippedAfter, agScore, lvIndels, refSpan;
    uint8_t  usedAffineGapScoring, usedGaplessClipping;
};

struct SgPairScoreSet {              // IntersectingPairedEndAligner::ScoreSet
    int64_t  bestResultGenomeLocation[2], bestResultOrigGenomeLocation[2];
    int      bestResultDirection[2];
    unsigned bestResultScore[2];
    int      bestResultUsedAffineGapScoring[2], bestResultBasesClippedBefore[2], bestResultBasesClippedAfter[2], bestResultAGScore[2],
             bestResultSeedOffset[2], bestResultLVIndels[2], bestResultUsedGaplessClipping[2], bestResultRefSpan[2];
    double   bestResultMatchProbability[2];
    double   probabilityOfBestPair, probabilityOfAllPairs;
    int      bestPairScore, bestPairAGScore;

    SG_HD void init(int64_t invalid) {
        for (int i = 0; i < 2; i++) {
            bestResultGenomeLocation[i] = invalid; bestResultOrigGenomeLocation[i] = invalid;
            bestResultScore[i] = (unsigned)SG_SCORE_ABOVE_LIMIT; bestResultDirection[i] = 0; bestResultUsedAffineGapScoring[i] = 0;
            bestResultBasesClippedBefore[i] = 0; bestResultBasesClippedAfter[i] = 0; bestResultAGScore[i] = 0; bestResultSeedOffset[i] = 0;
            bestResultLVIndels[i] = 0; bestResultMatchProbability[i] = 0.0; bestResultUsedGaplessClipping[i] = 0; bestResultRefSpan[i] = 0;
        }
        probabilityOfBestPair = 0; probabilityOfAllPairs = 0; bestPairScore = SG_TOO_BIG_SCORE; bestPairAGScore = 0;
    }
    SG_HD void initFrom(const snapgpu_paired_result *r) {
        for (int i = 0; i < 2; i++) {
            bestResultGenomeLocation[i] = r->location[i]; bestResultOrigGenomeLocation[i] = r->origLocation[i];
            bestResultScore[i] = (unsigned)r->score[i]; bestResultDirection[i] = r->direction[i];
            bestResultUsedAffineGapScoring[i] = r->usedAffineGapScoring[i]; bestResultBasesClippedBefore[i] = r->basesClippedBefore[i];
            bestResultBasesClippedAfter[i] = r->basesClippedAfter[i]; bestResultAGScore[i] = r->agScore[i]; bestResultSeedOffset[i] = r->seedOffset[i];
            bestResultLVIndels[i] = r->lvIndels[i]; bestResultMatchProbability[i] = r->matchProbability[i];
            bestResultUsedGaplessClipping[i] = r->usedGaplessClipping[i]; bestResultRefSpan[i] = r->refSpan[i];
        }
        probabilityOfBestPair = r->matchProbability[0] * r->matchProbability[1];
        probabilityOfAllPairs = r->probabilityAllPairs;
        bestPairScore = r->score[0] + r->score[1];
        bestPairAGScore = r->agScore[0] + r->agScore[1];
    }
    SG_HD void updateProbabilityOfAllPairs(double oldP) { double v = probabilityOfAllPairs - oldP; probabilityOfAllPairs = v > 0 ? v : 0; }   // :3873
    SG_HD void updateProbabilityOfBestPair(double newP, bool updateAll = true) { probabilityOfBestPair = newP; if (updateAll) probabilityOfAllPairs += probabilityOfBestPair; }
    SG_HD bool updateBestHitIfNeeded(int pairScore, int pairAGScore, double pairProbability, int fewerEndScore, int readWithMoreHits,
                                     int64_t fewerEndGenomeLocationOffset, const SgScoringCandidate *c, const SgMateCandidate *m) {   // :3878-3918
        probabilityOfAllPairs += pairProbability;
        const int f = 1 - readWithMoreHits, mo = readWithMoreHits;
        if (pairAGScore > bestPairAGScore || (pairAGScore == bestPairAGScore && pairProbability > probabilityOfBestPair)) {
            bestPairScore = pairScore; bestPairAGScore = pairAGScore; probabilityOfBestPair = pairProbability;
            bestResultGenomeLocation[f] = c->readWithFewerHitsGenomeLocation + fewerEndGenomeLocationOffset;
            bestResultGenomeLocation[mo] = m->readWithMoreHitsGenomeLocation + m->genomeOffset;
            bestResultOrigGenomeLocation[f] = c->readWithFewerHitsGenomeLocation;
            bestResultOrigGenomeLocation[mo] = m->readWithMoreHitsGenomeLocation;
            bestResultScore[f] = (unsigned)fewerEndScore; bestResultScore[mo] = (unsigned)m->score;
            // setPairDirection = {{FORWARD, RC}, {RC, FORWARD}}
            bestResultDirection[f] = (c->whichSetPair == 0) ? f : 1 - f;
            bestResultDirection[mo] = (c->whichSetPair == 0) ? mo : 1 - mo;
            bestResultUsedAffineGapScoring[f] = c->usedAffineGapScoring; bestResultUsedAffineGapScoring[mo] = m->usedAffineGapScoring;
            bestResultUsedGaplessClipping[f] = c->usedGaplessClipping; bestResultUsedGaplessClipping[mo] = m->usedGaplessClipping;
            bestResultBasesClippedBefore[f] = c->basesClippedBefore; bestResultBasesClippedAfter[f] = c->basesClippedAfter;
            bestResultBasesClippedBefore[mo] = m->basesClippedBefore; bestResultBasesClippedAfter[mo] = m->basesClippedAfter;
            bestResultAGScore[f] = c->agScore; bestResultAGScore[mo] = m->agScore;
            bestResultSeedOffset[f] = (int)c->seedOffset; bestResultSeedOffset[mo] = (int)m->seedOffset;
            bestResultMatchProbability[f] = c->matchProbability; bestResultMatchProbability[mo] = m->matchProbability;
            bestResultLVIndels[f] = c->lvIndels; bestResultLVIndels[mo] = m->lvIndels;
            bestResultRefSpan[f] = c->refSpan; bestResultRefSpan[mo] = m->refSpan;
            return true;
        }
        return false;
    }
    SG_HD bool updateBestHitIfNeededR(int pairScore, int pairAGScore, double pairProbability, const snapgpu_paired_result *n) {   // :3920-3948
        probabilityOfAllPairs += pairProbability;
        if (pairAGScore > bestPairAGScore || (pairAGScore == bestPairAGScore && pairProbability > probabilityOfBestPair)) {
            bestPairScore = pairScore; bestPairAGScore = pairAGScore; probabilityOfBestPair = pairProbability;
            for (int r = 0; r < 2; r++) {
                bestResultGenomeLocation[r] = n->location[r]; bestResultOrigGenomeLocation[r] = n->origLocation[r];
                bestResultScore[r] = (unsigned)n->score[r]; bestResultDirection[r] = n->direction[r];
                bestResultUsedAffineGapScoring[r] = n->usedAffineGapScoring[r]; bestResultUsedGaplessClipping[r] = n->usedGaplessClipping[r];
                bestResultBasesClippedBefore[r] = n->basesClippedBefore[r]; bestResultBasesClippedAfter[r] = n->basesClippedAfter[r];
                bestResultAGScore[r] = n->agScore[r]; bestResultSeedOffset[r] = n->seedOffset[r]; bestResultMatchProbability[r] = n->matchProbability[r];
                bestResultLVIndels[r] = n->lvIndels[r]; bestResultRefSpan[r] = n->refSpan[r];
            }
            return true;
        }
        return false;
    }
    SG_HDN void fillInResult(const SgTables &T, snapgpu_paired_result *r, const uint32_t *popularSeedsSkipped) const {   // :3951-3973
        const uint32_t p0 = popularSeedsSkipped[0], p1 = popularSeedsSkipped[1];    // (may alias r->popularSeedsSkipped)
        for (int w = 0; w < 2; w++) {
            r->location[w] = bestResultGenomeLocation[w]; r->origLocation[w] = bestResultOrigGenomeLocation[w];
            r->direction[w] = bestResultDirection[w];
            r->mapq[w] = sg_compute_mapq(T, probabilityOfAllPairs, probabilityOfBestPair, (int)(p0 + p1));
            r->status[w] = r->mapq[w] > SG_MAPQ_LIMIT_FOR_SINGLE_HIT ? SNAPGPU_SINGLE_HIT : SNAPGPU_MULTIPLE_HITS;
            r->score[w] = (int)bestResultScore[w]; r->clippingForReadAdjustment[w] = 0;
            r->usedAffineGapScoring[w] = bestResultUsedAffineGapScoring[w]; r->usedGaplessClipping[w] = bestResultUsedGaplessClipping[w];
            r->basesClippedBefore[w] = bestResultBasesClippedBefore[w]; r->basesClippedAfter[w] = bestResultBasesClippedAfter[w];
            r->agScore[w] = bestResultAGScore[w]; r->seedOffset[w] = bestResultSeedOffset[w]; r->lvIndels[w] = bestResultLVIndels[w];
            r->matchProbability[w] = bestResultMatchProbability[w];
            r->refSpan[w] = bestResultRefSpan[w];
        }
        r->popularSeedsSkipped[0] = p0; r->popularSeedsSkipped[1] = p1;
        r->probabilityAllPairs = probabilityOfAllPairs;
    }
};

// Per-worker scratch of the paired path.
struct SgPairedScratch {
    uint8_t *rcRead[2], *rcQual[2], *revRead[2][2];
    uint8_t *seedUsed;
    SgHitSet hitSets[2][2];
    SgScoringCandidate *candPool;    // [poolSize]
    SgMateCandidate *mates[2];       // [poolSize/2] each
    SgMergeAnchor *anchors;          // [poolSize]
    int32_t *scoreLists;             // [MAX_K + extraSearchDepth + 2] heads (pool index or -1)
    snapgpu_paired_result *lvCandidates;   // [agCandCap + 1]: the phase-4 candidates, then the pair's firstALTResult (SgPairedAligner::altResult)
    snapgpu_single_result *singleCandidates;   // [agCandCap] candidatesForAffineGap of the single-end Hamming pass
    uint8_t *agBt[2];                // the Chimeric aligner's own AffineGapVectorized objects used by the intersecting aligner
};

SG_HD size_t sg_paired_scratch_bytes(const SgParams &p, const SgPairedParams &pp)
{
    size_t agCols = sg_align_up((size_t)p.maxReadLen * 3 / 2 + 64, 64), agRows = (size_t)p.maxReadLen + SG_MAX_K + 1;
    size_t rl = sg_align_up((size_t)p.maxReadLen + 16, 256);
    size_t b = rl * 8 + sg_align_up(((size_t)p.maxReadLen + 7) / 8 + 128, 256);
    b += 4 * (sg_align_up(sizeof(SgHitLookup) * pp.maxSeedsToUse, 256) + 2 * sg_align_up(4 * (size_t)pp.maxSeedsToUse, 256));
    b += sg_align_up(sizeof(SgScoringCandidate) * (size_t)pp.poolCap, 256);
    b += 2 * sg_align_up(sizeof(SgMateCandidate) * (size_t)(pp.poolCap / 2), 256);
    b += sg_align_up(sizeof(SgMergeAnchor) * (size_t)pp.poolCap, 256);
    b += sg_align_up(4 * (SG_MAX_K + 64), 256);
    b += sg_align_up(sizeof(snapgpu_paired_result) * ((size_t)pp.agCandCap + 1), 256);
    b += sg_align_up(sizeof(snapgpu_single_result) * (size_t)pp.agCandCap, 256);
    b += 2 * sg_align_up(agRows * agCols, 256);
    return b;
}

SG_HD void sg_paired_scratch_carve(const SgParams &p, const SgPairedParams &pp, uint8_t *base, SgPairedScratch *s)
{
    size_t agCols = sg_align_up((size_t)p.maxReadLen * 3 / 2 + 64, 64), agRows = (size_t)p.maxReadLen + SG_MAX_K + 1;
    size_t rl = sg_align_up((size_t)p.maxReadLen + 16, 256);
    uint8_t *q = base;
    for (int r = 0; r < 2; r++) { s->rcRead[r] = q; q += rl; s->rcQual[r] = q; q += rl; s->revRead[r][0] = q; q += rl; s->revRead[r][1] = q; q += rl; }
    s->seedUsed = q; q += sg_align_up(((size_t)p.maxReadLen + 7) / 8 + 128, 256);
    for (int r = 0; r < 2; r++) for (int d = 0; d < 2; d++) {
        SgHitSet &h = s->hitSets[r][d];
        h.lookups = (SgHitLookup *)q; q += sg_align_up(sizeof(SgHitLookup) * pp.maxSeedsToUse, 256);
        h.exhausted = (uint32_t *)q; q += sg_align_up(4 * (size_t)pp.maxSeedsToUse, 256);
        h.missCount = (uint32_t *)q; q += sg_align_up(4 * (size_t)pp.maxSeedsToUse, 256);
        h.nLookupsUsed = 0; h.currentDisjointHitSet = -1; h.mostRecentLocationReturned = 0;
    }
    s->candPool = (SgScoringCandidate *)q; q += sg_align_up(sizeof(SgScoringCandidate) * (size_t)pp.poolCap, 256);
    for (int k = 0; k < 2; k++) { s->mates[k] = (SgMateCandidate *)q; q += sg_align_up(sizeof(SgMateCandidate) * (size_t)(pp.poolCap / 2), 256); }
    s->anchors = (SgMergeAnchor *)q; q += sg_align_up(sizeof(SgMergeAnchor) * (size_t)pp.poolCap, 256);
    s->scoreLists = (int32_t *)q; q += sg_align_up(4 * (SG_MAX_K + 64), 256);
    s->lvCandidates = (snapgpu_paired_result *)q; q += sg_align_up(sizeof(snapgpu_paired_result) * ((size_t)pp.agCandCap + 1), 256);
    s->singleCandidates = (snapgpu_single_result *)q; q += sg_align_up(sizeof(snapgpu_single_result) * (size_t)pp.agCandCap, 256);
    s->agBt[0] = q; q += sg_align_up(agRows * agCols, 256);
    s->agBt[1] = q; q += sg_align_up(agRows * agCols, 256);
}

// The IntersectingPairedEndAligner + ChimericPairedEndAligner member state for one pair.
struct SgPairedAligner {
    SgAligner *single;               // the Chimeric aligner's BaseAligner (its own scratch incl. its own AG traceback arrays)
    const SgIndexView *ix; const SgParams *pr; const SgPairedParams *pp; const SgTables *tb;
    SgPairedScratch ps;
    SgAgParams ag;
    int maxK;                        // IntersectingPairedEndAligner::maxK for this call
    const uint8_t *readData[2][2], *readQual[2][2];
    uint32_t readLen[2];
    uint32_t lowestFreeScoringCandidatePoolEntry, lowestFreeScoringMateCandidate[2], firstFreeMergeAnchor;
    int countOfHashTableLookups[2];
    int64_t totalHashTableHits[2][2];
    uint32_t readWithMoreHits, readWithFewerHits;
    int64_t invalidLocation;
    uint32_t lvCalls, agCalls;       // nLocationsScoredLandauVishkin / AffineGap
    int error;                       // 1: a pool overflowed (the reference soft_exit()s there)
    // working storage of align / alignLV / alignAffineGap (their stack objects in the reference): members, so that on the device
    // they are part of the per-warp state rather than per-thread stack
    SgPairScoreSet wsAll, wsNonAlt;
    snapgpu_single_result wsSingle[2];
    snapgpu_paired_result wsKey;

    SG_HD bool isALT(int64_t loc) const { return loc >= ix->altFirstLocation; }
    // the pair's firstALTResult.  Read only where its status is not NotFound -- but for popularSeedsSkipped, which the phase-4 emission takes
    // from it as it stands (:2842), so that one is reset per pair too
    SG_HD snapgpu_paired_result *altResult() const { return ps.lvCandidates + pp->agCandCap; }
    SG_HD bool isSeedUsed(int64_t i) const { return (ps.seedUsed[i / 8] & (1 << (i % 8))) != 0; }
    SG_HD void setSeedUsed(int64_t i) { ps.seedUsed[i / 8] |= (uint8_t)(1 << (i % 8)); }
    SG_HD static int setPairDirection(uint32_t whichSetPair, uint32_t whichRead) { return whichSetPair == 0 ? (int)whichRead : 1 - (int)whichRead; }

    // computeScoreLimit (:3975-3988); 64-bit arithmetic like the reference's GenomeDistance
    SG_HD int computeScoreLimit(bool nonALTAlignment, const SgPairScoreSet *all, const SgPairScoreSet *nonAlt, int64_t maxBigIndelSeen) const {
        const int64_t gap = pr->maxScoreGapToPreferNonAltAlignment;
        int64_t inner = nonALTAlignment ? (((int64_t)all->bestPairScore + gap) < (int64_t)nonAlt->bestPairScore ? ((int64_t)all->bestPairScore + gap) : (int64_t)nonAlt->bestPairScore)
                                        : ((int64_t)all->bestPairScore < ((int64_t)nonAlt->bestPairScore - gap) ? (int64_t)all->bestPairScore : ((int64_t)nonAlt->bestPairScore - gap));
        int64_t a = (int64_t)maxK + maxBigIndelSeen;
        int64_t v = (int64_t)pr->extraSearchDepth + (a < inner ? a : inner);
        return (int)(v < SG_MAX_K - 1 ? v : SG_MAX_K - 1);
    }
};

// IntersectingPairedEndAligner::scoreLocationWithAffineGap (:3119-3282).  useAltLiftover is always false here.
template <int AGM = 0>
SG_HDN void sg_paired_score_location_ag(SgPairedAligner &P, uint32_t whichRead, int direction, int64_t genomeLocation, uint32_t seedOffset, int scoreLimit,
                                        int *score, double *matchProbability, int *genomeLocationOffset, int *basesClippedBefore, int *basesClippedAfter,
                                        int *agScore, int *genomeSpan)
{
    const SgIndexView &ix = *P.ix; const SgParams &pr = *P.pr; const SgTables &T = *P.tb;
    const int readLen = (int)P.readLen[whichRead];
    const int64_t genomeDataLength = (int64_t)readLen + SG_MAX_K;
    const uint8_t *data = sg_get_substring(ix, genomeLocation, genomeDataLength);
    *genomeLocationOffset = 0;
    *genomeSpan = 0;
    if (data == (const uint8_t *)0) { *score = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0; *genomeLocationOffset = 0; *agScore = SG_SCORE_ABOVE_LIMIT; return; }
    *basesClippedBefore = 0; *basesClippedAfter = 0;
    double matchProb1 = 1.0, matchProb2 = 1.0;
    int score1 = 0, score2 = 0;
    const int seedLen = (int)ix.seedLen;
    int agScore1 = seedLen, agScore2 = 0;
    const int tailStart = (int)seedOffset + seedLen;
    int textLen = (int)(genomeDataLength - tailStart), textRem = readLen - tailStart;
    const uint8_t *readToScore = P.readData[whichRead][direction], *qualToScore = P.readQual[whichRead][direction];
    // the intersecting aligner scores with the Chimeric aligner's AffineGapVectorized objects: their own traceback arrays
    SgScratch sc = P.single->sc;
    sc.agBt[0] = P.ps.agBt[0]; sc.agBt[1] = P.ps.agBt[1];
    SgAgResult ar;
    if (tailStart != readLen) {
        int patternLen = readLen - tailStart;
        bool banded = (patternLen >= (3 * (2 * scoreLimit + 1))) && !pr.noBandedAffineGap;
        ar.textOffset = textRem; ar.patternOffset = *basesClippedAfter; ar.nEdits = score1; ar.matchProbability = matchProb1; ar.agScore = -1;
        sg_ag_dispatch<AGM>(T, sc, P.ag, 1, banded, data + tailStart, textLen, readToScore + tailStart, qualToScore + tailStart, patternLen, scoreLimit, readLen,
                       direction != 0, P.pp->useSoftClip != 0, &ar, sg_lane());
        agScore1 = ar.agScore; textRem = ar.textOffset; *basesClippedAfter = ar.patternOffset; score1 = ar.nEdits; matchProb1 = ar.matchProbability;
        agScore1 += (seedLen - readLen);
        P.agCalls++;
    }
    if (score1 != SG_SCORE_ABOVE_LIMIT) {
        if (seedOffset != 0) {
            int limitLeft = scoreLimit - score1;
            int patternLen = (int)seedOffset;
            bool banded = (patternLen >= (3 * (2 * limitLeft + 1))) && !pr.noBandedAffineGap;
            ar.textOffset = *genomeLocationOffset; ar.patternOffset = *basesClippedBefore; ar.nEdits = score2; ar.matchProbability = matchProb2; ar.agScore = -1;
            sg_ag_dispatch<AGM>(T, sc, P.ag, -1, banded, data + seedOffset, (int)seedOffset + limitLeft, P.ps.revRead[whichRead][direction] + readLen - seedOffset,
                           P.readQual[whichRead][1 - direction] + readLen - seedOffset, patternLen, limitLeft, readLen, direction != 0,
                           P.pp->useSoftClip != 0, &ar, sg_lane());
            agScore2 = ar.agScore; *genomeLocationOffset = ar.textOffset; *basesClippedBefore = ar.patternOffset; score2 = ar.nEdits; matchProb2 = ar.matchProbability;
            agScore2 -= readLen;
            if (score2 == SG_SCORE_ABOVE_LIMIT) { *score = SG_SCORE_ABOVE_LIMIT; *genomeLocationOffset = 0; *agScore = -1; }
        }
    } else {
        *score = SG_SCORE_ABOVE_LIMIT; *genomeLocationOffset = 0; *agScore = -1;
    }
    if (score1 != SG_SCORE_ABOVE_LIMIT && score2 != SG_SCORE_ABOVE_LIMIT) {
        *score = score1 + score2;
        *matchProbability = matchProb1 * matchProb2 * T.snpPowSeedLen;
        *genomeSpan = ((int)seedOffset - *genomeLocationOffset) + seedLen + (readLen - tailStart - textRem);
        *agScore = agScore1 + agScore2;
    } else {
        *score = SG_SCORE_ABOVE_LIMIT; *agScore = -1; *matchProbability = 0.0;
    }
}

// IntersectingPairedEndAligner::scoreLocation (:3283-3399)
SG_HDN void sg_paired_score_location(SgPairedAligner &P, uint32_t whichRead, int direction, int64_t genomeLocation, uint32_t seedOffset, int scoreLimit,
                                     int *score, double *matchProbability, int *genomeLocationOffset, uint8_t *usedAffineGapScoring,
                                     int *basesClippedBefore, int *basesClippedAfter, int *agScore, int *totalIndelsLV, uint8_t *usedGaplessClipping, int *genomeSpan)
{
    const SgIndexView &ix = *P.ix; const SgParams &pr = *P.pr; const SgTables &T = *P.tb;
    if (pr.noUkkonen) scoreLimit = P.maxK + (int)pr.extraSearchDepth;
    const int readLen = (int)P.readLen[whichRead];
    const int64_t genomeDataLength = (int64_t)readLen + SG_MAX_K;
    const uint8_t *data = sg_get_substring(ix, genomeLocation, genomeDataLength);
    *genomeLocationOffset = 0; *genomeSpan = 0; *usedGaplessClipping = 0;
    if (data == (const uint8_t *)0) { *score = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0; *genomeLocationOffset = 0; *agScore = SG_SCORE_ABOVE_LIMIT; return; }
    *basesClippedBefore = 0; *basesClippedAfter = 0;
    double matchProb1 = 1.0, matchProb2 = 1.0;
    int score1 = 0, score2 = 0;
    const int seedLen = (int)ix.seedLen;
    const int tailStart = (int)seedOffset + seedLen;
    int agScore1 = seedLen, agScore2 = 0;
    const int textLen = (int)(genomeDataLength - tailStart);
    int totalIndels1 = 0, totalIndels2 = 0, textSpan1 = 0, textSpan2 = 0;
    const uint8_t *readToScore = P.readData[whichRead][direction], *qualToScore = P.readQual[whichRead][direction];
    P.lvCalls++;
    SgLvResult lv;
    sg_lv_compute(T, P.single->sc, 1, data + tailStart, textLen, readToScore + tailStart, qualToScore + tailStart, readLen - tailStart, scoreLimit, &lv, sg_lane());
    score1 = lv.score; matchProb1 = lv.matchProbability; totalIndels1 = lv.totalIndels; textSpan1 = lv.textSpan;
    agScore1 = (seedLen + readLen - tailStart - score1) * pr.matchReward - score1 * pr.subPenalty;
    if (score1 != SG_SCORE_ABOVE_LIMIT) {
        int limitLeft = scoreLimit - score1;
        sg_lv_compute(T, P.single->sc, -1, data + seedOffset, (int)seedOffset + SG_MAX_K, P.ps.revRead[whichRead][direction] + readLen - seedOffset,
                      P.readQual[whichRead][1 - direction] + readLen - seedOffset, (int)seedOffset, limitLeft, &lv, sg_lane());
        score2 = lv.score; matchProb2 = lv.matchProbability; *genomeLocationOffset = lv.netIndel; totalIndels2 = lv.totalIndels; textSpan2 = lv.textSpan;
        agScore2 = ((int)seedOffset - score2) * pr.matchReward - score2 * pr.subPenalty;
    }
    if (0 != *genomeLocationOffset && (const uint8_t *)0 == sg_get_substring(ix, genomeLocation + *genomeLocationOffset, genomeDataLength)) {
        score2 = SG_SCORE_ABOVE_LIMIT;
    }
    if (score1 != SG_SCORE_ABOVE_LIMIT && score2 != SG_SCORE_ABOVE_LIMIT) {
        *score = score1 + score2;
        *matchProbability = matchProb1 * matchProb2 * T.snpPowSeedLen;
        *agScore = agScore1 + agScore2;
        *genomeSpan = textSpan1 + seedLen + textSpan2;
        *totalIndelsLV = totalIndels1 + totalIndels2;
    } else {
        *score = SG_SCORE_ABOVE_LIMIT; *agScore = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0.0;
    }
    if (pr.noEditDistance) {         // -ne: score with affine gap too and throw the result away (:3390-3398)
        int ts, tag, off, cb, ca, span; double mp;
        sg_paired_score_location_ag(P, whichRead, direction, genomeLocation, seedOffset, scoreLimit, &ts, &mp, &off, &cb, &ca, &tag, &span);
    }
    (void)usedAffineGapScoring;
}

// IntersectingPairedEndAligner::scoreLocationWithHammingDistance (:3401-3497).  Note what it does NOT set: the clip counts
// stay 0 (the gapless scorer's pattern offsets go to locals), only the reverse extension's text offset is returned.
SG_HDN void sg_paired_score_location_hamming(SgPairedAligner &P, uint32_t whichRead, int direction, int64_t genomeLocation, uint32_t seedOffset, int scoreLimit,
                                             int *score, double *matchProbability, int *genomeLocationOffset, int *basesClippedBefore, int *basesClippedAfter,
                                             int *agScore, uint8_t *usedGaplessClipping, int *scoreGapless)
{
    const SgIndexView &ix = *P.ix; const SgParams &pr = *P.pr; const SgTables &T = *P.tb;
    if (pr.noUkkonen) scoreLimit = P.maxK + (int)pr.extraSearchDepth;
    const int readLen = (int)P.readLen[whichRead];
    const int64_t genomeDataLength = (int64_t)readLen + SG_MAX_K;
    const uint8_t *data = sg_get_substring(ix, genomeLocation, genomeDataLength);
    *genomeLocationOffset = 0;
    *usedGaplessClipping = 0;
    if (data == (const uint8_t *)0) { *score = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0; *genomeLocationOffset = 0; *agScore = SG_SCORE_ABOVE_LIMIT; return; }
    *basesClippedBefore = 0; *basesClippedAfter = 0;
    double matchProb1 = 1.0, matchProb2 = 1.0;
    int score1 = 0, score2 = 0;
    const int seedLen = (int)ix.seedLen;
    const int tailStart = (int)seedOffset + seedLen;
    int agScore1 = seedLen, agScore2 = 0;
    const int textLen = (int)(genomeDataLength - tailStart);
    int score1Gapless = 0, score2Gapless = 0;
    SgGaplessOut g;
    if (tailStart != readLen) {
        g.nEdits = score1; g.matchProbability = matchProb1; g.nEditsGapless = score1Gapless;
        agScore1 = sg_gapless_compute(T, P.ag, 1, data + tailStart, textLen, P.readData[whichRead][direction] + tailStart, P.readQual[whichRead][direction] + tailStart,
                                      readLen - tailStart, readLen, scoreLimit, &g);
        score1 = g.nEdits; matchProb1 = g.matchProbability; score1Gapless = g.nEditsGapless;
        agScore1 += (seedLen - readLen);
    }
    if (score1Gapless != SG_SCORE_ABOVE_LIMIT) {
        int limitLeft = scoreLimit - score1Gapless;
        if (seedOffset != 0) {
            g.nEdits = score2; g.matchProbability = matchProb2; g.nEditsGapless = score2Gapless; g.textOffset = *genomeLocationOffset;
            agScore2 = sg_gapless_compute(T, P.ag, -1, data + seedOffset, (int)seedOffset + SG_MAX_K, P.ps.revRead[whichRead][direction] + readLen - seedOffset,
                                          P.readQual[whichRead][1 - direction] + readLen - seedOffset, (int)seedOffset, readLen, limitLeft, &g);
            score2 = g.nEdits; matchProb2 = g.matchProbability; score2Gapless = g.nEditsGapless; *genomeLocationOffset = g.textOffset;
            agScore2 -= readLen;
            if (score2Gapless == SG_SCORE_ABOVE_LIMIT) { *score = SG_SCORE_ABOVE_LIMIT; *genomeLocationOffset = 0; *agScore = SG_SCORE_ABOVE_LIMIT; }
        }
    }
    if (score1Gapless != SG_SCORE_ABOVE_LIMIT && score2Gapless != SG_SCORE_ABOVE_LIMIT) {
        *score = score1 + score2;
        *matchProbability = matchProb1 * matchProb2 * T.snpPowSeedLen;
        *agScore = agScore1 + agScore2;
        *scoreGapless = score1Gapless + score2Gapless;
        *usedGaplessClipping = 1;
    } else {
        *score = SG_SCORE_ABOVE_LIMIT; *agScore = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0.0; *scoreGapless = SG_SCORE_ABOVE_LIMIT;
    }
}

SG_HD void sg_paired_fill_candidate_result(snapgpu_paired_result *r, const SgPairedAligner &P, const SgScoringCandidate *c, const SgMateCandidate *m,
                                           int fewerEndScore, int fewerEndGenomeLocationOffset, const uint32_t *popularSeedsSkipped)
{
    const uint32_t mo = P.readWithMoreHits, f = P.readWithFewerHits;
    r->alignedAsPair = 1;
    r->direction[mo] = SgPairedAligner::setPairDirection(c->whichSetPair, mo);
    r->direction[f] = SgPairedAligner::setPairDirection(c->whichSetPair, f);
    r->location[mo] = m->readWithMoreHitsGenomeLocation + m->genomeOffset;
    r->location[f] = c->readWithFewerHitsGenomeLocation + fewerEndGenomeLocationOffset;
    r->origLocation[mo] = m->readWithMoreHitsGenomeLocation;
    r->origLocation[f] = c->readWithFewerHitsGenomeLocation;
    r->mapq[0] = r->mapq[1] = 0;
    r->score[mo] = m->score; r->score[f] = fewerEndScore;
    r->status[f] = r->status[mo] = SNAPGPU_MULTIPLE_HITS;
    r->usedAffineGapScoring[mo] = m->usedAffineGapScoring; r->usedAffineGapScoring[f] = c->usedAffineGapScoring;
    r->usedGaplessClipping[mo] = m->usedGaplessClipping; r->usedGaplessClipping[f] = c->usedGaplessClipping;
    r->basesClippedBefore[f] = c->basesClippedBefore; r->basesClippedAfter[f] = c->basesClippedAfter;
    r->basesClippedBefore[mo] = m->basesClippedBefore; r->basesClippedAfter[mo] = m->basesClippedAfter;
    r->agScore[mo] = m->agScore; r->agScore[f] = c->agScore;
    r->seedOffset[mo] = (int)m->seedOffset; r->seedOffset[f] = (int)c->seedOffset;
    r->lvIndels[mo] = m->lvIndels; r->lvIndels[f] = c->lvIndels;
    r->matchProbability[mo] = m->matchProbability; r->matchProbability[f] = c->matchProbability;
    r->popularSeedsSkipped[mo] = popularSeedsSkipped[mo]; r->popularSeedsSkipped[f] = popularSeedsSkipped[f];
    // refSpan is NOT filled in for these records by the reference (:1134-1163): it keeps whatever the buffer slot held
}

SG_HD void sg_paired_fill_best_result(snapgpu_paired_result *r, const SgPairScoreSet &s, const uint32_t *popularSeedsSkipped)
{
    r->alignedAsPair = 1;
    for (int k = 0; k < 2; k++) {
        r->direction[k] = s.bestResultDirection[k]; r->location[k] = s.bestResultGenomeLocation[k]; r->origLocation[k] = s.bestResultOrigGenomeLocation[k];
        r->mapq[k] = 0; r->score[k] = (int)s.bestResultScore[k]; r->status[k] = SNAPGPU_MULTIPLE_HITS;
        r->usedAffineGapScoring[k] = s.bestResultUsedAffineGapScoring[k]; r->basesClippedBefore[k] = s.bestResultBasesClippedBefore[k];
        r->basesClippedAfter[k] = s.bestResultBasesClippedAfter[k]; r->agScore[k] = s.bestResultAGScore[k]; r->seedOffset[k] = s.bestResultSeedOffset[k];
        r->popularSeedsSkipped[k] = popularSeedsSkipped[k]; r->lvIndels[k] = s.bestResultLVIndels[k]; r->matchProbability[k] = s.bestResultMatchProbability[k];
        r->usedGaplessClipping[k] = s.bestResultUsedGaplessClipping[k]; r->refSpan[k] = s.bestResultRefSpan[k];
    }
}

// IntersectingPairedEndAligner::alignLandauVishkin (:254-1435) and, with hamming = true, ::alignHamming (:1441-2487): the same
// function but for the scorer, the missing phase 2a and a few conditions.  Returns false if the phase-4 candidate buffer overflowed.
SG_HDN bool sg_paired_align_lv(SgPairedAligner &P, const uint8_t *const readBases[2], const uint8_t *const readQuals[2], const uint32_t lens[2],
                               snapgpu_paired_result *result, int *nLVCandidatesForAffineGap, bool hamming = false)
{
    const SgIndexView &ix = *P.ix; const SgParams &pr = *P.pr; const SgPairedParams &pp = *P.pp; const SgTables &T = *P.tb;
    SgPairedScratch &ps = P.ps;
    const uint32_t seedLen = ix.seedLen;
    const int maxK = P.maxK;
    const int esd = (int)pr.extraSearchDepth;
    const int maxLVCand = pr.useAffineGap ? (int)pp.agCandCap : 0;
    snapgpu_paired_result *alt = P.altResult();

    alt->status[0] = alt->status[1] = SNAPGPU_NOT_FOUND;
    if (!hamming) alt->refSpan[0] = alt->refSpan[1] = 0;
    result->clippingForReadAdjustment[0] = result->clippingForReadAdjustment[1] = 0;
    result->usedAffineGapScoring[0] = result->usedAffineGapScoring[1] = 0;
    result->basesClippedBefore[0] = result->basesClippedBefore[1] = 0;
    result->basesClippedAfter[0] = result->basesClippedAfter[1] = 0;
    result->agScore[0] = result->agScore[1] = 0;
    result->usedGaplessClipping[0] = result->usedGaplessClipping[1] = 0;
    if (!hamming) {
        result->refSpan[0] = result->refSpan[1] = 0;
        result->liftover[0] = result->liftover[1] = 0;
    }
    *nLVCandidatesForAffineGap = 0;

    int maxSeeds;
    if (pp.numSeedsFromCommandLine != 0) maxSeeds = (int)pp.numSeedsFromCommandLine;
    else maxSeeds = (int)((lens[0] > lens[1] ? lens[0] : lens[1]) * pr.seedCoverage / (int)seedLen);

    P.lowestFreeScoringCandidatePoolEntry = 0;
    for (int k = 0; k <= maxK + esd; k++) ps.scoreLists[k] = -1;
    P.lowestFreeScoringMateCandidate[0] = P.lowestFreeScoringMateCandidate[1] = 0;
    P.firstFreeMergeAnchor = 0;

    SgPairScoreSet &all = P.wsAll, &nonAlt = P.wsNonAlt;
    all.init(P.invalidLocation); nonAlt.init(P.invalidLocation);
    uint32_t popularSeedsSkipped[2];

    if (lens[0] < seedLen || lens[1] < seedLen) return true;

    uint32_t countOfNs = 0;
    for (uint32_t w = 0; w < 2; w++) {
        P.readLen[w] = lens[w];
        popularSeedsSkipped[w] = 0;
        P.countOfHashTableLookups[w] = 0;
        for (int d = 0; d < 2; d++) { P.totalHashTableHits[w][d] = 0; ps.hitSets[w][d].init(); }
        P.readData[w][0] = readBases[w]; P.readQual[w][0] = readQuals[w];
        P.readData[w][1] = ps.rcRead[w]; P.readQual[w][1] = ps.rcQual[w];
#if defined(__CUDA_ARCH__)
        // the derived strings (:347-372) are built 32 bases per step; every lane reads all of them afterwards
        #pragma unroll 1
        for (uint32_t i = (uint32_t)sg_lane(); i < lens[w]; i += 32) {
            const uint8_t b = readBases[w][i], c = sg_complement(b);
            ps.rcRead[w][lens[w] - i - 1] = c;
            ps.rcQual[w][lens[w] - i - 1] = readQuals[w][i];
            ps.revRead[w][0][lens[w] - i - 1] = b;
            ps.revRead[w][1][i] = c;
            countOfNs += (b == 'N') ? 1u : 0u;
        }
#else
        for (uint32_t i = 0; i < lens[w]; i++) {
            const uint8_t b = readBases[w][i], c = sg_complement(b);
            ps.rcRead[w][lens[w] - i - 1] = c;
            ps.rcQual[w][lens[w] - i - 1] = readQuals[w][i];
            ps.revRead[w][0][lens[w] - i - 1] = b;
            ps.revRead[w][1][i] = c;
            countOfNs += (b == 'N') ? 1u : 0u;
        }
#endif
    }
#if defined(__CUDA_ARCH__)
    countOfNs = __reduce_add_sync(0xffffffffu, countOfNs);
    __syncwarp();
#endif
    if ((int)countOfNs > maxK) return true;

    // ---- Phase 1: hash table lookups (:409-502) ----
    for (uint32_t w = 0; w < 2; w++) {
        int nextSeedToTest = 0;
        uint32_t wrapCount = 0;
        const int nPossibleSeeds = (int)lens[w] - (int)seedLen + 1;
        {
            const uint32_t ml = lens[0] > lens[1] ? lens[0] : lens[1];
#if defined(__CUDA_ARCH__)
            __syncwarp();
            for (uint32_t i = (uint32_t)sg_lane(); i < (ml + 7) / 8; i += 32) ps.seedUsed[i] = 0;
            __syncwarp();
#else
            for (uint32_t i = 0; i < (ml + 7) / 8; i++) ps.seedUsed[i] = 0;
#endif
        }
        bool beginsDisjointHitSet[2] = {true, true};
        while (P.countOfHashTableLookups[w] < nPossibleSeeds && P.countOfHashTableLookups[w] < maxSeeds) {
            if (nextSeedToTest >= nPossibleSeeds) {
                wrapCount++;
                beginsDisjointHitSet[0] = beginsDisjointHitSet[1] = true;
                if (wrapCount >= seedLen) break;
                nextSeedToTest = (int)T.wrapSeed[wrapCount];
            }
            while (nextSeedToTest < nPossibleSeeds && P.isSeedUsed(nextSeedToTest)) nextSeedToTest++;
            if (nextSeedToTest >= nPossibleSeeds) continue;
            P.setSeedUsed(nextSeedToTest);
            uint64_t sb, srcb;
            SgHits hits;
#if defined(__CUDA_ARCH__)
            if (!sg_warp_seed_pack(readBases[w] + nextSeedToTest, seedLen, sg_lane(), &sb, &srcb)) { nextSeedToTest++; continue; }
            sg_warp_lookup_seed32(ix, sb, srcb, sg_lane(), &hits, &P.single->work.entriesProbed, &P.single->work.overflowWords);
#else
            if (!sg_seed_pack(readBases[w] + nextSeedToTest, seedLen, &sb, &srcb)) { nextSeedToTest++; continue; }
            sg_lookup_seed32(ix, sb, srcb, &hits, &P.single->work.entriesProbed, &P.single->work.overflowWords);
#endif
            P.single->work.lookups++;
            P.countOfHashTableLookups[w]++;
            for (int dir = 0; dir < 2; dir++) {
                int offset = (dir == 0) ? nextSeedToTest : (int)lens[w] - (int)seedLen - nextSeedToTest;
                if ((int64_t)hits.nHits[dir] < (int64_t)pp.maxBigHits) {
                    P.totalHashTableHits[w][dir] += hits.nHits[dir];
                    ps.hitSets[w][dir].recordLookup((uint32_t)offset, hits.nHits[dir], hits.hits[dir], beginsDisjointHitSet[dir]);
                    beginsDisjointHitSet[dir] = false;
                } else {
                    popularSeedsSkipped[w]++;
                }
            }
            if ((maxSeeds - P.countOfHashTableLookups[w] + 1) * (int)seedLen + nextSeedToTest < nPossibleSeeds) {
                nextSeedToTest += (nPossibleSeeds - nextSeedToTest - 1) / (maxSeeds - P.countOfHashTableLookups[w] + 1);
            } else {
                nextSeedToTest += (int)seedLen;
            }
        }
    }

    P.readWithMoreHits = (P.totalHashTableHits[0][0] + P.totalHashTableHits[0][1] > P.totalHashTableHits[1][0] + P.totalHashTableHits[1][1]) ? 0u : 1u;
    P.readWithFewerHits = 1 - P.readWithMoreHits;
    const uint32_t MORE = P.readWithMoreHits, FEWER = P.readWithFewerHits;
    const int64_t maxSpacing = (int64_t)pp.maxSpacing;

    // ---- Phase 2: candidates from the fuzzy intersection of the hit sets (:530-717) ----
    int maxUsedBestPossibleScoreList = 0;
    for (uint32_t whichSetPair = 0; whichSetPair < 2; whichSetPair++) {
        SgHitSet *setPair[2];
        if (whichSetPair == 0) { setPair[0] = &ps.hitSets[0][0]; setPair[1] = &ps.hitSets[1][1]; }
        else { setPair[0] = &ps.hitSets[0][1]; setPair[1] = &ps.hitSets[1][0]; }
        uint32_t lastSeedOffsetForReadWithFewerHits = 0, lastSeedOffsetForReadWithMoreHits = 0;
        int64_t lastGenomeLocationForReadWithFewerHits, lastGenomeLocationForReadWithMoreHits;
        bool outOfMoreHitsLocations = false;
        if (setPair[FEWER]->getFirstHit(&lastGenomeLocationForReadWithFewerHits, &lastSeedOffsetForReadWithFewerHits)) continue;
        lastGenomeLocationForReadWithMoreHits = P.invalidLocation;
        SgMateCandidate *mates = ps.mates[whichSetPair];
        for (;;) {
            if (lastGenomeLocationForReadWithMoreHits > lastGenomeLocationForReadWithFewerHits + maxSpacing) {
                if (!setPair[MORE]->getNextHitLessThanOrEqualTo(lastGenomeLocationForReadWithFewerHits + maxSpacing,
                                                                &lastGenomeLocationForReadWithMoreHits, &lastSeedOffsetForReadWithMoreHits)) break;
            }
            if ((lastGenomeLocationForReadWithMoreHits + maxSpacing < lastGenomeLocationForReadWithFewerHits || outOfMoreHitsLocations) &&
                (0 == P.lowestFreeScoringMateCandidate[whichSetPair] ||
                 !SgHitSet::within(mates[P.lowestFreeScoringMateCandidate[whichSetPair] - 1].readWithMoreHitsGenomeLocation, lastGenomeLocationForReadWithFewerHits, maxSpacing))) {
                if (outOfMoreHitsLocations) break;
                if (!setPair[FEWER]->getNextHitLessThanOrEqualTo(lastGenomeLocationForReadWithMoreHits + maxSpacing, &lastGenomeLocationForReadWithFewerHits,
                                                                 &lastSeedOffsetForReadWithFewerHits)) break;
                continue;
            }
            while (lastGenomeLocationForReadWithMoreHits + maxSpacing >= lastGenomeLocationForReadWithFewerHits && !outOfMoreHitsLocations) {
                uint32_t bestPossibleScoreForReadWithMoreHits = pr.noTruncation ? 0u : setPair[MORE]->computeBestPossibleScoreForCurrentHit();
                if (P.lowestFreeScoringMateCandidate[whichSetPair] >= pp.poolCap / 2) { P.error = pp.poolCap < pp.poolSize ? 4 : 1; return true; }
                SgMateCandidate &m = mates[P.lowestFreeScoringMateCandidate[whichSetPair]];
                m.readWithMoreHitsGenomeLocation = lastGenomeLocationForReadWithMoreHits;
                m.bestPossibleScore = (int)bestPossibleScoreForReadWithMoreHits;
                m.seedOffset = lastSeedOffsetForReadWithMoreHits;
                m.score = SG_LOCATION_NOT_YET_SCORED; m.scoreLimit = -1; m.matchProbability = 0; m.genomeOffset = 0;
                m.usedAffineGapScoring = 0; m.usedGaplessClipping = 0; m.basesClippedBefore = 0; m.basesClippedAfter = 0; m.agScore = 0; m.lvIndels = 0;
                m.largestBigIndelDetected = 0;       // noMaxKForIndel is not exposed
                m.refSpan = 0;
                P.lowestFreeScoringMateCandidate[whichSetPair]++;
                if (!setPair[MORE]->getNextLowerHit(&lastGenomeLocationForReadWithMoreHits, &lastSeedOffsetForReadWithMoreHits)) {
                    lastGenomeLocationForReadWithMoreHits = 0;
                    outOfMoreHitsLocations = true;
                    break;
                }
            }
            int bestPossibleScoreForReadWithFewerHits = pr.noTruncation ? 0 : (int)setPair[FEWER]->computeBestPossibleScoreForCurrentHit();
            int lowestBestPossibleScoreOfAnyPossibleMate = maxK + esd;
            for (int i = (int)P.lowestFreeScoringMateCandidate[whichSetPair] - 1; i >= 0; i--) {
                if (mates[i].readWithMoreHitsGenomeLocation > lastGenomeLocationForReadWithFewerHits + maxSpacing) break;
                if (mates[i].bestPossibleScore < lowestBestPossibleScoreOfAnyPossibleMate) lowestBestPossibleScoreOfAnyPossibleMate = mates[i].bestPossibleScore;
            }
            if (lowestBestPossibleScoreOfAnyPossibleMate + bestPossibleScoreForReadWithFewerHits <= maxK + esd) {
                if (P.lowestFreeScoringCandidatePoolEntry >= pp.poolCap) { P.error = pp.poolCap < pp.poolSize ? 4 : 1; return true; }
                int bestPossibleScore = pr.noOrderedEvaluation ? 0 : lowestBestPossibleScoreOfAnyPossibleMate + bestPossibleScoreForReadWithFewerHits;
                SgScoringCandidate &c = ps.candPool[P.lowestFreeScoringCandidatePoolEntry];
                c.readWithFewerHitsGenomeLocation = lastGenomeLocationForReadWithFewerHits;
                c.whichSetPair = whichSetPair;
                c.scoringMateCandidateIndex = P.lowestFreeScoringMateCandidate[whichSetPair] - 1;
                c.seedOffset = lastSeedOffsetForReadWithFewerHits;
                c.bestPossibleScore = (uint32_t)bestPossibleScoreForReadWithFewerHits;
                c.scoreListNext = ps.scoreLists[bestPossibleScore];
                c.mergeAnchor = -1;
                c.usedAffineGapScoring = 0; c.usedGaplessClipping = 0; c.basesClippedBefore = 0; c.basesClippedAfter = 0; c.agScore = 0; c.lvIndels = 0;
                c.matchProbability = 1.0; c.largestBigIndelDetected = 0; c.refSpan = 0;
                ps.scoreLists[bestPossibleScore] = (int32_t)P.lowestFreeScoringCandidatePoolEntry;
                P.lowestFreeScoringCandidatePoolEntry++;
                if (bestPossibleScore > maxUsedBestPossibleScoreList) maxUsedBestPossibleScoreList = bestPossibleScore;
            }
            if (!setPair[FEWER]->getNextLowerHit(&lastGenomeLocationForReadWithFewerHits, &lastSeedOffsetForReadWithFewerHits)) break;
        }
    }

    // ---- Phase 2a: big-indel hints (:723-801) ----
    const int64_t maxKForIndels = (int64_t)pp.maxKForIndels;
    for (int whichSetPair = 0; whichSetPair < 2 && !hamming; whichSetPair++) {
        SgMateCandidate *mates = ps.mates[whichSetPair];
        int bottom = 0, top = 1;
        while (top < (int)P.lowestFreeScoringMateCandidate[whichSetPair]) {
            int64_t spread = mates[bottom].readWithMoreHitsGenomeLocation - mates[top].readWithMoreHitsGenomeLocation; if (spread < 0) spread = -spread;
            if (spread < maxKForIndels) {
                if (spread > mates[bottom].largestBigIndelDetected) mates[bottom].largestBigIndelDetected = spread;
                if (spread > mates[top].largestBigIndelDetected) mates[top].largestBigIndelDetected = spread;
                top++;
            } else if (bottom < top - 1) {
                bottom++;
            } else {
                bottom++; top++;
            }
        }
    }
    if (!hamming) {
        int bottom = 0, top = 1;
        while (top < (int)P.lowestFreeScoringCandidatePoolEntry) {
            if (ps.candPool[bottom].whichSetPair != ps.candPool[top].whichSetPair) { bottom = top; top = top + 1; continue; }
            int64_t spread = ps.candPool[bottom].readWithFewerHitsGenomeLocation - ps.candPool[top].readWithFewerHitsGenomeLocation; if (spread < 0) spread = -spread;
            if (spread < maxKForIndels) {
                if ((int)spread > ps.candPool[bottom].largestBigIndelDetected) ps.candPool[bottom].largestBigIndelDetected = (int)spread;
                if ((int)spread > ps.candPool[top].largestBigIndelDetected) ps.candPool[top].largestBigIndelDetected = (int)spread;
                top++;
            } else if (bottom < top - 1) {
                bottom++;
            } else {
                bottom++; top++;
            }
        }
    }

    // ---- Phase 3: score and merge (:806-1206) ----
    int currentBestPossibleScoreList = 0;
    bool doneScoring = false;
    for (;;) {
        int a1 = all.bestPairScore < nonAlt.bestPairScore - pr.maxScoreGapToPreferNonAltAlignment ? all.bestPairScore : nonAlt.bestPairScore - pr.maxScoreGapToPreferNonAltAlignment;
        int a2 = all.bestPairScore + pr.maxScoreGapToPreferNonAltAlignment < nonAlt.bestPairScore ? all.bestPairScore + pr.maxScoreGapToPreferNonAltAlignment : nonAlt.bestPairScore;
        int worst = a1 > a2 ? a1 : a2;
        if (!(currentBestPossibleScoreList <= maxUsedBestPossibleScoreList &&
              (unsigned)currentBestPossibleScoreList <= pr.extraSearchDepth + (unsigned)(maxK < worst ? maxK : worst))) break;
        if (ps.scoreLists[currentBestPossibleScoreList] == -1) { currentBestPossibleScoreList++; continue; }
        const int32_t ci = ps.scoreLists[currentBestPossibleScoreList];
        SgScoringCandidate *candidate = &ps.candPool[ci];
        int fewerEndScore; double fewerEndMatchProbability; int fewerEndGenomeLocationOffset;
        bool nonALTAlignment = (!pr.altAwareness) || !P.isALT(candidate->readWithFewerHitsGenomeLocation);
        int scoreLimit = P.computeScoreLimit(nonALTAlignment, &all, &nonAlt, hamming ? 0 : candidate->largestBigIndelDetected);
        if (currentBestPossibleScoreList > scoreLimit) { ps.scoreLists[currentBestPossibleScoreList] = candidate->scoreListNext; continue; }

        if (!hamming) {
            sg_paired_score_location(P, FEWER, SgPairedAligner::setPairDirection(candidate->whichSetPair, FEWER), candidate->readWithFewerHitsGenomeLocation,
                                     candidate->seedOffset, scoreLimit, &fewerEndScore, &fewerEndMatchProbability, &fewerEndGenomeLocationOffset,
                                     &candidate->usedAffineGapScoring, &candidate->basesClippedBefore, &candidate->basesClippedAfter, &candidate->agScore,
                                     &candidate->lvIndels, &candidate->usedGaplessClipping, &candidate->refSpan);
        } else {
            int fewerEndScoreGapless;
            sg_paired_score_location_hamming(P, FEWER, SgPairedAligner::setPairDirection(candidate->whichSetPair, FEWER), candidate->readWithFewerHitsGenomeLocation,
                                             candidate->seedOffset, scoreLimit, &fewerEndScore, &fewerEndMatchProbability, &fewerEndGenomeLocationOffset,
                                             &candidate->basesClippedBefore, &candidate->basesClippedAfter, &candidate->agScore, &candidate->usedGaplessClipping,
                                             &fewerEndScoreGapless);
        }
        candidate->matchProbability = fewerEndMatchProbability;

        if (fewerEndScore != SG_SCORE_ABOVE_LIMIT) {
            uint32_t mateIndex = candidate->scoringMateCandidateIndex;
            SgMateCandidate *mates = ps.mates[candidate->whichSetPair];
            for (;;) {
                SgMateCandidate *mate = &mates[mateIndex];
                if (!hamming) {
                    int64_t lim = candidate->largestBigIndelDetected < fewerEndScore ? candidate->largestBigIndelDetected : fewerEndScore;
                    if (mate->largestBigIndelDetected > lim) lim = mate->largestBigIndelDetected;
                    scoreLimit = P.computeScoreLimit(nonALTAlignment, &all, &nonAlt, lim);
                }
                const bool candGapless = hamming && candidate->usedGaplessClipping;
                if (!SgHitSet::within(mate->readWithMoreHitsGenomeLocation, candidate->readWithFewerHitsGenomeLocation, (int64_t)pp.minSpacing - 1) &&
                    ((mate->bestPossibleScore <= scoreLimit - fewerEndScore) || candGapless)) {
                    // (Hamming) a gapless-clipped fewer end does not lower the mate's limit: its reported score includes the clip (:1968-1990)
                    int mateScoreLimit = candGapless ? scoreLimit : scoreLimit - fewerEndScore;
                    if (mate->score == SG_LOCATION_NOT_YET_SCORED || (mate->score == SG_SCORE_ABOVE_LIMIT && mate->scoreLimit < scoreLimit - fewerEndScore) || candGapless) {
                        if (!hamming) {
                            sg_paired_score_location(P, MORE, SgPairedAligner::setPairDirection(candidate->whichSetPair, MORE), mate->readWithMoreHitsGenomeLocation,
                                                     mate->seedOffset, mateScoreLimit, &mate->score, &mate->matchProbability, &mate->genomeOffset,
                                                     &mate->usedAffineGapScoring, &mate->basesClippedBefore, &mate->basesClippedAfter, &mate->agScore, &mate->lvIndels,
                                                     &mate->usedGaplessClipping, &mate->refSpan);
                        } else {
                            int mateScoreGapless;
                            sg_paired_score_location_hamming(P, MORE, SgPairedAligner::setPairDirection(candidate->whichSetPair, MORE), mate->readWithMoreHitsGenomeLocation,
                                                             mate->seedOffset, mateScoreLimit, &mate->score, &mate->matchProbability, &mate->genomeOffset,
                                                             &mate->basesClippedBefore, &mate->basesClippedAfter, &mate->agScore, &mate->usedGaplessClipping,
                                                             &mateScoreGapless);
                        }
                        mate->scoreLimit = mateScoreLimit;
                    }
                    if (mate->score != SG_SCORE_ABOVE_LIMIT &&
                        ((fewerEndScore + mate->score <= scoreLimit) || candGapless || (hamming && mate->usedGaplessClipping))) {
                        double pairProbability = mate->matchProbability * fewerEndMatchProbability;
                        int pairScore = mate->score + fewerEndScore;
                        int pairAGScore = mate->agScore + candidate->agScore;
                        int32_t mergeAnchor = candidate->mergeAnchor;
                        if (mergeAnchor == -1) {
                            for (int32_t mc = ci - 1; mc >= 0 &&
                                 SgHitSet::within(ps.candPool[mc].readWithFewerHitsGenomeLocation, candidate->readWithFewerHitsGenomeLocation + fewerEndGenomeLocationOffset, 50) &&
                                 ps.candPool[mc].whichSetPair == candidate->whichSetPair; mc--) {
                                if (ps.candPool[mc].mergeAnchor != -1) { candidate->mergeAnchor = mergeAnchor = ps.candPool[mc].mergeAnchor; break; }
                            }
                            if (mergeAnchor == -1) {
                                for (int32_t mc = ci + 1; mc < (int32_t)P.lowestFreeScoringCandidatePoolEntry &&
                                     SgHitSet::within(ps.candPool[mc].readWithFewerHitsGenomeLocation, candidate->readWithFewerHitsGenomeLocation + fewerEndGenomeLocationOffset, 50) &&
                                     ps.candPool[mc].whichSetPair == candidate->whichSetPair; mc++) {
                                    if (ps.candPool[mc].mergeAnchor != -1) { candidate->mergeAnchor = mergeAnchor = ps.candPool[mc].mergeAnchor; break; }
                                }
                            }
                        }
                        bool eliminatedByMerge; double oldPairProbability; bool mergeReplacement = false;
                        const int64_t newMore = mate->readWithMoreHitsGenomeLocation + mate->genomeOffset;
                        const int64_t newFewer = candidate->readWithFewerHitsGenomeLocation + fewerEndGenomeLocationOffset;
                        if (mergeAnchor == -1) {
                            if (P.firstFreeMergeAnchor >= pp.poolCap) { P.error = pp.poolCap < pp.poolSize ? 4 : 1; return true; }
                            mergeAnchor = (int32_t)P.firstFreeMergeAnchor++;
                            SgMergeAnchor &an = ps.anchors[mergeAnchor];
                            an.locationForReadWithMoreHits = newMore; an.locationForReadWithFewerHits = newFewer;
                            an.matchProbability = pairProbability; an.pairScore = pairScore; an.pairAGScore = pairAGScore;
                            eliminatedByMerge = false; oldPairProbability = 0;
                            candidate->mergeAnchor = mergeAnchor;
                        } else {
                            // MergeAnchor::checkMerge (:3820-3871)
                            SgMergeAnchor &an = ps.anchors[mergeAnchor];
                            int64_t dM = an.locationForReadWithMoreHits - newMore; if (dM < 0) dM = -dM;
                            int64_t dF = an.locationForReadWithFewerHits - newFewer; if (dF < 0) dF = -dF;
                            bool rangeMatch = dM < 50 && dF < 50;
                            if (an.locationForReadWithMoreHits == P.invalidLocation || !rangeMatch) {
                                an.locationForReadWithMoreHits = newMore; an.locationForReadWithFewerHits = newFewer;
                                an.matchProbability = pairProbability; an.pairScore = pairScore; an.pairAGScore = pairAGScore;
                                oldPairProbability = 0.0; mergeReplacement = false; eliminatedByMerge = false;
                            } else if (pairAGScore > an.pairAGScore || (pairAGScore == an.pairAGScore && pairProbability > an.matchProbability)) {
                                oldPairProbability = an.matchProbability;
                                an.matchProbability = pairProbability; an.pairScore = pairScore; an.pairAGScore = pairAGScore;
                                mergeReplacement = true; eliminatedByMerge = false;
                            } else {
                                oldPairProbability = 0.0; mergeReplacement = false; eliminatedByMerge = true;
                            }
                        }
                        if (!eliminatedByMerge) {
                            all.updateProbabilityOfAllPairs(oldPairProbability);
                            if (nonALTAlignment) nonAlt.updateProbabilityOfAllPairs(oldPairProbability);
                            if (!mergeReplacement && (pairProbability > all.probabilityOfBestPair) && (maxLVCand > 0) &&
                                (!hamming || pairScore <= all.bestPairScore) && (esd >= all.bestPairScore - pairScore)) {
                                if (*nLVCandidatesForAffineGap >= maxLVCand) { *nLVCandidatesForAffineGap = maxLVCand + 1; return false; }
                                sg_paired_fill_best_result(&ps.lvCandidates[*nLVCandidatesForAffineGap], all, popularSeedsSkipped);
                                (*nLVCandidatesForAffineGap)++;
                            }
                            if (nonALTAlignment) {
                                nonAlt.updateBestHitIfNeeded(pairScore, pairAGScore, pairProbability, fewerEndScore, (int)MORE, fewerEndGenomeLocationOffset, candidate, mate);
                            }
                            bool updatedBestScore = all.updateBestHitIfNeeded(pairScore, pairAGScore, pairProbability, fewerEndScore, (int)MORE, fewerEndGenomeLocationOffset, candidate, mate);
                            if ((!updatedBestScore) && maxLVCand > 0 && (hamming ? (pairScore >= all.bestPairScore) : (pairScore <= (maxK + esd))) &&
                                (esd >= pairScore - all.bestPairScore)) {
                                if (*nLVCandidatesForAffineGap >= maxLVCand) { *nLVCandidatesForAffineGap = maxLVCand + 1; return false; }
                                sg_paired_fill_candidate_result(&ps.lvCandidates[*nLVCandidatesForAffineGap], P, candidate, mate, fewerEndScore, fewerEndGenomeLocationOffset, popularSeedsSkipped);
                                (*nLVCandidatesForAffineGap)++;
                            }
                            if ((pr.altAwareness ? nonAlt.probabilityOfAllPairs : all.probabilityOfAllPairs) >= 4.9) { doneScoring = true; break; }
                        }
                    }
                }
                if (mateIndex == 0 || !SgHitSet::within(mates[mateIndex - 1].readWithMoreHitsGenomeLocation, candidate->readWithFewerHitsGenomeLocation, maxSpacing)) break;
                mateIndex--;
            }
            if (doneScoring) break;
        }
        ps.scoreLists[currentBestPossibleScoreList] = candidate->scoreListNext;
    }

    const SgPairScoreSet *emit = ((!pr.altAwareness) || nonAlt.bestPairScore > all.bestPairScore + pr.maxScoreGapToPreferNonAltAlignment) ? &all : &nonAlt;
    if (emit->bestPairScore == SG_TOO_BIG_SCORE) {
        for (int w = 0; w < 2; w++) {
            result->location[w] = P.invalidLocation; result->origLocation[w] = P.invalidLocation; result->mapq[w] = 0; result->score[w] = SG_SCORE_ABOVE_LIMIT;
            result->status[w] = SNAPGPU_NOT_FOUND; result->clippingForReadAdjustment[w] = 0; result->usedAffineGapScoring[w] = 0; result->usedGaplessClipping[w] = 0;
            result->basesClippedBefore[w] = 0; result->basesClippedAfter[w] = 0; result->agScore[w] = SG_SCORE_ABOVE_LIMIT; result->seedOffset[w] = 0;
            result->lvIndels[w] = 0; result->popularSeedsSkipped[w] = popularSeedsSkipped[w]; result->matchProbability[w] = 0.0;
            alt->status[w] = SNAPGPU_NOT_FOUND;
        }
        result->probabilityAllPairs = 0.0;
    } else {
        emit->fillInResult(T, result, popularSeedsSkipped);
        if (pr.altAwareness && emit == &nonAlt &&
            (all.bestResultGenomeLocation[0] != nonAlt.bestResultGenomeLocation[0] || all.bestResultGenomeLocation[1] != nonAlt.bestResultGenomeLocation[1])) {
            all.fillInResult(T, alt, popularSeedsSkipped);
            alt->supplementary[0] = alt->supplementary[1] = 1;
        } else {
            alt->status[0] = alt->status[1] = SNAPGPU_NOT_FOUND;
        }
    }
    for (int w = 0; w < 2; w++) result->scorePriorToClipping[w] = result->score[w];
    return true;
}

// IntersectingPairedEndAligner::scoreLocationWithAffineGapLiftover (:2970-3118): the whole read from the projected start, forward and then back
// over what the forward pass aligned, with useAltLiftover set.  Liftover is rare, so it takes the general affine-gap form (usePacked = 0), the
// only one that honours the flag.  The reference counts no affine-gap call here.
template <int AGM = 0>
SG_HDN void sg_paired_score_location_ag_liftover(SgPairedAligner &P, uint32_t whichRead, int direction, int64_t genomeLocation, int scoreLimit, int *score,
                                                 double *matchProbability, int *genomeLocationOffset, int *basesClippedBefore, int *basesClippedAfter,
                                                 int *agScore, int *genomeSpan)
{
    const SgIndexView &ix = *P.ix; const SgParams &pr = *P.pr; const SgTables &T = *P.tb;
    const int readLen = (int)P.readLen[whichRead];
    const int64_t genomeDataLength = (int64_t)readLen + SG_MAX_K;
    const uint8_t *data = sg_get_substring(ix, genomeLocation, genomeDataLength);
    *genomeLocationOffset = 0;
    *genomeSpan = 0;
    if (data == (const uint8_t *)0) { *score = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0; *genomeLocationOffset = 0; *agScore = SG_SCORE_ABOVE_LIMIT; return; }
    *basesClippedBefore = 0; *basesClippedAfter = 0;
    SgScratch sc = P.single->sc;
    sc.agBt[0] = P.ps.agBt[0]; sc.agBt[1] = P.ps.agBt[1];
    SgAgParams ag = P.ag;
    ag.usePacked = 0; ag.altLiftover = 1;
    SgAgResult ar;
    int patternLen = readLen;
    bool banded = (patternLen >= (3 * (2 * scoreLimit + 1))) && !pr.noBandedAffineGap;
    ar.textOffset = 0; ar.patternOffset = 0; ar.nEdits = 0; ar.matchProbability = 1.0; ar.agScore = -1;
    sg_ag_dispatch<AGM>(T, sc, ag, 1, banded, data, (int)genomeDataLength, P.readData[whichRead][direction], P.readQual[whichRead][direction], patternLen, scoreLimit,
                        readLen, direction != 0, P.pp->useSoftClip != 0, &ar, sg_lane());
    const int textRem = ar.textOffset, score1 = ar.nEdits;
    *basesClippedAfter = ar.patternOffset;
    if (score1 != SG_SCORE_ABOVE_LIMIT && score1 <= SG_MAX_K - 1) {
        const int limitLeft = score1;
        patternLen = readLen - *basesClippedAfter;
        banded = (patternLen >= (3 * (2 * limitLeft + 1))) && !pr.noBandedAffineGap;
        ar.textOffset = 0; ar.patternOffset = 0; ar.nEdits = 0; ar.matchProbability = 1.0; ar.agScore = -1;
        sg_ag_dispatch<AGM>(T, sc, ag, -1, banded, data + readLen - textRem, readLen - textRem, P.ps.revRead[whichRead][direction] + *basesClippedAfter,
                            P.readQual[whichRead][1 - direction] + *basesClippedAfter, patternLen, limitLeft, readLen, direction != 0, P.pp->useSoftClip != 0, &ar, sg_lane());
        *basesClippedBefore = ar.patternOffset;
        if (ar.nEdits == SG_SCORE_ABOVE_LIMIT || ar.nEdits > SG_MAX_K - 1) {
            *score = SG_SCORE_ABOVE_LIMIT; *genomeLocationOffset = 0; *agScore = -1;
        } else {
            *score = ar.nEdits;
            *agScore = ar.agScore - readLen;
            *matchProbability = ar.matchProbability;
            *genomeLocationOffset = *basesClippedAfter + ar.textOffset - textRem;
            *genomeSpan = readLen - textRem - *genomeLocationOffset;
        }
    } else {
        *score = SG_SCORE_ABOVE_LIMIT; *genomeLocationOffset = 0; *agScore = -1;
    }
}

// The end of alignAffineGap (:2865-2966), soft clipping on: a pair on ALT contigs, or an ALT pair (firstALTResult) that beats the emitted one and
// projects to another contig, is projected onto the primary contig and rescored there; if either end fails, the result stays as it was.
template <int AGM = 0>
SG_HDN void sg_paired_alt_liftover(SgPairedAligner &P, snapgpu_paired_result *result)
{
    const SgIndexView &ix = *P.ix;
    const snapgpu_paired_result *alt = P.altResult();
    int bestAltScore = INT_MAX, bestResScore = INT_MAX, altProjContigNum = -1, resContigNum = -1;
    bool isResultALT = false;
    if (alt->status[0] != SNAPGPU_NOT_FOUND && alt->status[1] != SNAPGPU_NOT_FOUND) {
        bestAltScore = alt->score[0] + alt->score[1];
        altProjContigNum = sg_proj_contig_num_at(ix, alt->location[0]);
    }
    if (result->status[0] != SNAPGPU_NOT_FOUND && result->status[1] != SNAPGPU_NOT_FOUND) {
        bestResScore = result->score[0] + result->score[1];
        resContigNum = sg_contig_at(ix, result->location[0]);
        isResultALT = P.isALT(result->location[0]) && P.isALT(result->location[1]);
    }
    if (!(((bestAltScore < bestResScore) && (altProjContigNum != resContigNum)) || isResultALT)) return;
    const snapgpu_paired_result *src = isResultALT ? result : alt;
    const int projDirection = sg_proj_contig_rc(ix, src->location[0]);     // orientation of the ALT contig against its primary one
    int newDirection[2], newSeedOffset[2], newMapq[2];
    int64_t newStart[2];
    for (int r = 0; r < 2; r++) {
        newDirection[r] = (src->direction[r] != projDirection) ? SNAPGPU_RC : SNAPGPU_FORWARD;
        newSeedOffset[r] = (newDirection[r] != src->direction[r]) ? (int)P.readLen[r] - src->seedOffset[r] - 1 : src->seedOffset[r];
        newStart[r] = sg_proj_location(ix, src->location[r], src->refSpan[r], P.invalidLocation);
        newMapq[r] = isResultALT ? (src->mapq[r] <= 3 ? 70 : src->mapq[r]) : src->mapq[r];
    }
    if (newStart[0] == P.invalidLocation || newStart[1] == P.invalidLocation) return;
    snapgpu_paired_result &resultBeforeLiftover = P.wsKey;           // (the phase-4 sort is over)
    resultBeforeLiftover = *result;
    for (int r = 0; r < 2; r++) {
        int genomeOffset;
        result->usedAffineGapScoring[r] = 1;
        result->liftover[r] = 1;
        result->direction[r] = newDirection[r];
        result->location[r] = newStart[r];
        result->seedOffset[r] = newSeedOffset[r];
        result->mapq[r] = newMapq[r];
        sg_paired_score_location_ag_liftover<AGM>(P, (uint32_t)r, result->direction[r], result->location[r], SG_MAX_K - 1, &result->score[r], &result->matchProbability[r],
                                                  &genomeOffset, &result->basesClippedBefore[r], &result->basesClippedAfter[r], &result->agScore[r], &result->refSpan[r]);
        if (result->score[r] != SG_SCORE_ABOVE_LIMIT && result->score[r] <= SG_MAX_K - 1) result->location[r] += genomeOffset;
        else result->status[r] = SNAPGPU_NOT_FOUND;
    }
    if (result->status[0] == SNAPGPU_NOT_FOUND || result->status[1] == SNAPGPU_NOT_FOUND) *result = resultBeforeLiftover;
}

// IntersectingPairedEndAligner::alignAffineGap (:2489-2969), phase 4, with the pair's firstALTResult (P.altResult()).
template <int AGM = 0>
SG_HDN void sg_paired_align_ag(SgPairedAligner &P, snapgpu_paired_result *result, int *nLVCandidatesForAffineGap)
{
    const SgParams &pr = *P.pr; const SgPairedParams &pp = *P.pp; const SgTables &T = *P.tb;
    SgPairedScratch &ps = P.ps;
    snapgpu_paired_result *alt = P.altResult();
    if (result->status[0] == SNAPGPU_NOT_FOUND || result->status[1] == SNAPGPU_NOT_FOUND) return;
    if (P.readLen[0] < P.ix->seedLen || P.readLen[1] < P.ix->seedLen) return;
    // the RC / reversed strings built by alignLandauVishkin are still valid (same reads); the N check passed there
    const int maxK = P.maxK, esd = (int)pr.extraSearchDepth;
    const int maxKForSameAlignment = pr.gapOpenPenalty / (pr.subPenalty - pr.gapExtendPenalty);
    const int bestPairScore = result->score[0] + result->score[1];
    int scoreLimit, scoreLimitALT;
    if (result->usedGaplessClipping[0] || result->usedGaplessClipping[1]) scoreLimit = scoreLimitALT = SG_MAX_K - 1; else scoreLimit = scoreLimitALT = maxK + esd;
    int genomeOffset[2] = {0, 0};
    bool skipAffineGap[2] = {false, false};
    const double oldPairProbabilityBestResult = result->matchProbability[0] * result->matchProbability[1];
    const double oldPairProbabilityBestResultALT = (alt->status[0] != SNAPGPU_NOT_FOUND) ? alt->matchProbability[0] * alt->matchProbability[1] : 0.0;

    for (int r = 0; r < 2; r++) {
        if (result->usedGaplessClipping[r] || result->score[r] > maxKForSameAlignment) {
            result->usedAffineGapScoring[r] = 1;
            if (!result->usedGaplessClipping[r]) scoreLimit = scoreLimit > result->score[r] ? scoreLimit : result->score[r];
            sg_paired_score_location_ag<AGM>(P, (uint32_t)r, result->direction[r], result->origLocation[r], (uint32_t)result->seedOffset[r], scoreLimit, &result->score[r],
                                        &result->matchProbability[r], &genomeOffset[r], &result->basesClippedBefore[r], &result->basesClippedAfter[r],
                                        &result->agScore[r], &result->refSpan[r]);
            if (result->score[r] != SG_SCORE_ABOVE_LIMIT) {
                result->location[r] = result->origLocation[r] + genomeOffset[r];
                scoreLimit -= result->score[r];
            } else {
                result->status[r] = SNAPGPU_NOT_FOUND;
            }
            // the ALT pair's end is rescored only where the result's is, under its own limit (:2618-2644)
            if (alt->status[r] != SNAPGPU_NOT_FOUND && (alt->usedGaplessClipping[r] || alt->score[r] > maxKForSameAlignment)) {
                alt->usedAffineGapScoring[r] = 1;
                if (!alt->usedGaplessClipping[r]) scoreLimitALT = scoreLimitALT > alt->score[r] ? scoreLimitALT : alt->score[r];
                sg_paired_score_location_ag<AGM>(P, (uint32_t)r, alt->direction[r], alt->origLocation[r], (uint32_t)alt->seedOffset[r], scoreLimitALT, &alt->score[r],
                                                 &alt->matchProbability[r], &genomeOffset[r], &alt->basesClippedBefore[r], &alt->basesClippedAfter[r],
                                                 &alt->agScore[r], &alt->refSpan[r]);
                if (alt->score[r] != SG_SCORE_ABOVE_LIMIT) {
                    alt->location[r] = alt->origLocation[r] + genomeOffset[r];
                    scoreLimitALT -= alt->score[r];
                } else {
                    alt->status[r] = SNAPGPU_NOT_FOUND;
                }
            }
        } else {
            result->usedAffineGapScoring[r] = 0;
            skipAffineGap[r] = true;
        }
    }

    if (result->status[0] == SNAPGPU_NOT_FOUND || result->status[1] == SNAPGPU_NOT_FOUND || (result->score[0] > SG_MAX_K - 1) || (result->score[1] > SG_MAX_K - 1)) {
        for (int w = 0; w < 2; w++) {
            result->location[w] = P.invalidLocation; result->origLocation[w] = P.invalidLocation; result->mapq[w] = 0; result->score[w] = SG_SCORE_ABOVE_LIMIT;
            result->status[w] = SNAPGPU_NOT_FOUND; result->clippingForReadAdjustment[w] = 0; result->usedAffineGapScoring[w] = 0; result->usedGaplessClipping[w] = 0;
            result->basesClippedBefore[w] = 0; result->basesClippedAfter[w] = 0; result->agScore[w] = SG_SCORE_ABOVE_LIMIT; result->seedOffset[w] = 0;
            result->lvIndels[w] = 0; result->matchProbability[w] = 0.0;
            alt->status[w] = SNAPGPU_NOT_FOUND;
        }
        result->probabilityAllPairs = 0.0;
        return;
    }

    SgPairScoreSet &all = P.wsAll, &nonAlt = P.wsNonAlt;
    nonAlt.init(P.invalidLocation);
    bool nonALTAlignment = (!pr.altAwareness) || !P.isALT(result->location[0]);
    all.initFrom(result);
    bool altBestAlignment = false;
    if (alt->status[0] != SNAPGPU_NOT_FOUND && alt->status[1] != SNAPGPU_NOT_FOUND) {
        altBestAlignment = all.updateBestHitIfNeededR(alt->score[0] + alt->score[1], alt->agScore[0] + alt->agScore[1],
                                                      alt->matchProbability[0] * alt->matchProbability[1], alt);
    }
    if (nonALTAlignment) nonAlt.initFrom(result);
    if (!skipAffineGap[0] || !skipAffineGap[1]) {
        double newPairProbability = result->matchProbability[0] * result->matchProbability[1];
        if (altBestAlignment) {
            // the ALT pair's probability is in the total already (updateBestHitIfNeeded above)
            all.updateProbabilityOfAllPairs(oldPairProbabilityBestResultALT);
            all.updateProbabilityOfBestPair(alt->matchProbability[0] * alt->matchProbability[1], false);
        } else {
            all.updateProbabilityOfAllPairs(oldPairProbabilityBestResult);
            all.updateProbabilityOfBestPair(newPairProbability);
        }
        if (nonALTAlignment) {
            nonAlt.updateProbabilityOfAllPairs(oldPairProbabilityBestResult);
            nonAlt.updateProbabilityOfBestPair(newPairProbability);
        }
    }

    if ((*nLVCandidatesForAffineGap > 0) && (!skipAffineGap[0] || !skipAffineGap[1])) {
        scoreLimit = (maxK < bestPairScore ? maxK : bestPairScore) + esd;
        // qsort(..., compareByScore) on the sum of the two scores: glibc's qsort is a merge sort for these sizes, i.e. stable
        // (SURVEY 7.6); insertion sort keeps equal keys in order and n is small
        const int n = *nLVCandidatesForAffineGap;
        for (int i = 1; i < n; i++) {
            snapgpu_paired_result &key = P.wsKey;
            key = ps.lvCandidates[i];
            int ks = key.score[0] + key.score[1];
            int j = i - 1;
            while (j >= 0 && (ps.lvCandidates[j].score[0] + ps.lvCandidates[j].score[1]) > ks) { ps.lvCandidates[j + 1] = ps.lvCandidates[j]; j--; }
            ps.lvCandidates[j + 1] = key;
        }
        for (int i = 0; i < n; i++) {
            snapgpu_paired_result *lv = &ps.lvCandidates[i];
            int lvPairScore = lv->score[0] + lv->score[1];
            int lvPairIndels = lv->lvIndels[0] + lv->lvIndels[1];
            if (lv->usedGaplessClipping[0] || lv->usedGaplessClipping[1]) scoreLimit = SG_MAX_K - 1;
            else if ((lvPairScore > bestPairScore + esd) && (lvPairIndels > 1)) scoreLimit = maxK + esd;
            if ((lvPairScore <= bestPairScore + esd) || (lvPairIndels > 1) || lv->usedGaplessClipping[0] || lv->usedGaplessClipping[1]) {
                bool nonALT = (!pr.altAwareness) || !P.isALT(lv->location[0]);
                double oldPairProbability = lv->matchProbability[0] * lv->matchProbability[1];
                if (!skipAffineGap[0]) {
                    lv->usedAffineGapScoring[0] = 1;
                    if (!lv->usedGaplessClipping[0]) scoreLimit = scoreLimit > lv->score[0] ? scoreLimit : lv->score[0];
                    sg_paired_score_location_ag<AGM>(P, 0, lv->direction[0], lv->origLocation[0], (uint32_t)lv->seedOffset[0], scoreLimit, &lv->score[0], &lv->matchProbability[0],
                                                &genomeOffset[0], &lv->basesClippedBefore[0], &lv->basesClippedAfter[0], &lv->agScore[0], &lv->refSpan[0]);
                }
                if ((lv->score[0] != SG_SCORE_ABOVE_LIMIT) && (lv->score[0] <= SG_MAX_K - 1)) {
                    lv->location[0] = lv->origLocation[0] + genomeOffset[0];
                    if (!skipAffineGap[1]) {
                        lv->usedAffineGapScoring[1] = 1;
                        scoreLimit = scoreLimit - lv->score[0];
                        if (!lv->usedGaplessClipping[1]) scoreLimit = scoreLimit > lv->score[1] ? scoreLimit : lv->score[1];
                        sg_paired_score_location_ag<AGM>(P, 1, lv->direction[1], lv->origLocation[1], (uint32_t)lv->seedOffset[1], scoreLimit, &lv->score[1], &lv->matchProbability[1],
                                                    &genomeOffset[1], &lv->basesClippedBefore[1], &lv->basesClippedAfter[1], &lv->agScore[1], &lv->refSpan[1]);
                    }
                    if ((lv->score[1] != SG_SCORE_ABOVE_LIMIT) && (lv->score[1] <= SG_MAX_K - 1)) {
                        lv->location[1] = lv->origLocation[1] + genomeOffset[1];
                        double pairProbability = lv->matchProbability[0] * lv->matchProbability[1];
                        int pairScore = lv->score[0] + lv->score[1];
                        int pairAGScore = lv->agScore[0] + lv->agScore[1];
                        if (result->location[0] == lv->location[0] && result->location[1] == lv->location[1]) continue;
                        all.updateProbabilityOfAllPairs(oldPairProbability);
                        all.updateBestHitIfNeededR(pairScore, pairAGScore, pairProbability, lv);
                        if (nonALT) {
                            nonAlt.updateProbabilityOfAllPairs(oldPairProbability);
                            nonAlt.updateBestHitIfNeededR(pairScore, pairAGScore, pairProbability, lv);
                        }
                        scoreLimit = P.computeScoreLimit(nonALT, &all, &nonAlt, 0);
                    }
                }
            }
        }
    }

    const SgPairScoreSet *emit = ((!pr.altAwareness) || nonAlt.bestPairScore > all.bestPairScore + pr.maxScoreGapToPreferNonAltAlignment) ? &all : &nonAlt;
    emit->fillInResult(T, result, result->popularSeedsSkipped);
    if (pr.altAwareness && emit == &nonAlt &&
        (all.bestResultGenomeLocation[0] != nonAlt.bestResultGenomeLocation[0] || all.bestResultGenomeLocation[1] != nonAlt.bestResultGenomeLocation[1])) {
        all.fillInResult(T, alt, alt->popularSeedsSkipped);
        alt->supplementary[0] = alt->supplementary[1] = 1;
    } else {
        alt->status[0] = alt->status[1] = SNAPGPU_NOT_FOUND;
    }
    // without ALT contigs (projStart == NULL) nothing is ALT, the two score sets agree and there is nothing to lift over
    if (pp.useSoftClip && pr.altAwareness && P.ix->projStart) sg_paired_alt_liftover<AGM>(P, result);
}

// (re)derive the per-read strings and pointers alignLandauVishkin sets up (:347-372), for a worker that takes a pair over at the
// stage boundary below
SG_HDN void sg_paired_restore_reads(SgPairedAligner &P, const uint8_t *const readBases[2], const uint8_t *const readQuals[2], const uint32_t lens[2])
{
    SgPairedScratch &ps = P.ps;
    for (uint32_t w = 0; w < 2; w++) {
        P.readLen[w] = lens[w];
        P.readData[w][0] = readBases[w]; P.readQual[w][0] = readQuals[w];
        P.readData[w][1] = ps.rcRead[w]; P.readQual[w][1] = ps.rcQual[w];
#if defined(__CUDA_ARCH__)
        #pragma unroll 1
        for (uint32_t i = (uint32_t)sg_lane(); i < lens[w]; i += 32) {
#else
        for (uint32_t i = 0; i < lens[w]; i++) {
#endif
            const uint8_t b = readBases[w][i], c = sg_complement(b);
            ps.rcRead[w][lens[w] - i - 1] = c;
            ps.rcQual[w][lens[w] - i - 1] = readQuals[w][i];
            ps.revRead[w][0][lens[w] - i - 1] = b;
            ps.revRead[w][1][i] = c;
        }
    }
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
}

// ChimericPairedEndAligner::align (ChimericPairedEndAligner.cpp:126-448) around IntersectingPairedEndAligner::align (:169-252), cut in
// two at the point where the seed / Landau-Vishkin phases (alignLandauVishkin, incl. the Hamming retry) are over and the
// affine-gap phase and the single-end fallback begin.  What crosses the cut: `result`, the phase-4 candidate list
// (P.ps.lvCandidates[0, nLVCand)) and the return value of stage 1.  When that value has SG_STAGE_ALT_RESULT set, the last record of the
// list is the pair's firstALTResult: a launch form that hands the candidates over hands it over too, and stage 2 takes it back to its slot
// (P.altResult()).  sg_paired_align() is the two stages back to back; the
// device may run them in different kernels (sg_align_paired_kernel) so that each kernel's code stays small.
//   stage 1 returns 0: `result` is final (or P.error is set); 1: continue, both reads were long enough for the paired aligner;
//   2: continue, one read is too short (single-end fallback only).
SG_HDN int sg_paired_align_stage1(SgPairedAligner &P, const uint8_t *const readBases[2], const uint8_t *const readQuals[2], const uint32_t lens[2],
                                  snapgpu_paired_result *result, int *nLVCand)
{
    const SgParams &pr = *P.pr; const SgPairedParams &pp = *P.pp;
    result->status[0] = result->status[1] = SNAPGPU_NOT_FOUND;
    result->usedAffineGapScoring[0] = result->usedAffineGapScoring[1] = 0;
    result->basesClippedBefore[0] = result->basesClippedBefore[1] = 0;
    result->basesClippedAfter[0] = result->basesClippedAfter[1] = 0;
    result->clippingForReadAdjustment[0] = result->clippingForReadAdjustment[1] = 0;
    result->agScore[0] = result->agScore[1] = 0;
    result->liftover[0] = result->liftover[1] = 0;
    result->agForcedSingleAlignerCall = 0;
    const uint32_t minReadLength = pr.minReadLength;
    *nLVCand = 0;
    snapgpu_paired_result *alt = P.altResult();
    alt->status[0] = alt->status[1] = SNAPGPU_NOT_FOUND;                   // ChimericPairedEndAligner.cpp:162
    alt->popularSeedsSkipped[0] = alt->popularSeedsSkipped[1] = 0;

    if (lens[0] < minReadLength && lens[1] < minReadLength) {
        for (int w = 0; w < 2; w++) { result->location[w] = P.invalidLocation; result->mapq[w] = 0; result->score[w] = 0; result->status[w] = SNAPGPU_NOT_FOUND; }
        result->alignedAsPair = 0;
        return 0;
    }
    if (lens[0] >= minReadLength && lens[1] >= minReadLength) {
        P.maxK = (int)pr.maxK;
        bool fit = sg_paired_align_lv(P, readBases, readQuals, lens, result, nLVCand);
        if (!fit || P.error) { P.error = P.error ? P.error : (pp.agCandCap < SG_MAX_AG_CANDIDATES ? 4 : 2); return 0; }      // buffer growth + retry (PairedAligner.cpp:727-780) is not implemented
        if (pr.useAffineGap && pp.useSoftClip && (result->status[0] == SNAPGPU_NOT_FOUND || result->status[1] == SNAPGPU_NOT_FOUND)) {
            // IntersectingPairedEndAligner.cpp:220-233: try again with Hamming scoring that clips a poorly matching start / end
            fit = sg_paired_align_lv(P, readBases, readQuals, lens, result, nLVCand, true);
            if (!fit || P.error) { P.error = P.error ? P.error : (pp.agCandCap < SG_MAX_AG_CANDIDATES ? 4 : 2); return 0; }
        }
        if (alt->status[0] != SNAPGPU_NOT_FOUND || alt->status[1] != SNAPGPU_NOT_FOUND || alt->popularSeedsSkipped[0] || alt->popularSeedsSkipped[1]) {
            // the firstALTResult crosses the cut as one more candidate record (its slot follows the candidates: nLVCand <= agCandCap).  It
            // swaps places with what that candidate slot held, and stage 2 swaps them back: candidate records keep a field the reference
            // never writes (refSpan, see sg_paired_fill_candidate_result), so the buffer must not remember the ALT record
            if (*nLVCand != (int)pp.agCandCap) {
                snapgpu_paired_result &held = P.wsKey;
                held = P.ps.lvCandidates[*nLVCand]; P.ps.lvCandidates[*nLVCand] = *alt; *alt = held;
            }
            (*nLVCand)++;
            return 1 | SG_STAGE_ALT_RESULT;
        }
        return 1;
    }
    return 2;
}

// stage 2 (the affine-gap phase of the intersecting aligner) returns 0: `result` is final; 1: continue with the single-end
// aligner on both reads (stage 3); 2: the same, comparing its result with the pair's (compareWithSingleEndAlignment).
// Only `result` and that value cross this cut.
template <int AGM = 0>
SG_HDN int sg_paired_align_stage2(SgPairedAligner &P, snapgpu_paired_result *result, int stage, int nLVCand)
{
    const SgParams &pr = *P.pr; const SgPairedParams &pp = *P.pp;
    bool compareWithSingleEndAlignment = false;
    snapgpu_paired_result *alt = P.altResult();
    if (stage & SG_STAGE_ALT_RESULT) {
        nLVCand--;
        if (nLVCand != (int)pp.agCandCap) {
            snapgpu_paired_result &held = P.wsKey;
            held = P.ps.lvCandidates[nLVCand]; P.ps.lvCandidates[nLVCand] = *alt; *alt = held;
        }
        stage &= ~SG_STAGE_ALT_RESULT;
    } else {
        alt->status[0] = alt->status[1] = SNAPGPU_NOT_FOUND;
        alt->popularSeedsSkipped[0] = alt->popularSeedsSkipped[1] = 0;
    }
    if (stage == 1) {
        P.maxK = (int)pr.maxK;
        if (pr.useAffineGap) sg_paired_align_ag<AGM>(P, result, &nLVCand);
        result->alignedAsPair = 1;
        if (pp.forceSpacing) {
            if (result->status[0] == SNAPGPU_NOT_FOUND) result->alignedAsPair = 0;
            return 0;
        }
        int maxScore = result->score[0] > result->score[1] ? result->score[0] : result->score[1];
        result->mapq[0] = result->mapq[0] <= pp.flattenMAPQAtOrBelow ? 0 : result->mapq[0];
        result->mapq[1] = result->mapq[1] <= pp.flattenMAPQAtOrBelow ? 0 : result->mapq[1];
        // an ALT pair at least minScoreGapRealignmentALT better than the result, or a lifted-over result, is not split up by the single-end
        // aligner (ChimericPairedEndAligner.cpp:225-242)
        const bool seenBetterAltResult = alt->status[0] != SNAPGPU_NOT_FOUND && alt->status[1] != SNAPGPU_NOT_FOUND &&
                                         alt->score[0] + alt->score[1] <= result->score[0] + result->score[1] - pp.minScoreGapRealignmentALT;
        const bool useAltLiftover = result->liftover[0] && result->liftover[1];
        if ((result->usedAffineGapScoring[0] || result->usedAffineGapScoring[1]) && maxScore >= pp.minScoreRealignment && !seenBetterAltResult && !useAltLiftover)
            compareWithSingleEndAlignment = true;
        if (result->status[0] != SNAPGPU_NOT_FOUND && result->status[1] != SNAPGPU_NOT_FOUND && !compareWithSingleEndAlignment) return 0;
    }
    return compareWithSingleEndAlignment ? 2 : 1;
}

// stage 3: ChimericPairedEndAligner.cpp:268-448, the single-end aligner on each read and the choice between its result and the pair's.
// (Its two writes to firstALTResult, :296 and :418, only decide whether -ea would write that record out, so they are not restated.)
SG_HDN void sg_paired_align_stage3(SgPairedAligner &P, const uint8_t *const readBases[2], const uint8_t *const readQuals[2], const uint32_t lens[2],
                                   snapgpu_paired_result *result, int stage)
{
    const SgParams &pr = *P.pr; const SgPairedParams &pp = *P.pp;
    SgAligner &S = *P.single;
    const uint32_t minReadLength = pr.minReadLength;
    const int maxKSingleEnd = (int)(pr.maxK / 2);
    const bool compareWithSingleEndAlignment = stage == 2;
    int pairAGScore = 0;
    const int sumPairScore = compareWithSingleEndAlignment ? result->score[0] + result->score[1] : 0;

    int scoreLimitLeft = maxKSingleEnd;
    if (compareWithSingleEndAlignment) {
        scoreLimitLeft = sumPairScore;
        if (result->status[0] != SNAPGPU_NOT_FOUND && result->status[1] != SNAPGPU_NOT_FOUND) result->agForcedSingleAlignerCall = 1;
    }

    snapgpu_single_result *singleResult = P.wsSingle;
    memset(singleResult, 0, 2 * sizeof(snapgpu_single_result));
    int singleEndAGScore = 0;
    bool chooseSingleEndMapq = true;
    int nSingleCandsFirstRead = 0;
    for (int r = 0; r < 2; r++) {
        if (compareWithSingleEndAlignment) pairAGScore += result->agScore[r];
        S.maxK = (uint32_t)maxKSingleEnd;
        if (lens[r] < minReadLength) {
            result->status[r] = SNAPGPU_NOT_FOUND; result->mapq[r] = 0; result->direction[r] = SNAPGPU_FORWARD; result->location[r] = P.invalidLocation;
            result->score[r] = 0; result->usedAffineGapScoring[r] = 0; result->basesClippedBefore[r] = 0; result->basesClippedAfter[r] = 0; result->agScore[r] = 0;
            result->alignedAsPair = 0; result->clippingForReadAdjustment[r] = 0;
            chooseSingleEndMapq = false;
        } else {
            if (compareWithSingleEndAlignment) {
                if (scoreLimitLeft < 0) break;
                int m = result->score[r] < scoreLimitLeft ? result->score[r] : scoreLimitLeft;
                S.maxK = (uint32_t)(maxKSingleEnd < m ? maxKSingleEnd : m);
            }
            S.agCands = (snapgpu_single_result *)0;
            sg_align_read(S, readBases[r], readQuals[r], lens[r], &singleResult[r]);
            bool usedHammingScoringBaseAligner = false;
            if (pp.useSoftClip && pp.enableHammingScoringBaseAligner) {
                if (singleResult[r].status == SNAPGPU_NOT_FOUND && result->status[r] == SNAPGPU_NOT_FOUND) {
                    // ChimericPairedEndAligner.cpp:330-362: Hamming scoring in the base aligner for an end nothing else could place
                    usedHammingScoringBaseAligner = true;
                    S.agCands = P.ps.singleCandidates + nSingleCandsFirstRead;
                    S.nAgCands = 0; S.maxAgCands = (int)pp.agCandCap - nSingleCandsFirstRead; S.agCandsOverflow = 0;
                    sg_align_read(S, readBases[r], readQuals[r], lens[r], &singleResult[r], true);
                    if (S.agCandsOverflow) { P.error = pp.agCandCap < SG_MAX_AG_CANDIDATES ? 4 : 2; S.agCands = (snapgpu_single_result *)0; return; }
                    sg_align_affine_gap(S, &singleResult[r], S.nAgCands, S.agCands);
                    if (r == 0) nSingleCandsFirstRead = S.nAgCands;
                    S.agCands = (snapgpu_single_result *)0;
                }
            }
            if (compareWithSingleEndAlignment) {
                if (usedHammingScoringBaseAligner) {
                    // the mate's limit is not lowered when this end needed Hamming scoring (:369-379)
                } else if (singleResult[r].score != SG_SCORE_ABOVE_LIMIT && singleResult[r].score != (int)SG_UNUSED_SCORE) scoreLimitLeft -= singleResult[r].score;
                else scoreLimitLeft = SG_SCORE_ABOVE_LIMIT;
                singleEndAGScore += singleResult[r].agScore;
                if (result->agScore[r] >= singleResult[r].agScore) chooseSingleEndMapq = false;
            }
        }
    }
    S.maxK = (uint32_t)maxKSingleEnd;

    if (chooseSingleEndMapq) {
        for (int r = 0; r < 2; r++) {
            result->mapq[r] = result->mapq[r] < singleResult[r].mapq ? result->mapq[r] : singleResult[r].mapq;
            if (result->mapq[r] <= pp.flattenMAPQAtOrBelow) result->mapq[r] = 0;
        }
    }
    if (!compareWithSingleEndAlignment || (singleEndAGScore >= pairAGScore + pp.minAGScoreImprovement)) {
        for (int r = 0; r < 2; r++) {
            if (lens[r] < minReadLength) {
                result->status[r] = SNAPGPU_NOT_FOUND; result->mapq[r] = 0; result->direction[r] = SNAPGPU_FORWARD; result->location[r] = P.invalidLocation;
                result->score[r] = 0; result->usedAffineGapScoring[r] = 0; result->basesClippedBefore[r] = 0; result->basesClippedAfter[r] = 0; result->agScore[r] = 0;
                result->clippingForReadAdjustment[r] = 0;
            } else {
                result->status[r] = singleResult[r].status;
                result->mapq[r] = singleResult[r].mapq / 3;
                result->mapq[r] = result->mapq[r] <= 3 ? 0 : result->mapq[r];
                result->direction[r] = singleResult[r].direction;
                result->location[r] = singleResult[r].location;
                result->score[r] = singleResult[r].score;
                result->scorePriorToClipping[r] = singleResult[r].scorePriorToClipping;
                result->usedAffineGapScoring[r] = singleResult[r].usedAffineGapScoring;
                result->basesClippedBefore[r] = singleResult[r].basesClippedBefore;
                result->basesClippedAfter[r] = singleResult[r].basesClippedAfter;
                result->agScore[r] = singleResult[r].agScore;
            }
        }
        result->alignedAsPair = 0;
    }
}

SG_HD void sg_paired_align(SgPairedAligner &P, const uint8_t *const readBases[2], const uint8_t *const readQuals[2], const uint32_t lens[2],
                           snapgpu_paired_result *result)
{
    int nLVCand = 0;
    const int stage = sg_paired_align_stage1(P, readBases, readQuals, lens, result, &nLVCand);
    if (stage == 0) return;
    const int stage3 = sg_paired_align_stage2(P, result, stage, nLVCand);
    if (stage3 != 0) sg_paired_align_stage3(P, readBases, readQuals, lens, result, stage3);
}
