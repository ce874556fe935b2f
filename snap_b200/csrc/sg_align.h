// sg_align.h -- the per-read single-end state machine.  Scalar form, host+device.
// Restates BaseAligner::AlignRead (reference SNAPLib/BaseAligner.cpp:272-763), BaseAligner::score (:917-1534),
// the candidate table (:1810-1973, :2331-2379), ScoreSet (:2143-2323) and scoreLimit (:2555-2570) for the
// configuration `snap single` runs by default: no secondary results (-om unset), no Hamming pass.
// Everything that decides *which* candidate is scored *when* (FIFO weight lists, per-seed score() calls, the
// lowest-possible-score bound, early exits) is kept in the reference's order, because results depend on it.
#pragma once
#include "sg_common.h"
#include "sg_seed.h"
#include "sg_lv.h"
#include "sg_ag.h"
#if defined(__CUDACC__)
#include "sg_warp.cuh"
#include "sg_warp_ag.cuh"
#endif

// Affine-gap leaf dispatch: on the device with a converged warp (lane >= 0) the rows are spread over the lanes.
template <int AGM = 0>
SG_HD void sg_ag_dispatch(const SgTables &T, const SgScratch &S, const SgAgParams &P, int dir, bool banded,
                          const uint8_t *text, int textLen, const uint8_t *pattern, const uint8_t *quality, int patternLen,
                          int w, int scoreInit, bool isRC, bool useClippingOptimizations, SgAgResult *out, int lane)
{
#if defined(__CUDA_ARCH__)
    // every device caller is a converged warp (lane >= 0); the scalar form is not compiled into the kernels
    sg_warp_ag_compute<AGM>(T, S, P, dir, banded, text, textLen, pattern, quality, patternLen, w, scoreInit, isRC, useClippingOptimizations, out, lane);
#else
    (void)lane;
    sg_ag_compute(T, S, P, dir, banded, text, textLen, pattern, quality, patternLen, w, scoreInit, isRC, useClippingOptimizations, out);
#endif
}

struct SgScoreSet {                  // BaseAligner::ScoreSet, BaseAligner.h:260-329
    int      bestScore;
    int64_t  bestScoreGenomeLocation, bestScoreOrigGenomeLocation;
    int      bestScoreDirection;
    int      bestScoreUsedAffineGapScoring;
    int      bestScoreBasesClippedBefore, bestScoreBasesClippedAfter;
    int      bestScoreAGScore;
    int      bestScoreSeedOffset;
    double   bestScoreMatchProbability;
    double   probabilityOfAllCandidates, probabilityOfBestCandidate;

    SG_HD void init(int64_t invalidLocation) {   // :2099-2114
        bestScore = SG_UNUSED_SCORE;
        bestScoreGenomeLocation = invalidLocation; bestScoreOrigGenomeLocation = invalidLocation;
        bestScoreDirection = 0; bestScoreUsedAffineGapScoring = 0;
        bestScoreBasesClippedBefore = 0; bestScoreBasesClippedAfter = 0;
        bestScoreAGScore = -1; bestScoreSeedOffset = 0; bestScoreMatchProbability = 0.0;
        probabilityOfAllCandidates = 0; probabilityOfBestCandidate = 0;
    }
    SG_HD void updateProbabilitiesForNearbyMatch(double p) {            // :2132-2135
        double v = probabilityOfAllCandidates - p;
        probabilityOfAllCandidates = v > 0.0 ? v : 0.0;
    }
    SG_HD void updateProbabilitiesForNewMatch(double newP, double nearbyP) {   // :2137-2141
        double v = probabilityOfAllCandidates - nearbyP;
        probabilityOfAllCandidates = v > 0.0 ? v : 0.0;
        probabilityOfAllCandidates += newP;
    }
    // ScoreSet::updateBestScore with secondaryResults == NULL and candidatesForAffineGap == NULL (:2143-2299)
    SG_HD void updateBestScore(int64_t genomeLocation, int64_t origGenomeLocation, unsigned score, bool useAffineGap, int agScore,
                               double matchProbability, const SgElem *el) {
        bool seenNewBestScore;
        if (useAffineGap) {
            seenNewBestScore = (agScore > bestScoreAGScore) || (bestScoreAGScore == agScore && matchProbability > probabilityOfBestCandidate);
        } else {
            seenNewBestScore = (score < (unsigned)bestScore) || (score == (unsigned)bestScore && matchProbability > probabilityOfBestCandidate);
        }
        if (seenNewBestScore) {
            bestScore = (int)score;
            bestScoreAGScore = agScore;
            probabilityOfBestCandidate = matchProbability;
            bestScoreGenomeLocation = genomeLocation;
            bestScoreOrigGenomeLocation = origGenomeLocation;
            bestScoreDirection = el->direction;
            bestScoreUsedAffineGapScoring = el->usedAffineGapScoring;
            bestScoreBasesClippedBefore = el->basesClippedBefore;
            bestScoreBasesClippedAfter = el->basesClippedAfter;
            bestScoreSeedOffset = el->seedOffset;
            bestScoreMatchProbability = el->matchProbabilityForBestScore;
        }
    }
    // ScoreSet::updateBestScore with a candidatesForAffineGap buffer (the Hamming pass, :1444-1456): the displaced best / the
    // near-best candidate is appended when it is within extraSearchDepth of the best (:2202-2226, :2273-2297).
    // Returns false if the buffer is full (the reference's caller then reports an overflow).
    SG_HD bool updateBestScoreRecording(int64_t genomeLocation, int64_t origGenomeLocation, unsigned score, bool useAffineGap, int agScore,
                                        double matchProbability, const SgElem *el, snapgpu_single_result *cands, int *nCands, int maxCands, int extraSearchDepth) {
        bool seenNewBestScore;
        if (useAffineGap) {
            seenNewBestScore = (agScore > bestScoreAGScore) || (bestScoreAGScore == agScore && matchProbability > probabilityOfBestCandidate);
        } else {
            seenNewBestScore = (score < (unsigned)bestScore) || (score == (unsigned)bestScore && matchProbability > probabilityOfBestCandidate);
        }
        if (seenNewBestScore) {
            if ((unsigned)bestScore >= score) {
                if ((unsigned)bestScore >= score && (int)((unsigned)bestScore - score) <= extraSearchDepth) {
                    if (*nCands >= maxCands) { *nCands = maxCands + 1; return false; }
                    snapgpu_single_result *r = &cands[*nCands];
                    r->direction = bestScoreDirection; r->location = bestScoreGenomeLocation; r->origLocation = bestScoreOrigGenomeLocation;
                    r->mapq = 0; r->score = bestScore; r->status = SNAPGPU_MULTIPLE_HITS; r->clippingForReadAdjustment = 0;
                    r->usedAffineGapScoring = bestScoreUsedAffineGapScoring; r->basesClippedBefore = bestScoreBasesClippedBefore;
                    r->basesClippedAfter = bestScoreBasesClippedAfter; r->agScore = bestScoreAGScore; r->matchProbability = bestScoreMatchProbability;
                    r->seedOffset = bestScoreSeedOffset;
                    (*nCands)++;
                }
            }
            bestScore = (int)score;
            bestScoreAGScore = agScore;
            probabilityOfBestCandidate = matchProbability;
            bestScoreGenomeLocation = genomeLocation;
            bestScoreOrigGenomeLocation = origGenomeLocation;
            bestScoreDirection = el->direction;
            bestScoreUsedAffineGapScoring = el->usedAffineGapScoring;
            bestScoreBasesClippedBefore = el->basesClippedBefore;
            bestScoreBasesClippedAfter = el->basesClippedAfter;
            bestScoreSeedOffset = el->seedOffset;
            bestScoreMatchProbability = el->matchProbabilityForBestScore;
        } else {
            if ((int)((unsigned)bestScore - score) <= extraSearchDepth && score != (unsigned)SG_SCORE_ABOVE_LIMIT && (unsigned)bestScore >= score) {
                if (*nCands >= maxCands) { *nCands = maxCands + 1; return false; }
                snapgpu_single_result *r = &cands[*nCands];
                r->direction = el->direction; r->location = genomeLocation; r->origLocation = origGenomeLocation;
                r->mapq = 0; r->score = (int)score; r->status = SNAPGPU_MULTIPLE_HITS; r->clippingForReadAdjustment = 0;
                r->usedAffineGapScoring = el->usedAffineGapScoring; r->basesClippedBefore = el->basesClippedBefore;
                r->basesClippedAfter = el->basesClippedAfter; r->agScore = el->agScore; r->seedOffset = el->seedOffset;
                r->matchProbability = el->matchProbabilityForBestScore;
                (*nCands)++;
            }
        }
        return true;
    }
    // ScoreSet::updateBestScore with a secondaryResults buffer and candidatesForAffineGap == NULL (`-om` on the single-end path, :1457-1467):
    // the displaced best (:2176-2200) or the near-best candidate (:2247-2271) is appended when it is within
    // maxEditDistanceForSecondaryResults of the best.  Returns false when the buffer is full (*overflowedSecondaryBuffer, :2177-2180).
    SG_HD bool updateBestScoreSecondary(int64_t genomeLocation, int64_t origGenomeLocation, unsigned score, bool useAffineGap, int agScore,
                                        double matchProbability, const SgElem *el, snapgpu_single_result *sec, int *nSec, int maxSec, int maxEditDistanceForSecondaryResults) {
        bool seenNewBestScore;
        if (useAffineGap) {
            seenNewBestScore = (agScore > bestScoreAGScore) || (bestScoreAGScore == agScore && matchProbability > probabilityOfBestCandidate);
        } else {
            seenNewBestScore = (score < (unsigned)bestScore) || (score == (unsigned)bestScore && matchProbability > probabilityOfBestCandidate);
        }
        if (seenNewBestScore) {
            if ((unsigned)bestScore >= score) {
                if ((int)((unsigned)bestScore - score) <= maxEditDistanceForSecondaryResults) {
                    if (maxSec <= *nSec) return false;
                    snapgpu_single_result *r = &sec[*nSec];
                    r->direction = bestScoreDirection; r->location = bestScoreGenomeLocation; r->origLocation = bestScoreOrigGenomeLocation;
                    r->mapq = 0; r->score = bestScore; r->status = SNAPGPU_MULTIPLE_HITS; r->clippingForReadAdjustment = 0;
                    r->usedAffineGapScoring = bestScoreUsedAffineGapScoring; r->basesClippedBefore = bestScoreBasesClippedBefore;
                    r->basesClippedAfter = bestScoreBasesClippedAfter; r->agScore = bestScoreAGScore; r->matchProbability = bestScoreMatchProbability;
                    r->seedOffset = bestScoreSeedOffset;
                    r->scorePriorToClipping = 0; r->supplementary = 0; r->probabilityAllCandidates = 0; r->popularSeedsSkipped = 0; r->reserved = 0;
                    (*nSec)++;
                }
            }
            bestScore = (int)score;
            bestScoreAGScore = agScore;
            probabilityOfBestCandidate = matchProbability;
            bestScoreGenomeLocation = genomeLocation;
            bestScoreOrigGenomeLocation = origGenomeLocation;
            bestScoreDirection = el->direction;
            bestScoreUsedAffineGapScoring = el->usedAffineGapScoring;
            bestScoreBasesClippedBefore = el->basesClippedBefore;
            bestScoreBasesClippedAfter = el->basesClippedAfter;
            bestScoreSeedOffset = el->seedOffset;
            bestScoreMatchProbability = el->matchProbabilityForBestScore;
        } else {
            if (-1 != maxEditDistanceForSecondaryResults && (int)((unsigned)bestScore - score) <= maxEditDistanceForSecondaryResults &&
                score != (unsigned)SG_SCORE_ABOVE_LIMIT && (unsigned)bestScore >= score) {
                if (maxSec <= *nSec) return false;
                snapgpu_single_result *r = &sec[*nSec];
                r->direction = el->direction; r->location = genomeLocation; r->origLocation = origGenomeLocation;
                r->mapq = 0; r->score = (int)score; r->status = SNAPGPU_MULTIPLE_HITS; r->clippingForReadAdjustment = 0;
                r->usedAffineGapScoring = el->usedAffineGapScoring; r->basesClippedBefore = el->basesClippedBefore;
                r->basesClippedAfter = el->basesClippedAfter; r->agScore = el->agScore; r->seedOffset = el->seedOffset;
                r->matchProbability = el->matchProbabilityForBestScore;
                r->scorePriorToClipping = 0; r->supplementary = 0; r->probabilityAllCandidates = 0; r->popularSeedsSkipped = 0; r->reserved = 0;
                (*nSec)++;
            }
        }
        return true;
    }
    SG_HD void initFrom(const snapgpu_single_result *r) {               // ScoreSet::init(SingleAlignmentResult*), :2116-2130
        bestScore = r->score; bestScoreGenomeLocation = r->location; bestScoreOrigGenomeLocation = r->origLocation;
        bestScoreDirection = r->direction; bestScoreUsedAffineGapScoring = r->usedAffineGapScoring;
        bestScoreBasesClippedBefore = r->basesClippedBefore; bestScoreBasesClippedAfter = r->basesClippedAfter;
        bestScoreAGScore = r->agScore; bestScoreSeedOffset = r->seedOffset; bestScoreMatchProbability = r->matchProbability;
        probabilityOfAllCandidates = r->probabilityAllCandidates; probabilityOfBestCandidate = r->matchProbability;
    }
    SG_HD void updateProbabilityOfAllMatches(double oldP) { double v = probabilityOfAllCandidates - oldP; probabilityOfAllCandidates = 0 > v ? 0 : v; }   // BaseAligner.h:282
    SG_HD void updateProbabilityOfBestMatch(double newP) { probabilityOfBestCandidate = newP; probabilityOfAllCandidates += newP; }
    SG_HD bool updateBestScoreFromResult(const snapgpu_single_result *r) {   // BaseAligner.h:308-326 (probabilityOfBestCandidate is NOT touched there)
        probabilityOfAllCandidates += r->matchProbability;
        if (r->agScore > bestScoreAGScore || (r->agScore == bestScoreAGScore && r->matchProbability > bestScoreMatchProbability)) {
            bestScore = r->score; bestScoreAGScore = r->agScore; bestScoreMatchProbability = r->matchProbability;
            bestScoreGenomeLocation = r->location; bestScoreOrigGenomeLocation = r->origLocation; bestScoreDirection = r->direction;
            bestScoreUsedAffineGapScoring = r->usedAffineGapScoring; bestScoreBasesClippedBefore = r->basesClippedBefore;
            bestScoreBasesClippedAfter = r->basesClippedAfter; bestScoreSeedOffset = r->seedOffset;
            return true;
        }
        return false;
    }
    SG_HDN void fillIn(const SgTables &T, snapgpu_single_result *r, int popularSeedsSkipped) const {   // :2301-2323
        r->agScore = bestScoreAGScore;
        r->basesClippedAfter = bestScoreBasesClippedAfter;
        r->basesClippedBefore = bestScoreBasesClippedBefore;
        r->clippingForReadAdjustment = 0;
        r->direction = bestScoreDirection;
        r->location = bestScoreGenomeLocation;
        r->origLocation = bestScoreOrigGenomeLocation;
        r->mapq = sg_compute_mapq(T, probabilityOfAllCandidates, probabilityOfBestCandidate, popularSeedsSkipped);
        r->score = bestScore;
        r->usedAffineGapScoring = bestScoreUsedAffineGapScoring;
        r->seedOffset = bestScoreSeedOffset;
        r->matchProbability = bestScoreMatchProbability;
        r->popularSeedsSkipped = (uint32_t)popularSeedsSkipped;
        r->status = (r->mapq >= SG_MAPQ_LIMIT_FOR_SINGLE_HIT) ? SNAPGPU_SINGLE_HIT : SNAPGPU_MULTIPLE_HITS;
        r->probabilityAllCandidates = probabilityOfAllCandidates;
    }
};

// The BaseAligner member state that lives across AlignRead()/score() for one read.
struct SgAligner {
    const SgIndexView *ix;
    const SgParams    *pr;
    const SgTables    *tb;
    SgScratch          sc;
    SgAgParams         ag;
    SgWork             work;
    uint32_t           maxK;         // BaseAligner::maxK: pr->maxK unless the paired caller lowered it (setMaxK, BaseAligner.h:118)

    // per-read state
    const uint8_t *readData[2], *readQual[2];   // [FORWARD] = input, [RC] = rcRead/rcQual
    uint32_t readLen;
    uint32_t nUsedElements, highestUsedWeightList, wrapCount, nAddedToHashTable, popularSeedsSkipped;
    uint32_t lowestPossibleScoreOfAnyUnseenLocation[2], currRoundLowestPossibleScoreOfAnyUnseenLocation[2];
    uint32_t mostSeedsContainingAnyParticularBase[2], nSeedsApplied[2];
    SgScoreSet all, nonAlt;
    int64_t invalidLocation;
    // candidatesForAffineGap of the Hamming pass (only the paired caller provides a buffer)
    snapgpu_single_result *agCands; int nAgCands, maxAgCands; int agCandsOverflow;
    SgScoreSet wsAll, wsNonAlt; snapgpu_single_result wsKey;     // working storage of alignAffineGap (stack objects in the reference)
    int deferred;                    // set by the DEFER instantiation when the read needs affine-gap scoring (see sg_align_read_t)
    // secondary alignments (`-om`; the SEC instantiation only): the caller's secondaryResults buffer and the three options that shape it
    snapgpu_single_result *secResults; int nSec, maxSec, secOverflow;
    int secMaxEditDist;              // maxEditDistanceForSecondaryResults = -om
    int secMaxResults;               // maxSecondaryResults = -omax
    int secMaxPerContig;             // maxSecondaryAlignmentsPerContig = -mpc (<= 0: no limit)

    // ---- weight lists: doubly linked FIFO per weight; link values are element indices or SG_SENTINEL+w ----
    SG_HD uint32_t getNext(uint32_t n) const { return (n & SG_SENTINEL) ? sc.listNext[n & ~SG_SENTINEL] : sc.pool[n].weightNext; }
    SG_HD uint32_t getPrev(uint32_t n) const { return (n & SG_SENTINEL) ? sc.listPrev[n & ~SG_SENTINEL] : sc.pool[n].weightPrev; }
    SG_HD void setNext(uint32_t n, uint32_t v) { if (n & SG_SENTINEL) sc.listNext[n & ~SG_SENTINEL] = v; else sc.pool[n].weightNext = v; }
    SG_HD void setPrev(uint32_t n, uint32_t v) { if (n & SG_SENTINEL) sc.listPrev[n & ~SG_SENTINEL] = v; else sc.pool[n].weightPrev = v; }

    SG_HD bool isALT(int64_t loc) const { return loc >= ix->altFirstLocation; }

    // BaseAligner::scoreLimit (:2555-2570).  All quantities are non-negative, so the reference's mixed
    // signed/unsigned __min chain reduces to plain integer minima.
    SG_HD int scoreLimit(bool forALT) const {
        int esd = (int)pr->extraSearchDepth, maxK = (int)this->maxK;
        if (pr->noUkkonen) { int v = maxK + esd; return v < SG_MAX_K - 1 ? v : SG_MAX_K - 1; }
        int inner;
        if (forALT) {
            int g = pr->maxScoreGapToPreferNonAltAlignment < nonAlt.bestScore ? pr->maxScoreGapToPreferNonAltAlignment : nonAlt.bestScore;
            int t = nonAlt.bestScore - g;
            inner = all.bestScore < t ? all.bestScore : t;
        } else {
            int t = all.bestScore + pr->maxScoreGapToPreferNonAltAlignment;
            inner = t < nonAlt.bestScore ? t : nonAlt.bestScore;
        }
        int v = esd + (maxK < inner ? maxK : inner);
        return v < SG_MAX_K - 1 ? v : SG_MAX_K - 1;
    }

    // ---- candidate lookup table (our own open-addressing map standing in for the epoch-cleared chained table,
    //      :340-364; only the key -> element mapping is observable) ----
    SG_HD uint32_t tableHash(uint32_t baseLoc, uint32_t dir) const {
        uint32_t k = (baseLoc / SG_ELEM_SIZE) * 2u + dir;
        k *= 0x9E3779B1u;
        return (k >> 7) & (pr->tableSlots - 1);
    }
    // findElement (:1810-1840): returns element index or ~0u
    SG_HD uint32_t findElement(uint32_t genomeLocation32, uint32_t dir) const {
        uint32_t base = genomeLocation32 - genomeLocation32 % SG_ELEM_SIZE;
        uint32_t s = tableHash(base, dir);
        for (;;) {
            uint32_t v = sc.table[s];
            if (v == 0) return ~0u;
            const SgElem &el = sc.pool[v - 1];
            if (el.baseGenomeLocation == base && el.direction == dir) return v - 1;
            s = (s + 1) & (pr->tableSlots - 1);
        }
    }
    // allocateNewCandidate (:1884-1973)
    SG_HD uint32_t allocateNewCandidate(uint32_t genomeLocation32, uint32_t dir, uint32_t lowestPossibleScore, int seedOffset) {
        uint32_t low = genomeLocation32 % SG_ELEM_SIZE;
        uint32_t base = genomeLocation32 - low;
        uint32_t ei = nUsedElements++;
        SgElem &el = sc.pool[ei];
        el.candidatesUsed = (uint64_t)1 << low;
        el.candidatesScored = 0;
        el.lowestPossibleScore = lowestPossibleScore;
        el.direction = (uint8_t)dir;
        el.weight = 1;
        el.baseGenomeLocation = base;
        el.bestScore = SG_UNUSED_SCORE;
        el.allExtantCandidatesScored = 0;
        el.matchProbabilityForBestScore = 0;
        el.usedAffineGapScoring = 0;
        el.basesClippedBefore = 0;
        el.basesClippedAfter = 0;
        el.agScore = 0;
        el.seedOffset = 0;
        el.bestScoreGenomeLocation = 0;
        // insert at the tail of weight list 1
        uint32_t head = SG_SENTINEL | 1u;
        uint32_t tail = getPrev(head);
        el.weightNext = head;
        el.weightPrev = tail;
        setPrev(head, ei);
        setNext(tail, ei);
        el.candSeedOffset[low] = (uint16_t)seedOffset;
        if (highestUsedWeightList < 1) highestUsedWeightList = 1;
        uint32_t s = tableHash(base, dir);
        while (sc.table[s] != 0) s = (s + 1) & (pr->tableSlots - 1);
        sc.table[s] = ei + 1;
        el.slot = s;
        return ei;
    }
    // incrementWeight (:2341-2379)
    SG_HD void incrementWeight(uint32_t ei) {
        SgElem &el = sc.pool[ei];
        if (el.allExtantCandidatesScored) return;
        if (el.weight >= pr->numWeightLists - 1) return;
        setPrev(el.weightNext, el.weightPrev);
        setNext(el.weightPrev, el.weightNext);
        el.weight++;
        if (highestUsedWeightList < el.weight) highestUsedWeightList = el.weight;
        uint32_t head = SG_SENTINEL | el.weight;
        uint32_t tail = getPrev(head);
        el.weightNext = head;
        el.weightPrev = tail;
        setPrev(head, ei);
        setNext(tail, ei);
    }
    // clearCandidates (:2331-2339), plus un-marking our lookup table
    SG_HD void clearCandidates() {
#if defined(__CUDA_ARCH__)
        {
            const uint32_t lane = (uint32_t)sg_lane(), nUsed = nUsedElements, nLists = pr->numWeightLists;
            #pragma unroll 1
            for (uint32_t i = lane; i < nUsed; i += 32) sc.table[sc.pool[i].slot] = 0;
            #pragma unroll 1
            for (uint32_t i = 1 + lane; i < nLists; i += 32) {
                sc.listNext[i] = SG_SENTINEL | i;
                sc.listPrev[i] = SG_SENTINEL | i;
            }
            __syncwarp();                // (this object is shared by the warp's lanes: no lane may still be reading nUsedElements)
            nUsedElements = 0;
            highestUsedWeightList = 0;
            __syncwarp();
            return;
        }
#endif
        for (uint32_t i = 0; i < nUsedElements; i++) sc.table[sc.pool[i].slot] = 0;
        nUsedElements = 0;
        highestUsedWeightList = 0;
        for (uint32_t i = 1; i < pr->numWeightLists; i++) {
            sc.listNext[i] = SG_SENTINEL | i;
            sc.listPrev[i] = SG_SENTINEL | i;
        }
    }

    SG_HD bool isSeedUsed(uint32_t i) const { return (sc.seedUsed[i / 8] & (1 << (i % 8))) != 0; }
    SG_HD void setSeedUsed(uint32_t i) { sc.seedUsed[i / 8] |= (uint8_t)(1 << (i % 8)); }
};

// Result of scoring one candidate location: the block :1117-1334 of BaseAligner::score.
struct SgCandScore {
    unsigned score; double matchProbability; int64_t genomeLocation; int usedAffineGapScoring;
    int basesClippedBefore, basesClippedAfter, agScore;
};

// HAM: the Hamming / gapless pass (AlignRead(..., useHamming = true)); a template parameter so that the stock pass carries none of its code.
// DEFER: an instantiation WITHOUT the affine-gap code: at the point where the reference would rescore with affine gap it sets
// A.deferred and unwinds; the caller then aligns that read again from scratch with the full instantiation (two-pass launch).
// sg_score inlines this in the DEFER instantiation and calls the out-of-line sg_score_candidate below in the others (see there).
// AGM: the affine-gap forms the kernel carries (sg_warp_ag_compute); 1 in the second pass of the two-pass launch.
template <bool HAM, bool DEFER, int AGM = 0>
SG_HD void sg_score_candidate_inl(SgAligner &A, const SgElem &el, int64_t genomeLocationIn, int seedOffset, int scoreLimitForThisElement, SgCandScore *o)
{
    const bool useHamming = HAM;
    const SgIndexView &ix = *A.ix; const SgParams &pr = *A.pr; const SgTables &T = *A.tb;
    int64_t genomeLocation = genomeLocationIn;
    unsigned score = (unsigned)SG_SCORE_ABOVE_LIMIT;
    double matchProbability = 0.0;
    const int dirn = el.direction;
    int readLen = (int)A.readLen;
    int64_t genomeDataLength = (int64_t)readLen + SG_MAX_K;
    const uint8_t *data = sg_get_substring(ix, genomeLocation, genomeDataLength);
    int usedAffineGapScoring = 0, basesClippedBefore = 0, basesClippedAfter = 0, agScore = -1;

    if (data != (const uint8_t *)0) {
        const uint8_t *readToScore = A.readData[dirn];
        const uint8_t *qualToScore = A.readQual[dirn];
        const uint8_t *oppQual = A.readQual[1 - dirn];
        const uint8_t *revRead = A.sc.revRead[dirn];
        double matchProb1 = 1.0, matchProb2 = 1.0;
        int score1 = 0, score2 = 0;
        int seedLen = (int)ix.seedLen;
        int tailStart = seedOffset + seedLen;
        int agScore1 = seedLen, agScore2 = 0;
        int maxKForSameAlignment = pr.gapOpenPenalty / (pr.subPenalty - pr.gapExtendPenalty);
        int genomeLocationOffset = 0;
        int64_t tl = genomeDataLength - tailStart;
        int textLen = (int)(tl < 0x7ffffff0 ? tl : 0x7ffffff0);

        int score1Gapless = 0, score2Gapless = 0;
        if (!useHamming) {
            SgLvResult lv;
            sg_lv_compute(T, A.sc, 1, data + tailStart, textLen, readToScore + tailStart, qualToScore + tailStart, readLen - tailStart,
                          scoreLimitForThisElement, &lv, sg_lane());
            score1 = lv.score; matchProb1 = lv.matchProbability;
            agScore1 = (seedLen + readLen - tailStart - score1) * pr.matchReward - score1 * pr.subPenalty;
            if (score1 != SG_SCORE_ABOVE_LIMIT) {
                int limitLeft = scoreLimitForThisElement - score1;
                sg_lv_compute(T, A.sc, -1, data + seedOffset, seedOffset + SG_MAX_K, revRead + readLen - seedOffset, oppQual + readLen - seedOffset,
                              seedOffset, limitLeft, &lv, sg_lane());
                score2 = lv.score; matchProb2 = lv.matchProbability; genomeLocationOffset = lv.netIndel;
                agScore2 = (seedOffset - score2) * pr.matchReward - score2 * pr.subPenalty;
            }
            A.work.lvCalls++;
        } else {
            // the Hamming / gapless pass (:1177-1199): extend from the seed without indels, clipping the poorly matching end
            SgGaplessOut g;
            if (tailStart != readLen) {
                g.nEdits = score1; g.matchProbability = matchProb1; g.nEditsGapless = score1Gapless;
                agScore1 = sg_gapless_compute(T, A.ag, 1, data + tailStart, textLen, readToScore + tailStart, qualToScore + tailStart, readLen - tailStart,
                                              readLen, scoreLimitForThisElement, &g);
                score1 = g.nEdits; matchProb1 = g.matchProbability; score1Gapless = g.nEditsGapless;
                agScore1 += (seedLen - readLen);
            }
            if (score1Gapless != SG_SCORE_ABOVE_LIMIT) {
                int limitLeft = scoreLimitForThisElement - score1Gapless;
                if (seedOffset != 0) {
                    g.nEdits = score2; g.matchProbability = matchProb2; g.nEditsGapless = score2Gapless; g.textOffset = genomeLocationOffset;
                    agScore2 = sg_gapless_compute(T, A.ag, -1, data + seedOffset, seedOffset + SG_MAX_K, revRead + readLen - seedOffset,
                                                  oppQual + readLen - seedOffset, seedOffset, readLen, limitLeft, &g);
                    score2 = g.nEdits; matchProb2 = g.matchProbability; score2Gapless = g.nEditsGapless; genomeLocationOffset = g.textOffset;
                    agScore2 -= readLen;
                    if (score2Gapless == SG_SCORE_ABOVE_LIMIT) genomeLocationOffset = 0;
                }
            }
        }

        if (!useHamming && score1 != SG_SCORE_ABOVE_LIMIT && score2 != SG_SCORE_ABOVE_LIMIT) {
            // :1203
            if (pr.noEditDistance || (pr.useAffineGap && (score1 + score2 > maxKForSameAlignment && el.lowestPossibleScore <= (unsigned)A.all.bestScore))) {
                if (DEFER) { A.deferred = 1; return; }
                score1 = 0; score2 = 0; agScore1 = seedLen; agScore2 = 0;
                usedAffineGapScoring = 1;
                A.work.agCalls++;
                SgAgResult ar;
                ar.textOffset = 0; ar.patternOffset = 0; ar.nEdits = 0; ar.matchProbability = 1.0; ar.agScore = -1;
                if (tailStart != readLen) {
                    int patternLen = readLen - tailStart;
                    bool banded = (patternLen >= (3 * (2 * scoreLimitForThisElement + 1))) && !pr.noBandedAffineGap;
                    sg_ag_dispatch<AGM>(T, A.sc, A.ag, 1, banded, data + tailStart, textLen, readToScore + tailStart, qualToScore + tailStart,
                                        patternLen, scoreLimitForThisElement, readLen, dirn != 0, false, &ar, sg_lane());
                    agScore1 = ar.agScore; basesClippedAfter = ar.patternOffset; score1 = ar.nEdits; matchProb1 = ar.matchProbability;
                    agScore1 += (seedLen - readLen);
                }
                if (score1 != SG_SCORE_ABOVE_LIMIT) {
                    if (seedOffset != 0) {
                        int limitLeft = scoreLimitForThisElement - score1;
                        int patternLen = seedOffset;
                        bool banded = (patternLen >= (3 * (2 * limitLeft + 1))) && !pr.noBandedAffineGap;
                        ar.textOffset = genomeLocationOffset; ar.patternOffset = basesClippedBefore; ar.matchProbability = matchProb2;
                        sg_ag_dispatch<AGM>(T, A.sc, A.ag, -1, banded, data + seedOffset, seedOffset + limitLeft, revRead + readLen - seedOffset,
                                            oppQual + readLen - seedOffset, seedOffset, limitLeft, readLen, dirn != 0, false, &ar, sg_lane());
                        agScore2 = ar.agScore; genomeLocationOffset = ar.textOffset; basesClippedBefore = ar.patternOffset;
                        score2 = ar.nEdits; matchProb2 = ar.matchProbability;
                        agScore2 -= readLen;
                    }
                }
            }
        }

        bool foundAlignment = useHamming ? (score1Gapless != SG_SCORE_ABOVE_LIMIT && score2Gapless != SG_SCORE_ABOVE_LIMIT)
                                         : (score1 != SG_SCORE_ABOVE_LIMIT && score2 != SG_SCORE_ABOVE_LIMIT);
        if (foundAlignment && genomeLocationOffset != 0 &&
            (const uint8_t *)0 == sg_get_substring(ix, genomeLocation + genomeLocationOffset, genomeDataLength)) {
            foundAlignment = false;
        }
        if (foundAlignment) {
            score = (unsigned)(score1 + score2);
            matchProbability = matchProb1 * matchProb2 * T.snpPowSeedLen;
            genomeLocation += genomeLocationOffset;
            agScore = agScore1 + agScore2;
        } else {
            score = (unsigned)SG_SCORE_ABOVE_LIMIT;
            agScore = SG_SCORE_ABOVE_LIMIT;
            matchProbability = 0.0;
        }
    } else {
        matchProbability = 0.0;
    }
    o->score = score; o->matchProbability = matchProbability; o->genomeLocation = genomeLocation;
    o->usedAffineGapScoring = usedAffineGapScoring; o->basesClippedBefore = basesClippedBefore; o->basesClippedAfter = basesClippedAfter;
    o->agScore = agScore;
}

// The call boundary of the full instantiations.  The first pass of the two-pass launch (DEFER, 40 registers at 6 CTAs per SM) does
// without it: every candidate crossed it there, and the registers saved and restored around it went through the per-lane stack, which
// every lane of the warp writes -- a 128-byte line per warp-uniform word.  Inlined, sg_align_kernel<6, 1> has a 624-byte frame instead
// of 720 and takes 20.0 ms instead of 22.1 per 1 M-read step on an H100 SXM (700 W; DESIGN.md section 8).
template <bool HAM, bool DEFER, int AGM = 0>
SG_HDN void sg_score_candidate(SgAligner &A, const SgElem &el, int64_t genomeLocationIn, int seedOffset, int scoreLimitForThisElement, SgCandScore *o)
{
    sg_score_candidate_inl<HAM, DEFER, AGM>(A, el, genomeLocationIn, seedOffset, scoreLimitForThisElement, o);
}

// BaseAligner::score (:917-1534).  Returns true iff a result was reached.
// SEC: the caller gave a secondaryResults buffer (`-om`): candidates within A.secMaxEditDist of the best are recorded as they are scored and the
// "nothing can rescue MAPQ" stop (:1512) is off; an overflow of the buffer sets A.secOverflow and ends the read (the reference returns false
// from AlignRead and its caller starts over with a larger buffer, SingleAligner.cpp:250-263).
template <bool HAM, bool DEFER, bool SEC = false, int AGM = 0>
SG_HDN bool sg_score(SgAligner &A, bool forceResult, snapgpu_single_result *primaryResult)
{
    const bool useHamming = HAM;
    const SgParams &pr = *A.pr; const SgTables &T = *A.tb;
    if (0 == A.mostSeedsContainingAnyParticularBase[0] && 0 == A.mostSeedsContainingAnyParticularBase[1]) {
        primaryResult->status = SNAPGPU_NOT_FOUND;
        primaryResult->mapq = 0;
        return true;
    }
    for (int direction = 0; direction < 2; direction++) {
        if (0 != A.mostSeedsContainingAnyParticularBase[direction]) {
            // EXACT_DISJOINT_MISS_COUNT is #defined at BaseAligner.cpp:42, so the bound is the number of seeds applied in
            // the current wrap round (:997-1000), not nSeedsApplied / mostSeedsContainingAnyParticularBase (:1002-1004).
            uint32_t v = A.currRoundLowestPossibleScoreOfAnyUnseenLocation[direction];
            if (A.lowestPossibleScoreOfAnyUnseenLocation[direction] < v) A.lowestPossibleScoreOfAnyUnseenLocation[direction] = v;
        }
    }

    uint32_t weightListToCheck = A.highestUsedWeightList;
    do {
        while (weightListToCheck > 0 && A.sc.listNext[weightListToCheck] == (SG_SENTINEL | weightListToCheck)) {
            weightListToCheck--;
            A.highestUsedWeightList = weightListToCheck;
        }
        uint32_t lpsMin = A.lowestPossibleScoreOfAnyUnseenLocation[0] < A.lowestPossibleScoreOfAnyUnseenLocation[1]
                              ? A.lowestPossibleScoreOfAnyUnseenLocation[0] : A.lowestPossibleScoreOfAnyUnseenLocation[1];
        int slT = A.scoreLimit(true), slF = A.scoreLimit(false);
        int slMax = slT > slF ? slT : slF;
        if ((lpsMin > (uint32_t)slMax && !pr.noTruncation) || forceResult) {
            if (weightListToCheck < pr.minWeightToCheck) {
                const SgScoreSet *fin;
                if (!pr.altAwareness || A.nonAlt.bestScore > A.all.bestScore + pr.maxScoreGapToPreferNonAltAlignment) {
                    fin = &A.all;
                } else {
                    fin = &A.nonAlt;
                }
                primaryResult->score = fin->bestScore;
                if (fin->bestScore <= (int)A.maxK || (useHamming && fin->bestScore != (int)SG_UNUSED_SCORE)) {
                    fin->fillIn(T, primaryResult, (int)A.popularSeedsSkipped);
                    primaryResult->supplementary = 0;
                    return true;
                } else {
                    primaryResult->status = SNAPGPU_NOT_FOUND;
                    primaryResult->mapq = 0;
                    return true;
                }
            }
            forceResult = true;
        } else if (weightListToCheck == 0) {
            return false;
        }

        uint32_t ei = A.sc.listNext[weightListToCheck];
        SgElem &el = A.sc.pool[ei];
        int scoreLimitForThisElement = A.scoreLimit(pr.altAwareness && A.isALT((int64_t)el.baseGenomeLocation));
        if (el.lowestPossibleScore <= (uint32_t)scoreLimitForThisElement) {
            uint64_t candidatesMask = el.candidatesUsed;
            while (candidatesMask != 0) {
                uint32_t candidateIndexToScore = 0;
#if defined(__CUDA_ARCH__)
                candidateIndexToScore = (uint32_t)(__ffsll((long long)candidatesMask) - 1);                       // _BitScanForward64
#else
                { uint64_t m = candidatesMask; while (!(m & 1)) { m >>= 1; candidateIndexToScore++; } }   // _BitScanForward64
#endif
                uint64_t candidateBit = (uint64_t)1 << candidateIndexToScore;
                candidatesMask &= ~candidateBit;
                if ((el.candidatesScored & candidateBit) != 0) continue;
                bool anyNearbyCandidatesAlreadyScored = el.candidatesScored != 0;
                el.candidatesScored |= candidateBit;

                int64_t genomeLocation = (int64_t)el.baseGenomeLocation + candidateIndexToScore;
                int64_t origGenomeLocation = genomeLocation;
                int64_t elementGenomeLocation = genomeLocation;
                bool genomeLocationIsNonALT = (!pr.altAwareness) || !A.isALT(genomeLocation);

                SgCandScore cs;
                if (DEFER) sg_score_candidate_inl<HAM, DEFER>(A, el, genomeLocation, (int)el.candSeedOffset[candidateIndexToScore], scoreLimitForThisElement, &cs);
                else sg_score_candidate<HAM, DEFER, AGM>(A, el, genomeLocation, (int)el.candSeedOffset[candidateIndexToScore], scoreLimitForThisElement, &cs);
                if (DEFER && A.deferred) return true;
                unsigned score = cs.score;
                double matchProbability = cs.matchProbability;
                genomeLocation = cs.genomeLocation;

                if (anyNearbyCandidatesAlreadyScored) {
                    if (useHamming && matchProbability <= el.matchProbabilityForBestScore) continue;      // :1362
                    if (el.bestScore < score || (el.bestScore == score && matchProbability <= el.matchProbabilityForBestScore)) {
                        continue;
                    }
                }
                el.bestScoreGenomeLocation = genomeLocation;
                el.usedAffineGapScoring = (uint8_t)cs.usedAffineGapScoring;
                el.basesClippedBefore = cs.basesClippedBefore;
                el.basesClippedAfter = cs.basesClippedAfter;
                el.agScore = cs.agScore;
                el.seedOffset = (int)el.candSeedOffset[candidateIndexToScore];

                uint32_t nearby = ~0u;
                if ((unsigned)SG_SCORE_ABOVE_LIMIT != score && score < 2) {
                    int64_t half = SG_ELEM_SIZE / 2;
                    int64_t nearbyGenomeLocation = elementGenomeLocation + (2 * ((elementGenomeLocation % SG_ELEM_SIZE) / half) - 1) * half;
                    // the reference keys its table on the 64-bit location, so a (negative / >32-bit) neighbour never matches
                    if (nearbyGenomeLocation >= 0 && nearbyGenomeLocation <= 0xffffffffLL) {
                        nearby = A.findElement((uint32_t)nearbyGenomeLocation, el.direction);
                    }
                }
                if (nearby != ~0u && A.sc.pool[nearby].candidatesScored != 0) {
                    SgElem &ne = A.sc.pool[nearby];
                    int64_t dist = genomeLocation - ne.bestScoreGenomeLocation; if (dist < 0) dist = -dist;
                    if (!(dist <= SG_MAX_MERGE_DIST)) {
                        nearby = ~0u;
                    } else {
                        if (useHamming && ne.matchProbabilityForBestScore >= matchProbability) continue;      // :1418
                        if (ne.bestScore < score || (ne.bestScore == score && ne.matchProbabilityForBestScore >= matchProbability)) {
                            continue;
                        }
                        A.all.updateProbabilitiesForNearbyMatch(ne.matchProbabilityForBestScore);
                        if (genomeLocationIsNonALT) A.nonAlt.updateProbabilitiesForNearbyMatch(ne.matchProbabilityForBestScore);
                        anyNearbyCandidatesAlreadyScored = true;
                        ne.matchProbabilityForBestScore = 0;
                    }
                }

                A.all.updateProbabilitiesForNewMatch(matchProbability, el.matchProbabilityForBestScore);
                if (genomeLocationIsNonALT) A.nonAlt.updateProbabilitiesForNewMatch(matchProbability, el.matchProbabilityForBestScore);
                el.matchProbabilityForBestScore = matchProbability;
                el.bestScore = score;

                if (useHamming && A.agCands != (snapgpu_single_result *)0) {
                    // :1444-1456: both score sets append to the same candidatesForAffineGap buffer
                    bool ok = A.all.updateBestScoreRecording(genomeLocation, origGenomeLocation, score, pr.useAffineGap != 0, cs.agScore, matchProbability, &el,
                                                             A.agCands, &A.nAgCands, A.maxAgCands, (int)pr.extraSearchDepth);
                    if (ok && genomeLocationIsNonALT) {
                        ok = A.nonAlt.updateBestScoreRecording(genomeLocation, origGenomeLocation, score, pr.useAffineGap != 0, cs.agScore, matchProbability, &el,
                                                               A.agCands, &A.nAgCands, A.maxAgCands, (int)pr.extraSearchDepth);
                    }
                    if (!ok || A.nAgCands >= A.maxAgCands) { A.agCandsOverflow = 1; return true; }      // :1475-1478 (the reference returns false = overflow)
                } else if (SEC) {
                    // :1457-1467: both score sets append to the same secondaryResults buffer (so, without ALT contigs, every record appears twice --
                    // the reference's own behaviour); the third call (:1480-1486) passes no buffer and finds nothing left to update
                    bool ok = A.all.updateBestScoreSecondary(genomeLocation, origGenomeLocation, score, pr.useAffineGap != 0, cs.agScore, matchProbability, &el,
                                                             A.secResults, &A.nSec, A.maxSec, A.secMaxEditDist);
                    if (ok && genomeLocationIsNonALT) {
                        ok = A.nonAlt.updateBestScoreSecondary(genomeLocation, origGenomeLocation, score, pr.useAffineGap != 0, cs.agScore, matchProbability, &el,
                                                               A.secResults, &A.nSec, A.maxSec, A.secMaxEditDist);
                    }
                    if (!ok) { A.secOverflow = 1; return true; }                                        // :1471-1473
                } else {
                    A.all.updateBestScore(genomeLocation, origGenomeLocation, score, pr.useAffineGap != 0, cs.agScore, matchProbability, &el);
                    if (genomeLocationIsNonALT) {
                        // the reference calls this twice more (:1463, :1484); with no secondary buffers the repeats are no-ops
                        A.nonAlt.updateBestScore(genomeLocation, origGenomeLocation, score, pr.useAffineGap != 0, cs.agScore, matchProbability, &el);
                    }
                }

                if (pr.stopOnFirstHit && ((A.all.bestScore <= (int)A.maxK) || (useHamming && A.all.bestScore != (int)SG_UNUSED_SCORE))) {
                    (pr.altAwareness ? A.nonAlt : A.all).fillIn(T, primaryResult, (int)A.popularSeedsSkipped);
                    primaryResult->status = SNAPGPU_MULTIPLE_HITS;
                    primaryResult->mapq = 0;
                    return true;
                }
                if ((pr.altAwareness ? A.nonAlt.probabilityOfAllCandidates : A.all.probabilityOfAllCandidates) >= 4.9 && (!SEC || -1 == A.secMaxEditDist)) {
                    (pr.altAwareness ? A.nonAlt : A.all).fillIn(T, primaryResult, (int)A.popularSeedsSkipped);
                    return true;
                }
            }
        }
        // remove the element from its weight list
        el.allExtantCandidatesScored = 1;
        A.setPrev(el.weightNext, el.weightPrev);
        A.setNext(el.weightPrev, el.weightNext);
        el.weightNext = el.weightPrev = ei;
    } while (forceResult);
    return false;
}

// BaseAligner::finalizeSecondaryResults (:2422-2553) with ignoreAlignmentAdjustmentsForOm (the default; the adjuster is not implemented, sg_derive_params
// refuses it): drop what is no longer within -om of the best (the last record moves into the hole, :2468-2485), cap the records per contig
// (-mpc, :2487-2547) and the total (-omax, :2549-2552).  The two qsort() calls are glibc's merge sort, i.e. stable: insertion sorts here.
SG_HDN void sg_finalize_secondary(SgAligner &A, snapgpu_single_result *primaryResult)
{
    const SgIndexView &ix = *A.ix; const SgParams &pr = *A.pr;
    snapgpu_single_result *sec = A.secResults;
    int n = A.nSec;
    const int bestScore = primaryResult->score;
    const int bound = bestScore + A.secMaxEditDist;
    const int worstScoreToKeep = (int)A.maxK < bound ? (int)A.maxK : bound;
    int i = 0;
    while (i < n) {
        if (sec[i].score > worstScoreToKeep) {
            sec[i] = sec[n - 1];
            n--;
        } else {
            sec[i].scorePriorToClipping = sec[i].score;
            sec[i].supplementary = (pr.altAwareness && A.isALT(sec[i].location)) ? 1 : 0;
            i++;
        }
    }
    if (A.secMaxPerContig > 0 && primaryResult->status != SNAPGPU_NOT_FOUND) {
        // Genome::getContigNumAtLocation (Genome.cpp:573-600) is a binary search over the contigs' beginningLocation
        #define SG_CONTIG_OF(LOC, OUT) { int lo_ = 0, hi_ = (int)ix.nContigs - 1; OUT = -1; const int64_t l_ = (LOC); \
            while (lo_ <= hi_) { const int mid_ = (lo_ + hi_) / 2; const int64_t b_ = ix.contigStart[mid_]; \
                if (b_ <= l_ && (mid_ == (int)ix.nContigs - 1 || ix.contigStart[mid_ + 1] > l_)) { OUT = mid_; break; } \
                else if (b_ <= l_) lo_ = mid_ + 1; else hi_ = mid_ - 1; } }
        int primaryContig; SG_CONTIG_OF(primaryResult->location, primaryContig);
        // :2498-2511 counts per contig with an epoch-stamped array; what matters is only whether any contig (the primary's starts at one) exceeds the cap
        bool anyContigHasTooManyResults = false;
        for (i = 0; i < n && !anyContigHasTooManyResults; i++) {
            int ci; SG_CONTIG_OF(sec[i].location, ci);
            int hits = (ci == primaryContig) ? 1 : 0;
            for (int j = 0; j <= i; j++) { int cj; SG_CONTIG_OF(sec[j].location, cj); if (cj == ci) hits++; }
            if (hits > A.secMaxPerContig) anyContigHasTooManyResults = true;
        }
        if (anyContigHasTooManyResults) {
            // qsort(compareByContigAndScore), AlignmentResult.cpp:29-50
            for (i = 1; i < n; i++) {
                snapgpu_single_result &key = A.wsKey;
                key = sec[i];
                int ck; SG_CONTIG_OF(key.location, ck);
                int j = i - 1;
                for (; j >= 0; j--) {
                    int cj; SG_CONTIG_OF(sec[j].location, cj);
                    if (cj > ck || (cj == ck && sec[j].score > key.score)) sec[j + 1] = sec[j]; else break;
                }
                sec[j + 1] = key;
            }
            int currentContigNum = -1, currentContigCount = 0, destResult = 0;
            for (int sourceResult = 0; sourceResult < n; sourceResult++) {
                int contigNum; SG_CONTIG_OF(sec[sourceResult].location, contigNum);
                if (contigNum != currentContigNum) {
                    currentContigNum = contigNum;
                    currentContigCount = (contigNum == primaryContig) ? 1 : 0;
                }
                currentContigCount++;
                if (currentContigCount <= A.secMaxPerContig) {
                    if (destResult != sourceResult) sec[destResult] = sec[sourceResult];
                    destResult++;
                }
            }
            n = destResult;
        }
        #undef SG_CONTIG_OF
    }
    if (n > A.secMaxResults) {
        // qsort(compareByScore), AlignmentResult.cpp:53-65, then truncate
        for (i = 1; i < n; i++) {
            snapgpu_single_result &key = A.wsKey;
            key = sec[i];
            int j = i - 1;
            while (j >= 0 && sec[j].score > key.score) { sec[j + 1] = sec[j]; j--; }
            sec[j + 1] = key;
        }
        n = A.secMaxResults;
    }
    A.nSec = n;
}

// BaseAligner::AlignRead (:272-763) for one read with the stock loop's arguments (SingleAligner.cpp:250).
// `result` must be caller-zeroed POD; on return it holds what the reference would have put in primaryResult.
template <bool HAM, bool DEFER = false, bool SEC = false, int AGM = 0>
SG_HDN void sg_align_read_t(SgAligner &A, const uint8_t *readData, const uint8_t *readQuality, uint32_t readLen, snapgpu_single_result *primaryResult)
{
    const SgIndexView &ix = *A.ix; const SgParams &pr = *A.pr; const SgTables &T = *A.tb;
    const uint32_t seedLen = ix.seedLen;
    A.all.bestScore = A.nonAlt.bestScore = SG_TOO_BIG_SCORE;

    uint32_t maxSeedsToUse;
    if (0 != pr.numSeedsFromCommandLine) {
        maxSeedsToUse = pr.numSeedsFromCommandLine;
    } else {
        maxSeedsToUse = (uint32_t)(int)(2 * pr.seedCoverage * readLen / (int)seedLen);
    }

    primaryResult->location = A.invalidLocation;
    primaryResult->direction = SNAPGPU_FORWARD;
    primaryResult->score = SG_UNUSED_SCORE;
    primaryResult->status = SNAPGPU_NOT_FOUND;
    primaryResult->clippingForReadAdjustment = 0;
    primaryResult->usedAffineGapScoring = 0;
    primaryResult->basesClippedBefore = 0;
    primaryResult->basesClippedAfter = 0;
    primaryResult->agScore = 0;
    primaryResult->seedOffset = 0;
    primaryResult->supplementary = 0;

    A.popularSeedsSkipped = 0;
    A.nAddedToHashTable = 0;
    A.readLen = readLen;
    if (DEFER) A.deferred = 0;
    if (SEC) { A.nSec = 0; A.secOverflow = 0; }            // :318-320

    if ((int)readLen < (int)seedLen) {
        return;                      // :360-366, "hopeless"
    }

    uint32_t countOfNs = 0;
#if defined(__CUDA_ARCH__)
    if (sg_lane() >= 0) {
        // the four derived strings (:388-396) are built 32 bases per step; every lane reads all of them afterwards
        #pragma unroll 1
        for (uint32_t i = sg_lane(); i < (readLen + 7) / 8; i += 32) A.sc.seedUsed[i] = 0;
        #pragma unroll 1
        for (uint32_t i = sg_lane(); i < readLen; i += 32) {
            uint8_t baseByte = readData[i];
            uint8_t complement = sg_complement(baseByte);
            A.sc.rcRead[readLen - i - 1] = complement;
            A.sc.rcQual[readLen - i - 1] = readQuality[i];
            A.sc.revRead[0][readLen - i - 1] = baseByte;
            A.sc.revRead[1][i] = complement;
            countOfNs += (baseByte == 'N') ? 1u : 0u;
        }
        countOfNs = __reduce_add_sync(0xffffffffu, countOfNs);
        __syncwarp();
    } else
#endif
    {
        for (uint32_t i = 0; i < (readLen + 7) / 8; i++) A.sc.seedUsed[i] = 0;
        for (uint32_t i = 0; i < readLen; i++) {
            uint8_t baseByte = readData[i];
            uint8_t complement = sg_complement(baseByte);
            A.sc.rcRead[readLen - i - 1] = complement;
            A.sc.rcQual[readLen - i - 1] = readQuality[i];
            A.sc.revRead[0][readLen - i - 1] = baseByte;
            A.sc.revRead[1][i] = complement;
            countOfNs += (baseByte == 'N') ? 1u : 0u;                  // nTable, :212-214
        }
    }
    if (countOfNs > A.maxK) {
        return;                      // :398-402
    }
    if (countOfNs > 0) {             // :407-420
        int minSeedToConsiderNing = 0;
        for (int i = 0; i < (int)readLen; i++) {
            if (sg_base_value(readData[i]) > 3) {
                int limit = (i + (int)seedLen - 1) < ((int)readLen - 1) ? (i + (int)seedLen - 1) : ((int)readLen - 1);
                int j0 = minSeedToConsiderNing > (i - (int)seedLen + 1) ? minSeedToConsiderNing : (i - (int)seedLen + 1);
                for (int j = j0; j <= limit; j++) A.setSeedUsed((uint32_t)j);
                minSeedToConsiderNing = limit + 1;
                if (minSeedToConsiderNing >= (int)readLen) break;
            }
        }
    }

    A.readData[0] = readData;   A.readQual[0] = readQuality;
    A.readData[1] = A.sc.rcRead; A.readQual[1] = A.sc.rcQual;

    A.clearCandidates();

    uint32_t nPossibleSeeds = readLen - seedLen + 1;
    uint32_t nextSeedToTest = 0;
    A.wrapCount = 0;
    A.lowestPossibleScoreOfAnyUnseenLocation[0] = A.lowestPossibleScoreOfAnyUnseenLocation[1] = 0;
    A.currRoundLowestPossibleScoreOfAnyUnseenLocation[0] = A.currRoundLowestPossibleScoreOfAnyUnseenLocation[1] = 0;
    A.mostSeedsContainingAnyParticularBase[0] = A.mostSeedsContainingAnyParticularBase[1] = 1;
    A.all.init(A.invalidLocation);
    if (pr.altAwareness) A.nonAlt.init(A.invalidLocation);
    A.nSeedsApplied[0] = A.nSeedsApplied[1] = 0;

    while (A.nSeedsApplied[0] + A.nSeedsApplied[1] < maxSeedsToUse) {
        if (nextSeedToTest >= nPossibleSeeds) {
            A.wrapCount++;
            if (A.wrapCount >= seedLen) {
                sg_score<HAM, DEFER, SEC, AGM>(A, true, primaryResult);
                primaryResult->scorePriorToClipping = primaryResult->score;     // finalizeSecondaryResults, :2442
                if (SEC && !A.secOverflow) sg_finalize_secondary(A, primaryResult);
                return;
            }
            nextSeedToTest = T.wrapSeed[A.wrapCount];
            A.mostSeedsContainingAnyParticularBase[0] = A.mostSeedsContainingAnyParticularBase[1] = A.wrapCount + 1;
            A.currRoundLowestPossibleScoreOfAnyUnseenLocation[0] = A.currRoundLowestPossibleScoreOfAnyUnseenLocation[1] = 0;
        }
        while (nextSeedToTest < nPossibleSeeds && A.isSeedUsed(nextSeedToTest)) nextSeedToTest++;
        if (nextSeedToTest >= nPossibleSeeds) continue;
        A.setSeedUsed(nextSeedToTest);

        uint64_t sb, srcb;
        SgHits hits;
#if defined(__CUDA_ARCH__)
        if (!sg_warp_seed_pack(readData + nextSeedToTest, seedLen, sg_lane(), &sb, &srcb)) continue;
        sg_warp_lookup_seed32(ix, sb, srcb, sg_lane(), &hits, &A.work.entriesProbed, &A.work.overflowWords);
#else
        if (!sg_seed_pack(readData + nextSeedToTest, seedLen, &sb, &srcb)) continue;
        sg_lookup_seed32(ix, sb, srcb, &hits, &A.work.entriesProbed, &A.work.overflowWords);
#endif
        A.work.lookups++;

        bool appliedEitherSeed = false;
        for (uint32_t direction = 0; direction < 2; direction++) {
            if (hits.nHits[direction] > pr.maxHits && !pr.explorePopularSeeds) {
                A.work.popularIgnored++;
                A.popularSeedsSkipped++;
            } else {
                uint32_t offset = (direction == 0) ? nextSeedToTest : (readLen - seedLen - nextSeedToTest);
                uint32_t limit = hits.nHits[direction] < pr.maxHits ? hits.nHits[direction] : pr.maxHits;
                A.work.overflowWords += (hits.nHits[direction] > 1) ? limit : 0;
                const uint32_t *hitList = hits.hits[direction];
#if defined(__CUDA_ARCH__)
                // long lists go through shared memory, one bulk asynchronous copy (TMA) per chunk (sg_warp_stage_hits)
                const bool stageHits = pr.tmaMinHits != 0 && limit >= pr.tmaMinHits && A.sc.hitStageWords != 0;
                uint32_t stagedFrom = 0, stagedN = 0, stagedLead = 0;
#endif
                #pragma unroll 1
                for (uint32_t i = 0; i < limit; i++) {
#if defined(__CUDA_ARCH__)
                    uint32_t hitWord;
                    if (stageHits) {
                        if (i >= stagedFrom + stagedN) {
                            stagedFrom = i;
                            stagedN = sg_warp_stage_hits(A.sc, hitList + i, limit - i, sg_lane(), &stagedLead);
                        }
                        hitWord = A.sc.hitStage[stagedLead + (i - stagedFrom)];
                    } else {
                        hitWord = hitList[i];
                    }
                    uint32_t genomeLocationOfThisHit = hitWord - offset;
#else
                    uint32_t genomeLocationOfThisHit = hitList[i] - offset;       // 32-bit wrap like the reference
#endif
                    uint32_t ei = A.findElement(genomeLocationOfThisHit, direction);
                    if (ei != ~0u) {
                        // findCandidate (:1873-1878)
                        SgElem &el = A.sc.pool[ei];
                        uint32_t low = genomeLocationOfThisHit % SG_ELEM_SIZE;
                        uint64_t bit = (uint64_t)1 << low;
                        el.allExtantCandidatesScored = (uint8_t)(el.allExtantCandidatesScored && ((el.candidatesUsed & bit) != 0));
                        el.candidatesUsed |= bit;
                        if (!pr.noOrderedEvaluation) A.incrementWeight(ei);
                        el.candSeedOffset[low] = (uint16_t)offset;
                    } else {
                        bool candidateIsALT = pr.altAwareness && A.isALT((int64_t)genomeLocationOfThisHit);
                        if (A.lowestPossibleScoreOfAnyUnseenLocation[direction] <= (uint32_t)A.scoreLimit(candidateIsALT) || pr.noTruncation) {
                            A.allocateNewCandidate(genomeLocationOfThisHit, direction, A.lowestPossibleScoreOfAnyUnseenLocation[direction], (int)offset);
                            A.nAddedToHashTable++;
                        }
                    }
                }
                A.nSeedsApplied[direction]++;
                A.currRoundLowestPossibleScoreOfAnyUnseenLocation[direction]++;
                appliedEitherSeed = true;
            }
        }
        nextSeedToTest += seedLen;

        if (appliedEitherSeed) {
            if (sg_score<HAM, DEFER, SEC, AGM>(A, false, primaryResult)) {
                primaryResult->scorePriorToClipping = primaryResult->score;
                if (SEC && !A.secOverflow) sg_finalize_secondary(A, primaryResult);
                return;
            }
        }
    }
    sg_score<HAM, DEFER, SEC, AGM>(A, true, primaryResult);
    primaryResult->scorePriorToClipping = primaryResult->score;
    if (SEC && !A.secOverflow) sg_finalize_secondary(A, primaryResult);
}

SG_HD void sg_align_read(SgAligner &A, const uint8_t *readData, const uint8_t *readQuality, uint32_t readLen, snapgpu_single_result *primaryResult,
                         bool useHamming = false)
{
    if (useHamming) sg_align_read_t<true>(A, readData, readQuality, readLen, primaryResult);
    else sg_align_read_t<false>(A, readData, readQuality, readLen, primaryResult);
}

// BaseAligner::scoreLocationWithAffineGap (:766-915): the affine-gap rescoring used by alignAffineGap below.  Note the
// asymmetry it has in the reference: the forward call passes useClippingOptimizations = true and no text offset, the
// reverse call leaves useClippingOptimizations at its default (false).
SG_HDN void sg_single_score_location_ag(SgAligner &A, int direction, int64_t genomeLocation, uint32_t seedOffset, int scoreLimit, int *score,
                                        double *matchProbability, int *genomeLocationOffset, int *basesClippedBefore, int *basesClippedAfter, int *agScore)
{
    const SgIndexView &ix = *A.ix; const SgParams &pr = *A.pr; const SgTables &T = *A.tb;
    const int readLen = (int)A.readLen;
    const int64_t genomeDataLength = (int64_t)readLen + SG_MAX_K;
    const uint8_t *data = sg_get_substring(ix, genomeLocation, genomeDataLength);
    *genomeLocationOffset = 0;
    if (data == (const uint8_t *)0) { *score = SG_SCORE_ABOVE_LIMIT; *matchProbability = 0; *genomeLocationOffset = 0; *agScore = SG_SCORE_ABOVE_LIMIT; return; }
    *basesClippedBefore = 0; *basesClippedAfter = 0;
    double matchProb1 = 1.0, matchProb2 = 1.0;
    int score1 = 0, score2 = 0;
    const int seedLen = (int)ix.seedLen;
    const int tailStart = (int)seedOffset + seedLen;
    int agScore1 = seedLen, agScore2 = 0;
    const int textLen = (int)(genomeDataLength - tailStart);
    const uint8_t *readToScore = A.readData[direction], *qualToScore = A.readQual[direction];
    SgAgResult ar;
    if (tailStart != readLen) {
        int patternLen = readLen - tailStart;
        bool banded = (patternLen >= (3 * (2 * scoreLimit + 1))) && !pr.noBandedAffineGap;
        ar.textOffset = 0; ar.patternOffset = *basesClippedAfter; ar.nEdits = score1; ar.matchProbability = matchProb1; ar.agScore = -1;
        sg_ag_dispatch(T, A.sc, A.ag, 1, banded, data + tailStart, textLen, readToScore + tailStart, qualToScore + tailStart, patternLen, scoreLimit, readLen,
                       direction != 0, true, &ar, sg_lane());
        agScore1 = ar.agScore; *basesClippedAfter = ar.patternOffset; score1 = ar.nEdits; matchProb1 = ar.matchProbability;
        agScore1 += (seedLen - readLen);
        A.work.agCalls++;
    }
    if (score1 != SG_SCORE_ABOVE_LIMIT) {
        if (seedOffset != 0) {
            int limitLeft = scoreLimit - score1;
            int patternLen = (int)seedOffset;
            bool banded = (patternLen >= (3 * (2 * limitLeft + 1))) && !pr.noBandedAffineGap;
            ar.textOffset = *genomeLocationOffset; ar.patternOffset = *basesClippedBefore; ar.nEdits = score2; ar.matchProbability = matchProb2; ar.agScore = -1;
            sg_ag_dispatch(T, A.sc, A.ag, -1, banded, data + seedOffset, (int)seedOffset + limitLeft, A.sc.revRead[direction] + readLen - seedOffset,
                           A.readQual[1 - direction] + readLen - seedOffset, patternLen, limitLeft, readLen, direction != 0, false, &ar, sg_lane());
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
        *agScore = agScore1 + agScore2;
    } else {
        *score = SG_SCORE_ABOVE_LIMIT; *agScore = -1; *matchProbability = 0.0;
    }
}

// BaseAligner::alignAffineGap (:1536-1784) for the read the aligner has just run AlignRead on (its RC / reversed strings and
// its member score sets, which scoreLimit() reads at :1757, are still in place).  No ALT result.
SG_HDN void sg_align_affine_gap(SgAligner &A, snapgpu_single_result *result, int nCands, snapgpu_single_result *cands)
{
    const SgParams &pr = *A.pr; const SgTables &T = *A.tb;
    if (result->status == SNAPGPU_NOT_FOUND) return;
    const int bestScore = result->score;
    int scoreLimitForCandidate = SG_MAX_K - 1;
    int genomeOffset = 0;
    bool skipAffineGap = false;
    const double oldProbabilityBestResult = result->matchProbability;
    const int maxKForSameAlignment = pr.gapOpenPenalty / (pr.subPenalty - pr.gapExtendPenalty);
    result->usedAffineGapScoring = 0;
    if (result->score > maxKForSameAlignment) {
        result->usedAffineGapScoring = 1;
        sg_single_score_location_ag(A, result->direction, result->origLocation, (uint32_t)result->seedOffset, scoreLimitForCandidate, &result->score,
                                    &result->matchProbability, &genomeOffset, &result->basesClippedBefore, &result->basesClippedAfter, &result->agScore);
        if (result->score != SG_SCORE_ABOVE_LIMIT) result->location = result->origLocation + genomeOffset;
        else result->status = SNAPGPU_NOT_FOUND;
    } else {
        skipAffineGap = true;
    }
    if (result->status == SNAPGPU_NOT_FOUND || result->score > SG_MAX_K - 1) {
        result->location = A.invalidLocation; result->mapq = 0; result->score = SG_SCORE_ABOVE_LIMIT; result->status = SNAPGPU_NOT_FOUND;
        result->clippingForReadAdjustment = 0; result->usedAffineGapScoring = 0; result->basesClippedBefore = 0; result->basesClippedAfter = 0;
        result->agScore = SG_SCORE_ABOVE_LIMIT; result->seedOffset = 0; result->matchProbability = 0.0;
        return;
    }
    SgScoreSet &all = A.wsAll, &nonAlt = A.wsNonAlt;
    nonAlt.init(A.invalidLocation);              // ScoreSet::ScoreSet() (default ctor calls init())
    const bool nonALTAlignment = (!pr.altAwareness) || !A.isALT(result->location);
    all.initFrom(result);
    if (nonALTAlignment) nonAlt.initFrom(result);
    if (!skipAffineGap) {
        const double newProbability = result->matchProbability;
        all.updateProbabilityOfAllMatches(oldProbabilityBestResult);
        all.updateProbabilityOfBestMatch(newProbability);
        if (nonALTAlignment) {
            nonAlt.updateProbabilityOfAllMatches(oldProbabilityBestResult);
            nonAlt.updateProbabilityOfBestMatch(newProbability);
        }
    }
    if (nCands > 0 && !skipAffineGap) {
        scoreLimitForCandidate = ((int)A.maxK < bestScore ? (int)A.maxK : bestScore) + (int)pr.extraSearchDepth;
        // qsort(compareByScore): stable (glibc merge sort, SURVEY 7.6)
        for (int i = 1; i < nCands; i++) {
            snapgpu_single_result &key = A.wsKey;
            key = cands[i];
            int j = i - 1;
            while (j >= 0 && cands[j].score > key.score) { cands[j + 1] = cands[j]; j--; }
            cands[j + 1] = key;
        }
        for (int i = 0; i < nCands; i++) {
            snapgpu_single_result *c = &cands[i];
            const bool nonALT = (!pr.altAwareness) || !A.isALT(c->location);
            const double oldProbability = c->matchProbability;
            c->usedAffineGapScoring = 1;
            sg_single_score_location_ag(A, c->direction, c->origLocation, (uint32_t)c->seedOffset, scoreLimitForCandidate, &c->score, &c->matchProbability,
                                        &genomeOffset, &c->basesClippedBefore, &c->basesClippedAfter, &c->agScore);
            if (c->score != SG_SCORE_ABOVE_LIMIT && (c->score <= SG_MAX_K - 1)) {
                c->location = c->origLocation + genomeOffset;
                if (result->location == c->location) continue;
                all.updateProbabilityOfAllMatches(oldProbability);
                all.updateBestScoreFromResult(c);
                if (nonALT) {
                    nonAlt.updateProbabilityOfAllMatches(oldProbability);
                    nonAlt.updateBestScoreFromResult(c);
                }
                scoreLimitForCandidate = A.scoreLimit(pr.altAwareness && !nonALT);       // the MEMBER score sets (:1757)
            }
        }
    }
    const SgScoreSet *emit = ((!pr.altAwareness) || nonAlt.bestScore > all.bestScore + pr.maxScoreGapToPreferNonAltAlignment) ? &all : &nonAlt;
    emit->fillIn(T, result, (int)result->popularSeedsSkipped);
}
