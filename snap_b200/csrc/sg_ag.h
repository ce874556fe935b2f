// sg_ag.h -- affine-gap seed extension, scalar *literal* restatement of the reference's striped SSE2 kernels:
// AffineGapVectorized<TEXT_DIRECTION>::computeScore (reference SNAPLib/AffineGapVectorized.h:821-1339) and
// computeScoreBanded (:256-819).  The reference's results depend on details of its Farrar layout -- the order in
// which the lazy-F loop visits vectors and the *joint* convergence test over the 8 lanes (:1080-1112), whole-vector
// band edges and state carried in H/E between rows in the banded variant (:447-528) -- so this restatement keeps
// the striped coordinates (vector index, lane) and walks them in the same order.  All cell values stay far from
// int16 saturation except the INT16_MIN padding profile, which is handled explicitly.
#pragma once
#include "sg_common.h"

// Counting points of the scalar form (tools/narrow_band_counts.py defines them; empty everywhere else): one call, and one
// (row, segment) unit with the number of lazy-F rounds it entered.
#ifndef SG_AG_CALL_HOOK
#define SG_AG_CALL_HOOK(banded, numVec, w, patternLen, textLen)
#endif
#ifndef SG_AG_UNIT_HOOK
#define SG_AG_UNIT_HOOK(row, seg, nVecHere, rounds) ((void)(rounds))
#endif
#include "sg_seed.h"

struct SgAgParams {
    int matchReward, subPenalty /* negative */, gapOpenPenalty /* open+extend */, gapExtendPenalty, fivePrimeEndBonus, threePrimeEndBonus;
    int usePacked;                   // device: take the specialised forms (packed s16x2 for unbanded problems, sg_warp_ag_rows_banded4 for
                                     // narrow bands); results are identical either way, which is faster depends on the kernel (DESIGN.md 6)
    int altLiftover;                 // the reference's useAltLiftover: no quality-aware end adjustment (AffineGapVectorized.h:691, 1212).
                                     // Only the general form honours it; its callers set usePacked = 0.
};

SG_HD SgAgParams sg_ag_params(int matchReward, int subPenalty, int gapOpen, int gapExtend, int five, int three)
{
    SgAgParams p;                    // AffineGapVectorized::init, :105-133
    p.matchReward = matchReward; p.subPenalty = -subPenalty; p.gapOpenPenalty = gapOpen + gapExtend;
    p.gapExtendPenalty = gapExtend; p.fivePrimeEndBonus = five; p.threePrimeEndBonus = three;
    p.usePacked = 0; p.altLiftover = 0;
    return p;
}

// The specialised device forms (packed s16x2 rows, narrow-band rows) do plain 16-bit arithmetic where the reference saturates, and
// the packed one pads with -16384 instead of INT16_MIN.  That is exact as long as no cell value can come near either: true for any
// sane scoring scheme, checked here so that an exotic one falls back to the general form (which saturates like the reference).
// The guard is about saturation only: every form keeps the query profile at full int16 width, so any match reward or substitution
// penalty is represented exactly.  tests/test_scoring_schemes.py pins which side of it each tested scheme falls on.
SG_HD bool sg_ag_small_scores(const SgAgParams &P, uint32_t maxReadLen)
{
    const long long top = (long long)(P.matchReward > 0 ? P.matchReward : 0) * ((long long)maxReadLen + SG_MAX_K + 1)
                          + (P.fivePrimeEndBonus > P.threePrimeEndBonus ? P.fivePrimeEndBonus : P.threePrimeEndBonus);
    const long long step = (long long)(-P.subPenalty > P.gapOpenPenalty ? -P.subPenalty : P.gapOpenPenalty);
    return P.matchReward >= 0 && P.subPenalty <= 0 && P.gapOpenPenalty >= 0 && P.gapExtendPenalty >= 0 && top < 12000 && step < 4000;
}

struct SgAgResult {
    int agScore, textOffset, patternOffset, nEdits;
    double matchProbability;
#ifdef SG_AG_POISON_CHECK
    int poisoned;
#endif
};

// ntTransitionMatrix (:123-132): equal ACGT -> match, different ACGT -> sub, anything with N (value 4) -> -1.
SG_HD int sg_ag_sub(const SgAgParams &P, uint32_t tb, uint32_t pb)
{
    if (tb > 3 || pb > 3) return -1;
    return tb == pb ? P.matchReward : P.subPenalty;
}

SG_HD int sg_sat16(int v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }

// One main-loop cell update (:1033-1072 / :487-526).  Returns new h; updates e (stored), f (register), action bits.
SG_HD int sg_ag_cell(const SgAgParams &P, int hdiag, int prof, int16_t *Ecell, int *f, uint8_t *act)
{
    int m = (hdiag > 0) ? sg_sat16(hdiag + prof) : 0;
    int e = *Ecell;
    uint8_t a = (e > m) ? 1 : 0;
    int h = m > e ? m : e;
    if (*f > h) a |= 2;
    if (*f > h) h = *f;
    int e2 = sg_sat16(e - P.gapExtendPenalty);
    int temp = sg_sat16(m - P.gapOpenPenalty);
    if (temp < 0) temp = 0;
    if (e2 > temp) a |= 4;
    *Ecell = (int16_t)(e2 > temp ? e2 : temp);
    int f2 = sg_sat16(*f - P.gapExtendPenalty);
    if (f2 > temp) a |= 32;
    *f = f2 > temp ? f2 : temp;
    *act = a;
    return h;
}

// Shared tail: local-vs-global choice, clipping heuristics and traceback (:1161-1338 / :642-818).
// btIndex(row, col) maps to the striped byte holding the 6 action bits.
struct SgAgLayout {
    int numVec, segLen, numSeg, banded, w, patternLen, nRows;
    // Was cell (row, col) written by the DP of this call?  Rows past the last one the row loop reached were not
    // (the clipping heuristics can start the traceback there); in the banded variant only whole in-band vectors are (:483).
    SG_HD bool computed(int row, int col) const {
        if (row >= nRows) return false;
        if (!banded) return true;
        int bandBeg = (row - w) > 0 ? (row - w) : 0;
        int bandEnd = (row + w) < (patternLen - 1) ? (row + w) : (patternLen - 1);
        int seg = col / segLen;
        if (seg < bandBeg / segLen || seg > bandEnd / segLen) return false;
        int k = (col % segLen) % numVec;
        return seg * segLen + k <= bandEnd;
    }
    SG_HD int cellIndex(int col) const {
        if (!banded) return (col % numVec) * SG_VEC + (col / numVec);
        int vecIdx = (col / segLen) * numVec + ((col % segLen) % numVec);
        int elemIdx = (col % segLen) / numVec;
        return vecIdx * SG_VEC + elemIdx;
    }
    SG_HD int rowStride() const { return banded ? numVec * numSeg * SG_VEC : numVec * SG_VEC; }
};

// Row pruning of the unbanded DP (ours; the reference walks all textLen rows).  After row i: every cell of a row r >= patternLen
// lies on a path that consumed r+1 text characters against at most patternLen pattern characters, so it holds at least
// r+1-patternLen vertical-gap steps and H(r, .) <= max(0, scoreInit + matchReward*patternLen - open - (r - patternLen)*ext),
// non-increasing in r.  Once that bound is below both running bests no later row can replace them (local needs >, global
// needs >=).  The only other use of later rows is the traceback, which the clipping heuristics of sg_ag_finish may start
// up to patternLen-1-bestLocalPatternOffset rows below the best local row: those rows are kept.
SG_HD bool sg_ag_can_stop_after_row(const SgAgParams &P, int i, int patternLen, int scoreInit, int bestLocalScore, int bestLocalTextOffset,
                                    int bestLocalPatternOffset, int bestGlobalScore)
{
    if (i + 1 < patternLen) return false;
    int ub = scoreInit + (P.matchReward > 0 ? P.matchReward : 0) * patternLen - P.gapOpenPenalty - (i + 1 - patternLen) * P.gapExtendPenalty;
    if (ub < 0) ub = 0;              // H is floored at 0
    if (!(ub < bestLocalScore && ub < bestGlobalScore)) return false;
    return i >= bestLocalTextOffset + (patternLen - 1 - bestLocalPatternOffset);
}

SG_HDN void sg_ag_finish(const SgTables &T, const SgAgParams &P, const SgAgLayout &lay, const uint8_t *bt, int dir,
                         const uint8_t *text /* already decremented for dir==-1 */, const uint8_t *pattern, const uint8_t *quality,
                         int patternLen, int scoreInit, int endBonus, bool useClippingOptimizations,
                         int bestLocalAlignmentScore, int bestLocalAlignmentTextOffset, int bestLocalAlignmentPatternOffset,
                         int bestGlobalAlignmentScore, int bestGlobalAlignmentTextOffset, SgAgResult *out)
{
    int score;
    int oPat, oText;
    if ((bestLocalAlignmentScore != bestGlobalAlignmentScore) && (bestLocalAlignmentScore >= bestGlobalAlignmentScore + endBonus)) {
        oPat = bestLocalAlignmentPatternOffset;
        oText = bestLocalAlignmentTextOffset;
        score = bestLocalAlignmentScore;
        if (useClippingOptimizations) {
            int patternOffsetAdj = oPat - 1;
            int textOffsetAdj = oText;
            int countEndMatches = 0;
            while ((patternOffsetAdj + 1 != patternLen) && pattern[patternOffsetAdj + 1] == text[(textOffsetAdj + 1) * dir]) {
                countEndMatches++; patternOffsetAdj++; textOffsetAdj++;
            }
            if (countEndMatches >= 3) {
                oPat = patternOffsetAdj; oText = textOffsetAdj;
            } else {
                patternOffsetAdj = oPat + 1;
                textOffsetAdj = oText;
                countEndMatches = 0;
                while ((patternOffsetAdj < patternLen) && pattern[patternOffsetAdj] == text[textOffsetAdj * dir]) {
                    countEndMatches++; patternOffsetAdj++; textOffsetAdj++;
                }
                if (countEndMatches >= 3) {
                    oPat = patternOffsetAdj - 1; oText = textOffsetAdj - 1;
                }
            }
            if (oPat == bestLocalAlignmentPatternOffset && oText == bestLocalAlignmentTextOffset && !P.altLiftover) {
                patternOffsetAdj = oPat;
                while (patternOffsetAdj != patternLen - 1 && (int8_t)quality[patternOffsetAdj] >= 65 && (int8_t)quality[patternOffsetAdj + 1] >= 65) {
                    patternOffsetAdj += 1;
                }
                if (patternOffsetAdj == patternLen - 1) {
                    oPat = patternOffsetAdj;
                } else if (patternOffsetAdj >= oPat + 2) {
                    int tmpOffset = patternOffsetAdj + 1;
                    int countRemHighQualityBases = 0;
                    int remPatternLen = patternLen - tmpOffset;
                    while (tmpOffset != patternLen - 1) {
                        if ((int8_t)quality[tmpOffset] >= 65) countRemHighQualityBases++;
                        tmpOffset++;
                    }
                    float ratio = ((float)countRemHighQualityBases) / (float)remPatternLen;
                    if ((double)ratio < 0.1) oPat = patternOffsetAdj;
                }
            }
        }
    } else {
        oPat = patternLen - 1;
        oText = bestGlobalAlignmentTextOffset;
        score = bestGlobalAlignmentScore;
    }

    out->patternOffset = oPat; out->textOffset = oText;
    if (score > scoreInit) {
        int rowIdx = oText, colIdx = oPat;
        int action = 0, prevAction = 0;          // M=0 D=1 I=2 X=3
        int actionCount = 1;
        int nMatches = 0, nMismatches = 0, nGaps = 0;
        double mp = 1.0;
        const int stride = lay.rowStride();
        // striped position of colIdx, maintained incrementally (no divisions in the loop): segment, SSE lane, vector
        int cSeg = colIdx / lay.segLen, cLane = (colIdx % lay.segLen) / lay.numVec, cVec = (colIdx % lay.segLen) % lay.numVec;
        while (rowIdx >= 0 && colIdx >= 0) {
            int matrixIdx = action << 1;
            const int cIdx = (cSeg * lay.numVec + cVec) * SG_VEC + cLane;
            // A traceback step can land on a cell this call never wrote.  The reference then reads whatever an *earlier*
            // call of the same object left in its never-cleared backtraceAction array (:1374); we keep the array persistent
            // per worker and per direction with the same linear layout, so the same stale bits are read whenever the
            // history is the same (always true within one read; across reads it depends on which thread/warp ran what).
            uint8_t cell = bt[(size_t)rowIdx * stride + cIdx];
#ifdef SG_AG_POISON_CHECK
            if (!lay.computed(rowIdx, colIdx)) out->poisoned = 1;
#endif
            action = (cell >> matrixIdx) & 3;
            if (action == 0) {
                if (pattern[colIdx] != text[rowIdx * dir]) {
                    mp *= T.phred[quality[colIdx]];
                    nMismatches++;
                } else {
                    nMatches++;
                }
                rowIdx--; colIdx--;
                if (--cVec < 0) { cVec = lay.numVec - 1; if (--cLane < 0) { cLane = SG_VEC - 1; cSeg--; } }
            } else if (action == 1) {
                rowIdx--;
            } else {
                colIdx--;
                if (--cVec < 0) { cVec = lay.numVec - 1; if (--cLane < 0) { cLane = SG_VEC - 1; cSeg--; } }
                action = 2;
            }
            if (prevAction != 0) {
                if (prevAction == action) {
                    actionCount++;
                } else {
                    nGaps += actionCount;
                    mp *= T.indel[actionCount];
                    actionCount = 1;
                }
            }
            prevAction = action;
        }
        if (rowIdx >= 0) {
            actionCount = rowIdx + 1;
            nGaps += actionCount;
            mp *= T.indel[actionCount];
        }
        if (colIdx >= 0) {
            actionCount = colIdx + 1;
            nGaps += actionCount;
            mp *= T.indel[actionCount];
        }
        out->nEdits = nMismatches + nGaps;
        mp *= T.perfect[nMatches];
        oText += 1; oPat += 1;
        oText = patternLen - oText;
        oPat = patternLen - oPat;
        mp *= T.indel[oPat];
        out->textOffset = oText; out->patternOffset = oPat;
        out->matchProbability = mp;
        out->agScore = score;
    } else {
        out->agScore = -1;
    }
}

// Lazy-F pass over vectors [vecBase, vecBase+nVecHere) of the current row (:1080-1112 / :534-569).
// Returns true if it converged (the reference's `goto got_answer`).
SG_HD bool sg_ag_lazy_pass(const SgAgParams &P, int16_t *Hcur, uint8_t *btRow, int vecBase, int nVecHere, int *f, int *maxv)
{
    for (int v = 0; v < nVecHere; v++) {
        bool anyLive = false;
        for (int l = 0; l < SG_VEC; l++) {
            int idx = (vecBase + v) * SG_VEC + l;
            int h = Hcur[idx];
            uint8_t a = btRow[idx];
            if (f[l] > h) { a |= 2; h = f[l]; }
            Hcur[idx] = (int16_t)h;
            if (h > maxv[l]) maxv[l] = h;
            int temp = h - P.gapOpenPenalty; if (temp < 0) temp = 0;      // _mm_subs_epu16 on non-negative values
            int fl = f[l] - P.gapExtendPenalty; if (fl < 0) fl = 0;
            f[l] = fl;
            if (fl > temp) { a |= 32; anyLive = true; }
            btRow[idx] = a;
        }
        if (!anyLive) return true;
    }
    return false;
}

SG_HDN void sg_ag_compute(const SgTables &T, const SgScratch &S, const SgAgParams &P, int dir, bool banded,
                          const uint8_t *text, int textLen, const uint8_t *pattern, const uint8_t *quality, int patternLen,
                          int w, int scoreInit, bool isRC, bool useClippingOptimizations, SgAgResult *out)
{
    // `out` is in/out like the reference's o_* pointers: on the two early returns below textOffset / patternOffset
    // (and for w < 0 also matchProbability) are left as the caller initialised them (:860-893).
    out->agScore = -1;
    if (w > SG_MAX_K - 1) w = SG_MAX_K - 1;
    if (text == (const uint8_t *)0) { out->matchProbability = 0.0; out->nEdits = -1; return; }
    if (w < 0) { out->nEdits = SG_SCORE_ABOVE_LIMIT; return; }
    out->matchProbability = 1.0;
    out->textOffset = -1; out->patternOffset = -1; out->nEdits = -1;
    if (dir == -1) text--;

    SgAgLayout lay;
    lay.banded = banded ? 1 : 0;
    if (banded) {
        int bandWidth = (2 * w + 1) < patternLen ? (2 * w + 1) : patternLen;
        lay.numVec = (bandWidth + SG_VEC - 1) / SG_VEC;
        lay.segLen = lay.numVec * SG_VEC;
        lay.numSeg = (patternLen + lay.segLen - 1) / lay.segLen;
    } else {
        lay.numVec = (patternLen + SG_VEC - 1) / SG_VEC;
        lay.segLen = lay.numVec * SG_VEC;
        lay.numSeg = 1;
    }
    lay.w = w; lay.patternLen = patternLen;
    const int numVec = lay.numVec, segLen = lay.segLen, numSeg = lay.numSeg;
    const int stride = lay.rowStride();
    SG_AG_CALL_HOOK(banded, numVec, w, patternLen, textLen);

    int endBonus;                    // :950-966
    if (!isRC) endBonus = (dir == -1) ? P.fivePrimeEndBonus : P.threePrimeEndBonus;
    else       endBonus = (dir == -1) ? P.threePrimeEndBonus : P.fivePrimeEndBonus;

    int16_t *Hptr = S.agH, *Hm1ptr = S.agHm1, *E = S.agE;
    uint8_t *bt = S.agBt[dir == 1 ? 0 : 1];
#ifdef SG_AG_POISON_CHECK
    out->poisoned = 0;
#endif

    // first row (:971-983 / :399-414); scoreFirstRow[] deliberately persists across vecIdx like the reference's
    {
        int scoreFirstRow[SG_VEC];
        for (int l = 0; l < SG_VEC; l++) scoreFirstRow[l] = 0;
        for (int segIdx = 0; segIdx < numSeg; segIdx++) {
            for (int vecIdx = 0; vecIdx < numVec; vecIdx++) {
                for (int l = 0; l < SG_VEC; l++) {
                    int patternIdx = segIdx * segLen + l * numVec + vecIdx;
                    if (patternIdx < patternLen) {
                        int v = scoreInit - P.gapOpenPenalty - patternIdx * P.gapExtendPenalty;
                        scoreFirstRow[l] = v > 0 ? v : 0;
                    }
                    int idx = (segIdx * numVec + vecIdx) * SG_VEC + l;
                    Hptr[idx] = (int16_t)scoreFirstRow[l];
                    Hm1ptr[idx] = 0;     // banded zeroes Hminus1 (:411); the full variant overwrites it before use
                    E[idx] = 0;
                }
            }
        }
    }

    int bestGlobalAlignmentScore = -1, bestGlobalAlignmentTextOffset = -1;
    int bestLocalAlignmentScore = -1, bestLocalAlignmentTextOffset = -1, bestLocalAlignmentPatternOffset = -1;

    lay.nRows = 0;
    for (int i = 0; i < textLen; i++) {
        lay.nRows = i + 1;
        const uint32_t tb = sg_base_value(text[i * dir]);
        uint8_t *btRow = bt + (size_t)i * stride;
        int f[SG_VEC], maxv[SG_VEC], X[SG_VEC], h[SG_VEC];
        for (int l = 0; l < SG_VEC; l++) { f[l] = 0; maxv[l] = 0; X[l] = 0; }
        int localAlignmentPatternOffset = -1;

        int bandBeg = 0, bandEnd = patternLen - 1, segBeg = 0, segEnd = 0;
        if (banded) {
            bandBeg = (i - w) > 0 ? (i - w) : 0;
            bandEnd = (i + w) < (patternLen - 1) ? (i + w) : (patternLen - 1);
            segBeg = bandBeg / segLen;
            segEnd = bandEnd / segLen;
        }

        for (int j = segBeg; j <= segEnd; j++) {
            // h = shifted last vector of this segment from the previous row, lane 0 = initial value
            for (int l = SG_VEC - 1; l > 0; l--) h[l] = Hptr[(j * numVec + numVec - 1) * SG_VEC + l - 1];
            int hInit;
            if (j == 0) {
                hInit = scoreInit;
                if (i > 0) { hInit = scoreInit - P.gapOpenPenalty - (i - 1) * P.gapExtendPenalty; if (hInit < 0) hInit = 0; }
            } else {
                if (bandBeg > j * segLen) hInit = 0;
                else hInit = Hptr[(j * numVec - 1) * SG_VEC + (SG_VEC - 1)];
            }
            h[0] = hInit;

            int nVecHere = numVec;
            if (banded) {
                int lim = bandEnd - j * segLen + 1;   // k with j*segLen + k <= bandEnd
                if (lim < nVecHere) nVecHere = lim;
                if (nVecHere < 0) nVecHere = 0;
            }
            for (int k = 0; k < nVecHere; k++) {
                for (int l = 0; l < SG_VEC; l++) {
                    int col = j * segLen + l * numVec + k;
                    int prof = (col < patternLen) ? sg_ag_sub(P, tb, sg_base_value(pattern[col])) : -32768;
                    int idx = (j * numVec + k) * SG_VEC + l;
                    uint8_t a;
                    int hh = sg_ag_cell(P, h[l], prof, &E[idx], &f[l], &a);
                    if (hh > maxv[l]) maxv[l] = hh;
                    Hm1ptr[idx] = (int16_t)hh;
                    btRow[idx] = a;
                    h[l] = Hptr[idx];
                }
            }

            // lazy F
            int passes = banded ? (SG_VEC - 1) : SG_VEC, rounds = 0;
            for (int kk = 0; kk < passes; kk++) {
                rounds++;
                if (banded) { if (f[SG_VEC - 1] > X[0]) X[0] = f[SG_VEC - 1]; }   // X = max(X, f >> 7 lanes) (:537)
                for (int l = SG_VEC - 1; l > 0; l--) f[l] = f[l - 1];
                f[0] = 0;
                if (sg_ag_lazy_pass(P, Hm1ptr, btRow, j * numVec, nVecHere, f, maxv)) break;
            }
            SG_AG_UNIT_HOOK(i, j, nVecHere, rounds);
            if (banded) { for (int l = 0; l < SG_VEC; l++) f[l] = X[l]; }          // pass f on to the next segment (:572)
        }

        int maxScoreRow = 0;
        for (int l = 0; l < SG_VEC; l++) if (maxv[l] > maxScoreRow) maxScoreRow = maxv[l];

        if (!banded || bandEnd == patternLen - 1) {
            int globalAlignmentScore = Hm1ptr[lay.cellIndex(banded ? bandEnd : patternLen - 1)];
            if (globalAlignmentScore >= bestGlobalAlignmentScore) {
                bestGlobalAlignmentScore = globalAlignmentScore;
                bestGlobalAlignmentTextOffset = i;
            }
        }

        if (maxScoreRow == 0) break;

        if (maxScoreRow > bestLocalAlignmentScore) {
            for (int j = segBeg; j <= segEnd; j++) {
                int nVecHere = numVec;
                if (banded) {
                    int lim = bandEnd - j * segLen + 1;
                    if (lim < nVecHere) nVecHere = lim;
                }
                for (int k = 0; k < nVecHere; k++) {
                    int top = -1;
                    for (int l = 0; l < SG_VEC; l++) if (Hm1ptr[(j * numVec + k) * SG_VEC + l] == maxScoreRow) top = l;
                    if (top >= 0) {
                        int patternOffset = j * segLen + top * numVec + k;
                        if (patternOffset > localAlignmentPatternOffset) localAlignmentPatternOffset = patternOffset;
                    }
                }
            }
            bestLocalAlignmentScore = maxScoreRow;
            bestLocalAlignmentTextOffset = i;
            bestLocalAlignmentPatternOffset = localAlignmentPatternOffset;
        }

        if (!banded && sg_ag_can_stop_after_row(P, i, patternLen, scoreInit, bestLocalAlignmentScore, bestLocalAlignmentTextOffset,
                                                bestLocalAlignmentPatternOffset, bestGlobalAlignmentScore)) break;

        int16_t *tmp = Hm1ptr; Hm1ptr = Hptr; Hptr = tmp;
    }

    sg_ag_finish(T, P, lay, bt, dir, text, pattern, quality, patternLen, scoreInit, endBonus, useClippingOptimizations,
                 bestLocalAlignmentScore, bestLocalAlignmentTextOffset, bestLocalAlignmentPatternOffset,
                 bestGlobalAlignmentScore, bestGlobalAlignmentTextOffset, out);
}

// AffineGapVectorized<dir>::computeGaplessScore (AffineGapVectorized.h:139-255): Hamming extension from the seed with the
// poorly matching end clipped at the prefix of maximum score.  In/out like the reference: *o_nEdits, *o_textOffset,
// *o_patternOffset, *matchProbability and *o_nEditsGapless are only written on the paths that write them there
// (pass NULL for the ones the caller passes NULL for).  `dir` = +1 forward text, -1 text read backwards from text-1.
struct SgGaplessOut { int nEdits, textOffset, patternOffset, nEditsGapless; double matchProbability; };

SG_HDN int sg_gapless_compute(const SgTables &T, const SgAgParams &P, int dir, const uint8_t *text, int textLen, const uint8_t *pattern,
                              const uint8_t *quality, int patternLen, int scoreInit, int scoreLimit, SgGaplessOut *o)
{
    (void)textLen;
    if (scoreLimit < 0 || (const uint8_t *)0 == text) {
        o->nEdits = SG_SCORE_ABOVE_LIMIT; o->nEditsGapless = SG_SCORE_ABOVE_LIMIT;
        return SG_SCORE_ABOVE_LIMIT;
    }
    o->matchProbability = 1.0;
    if (dir == -1) text--;
    int gapLessScore = scoreInit, maxScore = scoreInit, best = 0;
    #pragma unroll 1
    for (int i = 0; i < patternLen; i++) {
        gapLessScore += (pattern[i] == text[i * dir]) ? P.matchReward : P.subPenalty;
        if (gapLessScore > maxScore) { maxScore = gapLessScore; best = i; }
    }
    if (maxScore > scoreInit) {
        int nEdits = 0, nMatches = 0;
        double mp = 1.0;
        #pragma unroll 1
        for (int i = 0; i <= best; i++) {
            if (pattern[i] != text[i * dir]) { nEdits += 1; mp *= T.phred[quality[i]]; }
            else nMatches++;
        }
        mp *= T.perfect[nMatches];
        int po = patternLen - (best + 1);
        o->patternOffset = po;
        o->textOffset = po;
        o->nEditsGapless = (nEdits <= scoreLimit) ? nEdits : -1;
        o->nEdits = nEdits + po;
        mp *= T.indel[po];
        o->matchProbability = mp;
        return maxScore;
    }
    o->nEdits = SG_SCORE_ABOVE_LIMIT; o->nEditsGapless = SG_SCORE_ABOVE_LIMIT;
    return SG_SCORE_ABOVE_LIMIT;
}
