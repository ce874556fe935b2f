// sg_warp_ag.cuh -- affine-gap seed extension, one warp per (text, pattern) pair (device only).
//
// Same results as the scalar restatement in sg_ag.h (which itself walks the reference's striped SSE2 coordinates,
// AffineGapVectorized.h:256-819 / :821-1339), bit for bit, with the work of one DP row spread over the warp:
//
//   lane = q*8 + l      l = the SSE lane of the reference's 8 x int16 vector, q = one of 4 consecutive vectors.
//
// A block of 4 striped vectors (32 cells, contiguous in the H / E / traceback arrays => coalesced 64 B / 32 B rows)
// is processed per step.  Everything in a cell except the horizontal-gap value F is independent of the other cells of
// the row; F is a max-plus prefix over the vectors of one SSE lane (f' = max(f - ext, temp)), which the 4 sub-lanes
// resolve with 3 shuffles, carrying the block's outgoing F to the next block.  The lazy-F loop of the reference
// decays F by a constant per vector independently of H, so a whole block of it is evaluated at once and the
// reference's "stop at the first vector where no lane can still change H" is recovered from a ballot: only vectors up to
// that one are committed.  Integer DP on int16-range values: DPX-style min/max, no tensor cores.
#pragma once
#include "sg_ag.h"
#include "sg_warp_ag_packed.cuh"
#include "sg_warp_ag_duo.cuh"


__device__ __forceinline__ int sg_shfl(int v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// The banded DP for bands of up to 32 columns (numVec <= 4, i.e. w <= 15: every `snap single -d 14` rescoring): each
// (row, segment) is ONE block of 4 vectors, every lane owns one cell, which stays in registers through the main pass and all
// lazy-F passes and is written once.  Exactly the nBlocks == 1 case of the general row loop in sg_warp_ag_compute, in a
// function of its own so that its loop carries no state of the other cases (registers: the kernels run at 64 per thread,
// and the general function spills inside its loops) and its code is one small contiguous piece.
__device__ __noinline__ void sg_warp_ag_rows_banded4(const SgScratch &S, int open, int ext, int dir, const uint8_t *text, int textLen, int patternLen,
                                                     int w, int scoreInit, SgAgLayout &lay, uint8_t *bt, int lane, SgAgBests *res)
{
    const int numVec = lay.numVec, segLen = lay.segLen;
    const int stride = lay.rowStride();
    const int l = lane & 7, q = lane >> 3;
    int16_t *Hptr = S.agH, *Hm1ptr = S.agHm1, *E = S.agE;
    const int16_t *prof = S.agProf;
    int bestG = -1, bestGT = -1, bestL = -1, bestLT = -1, bestLP = -1;
    const int globalIdx = lay.cellIndex(patternLen - 1);
    int segBegTrack = 0, segEndTrack = ((w < patternLen - 1) ? w : (patternLen - 1)) / segLen;
    const int laneUp = (lane & 24) | ((l + 7) & 7);

    #pragma unroll 1
    for (int i = 0; i < textLen; i++) {
        const uint32_t tb = sg_base_value(text[i * dir]);
        uint8_t *btRow = bt + (size_t)i * stride;
        const int16_t *profRow = prof + tb * stride;
        int myMax = 0, myMaxCol = -1, X0 = 0;
        const int bandBeg = (i - w) > 0 ? (i - w) : 0;
        const int bandEnd = (i + w) < (patternLen - 1) ? (i + w) : (patternLen - 1);
        while (bandBeg >= (segBegTrack + 1) * segLen) segBegTrack++;
        while (bandEnd >= (segEndTrack + 1) * segLen) segEndTrack++;

        #pragma unroll 1
        for (int j = segBegTrack; j <= segEndTrack; j++) {
            const int vbase = j * numVec;
            int nVecHere = bandEnd - j * segLen + 1;
            if (nVecHere > numVec) nVecHere = numVec;
            if (nVecHere < 0) nVecHere = 0;
            int hInit;
            if (j == 0) {
                hInit = scoreInit;
                if (i > 0) { hInit = scoreInit - open - (i - 1) * ext; if (hInit < 0) hInit = 0; }
            } else {
                hInit = (bandBeg > j * segLen) ? 0 : (int)Hptr[(vbase - 1) * SG_VEC + (SG_VEC - 1)];
            }
            const int fcarry = (j > segBegTrack) ? (l == 0 ? X0 : 0) : 0;       // (X0, 0, ..., 0) passed on from the previous segment (:572)
            const bool valid = q < nVecHere;
            const int idx = (vbase + q) * SG_VEC + l;
            int temp = 0, h = 0, act = 0;
            if (valid) {
                int hdiag;
                if (q == 0) hdiag = (l == 0) ? hInit : (int)Hptr[(vbase + numVec - 1) * SG_VEC + l - 1];
                else hdiag = Hptr[idx - SG_VEC];
                const int pv = profRow[idx];
                const int m = (hdiag > 0) ? hdiag + pv : 0;      // (no saturation can occur here: sg_ag_small_scores)
                const int e = E[idx];
                act = (e > m) ? 1 : 0;
                h = m > e ? m : e;
                const int e2 = e - ext;
                temp = m - open; if (temp < 0) temp = 0;
                if (e2 > temp) act |= 4;
                E[idx] = (int16_t)(e2 > temp ? e2 : temp);
            }
            const int t0 = sg_shfl(temp, l), t1 = sg_shfl(temp, 8 + l), t2 = sg_shfl(temp, 16 + l), t3 = sg_shfl(temp, 24 + l);
            int fin = fcarry - q * ext;
            if (q > 0) { int v = t0 - (q - 1) * ext; if (v > fin) fin = v; }
            if (q > 1) { int v = t1 - (q - 2) * ext; if (v > fin) fin = v; }
            if (q > 2) { int v = t2; if (v > fin) fin = v; }
            if (valid) {
                if (fin > h) { act |= 2; h = fin; }
                if (fin - ext > temp) act |= 32;
            }
            int fl = fcarry - nVecHere * ext;            // f register of SSE lane l after the main pass
            { int v = t0 - (nVecHere - 1) * ext; if (nVecHere > 0 && v > fl) fl = v; }
            { int v = t1 - (nVecHere - 2) * ext; if (nVecHere > 1 && v > fl) fl = v; }
            { int v = t2 - (nVecHere - 3) * ext; if (nVecHere > 2 && v > fl) fl = v; }
            { int v = t3 - (nVecHere - 4) * ext; if (nVecHere > 3 && v > fl) fl = v; }
            if (fl < 0) fl = 0;
            // lazy F (:534-569).  Counted on `snap single -d 14`: 4.4 rounds per (row, segment) -- with gap-extend 1
            // against gap-open 7 the cells right of the diagonal stay within reach of F round after round -- so the round is kept to
            // the bone: a lane outside the unit holds an H nothing beats (no `valid` tests), "my vector is at or before the first one
            // with no live lane" is one mask test on the vote, and X (:572) is taken after the loop in closed form -- lane 7 holds SSE
            // lane 7-r's f, r rounds decayed, at the top of round r -- instead of by a shuffle per round.
            const unsigned stopBits = 0x80808080u & (nVecHere >= 4 ? 0xffffffffu : ((1u << (8 * nVecHere)) - 1u));
            const unsigned beforeMe = 0x80808080u & ((1u << (8 * q)) - 1u);
            const int dRound = nVecHere * ext, fl0 = fl;
            // 0x3fff beats every F: F is a decayed cell value, and sg_ag_small_scores keeps cell values below 12000 for this form
            if (!valid) h = 0x3fff;
            int nRounds = 0;
            #pragma unroll 1
            for (int kk = 0; kk < SG_VEC - 1; kk++) {
                nRounds++;
                { const int up = sg_shfl(fl, laneUp); fl = (l == 0) ? 0 : up; }
                int fv = fl - q * ext; if (fv < 0) fv = 0;
                const int newh = fv > h ? fv : h;
                int tmp2 = newh - open; if (tmp2 < 0) tmp2 = 0;
                int fn = fv - ext; if (fn < 0) fn = 0;
                const bool live = fn > tmp2;
                const unsigned liveMask = __ballot_sync(0xffffffffu, live);
                // lowest all-zero byte of the ballot among the unit's vectors = first vector at which no lane is live
                const unsigned zb = (liveMask - 0x01010101u) & ~liveMask & stopBits;
                if (!(zb & beforeMe)) {
                    if (fv > h) act |= 2;
                    if (live) act |= 32;
                    h = newh;
                }
                if (zb) break;
                fl = fl - dRound; if (fl < 0) fl = 0;
            }
            if (j < segEndTrack) {        // X only feeds the next segment of this row
                int v = fl0 - (7 - l) * dRound;
                if (v < 0 || (7 - l) >= nRounds) v = 0;
                v = __reduce_max_sync(0xffffffffu, v);
                if (v > X0) X0 = v;
            }
            if (valid) {
                const int col = j * segLen + l * numVec + q;
                if (h > myMax || (h == myMax && col > myMaxCol)) { myMax = h; myMaxCol = col; }
                Hm1ptr[idx] = (int16_t)h;
                btRow[idx] = (uint8_t)act;
            }
            __syncwarp();
        }

        const int maxScoreRow = __reduce_max_sync(0xffffffffu, myMax);
        if (bandEnd == patternLen - 1) {
            const int globalAlignmentScore = Hm1ptr[globalIdx];
            if (globalAlignmentScore >= bestG) { bestG = globalAlignmentScore; bestGT = i; }
        }
        lay.nRows = i + 1;
        if (maxScoreRow == 0) break;
        if (maxScoreRow > bestL) {
            bestL = maxScoreRow; bestLT = i;
            bestLP = __reduce_max_sync(0xffffffffu, (myMax == maxScoreRow) ? myMaxCol : -1);
        }
        int16_t *tmp = Hm1ptr; Hm1ptr = Hptr; Hptr = tmp;
    }
    __syncwarp();
    res->gScore = bestG; res->gText = bestGT; res->lScore = bestL; res->lText = bestLT; res->lPat = bestLP;
}


// AGM: 2 = the caller's kernel may take the unrolled packed instantiation (only stage 2 of the paired launch carries that code);
//      3 = 2 + the experimental narrow-band form of sg_warp_ag_duo.cuh when SgAgParams.usePacked has bit 2 set (leaf tests only)
template <int AGM = 0>
__device__ __noinline__ void sg_warp_ag_compute(const SgTables &T, const SgScratch &S, const SgAgParams &P, int dir, bool banded,
                                                const uint8_t *text, int textLen, const uint8_t *pattern, const uint8_t *quality, int patternLen,
                                                int w, int scoreInit, bool isRC, bool useClippingOptimizations, SgAgResult *out, int lane)
{
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
    lay.w = w; lay.patternLen = patternLen; lay.nRows = 0;
    const int numVec = lay.numVec, segLen = lay.segLen, numSeg = lay.numSeg;
    const int stride = lay.rowStride();
    const int l = lane & 7, q = lane >> 3;
    const int open = P.gapOpenPenalty, ext = P.gapExtendPenalty;

    int endBonus;
    if (!isRC) endBonus = (dir == -1) ? P.fivePrimeEndBonus : P.threePrimeEndBonus;
    else       endBonus = (dir == -1) ? P.threePrimeEndBonus : P.fivePrimeEndBonus;

    int16_t *Hptr = S.agH, *Hm1ptr = S.agHm1, *E = S.agE;
    uint8_t *bt = S.agBt[dir == 1 ? 0 : 1];

    // first row (:971-983 / :399-414): per SSE lane the "last value assigned" persists across vectors and segments
    if (q == 0) {
        int last = 0;
        for (int segIdx = 0; segIdx < numSeg; segIdx++) {
            for (int vecIdx = 0; vecIdx < numVec; vecIdx++) {
                int patternIdx = segIdx * segLen + l * numVec + vecIdx;
                if (patternIdx < patternLen) {
                    int v = scoreInit - open - patternIdx * ext;
                    last = v > 0 ? v : 0;
                }
                int idx = (segIdx * numVec + vecIdx) * SG_VEC + l;
                Hptr[idx] = (int16_t)last;
                Hm1ptr[idx] = 0;
                E[idx] = 0;
            }
        }
    }
#ifndef SG_AG_NO_PACKED
    if (!banded && numVec <= SG_AGP_MAX_VEC && (P.usePacked & 3)) {
        // unbanded, up to 192 columns: the packed (two cells per lane, DPX s16x2) register-resident form
        __syncwarp();
        SgAgBests bb;
        if (AGM >= 2 && (P.usePacked & 3) == 2) sg_warp_ag_rows_packed<true>(S, P, dir, text, textLen, pattern, patternLen, scoreInit, lay, bt, lane, &bb);
        else sg_warp_ag_rows_packed<false>(S, P, dir, text, textLen, pattern, patternLen, scoreInit, lay, bt, lane, &bb);
        sg_ag_finish(T, P, lay, bt, dir, text, pattern, quality, patternLen, scoreInit, endBonus, useClippingOptimizations,
                     bb.lScore, bb.lText, bb.lPat, bb.gScore, bb.gText, out);
        return;
    }
#endif
    if (AGM == 3 && banded && numVec <= 4 && (P.usePacked & 3) && (P.usePacked & 4)) {
        // bands of up to 32 columns, the experimental form: two (row, segment) units per step, two cells per lane, lazy F without
        // its loop (sg_warp_ag_duo.cuh).  Same results; 12 % fewer instructions than the one-cell-per-lane form below but 4 % slower
        // in the single-end kernel and 10 % in the paired one (instruction-fetch stalls: its step is 530 instructions of straight-line
        // code against a 6 KB L0), so only the leaf-test kernel (AGM 3) and the SIMT emulator of the CPU suite instantiate it.
        __syncwarp();
        SgAgBests bb;
        sg_warp_ag_rows_banded_duo(S, P, dir, text, textLen, pattern, patternLen, w, scoreInit, lay, bt, lane, &bb);
        sg_ag_finish(T, P, lay, bt, dir, text, pattern, quality, patternLen, scoreInit, endBonus, useClippingOptimizations,
                     bb.lScore, bb.lText, bb.lPat, bb.gScore, bb.gText, out);
        return;
    }
    // striped query profile (the reference's qProfile, :921-935 / :348-365) as int16 with the reference's INT16_MIN padding: any
    // match reward or substitution penalty of the scheme fits
    int16_t *prof = S.agProf;
    for (int idx = lane; idx < stride; idx += 32) {
        const int vec = idx >> 3, ll = idx & 7;
        const int col = (vec / numVec) * segLen + ll * numVec + (vec % numVec);
        const uint32_t pb = (col < patternLen) ? sg_base_value(pattern[col]) : 5u;
        for (uint32_t t = 0; t < 5; t++) prof[t * stride + idx] = (pb == 5u) ? (int16_t)-32768 : (int16_t)sg_ag_sub(P, t, pb);
    }
    __syncwarp();

    if (banded && numVec <= 4 && (P.usePacked & 3)) {      // (same switch as the packed form)
        SgAgBests bb;
        sg_warp_ag_rows_banded4(S, open, ext, dir, text, textLen, patternLen, w, scoreInit, lay, bt, lane, &bb);
        sg_ag_finish(T, P, lay, bt, dir, text, pattern, quality, patternLen, scoreInit, endBonus, useClippingOptimizations,
                     bb.lScore, bb.lText, bb.lPat, bb.gScore, bb.gText, out);
        return;
    }

    int bestGlobalAlignmentScore = -1, bestGlobalAlignmentTextOffset = -1;
    int bestLocalAlignmentScore = -1, bestLocalAlignmentTextOffset = -1, bestLocalAlignmentPatternOffset = -1;
    const int globalIdx = lay.cellIndex(patternLen - 1);     // where the last pattern column lives (constant)
    // band edges advance by at most one column per row, so the segments they fall in are tracked without dividing
    int segBegTrack = 0, segEndTrack = banded ? (((w < patternLen - 1) ? w : (patternLen - 1)) / segLen) : 0;

    #pragma unroll 1
    for (int i = 0; i < textLen; i++) {
        lay.nRows = i + 1;
        const uint32_t tb = sg_base_value(text[i * dir]);
        uint8_t *btRow = bt + (size_t)i * stride;
        const int16_t *profRow = prof + tb * stride;
        int myMax = 0;                   // running max of H over the cells this lane committed in this row
        int myMaxCol = -1;               // ... and the largest column at which this lane saw it
        int X0 = 0;                      // lane 0 of the reference's X register
        int fcarry = 0;                  // F entering the next vector of my SSE lane (identical in the 4 sub-lanes)

        int bandBeg = 0, bandEnd = patternLen - 1, segBeg = 0, segEnd = 0;
        if (banded) {
            bandBeg = (i - w) > 0 ? (i - w) : 0;
            bandEnd = (i + w) < (patternLen - 1) ? (i + w) : (patternLen - 1);
            while (bandBeg >= (segBegTrack + 1) * segLen) segBegTrack++;
            while (bandEnd >= (segEndTrack + 1) * segLen) segEndTrack++;
            segBeg = segBegTrack;
            segEnd = segEndTrack;
        }

        #pragma unroll 1
        for (int j = segBeg; j <= segEnd; j++) {
            const int vbase = j * numVec;
            int nVecHere = numVec;
            if (banded) {
                int lim = bandEnd - j * segLen + 1;
                if (lim < nVecHere) nVecHere = lim;
                if (nVecHere < 0) nVecHere = 0;
            }
            int hInit;
            if (j == 0) {
                hInit = scoreInit;
                if (i > 0) { hInit = scoreInit - open - (i - 1) * ext; if (hInit < 0) hInit = 0; }
            } else {
                if (bandBeg > j * segLen) hInit = 0;
                else hInit = Hptr[(vbase - 1) * SG_VEC + (SG_VEC - 1)];
            }
            // f entering vector 0 of this segment: 0, or (X0, 0, ..., 0) passed on from the previous segment (:572)
            fcarry = (banded && j > segBeg) ? (l == 0 ? X0 : 0) : 0;

            const int nBlocks = (nVecHere + 3) >> 2;
            const int passes = banded ? (SG_VEC - 1) : SG_VEC;
            if (nBlocks == 1) {
                // ---- up to 4 vectors in this segment (band half-width <= 15): every lane owns one cell, which stays in
                //      registers through the main pass and all lazy-F passes and is written once ----
                const int k = q;
                const bool valid = k < nVecHere;
                const int idx = (vbase + k) * SG_VEC + l;
                int temp = 0, h = 0, act = 0;
                if (valid) {
                    int hdiag;
                    if (k == 0) hdiag = (l == 0) ? hInit : (int)Hptr[(vbase + numVec - 1) * SG_VEC + l - 1];
                    else hdiag = Hptr[idx - SG_VEC];
                    const int pv = profRow[idx];
                    const int m = (hdiag > 0) ? sg_sat16(hdiag + pv) : 0;
                    const int e = E[idx];
                    act = (e > m) ? 1 : 0;
                    h = m > e ? m : e;
                    const int e2 = sg_sat16(e - ext);
                    temp = sg_sat16(m - open); if (temp < 0) temp = 0;
                    if (e2 > temp) act |= 4;
                    E[idx] = (int16_t)(e2 > temp ? e2 : temp);
                }
                const int t0 = sg_shfl(temp, l), t1 = sg_shfl(temp, 8 + l), t2 = sg_shfl(temp, 16 + l), t3 = sg_shfl(temp, 24 + l);
                int fin = fcarry - q * ext;
                if (q > 0) { int v = t0 - (q - 1) * ext; if (v > fin) fin = v; }
                if (q > 1) { int v = t1 - (q - 2) * ext; if (v > fin) fin = v; }
                if (q > 2) { int v = t2; if (v > fin) fin = v; }
                if (valid) {
                    if (fin > h) { act |= 2; h = fin; }
                    if (sg_sat16(fin - ext) > temp) act |= 32;
                }
                int fl = fcarry - nVecHere * ext;            // f register of SSE lane l after the main pass
                { int v = t0 - (nVecHere - 1) * ext; if (nVecHere > 0 && v > fl) fl = v; }
                { int v = t1 - (nVecHere - 2) * ext; if (nVecHere > 1 && v > fl) fl = v; }
                { int v = t2 - (nVecHere - 3) * ext; if (nVecHere > 2 && v > fl) fl = v; }
                { int v = t3 - (nVecHere - 4) * ext; if (nVecHere > 3 && v > fl) fl = v; }
                if (fl < 0) fl = 0;
                const unsigned validBytes = nVecHere >= 4 ? 0xffffffffu : ((1u << (8 * nVecHere)) - 1u);
                #pragma unroll 1
                for (int kk = 0; kk < passes; kk++) {
                    if (banded && j < segEnd) { int f7 = sg_shfl(fl, 7); if (f7 > X0) X0 = f7; }      // X0 only feeds the next segment of this row
                    { int up = sg_shfl(fl, (lane & 24) | ((l + 7) & 7)); fl = (l == 0) ? 0 : up; }
                    int fv = fl - k * ext; if (fv < 0) fv = 0;
                    const bool a2 = valid && fv > h;
                    const int newh = a2 ? fv : h;
                    int tmp2 = newh - open; if (tmp2 < 0) tmp2 = 0;
                    int fn = fv - ext; if (fn < 0) fn = 0;
                    const bool live = valid && fn > tmp2;
                    const unsigned liveMask = __ballot_sync(0xffffffffu, live);
                    // lowest all-zero byte of the ballot among the valid vectors = first vector at which no lane is live
                    const unsigned zb = (liveMask - 0x01010101u) & ~liveMask & 0x80808080u & validBytes;
                    const int firstConv = zb ? ((__ffs(zb) - 1) >> 3) : 4;
                    if (q <= firstConv) { h = newh; act |= (a2 ? 2 : 0) | (live ? 32 : 0); }
                    if (firstConv < 4) break;
                    fl = fl - nVecHere * ext; if (fl < 0) fl = 0;
                }
                if (valid) {
                    const int col = j * segLen + l * numVec + k;
                    if (h > myMax || (h == myMax && col > myMaxCol)) { myMax = h; myMaxCol = col; }
                    Hm1ptr[idx] = (int16_t)h;
                    btRow[idx] = (uint8_t)act;
                }
                __syncwarp();
                continue;
            }


            // ---------------- main pass, 4 vectors per step ----------------
            for (int b = 0; b < nBlocks; b++) {
                const int k = 4 * b + q;
                const bool valid = k < nVecHere;
                const int idx = (vbase + k) * SG_VEC + l;
                int temp = 0, h1 = 0, act = 0;
                if (valid) {
                    int hdiag;
                    if (k == 0) hdiag = (l == 0) ? hInit : (int)Hptr[(vbase + numVec - 1) * SG_VEC + l - 1];
                    else hdiag = Hptr[idx - SG_VEC];
                    const int pv = profRow[idx];
                    const int m = (hdiag > 0) ? sg_sat16(hdiag + pv) : 0;
                    const int e = E[idx];
                    act = (e > m) ? 1 : 0;
                    h1 = m > e ? m : e;
                    const int e2 = sg_sat16(e - ext);
                    temp = sg_sat16(m - open); if (temp < 0) temp = 0;
                    if (e2 > temp) act |= 4;
                    E[idx] = (int16_t)(e2 > temp ? e2 : temp);
                }
                // F entering vector k of SSE lane l: max(fcarry - q*ext, temp[k'] - (q-1-q')*ext for q' < q in this block).
                // (the reference's saturating f - ext only ever matters through max(.., temp >= 0), so plain ints are exact)
                const int t0 = sg_shfl(temp, l), t1 = sg_shfl(temp, 8 + l), t2 = sg_shfl(temp, 16 + l), t3 = sg_shfl(temp, 24 + l);
                int fin = fcarry - q * ext;
                if (q > 0) { int v = t0 - (q - 1) * ext; if (v > fin) fin = v; }
                if (q > 1) { int v = t1 - (q - 2) * ext; if (v > fin) fin = v; }
                if (q > 2) { int v = t2; if (v > fin) fin = v; }
                // the reference's f register is max(f - ext, temp) >= 0 after the first vector and 0 (or X) before it
                if (b > 0 || q > 0) { if (fin < 0) fin = 0; }
                if (valid) {
                    int h = h1;
                    if (fin > h) { act |= 2; h = fin; }
                    const int f2 = sg_sat16(fin - ext);
                    if (f2 > temp) act |= 32;
                    const int col = j * segLen + l * numVec + k;
                    if (h > myMax || (h == myMax && col > myMaxCol)) { myMax = h; myMaxCol = col; }
                    Hm1ptr[idx] = (int16_t)h;
                    btRow[idx] = (uint8_t)act;
                }
                // carry out of this block = F entering vector 4b+4 (only vectors < nVecHere contribute)
                int nv = nVecHere - 4 * b; if (nv > 4) nv = 4;
                int c = fcarry - nv * ext;
                { int v = t0 - (nv - 1) * ext; if (nv > 0 && v > c) c = v; }
                { int v = t1 - (nv - 2) * ext; if (nv > 1 && v > c) c = v; }
                { int v = t2 - (nv - 3) * ext; if (nv > 2 && v > c) c = v; }
                { int v = t3 - (nv - 4) * ext; if (nv > 3 && v > c) c = v; }
                if (c < 0) c = 0;
                fcarry = c;
            }
            __syncwarp();

            // ---------------- lazy F (:1080-1112 / :534-569) ----------------
            int fl = fcarry;                 // f register of SSE lane l after the main pass
            bool converged = false;
            for (int kk = 0; kk < passes && !converged; kk++) {
                if (banded && j < segEnd) { int f7 = sg_shfl(fl, 7); if (f7 > X0) X0 = f7; }
                { int up = sg_shfl(fl, (lane & 24) | ((l + 7) & 7)); fl = (l == 0) ? 0 : up; }      // f = f << one lane
                for (int b = 0; b < nBlocks && !converged; b++) {
                    const int v = 4 * b + q;
                    const bool valid = v < nVecHere;
                    const int idx = (vbase + v) * SG_VEC + l;
                    int fv = fl - v * ext; if (fv < 0) fv = 0;
                    int h = 0, act = 0, newh = 0;
                    bool live = false, a2 = false;
                    if (valid) {
                        h = Hm1ptr[idx];
                        act = btRow[idx];
                        a2 = fv > h;
                        newh = a2 ? fv : h;
                        int temp = newh - open; if (temp < 0) temp = 0;
                        int fn = fv - ext; if (fn < 0) fn = 0;
                        live = fn > temp;
                    }
                    const unsigned liveMask = __ballot_sync(0xffffffffu, live);
                    // first vector of this block (in order) at which no SSE lane is live any more: the lowest all-zero
                    // byte of the ballot among the valid vectors
                    int nv = nVecHere - 4 * b; if (nv > 4) nv = 4;
                    const unsigned zeroBytes = (liveMask - 0x01010101u) & ~liveMask & 0x80808080u & (nv >= 4 ? 0xffffffffu : ((1u << (8 * nv)) - 1u));
                    const int firstConv = zeroBytes ? ((__ffs(zeroBytes) - 1) >> 3) : 4;
                    if (valid && q <= firstConv && (a2 || live)) {      // nothing to write when the cell is unchanged
                        Hm1ptr[idx] = (int16_t)newh;
                        btRow[idx] = (uint8_t)(act | (a2 ? 2 : 0) | (live ? 32 : 0));
                        if (a2) {
                            const int col = j * segLen + l * numVec + v;
                            if (newh > myMax || (newh == myMax && col > myMaxCol)) { myMax = newh; myMaxCol = col; }
                        }
                    }
                    if (firstConv < 4) converged = true;
                }
                if (!converged) { fl = fl - nVecHere * ext; if (fl < 0) fl = 0; }
            }
            __syncwarp();
        }

        const int maxScoreRow = __reduce_max_sync(0xffffffffu, myMax);

        if (!banded || bandEnd == patternLen - 1) {
            int globalAlignmentScore = Hm1ptr[globalIdx];
            if (globalAlignmentScore >= bestGlobalAlignmentScore) {
                bestGlobalAlignmentScore = globalAlignmentScore;
                bestGlobalAlignmentTextOffset = i;
            }
        }

        if (maxScoreRow == 0) break;

        if (maxScoreRow > bestLocalAlignmentScore) {
            // the largest column holding the row maximum (:1137-1148): H only grows within a row, so the (max, column)
            // pair each lane kept while committing cells is exact
            const int best = __reduce_max_sync(0xffffffffu, (myMax == maxScoreRow) ? myMaxCol : -1);
            bestLocalAlignmentScore = maxScoreRow;
            bestLocalAlignmentTextOffset = i;
            bestLocalAlignmentPatternOffset = best;
        }

        if (!banded && sg_ag_can_stop_after_row(P, i, patternLen, scoreInit, bestLocalAlignmentScore, bestLocalAlignmentTextOffset,
                                                bestLocalAlignmentPatternOffset, bestGlobalAlignmentScore)) break;      // row pruning, see sg_ag.h

        int16_t *tmp = Hm1ptr; Hm1ptr = Hptr; Hptr = tmp;
    }
    __syncwarp();

    sg_ag_finish(T, P, lay, bt, dir, text, pattern, quality, patternLen, scoreInit, endBonus, useClippingOptimizations,
                 bestLocalAlignmentScore, bestLocalAlignmentTextOffset, bestLocalAlignmentPatternOffset,
                 bestGlobalAlignmentScore, bestGlobalAlignmentTextOffset, out);
}
