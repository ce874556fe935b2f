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
//
// A band of 2w+1 <= segLen columns touches at most two segments in a row, so a row is a first unit and, when the band crosses a
// segment boundary, a second one that takes the first one's X.  The function is instruction-issue bound (DESIGN.md section 8), so
// what does not change from unit to unit is a per-lane constant (the offset of a lane's diagonal predecessor, the lazy-F shuffle
// source), and the kernels' 64 registers decide which ones: values used once per unit are recomputed rather than held.  A unit has
// no branches but its lazy-F loop: lanes outside the unit load from a cell of the unit (their values are never used) and do not
// store.
#ifdef __CUDA_ARCH__
#define SG_ASSUME_GLOBAL(p) __builtin_assume(__isGlobal(p))      // arena memory: global loads and stores, not generic ones
#else
#define SG_ASSUME_GLOBAL(p) ((void)0)
#endif
__device__ __noinline__ void sg_warp_ag_rows_banded4(const SgScratch &S, int open, int ext, int dir, const uint8_t *text, int textLen, int patternLen,
                                                     int w, int scoreInit, SgAgLayout &lay, uint8_t *bt, int lane, SgAgBests *res)
{
    const int BIG = 1 << 20;             // pushes a term below every F (F and cell values stay below 12000: sg_ag_small_scores)
    const int numVec = lay.numVec, segLen = lay.segLen;
    const int stride = lay.rowStride();
    const int l = lane & 7, q = lane >> 3;
    int16_t *Hptr = S.agH, *Hm1ptr = S.agHm1;
    int16_t *const E = S.agE;
    const int16_t *const prof = S.agProf;
    SG_ASSUME_GLOBAL(Hptr); SG_ASSUME_GLOBAL(Hm1ptr); SG_ASSUME_GLOBAL(E); SG_ASSUME_GLOBAL(prof); SG_ASSUME_GLOBAL(bt);
    int bestG = -1, bestGT = -1, bestLT = -1;
    int bestKey = -1;                    // (best local score << 16) | its column, -1 before the first
    // column patternLen-1 is lane gLane of its segment's unit, and that unit is the last one of every row whose band reaches it
    const int gLane = lay.cellIndex(patternLen - 1) % segLen;

    // per-lane constants.  Cell of lane (q, l) in the unit of segment j: j*segLen + lane.  Its diagonal predecessor (the previous
    // row's H one column left): vector q-1 of the same SSE lane, or for q = 0 the segment's last vector in SSE lane l-1, or for
    // lane 0 the previous segment's last cell (the reference's hInit)
    const int diagOff = q ? -SG_VEC : (l ? segLen - SG_VEC - 1 : -1);
    const int laneUp = (lane & 24) | ((l + 7) & 7);
    const int qExt = q * ext;

    int begOff = 0;                                                  // first cell of the row's first segment
    int endOff = (((w < patternLen - 1) ? w : (patternLen - 1)) / segLen) * segLen;   // ... and of its last
    // H left of column 0 (the reference's hInit of segment 0): scoreInit in row 0, scoreInit - open - (i-1)*ext after; it only
    // enters through hdiag > 0 ? .. : 0, so it needs no clamp at 0
    int rowInit = scoreInit;
    const uint8_t *tp = text;
    uint8_t *btRow = bt;
    int i = 0;

    #pragma unroll 1
    for (; i < textLen; i++) {
        const int16_t *profRow = prof + (int)sg_base_value(*tp) * stride;
        tp += dir;
        const int bandBeg = (i - w) > 0 ? (i - w) : 0;
        const int bandEnd = (i + w) < (patternLen - 1) ? (i + w) : (patternLen - 1);
        // band edges advance by at most one column per row
        if (bandBeg >= begOff + segLen) begOff += segLen;
        if (bandEnd >= endOff + segLen) endOff += segLen;
        int key = 0;                     // max over my committed cells of (H << 16) | column: the row maximum and its largest column
        int X0 = 0, h = 0;

        // one unit, or two with the first one's X carried into the second; none once the band has left the last segment
        #pragma unroll 1
        for (int jOff = begOff; jOff <= endOff; jOff += segLen) {
            const int nv = (bandEnd - jOff + 1) < numVec ? (bandEnd - jOff + 1) : numVec;     // vectors of this segment in the band, >= 1
            const bool valid = q < nv;
            const bool ownInit = lane == 0 && (jOff == 0 || bandBeg > jOff);
            const int hInit = (jOff == 0) ? rowInit : 0;
            const int cell = jOff + (valid ? lane : 0);
            const int dcell = (valid && !ownInit) ? cell + diagOff : jOff;
            const int hd = Hptr[dcell];
            const int pv = profRow[cell];
            const int e = E[cell];
            const int hdiag = ownInit ? hInit : hd;
            const int m = (hdiag > 0) ? hdiag + pv : 0;      // (no saturation can occur here: sg_ag_small_scores)
            const int hme = m > e ? m : e;
            const int e2 = e - ext;
            int temp = m - open; if (temp < 0) temp = 0;
            if (valid) E[cell] = (int16_t)(e2 > temp ? e2 : temp);
            int act = ((e > m) ? 1 : 0) | ((e2 > temp) ? 4 : 0);
            // F leaving vector q of SSE lane l is max(fcarry - (q+1)*ext, temp[q'] - (q-q')*ext for q' <= q): a prefix max of
            // temp + q*ext over the 4 vectors (a shuffle up returns a lane's own value where it has no source, which a max absorbs)
            const int fcarry = (l == 0) ? X0 : 0;          // (X0, 0, ..., 0) passed on from the previous segment (:572)
            int s = temp + qExt;
            { const int v = __shfl_up_sync(0xffffffffu, s, 8); if (v > s) s = v; }
            { const int v = __shfl_up_sync(0xffffffffu, s, 16); if (v > s) s = v; }
            const int fout = ((fcarry - ext) > s ? (fcarry - ext) : s) - qExt;
            const int fup = __shfl_up_sync(0xffffffffu, fout, 8);
            const int fin = q ? fup : fcarry;              // F entering my vector
            h = hme > fin ? hme : fin;
            if (fin - ext > temp) act |= 32;
            // f register of SSE lane l after the main pass: F leaving the unit's last vector
            const int fl0 = sg_shfl(fout, ((nv - 1) << 3) | l);
            // lazy F (:534-569).  Counted on `snap single -d 14`: 4.4 rounds per (row, segment) -- with gap-extend 1 against
            // gap-open 7 the cells right of the diagonal stay within reach of F round after round -- so the round is kept to the
            // bone.  f carries -q*ext and is never clamped at 0: every use of it (max with H >= 0, f > H, f - ext > max(.., 0))
            // gives the same answer for a negative f as for 0.  Lane 7 carries BIG less, so that SSE lane 0 takes a value below 0.
            // A lane outside the unit votes in a byte the stop mask ignores.  Every round but the last commits in every lane; the
            // last commits up to the first vector with no live lane.  H rises only where F beat it, so bit 2 is read off H.
            const unsigned stopBits = 0x80808080u >> (32 - 8 * nv);
            const int dRound = nv * ext, dec = dRound + ((l == 7) ? BIG : 0);
            int f = fl0 - qExt - ((l == 7) ? BIG : 0);
            int nRounds = 0;
            bool liveAny = false;
            #pragma unroll 1
            for (;;) {
                f = sg_shfl(f, laneUp);
                nRounds++;
                const int newh = f > h ? f : h;
                int tmp2 = newh - open; if (tmp2 < 0) tmp2 = 0;
                const bool live = f - ext > tmp2;
                const unsigned liveMask = __ballot_sync(0xffffffffu, live);
                // lowest all-zero byte of the ballot among the unit's vectors = first vector at which no lane is live
                const unsigned zb = (liveMask - 0x01010101u) & ~liveMask & stopBits;
                if (zb) {
                    const unsigned beforeMe = 0x80808080u & ((1u << (lane & 24)) - 1u);     // the bytes of the vectors before mine
                    if (!(zb & beforeMe)) { h = newh; liveAny |= live; }
                    break;
                }
                h = newh; liveAny |= live;
                if (nRounds == SG_VEC - 1) break;
                f -= dec;
            }
            if (h > hme) act |= 2;
            if (liveAny) act |= 32;
            if (valid) {
                Hm1ptr[cell] = (int16_t)h;
                btRow[cell] = (uint8_t)act;
                const int k = (h << 16) | (jOff + l * numVec + q);     // (a lane's columns rise from unit to unit: ties go to the later)
                if (k > key) key = k;
            }
            if (jOff < endOff) {
                // X (:572) only feeds the next segment of this row, in closed form: lane 7 holds SSE lane 7-r's f, r rounds
                // decayed, at the top of round r
                int v = fl0 - (7 - l) * dRound;
                if (v < 0 || (7 - l) >= nRounds) v = 0;
                X0 = __reduce_max_sync(0xffffffffu, v);
            }
        }
        __syncwarp();

        const int rowKey = __reduce_max_sync(0xffffffffu, key);
        if (bandEnd == patternLen - 1) {
            // the last unit holds the cell in lane gLane; with no unit in the row, the reference reads the row two rows back
            const int globalAlignmentScore = (begOff <= endOff) ? sg_shfl(h, gLane) : (int)Hm1ptr[endOff + gLane];
            if (globalAlignmentScore >= bestG) { bestG = globalAlignmentScore; bestGT = i; }
        }
        const int maxScoreRow = rowKey >> 16;
        if (maxScoreRow == 0) break;
        if (maxScoreRow > (bestKey >> 16)) { bestKey = rowKey; bestLT = i; }
        int16_t *tmp = Hm1ptr; Hm1ptr = Hptr; Hptr = tmp;
        btRow += stride;
        rowInit -= (i == 0) ? open : ext;
    }
    lay.nRows = (i < textLen) ? i + 1 : i;
    __syncwarp();
    res->gScore = bestG; res->gText = bestGT; res->lScore = bestKey < 0 ? -1 : bestKey >> 16; res->lText = bestLT;
    res->lPat = bestKey < 0 ? -1 : bestKey & 0xffff;
}


// AGM, the forms the caller's kernel carries beyond the general, packed and banded4 ones (bits, so that no other kernel grows):
//      1 = the two-unit narrow-band form of sg_warp_ag_duo.cuh, taken when SgAgParams.usePacked has bit 2 set (the single-end second
//          pass, SNAPGPU_SINGLE_AG_NARROW=duo);
//      2 = the unrolled packed instantiation (stage 2 of the paired launch);
//      3 = both (the leaf-test kernel and the SIMT emulator of the CPU suite)
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
        if ((AGM & 2) && (P.usePacked & 3) == 2) sg_warp_ag_rows_packed<true>(S, P, dir, text, textLen, pattern, patternLen, scoreInit, lay, bt, lane, &bb);
        else sg_warp_ag_rows_packed<false>(S, P, dir, text, textLen, pattern, patternLen, scoreInit, lay, bt, lane, &bb);
        sg_ag_finish(T, P, lay, bt, dir, text, pattern, quality, patternLen, scoreInit, endBonus, useClippingOptimizations,
                     bb.lScore, bb.lText, bb.lPat, bb.gScore, bb.gText, out);
        return;
    }
#endif
    if ((AGM & 1) && banded && numVec <= 4 && (P.usePacked & 3) && (P.usePacked & 4)) {
        // bands of up to 32 columns: two (row, segment) units per step, two cells per lane (sg_warp_ag_duo.cuh).  Same results as
        // sg_warp_ag_rows_banded4 below; slower than it on H100 (DESIGN.md section 8), so the second pass takes it only under
        // SNAPGPU_SINGLE_AG_NARROW=duo.
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
