// sg_warp_ag_duo.cuh -- the banded affine-gap DP for bands of up to 32 columns (numVec <= 4: every `snap single -d 14` rescoring),
// two (row, segment) units per step, two cells per lane as s16x2 on the DPX min/max unit.  The single-end second pass takes it under
// SNAPGPU_SINGLE_AG_NARROW=duo; the leaf-test kernel and the SIMT emulator of the CPU suite under SgAgParams.usePacked bit 2.
//
// A band of 2w+1 <= segLen columns touches at most two of the reference's segments in a row, and the reference computes both
// whole (AffineGapVectorized.h:256-819: vectors 0 .. nVecHere-1 of every segment between the one holding the band's first column and
// the one holding its last, in-band or not), the second after the first because the horizontal-gap register leaving segment j's
// lazy-F loop (X, :572) enters segment j+1.  sg_warp_ag_rows_banded4 therefore spends one block of 32 one-cell lanes per
// (row, segment), twice per row.  Here the warp is two half-warps of 16 lanes x 2 cells:
//
//   lane = half*16 + q*4 + a      q = vector within the segment, a = the pair of SSE lanes (2a, 2a+1), lo / hi half of a word
//
// half h owns the segments j = h (mod 2) and the schedule is skewed by one row per segment -- unit (row i, segment j) runs at step
// i + j -- so both halves work at once: while one finishes row i in segment j+1 the other already runs row i+1 in segment j.
// Everything unit (i, j+1) needs from unit (i, j) (the X register, the previous row's last cell for its diagonal) was produced a
// step earlier; segments j and j+2 are never live in overlapping steps (2w+1 <= segLen), so a half never has two units to run.
// Same cells, same commit rule, same stale reads (H and E stay in the reference's two ping-pong rows in memory) as
// sg_warp_ag_rows_banded4 and therefore as the reference; the only cell two concurrent units share -- the previous row's last
// cell of segment j, read by (i, j+1) and overwritten by (i+1, j) -- is read before the step's writes.
//
// The lazy-F loop (4.4 rounds per unit on `snap single -d 14`: with gap-extend 1 against gap-open 7 the cells right of the
// diagonal stay within reach of F) runs once per step for both units, as long as the longer of the two (6.3 rounds per step), and
// commits as it goes like banded4's.  Every loop is `#pragma unroll 1`: the kernel is instruction-fetch bound, and a step of
// straight-line code (7 rounds evaluated and reduced at the end, as an earlier form of this function did) outgrows the L0 cache.
// Counted on `snap single -d 14` (tools/narrow_band_counts.py): 0.61 steps per banded4 unit, but at 64 registers the step spills
// (~360 instructions outside the loop, 47 per round, against banded4's ~185 per unit and 28 per round), so it is not faster.
#pragma once

__device__ __noinline__ void sg_warp_ag_rows_banded_duo(const SgScratch &S, const SgAgParams &P, int dir, const uint8_t *text, int textLen,
                                                        const uint8_t *pattern, int patternLen, int w, int scoreInit, SgAgLayout &lay, uint8_t *bt,
                                                        int lane, SgAgBests *res)
{
    const unsigned FULL = 0xffffffffu;
    const int numVec = lay.numVec, segLen = lay.segLen, numSeg = lay.numSeg;
    const int stride = lay.rowStride();                  // cells per row
    const int strideW = stride >> 1;                     // 32-bit words per row of H / E
    const int half = lane >> 4, q = (lane >> 2) & 3, a = lane & 3;
    const int open = P.gapOpenPenalty, ext = P.gapExtendPenalty;
    const unsigned nOpen2 = sg_pk2(-open), nExt2 = sg_pk2(-ext), nQExt2 = sg_pk2(-q * ext);
    const unsigned aMask = (a == 0) ? 0xffff0000u : 0xffffffffu;       // SSE lane 0 takes 0 when f moves up a lane
    unsigned *prof = (unsigned *)S.agProf;               // [5][strideW] packed substitution scores of the pattern columns

    for (int x = lane; x < strideW; x += 32) {
        const int vec = x >> 2, aa = x & 3;
        const int c0 = (vec / numVec) * segLen + (2 * aa) * numVec + (vec % numVec), c1 = c0 + numVec;
        const uint32_t p0 = (c0 < patternLen) ? sg_base_value(pattern[c0]) : 5u;
        const uint32_t p1 = (c1 < patternLen) ? sg_base_value(pattern[c1]) : 5u;
        for (uint32_t t = 0; t < 5; t++) {
            prof[t * strideW + x] = sg_pk(p0 == 5u ? SG_AGP_PAD : sg_ag_sub(P, t, p0), p1 == 5u ? SG_AGP_PAD : sg_ag_sub(P, t, p1));
        }
    }
    __syncwarp();

    int bestG = -1, bestGT = -1, bestL = -1, bestLT = -1, bestLP = -1;
    const int globalIdx = lay.cellIndex(patternLen - 1);
    int jU = half;                                       // the segment this half is on
#ifdef WS_TRACE_DUO
    if (lane == 0) fprintf(stderr, "duo P=%d w=%d numVec=%d numSeg=%d textLen=%d\n", patternLen, w, numVec, numSeg, textLen);
#endif
    int x0in = 0;                                        // X leaving the other half's previous unit
    int prevKey = 0;                                     // (my cells' maximum << 16) | (largest column holding it + 1) in my previous unit
    const int emptyRow = numSeg * segLen + w;            // first row whose band starts beyond the last segment
    const int lastStep = textLen + numSeg + 2;           // (a bound, never reached: the last row's last unit ends the loop)

    #pragma unroll 1
    for (int t = 0; t < lastStep && textLen > 0; t++) {
        int i = t - jU;
        int bandBeg = (i - w) > 0 ? (i - w) : 0;
        int bandEnd = (i + w) < (patternLen - 1) ? (i + w) : (patternLen - 1);
        if (i >= 0 && bandBeg >= (jU + 1) * segLen) {    // the band has left my segment: on to the next one of my parity
            jU += 2; i -= 2;
            bandBeg = (i - w) > 0 ? (i - w) : 0;
            bandEnd = (i + w) < (patternLen - 1) ? (i + w) : (patternLen - 1);
        }
        const bool active = i >= 0 && i < textLen && jU < numSeg && bandEnd >= jU * segLen && bandBeg < (jU + 1) * segLen;
        const bool notFirst = bandBeg < jU * segLen;             // j > the row's first segment
        const bool notLast = bandEnd >= (jU + 1) * segLen;       // j < the row's last segment
        const int vbase = jU * numVec;
        int nVecHere = bandEnd - jU * segLen + 1;
        if (nVecHere > numVec) nVecHere = numVec;
        if (nVecHere < 1) nVecHere = 1;
        const bool valid = active && q < nVecHere;
        const unsigned *Hr = (const unsigned *)((i & 1) ? S.agHm1 : S.agH);
        unsigned *Hw = (unsigned *)((i & 1) ? S.agH : S.agHm1);
        unsigned *Ew = (unsigned *)S.agE;
        const int x = (vbase + q) * 4 + a;                       // my word of the row
        const unsigned ends = __ballot_sync(FULL, active && !notLast);   // which unit, if any, is the last of its row (used at the bottom)

        // ---------------- main pass ----------------
        unsigned hd = 0, e = 0, pv = 0;
        int hInit = 0;
        if (valid) {
            hd = Hr[(q == 0) ? (vbase + numVec - 1) * 4 + a : x - 4];
            e = Ew[x];
            pv = prof[sg_base_value(text[i * dir]) * strideW + x];
            if (q == 0 && a == 0) {
                if (jU == 0) {
                    hInit = scoreInit;
                    if (i > 0) { hInit = scoreInit - open - (i - 1) * ext; if (hInit < 0) hInit = 0; }
                } else if (!(bandBeg > jU * segLen)) {
                    hInit = ((const int16_t *)Hr)[(vbase - 1) * SG_VEC + (SG_VEC - 1)];
                }
            }
        }
        {
            // vector 0 takes the previous row's LAST vector of the segment moved up one SSE lane, hInit entering lane 0
            const unsigned below = __shfl_up_sync(FULL, hd, 1);
            if (q == 0) hd = (hd << 16) | (a == 0 ? ((unsigned)hInit & 0xffffu) : (below >> 16));
        }
        const unsigned m = __vadd2(hd, pv) & sg_nzmask2(hd);                   // (hdiag > 0) ? hdiag + profile : 0
        bool mgeHi, mgeLo, tgeHi, tgeLo, hgeHi, hgeLo, t2Hi, t2Lo;
        const unsigned h1 = __vibmax_s16x2(m, e, &mgeHi, &mgeLo);              // bit 1: e > m
        unsigned temp = __viaddmax_s16x2_relu(m, nOpen2, 0u);                  // max(m - open, 0)
        const unsigned e2 = __vadd2(e, nExt2);
        const unsigned ne = __vibmax_s16x2(temp, e2, &tgeHi, &tgeLo);          // bit 4: e - ext > temp
        if (valid) Ew[x] = ne; else temp = 0u;
        // F entering each vector of the segment: f' = max(f - ext, temp), starting from (X, 0, ..., 0) handed on by the row's
        // previous segment (:572); the four temps arrive by four independent shuffles
        const int hb = (lane & 16) | a;
        const unsigned t0 = __shfl_sync(FULL, temp, hb), t1 = __shfl_sync(FULL, temp, hb | 4), t2 = __shfl_sync(FULL, temp, hb | 8),
                       t3 = __shfl_sync(FULL, temp, hb | 12);
        const unsigned fcarry = (notFirst && a == 0) ? ((unsigned)x0in & 0xffffu) : 0u;
        const unsigned p1 = __viaddmax_s16x2(fcarry, nExt2, t0), p2 = __viaddmax_s16x2(p1, nExt2, t1), p3 = __viaddmax_s16x2(p2, nExt2, t2),
                       p4 = __viaddmax_s16x2(p3, nExt2, t3);
        const unsigned fin = (q == 0) ? fcarry : (q == 1) ? p1 : (q == 2) ? p2 : p3;
        const unsigned hMain = __vibmax_s16x2(h1, fin, &hgeHi, &hgeLo);        // bit 2: f > h
        (void)__vibmax_s16x2(temp, __vadd2(fin, nExt2), &t2Hi, &t2Lo);         // bit 32: f - ext > temp
        unsigned act = ((mgeLo ? 0u : 1u) | (hgeLo ? 0u : 2u) | (tgeLo ? 0u : 4u) | (t2Lo ? 0u : 32u)) |
                       (((mgeHi ? 0u : 1u) | (hgeHi ? 0u : 2u) | (tgeHi ? 0u : 4u) | (t2Hi ? 0u : 32u)) << 8);
        // f register of the SSE lanes after the main pass (the same in all four vectors' lanes)
        const unsigned fl0 = __vimax_s16x2_relu((nVecHere == 1) ? p1 : (nVecHere == 2) ? p2 : (nVecHere == 3) ? p3 : p4, 0u);

        // ---------------- lazy F (:534-569), both halves' units in one loop ----------------
        // The reference runs up to 7 rounds (f moves up one SSE lane and decays by nVecHere*ext per round) over the vectors in
        // order, updating H and the traceback bits, and stops after the first (round, vector) in which no lane can still change a
        // later cell.  One ballot per round carries both halves' live lanes (bit half*16 + q*4 + a); per half, the lowest all-zero
        // nibble is the first vector with no live lane, and a lane commits the round only if its vector is at or before it -- the
        // rule of sg_warp_ag_rows_banded4, a nibble per vector instead of a byte.  A vector outside its half's unit votes live
        // (`fill`), so it never stops the loop.  A half that has stopped, or has no unit, commits nothing more; the loop ends when
        // both halves have stopped.  A lane commits rounds 0 .. k-1 and no later one, so H only grows and the bits are taken
        // after the loop: 2 if H grew, 32 if f - ext beat H - open in a committed round (liveAcc > 0).
        const unsigned nD2 = sg_pk2(-nVecHere * ext);
        // Every read of the rows in memory (hInit above all, see the header) before any write of this step.  Without this barrier,
        // and with bit 32 taken by a DPX max against 0 after the loop, the device gave other results than the SIMT emulator on ~3 % of
        // narrow-band jobs (tests/test_gpu_scoring_schemes.py, form 5); with both changes the two agree.
        __syncwarp();
        const unsigned fill = ~__ballot_sync(FULL, valid);
        const unsigned myHalf = half ? 0x88880000u : 0x00008888u;
        const unsigned beforeMe = (0x8888u & ((1u << (4 * q)) - 1u)) << (16 * half);    // nibble tops of my half's vectors before mine
        unsigned seen = ((fill & 0xffffu) == 0xffffu ? 0x8u : 0u) | ((fill >> 16) == 0xffffu ? 0x80000u : 0u);   // halves stopped
        bool stopped = (seen & myHalf) != 0u;
        unsigned h = hMain, fl = fl0, liveAcc = 0u;
        int nExec = SG_VEC - 1;                                  // rounds my half entered
        #pragma unroll 1
        for (int kk = 0; kk < SG_VEC - 1; kk++) {
            const unsigned below = __shfl_up_sync(FULL, fl, 1);
            const unsigned flS = __byte_perm(fl, below, 0x1076) & aMask;                  // f = f << one SSE lane
            const unsigned fv = __viaddmax_s16x2_relu(flS, nQExt2, 0u);
            const unsigned newh = __vmaxs2(h, fv);                                        // f > h: take it
            const unsigned tmp2 = __viaddmax_s16x2_relu(newh, nOpen2, 0u);
            const unsigned fn = __viaddmax_s16x2_relu(fv, nExt2, 0u);
            bool lgeHi, lgeLo;
            (void)__vibmax_s16x2(tmp2, fn, &lgeHi, &lgeLo);                               // live: f - ext > h - open
            const unsigned vote = __ballot_sync(FULL, !(lgeLo && lgeHi)) | fill;
            const unsigned zb = __vsub2(vote, 0x11111111u) & ~vote & 0x88888888u;         // (no borrow between the halves)
            if (!stopped && !(zb & beforeMe)) { h = newh; liveAcc = __vmaxs2(liveAcc, __vsub2(fn, tmp2)); }
            if (!stopped && (zb & myHalf)) { stopped = true; nExec = kk + 1; }
            seen |= zb;
            if ((seen & 0xffffu) && (seen >> 16)) break;
            fl = __viaddmax_s16x2_relu(flS, nD2, 0u);
        }
        {
            bool geHi, geLo;
            (void)__vibmax_s16x2(hMain, h, &geHi, &geLo);                                  // bit 2: some round's f beat H
            act |= ((geLo ? 0u : 2u) | ((liveAcc & 0xffffu) ? 32u : 0u)) | (((geHi ? 0u : 2u) | ((liveAcc >> 16) ? 32u : 0u)) << 8);   // bit 32
        }
        // X (:572): the largest value lane 7 held at the top of a round that was entered = SSE lane 7-r's f, r rounds decayed
        {
            const int rLo = 7 - 2 * a, rHi = 6 - 2 * a;
            const unsigned c = __viaddmax_s16x2_relu(fl0, sg_pk(-rLo * nVecHere * ext, -rHi * nVecHere * ext), 0u);
            int v = 0;
            if (rLo < nExec) v = (int)(c & 0xffffu);
            if (rHi < nExec) { const int u = (int)(c >> 16); if (u > v) v = u; }
            if (!(active && notLast)) v = 0;
            const int xa = __reduce_max_sync(FULL, half ? 0 : v), xb = __reduce_max_sync(FULL, half ? v : 0);
            x0in = half ? xa : xb;               // X leaving the OTHER half's unit: what enters mine one step later, if my row has a previous segment
        }

        // ---------------- write my cells once; my maximum and the largest column holding it ----------------
        int curKey = 0;                                                         // (maximum << 16) | (column + 1)
        if (valid) {
            Hw[x] = h;
            *(uint16_t *)(bt + (size_t)i * stride + 2 * x) = (uint16_t)act;
            const int lo = (int)(short)(h & 0xffffu), hi = (int)(short)(h >> 16);
            const int colLo = jU * segLen + (2 * a) * numVec + q;
            curKey = (hi >= lo) ? ((hi << 16) | (colLo + numVec + 1)) : ((lo << 16) | (colLo + 1));
        }
        __syncwarp();

        // ---------------- end of a row: at most one of the two units is the last of its row ----------------
        if (ends) {
            const int hc = (ends & 0xffffu) ? 0 : 1;
            const int jc = __shfl_sync(FULL, jU, hc * 16);
            const int ic = t - jc;
            const int bandBegC = (ic - w) > 0 ? (ic - w) : 0;
            const int bandEndC = (ic + w) < (patternLen - 1) ? (ic + w) : (patternLen - 1);
            const bool twoSegs = bandBegC < jc * segLen;
            // the row's maximum and the largest column holding it (:1137-1148), over this unit and, if the row has two, the one
            // the other half ran a step ago
            const int rowKey = __reduce_max_sync(FULL, (half == hc) ? curKey : twoSegs ? prevKey : 0);
            const int maxScoreRow = rowKey >> 16;
            if (bandEndC == patternLen - 1) {
                const int globalAlignmentScore = ((ic & 1) ? S.agH : S.agHm1)[globalIdx];
                if (globalAlignmentScore >= bestG) { bestG = globalAlignmentScore; bestGT = ic; }
            }
            lay.nRows = ic + 1;
            if (maxScoreRow == 0) break;
            if (maxScoreRow > bestL) { bestL = maxScoreRow; bestLT = ic; bestLP = (rowKey & 0xffff) - 1; }
            if (ic == textLen - 1) break;
            if (ic + 1 == emptyRow) {
                // the band has left the pattern's last segment: the reference's row loop visits no segment, still looks at the
                // (two rows old) last-column cell for the global score, finds a row maximum of 0 and stops
                const int globalAlignmentScore = ((emptyRow & 1) ? S.agH : S.agHm1)[globalIdx];
                if (globalAlignmentScore >= bestG) { bestG = globalAlignmentScore; bestGT = emptyRow; }
                lay.nRows = emptyRow + 1;
                break;
            }
        }
        prevKey = curKey;
    }
    __syncwarp();
    res->gScore = bestG; res->gText = bestGT; res->lScore = bestL; res->lText = bestLT; res->lPat = bestLP;
}
